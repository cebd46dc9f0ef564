"""The data and the reference of tests/test_gpu_row_movement.py, checked without a GPU: the wide table holds what it claims
(NaN payloads, signed zeros, subnormals, the decimal(38, 10) extremes and sign crossings, the string edge cases at their byte
lengths, the three validity variants), and the comparison notices a single wrong bit.  A data bug must not pass for a green GPU
run."""
import numpy as np
import pyarrow as pa
import pytest

from test_gpu_key_types import F32_NAN_BITS, F64_NAN_BITS, raw_bits
from test_gpu_row_movement import (ALL_FIXED, DEC38_SPECIALS, DEC38_TOP, F32_SUBNORMALS, F64_SUBNORMALS, FIXED_TYPES, STR_SPECIALS, STRINGS,
                                   TILE, TILE_NULLS, TYPES, WIDTHS, assert_same, dec38_words, fixed_names, take_rows, wide_table)

N = 9000


@pytest.fixture(scope="module")
def table():
    return wide_table(N)


def _words(table, name):
    valid, words = raw_bits(table.column(name))
    return valid, words


@pytest.mark.parametrize("variant", ["t", "n"])
@pytest.mark.parametrize("tname,nan_bits,sub_bits,width", [("float64", F64_NAN_BITS, F64_SUBNORMALS, 64), ("float32", F32_NAN_BITS, F32_SUBNORMALS, 32)])
def test_float_columns_keep_every_payload(table, tname, nan_bits, sub_bits, width, variant):
    """The float columns hold every NaN payload of both signs, +-0.0, +-inf and subnormals at valid positions -- through the
    Arrow array and through the host image the GPU batch is imported from."""
    from spark_b200.columnar import HostColumn
    valid, (w,) = _words(table, "%s_%s" % (tname, variant))
    sign = 1 << (width - 1)
    inf = 0x7FF0000000000000 if width == 64 else 0x7F800000
    want = set(nan_bits) | set(sub_bits) | {0, sign, inf, inf | sign}
    assert want <= set(w[valid].tolist())
    host = np.ascontiguousarray(HostColumn.from_arrow(table.column("%s_%s" % (tname, variant))).data)
    hw = host.view(np.uint64 if width == 64 else np.uint32)
    assert want <= set(hw[valid].tolist())
    assert np.array_equal(hw[valid].astype(np.uint64), w[valid])


def test_decimal38_extremes_and_sign_crossings(table):
    valid, (lo, hi) = _words(table, "dec38_10_n")
    assert valid.all()
    got = set(zip(lo.view(np.int64).tolist(), hi.view(np.int64).tolist()))
    want = set(map(tuple, dec38_words(DEC38_SPECIALS).tolist()))
    assert want <= got
    assert (DEC38_TOP in DEC38_SPECIALS) and (-DEC38_TOP in DEC38_SPECIALS)
    his = hi.view(np.int64)
    assert {0, -1, 1} <= set(his.tolist())                    # high words 0, -1 and a crossing of 2^64
    assert ((lo.view(np.int64) < 0) & (his == 0)).any()         # low word's bit 63 set under a positive high word
    assert table.schema.field("dec38_10_n").type == pa.decimal128(38, 10)
    # every value is inside decimal(38)
    v = [(int(h) << 64) | (int(l) & ((1 << 64) - 1)) for l, h in zip(lo.view(np.int64)[:2000], his[:2000])]
    assert all(-DEC38_TOP <= x <= DEC38_TOP for x in v)


def test_string_edge_cases(table):
    lengths = {len(s.encode()) for s in STR_SPECIALS}
    assert {0, 1, 3, 4, 5, 15, 16, 17, 31, 32, 33} <= lengths and max(lengths) > 100
    assert any("\x00" in s and len(s) > 1 for s in STR_SPECIALS)
    utf8_widths = {len(ch.encode()) for s in STR_SPECIALS for ch in s}
    assert utf8_widths == {1, 2, 3, 4}
    vals = table.column("str_n").to_pylist()
    assert table.column("str_n").null_count == 0
    assert set(STR_SPECIALS) <= set(vals)


def test_validity_variants(table):
    for name in ALL_FIXED[1:] + STRINGS:
        col = table.column(name).combine_chunks()
        variant = name.rsplit("_", 1)[1]
        valid = np.asarray(col.is_valid())
        if variant == "n":
            assert col.null_count == 0 and col.buffers()[0] is None, name
        elif variant == "a":
            assert col.null_count == N, name
        else:
            for p in TILE_NULLS:
                assert not valid[p::TILE].any(), (name, p)
            assert 0.03 < 1 - valid.mean() < 0.08, name


def test_widths_cross_the_column_group_limits():
    assert [len(fixed_names(w)) for w in WIDTHS] == [12, 13, 16, 17, 25]
    first = fixed_names(13)
    assert first[0] == "row" and {c.rsplit("_", 1)[0] for c in first[1:]} == set(FIXED_TYPES)
    assert not any(c.startswith("dec38") for c in fixed_names(25, dec128=False))
    assert len(ALL_FIXED) == 1 + 3 * len(TYPES)


def test_take_rows_is_a_bit_exact_take(table):
    rng = np.random.default_rng(3)
    idx = rng.integers(-1, N, 5000)
    got = take_rows(table, idx)
    ok = idx >= 0
    for name in ALL_FIXED:
        sv, sw = raw_bits(table.column(name))
        gv, gw = raw_bits(got.column(name))
        assert np.array_equal(gv, ok & sv[np.where(ok, idx, 0)]), name
        for a, b in zip(gw, sw):
            assert np.array_equal(a[gv], b[idx[gv]]), name
    for name in STRINGS:
        src = table.column(name).to_pylist()
        assert got.column(name).to_pylist() == [src[i] if i >= 0 else None for i in idx]


@pytest.mark.parametrize("name,flip", [("float64_t", 1), ("float64_n", 1 << 63), ("float32_n", 1), ("dec38_10_n", 1 << 64), ("int16_n", 1 << 8)])
def test_comparison_sees_one_wrong_bit(table, name, flip):
    """One flipped bit -- a NaN payload bit, the sign of a zero, the high word of a decimal(38, 10), the high byte of an int16 --
    fails assert_same."""
    t = table.slice(0, 200)
    valid, _ = raw_bits(t.column(name))
    r = int(np.nonzero(valid)[0][5])
    col = t.column(name).combine_chunks()
    assert col.offset == 0
    width = 16 if pa.types.is_decimal(col.type) else col.type.bit_width // 8
    raw = bytearray(np.frombuffer(col.buffers()[1], np.uint8, count=len(col) * width).tobytes())
    v = int.from_bytes(raw[r * width:(r + 1) * width], "little") ^ flip
    raw[r * width:(r + 1) * width] = v.to_bytes(width, "little")
    bad = pa.Array.from_buffers(col.type, len(col), [col.buffers()[0], pa.py_buffer(bytes(raw))])
    t2 = t.set_column(t.column_names.index(name), name, bad)
    assert_same(t, t)
    with pytest.raises(AssertionError):
        assert_same(t2, t)


def test_comparison_sees_string_bytes_and_validity(table):
    t = table.slice(0, 300)
    vals = t.column("str_n").to_pylist()
    i = vals.index("a\x00b")
    vals[i] = "a\x00c"
    with pytest.raises(AssertionError):
        assert_same(t.set_column(t.column_names.index("str_n"), "str_n", pa.array(vals, pa.string())), t)
    v2 = t.column("int8_n").to_pylist()
    v2[3] = None
    with pytest.raises(AssertionError):
        assert_same(t.set_column(t.column_names.index("int8_n"), "int8_n", pa.array(v2, pa.int8())), t)


def test_decimal128_column_compiles_as_a_bare_reference():
    """Filter and expand pass every column through as a bare reference; a decimal(38, s) one has no value class and compiles
    to a COL node of vtype 0, like a string column."""
    from spark_b200 import _capi as capi
    from spark_b200.expressions import AttributeReference, CompiledExpr, Schema
    for t in (capi.SB_DECIMAL128, capi.SB_STRING):
        ce = CompiledExpr(AttributeReference("d"), Schema(["x", "d"], [capi.SB_INT64, t], set()))
        assert ce.c.n == 1 and ce.c.nodes[0].arg == 1 and ce.c.nodes[0].vtype == 0
