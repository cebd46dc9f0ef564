"""CPU pins for the key-type parity tests (tests/test_gpu_key_types.py): the bit comparator, the data generators, and the
oracle's own answers on small hand-written vectors -- signed zeros and NaN payloads, 64-bit keys with bit 63 set, decimal
keys and hashes, and the sort order of the special float values.  No GPU needed."""
import numpy as np
import pyarrow as pa
import pytest

from oracle import oracle as O
from test_gpu_key_types import (F32_NAN_BITS, F64_NAN_BITS, TYPE_NAMES, TYPES, _f32, _f64, assert_bits_equal, distinct, key_column,
                                make_array, raw_bits, specials)

I64_MIN, I64_MAX = -2 ** 63, 2 ** 63 - 1


def _bits64(arr):
    return [int(x) for x in raw_bits(arr)[1][0]]


# ------------------------------------------------------------------------------------------------ the comparator
def test_comparator_rejects_signed_zero():
    a = pa.table({"x": make_array("float64", np.array([0.0, 1.0]))})
    b = pa.table({"x": make_array("float64", np.array([-0.0, 1.0]))})
    assert_bits_equal(a, a)
    with pytest.raises(AssertionError):
        assert_bits_equal(a, b)
    with pytest.raises(AssertionError):
        assert_bits_equal(pa.table({"x": make_array("float32", np.array([0.0], np.float32))}),
                          pa.table({"x": make_array("float32", np.array([-0.0], np.float32))}))


@pytest.mark.parametrize("width", [32, 64])
def test_comparator_rejects_a_different_nan_payload(width):
    bits = F32_NAN_BITS if width == 32 else F64_NAN_BITS
    conv, tn = (_f32, "float32") if width == 32 else (_f64, "float64")
    a = pa.table({"x": make_array(tn, conv([bits[0]]))})
    for other in bits[1:]:
        with pytest.raises(AssertionError):
            assert_bits_equal(a, pa.table({"x": make_array(tn, conv([other]))}))


def test_comparator_checks_validity_types_and_is_order_insensitive_only_when_asked():
    a = pa.table({"x": pa.array([1, 2, 3], pa.int64())})
    assert_bits_equal(a, pa.table({"x": pa.array([3, 1, 2], pa.int64())}))
    with pytest.raises(AssertionError):
        assert_bits_equal(a, pa.table({"x": pa.array([3, 1, 2], pa.int64())}), ordered=True)
    with pytest.raises(AssertionError):
        assert_bits_equal(a, pa.table({"x": pa.array([1, 2, None], pa.int64())}))
    with pytest.raises(AssertionError):
        assert_bits_equal(a, pa.table({"x": pa.array([1, 2, 3], pa.int32())}))
    d = pa.table({"x": make_array(pa.decimal128(7, 2), np.array([1, -1]))})
    with pytest.raises(AssertionError):
        assert_bits_equal(d, pa.table({"x": make_array(pa.decimal128(9, 2), np.array([1, -1]))}))
    with pytest.raises(AssertionError):     # the high word of a decimal counts too
        assert_bits_equal(d, pa.table({"x": pa.Array.from_buffers(pa.decimal128(7, 2), 2, [None, pa.py_buffer(
            np.array([1, 0, -1, 0], np.int64).tobytes())])}))


def test_raw_bits_of_a_sliced_column():
    arr = make_array("int16", np.array([5, -1, 7, 9], np.int16), np.array([True, True, False, True])).slice(1)
    valid, (w,) = raw_bits(arr)
    assert valid.tolist() == [True, False, True] and w.tolist() == [0xFFFF, 0, 9]


# ------------------------------------------------------------------------------------------------ the generators
@pytest.mark.parametrize("tname", TYPE_NAMES)
def test_generated_columns_carry_every_special_and_nulls(tname):
    rng = np.random.default_rng(0)
    arr = key_column(tname, 2000, rng)
    assert arr.type == TYPES[tname] and arr.null_count > 0
    valid, words = raw_bits(arr)
    sp = specials(tname)
    if tname.startswith("dec"):
        want = sp.astype(np.int64).view(np.uint64)
    else:
        want = np.ascontiguousarray(sp).view({1: np.uint8, 2: np.uint16, 4: np.uint32, 8: np.uint64}[sp.dtype.itemsize]).astype(np.uint64)
    assert set(want.tolist()) <= set(words[0][valid].tolist())
    if tname != "bool":                                               # the EMPTY sentinel's pattern (all ones) is a value
        assert ((1 << (8 * sp.dtype.itemsize)) - 1) in want.tolist() if not tname.startswith("dec") else -1 in sp.tolist()
    if tname == "float64":
        assert {0xFFFFFFFFFFFFFFFF, 0x8000000000000000, 0xFFF8000000000000, 0x7FF0000000000001} <= set(words[0].tolist())
    if tname == "float32":
        assert {0xFFFFFFFF, 0x80000000, 0xFFC00000, 0x7F800001} <= set(words[0].tolist())


def test_distinct_keeps_signed_zeros_and_nan_payloads_apart():
    v = np.concatenate([_f64([0, 1 << 63, 0, F64_NAN_BITS[0], F64_NAN_BITS[1], F64_NAN_BITS[0]])])
    assert [int(x) for x in distinct(v).view(np.uint64)] == [0, 1 << 63, F64_NAN_BITS[0], F64_NAN_BITS[1]]


def test_oracle_columns_keep_nan_payloads_through_nulls_and_take():
    v = _f64(F64_NAN_BITS + [1 << 63])
    arr = make_array("float64", v, np.array([True, True, True, False, True, True]))
    c = O.Col.from_arrow(arr)
    assert [int(x) for x in c.values.view(np.uint64)[[0, 1, 2, 4, 5]]] == F64_NAN_BITS[:3] + [F64_NAN_BITS[4], 1 << 63]
    t = c.take(np.array([5, 4, -1, 1]))
    assert _bits64(t.to_arrow())[:2] == [1 << 63, F64_NAN_BITS[4]] and t.valid.tolist() == [True, True, False, True]


# ------------------------------------------------------------------------------------------------ decimal columns in the oracle
def test_oracle_takes_decimal64_columns_as_unscaled_longs():
    arr = make_array(pa.decimal128(7, 2), np.array([-9999999, 9999999, -1, 0]), np.array([True, True, True, False]))
    c = O.Col.from_arrow(arr)
    assert c.type == O.SO_DECIMAL64 and c.values.tolist() == [-9999999, 9999999, -1, 0] and c.valid.tolist() == [True, True, True, False]
    back = c.take(np.array([2, 0, 3, -1])).to_arrow()
    assert back.type == pa.decimal128(7, 2)
    assert back.to_pylist()[:2] == [arr[2].as_py(), arr[0].as_py()] and back.null_count == 2
    assert O.Col.from_arrow(pa.array([1, None], pa.timestamp("us"))).to_arrow().type == pa.timestamp("us")
    with pytest.raises(NotImplementedError):
        O.Col.from_arrow(pa.array([1], pa.decimal128(19, 0)))


def test_oracle_join_sort_and_group_keep_decimal_types():
    t = pa.table({"k": make_array(pa.decimal128(18, 0), np.array([5, -(10 ** 18 - 1), 5, -1])), "v": pa.array([1, 2, 3, 4])})
    b = pa.table({"k2": make_array(pa.decimal128(18, 0), np.array([5, -1])), "w": pa.array([10, 20])})
    j = O.hash_join(t, b, ["k"], ["k2"], "inner")
    assert j.schema.field("k").type == pa.decimal128(18, 0) and j.schema.field("k2").type == pa.decimal128(18, 0)
    assert sorted(zip(j.column("v").to_pylist(), j.column("w").to_pylist())) == [(1, 10), (3, 10), (4, 20)]
    s = O.sort(t, [("k", True, True)])
    assert s.column("v").to_pylist() == [2, 4, 1, 3] and s.schema.field("k").type == pa.decimal128(18, 0)
    g = O.hash_aggregate(t, ["k"], [("count_star", None, "n")])
    assert g.schema.field("k").type == pa.decimal128(18, 0) and sorted(g.column("n").to_pylist()) == [1, 1, 2]


# ------------------------------------------------------------------------------------------------ the oracle's answers
def test_signed_zeros_and_nan_payloads_group_together_and_come_out_normalised():
    v = _f64([0, 1 << 63, F64_NAN_BITS[1], F64_NAN_BITS[2], F64_NAN_BITS[4], 0x3FF0000000000000])
    t = pa.table({"k": make_array("float64", v), "x": pa.array([1, 2, 3, 4, 5, 6])})
    g = O.hash_aggregate(t, ["k"], [("sum", "x", "s")])
    rows = dict(zip(_bits64(g.column("k")), g.column("s").to_pylist()))
    assert rows == {0: 3, 0x7FF8000000000000: 12, 0x3FF0000000000000: 6}
    v32 = _f32([0x80000000, 0, F32_NAN_BITS[1], F32_NAN_BITS[2]])
    g = O.hash_aggregate(pa.table({"k": make_array("float32", v32), "x": pa.array([1, 2, 3, 4])}), ["k"], [("sum", "x", "s")])
    assert dict(zip([int(w) for w in raw_bits(g.column("k"))[1][0]], g.column("s").to_pylist())) == {0: 3, 0x7FC00000: 7}


def test_signed_zeros_and_nan_payloads_join_together_keeping_their_bits():
    p = pa.table({"k": make_array("float64", _f64([1 << 63, F64_NAN_BITS[2], 0x3FF0000000000000])), "p": pa.array([0, 1, 2])})
    b = pa.table({"k2": make_array("float64", _f64([0, F64_NAN_BITS[1]])), "b": pa.array([0, 1])})
    j = O.hash_join(p, b, ["k"], ["k2"], "inner")
    assert sorted(zip(j.column("p").to_pylist(), _bits64(j.column("k")), _bits64(j.column("k2")))) == \
        [(0, 1 << 63, 0), (1, F64_NAN_BITS[2], F64_NAN_BITS[1])]
    assert O.hash_join(p, b, ["k"], ["k2"], "left_anti").column("p").to_pylist() == [2]


def test_int64_keys_with_bit_63_set_stay_distinct():
    t = pa.table({"k": pa.array([I64_MIN, -1, I64_MAX, -1, I64_MIN, 0], pa.int64()), "x": pa.array([1, 2, 4, 8, 16, 32])})
    g = O.hash_aggregate(t, ["k"], [("sum", "x", "s")])
    assert dict(zip(g.column("k").to_pylist(), g.column("s").to_pylist())) == {I64_MIN: 17, -1: 10, I64_MAX: 4, 0: 32}
    g2 = O.hash_aggregate(t.append_column("k2", pa.array([I64_MAX, I64_MAX, I64_MIN, I64_MAX, I64_MAX, -1])), ["k", "k2"], [("sum", "x", "s")])
    assert g2.num_rows == 4


def _hash_long(v, seed):
    m = 0xFFFFFFFF
    rotl = lambda x, r: ((x << r) | (x >> (32 - r))) & m

    def mix_k1(k):
        return (rotl((k * 0xCC9E2D51) & m, 15) * 0x1B873593) & m

    def mix_h1(h, k):
        return (rotl(h ^ k, 13) * 5 + 0xE6546B64) & m
    u = v & 0xFFFFFFFFFFFFFFFF
    h = mix_h1(mix_h1(seed & m, mix_k1(u & m)), mix_k1(u >> 32))
    h ^= 8
    h ^= h >> 16; h = (h * 0x85EBCA6B) & m
    h ^= h >> 13; h = (h * 0xC2B2AE35) & m
    h ^= h >> 16
    return h - (1 << 32) if h >= 1 << 31 else h


def test_murmur3_of_a_decimal64_is_hash_long_of_its_unscaled_value():
    """hash.scala: a decimal with precision <= 18 hashes as hashLong(unscaledValue): checked against a Python restatement of
    Murmur3_x86_32.hashLong (common/unsafe/.../hash/Murmur3_x86_32.java), whatever the precision and scale."""
    vals = np.array([0, 1, -1, 123456, -(10 ** 18 - 1), 10 ** 18 - 1], np.int64)
    for prec, scale in ((7, 2), (18, 0), (18, 6)):
        small = vals if prec == 18 else np.array([0, 1, -1, 123456, -9999999, 9999999], np.int64)
        t = pa.table({"k": make_array(pa.decimal128(prec, scale), small)})
        want = [O.lib().so_murmur3_long(int(x), 42) for x in small]
        assert O.hash_rows(t, ["k"]).tolist() == want
        assert O.hash_rows(t, ["k"]).tolist() == O.hash_rows(pa.table({"k": pa.array(small)}), ["k"]).tolist()


def test_sort_order_of_nan_infinities_and_signed_zeros():
    """SQLOrderingUtil.compareDoubles / DoublePrefixComparator: -inf < -1 < -0.0 == 0.0 < 1 < inf < NaN, every NaN payload one
    value; ties keep their arrival order."""
    v = _f64([F64_NAN_BITS[1], 0x7FF0000000000000, 1 << 63, 0xBFF0000000000000, 0, F64_NAN_BITS[2], 0xFFF0000000000000, 0x3FF0000000000000])
    t = pa.table({"k": make_array("float64", v), "row": pa.array(range(8))})
    asc = O.sort(t, [("k", True, True)]).column("row").to_pylist()
    assert asc == [6, 3, 2, 4, 7, 1, 0, 5]
    assert O.sort(t, [("k", False, False)]).column("row").to_pylist() == [0, 5, 1, 7, 2, 4, 3, 6]
    assert O.take_ordered(t, [("k", True, True)], 8).column("row").to_pylist() == asc
    assert O.take_ordered(t.append_column("g", pa.array([0] * 8)), [("g", True, True), ("k", True, True)], 8).column("row").to_pylist() == asc
    v32 = _f32([F32_NAN_BITS[1], 0x7F800000, 0x80000000, 0, 0xFF800000])
    t32 = pa.table({"k": make_array("float32", v32), "row": pa.array(range(5))})
    assert O.sort(t32, [("k", True, True)]).column("row").to_pylist() == [4, 2, 3, 1, 0]
