"""GPU parity for every fixed-width key type and key layout: joins, grouping, hash and range partitioning, sort and top-N,
compared with the oracle BIT FOR BIT.

Every operator turns its key columns into machine words first (join.cu packing / hashing, the aggregate's packed and wide
layouts, the Murmur3 partition hash, the order-preserving sort key), and a wrong word gives a wrong answer quietly.  The data
of every type holds its extremes (MIN, MAX, -1 -- which is also the aggregate table's EMPTY sentinel 0xFF..FF -- and 0), NULLs
and, for floats, +-0.0, +-inf and NaNs with several payloads and both signs.  `assert_bits_equal` compares the raw values and
validity of every column, so -0.0 is not 0.0 and one NaN payload is not another: key columns that come out of an aggregate
must be normalised (NormalizeFloatingNumbers), columns that pass through a join must keep their original bits.
"""
import zlib

import numpy as np
import pyarrow as pa
import pytest

from oracle import oracle as O

pytestmark = pytest.mark.gpu

# ------------------------------------------------------------------------------------------------ data
TYPES = {"bool": pa.bool_(), "int8": pa.int8(), "int16": pa.int16(), "int32": pa.int32(), "int64": pa.int64(),
         "date32": pa.date32(), "timestamp": pa.timestamp("us"), "dec7_2": pa.decimal128(7, 2), "dec18_0": pa.decimal128(18, 0),
         "float32": pa.float32(), "float64": pa.float64()}
TYPE_NAMES = list(TYPES)
_STORAGE = {"bool": np.uint8, "int8": np.int8, "int16": np.int16, "int32": np.int32, "int64": np.int64, "date32": np.int32,
            "timestamp": np.int64, "dec7_2": np.int64, "dec18_0": np.int64, "float32": np.float32, "float64": np.float64}

F64_NAN_BITS = [0x7FF8000000000000, 0xFFF8000000000000, 0x7FF0000000000001, 0x7FF4000000000000, 0xFFFFFFFFFFFFFFFF]
F32_NAN_BITS = [0x7FC00000, 0xFFC00000, 0x7F800001, 0x7FC00001, 0xFFFFFFFF]


def _f64(bits):
    return np.array(bits, dtype=np.uint64).view(np.float64)


def _f32(bits):
    return np.array(bits, dtype=np.uint32).view(np.float32)


def specials(tname):
    """The values of a type every data set contains: extremes, -1 (the EMPTY sentinel's bit pattern), 0, and for floats
    signed zeros, infinities and NaN payloads of both signs."""
    if tname == "bool":
        return np.array([0, 1], np.uint8)
    if tname in ("dec7_2", "dec18_0"):
        top = 10 ** (7 if tname == "dec7_2" else 18) - 1
        return np.array([-top, top, -1, 0, 1, -top + 1], np.int64)
    if tname == "float64":
        fin = np.array([0.0, -0.0, np.inf, -np.inf, -1.0, 1.0, np.finfo(np.float64).max, -np.finfo(np.float64).max, 5e-324, -5e-324])
        return np.concatenate([fin, _f64(F64_NAN_BITS)])
    if tname == "float32":
        fin = np.array([0.0, -0.0, np.inf, -np.inf, -1.0, 1.0, np.finfo(np.float32).max, -np.finfo(np.float32).max, 1e-45, -1e-45],
                       np.float32)
        return np.concatenate([fin, _f32(F32_NAN_BITS)])
    info = np.iinfo(_STORAGE[tname])
    return np.array([info.min, info.max, -1, 0, 1, info.min + 1, info.max - 1], _STORAGE[tname])


def pool(tname, m, rng):
    """`m` distinct-ish values of a type: its specials first, then random ones (floats: quarter-integers, so that the
    random part of a data set still repeats)."""
    sp = specials(tname)
    k = max(0, m - len(sp))
    if tname == "bool":
        rnd = np.zeros(0, np.uint8)
    elif tname in ("float32", "float64"):
        rnd = (rng.integers(-4000, 4000, k) / 4.0).astype(_STORAGE[tname])
    elif tname == "dec7_2":
        rnd = rng.integers(-10 ** 7 + 1, 10 ** 7, k)
    elif tname == "dec18_0":
        rnd = rng.integers(-10 ** 18 + 1, 10 ** 18, k)
    else:
        info = np.iinfo(_STORAGE[tname])
        rnd = rng.integers(int(info.min), int(info.max), k, dtype=np.int64, endpoint=True)
    return np.concatenate([sp, rnd.astype(_STORAGE[tname])])


def make_array(tname, values, valid=None):
    """Arrow array of a type from storage values (unscaled longs for decimals, days / microseconds for dates and timestamps),
    built from buffers so that every bit -- NaN payloads included -- arrives as given."""
    t = TYPES[tname] if isinstance(tname, str) else tname
    values = np.asarray(values)
    n = len(values)
    vb = None if valid is None or bool(np.all(valid)) else pa.py_buffer(np.packbits(np.asarray(valid, bool), bitorder="little").tobytes())
    if pa.types.is_boolean(t):
        return pa.array(values.astype(bool), mask=None if vb is None else ~np.asarray(valid, bool))
    if pa.types.is_decimal(t):
        wide = np.empty((n, 2), np.int64)
        wide[:, 0] = values.astype(np.int64)
        wide[:, 1] = wide[:, 0] >> 63
        return pa.Array.from_buffers(t, n, [vb, pa.py_buffer(wide.tobytes())])
    return pa.Array.from_buffers(t, n, [vb, pa.py_buffer(np.ascontiguousarray(values).tobytes())])


def key_column(tname, n, rng, null_frac=0.05, m=300, values=None):
    """n keys drawn from pool(tname, m) (or from `values`), every special present at least once, NULLs at null_frac."""
    src = pool(tname, m, rng) if values is None else values
    v = src[rng.integers(0, len(src), n)]
    head = min(n, len(src))
    v[:head] = src[:head]
    valid = rng.random(n) >= null_frac if null_frac else None
    if valid is not None:
        valid[:min(n, 2 * len(specials(tname)))] = True
    return make_array(tname, v, valid)


# ------------------------------------------------------------------------------------------------ bit-exact comparison
def raw_bits(arr):
    """(valid bool[n], [uint64[n] words]) of an Arrow column: the raw value bits (NULL slots zeroed), decimals as two words."""
    if isinstance(arr, pa.ChunkedArray):
        arr = arr.combine_chunks() if arr.num_chunks != 1 else arr.chunk(0)
    n, t = len(arr), arr.type
    valid = np.asarray(arr.is_valid()) if arr.null_count else np.ones(n, bool)
    if pa.types.is_boolean(t):
        words = [np.asarray(arr.fill_null(False)).astype(np.uint64)]
    elif pa.types.is_decimal(t):
        w = np.frombuffer(arr.buffers()[1], np.uint64, count=2 * (arr.offset + n))[2 * arr.offset:].reshape(n, 2)
        words = [w[:, 0].copy(), w[:, 1].copy()]
    else:
        dt = {1: np.uint8, 2: np.uint16, 4: np.uint32, 8: np.uint64}[t.bit_width // 8]
        words = [np.frombuffer(arr.buffers()[1], dt, count=arr.offset + n)[arr.offset:].astype(np.uint64)]
    for w in words:
        w[~valid] = 0
    return valid, words


def _flat(table):
    cols = []
    for i in range(table.num_columns):
        valid, words = raw_bits(table.column(i))
        cols.append((table.column_names[i], valid, words))
    return cols


def assert_bits_equal(got, want, ordered=False, check_types=True):
    """Tables equal bit for bit: same column types, row count, validity and raw value bits.  Unordered: both sides are
    sorted by every column's bits first (a multiset comparison, like checkAnswer's, but exact)."""
    assert got.num_columns == want.num_columns, (got.schema, want.schema)
    if check_types:
        for i in range(want.num_columns):
            assert got.schema.field(i).type == want.schema.field(i).type, \
                "column %d (%s): type %s != %s" % (i, want.column_names[i], got.schema.field(i).type, want.schema.field(i).type)
    assert got.num_rows == want.num_rows, "row count %d != %d" % (got.num_rows, want.num_rows)
    g, w = _flat(got), _flat(want)
    if not ordered and want.num_rows > 1:
        def order(cols):
            keys = []
            for _, valid, words in cols:
                keys.append(valid)
                keys.extend(words)
            return np.lexsort(keys[::-1])
        gp, wp = order(g), order(w)
    else:
        gp = wp = np.arange(want.num_rows)
    for (name, gv, gw), (_, wv, ww) in zip(g, w):
        gv, wv = gv[gp], wv[wp]
        bad = np.nonzero(gv != wv)[0]
        assert len(bad) == 0, "column %s row %d: valid %s vs %s" % (name, bad[0], gv[bad[0]], wv[bad[0]])
        for a, b in zip(gw, ww):
            a, b = a[gp], b[wp]
            bad = np.nonzero(a != b)[0]
            assert len(bad) == 0, "column %s row %d: bits %#x vs %#x (%d rows differ)" % (name, bad[0], int(a[bad[0]]), int(b[bad[0]]), len(bad))


# ------------------------------------------------------------------------------------------------ runners
def _seed(*parts):
    return zlib.crc32(repr(parts).encode())


def distinct(vals):
    """The values of `vals` with distinct bit patterns, first occurrences in order (so -0.0 / 0.0 and NaN payloads all stay)."""
    u = np.ascontiguousarray(vals).view({1: np.uint8, 2: np.uint16, 4: np.uint32, 8: np.uint64}[vals.dtype.itemsize])
    return vals[np.sort(np.unique(u, return_index=True)[1])]


def _batch(t, stream):
    from spark_b200.columnar import ColumnarBatch
    return ColumnarBatch.from_arrow(t, stream)


def _misaligned_device_batch(table):
    """A NULL-free fixed-width table borrowed from device memory (sb_table_import_device) with every column starting one
    element past a 256-byte-aligned allocation, so no data pointer is 16-byte aligned.  Returns (batch, buffers to keep alive)."""
    import ctypes as C
    import torch
    from spark_b200 import _capi as capi
    from spark_b200.columnar import ColumnarBatch, HostColumn
    cols, keep = (capi.sb_column * table.num_columns)(), []
    for i in range(table.num_columns):
        h = HostColumn.from_arrow(table.column(i))
        assert h.validity is None and h.offsets is None
        raw = np.ascontiguousarray(h.data).view(np.uint8)
        w = h.data.dtype.itemsize
        buf = torch.zeros(len(raw) + 2 * w, dtype=torch.uint8, device="cuda")
        buf[w:w + len(raw)] = torch.from_numpy(raw.copy()).cuda()   # a writable copy: Arrow buffers are read-only
        keep.append(buf)
        cols[i] = h.c()
        cols[i].data = buf.data_ptr() + w
    torch.cuda.synchronize()
    out = C.c_void_p()
    capi.check(capi.load().sb_table_import_device(cols, table.num_columns, C.byref(out)))
    batch = ColumnarBatch(out, table.column_names, [f.type for f in table.schema])
    for i in range(table.num_columns):
        assert batch.column_desc(i).data % 16 != 0
    return batch, keep


def _gpu_join(probe, build, pk, bk, how, stream, misaligned=False):
    from spark_b200.execution import BroadcastHashJoinExec, LocalTableScanExec
    pb, keep = _misaligned_device_batch(probe) if misaligned else (_batch(probe, stream), None)
    bb = _batch(build, stream)
    try:
        return BroadcastHashJoinExec(pk, bk, how, "right", LocalTableScanExec(pb), LocalTableScanExec(bb)).collect(stream)
    finally:
        pb.close()
        del keep


def _check_join(probe, build, pk, bk, how, stream, misaligned=False):
    got = _gpu_join(probe, build, pk, bk, how, stream, misaligned)
    want = O.hash_join(probe, build, pk, bk, how)
    assert_bits_equal(got, want)
    return got


HOWS = ["inner", "left_outer", "left_semi", "left_anti", "full_outer", "existence"]
CAND_N = (1 << 20) + 13          # >= 2^20 streamed rows take the candidate pass; not a multiple of 16 or 32 (ragged tail)


# ------------------------------------------------------------------------------------------------ joins
@pytest.mark.parametrize("how", HOWS)
@pytest.mark.parametrize("tname", TYPE_NAMES)
def test_join_single_key_short_streamed_side(gpu, stream, tname, how):
    """Every type as the only key, NULLs and duplicates on both sides: -0.0 meets 0.0, NaN meets NaN whatever its payload
    (NormalizeFloatingNumbers on join keys), and the output keeps each side's own bits."""
    rng = np.random.default_rng(TYPE_NAMES.index(tname) * 10 + HOWS.index(how))
    vals = pool(tname, 200, rng)
    probe = pa.table({"k": key_column(tname, 4000, rng, values=vals), "p": np.arange(4000, dtype=np.int64)})
    nb = 60 if tname == "bool" else 1500
    build = pa.table({"k2": key_column(tname, nb, rng, values=vals[::-1].copy()), "b": np.arange(nb, dtype=np.int32)})
    _check_join(probe, build, ["k"], ["k2"], how, stream)


@pytest.mark.parametrize("nullable", [False, True])
@pytest.mark.parametrize("variant", [0, 1])
@pytest.mark.parametrize("tname", TYPE_NAMES)
def test_join_single_key_candidate_pass(gpu, stream, sbconfig, tname, variant, nullable):
    """The candidate pass over 2^20 + 13 streamed rows, both geometries (`join_cand` 0: 16-row fast_key loads for NULL-free
    integer keys; 1: lane-strided, KW 8 / 4 / general).  NULL-free keys also run over a probe borrowed from device memory one
    element past an aligned allocation: its key column is not 16-byte aligned, so fast_key's 16-byte loads must not be used."""
    sbconfig("join_cand", variant)
    rng = np.random.default_rng(1000 + TYPE_NAMES.index(tname) * 4 + variant * 2 + nullable)
    vals = pool(tname, 3000, rng)
    # one build row per bit pattern (bool / int8 have few values): an integer key has at most one partner; -0.0 / 0.0 and the NaN
    # payloads stay separate rows, which normalisation makes duplicate keys
    bk = distinct(vals[:1500])
    build = pa.table({"k2": key_column(tname, len(bk), rng, null_frac=0.02 if nullable else 0, values=bk),
                      "b": np.arange(len(bk), dtype=np.int64)})
    probe = pa.table({"k": key_column(tname, CAND_N, rng, null_frac=0.03 if nullable else 0, values=vals), "p": np.arange(CAND_N, dtype=np.int64)})
    hows = ["inner", "left_anti"] + (["left_semi", "left_outer", "full_outer"] if tname in ("int32", "float32", "float64", "dec18_0") else [])
    for how in hows:
        _check_join(probe, build, ["k"], ["k2"], how, stream)
    if not nullable:
        _check_join(probe, build, ["k"], ["k2"], "inner", stream, misaligned=True)


def _shape_keys(shape, tname, rng):
    """Build keys for each relation shape: dense unique keys (direct-address table), strictly ascending keys (sorted rank mode,
    int32 crossing zero), duplicates (bitmap + slot table) and sparse keys (Bloom filter)."""
    info = np.iinfo(_STORAGE[tname])
    if shape == "dense":
        return rng.permutation(np.arange(-3000, 3000)).astype(_STORAGE[tname])
    if shape == "sorted":
        return np.sort(rng.choice(np.arange(-200_000, 200_000), 6000, replace=False)).astype(_STORAGE[tname])
    if shape == "dups":
        k = rng.integers(-5000, 5000, 6000)
        k[:500] = k[500:1000]
        return k.astype(_STORAGE[tname])
    k = rng.integers(int(info.min), int(info.max), 6000, dtype=np.int64, endpoint=True).astype(_STORAGE[tname])
    k[:4] = [info.min, info.max, -1, 0]
    return k


@pytest.mark.parametrize("shape", ["dense", "sorted", "dups", "sparse"])
@pytest.mark.parametrize("tname", ["int32", "int64", "date32", "timestamp", "dec18_0"])
def test_join_build_shapes(gpu, stream, tname, shape):
    rng = np.random.default_rng(_seed((tname, shape)))
    bk = _shape_keys(shape, tname, rng)
    build = pa.table({"k2": make_array(tname, bk), "b": np.arange(len(bk), dtype=np.int64)})
    near = bk[rng.integers(0, len(bk), CAND_N)]
    far = _shape_keys("sparse", tname, rng)[rng.integers(0, 6000, CAND_N)]
    pk = np.where(rng.random(CAND_N) < 0.5, near, far)
    for valid, hows in ((None, ("inner", "left_outer", "left_anti")), (rng.random(CAND_N) >= 0.02, ("inner", "left_anti"))):
        probe = pa.table({"k": make_array(tname, pk, valid), "p": np.arange(CAND_N, dtype=np.int64)})
        for how in hows:
            _check_join(probe, build, ["k"], ["k2"], how, stream)
    _check_join(pa.table({"k": make_array(tname, pk[:5000]), "p": np.arange(5000, dtype=np.int64)}), build, ["k"], ["k2"], "inner", stream)


@pytest.mark.parametrize("span,ascending", [((1 << 23) - 1, False), (1 << 23, False), ((1 << 30) - 1, True), (1 << 30, True)])
def test_join_exact_bitmap_limits(gpu, stream, span, ascending):
    """Relations whose key range is just inside and just outside the exact bitmap's limits (2^23 for any keys, 2^30 for
    ascending sparse ones): both sides of each limit must give the same answer.  The bitmap's overall cap of 2^31 is reached
    only by a relation of about 2^25 dense-enough keys (64 range per key) and is not tested here."""
    rng = np.random.default_rng(span)
    mid = np.unique(rng.integers(1, span, 3000))
    bk = np.concatenate([[-7], mid - 7, [span - 7]]).astype(np.int64)    # range = span + 1 keys
    if not ascending:
        bk = rng.permutation(bk)
    build = pa.table({"k2": bk, "b": np.arange(len(bk), dtype=np.int64)})
    pk = np.where(rng.random(CAND_N) < 0.5, bk[rng.integers(0, len(bk), CAND_N)], rng.integers(-20, span + 20, CAND_N))
    probe = pa.table({"k": pk, "p": np.arange(CAND_N, dtype=np.int64)})
    for how in ("inner", "left_semi", "left_anti"):
        _check_join(probe, build, ["k"], ["k2"], how, stream)


PACKED = {
    "i32_i32": ["int32", "int32"],                          # exactly 64 packed bits, negative values in both fields
    "i32_i16_i8_bool": ["int32", "int16", "int8", "bool"],  # exactly 64 packed bits
    "f32_i32": ["float32", "int32"],                        # a float inside a packed word
    "i16_i32": ["int16", "int32"],                          # fields of two widths, negative values in both
    "f64_i64": ["float64", "int64"],                        # wide (hash + verify) with a float column
    "i64_f64_i32": ["int64", "float64", "int32"],
}


@pytest.mark.parametrize("n", [20_000, CAND_N])
@pytest.mark.parametrize("layout", list(PACKED))
def test_join_multi_key_layouts(gpu, stream, layout, n):
    """Multi-column keys: packed into one word up to 64 bits, hashed and verified above.  Streamed rows are build rows with
    one column changed to another pool value, so keys agree on every column but one."""
    types = PACKED[layout]
    rng = np.random.default_rng(_seed((layout, n)))
    nb = 3000
    pools = [pool(t, 40, rng) for t in types]
    bcols = [p[rng.integers(0, len(p), nb)] for p in pools]
    pick = rng.integers(0, nb, n)
    pcols = [c[pick].copy() for c in bcols]
    change = rng.integers(-1, len(types), n)                 # -1: the row is a build key as it is
    for i, p in enumerate(pools):
        sel = change == i
        pcols[i][sel] = p[rng.integers(0, len(p), int(sel.sum()))]
    bnames = ["b%d" % i for i in range(len(types))]
    pnames = ["p%d" % i for i in range(len(types))]
    build = pa.table({**{nm: make_array(t, c) for nm, t, c in zip(bnames, types, bcols)}, "brow": np.arange(nb, dtype=np.int64)})
    pvalid = rng.random(n) >= 0.02
    probe = pa.table({**{nm: make_array(t, c, pvalid if i == 0 else None) for i, (nm, t, c) in enumerate(zip(pnames, types, pcols))},
                      "prow": np.arange(n, dtype=np.int64)})
    for how in ("inner", "left_anti", "left_outer") if n > 20_000 else HOWS:
        _check_join(probe, build, pnames, bnames, how, stream)


@pytest.mark.parametrize("ptype,btype", [("date32", "date32"), ("timestamp", "timestamp"), (pa.decimal128(12, 2), pa.decimal128(7, 2)),
                                         ("dec18_0", "dec18_0")])
def test_inner_join_build_key_column_keeps_its_type(gpu, stream, ptype, btype):
    """A unique dense relation settles the inner join in the candidate pass, and the build side's key column is then taken
    from the streamed key column: it must keep the BUILD column's type, precision and scale."""
    rng = np.random.default_rng(77)
    bk = rng.permutation(np.arange(-20_000, 20_000)).astype(np.int64)
    if btype == "date32":
        bk = bk.astype(np.int32)
    build = pa.table({"k2": make_array(btype, bk), "b": np.arange(len(bk), dtype=np.int64)})
    pk = rng.integers(-25_000, 25_000, CAND_N).astype(bk.dtype)
    probe = pa.table({"k": make_array(ptype, pk), "p": np.arange(CAND_N, dtype=np.int64)})
    got = _check_join(probe, build, ["k"], ["k2"], "inner", stream)
    assert got.schema.field("k2").type == build.schema.field("k2").type


# ------------------------------------------------------------------------------------------------ grouping
AGG_ENVS = [{"agg_tier": 1, "agg_rtc_min_rows": 0}, {"agg_tier": 2, "agg_rtc_min_rows": 0}, {"agg_rtc": 0}, {"agg_rtc_min_rows": 0}]
AGG_ENV_IDS = ["tier1", "tier2", "generic", "rtc"]


def _aggs():
    from spark_b200.expressions import Count, Min, Sum, col
    return [(Count(), "n"), (Sum(col("v")), "s"), (Min(col("v")), "mn")]


_OAGGS = [("count_star", None, "n"), ("sum", "v", "s"), ("min", "v", "mn")]


def _check_group(t, keys, stream, sbconfig, env):
    from spark_b200.execution import HashAggregateExec, LocalTableScanExec
    for k, v in env.items():
        sbconfig(k, v)
    got = HashAggregateExec(keys, _aggs(), LocalTableScanExec(_batch(t, stream))).collect(stream)
    want = O.hash_aggregate(t, keys, _OAGGS)
    assert_bits_equal(got, want)
    return got


@pytest.mark.parametrize("env", AGG_ENVS, ids=AGG_ENV_IDS)
@pytest.mark.parametrize("tname", TYPE_NAMES)
def test_group_by_single_key(gpu, stream, sbconfig, tname, env):
    """Every type as the only grouping key; keys come out normalised (-0.0 as 0.0, every NaN as the canonical NaN)."""
    rng = np.random.default_rng(2000 + TYPE_NAMES.index(tname))
    n = 50_000
    t = pa.table({"k": key_column(tname, n, rng, m=500), "v": rng.integers(-100, 100, n)})
    got = _check_group(t, ["k"], stream, sbconfig, env)
    if tname in ("float32", "float64"):
        valid, (w,) = raw_bits(got.column("k"))
        canon = 0x7FC00000 if tname == "float32" else 0x7FF8000000000000
        negzero = 0x80000000 if tname == "float32" else 0x8000000000000000
        vals = got.column("k").to_numpy(zero_copy_only=False)
        assert not np.any(w == negzero) and np.all(w[valid & np.isnan(vals)] == canon)
        assert np.count_nonzero(valid & np.isnan(vals)) == 1 and np.count_nonzero(valid & (vals == 0)) == 1


def _i64_pool():
    return np.array([np.iinfo(np.int64).min, -1, np.iinfo(np.int64).max, 0, 1, -(1 << 62), 1 << 62, np.iinfo(np.int64).min + 1], np.int64)


LAYOUTS = {   # (types, nullable flags): what the aggregate's key packing makes of them
    "packed_56_3flags": (["int32", "int16", "int8"], [True, True, True]),                   # 59 bits: one packed word
    "packed_62": (["int16", "int8", "int8", "int8", "int8", "int8"], [True] * 6),          # 62 bits: the widest packed layout
    "wide_64": (["int32", "int16", "int8", "bool"], [False] * 4),                           # 64 bits: two words
    "wide_65": (["int32", "int32"], [True, False]),                                         # 65 bits
    "two_words_i64": (["int64", "int32"], [True, True]),                                    # bit 63 spills into word 1
    "two_words_f64_f32": (["float64", "float32", "int8"], [True, True, False]),
    "three_words": (["int64", "int64", "int32"], [True, False, True]),
    "four_words": (["int64", "int64", "int64", "int32"], [True, True, True, False]),
    "four_words_f64": (["float64", "int64", "timestamp", "int16"], [False, False, False, True]),
}


@pytest.mark.parametrize("env", AGG_ENVS, ids=AGG_ENV_IDS)
@pytest.mark.parametrize("layout", list(LAYOUTS))
def test_group_by_key_layouts(gpu, stream, sbconfig, layout, env):
    """Grouping keys at every packing boundary and word count (AGG_MAX_WORDS = 4); 64-bit keys take values with bit 63 set
    (INT64_MIN, -1) next to INT64_MAX, which must stay distinct groups."""
    types, nullable = LAYOUTS[layout]
    rng = np.random.default_rng(_seed(layout))
    n = 40_000
    cols = {}
    for i, (tn, nl) in enumerate(zip(types, nullable)):
        vals = _i64_pool() if tn == "int64" else pool(tn, 6, rng)
        cols["k%d" % i] = key_column(tn, n, rng, null_frac=0.05 if nl else 0, values=vals)
    cols["v"] = rng.integers(-100, 100, n)
    t = pa.table(cols)
    _check_group(t, list(cols)[:-1], stream, sbconfig, env)


def test_group_by_keys_beyond_four_words_is_refused(gpu, stream):
    """Four nullable int64 keys and one more need a fifth 63-bit word: refused with SB_ERR_UNSUPPORTED, not answered."""
    from spark_b200 import _capi as capi
    from spark_b200.execution import HashAggregateExec, LocalTableScanExec
    rng = np.random.default_rng(5)
    n = 1000
    cols = {"k%d" % i: key_column("int64", n, rng, values=_i64_pool()) for i in range(4)}
    cols["k4"] = key_column("int8", n, rng)
    cols["v"] = rng.integers(0, 10, n)
    t = pa.table(cols)
    with pytest.raises(capi.SparkB200Error) as e:
        HashAggregateExec(["k0", "k1", "k2", "k3", "k4"], _aggs(), LocalTableScanExec(_batch(t, stream))).collect(stream)
    assert e.value.code == 5      # SB_ERR_UNSUPPORTED


@pytest.mark.parametrize("keys", [["float64"], ["float32", "int64"], ["int64", "float64", "dec7_2"]])
def test_group_by_partial_then_final(gpu, stream, keys):
    """Partial aggregation of two halves, then Final over their concatenation: the normalised keys of one half must meet the
    other half's -- the Final stage groups keys that the Partial stages already normalised."""
    from spark_b200.columnar import ColumnarBatch
    from spark_b200.execution import HashAggregateExec, LocalTableScanExec
    rng = np.random.default_rng(len(keys))
    n = 30_000
    cols = {"k%d" % i: key_column(tn, n, rng, values=_i64_pool() if tn == "int64" else pool(tn, 20, rng)) for i, tn in enumerate(keys)}
    cols["v"] = rng.integers(-100, 100, n)
    t = pa.table(cols)
    names = list(cols)[:-1]
    parts = []
    for half in (t.slice(0, n // 2), t.slice(n // 2)):
        parts.append(HashAggregateExec(names, _aggs(), LocalTableScanExec(_batch(half, stream)), mode="partial").collect(stream))
    both = pa.concat_tables(parts)
    got = HashAggregateExec(names, _aggs(), LocalTableScanExec(ColumnarBatch.from_arrow(both, stream)), mode="final").collect(stream)
    assert_bits_equal(got, O.hash_aggregate(t, names, _OAGGS))


# ------------------------------------------------------------------------------------------------ hash partitioning
@pytest.mark.parametrize("nparts", [1, 200, 2048])
@pytest.mark.parametrize("tname", TYPE_NAMES)
def test_hash_partition_ids(gpu, stream, tname, nparts):
    """Pmod(Murmur3Hash(key, 42), n) for every type: decimal(p <= 18) hashes its unscaled long, -0.0 hashes as 0.0 and every
    NaN as the canonical one."""
    from spark_b200.execution import HashPartitioning, LocalTableScanExec, ShuffleExchangeExec
    rng = np.random.default_rng(3000 + TYPE_NAMES.index(tname))
    t = pa.table({"k": key_column(tname, 30_000, rng, m=2000)})
    b = _batch(t, stream)
    pids = ShuffleExchangeExec(HashPartitioning(["k"], nparts), LocalTableScanExec(b)).partition_ids(b, stream)
    want = O.partition_ids(t, ["k"], nparts)
    assert np.array_equal(pids, want), np.nonzero(pids != want)[0][:10]


def test_hash_partition_all_types_together(gpu, stream):
    from spark_b200.execution import HashPartitioning, LocalTableScanExec, ShuffleExchangeExec
    rng = np.random.default_rng(31)
    t = pa.table({tn: key_column(tn, 20_000, rng, m=100) for tn in TYPE_NAMES})
    b = _batch(t, stream)
    for keys in (TYPE_NAMES[:8], TYPE_NAMES[3:]):        # at most 8 partitioning keys
        ex = ShuffleExchangeExec(HashPartitioning(keys, 200), LocalTableScanExec(b))
        assert np.array_equal(ex.partition_ids(b, stream), O.partition_ids(t, keys, 200))
        got = ex.executeColumnar(stream).to_arrow(stream)
        want, offs = O.hash_partition(t, keys, 200)
        assert np.array_equal(ex.partition_offsets, offs)
        assert_bits_equal(got, want, ordered=True)


# ------------------------------------------------------------------------------------------------ sort and top-N
@pytest.mark.parametrize("asc", [True, False])
@pytest.mark.parametrize("nullable", [False, True])
@pytest.mark.parametrize("tname", ["int8", "int16", "timestamp", "dec7_2", "dec18_0", "float32", "float64"])
def test_sort_single_column(gpu, stream, tname, nullable, asc):
    """Single-column sorts; NULL-free integer-like keys rebuild the sorted key column from the sorted keys (unkey_kernel), and
    that column must be bit-exact.  Float keys: -0.0 and 0.0 are ties kept in arrival order, every NaN sorts last as one value."""
    from spark_b200.execution import LocalTableScanExec, SortExec
    rng = np.random.default_rng(_seed((tname, nullable, asc)))
    n = 50_000
    t = pa.table({"k": key_column(tname, n, rng, null_frac=0.1 if nullable else 0, m=3000), "row": np.arange(n, dtype=np.int64)})
    got = SortExec([("k", asc, True)], LocalTableScanExec(_batch(t, stream))).collect(stream)
    assert_bits_equal(got, O.sort(t, [("k", asc, True)]), ordered=True)


TOPN_TYPES = ["float64", "float32", "int8", "bool", "date32", "dec18_0"]


@pytest.mark.parametrize("asc", [True, False])
@pytest.mark.parametrize("n,k", [(65536, 8192), (65536, 8193), (65537, 8192), (65537, 8193)])
@pytest.mark.parametrize("tname", TOPN_TYPES)
def test_top_n_against_take_ordered(gpu, stream, tname, n, k, asc):
    """TakeOrderedAndProject against the oracle's full stable ordering.  The radix select runs only when n > 65536 and
    k * 8 <= n: these four shapes sit on both sides of both conditions."""
    from spark_b200.execution import LocalTableScanExec, TakeOrderedAndProjectExec
    from spark_b200.expressions import SortOrder
    rng = np.random.default_rng(_seed((tname, n, k, asc)))
    t = pa.table({"k": key_column(tname, n, rng, null_frac=0, m=500), "row": np.arange(n, dtype=np.int64)})
    got = TakeOrderedAndProjectExec(k, [SortOrder("k", asc)], None, LocalTableScanExec(_batch(t, stream))).collect(stream)
    assert_bits_equal(got, O.take_ordered(t, [("k", asc, True)], k), ordered=True)


@pytest.mark.parametrize("case", ["tie_run", "constant_first_key"])
@pytest.mark.parametrize("tname", ["float64", "int64", "dec18_0"])
def test_top_n_ties(gpu, stream, tname, case):
    """k lands inside a long run of equal first keys (the select narrows to that one key: the rows equal to the bound must be
    kept), and a first key that is the same on every row (the select loop runs all 8 bytes)."""
    from spark_b200.execution import LocalTableScanExec, TakeOrderedAndProjectExec
    from spark_b200.expressions import SortOrder
    rng = np.random.default_rng(_seed((tname, case)))
    n = 200_003
    vals = pool(tname, 50, rng)
    v = vals[rng.integers(0, len(vals), n)]
    run = vals[3]
    if case == "tie_run":
        v[rng.random(n) < 0.7] = run
    else:
        v[:] = run
    t = pa.table({"k": make_array(tname, v), "g": rng.integers(0, 5, n), "row": np.arange(n, dtype=np.int64)})
    for k in (20_000, n // 8, n // 8 + 1):
        for orders in ([("k", True, True)], [("k", False, True), ("g", True, True)]):
            got = TakeOrderedAndProjectExec(k, [SortOrder(*o) for o in orders], None, LocalTableScanExec(_batch(t, stream))).collect(stream)
            assert_bits_equal(got, O.take_ordered(t, orders, k), ordered=True)


@pytest.mark.parametrize("asc,nulls_first", [(True, True), (False, False)])
@pytest.mark.parametrize("tname", ["int8", "int16", "int32", "float32", "timestamp", "dec7_2"])
def test_range_partition(gpu, stream, tname, asc, nulls_first):
    """RangePartitioner.getPartition over the remaining radix types, with NULL and NaN among the bounds."""
    from spark_b200.execution import LocalTableScanExec, RangePartitioning, ShuffleExchangeExec
    rng = np.random.default_rng(_seed((tname, asc)))
    n = 40_000
    t = pa.table({"k": key_column(tname, n, rng, null_frac=0.1, m=1000), "row": np.arange(n, dtype=np.int64)})
    sample = pa.table({"k": pa.concat_arrays([t.column("k").combine_chunks().slice(0, 40), pa.nulls(1, TYPES[tname])])})
    bounds_t = O.sort(sample, [("k", asc, nulls_first)])
    ex = ShuffleExchangeExec(RangePartitioning(("k", asc, nulls_first), _batch(bounds_t, stream)), LocalTableScanExec(_batch(t, stream)))
    got = ex.executeColumnar(stream).to_arrow(stream)
    want, offs = O.range_partition(t, ("k", asc, nulls_first), bounds_t.column("k").combine_chunks())
    assert np.array_equal(ex.partition_offsets, offs)
    assert_bits_equal(got, want, ordered=True)
