"""GPU parity for every path that carries columns to their new rows, over every column type, BIT FOR BIT.

Every operator has two halves: what it computes from its keys, and moving the OTHER columns to their new rows unchanged.  The
second half is spread over several kernels that pick a path by column width, column count, alignment, bucket count and row
count: `gather_fixed_kernel` (one branch per width, groups of GATHER_MAX_COLS = 12 columns, validity by ballot, -1 -> NULL)
behind slice, sort, top-N, window, filter, expand and every join output; the shuffle's regroup (copy-engine kernel with 4096- or
8192-row tiles, load/store kernel, two-level split above 256 buckets, chunks of SCATTER_MAX_COLS = 16 columns, strings and
decimal128 by a row-id gather afterwards); and `sb_table_concat`.

Every operation here is a selection or a permutation of rows, so the reference is plain: an expected row index vector computed
on the host (-1 = NULL), applied with numpy `take` to the raw buffers of the input.  The comparison is on bits: values at valid
positions (NaN payloads and -0.0 kept), validity, string bytes and Arrow types (decimal precision and scale, timestamp unit).
"""
import functools
import zlib

import numpy as np
import pyarrow as pa
import pytest

from oracle import oracle as O
from test_gpu_key_types import CAND_N, _misaligned_device_batch, assert_bits_equal, make_array, raw_bits, specials
from test_gpu_round2 import one_rank_comm  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu

# ------------------------------------------------------------------------------------------------ data
TYPES = {"bool": pa.bool_(), "int8": pa.int8(), "int16": pa.int16(), "int32": pa.int32(), "int64": pa.int64(),
         "date32": pa.date32(), "timestamp": pa.timestamp("us"), "dec7_2": pa.decimal128(7, 2), "dec18_0": pa.decimal128(18, 0),
         "dec38_10": pa.decimal128(38, 10), "float32": pa.float32(), "float64": pa.float64()}
FIXED_TYPES = list(TYPES)
VARIANTS = ["t", "n", "a"]     # NULLs on tile edges + 5% random / no validity buffer / all NULL
TILE = 4096
TILE_NULLS = [0, 7, 8, 31, 32, 63]
# the fixed-width columns in table order: the row id, then every type once per validity variant (variant-major, so that the
# first 13 columns already hold every type)
ALL_FIXED = ["row"] + ["%s_%s" % (t, v) for v in VARIANTS for t in FIXED_TYPES]
STRINGS = ["str_%s" % v for v in VARIANTS]
WIDTHS = [12, 13, 16, 17, 25]  # fixed-width columns: both sides of GATHER_MAX_COLS = 12 and SCATTER_MAX_COLS = 16, and two groups

DEC38_TOP = 10 ** 38 - 1
# decimal(38, 10) specials as 128-bit integers: the extremes, high words 0 and -1, and values on both sides of the sign crossing
# of the low word (2^63) and of the high word (2^64)
DEC38_SPECIALS = [DEC38_TOP, -DEC38_TOP, 0, 1, -1, (1 << 63) - 1, 1 << 63, (1 << 64) - 1, 1 << 64, -(1 << 63), -(1 << 63) - 1,
                  -(1 << 64), -(1 << 64) + 1, DEC38_TOP - (1 << 64), -DEC38_TOP + (1 << 64)]
F64_SUBNORMALS = [0x000FFFFFFFFFFFFF, 0x800FFFFFFFFFFFFF, 0x0000000000000001, 0x8000000000000001]
F32_SUBNORMALS = [0x007FFFFF, 0x807FFFFF, 0x00000001, 0x80000001]


def _str_specials():
    """Strings at every edge a byte copy can get wrong: empty, embedded NUL, 1- to 4-byte UTF-8 sequences, byte lengths around
    4, 16 and 32, and one longer than 100 bytes."""
    out = ["", "\x00", "a\x00b", "\x00\x00\x00", "é", "€", "\U0001F600", "aé€\U0001F600"]
    for k in (1, 3, 4, 5, 15, 16, 17, 31, 32, 33):
        out.append("".join(chr(ord("a") + (i * 7 + k) % 26) for i in range(k)))
    out += ["é" * 8, "€" * 11, "\U0001F600" * 8 + "x", ("ab\x00€\U0001F600é" * 12)]    # 16, 33, 33 and 132 bytes
    return out


STR_SPECIALS = _str_specials()


def dec38_words(values):
    """(n, 2) int64 low / high words of 128-bit two's complement integers."""
    v = [int(x) & ((1 << 128) - 1) for x in values]
    lo = np.array([x & ((1 << 64) - 1) for x in v], np.uint64).view(np.int64)
    hi = np.array([x >> 64 for x in v], np.uint64).view(np.int64)
    return np.stack([lo, hi], axis=1)


def _fixed_values(tname, n, rng):
    """n storage values of a type: random bit patterns over the type's whole range with its specials at the head and
    scattered over the column.  decimal(38, 10): (n, 2) words."""
    if tname == "dec38_10":
        sp = dec38_words(DEC38_SPECIALS)
        w = np.empty((n, 2), np.int64)
        w[:, 0] = rng.integers(np.iinfo(np.int64).min, np.iinfo(np.int64).max, n, dtype=np.int64, endpoint=True)
        w[:, 1] = rng.integers(-(1 << 62), 1 << 62, n)      # |value| < 2^126 < 10^38 - 1
    else:
        sp = specials(tname)
        if tname == "float64":
            sp = np.concatenate([sp, np.array(F64_SUBNORMALS, np.uint64).view(np.float64)])
        elif tname == "float32":
            sp = np.concatenate([sp, np.array(F32_SUBNORMALS, np.uint32).view(np.float32)])
        if tname == "bool":
            w = rng.integers(0, 2, n).astype(np.uint8)
        elif tname in ("float32", "float64"):
            ut = np.uint32 if tname == "float32" else np.uint64
            w = rng.integers(0, np.iinfo(ut).max, n, dtype=ut, endpoint=True).view(sp.dtype)
        elif tname in ("dec7_2", "dec18_0"):
            top = 10 ** (7 if tname == "dec7_2" else 18) - 1
            w = rng.integers(-top, top, n, endpoint=True)
        else:
            info = np.iinfo(sp.dtype)
            w = rng.integers(int(info.min), int(info.max), n, dtype=np.int64, endpoint=True).astype(sp.dtype)
    if n:
        k = min(n, len(sp))
        w[:k] = sp[:k]
        spots = rng.integers(0, n, min(n, 8 * len(sp)))
        w[spots] = sp[np.arange(len(spots)) % len(sp)]
    return w


def validity(variant, n, rng):
    if variant == "n":
        return None
    if variant == "a":
        return np.zeros(n, bool)
    valid = rng.random(n) >= 0.05
    for p in TILE_NULLS:
        valid[p::TILE] = False
    return valid


def _array(tname, values, valid):
    if tname == "dec38_10":
        vb = None if valid is None or valid.all() else pa.py_buffer(np.packbits(valid, bitorder="little").tobytes())
        return pa.Array.from_buffers(TYPES[tname], len(values), [vb, pa.py_buffer(np.ascontiguousarray(values).tobytes())])
    return make_array(TYPES[tname], values, valid)


def _strings(n, rng):
    pool = np.array(STR_SPECIALS + ["s%d" % i for i in range(40)] + ["x" * k for k in range(2, 70, 3)], dtype=object)
    v = pool[rng.integers(0, len(pool), n)]
    k = min(n, len(STR_SPECIALS))
    v[:k] = STR_SPECIALS[:k]
    return v


@functools.lru_cache(maxsize=3)
def _full_table(n, seed):
    """Every column the tests draw from, n rows: `row` (int64 row id), every fixed-width type in each validity variant, a string
    column in each variant, `k` (NULL-free int32 sort key with ties), `g` (NULL-free int32 window partition) and `f` (int64
    filter input)."""
    rng = np.random.default_rng(seed)
    cols = {"row": pa.array(np.arange(n, dtype=np.int64))}
    for v in VARIANTS:
        for t in FIXED_TYPES:
            cols["%s_%s" % (t, v)] = _array(t, _fixed_values(t, n, rng), validity(v, n, rng))
    for v in VARIANTS:
        valid = validity(v, n, rng)
        cols["str_%s" % v] = pa.array(_strings(n, rng).tolist(), type=pa.string(), mask=None if valid is None else ~valid)
    cols["k"] = pa.array(rng.integers(-60, 60, n).astype(np.int32))
    cols["g"] = pa.array(np.sort(rng.integers(0, max(1, n // 300), n)).astype(np.int32)[rng.permutation(n)])
    cols["f"] = pa.array(rng.integers(0, 2, n).astype(np.int64))
    return pa.table(cols)


def fixed_names(width, dec128=True):
    names = [c for c in ALL_FIXED if dec128 or not c.startswith("dec38")]
    assert width <= len(names)
    return names[:width]


def wide_table(n, width=len(ALL_FIXED), strings=True, dec128=True, seed=1, extra=()):
    """`width` fixed-width columns (the row id first), optionally without decimal(38, 10), plus the three string columns."""
    names = fixed_names(width, dec128) + (STRINGS if strings else []) + list(extra)
    return _full_table(n, seed).select(names)


# ------------------------------------------------------------------------------------------------ reference and comparison
def _storage(arr):
    """Raw storage values of a fixed-width Arrow array: (n,) of the type's width, (n, 2) int64 for decimals, uint8 for bool."""
    n, t = len(arr), arr.type
    if pa.types.is_boolean(t):
        return np.asarray(arr.fill_null(False)).astype(np.uint8)
    if pa.types.is_decimal(t):
        return np.frombuffer(arr.buffers()[1], np.int64, count=2 * (arr.offset + n))[2 * arr.offset:].reshape(n, 2)
    dt = {1: np.uint8, 2: np.uint16, 4: np.uint32, 8: np.uint64}[t.bit_width // 8]
    return np.frombuffer(arr.buffers()[1], dt, count=arr.offset + n)[arr.offset:]


def take_rows(table, idx):
    """The table whose row i is input row idx[i] (idx[i] < 0: NULL in every column), built with numpy `take` on the raw buffers
    of the fixed-width columns and Arrow's `take` on the strings."""
    idx = np.asarray(idx, np.int64)
    ok = idx >= 0
    cols = {}
    for name in table.column_names:
        arr = table.column(name)
        arr = arr.combine_chunks() if arr.num_chunks != 1 else arr.chunk(0)
        src_valid = np.asarray(arr.is_valid()) if arr.null_count else np.ones(len(arr), bool)
        j = np.where(ok, idx, 0)
        valid = ok & src_valid[j] if len(arr) else np.zeros(len(idx), bool)
        if pa.types.is_string(arr.type):
            cols[name] = arr.take(pa.array(idx, mask=~ok))
            continue
        if len(arr):
            vals = _storage(arr)[j]
        else:       # nothing to take from: every index is -1
            vals = np.zeros((len(idx), 2) if pa.types.is_decimal(arr.type) else len(idx), np.int64 if pa.types.is_decimal(arr.type) else
                            {1: np.uint8, 2: np.uint16, 4: np.uint32, 8: np.uint64}[max(1, arr.type.bit_width // 8)])
        vb = None if valid.all() else pa.py_buffer(np.packbits(valid, bitorder="little").tobytes())
        if pa.types.is_boolean(arr.type):
            cols[name] = pa.array(vals.astype(bool), mask=~valid)
        else:
            cols[name] = pa.Array.from_buffers(arr.type, len(idx), [vb, pa.py_buffer(np.ascontiguousarray(vals).tobytes())])
    return pa.table(cols)


def _is_string(t):
    return pa.types.is_string(t) or pa.types.is_binary(t)


def assert_same(got, want):
    """Equal bit for bit, row order included: fixed-width columns through assert_bits_equal, strings byte for byte."""
    assert got.num_columns == want.num_columns, (got.column_names, want.column_names)
    assert got.num_rows == want.num_rows, "row count %d != %d" % (got.num_rows, want.num_rows)
    for i in range(want.num_columns):
        assert got.schema.field(i).type == want.schema.field(i).type, \
            "column %d (%s): type %s != %s" % (i, want.column_names[i], got.schema.field(i).type, want.schema.field(i).type)
    fixed = [i for i in range(want.num_columns) if not _is_string(want.schema.field(i).type)]
    g = pa.table([got.column(i) for i in fixed], names=[want.column_names[i] for i in fixed])
    w = pa.table([want.column(i) for i in fixed], names=[want.column_names[i] for i in fixed])
    assert_bits_equal(g, w, ordered=True)
    for i in range(want.num_columns):
        if i in fixed:
            continue
        gv = np.asarray(got.column(i).is_valid())
        wv = np.asarray(want.column(i).is_valid())
        bad = np.nonzero(gv != wv)[0]
        assert len(bad) == 0, "column %s row %d: valid %s vs %s" % (want.column_names[i], bad[0], gv[bad[0]], wv[bad[0]])
        glen, gbytes = _string_bytes(got.column(i), wv)
        wlen, wbytes = _string_bytes(want.column(i), wv)
        bad = np.nonzero(glen != wlen)[0]
        assert len(bad) == 0, "column %s: byte length %d vs %d at the %d-th valid row" % (want.column_names[i], glen[bad[0]], wlen[bad[0]], bad[0])
        bad = np.nonzero(gbytes != wbytes)[0]
        assert len(bad) == 0, "column %s: %d string bytes differ, the first at byte %d of the valid rows" % (want.column_names[i], len(bad), bad[0])


def _string_bytes(col, valid):
    """(byte length of every valid row, the bytes of the valid rows end to end) read from the raw offsets and data buffers,
    without trusting them: offsets that are not monotone or point outside the data fail the comparison instead of crashing Arrow."""
    arr = col.combine_chunks() if col.num_chunks != 1 else col.chunk(0)
    n = len(arr)
    offs = np.frombuffer(arr.buffers()[1], np.int32, count=arr.offset + n + 1)[arr.offset:].astype(np.int64) if n else np.zeros(1, np.int64)
    data = np.frombuffer(arr.buffers()[2], np.uint8) if arr.buffers()[2] is not None else np.zeros(0, np.uint8)
    lens = np.diff(offs)
    assert (lens >= 0).all() and offs[0] >= 0 and offs[-1] <= len(data), "string offsets out of order or out of bounds"
    starts, lens = offs[:-1][valid], lens[valid]
    total = int(lens.sum())
    pos = np.repeat(starts - (np.cumsum(lens) - lens), lens) + np.arange(total)
    return lens, data[pos]


def assert_moved(got, src, idx):
    assert_same(got, take_rows(src, idx))


def _seed(*parts):
    return zlib.crc32(repr(parts).encode())


def _batch(t, stream):
    from spark_b200.columnar import ColumnarBatch
    return ColumnarBatch.from_arrow(t, stream)


# ------------------------------------------------------------------------------------------------ shuffle regroup
NPARTS = [1, 7, 63, 64, 256, 257, 2048]
ROWS = [0, 1, 4095, 4096, 4097, 8191, 8192, 8193, 100_003]
LAYOUTS = {"fixed": (False, False), "dec128": (True, False), "strings": (False, True), "all": (True, True)}   # (decimal128, strings)


def _check_hash_shuffle(t, nparts, stream, batch=None):
    """HashPartitioning on the row id: offsets from a bincount of the partition ids, rows in stable-argsort order (arrival order
    inside a bucket)."""
    from spark_b200.execution import HashPartitioning, LocalTableScanExec, ShuffleExchangeExec
    b = batch if batch is not None else _batch(t, stream)
    ex = ShuffleExchangeExec(HashPartitioning(["row"], nparts), LocalTableScanExec(b))
    got = ex.collect(stream)
    pid = O.partition_ids(t.select(["row"]), ["row"], nparts)
    assert np.array_equal(ex.partition_offsets, np.concatenate([[0], np.cumsum(np.bincount(pid, minlength=nparts))]))
    assert_moved(got, t, np.argsort(pid, kind="stable"))


def _check_round_robin(t, nparts, start, stream):
    from spark_b200.execution import LocalTableScanExec, RoundRobinPartitioning, ShuffleExchangeExec
    ex = ShuffleExchangeExec(RoundRobinPartitioning(nparts, start), LocalTableScanExec(_batch(t, stream)))
    got = ex.collect(stream)
    want_rows, offs = O.round_robin_partition(t.select(["row"]), nparts, start)
    assert np.array_equal(ex.partition_offsets, offs)
    assert_moved(got, t, np.asarray(want_rows.column("row")))


@pytest.mark.parametrize("ldst", [0, 1])
@pytest.mark.parametrize("nparts", NPARTS)
def test_shuffle_fanout(gpu, stream, sbconfig, nparts, ldst):
    """Every fan-out: one bucket, the 512-thread tiles (nparts < 64), the 1024-thread tiles (nparts >= 64 with rows of 32 bytes
    or more), the 256-bucket limit and the two-level split above it, over 25 fixed-width columns (two scatter chunks),
    decimal(38, 10) and strings (the row-id gather), both regroup kernels."""
    sbconfig("regroup_ldst", ldst)
    t = wide_table(100_003, width=25)
    _check_hash_shuffle(t, nparts, stream)
    if nparts in (7, 257):
        _check_round_robin(t, nparts, 3, stream)


@pytest.mark.parametrize("ldst", [0, 1])
@pytest.mark.parametrize("n", ROWS)
def test_shuffle_row_counts(gpu, stream, sbconfig, n, ldst):
    """Row counts around the 4096- and 8192-row tiles: empty, one row, one short of a tile, exactly a tile, one more."""
    sbconfig("regroup_ldst", ldst)
    t = wide_table(n, width=17)
    for nparts in (7, 64, 300):
        _check_hash_shuffle(t, nparts, stream)


@pytest.mark.parametrize("ldst", [0, 1])
@pytest.mark.parametrize("layout", list(LAYOUTS))
@pytest.mark.parametrize("width", WIDTHS)
def test_shuffle_widths(gpu, stream, sbconfig, width, layout, ldst):
    """Column counts on both sides of the 16-column scatter chunk, with and without decimal(38, 10) and string columns (with
    and without the row-id gather)."""
    sbconfig("regroup_ldst", ldst)
    dec128, strings = LAYOUTS[layout]
    t = wide_table(20_011, width=width, strings=strings, dec128=dec128)
    for nparts in (7, 64, 257):
        _check_hash_shuffle(t, nparts, stream)


@pytest.mark.parametrize("nparts", [7, 64, 300])
def test_shuffle_misaligned_source(gpu, stream, nparts):
    """Sources that are not 16-byte aligned cannot feed the copy engine: the load/store kernel takes them whatever the
    setting.  Every NULL-free fixed-width type, decimal(38, 10) included (moved by the row-id gather)."""
    t = _full_table(30_007, 1).select(["row"] + ["%s_n" % tn for tn in FIXED_TYPES])
    batch, keep = _misaligned_device_batch(t)
    try:
        _check_hash_shuffle(t, nparts, stream, batch=batch)
    finally:
        batch.close()
        del keep


@pytest.mark.parametrize("strings", [False, True])
def test_fused_exchange_wide_table(one_rank_comm, stream, strings):  # noqa: F811
    """sb_shuffle_exchange on a one-rank communicator.  Without strings and decimal(38, 10) the multisplit's stores go straight
    into the receive window (the REMOTE regroup kernel), with more than 16 pieces (two scatter chunks); with them the exchange
    partitions and runs the all-to-all.  Either way the result is the shuffle of the whole table."""
    from spark_b200.execution import HashPartitioning, LocalTableScanExec, ShuffleExchangeExec
    t = wide_table(100_003) if strings else wide_table(100_003, width=34, strings=False, dec128=False)
    for nparts in (7, 257):
        ex = ShuffleExchangeExec(HashPartitioning(["row"], nparts), LocalTableScanExec(_batch(t, stream)), fused=True)
        got = ex.collect(stream)
        pid = O.partition_ids(t.select(["row"]), ["row"], nparts)
        assert np.array_equal(ex.partition_offsets, np.concatenate([[0], np.cumsum(np.bincount(pid, minlength=nparts))]))
        assert_moved(got, t, np.argsort(pid, kind="stable"))


# ------------------------------------------------------------------------------------------------ gather via slice; concat
SLICE_BEGINS = [0, 1, 7, 8, 31, 33, 2047]
SLICE_LENGTHS = [0, 1, 2047, 2048, 2049]     # around the 256 x 8-row gather block


@pytest.mark.parametrize("width", WIDTHS + [len(ALL_FIXED)])
def test_slice(gpu, stream, width):
    t = wide_table(4200, width=width)
    b = _batch(t, stream)
    try:
        for begin in SLICE_BEGINS:
            for length in SLICE_LENGTHS:
                s = b.slice(begin, begin + length, stream)
                try:
                    assert_moved(s.to_arrow(stream), t, np.arange(begin, begin + length))
                finally:
                    s.close()
    finally:
        b.close()


CONCAT_PIECES = [[0, 1, 31, 33, 4097], [4097, 33, 0, 31, 1], [31], [0, 0], [1, 4097, 1]]


@pytest.mark.parametrize("pieces", CONCAT_PIECES, ids=["-".join(map(str, p)) for p in CONCAT_PIECES])
def test_concat(gpu, stream, pieces):
    """Pieces imported one by one: some carry a validity buffer and some do not (a piece without NULLs has none), one string
    piece holds 0 bytes (every string empty) and an empty piece holds nothing at all."""
    from spark_b200.columnar import ColumnarBatch
    t = wide_table(8400, seed=2)
    # a 31-row piece is rows 1000..1030, where every string is empty (or NULL)
    for name in ("str_n", "str_t"):
        vals = t.column(name).to_pylist()
        vals[1000:1031] = [None if v is None else "" for v in vals[1000:1031]]
        t = t.set_column(t.column_names.index(name), name, pa.array(vals, pa.string()))
    idx, parts = [], []
    cur = 0
    for k in pieces:
        s = 1000 if k == 31 else cur
        parts.append(_batch(t.slice(s, k), stream))
        idx.append(np.arange(s, s + k))
        cur = (cur + k + 1) % 4000
    try:
        cat = ColumnarBatch.concat(parts, stream)
        try:
            assert_moved(cat.to_arrow(stream), t, np.concatenate(idx))
        finally:
            cat.close()
    finally:
        for p in parts:
            p.close()


@pytest.mark.parametrize("cuts", [[0, 1, 32, 65, 4162, 4200], [0, 4200], [0, 0, 2048, 2048, 4200]])
def test_slice_then_concat_is_identity(gpu, stream, cuts):
    from spark_b200.columnar import ColumnarBatch
    t = wide_table(4200)
    b = _batch(t, stream)
    parts = [b.slice(cuts[i], cuts[i + 1], stream) for i in range(len(cuts) - 1)]
    try:
        cat = ColumnarBatch.concat(parts, stream)
        try:
            assert_moved(cat.to_arrow(stream), t, np.arange(t.num_rows))
        finally:
            cat.close()
    finally:
        for p in parts:
            p.close()
        b.close()


# ------------------------------------------------------------------------------------------------ join outputs
JOIN_HOWS = ["inner", "left_outer", "full_outer", "right_outer", "left_semi", "left_anti", "existence"]
_ORACLE_HOW = {"right_outer": "build_outer"}


def _join_sides(n_probe, n_build, width, seed, all_match=False):
    rng = np.random.default_rng(seed)
    probe = wide_table(n_probe, width=width, seed=seed)
    build = wide_table(n_build, width=width, seed=seed + 1)
    build = build.rename_columns(["b_" + c for c in build.column_names])
    if all_match:     # unique build keys, every streamed key among them
        bk = rng.permutation(n_build).astype(np.int64)
        pk = rng.integers(0, n_build, n_probe)
        pmask = None
    else:             # duplicates on both sides, unmatched rows on both sides, a few NULL streamed keys
        bk = rng.integers(0, 2 * n_build // 3, n_build)
        pk = rng.integers(0, n_build, n_probe)
        pmask = rng.random(n_probe) < 0.01
    probe = probe.append_column("k", pa.array(pk, pa.int64(), mask=pmask))
    build = build.append_column("k2", pa.array(bk, pa.int64()))
    return probe, build


def _check_join_rows(probe, build, how, stream):
    from spark_b200.execution import BroadcastHashJoinExec, LocalTableScanExec
    got = BroadcastHashJoinExec(["k"], ["k2"], how, "right", LocalTableScanExec(_batch(probe, stream)),
                                LocalTableScanExec(_batch(build, stream))).collect(stream)
    pairs = O.hash_join(probe.select(["k", "row"]), build.select(["k2", "b_row"]), ["k"], ["k2"], _ORACLE_HOW.get(how, how))
    pidx = np.asarray(pairs.column("row").fill_null(-1))
    if how in ("left_semi", "left_anti"):
        want = take_rows(probe, pidx)
    elif how == "existence":
        want = take_rows(probe, pidx).append_column("exists", pairs.column("exists"))
    else:
        bidx = np.asarray(pairs.column("b_row").fill_null(-1))
        want = take_rows(probe, pidx)
        bt = take_rows(build, bidx)
        for name in bt.column_names:
            want = want.append_column(name, bt.column(name))
    # the output order is not specified: order both sides by (streamed row id, build row id), unique per output row
    def order(t):
        keys = [np.asarray(t.column("row").fill_null(-1))]
        if "b_row" in t.column_names:
            keys.insert(0, np.asarray(t.column("b_row").fill_null(-1)))
        return np.lexsort(keys)
    assert got.num_rows == want.num_rows, "row count %d != %d" % (got.num_rows, want.num_rows)
    assert_same(got.take(pa.array(order(got))), want.take(pa.array(order(want))))


@pytest.mark.parametrize("how", JOIN_HOWS)
def test_join_outputs(gpu, stream, how):
    """Every payload type on both sides of every join type: matched rows, NULL-filled outer rows (negative gather indices) and
    the probe columns of semi, anti and existence joins."""
    probe, build = _join_sides(30_011, 9_001, len(ALL_FIXED), _seed("join", how) % 1000)
    _check_join_rows(probe, build, how, stream)


@pytest.mark.parametrize("all_match", [False, True])
@pytest.mark.parametrize("how", ["inner", "left_outer"])
def test_join_outputs_candidate_pass(gpu, stream, how, all_match):
    """2^20 + 13 streamed rows take the candidate pass; when every streamed row finds its one partner the streamed half of the
    output shares the input's buffers (no gather) and the build half is one lookup per row."""
    probe, build = _join_sides(CAND_N, 50_000, 13, 7 + all_match, all_match=all_match)
    _check_join_rows(probe.select(fixed_names(13) + ["str_t", "k"]), build.select(["b_" + c for c in fixed_names(13)] + ["b_str_t", "k2"]),
                     how, stream)


# ------------------------------------------------------------------------------------------------ filter, expand, sort, top-N, lag / lead
FILTERS = {"none": lambda n, rng: np.zeros(n, np.int64), "all": lambda n, rng: np.ones(n, np.int64),
           "every_32nd": lambda n, rng: (np.arange(n) % 32 == 5).astype(np.int64), "half": lambda n, rng: rng.integers(0, 2, n)}


@pytest.mark.parametrize("kind", list(FILTERS))
def test_filter(gpu, stream, kind):
    from spark_b200.execution import FilterExec, LocalTableScanExec
    from spark_b200.expressions import Literal, col
    n = 50_021
    t = wide_table(n)
    f = FILTERS[kind](n, np.random.default_rng(5))
    t = t.append_column("f", pa.array(f, pa.int64()))
    got = FilterExec(col("f") > Literal(0), LocalTableScanExec(_batch(t, stream))).collect(stream)
    assert_moved(got, t, np.nonzero(f > 0)[0])


def _partner(name):
    """A column of the same type in another validity variant (expand's second projection list)."""
    if name == "row":
        return name
    base, v = name.rsplit("_", 1)
    return "%s_%s" % (base, {"t": "n", "n": "a", "a": "t"}[v])


def test_expand(gpu, stream):
    """Two projection lists of every column: list 0 the columns themselves, list 1 the same type in another validity variant;
    input row r yields output rows 2r and 2r + 1."""
    from spark_b200.execution import ExpandExec, LocalTableScanExec
    from spark_b200.expressions import col
    n = 20_011
    t = wide_table(n)
    names = t.column_names
    got = ExpandExec([[col(c) for c in names], [col(_partner(c)) for c in names]], names, LocalTableScanExec(_batch(t, stream))).collect(stream)
    j = np.arange(2 * n)
    want = {}
    for c in names:
        both = pa.table({c: pa.concat_arrays([t.column(c).combine_chunks(), t.column(_partner(c)).combine_chunks()])})
        want[c] = take_rows(both, (j % 2) * n + j // 2).column(0)
    assert_same(got, pa.table(want))


def _sorted_order(t, asc):
    k = np.asarray(t.column("k")).astype(np.int64)
    return np.lexsort((np.asarray(t.column("row")), k if asc else -k))


@pytest.mark.parametrize("asc", [True, False])
@pytest.mark.parametrize("width", [13, len(ALL_FIXED)])
def test_sort_carries_every_column(gpu, stream, width, asc):
    """A NULL-free int key with ties (stable: ties keep arrival order): the sorted key column is rebuilt from the sorted keys,
    every other column is gathered."""
    from spark_b200.execution import LocalTableScanExec, SortExec
    t = wide_table(100_003, width=width, extra=("k",))
    got = SortExec([("k", asc, True)], LocalTableScanExec(_batch(t, stream))).collect(stream)
    assert_moved(got, t, _sorted_order(t, asc))


@pytest.mark.parametrize("limit", [1, 5000, 20_000])
def test_top_n_carries_every_column(gpu, stream, limit):
    from spark_b200.execution import LocalTableScanExec, TakeOrderedAndProjectExec
    from spark_b200.expressions import SortOrder
    t = wide_table(100_003, extra=("k",))
    for asc in (True, False):
        got = TakeOrderedAndProjectExec(limit, [SortOrder("k", asc)], None, LocalTableScanExec(_batch(t, stream))).collect(stream)
        assert_moved(got, t, _sorted_order(t, asc)[:limit])


@pytest.mark.parametrize("offset", [1, 2])
@pytest.mark.parametrize("func", ["lag", "lead"])
def test_lag_lead_carries_every_column(gpu, stream, func, offset):
    """lag / lead of every column with the default NULL: rows outside the partition are a negative gather index."""
    from spark_b200.execution import LocalTableScanExec, WindowExec, WindowFunction
    n = 30_011
    t = wide_table(n, extra=("g",))
    payload = t.column_names[:-1]
    wins = [WindowFunction(func, c, param=offset, name="%s_%s" % (func, c)) for c in payload]
    got = WindowExec(wins, ["g"], [("row", True, True)], LocalTableScanExec(_batch(t, stream))).collect(stream)
    g = np.asarray(t.column("g"))
    perm = np.lexsort((np.asarray(t.column("row")), g))
    src = np.arange(n) + (offset if func == "lead" else -offset)
    inside = (src >= 0) & (src < n)
    same = np.zeros(n, bool)
    same[inside] = g[perm[src[inside]]] == g[perm[inside]]
    idx = np.where(same, perm[np.clip(src, 0, max(n - 1, 0))], -1)
    want = take_rows(t, perm)
    moved = take_rows(t.select(payload), idx)
    for c in payload:
        want = want.append_column("%s_%s" % (func, c), moved.column(c))
    assert_same(got, want)
