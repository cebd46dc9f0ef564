"""CPU half of the fixed-width scan matrix (the GPU half is tests/test_gpu_scan_types.py): the Parquet files of every type,
encoding, page layout and NULL pattern the GPU scan is tested on, written by pyarrow (parquet-cpp), walked with the product's
page walker (sb_parquet_chunk_pages, host only), decoded with the oracle's restatement of the page decoding and compared BIT FOR
BIT with pyarrow's reader.  The generators are checked here too -- the dictionary bit widths, hybrid run shapes, NULL layouts
and page offsets they are meant to produce do occur -- so a wrong expectation fails before it reaches the GPU.

Spark's view of the columns (VectorizedParquetRecordReader / ParquetVectorUpdaterFactory): INT32 narrows to byte / short,
decimals keep precision and scale (INT32-stored ones sign-extend into a long), TIMESTAMP(MILLIS) is read in microseconds
(LongAsMicrosUpdater) and TIMESTAMP(NANOS), INT96, FIXED_LEN_BYTE_ARRAY, unsigned integers and TIME are refused."""
import os

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq
import pytest

from oracle import parquet_oracle as PO
from parquet_delta_oracle import decode_column_chunk as oracle_decode_chunk
from test_gpu_key_types import assert_bits_equal

# ------------------------------------------------------------------------------------------------ types and values
DECIMALS = [(p, s) for p in (1, 7, 9, 10, 18) for s in sorted({0, 2, p}) if s <= p]
TYPES = dict([("bool", pa.bool_()), ("int8", pa.int8()), ("int16", pa.int16()), ("int32", pa.int32()), ("int64", pa.int64()),
              ("date32", pa.date32()), ("float32", pa.float32()), ("float64", pa.float64()), ("ts_us", pa.timestamp("us")),
              ("ts_ms", pa.timestamp("ms")), ("ts_s", pa.timestamp("s"))] +
             [("dec%d_%d" % ps, pa.decimal128(*ps)) for ps in DECIMALS])
# columns whose physical type is INT32 / INT64 (DELTA_BINARY_PACKED candidates)
DELTA_TYPES = [t for t in TYPES if t not in ("bool", "float32", "float64")]

F64_NAN_BITS = [0x7FF8000000000000, 0xFFF8000000000000, 0x7FF0000000000001, 0xFFF0000000000001, 0x7FF4000000000000, 0xFFFFFFFFFFFFFFFF]
F32_NAN_BITS = [0x7FC00000, 0xFFC00000, 0x7F800001, 0xFF800001, 0x7FC00001, 0xFFFFFFFF]
_STORAGE = {pa.bool_(): np.uint8, pa.int8(): np.int8, pa.int16(): np.int16, pa.int32(): np.int32, pa.int64(): np.int64,
            pa.date32(): np.int32, pa.float32(): np.float32, pa.float64(): np.float64}


def storage_dtype(t):
    return np.int64 if pa.types.is_timestamp(t) or pa.types.is_decimal(t) else _STORAGE[t]


def specials(t):
    """Edge values of an Arrow type, as storage values (days, the type's own time unit, unscaled decimals, raw float bits)."""
    if pa.types.is_boolean(t):
        return np.array([0, 1, 1, 0], np.uint8)
    if pa.types.is_decimal(t):
        top = 10 ** t.precision - 1
        return np.array([-top, top, -1, 0, 1, -top + 1, top - 1], np.int64)
    if pa.types.is_timestamp(t):      # MIN / MAX that still fit int64 microseconds after Spark's conversion, and before 1970
        lim = (2 ** 63 - 1) // {"us": 1, "ms": 1000, "s": 1_000_000}[t.unit]
        return np.array([-lim, lim, -1, 0, 1, -86_400 * 365, -lim + 1], np.int64)
    if pa.types.is_floating(t):
        ft = np.float64 if t == pa.float64() else np.float32
        fi = np.finfo(ft)
        nan = np.array(F64_NAN_BITS if ft == np.float64 else F32_NAN_BITS, np.uint64 if ft == np.float64 else np.uint32).view(ft)
        big = ft(2.0 ** 53) if ft == np.float64 else ft(2.0 ** 24)
        fin = np.array([0.0, -0.0, np.inf, -np.inf, -1.0, 1.0, fi.max, -fi.max, fi.tiny, -fi.tiny, fi.smallest_subnormal,
                        -fi.smallest_subnormal, fi.tiny - fi.smallest_subnormal, np.nextafter(big, ft(np.inf)), big], ft)
        return np.concatenate([fin, nan])
    info = np.iinfo(_STORAGE[t])
    return np.array([info.min, info.max, -1, 0, 1, info.min + 1, info.max - 1], _STORAGE[t])


def random_values(t, n, rng, distinct=None):
    """n storage values of a type, its specials first; `distinct` draws them from a pool of that many (dictionary-friendly)"""
    sp = specials(t)
    dt = storage_dtype(t)
    if pa.types.is_boolean(t):
        v = rng.integers(0, 2, n).astype(np.uint8)
    elif pa.types.is_floating(t):
        v = (rng.integers(-4000, 4000, n) / 4.0).astype(dt)
    elif pa.types.is_decimal(t):
        top = 10 ** t.precision
        v = rng.integers(-top + 1, top, n, dtype=np.int64)
    else:
        lo, hi = (int(sp.min()), int(sp.max())) if not pa.types.is_date32(t) else (-800_000, 800_000)
        v = rng.integers(lo, hi, n, dtype=np.int64, endpoint=True).astype(dt)
    if distinct is not None:
        v = np.concatenate([sp, v[:distinct]])[rng.integers(0, len(sp) + min(distinct, n), n)].astype(dt)
    v[:min(n, len(sp))] = sp[:n]
    return v.astype(dt)


def make_array(t, values, valid=None):
    """Arrow array from storage values, built from buffers so that every bit -- NaN payloads included -- arrives as given"""
    values = np.asarray(values)
    n = len(values)
    has_nulls = valid is not None and not bool(np.all(valid))
    vb = pa.py_buffer(np.packbits(np.asarray(valid, bool), bitorder="little").tobytes()) if has_nulls else None
    if pa.types.is_boolean(t):
        return pa.array(values.astype(bool), mask=~np.asarray(valid, bool) if has_nulls else None)
    if pa.types.is_decimal(t):
        wide = np.empty((n, 2), np.int64)
        wide[:, 0] = values.astype(np.int64)
        wide[:, 1] = wide[:, 0] >> 63
        return pa.Array.from_buffers(t, n, [vb, pa.py_buffer(wide.tobytes())])
    return pa.Array.from_buffers(t, n, [vb, pa.py_buffer(np.ascontiguousarray(values.astype(storage_dtype(t))).tobytes())])


def table(cols, required=()):
    """pa.table of the columns; those named in `required` are non-nullable (no definition levels in their pages)"""
    return pa.table(list(cols.values()), schema=pa.schema([pa.field(k, v.type, nullable=k not in required) for k, v in cols.items()]))


def spark_type(t):
    """the Arrow type the GPU scan returns for a column of Arrow type t"""
    return pa.timestamp("us") if pa.types.is_timestamp(t) else t


# ------------------------------------------------------------------------------------------------ NULL patterns
NULL_PATTERNS = ["none", "all", "alternating", "runs", "page_edges", "null_page"]


def null_mask(pattern, n, page_starts, rng):
    """valid[n] of a pattern; page_starts: first row of every page (row-group relative rows already made absolute)"""
    if pattern == "none":
        return np.ones(n, bool)
    if pattern == "all":
        return np.zeros(n, bool)
    if pattern == "alternating":        # definition levels bit-packed
        return np.arange(n) % 2 == 0
    if pattern == "runs":               # runs of 8 .. 40 equal levels: definition levels RLE
        lens = rng.integers(8, 41, n // 8 + 2)
        return (np.repeat(np.arange(len(lens)) % 2 == 0, lens)[:n]).copy()
    v = rng.random(n) >= 0.1
    if pattern == "page_edges":         # the first and the last row of every page NULL
        starts = np.asarray(page_starts)
        v[starts] = False
        v[starts[1:] - 1] = False
        v[n - 1] = False
        return v
    if pattern == "null_page":          # the second page of every row group entirely NULL, between pages with values
        for a, b in zip(page_starts, list(page_starts[1:]) + [n]):
            if a in page_starts[1::3]:
                v[a:b] = False
        return v
    raise ValueError(pattern)


def page_starts_of(n, row_group_size, page_rows):
    starts = []
    for g in range(0, n, row_group_size):
        starts.extend(range(g, min(n, g + row_group_size), page_rows))
    return starts


# ------------------------------------------------------------------------------------------------ the matrix
# every type, NULL-free and NULLable (the pattern rotates with the file), written PLAIN, dictionary, dictionary with fallback to
# PLAIN inside a chunk, and DELTA_BINARY_PACKED (BOOLEAN: RLE), data page V1 and V2; rows per page and per row group are not
# multiples of 8, 256 or 1024, and pages are longer than expand_rows' 1024-row tiles
ENCODINGS = ["plain", "dict", "fallback", "delta"]
VERSIONS = ["1.0", "2.0"]
MATRIX_ROWS, MATRIX_RG, MATRIX_PAGE = 6007, 4001, 1337


def matrix_table(seed, rotate=0, n=MATRIX_ROWS, row_group_size=MATRIX_RG, page_rows=MATRIX_PAGE):
    rng = np.random.default_rng(seed)
    starts = page_starts_of(n, row_group_size, page_rows)
    cols = {}
    for i, (name, t) in enumerate(TYPES.items()):
        vals = random_values(t, n, rng, distinct=None if i % 2 else 200)
        cols[name] = make_array(t, vals)
        pattern = NULL_PATTERNS[1 + (i + rotate) % (len(NULL_PATTERNS) - 1)]
        cols[name + "_n"] = make_array(t, random_values(t, n, rng, distinct=300), null_mask(pattern, n, starts, rng))
    return table(cols, required=list(TYPES))


def write_matrix(dirname, encoding, version, compression="NONE", n=MATRIX_ROWS, seed=None):
    rot = ENCODINGS.index(encoding) + 2 * VERSIONS.index(version)
    t = matrix_table(seed if seed is not None else 1000 + rot, rotate=rot, n=n)
    kw = dict(use_dictionary=encoding in ("dict", "fallback"), dictionary_pagesize_limit=1 << 26)
    if encoding == "fallback":          # a dictionary page of a few hundred bytes: high-cardinality chunks fall back to PLAIN
        kw["dictionary_pagesize_limit"] = 512
    if encoding == "delta":
        kw["column_encoding"] = {c: ("RLE" if c.startswith("bool") else "DELTA_BINARY_PACKED") for c in t.column_names
                                 if c.split("_n")[0] in DELTA_TYPES or c.startswith("bool")}
    path = os.path.join(dirname, "m-%s-v%s-%s.parquet" % (encoding, version, compression))
    pq.write_table(t, path, compression=compression, data_page_version=version, row_group_size=MATRIX_RG, max_rows_per_page=MATRIX_PAGE,
                   data_page_size=1 << 30, store_decimal_as_integer=True, **kw)
    return t, path


# dictionary sizes 1, 2, 3, 2^k and 2^k + 1 (k <= 20): index bit widths 0 .. 21, one row group each
DICT_SIZES = sorted({1, 2, 3} | {2 ** k for k in range(1, 21)} | {2 ** k + 1 for k in range(1, 21)})


def dict_bit_width(size):
    """the index bit width parquet-cpp writes (at least 1; parquet-mr writes 0 for a dictionary of one entry, see
    one_entry_dictionary_chunk)"""
    return max(1, (size - 1).bit_length())


def one_entry_dictionary_chunk(n, value, physical=2):
    """a hand-built column chunk the way parquet-mr writes a one-entry dictionary: [PLAIN dictionary value][one data page whose
    values are the bit width 0 alone] -- every index is 0 without a single run"""
    import ctypes as C
    import spark_b200._capi as capi
    from spark_b200.scan import EncodedColumnChunk
    dt = np.int64 if physical == 2 else np.int32
    data = np.concatenate([np.frombuffer(np.array([value], dt).tobytes(), np.uint8), np.zeros(1, np.uint8)])
    pages = (capi.sb_page * 1)()
    pages[0].encoding, pages[0].num_values, pages[0].values_offset, pages[0].values_bytes = capi.SB_ENC_RLE_DICTIONARY, n, data.nbytes - 1, 1
    sbt = capi.SB_INT64 if physical == 2 else capi.SB_INT32
    return EncodedColumnChunk(sbt, 0, physical, data, C.cast(pages, C.POINTER(capi.sb_page)), 1, 0, 1)


def write_dict_widths(dirname):
    path = os.path.join(dirname, "widths.parquet")
    rng = np.random.default_rng(7)
    schema = pa.schema([pa.field("i32", pa.int32(), nullable=False), pa.field("f64", pa.float64(), nullable=False)])
    tables = []
    with pq.ParquetWriter(path, schema, compression="NONE", use_dictionary=True, dictionary_pagesize_limit=1 << 30,
                          data_page_size=1 << 30, max_rows_per_page=1 << 22) as w:      # one page per chunk: its bit width is the dictionary's
        for size in DICT_SIZES:
            n = size + 17
            idx = np.concatenate([rng.permutation(size), rng.integers(0, size, n - size)])
            pool = rng.choice(2 ** 31 - 1, size, replace=False).astype(np.int32) - (2 ** 30)
            t = pa.table({"i32": pa.array(pool[idx]), "f64": pa.array(pool[idx].astype(np.float64) * -0.25)}, schema=schema)
            w.write_table(t, row_group_size=n)
            tables.append(t)
    return tables, path


HYBRID_ROWS = 200_005


def hybrid_table():
    """one page per column: a dictionary-index run of > 2^16 repeats; alternating short RLE and bit-packed runs (far more than
    SCAN_RUNS = 64 runs in the page); a last bit-packed group padded past the page's end; definition levels in long RLE runs,
    in alternating RLE / bit-packed runs, and bit-packed only"""
    n = HYBRID_ROWS
    rng = np.random.default_rng(11)
    long = np.concatenate([np.full(150_000, 5, np.int32), rng.integers(0, 40, n - 150_000).astype(np.int32)])
    blocks = []
    for i in range(n // 16 + 1):        # 8 repeats of one value, then 8 values without repeats
        blocks.append(np.full(8, rng.integers(0, 500), np.int32))
        blocks.append(500 + rng.permutation(500)[:8].astype(np.int32))
    alt = np.concatenate(blocks)[:n]
    padded = rng.integers(0, 3000, n).astype(np.int32)        # n % 8 == 5: the last group holds 5 values
    lens = np.where(np.arange(n // 8) % 2 == 0, 8, 1)
    mixed_valid = np.repeat(np.arange(len(lens)) % 4 < 2, lens)
    mixed_valid = np.concatenate([mixed_valid, np.arange(n) % 2 == 0])[:n]
    mixed_valid[: 8 * 20] = np.repeat(np.arange(20) % 2 == 0, 8)
    return table({
        "long_run": pa.array(long), "alternating": pa.array(alt), "padded": pa.array(padded),
        "def_long": make_array(pa.int64(), rng.integers(-5, 5, n), np.concatenate([np.zeros(70_000, bool), rng.random(n - 70_000) < 0.9])),
        "def_mixed": make_array(pa.int32(), rng.integers(0, 100, n).astype(np.int32), mixed_valid),
        "def_packed": make_array(pa.float64(), rng.integers(0, 50, n) / 8.0, np.arange(n) % 3 != 1),
    }, required=["long_run", "alternating", "padded"])


def write_hybrid(dirname, version="1.0"):
    t = hybrid_table()
    path = os.path.join(dirname, "hybrid-v%s.parquet" % version)
    pq.write_table(t, path, compression="NONE", use_dictionary=True, dictionary_pagesize_limit=1 << 30, data_page_size=1 << 30,
                   max_rows_per_page=1 << 21, data_page_version=version)
    return t, path


GEOMETRY_PAGE = 1004      # a multiple of 4 (not of 8): row starts of 4- and 8-byte pages fall on and off 16-byte boundaries
GEOMETRY_TYPES = ["int32", "int64", "float32", "float64", "date32", "ts_us", "dec18_2", "dec10_0"]


def write_geometry(dirname, compression="NONE"):
    """NULL-free PLAIN pages of 4- and 8-byte columns whose values start at chunk offsets both on and off 16-byte boundaries
    (scan_decode_kernel's 16-byte copy and its element-wise path), in two row groups"""
    rng = np.random.default_rng(3)
    n = 40 * GEOMETRY_PAGE + 7
    t = table({c: make_array(TYPES[c], random_values(TYPES[c], n, rng)) for c in GEOMETRY_TYPES}, required=GEOMETRY_TYPES)
    path = os.path.join(dirname, "geometry-%s.parquet" % compression)
    pq.write_table(t, path, compression=compression, use_dictionary=False, max_rows_per_page=GEOMETRY_PAGE, data_page_size=1 << 30,
                   row_group_size=24 * GEOMETRY_PAGE, store_decimal_as_integer=True)
    return t, path


def plain_copy_paths(ch):
    """for every NULL-free PLAIN page whose physical width is its column width: does it take the 16-byte copy (values offset
    and output offset both multiples of 16, for a 16-byte aligned device buffer)?"""
    import spark_b200._capi as capi
    w = capi.TYPE_WIDTH[ch.type]
    pw = {1: 4, 2: 8, 4: 4, 5: 8}.get(ch.physical, 0)
    out, row = [], 0
    for p in page_tuples(ch):
        if p[0] == capi.SB_ENC_PLAIN and p[5] == 0 and pw == w:
            out.append(p[2] % 16 == 0 and (row * w) % 16 == 0)
        row += p[1]
    return out


STRIPE_ROWS = 1_000_003
STRIPE_LAYOUTS = {"one_page": 1 << 21, "few_pages": 10_007, "many_pages": 1009}     # max rows per page


def stripe_table():
    rng = np.random.default_rng(5)
    base = rng.integers(-3000, 3000, STRIPE_ROWS).astype(np.int32)
    runs = np.repeat(rng.integers(-3000, 3000, STRIPE_ROWS // 100 + 1), 100)[:STRIPE_ROWS].astype(np.int32)
    return table({"v": pa.array(np.where((np.arange(STRIPE_ROWS) // 5000) % 2 == 0, base, runs))}, required=["v"])


def write_stripes(dirname):
    t = stripe_table()
    paths = {}
    for name, rows in STRIPE_LAYOUTS.items():
        paths[name] = os.path.join(dirname, "stripe-%s.parquet" % name)
        pq.write_table(t, paths[name], compression="NONE", use_dictionary=True, dictionary_pagesize_limit=1 << 30, data_page_size=1 << 30,
                       max_rows_per_page=rows, row_group_size=STRIPE_ROWS)
    return t, paths


def expected_nparts(num_sms, npages):
    """scan_decode_kernel's blocks per page (scan.cu: enough blocks for 6 per SM, 1 .. 16 per page)"""
    return min(16, max(1, -(-6 * num_sms // npages)))


# ------------------------------------------------------------------------------------------------ references
def page_tuples(ch):
    return [(ch.pages[i].encoding, ch.pages[i].num_values, ch.pages[i].values_offset, ch.pages[i].values_bytes,
             ch.pages[i].def_offset, ch.pages[i].def_bytes) for i in range(ch.npages)]


def oracle_column(ch, t, pcol):
    """the oracle's restatement of the page decoding of one column chunk, as the Arrow column Spark would see"""
    vals, valid = oracle_decode_chunk(ch.data, page_tuples(ch), ch.dict_offset, ch.dict_count, ch.physical)
    if pa.types.is_boolean(t):
        vals = vals.astype(np.uint8)
    elif pa.types.is_decimal(t) or pa.types.is_timestamp(t):
        vals = vals.astype(np.int64)       # INT32-stored decimals sign-extend
        if pa.types.is_timestamp(t):
            vals = vals * np.int64(timestamp_multiplier(pcol))
    else:
        vals = vals.astype(_STORAGE[t])    # INT32 narrows to byte / short
    if valid is not None and not valid.all():
        vals = np.where(valid, vals, np.zeros(1, vals.dtype))
    return make_array(spark_type(t), vals, valid)


def timestamp_multiplier(pcol):
    return 1000 if '"timeUnit": "milliseconds"' in pcol.logical_type.to_json() else 1


def pyarrow_column(col):
    """pyarrow's reader, converted the way Spark converts: timestamps in microseconds"""
    col = col.combine_chunks() if isinstance(col, pa.ChunkedArray) else col
    return col.cast(pa.timestamp("us")) if pa.types.is_timestamp(col.type) else col


def oracle_table(path, rg=None):
    """the oracle's decoding of every column of a file (or of one row group), as a table of Spark's Arrow types"""
    from spark_b200.scan import ParquetScanExec
    scan = ParquetScanExec(path)
    pf = scan.file
    groups = [rg] if rg is not None else range(pf.metadata.num_row_groups)
    parts = []
    for g in groups:
        cols = {}
        for f, ch in zip(scan.fields, scan.row_group_chunks(g)):
            cols[f.name] = oracle_column(ch, f.type, pf.schema.column(pf.schema.names.index(f.name)))
        parts.append(pa.table(cols))
    return pa.concat_tables(parts).combine_chunks()


def pyarrow_table(path, rg=None):
    pf = pq.ParquetFile(path)
    t = pf.read() if rg is None else pf.read_row_group(rg)
    return pa.table({c: pyarrow_column(t.column(c)) for c in t.column_names})


def spark_input(t):
    """the written table as Spark reads it back (timestamps in microseconds)"""
    return pa.table({c: pyarrow_column(t.column(c)) for c in t.column_names})


def hybrid_runs(buf, bw, count):
    """[(kind, values)] of an RLE / bit-packed hybrid stream: 'rle' or 'bp' (values = 8 * groups, padding included)"""
    b = np.asarray(buf, np.uint8)
    out, pos, got = [], 0, 0
    while got < count and pos < len(b):
        h, pos = PO.read_uvarint(b, pos)
        if h & 1:
            out.append(("bp", (h >> 1) * 8))
            pos += (h >> 1) * bw
        else:
            out.append(("rle", h >> 1))
            pos += (bw + 7) // 8
        got += out[-1][1]
    return out


def chunks_of(path, rg=0):
    from spark_b200.scan import ParquetScanExec
    scan = ParquetScanExec(path)
    return scan, dict(zip(scan.columns, scan.row_group_chunks(rg)))


# ------------------------------------------------------------------------------------------------ tests
@pytest.mark.parametrize("version", VERSIONS)
@pytest.mark.parametrize("encoding", ENCODINGS)
def test_matrix_oracle_equals_pyarrow(tmp_path, encoding, version):
    t, path = write_matrix(str(tmp_path), encoding, version)
    want = pyarrow_table(path)
    got = oracle_table(path)
    assert_bits_equal(got, want, ordered=True)
    if encoding != "dict" and encoding != "fallback":       # parquet-cpp's dictionary may merge NaN payloads and signed zeros
        assert_bits_equal(got, spark_input(t), ordered=True)
    else:
        ints = [c for c in t.column_names if not pa.types.is_floating(t.schema.field(c).type)]
        assert_bits_equal(got.select(ints), spark_input(t).select(ints), ordered=True)


@pytest.mark.parametrize("encoding", ENCODINGS)
def test_matrix_files_hold_the_intended_pages(tmp_path, encoding):
    """page row counts, encodings, NULL layouts and PLAIN value offsets the GPU tests rely on"""
    import spark_b200._capi as capi
    t, path = write_matrix(str(tmp_path), encoding, "1.0")
    scan = ParquetScanExec_(path)
    rows = [MATRIX_PAGE] * 3
    seen = set()
    for rg in range(scan.meta.num_row_groups):
        for name, ch in zip(scan.columns, scan.row_group_chunks(rg)):
            pages = page_tuples(ch)
            counts = [p[1] for p in pages]
            if encoding != "fallback":     # (the fallback to PLAIN flushes the dictionary-encoded rows as a page of their own)
                assert counts[:-1] == rows[:len(counts) - 1], (name, counts)
                assert all(c % 8 for c in counts[:-1]), counts
            assert all(p[5] == 0 for p in pages) == (name in TYPES), name          # definition levels only where NULLs may be
            encs = {p[0] for p in pages}
            seen |= {(name.split("_n")[0], e) for e in encs}
    if encoding == "dict":
        assert all((c, capi.SB_ENC_RLE_DICTIONARY) in seen for c in TYPES if c != "bool")
    if encoding == "fallback":          # high-cardinality chunks: dictionary pages first, then PLAIN in the same chunk
        both = [c for c in TYPES if (c, capi.SB_ENC_RLE_DICTIONARY) in seen and (c, capi.SB_ENC_PLAIN) in seen]
        assert len(both) >= 5, both
    if encoding == "delta":
        assert all((c, capi.SB_ENC_DELTA_BINARY_PACKED) in seen for c in DELTA_TYPES)
        assert ("bool", capi.SB_ENC_RLE_BOOLEAN) in seen


def ParquetScanExec_(path):
    from spark_b200.scan import ParquetScanExec
    return ParquetScanExec(path)


def write_nulls(dirname):
    """an all-NULL dictionary chunk (its dictionary page is empty), definition levels only bit-packed, and in RLE runs"""
    rng = np.random.default_rng(1)
    starts = page_starts_of(MATRIX_ROWS, MATRIX_RG, MATRIX_PAGE)
    t = pa.table({"a": make_array(pa.int32(), np.zeros(MATRIX_ROWS, np.int32), np.zeros(MATRIX_ROWS, bool)),
                  "b": make_array(pa.int64(), np.arange(MATRIX_ROWS), null_mask("alternating", MATRIX_ROWS, starts, rng)),
                  "c": make_array(pa.int64(), np.arange(MATRIX_ROWS), null_mask("runs", MATRIX_ROWS, starts, rng))})
    path = os.path.join(dirname, "nulls.parquet")
    pq.write_table(t, path, compression="NONE", use_dictionary=True, max_rows_per_page=MATRIX_PAGE, row_group_size=MATRIX_RG)
    return path


def test_null_patterns_land_where_intended(tmp_path):
    """page edges NULL, one page of every row group all NULL, an all-NULL chunk whose dictionary is empty; definition levels
    both bit-packed and RLE"""
    rng = np.random.default_rng(0)
    starts = page_starts_of(MATRIX_ROWS, MATRIX_RG, MATRIX_PAGE)
    v = null_mask("page_edges", MATRIX_ROWS, starts, rng)
    assert not v[starts].any() and not v[np.array(starts[1:]) - 1].any()
    v = null_mask("null_page", MATRIX_ROWS, starts, rng)
    assert not v[MATRIX_PAGE:2 * MATRIX_PAGE].any() and v[:MATRIX_PAGE].any() and v[2 * MATRIX_PAGE:3 * MATRIX_PAGE].any()
    path = write_nulls(str(tmp_path))
    _, ch = chunks_of(path)
    assert ch["a"].dict_offset >= 0 and ch["a"].dict_count == 0
    kinds = {}
    for name in "bc":
        p = page_tuples(ch[name])[0]
        kinds[name] = {k for k, _ in hybrid_runs(ch[name].data[p[4]:p[4] + p[5]], 1, p[1])}
    assert kinds["b"] == {"bp"} and "rle" in kinds["c"], kinds
    assert_bits_equal(oracle_table(path), pyarrow_table(path), ordered=True)


def test_dictionary_index_widths_0_to_21(tmp_path):
    tables, path = write_dict_widths(str(tmp_path))
    from spark_b200.scan import ParquetScanExec
    import spark_b200._capi as capi
    scan = ParquetScanExec(path)
    widths = set()
    for rg, size in enumerate(DICT_SIZES):
        for name, ch in zip(scan.columns, scan.row_group_chunks(rg)):
            assert ch.dict_count == size, (name, size, ch.dict_count)
            for p in page_tuples(ch):
                assert p[0] == capi.SB_ENC_RLE_DICTIONARY, (name, size, "fell back to PLAIN")
                assert int(ch.data[p[2]]) == dict_bit_width(size), (name, size, int(ch.data[p[2]]))
                widths.add(int(ch.data[p[2]]))
        assert_bits_equal(oracle_table(path, rg), pyarrow_table(path, rg), ordered=True)
        assert_bits_equal(oracle_table(path, rg), tables[rg], ordered=True)
    assert widths == set(range(1, 22))
    ch = one_entry_dictionary_chunk(3001, -7)
    vals, valid = oracle_decode_chunk(ch.data, page_tuples(ch), ch.dict_offset, ch.dict_count, ch.physical)
    assert valid is None and int(ch.data[page_tuples(ch)[0][2]]) == 0 and np.array_equal(vals, np.full(3001, -7))


@pytest.mark.parametrize("version", VERSIONS)
def test_hybrid_stream_shapes(tmp_path, version):
    t, path = write_hybrid(str(tmp_path), version)
    _, ch = chunks_of(path)
    shapes = {}
    for name, c in ch.items():
        (p,) = page_tuples(c)                 # one page per chunk
        assert p[1] == HYBRID_ROWS
        nvals = HYBRID_ROWS if p[5] == 0 else int(t.column(name).combine_chunks().is_valid().to_numpy(zero_copy_only=False).sum())
        shapes[name] = hybrid_runs(c.data[p[2] + 1:p[2] + p[3]], int(c.data[p[2]]), nvals)
        if p[5]:
            shapes[name + ".def"] = hybrid_runs(c.data[p[4]:p[4] + p[5]], 1, HYBRID_ROWS)
    assert max(n for k, n in shapes["long_run"] if k == "rle") > 1 << 16
    alt = shapes["alternating"]
    assert len(alt) > 100 * 64 and {k for k, _ in alt} == {"rle", "bp"}
    assert shapes["padded"][-1][0] == "bp" and sum(n for _, n in shapes["padded"]) > HYBRID_ROWS
    assert max(n for k, n in shapes["def_long.def"] if k == "rle") > 1 << 16
    mixed = shapes["def_mixed.def"]
    assert len(mixed) > 64 and {k for k, _ in mixed} == {"rle", "bp"}
    assert {k for k, _ in shapes["def_packed.def"]} == {"bp"}
    assert_bits_equal(oracle_table(path), pyarrow_table(path), ordered=True)
    assert_bits_equal(oracle_table(path), t, ordered=True)


def test_geometry_pages_take_both_plain_copy_paths(tmp_path):
    t, path = write_geometry(str(tmp_path))
    scan = ParquetScanExec_(path)
    assert scan.meta.num_row_groups == 2
    paths = set()
    for rg in range(2):
        for ch in scan.row_group_chunks(rg):
            paths |= set(plain_copy_paths(ch))
    assert paths == {True, False}
    assert_bits_equal(oracle_table(path), pyarrow_table(path), ordered=True)
    assert_bits_equal(oracle_table(path), spark_input(t), ordered=True)


def test_stripe_layouts_page_counts(tmp_path):
    """one page, ~100 pages and ~1000 pages of the same NULL-free dictionary column: on a 132-SM H100 these decode with 16,
    8 and 1 blocks per page"""
    t, paths = write_stripes(str(tmp_path))
    npages = {}
    for name, path in paths.items():
        _, ch = chunks_of(path)
        npages[name] = ch["v"].npages
        assert all(p[0] == 1 and p[5] == 0 for p in page_tuples(ch["v"]))
        assert_bits_equal(oracle_table(path), t, ordered=True)
    assert npages["one_page"] == 1 and 50 <= npages["few_pages"] <= 200 and npages["many_pages"] >= 6 * 132
    assert [expected_nparts(132, npages[k]) for k in STRIPE_LAYOUTS] == [16, 8, 1]


# ---- refusals: SparkB200Error(5) naming the column, when the scan is created (before any device call)
REFUSED = {
    "ts_nanos": (pa.array([0, -1, 10 ** 18], pa.timestamp("ns")), {}),
    "int96": (pa.array([0, -1, 10 ** 18], pa.timestamp("ns")), dict(use_deprecated_int96_timestamps=True)),
    "flba_decimal": (pa.array([0, 1, -1], pa.decimal128(9, 2)), dict(store_decimal_as_integer=False)),
    "decimal_p19": (pa.array([0, 1, -1], pa.decimal128(19, 2)), dict(store_decimal_as_integer=True)),
    "uint8": (pa.array([0, 1, 255], pa.uint8()), {}),
    "uint16": (pa.array([0, 1, 65535], pa.uint16()), {}),
    "uint32": (pa.array([0, 1, 2 ** 32 - 1], pa.uint32()), {}),
    "uint64": (pa.array([0, 1, 2 ** 64 - 1], pa.uint64()), {}),
    "time32": (pa.array([0, 1, 86_399_999], pa.time32("ms")), {}),
    "time64": (pa.array([0, 1, 86_399_999_999], pa.time64("us")), {}),
}


@pytest.mark.parametrize("name", list(REFUSED))
def test_unsupported_columns_are_refused_naming_the_column(tmp_path, name):
    from spark_b200 import _capi as capi
    from spark_b200.scan import ParquetScanExec
    arr, kw = REFUSED[name]
    col = "bad_" + name
    path = os.path.join(str(tmp_path), "r.parquet")
    pq.write_table(pa.table({"ok": pa.array([1, 2, 3], pa.int32()), col: arr}), path, compression="NONE", **kw)
    with pytest.raises(capi.SparkB200Error) as e:
        ParquetScanExec(path)
    assert e.value.code == 5 and col in str(e.value), str(e.value)
    assert ParquetScanExec(path, columns=["ok"]).row_group_chunks(0)[0].npages == 1      # the other columns still read


def test_scan_types_are_sparks(tmp_path):
    """the SB type, scale word and multiplier the scan hands the kernel: decimals keep their precision, TIMESTAMP(MILLIS)
    (which is how pyarrow writes timestamp[ms] and timestamp[s]) is multiplied by 1000"""
    from spark_b200 import _capi as capi
    from spark_b200.scan import ParquetScanExec
    t, path = write_matrix(str(tmp_path), "plain", "1.0", n=100)
    scan = ParquetScanExec(path)
    by = dict(zip(scan.columns, scan.types))
    assert by["ts_us"] == (capi.SB_TIMESTAMP, 0, 1)
    assert by["ts_ms"] == by["ts_s"] == (capi.SB_TIMESTAMP, 0, 1000)
    for p, s in DECIMALS:
        assert by["dec%d_%d" % (p, s)] == (capi.SB_DECIMAL64, (p << 8) | s, 0)
    ch = dict(zip(scan.columns, scan.row_group_chunks(0)))
    assert ch["ts_ms"].c().value_multiplier == 1000 and ch["dec7_2"].c().scale == (7 << 8) | 2
