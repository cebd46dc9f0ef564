"""GPU half of the fixed-width scan matrix (files and references: tests/test_scan_types_cpu.py): every column the GPU scan
decodes is compared BIT FOR BIT -- raw value bits, validity and Arrow type, decimal precision and timestamp unit included --
with two references that never see the GPU's result type: pyarrow's reader (timestamps converted to microseconds as Spark
converts them) and the oracle's restatement of the page decoding of the same page bytes (oracle/parquet_oracle.py,
tests/parquet_delta_oracle.py).  Plus the block striping of one page over several blocks, the types reaching the operators
downstream, and the write-side twin (sb_scan_encode) as the identity on every type it takes, NaN payloads and -0.0 included."""
import ctypes as C
import os

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq
import pytest

import test_scan_types_cpu as M
from test_gpu_key_types import assert_bits_equal

pytestmark = pytest.mark.gpu


def _scan_all(path, stream):
    """the file through executeColumnar, and row group by row group through batches()"""
    from spark_b200.scan import ParquetScanExec
    scan = ParquetScanExec(path)
    whole = scan.collect(stream)
    parts = []
    for b in scan.batches(stream):
        parts.append(b.to_arrow(stream))
        b.close()
    return whole, parts


def _check_file(path, stream, oracle_path=None, input_table=None):
    """GPU == oracle (on the uncompressed twin's page bytes for a compressed file) == pyarrow, whole file and per row group"""
    oracle_path = oracle_path or path
    got, parts = _scan_all(path, stream)
    assert_bits_equal(got, M.oracle_table(oracle_path), ordered=True)
    assert_bits_equal(got, M.pyarrow_table(path), ordered=True)
    for rg, part in enumerate(parts):
        assert_bits_equal(part, M.oracle_table(oracle_path, rg), ordered=True)
    if input_table is not None:
        assert_bits_equal(got, M.spark_input(input_table), ordered=True)
    return got


@pytest.mark.parametrize("compression", ["NONE", "SNAPPY"])
@pytest.mark.parametrize("version", M.VERSIONS)
@pytest.mark.parametrize("encoding", M.ENCODINGS)
def test_every_type_encoding_page_version_and_null_pattern(gpu, stream, tmp_path, encoding, version, compression):
    d = str(tmp_path)
    t, plain = M.write_matrix(d, encoding, version, "NONE")
    path = plain if compression == "NONE" else M.write_matrix(d, encoding, version, compression)[1]
    got = _check_file(path, stream, oracle_path=plain)
    if encoding in ("plain", "delta"):     # no dictionary that could merge NaN payloads or signed zeros: the input itself
        assert_bits_equal(got, M.spark_input(t), ordered=True)


def test_single_row(gpu, stream, tmp_path):
    t, path = M.write_matrix(str(tmp_path), "dict", "1.0", n=1, seed=5)
    _check_file(path, stream, input_table=t)


def test_null_layouts_and_the_all_null_chunk(gpu, stream, tmp_path):
    path = M.write_nulls(str(tmp_path))
    _check_file(path, stream)


def test_dictionary_index_widths(gpu, stream, tmp_path):
    """bit widths 1 .. 21 from parquet-cpp, one row group per dictionary size, and 0 from a parquet-mr-style one-entry chunk"""
    from spark_b200.scan import decode_chunks
    tables, path = M.write_dict_widths(str(tmp_path))
    got, parts = _scan_all(path, stream)
    for rg, part in enumerate(parts):
        assert_bits_equal(part, M.oracle_table(path, rg), ordered=True)
        assert_bits_equal(part, tables[rg], ordered=True)
    for n in (1, 1000, 70_001):
        ch = M.one_entry_dictionary_chunk(n, -7)
        b = decode_chunks(["v"], [ch], stream, [pa.int64()])
        assert_bits_equal(b.to_arrow(stream), pa.table({"v": pa.array(np.full(n, -7, np.int64))}), ordered=True)
        b.close()


@pytest.mark.parametrize("version", M.VERSIONS)
def test_hybrid_stream_shapes(gpu, stream, tmp_path, version):
    t, path = M.write_hybrid(str(tmp_path), version)
    _check_file(path, stream, input_table=t)


@pytest.mark.parametrize("compression", ["NONE", "SNAPPY"])
def test_plain_pages_on_and_off_16_byte_boundaries(gpu, stream, tmp_path, compression):
    t, plain = M.write_geometry(str(tmp_path))
    path = plain if compression == "NONE" else M.write_geometry(str(tmp_path), compression)[1]
    _check_file(path, stream, oracle_path=plain, input_table=t)


def test_one_page_striped_over_blocks_decodes_like_many_pages(gpu, stream, tmp_path):
    """the same NULL-free dictionary column as one page (16 blocks), ~100 pages (1 < blocks per page < 16) and ~1000 pages (one
    block each): bit-identical answers, and all three striping regimes reached on this device"""
    from spark_b200 import _capi as capi
    info = (C.c_int64 * 4)()
    capi.check(capi.load().sb_device_info(info))
    sms = int(info[0])
    t, paths = M.write_stripes(str(tmp_path))
    regimes, results = [], []
    for name, path in paths.items():
        _, ch = M.chunks_of(path)
        regimes.append(M.expected_nparts(sms, ch["v"].npages))
        results.append(_check_file(path, stream, input_table=t))
    assert regimes[0] == 16 and 1 < regimes[1] < 16 and regimes[2] == 1, (sms, regimes)
    for r in results[1:]:
        assert_bits_equal(r, results[0], ordered=True)


# ---- downstream: the scanned types reach the operators
def test_sum_and_avg_of_a_scanned_decimal_7_2(gpu, stream, tmp_path):
    """Sum and Average derive their result types from the input's precision: decimal(7,2) -> decimal(17,2) and decimal(11,6).
    The scanned column gives what the same values imported from Arrow give, and the exact answers (Average rounds HALF_UP)"""
    import decimal as D
    from spark_b200.columnar import ColumnarBatch
    from spark_b200.execution import HashAggregateExec, LocalTableScanExec
    from spark_b200.expressions import Average, Sum, col
    from spark_b200.scan import ParquetScanExec
    rng = np.random.default_rng(2)
    n = 20_011
    v = M.random_values(pa.decimal128(7, 2), n, rng)
    k = rng.integers(0, 7, n).astype(np.int32)
    valid = rng.random(n) > 0.1
    t = pa.table({"k": pa.array(k), "d": M.make_array(pa.decimal128(7, 2), v, valid)})
    path = os.path.join(str(tmp_path), "dec.parquet")
    pq.write_table(t, path, compression="NONE", store_decimal_as_integer=True, max_rows_per_page=3001)
    aggs = [(Sum(col("d")), "s"), (Average(col("d")), "a")]
    got = HashAggregateExec(["k"], aggs, ParquetScanExec(path)).collect(stream)
    imported = ColumnarBatch.from_arrow(t, stream)
    want = HashAggregateExec(["k"], aggs, LocalTableScanExec(imported)).collect(stream)
    imported.close()
    assert got.schema.types == [pa.int32(), pa.decimal128(17, 2), pa.decimal128(11, 6)], got.schema
    assert_bits_equal(got, want)
    exact = {}
    for key in range(7):
        sel = (k == key) & valid
        total = int(v[sel].sum())
        avg = (D.Decimal(total).scaleb(-2) / D.Decimal(int(sel.sum()))).quantize(D.Decimal("1e-6"), rounding=D.ROUND_HALF_UP)
        exact[key] = (D.Decimal(total).scaleb(-2), avg)
    rows = got.to_pylist()
    assert len(rows) == 7 and all((r["s"], r["a"]) == exact[r["k"]] for r in rows), rows


def test_filter_on_a_scanned_millisecond_timestamp(gpu, stream, tmp_path):
    from oracle import oracle as O
    from spark_b200.execution import FilterExec
    from spark_b200.expressions import GreaterThanOrEqual, Literal, col
    from spark_b200.scan import ParquetScanExec
    rng = np.random.default_rng(4)
    n = 10_007
    ms = rng.integers(-2_000_000_000_000, 2_000_000_000_000, n)
    t = pa.table({"ts": M.make_array(pa.timestamp("ms"), ms, rng.random(n) > 0.05), "row": pa.array(np.arange(n, dtype=np.int64))})
    path = os.path.join(str(tmp_path), "ts.parquet")
    pq.write_table(t, path, compression="NONE")
    cut = int(np.median(ms)) * 1000 + 1                     # microseconds: only the converted column splits here
    cond = GreaterThanOrEqual(col("ts"), Literal(cut))
    got = FilterExec(cond, ParquetScanExec(path)).collect(stream)
    want = O.filter_table(M.spark_input(t), cond.sexpr())
    assert 0.4 * n < want.num_rows < 0.6 * n
    assert_bits_equal(got, want, ordered=True)


# ---- the write-side twin
ENCODE_TYPES = {"int8": pa.int8(), "int16": pa.int16(), "int32": pa.int32(), "date32": pa.date32(), "int64": pa.int64(),
                "timestamp": pa.timestamp("us"), "dec18_2": pa.decimal128(18, 2), "dec7_2": pa.decimal128(7, 2),
                "float32": pa.float32(), "float64": pa.float64()}


def _encode_values(t, size, n, rng):
    """n values over exactly min(size, what the type holds) distinct bit patterns (floats: their specials first: NaN payloads,
    -0.0 and 0.0 are distinct entries)"""
    if pa.types.is_floating(t) or pa.types.is_decimal(t) or pa.types.is_timestamp(t):
        pool = M.random_values(t, max(size, 64) * 4, rng)
    else:
        info = np.iinfo(M.storage_dtype(t))
        pool = np.concatenate([M.specials(t), rng.integers(int(info.min), int(info.max), 4 * size + 64, dtype=np.int64, endpoint=True)])
        pool = pool.astype(M.storage_dtype(t))
    u = np.ascontiguousarray(pool).view({1: np.uint8, 2: np.uint16, 4: np.uint32, 8: np.uint64}[pool.dtype.itemsize])
    pool = pool[np.sort(np.unique(u, return_index=True)[1])][:size]
    v = pool[np.concatenate([np.arange(len(pool)), rng.integers(0, len(pool), n - len(pool))])]
    return v, len(pool)


@pytest.mark.parametrize("tname", list(ENCODE_TYPES))
def test_encode_decode_is_the_identity_on_every_type(gpu, stream, tname):
    """sb_scan_encode -> decode_chunks returns every bit it was given (dictionary sizes 1 .. 2^16 + 1, pages of 8 .. 1000 rows,
    PLAIN for the 4- and 8-byte types), and the oracle's restatement decodes the same bytes to the same bits"""
    from parquet_delta_oracle import decode_column_chunk
    from spark_b200.columnar import ColumnarBatch
    from spark_b200.scan import decode_chunks, encode_column
    t = ENCODE_TYPES[tname]
    rng = np.random.default_rng(len(tname))
    for size in (1, 2, 255, 256, 257, 2 ** 16 + 1):
        n = max(3 * size, 2003)
        v, distinct = _encode_values(t, size, n, rng)
        table = pa.table({"c": M.make_array(t, v)})
        batch = ColumnarBatch.from_arrow(table, stream)
        try:
            for page_rows in (8, 504, 512, 1000):
                for dictionary in (True, False) if t.bit_width >= 32 and size == 257 else (True,):
                    ch = encode_column(batch, "c", dictionary=dictionary, page_rows=page_rows, stream=stream)
                    if dictionary:
                        assert ch.dict_count == distinct, (size, ch.dict_count, distinct)
                    back = decode_chunks(["c"], [ch], stream, [t])
                    assert_bits_equal(back.to_arrow(stream), table, ordered=True)
                    back.close()
                    vals, valid = decode_column_chunk(ch.data, M.page_tuples(ch), ch.dict_offset, ch.dict_count, ch.physical)
                    want = np.ascontiguousarray(v).astype(np.int64 if pa.types.is_decimal(t) else v.dtype)
                    got = vals.astype(want.dtype) if vals.dtype.kind in "iu" and want.dtype.kind in "iu" else vals.view(want.dtype)
                    assert valid is None and np.array_equal(got.view(np.uint8), want.view(np.uint8)), (tname, size, page_rows)
        finally:
            batch.close()
