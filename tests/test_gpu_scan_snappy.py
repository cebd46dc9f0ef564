"""GPU parity of the Snappy scan path: Parquet files written SNAPPY by pyarrow (and by parquet-mr: the reference's goldens),
decompressed and decoded on the GPU by sb_scan_decode_compressed, compared bit for bit (values and validity) with pyarrow's
reader and with the same data written NONE through the uncompressed path; hand-built chunks carrying every Snappy element form
and every malformed stream of tests/snappy_streams.py; Q1 and a join + GROUP BY over SNAPPY files."""
import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq
import pytest

import snappy_streams as SS
from test_scan_cpu import CASES, _table
from test_scan_snappy_cpu import (DECIMAL32, DECIMAL32_DICT_FIRST, DECIMAL32_DICT_LAST, THRIFT_FLAT, golden, thrift_compat_rows)
from test_scan_strings_cpu import STRING_CASES, _zz, case_id, string_values, write_strings

pytestmark = pytest.mark.gpu


def _collect(path, stream, columns=None):
    from spark_b200.scan import ParquetScanExec
    return ParquetScanExec(path, columns=columns).collect(stream)


def _same(got, want):
    """bit for bit: validity, and values (doubles compared as bits)"""
    assert got.num_rows == want.num_rows
    for name in want.column_names:
        g, w = got.column(name).combine_chunks(), want.column(name).combine_chunks()
        assert g.null_count == w.null_count, name
        assert np.array_equal(np.asarray(g.is_valid()), np.asarray(w.is_valid())), name
        if pa.types.is_floating(w.type):
            gv, wv = np.asarray(g.fill_null(0)), np.asarray(w.cast(g.type).fill_null(0))
            assert np.array_equal(gv.view(np.uint8), wv.view(np.uint8)), name
        else:
            assert g.to_pylist() == w.cast(g.type).to_pylist(), name


def _snappy_and_none(tmp_path, table, **kw):
    a, b = str(tmp_path / "snappy.parquet"), str(tmp_path / "none.parquet")
    pq.write_table(table, a, compression="SNAPPY", **kw)
    pq.write_table(table, b, compression="NONE", **kw)
    return a, b


def _check_file_pair(stream, a, b, columns=None):
    got = _collect(a, stream, columns)
    _same(got, pq.read_table(a, columns=columns))
    _same(got, _collect(b, stream, columns))
    return got


@pytest.mark.parametrize("case", CASES, ids=lambda c: "v%s-dict%s-n%d" % (c["version"], "sel" if isinstance(c["use_dictionary"], list) else c["use_dictionary"], c["n"]))
def test_fixed_width_cases_written_snappy(gpu, stream, tmp_path, case):
    t = _table(case["n"], seed=case["n"])
    a, b = _snappy_and_none(tmp_path, t, use_dictionary=case["use_dictionary"], data_page_version=case["version"], data_page_size=16 * 1024)
    _check_file_pair(stream, a, b)


@pytest.mark.parametrize("case", STRING_CASES, ids=case_id)
def test_string_cases_written_snappy(gpu, stream, tmp_path, case):
    n = 6000
    vals = string_values(n, seed=len(case_id(case)), nullable=case["nullable"])
    t = write_strings(str(tmp_path / "x.parquet"), vals, case["enc"], case["version"], row_group_size=-(-n // case["rgs"]))
    kw = dict(use_dictionary=["s"]) if case["enc"] == "DICTIONARY" else dict(use_dictionary=False, column_encoding={"s": case["enc"]})
    a, b = _snappy_and_none(tmp_path, t, data_page_version=case["version"], data_page_size=4096, row_group_size=-(-n // case["rgs"]), **kw)
    _check_file_pair(stream, a, b)


@pytest.mark.parametrize("shape", ["rows-2^20+3", "8k-pages", "4m-pages", "random-doubles", "constant", "all-null"])
def test_sizes_and_shapes(gpu, stream, tmp_path, shape):
    rng = np.random.default_rng(7)
    n = (1 << 20) + 3 if shape in ("rows-2^20+3", "4m-pages", "random-doubles", "constant") else 200_000
    kw = dict(use_dictionary=False)
    if shape == "rows-2^20+3":
        t = pa.table({"k": pa.array(np.arange(n) // 7), "s": pa.array(["key-%07d" % (i % 5000) for i in range(n)]),
                      "f": pa.array(rng.integers(0, 1000, n) / 100.0, mask=rng.random(n) < 0.1)})
        kw = dict(use_dictionary=["f"])
    elif shape == "8k-pages":
        t = pa.table({"x": pa.array(np.cumsum(rng.integers(0, 9, n))), "y": pa.array(rng.integers(0, 3, n).astype(np.int32))})
        kw["data_page_size"] = 8 * 1024
    elif shape == "4m-pages":
        t = pa.table({"x": pa.array(np.cumsum(rng.integers(0, 9, n)).astype(np.int64) % 100_000)})
        kw["data_page_size"] = 4 << 20
    elif shape == "random-doubles":
        t = pa.table({"d": pa.array(rng.standard_normal(n))})
    elif shape == "constant":
        t = pa.table({"c": pa.array(np.full(n, 3.25)), "i": pa.array(np.full(n, 7, np.int32))})
    else:
        t = pa.table({"z": pa.array([None] * n, pa.int64()), "w": pa.array([None] * n, pa.string())})
        kw = dict(use_dictionary=True)
    a, b = _snappy_and_none(tmp_path, t, **kw)
    _check_file_pair(stream, a, b)


def test_mixed_codecs_in_one_row_group_and_compressed_dictionary(gpu, stream, tmp_path):
    n = 50_000
    rng = np.random.default_rng(2)
    t = pa.table({"a": pa.array(rng.integers(0, 30, n)), "b": pa.array(["v%d" % (i % 77) for i in range(n)]), "c": pa.array(rng.standard_normal(n))})
    a, b = str(tmp_path / "mix.parquet"), str(tmp_path / "none.parquet")
    pq.write_table(t, a, compression={"a": "SNAPPY", "b": "SNAPPY", "c": "NONE"}, use_dictionary=["a", "b"])
    pq.write_table(t, b, compression="NONE", use_dictionary=["a", "b"])
    from spark_b200.scan import ParquetScanExec
    chunks = ParquetScanExec(a).row_group_file_chunks(0)
    assert [ch.codec for ch in chunks] == [1, 1, 0]
    assert any(ch.spans[i].page_type == 2 and ch.spans[i].values_compressed for ch in chunks[:2] for i in range(ch.npages))
    _check_file_pair(stream, a, b)


# ---- hand-built chunks -------------------------------------------------------------------------------------------------------

def _v1_page(body, uncompressed, num_values, encoding=0):
    inner = b"\x15" + _zz(num_values) + b"\x15" + _zz(encoding) + b"\x15" + _zz(3) + b"\x15" + _zz(3) + b"\x00"
    return b"\x15" + _zz(0) + b"\x15" + _zz(uncompressed) + b"\x15" + _zz(len(body)) + b"\x2c" + inner + b"\x00" + body


def _v2_page(levels, values, uncompressed_values, num_values, num_nulls, is_compressed, encoding=0):
    inner = (b"\x15" + _zz(num_values) + b"\x15" + _zz(num_nulls) + b"\x15" + _zz(num_values) + b"\x15" + _zz(encoding) + b"\x15" + _zz(len(levels))
             + b"\x15" + _zz(0) + (b"\x11" if is_compressed else b"\x12") + b"\x00")
    body = levels + values
    return (b"\x15" + _zz(3) + b"\x15" + _zz(len(levels) + uncompressed_values) + b"\x15" + _zz(len(body)) + b"\x5c" + inner + b"\x00" + body)


def _decode(chunk: bytes, stream, physical, sb_type, max_def=0):
    from spark_b200 import _capi as capi
    from spark_b200.scan import CompressedColumnChunk, decode_file_chunks
    ch = CompressedColumnChunk.from_file_bytes(np.frombuffer(chunk, np.uint8).copy(), sb_type, 0, capi.SB_PHYS[physical], capi.SB_CODEC["SNAPPY"], max_def)
    b = decode_file_chunks(["x"], [ch], stream)
    try:
        return b.to_arrow(stream).column("x").combine_chunks()
    finally:
        b.close()


def test_every_valid_element_form_decodes(gpu, stream):
    """each stream of snappy_streams.valid_streams() as the body of a PLAIN INT32 page, then all of them as one chunk"""
    from spark_b200 import _capi as capi
    pages, want = b"", []
    for name, (s, out) in SS.valid_streams().items():
        n = len(out) // 4
        page = _v1_page(s, len(out), n)
        got = _decode(page, stream, "INT32", capi.SB_INT32)
        w = np.frombuffer(out[:4 * n], np.int32).tolist()
        assert got.to_pylist() == w, name
        pages += page
        want += w
    assert _decode(pages, stream, "INT32", capi.SB_INT32).to_pylist() == want


@pytest.mark.parametrize("name", sorted(SS.malformed_streams()))
def test_malformed_stream_is_invalid_and_names_the_page(gpu, stream, name):
    from spark_b200 import _capi as capi
    s, declared, status = SS.malformed_streams()[name]
    good = SS.Writer().literal(b"\x01\x00\x00\x00\x02\x00\x00\x00")
    chunk = _v1_page(good.stream(), 8, 2) + _v1_page(s, declared, declared // 4)
    with pytest.raises(capi.SparkB200Error) as e:
        _decode(chunk, stream, "INT32", capi.SB_INT32)
    want = {SS.BAD_PREAMBLE: "preamble", SS.LENGTH_MISMATCH: "uncompressed size", SS.INPUT_OVERRUN: "past the end of the input",
            SS.BAD_OFFSET: "copy offset", SS.OUTPUT_OVERRUN: "past the declared length", SS.LEFTOVER: "left over",
            SS.SHORT: "ends before"}[status]
    assert e.value.code == 2 and "page 1" in str(e.value) and want in str(e.value), str(e.value)
    assert _decode(_v1_page(good.stream(), 8, 2), stream, "INT32", capi.SB_INT32).to_pylist() == [1, 2]   # the stream is still usable


def test_v2_pages_with_uncompressed_values_inside_a_snappy_chunk(gpu, stream):
    """V2 pages whose is_compressed is false sit in a SNAPPY chunk next to compressed V1 and V2 pages; an optional INT64 column"""
    from spark_b200 import _capi as capi
    vals = np.arange(1, 41, dtype=np.int64) * 1000003
    levels = b"\x50\x01"                             # RLE run of 40 definition levels = 1
    raw = vals[:40].tobytes()
    v1_body = np.uint32(len(levels)).tobytes() + levels + raw
    w = SS.Writer().literal(v1_body[:9]).literal(v1_body[9:])
    chunk = (_v1_page(w.stream(), len(v1_body), 40)
             + _v2_page(levels, raw, len(raw), 40, 0, is_compressed=False)
             + _v2_page(levels, SS.Writer().literal(raw).stream(), len(raw), 40, 0, is_compressed=True))
    got = _decode(chunk, stream, "INT64", capi.SB_INT64, max_def=1)
    assert got.null_count == 0 and got.to_pylist() == vals.tolist() * 3


# ---- the reference's goldens -----------------------------------------------------------------------------------------------

def test_parquet_thrift_compat_golden(gpu, stream):
    from spark_b200 import _capi as capi
    path = golden("parquet-thrift-compat.snappy.parquet")
    got = _collect(path, stream, THRIFT_FLAT)
    want = thrift_compat_rows()
    for name in THRIFT_FLAT:
        g = got.column(name).to_pylist()
        if name.endswith("DoubleColumn"):
            assert [None if v is None else round(v, 9) for v in g] == want[name], name
        else:
            text = [v.decode() if isinstance(v, bytes) else v for v in want[name]]
            assert [v.decode() if isinstance(v, bytes) else v for v in g] == text, name
    _same(got, pq.read_table(path, columns=THRIFT_FLAT))
    with pytest.raises(capi.SparkB200Error) as e:
        _collect(path, stream, ["stringsColumn"])
    assert e.value.code == 5


def test_decimal32_written_as_64_bit_goldens(gpu, stream):
    got = _collect(golden("decimal32-written-as-64-bit.snappy.parquet"), stream).column("_c0")
    assert [None if v is None else int(v.scaleb(1)) for v in got.to_pylist()] == DECIMAL32
    got = _collect(golden("decimal32-written-as-64-bit-dict.snappy.parquet"), stream).column("_c0").to_pylist()
    assert len(got) == 2048
    unscaled = [None if v is None else int(v.scaleb(1)) for v in got]
    assert unscaled[:10] == DECIMAL32_DICT_FIRST and unscaled[-10:] == DECIMAL32_DICT_LAST


# ---- downstream ------------------------------------------------------------------------------------------------------------

def test_q1_over_a_snappy_file_equals_uncompressed_and_oracle(gpu, stream, tmp_path):
    from oracle import oracle as O
    from spark_b200 import tpch
    from spark_b200.scan import ParquetScanExec
    from util import assert_tables_equal
    t = tpch.lineitem_q1_table(1 << 22, seed=3)
    a, b = _snappy_and_none(tmp_path, t, row_group_size=1 << 20)
    assert pq.ParquetFile(a).metadata.num_row_groups == 4

    def q1(path):
        return tpch.q1_final_plan(tpch.q1_partial_plan(ParquetScanExec(path), fused=True), sort=True).collect(stream)

    _same(_collect(a, stream), _collect(b, stream))  # the scanned columns bit for bit, doubles included
    got = q1(a)
    assert_tables_equal(got, q1(b), ordered=True)    # the floating sums depend on the aggregate's atomic order
    f = O.filter_table(t, ("le", ("col", "l_shipdate"), ("lit", tpch.Q1_CUTOFF, np.int32)))
    dp = ("mul", ("col", "l_extendedprice"), ("sub", ("lit", 1.0), ("col", "l_discount")))
    p = O.project(f, [(c, ("col", c)) for c in ["l_returnflag", "l_linestatus", "l_quantity", "l_extendedprice", "l_discount"]] +
                  [("disc_price", dp), ("charge", ("mul", dp, ("add", ("lit", 1.0), ("col", "l_tax"))))])
    want = O.sort(O.hash_aggregate(p, tpch.Q1_KEYS, tpch.q1_oracle_aggs()), [("l_returnflag", True, True), ("l_linestatus", True, True)])
    assert_tables_equal(got, want, ordered=True, rtol=1e-9)


def test_q3_join_group_by_over_snappy_string_columns(gpu, stream, tmp_path):
    from oracle import tpch_oracle as TO
    from spark_b200 import tpch
    from spark_b200.execution import HashAggregateExec
    from spark_b200.expressions import Count
    from spark_b200.scan import ParquetScanExec
    from test_gpu_string_predicates import _with_string_filter
    from util import assert_tables_equal
    sf = 0.05
    customer, orders = tpch.customer_table(sf), tpch.orders_table(sf)
    lineitem = tpch.lineitem_join_table(orders, sf)
    customer_s = customer.set_column(customer.schema.get_field_index("c_mktsegment"), "c_mktsegment",
                                     pa.array([tpch.SEGMENTS[c] for c in customer.column("c_mktsegment").to_numpy()]))

    def scan(name, t):
        path = str(tmp_path / (name + ".parquet"))
        pq.write_table(t, path, compression="SNAPPY", use_dictionary=False, data_page_size=64 * 1024, row_group_size=100_000)
        return ParquetScanExec(path)

    got = _with_string_filter(tpch.q3_plan(scan("customer", customer_s), scan("orders", orders), scan("lineitem", lineitem)),
                              "c_mktsegment", "BUILDING").collect(stream)
    want, _ = TO.q3(customer, orders, lineitem, tpch.Q3_SEGMENT, tpch.Q3_DATE)
    assert_tables_equal(got, want, ordered=True)
    counts = HashAggregateExec(["c_mktsegment"], [(Count(), "n")], scan("customer", customer_s)).collect(stream)
    want_counts = customer_s.group_by("c_mktsegment").aggregate([("c_mktsegment", "count")])
    assert dict(zip(counts.column("c_mktsegment").to_pylist(), counts.column("n").to_pylist())) == \
        dict(zip(want_counts.column("c_mktsegment").to_pylist(), want_counts.column("c_mktsegment_count").to_pylist()))
