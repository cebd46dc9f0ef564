"""GPU parity of the BYTE_ARRAY and DELTA_* scan path: Parquet files written by pyarrow (and one by parquet-mr), column chunks
shipped to the GPU encoded, decoded by sb_scan_decode, compared bit for bit with pyarrow's reader and with the oracle's
restatement of the reference reader -- every case of tests/test_scan_strings_cpu.py plus the edges (NULL-only pages, empty
strings, 1 MB values, one-entry dictionaries, a dictionary -> PLAIN fallback, 2^20 + 3 rows), an arena that would overflow
int32 offsets, and TPC-H Q3 / Q5, a GROUP BY and an ORDER BY over string columns that come out of the scan."""

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq
import pytest

from test_scan_strings_cpu import (DELTA_CASES, GOLDEN, STRING_CASES, STRING_ENCODINGS, case_id, delta_values, oracle_column,
                                   string_values, write_delta_ints, write_strings)

pytestmark = pytest.mark.gpu


def _collect(path, stream, columns=None):
    from spark_b200.scan import ParquetScanExec
    return ParquetScanExec(path, columns=columns).collect(stream)


def _check_strings(path, stream, name="s", oracle=True):
    from spark_b200.scan import ParquetScanExec
    got = _collect(path, stream).column(name).combine_chunks()
    want = pq.read_table(path).column(name).combine_chunks()
    assert got.type == (pa.binary() if pa.types.is_binary(want.type) else pa.string())
    assert got.null_count == want.null_count
    assert got.to_pylist() == want.to_pylist()
    # the arena itself, byte for byte (NULL rows take no bytes)
    arena = b"".join(v.encode() if isinstance(v, str) else v for v in want.to_pylist() if v is not None)
    offsets = np.frombuffer(got.buffers()[1], np.int32)[:len(got) + 1]
    assert offsets[0] == 0 and offsets[-1] == len(arena)
    assert got.buffers()[2].to_pybytes()[:len(arena)] == arena
    if oracle:
        chunks, _ = oracle_column(ParquetScanExec(path, columns=[name]), name)
        assert [v.encode() if isinstance(v, str) else v for v in got.to_pylist()] == [v for part in chunks for v in part]
    return got


@pytest.mark.parametrize("case", STRING_CASES, ids=case_id)
def test_string_scan_equals_pyarrow_and_oracle(gpu, stream, tmp_path, case):
    n = 6000
    path = str(tmp_path / "s.parquet")
    write_strings(path, string_values(n, seed=len(case_id(case)), nullable=case["nullable"]), case["enc"], case["version"],
                  row_group_size=-(-n // case["rgs"]))
    _check_strings(path, stream)
    t = _collect(path, stream)
    assert t.column("i").to_pylist() == list(range(n))          # a fixed-width column decoded in the same call


@pytest.mark.parametrize("enc", STRING_ENCODINGS)
@pytest.mark.parametrize("n", [1, 4097, (1 << 20) + 3])
def test_string_scan_row_counts(gpu, stream, tmp_path, enc, n):
    path = str(tmp_path / "n.parquet")
    vals = string_values(n, seed=n) if n < 10_000 else ["k%08d/%s" % (i, "x" * (i % 17)) if i % 9 else None for i in range(n)]
    write_strings(path, vals, enc, "2.0" if n % 2 else "1.0", data_page_size=64 * 1024)
    _check_strings(path, stream, oracle=n < 10_000)


@pytest.mark.parametrize("enc", STRING_ENCODINGS)
def test_binary_edges(gpu, stream, tmp_path, enc):
    """0x00 / 0xFF bytes in a binary column (it comes back as binary), values of 1 MB and more (larger than a page), an
    all-NULL stretch and a stretch of empty values."""
    rng = np.random.default_rng(5)
    big = [bytes(rng.integers(0, 256, (1 << 20) + k, dtype=np.uint8)) for k in (0, 7)]
    vals = [b"\x00", b"\xff\xfe\x00\xff", b""] * 50 + [big[0], None, big[1]] + [None] * 3000 + [b""] * 3000 + [b"tail\xff"]
    path = str(tmp_path / "b.parquet")
    kw = dict(use_dictionary=["b"]) if enc == "DICTIONARY" else dict(use_dictionary=False, column_encoding={"b": enc})
    pq.write_table(pa.table({"b": pa.array(vals, pa.binary())}), path, compression="NONE", data_page_size=64 * 1024, **kw)
    got = _check_strings(path, stream, name="b")
    assert got.to_pylist()[150] == big[0] and got.to_pylist()[151] is None


def test_one_entry_dictionary_and_fallback_to_plain(gpu, stream, tmp_path):
    path = str(tmp_path / "one.parquet")
    pq.write_table(pa.table({"s": pa.array(["ASIA"] * 5000 + [None] * 10)}), path, compression="NONE", use_dictionary=True)
    _check_strings(path, stream)
    path = str(tmp_path / "fb.parquet")
    vals = ["v%07d-%s" % (i, "x" * (i % 13)) for i in range(300_000)]
    pq.write_table(pa.table({"s": pa.array(vals)}), path, compression="NONE", use_dictionary=True)
    from spark_b200.scan import ParquetScanExec
    encs = {ch.pages[i].encoding for ch in ParquetScanExec(path).row_group_chunks(0) for i in range(ch.npages)}
    assert encs == {0, 1}                                          # dictionary pages, then PLAIN once the dictionary is full
    _check_strings(path, stream, oracle=False)


def test_sorted_keys_with_long_shared_prefixes(gpu, stream, tmp_path):
    vals = sorted("warehouse/region-%02d/store-%05d/sku-%09d" % (i % 7, i // 13, i) for i in range(200_000))
    path = str(tmp_path / "dba.parquet")
    write_strings(path, vals, "DELTA_BYTE_ARRAY", data_page_size=256 * 1024)
    _check_strings(path, stream, oracle=False)


@pytest.mark.parametrize("version", ["1.0", "2.0"])
@pytest.mark.parametrize("typ,shape", DELTA_CASES, ids=["%s-%s" % c for c in DELTA_CASES])
def test_delta_binary_packed_ints(gpu, stream, tmp_path, typ, shape, version):
    from spark_b200.scan import ParquetScanExec
    path = str(tmp_path / "d.parquet")
    write_delta_ints(path, delta_values(typ, shape), typ, version, nullable=shape in ("unaligned", "negative_deltas"))
    got = _collect(path, stream).column("x").combine_chunks()
    want = pq.read_table(path).column("x").combine_chunks()
    assert got.null_count == want.null_count and got.to_pylist() == want.to_pylist()
    vals, valid = oracle_column(ParquetScanExec(path), "x")
    ok = np.asarray(want.is_valid())
    g = np.asarray((got.cast(pa.int32()) if typ == "date32" else got).fill_null(0))
    assert np.array_equal(g[ok], vals[0][ok])


def test_delta_binary_packed_many_pages_and_row_groups(gpu, stream, tmp_path):
    rng = np.random.default_rng(3)
    n = (1 << 20) + 3
    x = np.cumsum(rng.integers(-1000, 100_000, n)).astype(np.int64)
    path = str(tmp_path / "big.parquet")
    pq.write_table(pa.table({"x": x, "y": (x % 100_000).astype(np.int32)}), path, compression="NONE", use_dictionary=False,
                   column_encoding={"x": "DELTA_BINARY_PACKED", "y": "DELTA_BINARY_PACKED"}, data_page_size=64 * 1024, row_group_size=400_000)
    got = _collect(path, stream)
    assert np.array_equal(got.column("x").to_numpy(), x) and np.array_equal(got.column("y").to_numpy(), (x % 100_000).astype(np.int32))


def test_parquet_mr_fixture(gpu, stream):
    t = _collect(GOLDEN, stream, columns=["id", "name"])
    assert t.column("id").to_pylist() == [1, 2, 3]
    assert t.column("name").to_pylist() == ["Alice", "Bob", "Cecilia"]


def test_arena_larger_than_int32_offsets_is_unsupported(gpu, stream):
    """A dictionary of one 64 KiB string and a bit-width-0 page of 40 000 rows decode to 2.6 GB: refused, no wrap, no fault."""
    from spark_b200 import _capi as capi
    from spark_b200.scan import EncodedColumnChunk, decode_chunks
    entry = 64 * 1024
    data = np.zeros(4 + entry + 1, np.uint8)
    data[:4] = np.frombuffer(np.uint32(entry).tobytes(), np.uint8)
    data[4:4 + entry] = ord("x")
    data[4 + entry] = 0                                            # bit width 0: every index is 0
    pages = (capi.sb_page * 1)()
    pages[0].encoding, pages[0].num_values, pages[0].values_offset, pages[0].values_bytes = capi.SB_ENC_RLE_DICTIONARY, 40_000, 4 + entry, 1
    ch = EncodedColumnChunk(capi.SB_STRING, 0, capi.SB_PHYS["BYTE_ARRAY"], data, pages, 1, 0, 1)
    with pytest.raises(capi.SparkB200Error) as e:
        decode_chunks(["s"], [ch], stream)
    assert e.value.code == 5 and "2^31 - 1" in str(e.value)
    pages[0].num_values = 1000                                    # 64 MB: decodes
    b = decode_chunks(["s"], [ch], stream)
    try:
        s = b.to_arrow(stream).column("s")
        assert len(s) == 1000 and s[999].as_py() == "x" * entry
    finally:
        b.close()


# ---- downstream: TPC-H Q3 / Q5 with string c_mktsegment / r_name read from Parquet --------------------------------------------

@pytest.mark.parametrize("enc", STRING_ENCODINGS)
def test_q3_q5_group_by_order_by_over_scanned_strings(gpu, stream, tmp_path, enc):
    from oracle import tpch_oracle as TO
    from spark_b200 import tpch
    from spark_b200.execution import HashAggregateExec, SortExec
    from spark_b200.expressions import Count
    from spark_b200.scan import ParquetScanExec
    from test_gpu_string_predicates import REGIONS, _with_string_filter
    from util import assert_tables_equal
    sf = 0.05
    customer, orders = tpch.customer_table(sf), tpch.orders_table(sf)
    lineitem = tpch.lineitem_join_table(orders, sf)
    supplier, nation, region = tpch.supplier_table(sf), tpch.nation_table(), tpch.region_table()
    customer_s = customer.set_column(customer.schema.get_field_index("c_mktsegment"), "c_mktsegment",
                                     pa.array([tpch.SEGMENTS[c] for c in customer.column("c_mktsegment").to_numpy()]))
    region_s = region.set_column(region.schema.get_field_index("r_name"), "r_name", pa.array([REGIONS[c] for c in region.column("r_name").to_numpy()]))

    def scan(name, t):
        path = str(tmp_path / (name + ".parquet"))
        strs = [f.name for f in t.schema if pa.types.is_string(f.type)]
        kw = dict(use_dictionary=strs) if enc == "DICTIONARY" else dict(use_dictionary=False, column_encoding={s: enc for s in strs})
        pq.write_table(t, path, compression="NONE", data_page_size=64 * 1024, row_group_size=100_000, **kw)
        return ParquetScanExec(path)

    got = _with_string_filter(tpch.q3_plan(scan("customer", customer_s), scan("orders", orders), scan("lineitem", lineitem)),
                              "c_mktsegment", "BUILDING").collect(stream)
    want, _ = TO.q3(customer, orders, lineitem, tpch.Q3_SEGMENT, tpch.Q3_DATE)
    assert_tables_equal(got, want, ordered=True)
    got = _with_string_filter(tpch.q5_plan(scan("customer", customer_s), scan("orders", orders), scan("lineitem", lineitem),
                                           scan("supplier", supplier), scan("nation", nation), scan("region", region_s)),
                              "r_name", "ASIA").collect(stream)
    want = TO.q5(customer, orders, lineitem, supplier, nation, region, tpch.Q5_REGION, tpch.Q5_DATE_LO, tpch.Q5_DATE_HI)
    assert want.num_rows == 5
    assert_tables_equal(got, want, ordered=True)
    # GROUP BY and ORDER BY on the scanned string column
    c = scan("customer", customer_s)
    counts = HashAggregateExec(["c_mktsegment"], [(Count(), "n")], c).collect(stream)
    want_counts = customer_s.group_by("c_mktsegment").aggregate([("c_mktsegment", "count")])
    assert dict(zip(counts.column("c_mktsegment").to_pylist(), counts.column("n").to_pylist())) == \
        dict(zip(want_counts.column("c_mktsegment").to_pylist(), want_counts.column("c_mktsegment_count").to_pylist()))
    srt = SortExec([("c_mktsegment", True, True)], c).collect(stream)
    assert srt.column("c_mktsegment").to_pylist() == sorted(customer_s.column("c_mktsegment").to_pylist(), key=lambda s: s.encode())
