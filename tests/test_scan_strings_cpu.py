"""CPU tests of the BYTE_ARRAY and DELTA_* side of the scan boundary: the product's page walker (sb_parquet_chunk_pages, host
only) and the oracle's restatement of the page decoding (tests/parquet_delta_oracle.py), both against files written -- and read
back -- by pyarrow (parquet-cpp), and against one string file written by parquet-mr (tests/golden/timestamp-nanos.parquet)."""
import ctypes as C
import os

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq
import pytest

import parquet_delta_oracle as DO

# The reference's sql/core/src/test/resources/test-data/timestamp-nanos.parquet, byte for byte (784 bytes, sha256 16d726f5...0786e):
# written by parquet-mr 1.12.3, uncompressed; `id` INT64 required, `name` BYTE_ARRAY optional PLAIN = Alice, Bob, Cecilia.  The one
# string file here from a writer other than pyarrow.
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "timestamp-nanos.parquet")
GOLDEN_SHA256 = "16d726f55f2a31e8d12db62f5e9070be42a03653b1d704ac0b3c4e8633d0786e"
STRING_ENCODINGS = ["PLAIN", "DICTIONARY", "DELTA_LENGTH_BYTE_ARRAY", "DELTA_BYTE_ARRAY"]
INT32_MIN, INT32_MAX = -2 ** 31, 2 ** 31 - 1
INT64_MIN, INT64_MAX = -2 ** 63, 2 ** 63 - 1


def string_values(n, seed=0, nullable=True):
    """NULLs (some pages all NULL), empty strings (a stretch of only empty strings), 0x00 / 0xFF bytes, multi-byte UTF-8,
    repeated values and sorted keys with long shared prefixes."""
    rng = np.random.default_rng(seed)
    words = ["", "a", "ASIA", "BUILDING", "z" * 40, "été", "日本語", "\U0001f600x", "nul\x00byte", "\x7f" * 3]
    out = []
    for i in range(n):
        k = int(rng.integers(0, 4))
        if k == 0:
            out.append(words[int(rng.integers(0, len(words)))])
        elif k == 1:
            out.append("common-prefix/of/a/sorted/key/%09d" % i)
        elif k == 2:
            out.append("".join(chr(int(c)) for c in rng.integers(32, 0x2FF, int(rng.integers(0, 30)))))
        else:
            out.append(words[i % 3])
    if n > 200:
        out[100:180] = [""] * 80                                # a page's worth of empty strings
    if nullable:
        mask = rng.random(n) < 0.2
        if n > 3000:
            mask[1000:3000] = True                              # whole pages of NULLs
        out = [None if m else v for v, m in zip(out, mask)]
    return out


def write_strings(path, values, encoding, version="1.0", row_group_size=None, data_page_size=4096, binary=False):
    typ = pa.binary() if binary else pa.string()
    arr = pa.array([None if v is None else (v.encode("utf-8", "surrogatepass") if binary else v) for v in values], typ)
    t = pa.table({"s": arr, "i": pa.array(np.arange(len(values), dtype=np.int64))})
    kw = dict(use_dictionary=["s"]) if encoding == "DICTIONARY" else dict(use_dictionary=False, column_encoding={"s": encoding})
    pq.write_table(t, path, compression="NONE", data_page_version=version, data_page_size=data_page_size,
                   row_group_size=row_group_size or max(1, len(values)), **kw)
    return t


def page_tuples(ch):
    return [(ch.pages[i].encoding, ch.pages[i].num_values, ch.pages[i].values_offset, ch.pages[i].values_bytes,
             ch.pages[i].def_offset, ch.pages[i].def_bytes) for i in range(ch.npages)]


def oracle_column(scan, name):
    """the oracle's decode of every row group of one column"""
    idx = scan.columns.index(name)
    out, valid = [], []
    for rg in range(scan.meta.num_row_groups):
        ch = scan.row_group_chunks(rg)[idx]
        v, ok = DO.decode_column_chunk(ch.data, page_tuples(ch), ch.dict_offset, ch.dict_count, ch.physical)
        out.append(v)
        valid.append(ok)
    return out, valid


STRING_CASES = [dict(enc=e, version=v, nullable=nl, rgs=rgs) for e in STRING_ENCODINGS for v in ("1.0", "2.0")
                for nl in (False, True) for rgs in (1, 3)]


def case_id(c):
    return "%s-v%s-%s-rg%d" % (c["enc"], c["version"], "opt" if c["nullable"] else "req", c["rgs"])


@pytest.mark.parametrize("case", STRING_CASES, ids=case_id)
def test_string_pages_walker_and_oracle_against_pyarrow(tmp_path, case):
    from spark_b200.scan import ParquetScanExec
    n = 6000
    vals = string_values(n, seed=len(case_id(case)), nullable=case["nullable"])
    path = str(tmp_path / "s.parquet")
    write_strings(path, vals, case["enc"], case["version"], row_group_size=-(-n // case["rgs"]))
    if not case["nullable"]:   # pyarrow writes a column of a table without NULLs as optional; the walker handles both
        assert None not in vals
    scan = ParquetScanExec(path, columns=["s"])
    assert scan.meta.num_row_groups == case["rgs"]
    chunks, _ = oracle_column(scan, "s")
    got = [v for part in chunks for v in part]
    want = [None if v is None else v.encode("utf-8") for v in pq.read_table(path).column("s").to_pylist()]
    assert got == want
    encs = {e for rg in range(case["rgs"]) for e in (p[0] for p in page_tuples(scan.row_group_chunks(rg)[0]))}
    expect = {"PLAIN": DO.ENC_PLAIN, "DICTIONARY": DO.ENC_RLE_DICTIONARY, "DELTA_LENGTH_BYTE_ARRAY": DO.ENC_DELTA_LENGTH_BYTE_ARRAY,
              "DELTA_BYTE_ARRAY": DO.ENC_DELTA_BYTE_ARRAY}[case["enc"]]
    assert encs == {expect}
    if case["enc"] != "DICTIONARY":                                         # small data_page_size: many pages of values
        assert scan.row_group_chunks(0)[0].npages > 1


def test_dictionary_falls_back_to_plain_inside_one_chunk(tmp_path):
    from spark_b200.scan import ParquetScanExec
    n = 60_000
    vals = ["v%07d-%s" % (i, "x" * (i % 13)) for i in range(n)]           # high cardinality: the dictionary overflows
    path = str(tmp_path / "fb.parquet")
    t = pa.table({"s": pa.array(vals)})
    pq.write_table(t, path, compression="NONE", use_dictionary=True, dictionary_pagesize_limit=64 * 1024, data_page_size=16 * 1024)
    scan = ParquetScanExec(path)
    encs = [p[0] for p in page_tuples(scan.row_group_chunks(0)[0])]
    assert DO.ENC_RLE_DICTIONARY in encs and DO.ENC_PLAIN in encs
    got, _ = oracle_column(scan, "s")
    assert [v.decode() for v in got[0]] == vals


# ---- DELTA_BINARY_PACKED: the data shapes of ParquetDeltaEncodingSuite.scala:81-159 (block 128, 4 miniblocks) ----------------

def delta_shapes(lo, hi, seed=0):
    rng = np.random.default_rng(seed)
    block, mini = 128, 32

    def rnd(k):
        return [int(x) for x in rng.integers(lo, hi, k, endpoint=True)]

    return {
        "aligned_to_block": rnd(5 * block),
        "partial_block": rnd(block - 3),
        "partial_miniblock": rnd(mini - 3),
        "negative_deltas": [10 - (i * 32 - int(rng.integers(0, 6))) for i in range(block)],
        "equal_deltas": [i * 32 for i in range(block)] + [0] * block,
        "equal_values": [3] * block + [0] * block,
        "zero_delta_per_block": [(i - 1) // block for i in range(5 * block + 1)],
        "unaligned": [int(x) - 10 for x in rng.integers(0, 20, 5 * block + 3)],
        "min_max": [lo if i % 2 == 0 else hi for i in range(10)],
        "one_two_min_three": [1, 2, lo, 3],
    }


DELTA_CASES = [(t, s) for t in ("int32", "int64", "date32") for s in delta_shapes(0, 1)]


def write_delta_ints(path, values, typ, version="1.0", nullable=False, data_page_size=1024 * 1024):
    at = {"int32": pa.int32(), "int64": pa.int64(), "date32": pa.date32()}[typ]
    arr = pa.array(values, pa.int32() if typ == "date32" else at)
    if typ == "date32":
        arr = arr.cast(pa.date32())
    if nullable:
        mask = np.arange(len(values)) % 7 == 3
        arr = pa.array([None if m else v for v, m in zip(arr.to_pylist(), mask)], at)
    pq.write_table(pa.table({"x": arr}), path, compression="NONE", use_dictionary=False, column_encoding={"x": "DELTA_BINARY_PACKED"},
                   data_page_version=version, data_page_size=data_page_size)
    return arr


def delta_values(typ, shape):
    lo, hi = (INT64_MIN, INT64_MAX) if typ == "int64" else (INT32_MIN, INT32_MAX)
    if typ == "date32":
        lo, hi = -719162, 2932896         # 0001-01-01 .. 9999-12-31
    v = delta_shapes(lo, hi, seed=len(shape))[shape]
    if typ == "date32" and shape == "one_two_min_three":
        v = [1, 2, lo, 3]
    return v


@pytest.mark.parametrize("typ,shape", DELTA_CASES, ids=["%s-%s" % c for c in DELTA_CASES])
def test_delta_binary_packed_walker_and_oracle(tmp_path, typ, shape):
    from spark_b200.scan import ParquetScanExec
    path = str(tmp_path / "d.parquet")
    arr = write_delta_ints(path, delta_values(typ, shape), typ, nullable=shape == "unaligned")
    scan = ParquetScanExec(path)
    ch = scan.row_group_chunks(0)[0]
    assert {p[0] for p in page_tuples(ch)} == {DO.ENC_DELTA_BINARY_PACKED}
    vals, valid = DO.decode_column_chunk(ch.data, page_tuples(ch), ch.dict_offset, ch.dict_count, ch.physical)
    want = pq.read_table(path).column("x").combine_chunks()
    if pa.types.is_date32(want.type):
        want = want.cast(pa.int32())
    ok = np.asarray(want.is_valid())
    assert np.array_equal(valid if valid is not None else np.ones(len(vals), bool), ok)
    assert vals[ok].tolist() == [v for v in want.to_pylist() if v is not None]


def test_int32_min_round_trips_through_wrapping_deltas():
    """1, 2, INT32_MIN, 3 (ParquetDeltaEncodingSuite.scala:298-313): the deltas wrap; the INT32 value is the low 32 bits."""
    import io
    buf = io.BytesIO()
    pq.write_table(pa.table({"x": pa.array([1, 2, INT32_MIN, 3], pa.int32())}), buf, compression="NONE", use_dictionary=False,
                   column_encoding={"x": "DELTA_BINARY_PACKED"})
    md = pq.ParquetFile(io.BytesIO(buf.getvalue())).metadata.row_group(0).column(0)
    data = np.frombuffer(buf.getvalue(), np.uint8)[md.data_page_offset:md.data_page_offset + md.total_compressed_size]
    from spark_b200.scan import EncodedColumnChunk
    ch = EncodedColumnChunk.from_file_bytes(data.copy(), 4, 0, 1, 1)
    vals, _ = DO.decode_column_chunk(ch.data, page_tuples(ch), ch.dict_offset, ch.dict_count, ch.physical)
    assert vals.tolist() == [1, 2, INT32_MIN, 3]


# ---- hand-written pages: the Thrift compact PageHeader of one data page (fields of read_page_header in csrc/scan.cu) -------

def _zz(v):
    return _uvarint((v << 1) ^ (v >> 63))


def _uvarint(v):
    v &= (1 << 64) - 1
    out = bytearray()
    while True:
        b = v & 0x7F
        v >>= 7
        if v:
            out.append(b | 0x80)
        else:
            out.append(b)
            return bytes(out)


def data_page(body: bytes, num_values: int, encoding: int) -> bytes:
    """PageHeader{1: type DATA_PAGE, 2/3: sizes, 5: DataPageHeader{1: num_values, 2: encoding, 3/4: RLE levels}} + body"""
    n = len(body)
    inner = b"\x15" + _zz(num_values) + b"\x15" + _zz(encoding) + b"\x15" + _zz(3) + b"\x15" + _zz(3) + b"\x00"
    return b"\x15" + _zz(0) + b"\x15" + _zz(n) + b"\x15" + _zz(n) + b"\x2c" + inner + b"\x00" + body


def walk(chunk: bytes, max_def=0):
    from spark_b200 import _capi as capi
    lib = capi.load()
    buf = np.frombuffer(chunk, np.uint8).copy()
    pages = (capi.sb_page * 8)()
    n, doff, dc = C.c_int32(), C.c_int64(), C.c_int32()
    rc = lib.sb_parquet_chunk_pages(buf.ctypes.data, buf.nbytes, max_def, pages, 8, C.byref(n), C.byref(doff), C.byref(dc))
    return rc, lib.sb_last_error().decode() if rc else "", [pages[i] for i in range(n.value)]


def delta_header(block, minis, total, first=0):
    return _uvarint(block) + _uvarint(minis) + _uvarint(total) + _zz(first)


@pytest.mark.parametrize("block,minis,total,what", [(1 << 30, 1, 1, "block size"), (128, 256, 1, "miniblock count"),
                                                    (128, 4, (1 << 32) - 1, "total count")],
                         ids=["block-2^30", "minis-above-block", "total-negative"])
def test_crafted_delta_headers_are_invalid(block, minis, total, what):
    """ParquetDeltaEncodingSuite.scala:175-207: the three headers the reference reader rejects before allocating anything
    (the negative total is -1 written as an unsigned 32-bit varint)."""
    from spark_b200 import _capi as capi
    rc, msg, _ = walk(data_page(delta_header(block, minis, total) + b"\x00" * 8, 100, 5))
    assert rc == 2 and what in msg and "page 0" in msg, (rc, msg)      # SB_ERR_INVALID
    ok, _, pages = walk(data_page(delta_header(128, 4, 1) + b"\x00" * 8, 100, 5))
    assert ok == capi.SB_OK and pages[0].encoding == capi.SB_ENC_DELTA_BINARY_PACKED


def test_miniblock_size_must_be_a_multiple_of_8():
    rc, msg, _ = walk(data_page(delta_header(128, 32, 1), 10, 5))
    assert rc == 2 and "multiple of 8" in msg


def test_delta_byte_array_page_continuing_the_previous_value_is_unsupported():
    """PARQUET-246: a first prefix length other than 0 would take bytes of the previous page's last value."""
    from spark_b200 import _capi as capi
    suffixes = delta_header(128, 4, 1, 3) + b"abc"
    rc, msg, _ = walk(data_page(delta_header(128, 4, 1, 2) + suffixes, 1, 7))
    assert rc == 5 and "PARQUET-246" in msg, (rc, msg)
    rc, _, pages = walk(data_page(delta_header(128, 4, 1, 0) + suffixes, 1, 7))
    assert rc == capi.SB_OK and pages[0].encoding == capi.SB_ENC_DELTA_BYTE_ARRAY
    assert DO.decode_delta_byte_array(np.frombuffer(delta_header(128, 4, 1, 0) + suffixes, np.uint8)) == [b"abc"]


def test_other_encodings_and_types_stay_refused(tmp_path):
    from spark_b200 import _capi as capi
    from spark_b200.scan import ParquetScanExec
    rc, msg, _ = walk(data_page(b"\x00" * 16, 4, 9))                 # BYTE_STREAM_SPLIT
    assert rc == 5 and "encoding 9" in msg
    path = str(tmp_path / "bss.parquet")
    pq.write_table(pa.table({"f": pa.array(np.arange(100, dtype=np.float32))}), path, compression="NONE", use_dictionary=False,
                   column_encoding={"f": "BYTE_STREAM_SPLIT"})
    with pytest.raises(capi.SparkB200Error) as e:
        ParquetScanExec(path).row_group_chunks(0)
    assert e.value.code == 5
    path = str(tmp_path / "flba.parquet")
    pq.write_table(pa.table({"d": pa.array([1, 2], pa.decimal128(30, 2)), "b": pa.array([b"ab", b"cd"], pa.binary(2))}), path,
                   compression="NONE")
    for col in ("d", "b"):
        with pytest.raises(capi.SparkB200Error) as e:
            ParquetScanExec(path, columns=[col]).row_group_chunks(0)
        assert e.value.code == 5
    path = str(tmp_path / "int96.parquet")
    pq.write_table(pa.table({"t": pa.array([1, 2], pa.timestamp("ns"))}), path, compression="NONE", use_deprecated_int96_timestamps=True)
    with pytest.raises(capi.SparkB200Error) as e:
        ParquetScanExec(path).row_group_chunks(0)
    assert e.value.code == 5
    path = str(tmp_path / "snappy.parquet")
    pq.write_table(pa.table({"s": pa.array(["x"] * 100)}), path, compression="SNAPPY")
    with pytest.raises(capi.SparkB200Error):
        ParquetScanExec(path).row_group_chunks(0)


def test_parquet_mr_string_fixture():
    """tests/golden/timestamp-nanos.parquet: parquet-mr 1.12.3, optional PLAIN BYTE_ARRAY `name`."""
    import hashlib
    from spark_b200.scan import ParquetScanExec
    with open(GOLDEN, "rb") as f:
        assert hashlib.sha256(f.read()).hexdigest() == GOLDEN_SHA256       # the reference's file, unchanged
    scan = ParquetScanExec(GOLDEN, columns=["id", "name"])
    ids, _ = oracle_column(scan, "id")
    names, _ = oracle_column(scan, "name")
    assert ids[0].tolist() == [1, 2, 3]
    assert names[0] == [b"Alice", b"Bob", b"Cecilia"]
    ch = scan.row_group_chunks(0)[1]
    assert ch.physical == 6 and ch.npages == 1 and page_tuples(ch)[0][0] == DO.ENC_PLAIN and page_tuples(ch)[0][5] > 0
