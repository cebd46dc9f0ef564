"""CPU tests of the compressed side of the scan boundary: the span walker (sb_parquet_page_spans, host only) against pyarrow's
footer and libsnappy (pa.Codec), the refusals of codecs other than SNAPPY, and the test Snappy writer (tests/snappy_streams.py)
against libsnappy."""
import ctypes as C
import hashlib
import os

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq
import pytest

import snappy_streams as SS
from test_scan_cpu import _table
from test_scan_strings_cpu import _zz, string_values

GOLDEN_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
# The reference's sql/core/src/test/resources/test-data/ files, byte for byte (ParquetThriftCompatibilitySuite, ParquetIOSuite)
GOLDENS = {
    "parquet-thrift-compat.snappy.parquet": "2ed64edd7afdb1042700ce21a82b8c9f3a73b662f819f1bbdcc030fc7b58541e",
    "decimal32-written-as-64-bit.snappy.parquet": "2ee38fafbdf6b038ced1973b523fb375084e3407648d0b9d94d0e4f1a13faa98",
    "decimal32-written-as-64-bit-dict.snappy.parquet": "af33490a3f798039531094ceec35895b308b264005b18aa2ca3866322953eddf",
}
# ParquetThriftCompatibilitySuite.scala:35-71: the flat columns of row i
SUITS = ["SPADES", "HEARTS", "DIAMONDS", "CLUBS"]
THRIFT_FLAT = ["boolColumn", "byteColumn", "shortColumn", "intColumn", "longColumn", "doubleColumn", "binaryColumn", "stringColumn",
               "enumColumn", "maybeBoolColumn", "maybeByteColumn", "maybeShortColumn", "maybeIntColumn", "maybeLongColumn",
               "maybeDoubleColumn", "maybeBinaryColumn", "maybeStringColumn", "maybeEnumColumn"]


def golden(name):
    path = os.path.join(GOLDEN_DIR, name)
    with open(path, "rb") as f:
        assert hashlib.sha256(f.read()).hexdigest() == GOLDENS[name]
    return path


def thrift_compat_rows(n=10):
    def row(i):
        flat = [i % 2 == 0, i, i + 1, i + 2, i * 10, i + 0.2, "val_%d" % i, "val_%d" % i, SUITS[i % 4].encode()]
        return flat + [None if i % 3 == 0 else v for v in flat]
    return {name: [row(i)[k] for i in range(n)] for k, name in enumerate(THRIFT_FLAT)}


DECIMAL32 = [792059492, 986842987, 540247998, None, 357991078, 494131059, 92536396, 426847157, -999999999, 204486094]
DECIMAL32_DICT_FIRST = [751, 937, 511, None, 337, 467, 84, 403, -999, 190]
DECIMAL32_DICT_LAST = [866, 20, 492, 76, 824, 604, 343, 820, 864, 243]


def write_snappy(tmp_path, table, name="t.parquet", **kw):
    path = str(tmp_path / name)
    kw.setdefault("compression", "SNAPPY")
    pq.write_table(table, path, **kw)
    return path


def spans_of(chunk):
    return [chunk.spans[i] for i in range(chunk.npages)]


def check_spans_against_footer(path, columns=None):
    from spark_b200.scan import ParquetScanExec
    scan = ParquetScanExec(path, columns=columns)
    snappy = pa.Codec("snappy")
    for rg in range(scan.meta.num_row_groups):
        g = scan.meta.row_group(rg)
        metas = {g.column(i).path_in_schema: g.column(i) for i in range(g.num_columns)}
        for f, ch in zip(scan.fields, scan.row_group_file_chunks(rg)):
            cm = metas[f.name]
            spans = spans_of(ch)
            assert sum(s.header_bytes + s.compressed_bytes for s in spans) == cm.total_compressed_size == ch.nbytes
            assert sum(s.num_values for s in spans if s.page_type != 2) == cm.num_values
            if cm.has_dictionary_page:                  # old parquet-mr writers leave dictionary_page_offset unset
                assert any(s.page_type == 2 for s in spans)
            for s in spans:
                body = ch.data[s.body_offset:s.body_offset + s.compressed_bytes].tobytes()
                if s.values_compressed:
                    values = snappy.decompress(body[s.levels_bytes:], decompressed_size=s.uncompressed_bytes - s.levels_bytes).to_pybytes()
                    assert len(values) == s.uncompressed_bytes - s.levels_bytes
                else:
                    assert s.compressed_bytes == s.uncompressed_bytes
    return scan


SPAN_CASES = [dict(version=v, dictionary=d, nullable=nl) for v in ("1.0", "2.0") for d in ("dict", "plain", "delta") for nl in (False, True)]


@pytest.mark.parametrize("case", SPAN_CASES, ids=lambda c: "v%s-%s-%s" % (c["version"], c["dictionary"], "opt" if c["nullable"] else "req"))
def test_span_walker_against_pyarrow_footer_and_libsnappy(tmp_path, case):
    n = 30_000
    rng = np.random.default_rng(len(str(case)))
    mask = (rng.random(n) < 0.2) if case["nullable"] else None
    t = pa.table({"i64": pa.array(np.cumsum(rng.integers(-5, 50, n)), mask=mask), "i32": pa.array(rng.integers(0, 40, n).astype(np.int32), mask=mask),
                  "s": pa.array(string_values(n, seed=1, nullable=case["nullable"])), "d": pa.array(rng.standard_normal(n), mask=mask)})
    kw = dict(data_page_version=case["version"], data_page_size=16 * 1024)
    if case["dictionary"] == "dict":
        kw["use_dictionary"] = True
    elif case["dictionary"] == "plain":
        kw["use_dictionary"] = False
    else:
        kw.update(use_dictionary=False, column_encoding={"i64": "DELTA_BINARY_PACKED", "i32": "DELTA_BINARY_PACKED", "s": "DELTA_BYTE_ARRAY",
                                                         "d": "PLAIN"})
    scan = check_spans_against_footer(write_snappy(tmp_path, t, **kw))
    chunks = scan.row_group_file_chunks(0)
    assert all(ch.codec == 1 for ch in chunks) and max(ch.npages for ch in chunks) > 1
    if case["version"] == "2.0" and case["nullable"]:
        assert any(s.levels_bytes > 0 for ch in chunks for s in spans_of(ch))


@pytest.mark.parametrize("name", sorted(GOLDENS))
def test_span_walker_on_reference_goldens(name):
    path = golden(name)
    columns = THRIFT_FLAT if name.startswith("parquet-thrift") else None
    scan = check_spans_against_footer(path, columns)
    if name.startswith("parquet-thrift"):   # tiny pages grow under Snappy: sizes alone cannot tell a compressed page
        assert any(s.compressed_bytes >= s.uncompressed_bytes for ch in scan.row_group_file_chunks(0) for s in spans_of(ch))


@pytest.mark.parametrize("codec", ["GZIP", "ZSTD", "LZ4", "BROTLI"])
def test_other_codecs_are_refused_before_any_device_call(tmp_path, codec):
    from spark_b200 import _capi as capi
    from spark_b200.scan import ParquetScanExec
    path = write_snappy(tmp_path, _table(2000), compression=codec)
    with pytest.raises(capi.SparkB200Error) as e:
        ParquetScanExec(path).collect()                 # no capi.init: a device call would fail differently
    assert e.value.code == 5 and codec in str(e.value).upper()


def test_nested_column_is_refused_by_name(tmp_path):
    from spark_b200 import _capi as capi
    from spark_b200.scan import ParquetScanExec
    with pytest.raises(capi.SparkB200Error) as e:
        ParquetScanExec(golden("parquet-thrift-compat.snappy.parquet"), columns=["intColumn", "stringsColumn"]).collect()
    assert e.value.code == 5 and "stringsColumn" in str(e.value)


def _page(body, uncompressed, num_values=1):
    inner = b"\x15" + _zz(num_values) + b"\x15" + _zz(0) + b"\x15" + _zz(3) + b"\x15" + _zz(3) + b"\x00"
    return b"\x15" + _zz(0) + b"\x15" + _zz(uncompressed) + b"\x15" + _zz(len(body)) + b"\x2c" + inner + b"\x00" + body


def spans(chunk: bytes, codec=1, max_def=0):
    from spark_b200 import _capi as capi
    lib = capi.load()
    buf = np.frombuffer(chunk, np.uint8).copy()
    out = (capi.sb_page_span * 8)()
    n = C.c_int32()
    rc = lib.sb_parquet_page_spans(buf.ctypes.data, buf.nbytes, codec, max_def, out, 8, C.byref(n))
    return rc, lib.sb_last_error().decode() if rc else "", [out[i] for i in range(n.value)]


def test_unknown_codec_and_overrunning_body_are_refused():
    body = SS.Writer().literal(b"abcd").stream()
    rc, msg, sp = spans(_page(body, 4))
    assert rc == 0 and len(sp) == 1 and sp[0].values_compressed == 1 and sp[0].uncompressed_bytes == 4
    assert sp[0].header_bytes + sp[0].compressed_bytes == len(_page(body, 4))
    rc, msg, _ = spans(_page(body, 4), codec=9)
    assert rc == 5 and "codec 9" in msg
    rc, msg, _ = spans(_page(body, 4), codec=6)
    assert rc == 5 and "ZSTD" in msg
    rc, msg, _ = spans(_page(body, 4)[:-1])                              # the body runs past the chunk
    assert rc == 2 and "overruns" in msg
    rc, msg, sp = spans(_page(b"\x00" * 4, 4), codec=0)                  # UNCOMPRESSED: stored as they are
    assert rc == 0 and sp[0].values_compressed == 0
    rc, msg, _ = spans(_page(b"\x00" * 4, 5), codec=0)
    assert rc == 2 and "stored bytes" in msg


def test_writer_streams_decompress_under_libsnappy():
    snappy = pa.Codec("snappy")
    streams = SS.valid_streams()
    assert len(streams) > 100
    for name, (stream, want) in streams.items():
        got = snappy.decompress(stream, decompressed_size=len(want)).to_pybytes() if want else b""
        assert got == want, name
    preambles = {len(stream) - len(SS.Writer().literal(b"pre").elements) for n, (stream, _) in streams.items() if n.startswith("preamble")}
    assert preambles == {1, 2, 3, 4, 5}


@pytest.mark.parametrize("name", sorted(SS.malformed_streams()))
def test_malformed_streams_have_the_verdict_of_the_rule(name):
    """accepted exactly when libsnappy accepts the stream and its preamble equals the declared size: every one of these fails"""
    stream, declared, status = SS.malformed_streams()[name]
    snappy = pa.Codec("snappy")
    preamble_ok = True
    try:
        v, shift, k = 0, 0, 0
        while True:
            b = stream[k]
            v |= (b & 0x7F) << shift
            k += 1
            shift += 7
            if b < 0x80:
                break
        preamble_ok = k <= 5 and v < 1 << 32 and v == declared
    except IndexError:
        preamble_ok = False
    libsnappy_ok = True
    try:
        snappy.decompress(stream, decompressed_size=max(declared, 1))
    except Exception:
        libsnappy_ok = False
    assert not (libsnappy_ok and preamble_ok), name
    assert (status == SS.LENGTH_MISMATCH) == (libsnappy_ok and not preamble_ok) or status == SS.LENGTH_MISMATCH
