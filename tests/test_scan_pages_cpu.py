"""CPU tests of the page header walk shared by sb_parquet_chunk_pages and sb_parquet_page_spans (host only): malformed headers are
refused the same way by both, and on every uncompressed file the other scan tests write, the descriptors sb_parquet_chunk_pages
returns are the ones the spans of sb_parquet_page_spans describe."""
import os
import subprocess
import sys

import numpy as np
import pytest

from test_scan_cpu import CASES, write_case
from test_scan_snappy_cpu import spans
from test_scan_strings_cpu import (DELTA_CASES, GOLDEN, STRING_CASES, _zz, case_id, delta_values, page_tuples, string_values, walk,
                                   write_delta_ints, write_strings)
from test_scan_types_cpu import (ENCODINGS, VERSIONS, write_dict_widths, write_geometry, write_hybrid, write_matrix, write_nulls,
                                 write_stripes)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---- hand-written pages: the Thrift compact PageHeader fields read_page_header in csrc/scan.cu reads -------------------------

def header(page_type, uncompressed, compressed, field=None, inner=b""):
    """PageHeader{1: type, 2: uncompressed_page_size, 3: compressed_page_size, field: the inner header struct's fields}"""
    out = b"\x15" + _zz(page_type) + b"\x15" + _zz(uncompressed) + b"\x15" + _zz(compressed)
    if field is not None:
        out += bytes([(field - 3) << 4 | 12]) + inner + b"\x00"
    return out + b"\x00"


def i32_fields(*values):
    """fields 1, 2, ... of a struct, each an i32"""
    return b"".join(b"\x15" + _zz(v) for v in values)


def v1_page(body, num_values, encoding=0):
    """DataPageHeader{num_values, encoding, RLE definition and repetition levels}"""
    return header(0, len(body), len(body), 5, i32_fields(num_values, encoding, 3, 3)) + body


def v2_page(body, num_values, def_len=0, is_compressed=True, uncompressed=None):
    """DataPageHeaderV2{num_values, num_nulls 0, num_rows, PLAIN, def_len, rep_len 0, is_compressed}"""
    inner = i32_fields(num_values, 0, num_values, 0, def_len, 0) + (b"\x11" if is_compressed else b"\x12")
    return header(3, len(body) if uncompressed is None else uncompressed, len(body), 8, inner) + body


def dictionary_page(body, num_values):
    """DictionaryPageHeader{num_values, PLAIN}"""
    return header(2, len(body), len(body), 7, i32_fields(num_values, 0)) + body


CHILD = """
import ctypes as C, sys
import numpy as np
sys.path.insert(0, sys.argv[1])
from spark_b200 import _capi as capi
lib = capi.load()
buf = np.frombuffer(bytes.fromhex(sys.argv[2]), np.uint8).copy()
n = C.c_int32()
if sys.argv[3] == "pages":
    out, doff, dc = (capi.sb_page * 8)(), C.c_int64(), C.c_int32()
    rc = lib.sb_parquet_chunk_pages(buf.ctypes.data, buf.nbytes, 0, out, 8, C.byref(n), C.byref(doff), C.byref(dc))
else:
    out = (capi.sb_page_span * 8)()
    rc = lib.sb_parquet_page_spans(buf.ctypes.data, buf.nbytes, 0, 0, out, 8, C.byref(n))
print(rc, lib.sb_last_error().decode() if rc else "")
"""


@pytest.mark.parametrize("walker", ["pages", "spans"])
@pytest.mark.parametrize("size", [-7, -1000])
def test_negative_page_size_is_refused(walker, size):
    """An INDEX_PAGE header whose two sizes are negative: the body would start before the header (-7 steps back onto it, a
    larger size reads before the chunk).  The walk runs in a child process, so a walker that loops ends in the timeout."""
    chunk = header(1, size, size)
    if size == -7:
        assert chunk == bytes.fromhex("1502150d150d00")
    flags = ["-s"] if sys.flags.no_user_site else []
    r = subprocess.run([sys.executable] + flags + ["-c", CHILD, ROOT, chunk.hex(), walker], capture_output=True, text=True, timeout=60)
    assert r.returncode == 0, r.stderr
    rc, msg = r.stdout.strip().split(" ", 1)
    assert rc == "2" and "overruns the column chunk" in msg, r.stdout       # SB_ERR_INVALID


NEGATIVE_COUNTS = {
    "v1": v1_page(np.arange(20, dtype=np.int32).tobytes(), 20) + v1_page(b"", -10),
    "v2": v2_page(b"", -10),
    "dictionary": dictionary_page(b"", -3) + v1_page(b"\x01", 4, encoding=8),
}


@pytest.mark.parametrize("name", sorted(NEGATIVE_COUNTS))
def test_negative_value_count_is_refused_by_both_walkers(name):
    """a negative num_values would let the pages of a column hold fewer rows than one of them writes"""
    chunk = NEGATIVE_COUNTS[name]
    for rc, msg, _ in (walk(chunk), spans(chunk, codec=0)):
        assert rc == 2 and "negative value count" in msg, (rc, msg)


def test_uncompressed_v2_page_must_store_its_uncompressed_size():
    """a V2 page marked is_compressed = false stores its values as they are: both sizes must agree on every path"""
    body = np.arange(2, dtype=np.int32).tobytes()
    stored = v2_page(body, 2, is_compressed=False, uncompressed=12)
    for rc, msg, _ in (walk(stored), spans(stored, codec=1), spans(stored, codec=0)):
        assert rc == 2 and "8 stored bytes for 12" in msg, (rc, msg)
    rc, _, pages = walk(v2_page(body, 2, is_compressed=False))
    assert rc == 0 and [(p.num_values, p.values_bytes) for p in pages] == [(2, 8)]
    for page in (v2_page(body, 2, is_compressed=False), v1_page(body, 2), dictionary_page(body, 2)):     # the pages end where their bytes do
        rc, _, sp = spans(page, codec=0)
        assert rc == 0 and [s.header_bytes + s.compressed_bytes for s in sp] == [len(page)]
    rc, msg, _ = walk(v2_page(body, 2, is_compressed=True, uncompressed=12))  # a compressed page: not decoded on this path
    assert rc == 5 and "compressed Parquet pages are not decoded" in msg, (rc, msg)


def test_negative_v2_level_length_is_refused_by_both_walkers():
    chunk = v2_page(np.arange(4, dtype=np.int32).tobytes(), 4, def_len=-4)
    for rc, msg, _ in (walk(chunk, max_def=1), spans(chunk, codec=0, max_def=1)):
        assert rc == 2 and "levels overrun the page" in msg, (rc, msg)


# ---- both walkers over real files ----------------------------------------------------------------------------------------------

def pages_from_spans(data, spans_, max_def_level):
    """the descriptors the spans of an uncompressed chunk describe: a V1 page of an optional column starts with the 4-byte
    length of its definition levels, a V2 page's level bytes are counted by its span"""
    pages, dict_offset, dict_count = [], -1, 0
    for s in spans_:
        assert s.values_compressed == 0 and s.compressed_bytes == s.uncompressed_bytes
        body, end = s.body_offset, s.body_offset + s.uncompressed_bytes
        if s.page_type == 2:
            dict_offset, dict_count = body, s.num_values
            continue
        def_offset = def_bytes = 0
        if s.page_type == 0 and max_def_level > 0:
            def_offset, def_bytes = body + 4, int.from_bytes(data[body:body + 4].tobytes(), "little")
            values = def_offset + def_bytes
        else:
            if s.levels_bytes > 0:
                def_offset, def_bytes = body, s.levels_bytes
            values = body + s.levels_bytes
        pages.append((s.encoding, s.num_values, values, end - values, def_offset, def_bytes))
    return pages, dict_offset, dict_count


def assert_walkers_agree(path, columns=None):
    from spark_b200.scan import ParquetScanExec
    scan = ParquetScanExec(path, columns=columns)
    npages = 0
    for rg in range(scan.meta.num_row_groups):
        for ch, fc in zip(scan.row_group_chunks(rg), scan.row_group_file_chunks(rg)):
            assert fc.codec == 0 and np.array_equal(ch.data, fc.data)
            got = (page_tuples(ch), ch.dict_offset, ch.dict_count)
            assert got == pages_from_spans(fc.data, [fc.spans[i] for i in range(fc.npages)], fc.max_def_level)
            npages += ch.npages
    assert npages > 0


@pytest.mark.parametrize("case", CASES, ids=lambda c: "v%s-n%d-%s" % (c["version"], c["n"], c["use_dictionary"]))
def test_walkers_agree_on_mixed_type_files(tmp_path, case):
    assert_walkers_agree(write_case(str(tmp_path), case)[1])


@pytest.mark.parametrize("case", STRING_CASES, ids=case_id)
def test_walkers_agree_on_string_files(tmp_path, case):
    path = str(tmp_path / "s.parquet")
    write_strings(path, string_values(6000, seed=len(case_id(case)), nullable=case["nullable"]), case["enc"], case["version"],
                  row_group_size=-(-6000 // case["rgs"]))
    assert_walkers_agree(path)


@pytest.mark.parametrize("typ,shape", DELTA_CASES, ids=["%s-%s" % c for c in DELTA_CASES])
def test_walkers_agree_on_delta_files(tmp_path, typ, shape):
    path = str(tmp_path / "d.parquet")
    write_delta_ints(path, delta_values(typ, shape), typ, nullable=shape == "unaligned")
    assert_walkers_agree(path)


@pytest.mark.parametrize("version", VERSIONS)
@pytest.mark.parametrize("encoding", ENCODINGS)
def test_walkers_agree_on_type_matrix_files(tmp_path, encoding, version):
    assert_walkers_agree(write_matrix(str(tmp_path), encoding, version)[1])


def test_walkers_agree_on_page_layout_files(tmp_path):
    d = str(tmp_path)
    paths = [write_dict_widths(d)[1], write_hybrid(d, "1.0")[1], write_hybrid(d, "2.0")[1], write_geometry(d)[1], write_nulls(d)]
    for path in paths + list(write_stripes(d)[1].values()):
        assert_walkers_agree(path)


def test_walkers_agree_on_the_parquet_mr_golden():
    assert_walkers_agree(GOLDEN, columns=["id", "name"])
