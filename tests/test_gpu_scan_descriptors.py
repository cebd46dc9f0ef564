"""sb_scan_decode and sb_scan_decode_compressed take page descriptors from their caller (the JNI scanDecode builds them from Java
arrays): malformed ones are refused with SB_ERR_INVALID before any kernel is launched, and the stream decodes the next call."""
import ctypes as C

import numpy as np
import pytest

from test_scan_pages_cpu import v1_page

pytestmark = pytest.mark.gpu

VALUES = np.arange(-10, 30, dtype=np.int32)     # 40 rows of PLAIN INT32


def int32_chunk(pages, values=VALUES):
    """one INT32 column over the bytes of `values`; pages: (num_values, values_offset, values_bytes, def_offset, def_bytes)"""
    from spark_b200 import _capi as capi
    from spark_b200.scan import EncodedColumnChunk
    arr = (capi.sb_page * len(pages))()
    for i, (n, voff, vbytes, doff, dbytes) in enumerate(pages):
        arr[i].encoding, arr[i].num_values = capi.SB_ENC_PLAIN, n
        arr[i].values_offset, arr[i].values_bytes, arr[i].def_offset, arr[i].def_bytes = voff, vbytes, doff, dbytes
    return EncodedColumnChunk(capi.SB_INT32, 0, capi.SB_PHYS["INT32"], values.view(np.uint8).copy(), arr, len(pages), -1, 0)


def string_chunk(num_values):
    """one PLAIN BYTE_ARRAY page holding "ab" once"""
    from spark_b200 import _capi as capi
    from spark_b200.scan import EncodedColumnChunk
    data = np.frombuffer(b"\x02\x00\x00\x00ab", np.uint8).copy()
    arr = (capi.sb_page * 1)()
    arr[0].encoding, arr[0].num_values, arr[0].values_offset, arr[0].values_bytes = capi.SB_ENC_PLAIN, num_values, 0, 6
    return EncodedColumnChunk(capi.SB_STRING, 0, capi.SB_PHYS["BYTE_ARRAY"], data, arr, 1, -1, 0)


VALID = [(20, 0, 80, 0, 0), (20, 80, 80, 0, 0)]
REFUSED = {
    # pages of 60 and -20 rows: the column would hold 40 rows and the first page write 60
    "negative-num-values": ([int32_chunk([(60, 0, 160, 0, 0), (-20, 0, 0, 0, 0)])], "negative value count"),
    "negative-def-offset": ([int32_chunk([(40, 0, 160, -8, 4)])], "offsets outside the chunk"),
    "negative-values-bytes": ([int32_chunk([(40, 16, -16, 0, 0)])], "offsets outside the chunk"),
    "negative-def-bytes": ([int32_chunk([(40, 0, 160, 0, -4)])], "offsets outside the chunk"),
    # the second column's pages hold more rows than the first column
    "pages-overrun-the-column": ([int32_chunk(VALID), int32_chunk(VALID + [(20, 0, 80, 0, 0)])], "has 60 rows, chunk 0 has 40"),
    "string-negative-num-values": ([string_chunk(-1)], "negative value count"),
}


@pytest.mark.parametrize("name", sorted(REFUSED))
def test_malformed_descriptors_are_refused_before_any_launch(gpu, stream, name):
    from spark_b200 import _capi as capi
    from spark_b200.scan import decode_chunks
    chunks, what = REFUSED[name]
    launches = capi.kernel_launch_count()
    with pytest.raises(capi.SparkB200Error) as e:
        decode_chunks(["c%d" % i for i in range(len(chunks))], chunks, stream)
    assert e.value.code == 2 and what in str(e.value), str(e.value)
    assert capi.kernel_launch_count() == launches
    b = decode_chunks(["x"], [int32_chunk(VALID)], stream)      # the same stream decodes the next call
    assert b.to_arrow(stream).column("x").to_pylist() == VALUES.tolist()
    b.close()


def test_negative_span_value_count_is_refused_before_any_launch(gpu, stream):
    from spark_b200 import _capi as capi
    from spark_b200.scan import CompressedColumnChunk, decode_file_chunks
    body = VALUES.tobytes()
    buf = np.frombuffer(v1_page(body, len(VALUES)), np.uint8).copy()
    ch = CompressedColumnChunk.from_file_bytes(buf, capi.SB_INT32, 0, capi.SB_PHYS["INT32"], capi.SB_CODEC["UNCOMPRESSED"], 0)
    assert ch.npages == 1
    b = decode_file_chunks(["x"], [ch], stream)
    assert b.to_arrow(stream).column("x").to_pylist() == VALUES.tolist()
    b.close()
    ch.spans[0].num_values = -1
    launches = capi.kernel_launch_count()
    with pytest.raises(capi.SparkB200Error) as e:
        decode_file_chunks(["x"], [ch], stream)
    assert e.value.code == 2 and "negative value count" in str(e.value), str(e.value)
    assert capi.kernel_launch_count() == launches
