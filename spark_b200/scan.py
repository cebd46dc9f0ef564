"""FileSourceScanExec mirror for Parquet: column chunks go to the GPU ENCODED and are decoded there (csrc/scan.cu).

Reference: FileSourceScanExec.doExecuteColumnar (sql/core/src/main/scala/org/apache/spark/sql/execution/DataSourceScanExec.scala:735-760)
hands out the ColumnarBatches of VectorizedParquetRecordReader (sql/core/src/main/java/.../parquet/VectorizedParquetRecordReader.java);
one batch here is one row group.  The footer (schema, column-chunk byte ranges, codecs) is read with pyarrow's metadata reader --
the role parquet-mr's ParquetFileReader plays for the reference; every data byte goes through sb_parquet_chunk_pages +
sb_scan_decode (uncompressed row groups) or sb_parquet_page_spans + sb_scan_decode_compressed (SNAPPY pages, decompressed on the
GPU).
"""
from __future__ import annotations

import ctypes as C
import mmap

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq

from . import _capi as capi
from .columnar import ColumnarBatch, _h
from .execution import SparkPlan

_PHYS = {"BOOLEAN": capi.SB_PHYS["BOOLEAN"], "INT32": capi.SB_PHYS["INT32"], "INT64": capi.SB_PHYS["INT64"],
         "FLOAT": capi.SB_PHYS["FLOAT"], "DOUBLE": capi.SB_PHYS["DOUBLE"], "BYTE_ARRAY": capi.SB_PHYS["BYTE_ARRAY"]}


def _is_bytes(arrow_type):
    return (pa.types.is_string(arrow_type) or pa.types.is_large_string(arrow_type) or pa.types.is_binary(arrow_type)
            or pa.types.is_large_binary(arrow_type))


# Parquet TIMESTAMP units -> the factor that makes microseconds (ParquetVectorUpdaterFactory: MILLIS through LongAsMicrosUpdater;
# NANOS is refused unless a legacy flag reads it as a plain long, which the GPU scan does not offer)
_TIMESTAMP_MULTIPLIER = {"microseconds": 1, "milliseconds": 1000}


def _sb_type(name, arrow_type, pcol):
    """(SB_* type, sb scale word, value multiplier) of a flat column: Arrow type `arrow_type`, Parquet column `pcol`
    (pyarrow's ColumnSchema).  What the GPU scan cannot read as Spark would is SparkB200Error(5) naming the column."""
    def refuse(why):
        return capi.SparkB200Error(5, "column %s (%s, Parquet %s %s): %s" % (name, arrow_type, pcol.physical_type, pcol.logical_type, why))
    if _is_bytes(arrow_type):      # BYTE_ARRAY -> int32 offsets + byte arena; a binary column comes back as binary
        return capi.SB_STRING, 0, 0
    if pcol.physical_type not in _PHYS:
        raise refuse("physical type %s is not supported by the GPU scan" % pcol.physical_type)
    if pa.types.is_decimal(arrow_type):
        if arrow_type.precision > 18:
            raise refuse("decimal precision %d > 18 is not supported by the GPU scan" % arrow_type.precision)
        return capi.SB_DECIMAL64, capi.decimal_type(arrow_type.precision, arrow_type.scale), 0
    if pa.types.is_timestamp(arrow_type):
        unit = pcol.logical_type.to_json()
        mul = next((m for u, m in _TIMESTAMP_MULTIPLIER.items() if '"timeUnit": "%s"' % u in unit), None)
        if pcol.physical_type != "INT64" or mul is None:
            raise refuse("only INT64 TIMESTAMP(MILLIS) and TIMESTAMP(MICROS) are read as timestamps")
        return capi.SB_TIMESTAMP, 0, mul
    if pa.types.is_unsigned_integer(arrow_type) or pa.types.is_time(arrow_type):
        raise refuse("the GPU scan has no Spark type for it")
    from .columnar import sb_type_of
    try:
        return sb_type_of(arrow_type), 0, 0
    except capi.SparkB200Error as e:
        raise refuse(str(e)) from None


class EncodedColumnChunk:
    """Host image of one column chunk + its page descriptors (keeps the buffers alive for the C struct)."""

    def __init__(self, sb_type, scale, physical, data: np.ndarray, pages, npages, dict_offset, dict_count, multiplier=0):
        self.type, self.scale, self.physical, self.multiplier = sb_type, scale, physical, multiplier
        self.data, self.pages, self.npages = data, pages, npages
        self.dict_offset, self.dict_count = dict_offset, dict_count

    @property
    def nbytes(self):
        return int(self.data.nbytes)

    def c(self) -> capi.sb_column_chunk:
        s = capi.sb_column_chunk()
        s.type, s.scale, s.physical_type, s.npages = self.type, self.scale, self.physical, self.npages
        s.data = self.data.ctypes.data
        s.data_bytes = self.data.nbytes
        s.pages = C.cast(self.pages, C.POINTER(capi.sb_page))
        s.dict_offset, s.dict_count = self.dict_offset, self.dict_count
        s.value_multiplier = self.multiplier
        return s

    @staticmethod
    def from_file_bytes(buf: np.ndarray, sb_type, scale, physical, max_def_level, pages_cap=None, multiplier=0) -> "EncodedColumnChunk":
        lib = capi.load()
        cap = pages_cap or max(16, buf.nbytes // 512 + 16)
        pages = (capi.sb_page * cap)()
        npages, doff, dcount = C.c_int32(), C.c_int64(), C.c_int32()
        capi.check(lib.sb_parquet_chunk_pages(buf.ctypes.data, buf.nbytes, max_def_level, pages, cap, C.byref(npages), C.byref(doff), C.byref(dcount)))
        return EncodedColumnChunk(sb_type, scale, physical, buf, pages, npages.value, doff.value, dcount.value, multiplier)


class CompressedColumnChunk:
    """Host bytes of one column chunk as it lies in the file + the spans of its pages (sb_parquet_page_spans)."""

    def __init__(self, sb_type, scale, physical, codec, max_def_level, data: np.ndarray, spans, npages, multiplier=0):
        self.type, self.scale, self.physical, self.codec, self.max_def_level = sb_type, scale, physical, codec, max_def_level
        self.multiplier = multiplier
        self.data, self.spans, self.npages = data, spans, npages

    @property
    def nbytes(self):
        return int(self.data.nbytes)

    def c(self) -> capi.sb_compressed_chunk:
        s = capi.sb_compressed_chunk()
        s.type, s.scale, s.physical_type, s.codec = self.type, self.scale, self.physical, self.codec
        s.max_def_level, s.npages, s.value_multiplier = self.max_def_level, self.npages, self.multiplier
        s.data = self.data.ctypes.data
        s.data_bytes = self.data.nbytes
        s.spans = C.cast(self.spans, C.POINTER(capi.sb_page_span))
        return s

    @staticmethod
    def from_file_bytes(buf: np.ndarray, sb_type, scale, physical, codec, max_def_level, cap=None, multiplier=0) -> "CompressedColumnChunk":
        lib = capi.load()
        cap = cap or max(16, buf.nbytes // 64 + 16)          # a page header alone takes more than 16 bytes
        spans = (capi.sb_page_span * cap)()
        n = C.c_int32()
        capi.check(lib.sb_parquet_page_spans(buf.ctypes.data, buf.nbytes, codec, max_def_level, spans, cap, C.byref(n)))
        return CompressedColumnChunk(sb_type, scale, physical, codec, max_def_level, buf, spans, n.value, multiplier)


def decode_chunks(names, chunks, stream=None, arrow_types=None) -> ColumnarBatch:
    lib = capi.load()
    arr = (capi.sb_column_chunk * len(chunks))()
    for i, ch in enumerate(chunks):
        arr[i] = ch.c()
    h = C.c_void_p()
    capi.check(lib.sb_scan_decode(arr, len(chunks), _h(stream), C.byref(h)))
    return ColumnarBatch(h, list(names), arrow_types)


def decode_file_chunks(names, chunks, stream=None, arrow_types=None) -> ColumnarBatch:
    """sb_scan_decode_compressed of CompressedColumnChunks (each chunk's codec is its own)"""
    lib = capi.load()
    arr = (capi.sb_compressed_chunk * len(chunks))()
    for i, ch in enumerate(chunks):
        arr[i] = ch.c()
    h = C.c_void_p()
    capi.check(lib.sb_scan_decode_compressed(arr, len(chunks), _h(stream), C.byref(h)))
    return ColumnarBatch(h, list(names), arrow_types)


class ParquetScanExec(SparkPlan):
    """Scan of a Parquet file: `batches()` yields one HBM-resident ColumnarBatch per row group; executeColumnar concatenates
    them (for plans that want the partition as one batch).  Pages may be uncompressed or SNAPPY-compressed (per column);
    other codecs and nested columns are refused with SparkB200Error(5), and so is, when the scan is created, a column the GPU
    scan cannot read as Spark does (INT96, FIXED_LEN_BYTE_ARRAY, TIMESTAMP(NANOS), unsigned integers, TIME, decimal precision
    above 18).  TIMESTAMP(MILLIS) comes back in microseconds, decimals keep their precision."""

    def __init__(self, path, columns=None):
        self.path = path
        self.file = pq.ParquetFile(path)
        self.meta = self.file.metadata
        schema = self.file.schema_arrow
        self.columns = list(columns) if columns is not None else list(schema.names)
        self.fields = [schema.field(c) for c in self.columns]
        pnames = self.file.schema.names
        self.types = [_sb_type(f.name, f.type, self.file.schema.column(pnames.index(f.name))) if f.name in pnames else None
                      for f in self.fields]         # (type, scale, multiplier) of every flat column; nested ones fail in _column_metas
        self._f = open(path, "rb")
        self._mm = mmap.mmap(self._f.fileno(), 0, access=mmap.ACCESS_READ)
        self._bytes = np.frombuffer(self._mm, dtype=np.uint8)

    def _column_metas(self, rg: int):
        """(field, column-chunk metadata) of every selected column of row group rg; nested columns are refused"""
        g = self.meta.row_group(rg)
        by_name = {g.column(i).path_in_schema: g.column(i) for i in range(g.num_columns)}
        out = []
        for f in self.fields:
            if f.name not in by_name:
                raise capi.SparkB200Error(5, "column %s is nested (%s); the GPU scan reads flat columns" % (f.name, f.type))
            cm = by_name[f.name]
            if cm.physical_type not in _PHYS:
                raise capi.SparkB200Error(5, "column %s: physical type %s is not supported by the GPU scan" % (f.name, cm.physical_type))
            if (cm.physical_type == "BYTE_ARRAY") != _is_bytes(f.type):
                raise capi.SparkB200Error(5, "column %s: physical type %s with Arrow type %s is not supported by the GPU scan" % (f.name, cm.physical_type, f.type))
            out.append((f, cm))
        return out

    def _chunk_bytes(self, f, cm):
        start = cm.dictionary_page_offset if cm.has_dictionary_page and cm.dictionary_page_offset else cm.data_page_offset
        start = min(start, cm.data_page_offset)
        t, scale, mul = self.types[self.columns.index(f.name)]
        max_def = self.file.schema.column(self.file.schema.names.index(f.name)).max_definition_level
        return self._bytes[start:start + cm.total_compressed_size], t, scale, mul, max_def

    def row_group_chunks(self, rg: int):
        """host page descriptors of the row group's chunks, which must be uncompressed"""
        out = []
        for f, cm in self._column_metas(rg):
            if cm.compression != "UNCOMPRESSED":
                raise capi.SparkB200Error(5, "column %s is %s-compressed; the GPU scan reads uncompressed pages" % (f.name, cm.compression))
            buf, t, scale, mul, max_def = self._chunk_bytes(f, cm)
            out.append(EncodedColumnChunk.from_file_bytes(buf, t, scale, _PHYS[cm.physical_type], max_def, multiplier=mul))
        return out

    def row_group_file_chunks(self, rg: int):
        """the row group's chunks as they lie in the file, with the spans of their pages (UNCOMPRESSED or SNAPPY)"""
        out = []
        for f, cm in self._column_metas(rg):
            codec = capi.SB_CODEC.get(cm.compression)
            if codec not in (capi.SB_CODEC["UNCOMPRESSED"], capi.SB_CODEC["SNAPPY"]):
                raise capi.SparkB200Error(5, "column %s is %s-compressed; the GPU scan reads UNCOMPRESSED and SNAPPY pages" % (f.name, cm.compression))
            buf, t, scale, mul, max_def = self._chunk_bytes(f, cm)
            out.append(CompressedColumnChunk.from_file_bytes(buf, t, scale, _PHYS[cm.physical_type], codec, max_def, multiplier=mul))
        return out

    def batches(self, stream=None):
        types = [f.type for f in self.fields]
        for rg in range(self.meta.num_row_groups):
            if all(cm.compression == "UNCOMPRESSED" for _, cm in self._column_metas(rg)):
                yield decode_chunks(self.columns, self.row_group_chunks(rg), stream, types)          # no synchronisation
            else:
                yield decode_file_chunks(self.columns, self.row_group_file_chunks(rg), stream, types)

    def executeColumnar(self, stream=None):
        bs = list(self.batches(stream))
        if len(bs) == 1:
            return bs[0]
        try:
            return ColumnarBatch.concat(bs, stream)
        finally:
            for b in bs:
                b.close()


def encode_column(batch: ColumnarBatch, name: str, dictionary: bool, page_rows: int = 1 << 20, stream=None, pinned=False) -> EncodedColumnChunk:
    """Write-side twin (tests, bench.py): encodes one NULL-free fixed-width column the way a Parquet writer would -- a sorted
    dictionary + pages of bit-packed indices (RLE_DICTIONARY), or PLAIN pages -- entirely on the GPU (distinct values through the
    hash aggregate, order through the radix sort, indices + bit packing in sb_scan_encode) and brings the chunk to the host.
    The dictionary of a float column is built on its bit patterns (the aggregate and the sort would fold -0.0 into 0.0 and every
    NaN into one), so decoding gives back every bit that was encoded."""
    from .execution import HashAggregateExec, LocalTableScanExec, SortExec
    from .columnar import PinnedArray
    lib = capi.load()
    col = batch.column_index(name)
    d = batch.column_desc(col)
    n = batch.num_rows
    dict_batch = None
    if dictionary:
        if d.type in (capi.SB_FLOAT32, capi.SB_FLOAT64):      # the same device buffer seen as integers of its width
            bits = capi.sb_column()
            bits.type = capi.SB_INT32 if d.type == capi.SB_FLOAT32 else capi.SB_INT64
            bits.length, bits.data = d.length, d.data
            h = C.c_void_p()
            capi.check(lib.sb_table_import_device(C.byref(bits), 1, C.byref(h)))
            one = ColumnarBatch(h, [name], [pa.int32() if d.type == capi.SB_FLOAT32 else pa.int64()])
        else:
            one = batch.select([name])
        try:
            dict_batch = SortExec([(name, True, True)], HashAggregateExec([name], [], LocalTableScanExec(one), mode="complete")).executeColumnar(stream)
        finally:
            one.close()
    cap = max(1, (n + page_rows - 1) // page_rows)
    pages = (capi.sb_page * cap)()
    npages, doff, dcount = C.c_int32(), C.c_int64(), C.c_int32()
    h = C.c_void_p()
    try:
        capi.check(lib.sb_scan_encode(batch.handle, col, dict_batch.handle if dict_batch else None, page_rows, _h(stream), C.byref(h), pages, cap,
                                      C.byref(npages), C.byref(doff), C.byref(dcount)))
    finally:
        if dict_batch:
            dict_batch.close()
    chunk = ColumnarBatch(h, ["bytes"], [pa.int8()])
    try:
        nbytes = chunk.num_rows
        if pinned:
            keep = PinnedArray(max(nbytes, 1), np.uint8)
            host = keep.array[:nbytes]
        else:
            keep = None
            host = np.empty(nbytes, np.uint8)
        capi.check(lib.sb_table_export_host(chunk.handle, 0, host.ctypes.data if nbytes else None, None, None, None, _h(stream)))
    finally:
        chunk.close()
    width = capi.TYPE_WIDTH[d.type]
    phys = (capi.SB_PHYS["DOUBLE"] if d.type == capi.SB_FLOAT64 else capi.SB_PHYS["FLOAT"] if d.type == capi.SB_FLOAT32
            else capi.SB_PHYS["INT64"] if width == 8 else capi.SB_PHYS["INT32"])
    ech = EncodedColumnChunk(d.type, d.scale, phys, host, pages, npages.value, doff.value, dcount.value)
    ech._keep = keep
    return ech
