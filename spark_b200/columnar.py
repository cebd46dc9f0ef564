"""ColumnarBatch / ColumnVector mirrors: HBM-resident Arrow-layout batches behind sb_table handles.

Mirrors sql/catalyst/src/main/java/org/apache/spark/sql/vectorized/ColumnarBatch.java:30-128 and
ArrowColumnVector.java:42-47 of the reference: a batch is an ordered set of named column vectors plus a
row count; whoever creates a batch closes it (SparkPlan.scala:355-358).
"""
from __future__ import annotations

import ctypes as C
import datetime

import numpy as np
import pyarrow as pa

from . import _capi as capi

_ARROW2SB = {pa.bool_(): capi.SB_BOOL, pa.int8(): capi.SB_INT8, pa.int16(): capi.SB_INT16,
             pa.int32(): capi.SB_INT32, pa.int64(): capi.SB_INT64, pa.float32(): capi.SB_FLOAT32,
             pa.float64(): capi.SB_FLOAT64, pa.date32(): capi.SB_DATE32, pa.string(): capi.SB_STRING,
             pa.binary(): capi.SB_STRING}
_SB2ARROW = {capi.SB_BOOL: pa.bool_(), capi.SB_INT8: pa.int8(), capi.SB_INT16: pa.int16(), capi.SB_INT32: pa.int32(),
             capi.SB_INT64: pa.int64(), capi.SB_FLOAT32: pa.float32(), capi.SB_FLOAT64: pa.float64(),
             capi.SB_DATE32: pa.date32(), capi.SB_TIMESTAMP: pa.timestamp("us"), capi.SB_STRING: pa.string()}
_SB2NP = {capi.SB_BOOL: np.uint8, capi.SB_INT8: np.int8, capi.SB_INT16: np.int16, capi.SB_INT32: np.int32,
          capi.SB_INT64: np.int64, capi.SB_FLOAT32: np.float32, capi.SB_FLOAT64: np.float64,
          capi.SB_DATE32: np.int32, capi.SB_TIMESTAMP: np.int64, capi.SB_DECIMAL64: np.int64}


def sb_type_of(arrow_type) -> int:
    if pa.types.is_timestamp(arrow_type):
        return capi.SB_TIMESTAMP
    if pa.types.is_decimal(arrow_type):      # Decimal.scala: precision <= 18 is a long of unscaled values, else 128 bits
        return capi.SB_DECIMAL64 if arrow_type.precision <= 18 else capi.SB_DECIMAL128
    try:
        return _ARROW2SB[arrow_type]
    except KeyError:
        raise capi.SparkB200Error(capi.SB_OK + 5, "unsupported Arrow type %s" % arrow_type)


class Stream:
    """One CUDA stream per Spark task thread (sb_stream)."""

    def __init__(self):
        lib = capi.init()
        h = C.c_void_p()
        capi.check(lib.sb_stream_create(C.byref(h)))
        self.handle = h

    def synchronize(self):
        capi.check(capi.load().sb_stream_synchronize(self.handle))

    def record_start(self):
        capi.check(capi.load().sb_stream_record_start(self.handle))

    def record_stop(self):
        capi.check(capi.load().sb_stream_record_stop(self.handle))

    def elapsed_ms(self) -> float:
        ms = C.c_float()
        capi.check(capi.load().sb_stream_elapsed_ms(self.handle, C.byref(ms)))
        return float(ms.value)

    def close(self):
        if self.handle:
            capi.load().sb_stream_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def _h(stream):
    return stream.handle if stream is not None else None


class PinnedArray:
    """numpy view over sb_host_alloc'd (page-locked) memory, so H2D copies are DMA at PCIe speed."""

    def __init__(self, n, dtype):
        lib = capi.init()
        self.dtype = np.dtype(dtype)
        self.nbytes = int(n) * self.dtype.itemsize
        p = C.c_void_p()
        capi.check(lib.sb_host_alloc(max(self.nbytes, 1), C.byref(p)))
        self.ptr = p
        buf = (C.c_char * max(self.nbytes, 1)).from_address(p.value)
        self.array = np.frombuffer(buf, dtype=self.dtype, count=int(n))

    def close(self):
        if self.ptr:
            self.array = None
            capi.load().sb_host_free(self.ptr)
            self.ptr = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class HostColumn:
    """Host image of one column (Arrow layout) ready for sb_table_import_host."""

    def __init__(self, sb_type, data, validity_bitmap=None, offsets=None, null_count=0, length=None):
        self.type = sb_type
        self.data = data
        self.validity = validity_bitmap
        self.offsets = offsets
        self.null_count = null_count
        self.length = length if length is not None else (len(offsets) - 1 if offsets is not None else len(data))

    @staticmethod
    def from_arrow(arr) -> "HostColumn":
        if isinstance(arr, pa.ChunkedArray):
            arr = arr.combine_chunks() if arr.num_chunks != 1 else arr.chunk(0)
        t = sb_type_of(arr.type)
        n = len(arr)
        validity = None
        if arr.null_count:
            validity = np.packbits(np.asarray(arr.is_valid()), bitorder="little")
        if t == capi.SB_STRING:
            if arr.offset:
                arr = pa.concat_arrays([arr])
            bufs = arr.buffers()
            offs = np.frombuffer(bufs[1], dtype=np.int32, count=n + 1).copy() if n else np.zeros(1, np.int32)
            data = np.frombuffer(bufs[2], dtype=np.uint8).copy() if bufs[2] is not None else np.zeros(0, np.uint8)
            return HostColumn(t, data, validity, offs, arr.null_count, n)
        if t in (capi.SB_DECIMAL64, capi.SB_DECIMAL128):
            # Arrow decimal128: 16-byte little-endian two's complement unscaled values
            raw = np.frombuffer(pa.concat_arrays([arr]).buffers()[1], dtype=np.int64, count=2 * n).reshape(n, 2) if n else np.zeros((0, 2), np.int64)
            vals = np.ascontiguousarray(raw[:, 0]) if t == capi.SB_DECIMAL64 else np.ascontiguousarray(raw).reshape(-1)
            if arr.null_count:
                vals = vals.copy()
                nulls = ~np.asarray(arr.is_valid())
                if t == capi.SB_DECIMAL64:
                    vals[nulls] = 0
                else:
                    vals.reshape(n, 2)[nulls] = 0
            h = HostColumn(t, vals, validity, None, arr.null_count, n)
            h.scale = (arr.type.precision << 8) | arr.type.scale
            return h
        if t == capi.SB_BOOL:
            vals = np.asarray(arr.fill_null(False)).astype(np.uint8)
        elif t == capi.SB_DATE32:
            vals = np.asarray(arr.cast(pa.int32()).fill_null(0))
        elif t == capi.SB_TIMESTAMP:
            vals = np.asarray(arr.cast(pa.int64()).fill_null(0))
        else:
            vals = np.asarray(arr.fill_null(0)) if arr.null_count else np.asarray(arr)
        return HostColumn(t, np.ascontiguousarray(vals, dtype=_SB2NP[t]), validity, None, arr.null_count, n)

    def c(self) -> capi.sb_column:
        s = capi.sb_column()
        s.type = self.type
        s.scale = getattr(self, "scale", 0)
        s.length = self.length
        s.null_count = self.null_count
        s.data = self.data.ctypes.data if self.data is not None and self.data.size else None
        s.validity = self.validity.ctypes.data if self.validity is not None else None
        s.offsets = self.offsets.ctypes.data if self.offsets is not None else None
        return s


class ColumnarBatch:
    """An HBM-resident batch: sb_table handle + column names (+ Arrow types for the way back)."""

    def __init__(self, handle, names, arrow_types=None):
        self.handle = handle
        self.names = list(names)
        self.arrow_types = list(arrow_types) if arrow_types is not None else [None] * len(self.names)

    # ---- construction -------------------------------------------------------------------------
    @staticmethod
    def from_host_columns(names, cols, stream=None, arrow_types=None) -> "ColumnarBatch":
        lib = capi.init()
        arr = (capi.sb_column * max(1, len(cols)))()
        for i, c in enumerate(cols):
            arr[i] = c.c()
        h = C.c_void_p()
        capi.check(lib.sb_table_import_host(arr, len(cols), _h(stream), C.byref(h)))
        if stream is None:
            capi.check(lib.sb_stream_synchronize(None))
        return ColumnarBatch(h, names, arrow_types)

    @staticmethod
    def from_arrow(table: pa.Table, stream=None) -> "ColumnarBatch":
        """RowToColumnarExec replacement (Columnar.scala:503-546): host Arrow buffers -> HBM."""
        cols = [HostColumn.from_arrow(table.column(i)) for i in range(table.num_columns)]
        b = ColumnarBatch.from_host_columns(table.column_names, cols, stream, [f.type for f in table.schema])
        if stream is not None:
            stream.synchronize()   # host staging arrays may be temporaries
        return b

    @staticmethod
    def from_numpy(columns: dict, stream=None, types=None) -> "ColumnarBatch":
        names, cols, ats = [], [], []
        for name, a in columns.items():
            t = (types or {}).get(name)
            if t is None:
                t = {np.dtype(np.int8): capi.SB_INT8, np.dtype(np.int16): capi.SB_INT16, np.dtype(np.int32): capi.SB_INT32,
                     np.dtype(np.int64): capi.SB_INT64, np.dtype(np.float32): capi.SB_FLOAT32,
                     np.dtype(np.float64): capi.SB_FLOAT64, np.dtype(np.uint8): capi.SB_BOOL}[a.dtype]
            names.append(name)
            cols.append(HostColumn(t, np.ascontiguousarray(a)))
            ats.append(_SB2ARROW[t])
        return ColumnarBatch.from_host_columns(names, cols, stream, ats)

    # ---- inspection -----------------------------------------------------------------------------
    @property
    def num_rows(self) -> int:
        n = C.c_int64()
        capi.check(capi.load().sb_table_num_rows(self.handle, C.byref(n)))
        return int(n.value)

    @property
    def num_cols(self) -> int:
        n = C.c_int32()
        capi.check(capi.load().sb_table_num_columns(self.handle, C.byref(n)))
        return int(n.value)

    def column_desc(self, i) -> capi.sb_column:
        d = capi.sb_column()
        capi.check(capi.load().sb_table_column(self.handle, i, C.byref(d)))
        return d

    def column_index(self, name) -> int:
        try:
            return self.names.index(name)
        except ValueError:
            raise KeyError("no column %r in %r" % (name, self.names))

    # ---- ColumnarToRowExec replacement: HBM -> host Arrow -----------------------------------------
    def column_to_numpy(self, i, stream=None):
        """Returns (values ndarray | (offsets, bytes) for strings, valid bool ndarray | None)."""
        lib = capi.load()
        d = self.column_desc(i)
        n = int(d.length)
        bm = np.zeros((n + 7) // 8 + 1, np.uint8) if d.validity else None
        nulls = C.c_int64()
        if d.type == capi.SB_STRING:
            sb = C.c_int64()
            capi.check(lib.sb_table_string_bytes(self.handle, i, C.byref(sb)))
            offs = np.zeros(n + 1, np.int32)
            data = np.zeros(max(int(sb.value), 1), np.uint8)
            capi.check(lib.sb_table_export_host(self.handle, i, data.ctypes.data, bm.ctypes.data if bm is not None else None,
                                                offs.ctypes.data, C.byref(nulls), _h(stream)))
            vals = (offs, data[: int(sb.value)])
        else:
            vals = np.zeros(2 * n, np.int64) if d.type == capi.SB_DECIMAL128 else np.zeros(n, _SB2NP[d.type])
            capi.check(lib.sb_table_export_host(self.handle, i, vals.ctypes.data if n else None,
                                                bm.ctypes.data if bm is not None else None, None, C.byref(nulls), _h(stream)))
        valid = None
        if bm is not None:
            valid = np.unpackbits(bm, bitorder="little")[:n].astype(bool)
        return vals, valid

    def to_arrow(self, stream=None) -> pa.Table:
        out = {}
        for i, name in enumerate(self.names):
            d = self.column_desc(i)
            vals, valid = self.column_to_numpy(i, stream)
            mask = None if valid is None else ~valid
            if d.type == capi.SB_STRING:
                offs, data = vals
                vb = None if valid is None else pa.py_buffer(np.packbits(valid, bitorder="little").tobytes())
                at = self.arrow_types[i] if i < len(self.arrow_types) else None
                typ = pa.binary() if at is not None and (pa.types.is_binary(at) or pa.types.is_large_binary(at)) else pa.string()
                arr = pa.Array.from_buffers(typ, int(d.length), [vb, pa.py_buffer(offs.tobytes()), pa.py_buffer(data.tobytes())])
            elif d.type in (capi.SB_DECIMAL64, capi.SB_DECIMAL128):
                n = int(d.length)
                prec, scale = (d.scale >> 8) & 0xff, d.scale & 0xff
                if prec == 0:
                    prec = 18 if d.type == capi.SB_DECIMAL64 else 38
                if d.type == capi.SB_DECIMAL64:
                    wide = np.empty((n, 2), np.int64)
                    wide[:, 0] = vals
                    wide[:, 1] = vals >> 63            # sign extension
                else:
                    wide = vals.reshape(n, 2)
                vb = None if valid is None else pa.py_buffer(np.packbits(valid, bitorder="little").tobytes())
                arr = pa.Array.from_buffers(pa.decimal128(prec, scale), n, [vb, pa.py_buffer(np.ascontiguousarray(wide).tobytes())])
            elif d.type == capi.SB_BOOL:
                arr = pa.array(vals.astype(bool), mask=mask)
            elif d.type == capi.SB_DATE32:
                arr = pa.array(vals, mask=mask).cast(pa.date32())
            elif d.type == capi.SB_TIMESTAMP:
                arr = pa.array(vals, mask=mask).cast(pa.timestamp("us"))
            else:
                arr = pa.array(vals, mask=mask)
            key = name
            k = 1
            while key in out:   # Arrow tables need unique names; joins may duplicate them
                key = "%s_%d" % (name, k)
                k += 1
            out[key] = arr
        return pa.table(out)

    # ---- cheap structural ops -----------------------------------------------------------------------
    def select(self, names) -> "ColumnarBatch":
        idx = [self.column_index(n) for n in names]
        arr = (C.c_int32 * max(1, len(idx)))(*idx)
        h = C.c_void_p()
        capi.check(capi.load().sb_table_select(self.handle, arr, len(idx), C.byref(h)))
        return ColumnarBatch(h, names, [self.arrow_types[i] for i in idx])

    def rename(self, names) -> "ColumnarBatch":
        capi.check(capi.load().sb_table_retain(self.handle))
        return ColumnarBatch(C.c_void_p(self.handle.value), names, self.arrow_types)

    def zip(self, other) -> "ColumnarBatch":
        h = C.c_void_p()
        capi.check(capi.load().sb_table_zip(self.handle, other.handle, C.byref(h)))
        return ColumnarBatch(h, self.names + other.names, self.arrow_types + other.arrow_types)

    def slice(self, begin, end, stream=None) -> "ColumnarBatch":
        h = C.c_void_p()
        capi.check(capi.load().sb_table_slice(self.handle, begin, end, _h(stream), C.byref(h)))
        return ColumnarBatch(h, self.names, self.arrow_types)

    @staticmethod
    def concat(batches, stream=None) -> "ColumnarBatch":
        """Row-wise concatenation on the device (the reduce side of an exchange stitches fetched blocks this way)."""
        batches = list(batches)
        if not batches:
            raise ValueError("concat of zero batches")
        arr = (C.c_void_p * len(batches))(*[b.handle for b in batches])
        h = C.c_void_p()
        capi.check(capi.load().sb_table_concat(arr, len(batches), _h(stream), C.byref(h)))
        return ColumnarBatch(h, batches[0].names, batches[0].arrow_types)

    def close(self):
        if self.handle:
            capi.load().sb_table_release(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def date_to_days(d) -> int:
    if isinstance(d, datetime.date):
        return (d - datetime.date(1970, 1, 1)).days
    return int(d)
