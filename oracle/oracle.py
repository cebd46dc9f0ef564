"""CPU ORACLE -- test infrastructure, NOT product code.

Python face of ``spark_oracle.c`` plus numpy restatements of the expression / operator semantics of
apache/spark's shuffle / sort / hash-aggregate / hash-join path.  Only ``tests/``,
``__graft_entry__.smoke()`` and ``bench.py``'s cpu_baseline / ``--impl reference`` legs may import
this module; ``spark_b200`` never does.

Parity status: pinned operator-by-operator against the reference's own known-answer vectors
(tests/test_oracle_golden.py); TPC-H answers and the round-robin start offset are "parity unpinned"
(the reference holds no goldens for them) -- see the header of spark_oracle.c and DESIGN.md.

Tables are ``pyarrow.Table`` objects (Arrow layout == the layout of the reference's
ArrowColumnVector, sql/catalyst/src/main/java/org/apache/spark/sql/vectorized/ArrowColumnVector.java:42-47).
Expressions are nested tuples, e.g. ``("mul", ("col", "p"), ("sub", ("lit", 1.0), ("col", "d")))``.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np
import pyarrow as pa

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None

SO_BOOL, SO_INT8, SO_INT16, SO_INT32, SO_INT64, SO_FLOAT32, SO_FLOAT64, SO_DATE32, SO_TIMESTAMP, \
    SO_DECIMAL64, SO_STRING = range(1, 12)


class so_column(C.Structure):
    _fields_ = [("type", C.c_int32), ("scale", C.c_int32), ("length", C.c_int64), ("null_count", C.c_int64),
                ("data", C.c_void_p), ("validity", C.c_void_p), ("offsets", C.c_void_p)]


class so_sort_order(C.Structure):
    _fields_ = [("col", C.c_int32), ("ascending", C.c_int32), ("nulls_first", C.c_int32), ("pad", C.c_int32)]


def build(force: bool = False) -> str:
    """Compile the C restatement (gcc) next to its source."""
    so = os.path.join(_HERE, "libspark_oracle.so")
    src = os.path.join(_HERE, "spark_oracle.c")
    hdr = os.path.join(_HERE, "..", "include", "sb_synth.h")   # the synthetic dataset's definition (pure functions)
    newest = max(os.path.getmtime(src), os.path.getmtime(hdr))
    if force or not os.path.exists(so) or os.path.getmtime(so) < newest:
        cc = "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else "gcc"
        base = [cc, "-O2", "-fPIC", "-shared", "-ffp-contract=off", "-o", so, src, "-lm"]
        r = subprocess.run(base[:2] + ["-fopenmp"] + base[2:], capture_output=True, text=True)
        if r.returncode != 0:
            r = subprocess.run(base, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("oracle build failed:\n" + r.stderr)
    return so


def lib():
    global _LIB
    if _LIB is None:
        so = os.path.join(_HERE, "libspark_oracle.so")   # built by __graft_entry__.build(); the tree may be read-only after that
        L = C.CDLL(so if os.path.exists(so) else build())
        i32, i64, p = C.c_int32, C.c_int64, C.c_void_p
        L.so_threads.restype = i32
        L.so_set_threads.argtypes = [i32]; L.so_set_threads.restype = None
        L.so_murmur3_int.restype = i32; L.so_murmur3_int.argtypes = [i32, i32]
        L.so_murmur3_long.restype = i32; L.so_murmur3_long.argtypes = [i64, i32]
        L.so_murmur3_bytes.restype = i32; L.so_murmur3_bytes.argtypes = [C.c_char_p, i32, i32]
        L.so_murmur3_words.restype = i32; L.so_murmur3_words.argtypes = [C.c_char_p, i32, i32]
        L.so_double_prefix.restype = i64; L.so_double_prefix.argtypes = [C.c_double]
        L.so_hash_rows.argtypes = [p, i32, i64, i32, p]
        L.so_partition_ids.argtypes = [p, i32, i64, i32, p]
        L.so_partition_scatter.argtypes = [p, i64, i32, p, p]
        L.so_round_robin_ids.argtypes = [i64, i32, i32, p]
        L.so_sort_prefix.argtypes = [p, i64, i32, i32, p, p]
        L.so_radix_sort_key_prefix.restype = i32; L.so_radix_sort_key_prefix.argtypes = [p, p, i64, i32, i32, i32, i32]
        L.so_radix_sort.restype = i32; L.so_radix_sort.argtypes = [p, i64, i32, i32, i32, i32]
        L.so_inmemory_sorter_radix.argtypes = [p, p, i64, i32, i32, i32, p]
        L.so_sort_rows.argtypes = [p, p, i32, i64, p]
        L.so_group_ids.restype = i64; L.so_group_ids.argtypes = [p, i32, i64, p, p]
        L.so_agg_sum_i64.argtypes = [p, p, i64, i64, p, p]
        L.so_agg_sum_f64.argtypes = [p, p, i64, i64, p, p]
        L.so_agg_count.argtypes = [p, p, i64, i64, p]
        L.so_agg_minmax_i64.argtypes = [p, p, i64, i64, i32, p, p]
        L.so_agg_minmax_f64.argtypes = [p, p, i64, i64, i32, p, p]
        L.so_hash_join.restype = i64; L.so_hash_join.argtypes = [p, p, i32, i64, i64, i32, p, p]
        L.so_q1_partial_final.restype = i32
        L.so_q1_partial_final.argtypes = [p, p, p, p, p, p, p, i64, i32, i32, p, p, p, p]
        L.so_synth_fill.restype = None; L.so_synth_fill.argtypes = [i32, i32, i64, i64, i64, C.c_uint64, p]
        L.so_synth_rows.restype = i64; L.so_synth_rows.argtypes = [i32, i64]
        L.so_q3.restype = i32
        L.so_q3.argtypes = [p, p, i64, p, p, p, p, i64, p, p, p, p, i64, i32, i32, i32, p, p, p, p, p]
        L.so_q5.restype = None
        L.so_q5.argtypes = [p, p, i64, p, p, p, i64, p, p, p, p, i64, p, p, i64, p, i32, i32, i32, p, p]
        _LIB = L
    return _LIB


# --------------------------------------------------------------------------- columns
_ARROW2SO = {pa.int8(): SO_INT8, pa.int16(): SO_INT16, pa.int32(): SO_INT32, pa.int64(): SO_INT64,
             pa.float32(): SO_FLOAT32, pa.float64(): SO_FLOAT64, pa.date32(): SO_DATE32,
             pa.string(): SO_STRING, pa.binary(): SO_STRING, pa.bool_(): SO_BOOL}
_NP = {SO_BOOL: np.uint8, SO_INT8: np.int8, SO_INT16: np.int16, SO_INT32: np.int32, SO_INT64: np.int64,
       SO_FLOAT32: np.float32, SO_FLOAT64: np.float64, SO_DATE32: np.int32, SO_TIMESTAMP: np.int64,
       SO_DECIMAL64: np.int64}


class Col:
    """One column held as numpy values + numpy bool validity (None = all valid)."""

    def __init__(self, so_type, values, valid=None, offsets=None, arrow_type=None):
        self.type = so_type
        self.values = np.ascontiguousarray(values)
        self.valid = None if valid is None or bool(np.all(valid)) else np.ascontiguousarray(valid, dtype=bool)
        self.offsets = None if offsets is None else np.ascontiguousarray(offsets, dtype=np.int32)
        # decimal(p, s) / timestamp unit of the values: set by from_arrow, kept by take(), restored by to_arrow().  Cols built from
        # the C oracle's outputs have none: a decimal or timestamp result comes back as plain int64
        self.arrow_type = arrow_type
        self._keep = []

    def __len__(self):
        return len(self.offsets) - 1 if self.type == SO_STRING else len(self.values)

    @staticmethod
    def from_arrow(arr) -> "Col":
        if isinstance(arr, pa.ChunkedArray):
            arr = arr.combine_chunks() if arr.num_chunks != 1 else arr.chunk(0)
        t = arr.type
        if pa.types.is_timestamp(t):
            so = SO_TIMESTAMP
        elif pa.types.is_decimal(t):
            if t.precision > 18:
                raise NotImplementedError("decimal(p > 18) columns: only decimal(p <= 18) is a long of unscaled values")
            so = SO_DECIMAL64
        else:
            so = _ARROW2SO[t]
        valid = None
        if arr.null_count:
            valid = np.asarray(arr.is_valid())
        if so == SO_DECIMAL64:   # Decimal.scala: precision <= 18 is held as the unscaled long (low half of Arrow's 16 bytes)
            n = len(arr)
            raw = np.frombuffer(pa.concat_arrays([arr]).buffers()[1], dtype=np.int64, count=2 * n).reshape(n, 2)
            vals = np.where(valid, raw[:, 0], 0) if valid is not None else raw[:, 0]
            return Col(so, vals.astype(np.int64), valid, arrow_type=t)
        if so == SO_STRING:
            n = len(arr)
            arr = pa.concat_arrays([arr]) if arr.offset else arr
            bufs = arr.buffers()
            offs = np.frombuffer(bufs[1], dtype=np.int32, count=n + 1) if n + 1 > 0 and bufs[1] is not None else np.zeros(1, np.int32)
            data = np.frombuffer(bufs[2], dtype=np.uint8) if bufs[2] is not None else np.zeros(0, np.uint8)
            return Col(so, data, valid, offs)
        if so == SO_BOOL:
            vals = np.asarray(arr.fill_null(False)).astype(np.uint8)
        elif so == SO_DATE32:
            vals = np.asarray(arr.cast(pa.int32()).fill_null(0))
        elif so == SO_TIMESTAMP:
            vals = np.asarray(arr.cast(pa.int64()).fill_null(0))
        else:
            vals = np.asarray(arr.fill_null(0))
        return Col(so, vals.astype(_NP[so], copy=False), valid, arrow_type=t if so == SO_TIMESTAMP else None)

    def to_arrow(self):
        mask = None if self.valid is None else ~self.valid
        if self.type == SO_STRING:
            n = len(self)
            vb = None
            if self.valid is not None:
                vb = pa.py_buffer(np.packbits(self.valid, bitorder="little").tobytes())
            return pa.Array.from_buffers(pa.string(), n, [vb, pa.py_buffer(self.offsets.tobytes()),
                                                          pa.py_buffer(self.values.tobytes())])
        if self.type == SO_BOOL:
            return pa.array(self.values.astype(bool), mask=mask)
        if self.type == SO_DECIMAL64 and self.arrow_type is not None:
            n = len(self.values)
            wide = np.empty((n, 2), np.int64)
            wide[:, 0] = self.values
            wide[:, 1] = self.values >> 63            # sign extension to Arrow's 16-byte two's complement
            vb = None if self.valid is None else pa.py_buffer(np.packbits(self.valid, bitorder="little").tobytes())
            return pa.Array.from_buffers(self.arrow_type, n, [vb, pa.py_buffer(wide.tobytes())])
        a = pa.array(self.values, mask=mask)
        if self.type == SO_DATE32:
            a = a.cast(pa.date32())
        elif self.type == SO_TIMESTAMP and self.arrow_type is not None:
            a = a.cast(self.arrow_type)
        return a

    def bitmap(self):
        if self.valid is None:
            return None
        return np.packbits(self.valid, bitorder="little")

    def c(self) -> so_column:
        s = so_column()
        s.type = self.type
        s.scale = 0
        s.length = len(self)
        s.null_count = 0 if self.valid is None else int((~self.valid).sum())
        s.data = self.values.ctypes.data if self.values.size else None
        bm = self.bitmap()
        self._keep = [bm]
        s.validity = bm.ctypes.data if bm is not None else None
        s.offsets = self.offsets.ctypes.data if self.offsets is not None else None
        return s

    def take(self, idx) -> "Col":
        """Gather rows; idx < 0 yields NULL (outer-join padding)."""
        idx = np.asarray(idx, dtype=np.int64)
        neg = idx < 0
        safe = np.where(neg, 0, idx)
        if self.type == SO_STRING:
            arr = self.to_arrow().take(pa.array(safe))
            c = Col.from_arrow(arr)
            valid = np.ones(len(idx), bool) if c.valid is None else c.valid.copy()
            valid[neg] = False
            c.valid = None if valid.all() else valid
            return c
        if len(self) == 0:
            vals = np.zeros(len(idx), dtype=self.values.dtype)
            valid = ~neg
        else:
            vals = self.values[safe]
            valid = (np.ones(len(idx), bool) if self.valid is None else self.valid[safe]) & ~neg
        return Col(self.type, vals, valid, arrow_type=self.arrow_type)


def _cols(table, names):
    return [Col.from_arrow(table.column(n)) for n in names]


def _carray(cols):
    arr = (so_column * max(1, len(cols)))()
    for i, c in enumerate(cols):
        arr[i] = c.c()
    return arr


def table_from_cols(names, cols):
    return pa.table({n: c.to_arrow() for n, c in zip(names, cols)})


def take_table(table, idx):
    return table_from_cols(table.column_names, [Col.from_arrow(table.column(n)).take(idx) for n in table.column_names])


# --------------------------------------------------------------------------- hashing / partitioning
def hash_rows(table, key_cols, seed=42):
    """Murmur3Hash(exprs, seed) per row (hash.scala:400-409, 707-760)."""
    cols = _cols(table, key_cols)
    n = table.num_rows
    out = np.empty(n, np.int32)
    lib().so_hash_rows(_carray(cols), len(cols), n, seed, out.ctypes.data)
    return out


def partition_ids(table, key_cols, num_partitions):
    """HashPartitioning.partitionIdExpression (partitioning.scala:339-341)."""
    cols = _cols(table, key_cols)
    n = table.num_rows
    out = np.empty(n, np.int32)
    lib().so_partition_ids(_carray(cols), len(cols), n, num_partitions, out.ctypes.data)
    return out


def scatter_by_pid(pid, num_partitions):
    pid = np.ascontiguousarray(pid, np.int32)
    perm = np.empty(len(pid), np.int64)
    offs = np.empty(num_partitions + 1, np.int64)
    lib().so_partition_scatter(pid.ctypes.data, len(pid), num_partitions, perm.ctypes.data, offs.ctypes.data)
    return perm, offs


def hash_partition(table, key_cols, num_partitions):
    """ShuffleExchangeExec with HashPartitioning, map side: rows grouped by partition id, arrival
    order kept inside a partition.  Returns (reordered table, offsets[n+1])."""
    pid = partition_ids(table, key_cols, num_partitions)
    perm, offs = scatter_by_pid(pid, num_partitions)
    return take_table(table, perm), offs


def round_robin_partition(table, num_partitions, start):
    """RoundRobinPartitioning ids (ShuffleExchangeExec.scala:428-442); `start` is the
    XORShiftRandom(mapPartitionId).nextInt(n) draw -- parity unpinned, supplied by the caller."""
    n = table.num_rows
    pid = np.empty(n, np.int32)
    lib().so_round_robin_ids(n, num_partitions, start, pid.ctypes.data)
    perm, offs = scatter_by_pid(pid, num_partitions)
    return take_table(table, perm), offs


def range_partition_ids(table, order, bounds):
    """RangePartitioner.getPartition (core/src/main/scala/org/apache/spark/Partitioner.scala:241-260): the partition of a row
    is the number of range bounds its key is strictly greater than under the sort ordering (NULL placement and double
    ordering as in the sort).  order = (col, ascending, nulls_first); bounds = pyarrow array of the sorted bounds."""
    name, asc, nf = order
    nb = len(bounds)
    both = pa.table({"k": pa.concat_arrays([table.column(name).combine_chunks() if isinstance(table.column(name), pa.ChunkedArray) else table.column(name),
                                            bounds.cast(table.column(name).type)]), "i": np.arange(table.num_rows + nb)})
    n = table.num_rows
    pid = np.zeros(n, np.int32)
    cols = _cols(both, ["k", "i"])
    ords = (so_sort_order * 1)()
    ords[0].col = 0; ords[0].ascending = int(asc); ords[0].nulls_first = int(nf)
    # stable sort of keys ++ bounds: a bound counts for a key iff it sorts strictly before it, i.e. ties must put keys first
    perm = np.empty(n + nb, np.int64)
    # order rows so that for equal values keys (index < n) precede bounds (index >= n): arrival order already does that
    lib().so_sort_rows(_carray(cols), ords, 1, n + nb, perm.ctypes.data)
    is_bound = perm >= n
    bounds_before = np.cumsum(is_bound) - is_bound
    pid_sorted = bounds_before
    out = np.empty(n + nb, np.int64)
    out[perm] = pid_sorted
    return out[:n].astype(np.int32)


def range_partition(table, order, bounds):
    pid = range_partition_ids(table, order, bounds)
    perm, offs = scatter_by_pid(pid, len(bounds) + 1)
    return take_table(table, perm), offs


# --------------------------------------------------------------------------- sort
_RADIX_TYPES = {SO_BOOL, SO_INT8, SO_INT16, SO_INT32, SO_INT64, SO_FLOAT32, SO_FLOAT64, SO_DATE32,
                SO_TIMESTAMP, SO_DECIMAL64}


def sort_prefix(col: Col, ascending=True, nulls_first=True):
    n = len(col)
    prefix = np.empty(n, np.int64)
    isnull = np.empty(n, np.uint8)
    cc = col.c()
    lib().so_sort_prefix(C.byref(cc), n, int(ascending), int(nulls_first), prefix.ctypes.data, isnull.ctypes.data)
    return prefix, isnull


def sort_permutation(table, orders):
    """SortExec for one partition.  orders = [(col, ascending, nulls_first), ...].
    One radix-eligible column -> UnsafeInMemorySorter radix path (SortExec.scala:82-83,
    SortPrefixUtils.scala:123-137); otherwise the stable full-row comparison sort (TimSort path)."""
    n = table.num_rows
    perm = np.empty(n, np.int64)
    names = table.column_names
    if len(orders) == 1:
        name, asc, nf = orders[0]
        col = Col.from_arrow(table.column(name))
        if col.type in _RADIX_TYPES:
            prefix, isnull = sort_prefix(col, asc, nf)
            sgn = col.type not in (SO_FLOAT32, SO_FLOAT64)     # PrefixComparators: DOUBLE is unsigned
            lib().so_inmemory_sorter_radix(prefix.ctypes.data, isnull.ctypes.data, n, int(not asc), int(sgn),
                                           int(nf), perm.ctypes.data)
            return perm
    cols = _cols(table, names)
    ords = (so_sort_order * len(orders))()
    for i, (name, asc, nf) in enumerate(orders):
        ords[i].col = names.index(name); ords[i].ascending = int(asc); ords[i].nulls_first = int(nf)
    lib().so_sort_rows(_carray(cols), ords, len(orders), n, perm.ctypes.data)
    return perm


def sort(table, orders):
    return take_table(table, sort_permutation(table, orders))


def take_ordered(table, orders, k):
    """TakeOrderedAndProjectExec (limit.scala:347-386): top-k by the full ordering."""
    cols = _cols(table, table.column_names)
    names = table.column_names
    n = table.num_rows
    perm = np.empty(n, np.int64)
    ords = (so_sort_order * len(orders))()
    for i, (name, asc, nf) in enumerate(orders):
        ords[i].col = names.index(name); ords[i].ascending = int(asc); ords[i].nulls_first = int(nf)
    lib().so_sort_rows(_carray(cols), ords, len(orders), n, perm.ctypes.data)
    return take_table(table, perm[:k])


# --------------------------------------------------------------------------- expressions
def _wrap(a, dtype):
    return a.astype(dtype, copy=False)


def _dcmp(x, y):
    """SQLOrderingUtil.compareDoubles: NaN == NaN, NaN largest, -0.0 == 0.0."""
    xn, yn = np.isnan(x), np.isnan(y)
    with np.errstate(invalid="ignore"):
        r = np.where(x == y, 0, np.where(x < y, -1, 1))
    r = np.where(xn & yn, 0, np.where(xn, 1, np.where(yn, -1, r)))
    return r


def eval_expr(e, table):
    """Evaluate a tuple expression -> (values ndarray, valid bool ndarray).  Null-propagating
    arithmetic/comparison, Kleene AND/OR (predicates.scala And/Or), non-ANSI wrap-around integers,
    Divide -> NULL on zero divisor (arithmetic.scala DivModLike)."""
    n = table.num_rows
    op = e[0]
    if op == "col":
        c = Col.from_arrow(table.column(e[1]))
        v = c.values
        if c.type == SO_BOOL:
            v = v.astype(bool)
        return v, (np.ones(n, bool) if c.valid is None else c.valid)
    if op == "lit":
        val = e[1]
        dt = e[2] if len(e) > 2 else None
        if val is None:                      # a typed NULL keeps its class
            return np.zeros(n, dt or np.int64), np.zeros(n, bool)
        if dt is None:
            dt = np.float64 if isinstance(val, float) else (bool if isinstance(val, bool) else np.int64)
        return np.full(n, val, dtype=dt), np.ones(n, bool)
    if op in ("add", "sub", "mul"):
        a, av = eval_expr(e[1], table); b, bv = eval_expr(e[2], table)
        dt = np.result_type(a.dtype, b.dtype)
        a = a.astype(dt); b = b.astype(dt)
        with np.errstate(over="ignore", invalid="ignore"):
            r = a + b if op == "add" else (a - b if op == "sub" else a * b)
        return r, av & bv
    if op == "div":
        a, av = eval_expr(e[1], table); b, bv = eval_expr(e[2], table)
        a = a.astype(np.float64); b = b.astype(np.float64)
        nz = b != 0
        with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
            r = np.where(nz, a / np.where(nz, b, 1.0), 0.0)
        return r, av & bv & nz
    if op == "neg":
        a, av = eval_expr(e[1], table)
        with np.errstate(over="ignore"):
            return -a, av
    if op in ("eq", "ne", "lt", "le", "gt", "ge"):
        a, av = eval_expr(e[1], table); b, bv = eval_expr(e[2], table)
        if a.dtype.kind == "f" or b.dtype.kind == "f":
            c = _dcmp(a.astype(np.float64), b.astype(np.float64))
        else:
            dt = np.result_type(a.dtype, b.dtype)
            a = a.astype(dt); b = b.astype(dt)
            c = np.where(a == b, 0, np.where(a < b, -1, 1))
        r = {"eq": c == 0, "ne": c != 0, "lt": c < 0, "le": c <= 0, "gt": c > 0, "ge": c >= 0}[op]
        return r, av & bv
    if op == "and":
        a, av = eval_expr(e[1], table); b, bv = eval_expr(e[2], table)
        a = a.astype(bool); b = b.astype(bool)
        false_a, false_b = av & ~a, bv & ~b
        valid = (av & bv) | false_a | false_b
        return (a & b) & av & bv, valid
    if op == "or":
        a, av = eval_expr(e[1], table); b, bv = eval_expr(e[2], table)
        a = a.astype(bool); b = b.astype(bool)
        true_a, true_b = av & a, bv & b
        valid = (av & bv) | true_a | true_b
        return true_a | true_b, valid
    if op == "not":
        a, av = eval_expr(e[1], table)
        return ~a.astype(bool), av
    if op == "isnull":
        a, av = eval_expr(e[1], table)
        return ~av, np.ones(n, bool)
    if op == "isnotnull":
        a, av = eval_expr(e[1], table)
        return av.copy(), np.ones(n, bool)
    if op == "cast_f64":
        a, av = eval_expr(e[1], table)
        return a.astype(np.float64), av
    if op in ("cast_i64", "cast_i32"):
        a, av = eval_expr(e[1], table)
        dt = np.int64 if op == "cast_i64" else np.int32
        if a.dtype.kind == "f":
            return _java_double_to_int(a.astype(np.float64), dt), av
        return a.astype(dt), av          # long -> int keeps the low 32 bits (JLS 5.1.3 narrowing)
    raise ValueError("unknown expression op %r" % (op,))


def _java_double_to_int(a, dt):
    """Java's (long) d / (int) d (JLS 5.1.3, what Cast.scala:1159-1161 `numeric.toLong` / `toInt` run): NaN -> 0, otherwise
    rounded toward zero and saturated at the target's range.  numpy's astype would give INT64_MIN for NaN and +-inf."""
    info = np.iinfo(dt)
    hi = float(info.max) + 1.0                  # 2^31 / 2^63, exact in double
    out = np.zeros(len(a), dt)
    with np.errstate(invalid="ignore"):
        big, small = a >= hi, a <= -hi
        mid = ~(big | small | np.isnan(a))
    out[big], out[small] = info.max, info.min
    out[mid] = np.trunc(a[mid]).astype(dt)
    return out


def _col_from_eval(v, valid):
    if v.dtype == bool:
        return Col(SO_BOOL, v.astype(np.uint8), valid)
    so = {np.dtype(np.int8): SO_INT8, np.dtype(np.int16): SO_INT16, np.dtype(np.int32): SO_INT32,
          np.dtype(np.int64): SO_INT64, np.dtype(np.float32): SO_FLOAT32, np.dtype(np.float64): SO_FLOAT64}[v.dtype]
    return Col(so, v, valid)


def filter_table(table, predicate):
    """FilterExec: keep rows whose predicate is TRUE (NULL drops the row)."""
    v, valid = eval_expr(predicate, table)
    keep = np.nonzero(v.astype(bool) & valid)[0]
    return take_table(table, keep)


def filter_mask(table, predicate):
    """Boolean mask of the rows a FilterExec keeps (predicate TRUE, not NULL)."""
    v, valid = eval_expr(predicate, table)
    return v.astype(bool) & valid


def project(table, named_exprs):
    """ProjectExec: named_exprs = [(name, expr)]; ("col", x) keeps the source type (dates, strings)."""
    out = {}
    for name, e in named_exprs:
        if e[0] == "col":
            out[name] = table.column(e[1])
        else:
            v, valid = eval_expr(e, table)
            out[name] = _col_from_eval(v, valid).to_arrow()
    return pa.table(out)


# --------------------------------------------------------------------------- hash aggregate
def normalize_floats(col: Col) -> Col:
    """NormalizeNaNAndZero (sql/catalyst/.../optimizer/NormalizeFloatingNumbers.scala:180-199): -0.0 -> 0.0 and every NaN -> the
    canonical Float.NaN / Double.NaN (0x7fc00000 / 0x7ff8000000000000).  The aggregation strategy applies it to the grouping
    expressions (sql/core/.../execution/SparkStrategies.scala:736-745), so a group key comes out normalised."""
    if col.type not in (SO_FLOAT32, SO_FLOAT64):
        return col
    v = col.values.copy()
    with np.errstate(invalid="ignore"):
        v[v == 0] = 0.0
    v[np.isnan(v)] = np.nan      # numpy's nan is the canonical quiet NaN in both widths
    return Col(col.type, v, col.valid)


def _group(table, key_cols):
    n = table.num_rows
    cols = _cols(table, key_cols)
    for c in cols:
        if c.type == SO_STRING:
            raise NotImplementedError("string group keys: dictionary-encode to integer codes first")
    gid = np.empty(n, np.int64)
    first = np.empty(max(n, 1), np.int64)
    if len(cols) == 0:
        gid[:] = 0
        return gid, np.zeros(1, np.int64), 1        # no grouping keys: one group even for empty input
    ng = lib().so_group_ids(_carray(cols), len(cols), n, gid.ctypes.data, first.ctypes.data)
    return gid, first[:ng], ng


def hash_aggregate(table, key_cols, aggs, mode="complete"):
    """HashAggregateExec.  aggs = [(func, input, out_name)] with func in
    sum/avg/count/count_star/min/max; `input` is a column name (Complete/Partial) -- for Final mode
    the table holds the Partial output (keys ++ buffers named as produced below).
    Buffer layout (AggUtils.scala:170-205): sum -> <name>#sum ; avg -> <name>#sum, <name>#count ;
    count -> <name>#count ; min/max -> <name>#val.
    Result types: Sum(integral) long, Sum(fp) double, Avg double, Count long (Sum.scala:80-88,
    Average.scala:80, Count.scala:54)."""
    L = lib()
    gid, first, ng = _group(table, key_cols)
    n = table.num_rows
    out_names, out_cols = [], []
    for k in key_cols:
        out_names.append(k); out_cols.append(normalize_floats(Col.from_arrow(table.column(k)).take(first)))
    gp = gid.ctypes.data

    def sum_of(col):
        cc = col.c()
        if col.type in (SO_FLOAT32, SO_FLOAT64):
            o = np.empty(ng, np.float64); ov = np.empty(ng, np.uint8)
            L.so_agg_sum_f64(gp, C.byref(cc), n, ng, o.ctypes.data, ov.ctypes.data)
            return Col(SO_FLOAT64, o, ov.astype(bool))
        o = np.empty(ng, np.int64); ov = np.empty(ng, np.uint8)
        L.so_agg_sum_i64(gp, C.byref(cc), n, ng, o.ctypes.data, ov.ctypes.data)
        return Col(SO_INT64, o, ov.astype(bool))

    def count_of(col):
        o = np.empty(ng, np.int64)
        if col is None:
            L.so_agg_count(gp, None, n, ng, o.ctypes.data)
        else:
            cc = col.c()
            L.so_agg_count(gp, C.byref(cc), n, ng, o.ctypes.data)
        return Col(SO_INT64, o)

    def minmax_of(col, is_max):
        cc = col.c()
        if col.type in (SO_FLOAT32, SO_FLOAT64):
            o = np.empty(ng, np.float64); ov = np.empty(ng, np.uint8)
            L.so_agg_minmax_f64(gp, C.byref(cc), n, ng, int(is_max), o.ctypes.data, ov.ctypes.data)
            return Col(SO_FLOAT64 if col.type == SO_FLOAT64 else SO_FLOAT32,
                       o.astype(_NP[col.type]), ov.astype(bool))
        o = np.empty(ng, np.int64); ov = np.empty(ng, np.uint8)
        L.so_agg_minmax_i64(gp, C.byref(cc), n, ng, int(is_max), o.ctypes.data, ov.ctypes.data)
        return Col(col.type, o.astype(_NP[col.type]), ov.astype(bool))

    for func, inp, name in aggs:
        if mode in ("complete", "partial"):
            col = None if func == "count_star" else Col.from_arrow(table.column(inp))
            if func == "sum":
                bufs = [("#sum", sum_of(col))]
            elif func == "avg":
                s = sum_of(Col(SO_FLOAT64, col.values.astype(np.float64), col.valid))
                # Average buffer sum starts at 0, never NULL (Average.scala:93-97)
                s = Col(SO_FLOAT64, np.where(s.valid, s.values, 0.0) if s.valid is not None else s.values)
                bufs = [("#sum", s), ("#count", count_of(col))]
            elif func in ("count", "count_star"):
                bufs = [("#count", count_of(col))]
            elif func in ("min", "max"):
                bufs = [("#val", minmax_of(col, func == "max"))]
            else:
                raise ValueError(func)
        else:  # final: merge buffers
            if func == "sum":
                bufs = [("#sum", sum_of(Col.from_arrow(table.column(name + "#sum"))))]
            elif func == "avg":
                s = sum_of(Col.from_arrow(table.column(name + "#sum")))
                s = Col(SO_FLOAT64, np.where(s.valid, s.values, 0.0) if s.valid is not None else s.values)
                c = sum_of(Col.from_arrow(table.column(name + "#count")))
                c = Col(SO_INT64, np.where(c.valid, c.values, 0) if c.valid is not None else c.values)
                bufs = [("#sum", s), ("#count", c)]
            elif func in ("count", "count_star"):
                c = sum_of(Col.from_arrow(table.column(name + "#count")))
                c = Col(SO_INT64, np.where(c.valid, c.values, 0) if c.valid is not None else c.values)
                bufs = [("#count", c)]
            elif func in ("min", "max"):
                bufs = [("#val", minmax_of(Col.from_arrow(table.column(name + "#val")), func == "max"))]
            else:
                raise ValueError(func)
        if mode == "partial":
            for suf, c in bufs:
                out_names.append(name + suf); out_cols.append(c)
        else:  # evaluate (Sum.scala:180, Average.scala:109-127, Count.scala)
            if func == "avg":
                s, c = bufs[0][1], bufs[1][1]
                nz = c.values != 0
                with np.errstate(divide="ignore", invalid="ignore"):
                    r = np.where(nz, s.values / np.where(nz, c.values, 1), 0.0)
                out_names.append(name); out_cols.append(Col(SO_FLOAT64, r, nz))
            else:
                out_names.append(name); out_cols.append(bufs[0][1])
    return table_from_cols(out_names, out_cols)


# --------------------------------------------------------------------------- hash join
JOIN_TYPES = {"inner": 0, "left_outer": 1, "left_semi": 2, "left_anti": 3}


def hash_join(probe, build, probe_keys, build_keys, join_type="inner", condition=None):
    """Equi-join with `probe` as the streamed side and `build` as the hashed side
    (BroadcastHashJoinExec / ShuffledHashJoinExec; SortMergeJoinExec gives the same multiset).
    join_type: inner | left_outer | left_semi | left_anti | full_outer | build_outer (the hashed side preserved) | existence |
    left_anti_null_aware.  `condition` (an expression over probe ++ build columns) is HashJoin.boundCondition
    (HashJoin.scala:144-172): only key matches for which it is TRUE are matches.
    Output columns: probe columns ++ build columns (semi/anti: probe columns only; existence: probe ++ `exists`)."""
    L = lib()
    pk = _cols(probe, probe_keys); bk = _cols(build, build_keys)
    pa_, ba_ = _carray(pk), _carray(bk)
    np_, nb_ = probe.num_rows, build.num_rows
    cnt = L.so_hash_join(ba_, pa_, len(pk), nb_, np_, 0, None, None)          # every key match (inner pairs)
    pi = np.empty(cnt, np.int64); bi = np.empty(cnt, np.int64)
    L.so_hash_join(ba_, pa_, len(pk), nb_, np_, 0, pi.ctypes.data, bi.ctypes.data)
    names = list(probe.column_names) + list(build.column_names)

    def joined(p_idx, b_idx):
        cols = [Col.from_arrow(probe.column(n)).take(p_idx) for n in probe.column_names]
        cols += [Col.from_arrow(build.column(n)).take(b_idx) for n in build.column_names]
        return table_from_cols(names, cols)
    if condition is not None and cnt:
        keep = filter_mask(joined(pi, bi), condition)
        pi, bi = pi[keep], bi[keep]
    p_matched = np.zeros(np_, bool); p_matched[pi] = True
    b_matched = np.zeros(nb_, bool); b_matched[bi] = True
    if join_type == "inner":
        return joined(pi, bi)
    if join_type in ("left_semi", "left_anti", "left_anti_null_aware"):
        if join_type == "left_semi":
            sel = np.nonzero(p_matched)[0]
        elif join_type == "left_anti":
            sel = np.nonzero(~p_matched)[0]
        else:   # BroadcastHashJoinExec.scala:137-162
            bnull = np.zeros(nb_, bool)
            for c in bk:
                if c.valid is not None:
                    bnull |= ~c.valid
            pnull = np.zeros(np_, bool)
            for c in pk:
                if c.valid is not None:
                    pnull |= ~c.valid
            sel = np.arange(np_) if nb_ == 0 else (np.zeros(0, np.int64) if bnull.any() else np.nonzero(~p_matched & ~pnull)[0])
        return table_from_cols(list(probe.column_names), [Col.from_arrow(probe.column(n)).take(sel.astype(np.int64)) for n in probe.column_names])
    if join_type == "existence":
        cols = [Col.from_arrow(probe.column(n)) for n in probe.column_names] + [Col(SO_BOOL, p_matched.astype(np.uint8))]
        return table_from_cols(list(probe.column_names) + ["exists"], cols)
    up = np.nonzero(~p_matched)[0] if join_type in ("left_outer", "full_outer") else np.zeros(0, np.int64)
    ub = np.nonzero(~b_matched)[0] if join_type in ("build_outer", "full_outer") else np.zeros(0, np.int64)
    p_idx = np.concatenate([pi, up, np.full(len(ub), -1)]).astype(np.int64)
    b_idx = np.concatenate([bi, np.full(len(up), -1), ub]).astype(np.int64)
    return joined(p_idx, b_idx)


# --------------------------------------------------------------------------- comparison helpers
def canonical_rows(table, float_digits=None):
    """Rows sorted like the reference's checkAnswer (QueryTest.scala / RowComparisonUtils.scala:87-112):
    order-insensitive comparison by sorting rows."""
    cols = []
    for name in table.column_names:
        a = table.column(name).to_pylist()
        cols.append(a)
    rows = list(zip(*cols)) if cols else []

    def key(r):
        return tuple((x is None, 0 if x is None else (repr(x) if not isinstance(x, (int, float)) else x)) for x in r)
    return sorted(rows, key=lambda r: tuple((x is None, "" if x is None else str(type(x)), 0 if x is None else x) for x in r))


# --------------------------------------------------------------------------- RangePartitioner.determineBounds
def determine_bounds(candidates, partitions, key=None):
    """RangePartitioner.determineBounds (core/src/main/scala/org/apache/spark/Partitioner.scala:357-388), line by line:
    candidates = [(key, weight float32)], unordered; `key` maps a candidate key to its sort key (None = natural order).
    Pinned by PartitioningSuite.scala:119-125 (tests/test_oracle_golden.py)."""
    keyf = key or (lambda x: x)
    ordered = sorted(candidates, key=lambda kw: keyf(kw[0]))           # sortBy(_._1) is stable, like sorted()
    num = len(ordered)
    sum_weights = sum(float(np.float32(w)) for _, w in ordered)
    step = sum_weights / partitions if partitions else 0.0
    cum, target = 0.0, step
    bounds = []
    i = j = 0
    previous = None
    have_prev = False
    while i < num and j < partitions - 1:
        k, w = ordered[i]
        cum += float(np.float32(w))
        if cum >= target:
            if not have_prev or keyf(k) > keyf(previous):               # skip duplicate values
                bounds.append(k)
                target += step
                j += 1
                previous, have_prev = k, True
        i += 1
    return bounds


# --------------------------------------------------------------------------- AQE: ShufflePartitionsUtil.coalescePartitions
def coalesce_partitions(bytes_by_partition, advisory_target_size, min_num_partitions=1, min_partition_size=0,
                        max_reducer_partitions_per_task=2 ** 31 - 1):
    """ShufflePartitionsUtil.coalescePartitions without skew specs (sql/core/.../adaptive/ShufflePartitionsUtil.scala:45-126,
    263-369).  bytes_by_partition: one list per shuffle.  Returns, per shuffle, [(start, end, dataSize)] or [] for "no coalescing".
    Pinned by ShufflePartitionsUtilSuite.scala:54-300 (tests/test_oracle_golden.py)."""
    import math
    stats = [list(b) for b in bytes_by_partition]
    if not stats:
        return []
    total = sum(sum(b) for b in stats)
    max_target = int(math.ceil(total / float(min_num_partitions)))
    target = max(min(max_target, advisory_target_size), min_partition_size)
    if len({len(b) for b in stats}) > 1:
        return []
    n = len(stats[0])
    specs = []
    coalesced = latest_size = 0
    i = latest_split = 0

    def create(force=False):
        if coalesced > 0 or force:
            specs.append([latest_split, i])

    def within(a, b):
        return b - a <= max_reducer_partitions_per_task
    while i < n:
        cur = sum(b[i] for b in stats)
        if i > latest_split and i - latest_split >= max_reducer_partitions_per_task:
            create()
            latest_split, latest_size, coalesced = i, coalesced, cur
        elif i > latest_split and coalesced + cur > target:
            if coalesced < min_partition_size:
                if latest_size > 0 and latest_size < cur and within(specs[-1][0], i):
                    specs[-1][1] = i
                    latest_split = i
                    latest_size += coalesced
                    coalesced = cur
                else:
                    coalesced += cur
            else:
                create()
                latest_split, latest_size, coalesced = i, coalesced, cur
        else:
            coalesced += cur
        i += 1
    if coalesced < min_partition_size and latest_size > 0 and within(specs[-1][0], n):
        specs[-1][1] = n
    else:
        create(not specs)
    if len(specs) >= n:
        return []
    return [[(a, b, sum(st[a:b])) for a, b in specs] for st in stats]


# --------------------------------------------------------------------------- string keys
def binary_compare(a: bytes, b: bytes) -> int:
    """UTF8String.binaryCompare (common/unsafe/.../types/UTF8String.java:2075) -> ByteArray.compareBinary
    (common/unsafe/.../types/ByteArray.java): compare as UNSIGNED bytes up to the shorter length, then the shorter one first."""
    m = min(len(a), len(b))
    for i in range(m):
        if a[i] != b[i]:
            return (a[i] & 0xFF) - (b[i] & 0xFF)
    return len(a) - len(b)


def string_codes(column):
    """Order-preserving dictionary codes of a string column: (int32 arrow array, NULL where the string is NULL; the sorted list
    of distinct values as bytes).  code(a) < code(b) <=> binary_compare(a, b) < 0 -- how grouping (equality), joins (equality) and
    sorts (SortOrder on StringType: UTF8String.compareTo) see the column."""
    import functools
    vals = [None if v is None else (v if isinstance(v, bytes) else v.encode("utf-8")) for v in column.to_pylist()]
    dictionary = sorted({v for v in vals if v is not None}, key=functools.cmp_to_key(binary_compare))
    rank = {v: i for i, v in enumerate(dictionary)}
    return pa.array([None if v is None else rank[v] for v in vals], type=pa.int32()), dictionary


def encode_string_columns(table, cols, dictionaries=None):
    """table with the string columns `cols` replaced by their codes; returns (table, {col: dictionary}).  dictionaries: encode
    against existing ones instead (values outside get -1, like a probe-side key the build side never saw)."""
    out, dicts = table, {}
    for c in cols:
        i = table.column_names.index(c)
        if dictionaries is None:
            codes, d = string_codes(table.column(c))
        else:
            d = dictionaries[c]
            rank = {v: k for k, v in enumerate(d)}
            vals = [None if v is None else (v if isinstance(v, bytes) else v.encode("utf-8")) for v in table.column(c).to_pylist()]
            codes = pa.array([None if v is None else rank.get(v, -1) for v in vals], type=pa.int32())
        out = out.set_column(i, c, codes)
        dicts[c] = d
    return out, dicts


def decode_string_columns(table, dicts, as_type=None):
    out = table
    for c, d in dicts.items():
        if c not in table.column_names:
            continue
        i = table.column_names.index(c)
        codes = table.column(c).to_pylist()
        vals = [None if (k is None or k < 0) else d[k] for k in codes]
        t = as_type or pa.string()
        out = out.set_column(i, c, pa.array([None if v is None else (v.decode("utf-8") if t == pa.string() else v) for v in vals], type=t))
    return out


# --------------------------------------------------------------------------- ExpandExec / WindowExec (test sizes: plain Python loops)
def expand(table, projections, names):
    """ExpandExec.doExecute (sql/core/.../execution/ExpandExec.scala:85-97): `iter.flatMap { input => groups.iterator.map(_(input)) }`:
    for every input row, one output row per projection list, list 0 first.  projections: lists of expression s-exprs (eval_expr)."""
    n = table.num_rows
    cols = []
    for c in range(len(names)):
        per_list = []
        for plist in projections:
            e = plist[c]
            if e[0] == "col":
                per_list.append(table.column(e[1]).to_pylist())
            else:
                v, valid = eval_expr(e, table)
                per_list.append([v[i].item() if valid[i] else None for i in range(n)])
        cols.append([per_list[l][r] for r in range(n) for l in range(len(projections))])
    out = {}
    for c, name in enumerate(names):
        e0 = projections[0][c]
        t = table.column(e0[1]).type if e0[0] == "col" else None
        out[name] = pa.array(cols[c], type=t) if t is not None else pa.array(cols[c])
    return pa.table(out)


def _norm_key(v):
    if isinstance(v, float):
        if v != v:
            return ("nan",)
        if v == 0.0:
            return 0.0
    return v


def _window_layout(table, partition_cols, orders):
    """The sorted input of a WindowExec and, per sorted row, its partition [seg_start, seg_end) and peer group
    [peer_start, peer_end), plus the single ORDER BY key's values for RANGE frames with value offsets (None otherwise)."""
    key_cols = list(partition_cols) + [o[0] for o in orders]
    str_cols = [c for c in dict.fromkeys(key_cols) if pa.types.is_string(table.column(c).type) or pa.types.is_binary(table.column(c).type)]
    enc, _ = encode_string_columns(table, str_cols) if str_cols else (table, {})
    sort_orders = [(c, True, True) for c in partition_cols] + list(orders)
    n = table.num_rows
    perm = sort_permutation(enc, sort_orders) if sort_orders and n else np.arange(n, dtype=np.int64)
    srt = take_table(table, perm)
    senc = take_table(enc, perm)
    pk = list(zip(*[[_norm_key(v) for v in senc.column(c).to_pylist()] for c in partition_cols])) if partition_cols else [()] * n
    ok = list(zip(*[[_norm_key(v) for v in senc.column(o[0]).to_pylist()] for o in orders])) if orders else [()] * n
    seg_start, seg_end, peer_start, peer_end = [0] * n, [0] * n, [0] * n, [0] * n
    i = 0
    while i < n:
        j = i
        while j < n and pk[j] == pk[i]:
            j += 1
        a = i
        while a < j:
            b = a
            while b < j and ok[b] == ok[a]:
                b += 1
            for r in range(a, b):
                seg_start[r], seg_end[r], peer_start[r], peer_end[r] = i, j, a, b
            a = b
        i = j
    okey_vals = None
    if len(orders) == 1:
        okey_vals = srt.column(orders[0][0]).to_pylist()
        if okey_vals and not isinstance(next((v for v in okey_vals if v is not None), 0), (int, float)):
            okey_vals = [None if v is None else (v.toordinal() - 719163) for v in okey_vals] if pa.types.is_date(srt.column(orders[0][0]).type) else None
    return srt, seg_start, seg_end, peer_start, peer_end, okey_vals


def _frame_bounds(frame, orders, okey_vals, s, e, peer_start, peer_end, r):
    """[lo, hi] (sorted rows, empty when lo > hi) of row r's frame in the partition [s, e)."""
    kind, lower, upper = frame
    if kind != "range":
        return (s if lower is None else max(s, r + lower)), (e - 1 if upper is None else min(e - 1, r + upper))
    # RANGE: UNBOUNDED -> partition end, CURRENT ROW (0) -> peer group end, else a VALUE offset over the single ORDER BY key:
    # bound = key + offset for ASC, key - offset for DESC (WindowEvaluatorFactoryBase.createBoundOrdering); the frame is
    # the rows whose keys lie between the bounds in the sort order; a NULL key has only its peers (RangeBoundOrdering)
    ov = okey_vals[r] if okey_vals is not None else None
    asc, nf = (orders[0][1], orders[0][2]) if orders else (True, True)

    def side(q, bound):     # -1 the key of row q sorts before the bound, 0 equal, +1 after
        k = okey_vals[q]
        if k is None:
            return -1 if nf else 1
        c = int(_dcmp(float(k), float(bound))) if isinstance(k, float) or isinstance(bound, float) else (k > bound) - (k < bound)
        return c if asc else -c

    def first(pred):        # first position in [s, e) where pred holds (pred is monotone over the sorted partition)
        a, b = s, e
        while a < b:
            m = (a + b) // 2
            if pred(m):
                b = m
            else:
                a = m + 1
        return a

    if lower is None:
        lo = s
    elif lower == 0 or ov is None:
        lo = peer_start[r]
    else:
        bl = ov + lower if asc else ov - lower
        lo = first(lambda q: side(q, bl) >= 0)
    if upper is None:
        hi = e - 1
    elif upper == 0 or ov is None:
        hi = peer_end[r] - 1
    else:
        bu = ov + upper if asc else ov - upper
        hi = first(lambda q: side(q, bu) > 0) - 1
    return lo, hi


def _default_frame(frame, orders):
    """SpecifiedWindowFrame.defaultWindowFrame (windowExpressions.scala): RANGE UNBOUNDED PRECEDING..CURRENT ROW with an ORDER BY,
    the whole partition without."""
    if frame is not None:
        return frame
    return ("range", None, 0) if orders else ("rows", None, None)


def window_frames(table, partition_cols, orders, spec):
    """[(lo, hi)] of every output row of window(table, partition_cols, orders, [spec]), as positions in its sorted order (empty
    frame when lo > hi).  spec is one of window()'s spec tuples; only its frame is read."""
    _, seg_start, seg_end, peer_start, peer_end, okey_vals = _window_layout(table, partition_cols, orders)
    frame = _default_frame(spec[2], orders)
    return [_frame_bounds(frame, orders, okey_vals, seg_start[r], seg_end[r], peer_start, peer_end, r) for r in range(len(seg_start))]


def window(table, partition_cols, orders, specs):
    """WindowExec (sql/core/.../window/WindowExec.scala:90-110 + WindowEvaluatorFactoryBase + WindowFunctionFrame.scala), one
    partition at a time, the way the reference's frame classes walk it: growing frames accumulate as their upper bound moves,
    shrinking frames are accumulated from the partition's end, sliding frames are re-evaluated over their rows.
    orders: [(col, ascending, nulls_first)]; specs: [(func, col, (kind, lower, upper) | None, param, out_name)] with kind 'rows' |
    'range', None bound = UNBOUNDED, 0 = CURRENT ROW, negative = PRECEDING (rows).  Default frame: _default_frame.
    Output: rows sorted by partition keys (ASC NULLS FIRST) ++ orders, plus one column per spec."""
    srt, seg_start, seg_end, peer_start, peer_end, okey_vals = _window_layout(table, partition_cols, orders)
    n = table.num_rows
    out = {name: srt.column(name) for name in srt.column_names}
    seg_bounds = []
    i = 0
    while i < n:
        seg_bounds.append((i, seg_end[i]))
        i = seg_end[i]

    def better(func, x, y):   # is y a better min / max than x?  doubles order like SQLOrderingUtil.compareDoubles
        c = int(_dcmp(y, x)) if isinstance(x, float) else (y > x) - (y < x)
        return c < 0 if func == "min" else c > 0

    for func, col, frame, param, name in specs:
        vals = srt.column(col).to_pylist() if col is not None else None
        frame = _default_frame(frame, orders)
        kind, lower, upper = frame
        res = [None] * n
        for s, e in seg_bounds:
            size = e - s
            if func in ("row_number", "rank", "dense_rank", "percent_rank", "cume_dist", "ntile"):
                dense = 0
                bs, pad = (size // param, size % param) if func == "ntile" else (0, 0)
                row_number = bucket = threshold = 0                       # NTile state (windowExpressions.scala NTile)
                for r in range(s, e):
                    rank = peer_start[r] - s + 1
                    if peer_start[r] == r:
                        dense += 1                                        # DenseRank: +1 at every change of the order key
                    if func == "row_number":
                        res[r] = r - s + 1
                    elif func == "rank":
                        res[r] = rank
                    elif func == "dense_rank":
                        res[r] = dense
                    elif func == "percent_rank":                          # (rank - 1) / (n - 1), 0.0 for a single row
                        res[r] = (rank - 1) / (size - 1) if size > 1 else 0.0
                    elif func == "cume_dist":                             # rows up to and including the peers / n
                        res[r] = (peer_end[r] - s) / size
                    else:
                        over = row_number >= threshold
                        nb = bucket + (1 if over else 0)
                        threshold = threshold + ((bs + (1 if bucket < pad else 0)) if over else 0)
                        bucket = nb
                        row_number += 1
                        res[r] = bucket
                continue
            if func in ("lag", "lead"):                                   # FrameLessOffsetWindowFunctionFrame: NULL outside the partition
                for r in range(s, e):
                    q = r - param if func == "lag" else r + param
                    res[r] = vals[q] if s <= q < e else None
                continue

            def bounds(r):
                return _frame_bounds(frame, orders, okey_vals, s, e, peer_start, peer_end, r)

            if func in ("first_value", "last_value"):
                for r in range(s, e):
                    lo, hi = bounds(r)
                    res[r] = None if lo > hi else vals[lo if func == "first_value" else hi]
                continue

            def finish(acc_sum, acc_cnt, acc_best):
                if func == "count":
                    return acc_cnt
                if func == "sum":
                    return None if acc_cnt == 0 else (float(acc_sum) if is_f else _wrap64(acc_sum))
                if func == "avg":
                    return None if acc_cnt == 0 else acc_sum / acc_cnt
                return acc_best

            is_f = pa.types.is_floating(srt.column(col).type)
            zero = 0.0 if (is_f or func == "avg") else 0
            conv = (lambda x: float(x)) if (is_f or func == "avg") else (lambda x: x)

            def fold(rows_iter, acc):
                sm, cnt, best = acc
                for q in rows_iter:
                    x = vals[q]
                    if x is None:
                        continue
                    sm += conv(x)
                    cnt += 1
                    if func in ("min", "max") and (best is None or better(func, best, x)):
                        best = x
                return sm, cnt, best

            if lower is None:            # growing frame (UnboundedPrecedingWindowFunctionFrame): rows are added as the upper bound moves
                acc, nxt = (zero, 0, None), s
                for r in range(s, e):
                    lo, hi = bounds(r)
                    acc = fold(range(nxt, hi + 1), acc)
                    nxt = max(nxt, hi + 1)
                    res[r] = finish(*acc)
            elif upper is None:          # shrinking frame (UnboundedFollowingWindowFunctionFrame), accumulated from the partition's end
                acc, nxt = (zero, 0, None), e - 1
                for r in range(e - 1, s - 1, -1):
                    lo, hi = bounds(r)
                    acc = fold(range(nxt, lo - 1, -1), acc)
                    nxt = min(nxt, lo - 1)
                    res[r] = finish(*acc)
            else:                        # sliding frame (SlidingWindowFunctionFrame): re-evaluated over its rows
                for r in range(s, e):
                    lo, hi = bounds(r)
                    res[r] = finish(*fold(range(lo, hi + 1), (zero, 0, None)))
        if func in ("row_number", "rank", "dense_rank", "ntile"):
            out[name] = pa.array(res, type=pa.int32())
        elif func in ("percent_rank", "cume_dist", "avg"):
            out[name] = pa.array(res, type=pa.float64())
        elif func == "count":
            out[name] = pa.array(res, type=pa.int64())
        elif func == "sum":
            t = srt.column(col).type
            out[name] = pa.array(res, type=pa.float64() if pa.types.is_floating(t) else pa.int64())
        else:
            out[name] = pa.array(res, type=srt.column(col).type)
    return pa.table(out)


def _wrap64(x):
    x &= (1 << 64) - 1
    return x - (1 << 64) if x >= (1 << 63) else x


# --------------------------------------------------------------------------- decimal SUM / AVG (exact integer arithmetic)
def decimal_aggregate(table, key_cols, aggs):
    """Sum / Average over DecimalType columns, Complete mode (Sum.scala:80-178, Average.scala:80-135, non-ANSI):
      sum(decimal(p, s)) : decimal(min(p + 10, 38), s); NULL when no non-NULL input; NULL when |sum| >= 10^precision
      avg(decimal(p, s)) : decimal(min(p + 4, 38), s + 4) = sum / count rounded HALF_UP (Decimal./ rounds to 39 digits first, which
                           cannot move the second rounding for a count below 2^63); NULL when no non-NULL input or on overflow
    aggs = [(func, column, out_name)] with func in sum | avg | count | min | max (the last three: same type / bigint).
    Groups by key_cols (non-decimal keys) with the oracle's grouping; arithmetic on Python integers."""
    import decimal as D
    gid, first, ng = _group(table, key_cols)
    out = {k: take_table(table.select([k]), first).column(0) for k in key_cols}
    for func, col, name in aggs:
        arr = table.column(col)
        t = arr.type
        vals = arr.to_pylist()
        if pa.types.is_decimal(t):
            p, s = t.precision, t.scale
            unscaled = [None if v is None else int(v.scaleb(s)) for v in vals]
        else:
            p = s = None
            unscaled = vals
        sums, cnts, mins, maxs = [0] * ng, [0] * ng, [None] * ng, [None] * ng
        for g, v in zip(gid.tolist(), unscaled):
            if v is None:
                continue
            sums[g] += v
            cnts[g] += 1
            mins[g] = v if mins[g] is None or v < mins[g] else mins[g]
            maxs[g] = v if maxs[g] is None or v > maxs[g] else maxs[g]
        if func == "count":
            out[name] = pa.array(cnts, type=pa.int64())
            continue
        if func in ("min", "max"):
            src = mins if func == "min" else maxs
            out[name] = pa.array([None if v is None else D.Decimal(v).scaleb(-s) for v in src], type=t) if p else pa.array(src, type=t)
            continue
        assert p is not None, "decimal_aggregate: sum / avg take decimal columns"
        with D.localcontext() as ctx:
            ctx.prec = 80
            if func == "sum":
                rp = min(p + 10, 38)
                res = [None if c == 0 or abs(x) >= 10 ** rp else D.Decimal(x).scaleb(-s) for x, c in zip(sums, cnts)]
                out[name] = pa.array(res, type=pa.decimal128(rp, s))
            else:
                rp, rs = min(p + 4, 38), s + 4
                res = []
                for x, c in zip(sums, cnts):
                    if c == 0:
                        res.append(None)
                        continue
                    num, den = abs(x) * 10 ** 4, c
                    q, r = divmod(num, den)
                    if 2 * r >= den:
                        q += 1
                    q = -q if x < 0 else q
                    res.append(None if abs(q) >= 10 ** rp else D.Decimal(q).scaleb(-rs))
                out[name] = pa.array(res, type=pa.decimal128(rp, rs))
    return pa.table(out)
