"""SparkPlan operator mirrors that run on the GPU through the C ABI.

Each class has the name, constructor shape and `executeColumnar()` contract of the reference operator it
replaces (SQLX = sql/core/src/main/scala/org/apache/spark/sql/execution):

  FilterExec / ProjectExec           SQLX/basicPhysicalOperators.scala:245 / :47
  HashAggregateExec                  SQLX/aggregate/HashAggregateExec.scala:50
  ShuffleExchangeExec                SQLX/exchange/ShuffleExchangeExec.scala:190
  SortExec                           SQLX/SortExec.scala:39
  TakeOrderedAndProjectExec          SQLX/limit.scala:310
  BroadcastHashJoinExec              SQLX/joins/BroadcastHashJoinExec.scala:40
  SortMergeJoinExec                  SQLX/joins/SortMergeJoinExec.scala:39   (same multiset, hash build/probe)
  B200ColumnarRule                   a ColumnarRule (SQLX/Columnar.scala:47-50): preColumnarTransitions collapses
                                     Filter/Project into the consuming HashAggregateExec, like WholeStageCodegen

In a Spark deployment these bodies live in the Scala plugin (scala/, INTEGRATION.md) and call the same sb_*
functions through JNI; this module is the binding used by the tests and bench.py.  One "partition" here is
one ColumnarBatch on one GPU.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _capi as capi
from .columnar import ColumnarBatch, Stream, _h
from .expressions import (AggregateFunction, AttributeReference, CompiledExpr, CompiledStringProgram, Expression, Schema, SortOrder,
                          StringFunction)


def _binary_names(names, arrow_types):
    import pyarrow as pa
    return {n for n, t in zip(names, arrow_types) if t is not None and (pa.types.is_binary(t) or pa.types.is_large_binary(t))}


def _schema_of(batch: ColumnarBatch) -> Schema:
    return Schema(batch.names, [batch.column_desc(i).type for i in range(len(batch.names))], _binary_names(batch.names, batch.arrow_types))


class SparkPlan:
    children = ()

    def executeColumnar(self, stream: Stream = None) -> ColumnarBatch:
        raise NotImplementedError

    # the reference's public entry point is execute*/collect; to_arrow is ColumnarToRowExec + collect
    def collect(self, stream=None):
        b = self.executeColumnar(stream)
        try:
            return b.to_arrow(stream)
        finally:
            b.close()


class LocalTableScanExec(SparkPlan):
    """Leaf that hands out an existing HBM batch (the scan/RowToColumnar boundary)."""

    def __init__(self, batch: ColumnarBatch):
        self.batch = batch

    def executeColumnar(self, stream=None):
        return self.batch.rename(self.batch.names)


class FilterExec(SparkPlan):
    def __init__(self, condition: Expression, child: SparkPlan):
        self.condition = condition
        self.child = child
        self.children = (child,)

    def executeColumnar(self, stream=None):
        inp = self.child.executeColumnar(stream)
        try:
            return _filter_project(inp, self.condition, [(n, AttributeReference(n)) for n in inp.names], stream)
        finally:
            inp.close()


class ProjectExec(SparkPlan):
    def __init__(self, projectList, child: SparkPlan):
        """projectList: [(name, Expression)] (Alias(expr, name)) or bare attribute names."""
        self.projectList = [(p, AttributeReference(p)) if isinstance(p, str) else p for p in projectList]
        self.child = child
        self.children = (child,)

    def executeColumnar(self, stream=None):
        # Project over Filter is one stage in the reference (whole-stage codegen fuses them, WholeStageCodegenExec.scala);
        # here it is one native call: only the projected columns of the surviving rows are ever materialised
        cond = None
        child = self.child
        if isinstance(child, FilterExec):
            cond, child = child.condition, child.child
        if cond is None and isinstance(child, BroadcastHashJoinExec) and child.condition is None:
            # ColumnPruning (sql/catalyst/.../optimizer/Optimizer.scala, object ColumnPruning) would have put this projection below the
            # join as well: the join materialises only the attributes somebody above it reads
            child.requiredOutput = {a for _, e in self.projectList for a in e.references()}
        inp = child.executeColumnar(stream)
        try:
            return _filter_project(inp, cond, self.projectList, stream)
        finally:
            inp.close()


def _filter_project(inp: ColumnarBatch, condition, project_list, stream) -> ColumnarBatch:
    if _has_string_function(condition) or any(_has_string_function(e) for _, e in project_list):
        return _filter_project_strings(inp, condition, project_list, stream)
    return _filter_project_native(inp, condition, project_list, stream)


def _has_string_function(e) -> bool:
    return e is not None and (isinstance(e, StringFunction) or any(_has_string_function(c) for c in e.children))


def _hoist_string_functions(e: Expression, hidden):
    """`e` with every string function that is an operand of a numeric or boolean node replaced by a hidden column; (name,
    function) pairs are appended to `hidden`."""
    import copy
    if isinstance(e, StringFunction):
        name = "\0sf%d" % len(hidden)
        hidden.append((name, e))
        return AttributeReference(name)
    if not _has_string_function(e):
        return e
    e2 = copy.copy(e)
    for attr in ("left", "right", "child"):
        if hasattr(e2, attr):
            setattr(e2, attr, _hoist_string_functions(getattr(e2, attr), hidden))
    if hasattr(e2, "left"):
        e2.children = (e2.left, e2.right)
    elif hasattr(e2, "child"):
        e2.children = (e2.child,)
    return e2


def _string_project(inp: ColumnarBatch, items, stream) -> ColumnarBatch:
    """sb_string_project: one string column per (name, string function) of `items`, over every row of `inp`."""
    import pyarrow as pa
    schema = _schema_of(inp)
    for _, e in items:
        for a in e.references():
            if a in schema.binary:
                raise capi.SparkB200Error(5, "string functions over the binary column %r are not supported on the GPU" % a)
    progs = [CompiledStringProgram(e, schema) for _, e in items]
    arr = (capi.sb_expr * max(1, len(progs)))()
    for i, p in enumerate(progs):
        arr[i] = p.c
    h = C.c_void_p()
    capi.check(capi.load().sb_string_project(inp.handle, arr, len(progs), _h(stream), C.byref(h)))
    return ColumnarBatch(h, [n for n, _ in items], [pa.string()] * len(items))


def _with_hidden(inp: ColumnarBatch, hidden, stream) -> ColumnarBatch:
    """inp ++ the hidden string columns (a new reference to inp when there are none)."""
    if not hidden:
        return inp.rename(inp.names)
    h = _string_project(inp, hidden, stream)
    try:
        return inp.zip(h)
    finally:
        h.close()


def _filter_project_strings(inp: ColumnarBatch, condition, project_list, stream) -> ColumnarBatch:
    """Filter + projection when string functions take part.  A string function inside the condition is materialised as a hidden
    column over all rows, the condition runs over inp ++ hidden, and the hidden columns are dropped with the rows.  The projections
    then run over the surviving rows only: string-valued outputs through sb_string_project, the rest through sb_filter_project (a
    string function inside them hoisted the same way), joined with sb_table_zip in the projection's order."""
    cur = inp.rename(inp.names)
    try:
        if condition is not None:
            hidden = []
            cond = _hoist_string_functions(condition, hidden)
            wide = _with_hidden(cur, hidden, stream)
            try:
                kept = _filter_project_native(wide, cond, [(n, AttributeReference(n)) for n in inp.names], stream)
            finally:
                wide.close()
            cur.close()
            cur = kept
        if not project_list:
            return _filter_project_native(cur, None, [], stream)
        strings = [(i, n, e) for i, (n, e) in enumerate(project_list) if isinstance(e, StringFunction)]
        others = [(i, n, e) for i, (n, e) in enumerate(project_list) if not isinstance(e, StringFunction)]
        parts = []
        try:
            if others:
                hidden = []
                exprs = [("\0p%d" % i, _hoist_string_functions(e, hidden)) for i, _, e in others]
                wide = _with_hidden(cur, hidden, stream)
                try:
                    parts.append(_filter_project_native(wide, None, exprs, stream))
                finally:
                    wide.close()
            if strings:
                parts.append(_string_project(cur, [("\0p%d" % i, e) for i, _, e in strings], stream))
            out = parts[0] if len(parts) == 1 else parts[0].zip(parts[1])
            if len(parts) == 2:
                parts[0].close()
                parts[1].close()
            parts = [out]
            sel = out.select(["\0p%d" % i for i in range(len(project_list))])
            try:
                return sel.rename([n for n, _ in project_list])
            finally:
                sel.close()
        finally:
            for b in parts:
                b.close()
    finally:
        cur.close()


def _filter_project_native(inp: ColumnarBatch, condition, project_list, stream) -> ColumnarBatch:
    lib = capi.load()
    schema = _schema_of(inp)
    pred = CompiledExpr(condition, schema) if condition is not None else None
    projs = [CompiledExpr(e, schema) for _, e in project_list]
    arr = (capi.sb_expr * max(1, len(projs)))()
    for i, p in enumerate(projs):
        arr[i] = p.c
    h = C.c_void_p()
    capi.check(lib.sb_filter_project(inp.handle, C.byref(pred.c) if pred else None, arr, len(projs), _h(stream), C.byref(h)))
    ats = []
    for _, e in project_list:
        ats.append(inp.arrow_types[schema.index(e.name)] if isinstance(e, AttributeReference) else None)
    return ColumnarBatch(h, [n for n, _ in project_list], ats)


class HashAggregateExec(SparkPlan):
    """groupingExpressions: attribute names; aggregateExpressions: [(AggregateFunction, result_name)];
    mode: 'partial' | 'final' | 'complete'.  `condition` / expression inputs are the fused child
    FilterExec / ProjectExec (set by B200ColumnarRule or directly)."""

    def __init__(self, groupingExpressions, aggregateExpressions, child: SparkPlan, mode="complete", condition=None,
                 expected_groups=0):
        self.groupingExpressions = list(groupingExpressions)
        self.aggregateExpressions = list(aggregateExpressions)
        self.child = child
        self.children = (child,)
        self.mode = mode
        self.condition = condition
        self.expected_groups = expected_groups

    def output_names(self, schema=None):
        """keys ++ buffers (partial) or results.  A decimal SUM carries Spark's (sum, isEmpty) buffer (Sum.scala:91-100): in
        update modes that is known from the input column's type, in the merge modes from the Partial table's own columns."""
        names = list(self.groupingExpressions)
        pos = len(names)
        for fn, name in self.aggregateExpressions:
            dec = False
            if schema is not None and fn.func in ("sum", "avg"):
                if self.mode in ("final", "partial_merge"):
                    dec = pos < len(schema.types) and schema.types[pos] in (capi.SB_DECIMAL64, capi.SB_DECIMAL128)
                else:
                    dec = isinstance(fn.child, AttributeReference) and schema.types[schema.index(fn.child.name)] in (capi.SB_DECIMAL64, capi.SB_DECIMAL128)
            moment = fn.func in ("var_pop", "var_samp", "stddev_pop", "stddev_samp")
            pos += 2 if (fn.func == "avg" or (dec and fn.func == "sum")) else (3 if moment else 1)
            if self.mode in ("partial", "partial_merge"):
                bufs = [name + "#n", name + "#avg", name + "#m2"] if moment else {
                    "sum": [name + "#sum"], "avg": [name + "#sum", name + "#count"], "count": [name + "#count"],
                    "count_star": [name + "#count"], "min": [name + "#val"], "max": [name + "#val"]}[fn.func]
                if dec and fn.func == "sum":
                    bufs = [name + "#sum", name + "#isEmpty"]
                names += bufs
            else:
                names.append(name)
        return names

    def executeColumnar(self, stream=None):
        if isinstance(self.child, BroadcastHashJoinExec) and self.child.condition is None and self.mode not in ("final", "partial_merge"):
            # ColumnPruning: the join below materialises only what the aggregate reads
            need = set(self.groupingExpressions)
            for fn, _ in self.aggregateExpressions:
                if fn.child is not None:
                    need |= fn.child.references()
            if self.condition is not None:
                need |= self.condition.references()
            self.child.requiredOutput = need
        inp = self.child.executeColumnar(stream)
        try:
            return self.run(inp, stream)
        finally:
            inp.close()

    def _compile(self, schema: Schema):
        """Lower the plan to the C structs once per input schema (the Scala operator does this in doPrepare)."""
        keep = []
        key_idx = [schema.index(k) for k in self.groupingExpressions]
        key_arr = (C.c_int32 * max(1, len(key_idx)))(*key_idx)
        specs = (capi.sb_agg_spec * max(1, len(self.aggregateExpressions)))()
        for i, (fn, _name) in enumerate(self.aggregateExpressions):
            specs[i].func = capi.SB_AGG[fn.func]
            if not getattr(fn, "null_on_divide_by_zero", True):
                specs[i].flags = capi.SB_AGG_FLAG_NAN_ON_DIVIDE_BY_ZERO
            if self.mode not in ("final", "partial_merge") and fn.child is not None:   # merge modes read buffers positionally
                ce = CompiledExpr(fn.child, schema)
                keep.append(ce)
                specs[i].input = ce.c
        plan = capi.sb_agg_plan()
        plan.mode = capi.SB_AGG_MODE[self.mode]
        plan.nkeys = len(key_idx)
        plan.key_cols = C.cast(key_arr, C.POINTER(C.c_int32))
        plan.naggs = len(self.aggregateExpressions)
        plan.aggs = C.cast(specs, C.POINTER(capi.sb_agg_spec))
        if self.condition is not None:
            fc = CompiledExpr(self.condition, schema)
            keep.append(fc)
            plan.filter = C.pointer(fc.c)
        plan.expected_groups = self.expected_groups
        return plan, key_idx, (keep, key_arr, specs)

    def new_state(self, first_batch: ColumnarBatch) -> "AggregationState":
        return AggregationState(self, _schema_of(first_batch), first_batch.arrow_types)

    def execute_batches(self, batches, stream=None) -> ColumnarBatch:
        """doExecuteColumnar over an iterator of batches: every batch is folded into one state and closed."""
        state = None
        try:
            for b in batches:
                if state is None:
                    state = self.new_state(b)
                state.update(b, stream)
                b.close()
            if state is None:
                raise capi.SparkB200Error(2, "execute_batches needs at least one (possibly empty) batch")
            return state.finish(stream)
        finally:
            if state is not None:
                state.close()

    def run(self, inp: ColumnarBatch, stream=None) -> ColumnarBatch:
        lib = capi.load()
        schema = _schema_of(inp)
        sig = (tuple(schema.names), tuple(schema.types))
        cache = self.__dict__.setdefault("_compiled", {})
        if sig not in cache:
            cache[sig] = self._compile(schema)
        plan, key_idx, _keepalive = cache[sig]
        h = C.c_void_p()
        capi.check(lib.sb_hash_aggregate(inp.handle, C.byref(plan), _h(stream), C.byref(h)))
        names = self.output_names(schema)
        ats = [inp.arrow_types[i] for i in key_idx] + [None] * (len(names) - len(key_idx))
        return ColumnarBatch(h, names, ats)


class AggregationState:
    """The aggregation map a task keeps while it drains its iterator of batches
    (TungstenAggregationIterator.processInputs, TungstenAggregationIterator.scala:206-281): sb_hash_agg_* state.
    `update` folds one ColumnarBatch in and the batch can be closed right away; `finish` returns what the
    operator's mode promises (partial: keys ++ buffers, complete / final: keys ++ results)."""

    def __init__(self, agg: "HashAggregateExec", schema: Schema, arrow_types=None):
        lib = capi.load()
        self.agg = agg
        self.plan, self.key_idx, self._keepalive = agg._compile(schema)
        self.schema = schema
        self.arrow_types = arrow_types
        h = C.c_void_p()
        capi.check(lib.sb_hash_agg_create(C.byref(self.plan), C.byref(h)))
        self.handle = h

    def update(self, batch: ColumnarBatch, stream=None):
        capi.check(capi.load().sb_hash_agg_update(self.handle, batch.handle, _h(stream)))

    def merge(self, partial: ColumnarBatch, stream=None):
        capi.check(capi.load().sb_hash_agg_merge(self.handle, partial.handle, _h(stream)))

    def finish(self, stream=None) -> ColumnarBatch:
        h = C.c_void_p()
        capi.check(capi.load().sb_hash_agg_finish(self.handle, _h(stream), C.byref(h)))
        names = self.agg.output_names(self.schema)
        ats = [self.arrow_types[i] if self.arrow_types else None for i in self.key_idx] + [None] * (len(names) - len(self.key_idx))
        return ColumnarBatch(h, names, ats)

    def close(self):
        if self.handle:
            capi.load().sb_hash_agg_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class HashPartitioning:
    def __init__(self, expressions, numPartitions):
        self.expressions = list(expressions)
        self.numPartitions = numPartitions


class RoundRobinPartitioning:
    def __init__(self, numPartitions, start=0):
        self.numPartitions = numPartitions
        self.start = start   # XORShiftRandom(mapPartitionId).nextInt(n) in the reference: parity unpinned


class SinglePartition:
    numPartitions = 1


class RangePartitioning:
    """RangePartitioning(ordering, numPartitions) with explicit range bounds (a one-column ColumnarBatch holding the
    numPartitions - 1 sorted bounds; in Spark the RangePartitioner samples them on the JVM side)."""

    def __init__(self, ordering, bounds: ColumnarBatch):
        self.ordering = ordering if isinstance(ordering, SortOrder) else SortOrder(*ordering)
        self.bounds = bounds
        self.numPartitions = bounds.num_rows + 1


def range_bounds(batch: ColumnarBatch, ordering, numPartitions: int, stream=None, samplePointsPerPartitionHint: int = 100,
                 inputPartitions: int = None, seed: int = 0) -> ColumnarBatch:
    """RangePartitioner's bounds for a global sort (Partitioner.scala:203-236; ShuffleExchangeExec.scala:381-401 uses
    spark.sql.execution.rangeExchange.sampleSizePerPartition = 100): sample this rank's batch, all-gather the candidates when a
    communicator is up, determineBounds.  Returns the one-column bounds batch RangePartitioning takes."""
    import math
    lib = capi.load()
    ordering = ordering if isinstance(ordering, SortOrder) else SortOrder(*ordering)
    rank, world = C.c_int32(), C.c_int32()
    capi.check(lib.sb_comm_rank(C.byref(rank), C.byref(world)))
    nin = inputPartitions or max(1, world.value)
    sample_size = min(float(samplePointsPerPartitionHint) * numPartitions, 1e6)
    per_partition = int(math.ceil(3.0 * sample_size / nin))
    orders = _orders_c(batch, [ordering])
    h = C.c_void_p()
    capi.check(lib.sb_range_sample(batch.handle, orders, per_partition, seed + rank.value, _h(stream), C.byref(h)))
    sample = ColumnarBatch(h, [ordering.child, "weight"], [batch.arrow_types[batch.column_index(ordering.child)], None])
    try:
        if world.value > 1:
            g = C.c_void_p()
            capi.check(lib.sb_all_gather(sample.handle, _h(stream), C.byref(g)))
            sample.close()
            sample = ColumnarBatch(g, [ordering.child, "weight"], sample.arrow_types)
        o2 = (capi.sb_sort_order * 1)()
        o2[0].col, o2[0].ascending, o2[0].nulls_first = 0, int(ordering.ascending), int(ordering.nulls_first)
        b = C.c_void_p()
        capi.check(lib.sb_range_determine_bounds(sample.handle, o2, numPartitions, _h(stream), C.byref(b)))
        return ColumnarBatch(b, [ordering.child], [sample.arrow_types[0]])
    finally:
        sample.close()


class ShuffleExchangeExec(SparkPlan):
    """Map side always runs on the local GPU (partition ids + regrouping).  With a communicator
    (sb_comm_init done, world size > 1) the buckets are exchanged with the NCCL all-to-all and the
    result holds the partitions this rank owns (contiguous ownership: rank r owns partitions [ceil(r n / R), ceil((r + 1) n / R)),
    sb_exchange_plan), partition-contiguous."""

    def __init__(self, outputPartitioning, child: SparkPlan, fused=None):
        self.outputPartitioning = outputPartitioning
        self.child = child
        self.children = (child,)
        self.partition_offsets = None
        # fused: map side and transport in one call (sb_shuffle_exchange: the multisplit's stores go straight into the owners'
        # receive windows over NVLink).  None = whenever more than one rank is up and the partitioning is a hash partitioning.
        self.fused = fused

    def executeColumnar(self, stream=None):
        inp = self.child.executeColumnar(stream)
        try:
            return self.run(inp, stream)
        finally:
            inp.close()

    def map_side(self, inp: ColumnarBatch, stream=None):
        lib = capi.load()
        p = self.outputPartitioning
        n = p.numPartitions
        offs = (C.c_int64 * (n + 1))()
        h = C.c_void_p()
        if isinstance(p, HashPartitioning):
            idx = [inp.column_index(k) for k in p.expressions]
            arr = (C.c_int32 * max(1, len(idx)))(*idx)
            capi.check(lib.sb_hash_partition(inp.handle, arr, len(idx), n, _h(stream), C.byref(h), offs))
        elif isinstance(p, RoundRobinPartitioning):
            capi.check(lib.sb_round_robin_partition(inp.handle, p.start, n, _h(stream), C.byref(h), offs))
        elif isinstance(p, RangePartitioning):
            capi.check(lib.sb_range_partition(inp.handle, _orders_c(inp, [p.ordering]), p.bounds.handle, _h(stream), C.byref(h), offs))
        else:
            capi.check(lib.sb_round_robin_partition(inp.handle, 0, 1, _h(stream), C.byref(h), offs))
        return ColumnarBatch(h, inp.names, inp.arrow_types), np.array(list(offs), dtype=np.int64)

    def run(self, inp: ColumnarBatch, stream=None) -> ColumnarBatch:
        lib = capi.load()
        rank, world = C.c_int32(), C.c_int32()
        capi.check(lib.sb_comm_rank(C.byref(rank), C.byref(world)))
        p = self.outputPartitioning
        if isinstance(p, HashPartitioning) and (self.fused or (self.fused is None and world.value > 1)):
            n = p.numPartitions
            idx = [inp.column_index(k) for k in p.expressions]
            arr = (C.c_int32 * max(1, len(idx)))(*idx)
            out_offs = (C.c_int64 * (n + 1))()
            h = C.c_void_p()
            capi.check(lib.sb_shuffle_exchange(inp.handle, arr, len(idx), n, _h(stream), C.byref(h), out_offs))
            self.partition_offsets = np.array(list(out_offs), dtype=np.int64)
            return ColumnarBatch(h, inp.names, inp.arrow_types)
        part, offs = self.map_side(inp, stream)
        if world.value <= 1:
            self.partition_offsets = offs
            return part
        try:
            n = self.outputPartitioning.numPartitions
            in_offs = (C.c_int64 * (n + 1))(*offs.tolist())
            out_offs = (C.c_int64 * (n + 1))()
            h = C.c_void_p()
            capi.check(lib.sb_all_to_all(part.handle, in_offs, n, _h(stream), C.byref(h), out_offs))
            self.partition_offsets = np.array(list(out_offs), dtype=np.int64)
            return ColumnarBatch(h, part.names, part.arrow_types)
        finally:
            part.close()

    # ---- ShuffleExchangeLike members AQE reads (ShuffleExchangeExec.scala:55-151, 235-262) --------------------------------------
    @property
    def numPartitions(self):
        return self.outputPartitioning.numPartitions

    def mapOutputStatistics(self, inp: ColumnarBatch, stream=None) -> np.ndarray:
        """MapOutputStatistics.bytesByPartitionId of this exchange for the given input: runs the map side and sums the
        partition sizes over all ranks (sb_map_output_statistics; collective when a communicator is up)."""
        lib = capi.load()
        part, offs = self.map_side(inp, stream)
        try:
            n = self.numPartitions
            in_offs = (C.c_int64 * (n + 1))(*offs.tolist())
            out = (C.c_int64 * n)()
            capi.check(lib.sb_map_output_statistics(part.handle, in_offs, n, _h(stream), out))
            return np.array(list(out), dtype=np.int64)
        finally:
            part.close()

    def partition_ids(self, inp: ColumnarBatch, stream=None) -> np.ndarray:
        """Partition id of every input row (for parity checks against Pmod(Murmur3Hash(keys), n))."""
        import torch
        lib = capi.load()
        p = self.outputPartitioning
        idx = [inp.column_index(k) for k in p.expressions]
        arr = (C.c_int32 * max(1, len(idx)))(*idx)
        out = torch.empty(max(inp.num_rows, 1), dtype=torch.int32, device="cuda")
        capi.check(lib.sb_partition_ids(inp.handle, arr, len(idx), p.numPartitions, _h(stream), C.c_void_p(out.data_ptr())))
        capi.check(lib.sb_stream_synchronize(_h(stream)))
        return out[: inp.num_rows].cpu().numpy()


class CoalescedPartitionSpec:
    """CoalescedPartitionSpec(startReducerIndex, endReducerIndex, dataSize) (SQLX/ShufflePartitionSpec... in ShuffledRowRDD.scala)."""

    def __init__(self, start, end, dataSize=None):
        self.startReducerIndex, self.endReducerIndex, self.dataSize = start, end, dataSize

    def __eq__(self, o):
        return (self.startReducerIndex, self.endReducerIndex, self.dataSize) == (o.startReducerIndex, o.endReducerIndex, o.dataSize)

    def __repr__(self):
        return "CoalescedPartitionSpec(%d, %d, %r)" % (self.startReducerIndex, self.endReducerIndex, self.dataSize)


def coalesce_shuffle_partitions(bytes_by_partition, advisoryTargetSize=64 << 20, minNumPartitions=1, minPartitionSize=1 << 20,
                                maxReducerPartitionsPerTask=2 ** 31 - 1):
    """CoalesceShufflePartitions (SQLX/adaptive/CoalesceShufflePartitions.scala) for one coalesce group: bytes_by_partition is one
    array per shuffle of the group.  Returns per shuffle a list of CoalescedPartitionSpec, or [] when the layout stays as it is.
    Defaults are the reference's: advisoryPartitionSizeInBytes 64 MB, coalescePartitions.minPartitionSize 1 MB."""
    lib = capi.load()
    arrs = [np.ascontiguousarray(b, dtype=np.int64) for b in bytes_by_partition]
    ns, npart = len(arrs), len(arrs[0]) if arrs else 0
    if ns == 0 or any(len(a) != npart for a in arrs):
        return []
    ptrs = (C.POINTER(C.c_int64) * ns)(*[a.ctypes.data_as(C.POINTER(C.c_int64)) for a in arrs])
    st, en = (C.c_int32 * max(1, npart))(), (C.c_int32 * max(1, npart))()
    sizes = (C.c_int64 * max(1, ns * npart))()
    n = C.c_int32()
    capi.check(lib.sb_coalesce_partitions(ptrs, ns, npart, advisoryTargetSize, minNumPartitions, minPartitionSize, maxReducerPartitionsPerTask,
                                          st, en, sizes, C.byref(n)))
    return [[CoalescedPartitionSpec(st[k], en[k], sizes[s * n.value + k]) for k in range(n.value)] for s in range(ns)] if n.value else []


class AQEShuffleReadExec(SparkPlan):
    """AQEShuffleReadExec over coalesced specs (SQLX/adaptive/AQEShuffleReadExec.scala:268-284): hands out the exchange's output
    as one batch per CoalescedPartitionSpec (a partition-contiguous exchange result makes every spec one row slice)."""

    def __init__(self, child: "ShuffleExchangeExec", partitionSpecs):
        self.child = child
        self.partitionSpecs = list(partitionSpecs)
        self.children = (child,)

    def batches(self, stream=None):
        out = self.child.executeColumnar(stream)
        try:
            offs = self.child.partition_offsets
            for spec in self.partitionSpecs:
                yield out.slice(int(offs[spec.startReducerIndex]), int(offs[spec.endReducerIndex]), stream)
        finally:
            out.close()

    def executeColumnar(self, stream=None):
        return self.child.executeColumnar(stream)


def _orders_c(batch: ColumnarBatch, sortOrder):
    arr = (capi.sb_sort_order * max(1, len(sortOrder)))()
    for i, o in enumerate(sortOrder):
        arr[i].col = batch.column_index(o.child)
        arr[i].ascending = int(o.ascending)
        arr[i].nulls_first = int(o.nulls_first)
    return arr


class SortExec(SparkPlan):
    def __init__(self, sortOrder, child: SparkPlan, global_=False):
        self.sortOrder = [o if isinstance(o, SortOrder) else SortOrder(*o) for o in sortOrder]
        self.child = child
        self.children = (child,)
        self.global_ = global_

    def executeColumnar(self, stream=None):
        inp = self.child.executeColumnar(stream)
        try:
            h = C.c_void_p()
            capi.check(capi.load().sb_sort(inp.handle, _orders_c(inp, self.sortOrder), len(self.sortOrder), _h(stream), C.byref(h)))
            return ColumnarBatch(h, inp.names, inp.arrow_types)
        finally:
            inp.close()


class TakeOrderedAndProjectExec(SparkPlan):
    def __init__(self, limit, sortOrder, projectList, child: SparkPlan):
        self.limit = limit
        self.sortOrder = [o if isinstance(o, SortOrder) else SortOrder(*o) for o in sortOrder]
        self.projectList = projectList
        self.child = child
        self.children = (child,)

    def executeColumnar(self, stream=None):
        inp = self.child.executeColumnar(stream)
        try:
            h = C.c_void_p()
            capi.check(capi.load().sb_top_n(inp.handle, _orders_c(inp, self.sortOrder), len(self.sortOrder), self.limit,
                                            _h(stream), C.byref(h)))
            top = ColumnarBatch(h, inp.names, inp.arrow_types)
            if self.projectList is None:
                return top
            try:
                return top.select(self.projectList)
            finally:
                top.close()
        finally:
            inp.close()


class HashedRelation:
    """Build side resident in HBM (HashedRelation.scala:136-168): sb_hash_table handle.  `condition` is the FilterExec below the
    build side fused into the build (rows failing it stay out of the relation; nothing is materialised); `out_names` the columns
    of the build batch that reach the join output (the ProjectExec below / above, fused)."""

    def __init__(self, batch: ColumnarBatch, keys, stream=None, condition=None, out_names=None):
        lib = capi.load()
        idx = [batch.column_index(k) for k in keys]
        arr = (C.c_int32 * max(1, len(idx)))(*idx)
        h = C.c_void_p()
        if condition is not None:
            ce = CompiledExpr(condition, _schema_of(batch))
            capi.check(lib.sb_join_build_filtered(batch.handle, arr, len(idx), C.byref(ce.c), _h(stream), C.byref(h)))
        else:
            capi.check(lib.sb_join_build(batch.handle, arr, len(idx), _h(stream), C.byref(h)))
        self.handle = h
        self.out_cols = None if out_names is None else [batch.column_index(n) for n in out_names]
        sel = range(len(batch.names)) if self.out_cols is None else self.out_cols
        self.names = [batch.names[i] for i in sel]
        self.arrow_types = [batch.arrow_types[i] for i in sel]
        self.types = [batch.column_desc(i).type for i in sel]

    def close(self):
        if self.handle:
            capi.load().sb_hash_table_release(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def _peel(plan):
    """(source, condition, names): `plan` seen as [ProjectExec of bare attributes] over [FilterExec] over source -- the part of
    the pipeline below a join that whole-stage codegen fuses into it on the CPU path (no rename, no computed column)."""
    names = cond = None
    if isinstance(plan, ProjectExec) and all(isinstance(e, AttributeReference) and e.name == n for n, e in plan.projectList):
        names = [n for n, _ in plan.projectList]
        plan = plan.child
    if isinstance(plan, FilterExec):
        cond = plan.condition
        plan = plan.child
    return plan, cond, names


_STREAM_LEFT = {"inner": "inner", "left_outer": "left_outer", "left_semi": "left_semi", "left_anti": "left_anti", "full_outer": "full_outer",
                "right_outer": "build_outer", "existence": "existence", "left_anti_null_aware": "left_anti_null_aware"}
_STREAM_RIGHT = {"inner": "inner", "right_outer": "left_outer", "left_outer": "build_outer", "full_outer": "full_outer"}


class ReusedExchangeExec(SparkPlan):
    """ReusedExchangeExec (SQLX/exchange/Exchange.scala:50-80): one subplan, several parents.  The child runs for the first parent that
    asks; the batch is shared with the other `uses - 1` and released after the last (the creation side of a runtime filter and the
    build side of the join it was derived from are the same broadcast)."""

    def __init__(self, child: SparkPlan, uses: int = 2):
        self.child, self.children, self.uses = child, (child,), uses
        self._batch, self._left = None, 0

    def executeColumnar(self, stream=None):
        if self._batch is None:
            self._batch, self._left = self.child.executeColumnar(stream), self.uses
        out = self._batch.rename(self._batch.names)      # a new handle over the same buffers
        self._left -= 1
        if self._left == 0:
            self._batch.close()
            self._batch = None
        return out


class RuntimeFilter:
    """What InjectRuntimeFilter (sql/catalyst/.../optimizer/InjectRuntimeFilter.scala:47-100) plans on the application side of a join:
    `applicationKey IN (creation side's creationKey)`, evaluated as a might-contain test.  Here the creation side becomes a single-key
    HashedRelation and its prefilter (exact bitmap or Bloom) is tested on the streamed column of the rows that survive the join's own
    candidate pass (short inputs: of every row)."""

    def __init__(self, applicationKey: str, creationKey: str, creationPlan: SparkPlan):
        self.applicationKey, self.creationKey, self.creationPlan = applicationKey, creationKey, creationPlan


class BroadcastHashJoinExec(SparkPlan):
    """leftKeys / rightKeys: attribute names; joinType: inner | left_outer | right_outer | full_outer | left_semi | left_anti |
    existence | left_anti_null_aware; buildSide: 'right' (left is streamed) or 'left'; condition: residual predicate over
    left ++ right attributes (HashJoin.boundCondition).  Output: left ++ right columns whatever the build side is
    (HashJoin.scala:55-70); existence: left columns ++ `exists`."""

    def __init__(self, leftKeys, rightKeys, joinType, buildSide, left: SparkPlan, right: SparkPlan, condition=None, runtimeFilters=None):
        self.runtimeFilters = list(runtimeFilters or [])    # on the STREAMED side (inner / left semi joins)
        self.requiredOutput = None                          # attribute names read above the join (set by the ProjectExec over it)
        self.leftKeys, self.rightKeys = list(leftKeys), list(rightKeys)
        table = _STREAM_LEFT if buildSide == "right" else _STREAM_RIGHT
        if buildSide not in ("left", "right") or joinType not in table:
            raise capi.SparkB200Error(5, "join type %r with buildSide=%r is not supported" % (joinType, buildSide))
        self.joinType, self.buildSide, self.condition = joinType, buildSide, condition
        self.native_type = table[joinType]
        self.left, self.right = left, right
        self.children = (left, right)

    def executeColumnar(self, stream=None):
        build_plan, stream_plan = (self.right, self.left) if self.buildSide == "right" else (self.left, self.right)
        build_keys, stream_keys = (self.rightKeys, self.leftKeys) if self.buildSide == "right" else (self.leftKeys, self.rightKeys)
        # Filter / Project directly below the join are fused into build and probe (nothing between scan and join output is
        # materialised); a residual condition keeps the children as they are
        fuse = self.condition is None and self.native_type not in ("existence", "left_anti_null_aware")
        b_src, b_cond, b_names = _peel(build_plan) if fuse else (build_plan, None, None)
        s_src, s_cond, s_names = _peel(stream_plan) if fuse else (stream_plan, None, None)
        need = self.requiredOutput if fuse else None
        build = b_src.executeColumnar(stream)
        try:
            if need is not None:
                b_all = b_names if b_names is not None else build.names
                b_names = [n for n in b_all if n in need] or b_all[:1]      # never a table without columns
            rel = HashedRelation(build, build_keys, stream, b_cond, b_names)
        finally:
            build.close()
        rf_rels = []
        try:
            for rf in self.runtimeFilters:
                cb = rf.creationPlan.executeColumnar(stream)
                try:
                    rf_rels.append((rf.applicationKey, HashedRelation(cb, [rf.creationKey], stream, None, [rf.creationKey])))
                finally:
                    cb.close()
            probe = s_src.executeColumnar(stream)
            try:
                if need is not None:
                    s_all = s_names if s_names is not None else probe.names
                    s_names = [n for n in s_all if n in need] or s_all[:1]
                out = probe_join(rel, probe, stream_keys, self.native_type, stream, self.condition, probe_filter=s_cond, probe_out=s_names,
                                 runtime_filters=rf_rels)
            finally:
                probe.close()
        finally:
            rel.close()
            for _, r in rf_rels:
                r.close()
        if self.buildSide == "left" and self.native_type in ("inner", "left_outer", "build_outer", "full_outer"):
            nl = len(rel.names)      # streamed ++ build came back: restore left ++ right
            order = list(range(len(out.names) - nl, len(out.names))) + list(range(len(out.names) - nl))
            arr = (C.c_int32 * len(order))(*order)
            h = C.c_void_p()
            try:
                capi.check(capi.load().sb_table_select(out.handle, arr, len(order), C.byref(h)))
                return ColumnarBatch(h, [out.names[i] for i in order], [out.arrow_types[i] for i in order])
            finally:
                out.close()
        return out


def probe_join(rel: HashedRelation, probe: ColumnarBatch, keys, joinType, stream=None, condition=None, probe_filter=None, probe_out=None,
               runtime_filters=None, **_ignored) -> ColumnarBatch:
    lib = capi.load()
    idx = [probe.column_index(k) for k in keys]
    arr = (C.c_int32 * max(1, len(idx)))(*idx)
    h = C.c_void_p()
    p_sel = list(range(len(probe.names))) if probe_out is None else [probe.column_index(n) for n in probe_out]
    p_names = [probe.names[i] for i in p_sel]
    p_types = [probe.arrow_types[i] for i in p_sel]
    if condition is not None:
        # the residual condition sees the joined row as the kernels lay it out: streamed columns ++ build columns
        schema = Schema(probe.names + rel.names, [probe.column_desc(i).type for i in range(len(probe.names))] + rel.types,
                        _binary_names(probe.names + rel.names, probe.arrow_types + rel.arrow_types))
        ce = CompiledExpr(condition, schema)
        capi.check(lib.sb_join_probe_condition(rel.handle, probe.handle, arr, len(idx), capi.SB_JOIN[joinType], C.byref(ce.c), _h(stream), C.byref(h)))
    elif probe_filter is not None or probe_out is not None or rel.out_cols is not None or runtime_filters:
        opt = capi.sb_join_options()
        keep = []
        if runtime_filters:
            rc_ = (C.c_int32 * len(runtime_filters))(*[probe.column_index(k) for k, _ in runtime_filters])
            rr_ = (C.c_void_p * len(runtime_filters))(*[r.handle for _, r in runtime_filters])
            keep += [rc_, rr_]
            opt.n_runtime_filters = len(runtime_filters)
            opt.runtime_filter_cols = C.cast(rc_, C.POINTER(C.c_int32))
            opt.runtime_filter_relations = C.cast(rr_, C.POINTER(C.c_void_p))
        if probe_filter is not None:
            fe = CompiledExpr(probe_filter, _schema_of(probe))
            keep.append(fe)
            opt.probe_filter = C.pointer(fe.c)
        if probe_out is not None:
            pa_ = (C.c_int32 * max(1, len(p_sel)))(*p_sel)
            keep.append(pa_)
            opt.probe_out_cols = C.cast(pa_, C.POINTER(C.c_int32))
            opt.n_probe_out = len(p_sel)
        if rel.out_cols is not None:
            ba_ = (C.c_int32 * max(1, len(rel.out_cols)))(*rel.out_cols)
            keep.append(ba_)
            opt.build_out_cols = C.cast(ba_, C.POINTER(C.c_int32))
            opt.n_build_out = len(rel.out_cols)
        capi.check(lib.sb_join_probe_ex(rel.handle, probe.handle, arr, len(idx), capi.SB_JOIN[joinType], C.byref(opt), _h(stream), C.byref(h)))
    else:
        capi.check(lib.sb_join_probe(rel.handle, probe.handle, arr, len(idx), capi.SB_JOIN[joinType], _h(stream), C.byref(h)))
    if joinType in ("left_semi", "left_anti", "left_anti_null_aware"):
        return ColumnarBatch(h, p_names, p_types)
    if joinType == "existence":
        import pyarrow as pa
        return ColumnarBatch(h, p_names + ["exists"], p_types + [pa.bool_()])
    return ColumnarBatch(h, p_names + rel.names, p_types + rel.arrow_types)


class ShuffledHashJoinExec(BroadcastHashJoinExec):
    """ShuffledHashJoinExec (SQLX/joins/ShuffledHashJoinExec.scala:38-130): the same build / probe over co-partitioned children;
    unlike the broadcast join it may preserve the build side (full outer, and outer joins that hash the preserved side)."""


class SortMergeJoinExec(BroadcastHashJoinExec):
    """The reference sorts both sides and merges (SortMergeJoinExec.scala:1213-1360); the GPU engine produces
    the same multiset with a hash build/probe and therefore does not report an outputOrdering."""

    def __init__(self, leftKeys, rightKeys, joinType, left, right, condition=None):
        super().__init__(leftKeys, rightKeys, joinType, "right", left, right, condition)


class B200ColumnarRule:
    """preColumnarTransitions: collapse Project/Filter chains under a HashAggregateExec into it (what
    CollapseCodegenStages + WholeStageCodegenExec do for the CPU path)."""

    def preColumnarTransitions(self, plan: SparkPlan) -> SparkPlan:
        for attr in ("child", "left", "right"):
            if hasattr(plan, attr):
                setattr(plan, attr, self.preColumnarTransitions(getattr(plan, attr)))
        if hasattr(plan, "child"):
            plan.children = (plan.child,)
        if isinstance(plan, HashAggregateExec) and plan.mode not in ("final", "partial_merge"):
            # Walk down the Project / Filter chain keeping ONE map from the names visible at the current level to expressions over
            # the level below (composed top-down: an upper alias is rewritten through every Project met beneath it), and the
            # conjunction of every Filter met so far rewritten the same way.  What is left at the bottom is expressed over the
            # source's attributes, which is what the fused kernel evaluates.
            child = plan.child
            agg_inputs = [fn.child for fn, _ in plan.aggregateExpressions]
            groups = {g: AttributeReference(g) for g in plan.groupingExpressions}
            cond = plan.condition
            changed = False
            while True:
                if isinstance(child, ProjectExec):
                    m = {n: e for n, e in child.projectList}
                    agg_inputs = [None if e is None else _substitute(e, m) for e in agg_inputs]
                    groups = {g: _substitute(e, m) for g, e in groups.items()}
                    if cond is not None:
                        cond = _substitute(cond, m)
                    child = child.child
                    changed = True
                elif isinstance(child, FilterExec):
                    cond = child.condition if cond is None else (cond & child.condition)
                    child = child.child
                    changed = True
                else:
                    break
            # grouping keys must still be plain attributes of the source under their own names (the native plan groups by input columns)
            group_ok = all(isinstance(e, AttributeReference) and e.name == g for g, e in groups.items())
            if changed and group_ok:
                aggs = [(fn if e is None else type(fn)(e), name) for (fn, name), e in zip(plan.aggregateExpressions, agg_inputs)]
                return HashAggregateExec(plan.groupingExpressions, aggs, child, plan.mode, cond, plan.expected_groups)
        return plan

    def postColumnarTransitions(self, plan: SparkPlan) -> SparkPlan:
        return plan

    # ---- runtime filters -------------------------------------------------------------------------------------------------------
    maxRuntimeFilters = 2      # per join; the reference caps the whole query (spark.sql.optimizer.runtimeFilter.number.threshold = 10)

    def injectRuntimeFilters(self, plan: SparkPlan) -> SparkPlan:
        """The physical-plan face of InjectRuntimeFilter (sql/catalyst/.../optimizer/InjectRuntimeFilter.scala:196-260, 411-460): for an
        inner join J2 whose streamed side is (Projects / Filters over) another inner or left-semi join J1, and whose build side has a
        selective predicate (a FilterExec somewhere below it), rows of J1's STREAMED input whose J2 key cannot be in J2's build side
        never reach the output -- so J1 tests that key against the relation's prefilter right after its candidate pass.  J2's build subplan
        becomes a ReusedExchangeExec shared by J2 and the filter's creation side."""
        for attr in ("child", "left", "right"):
            if hasattr(plan, attr):
                setattr(plan, attr, self.injectRuntimeFilters(getattr(plan, attr)))
        if hasattr(plan, "child"):
            plan.children = (plan.child,)
        elif hasattr(plan, "left"):
            plan.children = (plan.left, plan.right)
        if not (isinstance(plan, BroadcastHashJoinExec) and plan.joinType == "inner" and plan.condition is None):
            return plan
        right_built = plan.buildSide == "right"
        build, streamed = (plan.right, plan.left) if right_built else (plan.left, plan.right)
        bkeys, skeys = (plan.rightKeys, plan.leftKeys) if right_built else (plan.leftKeys, plan.rightKeys)
        if not _has_filter(build):
            return plan
        # walk down the streamed side through operators that pass the key attribute through unchanged
        j1 = streamed
        while True:
            if isinstance(j1, ProjectExec):
                passed = {n for n, e in j1.projectList if isinstance(e, AttributeReference) and e.name == n}
                if not all(k in passed for k in skeys):
                    return plan
                j1 = j1.child
            elif isinstance(j1, FilterExec):
                j1 = j1.child
            else:
                break
        if not (isinstance(j1, BroadcastHashJoinExec) and j1.joinType in ("inner", "left_semi") and j1.condition is None):
            return plan
        j1_streamed = j1.left if j1.buildSide == "right" else j1.right
        names = _output_names(j1_streamed)
        if names is None:
            return plan
        injected = False
        for sk, bk in zip(skeys, bkeys):
            if sk in names and len(j1.runtimeFilters) < self.maxRuntimeFilters and all(f.applicationKey != sk for f in j1.runtimeFilters):
                if not isinstance(build, ReusedExchangeExec):
                    build = ReusedExchangeExec(build, uses=1)
                build.uses += 1
                j1.runtimeFilters.append(RuntimeFilter(sk, bk, build))
                injected = True
        if injected:
            if right_built:
                plan.right = build
            else:
                plan.left = build
            plan.children = (plan.left, plan.right)
        return plan


def _has_filter(plan) -> bool:
    """hasSelectivePredicate's stand-in (InjectRuntimeFilter.scala:262-275): the mirror keeps no statistics, a FilterExec anywhere in the
    creation side counts as selective."""
    return isinstance(plan, FilterExec) or any(_has_filter(c) for c in getattr(plan, "children", ()))


def _output_names(plan):
    """Attribute names a plan produces, when they can be told without running it (None otherwise)."""
    if isinstance(plan, LocalTableScanExec):
        return list(plan.batch.names)
    if isinstance(plan, ProjectExec):
        return [n for n, _ in plan.projectList]
    if isinstance(plan, (FilterExec, ReusedExchangeExec)):
        return _output_names(plan.child)
    if isinstance(plan, BroadcastHashJoinExec):
        l = _output_names(plan.left)
        if plan.joinType in ("left_semi", "left_anti", "left_anti_null_aware"):
            return l
        r = _output_names(plan.right)
        return None if l is None or r is None else l + r
    out = getattr(plan, "output_names", None)
    return list(out) if out is not None else None


def _substitute(e: Expression, mapping):
    import copy
    if isinstance(e, AttributeReference):
        return mapping.get(e.name, e)
    e2 = copy.copy(e)
    for attr in ("left", "right", "child"):
        if hasattr(e2, attr):
            setattr(e2, attr, _substitute(getattr(e2, attr), mapping))
    if hasattr(e2, "left"):
        e2.children = (e2.left, e2.right)
    elif hasattr(e2, "child"):
        e2.children = (e2.child,)
    return e2


# ------------------------------------------------------------------------------------------------ f4: Expand / SortAggregate / Window
class ExpandExec(SparkPlan):
    """ExpandExec(projections, output, child) (sql/core/.../execution/ExpandExec.scala:36): every input row yields one output row
    per projection list, list 0 first.  projections: [[Expression, ...], ...]; output: the column names.  ROLLUP / CUBE /
    GROUPING SETS and multi-DISTINCT aggregates plan it below a HashAggregateExec."""

    def __init__(self, projections, output, child: SparkPlan):
        self.projections = [list(p) for p in projections]
        self.output = list(output)
        assert all(len(p) == len(self.output) for p in self.projections), "every projection list must produce the output schema"
        self.child = child
        self.children = (child,)

    def executeColumnar(self, stream=None):
        inp = self.child.executeColumnar(stream)
        try:
            schema = _schema_of(inp)
            compiled = [CompiledExpr(e, schema) for p in self.projections for e in p]
            arr = (capi.sb_expr * len(compiled))()
            for i, c in enumerate(compiled):
                arr[i] = c.c
            h = C.c_void_p()
            capi.check(capi.load().sb_expand(inp.handle, arr, len(self.projections), len(self.output), _h(stream), C.byref(h)))
            ats = []
            for c in range(len(self.output)):
                e = self.projections[0][c]
                ats.append(inp.arrow_types[schema.index(e.name)] if isinstance(e, AttributeReference) else None)
            return ColumnarBatch(h, self.output, ats)
        finally:
            inp.close()


class SortAggregateExec(HashAggregateExec):
    """SortAggregateExec (sql/core/.../aggregate/SortAggregateExec.scala): the planner's choice when an aggregation buffer is not
    mutable in an UnsafeRow (AggUtils.createAggregate).  It differs from HashAggregateExec in HOW groups are found (sorted input,
    adjacent rows), not in what comes out -- one row per group, same buffer algebra -- so the device operator is the same."""


class WindowFunction:
    """One window expression: func in row_number | rank | dense_rank | percent_rank | cume_dist | ntile | lag | lead | sum |
    count | avg | min | max | first_value | last_value; child = input column name (None for the ranking functions);
    frame = ('rows' | 'range', lower, upper) with None = UNBOUNDED, 0 = CURRENT ROW, negative = PRECEDING (rows only);
    default frame like SpecifiedWindowFrame.defaultWindowFrame: with ORDER BY range(UNBOUNDED, CURRENT ROW), else the partition."""

    def __init__(self, func, child=None, frame=None, param=0, name=None):
        self.func, self.child, self.frame, self.param = func, child, frame, param
        self.name = name or func


class WindowExec(SparkPlan):
    """WindowExec(windowExpression, partitionSpec, orderSpec, child) (sql/core/.../window/WindowExec.scala:90).  Output: the
    child's rows sorted by partitionSpec ++ orderSpec (the child ordering the reference requires) ++ one column per window
    expression."""

    def __init__(self, windowExpression, partitionSpec, orderSpec, child: SparkPlan):
        self.windowExpression = list(windowExpression)
        self.partitionSpec = list(partitionSpec)
        self.orderSpec = [o if isinstance(o, SortOrder) else SortOrder(*o) for o in orderSpec]
        self.child = child
        self.children = (child,)

    def executeColumnar(self, stream=None):
        inp = self.child.executeColumnar(stream)
        try:
            part = (C.c_int32 * max(1, len(self.partitionSpec)))(*[inp.column_index(c) for c in self.partitionSpec])
            specs = (capi.sb_window_spec * max(1, len(self.windowExpression)))()
            out_types = []
            for i, w in enumerate(self.windowExpression):
                frame = w.frame
                if frame is None:
                    frame = ("range", None, 0) if self.orderSpec else ("rows", None, None)
                kind, lo, hi = frame
                specs[i].func = capi.SB_WIN[w.func]
                specs[i].col = inp.column_index(w.child) if w.child is not None else 0
                specs[i].frame_type = capi.SB_FRAME_RANGE if kind == "range" else capi.SB_FRAME_ROWS
                if kind == "range" and self.orderSpec and any(b not in (None, 0) for b in (lo, hi)):
                    # value offsets: doubles (as bits) over a floating-point ORDER BY key, integers otherwise
                    kt = inp.column_desc(inp.column_index(self.orderSpec[0].child)).type
                    if kt in (capi.SB_FLOAT32, capi.SB_FLOAT64):
                        import struct
                        specs[i].frame_type = capi.SB_FRAME_RANGE_F64
                        lo, hi = [b if b in (None, 0) else struct.unpack("<q", struct.pack("<d", float(b)))[0] for b in (lo, hi)]
                specs[i].lower = capi.SB_UNBOUNDED_PRECEDING if lo is None else lo
                specs[i].upper = capi.SB_UNBOUNDED_FOLLOWING if hi is None else hi
                specs[i].param = w.param
                keeps = w.func in ("lag", "lead", "min", "max", "first_value", "last_value")
                out_types.append(inp.arrow_types[inp.column_index(w.child)] if keeps else None)
            h = C.c_void_p()
            capi.check(capi.load().sb_window(inp.handle, part, len(self.partitionSpec), _orders_c(inp, self.orderSpec), len(self.orderSpec),
                                             specs, len(self.windowExpression), _h(stream), C.byref(h)))
            return ColumnarBatch(h, inp.names + [w.name for w in self.windowExpression], inp.arrow_types + out_types)
        finally:
            inp.close()
