package org.apache.spark.sql.b200

import org.apache.spark.rdd.RDD
import org.apache.spark.sql.catalyst.expressions._
import org.apache.spark.sql.catalyst.optimizer.{BuildLeft, BuildRight, BuildSide}
import org.apache.spark.sql.catalyst.plans._
import org.apache.spark.sql.catalyst.plans.physical._
import org.apache.spark.sql.execution._
import org.apache.spark.sql.execution.aggregate.BaseAggregateExec
import org.apache.spark.sql.execution.metric.{SQLMetric, SQLMetrics}
import org.apache.spark.sql.types.DataType
import org.apache.spark.sql.vectorized.ColumnarBatch

/**
 * HashAggregateExec on the GPU (SQLX/aggregate/HashAggregateExec.scala:50).  The partition's batches are folded one by one into
 * an aggregation state on the device (sb_hash_agg_create / update / finish == TungstenAggregationIterator.processInputs,
 * TungstenAggregationIterator.scala:206-281); each input batch is closed as soon as it has been consumed, nothing is
 * concatenated.  `condition` / `inputs` are the Filter / Project chain GpuSupport.collapse folded into the aggregate.
 */
case class GpuHashAggregateExec(
    cpu: BaseAggregateExec,                   // HashAggregateExec, or SortAggregateExec (same answer, same device operator)
    condition: Option[Expression],
    inputs: Seq[Option[Expression]],          // one per aggregate function: its argument over `child`'s attributes (None: count(*))
    child: SparkPlan) extends UnaryExecNode with GpuExec {
  override def output: Seq[Attribute] = cpu.output
  override def outputPartitioning: Partitioning = cpu.outputPartitioning
  override def requiredChildDistribution: Seq[Distribution] = cpu.requiredChildDistribution   // Partial -> Exchange -> Final unchanged
  override lazy val metrics: Map[String, SQLMetric] = Map(
    "numOutputRows" -> SQLMetrics.createMetric(sparkContext, "number of output rows"),
    "aggTime" -> SQLMetrics.createTimingMetric(sparkContext, "time in aggregation build"))     // HashAggregateExec.scala:70-86

  override protected def doExecuteColumnar(): RDD[ColumnarBatch] = {
    val numOutputRows = longMetric("numOutputRows")
    val aggTime = longMetric("aggTime")
    val mode = GpuSupport.mode(cpu)                       // SB_AGG_MODE_* (AggUtils.scala:131-208)
    val childTypes: Array[DataType] = child.output.map(_.dataType).toArray
    val outTypes: Array[DataType] = output.map(_.dataType).toArray
    val plan = GpuSupport.compileAgg(cpu, condition, inputs, child.output)   // serialisable description; lowered per task below
    child.executeColumnar().mapPartitions { batches =>
      val stream = taskStream()
      val start = System.nanoTime()
      val native = plan.lower()                            // sb_expr handles for this task
      val state = Native.aggCreate(mode, native.keyCols, native.funcs, native.inputExprs, native.filterExpr, 0L)
      try {
        var any = false
        while (batches.hasNext) {
          val in = DeviceTransfer.toDevice(batches.next(), childTypes, stream)
          try Native.aggUpdate(state, in.table, stream) finally in.close()
          any = true
        }
        if (!any && cpu.groupingExpressions.nonEmpty) {
          Iterator.empty                                   // a grouping aggregate over an empty partition emits nothing
        } else {
          if (!any) {                                      // global aggregate: one row even for empty input (AggregateCodegenSupport.scala:131)
            val empty = GpuSupport.emptyDeviceBatch(childTypes, stream)
            try Native.aggUpdate(state, empty.table, stream) finally empty.close()
          }
          val out = new DeviceBatch(Native.aggFinish(state, stream), outTypes)
          numOutputRows += out.numRows()
          aggTime += (System.nanoTime() - start) / 1000000
          Iterator.single(out: ColumnarBatch)
        }
      } finally {
        Native.aggDestroy(state)
        native.close()
      }
    }
  }
  override protected def withNewChildInternal(c: SparkPlan): SparkPlan = copy(child = c)
}

/** FilterExec / ProjectExec (basicPhysicalOperators.scala:245 / :47) as one pass per batch: sb_filter_project; with string-producing
 *  functions, sb_string_project too (GpuSupport.runStringStage). */
case class GpuFilterProjectExec(condition: Option[Expression], projectList: Seq[NamedExpression], child: SparkPlan)
  extends UnaryExecNode with GpuExec {
  override def output: Seq[Attribute] = projectList.map(_.toAttribute)
  override def outputPartitioning: Partitioning = child.outputPartitioning
  override protected def doExecuteColumnar(): RDD[ColumnarBatch] = {
    val childTypes = child.output.map(_.dataType).toArray
    val outTypes = output.map(_.dataType).toArray
    if (GpuSupport.hasStringFunction(condition, projectList)) {
      val stage = GpuSupport.compileStringStage(condition, projectList, child.output)
      child.executeColumnar().mapPartitions { batches =>
        val stream = taskStream()
        val native = stage.lower()
        Option(org.apache.spark.TaskContext.get()).foreach(_.addTaskCompletionListener[Unit](_ => native.close()))
        batches.map { b =>
          val in = DeviceTransfer.toDevice(b, childTypes, stream)
          try new DeviceBatch(GpuSupport.runStringStage(native, in.table, stream), outTypes): ColumnarBatch
          finally in.close()
        }
      }
    } else {
      val compiled = GpuSupport.compileFilterProject(condition, projectList, child.output)
      child.executeColumnar().mapPartitions { batches =>
        val stream = taskStream()
        val native = compiled.lower()
        Option(org.apache.spark.TaskContext.get()).foreach(_.addTaskCompletionListener[Unit](_ => native.close()))
        batches.map { b =>
          val in = DeviceTransfer.toDevice(b, childTypes, stream)
          try new DeviceBatch(Native.filterProject(in.table, native.filterExpr, native.inputExprs, stream), outTypes): ColumnarBatch
          finally in.close()
        }
      }
    }
  }
  override protected def withNewChildInternal(c: SparkPlan): SparkPlan = copy(child = c)
}

/** SortExec (SQLX/SortExec.scala:39): per-partition stable sort; a global sort sits on top of a range exchange as in the reference. */
case class GpuSortExec(sortOrder: Seq[SortOrder], global: Boolean, child: SparkPlan) extends UnaryExecNode with GpuExec {
  override def output: Seq[Attribute] = child.output
  override def outputOrdering: Seq[SortOrder] = sortOrder
  override def outputPartitioning: Partitioning = child.outputPartitioning
  override def requiredChildDistribution: Seq[Distribution] =
    if (global) OrderedDistribution(sortOrder) :: Nil else UnspecifiedDistribution :: Nil        // SortExec.scala:54-55
  override protected def doExecuteColumnar(): RDD[ColumnarBatch] = {
    val types = child.output.map(_.dataType).toArray
    val (cols, asc, nullsFirst) = GpuSupport.orders(sortOrder, child.output)
    child.executeColumnar().mapPartitions { batches =>
      val stream = taskStream()
      val in = GpuSupport.concatToDevice(batches, types, stream)      // a sort needs the whole partition
      if (in == null) Iterator.empty
      else try Iterator.single(new DeviceBatch(Native.sort(in.table, cols, asc, nullsFirst, stream), types): ColumnarBatch) finally in.close()
    }
  }
  override protected def withNewChildInternal(c: SparkPlan): SparkPlan = copy(child = c)
}

/** TakeOrderedAndProjectExec (SQLX/limit.scala:310-411): per-partition top k, single-partition exchange, final top k, project. */
case class GpuTakeOrderedAndProjectExec(limit: Int, sortOrder: Seq[SortOrder], projectList: Seq[NamedExpression], child: SparkPlan)
  extends UnaryExecNode with GpuExec {
  override def output: Seq[Attribute] = projectList.map(_.toAttribute)
  override def outputPartitioning: Partitioning = SinglePartition
  override def outputOrdering: Seq[SortOrder] = sortOrder
  override protected def doExecuteColumnar(): RDD[ColumnarBatch] = {
    val types = child.output.map(_.dataType).toArray
    val outTypes = output.map(_.dataType).toArray
    val (cols, asc, nullsFirst) = GpuSupport.orders(sortOrder, child.output)
    val proj = GpuSupport.compileFilterProject(None, projectList, child.output)
    val k = limit.toLong
    def topK(batches: Iterator[ColumnarBatch]): Iterator[ColumnarBatch] = {
      val stream = taskStream()
      val in = GpuSupport.concatToDevice(batches, types, stream)
      if (in == null) Iterator.empty
      else try Iterator.single(new DeviceBatch(Native.topN(in.table, cols, asc, nullsFirst, k, stream), types): ColumnarBatch) finally in.close()
    }
    val local = child.executeColumnar().mapPartitions(topK)
    val single = if (child.outputPartitioning.numPartitions == 1) local else GpuSupport.gatherToSinglePartition(local, types)
    single.mapPartitions { batches =>
      topK(batches).map { top =>
        val stream = taskStream()
        val native = proj.lower()
        val d = top.asInstanceOf[DeviceBatch]
        try new DeviceBatch(Native.filterProject(d.table, 0L, native.inputExprs, stream), outTypes): ColumnarBatch
        finally { d.close(); native.close() }
      }
    }
  }
  override protected def withNewChildInternal(c: SparkPlan): SparkPlan = copy(child = c)
}

/**
 * What InjectRuntimeFilter (sql/catalyst/.../optimizer/InjectRuntimeFilter.scala:47-100) plans as
 * FilterExec(BloomFilterMightContain(bloomSubquery, xxhash64(applicationKey))) on the application side of a join: here the
 * creation side (a GpuBroadcastExchangeExec shared with the join the filter was derived from) is built into a single-key
 * relation and its prefilter is tested on `applicationKey` of the STREAMED side of the join that carries the filter
 * (sb_join_options.runtime_filter_cols / runtime_filter_relations).  Planned by B200ColumnarRule.injectRuntimeFilters.
 */
case class GpuRuntimeFilter(applicationKey: Attribute, creationKey: Attribute, creation: SparkPlan)

/**
 * BroadcastHashJoinExec / ShuffledHashJoinExec / SortMergeJoinExec (SQLX/joins/HashJoin.scala:184-400) as build + probe.
 * The build side is the whole partition of one child (broadcast: every partition sees the same relation through
 * GpuBroadcastExchangeExec); the streamed side is probed batch by batch.  Output is left ++ right whatever the build side
 * (HashJoin.scala:55-70).
 */
case class GpuHashJoinExec(
    leftKeys: Seq[Expression],
    rightKeys: Seq[Expression],
    joinType: JoinType,
    buildSide: BuildSide,
    condition: Option[Expression],
    left: SparkPlan,
    right: SparkPlan,
    isNullAwareAntiJoin: Boolean,
    broadcast: Boolean,
    runtimeFilters: Seq[GpuRuntimeFilter] = Nil) extends BinaryExecNode with GpuExec {

  override def output: Seq[Attribute] = joinType match {                                 // HashJoin.scala:55-70
    case _: InnerLike => left.output ++ right.output
    case LeftOuter => left.output ++ right.output.map(_.withNullability(true))
    case RightOuter => left.output.map(_.withNullability(true)) ++ right.output
    case FullOuter => (left.output ++ right.output).map(_.withNullability(true))
    case j: ExistenceJoin => left.output :+ j.exists
    case LeftExistence(_) => left.output
    case x => throw new IllegalArgumentException(s"GpuHashJoinExec does not take join type $x")
  }
  override def outputPartitioning: Partitioning = if (buildSide == BuildRight) left.outputPartitioning else right.outputPartitioning
  override def requiredChildDistribution: Seq[Distribution] =
    if (broadcast) {
      val mode = org.apache.spark.sql.execution.joins.HashedRelationBroadcastMode(if (buildSide == BuildRight) rightKeys else leftKeys,
        isNullAwareAntiJoin)
      if (buildSide == BuildRight) UnspecifiedDistribution :: BroadcastDistribution(mode) :: Nil
      else BroadcastDistribution(mode) :: UnspecifiedDistribution :: Nil                 // BroadcastHashJoinExec.scala:62-72
    } else ClusteredDistribution(leftKeys) :: ClusteredDistribution(rightKeys) :: Nil    // ShuffledJoin.scala:38-45

  override protected def doExecuteColumnar(): RDD[ColumnarBatch] = {
    val (buildPlan, streamPlan, buildKeys, streamKeys) =
      if (buildSide == BuildRight) (right, left, rightKeys, leftKeys) else (left, right, leftKeys, rightKeys)
    val buildTypes = buildPlan.output.map(_.dataType).toArray
    val streamTypes = streamPlan.output.map(_.dataType).toArray
    val outTypes = output.map(_.dataType).toArray
    val buildOrd = GpuSupport.ordinals(buildKeys, buildPlan.output)
    val streamOrd = GpuSupport.ordinals(streamKeys, streamPlan.output)
    val native = GpuSupport.nativeJoinType(joinType, buildSide, isNullAwareAntiJoin)     // SB_JOIN_* as seen from the streamed side
    // the residual condition is evaluated on the joined row as the kernels lay it out: streamed columns ++ build columns
    val cond = condition.map(c => GpuSupport.compileFilterProject(Some(c), Nil, streamPlan.output ++ buildPlan.output))
    val reorder: Array[Int] =                                                             // streamed ++ build -> left ++ right
      if (buildSide == BuildRight || !GpuSupport.emitsBothSides(joinType)) null
      else (streamTypes.length until streamTypes.length + buildTypes.length).toArray ++ streamTypes.indices

    def join(buildBatches: Iterator[ColumnarBatch], streamBatches: Iterator[ColumnarBatch]): Iterator[ColumnarBatch] = {
      val stream = taskStream()
      val b = GpuSupport.concatToDevice(buildBatches, buildTypes, stream, orEmpty = true)
      val relation = try Native.joinBuild(b.table, buildOrd, stream) finally b.close()   // the relation retains the build table
      val lowered = cond.map(_.lower())
      // runtime filters: one single-key relation per filter, built from the creation side's broadcast (the executor's device copy)
      val usable = if (lowered.isEmpty && (native == 0 || native == 2)   /* SB_JOIN_INNER, SB_JOIN_LEFT_SEMI */) runtimeFilters else Nil
      val rfCols = usable.map(f => GpuSupport.ordinals(Seq(f.applicationKey), streamPlan.output)(0)).toArray
      val rfRelations = usable.map { f =>
        val types = f.creation.output.map(_.dataType).toArray
        val c = GpuSupport.concatToDevice(GpuBroadcastExchangeExec.batchesOf(f.creation.executeBroadcast[Array[Long]]().value, types), types,
          stream, orEmpty = true)
        try Native.joinBuild(c.table, GpuSupport.ordinals(Seq(f.creationKey), f.creation.output), stream) finally c.close()
      }.toArray
      Option(org.apache.spark.TaskContext.get()).foreach(_.addTaskCompletionListener[Unit] { _ =>
        Native.hashTableRelease(relation); rfRelations.foreach(Native.hashTableRelease); lowered.foreach(_.close()) })
      // build-side-preserving joins emit the unmatched build rows once: they need the whole streamed partition in one probe
      val whole = GpuSupport.preservesBuildSide(joinType, buildSide)
      val inputs = if (whole) Iterator.single(GpuSupport.concatToDevice(streamBatches, streamTypes, stream, orEmpty = true): ColumnarBatch)
                   else streamBatches
      inputs.map { sb =>
        val p = DeviceTransfer.toDevice(sb, streamTypes, stream)
        try {
          val t = lowered match {
            case Some(l) => Native.joinProbeCondition(relation, p.table, streamOrd, native, l.filterExpr, stream)
            case None if rfRelations.nonEmpty =>
              Native.joinProbeRuntimeFiltered(relation, p.table, streamOrd, native, 0L, null, null, rfCols, rfRelations, stream)
            case None => Native.joinProbe(relation, p.table, streamOrd, native, stream)
          }
          if (reorder == null) new DeviceBatch(t, outTypes): ColumnarBatch
          else try new DeviceBatch(Native.tableSelect(t, reorder), outTypes): ColumnarBatch finally Native.tableRelease(t)
        } finally p.close()
      }
    }
    if (broadcast) {
      val relationBatches = buildPlan.executeBroadcast[Array[Long]]()      // GpuBroadcastExchangeExec: device table handle per executor
      streamPlan.executeColumnar().mapPartitions { s =>
        join(GpuBroadcastExchangeExec.batchesOf(relationBatches.value, buildTypes), s)
      }
    } else if (buildSide == BuildRight) {
      left.executeColumnar().zipPartitions(right.executeColumnar()) { (l, r) => join(r, l) }
    } else {
      left.executeColumnar().zipPartitions(right.executeColumnar()) { (l, r) => join(l, r) }
    }
  }
  override protected def withNewChildrenInternal(l: SparkPlan, r: SparkPlan): SparkPlan = copy(left = l, right = r)
}

/**
 * ExpandExec (SQLX/ExpandExec.scala:36): every input row yields one output row per projection list, list 0 first -- sb_expand.
 * ROLLUP / CUBE / GROUPING SETS and multi-DISTINCT aggregates plan it below an aggregate.
 */
case class GpuExpandExec(projections: Seq[Seq[Expression]], output: Seq[Attribute], child: SparkPlan) extends UnaryExecNode with GpuExec {
  override def outputPartitioning: Partitioning = UnknownPartitioning(0)                         // ExpandExec.scala:55-61
  override protected def doExecuteColumnar(): RDD[ColumnarBatch] = {
    val childTypes = child.output.map(_.dataType).toArray
    val outTypes = output.map(_.dataType).toArray
    val programs = projections.flatten.map(e => ExprCompiler.compile(e, child.output))
    val (nlists, ncols) = (projections.length, output.length)
    child.executeColumnar().mapPartitions { batches =>
      val stream = taskStream()
      val exprs = programs.map(_.create()).toArray
      Option(org.apache.spark.TaskContext.get()).foreach(_.addTaskCompletionListener[Unit](_ => exprs.foreach(Native.exprFree)))
      batches.map { b =>
        val in = DeviceTransfer.toDevice(b, childTypes, stream)
        try new DeviceBatch(Native.expand(in.table, exprs, nlists, ncols, stream), outTypes): ColumnarBatch finally in.close()
      }
    }
  }
  override protected def withNewChildInternal(c: SparkPlan): SparkPlan = copy(child = c)
}

/**
 * WindowExec (SQLX/window/WindowExec.scala:90) -- sb_window.  The reference requires its child sorted by partitionSpec ++ orderSpec
 * (WindowExecBase.requiredChildOrdering) and plans a SortExec for that; the device operator sorts the partition itself, so only the
 * clustering requirement is kept and the output carries the ordering.
 */
case class GpuWindowExec(windowExpression: Seq[NamedExpression], partitionSpec: Seq[Expression], orderSpec: Seq[SortOrder], child: SparkPlan)
  extends UnaryExecNode with GpuExec {
  override def output: Seq[Attribute] = child.output ++ windowExpression.map(_.toAttribute)
  override def outputPartitioning: Partitioning = child.outputPartitioning
  override def outputOrdering: Seq[SortOrder] = partitionSpec.map(SortOrder(_, Ascending)) ++ orderSpec
  override def requiredChildDistribution: Seq[Distribution] =                                    // WindowExecBase.scala
    if (partitionSpec.isEmpty) AllTuples :: Nil else ClusteredDistribution(partitionSpec) :: Nil
  override protected def doExecuteColumnar(): RDD[ColumnarBatch] = {
    val childTypes = child.output.map(_.dataType).toArray
    val outTypes = output.map(_.dataType).toArray
    val w = GpuSupport.lowerWindow(org.apache.spark.sql.execution.window.WindowExec(windowExpression, partitionSpec, orderSpec, child)).get
    child.executeColumnar().mapPartitions { batches =>
      val stream = taskStream()
      val in = GpuSupport.concatToDevice(batches, childTypes, stream)      // a window needs the whole partition
      if (in == null) Iterator.empty
      else try Iterator.single(new DeviceBatch(Native.window(in.table, w.partition, w.orderCols, w.asc, w.nullsFirst, w.funcs, w.inputs,
        w.frameTypes, w.lowers, w.uppers, w.params, stream), outTypes): ColumnarBatch) finally in.close()
    }
  }
  override protected def withNewChildInternal(c: SparkPlan): SparkPlan = copy(child = c)
}

/** RowToColumnarExec replacement (Columnar.scala:503-546): the child's host batches become HBM batches. */
case class HostToDeviceExec(child: SparkPlan) extends UnaryExecNode with GpuExec {
  override def output: Seq[Attribute] = child.output
  override def outputPartitioning: Partitioning = child.outputPartitioning
  override def outputOrdering: Seq[SortOrder] = child.outputOrdering
  override protected def doExecuteColumnar(): RDD[ColumnarBatch] = {
    val types = child.output.map(_.dataType).toArray
    // a row-based child is converted by the reference's own RowToColumnarExec first (off-heap vectors), then copied
    val host = if (child.supportsColumnar) child.executeColumnar() else RowToColumnarExec(child).executeColumnar()
    host.mapPartitions(_.map(b => DeviceTransfer.toDevice(b, types, taskStream()): ColumnarBatch))
  }
  override protected def withNewChildInternal(c: SparkPlan): SparkPlan = copy(child = c)
}

/** The way back for ColumnarToRowExec (Columnar.scala:67-214): HBM batches become OffHeapColumnVector batches. */
case class DeviceToHostExec(child: SparkPlan) extends UnaryExecNode {
  override def output: Seq[Attribute] = child.output
  override def outputPartitioning: Partitioning = child.outputPartitioning
  override def outputOrdering: Seq[SortOrder] = child.outputOrdering
  override def supportsColumnar: Boolean = true
  override protected def doExecute(): RDD[org.apache.spark.sql.catalyst.InternalRow] =
    throw new IllegalStateException("DeviceToHostExec is columnar; ColumnarToRowExec above it makes the rows")
  override protected def doExecuteColumnar(): RDD[ColumnarBatch] = {
    val types = child.output.map(_.dataType).toArray
    child.executeColumnar().mapPartitions(_.map(b => DeviceTransfer.toHost(b, types, GpuExec.taskStream())))
  }
  override protected def withNewChildInternal(c: SparkPlan): SparkPlan = copy(child = c)
}
