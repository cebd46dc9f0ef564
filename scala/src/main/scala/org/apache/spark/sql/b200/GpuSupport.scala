package org.apache.spark.sql.b200

import scala.collection.mutable.ArrayBuffer

import org.apache.spark.rdd.RDD
import org.apache.spark.sql.catalyst.expressions._
import org.apache.spark.sql.catalyst.expressions.aggregate._
import org.apache.spark.sql.catalyst.optimizer.{BuildLeft, BuildRight, BuildSide}
import org.apache.spark.sql.catalyst.plans._
import org.apache.spark.sql.catalyst.plans.physical._
import org.apache.spark.sql.execution._
import org.apache.spark.sql.execution.aggregate.{BaseAggregateExec, HashAggregateExec, SortAggregateExec}
import org.apache.spark.sql.execution.window.WindowExec
import org.apache.spark.sql.execution.exchange.{BroadcastExchangeExec, ShuffleExchangeExec}
import org.apache.spark.sql.execution.joins.{BroadcastHashJoinExec, ShuffledHashJoinExec, SortMergeJoinExec}
import org.apache.spark.sql.internal.SQLConf
import org.apache.spark.sql.types._
import org.apache.spark.sql.vectorized.ColumnarBatch
import org.apache.spark.unsafe.types.UTF8String

/**
 * What the GPU path can run and how Catalyst objects become the POD structures of include/spark_b200.h.  Anything this object
 * says no to stays on the CPU operators (the plan is still valid: ApplyColumnarRulesAndInsertTransitions inserts the
 * transitions); nothing is ever executed by a CPU re-implementation inside the plugin.
 */
object GpuSupport {
  // ---- support checks ---------------------------------------------------------------------------------------------------
  private def typeOk(dt: DataType): Boolean = GpuExec.typeId(dt) > 0
  private def fixedWidth(dt: DataType): Boolean = typeOk(dt) && dt != StringType && dt != BinaryType
  private def outputOk(p: SparkPlan): Boolean = p.output.forall(a => typeOk(a.dataType))
  private def exprOk(e: Expression): Boolean = ExprCompiler.supported(e)
  /** SUM / AVG over decimals: a bare decimal(p <= 18) column (128-bit limb sums inside the library, csrc/decimal.cu); decimal
   *  arithmetic in the argument stays on the CPU */
  private def decimalInputOk(c: Expression): Boolean = c.dataType match {
    case d: DecimalType => d.precision <= 18 && c.isInstanceOf[AttributeReference]
    case _ => true
  }
  /** central moments read their input as DOUBLE: a double expression, or the analyzer's Cast to DOUBLE of an integer or float one
   *  (decimal, boolean, string, date and timestamp inputs are not taken) */
  private def momentInputOk(c: Expression): Boolean = exprOk(c) && (c match {
    case cast: Cast if cast.dataType == DoubleType =>
      cast.child.dataType match { case ByteType | ShortType | IntegerType | LongType | FloatType | DoubleType => true; case _ => false }
    case _ => c.dataType == DoubleType
  })
  /** grouping / join / sort keys: fixed-width types, and strings (order-preserving dictionary codes inside the library) */
  private def keyOk(dt: DataType): Boolean = fixedWidth(dt) || dt == StringType

  def supports(agg: HashAggregateExec): Boolean = aggregateOk(agg)
  /** SortAggregateExec differs from HashAggregateExec in how groups are found, not in what comes out: same device operator */
  def supports(agg: SortAggregateExec): Boolean = aggregateOk(agg)
  private def aggregateOk(agg: BaseAggregateExec): Boolean =
    !agg.isStreaming && outputOk(agg.child) &&
      agg.groupingExpressions.forall(g => g.isInstanceOf[AttributeReference] && keyOk(g.dataType)) &&
      agg.groupingExpressions.length <= 6 &&
      agg.aggregateExpressions.forall { ae =>
        !ae.isDistinct && ae.filter.isEmpty && (ae.aggregateFunction match {
          case Sum(c, _) => fixedWidth(c.dataType) && decimalInputOk(c) && exprOk(c)
          case Average(c, _) => fixedWidth(c.dataType) && decimalInputOk(c) && exprOk(c)
          case Count(cs) => cs.length <= 1 && cs.forall(exprOk)
          case Min(c) => fixedWidth(c.dataType) && exprOk(c)
          case Max(c) => fixedWidth(c.dataType) && exprOk(c)
          case VariancePop(c, _) => momentInputOk(c)
          case VarianceSamp(c, _) => momentInputOk(c)
          case StddevPop(c, _) => momentInputOk(c)
          case StddevSamp(c, _) => momentInputOk(c)
          case _ => false      // Skewness, Kurtosis, covariance / correlation and the Pandas forms stay on the CPU
        })
      }
  def supports(s: SortExec): Boolean = outputOk(s.child) &&
    s.sortOrder.forall(o => o.child.isInstanceOf[AttributeReference] && keyOk(o.child.dataType))
  def supports(t: TakeOrderedAndProjectExec): Boolean = t.offset == 0 && outputOk(t.child) &&
    t.sortOrder.forall(o => o.child.isInstanceOf[AttributeReference] && keyOk(o.child.dataType)) && t.projectList.forall(exprOk)
  private def joinOk(leftKeys: Seq[Expression], rightKeys: Seq[Expression], jt: JoinType, cond: Option[Expression], l: SparkPlan,
                     r: SparkPlan): Boolean =
    outputOk(l) && outputOk(r) && leftKeys.length <= 4 &&
      (leftKeys ++ rightKeys).forall(k => k.isInstanceOf[AttributeReference] && keyOk(k.dataType)) &&
      cond.forall(exprOk) &&       // keys of <= 64 bits are packed (HashJoin.rewriteKeyExpr), wider ones hashed and verified inside the library
      (jt match { case _: InnerLike | LeftOuter | RightOuter | FullOuter | LeftSemi | LeftAnti | _: ExistenceJoin => true; case _ => false })
  def supports(j: BroadcastHashJoinExec): Boolean = joinOk(j.leftKeys, j.rightKeys, j.joinType, j.condition, j.left, j.right)
  def supports(j: ShuffledHashJoinExec): Boolean = joinOk(j.leftKeys, j.rightKeys, j.joinType, j.condition, j.left, j.right)
  def supports(j: SortMergeJoinExec): Boolean = joinOk(j.leftKeys, j.rightKeys, j.joinType, j.condition, j.left, j.right)
  def supports(e: ShuffleExchangeExec): Boolean = outputOk(e.child) && !e.child.output.exists(_.dataType == StringType) &&
    !SQLConf.get.getConf(SQLConf.SKEW_JOIN_ENABLED) && (e.outputPartitioning match {
      case HashPartitioning(keys, _) => keys.forall(_.isInstanceOf[AttributeReference])
      case RoundRobinPartitioning(_) | SinglePartition => true
      case RangePartitioning(ordering, _) => ordering.length == 1 && ordering.head.child.isInstanceOf[AttributeReference] &&
        fixedWidth(ordering.head.child.dataType)
      case _ => false
    })
  def supports(b: BroadcastExchangeExec): Boolean = outputOk(b.child) && !b.child.output.exists(_.dataType == StringType)
  def supports(f: FilterExec): Boolean = outputOk(f.child) && hoistedOk(f.condition)
  /** an expression of a numeric / boolean program once every string-producing function inside it is a hidden column of its own
   *  (csrc/strfunc.cu): the condition of a FilterExec, a numeric output of a ProjectExec */
  private def hoistedOk(e: Expression): Boolean = {
    val hidden = new ArrayBuffer[(AttributeReference, Expression)]()
    exprOk(ExprCompiler.hoist(e, hidden)) && hidden.forall(h => ExprCompiler.stringProgramOk(h._2))
  }
  def supports(e: ExpandExec): Boolean = outputOk(e.child) && e.output.forall(a => fixedWidth(a.dataType) || a.dataType == StringType) &&
    e.projections.forall(_.forall(exprOk))
  def supports(w: WindowExec): Boolean = outputOk(w.child) && lowerWindow(w).isDefined

  // ---- WindowExec -> sb_window_spec arrays ---------------------------------------------------------------------------------------
  final case class WindowLowered(partition: Array[Int], orderCols: Array[Int], asc: Array[Boolean], nullsFirst: Array[Boolean],
                                 funcs: Array[Int], inputs: Array[Int], frameTypes: Array[Int], lowers: Array[Long], uppers: Array[Long],
                                 params: Array[Long])
  private def bound(e: Expression, lower: Boolean): Option[Long] = e match {
    case UnboundedPreceding => Some(Long.MinValue)                       // SB_UNBOUNDED_PRECEDING
    case UnboundedFollowing => Some(Long.MaxValue)                       // SB_UNBOUNDED_FOLLOWING
    case CurrentRow => Some(0L)
    case Literal(v: Int, IntegerType) => Some(v.toLong)
    case UnaryMinus(Literal(v: Int, IntegerType), _) => Some(-v.toLong)
    case _ => None
  }
  /** None when some expression has no device form (value-offset RANGE frames, ignoreNulls, expression inputs, ...) */
  def lowerWindow(w: WindowExec): Option[WindowLowered] = {
    val in = w.child.output
    def ord(e: Expression): Option[Int] = e match {
      case a: AttributeReference => Some(in.indexWhere(_.exprId == a.exprId)).filter(_ >= 0)
      case _ => None
    }
    if (!w.partitionSpec.forall(p => ord(p).isDefined && keyOk(p.dataType))) return None
    if (!w.orderSpec.forall(o => ord(o.child).isDefined && keyOk(o.child.dataType))) return None
    if (w.partitionSpec.length + w.orderSpec.length > 8) return None
    val specs = w.windowExpression.map {
      case Alias(WindowExpression(fn, WindowSpecDefinition(_, _, SpecifiedWindowFrame(ft, lo, hi))), _) =>
        val frameType = if (ft == RangeFrame) 1 else 0
        val bounds = for (l <- bound(lo, lower = true); h <- bound(hi, lower = false)) yield (l, h)
        val rangeOk = frameType == 0 || bounds.exists { case (l, h) => (l == Long.MinValue || l == 0L) && (h == Long.MaxValue || h == 0L) }
        def agg(code: Int, c: Expression): Option[(Int, Int, Int, Long, Long, Long)] =
          for (i <- ord(c); (l, h) <- bounds if rangeOk && fixedWidth(c.dataType) && !c.dataType.isInstanceOf[DecimalType]) yield (code, i, frameType, l, h, 0L)
        fn match {
          case _: RowNumber => Some((1, 0, 0, 0L, 0L, 0L))
          case _: Rank => Some((2, 0, 0, 0L, 0L, 0L))
          case _: DenseRank => Some((3, 0, 0, 0L, 0L, 0L))
          case _: PercentRank => Some((4, 0, 0, 0L, 0L, 0L))
          case _: CumeDist => Some((5, 0, 0, 0L, 0L, 0L))
          case NTile(Literal(n: Int, IntegerType)) => Some((6, 0, 0, 0L, 0L, n.toLong))
          case Lag(c, Literal(k: Int, IntegerType), Literal(null, _), false) => ord(c).map(i => (7, i, 0, 0L, 0L, math.abs(k).toLong))
          case Lead(c, Literal(k: Int, IntegerType), Literal(null, _), false) => ord(c).map(i => (8, i, 0, 0L, 0L, k.toLong))
          case AggregateExpression(Sum(c, _), Complete, false, None, _) => agg(9, c)
          case AggregateExpression(Count(Seq(c)), Complete, false, None, _) => agg(10, c)
          case AggregateExpression(Average(c, _), Complete, false, None, _) => agg(11, c)
          case AggregateExpression(Min(c), Complete, false, None, _) => agg(12, c).filter(_._4 == Long.MinValue)
          case AggregateExpression(Max(c), Complete, false, None, _) => agg(13, c).filter(_._4 == Long.MinValue)
          case AggregateExpression(First(c, false), Complete, false, None, _) => for (i <- ord(c); (l, h) <- bounds if rangeOk) yield (14, i, frameType, l, h, 0L)
          case AggregateExpression(Last(c, false), Complete, false, None, _) => for (i <- ord(c); (l, h) <- bounds if rangeOk) yield (15, i, frameType, l, h, 0L)
          case _ => None
        }
      case _ => None
    }
    if (specs.exists(_.isEmpty)) return None
    val f = specs.map(_.get)
    val (oc, asc, nf) = orders(w.orderSpec, in)
    Some(WindowLowered(ordinals(w.partitionSpec, in), oc, asc, nf, f.map(_._1).toArray, f.map(_._2).toArray, f.map(_._3).toArray,
      f.map(_._4).toArray, f.map(_._5).toArray, f.map(_._6).toArray))
  }
  def supports(p: ProjectExec): Boolean = outputOk(p.child) && p.projectList.forall(e =>
    typeOk(e.dataType) && (ExprCompiler.stringProgramOk(stripAlias(e)) || hoistedOk(e)))
  private def stripAlias(e: Expression): Expression = e match { case Alias(c, _) => stripAlias(c); case o => o }

  private def keyBits(dt: DataType): Int = dt match {
    case BooleanType | ByteType => 8
    case ShortType => 16
    case IntegerType | FloatType | DateType => 32
    case _ => 64
  }

  // ---- Filter / Project folding under an aggregate (composed top-down, like spark_b200/execution.py B200ColumnarRule) -------
  final case class Collapsed(condition: Option[Expression], inputs: Seq[Option[Expression]], source: SparkPlan)

  def collapse(agg: BaseAggregateExec): Collapsed = {
    // aggregate inputs: Partial / Complete read the function's children, Final / PartialMerge read the buffer columns positionally
    var inputs: Seq[Option[Expression]] = agg.aggregateExpressions.map { ae =>
      if (ae.mode == Final || ae.mode == PartialMerge) None else ae.aggregateFunction.children.headOption
    }
    var groups: Seq[Expression] = agg.groupingExpressions
    var cond: Option[Expression] = None
    var node = agg.child
    var continue = true
    while (continue) node match {
      case ProjectExec(list, c) if list.forall(exprOk) =>
        val m = AttributeMap(list.collect { case a: Alias => a.toAttribute -> a.child })
        def sub(e: Expression): Expression = e.transform { case a: AttributeReference => m.getOrElse(a, a) }
        val newGroups = groups.map(sub)
        if (newGroups.forall(_.isInstanceOf[AttributeReference])) {
          inputs = inputs.map(_.map(sub)); groups = newGroups; cond = cond.map(sub); node = c
        } else continue = false                       // a computed grouping key: keep the Project (the native plan groups by columns)
      case FilterExec(c0, c) if exprOk(c0) =>
        cond = Some(cond.map(And(_, c0)).getOrElse(c0)); node = c
      case _ => continue = false
    }
    Collapsed(cond, inputs, node)
  }

  def mode(agg: HashAggregateExec): Int = {             // SB_AGG_MODE_* ; AggUtils.scala:131-208 plans one mode per operator
    val modes = agg.aggregateExpressions.map(_.mode).distinct
    if (modes.isEmpty || modes == Seq(Partial)) 1
    else if (modes == Seq(Final)) 2
    else if (modes == Seq(Complete)) 3
    else if (modes == Seq(PartialMerge)) 4
    else throw new B200Exception(5, s"mixed aggregate modes $modes in one operator")
  }

  // ---- lowering: serialisable descriptions on the driver, sb_expr handles per task -----------------------------------------------
  final class NativeHandles(val keyCols: Array[Int], val funcs: Array[Int], val inputExprs: Array[Long], val filterExpr: Long) {
    def close(): Unit = { inputExprs.foreach(h => if (h != 0L) Native.exprFree(h)); if (filterExpr != 0L) Native.exprFree(filterExpr) }
  }
  final case class Lowerable(keyCols: Array[Int], funcs: Array[Int], inputs: Array[Option[ExprCompiler.Program]],
                             filter: Option[ExprCompiler.Program]) {
    def lower(): NativeHandles = new NativeHandles(keyCols, funcs, inputs.map(_.map(_.create()).getOrElse(0L)),
      filter.map(_.create()).getOrElse(0L))
  }

  def compileAgg(agg: HashAggregateExec, condition: Option[Expression], inputs: Seq[Option[Expression]], in: Seq[Attribute]): Lowerable = {
    val keyCols = agg.groupingExpressions.map(g => in.indexWhere(_.exprId == g.toAttribute.exprId)).toArray
    val funcs = agg.aggregateExpressions.map(_.aggregateFunction match {
      case _: Sum => 1
      case _: Average => 2
      case Count(cs) => if (cs.isEmpty || cs.forall(!_.nullable)) 4 else 3
      case _: Min => 5
      case _: Max => 6
      // SB_AGG_VAR_POP .. SB_AGG_STDDEV_SAMP; bits 16.. carry sb_agg_spec.flags (SB_AGG_FLAG_NAN_ON_DIVIDE_BY_ZERO = 1)
      case VariancePop(_, _) => 7
      case VarianceSamp(_, nullOnDivideByZero) => 8 | (if (nullOnDivideByZero) 0 else 1 << 16)
      case StddevPop(_, _) => 9
      case StddevSamp(_, nullOnDivideByZero) => 10 | (if (nullOnDivideByZero) 0 else 1 << 16)
    }).toArray
    Lowerable(keyCols, funcs, inputs.map(_.map(e => ExprCompiler.compile(e, in))).toArray, condition.map(ExprCompiler.compile(_, in)))
  }

  def compileFilterProject(condition: Option[Expression], projectList: Seq[NamedExpression], in: Seq[Attribute]): Lowerable =
    Lowerable(Array.empty, Array.empty, projectList.map(p => Option(ExprCompiler.compile(p, in))).toArray,
      condition.map(ExprCompiler.compile(_, in)))

  // ---- FilterExec / ProjectExec with string-producing functions: Native.stringProject for string-valued outputs and for the string
  // functions inside the condition and the numeric outputs (hidden columns), Native.filterProject for the rest, Native.tableZip to
  // join them and Native.tableSelect for the projection's order.  The condition runs first, so the projections see surviving rows only.
  def hasStringFunction(condition: Option[Expression], projectList: Seq[NamedExpression]): Boolean =
    (condition.toSeq ++ projectList).exists(_.find(ExprCompiler.stringFunction).isDefined)

  final class StringStageHandles(val condHidden: Array[Long], val cond: Long, val keep: Array[Long], val strings: Array[Long],
                                 val projHidden: Array[Long], val numeric: Array[Long], val order: Array[Int]) {
    def close(): Unit = (condHidden ++ keep ++ strings ++ projHidden ++ numeric :+ cond).foreach(h => if (h != 0L) Native.exprFree(h))
  }
  final case class StringStage(condHidden: Array[ExprCompiler.Program], cond: Option[ExprCompiler.Program], keep: Array[ExprCompiler.Program],
                               strings: Array[ExprCompiler.Program], projHidden: Array[ExprCompiler.Program],
                               numeric: Array[ExprCompiler.Program], order: Array[Int]) {
    def lower(): StringStageHandles = new StringStageHandles(condHidden.map(_.create()), cond.map(_.create()).getOrElse(0L),
      keep.map(_.create()), strings.map(_.create()), projHidden.map(_.create()), numeric.map(_.create()), order)
  }

  def compileStringStage(condition: Option[Expression], projectList: Seq[NamedExpression], in: Seq[Attribute]): StringStage = {
    val ch = new ArrayBuffer[(AttributeReference, Expression)]()
    val cond = condition.map(ExprCompiler.hoist(_, ch))
    val condIn = in ++ ch.map(_._1)
    val isString = projectList.map(p => ExprCompiler.stringFunction(stripAlias(p)))
    val ph = new ArrayBuffer[(AttributeReference, Expression)]()
    val numericExprs = projectList.zip(isString).collect { case (p, false) => ExprCompiler.hoist(p, ph) }
    val projIn = in ++ ph.map(_._1)
    var ni = -1
    var si = numericExprs.length - 1
    val order = isString.map(str => if (str) { si += 1; si } else { ni += 1; ni }).toArray   // numeric outputs first, then the strings
    StringStage(ch.map(h => ExprCompiler.compileString(h._2, in)).toArray, cond.map(ExprCompiler.compile(_, condIn)),
      in.map(a => ExprCompiler.compile(a, condIn)).toArray,
      projectList.zip(isString).collect { case (p, true) => ExprCompiler.compileString(p, in) }.toArray,
      ph.map(h => ExprCompiler.compileString(h._2, in)).toArray, numericExprs.map(ExprCompiler.compile(_, projIn)).toArray, order)
  }

  /** one batch through a lowered StringStage; returns a new table */
  def runStringStage(h: StringStageHandles, table: Long, stream: Long): Long = {
    def withHidden(t: Long, progs: Array[Long]): Long =            // t ++ the string columns of progs (a new reference)
      if (progs.isEmpty) { Native.tableRetain(t); t }
      else { val s = Native.stringProject(t, progs, stream); try Native.tableZip(t, s) finally Native.tableRelease(s) }
    Native.tableRetain(table)
    var cur = table
    try {
      if (h.cond != 0L) {
        val w = withHidden(cur, h.condHidden)
        val kept = try Native.filterProject(w, h.cond, h.keep, stream) finally Native.tableRelease(w)
        Native.tableRelease(cur)
        cur = kept
      }
      val parts = new ArrayBuffer[Long]()
      try {
        if (h.numeric.nonEmpty) {
          val w = withHidden(cur, h.projHidden)
          parts += (try Native.filterProject(w, 0L, h.numeric, stream) finally Native.tableRelease(w))
        }
        if (h.strings.nonEmpty) parts += Native.stringProject(cur, h.strings, stream)
        if (parts.isEmpty) Native.tableSelect(cur, Array.empty[Int])
        else if (parts.length == 1) Native.tableSelect(parts(0), h.order)
        else {
          val all = Native.tableZip(parts(0), parts(1))
          try Native.tableSelect(all, h.order) finally Native.tableRelease(all)
        }
      } finally parts.foreach(Native.tableRelease)
    } finally Native.tableRelease(cur)
  }

  def ordinals(keys: Seq[Expression], in: Seq[Attribute]): Array[Int] =
    keys.map { case a: AttributeReference => in.indexWhere(_.exprId == a.exprId) }.toArray

  def orders(sortOrder: Seq[SortOrder], in: Seq[Attribute]): (Array[Int], Array[Boolean], Array[Boolean]) =
    (ordinals(sortOrder.map(_.child), in), sortOrder.map(_.direction == Ascending).toArray,
      sortOrder.map(_.nullOrdering == NullsFirst).toArray)

  // ---- joins -------------------------------------------------------------------------------------------------------------
  def buildSideFor(j: SortMergeJoinExec): BuildSide = j.joinType match {
    case RightOuter => BuildLeft                      // hash the non-preserved side when there is one
    case _ => BuildRight
  }
  def emitsBothSides(jt: JoinType): Boolean = jt match { case _: InnerLike | LeftOuter | RightOuter | FullOuter => true; case _ => false }
  def preservesBuildSide(jt: JoinType, side: BuildSide): Boolean = jt match {
    case FullOuter => true
    case LeftOuter => side == BuildLeft
    case RightOuter => side == BuildRight
    case _ => false
  }
  /** SB_JOIN_* as seen from the streamed side (include/spark_b200.h) */
  def nativeJoinType(jt: JoinType, side: BuildSide, nullAware: Boolean): Int = jt match {
    case _: InnerLike => 0
    case LeftOuter => if (side == BuildRight) 1 else 5
    case RightOuter => if (side == BuildLeft) 1 else 5
    case FullOuter => 4
    case LeftSemi => 2
    case LeftAnti => if (nullAware) 7 else 3
    case _: ExistenceJoin => 6
    case x => throw new B200Exception(5, s"join type $x")
  }

  // ---- partitioning -----------------------------------------------------------------------------------------------------------
  sealed trait PartDesc extends Serializable { def apply(table: Long, n: Int, stream: Long, offs: Array[Long]): Long }
  final case class HashDesc(keys: Array[Int]) extends PartDesc {
    def apply(table: Long, n: Int, stream: Long, offs: Array[Long]): Long = Native.hashPartition(table, keys, n, stream, offs)
  }
  final case class RoundRobinDesc() extends PartDesc {
    // the start position is XORShiftRandom(partitionId).nextInt(n) in the reference (ShuffleExchangeExec.scala:428-442): unpinned
    def apply(table: Long, n: Int, stream: Long, offs: Array[Long]): Long =
      Native.roundRobinPartition(table, new org.apache.spark.util.random.XORShiftRandom(org.apache.spark.TaskContext.getPartitionId()).nextInt(n), n, stream, offs)
  }
  final case class RangeDesc(col: Int, ascending: Boolean, nullsFirst: Boolean, samplePoints: Int) extends PartDesc {
    def apply(table: Long, n: Int, stream: Long, offs: Array[Long]): Long = {
      // RangePartitioner: sample every input partition, all-gather the candidates, determineBounds (Partitioner.scala:203-236, 357-388)
      val perPartition = math.ceil(3.0 * math.min(samplePoints.toDouble * n, 1e6) / B200Plugin.worldSize()).toLong
      val sample = Native.rangeSample(table, col, ascending, nullsFirst, perPartition, org.apache.spark.TaskContext.getPartitionId(), stream)
      val all = try Native.allGather(sample, stream) finally Native.tableRelease(sample)
      val bounds = try Native.rangeDetermineBounds(all, ascending, nullsFirst, n, stream) finally Native.tableRelease(all)
      try Native.rangePartition(table, col, ascending, nullsFirst, bounds, stream, offs) finally Native.tableRelease(bounds)
    }
  }
  def describePartitioning(p: Partitioning, in: Seq[Attribute]): PartDesc = p match {
    case HashPartitioning(keys, _) => HashDesc(ordinals(keys, in))
    case RoundRobinPartitioning(_) => RoundRobinDesc()
    case SinglePartition => HashDesc(Array.empty)                      // every row hashes to the seed: one bucket
    case RangePartitioning(ordering, _) =>
      RangeDesc(ordinals(ordering.map(_.child), in).head, ordering.head.direction == Ascending, ordering.head.nullOrdering == NullsFirst,
        SQLConf.get.rangeExchangeSampleSizePerPartition)
  }

  /** [source rank][owned partition + 1] row offsets inside the received table (grouped by source, partition-contiguous inside) */
  def sourceBlockOffsets(counts: Array[Long], n: Int, lo: Int, hi: Int, world: Int): Array[Array[Long]] = {
    var base = 0L
    Array.tabulate(world) { src =>
      val offs = new Array[Long](hi - lo + 1)
      offs(0) = base
      var p = lo
      while (p < hi) { offs(p - lo + 1) = offs(p - lo) + counts(src * n + p); p += 1 }
      base = offs(hi - lo)
      offs
    }
  }

  // ---- batches ------------------------------------------------------------------------------------------------------------------
  /** All batches of a partition as ONE device table (operators that need the whole partition: sort, join build).  null when the
   *  partition is empty unless orEmpty. */
  def concatToDevice(batches: Iterator[ColumnarBatch], types: Array[DataType], stream: Long, orEmpty: Boolean = false): DeviceBatch = {
    val parts = new ArrayBuffer[DeviceBatch]()
    while (batches.hasNext) parts += DeviceTransfer.toDevice(batches.next(), types, stream)
    if (parts.isEmpty) return if (orEmpty) emptyDeviceBatch(types, stream) else null
    if (parts.length == 1) return parts.head
    try new DeviceBatch(Native.tableConcat(parts.map(_.table).toArray, stream), types) finally parts.foreach(_.close())
  }

  def emptyDeviceBatch(types: Array[DataType], stream: Long): DeviceBatch = {
    val n = types.length
    val t = Native.tableImportHost(types.map(GpuExec.typeId), new Array[Long](n), new Array[Long](n), new Array[Long](n), new Array[Long](n),
      new Array[Long](n), stream)
    new DeviceBatch(t, types)
  }

  /** SinglePartition exchange of small per-partition results (top-k candidates): all-gather, then only rank 0 keeps them. */
  def gatherToSinglePartition(rdd: RDD[ColumnarBatch], types: Array[DataType]): RDD[ColumnarBatch] =
    rdd.barrier().mapPartitions { batches =>
      val stream = GpuExec.taskStream()
      val in = concatToDevice(batches, types, stream, orEmpty = true)
      val all = try Native.allGather(in.table, stream) finally in.close()
      if (org.apache.spark.TaskContext.getPartitionId() == 0) Iterator.single(new DeviceBatch(all, types): ColumnarBatch)
      else { Native.tableRelease(all); Iterator.empty }
    }.coalesce(1)
}

/**
 * Catalyst expression -> postfix sb_expr program (include/spark_b200.h SB_OP_*): null-propagating arithmetic and comparisons,
 * Kleene AND / OR, casts between the numeric classes.  `supported` is the single source of truth for what may be offloaded.
 */
object ExprCompiler {
  final case class Program(ops: Array[Int], vtypes: Array[Int], args: Array[Int], args2: Array[Int], literals: Array[Long], bytes: Array[Byte],
                           outType: Int) {
    def create(): Long = Native.exprCreate(ops, vtypes, args, args2, literals, bytes, outType)
  }
  // String tests run on the GPU against foldable literals over a column of the UTF8_BINARY collation (byte order = Spark's order);
  // they become SB_OP_STR_* leaves that name the column, the literal bytes travel in the program's pool.
  private def binaryString(dt: DataType): Boolean = dt match {
    case st: StringType => st.isUTF8BinaryCollation
    case _ => false
  }
  private def strCol(e: Expression): Boolean = e match {
    case a: AttributeReference => binaryString(a.dataType)
    case _ => false
  }
  private def strLit(e: Expression): Boolean = e match {
    case Literal(v, dt) => v != null && binaryString(dt)
    case _ => false
  }
  private val strCmpOps: PartialFunction[Expression, Int] = {        // SB_OP_STR_EQ .. SB_OP_STR_GE
    case _: EqualTo => 50; case _: LessThan => 51; case _: LessThanOrEqual => 52; case _: GreaterThan => 53; case _: GreaterThanOrEqual => 54
  }
  private def strCompare(b: BinaryComparison): Boolean =
    strCmpOps.isDefinedAt(b) && ((strCol(b.left) && strLit(b.right)) || (strLit(b.left) && strCol(b.right)))
  private def vt(dt: DataType): Int = dt match {       // SB_VT_*
    case BooleanType => 1
    case ByteType | ShortType | IntegerType | DateType => 2
    case LongType | TimestampType | TimestampNTZType => 3
    case FloatType | DoubleType => 4
    case _ => -1
  }
  def supported(e: Expression): Boolean = e match {
    case b: BinaryComparison if strCompare(b) => true
    case In(c, list) if strCol(c) && list.forall(l => l.isInstanceOf[Literal] && binaryString(l.dataType)) => true
    case InSet(c, _) if strCol(c) => true
    case StartsWith(c, l) => strCol(c) && strLit(l)
    case EndsWith(c, l) => strCol(c) && strLit(l)
    case Contains(c, l) => strCol(c) && strLit(l)
    case Like(c, l, _) => strCol(c) && strLit(l)
    case OctetLength(c) => strCol(c)
    case Length(c) => strCol(c)
    case a: AttributeReference => GpuExec.typeId(a.dataType) > 0
    case Alias(c, _) => supported(c)
    case l: Literal => vt(l.dataType) > 0        // a NULL literal too: LIT_NULL carries its class (an untyped NULL has none)
    case Add(l, r, _) => vt(e.dataType) > 1 && supported(l) && supported(r)
    case Subtract(l, r, _) => vt(e.dataType) > 1 && supported(l) && supported(r)
    case Multiply(l, r, _) => vt(e.dataType) > 1 && supported(l) && supported(r)
    case Divide(l, r, _) => e.dataType == DoubleType && supported(l) && supported(r)
    case UnaryMinus(c, _) => vt(c.dataType) > 1 && supported(c)
    case b: BinaryComparison => vt(b.left.dataType) > 0 && vt(b.left.dataType) == vt(b.right.dataType) && supported(b.left) && supported(b.right)
    case And(l, r) => supported(l) && supported(r)
    case Or(l, r) => supported(l) && supported(r)
    case Not(c) => supported(c)
    case IsNull(c) => supported(c)
    case IsNotNull(c) => supported(c)
    case Cast(c, to, _, _) => vt(to) > 1 && vt(c.dataType) > 0 && supported(c)
    case _ => false
  }
  // ---- string-producing functions (csrc/strfunc.cu, SB_OP_SF_*): programs of their own, run by Native.stringProject.  Positions,
  // lengths and pad lengths are int literals; trim strings, pads and separators string literals (NULL gives the function's NULL);
  // string operands are UTF8_BINARY columns, string literals or other such functions.
  private def intLit(e: Expression): Boolean = e match { case Literal(_, IntegerType) => true; case _ => false }
  private def strArg(e: Expression): Boolean = e match { case Literal(_, dt) => binaryString(dt); case _ => false }
  private def strOperand(e: Expression): Boolean = e match {
    case a: AttributeReference => binaryString(a.dataType)
    case Literal(_, dt) => binaryString(dt)
    case _ => stringFunction(e)
  }
  def stringFunction(e: Expression): Boolean = binaryString(e.dataType) && (e match {
    case Substring(s, p, l) => strOperand(s) && intLit(p) && intLit(l)
    case Concat(cs) => cs.forall(strOperand)
    case ConcatWs(sep +: cs) => strArg(sep) && cs.forall(strOperand)
    case StringTrim(s, t) => strOperand(s) && t.forall(strArg)
    case StringTrimLeft(s, t) => strOperand(s) && t.forall(strArg)
    case StringTrimRight(s, t) => strOperand(s) && t.forall(strArg)
    case StringLPad(s, l, p) => strOperand(s) && intLit(l) && strArg(p)
    case StringRPad(s, l, p) => strOperand(s) && intLit(l) && strArg(p)
    case _ => false
  })
  /** byte ranges a value is assembled from (SB_SF_MAX_RANGES = 16); a node never has fewer than its operands together */
  private def ranges(e: Expression): Int = e match {
    case Concat(cs) => math.max(1, cs.map(ranges).sum)
    case ConcatWs(_ +: cs) => math.max(1, cs.map(ranges).sum + cs.length - 1)
    case StringLPad(s, _, _) => ranges(s) + 1
    case StringRPad(s, _, _) => ranges(s) + 1
    case Substring(s, _, _) => ranges(s)
    case StringTrim(s, _) => ranges(s)
    case StringTrimLeft(s, _) => ranges(s)
    case StringTrimRight(s, _) => ranges(s)
    case _ => 1
  }
  def stringProgramOk(e: Expression): Boolean = stringFunction(e) && ranges(e) <= 16
  /** `e` with every string function replaced by a hidden string column; the (column, function) pairs are appended to `out` */
  def hoist(e: Expression, out: ArrayBuffer[(AttributeReference, Expression)]): Expression = e.transformDown {
    case f if stringFunction(f) =>
      val a = AttributeReference(s"_sf${out.length}", f.dataType, f.nullable)()
      out += ((a, f))
      a
  }
  def compileString(e: Expression, in: Seq[Attribute]): Program = {
    val ops = new ArrayBuffer[Int](); val args = new ArrayBuffer[Int](); val args2 = new ArrayBuffer[Int](); val lits = new ArrayBuffer[Long]()
    val pool = new java.io.ByteArrayOutputStream()
    def emit(op: Int, arg: Int = 0, lit: Long = 0L, arg2: Int = 0): Unit = { ops += op; args += arg; lits += lit; args2 += arg2 }
    def slice(b: Array[Byte]): Long = { val off = pool.size().toLong; pool.write(b, 0, b.length); (off << 32) | b.length.toLong }
    def intOf(l: Expression): Option[Int] = Option(l.asInstanceOf[Literal].value).map(_.asInstanceOf[Int])
    def strOf(l: Expression): Option[Array[Byte]] = Option(l.asInstanceOf[Literal].value).map(_.asInstanceOf[UTF8String].getBytes)
    def nullString(): Unit = emit(71, 0, 0L, 1)                          // SB_OP_SF_LIT, arg2 = 1: NULL
    def trim(op: Int, s: Expression, t: Option[Expression]): Unit = t match {
      case None => go(s); emit(op)
      case Some(l) => strOf(l) match { case Some(b) => go(s); emit(op, 1, slice(b)); case None => nullString() }
    }
    def pad(op: Int, s: Expression, l: Expression, p: Expression): Unit = (intOf(l), strOf(p)) match {
      case (Some(n), Some(b)) => go(s); emit(op, n, slice(b))
      case _ => nullString()
    }
    def go(x: Expression): Unit = x match {
      case Alias(c, _) => go(c)
      case a: AttributeReference => emit(70, in.indexWhere(_.exprId == a.exprId))
      case Literal(null, _) => nullString()
      case Literal(v, _) => emit(71, 0, slice(v.asInstanceOf[UTF8String].getBytes))
      case Substring(s, p, l) => (intOf(p), intOf(l)) match {
        case (Some(pi), Some(li)) => go(s); emit(72, pi, 0L, li)
        case _ => nullString()
      }
      case Concat(cs) => if (cs.isEmpty) emit(71, 0, slice(Array.emptyByteArray)) else { cs.foreach(go); emit(73, cs.length) }
      case ConcatWs(sep +: cs) => strOf(sep) match {
        case None => nullString()
        case Some(b) => if (cs.isEmpty) emit(71, 0, slice(Array.emptyByteArray)) else { cs.foreach(go); emit(74, cs.length, slice(b)) }
      }
      case StringTrim(s, t) => trim(75, s, t)
      case StringTrimLeft(s, t) => trim(76, s, t)
      case StringTrimRight(s, t) => trim(77, s, t)
      case StringLPad(s, l, p) => pad(78, s, l, p)
      case StringRPad(s, l, p) => pad(79, s, l, p)
      case other => throw new B200Exception(5, s"string function $other is not supported on the GPU path")
    }
    go(e)
    Program(ops.toArray, Array.fill(ops.length)(0), args.toArray, args2.toArray, lits.toArray, pool.toByteArray, GpuExec.typeId(StringType))
  }

  def compile(e: Expression, in: Seq[Attribute]): Program = {
    val ops = new ArrayBuffer[Int](); val vts = new ArrayBuffer[Int](); val args = new ArrayBuffer[Int](); val lits = new ArrayBuffer[Long]()
    val args2 = new ArrayBuffer[Int](); val pool = new java.io.ByteArrayOutputStream()
    def emit(op: Int, v: Int, arg: Int = 0, lit: Long = 0L, arg2: Int = 0): Unit = { ops += op; vts += v; args += arg; lits += lit; args2 += arg2 }
    def slice(b: Array[Byte]): Long = { val off = pool.size().toLong; pool.write(b, 0, b.length); (off << 32) | b.length.toLong }
    def colOf(c: Expression): Int = in.indexWhere(_.exprId == c.asInstanceOf[AttributeReference].exprId)
    def bytesOf(l: Expression): Array[Byte] = l.asInstanceOf[Literal].value.asInstanceOf[UTF8String].getBytes
    def strTest(op: Int, c: Expression, l: Expression, arg2: Int = 0): Unit = emit(op, 1, colOf(c), slice(bytesOf(l)), arg2)
    def strIn(c: Expression, values: Seq[Any]): Unit = {                 // [count][length][bytes]... in the host's byte order
      val present = values.filter(_ != null).map(_.asInstanceOf[UTF8String].getBytes)
      val buf = java.nio.ByteBuffer.allocate(4 + present.map(4 + _.length).sum).order(java.nio.ByteOrder.nativeOrder())
      buf.putInt(present.length)
      present.foreach { b => buf.putInt(b.length); buf.put(b) }
      emit(55, 1, colOf(c), slice(buf.array()), if (present.length != values.length) 1 else 0)
    }
    def bin(op: Int, l: Expression, r: Expression, v: Int, arg: Int = 0): Unit = { go(l); go(r); emit(op, v, arg) }
    def go(x: Expression): Unit = x match {
      case b: BinaryComparison if strCompare(b) =>                       // the column on the left: 'x' < s is s > 'x'
        val flipped = strLit(b.left)
        val op = strCmpOps(b)
        val op2 = if (!flipped) op else op match { case 51 => 53; case 52 => 54; case 53 => 51; case 54 => 52; case o => o }
        if (flipped) strTest(op2, b.right, b.left) else strTest(op2, b.left, b.right)
      case In(c, list) if strCol(c) => strIn(c, list.map(_.asInstanceOf[Literal].value))
      case InSet(c, hset) if strCol(c) => strIn(c, hset.toSeq)
      case StartsWith(c, l) => strTest(56, c, l)
      case EndsWith(c, l) => strTest(57, c, l)
      case Contains(c, l) => strTest(58, c, l)
      case Like(c, l, esc) => strTest(59, c, l, esc.toInt)
      case OctetLength(c) => emit(60, 2, colOf(c))
      case Length(c) => emit(61, 2, colOf(c))        // SB_OP_STR_CHAR_LENGTH: code points as UTF8String.numChars counts them
      case a: AttributeReference => emit(1, vt(a.dataType), in.indexWhere(_.exprId == a.exprId))
      case Alias(c, _) => go(c)
      case Literal(null, dt) => emit(4, vt(dt))
      case Literal(v, dt) => vt(dt) match {
        case 4 => emit(3, 4, 0, java.lang.Double.doubleToRawLongBits(v.asInstanceOf[Number].doubleValue()))
        case 1 => emit(2, 1, 0, if (v.asInstanceOf[Boolean]) 1L else 0L)
        case t => emit(2, t, 0, v.asInstanceOf[Number].longValue())
      }
      case Add(l, r, _) => bin(10, l, r, vt(x.dataType))
      case Subtract(l, r, _) => bin(11, l, r, vt(x.dataType))
      case Multiply(l, r, _) => bin(12, l, r, vt(x.dataType))
      case Divide(l, r, _) => bin(13, l, r, 4)
      case UnaryMinus(c, _) => go(c); emit(14, vt(c.dataType))
      case b: BinaryComparison =>
        val op = b match { case _: EqualTo => 20; case _: LessThan => 22; case _: LessThanOrEqual => 23; case _: GreaterThan => 24
                           case _: GreaterThanOrEqual => 25; case other => throw new B200Exception(5, s"comparison $other") }
        bin(op, b.left, b.right, 1, vt(b.left.dataType))                 // arg = operand class (the kernels compare doubles with NaN largest)
      case And(l, r) => bin(30, l, r, 1)
      case Or(l, r) => bin(31, l, r, 1)
      case Not(c) => go(c); emit(32, 1)
      case IsNull(c) => go(c); emit(33, 1)
      case IsNotNull(c) => go(c); emit(34, 1)
      case Cast(c, to, _, _) => go(c); emit(vt(to) match { case 4 => 40; case 3 => 41; case _ => 42 }, vt(to), vt(c.dataType))   // arg = source class
      case other => throw new B200Exception(5, s"expression $other is not supported on the GPU path")
    }
    go(e)
    Program(ops.toArray, vts.toArray, args.toArray, args2.toArray, lits.toArray, pool.toByteArray, GpuExec.typeId(e.dataType))
  }
}
