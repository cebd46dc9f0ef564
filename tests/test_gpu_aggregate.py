"""GPU parity: HashAggregateExec (+ fused FilterExec/ProjectExec) vs the oracle."""
import numpy as np
import pyarrow as pa
import pytest

from oracle import oracle as O
from util import assert_tables_equal

pytestmark = pytest.mark.gpu


def _run(plan_fn, t, stream):
    from spark_b200.columnar import ColumnarBatch
    from spark_b200.execution import LocalTableScanExec
    batch = ColumnarBatch.from_arrow(t, stream)
    return plan_fn(LocalTableScanExec(batch)).collect(stream)


# configs[0] of BASELINE.json: SELECT k, SUM(v) GROUP BY k on a 1M-row two-column DataFrame
@pytest.mark.parametrize("groups", [4, 1024, 65536, 1 << 20])
@pytest.mark.parametrize("vtype", ["int64", "float64"])
def test_c1_group_by_sum(gpu, stream, groups, vtype):
    from spark_b200.execution import HashAggregateExec
    from spark_b200.expressions import Sum, col
    n = 1 << 20
    rng = np.random.default_rng(42)
    k = rng.integers(0, groups, n)
    v = rng.integers(-2 ** 31, 2 ** 31, n) if vtype == "int64" else rng.random(n) * 1e4
    t = pa.table({"k": k, "v": v})
    got = _run(lambda scan: HashAggregateExec(["k"], [(Sum(col("v")), "sum_v")], scan), t, stream)
    want = O.hash_aggregate(t, ["k"], [("sum", "v", "sum_v")])
    assert_tables_equal(got, want, key_cols=["k"])


def test_all_functions_nulls_and_null_keys(gpu, stream):
    from spark_b200.execution import HashAggregateExec
    from spark_b200.expressions import Average, Count, Max, Min, Sum, col
    n = 50000
    rng = np.random.default_rng(7)
    d = rng.standard_normal(n)
    d[rng.random(n) < 0.01] = np.nan
    t = pa.table({"k1": pa.array(rng.integers(0, 50, n).astype(np.int32), mask=rng.random(n) < 0.05),
                  "k2": pa.array(rng.integers(0, 3, n).astype(np.int8), mask=rng.random(n) < 0.05),
                  "v": pa.array(rng.integers(-10 ** 12, 10 ** 12, n), mask=rng.random(n) < 0.3),
                  "d": pa.array(d, mask=rng.random(n) < 0.3),
                  "i": pa.array(rng.integers(-1000, 1000, n).astype(np.int32), mask=rng.random(n) < 0.3)})
    aggs = [(Sum(col("v")), "sv"), (Sum(col("d")), "sd"), (Average(col("d")), "ad"), (Average(col("i")), "ai"),
            (Count(col("v")), "cv"), (Count(), "n"), (Min(col("v")), "mnv"), (Max(col("v")), "mxv"),
            (Min(col("d")), "mnd"), (Max(col("d")), "mxd"), (Min(col("i")), "mni")]
    oaggs = [("sum", "v", "sv"), ("sum", "d", "sd"), ("avg", "d", "ad"), ("avg", "i", "ai"), ("count", "v", "cv"),
             ("count_star", None, "n"), ("min", "v", "mnv"), ("max", "v", "mxv"), ("min", "d", "mnd"), ("max", "d", "mxd"),
             ("min", "i", "mni")]
    got = _run(lambda scan: HashAggregateExec(["k1", "k2"], aggs, scan), t, stream)
    want = O.hash_aggregate(t, ["k1", "k2"], oaggs)
    assert_tables_equal(got, want, key_cols=["k1", "k2"])


@pytest.mark.parametrize("ktype", ["int64", "float64", "date32", "bool"])
def test_single_key_types_including_sentinel_and_null(gpu, stream, ktype):
    from spark_b200.execution import HashAggregateExec
    from spark_b200.expressions import Count, Sum, col
    n = 20000
    rng = np.random.default_rng(11)
    if ktype == "int64":
        k = rng.integers(-5, 5, n)
        k[:10] = -1                      # 0xFFFF... is the table's EMPTY sentinel
        k[10:20] = 2 ** 63 - 1
        karr = pa.array(k, mask=rng.random(n) < 0.1)
    elif ktype == "float64":
        k = rng.integers(-3, 3, n).astype(np.float64)
        k[rng.random(n) < 0.1] = -0.0    # must group with 0.0 (NormalizeFloatingNumbers)
        k[rng.random(n) < 0.1] = np.nan
        karr = pa.array(k, mask=rng.random(n) < 0.1)
    elif ktype == "date32":
        karr = pa.array(rng.integers(0, 40, n).astype(np.int32), mask=rng.random(n) < 0.1).cast(pa.date32())
    else:
        karr = pa.array(rng.integers(0, 2, n).astype(bool), mask=rng.random(n) < 0.1)
    t = pa.table({"k": karr, "v": rng.integers(0, 100, n)})
    got = _run(lambda scan: HashAggregateExec(["k"], [(Sum(col("v")), "s"), (Count(), "c")], scan), t, stream)
    want = O.hash_aggregate(t, ["k"], [("sum", "v", "s"), ("count_star", None, "c")])
    if ktype == "float64":
        # compare NaN/-0.0 keys by bit-normalised value
        norm = lambda tb: tb.set_column(0, "k", pa.array([None if x is None else (float("nan") if x != x else x + 0.0)
                                                          for x in tb.column("k").to_pylist()]))
        got, want = norm(got), norm(want)
    assert_tables_equal(got, want, key_cols=["k"])


def test_partial_exchange_final_equals_complete(gpu, stream):
    """AggUtils.scala:131-208 mode algebra: Partial on two 'map tasks' -> concat -> Final == Complete."""
    from spark_b200.columnar import ColumnarBatch
    from spark_b200.execution import HashAggregateExec, LocalTableScanExec
    from spark_b200.expressions import Average, Count, Max, Sum, col
    n = 40000
    rng = np.random.default_rng(3)
    t = pa.table({"k": rng.integers(0, 300, n).astype(np.int32),
                  "v": pa.array(rng.integers(-1000, 1000, n), mask=rng.random(n) < 0.2), "d": rng.random(n)})
    aggs = [(Sum(col("v")), "s"), (Average(col("d")), "a"), (Count(col("v")), "c"), (Count(), "n"), (Max(col("d")), "mx")]
    oaggs = [("sum", "v", "s"), ("avg", "d", "a"), ("count", "v", "c"), ("count_star", None, "n"), ("max", "d", "mx")]
    parts = []
    for half in (t.slice(0, n // 2), t.slice(n // 2)):
        b = ColumnarBatch.from_arrow(half, stream)
        parts.append(HashAggregateExec(["k"], aggs, LocalTableScanExec(b), mode="partial").collect(stream))
        want_partial = O.hash_aggregate(half, ["k"], oaggs, "partial")
        assert_tables_equal(parts[-1], want_partial, key_cols=["k"])
    merged = pa.concat_tables(parts)
    b = ColumnarBatch.from_arrow(merged, stream)
    got = HashAggregateExec(["k"], aggs, LocalTableScanExec(b), mode="final").collect(stream)
    want = O.hash_aggregate(t, ["k"], oaggs, "complete")
    assert_tables_equal(got, want, key_cols=["k"])


def test_global_aggregate_without_keys_and_empty_input(gpu, stream):
    from spark_b200.execution import HashAggregateExec
    from spark_b200.expressions import Average, Count, Sum, col
    t = pa.table({"v": pa.array([1, 2, None, 4], type=pa.int64()), "d": [0.5, 1.5, 2.5, 3.5]})
    aggs = [(Sum(col("v")), "s"), (Average(col("d")), "a"), (Count(), "n")]
    got = _run(lambda scan: HashAggregateExec([], aggs, scan), t, stream)
    assert got.to_pydict() == {"s": [7], "a": [2.0], "n": [4]}
    empty = t.slice(0, 0)
    got = _run(lambda scan: HashAggregateExec([], aggs, scan), empty, stream)
    assert got.to_pydict() == {"s": [None], "a": [None], "n": [0]}     # one row even for empty input
    got = _run(lambda scan: HashAggregateExec(["v"], aggs[1:], scan), empty, stream)
    assert got.num_rows == 0


def _q1_oracle(t):
    from spark_b200 import tpch
    f = O.filter_table(t, ("le", ("col", "l_shipdate"), ("lit", tpch.Q1_CUTOFF, np.int32)))
    dp = ("mul", ("col", "l_extendedprice"), ("sub", ("lit", 1.0), ("col", "l_discount")))
    p = O.project(f, [(c, ("col", c)) for c in ["l_returnflag", "l_linestatus", "l_quantity", "l_extendedprice", "l_discount"]] +
                  [("disc_price", dp), ("charge", ("mul", dp, ("add", ("lit", 1.0), ("col", "l_tax"))))])
    return O.hash_aggregate(p, ["l_returnflag", "l_linestatus"], tpch.q1_oracle_aggs())


@pytest.mark.parametrize("fused", [True, False])
def test_tpch_q1_fused_and_unfused(gpu, stream, fused):
    """configs[1] shape at a size the oracle finishes in seconds; the fused plan (FilterExec/ProjectExec inside the
    aggregate kernel) and the operator-by-operator plan must both equal the oracle."""
    from spark_b200 import tpch
    from spark_b200.columnar import ColumnarBatch
    from spark_b200.execution import LocalTableScanExec
    t = tpch.lineitem_q1_table(600_000, seed=5)
    batch = ColumnarBatch.from_arrow(t, stream)
    partial = tpch.q1_partial_plan(LocalTableScanExec(batch), fused=fused)
    got = tpch.q1_final_plan(partial, sort=False).collect(stream)
    assert_tables_equal(got, _q1_oracle(t), key_cols=["l_returnflag", "l_linestatus"])


def test_fusion_rule_produces_same_result(gpu, stream):
    from spark_b200 import tpch
    from spark_b200.columnar import ColumnarBatch
    from spark_b200.execution import B200ColumnarRule, HashAggregateExec, LocalTableScanExec
    t = tpch.lineitem_q1_table(100_000, seed=6)
    batch = ColumnarBatch.from_arrow(t, stream)
    plan = tpch.q1_partial_plan(LocalTableScanExec(batch), fused=False)
    fused = B200ColumnarRule().preColumnarTransitions(plan)
    assert isinstance(fused, HashAggregateExec) and isinstance(fused.child, LocalTableScanExec) and fused.condition is not None
    got = tpch.q1_final_plan(fused, sort=False).collect(stream)
    assert_tables_equal(got, _q1_oracle(t), key_cols=["l_returnflag", "l_linestatus"])


def test_general_expressions_take_the_materialising_path(gpu, stream):
    """Predicate with OR / arithmetic and an aggregate input that is not a product form."""
    from spark_b200.execution import HashAggregateExec
    from spark_b200.expressions import Literal, Sum, col
    n = 30000
    rng = np.random.default_rng(8)
    t = pa.table({"k": rng.integers(0, 20, n).astype(np.int32), "a": pa.array(rng.integers(-50, 50, n), mask=rng.random(n) < 0.1),
                  "b": rng.integers(-50, 50, n), "x": rng.random(n), "y": pa.array(rng.random(n), mask=rng.random(n) < 0.1)})
    cond = ((col("a") + col("b")) > Literal(0)) | (col("x") < col("y"))
    aggs = [(Sum(col("a") * col("b") - Literal(3)), "s1"), (Sum((col("x") + col("y")) / (col("b"))), "s2")]
    got = _run(lambda scan: HashAggregateExec(["k"], aggs, scan, condition=cond), t, stream)
    f = O.filter_table(t, cond.sexpr())
    p = O.project(f, [("k", ("col", "k")), ("e1", aggs[0][0].child.sexpr()), ("e2", aggs[1][0].child.sexpr())])
    want = O.hash_aggregate(p, ["k"], [("sum", "e1", "s1"), ("sum", "e2", "s2")])
    assert_tables_equal(got, want, key_cols=["k"])


def test_filter_project_operator(gpu, stream):
    from spark_b200.execution import FilterExec, ProjectExec
    from spark_b200.expressions import Literal, col
    n = 10000
    rng = np.random.default_rng(2)
    t = pa.table({"a": pa.array(rng.integers(-100, 100, n).astype(np.int32), mask=rng.random(n) < 0.1),
                  "x": pa.array(rng.standard_normal(n), mask=rng.random(n) < 0.1),
                  "s": pa.array(["v%d" % i if i % 7 else None for i in range(n)])})
    cond = (col("a") >= Literal(-10)) & col("x").is_not_null()
    proj = [("a", col("a")), ("s", col("s")), ("e", col("x") * Literal(2.0) + col("a")), ("q", col("x") / col("a"))]
    got = _run(lambda scan: ProjectExec(proj, FilterExec(cond, scan)), t, stream)
    want = O.project(O.filter_table(t, cond.sexpr()), [(n_, e.sexpr()) for n_, e in proj])
    assert_tables_equal(got, want, ordered=True)


@pytest.mark.parametrize("env", [{"agg_rtc_min_rows": 0}, {"agg_rtc": 0},
                                 {"agg_tier": 2, "agg_rtc_min_rows": 0}, {"agg_tier": 1, "agg_rtc_min_rows": 0}, {"agg_tier": 2, "agg_rtc": 0},
                                 {"agg_tier": 1, "agg_rtc": 0}],
                         ids=["rtc-chain", "generic-chain", "rtc-smem-tier", "rtc-dict-tier", "generic-smem-tier", "generic-dict-tier"])
def test_every_update_kernel_variant_matches_the_oracle(gpu, stream, env, sbconfig):
    """The run-time specialised (NVRTC, StaticPlan) and generic (DynPlan) update kernels share one code base; each variant
    must produce the oracle's Q1 answer, including a ragged last tile and a NULL-able variant of the plan."""
    from spark_b200 import tpch
    from spark_b200.columnar import ColumnarBatch
    from spark_b200.execution import HashAggregateExec, LocalTableScanExec
    from spark_b200.expressions import Average, Count, Literal, Max, Sum, col
    from spark_b200 import _capi as capi
    for k, v in env.items():
        sbconfig(k, v)
    t = tpch.lineitem_q1_table(300_017, seed=21)          # not a multiple of any tile size
    batch = ColumnarBatch.from_arrow(t, stream)
    got = tpch.q1_final_plan(tpch.q1_partial_plan(LocalTableScanExec(batch), fused=True), sort=False).collect(stream)
    assert_tables_equal(got, _q1_oracle(t), key_cols=["l_returnflag", "l_linestatus"])
    if env.get("agg_rtc_min_rows") == 0:   # the specialised kernels really ran (the Final stage's 4 rows run generic: check the log of Partial)
        part = tpch.q1_partial_plan(LocalTableScanExec(batch), fused=True).executeColumnar(stream)
        part.close()
        assert capi.load().sb_hash_aggregate_last_plan().decode().startswith("rtc:"), capi.load().sb_hash_aggregate_last_plan()
    # same shape with NULLs in a key, an input and the filter column -> never matches a static table, exercises the validity loads
    rng = np.random.default_rng(3)
    n = t.num_rows
    t2 = t.set_column(0, "l_quantity", pa.array(np.asarray(t.column("l_quantity")), mask=rng.random(n) < 0.1))
    t2 = t2.set_column(4, "l_returnflag", pa.array(np.asarray(t.column("l_returnflag")), mask=rng.random(n) < 0.05))
    t2 = t2.set_column(6, "l_shipdate", pa.array(np.asarray(t.column("l_shipdate").cast(pa.int32())), mask=rng.random(n) < 0.05).cast(pa.date32()))
    b2 = ColumnarBatch.from_arrow(t2, stream)
    aggs = [(Sum(col("l_quantity")), "sq"), (Average(col("l_quantity")), "aq"), (Count(col("l_quantity")), "cq"), (Count(), "n"),
            (Max(col("l_extendedprice") * (Literal(1) - col("l_discount"))), "mx")]
    cond = col("l_shipdate") <= Literal(tpch.Q1_CUTOFF)
    got2 = HashAggregateExec(["l_returnflag", "l_linestatus"], aggs, LocalTableScanExec(b2), condition=cond).collect(stream)
    f = O.filter_table(t2, cond.sexpr())
    p = O.project(f, [("l_returnflag", ("col", "l_returnflag")), ("l_linestatus", ("col", "l_linestatus")), ("l_quantity", ("col", "l_quantity")),
                      ("dp", ("mul", ("col", "l_extendedprice"), ("sub", ("lit", 1.0), ("col", "l_discount"))))])
    want2 = O.hash_aggregate(p, ["l_returnflag", "l_linestatus"], [("sum", "l_quantity", "sq"), ("avg", "l_quantity", "aq"),
                                                                    ("count", "l_quantity", "cq"), ("count_star", None, "n"), ("max", "dp", "mx")])
    assert_tables_equal(got2, want2, key_cols=["l_returnflag", "l_linestatus"])


@pytest.mark.parametrize("groups", [5, 1000, 6000, 200_000])
@pytest.mark.parametrize("tier", ["auto", "smem", "dict"])
def test_cardinality_tiers_agree_with_the_oracle(gpu, stream, groups, tier, sbconfig):
    """Few groups (lane-private dictionary), a few thousand (shared-memory table), more than the shared-memory table holds
    (spill to the HBM table, then bypass): every tier and the sampled automatic choice give the oracle's answer.  Keys include
    NULL and -1 (the bit pattern of the table's EMPTY sentinel); inputs include NULLs; min/max/avg/count ride along."""
    from spark_b200.columnar import ColumnarBatch
    from spark_b200.execution import HashAggregateExec, LocalTableScanExec
    from spark_b200.expressions import Average, Count, Max, Min, Sum, col
    if tier != "auto":
        sbconfig("agg_tier", {"dict": 1, "smem": 2}[tier])
    n = 400_037
    rng = np.random.default_rng(groups)
    k = rng.integers(-1, groups - 1, n)
    t = pa.table({"k": pa.array(k, mask=rng.random(n) < 0.03),
                  "v": pa.array(rng.integers(-2 ** 40, 2 ** 40, n), mask=rng.random(n) < 0.1),
                  "d": pa.array(rng.standard_normal(n) * 1e3)})
    aggs = [(Sum(col("v")), "sv"), (Sum(col("d")), "sd"), (Average(col("d")), "ad"), (Count(col("v")), "cv"), (Count(), "n"),
            (Min(col("v")), "mn"), (Max(col("d")), "mx")]
    got = HashAggregateExec(["k"], aggs, LocalTableScanExec(ColumnarBatch.from_arrow(t, stream))).collect(stream)
    want = O.hash_aggregate(t, ["k"], [("sum", "v", "sv"), ("sum", "d", "sd"), ("avg", "d", "ad"), ("count", "v", "cv"),
                                       ("count_star", None, "n"), ("min", "v", "mn"), ("max", "d", "mx")])
    assert_tables_equal(got, want, key_cols=["k"])


@pytest.mark.parametrize("groups", [3, 20, 1024])
@pytest.mark.parametrize("vtype", ["i64", "f64"])
def test_groupby_sum_static_shapes_through_both_tiers(gpu, stream, groups, vtype, sbconfig):
    """BASELINE configs[0] shape (k int64, v int64/double, no NULLs): the run-time specialised kernels of every tier."""
    sbconfig("agg_rtc_min_rows", 0)
    from spark_b200.columnar import ColumnarBatch
    from spark_b200.execution import HashAggregateExec, LocalTableScanExec
    from spark_b200.expressions import Sum, col
    n = 600_011
    rng = np.random.default_rng(groups + 7)
    v = rng.integers(-2 ** 31, 2 ** 31, n) if vtype == "i64" else rng.random(n) * 1e4
    t = pa.table({"k": rng.integers(0, groups, n), "v": v})
    got = HashAggregateExec(["k"], [(Sum(col("v")), "s")], LocalTableScanExec(ColumnarBatch.from_arrow(t, stream))).collect(stream)
    want = O.hash_aggregate(t, ["k"], [("sum", "v", "s")])
    assert_tables_equal(got, want, key_cols=["k"])


@pytest.mark.parametrize("interpret_only", [False, True], ids=["typed-fast-path", "interpreter"])
@pytest.mark.parametrize("n", [1, 15, 16, 17, 4097, 100_003])
def test_filter_predicates_of_every_type(gpu, stream, n, interpret_only, sbconfig):
    """FilterExec (basicPhysicalOperators.scala:245): conjunctions of column-vs-literal comparisons take the typed 16-rows-per-thread
    kernel, everything else the interpreter; both must keep exactly the oracle's rows (NULL comparisons drop the row, NaN is the
    largest double and equals itself, literal-on-the-left flips the operator), at sizes around the 16-row vector width."""
    from spark_b200.execution import FilterExec
    from spark_b200.expressions import Literal, col
    if interpret_only:
        sbconfig("expr_interpret_only", 1)
    rng = np.random.default_rng(n)
    d = rng.standard_normal(n)
    d[rng.random(n) < 0.1] = np.nan
    t = pa.table({"i8": pa.array(rng.integers(-5, 5, n).astype(np.int8), mask=rng.random(n) < 0.2),
                  "i16": pa.array(rng.integers(-300, 300, n).astype(np.int16)),
                  "i32": pa.array(rng.integers(-10, 10, n).astype(np.int32), mask=rng.random(n) < 0.1),
                  "i64": pa.array(rng.integers(-2 ** 40, 2 ** 40, n), mask=rng.random(n) < 0.1),
                  "dt": pa.array(rng.integers(9000, 9100, n).astype(np.int32)).cast(pa.date32()),
                  "f32": pa.array(rng.standard_normal(n).astype(np.float32), mask=rng.random(n) < 0.1),
                  "f64": pa.array(d, mask=rng.random(n) < 0.1),
                  "row": np.arange(n, dtype=np.int64)})
    conds = [col("i32") >= Literal(-3),
             (col("i8") < Literal(2)) & (col("i16") != Literal(7)) & col("i64").is_not_null(),
             (Literal(9050) > col("dt")) & (col("i64") <= Literal(2 ** 39)),
             (col("f64") > Literal(0.25)) & (col("f32") <= Literal(0.5)),
             col("f64").eq(Literal(float("nan"))),
             (col("i32").eq(Literal(0))) & (col("f64") >= Literal(-1.0)) & (col("i8") > Literal(-4)) & (col("dt") >= Literal(9010)),
             (col("i32") >= Literal(-3)) | (col("i8") < Literal(0))]        # OR: never the fast path
    for cond in conds:
        got = _run(lambda scan: FilterExec(cond, scan), t, stream)
        want = O.filter_table(t, cond.sexpr())
        assert got.column("row").to_pylist() == want.column("row").to_pylist(), cond.sexpr()


def test_reference_sql_golden_answers(gpu, stream):
    """The aggregate answers the reference prints in group-by.sql.out / having.sql.out (tests/sql_goldens.py), computed by the GPU
    operators: Project (computed grouping keys) -> HashAggregate -> Filter (HAVING)."""
    import sql_goldens as G
    from spark_b200.columnar import ColumnarBatch
    from spark_b200.execution import FilterExec, HashAggregateExec, LocalTableScanExec, ProjectExec
    from spark_b200.expressions import Average, Count, Literal, Max, Min, Sum, col
    fns = {"count": lambda c: Count(col(c)), "count_star": lambda c: Count(), "sum": lambda c: Sum(col(c)), "avg": lambda c: Average(col(c)),
           "min": lambda c: Min(col(c)), "max": lambda c: Max(col(c))}

    def expr(e):
        if e[0] == "col":
            return col(e[1])
        if e[0] == "lit":
            return Literal(bool(e[1]) if e[2] is np.bool_ else e[1])
        l, r = expr(e[1]), expr(e[2])
        return {"add": lambda: l + r, "gt": lambda: l > r, "eq": lambda: l.eq(r)}[e[0]]()
    for name, table, keys, proj, aggs, post, want, where in G.CASES:
        plan = LocalTableScanExec(ColumnarBatch.from_arrow(table, stream))
        if proj:
            plan = ProjectExec([(c, col(c)) for c in table.column_names] + [(n, expr(e)) for n, e in proj], plan)
        plan = HashAggregateExec(keys or [], [(fns[f](c), n) for f, c, n in aggs], plan)
        if post is not None and post != "drop_keys":
            plan = FilterExec(expr(post), plan)
        got = plan.collect(stream)
        if post == "drop_keys":
            got = got.select([n for _, _, n in aggs])
        rows = list(zip(*[got.column(i).to_pylist() for i in range(got.num_columns)])) if got.num_rows else []
        assert len(rows) == len(want), (name, where, rows, want)
        for g, w in zip(G.norm(rows), G.norm(want)):
            for x, y in zip(g, w):
                if isinstance(y, float):
                    assert abs(x - y) <= 1e-6 * abs(y), (name, where, x, y)
                else:
                    assert x == y, (name, where, g, w)
