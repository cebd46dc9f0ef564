"""Every floating SUM / AVG the GPU computes, window frames and hash-aggregate groups, checked against the correctly rounded sum
of the group's or frame's own terms (tests/float_sums.py), on data where a lossy or order-leaking accumulator shows: values of
1e20 before a frame, +-inf and NaN before / inside / after frames, alternating +-1e16 cancellation, frames of only +-0.0, all-NULL
frames, single-row partitions.  Integer SUM is bit-exact modulo 2^64, COUNT exact."""
import math
import struct

import numpy as np
import pyarrow as pa
import pytest

from float_sums import check_avg, check_sum, wrap64
from oracle import oracle as O

pytestmark = pytest.mark.gpu

INF, NAN = math.inf, math.nan
I64_MAX, I64_MIN = 2 ** 63 - 1, -2 ** 63


def _bits(x):
    return struct.pack("<d", x)


# ---------------------------------------------------------------------------------------------------------------- window
def _regimes(rng):
    """Partitions of the window table as (double values, int64 values); None = NULL."""
    small = lambda k: [float(x) for x in rng.integers(1, 9, k)]
    d = [[1e20] + small(11), [-1e20] + small(10) + [1e20], [1e20, -1e20] + small(6),
         [INF] + small(9), small(4) + [NAN] + small(5), small(8) + [-INF], [1.0, INF, 2.0, 3.0, -INF, 4.0, 5.0, 6.0, 7.0, 8.0],
         small(3) + [NAN, None, INF] + small(6),
         [1e16, 0.5, -1e16, 0.25, 1e16, 1.5, -1e16, 0.125, -1e16, 3.0, 1e16, 0.75, 1e16, -1e16, 2.5, -1e16],
         [-0.0, -0.0, None, -0.0, 0.0, -0.0, -0.0, -0.0, None, -0.0], [-0.0] * 6,
         [None] * 5 + [2.5] + [None] * 6 + [-1.25] + [None] * 4, [None] * 7,
         [-0.0], [INF], [NAN], [None], [1e20], [3.0]]
    for _ in range(60):                                             # small random partitions, several magnitudes
        k = int(rng.integers(1, 40))
        x = rng.standard_normal(k) * 10.0 ** rng.integers(-3, 12)
        d.append([None if rng.random() < 0.1 else float(v) for v in x])
    big = rng.standard_normal(2600) * 1e3                           # crosses the 2048- and 4096-row scan tiles
    big[rng.integers(0, 2600, 12)] = 1e15
    d.append([None if rng.random() < 0.05 else float(v) for v in big])
    for _ in range(60):
        k = int(rng.integers(1, 30))
        d.append([None if rng.random() < 0.1 else float(v) for v in rng.standard_normal(k) * 100])
    ints = [lambda k: [int(x) for x in rng.integers(-1000, 1000, k)], lambda k: [I64_MAX] * k, lambda k: [I64_MIN] + [-1] * (k - 1),
            lambda k: [0xFFFFFFFF] * k, lambda k: [I64_MAX if i % 2 else I64_MIN for i in range(k)],
            lambda k: [int(x) for x in rng.integers(-2 ** 62, 2 ** 62, k)], lambda k: [-1] * k]
    out = []
    for i, vals in enumerate(d):
        v = ints[i % len(ints)](len(vals))
        out.append((vals, [None if x is None else y for x, y in zip(vals, v)]))
    return out


def _window_table(seed):
    rng = np.random.default_rng(seed)
    ps, ds, vs, os_, ks = [], [], [], [], []
    specials = [-INF, INF, NAN, -0.0, 0.0, None]
    for p, (dv, iv) in enumerate(_regimes(rng)):
        n = len(dv)
        ps += [p] * n
        ds += dv
        vs += iv
        os_ += [None if rng.random() < 0.05 else (j // 2) * 3 for j in range(n)]          # peers, gaps, NULL keys
        ks += [specials[int(rng.integers(0, 6))] if rng.random() < 0.15 else j * 0.75 for j in range(n)]
    n = len(ps)
    perm = rng.permutation(n)                                       # the sort has work to do; the row column is the tie-breaker
    take = lambda xs: [xs[i] for i in perm]
    dd = take(ds)
    return pa.table({"p": pa.array(take(ps), type=pa.int64()),
                     "o": pa.array(take(os_), type=pa.int32()),
                     "k": pa.array(take(ks), type=pa.float64()),
                     "d": pa.array(dd, type=pa.float64()),
                     "f": pa.array([None if x is None else float(np.float32(x)) for x in dd], type=pa.float32()),
                     "v": pa.array(take(vs), type=pa.int64()),
                     "row": pa.array(perm, type=pa.int64())})


def _window(table, part, orders, specs, stream):
    from spark_b200.columnar import ColumnarBatch
    from spark_b200.execution import LocalTableScanExec, WindowExec, WindowFunction
    fns = [WindowFunction(f, c, fr, p, name) for f, c, fr, p, name in specs]
    return WindowExec(fns, part, orders, LocalTableScanExec(ColumnarBatch.from_arrow(table, stream))).collect(stream)


ROWS_FRAMES = [("rows", None, 0), ("rows", None, None), ("rows", -1, 1), ("rows", -3, 0), ("rows", 0, 2), ("rows", 0, 0),
               ("rows", -4, -2), ("rows", 2, 5), ("rows", 0, None), ("rows", -2, None)]
RANGE_INT_FRAMES = [("range", None, 0), ("range", -3, 2), ("range", 0, None), ("range", -7, -3), ("range", 1, 4)]
RANGE_F64_FRAMES = [("range", None, 0), ("range", -1.5, 0.75), ("range", 0, None), ("range", -2.25, -0.5), ("range", 0.5, 3.0)]
ORDERINGS = {"rows": ([("row", True, True)], ROWS_FRAMES),
             "range-int-asc": ([("o", True, True)], RANGE_INT_FRAMES),
             "range-int-desc": ([("o", False, False)], RANGE_INT_FRAMES),
             "range-f64": ([("k", True, False)], RANGE_F64_FRAMES)}


@pytest.mark.parametrize("column", ["d", "f", "v"], ids=["float64", "float32", "int64"])
@pytest.mark.parametrize("ordering", list(ORDERINGS))
def test_window_sums_depend_only_on_their_frame(gpu, stream, ordering, column):
    """SUM / AVG / COUNT over growing, whole, sliding (also wholly before / after the row), shrinking and RANGE-offset frames.
    Every output row is checked against its own frame's terms (oracle.window_frames)."""
    t = _window_table(11)
    orders, frames = ORDERINGS[ordering]
    specs = []
    for i, fr in enumerate(frames):
        specs += [("sum", column, fr, 0, "s%d" % i), ("avg", column, fr, 0, "a%d" % i), ("count", column, fr, 0, "c%d" % i)]
    got = _window(t, ["p"], orders, specs, stream)
    srt = O.window(t, ["p"], orders, [])
    assert got.column("row").to_pylist() == srt.column("row").to_pylist()      # output order = partition keys ++ order spec
    vals = srt.column(column).to_pylist()
    if column == "f":
        vals = [None if x is None else float(x) for x in vals]
    nn = [x for x in vals if x is not None]
    pos = np.concatenate([[0], np.cumsum([x is not None for x in vals])]).tolist()
    for i, fr in enumerate(frames):
        frames_of = O.window_frames(t, ["p"], orders, specs[3 * i])
        s, a, c = (got.column(n).to_pylist() for n in ("s%d" % i, "a%d" % i, "c%d" % i))
        seen = set()
        for r, (lo, hi) in enumerate(frames_of):
            terms = nn[pos[lo]:pos[hi + 1]] if lo <= hi else []
            what = "%s row %d frame [%d, %d] of %s" % (column, r, lo, hi, fr)
            assert c[r] == len(terms), what
            if not terms:
                assert s[r] is None and a[r] is None, what
                continue
            if column == "v":
                assert s[r] == wrap64(sum(terms)), what
                key = (lo, hi, _bits(a[r]))
            else:
                key = (lo, hi, _bits(s[r]), _bits(a[r]))
            if key in seen:
                continue
            seen.add(key)
            if column != "v":
                check_sum(s[r], terms, "sum " + what)
            check_avg(a[r], [float(x) for x in terms], "avg " + what)


def test_window_running_sums_over_four_million_rows(gpu, stream):
    """n > 2048^2: the segmented scan recurses twice.  One partition of 3 M rows and many small ones; values are multiples of
    2^-10 with small numerators, so every partial sum is exact and running, whole-partition, sliding and shrinking SUM and
    COUNT must equal numpy's segmented cumulative sums bit for bit."""
    rng = np.random.default_rng(5)
    big = 3_000_000
    sizes = rng.integers(1, 50, 60_000)
    sizes = sizes[np.cumsum(sizes) <= 1_200_000]
    p = np.concatenate([np.zeros(big, np.int64), np.repeat(np.arange(1, len(sizes) + 1), sizes)])
    n = len(p)
    assert n > 2048 * 2048
    x = rng.integers(-1000, 1001, n) / 1024.0
    null = rng.random(n) < 0.05
    perm = rng.permutation(n)
    t = pa.table({"p": p[perm], "x": pa.array(x[perm], mask=null[perm]), "row": np.arange(n, dtype=np.int64)})
    specs = [("sum", "x", ("rows", None, 0), 0, "run"), ("sum", "x", ("rows", None, None), 0, "all"), ("count", "x", ("rows", None, 0), 0, "cnt"),
             ("sum", "x", ("rows", -5, 5), 0, "slide"), ("sum", "x", ("rows", 0, None), 0, "rest")]
    got = _window(t, ["p"], [("row", True, True)], specs, stream)
    order = np.lexsort((np.arange(n), p[perm]))
    assert np.array_equal(np.asarray(got.column("row")), order)
    ps, xs, ns = p[perm][order], np.where(null[perm], 0.0, x[perm])[order], (~null[perm][order]).astype(np.int64)
    G, C = np.concatenate([[0.0], np.cumsum(xs)]), np.concatenate([[0], np.cumsum(ns)])
    head = np.concatenate([[True], ps[1:] != ps[:-1]])
    s = np.maximum.accumulate(np.where(head, np.arange(n), 0))
    e = np.concatenate([np.flatnonzero(head)[1:], [n]])[np.cumsum(head) - 1] - 1
    i = np.arange(n)

    def expect(lo, hi, name, what):
        want, cnt = G[hi + 1] - G[lo], C[hi + 1] - C[lo]
        col = got.column(name)
        valid = np.asarray(col.is_valid())
        assert np.array_equal(valid, cnt > 0), what
        vals = np.asarray(col.fill_null(0.0))
        assert np.array_equal(vals[valid].view(np.int64), (want[valid] + 0.0).view(np.int64)), what
    assert np.array_equal(np.asarray(got.column("cnt")), C[i + 1] - C[s])
    expect(s, i, "run", "running sum")
    expect(s, e, "all", "whole-partition sum")
    expect(np.maximum(s, i - 5), np.minimum(e, i + 5), "slide", "sliding sum")
    expect(i, e, "rest", "shrinking sum")


# ------------------------------------------------------------------------------------------------------------ hash aggregate
def _agg_table(seed, many):
    """Special groups (keys 0..), then filler groups: 4 large ones (lane-private dictionary) or 40 000 small ones (more than the
    shared-memory table holds).  d float64, f = d as float32, v int64, e / g factors of the expression sums."""
    rng = np.random.default_rng(seed)
    groups = [[1e20, 1.0, 2.0, 3.0, -1e20, 4.0], [INF, 1.0, 2.0], [-INF, 5.0], [1.0, NAN, 2.0], [INF, -INF, 3.0],
              [1e16, 0.5, -1e16, 0.25] * 4, [-0.0] * 5, [-0.0, 0.0, -0.0], [None] * 4, [2.75], [-0.0], [NAN], [None, 1e20, None],
              [1e16, -1e16] * 8, [0.1] * 10]
    ints = [[I64_MAX] * 7, [0xFFFFFFFF] * 9, [-1] * 9, [I64_MIN, -1], [I64_MAX, 1], [I64_MAX, I64_MIN, -1, -1],
            [0xFFFFFFFF, 0xFFFFFFFF, 2, I64_MAX]]
    keys, ds, vs = [], [], []
    for gi, vals in enumerate(groups):
        iv = ints[gi % len(ints)]
        for j, x in enumerate(vals):
            keys.append(gi)
            ds.append(x)
            vs.append(None if x is None else iv[j % len(iv)])
    if many:
        sizes = rng.integers(3, 30, 40_000)
        fk = np.repeat(np.arange(40_000), sizes) + 100
    else:
        fk = rng.integers(100, 104, 400_000)
    m = len(fk)
    fd = rng.standard_normal(m) * 10.0 ** rng.integers(-2, 6, m)
    fnull = rng.random(m) < 0.05
    keys += fk.tolist()
    ds += [None if z else float(x) for x, z in zip(fd, fnull)]
    vs += [None if z else int(x) for x, z in zip(rng.integers(-2 ** 62, 2 ** 62, m), fnull)]
    for x in (I64_MAX, I64_MAX, 0xFFFFFFFF):                       # wrap-around and carries inside random groups too
        j = int(rng.integers(len(groups), len(keys)))
        vs[j] = x
    n = len(keys)
    perm = rng.permutation(n)
    take = lambda xs: [xs[i] for i in perm]
    dd = take(ds)
    return pa.table({"k": pa.array(take(keys), type=pa.int64()), "d": pa.array(dd, type=pa.float64()),
                     "f": pa.array([None if x is None else float(np.float32(x)) for x in dd], type=pa.float32()),
                     "v": pa.array(take(vs), type=pa.int64()),
                     "e": rng.integers(0, 11, n) / 100.0, "g": rng.choice([0.5, 1.0, 2.0, 4.0], n)})


def _terms_by_group(keys, vals):
    out = {}
    for k, x in zip(keys, vals):
        lst = out.setdefault(k, [])
        if x is not None:
            lst.append(x)
    return out


def _check_groups(got, key_cols, per_group, funcs):
    """per_group: {agg name: {key: terms}}; funcs: {agg name: 'sum' | 'avg' | 'isum' | 'count'}."""
    keys = list(zip(*[got.column(k).to_pylist() for k in key_cols])) if key_cols else [()]
    for name, func in funcs.items():
        res = got.column(name).to_pylist()
        groups = per_group[name]
        assert len(res) == len(groups), name
        for key, r in zip(keys, res):
            terms = groups[key[0] if key else None]
            what = "%s group %r" % (name, key)
            if func == "count":
                assert r == len(terms), what
            elif not terms:
                assert r is None, what
            elif func == "isum":
                assert r == wrap64(sum(terms)), what
            elif func == "sum":
                check_sum(r, terms, what)
            else:
                check_avg(r, [float(x) for x in terms], what)


def _agg_plan():
    from spark_b200.expressions import Average, Count, Literal, Sum, col
    aggs = [(Sum(col("d")), "sd"), (Average(col("d")), "ad"), (Sum(col("f")), "sf"), (Average(col("f")), "af"),
            (Sum(col("v")), "sv"), (Average(col("v")), "av"), (Count(col("d")), "cd"),
            (Sum(col("d") * (Literal(1.0) - col("e"))), "sp")]                      # fused Q1-shaped product
    funcs = {"sd": "sum", "ad": "avg", "sf": "sum", "af": "avg", "sv": "isum", "av": "avg", "cd": "count", "sp": "sum"}
    src = {"sd": "d", "ad": "d", "sf": "f", "af": "f", "sv": "v", "av": "v", "cd": "d"}
    return aggs, funcs, src


def _expected(t, key_cols, src, aggs):
    """{agg name: {key: non-NULL terms}}; the product's terms are the per-row products oracle.eval_expr computes."""
    keys = t.column(key_cols[0]).to_pylist() if key_cols else [None] * t.num_rows
    out = {name: _terms_by_group(keys, t.column(c).to_pylist()) for name, c in src.items()}
    out["sp"] = _terms_by_group(keys, _eval(t, aggs[-1][0].child.sexpr()))
    return out


def _eval(t, sexpr):
    v, valid = O.eval_expr(sexpr, t)
    return [float(x) if ok else None for x, ok in zip(v.tolist(), valid.tolist())]


@pytest.mark.parametrize("many", [False, True], ids=["dictionary-groups", "40k-groups"])
@pytest.mark.parametrize("rtc", [0, 1], ids=["generic", "rtc"])
@pytest.mark.parametrize("tier", [0, 1, 2], ids=["auto-tier", "dict-tier", "smem-tier"])
def test_aggregate_sums_against_exact_sums(gpu, stream, sbconfig, tier, rtc, many):
    """Every tier (lane-private dictionary DADDs, shared-memory CAS / carry adds, HBM atomics) on the generic and the NVRTC
    kernels: floating SUM / AVG within the exact-sum bound, int64 SUM bit-exact across 2^64, COUNT exact; then a materialised
    expression sum and Partial -> concat -> Final."""
    from spark_b200 import _capi as capi
    from spark_b200.columnar import ColumnarBatch
    from spark_b200.execution import HashAggregateExec, LocalTableScanExec
    from spark_b200.expressions import Sum, col
    if tier:
        sbconfig("agg_tier", tier)
    sbconfig("agg_rtc", rtc)
    sbconfig("agg_rtc_min_rows", 0)
    t = _agg_table(3 + many, many)
    aggs, funcs, src = _agg_plan()
    got = HashAggregateExec(["k"], aggs, LocalTableScanExec(ColumnarBatch.from_arrow(t, stream))).collect(stream)
    if rtc:
        assert capi.load().sb_hash_aggregate_last_plan().decode().startswith("rtc:"), capi.load().sb_hash_aggregate_last_plan()
    want = _expected(t, ["k"], src, aggs)
    _check_groups(got, ["k"], want, funcs)
    # an aggregate input that is no product form: evaluated into a column first
    expr = (col("d") + col("e")) / col("g")
    mat = HashAggregateExec(["k"], [(Sum(expr), "sm")], LocalTableScanExec(ColumnarBatch.from_arrow(t, stream))).collect(stream)
    _check_groups(mat, ["k"], {"sm": _terms_by_group(t.column("k").to_pylist(), _eval(t, expr.sexpr()))}, {"sm": "sum"})
    # Partial on two halves -> concat -> Final
    half = t.num_rows // 2
    parts = [HashAggregateExec(["k"], aggs, LocalTableScanExec(ColumnarBatch.from_arrow(h, stream)), mode="partial").collect(stream)
             for h in (t.slice(0, half), t.slice(half))]
    final = HashAggregateExec(["k"], aggs, LocalTableScanExec(ColumnarBatch.from_arrow(pa.concat_tables(parts), stream)), mode="final").collect(stream)
    _check_groups(final, ["k"], want, funcs)


@pytest.mark.parametrize("rtc", [0, 1], ids=["generic", "rtc"])
def test_global_aggregate_sums_of_each_regime(gpu, stream, sbconfig, rtc):
    """No grouping keys: one group per call, over each special group's rows on its own."""
    from spark_b200.columnar import ColumnarBatch
    from spark_b200.execution import HashAggregateExec, LocalTableScanExec
    sbconfig("agg_rtc", rtc)
    sbconfig("agg_rtc_min_rows", 0)
    t = _agg_table(7, False)
    aggs, funcs, src = _agg_plan()
    k = np.asarray(t.column("k"))
    for g in list(range(15)) + [100]:
        sub = t.filter(pa.array(k == g))
        got = HashAggregateExec([], aggs, LocalTableScanExec(ColumnarBatch.from_arrow(sub, stream))).collect(stream)
        assert got.num_rows == 1
        _check_groups(got, [], _expected(sub, [], src, aggs), funcs)
