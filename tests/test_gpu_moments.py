"""VAR_POP / VAR_SAMP / STDDEV_POP / STDDEV_SAMP in the GPU hash aggregate (csrc/moments.cu), against the sequential oracle
(tests/moments_oracle.py) where Spark's answer is exact, and against exact rationals everywhere else.

The bound for finite data.  Let a group have m terms x_i, exact mean mu and M2 = sum (x_i - mu)^2, and let u = 2^-53.  Pass 1 sums
the x_i in some order and divides by m: |m^ - mu| <= D with D = 2^-52 sum |x_i| (a sum of m terms errs by at most (m - 1) u sum |x|,
the division by one more rounding).  Pass 2 forms d_i = fl(x_i - m^) (relative error u), d_i^2 (2u more) and sums them in some
order ((m - 1) u), so S2 is within (m + 2) u sum d_i^2 of the exact sum of squared deviations from m^, and S1 within (m + 1) u sum |d_i|.
In exact arithmetic sum (x_i - m^)^2 - (sum (x_i - m^))^2 / m = M2 for ANY m^: the correction removes m (mu - m^)^2 exactly.  Both
terms are at most sum d_i^2 <= M2 + m D^2 (Cauchy-Schwarz for the second), so with the final subtraction and division
    |m2 - M2| <= 2 (m + 2) 2^-52 (M2 + m D^2).
The results divide by n or n - 1 (one more rounding) and stddev takes a correctly rounded square root (half an ulp more).  Values
near 1e9 with unit spread are in the data: there the naive sum x^2 - (sum x)^2 / n loses every digit and this bound keeps ~30 bits."""
import math
import struct
from fractions import Fraction

import numpy as np
import pyarrow as pa
import pytest

import moments_oracle as M

pytestmark = pytest.mark.gpu

NAN, INF = math.nan, math.inf
FUNCS = M.FUNCS


def _cls(func):
    from spark_b200 import expressions as E
    return {"var_pop": E.VariancePop, "var_samp": E.VarianceSamp, "stddev_pop": E.StddevPop, "stddev_samp": E.StddevSamp}[func]


def _col(name):
    from spark_b200.expressions import col
    return col(name)


def _bits(x):
    return None if x is None else struct.pack("<d", x)


def _moment_aggs(col, legacy=False, funcs=FUNCS):
    return [(_cls(f)(_col(col), null_on_divide_by_zero=not legacy), "%s_%s" % (f, col)) for f in funcs]


def _run(t, keys, aggs, stream, mode="complete", condition=None):
    from spark_b200.columnar import ColumnarBatch
    from spark_b200.execution import HashAggregateExec, LocalTableScanExec
    return HashAggregateExec(keys, aggs, LocalTableScanExec(ColumnarBatch.from_arrow(t, stream)), mode=mode, condition=condition).collect(stream)


def _by_key(res, keys):
    cols = [res.column(k).to_pylist() for k in keys]
    out = {}
    for i in range(res.num_rows):
        out[tuple(c[i] for c in cols)] = {n: res.column(n)[i].as_py() for n in res.column_names}
    return out


def _groups(t, keys, col):
    ks = list(zip(*[t.column(k).to_pylist() for k in keys])) if keys else [()] * t.num_rows
    out = {}
    for k, x in zip(ks, t.column(col).to_pylist()):
        out.setdefault(k, []).append(x)
    return out


# ---------------------------------------------------------------------------------------------- edges: bit for bit
EDGE_GROUPS = [
    [1.0, 2.0, 3.0],                        # the ExpressionDescription examples
    [1.0, 1.0, 2.0, 2.0, 3.0, 3.0],         # testData2.a
    [None, None, None],                     # all NULL
    [None, 4.5, None],                      # one row among NULLs
    [-7.25],
    [0.1] * 7,                              # constant, not representable
    [-0.0, 0.0, -0.0, 0.0],
    [-0.0] * 3,
    [0.0, None, 0.0],
    [1e300] * 4,
    [1.0, NAN, 2.0],
    [NAN],
    [NAN, NAN],
    [1.0, INF, 3.0],
    [-INF, 5.0],
    [INF, -INF, 1.0],
    [INF, INF],
]
EXACT = {0, 1, 2, 3, 4, 5, 6, 7, 8, 9}     # groups whose whole buffer Spark computes exactly; the rest: m2 NaN, avg not pinned


def _edge_table():
    k, x = [], []
    for g, vals in enumerate(EDGE_GROUPS):
        k += [g] * len(vals)
        x += vals
    perm = np.random.default_rng(3).permutation(len(k))
    return pa.table({"k": pa.array([k[i] for i in perm], type=pa.int32()), "x": pa.array([x[i] for i in perm], type=pa.float64())})


def _check_edge_buffers(got_rows, prefix="m"):
    for g, vals in enumerate(EDGE_GROUPS):
        want = M.buffer_of(vals)
        r = got_rows[(g,)]
        n, avg, m2 = r[prefix + "#n"], r[prefix + "#avg"], r[prefix + "#m2"]
        assert n == want[0], (g, n, want)
        if g in EXACT:
            assert _bits(avg) == _bits(want[1]) and _bits(m2) == _bits(want[2]), (g, (n, avg, m2), want)
        else:
            assert math.isnan(m2), (g, m2)


@pytest.mark.parametrize("tier", [0, 1, 2])
@pytest.mark.parametrize("legacy", [False, True])
def test_edge_groups_bit_exact(gpu, stream, sbconfig, tier, legacy):
    sbconfig("agg_tier", tier)
    t = _edge_table()
    rows = _by_key(_run(t, ["k"], _moment_aggs("x", legacy), stream), ["k"])
    assert len(rows) == len(EDGE_GROUPS)
    for g, vals in enumerate(EDGE_GROUPS):
        buf = M.buffer_of(vals)
        for f in FUNCS:
            got, want = rows[(g,)]["%s_x" % f], M.evaluate(f, buf, null_on_divide_by_zero=not legacy)
            if g in EXACT or want is None:
                assert _bits(got) == _bits(want), (g, f, got, want)
            else:
                assert math.isnan(got), (g, f, got)
    part = _run(t, ["k"], [(_cls("var_pop")(_col("x")), "m")], stream, mode="partial")
    assert part.column_names == ["k", "m#n", "m#avg", "m#m2"]
    _check_edge_buffers(_by_key(part, ["k"]))


def test_global_aggregate_of_nothing(gpu, stream):
    """No grouping keys: one row even for empty input, buffer (0.0, 0.0, 0.0) and NULL results."""
    t = pa.table({"x": pa.array([], type=pa.float64())})
    res = _run(t, [], _moment_aggs("x"), stream)
    assert res.num_rows == 1 and all(res.column(c)[0].as_py() is None for c in res.column_names)
    part = _run(t, [], [(_cls("var_samp")(_col("x")), "m")], stream, mode="partial")
    assert [_bits(part.column(c)[0].as_py()) for c in part.column_names] == [_bits(0.0)] * 3
    from spark_b200 import expressions as E
    t2 = pa.table({"x": pa.array([1.0, 2.0, 3.0])})
    res = _run(t2, [], _moment_aggs("x"), stream, condition=E.GreaterThan(E.col("x"), E.lit(5.0)))   # every row filtered out
    assert all(res.column(c)[0].as_py() is None for c in res.column_names)


# ---------------------------------------------------------------------------------------------- finite data: exact bound
def _finite_table(seed, ngroups, n, key_kind="int32", offset=True):
    rng = np.random.default_rng(seed)
    g = rng.integers(0, ngroups, n)
    # per group one regime: unit spread around 1e9, wide magnitudes, small integers
    regime = g % 3 if offset else 1 + g % 2
    x = np.where(regime == 0, 1e9 + rng.standard_normal(n), np.where(regime == 1, rng.standard_normal(n) * 10.0 ** rng.integers(-3, 6, n),
                                                                        rng.integers(-50, 50, n).astype(np.float64)))
    xs = [None if rng.random() < 0.03 else float(v) for v in x]
    big = [None if v is None else int(2 ** 53 + 12345 * int(i % 977) + (int(i) * 7919) % 1000) for i, v in enumerate(xs)]   # int64 > 2^53
    cols = {"x": pa.array(xs, type=pa.float64()), "b": pa.array(big, type=pa.int64()),
            "f": pa.array([None if v is None else float(np.float32(v / 1e6)) for v in xs], type=pa.float32()),
            "i": pa.array(rng.integers(-1000, 1000, n), type=pa.int32())}
    if key_kind == "int32":
        cols["k"] = pa.array(g, type=pa.int32())
        keys = ["k"]
    elif key_kind == "wide":                                        # two 64-bit keys: a two-word packed key
        cols["k"] = pa.array(g * 1_000_003 - 2 ** 40, type=pa.int64())
        cols["k2"] = pa.array([None if v % 11 == 0 else int(v) * 3 for v in g], type=pa.int64())
        keys = ["k", "k2"]
    elif key_kind == "string":
        cols["k"] = pa.array(["grp-%d" % v for v in g], type=pa.string())
        keys = ["k"]
    else:
        keys = []
    return pa.table(cols), keys


def _check_exact(res, t, keys, col, funcs, names=None, what=""):
    rows = _by_key(res, keys)
    groups = _groups(t, keys, col)
    assert len(rows) == len(groups), (what, len(rows), len(groups))
    for k, xs in groups.items():
        m, mean, m2x = M.exact_moments(xs)
        vals = [float(x) for x in xs if x is not None]
        err = M.m2_bound(m, m2x, Fraction(sum(abs(Fraction(v)) for v in vals))) if m else 0
        for f in funcs:
            name = (names or {}).get(f, "%s_%s" % (f, col))
            got = rows[k][name]
            if m == 0 or (m == 1 and f.endswith("_samp")):
                assert got is None, (what, k, f, got)
            else:
                M.check_result(f, got, m, m2x, err, (what, k))


def _check_buffers_exact(res, t, keys, col, prefix, what="", slack=1):
    rows = _by_key(res, keys)
    for k, xs in _groups(t, keys, col).items():
        m, mean, m2x = M.exact_moments(xs)
        r = rows[k]
        assert r[prefix + "#n"] == float(m), (what, k)
        if m == 0:
            assert (r[prefix + "#avg"], r[prefix + "#m2"]) == (0.0, 0.0)
            continue
        abs_sum = sum(abs(Fraction(float(x))) for x in xs if x is not None)
        assert abs(Fraction(r[prefix + "#m2"]) - m2x) <= slack * M.m2_bound(m, m2x, abs_sum), (what, k, r, float(m2x))
        assert abs(Fraction(r[prefix + "#avg"]) - mean) <= (m + 4) * M.EPS * abs_sum, (what, k, r, float(mean))


@pytest.mark.parametrize("tier", [0, 1, 2])
@pytest.mark.parametrize("shape", [("global", 1, "none"), ("seven", 7, "int32"), ("wide", 300, "wide"), ("string", 40, "string")])
def test_finite_data_within_exact_bound(gpu, stream, sbconfig, tier, shape):
    sbconfig("agg_tier", tier)
    name, ngroups, kind = shape
    t, keys = _finite_table(11 + ngroups, ngroups, 6000, kind)
    aggs = _moment_aggs("x") + _moment_aggs("b", funcs=("var_pop", "stddev_samp")) + _moment_aggs("f", funcs=("var_samp",))
    res = _run(t, keys, aggs, stream)
    _check_exact(res, t, keys, "x", FUNCS, what=name)
    _check_exact(res, t, keys, "b", ("var_pop", "stddev_samp"), what=name)
    _check_exact(res, t, keys, "f", ("var_samp",), what=name)


def test_many_groups_and_the_specialised_kernels(gpu, stream, sbconfig):
    """~60 000 groups (per-block shared accumulators do not fit: global atomics), and the NVRTC-specialised pass 1."""
    sbconfig("agg_rtc_min_rows", 1 << 16)
    t, keys = _finite_table(5, 60_000, 400_000)
    res = _run(t, keys, _moment_aggs("x", funcs=("var_pop", "stddev_samp")), stream)
    _check_exact(res, t, keys, "x", ("var_pop", "stddev_samp"), what="60k")
    from spark_b200 import _capi as capi
    assert capi.load().sb_hash_aggregate_last_plan().decode().startswith("rtc:")


def test_every_mode(gpu, stream):
    """Partial buffers, Partial -> Final and Partial -> PartialMerge -> Final on the GPU, and Final over buffers the oracle made
    (Spark's buffers), against the exact answers."""
    from spark_b200 import expressions as E
    t, keys = _finite_table(21, 7, 9000)
    aggs = [(E.VariancePop(E.col("x")), "vp"), (E.StddevSamp(E.col("x")), "ss")]
    names = {"var_pop": "vp", "stddev_samp": "ss"}
    part = _run(t, keys, aggs, stream, mode="partial")
    assert part.column_names == ["k", "vp#n", "vp#avg", "vp#m2", "ss#n", "ss#avg", "ss#m2"]
    _check_buffers_exact(part, t, keys, "x", "vp", "partial")
    halves = [_run(t.slice(0, 4000), keys, aggs, stream, mode="partial"), _run(t.slice(4000), keys, aggs, stream, mode="partial")]
    cat = pa.concat_tables(halves)
    _check_merged(_run(cat, keys, aggs, stream, mode="final"), cat, "partial->final")
    pm = _run(cat, keys, aggs, stream, mode="partial_merge")
    _check_merged(pm, cat, "partial->partial_merge")
    _check_merged(_run(pm, keys, aggs, stream, mode="final"), pm, "partial_merge->final")
    # Final over Spark's buffers: the oracle's Welford buffers of three row ranges, plus an empty partial per group
    kk, xx = t.column("k").to_pylist(), t.column("x").to_pylist()
    rows = []
    for lo, hi in ((0, 3000), (3000, 3001), (3001, 9000)):
        for k, buf in M.grouped_buffers(kk[lo:hi], xx[lo:hi]).items():
            rows.append((k,) + buf + buf)
    rows += [(k, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0) for k in range(7)]
    spark = pa.table({n: pa.array([r[i] for r in rows], type=pa.int32() if i == 0 else pa.float64())
                      for i, n in enumerate(["k", "vp#n", "vp#avg", "vp#m2", "ss#n", "ss#avg", "ss#m2"])})
    _check_merged(_run(spark, keys, aggs, stream, mode="final"), spark, "spark buffers")


def _check_merged(res, partials, what):
    """A merge of (n, avg, m2) partials against the exact merge of those buffers taken as exact: M2 = sum m2_i + sum n_i (avg_i - A)^2,
    A = sum n_i avg_i / N.  Pass 1 sums n_i avg_i (error D = (k + 2) 2^-52 sum n_i |avg_i| / N on A), pass 2 forms n_i d_i^2 (three
    roundings) and sums k terms: the update bound with k + 2 terms and m2_i summed alongside.  Partials made from rows near 1e9 carry
    avg_i to an ulp of 1e9, so the merged M2 is pinned to the buffers, not to the raw rows."""
    rows = _by_key(res, ["k"])
    bufs = {}
    p = partials.to_pylist()
    for r in p:
        bufs.setdefault(r["k"], []).append((r["vp#n"], r["vp#avg"], r["vp#m2"]))
    for k, bs in bufs.items():
        bs = [b for b in bs if b[0] != 0.0]
        N = sum(Fraction(b[0]) for b in bs)
        A = sum(Fraction(b[0]) * Fraction(b[1]) for b in bs) / N
        M2b = sum(Fraction(b[2]) + Fraction(b[0]) * (Fraction(b[1]) - A) ** 2 for b in bs)
        abs_sum = sum(Fraction(b[0]) * abs(Fraction(b[1])) for b in bs)
        D = (len(bs) + 2) * M.EPS * abs_sum / N
        err = 2 * (len(bs) + 4) * M.EPS * (M2b + N * D * D)
        r = rows[(k,)]
        if "vp" in r:
            M.check_result("var_pop", r["vp"], int(N), M2b, err, (what, k))
            M.check_result("stddev_samp", r["ss"], int(N), M2b, err, (what, k))
        else:
            assert r["vp#n"] == float(N), (what, k)
            assert abs(Fraction(r["vp#m2"]) - M2b) <= err, (what, k, r["vp#m2"], float(M2b))
            assert abs(Fraction(r["vp#avg"]) - A) <= (len(bs) + 4) * M.EPS * abs_sum / N, (what, k)


def test_constant_and_non_finite_groups_through_merges(gpu, stream):
    """Constant groups stay exact and non-finite ones NaN when their partials are merged on the GPU."""
    from spark_b200 import expressions as E
    t = _edge_table()
    aggs = [(E.VarianceSamp(E.col("x")), "m")]
    halves = [_run(t.slice(0, 20), ["k"], aggs, stream, mode="partial"), _run(t.slice(20), ["k"], aggs, stream, mode="partial")]
    merged = _by_key(_run(pa.concat_tables(halves), ["k"], aggs, stream, mode="partial_merge"), ["k"])
    for g, vals in enumerate(EDGE_GROUPS):
        n, avg, m2 = merged[(g,)]["m#n"], merged[(g,)]["m#avg"], merged[(g,)]["m#m2"]
        want = M.buffer_of(vals)
        assert n == want[0]
        present = [v for v in vals if v is not None]
        if present and all(not math.isnan(v) and not math.isinf(v) for v in present) and len(set(map(_bits, present))) == 1:
            assert _bits(m2) == _bits(0.0) and avg == present[0], (g, avg, m2)
        elif any(v is not None and (math.isnan(v) or math.isinf(v)) for v in vals):
            assert math.isnan(m2), (g, m2)
        elif not present:
            assert (avg, m2) == (0.0, 0.0)


def test_streaming_state_over_batches(gpu, stream):
    from spark_b200 import expressions as E
    from spark_b200.columnar import ColumnarBatch
    from spark_b200.execution import HashAggregateExec, LocalTableScanExec
    # merged partials carry avg to an ulp of itself, so the raw-row bound holds only without a large offset (see _check_merged)
    t, keys = _finite_table(31, 500, 30_000, offset=False)
    aggs = [(E.StddevPop(E.col("x")), "sp"), (E.VarianceSamp(E.col("i")), "vs"), (E.Sum(E.col("x")), "s")]
    batches = [ColumnarBatch.from_arrow(t.slice(o, 5000), stream) for o in range(0, 30_000, 5000)]
    res = HashAggregateExec(keys, aggs, LocalTableScanExec(batches[0])).execute_batches(batches, stream).to_arrow(stream)
    _check_exact(res, t, keys, "x", ("stddev_pop",), {"stddev_pop": "sp"}, "stream")
    _check_exact(res, t, keys, "i", ("var_samp",), {"var_samp": "vs"}, "stream")


def test_fused_filter(gpu, stream):
    from spark_b200 import expressions as E
    t, keys = _finite_table(41, 7, 8000)
    cond = E.And(E.GreaterThan(E.col("i"), E.lit(-300)), E.LessThan(E.col("x"), E.lit(1e8)))
    res = _run(t, keys, _moment_aggs("x"), stream, condition=cond)
    i, x = t.column("i").to_pylist(), t.column("x").to_pylist()
    keep = pa.array([a > -300 and v is not None and v < 1e8 for a, v in zip(i, x)])
    _check_exact(res, t.filter(keep), keys, "x", FUNCS, what="filter")


def test_mixed_plans(gpu, stream):
    """Moments next to SUM, AVG, MIN, MAX, COUNT and decimal SUM of the same and of other columns: the other aggregates' answers
    are those of the plan without the moments."""
    import decimal as D
    from spark_b200 import expressions as E
    t, keys = _finite_table(51, 7, 7000)
    rng = np.random.default_rng(51)
    t = t.append_column("d", pa.array([D.Decimal(int(v)).scaleb(-2) for v in rng.integers(-10 ** 8, 10 ** 8, t.num_rows)], type=pa.decimal128(12, 2)))
    others = [(E.Sum(E.col("i")), "si"), (E.Average(E.col("x")), "ax"), (E.Min(E.col("x")), "mnx"), (E.Max(E.col("b")), "mxb"), (E.Count(E.col("x")), "cx"),
              (E.Count(), "n"), (E.Sum(E.col("d")), "sd")]
    moments = [(E.VarianceSamp(E.col("x")), "vx"), (E.StddevPop(E.col("i")), "spi")]
    base = _by_key(_run(t, keys, others, stream), keys)
    for plan in (moments + others, others[:3] + moments + others[3:]):
        got = _by_key(_run(t, keys, plan, stream), keys)
        for k, row in base.items():
            for name, v in row.items():
                if name == "ax":
                    assert math.isclose(got[k][name], v, rel_tol=1e-12), (name, k)
                else:
                    assert got[k][name] == v, (name, k, got[k][name], v)
        _check_exact(_run(t, keys, plan, stream), t, keys, "x", ("var_samp",), {"var_samp": "vx"}, "mixed")
        _check_exact(_run(t, keys, plan, stream), t, keys, "i", ("stddev_pop",), {"stddev_pop": "spi"}, "mixed")
    # partial -> final of a mixed plan with a decimal sum in front of the moment buffers
    plan = [(E.Sum(E.col("d")), "sd"), (E.VarianceSamp(E.col("x")), "vx"), (E.Average(E.col("x")), "ax")]
    part = _run(t, keys, plan, stream, mode="partial")
    assert part.column_names == ["k", "sd#sum", "sd#isEmpty", "vx#n", "vx#avg", "vx#m2", "ax#sum", "ax#count"]
    fin = _run(part, keys, plan, stream, mode="final")
    _check_exact(fin, t, keys, "x", ("var_samp",), {"var_samp": "vx"}, "mixed final")
    assert _by_key(fin, keys)[(0,)]["sd"] == base[(0,)]["sd"]


def test_slot_budget_and_input_types_are_refused(gpu, stream):
    import decimal as D
    from spark_b200 import _capi as capi
    from spark_b200 import expressions as E
    n = 100
    t = pa.table({"k": pa.array(np.arange(n) % 3, type=pa.int32()),
                  **{"c%d" % j: pa.array(np.arange(n, dtype=np.float64) * (j + 1)) for j in range(6)},
                  "dec": pa.array([D.Decimal(i) for i in range(n)], type=pa.decimal128(10, 0)),
                  "s": pa.array(["a%d" % i for i in range(n)]), "bo": pa.array([i % 2 == 0 for i in range(n)]),
                  "dt": pa.array(np.arange(n, dtype=np.int32), type=pa.date32())})
    # five inputs: COUNT (shared: no NULLs) + 3 x 5 = 16 slots, answered; a sixth input needs 19
    ok = _run(t, ["k"], [(E.VariancePop(E.col("c%d" % j)), "v%d" % j) for j in range(5)], stream)
    assert ok.num_rows == 3
    with pytest.raises(capi.SparkB200Error) as e:
        _run(t, ["k"], [(E.VariancePop(E.col("c%d" % j)), "v%d" % j) for j in range(6)], stream)
    assert e.value.code == 5
    for c in ("dec", "s", "bo", "dt"):
        with pytest.raises(capi.SparkB200Error) as e:
            _run(t, ["k"], [(E.StddevSamp(E.col(c)), "r")], stream)
        assert e.value.code == 5, c
