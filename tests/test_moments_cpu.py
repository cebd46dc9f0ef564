"""The central-moment oracle (tests/moments_oracle.py) against the answers the reference's own tests and documentation give, and its
merge against its update: splitting a group into partitions and merging their buffers gives the group's buffer."""
import math
import random

import pytest

import moments_oracle as M

TESTDATA2_A = [1, 1, 2, 2, 3, 3]   # SQLTestData.testData2, column a


def _all(values, legacy=False):
    buf = M.buffer_of(values)
    return {f: M.evaluate(f, buf, null_on_divide_by_zero=not legacy) for f in M.FUNCS}


def test_stddev_of_testdata2():
    # DataFrameAggregateSuite "stddev" (:452-460): stddev / stddev_pop / stddev_samp of testData2.a
    r = _all(TESTDATA2_A)
    assert math.isclose(r["stddev_samp"], math.sqrt(4 / 5), rel_tol=1e-15)
    assert math.isclose(r["stddev_pop"], math.sqrt(4 / 6), rel_tol=1e-15)


def test_zero_stddev_is_null():
    # "zero stddev" (:462-467): no rows -> NULL for every function
    assert _all([]) == {f: None for f in M.FUNCS}
    assert M.buffer_of([]) == (0.0, 0.0, 0.0)


def test_moments_of_testdata2():
    # "moments" (:483-497): var_samp / variance 4/5, var_pop 4/6
    r = _all(TESTDATA2_A)
    assert math.isclose(r["var_samp"], 4 / 5, rel_tol=1e-15)
    assert math.isclose(r["var_pop"], 4 / 6, rel_tol=1e-15)


@pytest.mark.parametrize("legacy", [False, True])
def test_zero_moments(legacy):
    # "zero moments" (:528-): one row: population forms 0.0; sample forms NULL, or NaN under spark.sql.legacy.statisticalAggregate
    r = _all([1], legacy)
    assert r["var_pop"] == 0.0 and r["stddev_pop"] == 0.0
    for f in ("var_samp", "stddev_samp"):
        if legacy:
            assert math.isnan(r[f])
        else:
            assert r[f] is None
    n, avg, m2 = M.buffer_of([1])
    assert (n, avg, m2) == (1.0, 1.0, 0.0) and math.copysign(1.0, m2) == 1.0


def test_null_moments():
    # "null moments" (:626-): only NULL inputs -> NULL results, the initial buffer
    assert _all([None, None, None]) == {f: None for f in M.FUNCS}
    assert M.buffer_of([None, None]) == (0.0, 0.0, 0.0)


def test_expression_description_examples():
    # the ExpressionDescription examples over VALUES (1), (2), (3)
    r = _all([1, 2, 3])
    assert r["stddev_pop"] == 0.816496580927726
    assert r["stddev_samp"] == 1.0
    assert r["var_pop"] == 0.6666666666666666
    assert r["var_samp"] == 1.0


def test_constant_groups_are_exact():
    for c in (0.1, -0.0, 0.0, 1e300, -7.25):
        n, avg, m2 = M.buffer_of([c] * 9)
        assert n == 9.0 and avg == c and m2 == 0.0 and math.copysign(1.0, m2) == 1.0
    n, avg, m2 = M.buffer_of([-0.0, 0.0, -0.0])
    assert avg == 0.0 and math.copysign(1.0, avg) == 1.0 and m2 == 0.0


def test_non_finite_terms_give_nan_m2():
    for vals in ([1.0, math.nan, 2.0], [1.0, math.inf], [-math.inf, 3.0, 4.0], [math.inf, -math.inf], [math.inf]):
        assert math.isnan(M.buffer_of(vals)[2]), vals


def test_merge_of_any_split_gives_the_group_buffer():
    rng = random.Random(7)
    for trial in range(200):
        m = rng.randint(0, 40)
        scale = 10.0 ** rng.randint(-3, 9)
        xs = [None if rng.random() < 0.1 else rng.gauss(0, 1) * scale + (1e9 if trial % 3 == 0 else 0.0) for _ in range(m)]
        whole = M.buffer_of(xs)
        cuts = sorted(rng.randint(0, m) for _ in range(rng.randint(0, 5)))
        parts = [xs[a:b] for a, b in zip([0] + cuts, cuts + [m])]
        merged = M.merge_all([M.buffer_of(p) for p in parts])
        assert merged[0] == whole[0]
        k, mean, m2x = M.exact_moments(xs)
        if k == 0:
            assert merged == (0.0, 0.0, 0.0)
            continue
        abs_sum = sum(abs(x) for x in xs if x is not None)
        spread = max(abs(M.Fraction(x) - mean) for x in xs if x is not None)
        # both sides within a first-order bound of Welford's rounding (each step errs by a few ulps of |x| times |x - avg|) around
        # the group's exact M2, and their means within the bound of the mean
        err = 4 * (k + 2) * M.EPS * (m2x + M.Fraction(abs_sum) * spread)
        for buf in (whole, merged):
            assert abs(M.Fraction(buf[2]) - m2x) <= err, (trial, buf, float(m2x))
            assert abs(M.Fraction(buf[1]) - mean) <= (k + 4) * M.EPS * abs_sum, (trial, buf, float(mean))


def test_merge_with_empty_sides():
    b = M.buffer_of([1.0, 2.0, 4.0])
    assert M.merge(M.initial(), b) == b and M.merge(b, M.initial()) == b
    assert M.merge(M.initial(), M.initial()) == (0.0, 0.0, 0.0)
