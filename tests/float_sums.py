"""An exact reference for floating SUM / AVG results (helper module, not a test file).

A floating sum is order-dependent, so a GPU sum is not compared with another implementation's sum; it is checked against the
correctly rounded sum of the same terms (math.fsum) within a bound that holds for every summation order:

    |r - fsum(x)| <= max(m - 1, 1) * 2^-52 * fsum(|x|)

scaled by the group's or frame's own m non-NULL terms.  Special values are classified first (fsum raises on inf + -inf):
any NaN term or both infinities -> NaN; otherwise one infinity -> that infinity; otherwise only +-0.0 terms -> +0.0 with the
sign bit clear, because Spark starts every sum from +0.0 (Sum.scala: coalesce(sum, zero) + x; Average.scala: sum starts at
0.0).  AVG is r ~= s / m: the sum's bound divided by m plus one rounding of the quotient.  Callers widen terms the way the
reference does (float32 -> double, long -> double for AVG) and keep finite sums below DBL_MAX."""
import math

EPS = 2.0 ** -52


def _special(xs):
    """NaN / +inf / -inf when the special-value rules decide the result, None otherwise."""
    nan = pinf = ninf = False
    for x in xs:
        if x != x:
            nan = True
        elif x == math.inf:
            pinf = True
        elif x == -math.inf:
            ninf = True
    if nan or (pinf and ninf):
        return math.nan
    if pinf:
        return math.inf
    if ninf:
        return -math.inf
    return None


def _check(r, xs, m_div, what):
    xs = [float(x) for x in xs]
    m = len(xs)
    assert m > 0, "%s: no terms (the result must be NULL)" % what
    sp = _special(xs)
    if sp is not None:
        if sp != sp:
            assert r != r, "%s: %r, want NaN (terms %s)" % (what, r, xs[:8])
        else:
            assert r == sp, "%s: %r, want %r (terms %s)" % (what, r, sp, xs[:8])
        return
    if all(x == 0.0 for x in xs):
        assert r == 0.0 and math.copysign(1.0, r) == 1.0, "%s: %r, want +0.0 (terms %s)" % (what, r, xs[:8])
        return
    s, a = math.fsum(xs), math.fsum(abs(x) for x in xs)
    bound = max(m - 1, 1) * EPS * a
    if m_div:
        want, tol = s / m, bound / m * (1 + EPS) + EPS * abs(s) / m
    else:
        want, tol = s, bound
    assert abs(r - want) <= tol, "%s: %r, want %r within %.3g (%d terms, sum|x| %.6g)" % (what, r, want, tol, m, a)


def check_sum(r, xs, what="sum"):
    """r: the SUM of one group or frame; xs: its non-NULL terms as doubles."""
    _check(r, xs, False, what)


def check_avg(r, xs, what="avg"):
    """r: the AVG of one group or frame; xs: its non-NULL terms widened to double."""
    _check(r, xs, True, what)


def wrap64(x):
    """A Python int reduced modulo 2^64 to a signed long: Spark's non-ANSI long SUM."""
    x &= (1 << 64) - 1
    return x - (1 << 64) if x >= (1 << 63) else x
