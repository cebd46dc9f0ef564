"""Spark's central-moment aggregates restated sequentially, in Spark's order, over Python floats (IEEE doubles), plus the exact
rational references the GPU's answers are checked against.

Citations: sql/catalyst/src/main/scala/org/apache/spark/sql/catalyst/expressions/aggregate/CentralMomentAgg.scala
  initial values  :78-79    (n, avg, m2) = (0.0, 0.0, 0.0)
  update          :122-160  Welford's step; a NULL input leaves the buffer as it is
  merge           :83-120   Chan et al.'s pairwise merge, an empty side (n == 0) taken as is
  evaluate        :179-181 (stddev_pop), :215-218 (stddev_samp), :251-253 (var_pop), :285-288 (var_samp); divideByZeroEvalResult :67-69
"""
import math
from fractions import Fraction

FUNCS = ("var_pop", "var_samp", "stddev_pop", "stddev_samp")
EPS = Fraction(1, 2 ** 52)


def initial():
    return (0.0, 0.0, 0.0)


def update(buf, x):
    """updateExpressionsDef (:122-160); x is cast to DOUBLE first (ImplicitCastInputTypes)."""
    if x is None:
        return buf
    n, avg, m2 = buf
    x = float(x)
    new_n = n + 1.0
    delta = x - avg
    delta_n = delta / new_n
    new_avg = avg + delta_n
    new_m2 = m2 + delta * (delta - delta_n)
    return (new_n, new_avg, new_m2)


def merge(left, right):
    """mergeExpressions (:83-120)."""
    n1, avg1, m2_1 = left
    n2, avg2, m2_2 = right
    new_n = n1 + n2
    empty_l, empty_r = n1 == 0.0, n2 == 0.0
    delta = 0.0 if (empty_l or empty_r) else avg2 - avg1
    delta_n = 0.0 if new_n == 0.0 else delta / new_n
    new_avg = avg2 if empty_l else (avg1 if empty_r else avg1 + delta_n * n2)
    new_m2 = m2_1 + m2_2 + delta * delta_n * n1 * n2
    return (new_n, new_avg, new_m2)


def _sqrt(v):   # Sqrt of a double: NaN for NaN or a negative argument
    return math.sqrt(v) if v >= 0.0 else math.nan


def evaluate(func, buf, null_on_divide_by_zero=True):
    """evaluateExpression of StddevPop / StddevSamp / VariancePop / VarianceSamp; None is NULL."""
    n, _avg, m2 = buf
    if n == 0.0:
        return None
    if func in ("var_pop", "stddev_pop"):
        v = m2 / n
    else:
        if n == 1.0:
            return None if null_on_divide_by_zero else math.nan
        v = m2 / (n - 1.0)
    return _sqrt(v) if func.startswith("stddev") else v


def buffer_of(values):
    buf = initial()
    for x in values:
        buf = update(buf, x)
    return buf


def grouped_buffers(keys, values):
    """key -> buffer, rows folded in row order (one task's TungstenAggregationIterator)."""
    out = {}
    for k, x in zip(keys, values):
        out[k] = update(out.get(k, initial()), x)
    return out


def merge_all(buffers):
    acc = initial()
    for b in buffers:
        acc = merge(acc, b)
    return acc


# ---- exact references for finite data --------------------------------------------------------------------------------------
def exact_moments(xs):
    """(count, exact mean, exact M2 = sum (x - mean)^2) of a group's own doubles (NULLs dropped)."""
    fs = [Fraction(float(x)) for x in xs if x is not None]
    m = len(fs)
    if m == 0:
        return 0, Fraction(0), Fraction(0)
    mean = sum(fs) / m
    return m, mean, sum((f - mean) ** 2 for f in fs)


def m2_bound(m, m2_exact, abs_sum):
    """|m2 - M2| <= 2 (m + 2) 2^-52 (M2 + m D^2), D = 2^-52 sum |x| (derivation in tests/test_gpu_moments.py)."""
    d = EPS * abs_sum
    return 2 * (m + 2) * EPS * (m2_exact + m * d * d)


def check_result(func, got, m, m2_exact, err_m2, what=""):
    """A var / stddev result against the exact one: the m2 error divided by n or n - 1, one more rounding, and for stddev the
    square root's half ulp (taken as a full 2^-52 relative)."""
    den = m if func.endswith("_pop") else m - 1
    lo, hi = (m2_exact - err_m2) / den, (m2_exact + err_m2) / den
    lo = max(lo, Fraction(0)) * (1 - EPS)
    hi = hi * (1 + EPS)
    g = Fraction(got)
    if func.startswith("stddev"):
        assert g >= 0 and (g * (1 - EPS)) ** 2 <= hi and (g * (1 + EPS)) ** 2 >= lo, (what, func, got, float(lo), float(hi))
    else:
        assert lo <= g <= hi, (what, func, got, float(lo), float(hi))
