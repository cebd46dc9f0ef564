"""The exact floating-sum reference (tests/float_sums.py) and oracle.window_frames, pinned to known answers; and proof, without
a GPU, that the reference rejects a window sum computed as a difference of running sums S[hi] - S[lo-1]."""
import math

import numpy as np
import pyarrow as pa
import pytest

from float_sums import check_avg, check_sum, wrap64
from oracle import oracle as O

INF, NAN = math.inf, math.nan


@pytest.mark.parametrize("terms,want", [
    ([1.0, NAN, 2.0], NAN), ([INF, -INF, 1.0], NAN), ([NAN, INF], NAN), ([-INF, NAN], NAN),
    ([INF, 1e308, 1e308], INF), ([2.0, -INF, -1e308, -1e308], -INF), ([INF], INF), ([INF, INF, -5.0], INF)])
def test_special_values_decide_the_result(terms, want):
    for check in (check_sum, check_avg):
        check(want, terms)
        for wrong in (0.0, 1.0, -want if want == want else INF):
            with pytest.raises(AssertionError):
                check(wrong, terms)


def test_every_zero_term_gives_plus_zero():
    for terms in ([-0.0], [-0.0, -0.0, -0.0], [0.0, -0.0], [0.0]):
        check_sum(0.0, terms)
        check_avg(0.0, terms)
        with pytest.raises(AssertionError):
            check_sum(-0.0, terms)
        with pytest.raises(AssertionError):
            check_avg(-0.0, terms)


def test_cancelling_terms_against_the_correctly_rounded_sum():
    # left to right: 1e16 + 1 rounds to 1e16, so the naive sum is 1.0; the exact sum is 2.0; the bound is 3 * 2^-52 * (2e16 + 2)
    terms = [1e16, 1.0, -1e16, 1.0]
    assert math.fsum(terms) == 2.0
    bound = 3 * 2.0 ** -52 * (2e16 + 2)
    check_sum(1.0, terms)
    check_sum(2.0 + bound * 0.99, terms)
    with pytest.raises(AssertionError):
        check_sum(2.0 + bound * 1.01, terms)
    # 0.1 ten times: the naive sum is 0.9999999999999999, the correctly rounded one 1.0; both lie inside 9 * 2^-52
    tenth = [0.1] * 10
    check_sum(sum(tenth), tenth)
    check_sum(1.0, tenth)
    with pytest.raises(AssertionError):
        check_sum(1.0 + 1e-14, tenth)
    with pytest.raises(AssertionError):
        check_sum(0.5, [1.0])


def test_average_is_the_sum_over_the_count():
    check_avg(2.5, [1.0, 2.0, 3.0, 4.0])
    with pytest.raises(AssertionError):
        check_avg(10.0, [1.0, 2.0, 3.0, 4.0])
    big = [float(2 ** 63 - 1)] * 5                  # AVG of longs near INT64_MAX: a double near 9.22e18, not a wrapped sum
    check_avg(9.223372036854776e18, big)
    with pytest.raises(AssertionError):
        check_avg(float(wrap64(5 * (2 ** 63 - 1))) / 5, big)
    with pytest.raises(AssertionError):
        check_sum(0.0, [])


def test_wrap64():
    assert wrap64(2 ** 63) == -2 ** 63
    assert wrap64(3 * (2 ** 63 - 1)) == 2 ** 63 - 3
    assert wrap64(-2 ** 63 - 1) == 2 ** 63 - 1
    assert wrap64(sum([0xFFFFFFFF] * 4)) == 4 * 0xFFFFFFFF


FRAME_TABLE = pa.table({"p": pa.array([1, 1, 1, 1, 1, 2, 2, 2], type=pa.int32()),
                        "o": pa.array([1, 2, 2, 4, None, 7, 8, 10], type=pa.int32()),
                        "k": pa.array([0.5, -0.0, 0.0, NAN, None, INF, -INF, 1.0], type=pa.float64()),
                        "row": pa.array(range(8), type=pa.int64())})


@pytest.mark.parametrize("orders,frame,want", [
    # partition 1 sorts as o = NULL, 1, 2, 2, 4 (positions 0..4), partition 2 as 7, 8, 10 (5..7)
    ([("o", True, True)], ("rows", -1, 1), [(0, 1), (0, 2), (1, 3), (2, 4), (3, 4), (5, 6), (5, 7), (6, 7)]),
    ([("o", True, True)], ("rows", None, 0), [(0, 0), (0, 1), (0, 2), (0, 3), (0, 4), (5, 5), (5, 6), (5, 7)]),
    ([("o", True, True)], ("rows", -3, -1), [(0, -1), (0, 0), (0, 1), (0, 2), (1, 3), (5, 4), (5, 5), (5, 6)]),
    ([("o", True, True)], ("rows", 0, None), [(0, 4), (1, 4), (2, 4), (3, 4), (4, 4), (5, 7), (6, 7), (7, 7)]),
    ([("o", True, True)], ("range", 0, None), [(0, 4), (1, 4), (2, 4), (2, 4), (4, 4), (5, 7), (6, 7), (7, 7)]),
    ([("o", True, True)], None, [(0, 0), (0, 1), (0, 3), (0, 3), (0, 4), (5, 5), (5, 6), (5, 7)]),
    ([("o", True, True)], ("range", -1, 1), [(0, 0), (1, 3), (1, 3), (1, 3), (4, 4), (5, 6), (5, 6), (7, 7)]),
    # descending, NULLS LAST: 4, 2, 2, 1, NULL and 10, 8, 7; bounds are key - offset
    ([("o", False, False)], ("range", -1, 1), [(0, 0), (1, 3), (1, 3), (1, 3), (4, 4), (5, 5), (6, 7), (6, 7)]),
    # double key, NULLS LAST: -0.0 / 0.0 (peers), 0.5, NaN, NULL and -inf, 1.0, inf; inf +- 1 = inf, NaN +- 1 = NaN
    ([("k", True, False)], ("range", -1.0, 0.5), [(0, 2), (0, 2), (0, 2), (3, 3), (4, 4), (5, 5), (6, 6), (7, 7)]),
])
def test_window_frames_by_hand(orders, frame, want):
    assert O.window_frames(FRAME_TABLE, ["p"], orders, ("sum", "row", frame, 0, "s")) == want


def _prefix_difference(d, frames, seg_start):
    """What a kernel computing S[hi] - S[lo-1] over segmented running sums returns (the running sum starts at the first term)."""
    n = len(d)
    S = np.empty(n)
    for i in range(n):
        S[i] = d[i] if seg_start[i] == i else S[i - 1] + d[i]
    with np.errstate(invalid="ignore"):
        return [S[hi] - S[lo - 1] if lo > seg_start[i] else S[hi] for i, (lo, hi) in enumerate(frames)]


@pytest.mark.parametrize("func,frame", [("sum", ("rows", -1, 1)), ("avg", ("rows", -1, 1)), ("sum", ("rows", 0, None)),
                                        ("avg", ("rows", 0, None)), ("sum", ("rows", None, 0))])
def test_the_check_rejects_running_sum_differences_and_accepts_the_oracle(func, frame):
    d = [INF, 1.0, 2.0, 3.0, 4.0, 1e20, 1.0, 2.0, 3.0, 4.0, -0.0]
    t = pa.table({"p": pa.array([0] * 5 + [1] * 5 + [2], type=pa.int32()), "d": d, "row": pa.array(range(len(d)), type=pa.int64())})
    orders = [("row", True, True)]
    spec = (func, "d", frame, 0, "s")
    frames = O.window_frames(t, ["p"], orders, spec)
    seg_start = [0] * 5 + [5] * 5 + [10]
    check = check_sum if func == "sum" else check_avg

    def check_all(res):
        for i, (lo, hi) in enumerate(frames):
            check(res[i], d[lo:hi + 1], "row %d" % i)
    check_all(O.window(t, ["p"], orders, [spec]).column("s").to_pylist())
    bad = _prefix_difference(np.array(d), frames, seg_start)
    if func == "avg":
        bad = [s / (hi - lo + 1) for s, (lo, hi) in zip(bad, frames)]
    with pytest.raises(AssertionError):
        check_all(bad)
    if frame == ("rows", -1, 1):    # the frames of rows 2..4 of both partitions: 6, 9, 7 against NaN and 0
        want = [6.0, 9.0, 7.0] if func == "sum" else [2.0, 3.0, 3.5]
        got = O.window(t, ["p"], orders, [spec]).column("s").to_pylist()
        assert got[2:5] == want and got[7:10] == want
        assert all(x != x for x in bad[2:5]) and bad[7:10] == [0.0, 0.0, 0.0]
    if frame == ("rows", 0, None) and func == "avg":
        assert O.window(t, ["p"], orders, [spec]).column("s").to_pylist()[6] == 2.5 and bad[6] == 0.0
