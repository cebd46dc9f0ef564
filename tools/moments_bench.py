"""VAR_SAMP in the hash aggregate (csrc/moments.cu) on 2^28 float64 rows with int32 keys at 4, 1 000 and 10^6 groups: the whole
call, the pass-1 update kernel, the pass-2 kernel and the finish kernel (device events, best of 5 after 2 warm-ups), the whole call
of a SUM + COUNT plan over the same data, and pass 2's bytes (keys + values) over its time as a share of the H100 SXM's 3.35 TB/s.

The values are 1e9 + j * 2^-10 with j a random integer in [-4096, 4096]: exactly representable, unit-scale spread on a 1e9 offset
(where the naive sum x^2 - (sum x)^2 / n keeps no digit), and the exact per-group M2 follows from integer sums of j and j^2, so
every answer is checked against the bound of tests/test_gpu_moments.py.  One JSON line per group count; the card's name and power
limit come with the numbers.  Usage: python tools/moments_bench.py [--rows-log2 28]"""
import ctypes as C
import json
import os
import subprocess
import sys
from fractions import Fraction

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from spark_b200 import _capi as capi                                        # noqa: E402
from spark_b200.columnar import ColumnarBatch, Stream                        # noqa: E402
from spark_b200.execution import HashAggregateExec, LocalTableScanExec       # noqa: E402
from spark_b200.expressions import Count, Sum, VarianceSamp, col             # noqa: E402

HBM_TBS = 3.35
KERNELS = ("agg_update", "moment_pass2", "moment_finish")
EPS = Fraction(1, 2 ** 52)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return out.stdout.strip().splitlines()[0]
    except Exception as e:   # the numbers are still printed; the card is then unknown
        return "unknown (%s)" % e


def timed(lib, stream, fn, reps=5, warm=2):
    for _ in range(warm):
        fn().close()
    best = None
    capi.check(lib.sb_profile_enable(1))
    for _ in range(reps):
        capi.check(lib.sb_profile_reset())
        stream.record_start()
        out = fn()
        stream.record_stop()
        ms = stream.elapsed_ms()
        out.close()
        k = {}
        for name in KERNELS:
            t, c = C.c_double(), C.c_int64()
            capi.check(lib.sb_profile_get(name.encode(), C.byref(t), C.byref(c)))
            k[name] = t.value
        if best is None or ms < best[0]:
            best = (ms, k)
    capi.check(lib.sb_profile_enable(0))
    return best


def check(res, keys, j, ngroups):
    """every group's var_samp against the exact one: |m2 - M2| <= 2 (m + 2) 2^-52 (M2 + m D^2), D = 2^-52 sum |x|."""
    cnt = np.bincount(keys, minlength=ngroups)
    # float64 sums of integers below 2^53 (|j| <= 2^12, at most 2^28 rows): exact
    sj = np.bincount(keys, weights=j.astype(np.float64), minlength=ngroups)
    sjj = np.bincount(keys, weights=(j * j).astype(np.float64), minlength=ngroups)
    got_k = res.column("k").to_numpy()
    got_v = res.column("v").to_pylist()
    bad = 0
    for g, v in zip(got_k.tolist(), got_v):
        m = int(cnt[g])
        m2 = Fraction(int(sjj[g]), 2 ** 20) - Fraction(int(sj[g]) ** 2, m * 2 ** 20)
        d = EPS * (m * Fraction(10 ** 9) + Fraction(4096, 1024) * m)
        err = 2 * (m + 2) * EPS * (m2 + m * d * d)
        lo, hi = max(m2 - err, 0) / (m - 1) * (1 - EPS), (m2 + err) / (m - 1) * (1 + EPS)
        bad += not (v is not None and lo <= Fraction(v) <= hi)
    return bad


def main():
    rows_log2 = int(sys.argv[sys.argv.index("--rows-log2") + 1]) if "--rows-log2" in sys.argv else 28
    n = 1 << rows_log2
    lib = capi.init(0)
    stream = Stream()
    rng = np.random.default_rng(0)
    j = rng.integers(-4096, 4097, n, dtype=np.int64)
    x = 1e9 + j.astype(np.float64) * 2.0 ** -10
    name = card()
    for ngroups in (4, 1000, 1_000_000):
        keys = rng.integers(0, ngroups, n, dtype=np.int32)
        batch = ColumnarBatch.from_numpy({"k": keys, "x": x}, stream)
        stream.synchronize()
        moments = HashAggregateExec(["k"], [(VarianceSamp(col("x")), "v")], LocalTableScanExec(batch))
        sums = HashAggregateExec(["k"], [(Sum(col("x")), "s"), (Count(col("x")), "c")], LocalTableScanExec(batch))
        ms, k = timed(lib, stream, lambda: moments.run(batch, stream))
        ms_sum, _ = timed(lib, stream, lambda: sums.run(batch, stream))
        res = moments.run(batch, stream)
        tbl = res.to_arrow(stream)
        res.close()
        bad = check(tbl, keys, j, ngroups)
        pass2_bytes = n * (4 + 8)
        print(json.dumps({"case": "var_samp", "rows": n, "groups": ngroups, "card": name, "call_ms": ms, "sum_count_call_ms": ms_sum,
                          "ratio_to_sum_count": ms / ms_sum, "pass1_ms": k["agg_update"], "pass2_ms": k["moment_pass2"],
                          "finish_ms": k["moment_finish"], "pass2_bytes": pass2_bytes,
                          "pass2_frac_of_hbm": pass2_bytes / (k["moment_pass2"] / 1e3) / (HBM_TBS * 1e12) if k["moment_pass2"] > 0 else None,
                          "groups_checked": tbl.num_rows, "groups_outside_bound": bad}), flush=True)
        batch.close()
        if bad:
            raise SystemExit("%d groups outside the exact bound" % bad)
    stream.close()


if __name__ == "__main__":
    main()
