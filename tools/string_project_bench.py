"""ProjectExec of string-producing functions on the GPU (sb_string_project, csrc/strfunc.cu) on seeded numpy-built columns.

Cases: substring(c_phone, 1, 2) over 15-byte phones; concat(a, '-', b) over 10-byte values; trim over values of 10..40 bytes with
0..3 spaces on either side; lpad(x, 20, '0') over 1..10-digit values.  Row counts keep every arena under 2^31 bytes.  Kernel time
is the device time of the two string_project kernels per call (CUDA events, after warm-up); call time adds the length scan and the
host read-back of the arena size.  Bytes = input offsets + input arenas + output offsets + output arena (no validity: the inputs
have no NULLs), over the kernel time and against 3.35 TB/s.  Every output is checked against numpy.  One JSON line per case and one
for the card (its name and power limit, read in the same run).

    python tools/string_project_bench.py [--steps 10] [--warmup 3] [--scale 1.0]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_PEAK = 3.35e12          # H100 SXM data sheet


def gpu_card():
    q = "name,power.limit,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True, timeout=60)
    return dict(zip(q.split(","), [x.strip() for x in r.stdout.strip().splitlines()[0].split(",")])) if r.returncode == 0 else {"error": r.stderr}


def fixed(rng, n, w, alphabet):
    return rng.choice(np.frombuffer(alphabet, np.uint8), (n, w))


def case_substring(rng, n):
    ph = fixed(rng, n, 15, b"0123456789")
    ph[:, [2, 6, 10]] = ord("-")
    cols = {"c_phone": (np.arange(n + 1, dtype=np.int32) * 15, ph.ravel())}
    want = ph[:, :2].ravel()
    return cols, want, np.arange(n + 1, dtype=np.int64) * 2


def case_concat(rng, n):
    a, b = fixed(rng, n, 10, b"abcdefghij"), fixed(rng, n, 10, b"KLMNOPQRST")
    offs = np.arange(n + 1, dtype=np.int32) * 10
    want = np.concatenate([a, np.full((n, 1), ord("-"), np.uint8), b], axis=1).ravel()
    return {"a": (offs, a.ravel()), "b": (offs, b.ravel())}, want, np.arange(n + 1, dtype=np.int64) * 21


def case_trim(rng, n):
    core = rng.integers(4, 35, n)
    lead, trail = rng.integers(0, 4, n), rng.integers(0, 4, n)
    lens = core + lead + trail
    offs = np.zeros(n + 1, np.int64)
    np.cumsum(lens, out=offs[1:])
    arena = rng.choice(np.frombuffer(b"abcdefghijklmnopqrstuvwxyz", np.uint8), int(offs[-1]))
    pos = np.arange(int(offs[-1])) - np.repeat(offs[:-1], lens)
    row_len = np.repeat(lens, lens)
    pad = (pos < np.repeat(lead, lens)) | (pos >= row_len - np.repeat(trail, lens))
    arena[pad] = ord(" ")
    wo = np.zeros(n + 1, np.int64)
    np.cumsum(core, out=wo[1:])
    return {"s": (offs.astype(np.int32), arena)}, arena[~pad], wo


def case_lpad(rng, n):
    l = rng.integers(1, 11, n)
    offs = np.zeros(n + 1, np.int64)
    np.cumsum(l, out=offs[1:])
    arena = rng.choice(np.frombuffer(b"0123456789", np.uint8), int(offs[-1]))
    out = np.full((n, 20), ord("0"), np.uint8)
    out[np.arange(20)[None, :] >= (20 - l)[:, None]] = arena
    return {"x": (offs.astype(np.int32), arena)}, out.ravel(), np.arange(n + 1, dtype=np.int64) * 20


def cases(scale):
    from spark_b200.expressions import Concat, StringLPad, StringTrim, Substring, col
    return [("substring(c_phone, 1, 2)", case_substring, int(120e6 * scale), Substring(col("c_phone"), 1, 2)),
            ("concat(a, '-', b)", case_concat, int(100e6 * scale), Concat(col("a"), "-", col("b"))),
            ("trim(s), 10..40 bytes", case_trim, int(10e6 * scale), StringTrim(col("s"))),
            ("lpad(x, 20, '0')", case_lpad, int(60e6 * scale), StringLPad(col("x"), 20, "0"))]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--scale", type=float, default=1.0)
    args = ap.parse_args()
    from spark_b200 import _capi as capi
    from spark_b200.columnar import ColumnarBatch, HostColumn, Stream
    from spark_b200.expressions import CompiledStringProgram, Schema
    lib = capi.init(0)
    print(json.dumps({"card": gpu_card()}), flush=True)
    stream = Stream()
    rng = np.random.default_rng(2026)
    for label, make, n, expr in cases(args.scale):
        cols, want, want_offs = make(rng, n)
        names = list(cols)
        host = [HostColumn(capi.SB_STRING, cols[c][1], None, cols[c][0], 0, n) for c in names]
        batch = ColumnarBatch.from_host_columns(names, host, stream)
        stream.synchronize()
        prog = CompiledStringProgram(expr, Schema(names, [capi.SB_STRING] * len(names)))
        h = C.c_void_p()
        capi.check(lib.sb_string_project(batch.handle, C.byref(prog.c), 1, stream.handle, C.byref(h)))
        got = ColumnarBatch(h, ["o"]).to_arrow(stream).column("o").combine_chunks()
        _, go, gd = got.buffers()
        go = np.frombuffer(go, np.int32, n + 1)
        ok = bool(np.array_equal(go, want_offs) and np.array_equal(np.frombuffer(gd, np.uint8, int(want_offs[-1])), want))
        del got, go, gd
        for _ in range(args.warmup):
            capi.check(lib.sb_string_project(batch.handle, C.byref(prog.c), 1, stream.handle, C.byref(h)))
            capi.check(lib.sb_table_release(h))
        stream.synchronize()
        capi.check(lib.sb_profile_enable(1))
        capi.check(lib.sb_profile_reset())
        stream.record_start()
        for _ in range(args.steps):
            capi.check(lib.sb_string_project(batch.handle, C.byref(prog.c), 1, stream.handle, C.byref(h)))
            capi.check(lib.sb_table_release(h))
        stream.record_stop()
        call_ms = stream.elapsed_ms() / args.steps
        ms, launches = C.c_double(), C.c_int64()
        capi.check(lib.sb_profile_get(b"string_project", C.byref(ms), C.byref(launches)))
        capi.check(lib.sb_profile_enable(0))
        t = ms.value / args.steps
        in_bytes = sum(4 * (n + 1) + int(cols[c][1].size) for c in names)
        out_bytes = 4 * (n + 1) + int(want_offs[-1])
        nbytes = in_bytes + out_bytes
        print(json.dumps({"case": label, "rows": n, "in_bytes": in_bytes, "out_bytes": out_bytes, "kernel_ms": round(t, 3),
                          "call_ms": round(call_ms, 3), "GB_s": round(nbytes / (t * 1e-3) / 1e9, 1),
                          "hbm_share": round(nbytes / (t * 1e-3) / HBM_PEAK, 3), "verified": ok}), flush=True)
        batch.close()
    stream.close()


if __name__ == "__main__":
    main()
