"""FilterExec over one string column on the GPU (csrc/expr.cu predicate_kernel with the matchers of csrc/strpred.cuh), on seeded
host-generated data shaped like the TPC-H columns the predicates come from.

Each case uses the largest row count whose arena stays under 2^31 bytes (Arrow string offsets are int32).  Time is the device
time of the predicate evaluation ("filter_project" section, CUDA events) per call, after warm-up.  Algorithmic bytes =
4 (n + 1) offsets + arena + validity (none here) + n mask bytes.  The mask is checked against numpy (verdicts of the distinct
strings, computed with Python's bytes / re, gathered by row).  Prints one JSON line per case and one for the card.

    python tools/string_filter_bench.py [--steps 10] [--warmup 3] [--max-rows N]
"""
import argparse
import ctypes as C
import json
import os
import re
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_PEAK = 3.35e12          # H100 SXM data sheet
LIMIT = 2 ** 31


def pools(rng):
    """name -> list of distinct byte strings."""
    segments = ["AUTOMOBILE", "BUILDING", "FURNITURE", "MACHINERY", "HOUSEHOLD"]
    types = ["%s %s %s" % (a, b, c) for a in ("STANDARD", "SMALL", "MEDIUM", "LARGE", "ECONOMY", "PROMO")
             for b in ("ANODIZED", "BURNISHED", "PLATED", "POLISHED", "BRUSHED") for c in ("TIN", "NICKEL", "BRASS", "STEEL", "COPPER")]
    colors = ["almond", "antique", "aquamarine", "azure", "beige", "bisque", "black", "blanched", "blue", "blush", "brown", "burlywood",
              "chartreuse", "chiffon", "chocolate", "coral", "cornflower", "cream", "cyan", "dark", "deep", "dim", "dodger", "drab",
              "firebrick", "forest", "frosted", "gainsboro", "ghost", "goldenrod", "green", "grey", "honeydew", "hot", "indian", "ivory"]
    names = [" ".join(rng.choice(colors, 5, replace=False)) for _ in range(4096)]
    words = ["carefully", "final", "deposits", "special", "requests", "furiously", "ironic", "packages", "blithely", "pending",
             "accounts", "quickly", "express", "theodolites", "slyly", "regular", "instructions", "bold", "foxes", "even"]
    comments = []
    while len(comments) < 4096:
        want = int(rng.integers(19, 79))
        c = ""
        while len(c) < want:
            c += ("" if not c else " ") + str(rng.choice(words))
        comments.append(c[:want])
    shipmodes = ["REG AIR", "AIR", "RAIL", "SHIP", "TRUCK", "MAIL", "FOB"]
    enc = lambda xs: [x.encode() for x in xs]          # noqa: E731
    return {"segment": enc(segments), "p_type": enc(types), "p_name": enc(names), "comment": enc(comments), "shipmode": enc(shipmodes)}


def cases():
    from spark_b200.expressions import In, Like, Not, col
    s = col("s")
    return [("c_mktsegment = 'BUILDING'", "segment", s.eq("BUILDING"), lambda v: v == b"BUILDING"),
            ("p_type LIKE '%BRASS'", "p_type", Like(s, "%BRASS"), lambda v: re.fullmatch(r"(?s).*BRASS", v.decode()) is not None),
            ("p_type LIKE 'PROMO%'", "p_type", Like(s, "PROMO%"), lambda v: re.fullmatch(r"(?s)PROMO.*", v.decode()) is not None),
            ("p_name LIKE '%green%'", "p_name", Like(s, "%green%"), lambda v: re.fullmatch(r"(?s).*green.*", v.decode()) is not None),
            ("o_comment NOT LIKE '%special%requests%'", "comment", Not(Like(s, "%special%requests%")),
             lambda v: re.fullmatch(r"(?s).*special.*requests.*", v.decode()) is None),
            ("l_shipmode IN (7 literals)", "shipmode", In(s, ["MAIL", "SHIP", "AIR", "TRUCK", "FOB", "BARGE", "POST"]),
             lambda v: v in (b"MAIL", b"SHIP", b"AIR", b"TRUCK", b"FOB", b"BARGE", b"POST"))]


def build_column(pool, n_cap, rng):
    """(idx per row, offsets int32, arena uint8) for the largest n <= n_cap whose arena is < 2^31 bytes."""
    lens = np.array([len(p) for p in pool], np.int64)
    n = min(n_cap, int((LIMIT - 1) / lens.mean() * 1.02) + 4096)   # enough rows on average; trimmed to the limit below
    idx = rng.integers(0, len(pool), n).astype(np.int32)
    ends = np.cumsum(lens[idx])
    n = int(np.searchsorted(ends, LIMIT - 1, side="right"))
    n = min(n, n_cap)
    idx, ends = idx[:n], ends[:n]
    offs = np.zeros(n + 1, np.int32)
    offs[1:] = ends
    pool_arena = np.frombuffer(b"".join(pool), np.uint8)
    pool_off = np.concatenate([[0], np.cumsum(lens)])
    arena = np.empty(int(ends[-1]) if n else 0, np.uint8)
    chunk = 1 << 22
    for a in range(0, n, chunk):
        b = min(n, a + chunk)
        l = lens[idx[a:b]]
        start = offs[a]
        pos = np.repeat(pool_off[idx[a:b]] - (offs[a:b].astype(np.int64) - start), l) + np.arange(int(l.sum()))
        arena[start:start + len(pos)] = pool_arena[pos]
    return idx, offs, arena


def gpu_card():
    q = "name,power.limit,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True, timeout=60)
    return dict(zip(q.split(","), [x.strip() for x in r.stdout.strip().splitlines()[0].split(",")])) if r.returncode == 0 else {"error": r.stderr}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--max-rows", type=int, default=1 << 40)
    args = ap.parse_args()
    from spark_b200 import _capi as capi
    from spark_b200.columnar import ColumnarBatch, HostColumn, Stream
    from spark_b200.expressions import CompiledExpr, Schema, col
    lib = capi.init(0)
    print(json.dumps({"card": gpu_card()}), flush=True)
    stream = Stream()
    rng = np.random.default_rng(2026)
    P = pools(rng)
    schema = Schema(["s", "row"], [capi.SB_STRING, capi.SB_INT32])
    columns = {}
    for label, pool_name, expr, ref in cases():
        if pool_name not in columns:
            columns.clear()
            idx, offs, arena = build_column(P[pool_name], args.max_rows, rng)
            n = len(idx)
            host = [HostColumn(capi.SB_STRING, arena, None, offs, 0, n), HostColumn(capi.SB_INT32, np.arange(n, dtype=np.int32), None, None, 0, n)]
            columns[pool_name] = (idx, offs, arena, ColumnarBatch.from_host_columns(["s", "row"], host, stream))
            stream.synchronize()
        idx, offs, arena, batch = columns[pool_name]
        n = len(idx)
        want = np.array([bool(ref(v)) for v in P[pool_name]])[idx]
        pred = CompiledExpr(expr, schema)
        proj = CompiledExpr(col("row"), schema)
        res = {"case": label, "rows": n, "arena_bytes": int(arena.size)}
        nbytes = 4 * (n + 1) + int(arena.size) + 0 + n
        h = C.c_void_p()
        capi.check(lib.sb_filter_project(batch.handle, C.byref(pred.c), C.byref(proj.c), 1, stream.handle, C.byref(h)))
        got = ColumnarBatch(h, ["row"])
        rows = got.to_arrow(stream).column("row").to_numpy()
        got.close()
        ok = bool(np.array_equal(rows, np.flatnonzero(want)))
        for _ in range(args.warmup):
            capi.check(lib.sb_filter_project(batch.handle, C.byref(pred.c), None, 0, stream.handle, C.byref(h)))
            capi.check(lib.sb_table_release(h))
        stream.synchronize()
        capi.check(lib.sb_profile_enable(1))
        capi.check(lib.sb_profile_reset())
        for _ in range(args.steps):
            capi.check(lib.sb_filter_project(batch.handle, C.byref(pred.c), None, 0, stream.handle, C.byref(h)))
            capi.check(lib.sb_table_release(h))
        stream.synchronize()
        ms, launches = C.c_double(), C.c_int64()
        capi.check(lib.sb_profile_get(b"filter_project", C.byref(ms), C.byref(launches)))
        capi.check(lib.sb_profile_enable(0))
        t = ms.value / max(1, launches.value)
        res.update({"ms": round(t, 4), "GB_s": round(nbytes / (t * 1e-3) / 1e9, 1), "hbm_share": round(nbytes / (t * 1e-3) / HBM_PEAK, 3),
                    "verified": ok})
        res["algorithmic_bytes"] = nbytes
        res["matches"] = int(want.sum())
        print(json.dumps(res), flush=True)
    for v in columns.values():
        v[3].close()
    stream.close()


if __name__ == "__main__":
    main()
