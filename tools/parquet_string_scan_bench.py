"""Parquet BYTE_ARRAY / DELTA scan on the GPU: per encoding, the H2D copy of the encoded column chunk against the decode kernels.

    python tools/parquet_string_scan_bench.py [--rows N] [--steps K] [--warmup W]

Writes uncompressed files with pyarrow (one row group per file, pyarrow's default 1 MB pages) into a temporary directory, checks
that the GPU decode equals pq.read_table, then reports per case, after W warm-up steps and averaged over K steps:
  copy_ms      H2D of the encoded chunk from pinned memory (sb_table_import_host of its bytes, stream events);
  decode_ms    the scan kernels (sb_profile: scan_decode, scan_decode_strings, scan_copy_strings; the H2D excluded);
  call_ms      one whole sb_scan_decode (copy + kernels + the one synchronisation of a string column), stream events;
  decoded_GB_s decoded column bytes (offsets + arena, or values) / decode_ms;
  larger       which of copy and decode takes longer.
The first line is the card (name, power limit, max SM clock): they are part of every number.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import pyarrow as pa  # noqa: E402
import pyarrow.compute as pc  # noqa: E402
import pyarrow.parquet as pq  # noqa: E402


def gpu_card():
    q = "name,power.limit,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True, timeout=60)
    return dict(zip(q.split(","), [x.strip() for x in r.stdout.strip().splitlines()[0].split(",")])) if r.returncode == 0 else {"error": r.stderr}


WORDS = ("furiously quickly carefully blithely slyly final regular special pending express ironic bold even silent unusual "
         "deposits requests accounts packages instructions theodolites foxes pinto beans asymptotes platelets dependencies "
         "excuses ideas dolphins sheaves warhorses courts frets sauternes").split()


def comments(n, rng):
    """l_comment-like: 19-78 bytes of random words; a pool of 200 000 distinct comments, drawn with replacement."""
    pool = []
    for _ in range(200_000):
        target = int(rng.integers(19, 79))
        s = ""
        while len(s) < target:
            s += WORDS[int(rng.integers(0, len(WORDS)))] + " "
        pool.append(s[:target])
    return pa.array(pool).take(pa.array(rng.integers(0, len(pool), n)))


def cases(n, rng):
    segments = ["AUTOMOBILE", "BUILDING", "FURNITURE", "HOUSEHOLD", "MACHINERY"]
    types = ["%s %s %s" % (a, b, c) for a in ("STANDARD", "SMALL", "MEDIUM", "LARGE", "ECONOMY", "PROMO")
             for b in ("ANODIZED", "BURNISHED", "PLATED", "POLISHED", "BRUSHED") for c in ("TIN", "NICKEL", "BRASS", "STEEL", "COPPER")]
    seg = pa.array(segments).take(pa.array(rng.integers(0, 5, n)))
    ptype = pa.array(types).take(pa.array(rng.integers(0, len(types), n)))
    com = comments(n, rng)
    keys = pa.array(["customer#%012d" % i for i in range(n)])
    ints = pa.array(np.cumsum(rng.integers(0, 1000, n)).astype(np.int64))
    return [("c_mktsegment dictionary", seg, "DICTIONARY"), ("p_type dictionary", ptype, "DICTIONARY"),
            ("l_comment PLAIN", com, "PLAIN"), ("l_comment DELTA_LENGTH_BYTE_ARRAY", com, "DELTA_LENGTH_BYTE_ARRAY"),
            ("l_comment DELTA_BYTE_ARRAY", com, "DELTA_BYTE_ARRAY"), ("sorted key DELTA_BYTE_ARRAY", keys, "DELTA_BYTE_ARRAY"),
            ("int64 DELTA_BINARY_PACKED", ints, "DELTA_BINARY_PACKED")]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1 << 22)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    from spark_b200 import _capi as capi
    from spark_b200.columnar import ColumnarBatch, HostColumn, PinnedArray, Stream
    from spark_b200.scan import EncodedColumnChunk, ParquetScanExec, decode_chunks
    lib = capi.init(0)
    print(json.dumps({"card": gpu_card()}), flush=True)
    stream = Stream()
    rng = np.random.default_rng(2026)
    tmp = tempfile.mkdtemp(prefix="pq_string_bench_")
    for label, arr, enc in cases(args.rows, rng):
        path = os.path.join(tmp, "c.parquet")
        kw = dict(use_dictionary=True) if enc == "DICTIONARY" else dict(use_dictionary=False, column_encoding={"c": enc})
        pq.write_table(pa.table({"c": arr}), path, compression="NONE", row_group_size=args.rows, **kw)
        scan = ParquetScanExec(path)
        ch = scan.row_group_chunks(0)[0]
        pinned = PinnedArray(ch.nbytes, np.uint8)
        pinned.array[:] = ch.data
        ch = EncodedColumnChunk(ch.type, ch.scale, ch.physical, pinned.array, ch.pages, ch.npages, ch.dict_offset, ch.dict_count)
        b = decode_chunks(["c"], [ch], stream, [arr.type])
        ok = b.to_arrow(stream).column("c").combine_chunks().equals(pq.read_table(path).column("c").combine_chunks())
        b.close()
        # H2D of the chunk's bytes
        host = [HostColumn(capi.SB_INT8, pinned.array.view(np.int8), None, None, 0, ch.nbytes)]
        for _ in range(args.warmup):
            ColumnarBatch.from_host_columns(["b"], host, stream).close()
        stream.synchronize()
        copy = 0.0
        for _ in range(args.steps):
            stream.record_start()
            t = ColumnarBatch.from_host_columns(["b"], host, stream)
            stream.record_stop()
            copy += stream.elapsed_ms()
            t.close()
        # the decode
        for _ in range(args.warmup):
            decode_chunks(["c"], [ch], stream, [arr.type]).close()
        stream.synchronize()
        capi.check(lib.sb_profile_enable(1))
        capi.check(lib.sb_profile_reset())
        call = 0.0
        for _ in range(args.steps):
            stream.record_start()
            t = decode_chunks(["c"], [ch], stream, [arr.type])
            stream.record_stop()
            call += stream.elapsed_ms()
            t.close()
        stream.synchronize()
        prof = capi.profile_dump()
        capi.check(lib.sb_profile_enable(0))
        kern = {k: round(v[0] / args.steps, 4) for k, v in prof.items() if k.startswith("scan_")}
        decode = sum(kern.values())
        if pa.types.is_string(arr.type):
            decoded = 4 * (args.rows + 1) + int(pc.sum(pc.binary_length(arr)).as_py())
        else:
            decoded = 8 * args.rows
        copy /= args.steps
        res = {"case": label, "rows": args.rows, "chunk_MB": round(ch.nbytes / 1e6, 2), "pages": ch.npages, "copy_ms": round(copy, 4),
               "copy_GB_s": round(ch.nbytes / (copy * 1e-3) / 1e9, 1), "decode_ms": round(decode, 4), "kernels_ms": kern,
               "call_ms": round(call / args.steps, 4), "decoded_MB": round(decoded / 1e6, 1),
               "decoded_GB_s": round(decoded / (decode * 1e-3) / 1e9, 1), "larger": "decode" if decode > copy else "copy", "verified": bool(ok)}
        print(json.dumps(res), flush=True)
        scan = None
        pinned.close()
        os.remove(path)
    os.rmdir(tmp)
    stream.close()


if __name__ == "__main__":
    main()
