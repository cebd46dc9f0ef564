"""Parquet SNAPPY scan on the GPU: per case, the H2D copy of the compressed chunks against the Snappy kernels and the decode.

    python tools/parquet_snappy_scan_bench.py [--q1-rows N] [--rows N] [--steps K] [--warmup W]

Cases: the Q1 row group (the seven lineitem columns of tpch.lineitem_q1_table in one call, one row group) and the string cases
of tools/parquet_string_scan_bench.py, each written by pyarrow SNAPPY and NONE (default 1 MB pages) into a temporary directory.
Every decode is checked against pq.read_table.  Per case, after W warm-up steps and averaged over K steps:
  compressed_MB / uncompressed_MB   chunk bytes of the SNAPPY file, and the page bytes they decompress to;
  copy_ms        H2D of the SNAPPY chunks from pinned memory (sb_table_import_host of their bytes, stream events);
  snappy_ms      scan_snappy + scan_resolve_pages (sb_profile);
  decode_ms      the decode kernels that follow (sb_profile: scan_decode, scan_decode_strings, scan_copy_strings);
  call_ms        one whole sb_scan_decode_compressed (SNAPPY file) and sb_scan_decode (NONE file), stream events;
  decompressed_GB_s   uncompressed_MB / snappy_ms.
The first line is the card (name, power limit, max SM clock): they are part of every number.
"""
import argparse
import json
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

import pyarrow as pa  # noqa: E402
import pyarrow.parquet as pq  # noqa: E402

from parquet_string_scan_bench import cases, gpu_card  # noqa: E402


def timed(stream, fn, steps, warmup):
    for _ in range(warmup):
        fn().close()
    stream.synchronize()
    total = 0.0
    for _ in range(steps):
        stream.record_start()
        t = fn()
        stream.record_stop()
        total += stream.elapsed_ms()
        t.close()
    stream.synchronize()
    return total / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--q1-rows", type=int, default=1 << 24)
    ap.add_argument("--rows", type=int, default=1 << 22)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    from spark_b200 import _capi as capi, tpch
    from spark_b200.columnar import ColumnarBatch, HostColumn, PinnedArray, Stream
    from spark_b200.scan import CompressedColumnChunk, EncodedColumnChunk, ParquetScanExec, decode_chunks, decode_file_chunks
    lib = capi.init(0)
    print(json.dumps({"card": gpu_card()}), flush=True)
    stream = Stream()
    rng = np.random.default_rng(2026)
    tmp = tempfile.mkdtemp(prefix="pq_snappy_bench_")
    q1 = tpch.lineitem_q1_table(args.q1_rows, seed=7)
    work = [("Q1 row group", q1, dict(row_group_size=args.q1_rows))]
    for label, arr, enc in cases(args.rows, rng):
        kw = dict(use_dictionary=True) if enc == "DICTIONARY" else dict(use_dictionary=False, column_encoding={"c": enc})
        work.append((label, pa.table({"c": arr}), dict(row_group_size=args.rows, **kw)))
    for label, table, kw in work:
        paths = {}
        for codec in ("SNAPPY", "NONE"):
            paths[codec] = os.path.join(tmp, codec + ".parquet")
            pq.write_table(table, paths[codec], compression=codec, **kw)
        names, types = table.column_names, [f.type for f in table.schema]
        keep = []

        def pinned(ch):
            p = PinnedArray(max(ch.nbytes, 1), np.uint8)
            p.array[:ch.nbytes] = ch.data
            keep.append(p)
            return p.array[:ch.nbytes]

        snappy_scan, none_scan = ParquetScanExec(paths["SNAPPY"]), ParquetScanExec(paths["NONE"])
        sch = [CompressedColumnChunk(c.type, c.scale, c.physical, c.codec, c.max_def_level, pinned(c), c.spans, c.npages)
               for c in snappy_scan.row_group_file_chunks(0)]
        nch = [EncodedColumnChunk(c.type, c.scale, c.physical, pinned(c), c.pages, c.npages, c.dict_offset, c.dict_count)
               for c in none_scan.row_group_chunks(0)]
        want = pq.read_table(paths["NONE"])
        ok = True
        for b in (decode_file_chunks(names, sch, stream, types), decode_chunks(names, nch, stream, types)):
            ok &= b.to_arrow(stream).equals(want)
            b.close()
        compressed = sum(c.nbytes for c in sch)
        uncompressed = sum(c.spans[i].uncompressed_bytes for c in sch for i in range(c.npages))
        whole = PinnedArray(compressed, np.uint8)                 # the SNAPPY chunks back to back: one H2D of all their bytes
        whole.array[:] = np.concatenate([c.data for c in sch])
        keep.append(whole)
        host = [HostColumn(capi.SB_INT8, whole.array.view(np.int8), None, None, 0, compressed)]
        copy = timed(stream, lambda: ColumnarBatch.from_host_columns(["b"], host, stream), args.steps, args.warmup)
        for _ in range(args.warmup):
            decode_file_chunks(names, sch, stream, types).close()
        capi.check(lib.sb_profile_enable(1))
        capi.check(lib.sb_profile_reset())
        call_snappy = timed(stream, lambda: decode_file_chunks(names, sch, stream, types), args.steps, 0)
        prof = capi.profile_dump()
        capi.check(lib.sb_profile_enable(0))
        call_none = timed(stream, lambda: decode_chunks(names, nch, stream, types), args.steps, args.warmup)
        kern = {k: round(v[0] / args.steps, 4) for k, v in prof.items() if k.startswith("scan_")}
        snappy = kern.get("scan_snappy", 0.0) + kern.get("scan_resolve_pages", 0.0)
        decode = sum(v for k, v in kern.items() if k not in ("scan_snappy", "scan_resolve_pages"))
        res = {"case": label, "rows": table.num_rows, "columns": len(names), "pages": sum(c.npages for c in sch),
               "compressed_MB": round(compressed / 1e6, 2), "uncompressed_MB": round(uncompressed / 1e6, 2),
               "none_chunk_MB": round(sum(c.nbytes for c in nch) / 1e6, 2), "copy_ms": round(copy, 4), "snappy_ms": round(snappy, 4),
               "decode_ms": round(decode, 4), "kernels_ms": kern, "call_ms_snappy": round(call_snappy, 4), "call_ms_none": round(call_none, 4),
               "decompressed_GB_s": round(uncompressed / (snappy * 1e-3) / 1e9, 1) if snappy > 0 else None,
               "snappy_within_copy": snappy <= copy, "snappy_call_within_none": call_snappy <= call_none, "verified": bool(ok)}
        print(json.dumps(res), flush=True)
        for p in keep:
            p.close()
        snappy_scan = none_scan = None
        for p in paths.values():
            os.remove(p)
    os.rmdir(tmp)
    stream.close()


if __name__ == "__main__":
    main()
