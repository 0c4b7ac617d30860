"""Filtered top-k on the H100: int8 10M x 384, k = 20, L2, eligible sets of 100 % / 10 % / 1 % of the rows, random and clustered
(one contiguous block).  Measures, per set:
  * one query: vsb_scan_topk_filtered against vsb_scan_topk (ms per call, median of the timed calls);
  * a batch of B = 1024 queries through the filtered batch path against the same B queries as filtered single calls;
  * the bitmap upload alone: a filtered call with k = 0 (argument checks + one 1.25 MB host -> device copy + stream sync).
Every filtered batch must equal its single calls (rowids and distances).  Writes the JSON to --out (default
profiles/h100_filtered.json) with the card's name, power limit and max SM clock read in the same run.

    python tools/filtered_bench.py [--rows 10000000] [--dim 384] [--single 20] [--batch 1024]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info():
    q = "name,power.limit,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 else "unknown"


def timed(fn, reps):
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    return 1e3 * float(np.median(ts)), ts


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--dim", type=int, default=384)
    ap.add_argument("--k", type=int, default=20)
    ap.add_argument("--single", type=int, default=20, help="timed single queries per leg")
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_filtered.json"))
    a = ap.parse_args()
    import sqlite_vector_b200 as vs
    eng = vs.load_engine()
    if eng.device_count() < 1:
        raise SystemExit("filtered_bench needs a CUDA device")
    rng = np.random.Generator(np.random.PCG64(42))
    n, dim, k, B = a.rows, a.dim, a.k, a.batch
    x = np.frombuffer(rng.bytes(n * dim), dtype=np.int8).reshape(n, dim)
    q = np.frombuffer(rng.bytes(B * dim), dtype=np.int8).reshape(B, dim)
    ix = vs.Index(vs.api.I8, dim, n)
    for s in range(0, n, 1 << 20):
        ix.append_dense(x[s:s + (1 << 20)])
    ix.finalize()
    sets = {"all": np.ones(n, bool)}
    for sel in (0.1, 0.01):
        sets[f"random{sel}"] = rng.random(n) < sel
        blk = np.zeros(n, bool)
        a0 = int(n * 0.6)
        blk[a0:a0 + int(n * sel)] = True
        sets[f"clustered{sel}"] = blk
    res = {"gpu": gpu_info(), "rows": n, "dim": dim, "k": k, "batch": B, "metric": "L2", "type": "int8", "sets": {}}
    # warm-up of every path
    ix.scan_topk(vs.api.L2, q[0], k)
    ix.scan_topk(vs.api.L2, q, k, as_arrays=True)
    plain_ms, _ = timed(lambda: ix.scan_topk(vs.api.L2, q[1], k), a.single)
    plain_batch_ms, _ = timed(lambda: ix.scan_topk(vs.api.L2, q, k, as_arrays=True), 3)
    res["unfiltered"] = {"single_ms": plain_ms, "batch_ms": plain_batch_ms}
    for name, m in sets.items():
        bits = vs.api.row_bitmap(m)
        ix.scan_topk_filtered(vs.api.L2, q[0], k, bits)                                     # warm-up
        single_ms, _ = timed(lambda: ix.scan_topk_filtered(vs.api.L2, q[2], k, bits), a.single)
        upload_ms, _ = timed(lambda: ix.scan_topk_filtered(vs.api.L2, q[2], 0, bits), a.single)
        b0, f0 = ix.stat("batches"), ix.stat("fallbacks")
        batch_ms, _ = timed(lambda: ix.scan_topk_filtered(vs.api.L2, q, k, bits, as_arrays=True), 3)
        batched = ix.stat("batches") - b0
        fell = ix.stat("fallbacks") - f0
        got = ix.scan_topk_filtered(vs.api.L2, q, k, bits, as_arrays=True)
        t0 = time.perf_counter()
        singles = [ix.scan_topk_filtered(vs.api.L2, q[b], k, bits)[0] for b in range(B)]
        singles_ms = 1e3 * (time.perf_counter() - t0)
        same = all(np.array_equal(got[0][b, :got[2][b]], singles[b][0]) and np.array_equal(got[1][b, :got[2][b]], singles[b][1]) for b in range(B))
        res["sets"][name] = {"eligible": int(m.sum()), "single_ms": single_ms, "upload_ms": upload_ms, "batch_ms": batch_ms,
                             "batch_single_calls_ms": singles_ms, "batches": int(batched), "fallbacks": int(fell), "batch_equals_singles": bool(same)}
        print(name, json.dumps(res["sets"][name]), flush=True)
    res["bitmap_bytes"] = int(vs.api.row_bitmap(sets["all"]).nbytes)
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))
    ix.close()


if __name__ == "__main__":
    main()
