"""Batched L1 queries on one GPU: the L1 batch path (l1_batch_kernel + refine + replay) against the per-query path.

  python tools/l1_batch_bench.py [--n 10000000] [--dim 384] [--k 20] [--out profiles/h100_l1_batch.json]

For int8 and f32 columns of n x dim, batches of 1024 and 16 host queries through vsb_scan_topk (host in, host out):
  * queries/s of the batch (median of --reps timed calls after one warm-up call);
  * queries/s of the per-query path (option no_batch = 1) on --sample queries, timed in the same process;
  * the L1 kernel's device time per batch (CUDA events of the levels, stat "tc_us") and the element pairs it computed per
    second (rows scored x queries x dim / kernel time);
  * the L1 kernel alone over all rows with each tile width N (vsb_debug_tc_level, bounds 0: no hits), host-timed;
  * parity: int8 bit-exact against the oracle on 3 queries, f32 against the oracle under tests/fpcheck.py on 3 queries.
The GPU's name, power limit and maximum SM clock are read in the same run.  Prints one JSON document."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import sqlite_vector_b200 as vs  # noqa: E402
from oracle import pyoracle as po  # noqa: E402
from tests.fpcheck import assert_fp_topk  # noqa: E402


def gpu_info():
    q = "name,power.limit,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True, timeout=60)
    first = r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else ""
    return dict(zip(q.split(","), [v.strip() for v in first.split(",")])) if first else {"error": r.stderr.strip()[-200:]}


def column(vtype, n, dim, seed, chunk=1 << 20):
    """seeded column, generated in row chunks from random bytes (fast at 10M rows); f32 values are a / 16 + b / 4096 with
    random int8 a, b: few exact ties"""
    rng = np.random.Generator(np.random.PCG64(seed))
    out = np.empty((n, dim), dtype=np.int8 if vtype == po.I8 else np.float32)
    for a in range(0, n, chunk):
        m = min(chunk, n - a)
        r = np.frombuffer(rng.bytes(m * dim), dtype=np.int8).reshape(m, dim)
        if vtype == po.I8:
            out[a:a + m] = r
        else:
            s = np.frombuffer(rng.bytes(m * dim), dtype=np.int8).reshape(m, dim)
            out[a:a + m] = r.astype(np.float32) * np.float32(1 / 16) + s.astype(np.float32) * np.float32(1 / 4096)
    return out


def timed(fn, reps):
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    return ts


def leg(eng, oracle, vtype, n, dim, k, batches, reps, sample):
    name = "int8" if vtype == po.I8 else "f32"
    x = column(vtype, n, dim, 11)
    ix = vs.Index(vtype, dim, n)
    for a in range(0, n, 1 << 20):
        ix.append_dense(x[a:a + (1 << 20)])
    ix.finalize()
    qall = column(vtype, max(batches), dim, 12)
    out = {"type": name, "n": n, "dim": dim, "k": k}
    for B in batches:
        q = np.ascontiguousarray(qall[:B])
        ix.scan_topk(po.L1, q, k)                                            # warm-up: workspace, tensor maps, modules
        b0, f0, us0, rows0 = ix.stat("batches"), ix.stat("fallbacks"), ix.stat("tc_us"), ix.stat("tc_rows")
        res = None

        def run():
            nonlocal res
            res = ix.scan_topk(po.L1, q, k)
        ts = timed(run, reps)
        nb, nf = ix.stat("batches") - b0, ix.stat("fallbacks") - f0
        kern_s = (ix.stat("tc_us") - us0) * 1e-6 / reps
        rows = (ix.stat("tc_rows") - rows0) / reps
        med = float(np.median(ts))
        r = {"B": B, "batch_calls": reps, "batches": nb, "fallbacks": nf, "batch_ms": [round(t * 1e3, 3) for t in ts],
             "batch_qps": round(B / med, 1), "l1_kernel_ms_per_batch": round(kern_s * 1e3, 3), "l1_rows_per_batch": rows,
             "l1_pairs_per_s": float(rows * B * dim / kern_s) if kern_s > 0 else None}
        # per-query path in the same process
        old = eng.set_option("no_batch", 1)
        try:
            ix.scan_topk(po.L1, q[:2], k)
            s = min(sample, B)
            tq = timed(lambda: ix.scan_topk(po.L1, q[:s], k), 2)
            one = ix.scan_topk(po.L1, q[:3], k)
        finally:
            eng.set_option("no_batch", old)
        r["per_query_sample"] = s
        r["per_query_qps"] = round(s / min(tq), 1)
        r["speedup_vs_per_query"] = round(r["batch_qps"] / r["per_query_qps"], 2)
        # parity
        rowids = np.arange(1, n + 1, dtype=np.int64)
        ok = True
        for b in range(3):
            ok &= bool(np.array_equal(res[b][0], one[b][0]) and np.array_equal(res[b][1], one[b][1])) if vtype == po.I8 else True
            want_ids, want_d = oracle.scan_dense(po.L1, vtype, q[b], x, rowids, k)
            if vtype == po.I8:
                ok &= bool(np.array_equal(res[b][0], want_ids) and np.array_equal(res[b][1], want_d))
            else:
                try:
                    assert_fp_topk(res[b][0], res[b][1], want_ids, want_d, po.L1, lambda rr, b=b: oracle.distance(po.L1, vtype, q[b], x[rr - 1]))
                except AssertionError:
                    ok = False
        r["parity_oracle_3_queries"] = "bit-exact" if (ok and vtype == po.I8) else ("within fpcheck" if ok else "FAILED")
        # the kernel alone with each tile width, all rows, no hits
        n128 = (n // 128) * 128
        tiles = {}
        for N in ((32, 64, 128) if B > 32 else (32,)):
            ix.debug_tc_level(po.L1, q, np.zeros(B, np.float32), 0, n128, N=N, cap=16)
            tiles[str(N)] = round(min(timed(lambda: ix.debug_tc_level(po.L1, q, np.zeros(B, np.float32), 0, n128, N=N, cap=16), 3)) * 1e3, 3)
        r["kernel_alone_ms_by_N"] = tiles
        out[f"B{B}"] = r
        print(json.dumps({name: r}), file=sys.stderr, flush=True)
    ix.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--dim", type=int, default=384)
    ap.add_argument("--k", type=int, default=20)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--sample", type=int, default=64)
    ap.add_argument("--types", default="int8,f32")
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    eng = vs.load_engine()
    if eng.device_count() < 1:
        sys.exit("l1_batch_bench needs a CUDA device")
    doc = {"gpu": gpu_info(), "how": __doc__.split("\n\n")[0] + " (tools/l1_batch_bench.py)", "legs": []}
    oracle = po.Oracle()
    for t in a.types.split(","):
        doc["legs"].append(leg(eng, oracle, po.I8 if t == "int8" else po.F32, a.n, a.dim, a.k, (1024, 16), a.reps, a.sample))
    doc["gpu_after"] = gpu_info()
    s = json.dumps(doc, indent=1)
    print(s)
    if a.out:
        with open(a.out, "w") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()
