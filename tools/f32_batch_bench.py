"""Batched f32 queries on the tensor cores (TF32, option f32_batch) against the per-query path, on one GPU.

  python tools/f32_batch_bench.py [--n 10000000] [--dim 384] [--k 20] [--out profiles/h100_f32_batch.json]

For the north-star column, n x dim f32 N(0, 1) (seed 1234, generated in 1M-row chunks from one generator) with N(0, 1) queries
(seed 4321), L2, batches of 1024 and 16 host queries through vsb_scan_topk (host in, host out):
  * queries/s of the batch (median of --reps timed calls after one warm-up call);
  * queries/s of the per-query path (f32_batch = 0) on --sample queries, timed in the same process;
  * the scoring kernels' device time per batch (CUDA events of the levels, stat "tc_us") and the TF32 rate it implies
    (2 x rows scored x queries x dim / kernel time; the data sheet's 495 TFLOP/s dense TF32 is a reference, not a target);
  * candidates refined per query (stat "batch_cands" / queries) and the call's fallbacks;
  * parity: 3 queries against the oracle and --sample queries against the per-query path, both under tests/fpcheck.py.
Then a clustered column (--cn rows around 1000 centres, spread 0.1, queries drawn the same way) for the candidate count where
the TF32 slack admits the most.  The GPU's name, power limit and maximum SM clock are read in the same run.  Prints one JSON
document."""
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

CHUNK = 1 << 20


def gpu_info():
    q = "name,power.limit,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True, timeout=60)
    first = r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else ""
    return dict(zip(q.split(","), [v.strip() for v in first.split(",")])) if first else {"error": r.stderr.strip()[-200:]}


def normal(n, dim, seed):
    rng = np.random.Generator(np.random.PCG64(seed))
    out = np.empty((n, dim), dtype=np.float32)
    for a in range(0, n, CHUNK):
        out[a:a + CHUNK] = rng.standard_normal((min(CHUNK, n - a), dim), dtype=np.float32)
    return out


def clustered(n, dim, seed, c, spread=0.1):
    """n rows, each one of the centres c plus spread x N(0, 1)"""
    rng = np.random.Generator(np.random.PCG64(seed))
    out = np.empty((n, dim), dtype=np.float32)
    for a in range(0, n, CHUNK):
        m = min(CHUNK, n - a)
        out[a:a + m] = c[rng.integers(0, c.shape[0], m)] + np.float32(spread) * rng.standard_normal((m, dim), dtype=np.float32)
    return out


def index_of(x):
    ix = vs.Index(po.F32, x.shape[1], x.shape[0])
    for a in range(0, x.shape[0], CHUNK):
        ix.append_dense(x[a:a + CHUNK])
    ix.finalize()
    return ix


def timed(fn, reps):
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    return ts


def fp_ok(metric, got, want, dist_of_row):
    try:
        assert_fp_topk(got[0], got[1], want[0], want[1], metric, dist_of_row)
        return True
    except AssertionError:
        return False


def batch_leg(eng, oracle, ix, x, q, metric, k, reps, sample, parity):
    B, dim = q.shape
    eng.set_option("f32_batch", 1)
    ix.scan_topk(metric, q, k)                                                # warm-up: row norms, tensor maps, modules
    st0 = {s: ix.stat(s) for s in ("batches", "fallbacks", "tc_us", "tc_rows", "batch_cands")}
    res = None

    def run():
        nonlocal res
        res = ix.scan_topk(metric, q, k)
    ts = timed(run, reps)
    d = {s: ix.stat(s) - v for s, v in st0.items()}
    kern_s = d["tc_us"] * 1e-6 / reps
    rows = d["tc_rows"] / reps
    med = float(np.median(ts))
    r = {"B": B, "batch_calls": reps, "batches": d["batches"], "fallbacks": d["fallbacks"], "batch_ms": [round(t * 1e3, 3) for t in ts],
         "batch_qps": round(B / med, 1), "tc_kernel_ms_per_batch": round(kern_s * 1e3, 3), "tc_rows_per_batch": rows,
         "tf32_tflops": round(2.0 * rows * B * dim / kern_s / 1e12, 1) if kern_s > 0 else None,
         "tf32_datasheet_tflops_reference": 495, "candidates_refined_per_query": round(d["batch_cands"] / (reps * B), 1)}
    eng.set_option("f32_batch", 0)                                            # the per-query path, same process
    try:
        ix.scan_topk(metric, q[:2], k)
        s = min(sample, B)
        tq = timed(lambda: ix.scan_topk(metric, q[:s], k), 2)
        one = ix.scan_topk(metric, q[:s], k)
    finally:
        eng.set_option("f32_batch", 1)
    r["per_query_sample"] = s
    r["per_query_qps"] = round(s / min(tq), 1)
    r["speedup_vs_per_query"] = round(r["batch_qps"] / r["per_query_qps"], 2)

    def dist(b):
        return lambda rr: oracle.distance(metric, po.F32, q[b], x[rr - 1])
    r[f"parity_per_query_{s}_queries"] = "within fpcheck" if all(fp_ok(metric, res[b], one[b], dist(b)) for b in range(s)) else "FAILED"
    if parity:
        rowids = np.arange(1, x.shape[0] + 1, dtype=np.int64)
        ok = all(fp_ok(metric, res[b], oracle.scan_dense(metric, po.F32, q[b], x, rowids, k), dist(b)) for b in range(3))
        r["parity_oracle_3_queries"] = "within fpcheck" if ok else "FAILED"
    print(json.dumps(r), file=sys.stderr, flush=True)
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--cn", type=int, default=1_000_000)
    ap.add_argument("--dim", type=int, default=384)
    ap.add_argument("--k", type=int, default=20)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--sample", type=int, default=64)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    eng = vs.load_engine()
    if eng.device_count() < 1:
        sys.exit("f32_batch_bench needs a CUDA device")
    old = eng.set_option("f32_batch", 1)
    doc = {"gpu": gpu_info(), "how": __doc__.split("\n\n")[1].strip() + " (tools/f32_batch_bench.py)", "legs": []}
    oracle = po.Oracle()
    try:
        x = normal(a.n, a.dim, 1234)
        qall = normal(1024, a.dim, 4321)
        ix = index_of(x)
        leg = {"column": "normal", "n": a.n, "dim": a.dim, "k": a.k, "metric": "L2"}
        for B in (1024, 16):
            leg[f"B{B}"] = batch_leg(eng, oracle, ix, x, np.ascontiguousarray(qall[:B]), po.L2, a.k, a.reps, a.sample, True)
        doc["legs"].append(leg)
        ix.close()
        del x
        centres = normal(1000, a.dim, 99)
        xc = clustered(a.cn, a.dim, 1234, centres)
        qc = clustered(1024, a.dim, 4321, centres)        # the same centres: every query has a cluster of near rows
        ixc = index_of(xc)
        leg = {"column": "clustered, 1000 centres, spread 0.1", "n": a.cn, "dim": a.dim, "k": a.k}
        for metric in (po.L2, po.COS, po.DOT):
            leg[po.METRIC_NAMES[metric] + "_B1024"] = batch_leg(eng, oracle, ixc, xc, qc, metric, a.k, a.reps, a.sample, True)
        doc["legs"].append(leg)
        ixc.close()
    finally:
        eng.set_option("f32_batch", old)
    doc["gpu_after"] = gpu_info()
    s = json.dumps(doc, indent=1)
    print(s)
    if a.out:
        with open(a.out, "w") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()
