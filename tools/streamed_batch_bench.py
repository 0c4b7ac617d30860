"""Batched queries on a streamed column: one pass of the windows per batch, against the per-query streamed loop, the resident
batch path and the host link.

  python tools/streamed_batch_bench.py [--n 10000000] [--dim 384] [--window 1000000] [--out profiles/h100_streamed_batch.json]

The column is forced to stream (vsb_index_create_streamed with --window rows per window) although it would fit the device: a
column larger than the H100's 80 GB needs that much pinned host memory, so the forced window size stands in for it.
int8 leg, n x dim, k = 20, batches of 1024 and 16 host queries through vsb_scan_topk:
  * streamed batch: queries/s (median of --reps timed calls after one warm-up call), host-to-device GB/s of the window copies
    (stat stream_bytes / stream_us, device time from the first copy to the last level), scoring-kernel time (stat tc_us);
  * the per-query streamed loop (option no_batch) on 2 queries, the resident batch path on the same rows and queries;
  * a pinned host-to-device copy of one column's bytes (torch, CUDA events): the roofline of the streamed batch;
  * overlap: streamed batch time against copy time + resident batch time;
  * parity: streamed equal to resident on every query (rowids and distances), int8 bit-exact against the oracle on 3 queries.
bf16 DOT leg (dim 768, --bf16-n rows): the first batch, which adds the pass for the largest row norm, next to later batches.
The GPU's name, power limit and maximum SM clock are read in the same run.  Prints one JSON document."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import sqlite_vector_b200 as vs  # noqa: E402
from oracle import pyoracle as po  # noqa: E402
from tools.l1_batch_bench import gpu_info, timed  # noqa: E402

CHUNK = 1 << 20


def column(vtype, n, dim, seed):
    """seeded column from random bytes, in row chunks: int8 as drawn, bf16 from int8 / 16"""
    rng = np.random.Generator(np.random.PCG64(seed))
    out = np.empty((n, dim), dtype=np.int8 if vtype == po.I8 else np.uint16)
    for a in range(0, n, CHUNK):
        m = min(CHUNK, n - a)
        r = np.frombuffer(rng.bytes(m * dim), dtype=np.int8).reshape(m, dim)
        out[a:a + m] = r if vtype == po.I8 else po.convert(r.astype(np.float32) / 16, po.BF16)
    return out


def index(vtype, x, window):
    ix = vs.Index(vtype, x.shape[1], x.shape[0], window_rows=window)
    for a in range(0, x.shape[0], CHUNK):
        ix.append_dense(x[a:a + CHUNK])
    ix.finalize()
    return ix


def pinned_h2d_gbs(nbytes, reps=3):
    import torch
    h = torch.empty(nbytes, dtype=torch.uint8, pin_memory=True)
    d = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    d.copy_(h, non_blocking=True)
    torch.cuda.synchronize()
    best = None
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        d.copy_(h, non_blocking=True)
        e1.record()
        e1.synchronize()
        s = e0.elapsed_time(e1) * 1e-3
        best = s if best is None else min(best, s)
    del h, d
    torch.cuda.empty_cache()
    return nbytes / best / 1e9


def batch_leg(ix, q, metric, k, reps):
    """warm-up call, then reps timed calls; the counters' deltas over the timed calls"""
    ix.scan_topk(metric, q, k, as_arrays=True)
    names = ("batches", "fallbacks", "tc_us", "tc_rows", "stream_bytes", "stream_us")
    s0 = {s: ix.stat(s) for s in names}
    out = None

    def run():
        nonlocal out
        out = ix.scan_topk(metric, q, k, as_arrays=True)
    ts = timed(run, reps)
    d = {s: ix.stat(s) - s0[s] for s in names}
    med = float(np.median(ts))
    r = {"batch_ms": [round(t * 1e3, 2) for t in ts], "qps": round(q.shape[0] / med, 1), "batches": d["batches"], "fallbacks": d["fallbacks"],
         "scoring_kernel_ms_per_batch": round(d["tc_us"] * 1e-3 / reps, 3), "scored_rows_per_batch": d["tc_rows"] / reps}
    if d["stream_us"] > 0:
        r["stream_bytes_per_batch"] = d["stream_bytes"] / reps
        r["h2d_GBps"] = round(d["stream_bytes"] / (d["stream_us"] * 1e-6) / 1e9, 2)
    return r, med, out


def same(a, b):
    return bool(np.array_equal(a[0], b[0]) and np.array_equal(a[1].view(np.uint64), b[1].view(np.uint64)) and np.array_equal(a[2], b[2]))


def int8_leg(eng, oracle, n, dim, k, window, reps, link_gbs):
    x = column(po.I8, n, dim, 21)
    qall = column(po.I8, 1024, dim, 22)
    st = index(po.I8, x, window)
    res = index(po.I8, x, 0)
    pitch = st.query_pitch
    copy_s = n * pitch / (link_gbs * 1e9)
    out = {"type": "int8", "metric": "L2", "n": n, "dim": dim, "k": k, "window_rows": window, "column_GB": round(n * pitch / 1e9, 3),
           "windows": -(-n // window), "column_copy_ms_at_pinned_rate": round(copy_s * 1e3, 2)}
    for B in (1024, 16):
        q = np.ascontiguousarray(qall[:B])
        rs, t_st, o_st = batch_leg(st, q, po.L2, k, reps)
        rr, t_res, o_res = batch_leg(res, q, po.L2, k, reps)
        r = {"B": B, "streamed_batch": rs, "resident_batch": rr,
             "overlap": {"streamed_batch_ms": round(t_st * 1e3, 2), "copy_plus_resident_batch_ms": round((copy_s + t_res) * 1e3, 2),
                         "copy_ms": round(copy_s * 1e3, 2), "streamed_over_copy": round(t_st / copy_s, 3)}}
        old = eng.set_option("no_batch", 1)
        try:
            st.scan_topk(po.L2, q[:1], k)
            tq = timed(lambda: st.scan_topk(po.L2, q[:2], k), 2)
        finally:
            eng.set_option("no_batch", old)
        r["per_query_streamed"] = {"queries": 2, "qps": round(2 / min(tq), 3)}
        r["speedup_vs_per_query_streamed"] = round(rs["qps"] / r["per_query_streamed"]["qps"], 1)
        ok = True
        rowids = np.arange(1, n + 1, dtype=np.int64)
        for b in range(3):
            want_ids, want_d = oracle.scan_dense(po.L2, po.I8, q[b], x, rowids, k)
            c = o_st[2][b]
            ok &= bool(np.array_equal(o_st[0][b, :c], want_ids) and np.array_equal(o_st[1][b, :c], want_d))
        r["parity"] = {"streamed_equals_resident_all_queries": same(o_st, o_res), "int8_oracle_3_queries": "bit-exact" if ok else "FAILED"}
        out[f"B{B}"] = r
        print(json.dumps({"int8": r}), file=sys.stderr, flush=True)
    st.close()
    res.close()
    return out


def bf16_leg(n, dim, k, window, reps):
    x = column(po.BF16, n, dim, 31)
    q = np.ascontiguousarray(column(po.BF16, 1024, dim, 32))
    st = index(po.BF16, x, window)
    res = index(po.BF16, x, 0)
    out = {"type": "bf16", "metric": "DOT", "n": n, "dim": dim, "k": k, "B": 1024, "window_rows": window,
           "column_GB": round(n * st.query_pitch / 1e9, 3)}
    b0, s0 = st.stat("stream_bytes"), st.stat("stream_us")
    t0 = time.perf_counter()
    first = st.scan_topk(po.DOT, q, k, as_arrays=True)
    t1 = time.perf_counter()
    out["first_batch"] = {"ms": round((t1 - t0) * 1e3, 2), "stream_bytes": st.stat("stream_bytes") - b0,
                          "h2d_GBps": round((st.stat("stream_bytes") - b0) / ((st.stat("stream_us") - s0) * 1e-6) / 1e9, 2)}
    rs, _, o_st = batch_leg(st, q, po.DOT, k, reps)
    out["later_batches"] = rs
    res.scan_topk(po.DOT, q, k)
    rr, _, o_res = batch_leg(res, q, po.DOT, k, reps)
    out["resident_batch"] = rr
    out["parity_streamed_equals_resident_all_queries"] = same(o_st, o_res) and same(first, o_res)
    print(json.dumps({"bf16": out}), file=sys.stderr, flush=True)
    st.close()
    res.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--dim", type=int, default=384)
    ap.add_argument("--k", type=int, default=20)
    ap.add_argument("--window", type=int, default=1_000_000)
    ap.add_argument("--bf16-n", type=int, default=2_000_000)
    ap.add_argument("--bf16-window", type=int, default=250_000)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    eng = vs.load_engine()
    if eng.device_count() < 1:
        sys.exit("streamed_batch_bench needs a CUDA device")
    doc = {"gpu": gpu_info(), "how": __doc__.split("\n\n")[0] + " (tools/streamed_batch_bench.py)"}
    link = pinned_h2d_gbs(1 << 30)
    doc["pinned_h2d_GBps_1GiB"] = round(link, 2)
    doc["int8"] = int8_leg(eng, po.Oracle(), a.n, a.dim, a.k, a.window, a.reps, link)
    doc["bf16_dot"] = bf16_leg(a.bf16_n, 768, a.k, a.bf16_window, a.reps)
    doc["gpu_after"] = gpu_info()
    s = json.dumps(doc, indent=1)
    print(s)
    if a.out:
        with open(a.out, "w") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()
