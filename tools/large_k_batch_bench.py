"""Batched top-k for k > 256 on one H100 (DESIGN §3.12).  Workloads: int8 10M x 384, L2, at B = 16 and 1024 queries and
k = 257 / 1000 / 4096; bf16 10M x 768, dot, at B = 1024, k = 1000.  For each batch, after a warm-up call of the same batch: the
wall time of one vsb_scan_topk call, its split into the batch levels (host clock around the levels, sort and candidate copy,
which end in a synchronise) and the threaded host replay, the replay's threads, the candidates per query and the fallbacks; then
the same queries as single calls (the path the batch took before), with every batch answer compared with its single call bit
for bit.  Reads the card's name, power limit and
maximum SM clock in the same run.  Writes profiles/h100_large_k_batch.json (or --out).

    python tools/large_k_batch_bench.py [--n 10000000] [--out profiles/h100_large_k_batch.json]
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
import sqlite_vector_b200 as vs  # noqa: E402
from sqlite_vector_b200 import api  # noqa: E402

STATS = ("large_k_batches", "large_k_batch_fallbacks", "large_k_query_fallbacks", "large_k_queries", "large_k_cands",
         "large_k_levels_us", "large_k_replay_us")


def _same(a, b):
    return bool(np.array_equal(a[0], b[0]) and np.array_equal(np.asarray(a[1], np.float64).view(np.uint64), np.asarray(b[1], np.float64).view(np.uint64)))


def _build(vtype, n, dim, make):
    ix = vs.Index(vtype, dim, n)
    step = 1 << 18
    for s in range(0, n, step):
        ix.append_dense(make(min(step, n - s)))
    ix.finalize()
    return ix


def _run(ix, metric, qs, k):
    ix.scan_topk(metric, qs, k)                                          # warm-up: first-use buffers of this batch and k
    s0 = {s: ix.stat(s) for s in STATS}
    t0 = time.perf_counter()
    got = ix.scan_topk(metric, qs, k)
    wall = (time.perf_counter() - t0) * 1e3
    d = {s: ix.stat(s) - s0[s] for s in STATS}
    t0 = time.perf_counter()
    singles = [ix.scan_topk(metric, qs[b], k)[0] for b in range(len(qs))]
    single_ms = (time.perf_counter() - t0) * 1e3
    return {"B": len(qs), "k": k, "batch_ms": wall, "batch_ms_per_query": wall / len(qs), "single_calls_ms": single_ms,
            "single_ms_per_query": single_ms / len(qs), "speedup": single_ms / wall,
            "levels_ms": d["large_k_levels_us"] / 1e3, "replay_ms": d["large_k_replay_us"] / 1e3, "replay_threads": ix.stat("large_k_replay_threads"),
            "cands_per_query": d["large_k_cands"] / max(1, d["large_k_queries"]), "batches": d["large_k_batches"],
            "batch_fallbacks": d["large_k_batch_fallbacks"], "query_fallbacks": d["large_k_query_fallbacks"],
            "equal_to_single_calls": all(_same(got[b], singles[b]) for b in range(len(qs)))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_large_k_batch.json"))
    a = ap.parse_args()
    eng = vs.load_engine()
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    rec = {"gpu": smi.stdout.strip(), "backend": eng.backend_name(), "n": a.n, "runs": [],
           "note": "wall time of one call after a warm-up call of the same batch; levels_ms and replay_ms from the index counters"}
    rng = np.random.Generator(np.random.PCG64(21))
    ix = _build(api.I8, a.n, 384, lambda m: rng.integers(-128, 128, (m, 384), dtype=np.int8))
    qs = rng.integers(-128, 128, (1024, 384), dtype=np.int8)
    for B in (16, 1024):
        for k in (257, 1000, 4096):
            r = dict(_run(ix, api.L2, qs[:B], k), type="int8", dim=384, metric="L2")
            rec["runs"].append(r)
            print(json.dumps(r), flush=True)
    ix.close()
    # bf16 from small integers (exact in bf16): the high half of the float32 bits
    bf16 = lambda m: (rng.integers(-64, 64, (m, 768)).astype(np.float32).view(np.uint32) >> 16).astype(np.uint16)
    ix = _build(api.BF16, a.n, 768, bf16)
    r = dict(_run(ix, api.DOT, bf16(1024), 1000), type="bf16", dim=768, metric="DOT")
    rec["runs"].append(r)
    print(json.dumps(r), flush=True)
    ix.close()
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(rec, f)
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
