"""Large-k top-k on one H100 (DESIGN §3.11): int8 10M x 384, L2.  For each k, the median wall time of one vsb_scan_topk call
against the work the parent did for k > 256 (vsb_scan_all + vsb_replay_topk over every row) in the same process, the candidates
per query and the list regrows, the host replay and exchange-sort share; a 64-query batch at k = 1000; a streamed column in
1M-row windows at k = 1000.  Every timed answer is compared with the all-rows replay.  Writes profiles/h100_large_k.json (or --out).

    python tools/large_k_bench.py [--n 10000000] [--reps 5] [--out profiles/h100_large_k.json]
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


def _timed(fn, reps):
    ts, out = [], None
    for _ in range(reps):
        t0 = time.perf_counter()
        out = fn()
        ts.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(ts)), out


def _old(eng, ix, q, ids, k):
    d = ix.scan_all(api.L2, q)
    c = np.zeros(len(d), dtype=api.CAND_DTYPE)
    c["dist"], c["rowid"], c["seq"] = d, ids, np.arange(len(d))
    return eng.replay_topk(c, k)[:2]


def _same(a, b):
    return bool(np.array_equal(a[0], b[0]) and np.array_equal(np.asarray(a[1], np.float64).view(np.uint64), np.asarray(b[1], np.float64).view(np.uint64)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--dim", type=int, default=384)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--ks", default="20,257,1000,4096,16384")
    ap.add_argument("--window", type=int, default=1_000_000)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_large_k.json"))
    a = ap.parse_args()
    eng = vs.load_engine()
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    rec = {"gpu": smi.stdout.strip(), "backend": eng.backend_name(), "n": a.n, "dim": a.dim, "type": "int8", "metric": "L2", "k": {}}
    rng = np.random.Generator(np.random.PCG64(11))
    x = rng.integers(-128, 128, (a.n, a.dim), dtype=np.int8)
    qs = rng.integers(-128, 128, (64, a.dim), dtype=np.int8)
    ids = np.arange(1, a.n + 1, dtype=np.int64)
    ix = vs.Index(api.I8, a.dim, a.n)
    for s in range(0, a.n, 1 << 20):
        ix.append_dense(x[s:s + (1 << 20)])
    ix.finalize()
    ix.scan_topk(api.L2, qs[0], 20)
    for k in map(int, a.ks.split(",")):
        ix.scan_topk(api.L2, qs[1], k)                                   # warm-up: first-use buffers of this k
        c0, r0, q0 = ix.stat("large_k_cands"), ix.stat("large_k_regrows"), ix.stat("large_k_queries")
        ms, (res,) = _timed(lambda: ix.scan_topk(api.L2, qs[2], k), a.reps)
        e = {"topk_ms": ms, "cands_per_query": (ix.stat("large_k_cands") - c0) / max(1, ix.stat("large_k_queries") - q0),
             "regrows": ix.stat("large_k_regrows") - r0}
        old_ms, old = _timed(lambda: _old(eng, ix, qs[2], ids, k), 1 if k >= 4096 else 2)
        e["old_path_ms"], e["equal_to_old_path"] = old_ms, _same(res, old)
        if k > 256:
            (c,) = ix.scan_candidates(api.L2, qs[2], k, cap=max(1 << 16, 4 * int(e["cands_per_query"]) + 1024))
            e["replay_ms"], _ = _timed(lambda: eng.replay_topk(c, k), 3)
            # the exchange sort alone (+ k O(log k) fills): the k results, fed in reverse order
            rc = np.zeros(len(res[0]), dtype=api.CAND_DTYPE)
            rc["rowid"], rc["dist"] = res[0][::-1], res[1][::-1].astype(np.float32)
            e["exchange_sort_ms"], _ = _timed(lambda: eng.replay_topk(rc, k), 3)
            e["scan_all_ms"], _ = _timed(lambda: ix.scan_all(api.L2, qs[2]), 3)
        rec["k"][str(k)] = e
        print(k, json.dumps(e), flush=True)
    b_ms, got = _timed(lambda: ix.scan_topk(api.L2, qs, 1000), 1)
    rec["batch64_k1000"] = {"ms": b_ms, "per_query_ms": b_ms / 64,
                            "equal_to_old_path": all(_same(got[b], _old(eng, ix, qs[b], ids, 1000)) for b in (0, 31, 63))}
    print("batch", json.dumps(rec["batch64_k1000"]), flush=True)
    ix.close()
    st = vs.Index(api.I8, a.dim, a.n, window_rows=a.window)
    for s in range(0, a.n, 1 << 20):
        st.append_dense(x[s:s + (1 << 20)])
    st.finalize()
    st.scan_topk(api.L2, qs[3], 1000)
    r0 = st.stat("large_k_regrows")
    s_ms, (sres,) = _timed(lambda: st.scan_topk(api.L2, qs[4], 1000), 3)
    s20_ms, _ = _timed(lambda: st.scan_topk(api.L2, qs[4], 20), 3)
    rec["streamed_k1000"] = {"window_rows": a.window, "ms": s_ms, "k20_ms": s20_ms, "regrows": st.stat("large_k_regrows") - r0,
                             "equal_to_old_path": _same(sres, _old(eng, st, qs[4], ids, 1000))}
    print("streamed", json.dumps(rec["streamed_k1000"]), flush=True)
    st.close()
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(rec, f)
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
