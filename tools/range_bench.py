"""Range search on the H100: int8 10M x 384, L2 (the bench corpus).  Each query's radius is just above its 20th, 1 000th and
100 000th nearest distance (from that query's vsb_scan_all distances), so the k nearest rows (and their ties) qualify.  Measures:
  * one query: vsb_scan_range against vsb_scan_topk (k = 20) and against vsb_scan_all plus a host threshold and sort, which is
    what the stream module does for `WHERE distance < r ORDER BY distance` (ms per call, median);
  * a batch of B = 1024 range queries against the same B queries as single calls (the batch counters say which path ran);
  * SQL at 200k rows: vector_quantize_scan_range against vector_quantize_scan_stream(...) WHERE distance < r ORDER BY distance.
Every range result must equal the all-distances answer of its query.  Writes the JSON to --out (default profiles/h100_range.json)
with the card's name, power limit and max SM clock read in the same run.

    python tools/range_bench.py [--rows 10000000] [--dim 384] [--single 10] [--batch 1024] [--sql-rows 200000]
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
RANKS = (20, 1000, 100_000)
HBM_PEAK = 3.35e12   # H100 SXM5 80GB HBM3, bytes / s


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
    return 1e3 * float(np.median(ts))


def stream_answer(dist, ids, r):
    """vsb_scan_all distances -> the range answer, on the host (the stream module's WHERE distance < r ORDER BY distance)"""
    keep = np.nonzero(dist.astype(np.float64) < r)[0]
    sel = keep[np.argsort(dist[keep], kind="stable")]
    return ids[sel], dist[sel].astype(np.float64)


SQL_CHILD = r'''
import json, sqlite3, sys, time
import numpy as np
lib, n, dim, nq = sys.argv[1], int(sys.argv[2]), int(sys.argv[3]), int(sys.argv[4])
rng = np.random.Generator(np.random.PCG64(7))
x = rng.standard_normal((n, dim), dtype=np.float32)
q = rng.standard_normal((nq, dim), dtype=np.float32)
con = sqlite3.connect(":memory:", isolation_level=None)
con.enable_load_extension(True)
con.load_extension(lib)
con.execute("CREATE TABLE t (id INTEGER PRIMARY KEY, e BLOB)")
con.execute(f"SELECT vector_init('t', 'e', 'type=FLOAT32,dimension={dim},distance=L2')")
con.execute("BEGIN")
con.executemany("INSERT INTO t(id, e) VALUES (?, ?)", ((i + 1, x[i].tobytes()) for i in range(n)))
con.execute("COMMIT")
con.execute("SELECT vector_quantize('t', 'e', 'qtype=INT8')")
con.execute("SELECT vector_quantize_preload('t', 'e')")
out = {"rows": n, "legs": {}}
stream_sql = "SELECT id, distance FROM vector_quantize_scan_stream('t', 'e', ?) WHERE distance < ? AND id > 0 ORDER BY distance, id"
range_sql = "SELECT id, distance FROM vector_quantize_scan_range('t', 'e', ?, ?)"
con.execute(range_sql, (q[0].tobytes(), 1.0)).fetchall()
for rank in (20, 1000):
    ms_s, ms_r, sizes, same = [], [], [], True
    for b in range(nq):
        d = sorted(r[0] for r in con.execute("SELECT distance FROM vector_quantize_scan_stream('t', 'e', ?) WHERE id > 0", (q[b].tobytes(),)))
        r = float(np.nextafter(d[rank - 1], np.inf))
        t0 = time.perf_counter(); a = con.execute(stream_sql, (q[b].tobytes(), r)).fetchall(); ms_s.append((time.perf_counter() - t0) * 1e3)
        t0 = time.perf_counter(); c = con.execute(range_sql, (q[b].tobytes(), r)).fetchall(); ms_r.append((time.perf_counter() - t0) * 1e3)
        same &= (a == c)
        sizes.append(len(c))
    out["legs"][str(rank)] = {"stream_where_order_ms": float(np.median(ms_s)), "range_module_ms": float(np.median(ms_r)),
                              "rows_returned": [min(sizes), max(sizes)], "equal": bool(same)}
print("\n@@JSON@@" + json.dumps(out), flush=True)
'''


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--dim", type=int, default=384)
    ap.add_argument("--single", type=int, default=10, help="queries timed per single-query leg")
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--sql-rows", type=int, default=200_000)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_range.json"))
    a = ap.parse_args()
    import sqlite_vector_b200 as vs
    eng = vs.load_engine()
    if eng.device_count() < 1:
        raise SystemExit("range_bench needs a CUDA device")
    rng = np.random.Generator(np.random.PCG64(42))
    n, dim, B = a.rows, a.dim, a.batch
    x = np.frombuffer(rng.bytes(n * dim), dtype=np.int8).reshape(n, dim)
    q = np.frombuffer(rng.bytes(B * dim), dtype=np.int8).reshape(B, dim)
    ix = vs.Index(vs.api.I8, dim, n)
    for s in range(0, n, 1 << 20):
        ix.append_dense(x[s:s + (1 << 20)])
    ix.finalize()
    ids = np.arange(1, n + 1, dtype=np.int64)
    res = {"gpu": gpu_info(), "rows": n, "dim": dim, "batch": B, "metric": "L2", "type": "int8", "radius_ranks": list(RANKS),
           "how": "radius of a query = next double above its rank-th nearest distance (vsb_scan_all); medians over queries"}
    radii = np.zeros((len(RANKS), B))
    for b in range(B):
        d = np.partition(ix.scan_all(vs.api.L2, q[b]), [r - 1 for r in RANKS])
        for i, r in enumerate(RANKS):
            radii[i, b] = np.nextafter(float(d[r - 1]), np.inf)
    ix.scan_topk(vs.api.L2, q[0], 20)                                            # warm-up
    ix.scan_range(vs.api.L2, q[0], radii[0, 0])
    res["topk20_ms"] = timed(lambda: ix.scan_topk(vs.api.L2, q[1], 20), a.single)
    res["single"] = {}
    for i, rank in enumerate(RANKS):
        ms_range, ms_all, sizes, equal = [], [], [], True
        for b in range(a.single):
            ms_range.append(timed(lambda: ix.scan_range(vs.api.L2, q[b], radii[i, b]), 1))
            t0 = time.perf_counter()
            want = stream_answer(ix.scan_all(vs.api.L2, q[b]), ids, radii[i, b])
            ms_all.append((time.perf_counter() - t0) * 1e3)
            got = ix.scan_range(vs.api.L2, q[b], radii[i, b])[0]
            equal &= np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])
            sizes.append(len(got[0]))
        med = float(np.median(ms_range))
        res["single"][str(rank)] = {"range_ms": med, "scan_all_threshold_sort_ms": float(np.median(ms_all)), "rows_returned": [min(sizes), max(sizes)],
                                    "hbm_fraction": n * ix.query_pitch / (med * 1e-3) / HBM_PEAK, "equal": bool(equal)}
    res["batch"] = {}
    for i, rank in enumerate(RANKS[:2]):                                        # 100 000 rows overflow a batch bucket
        s0 = {k: ix.stat(k) for k in ("range_batches", "range_batch_fallbacks", "range_query_fallbacks")}
        t0 = time.perf_counter()
        got = ix.scan_range(vs.api.L2, q, radii[i])
        batch_ms = (time.perf_counter() - t0) * 1e3
        s1 = {k: ix.stat(k) - s0[k] for k in s0}
        t0 = time.perf_counter()
        singles = [ix.scan_range(vs.api.L2, q[b], radii[i, b])[0] for b in range(B)]
        singles_ms = (time.perf_counter() - t0) * 1e3
        equal = all(np.array_equal(got[b][0], singles[b][0]) and np.array_equal(got[b][1], singles[b][1]) for b in range(B))
        res["batch"][str(rank)] = {"batch_ms": batch_ms, "single_calls_ms": singles_ms, "speedup": singles_ms / batch_ms, "counters": s1,
                                   "rows_returned": [min(len(g[0]) for g in got), max(len(g[0]) for g in got)], "equal": bool(equal)}
    ix.close()
    if a.sql_rows > 0:
        p = subprocess.run([sys.executable, "-c", SQL_CHILD, os.path.join(ROOT, "sqlite_vector_b200", "lib", "vector"), str(a.sql_rows), str(dim), "5"],
                           capture_output=True, text=True, timeout=3000)
        line = [ln for ln in p.stdout.splitlines() if ln.startswith("@@JSON@@")]
        res["sql"] = json.loads(line[0][len("@@JSON@@"):]) if line else {"error": p.stderr[-2000:]}
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(res, f)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
