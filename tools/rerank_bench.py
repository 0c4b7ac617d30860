"""Reranking quantized candidates on the raw column (vsb_scan_topk_rows, DESIGN §3.13) on one H100.

Workload: the bench corpus (f32 10M x 384 from bench.py's seeded blocks, and its S8 int8 copy), L2, k = 20, candidates c in
{20, 100, 400, 2000}.  For each c:
  - single queries (--queries of them, after five warm-up queries): the quantized stage (vsb_scan_topk on the int8 column, c rows),
    the rows stage (vsb_scan_topk_rows on the f32 column) and their total, against vsb_scan_topk on the f32 column (the exact
    answer) and against the composed filtered call (vsb_scan_topk_filtered with the bitmap of the candidates' rowids);
  - a batch of 1024 queries: the same stages as one call each, against vsb_scan_topk of the batch on the f32 column (per-query
    loop: f32 L2 batches only with the f32_batch option) and the composed filtered call once per query;
  - the same with the f32 column streamed from pinned host memory (--stream-window rows per window): rows stage alone, and a few
    queries of the full-scan and filtered baselines, each of which is a pass of the column over PCIe;
  - recall@20 of the rerank against the exact f32 top-20, per c;
  - that the rerank equals the composed filtered call bit for bit (every single query, the batch's sampled queries).
Then through SQL at --sql-n rows: vector_quantize_scan_rerank against the composed statement.  Reads the card's name, power
limit and clocks in the same run.  Writes profiles/h100_rerank.json (or --out).

    python tools/rerank_bench.py [--n 10000000] [--queries 50] [--out profiles/h100_rerank.json]
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
import bench  # noqa: E402  (the corpus generator of the flagship workload)
import sqlite_vector_b200 as vs  # noqa: E402
from sqlite_vector_b200 import api  # noqa: E402

K, CANDS, BATCH = 20, (20, 100, 400, 2000), 1024


def _smi():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return r.stdout.strip()


def _same(a, b):
    return bool(np.array_equal(a[0], b[0]) and np.array_equal(np.asarray(a[1], np.float64).view(np.uint64),
                                                              np.asarray(b[1], np.float64).view(np.uint64)))


def _ms(fn, reps=1):
    t0 = time.perf_counter()
    for _ in range(reps):
        out = fn()
    return (time.perf_counter() - t0) * 1e3 / reps, out


def _mem_available_gb():
    with open("/proc/meminfo") as f:
        for ln in f:
            if ln.startswith("MemAvailable:"):
                return int(ln.split()[1]) / 2**20
    return 0.0


def _build(torch, n, dim, scale, window):
    """(f32 resident index, int8 index, f32 streamed index or None): blocks generated on the GPU, appended from device memory"""
    f32 = vs.Index(api.F32, dim, n)
    i8 = vs.Index(api.I8, dim, n)
    st = vs.Index(api.F32, dim, n, window_rows=window) if window > 0 else None
    for b, a0, rows in bench.corpus_blocks(n, 0, n):
        x = bench.gen_block_f32(torch, b, rows, dim, "cuda")
        x8 = bench.quantize_s8(torch, x, scale).contiguous()
        torch.cuda.synchronize()                 # the engine copies on its own streams, which do not wait for torch's
        f32.append_device(x.data_ptr(), rows)
        i8.append_device(x8.data_ptr(), rows)
        if st is not None:
            st.append_dense(x.cpu().numpy())
    for ix in (f32, i8, st):
        if ix is not None:
            ix.finalize()
    return f32, i8, st


def _recall(got, exact):
    return float(np.mean([len(set(g[0].tolist()) & set(e[0].tolist())) / max(1, len(e[0])) for g, e in zip(got, exact)]))


def single_queries(f32, i8, qf, q8, nq, c, label, baselines=True, base_queries=None):
    """per-query means of the stages; the rerank's answers"""
    for b in range(5):                                                              # warm-up: first-use buffers, clocks
        cand = i8.scan_topk(api.L2, q8[b], c)
        f32.scan_topk_rows(api.L2, qf[b], K, [cand[0][0]])
    tq = tr = 0.0
    res, equal = [], True
    for b in range(nq):
        dq, cd = _ms(lambda: i8.scan_topk(api.L2, q8[b], c))
        dr, rr = _ms(lambda: f32.scan_topk_rows(api.L2, qf[b], K, [cd[0][0]]))
        tq, tr = tq + dq, tr + dr
        res.append(rr[0])
    out = {"what": label, "c": c, "queries": nq, "quantized_ms": tq / nq, "rows_ms": tr / nq, "total_ms": (tq + tr) / nq}
    if baselines:
        m = nq if base_queries is None else base_queries
        tf = tc = 0.0
        for b in range(m):
            df, _ = _ms(lambda: f32.scan_topk(api.L2, qf[b], K))
            cd = i8.scan_topk(api.L2, q8[b], c)
            dc, want = _ms(lambda: f32.scan_topk_filtered(api.L2, qf[b], K, f32.rowid_bitmap(cd[0][0])[0]))
            tf, tc = tf + df, tc + dc
            equal = equal and _same(res[b], want[0])
        out.update({"f32_full_scan_ms": tf / m, "composed_filtered_ms": tc / m + out["quantized_ms"], "baseline_queries": m,
                    "rerank_equals_composed": equal})
    return out, res


def batch_queries(f32, i8, qf, q8, c, label, baselines=True):
    i8.scan_topk(api.L2, q8, c)                                                     # warm-up of this batch shape
    dq, cands = _ms(lambda: i8.scan_topk(api.L2, q8, c))
    lists = [cd[0] for cd in cands]
    f32.scan_topk_rows(api.L2, qf, K, lists)
    dr, res = _ms(lambda: f32.scan_topk_rows(api.L2, qf, K, lists))
    out = {"what": label, "c": c, "B": len(qf), "quantized_ms": dq, "rows_ms": dr, "total_ms": dq + dr}
    if baselines:
        df, _ = _ms(lambda: f32.scan_topk(api.L2, qf, K))
        t0 = time.perf_counter()
        equal = True
        for b in range(len(qf)):
            want = f32.scan_topk_filtered(api.L2, qf[b], K, f32.rowid_bitmap(lists[b])[0])
            if b % 64 == 0:
                equal = equal and _same(res[b], want[0])
        dc = (time.perf_counter() - t0) * 1e3
        out.update({"f32_batch_scan_ms": df, "composed_filtered_ms": dc + dq, "rerank_equals_composed_sampled": equal})
    return out, res


SQL_CHILD = r'''
import json, sqlite3, sys, time
import numpy as np
lib, n, dim, nq, k = sys.argv[1], int(sys.argv[2]), int(sys.argv[3]), int(sys.argv[4]), int(sys.argv[5])
con = sqlite3.connect(":memory:", isolation_level=None)
con.enable_load_extension(True)
con.load_extension(lib)
rng = np.random.Generator(np.random.PCG64(1234))
con.execute("CREATE TABLE t (id INTEGER PRIMARY KEY, e BLOB)")
con.execute("BEGIN")
for a in range(0, n, 20000):
    x = rng.standard_normal((min(20000, n - a), dim), dtype=np.float32)
    con.executemany("INSERT INTO t(id, e) VALUES (?, ?)", [(a + i + 1, x[i].tobytes()) for i in range(x.shape[0])])
con.execute("COMMIT")
con.execute(f"SELECT vector_init('t', 'e', 'type=FLOAT32,dimension={dim}')")
con.execute("SELECT vector_quantize('t', 'e')").fetchall()
con.execute("SELECT vector_quantize_preload('t', 'e')").fetchall()
qs = np.random.Generator(np.random.PCG64(4321)).standard_normal((nq, dim), dtype=np.float32)
new = "SELECT id, distance FROM vector_quantize_scan_rerank('t', 'e', ?, ?, ?)"
old = ("SELECT id, distance FROM vector_full_scan_filtered('t', 'e', ?, ?, "
       "(SELECT vector_rowid_set(id) FROM vector_quantize_scan('t', 'e', ?, ?)))")
out = {"n": n, "dim": dim, "k": k, "queries": nq, "runs": []}
for c in (20, 100, 400, 2000):
    def timed(sql, args):
        con.execute(sql, args(0)).fetchall()                              # warm-up (stages the raw column on first use)
        rows, t0 = [], time.perf_counter()
        for b in range(nq):
            rows.append(con.execute(sql, args(b)).fetchall())
        return (time.perf_counter() - t0) / nq * 1e3, rows
    ms_new, r_new = timed(new, lambda b: (qs[b].tobytes(), k, c))
    ms_old, r_old = timed(old, lambda b: (qs[b].tobytes(), k, qs[b].tobytes(), c))
    out["runs"].append({"c": c, "rerank_ms": ms_new, "composed_ms": ms_old, "equal": r_new == r_old})
print("@@JSON@@" + json.dumps(out), flush=True)
'''


def sql_bench(n, nq):
    lib = os.path.join(ROOT, "sqlite_vector_b200", "lib", "vector")
    p = subprocess.run([sys.executable, "-c", SQL_CHILD, lib, str(n), "384", str(nq), str(K)], capture_output=True, text=True)
    for ln in p.stdout.splitlines():
        if ln.startswith("@@JSON@@"):
            return json.loads(ln[8:])
    return {"error": (p.stderr or p.stdout)[-600:]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--dim", type=int, default=384)
    ap.add_argument("--queries", type=int, default=50)
    ap.add_argument("--stream-window", type=int, default=1 << 20, help="rows per window of the streamed f32 column; 0: skip")
    ap.add_argument("--stream-baseline-queries", type=int, default=3)
    ap.add_argument("--sql-n", type=int, default=200_000)
    ap.add_argument("--sql-queries", type=int, default=50)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_rerank.json"))
    a = ap.parse_args()
    import torch
    eng = vs.load_engine()
    rec = {"gpu_before": _smi(), "backend": eng.backend_name(), "n": a.n, "dim": a.dim, "k": K, "metric": "L2",
           "note": "host wall clock around each synchronous call, per-query means; composed = the quantized stage + "
                   "vsb_scan_topk_filtered with the bitmap of the candidates (bitmap built on the host inside the timing)",
           "single": [], "batch": [], "streamed_single": [], "streamed_batch": [], "recall_at_20": {}}
    amax = bench.corpus_absmax(torch, a.n, a.dim, 0, a.n, "cuda")
    scale = float(np.float32(127.0) / np.float32(amax))
    window = a.stream_window
    if window > 0 and _mem_available_gb() < 1.5 * a.n * a.dim * 4 / 2**30:      # the pinned arena plus room for the rest
        rec["streamed_note"] = f"not measured: {_mem_available_gb():.0f} GB of host memory available"
        window = 0
    t0 = time.perf_counter()
    f32, i8, st = _build(torch, a.n, a.dim, scale, window)
    rec["build_s"] = time.perf_counter() - t0
    g = torch.Generator(device="cuda").manual_seed(bench.SEED_QUERY)
    qf_t = torch.randn((BATCH, a.dim), generator=g, device="cuda", dtype=torch.float32)
    qf = qf_t.cpu().numpy()
    q8 = bench.quantize_s8(torch, qf_t, scale).cpu().numpy()
    nq = min(a.queries, BATCH)
    exact = [f32.scan_topk(api.L2, qf[b], K)[0] for b in range(nq)]
    for c in CANDS:
        r, res = single_queries(f32, i8, qf, q8, nq, c, "resident f32, single queries")
        rec["recall_at_20"][str(c)] = _recall(res, exact)
        r["recall_at_20"] = rec["recall_at_20"][str(c)]
        rec["single"].append(r)
        print(json.dumps(r), flush=True)
    for c in CANDS:
        r, _ = batch_queries(f32, i8, qf, q8, c, "resident f32, batch", baselines=(c == 100))
        rec["batch"].append(r)
        print(json.dumps(r), flush=True)
    if st is not None:
        rec["stream_window"] = a.stream_window
        rec["host_mem_available_gb"] = _mem_available_gb()
        for c in CANDS:
            r, _ = single_queries(st, i8, qf, q8, nq, c, "streamed f32, single queries", baselines=(c == 100),
                                  base_queries=a.stream_baseline_queries)
            r["rows_host_bytes_total"] = st.stat("rows_host_bytes")
            rec["streamed_single"].append(r)
            print(json.dumps(r), flush=True)
            r, _ = batch_queries(st, i8, qf, q8, c, "streamed f32, batch", baselines=False)
            rec["streamed_batch"].append(r)
            print(json.dumps(r), flush=True)
        st.close()
    for ix in (f32, i8):
        ix.close()
    rec["sql"] = sql_bench(a.sql_n, a.sql_queries)
    print(json.dumps(rec["sql"]), flush=True)
    rec["gpu_after"] = _smi()
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(rec, f)
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
