"""Grouped top-k in passes of several queries on the H100: int8 10M x 384, L2, k 10, on kept groupings of the key sets of
tools/grouping_bench.py (10 000 x 1 000 rows with limit 10, 1 000 000 x 10 rows with limit 100, 1 000 x 1 000 random rows with
limit 10), nq = 1, 8 and 64.  For each, the median over --reps of one call of nq queries (batch_ms) against nq single-query calls
(singles_ms) in the same process, alternating, with the scan, walk and replay times the counters report for each.  Then the same
column streamed in 1M-row windows at nq = 8, and through SQL at 200 000 rows and 2 000 keys, k 3: 64 queries in one
vector_full_scan_grouped_batch statement against 64 vector_full_scan_grouped statements.  Every answer is compared bit for bit.
Writes JSON to --out with the card's name, power limit and max SM clock read in the same run.

    python tools/grouped_batch_bench.py [--rows 10000000] [--reps 3] [--out file]
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
sys.path.insert(0, os.path.join(ROOT, "tools"))
from grouping_bench import gpu_info, key_sets, same  # noqa: E402

COUNTERS = ("grouped_scan_us", "grouped_walk_us", "grouped_replay_us", "grouped_passes")

SQL_CHILD = r'''
import json, sqlite3, sys, time
import numpy as np
lib, n, nkeys, reps = sys.argv[1], int(sys.argv[2]), int(sys.argv[3]), int(sys.argv[4])
rng = np.random.Generator(np.random.PCG64(5))
dim, B, k = 64, 64, 3
x = rng.standard_normal((n, dim), dtype=np.float32)
q = rng.standard_normal((B, dim), dtype=np.float32)
con = sqlite3.connect(":memory:", isolation_level=None)
con.enable_load_extension(True)
con.load_extension(lib)
con.execute("CREATE TABLE t (id INTEGER PRIMARY KEY, e BLOB, doc INTEGER)")
con.execute("SELECT vector_init('t','e','type=FLOAT32,dimension=64,distance=L2')")
con.executemany("INSERT INTO t VALUES (?, ?, ?)", ((i + 1, x[i].tobytes(), int(i % nkeys)) for i in range(n)))
groups = con.execute("SELECT vector_rowid_sets(doc, id) FROM t").fetchone()[0]
single = "SELECT key, id, distance FROM vector_full_scan_grouped('t','e',?,3,?,10)"
batch = "SELECT query, key, id, distance FROM vector_full_scan_grouped_batch('t','e',?,3,?,10)"
con.execute(single, (q[0].tobytes(), groups)).fetchall()          # warm: staged column, kept grouping
con.execute(batch, (q.tobytes(), groups)).fetchall()
tb, ts, equal = [], [], True
for _ in range(reps):
    t0 = time.perf_counter()
    got = con.execute(batch, (q.tobytes(), groups)).fetchall()
    tb.append(1e3 * (time.perf_counter() - t0))
    t0 = time.perf_counter()
    want = [(b,) + r for b in range(B) for r in con.execute(single, (q[b].tobytes(), groups)).fetchall()]
    ts.append(1e3 * (time.perf_counter() - t0))
    equal = equal and got == want
print("@@" + json.dumps({"rows": n, "keys": nkeys, "dim": dim, "type": "float32", "k": k, "limit": 10, "queries": B,
                         "batch_statement_ms": float(np.median(tb)), "single_statements_ms": float(np.median(ts)),
                         "answers_equal": bool(equal)}))
'''


def timed(ix, fn):
    c0 = {c: ix.stat(c) for c in COUNTERS}
    t0 = time.perf_counter()
    r = fn()
    ms = 1e3 * (time.perf_counter() - t0)
    return r, ms, {c: ix.stat(c) - c0[c] for c in COUNTERS}


def compare(ix, g, api, qs, k, limit, reps):
    """median times of one call of len(qs) queries and of len(qs) single calls, alternating; and whether they agree"""
    tb, ts, cb, cs, equal = [], [], [], [], True
    for _ in range(reps):
        got, ms, c = timed(ix, lambda: g.scan_topk(api.L2, qs, k, limit))
        tb.append(ms)
        cb.append(c)
        want, ms, c = timed(ix, lambda: [g.scan_topk(api.L2, q, k, limit)[0] for q in qs])
        ts.append(ms)
        cs.append(c)
        equal = equal and same(got, want)
    med = lambda cc, name: float(np.median([c[name] for c in cc])) / 1e3
    return {"batch_ms": float(np.median(tb)), "singles_ms": float(np.median(ts)),
            "batch_scan_ms": med(cb, "grouped_scan_us"), "singles_scan_ms": med(cs, "grouped_scan_us"),
            "batch_walk_ms": med(cb, "grouped_walk_us"), "singles_walk_ms": med(cs, "grouped_walk_us"),
            "batch_replay_ms": med(cb, "grouped_replay_us"), "singles_replay_ms": med(cs, "grouped_replay_us"),
            "batch_passes": int(np.median([c["grouped_passes"] for c in cb])), "answers_equal": bool(equal)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--dim", type=int, default=384)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--sql-rows", type=int, default=200_000)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_grouped_batch.json"))
    a = ap.parse_args()
    from sqlite_vector_b200 import api
    rng = np.random.Generator(np.random.PCG64(11))
    n, dim = a.rows, a.dim
    ix = api.Index(api.I8, dim, n)
    st = api.Index(api.I8, dim, n, window_rows=1 << 20)
    chunk = 1 << 20
    for r0 in range(0, n, chunk):
        x = rng.integers(-128, 128, (min(chunk, n - r0), dim)).astype(np.int8)
        ix.append_dense(x)
        st.append_dense(x)
    ix.finalize()
    st.finalize()
    qs = rng.integers(-128, 128, (64, dim)).astype(np.int8)
    out = {"gpu": gpu_info(), "rows": n, "dim": dim, "metric": "L2", "type": "int8", "k": 10, "reps": a.reps, "sets": {}}
    for sname, (keys, k, limit) in key_sets(n, rng).items():
        rec = {"keys": len(keys), "limit": limit}
        with ix.grouping(keys) as g:
            g.scan_topk(api.L2, qs[:8], k, limit)                # warm: the pass buffers
            for nq in (1, 8, 64):
                rec[f"nq{nq}"] = compare(ix, g, api, qs[:nq], k, limit, a.reps)
                print(sname, nq, json.dumps(rec[f"nq{nq}"]), flush=True)
        if sname == "docs1000":
            with st.grouping(keys) as g:
                g.scan_topk(api.L2, qs[:8], k, limit)
                s0 = st.stat("stream_bytes")
                r = compare(st, g, api, qs[:8], k, limit, a.reps)
                r["stream_gb_per_rep"] = (st.stat("stream_bytes") - s0) / a.reps / 1e9
                want = ix.scan_topk_grouped(api.L2, qs[:8], k, keys, limit)
                r["equal_resident"] = same(g.scan_topk(api.L2, qs[:8], k, limit), want)
                out["streamed_nq8"] = r
                print("streamed", json.dumps(r), flush=True)
        out["sets"][sname] = rec
    ix.close()
    st.close()
    p = subprocess.run([sys.executable, "-c", SQL_CHILD, os.path.join(ROOT, "sqlite_vector_b200", "lib", "vector"), str(a.sql_rows), "2000",
                        str(a.reps)], capture_output=True, text=True)
    line = [ln for ln in p.stdout.splitlines() if ln.startswith("@@")]
    out["sql"] = json.loads(line[0][2:]) if line else {"error": p.stderr[-2000:]}
    print("sql", json.dumps(out["sql"]), flush=True)
    out["gpu_after"] = gpu_info()
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
