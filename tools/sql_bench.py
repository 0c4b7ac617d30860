"""End-to-end latency THROUGH SQL: the same statements against our extension (sqlite_vector_b200/lib/vector.so, needs a
H100) and against the unmodified reference (oracle/_ref/avx2/vector.so, CPU), each in its own process (SQLite loads
extensions RTLD_GLOBAL and the reference exports every symbol).

  python tools/sql_bench.py --n 200000 --dim 384 --queries 50 [--which ours|ref|both]

Prints one JSON line per extension: first-use seconds (a 64-row table: process-wide one-time costs), build / quantize / preload seconds, ms per vector_quantize_scan and vector_full_scan
query (k = 20), and a checksum of the returned ids so that the two runs can be compared (quantized scans: identical ids;
distances are in quantized space for both)."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

CHILD = r'''
import json, sqlite3, sys, time
import numpy as np
lib, n, dim, nq, k = sys.argv[1], int(sys.argv[2]), int(sys.argv[3]), int(sys.argv[4]), int(sys.argv[5])
con = sqlite3.connect(":memory:", isolation_level=None)
con.enable_load_extension(True)
con.load_extension(lib)
out = {"lib": lib, "backend": con.execute("SELECT vector_backend()").fetchone()[0], "n": n, "dim": dim, "k": k}
rng = np.random.Generator(np.random.PCG64(1234))
# first use of the extension on a 64-row table, timed on its own: for our extension this is where the process pays for the CUDA
# context, the kernel images, streams and the first pinned buffers (once per process, not per statement)
t0 = time.perf_counter()
con.execute("CREATE TABLE w (id INTEGER PRIMARY KEY, e BLOB)")
xw = rng.standard_normal((64, dim), dtype=np.float32)
con.executemany("INSERT INTO w(id, e) VALUES (?, ?)", [(i + 1, xw[i].tobytes()) for i in range(64)])
con.execute(f"SELECT vector_init('w', 'e', 'type=FLOAT32,dimension={dim}')")
con.execute("SELECT vector_quantize('w', 'e')").fetchall()
con.execute("SELECT vector_quantize_preload('w', 'e')").fetchall()
con.execute("SELECT id FROM vector_quantize_scan('w', 'e', ?, 5)", (xw[0].tobytes(),)).fetchall()
out["first_use_s"] = time.perf_counter() - t0
t0 = time.perf_counter()
con.execute("CREATE TABLE t (id INTEGER PRIMARY KEY, e BLOB)")
con.execute("BEGIN")
B = 20000
for a in range(0, n, B):
    x = rng.standard_normal((min(B, n - a), dim), dtype=np.float32)
    con.executemany("INSERT INTO t(id, e) VALUES (?, ?)", [(a + i + 1, x[i].tobytes()) for i in range(x.shape[0])])
con.execute("COMMIT")
out["insert_s"] = time.perf_counter() - t0
con.execute(f"SELECT vector_init('t', 'e', 'type=FLOAT32,dimension={dim}')")
t0 = time.perf_counter(); con.execute("SELECT vector_quantize('t', 'e')").fetchall(); out["quantize_s"] = time.perf_counter() - t0
t0 = time.perf_counter(); con.execute("SELECT vector_quantize_preload('t', 'e')").fetchall(); out["preload_s"] = time.perf_counter() - t0
qs = np.random.Generator(np.random.PCG64(4321)).standard_normal((nq, dim), dtype=np.float32)
def timed(sql):
    con.execute(sql, (qs[0].tobytes(), k)).fetchall()          # warm-up (our extension stages the raw column on first use)
    ids, t0 = [], time.perf_counter()
    for b in range(nq):
        rows = con.execute(sql, (qs[b].tobytes(), k)).fetchall()
        ids.append([r[0] for r in rows])
    return (time.perf_counter() - t0) / nq * 1e3, ids
out["quantize_scan_ms"], idq = timed("SELECT id, distance FROM vector_quantize_scan('t', 'e', ?, ?)")
out["full_scan_ms"], idf = timed("SELECT id, distance FROM vector_full_scan('t', 'e', ?, ?)")
out["quantize_scan_ids_crc"] = int(np.bitwise_xor.reduce(np.asarray(idq, dtype=np.int64).reshape(-1) * 2654435761 % (1 << 61)))
out["full_scan_top1"] = [r[0] for r in idf[:5]]
print("@@JSON@@" + json.dumps(out), flush=True)
'''


def run(lib, a):
    p = subprocess.run([sys.executable, "-c", CHILD, lib, str(a.n), str(a.dim), str(a.queries), str(a.k)], capture_output=True, text=True)
    for ln in p.stdout.splitlines():
        if ln.startswith("@@JSON@@"):
            return json.loads(ln[8:])
    return {"lib": lib, "error": (p.stderr or p.stdout)[-400:]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=200_000)
    ap.add_argument("--dim", type=int, default=384)
    ap.add_argument("--queries", type=int, default=50)
    ap.add_argument("--k", type=int, default=20)
    ap.add_argument("--which", default="both", choices=["ours", "ref", "both"])
    a = ap.parse_args()
    libs = []
    if a.which in ("ours", "both"):
        libs.append(os.path.join(ROOT, "sqlite_vector_b200", "lib", "vector"))
    if a.which in ("ref", "both"):
        libs.append(os.path.join(ROOT, "oracle", "_ref", "avx2", "vector"))
    for lib in libs:
        print(json.dumps(run(lib, a)))


if __name__ == "__main__":
    main()
