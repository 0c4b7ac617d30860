"""Run SQL statements against an extension library in a SEPARATE process (one library per process:
SQLite dlopens extensions RTLD_GLOBAL and the reference exports every symbol, SURVEY trap 2)."""
import json
import os
import subprocess
import sys

CHILD = r'''
import json, sqlite3, sys
lib, stmts = sys.argv[1], json.loads(sys.stdin.read())
con = sqlite3.connect(":memory:", isolation_level=None)
con.enable_load_extension(True)
con.load_extension(lib)
out = []
def enc(v):
    if isinstance(v, bytes): return {"hex": v.hex()}
    if isinstance(v, float):
        if v != v: return {"f": "nan"}
        if v in (float("inf"), float("-inf")): return {"f": str(v)}
    return v
for s in stmts:
    try:
        if isinstance(s, list):
            sql, params = s[0], [bytes.fromhex(p["hex"]) if isinstance(p, dict) else p for p in s[1]]
        else:
            sql, params = s, []
        rows = con.execute(sql, params).fetchall()
        out.append({"rows": [[enc(v) for v in r] for r in rows]})
    except Exception as e:
        out.append({"error": str(e)})
try:
    import ctypes
    h = ctypes.CDLL(lib + ".so")                       # the same mapping SQLite loaded: its launch counter
    h.vsb_kernel_launches.restype = ctypes.c_int64
    out.append({"kernel_launches": int(h.vsb_kernel_launches())})
except (OSError, AttributeError):
    out.append({"kernel_launches": None})              # the reference build has no such symbol
print("\n@@JSON@@" + json.dumps(out), flush=True)
'''


def run_sql(lib_path: str, statements, timeout=600, env=None, want_launches=False):
    """lib_path without the .so suffix is fine (sqlite appends it).  REF_CPU is served from tests/golden/ref_sql.json.gz where
    oracle/_ref is not built (tests/refreplay.py).  Returns a list of {"rows": ...} | {"error": ...}
    (plus, with want_launches, the library's kernel launch count after the script as a last element)."""
    if os.path.abspath(lib_path) == REF_CPU:      # the reference extension: live where oracle/_ref is built, else recorded
        from tests import refreplay
        key = refreplay._key("sql", json.dumps(statements, sort_keys=True), json.dumps(env, sort_keys=True))
        live = (lambda: _run_sql(lib_path, statements, timeout, env)) if os.path.exists(REF_CPU + ".so") else None
        r = refreplay.recorded("sql", key, live)
    else:
        r = _run_sql(lib_path, statements, timeout, env)
    return r if want_launches else r[:-1]


def _run_sql(lib_path, statements, timeout, env):
    p = subprocess.run([sys.executable, "-c", CHILD, lib_path], input=json.dumps(statements), capture_output=True, text=True, timeout=timeout,
                       env=None if env is None else dict(os.environ, **env))
    if p.returncode != 0:
        raise RuntimeError(f"sql child failed: {p.stderr[-2000:]}")
    for ln in p.stdout.splitlines():          # the reference printf()s diagnostics to stdout; find our marker
        if ln.startswith("@@JSON@@"):
            return json.loads(ln[len("@@JSON@@"):])
    raise RuntimeError("no result line from sql child: " + p.stdout[-500:])


ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OURS = os.path.join(ROOT, "sqlite_vector_b200", "lib", "vector")
REF_CPU = os.path.join(ROOT, "oracle", "_ref", "cpu", "vector")


def blob(a):
    return {"hex": a.tobytes().hex()}


# BASELINE config 1 through SQL: the child builds the table itself (100k x 384 f32 would be 300 MB of hex over a pipe)
C1_CHILD = r'''
import json, sqlite3, sys, time
import numpy as np
lib, n, dim, k, nq, metric = sys.argv[1], int(sys.argv[2]), int(sys.argv[3]), int(sys.argv[4]), int(sys.argv[5]), sys.argv[6]
x = np.random.Generator(np.random.PCG64(1234)).standard_normal((n, dim), dtype=np.float32)
q = np.random.Generator(np.random.PCG64(4321)).standard_normal((nq, dim), dtype=np.float32)
con = sqlite3.connect(":memory:", isolation_level=None)
con.enable_load_extension(True)
con.load_extension(lib)
con.execute("CREATE TABLE c1 (id INTEGER PRIMARY KEY, e BLOB)")
con.execute(f"SELECT vector_init('c1', 'e', 'type=FLOAT32,dimension={dim},distance={metric}')")
con.execute("BEGIN")
con.executemany("INSERT INTO c1(id, e) VALUES (?, ?)", ((3 * i + 1, x[i].tobytes()) for i in range(n)))
con.execute("COMMIT")
out = {"full": [], "quant": [], "ms_full": [], "ms_quant": []}
for b in range(nq):
    t0 = time.perf_counter()
    rows = con.execute("SELECT id, distance FROM vector_full_scan('c1', 'e', ?, ?)", (q[b].tobytes(), k)).fetchall()
    out["ms_full"].append((time.perf_counter() - t0) * 1e3)
    out["full"].append(rows)
out["quantized_rows"] = con.execute("SELECT vector_quantize('c1', 'e')").fetchall()[0][0]
con.execute("SELECT vector_quantize_preload('c1', 'e')")
for b in range(nq):
    t0 = time.perf_counter()
    rows = con.execute("SELECT id, distance FROM vector_quantize_scan('c1', 'e', ?, ?)", (q[b].tobytes(), k)).fetchall()
    out["ms_quant"].append((time.perf_counter() - t0) * 1e3)
    out["quant"].append(rows)
print("\n@@JSON@@" + json.dumps(out), flush=True)
'''


def run_c1(lib_path: str, n=100_000, dim=384, k=20, nq=3, metric="L2", timeout=900):
    """vector_full_scan / vector_quantize_scan top-k of `nq` seeded queries over a seeded n x dim f32 table, through SQL"""
    p = subprocess.run([sys.executable, "-c", C1_CHILD, lib_path, str(n), str(dim), str(k), str(nq), metric], capture_output=True, text=True, timeout=timeout)
    if p.returncode != 0:
        raise RuntimeError(f"c1 child failed: {p.stderr[-2000:]}")
    for ln in p.stdout.splitlines():
        if ln.startswith("@@JSON@@"):
            return json.loads(ln[len("@@JSON@@"):])
    raise RuntimeError("no result line from c1 child: " + p.stdout[-500:])
