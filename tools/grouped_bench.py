"""Grouped top-k on the H100: int8 10M x 384, L2.  Key sets: 10 000 contiguous keys of 1 000 rows ("docs1000"), 1 000 000
contiguous keys of 10 rows ("docs10") and 1 000 keys of 1 000 random rows ("random1000"); k = 1 / 3 / 10; limit 10 / 100 / all.
Per call (median of the timed calls): the wall time and its split from the index counters into layout (host mapping, sort and
upload), scan (device events around the all-distances scan), walk (device events around walk, bounds and compaction, with the
copies of the key minimums and survivors) and replay (host).  Compared in the same run against:
  * vsb_scan_all + host grouping in numpy (every distance copied to the host, sorted by key and distance);
  * one vsb_scan_topk_filtered call per key where that is at most 1 000 calls;
  * SQL at 200k rows: vector_full_scan_grouped against the window-function statement over vector_full_scan_stream.
Sampled keys of every grouped answer are checked against filtered calls bit for bit.  Writes the JSON to --out (default
profiles/h100_grouped.json) with the card's name, power limit and max SM clock read in the same run.

    python tools/grouped_bench.py [--rows 10000000] [--dim 384] [--reps 5]
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

COUNTERS = ("grouped_layout_us", "grouped_scan_us", "grouped_walk_us", "grouped_replay_us", "grouped_cands", "grouped_keys_replayed")


def gpu_info():
    q = "name,power.limit,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 else "unknown"


def host_grouping(dist, flat, key_of, nkeys, k, limit):
    """the grouped answer from every distance on the host: per key the k smallest (distance, row), keys by their first"""
    d = dist[flat - 1]
    o = np.lexsort((flat, d, key_of))
    ks, ds = key_of[o], d[o]
    first = np.r_[0, np.flatnonzero(np.diff(ks)) + 1]
    rank = np.arange(len(ks)) - np.repeat(first, np.diff(np.r_[first, len(ks)]))
    keep = o[rank < k]
    mins = ds[first]
    order = np.argsort(mins, kind="stable")
    return ks[first][order][: limit or None], keep


SQL_CHILD = r'''
import json, sqlite3, sys, time
import numpy as np
lib, n, dim, k, reps = sys.argv[1], int(sys.argv[2]), int(sys.argv[3]), int(sys.argv[4]), int(sys.argv[5])
rng = np.random.Generator(np.random.PCG64(7))
x = rng.integers(-128, 128, (n, dim)).astype(np.int8)
q = rng.integers(-128, 128, dim).astype(np.int8).tobytes()
con = sqlite3.connect(":memory:", isolation_level=None)
con.enable_load_extension(True)
con.load_extension(lib)
con.execute("CREATE TABLE t (id INTEGER PRIMARY KEY, e BLOB, doc INTEGER)")
con.execute(f"SELECT vector_init('t', 'e', 'type=INT8,dimension={dim},distance=L2')")
con.execute("BEGIN")
con.executemany("INSERT INTO t(id, e, doc) VALUES (?, ?, ?)", ((i + 1, x[i].tobytes(), i // 100) for i in range(n)))
con.execute("COMMIT")
con.execute("CREATE INDEX t_doc ON t(doc)")
grouped = "SELECT key, id, distance FROM vector_full_scan_grouped('t', 'e', ?, ?, (SELECT vector_rowid_sets(doc, id) FROM t), NULL)"
window = ("SELECT doc, id, distance FROM (SELECT t.doc, s.id, s.distance, row_number() OVER (PARTITION BY t.doc ORDER BY s.distance, s.id) AS rn "
          "FROM vector_full_scan_stream('t', 'e', ?) AS s JOIN t ON t.id = s.id) WHERE rn <= ?")
out = {}
for name, sql, args in (("grouped", grouped, (q, k)), ("window", window, (q, k))):
    con.execute(sql, args).fetchall()
    ts, rows = [], None
    for _ in range(reps):
        t0 = time.perf_counter()
        rows = con.execute(sql, args).fetchall()
        ts.append((time.perf_counter() - t0) * 1e3)
    out[name] = {"ms": sorted(ts)[len(ts) // 2], "rows": len(rows)}
    out[name + "_set"] = sorted((r[0], r[1]) for r in rows)
out["same_rows"] = out.pop("grouped_set") == out.pop("window_set")
print("\n@@JSON@@" + json.dumps(out), flush=True)
'''


def grouped_call(vs, ix, q, k, flat, offsets, nkeys, limit, decode=False):
    """one vsb_scan_topk_grouped call on CSR keys (no per-key Python objects); the keys returned, and with decode the answer as
    Index.scan_topk_grouped returns it for one query"""
    api, lib = vs.api, ix.eng.lib
    res = api._vp()
    ix.eng.check(lib.vsb_scan_topk_grouped(ix.h, api.L2, api._ptr(q), 1, k, api._ptr(flat), api._ptr(offsets), nkeys, limit,
                                           api.C.byref(res)))
    try:
        nk, keys, offs, ids, dist = api._i(), api._vp(), api._vp(), api._vp(), api._vp()
        ix.eng.check(lib.vsb_grouped_get(res, 0, api.C.byref(nk), api.C.byref(keys), api.C.byref(offs), api.C.byref(ids), api.C.byref(dist)))
        if not decode or nk.value == 0:
            return nk.value, []
        m = nk.value
        o = np.ctypeslib.as_array(api.C.cast(offs, api.C.POINTER(api.C.c_int64)), (m + 1,))
        kk = np.ctypeslib.as_array(api.C.cast(keys, api.C.POINTER(api.C.c_int32)), (m,))
        rid = np.ctypeslib.as_array(api.C.cast(ids, api.C.POINTER(api.C.c_int64)), (int(o[-1]),))
        dd = np.ctypeslib.as_array(api.C.cast(dist, api.C.POINTER(api.C.c_double)), (int(o[-1]),))
        return m, [(int(kk[i]), rid[o[i]:o[i + 1]].copy(), dd[o[i]:o[i + 1]].copy()) for i in range(m)]
    finally:
        lib.vsb_grouped_free(res)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--dim", type=int, default=384)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--sql-rows", type=int, default=200_000)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_grouped.json"))
    a = ap.parse_args()
    import sqlite_vector_b200 as vs
    eng = vs.load_engine()
    if eng.device_count() < 1:
        raise SystemExit("grouped_bench needs a CUDA device")
    rng = np.random.Generator(np.random.PCG64(42))
    n, dim = a.rows, a.dim
    x = np.frombuffer(rng.bytes(n * dim), dtype=np.int8).reshape(n, dim)
    q = np.frombuffer(rng.bytes(dim), dtype=np.int8)
    ix = vs.Index(vs.api.I8, dim, n)
    for s in range(0, n, 1 << 20):
        ix.append_dense(x[s:s + (1 << 20)])
    ix.finalize()
    ar = np.arange(1, n + 1, dtype=np.int64)
    perm = rng.permutation(n)[: (n // 1000) * 1000] + 1
    sets = {"docs1000": ar[: (n // 1000) * 1000].reshape(-1, 1000),
            "docs10": ar[: (n // 10) * 10].reshape(-1, 10),
            "random1000": np.sort(perm[:1000 * 1000].reshape(1000, 1000), axis=1)}
    res = {"gpu": gpu_info(), "rows": n, "dim": dim, "metric": "L2", "type": "int8", "sets": {}}
    ix.scan_topk(vs.api.L2, q, 10)
    t_all = []
    for _ in range(a.reps):
        t0 = time.perf_counter()
        ix.scan_all(vs.api.L2, q)
        t_all.append(time.perf_counter() - t0)
    res["scan_all_ms"] = 1e3 * float(np.median(t_all))
    for name, keys in sets.items():
        nkeys = keys.shape[0]
        flat = np.ascontiguousarray(keys.reshape(-1), dtype=np.int64)
        offsets = np.arange(nkeys + 1, dtype=np.int64) * keys.shape[1]
        key_of = np.repeat(np.arange(nkeys), keys.shape[1])
        out = {"keys": nkeys, "rows_per_key": int(keys.shape[1]), "calls": {}}
        for k in (1, 3, 10):
            # host grouping of every distance (scan_all + numpy), one call per k
            t0 = time.perf_counter()
            d_all = ix.scan_all(vs.api.L2, q)
            host_order, _ = host_grouping(d_all, flat, key_of, nkeys, k, 0)
            host_ms = 1e3 * (time.perf_counter() - t0)
            for limit in (10, 100, 0):
                grouped_call(vs, ix, q, k, flat, offsets, nkeys, limit)              # warm-up (and the pair list's size)
                c0 = {c: ix.stat(c) for c in COUNTERS}
                ts = []
                for _ in range(a.reps):
                    t0 = time.perf_counter()
                    nret, _ = grouped_call(vs, ix, q, k, flat, offsets, nkeys, limit)
                    ts.append(time.perf_counter() - t0)
                per = {c.replace("grouped_", ""): (ix.stat(c) - c0[c]) / a.reps for c in COUNTERS}
                for c in ("layout_us", "scan_us", "walk_us", "replay_us"):
                    per[c.replace("_us", "_ms")] = per.pop(c) / 1e3
                # sampled keys against filtered calls, bit for bit; the returned keys against the host grouping's
                _, got = grouped_call(vs, ix, q, k, flat, offsets, nkeys, limit, decode=True)
                same = True
                for i in sorted(set([0, len(got) // 2, len(got) - 1])):
                    g, gi, gd = got[i]
                    bits, _ = ix.rowid_bitmap(keys[g])
                    (wi, wd), = ix.scan_topk_filtered(vs.api.L2, q, k, bits)
                    same &= bool(np.array_equal(gi, wi) and np.array_equal(gd.view(np.uint64), wd.view(np.uint64)))
                host_keys = host_order[: limit or None]
                out["calls"][f"k{k}_limit{limit or 'all'}"] = dict(
                    ms=1e3 * float(np.median(ts)), keys_returned=nret, host_grouping_ms=host_ms,
                    host_keys_agree=bool(len(host_keys) == nret and np.array_equal(host_keys, [g for g, _, _ in got])),
                    sampled_keys_equal_filtered=same, **per)
                print(name, k, limit, json.dumps(out["calls"][f"k{k}_limit{limit or 'all'}"]), flush=True)
        out["layout_pairs"] = ix.stat("grouped_pairs")
        if nkeys <= 1000:                                                             # one filtered call per key
            k = 10
            t0 = time.perf_counter()
            for g in range(nkeys):
                bits, _ = ix.rowid_bitmap(keys[g])
                ix.scan_topk_filtered(vs.api.L2, q, k, bits)          # bitmap built and uploaded per key, as a caller would
            out["filtered_per_key_ms_k10_all"] = 1e3 * (time.perf_counter() - t0)
        res["sets"][name] = out
    ix.close()
    lib = os.path.join(ROOT, "sqlite_vector_b200", "lib", "vector")
    p = subprocess.run([sys.executable, "-c", SQL_CHILD, lib, str(a.sql_rows), str(dim), "3", str(a.reps)], capture_output=True, text=True, timeout=3600)
    res["sql"] = {"rows": a.sql_rows, "rows_per_doc": 100, "k": 3}
    for ln in p.stdout.splitlines():
        if ln.startswith("@@JSON@@"):
            res["sql"].update(json.loads(ln[len("@@JSON@@"):]))
    if p.returncode != 0:
        res["sql"]["error"] = p.stderr[-2000:]
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps({k: v for k, v in res.items() if k != "sets"}))


if __name__ == "__main__":
    main()
