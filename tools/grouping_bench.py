"""Grouped top-k layouts on the H100: int8 10M x 384, L2, one query, the key sets of profiles/h100_grouped.json: 10 000 contiguous
keys of 1 000 rows ("docs1000", k 10, limit 10), 1 000 000 contiguous keys of 10 rows ("docs10", k 10, limit 100) and 1 000 keys of
1 000 random rows ("random1000", k 10, limit 10).  For each, the median over --reps of:
  * layout_ms: the device layout build (vsb_grouping_create, the "grouped_layout_us" it adds);
  * call_ms / call_layout_ms: a per-call vsb_scan_topk_grouped and the layout time inside it;
  * kept_ms: vsb_scan_topk_grouping on the kept layout;
  * parent_call_ms / parent_layout_ms: the same per-call grouped call of a library built from the parent commit (--parent, the
    host layout builder), alternating with the calls above on the same seeded column, keys and queries.
Every answer is compared with the parent's bit for bit.  Writes JSON to --out with the card's name, power limit and max SM clock
read in the same run.

    python tools/grouping_bench.py --parent <dir of the parent's libvsb200.so> [--rows 10000000] [--reps 5] [--out file]
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


def gpu_info():
    q = "name,power.limit,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 else "unknown"


def key_sets(n, rng):
    ar = np.arange(1, n + 1, dtype=np.int64)
    head = ar[:10_000_000]
    return {"docs1000": (np.array_split(head, 10_000), 10, 10), "docs10": (np.array_split(head, 1_000_000), 10, 100),
            "random1000": ([rng.choice(ar, 1000, replace=False) for _ in range(1000)], 10, 10)}


def parent_engine(api, path):
    """an Engine over the parent's library, which lacks the grouping symbols"""
    import ctypes
    eng = api.Engine.__new__(api.Engine)
    eng.path, eng.lib = path, ctypes.CDLL(path)
    for name, (res, args) in api._SIGNATURES.items():
        if hasattr(eng.lib, name):
            fn = getattr(eng.lib, name)
            fn.restype, fn.argtypes = res, args
    return eng


def same(a, b):
    if len(a) != len(b):
        return False
    for qa, qb in zip(a, b):
        if [g for g, _, _ in qa] != [g for g, _, _ in qb]:
            return False
        for (_, ia, da), (_, ib, db) in zip(qa, qb):
            if not (np.array_equal(ia, ib) and np.array_equal(da.view(np.uint64), db.view(np.uint64))):
                return False
    return True


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parent", required=True, help="directory holding the parent commit's libvsb200.so")
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--dim", type=int, default=384)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_grouping.json"))
    a = ap.parse_args()
    from sqlite_vector_b200 import api
    new_eng, old_eng = api.load_engine(), parent_engine(api, os.path.join(a.parent, "libvsb200.so"))
    rng = np.random.Generator(np.random.PCG64(11))
    n, dim = a.rows, a.dim
    ixs = {}
    for name, eng in (("new", new_eng), ("parent", old_eng)):
        ixs[name] = api.Index(api.I8, dim, n, engine=eng)
    chunk = 1 << 20
    for r0 in range(0, n, chunk):                               # the same seeded rows into both columns
        x = rng.integers(-128, 128, (min(chunk, n - r0), dim)).astype(np.int8)
        for ix in ixs.values():
            ix.append_dense(x)
    for ix in ixs.values():
        ix.finalize()
    q = rng.integers(-128, 128, dim).astype(np.int8)
    new, old = ixs["new"], ixs["parent"]
    out = {"gpu": gpu_info(), "rows": n, "dim": dim, "metric": "L2", "type": "int8", "reps": a.reps, "sets": {}}
    for sname, (keys, k, limit) in key_sets(n, rng).items():
        for ix in (new, old):                                   # warm-up: workspaces, distance buffers, rowid paths
            ix.scan_topk_grouped(api.L2, q, k, keys[:10], limit)
        rec = {"keys": len(keys), "pairs": int(sum(len(r) for r in keys)), "k": k, "limit": limit}
        t = {m: [] for m in ("layout_ms", "call_ms", "call_layout_ms", "kept_ms", "parent_call_ms", "parent_layout_ms")}
        equal = True
        g = None
        for _ in range(a.reps):
            l0 = old.stat("grouped_layout_us")
            t0 = time.perf_counter()
            want = old.scan_topk_grouped(api.L2, q, k, keys, limit)
            t["parent_call_ms"].append(1e3 * (time.perf_counter() - t0))
            t["parent_layout_ms"].append((old.stat("grouped_layout_us") - l0) / 1e3)
            l0 = new.stat("grouped_layout_us")
            t0 = time.perf_counter()
            got = new.scan_topk_grouped(api.L2, q, k, keys, limit)
            t["call_ms"].append(1e3 * (time.perf_counter() - t0))
            t["call_layout_ms"].append((new.stat("grouped_layout_us") - l0) / 1e3)
            if g is not None:
                g.close()
            l0 = new.stat("grouped_layout_us")
            g = new.grouping(keys)
            t["layout_ms"].append((new.stat("grouped_layout_us") - l0) / 1e3)
            t0 = time.perf_counter()
            kept = g.scan_topk(api.L2, q, k, limit)
            t["kept_ms"].append(1e3 * (time.perf_counter() - t0))
            equal = equal and same(got, want) and same(kept, want)
        g.close()
        rec.update({m: float(np.median(v)) for m, v in t.items()})
        rec["answers_equal_parent"] = bool(equal)
        out["sets"][sname] = rec
        print(sname, json.dumps(rec), flush=True)
    for ix in (new, old):
        ix.close()
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
