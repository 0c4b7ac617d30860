"""Run one fixed corpus of table-valued-function calls against two builds of the extension and diff the outputs statement by
statement.  Each build runs in its own process (tests/sqlrun.py), one after the other; valid calls need a CUDA device.

  python tools/sql_modules_diff.py --a build/parent/vector --b sqlite_vector_b200/lib/vector [--out DIR]

The corpus, for each of the 20 modules: valid calls at k (range: radius) = 0, 1, 20 and 300 plus the variants a module has (JSON
queries, explicit query_sets, a limit, fewer candidates than k); one call per single fault (argument count, each argument's type,
BLOB size and range, unknown table, NULL / short / JSON queries, a column that cannot be staged or was never quantized); and the
two-fault calls that pair a negative k, a negative limit or candidates out of range with a fault checked after the arguments.
Only those two-fault calls may differ between builds whose argument checks run in a different order; every other difference
is reported as unexpected and makes the exit code 1."""
import argparse
import json
import os
import struct
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tests.sqlrun import run_sql  # noqa: E402

DIM, ROWS = 8, 3000


def _hex(b: bytes) -> str:
    return "x'" + b.hex() + "'"


def setup():
    rng = np.random.Generator(np.random.PCG64(2026))
    x = rng.standard_normal((ROWS, DIM), dtype=np.float32)
    s = ["CREATE TABLE t (id INTEGER PRIMARY KEY, e BLOB)", "CREATE TABLE u (id INTEGER PRIMARY KEY, e BLOB)",
         "CREATE TABLE bad (id INTEGER PRIMARY KEY, e BLOB)"]
    for a in range(0, ROWS, 500):
        vals = ", ".join(f"({3 * i + 1}, {_hex(x[i].tobytes())})" for i in range(a, min(a + 500, ROWS)))
        s += [f"INSERT INTO t(id, e) VALUES {vals}", f"INSERT INTO u(id, e) VALUES {vals}"]
    s += [f"INSERT INTO bad(id, e) VALUES (1, {_hex(x[0].tobytes())}), (2, x'01')"]
    s += [f"SELECT vector_init('{t}', 'e', 'type=FLOAT32,dimension={DIM}')" for t in ("t", "u", "bad")]
    s += ["SELECT vector_quantize('t', 'e')", "SELECT vector_quantize_preload('t', 'e')"]
    q = rng.standard_normal((3, DIM), dtype=np.float32)
    return s, q


def modules():
    """(name, argument kinds in position order)"""
    for kind in ("full", "quantize"):
        b = f"vector_{kind}_scan"
        yield b, ["T", "C", "Q1", "K"]
        yield b + "_stream", ["T", "C", "Q1"]
        yield b + "_batch", ["T", "C", "Q3", "K"]
        yield b + "_filtered", ["T", "C", "Q1", "K", "ROWIDS"]
        yield b + "_batch_filtered", ["T", "C", "Q3", "K", "ROWIDS"]
        yield b + "_batch_sets", ["T", "C", "Q3", "K", "SETS", "QSETS"]
        yield b + "_grouped", ["T", "C", "Q1", "K", "GROUPS", "LIMIT"]
        yield b + "_range", ["T", "C", "Q1", "RADIUS"]
        yield b + "_range_filtered", ["T", "C", "Q1", "RADIUS", "ROWIDS"]
    yield "vector_quantize_scan_rerank", ["T", "C", "Q1", "K", "CAND"]
    yield "vector_quantize_scan_rerank_batch", ["T", "C", "Q3", "K", "CAND"]


def corpus(q):
    good = {"T": "'t'", "C": "'e'", "Q1": _hex(q[0].tobytes()), "Q3": _hex(q.tobytes()), "K": "20", "RADIUS": "20",
            "ROWIDS": "(SELECT vector_rowid_set(id) FROM t WHERE id % 3 = 1 AND id < 4000)",
            "SETS": "(SELECT vector_rowid_sets(id % 4, id) FROM t)", "QSETS": "NULL",
            "GROUPS": "(SELECT vector_rowid_sets(id % 50, id) FROM t)", "LIMIT": "NULL", "CAND": "50"}
    variants = {"Q1": ["'" + json.dumps([float(v) for v in q[1]]) + "'"], "Q3": ["'" + json.dumps([float(v) for v in q.ravel()]) + "'"],
                "QSETS": [_hex(struct.pack("<3q", 2, 0, 7))], "LIMIT": ["5", "0"], "CAND": ["5", "0"], "T": ["'u'"]}
    faults = {"T": ["1", "'nope'", "'bad'", "'u'"], "C": ["NULL", "'zz'"],
              "Q1": ["1.5", "NULL", "x''", "x'0102'", "'[1,2]'", "'[1,'"], "Q3": ["1.5", "x''", "x'0102'", "'[1,2,3]'"],
              "K": ["'k'", "2.5", "NULL", "-1", "4294967295"], "RADIUS": ["'r'", "NULL", "x'00'"],
              "ROWIDS": ["NULL", "'1,2'", "12", "x'010203'"], "SETS": ["NULL", "x'0100000000000000'"],
              "QSETS": ["'0'", "x'0300'", _hex(struct.pack("<q", 0))], "GROUPS": ["NULL", "x'0100000000000000'"],
              "LIMIT": ["'2'", "2.5", "-1"], "CAND": ["'many'", "2.5", "-1", "2147483648"]}
    later = {"T": ["'nope'", "'bad'", "'u'"], "Q1": ["x'0102'", "NULL"], "Q3": ["x'0102'"], "QSETS": [_hex(struct.pack("<q", 0))]}
    early = {"K": ["-1"], "LIMIT": ["-1"], "CAND": ["-1", "2147483648"]}
    out = []                                                         # (statement, tag)

    def call(name, args, tag, select="*"):
        out.append((f"SELECT {select} FROM {name}({', '.join(args)})", tag))

    for name, kinds in modules():
        base = [good[k] for k in kinds]
        vary = "K" if "K" in kinds else "RADIUS" if "RADIUS" in kinds else None
        for v in (["0", "1", "20", "300"] if vary else [None]):
            a = list(base)
            if vary:
                a[kinds.index(vary)] = v
            call(name, a, "valid")
            if name.endswith("_stream"):
                call(name, a, "valid", "count(*), sum(id), sum(distance)")
        for i, kd in enumerate(kinds):
            for v in variants.get(kd, []):
                a = list(base)
                a[i] = v
                call(name, a, "valid")
        for i, kd in enumerate(kinds):
            for v in faults.get(kd, []):
                a = list(base)
                a[i] = v
                call(name, a, "one fault")
        call(name, base[:-1], "one fault")
        call(name, base + ["1"], "one fault")
        # two faults: an argument checked on its own (k, limit, candidates) with a fault checked after the arguments
        for i, kd in enumerate(kinds):
            for e in early.get(kd, []):
                for j, kl in enumerate(kinds):
                    for v in later.get(kl, []):
                        a = list(base)
                        a[i], a[j] = e, v
                        call(name, a, "two faults")
        if "LIMIT" in kinds:
            a = list(base)
            a[kinds.index("K")], a[kinds.index("LIMIT")] = "-1", "-1"
            call(name, a, "two faults")
        if "CAND" in kinds:                                           # k = 0 used to return before candidates was checked
            a = list(base)
            a[kinds.index("K")], a[kinds.index("CAND")] = "0", "-1"
            call(name, a, "two faults")
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--a", required=True, help="first extension build (path without .so)")
    ap.add_argument("--b", required=True, help="second extension build")
    ap.add_argument("--out", default=None, help="directory for the full outputs and the differences (JSON)")
    args = ap.parse_args()
    s, q = setup()
    stmts = corpus(q)
    sql = s + [st for st, _ in stmts]
    ra = run_sql(args.a, sql)[len(s):]
    rb = run_sql(args.b, sql)[len(s):]
    diffs, counts = [], {}
    for (st, tag), a, b in zip(stmts, ra, rb):
        counts.setdefault(tag, [0, 0])
        counts[tag][0] += 1
        if a != b:
            counts[tag][1] += 1
            diffs.append({"statement": st, "tag": tag, "a": a, "b": b})
    unexpected = [d for d in diffs if d["tag"] != "two faults"]
    summary = {"statements": len(stmts), "by_tag": {t: {"statements": n, "differ": d} for t, (n, d) in counts.items()},
               "valid_with_rows": sum(1 for (_, t), r in zip(stmts, rb) if t == "valid" and r.get("rows")),
               "unexpected": len(unexpected)}
    for d in diffs:
        print(json.dumps({"tag": d["tag"], "statement": d["statement"][:160], "a": str(d["a"])[:160], "b": str(d["b"])[:160]}))
    print(json.dumps(summary))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "sql_modules_diff.json"), "w") as f:
            json.dump({"summary": summary, "differences": diffs, "statements": [st for st, _ in stmts], "a": ra, "b": rb}, f)
    return 1 if unexpected else 0


if __name__ == "__main__":
    sys.exit(main())
