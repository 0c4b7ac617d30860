"""Writes tests/golden/sql_large_k.json: top-k answers for k > 256 from the UNMODIFIED reference (oracle/_ref, built by
`make -C oracle` where the reference tree is readable).  Two tie-heavy small-integer tables of 1 100 rows (elements 0..2, rowids
1..n): vector_full_scan on an L2 table and vector_quantize_scan on a DOT table quantized to int8, each at k = 257, 300, 1000,
n - 1 and n + 5 (more than the table holds).  The filtered case: the reference has no filtered top-k, so its answer for the rows
`id IN (...)` is its own top-k over a table that holds exactly those rows (copied with INSERT ... SELECT ... WHERE id IN (...)),
which is what vector_*_scan_filtered promises.  The fixture stays compact: elements and queries as digit strings, answers as
rowids (base64 of little-endian uint16) plus run lengths of the (sorted) distances; tests/test_gpu_large_k.py rebuilds the SQL
with the same functions.

    make -C oracle && python tools/large_k_golden.py
"""
import base64
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tests.sqlrun import REF_CPU, run_sql  # noqa: E402
from tests.test_gpu_large_k import golden_query, golden_setup  # noqa: E402

# (table, vector_init options, vector_quantize options or None)
TABLES = [("tf", "type=FLOAT32,dimension=4,distance=L2", None), ("tq", "type=FLOAT32,dimension=4,distance=DOT", "qtype=INT8")]


def main(n=1100):
    rng = np.random.Generator(np.random.PCG64(20261017))
    tables, cases = [], []
    for tbl, opts, qopts in TABLES:
        x = rng.integers(0, 3, n * 4)                                 # 81 distinct rows: heavy ties
        keep = (np.nonzero(rng.random(n) < 0.4)[0] + 1).tolist()
        q = rng.integers(0, 3, 4)
        tables.append({"name": tbl, "opts": opts, "qopts": qopts, "dim": 4, "x": "".join(map(str, x)), "keep": keep,
                       "query": "".join(map(str, q))})
        for k in (257, 300, 1000, n - 1, n + 5):
            cases.append({"table": tbl, "quantized": qopts is not None, "k": k, "filtered": False})
        for k in (257, len(keep) + 3):
            cases.append({"table": tbl, "quantized": qopts is not None, "k": k, "filtered": True})
    gold = {"tables": tables, "cases": cases}
    setup = golden_setup(gold)
    res = run_sql(REF_CPU, setup + [golden_query(gold, e) for e in cases])
    assert all("error" not in r for r in res), [r for r in res if "error" in r][:2]
    for e, r in zip(cases, res[len(setup):]):
        e["ids"] = base64.b64encode(np.array([row[0] for row in r["rows"]], "<u2").tobytes()).decode()
        runs = []                                                      # distances ascending: [value, count] runs
        for row in r["rows"]:
            if runs and runs[-1][0] == row[1]:
                runs[-1][1] += 1
            else:
                runs.append([row[1], 1])
        e["dist"] = runs
    out = os.path.join(ROOT, "tests", "golden", "sql_large_k.json")
    with open(out, "w") as f:
        json.dump(gold, f, separators=(",", ":"))
    print(out, os.path.getsize(out), "bytes,", len(cases), "cases,", sum(c for e in cases for _, c in e["dist"]), "rows")


if __name__ == "__main__":
    main()
