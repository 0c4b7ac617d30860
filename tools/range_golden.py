"""Writes tests/golden/sql_range.json: range answers of the UNMODIFIED reference (oracle/_ref, built by `make -C oracle` where the
reference tree is readable).  The reference's only door to "every row closer than r" is a stream module:
    SELECT id, distance FROM vector_*_scan_stream(...) WHERE distance < r AND id > 0 [AND id IN (...)] ORDER BY distance, id
(id > 0 drops the stream cursor's leading (0, 0.0) row).  Positive increasing rowids, so rowid order is scan order.  f32 full scans
use small integer elements (exact distances on both sides), quantized scans INT8 / UINT8.  Radii per query: a row's exact
distance (that row is out), the next double above it (in), 0, the 25th percentile (negative for DOT), one above every row.

    make -C oracle && python tools/range_golden.py
"""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tests.sqlrun import REF_CPU, run_sql  # noqa: E402

TABLES = [("tf", "type=FLOAT32,dimension=8,distance=L2", None), ("td", "type=FLOAT32,dimension=8,distance=DOT", None),
          ("tq", "type=FLOAT32,dimension=16,distance=L2", "qtype=INT8"), ("tu", "type=FLOAT32,dimension=16,distance=DOT", "qtype=UINT8")]


def stream(c):
    return "vector_%s_scan_stream('%s', 'e', x'%s')" % ("quantize" if c["quantized"] else "full", c["table"], c["vector"])


def main(n=32):
    rng = np.random.Generator(np.random.PCG64(20261016))
    setup, queries = [], []
    for tbl, opts, qopts in TABLES:
        dim = int(opts.split("dimension=")[1].split(",")[0])
        x = (rng.integers(-3, 4, (n, dim)) if qopts is None else rng.standard_normal((n, dim))).astype(np.float32)
        setup += [f"CREATE TABLE {tbl} (id INTEGER PRIMARY KEY, e BLOB)", f"SELECT vector_init('{tbl}', 'e', '{opts}')",
                  "INSERT INTO %s VALUES %s" % (tbl, ", ".join(f"({2 * i + 3}, x'{v.tobytes().hex()}')" for i, v in enumerate(x)))]
        setup += [f"SELECT vector_quantize('{tbl}', 'e', '{qopts}')"] if qopts else []
        q = (rng.integers(-3, 4, dim) if qopts is None else rng.standard_normal(dim)).astype(np.float32)
        queries.append({"table": tbl, "quantized": qopts is not None, "vector": q.tobytes().hex()})
    alld = run_sql(REF_CPU, setup + [f"SELECT distance FROM {stream(c)} WHERE id > 0" for c in queries])[len(setup):]
    cases = []
    for c, res in zip(queries, alld):
        d = np.unique(np.array([row[0] for row in res["rows"]], dtype=np.float64))
        at = float(d[len(d) // 10])
        keep = [2 * i + 3 for i in range(n) if rng.random() < 0.4]
        for r in (at, float(np.nextafter(at, np.inf)), 0.0, float(np.percentile(d, 25)), float(d[-1]) + 1.0):
            cases += [dict(c, radius=r, filter=None), dict(c, radius=r, filter=keep)]
    where = lambda e: "" if e["filter"] is None else " AND id IN (%s)" % ",".join(map(str, e["filter"]))
    res = run_sql(REF_CPU, setup + [[f"SELECT id, distance FROM {stream(e)} WHERE distance < ? AND id > 0{where(e)} ORDER BY distance, id",
                                      [e["radius"]]] for e in cases])
    assert all("error" not in r for r in res), [r for r in res if "error" in r]
    for e, r in zip(cases, res[len(setup):]):
        e["rows"] = r["rows"]
    out = os.path.join(ROOT, "tests", "golden", "sql_range.json")
    with open(out, "w") as f:
        json.dump({"setup": setup, "cases": cases}, f)
    print(out, os.path.getsize(out), "bytes,", len(cases), "cases,", sum(len(e["rows"]) for e in cases), "rows")


if __name__ == "__main__":
    main()
