"""Listed rows without a GPU: the argument errors of vector_quantize_scan_rerank(_batch), and rows_distance_kernel's resources
(no local memory, registers for its 256-thread blocks)."""
import os
import re
import shutil
import subprocess

import pytest

from tests.sqlrun import OURS, run_sql

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "sqlite_vector_b200", "lib", "libvsb200.so")


def test_rerank_argument_errors():
    s = ["CREATE TABLE t (id INTEGER PRIMARY KEY, e BLOB)", "SELECT vector_init('t','e','type=FLOAT32,dimension=2')",
         "INSERT INTO t(id, e) VALUES (1, x'0000803f00000040')"]
    mark = len(s)
    q = "x'0000803f00000040'"
    for fn in ("vector_quantize_scan_rerank", "vector_quantize_scan_rerank_batch"):
        s += [f"SELECT * FROM {fn}('t','e',{q},3)",                         # 0 4 arguments: SQLite refuses the missing hidden column
              f"SELECT * FROM {fn}(1,'e',{q},3,10)",                        # 1
              f"SELECT * FROM {fn}('t','e',1.5,3,10)",                      # 2
              f"SELECT * FROM {fn}('t','e',{q},'k',10)",                    # 3
              f"SELECT * FROM {fn}('t','e',{q},3,'many')",                  # 4
              f"SELECT * FROM {fn}('t','e',{q},3,2.5)",                     # 5
              f"SELECT * FROM {fn}('nope','e',{q},3,10)",                   # 6
              f"SELECT * FROM {fn}('t','e',x'01020304',3,10)",              # 7 short input
              f"SELECT * FROM {fn}('t','e',{q},3,10)"]                      # 8 never quantized
    r = run_sql(OURS, s)[mark:]
    for i, fn in enumerate(("vector_quantize_scan_rerank", "vector_quantize_scan_rerank_batch")):
        e = [x.get("error") for x in r[9 * i: 9 * i + 9]]
        assert e[0] is not None
        assert e[1] == f"{fn}: argument 1 must be of type TEXT (got INTEGER)."
        assert e[2] == f"{fn}: argument 3 must be of type TEXT or BLOB (got REAL)."
        assert e[3] == f"{fn}: argument 4 must be of type INTEGER (got TEXT)."
        assert e[4] == f"{fn}: argument 5 must be of type INTEGER (got TEXT)."
        assert e[5] == f"{fn}: argument 5 must be of type INTEGER (got REAL)."
        assert e[6] == f"{fn}: unable to retrieve context."
        if fn.endswith("_batch"):
            assert e[7] == f"{fn}: input has 4 bytes, expected a positive multiple of 8 (dimension 2)."
        else:
            assert e[7] == f"{fn}: input vector has 4 bytes, expected 8."
        assert e[8].startswith("Quantization table not found for table 't' and column 'e'."), e[8]


def test_rows_kernel_spills_nothing():
    """rows_distance_kernel, every (type, metric): no local memory, registers for its 256-thread blocks on one SM"""
    if not shutil.which("cuobjdump"):
        pytest.skip("no cuobjdump here")
    res = subprocess.run(["cuobjdump", "-res-usage", LIB], capture_output=True, text=True, check=True, timeout=300).stdout
    parts = re.split(r"Function (\S+):", res)
    names = parts[1::2]
    dem = subprocess.run(["c++filt"], input="\n".join(names), capture_output=True, text=True, check=True).stdout.splitlines()
    seen = 0
    for d, body in zip(dem, parts[2::2]):
        if not re.search(r"\brows_distance_kernel<", d):
            continue
        seen += 1
        regs, local = int(re.search(r"REG:(\d+)", body).group(1)), int(re.search(r"LOCAL:(\d+)", body).group(1))
        assert local == 0 and -(-regs * 32 // 256) * 256 * 8 <= 65536, (d, regs, local)
    assert seen == 20, seen
