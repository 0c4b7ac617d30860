"""Range search without a GPU: the SQL argument checks of the four *_range modules and the built range kernels
(scan_range_kernel, range_sort_kernel: no spills, their planned CTAs fit an SM)."""
import os
import re
import shutil
import subprocess

import pytest

from tests.sqlrun import OURS, run_sql

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "sqlite_vector_b200", "lib", "libvsb200.so")
SETUP = ["CREATE TABLE t (id INTEGER PRIMARY KEY, e BLOB)", "SELECT vector_init('t','e','type=INT8,dimension=4')",
         "INSERT INTO t VALUES (1, x'01020304'), (2, x'02030405'), (5, x'00000000')"]


def test_range_modules_check_their_arguments():
    q = "x'01020304'"
    s = SETUP + [
        f"SELECT * FROM vector_full_scan_range('t','e',{q},'r')",
        f"SELECT * FROM vector_full_scan_range('t','e',{q},NULL)",
        f"SELECT * FROM vector_quantize_scan_range('t','e',{q},x'00')",
        f"SELECT * FROM vector_full_scan_range(1,'e',{q},2.5)",
        f"SELECT * FROM vector_quantize_scan_range('t','e',7,2.5)",
        f"SELECT * FROM vector_full_scan_range_filtered('t','e',{q},2.5,NULL)",
        f"SELECT * FROM vector_full_scan_range_filtered('t','e',{q},2.5,x'0102')",
        f"SELECT * FROM vector_quantize_scan_range_filtered('t','e',{q},'x',x'0100000000000000')",
        f"SELECT * FROM vector_quantize_scan_range_filtered('t','e',{q},2,'1,2')",
        f"SELECT * FROM vector_full_scan_range('t','e',{q})",
        f"SELECT * FROM vector_full_scan_range('nope','e',{q},1.0)",
        f"SELECT * FROM vector_full_scan_range('t','e',x'0102',1.0)",
    ]
    r = run_sql(OURS, s)[len(SETUP):]
    assert r[0]["error"] == "vector_full_scan_range: argument 4 must be of type INTEGER or FLOAT (got TEXT)."
    assert r[1]["error"] == "vector_full_scan_range: argument 4 must be of type INTEGER or FLOAT (got N/A)."
    assert r[2]["error"] == "vector_quantize_scan_range: argument 4 must be of type INTEGER or FLOAT (got BLOB)."
    assert r[3]["error"] == "vector_full_scan_range: argument 1 must be of type TEXT (got INTEGER)."
    assert r[4]["error"] == "vector_quantize_scan_range: argument 3 must be of type TEXT or BLOB (got INTEGER)."
    assert r[5]["error"] == "vector_full_scan_range_filtered: argument 5 must be of type BLOB (got N/A)."
    assert r[6]["error"] == "vector_full_scan_range_filtered: rowids has 2 bytes, expected a multiple of 8 (int64 rowids)."
    assert r[7]["error"] == "vector_quantize_scan_range_filtered: argument 4 must be of type INTEGER or FLOAT (got TEXT)."
    assert r[8]["error"] == "vector_quantize_scan_range_filtered: argument 5 must be of type BLOB (got TEXT)."
    assert "error" in r[9]                                     # 3 arguments: SQLite refuses the missing hidden column itself
    assert r[10]["error"] == "vector_full_scan_range: unable to retrieve context."
    assert r[11]["error"] == "vector_full_scan_range: input vector has 2 bytes, expected 4."


def test_range_kernels_spill_nothing_and_fit_their_ctas():
    """every scan_range_kernel instantiation (256 threads, one CTA per SM) and range_sort_kernel (1024 threads, one block per
    query) keeps no local memory and fits its registers on an SM"""
    if not shutil.which("cuobjdump"):
        pytest.skip("no cuobjdump here")
    res = subprocess.run(["cuobjdump", "-res-usage", LIB], capture_output=True, text=True, check=True, timeout=300).stdout
    parts = re.split(r"Function (\S+):", res)
    names = parts[1::2]
    dem = subprocess.run(["c++filt"], input="\n".join(names), capture_output=True, text=True, check=True).stdout.splitlines()
    threads = {"scan_range_kernel": 256, "range_sort_kernel": 1024}
    seen = {k: 0 for k in threads}
    for d, body in zip(dem, parts[2::2]):
        kind = next((k for k in threads if re.search(r"\b%s\b" % k, d)), None)
        if kind is None:
            continue
        seen[kind] += 1
        regs, local = int(re.search(r"REG:(\d+)", body).group(1)), int(re.search(r"LOCAL:(\d+)", body).group(1))
        per_warp = -(-regs * 32 // 256) * 256
        assert local == 0 and per_warp * (threads[kind] // 32) <= 65536, (d, regs, local)
    assert seen == {"scan_range_kernel": 40, "range_sort_kernel": 1}, seen
