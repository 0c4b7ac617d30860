"""Grouped top-k (vsb_scan_topk_grouped) without a GPU: its kernels keep no local memory and fit their blocks, and the SQL
modules check their arguments before they touch a device."""
import os
import re
import shutil
import subprocess

import pytest

LIB = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "sqlite_vector_b200", "lib", "libvsb200.so")


def test_grouped_kernels_spill_nothing_and_fit_their_blocks():
    if not shutil.which("cuobjdump") or not os.path.exists(LIB):
        pytest.skip("no cuobjdump or no build here")
    res = subprocess.run(["cuobjdump", "-res-usage", LIB], capture_output=True, text=True, check=True, timeout=300).stdout
    parts = re.split(r"Function (\S+):", res)
    dem = subprocess.run(["c++filt"], input="\n".join(parts[1::2]), capture_output=True, text=True, check=True).stdout.splitlines()
    kinds = ("grouped_walk_kernel<true>", "grouped_walk_kernel<false>", "grouped_bounds_kernel<true>", "grouped_bounds_kernel<false>",
             "grouped_count_kernel", "grouped_write_kernel")
    seen = set()
    for d, body in zip(dem, parts[2::2]):
        kind = next((k for k in kinds if k in d), None)
        if kind is None:
            continue
        seen.add(kind)
        regs, local = int(re.search(r"REG:(\d+)", body).group(1)), int(re.search(r"LOCAL:(\d+)", body).group(1))
        assert local == 0 and regs <= 64, (d, regs, local)                  # 256-thread blocks, several per SM
    assert seen == set(kinds), seen


SETUP = ["CREATE TABLE t (id INTEGER PRIMARY KEY, e BLOB, doc INTEGER)", "SELECT vector_init('t','e','type=INT8,dimension=4')",
         "INSERT INTO t VALUES (1, x'01020304', 3), (2, x'02030405', NULL), (5, x'00000000', 9), (7, x'01010101', 3)"]


def test_grouped_modules_check_their_arguments():
    from tests.sqlrun import OURS, run_sql
    q = "x'01020304'"
    pair = "x'03000000000000000100000000000000'"
    s = SETUP + [
        f"SELECT * FROM vector_full_scan_grouped('t','e',{q},3,NULL,NULL)",
        f"SELECT * FROM vector_full_scan_grouped('t','e',{q},3,x'0100000000000000',NULL)",
        f"SELECT * FROM vector_quantize_scan_grouped('t','e',{q},3,{pair},'2')",
        f"SELECT * FROM vector_quantize_scan_grouped('t','e',{q},3,{pair},-1)",
        f"SELECT * FROM vector_full_scan_grouped('t','e',{q},'k',{pair},NULL)",
        f"SELECT * FROM vector_full_scan_grouped('t','e',{q},-2,{pair},NULL)",
        f"SELECT * FROM vector_full_scan_grouped('t','e',x'0102',3,{pair},NULL)",
        f"SELECT * FROM vector_full_scan_grouped('t','e',{q},3,{pair})",
        f"SELECT * FROM vector_full_scan_grouped('u','e',{q},3,{pair},NULL)",
    ]
    r = run_sql(OURS, s)[len(SETUP):]
    assert r[0]["error"] == "vector_full_scan_grouped: argument 5 must be of type BLOB (got N/A)."
    assert r[1]["error"] == "vector_full_scan_grouped: groups has 8 bytes, expected a multiple of 16 (int64 key, int64 rowid pairs)."
    assert r[2]["error"] == "vector_quantize_scan_grouped: argument 6 must be of type INTEGER or NULL (got TEXT)."
    assert r[3]["error"] == "vector_quantize_scan_grouped: limit must not be negative."
    assert r[4]["error"] == "vector_full_scan_grouped: argument 4 must be of type INTEGER (got TEXT)."
    assert r[5]["error"] == "vector_full_scan_grouped: k must not be negative."
    assert r[6]["error"] == "vector_full_scan_grouped: input vector has 2 bytes, expected 4."
    assert "error" in r[7]                                     # 5 arguments: SQLite refuses the missing hidden column itself
    assert r[8]["error"] == "vector_full_scan_grouped: unable to retrieve context."
