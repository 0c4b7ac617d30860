"""Groupings and the device layout builder of grouped top-k without a GPU: the layout kernels keep no local memory and fit their
blocks, and the grouped SQL modules, which now keep a grouping between statements, still check their arguments first."""
import os
import re
import shutil
import subprocess

import pytest

LIB = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "sqlite_vector_b200", "lib", "libvsb200.so")


def test_layout_kernels_spill_nothing_and_fit_their_blocks():
    if not shutil.which("cuobjdump") or not os.path.exists(LIB):
        pytest.skip("no cuobjdump or no build here")
    res = subprocess.run(["cuobjdump", "-res-usage", LIB], capture_output=True, text=True, check=True, timeout=300).stdout
    parts = re.split(r"Function (\S+):", res)
    dem = subprocess.run(["c++filt"], input="\n".join(parts[1::2]), capture_output=True, text=True, check=True).stdout.splitlines()
    kinds = {"grouped_map_count_kernel": 256, "grouped_scan64_kernel": 1024, "grouped_map_write_kernel": 256,
             "grouped_sort_hist_kernel": 256, "grouped_sort_scan_kernel": 256, "grouped_sort_scatter_kernel": 256,
             "grouped_table_keys_kernel": 256, "grouped_uniq_count_kernel": 256, "grouped_uniq_write_kernel": 256,
             "grouped_koff_kernel": 256, "grouped_piece_count_kernel": 256, "grouped_piece_write_kernel": 256,
             "grouped_rows_kernel": 256}
    seen = set()
    for d, body in zip(dem, parts[2::2]):
        kind = next((k for k in kinds if k + "(" in d), None)
        if kind is None:
            continue
        seen.add(kind)
        regs, local = int(re.search(r"REG:(\d+)", body).group(1)), int(re.search(r"LOCAL:(\d+)", body).group(1))
        shared = int(re.search(r"SHARED:(\d+)", body).group(1))
        assert local == 0, (d, local)
        assert regs * kinds[kind] <= 65536 and regs <= 64, (d, regs)          # one block fits an SM's register file
        assert shared <= 48 * 1024, (d, shared)                               # static shared memory only
    assert seen == set(kinds), set(kinds) - seen


SETUP = ["CREATE TABLE t (id INTEGER PRIMARY KEY, e BLOB, doc INTEGER)", "SELECT vector_init('t','e','type=INT8,dimension=4')",
         "INSERT INTO t VALUES (1, x'01020304', 3), (2, x'02030405', NULL), (5, x'00000000', 9), (7, x'01010101', 3)"]


def test_grouped_modules_check_their_arguments_on_repeated_statements():
    """the same faulty statement twice, and once after a valid-looking one, gives the same error each time: a kept grouping never
    stands in for the checks"""
    from tests.sqlrun import OURS, run_sql
    q = "x'01020304'"
    pair = "x'03000000000000000100000000000000'"
    bad = [
        (f"SELECT * FROM vector_full_scan_grouped('t','e',{q},3,x'0100000000000000',NULL)",
         "vector_full_scan_grouped: groups has 8 bytes, expected a multiple of 16 (int64 key, int64 rowid pairs)."),
        (f"SELECT * FROM vector_quantize_scan_grouped('t','e',{q},3,{pair},-1)", "vector_quantize_scan_grouped: limit must not be negative."),
        (f"SELECT * FROM vector_full_scan_grouped('t','e',{q},-2,{pair},NULL)", "vector_full_scan_grouped: k must not be negative."),
        (f"SELECT * FROM vector_full_scan_grouped('t','e',x'0102',3,{pair},NULL)", "vector_full_scan_grouped: input vector has 2 bytes, expected 4."),
        (f"SELECT * FROM vector_full_scan_grouped('u','e',{q},3,{pair},NULL)", "vector_full_scan_grouped: unable to retrieve context."),
    ]
    s = list(SETUP)
    for sql, _ in bad:
        s += [sql, sql]
    r = run_sql(OURS, s)[len(SETUP):]
    for i, (_, err) in enumerate(bad):
        assert r[2 * i]["error"] == err and r[2 * i + 1]["error"] == err, (i, r[2 * i], r[2 * i + 1])
