"""Filtered top-k without a GPU: the SQL argument checks of the *_filtered modules, the vector_rowid_set aggregate, the row bitmap
of the Python mirror, and the built kernels that test the row filter (no spills, one CTA per SM)."""
import json
import os
import re
import shutil
import struct
import subprocess

import numpy as np
import pytest

from tests.sqlrun import OURS, run_sql

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "sqlite_vector_b200", "lib", "libvsb200.so")
SETUP = ["CREATE TABLE t (id INTEGER PRIMARY KEY, e BLOB, lang TEXT)", "SELECT vector_init('t','e','type=INT8,dimension=4')",
         "INSERT INTO t VALUES (1, x'01020304', 'en'), (2, x'02030405', NULL), (5, x'00000000', 'en'), (7, x'01010101', 'de')"]


def test_filtered_modules_check_their_arguments():
    q = "x'01020304'"
    s = SETUP + [
        f"SELECT * FROM vector_full_scan_filtered('t','e',{q},3,NULL)",
        f"SELECT * FROM vector_full_scan_filtered('t','e',{q},3,'1,2')",
        f"SELECT * FROM vector_full_scan_filtered('t','e',{q},3,x'01020304')",
        f"SELECT * FROM vector_quantize_scan_filtered('t','e',{q},3,12)",
        f"SELECT * FROM vector_full_scan_batch_filtered('t','e',{q},3,x'010203')",
        f"SELECT * FROM vector_quantize_scan_batch_filtered('t','e',{q},3,NULL)",
        f"SELECT * FROM vector_full_scan_filtered('t','e',{q},'k',x'0100000000000000')",
        f"SELECT * FROM vector_full_scan_filtered('t','e',{q},3)",
    ]
    r = run_sql(OURS, s)[len(SETUP):]
    assert r[0]["error"] == "vector_full_scan_filtered: argument 5 must be of type BLOB (got N/A)."
    assert r[1]["error"] == "vector_full_scan_filtered: argument 5 must be of type BLOB (got TEXT)."
    assert r[2]["error"] == "vector_full_scan_filtered: rowids has 4 bytes, expected a multiple of 8 (int64 rowids)."
    assert r[3]["error"] == "vector_quantize_scan_filtered: argument 5 must be of type BLOB (got INTEGER)."
    assert r[4]["error"] == "vector_full_scan_batch_filtered: rowids has 3 bytes, expected a multiple of 8 (int64 rowids)."
    assert r[5]["error"] == "vector_quantize_scan_batch_filtered: argument 5 must be of type BLOB (got N/A)."
    assert r[6]["error"] == "vector_full_scan_filtered: argument 4 must be of type INTEGER (got TEXT)."
    assert "error" in r[7]                                     # 4 arguments: SQLite refuses the missing hidden column itself


def test_vector_rowid_set_builds_int64_blobs_and_skips_nulls():
    r = run_sql(OURS, SETUP + ["SELECT vector_rowid_set(id) FROM t WHERE lang = 'en'",
                               "SELECT vector_rowid_set(CASE WHEN lang IS NULL THEN NULL ELSE id END) FROM t",
                               "SELECT vector_rowid_set(id) FROM t WHERE 0",
                               "SELECT length(vector_rowid_set(id)), typeof(vector_rowid_set(id)) FROM t WHERE 0",
                               "SELECT vector_rowid_set(x) FROM (SELECT -3 AS x UNION ALL SELECT 9223372036854775807)"])[len(SETUP):]

    def ids(cell):
        b = bytes.fromhex(cell["hex"])
        return list(struct.unpack("<%dq" % (len(b) // 8), b))
    assert ids(r[0]["rows"][0][0]) == [1, 5]
    assert ids(r[1]["rows"][0][0]) == [1, 5, 7]
    assert ids(r[2]["rows"][0][0]) == []
    assert r[3]["rows"] == [[0, "blob"]]
    assert sorted(ids(r[4]["rows"][0][0])) == [-3, 2**63 - 1]


def test_aggregate_context_slot_against_sqlite_header(tmp_path):
    """vector_rowid_set reaches sqlite3_aggregate_context through a slot of its own in sqlite_abi.h: pin it against the position a
    real sqlite3ext.h gives (tests/golden/sqlite3_api_slot_aggregate.json), and against a header on this machine if any"""
    abi = open(os.path.join(ROOT, "sqlite_vector_b200", "csrc", "sqlite_abi.h")).read()
    slot = int(re.search(r"#define VSQ_SLOT_AGGREGATE_CONTEXT (\d+)", abi).group(1))
    assert re.search(r"#define sqlite3_aggregate_context .*slot\[VSQ_SLOT_AGGREGATE_CONTEXT\]", abi)
    golden = json.load(open(os.path.join(ROOT, "tests", "golden", "sqlite3_api_slot_aggregate.json")))["slots"]
    assert golden["aggregate_context"] == slot
    hdr_dir = "/usr/include"
    if not os.path.exists(os.path.join(hdr_dir, "sqlite3ext.h")):
        return
    src = tmp_path / "chk.c"
    src.write_text('#include <stddef.h>\n#include "sqlite3ext.h"\n'
                   f'_Static_assert(offsetof(sqlite3_api_routines, aggregate_context) == {slot} * sizeof(void*), "slot");\n'
                   "int main(void){return 0;}\n")
    subprocess.run(["gcc", "-I", hdr_dir, "-c", str(src), "-o", str(tmp_path / "chk.o")], check=True)


def test_row_bitmap_layout():
    from sqlite_vector_b200.api import row_bitmap
    rng = np.random.Generator(np.random.PCG64(3))
    for n in (0, 1, 31, 32, 33, 1000):
        m = rng.random(n) < 0.3
        b = row_bitmap(m)
        assert b.dtype == np.uint32 and b.size == (n + 31) // 32
        got = np.array([(int(b[i >> 5]) >> (i & 31)) & 1 for i in range(n)], dtype=bool)
        assert np.array_equal(got, m)


def test_filter_kernels_spill_nothing_and_fit_one_cta_per_sm():
    """the kernels that test the row filter (scan_kernel, tc_scan_kernel, l1_batch_kernel, all_pairs_kernel) keep no local memory
    and leave room for their one CTA per SM; all_pairs_kernel takes the bitmap"""
    if not shutil.which("cuobjdump"):
        pytest.skip("no cuobjdump here")
    res = subprocess.run(["cuobjdump", "-res-usage", LIB], capture_output=True, text=True, check=True, timeout=300).stdout
    parts = re.split(r"Function (\S+):", res)
    names = parts[1::2]
    dem = subprocess.run(["c++filt"], input="\n".join(names), capture_output=True, text=True, check=True).stdout.splitlines()
    threads = {"scan_kernel": 256, "tc_scan_kernel": 288, "l1_batch_kernel": 288, "all_pairs_kernel": 256}
    seen = set()
    for d, body in zip(dem, parts[2::2]):
        kind = next((k for k in threads if re.search(r"\b%s\b" % k, d)), None)
        if kind is None:
            continue
        seen.add(kind)
        if kind == "all_pairs_kernel":
            assert "unsigned int const*, long long" in d, d
        regs, local = int(re.search(r"REG:(\d+)", body).group(1)), int(re.search(r"LOCAL:(\d+)", body).group(1))
        per_warp = -(-regs * 32 // 256) * 256
        assert local == 0 and per_warp * (threads[kind] // 32) <= 65536, (d, regs, local)
    assert seen == set(threads), seen
