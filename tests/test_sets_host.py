"""Per-query sets (vsb_scan_topk_sets) without a GPU: the kernels the call adds keep no local memory and fit their blocks, and
the scorers that gained the per-pair set test still fit one CTA per SM."""
import os
import re
import shutil
import struct
import subprocess

import pytest

LIB = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "sqlite_vector_b200", "lib", "libvsb200.so")


def test_sets_kernels_spill_nothing_and_fit_their_blocks():
    if not shutil.which("cuobjdump") or not os.path.exists(LIB):
        pytest.skip("no cuobjdump or no build here")
    res = subprocess.run(["cuobjdump", "-res-usage", LIB], capture_output=True, text=True, check=True, timeout=300).stdout
    parts = re.split(r"Function (\S+):", res)
    dem = subprocess.run(["c++filt"], input="\n".join(parts[1::2]), capture_output=True, text=True, check=True).stdout.splitlines()
    threads = {"sets_pairs_kernel": 256, "sets_union_kernel": 256, "sets_prefix_kernel": 1024, "sets_plan_kernel": 1024,
               "tc_scan_kernel": 288, "l1_batch_kernel": 288}
    seen = set()
    for d, body in zip(dem, parts[2::2]):
        kind = next((k for k in threads if re.search(r"\b%s\b" % k, d)), None)
        if kind is None:
            continue
        seen.add(kind)
        regs, local = int(re.search(r"REG:(\d+)", body).group(1)), int(re.search(r"LOCAL:(\d+)", body).group(1))
        per_warp = -(-regs * 32 // 256) * 256
        assert local == 0 and per_warp * (threads[kind] // 32) <= 65536, (d, regs, local)
    assert seen == set(threads), seen


SETUP = ["CREATE TABLE t (id INTEGER PRIMARY KEY, e BLOB, tenant INTEGER)", "SELECT vector_init('t','e','type=INT8,dimension=4')",
         "INSERT INTO t VALUES (1, x'01020304', 3), (2, x'02030405', NULL), (5, x'00000000', 9), (7, x'01010101', 3)"]


def test_sets_modules_check_their_arguments():
    from tests.sqlrun import OURS, run_sql
    q, q2 = "x'01020304'", "x'0102030401020304'"
    pair = "x'03000000000000000100000000000000'"
    s = SETUP + [
        f"SELECT * FROM vector_full_scan_batch_sets('t','e',{q},3,NULL,NULL)",
        f"SELECT * FROM vector_full_scan_batch_sets('t','e',{q},3,x'0100000000000000',NULL)",
        f"SELECT * FROM vector_quantize_scan_batch_sets('t','e',{q},3,{pair},'0')",
        f"SELECT * FROM vector_quantize_scan_batch_sets('t','e',{q},3,{pair},x'0300')",
        f"SELECT * FROM vector_full_scan_batch_sets('t','e',{q2},3,{pair},x'0300000000000000')",
        f"SELECT * FROM vector_full_scan_batch_sets('t','e',{q},'k',{pair},NULL)",
        f"SELECT * FROM vector_full_scan_batch_sets('t','e',{q},3,{pair})",
    ]
    r = run_sql(OURS, s)[len(SETUP):]
    assert r[0]["error"] == "vector_full_scan_batch_sets: argument 5 must be of type BLOB (got N/A)."
    assert r[1]["error"] == "vector_full_scan_batch_sets: sets has 8 bytes, expected a multiple of 16 (int64 set, int64 rowid pairs)."
    assert r[2]["error"] == "vector_quantize_scan_batch_sets: argument 6 must be of type BLOB or NULL (got TEXT)."
    assert r[3]["error"] == "vector_quantize_scan_batch_sets: query_sets has 2 bytes, expected a multiple of 8 (int64 set indexes)."
    assert r[4]["error"] == "vector_full_scan_batch_sets: query_sets holds 1 set indexes for 2 queries."
    assert r[5]["error"] == "vector_full_scan_batch_sets: argument 4 must be of type INTEGER (got TEXT)."
    assert "error" in r[6]                                     # 5 arguments: SQLite refuses the missing hidden column itself


def test_vector_rowid_sets_builds_pair_blobs_and_skips_nulls():
    from tests.sqlrun import OURS, run_sql
    r = run_sql(OURS, SETUP + ["SELECT vector_rowid_sets(tenant, id) FROM t",
                               "SELECT vector_rowid_sets(tenant, CASE WHEN id = 5 THEN NULL ELSE id END) FROM t",
                               "SELECT vector_rowid_sets(tenant, id) FROM t WHERE 0",
                               "SELECT typeof(vector_rowid_sets(tenant, id)) FROM t WHERE 0",
                               "SELECT vector_rowid_sets(-1, 9223372036854775807)",
                               "SELECT vector_rowid_sets(id) FROM t"])[len(SETUP):]

    def pairs(cell):
        b = bytes.fromhex(cell["hex"])
        v = struct.unpack("<%dq" % (len(b) // 8), b)
        return [tuple(v[i:i + 2]) for i in range(0, len(v), 2)]
    assert pairs(r[0]["rows"][0][0]) == [(3, 1), (9, 5), (3, 7)]
    assert pairs(r[1]["rows"][0][0]) == [(3, 1), (3, 7)]
    assert pairs(r[2]["rows"][0][0]) == []
    assert r[3]["rows"] == [["blob"]]
    assert pairs(r[4]["rows"][0][0]) == [(-1, 2**63 - 1)]
    assert "error" in r[5]                                     # one argument: no such function
