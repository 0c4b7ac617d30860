"""Batched grouped top-k without a GPU: the two vector_*_scan_grouped_batch modules check their arguments in the order every
module keeps (the count, then each argument in position order, then the context, the vectors, the quantization table and
staging), with no CUDA device visible; and the kernels the passes added or changed keep no local memory and fit their blocks."""
import os
import re
import shutil
import subprocess

import pytest

from tests.sqlrun import OURS, run_sql

LIB = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "sqlite_vector_b200", "lib", "libvsb200.so")
SETUP = ["CREATE TABLE t (id INTEGER PRIMARY KEY, e BLOB)", "SELECT vector_init('t','e','type=FLOAT32,dimension=2')",
         "INSERT INTO t(id, e) VALUES (1, x'0000803f00000040'), (2, x'01')"]
Q2 = "x'0000803f000000400000803f00000040'"                         # two queries of dimension 2
PAIRS = "x'03000000000000000100000000000000'"


@pytest.mark.parametrize("fn", ["vector_full_scan_grouped_batch", "vector_quantize_scan_grouped_batch"])
def test_batch_modules_check_arguments_in_order(fn):
    stmts = [f"SELECT * FROM {fn}('t','e',{Q2},3,{PAIRS})",                # the count
             f"SELECT * FROM {fn}('nope','e',x'01',-1,x'01',-1)",          # k first: before groups, limit, context, vectors
             f"SELECT * FROM {fn}('nope','e',x'01',3,x'01',-1)",           # groups before limit
             f"SELECT * FROM {fn}('nope','e',x'01',3,{PAIRS},-1)",         # limit before the context
             f"SELECT * FROM {fn}('nope','e',{Q2},3,{PAIRS},NULL)",        # the context
             f"SELECT * FROM {fn}('t','e',NULL,3,{PAIRS},NULL)",           # the vectors' type
             f"SELECT * FROM {fn}('t','e',x'010203',3,{PAIRS},NULL)",      # not whole queries
             f"SELECT * FROM {fn}('t','e','[1,2,3]',3,{PAIRS},NULL)",      # a JSON array of no whole queries
             f"SELECT * FROM {fn}('t','e',{Q2},3,{PAIRS},NULL)",           # quantization table / staging
             f"SELECT * FROM {fn}('t','e','[1,2,1,2]',0,{PAIRS},NULL)"]    # k = 0 still stages first
    errs = [o.get("error") for o in run_sql(OURS, SETUP + stmts, env={"CUDA_VISIBLE_DEVICES": ""})[len(SETUP):]]
    assert errs[:8] == [f"{fn} expects 6 arguments, but 5 were provided.",
                        f"{fn}: k must not be negative.",
                        f"{fn}: groups has 1 bytes, expected a multiple of 16 (int64 key, int64 rowid pairs).",
                        f"{fn}: limit must not be negative.",
                        f"{fn}: unable to retrieve context.",
                        f"{fn}: argument 3 must be of type TEXT or BLOB (got N/A).",
                        f"{fn}: input has 3 bytes, expected a positive multiple of 8 (dimension 2).",
                        f"{fn}: input has 12 bytes, expected a positive multiple of 8 (dimension 2)."], errs
    for e in errs[8:]:
        if "_quantize_" in fn:
            assert e.startswith("Quantization table not found for table 't' and column 'e'."), e
        else:
            assert e.startswith("Invalid vector blob found at rowid 2.") or e.startswith("vector_full_scan: "), e


def test_pass_kernels_spill_nothing_and_fit_their_blocks():
    if not shutil.which("cuobjdump") or not os.path.exists(LIB):
        pytest.skip("no cuobjdump or no build here")
    res = subprocess.run(["cuobjdump", "-res-usage", LIB], capture_output=True, text=True, check=True, timeout=300).stdout
    parts = re.split(r"Function (\S+):", res)
    dem = subprocess.run(["c++filt"], input="\n".join(parts[1::2]), capture_output=True, text=True, check=True).stdout.splitlines()
    # threads of a block: the grouped steps run 8 warps, the offsets kernels 1024 threads, the scan 8 warps
    kinds = {"grouped_walk_kernel": 256, "grouped_bounds_kernel": 256, "grouped_count_kernel": 256, "grouped_write_kernel": 256,
             "grouped_offsets_kernel": 1024, "lk_offsets_kernel": 1024, "scan_pass_kernel": 256}
    seen = set()
    for d, body in zip(dem, parts[2::2]):
        kind = next((k for k in kinds if k + "(" in d or k + "<" in d), None)
        if kind is None:
            continue
        seen.add(kind)
        regs, local = int(re.search(r"REG:(\d+)", body).group(1)), int(re.search(r"LOCAL:(\d+)", body).group(1))
        assert local == 0, (d, local)
        assert regs * kinds[kind] <= 65536 and regs <= 255, (d, regs)
    assert seen == set(kinds), set(kinds) - seen
