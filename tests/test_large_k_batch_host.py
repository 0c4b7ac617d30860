"""Large-k batches without a GPU: the built kernels of the batch path for k > 256 (plan_refine_kernel, lkb_bound_kernel,
lkb_sort_kernel) keep no local memory and fit their launch blocks on an SM."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "sqlite_vector_b200", "lib", "libvsb200.so")


def test_large_k_batch_kernels_spill_nothing_and_fit_their_blocks():
    if not shutil.which("cuobjdump"):
        pytest.skip("no cuobjdump here")
    res = subprocess.run(["cuobjdump", "-res-usage", LIB], capture_output=True, text=True, check=True, timeout=300).stdout
    parts = re.split(r"Function (\S+):", res)
    names = parts[1::2]
    dem = subprocess.run(["c++filt"], input="\n".join(names), capture_output=True, text=True, check=True).stdout.splitlines()
    threads = {"plan_refine_kernel": 256, "lkb_bound_kernel": 256, "lkb_sort_kernel": 512}
    seen = {k: 0 for k in threads}
    for d, body in zip(dem, parts[2::2]):
        kind = next((k for k in threads if re.search(r"\b%s\b" % k, d)), None)
        if kind is None:
            continue
        seen[kind] += 1
        regs, local = int(re.search(r"REG:(\d+)", body).group(1)), int(re.search(r"LOCAL:(\d+)", body).group(1))
        per_warp = -(-regs * 32 // 256) * 256
        assert local == 0 and per_warp * (threads[kind] // 32) <= 65536, (d, regs, local)
    # one plan_refine_kernel per element type (5) and metric class (L2, cosine, dot, L1)
    assert seen == {"plan_refine_kernel": 20, "lkb_bound_kernel": 1, "lkb_sort_kernel": 1}, seen
