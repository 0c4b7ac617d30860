"""Passes of several queries (DESIGN §3.1) without a GPU: scan_kernel (one query) and every width of scan_pass_kernel are built,
keep no local memory (no spills) and still fit one CTA of 256 threads per SM."""
import os
import re
import shutil
import subprocess

import pytest

LIB = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "sqlite_vector_b200", "lib", "libvsb200.so")


def test_every_pass_width_spills_nothing_and_fits_one_cta_per_sm():
    if not shutil.which("cuobjdump") or not os.path.exists(LIB):
        pytest.skip("no cuobjdump or no build here")
    res = subprocess.run(["cuobjdump", "-res-usage", LIB], capture_output=True, text=True, check=True, timeout=300).stdout
    parts = re.split(r"Function (\S+):", res)
    dem = subprocess.run(["c++filt"], input="\n".join(parts[1::2]), capture_output=True, text=True, check=True).stdout.splitlines()
    widths = {}
    for d, body in zip(dem, parts[2::2]):
        m = re.search(r"\bscan(_pass)?_kernel<(\d+), (\d+), (true|false)(?:, (\d+))?>", d)
        if m is None:
            continue
        w = int(m.group(5) or 1)
        widths[w] = widths.get(w, 0) + 1
        regs, local = int(re.search(r"REG:(\d+)", body).group(1)), int(re.search(r"LOCAL:(\d+)", body).group(1))
        per_warp = -(-regs * 32 // 256) * 256
        assert local == 0 and per_warp * 8 <= 65536, (d, regs, local)
    # 5 element types x 4 metric kernels x (staged, DIRECT) at each width
    assert widths == {1: 40, 2: 40, 4: 40, 8: 40}, widths
