"""The built library's L1 batch kernel, without a GPU: tools/sass_evidence.py over cuobjdump -sass."""
import json
import os
import re
import shutil
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
T_F32, T_F16, T_BF16, T_U8, T_I8 = 1, 2, 3, 4, 5


def test_l1_batch_kernel_is_tma_fed_integer_dp4a_without_spills():
    """l1_batch_kernel<VT, N> exists for all five element types and every tile width; each is fed by TMA tensor loads
    (UTMALDG); the int8 / uint8 ones add with IDP.4A; none spills to local memory and nothing uses mma.sync"""
    if not shutil.which("cuobjdump"):
        pytest.skip("no cuobjdump here")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "sass_evidence.py")], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    ev = json.loads(r.stdout)
    ks = ev["kernels"]
    l1 = {}
    for name, ops in ks.items():
        m = re.search(r"\bl1_batch_kernel<(\d+), (\d+)>$", name)
        if m:
            l1[(int(m.group(1)), int(m.group(2)))] = ops
    assert set(l1) == {(vt, n) for vt in (T_F32, T_F16, T_BF16, T_U8, T_I8) for n in (32, 64, 128)}, sorted(ks)
    for (vt, n), ops in l1.items():
        assert "UTMALDG" in ops, (vt, n, ops)
        assert ("IDP" in ops) == (vt in (T_U8, T_I8)), (vt, n, ops)
        assert not any(op in ops for op in ("HMMA", "IMMA", "HGMMA", "IGMMA")), (vt, n, ops)
    assert not ev["mma_sync_anywhere"]
    assert not [k for k in ev["local_memory_spills"] if "l1_batch_kernel" in k], ev["local_memory_spills"]
