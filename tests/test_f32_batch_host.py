"""The built library's TF32 scoring kernels for f32 columns (option f32_batch), without a GPU: cuobjdump -sass / -res-usage."""
import json
import os
import re
import shutil
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "sqlite_vector_b200", "lib", "libvsb200.so")
TK_TF32 = 4
MC_L2, MC_COS, MC_DOT, MC_TC_SCORES = 0, 1, 2, 4
TC_THREADS = 2 * 128 + 32          # kTcThreads: two consumer warpgroups and the TMA producer warp


def _demangled(names):
    out = subprocess.run(["c++filt"], input="\n".join(names), capture_output=True, text=True, check=True).stdout.splitlines()
    return {a: re.sub(r"\(.*$", "", b).replace("vsb::", "").replace("void ", "") for a, b in zip(names, out)}


def _tf32_kernels(text, pattern):
    """{(MC, N): what follows the kernel's header line, up to the next one} for tc_scan_kernel<TK_TF32, MC, N>"""
    parts = re.split(pattern, text)
    mangled = parts[1::2]
    dem = _demangled(mangled)
    out = {}
    for name, body in zip(mangled, parts[2::2]):
        m = re.fullmatch(r"tc_scan_kernel<(\d+), (\d+), (\d+)>", dem[name])
        if m and int(m.group(1)) == TK_TF32:
            out[(int(m.group(2)), int(m.group(3)))] = body
    return out


def test_tf32_scoring_kernels_are_hgmma_tf32_tma_fed_one_cta_per_sm_without_spills():
    """tc_scan_kernel<TK_TF32, MC, N> exists for L2, cosine, dot and the scores mode at N = 32, 64 and 128 (not 256); each
    multiplies with HGMMA on TF32 operands fed by TMA tensor loads (UTMALDG), spills nothing to local memory, and its
    registers leave room for one 288-thread CTA per SM"""
    if not shutil.which("cuobjdump"):
        pytest.skip("no cuobjdump here")
    want = {(mc, n) for mc in (MC_L2, MC_COS, MC_DOT, MC_TC_SCORES) for n in (32, 64, 128)}
    sass = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True, check=True, timeout=300).stdout
    kern = _tf32_kernels(sass, r"Function : (\S+)")
    assert set(kern) == want, sorted(kern)
    for key, body in kern.items():
        mma = re.findall(r"\bHGMMA\.(\S+)", body)
        assert mma and all(re.fullmatch(r"64x%dx8\.F32\.TF32" % key[1], m) for m in mma), (key, sorted(set(mma)))
        assert "UTMALDG" in body, key
        assert not re.search(r"\b(STL|LDL|HMMA|IMMA)\b", body), key
    res = subprocess.run(["cuobjdump", "-res-usage", LIB], capture_output=True, text=True, check=True, timeout=300).stdout
    usage = _tf32_kernels(res, r"Function (\S+):")
    assert set(usage) == want, sorted(usage)
    for key, line in usage.items():
        regs, local = int(re.search(r"REG:(\d+)", line).group(1)), int(re.search(r"LOCAL:(\d+)", line).group(1))
        # registers are allocated per warp in units of 256; an SM has 65536 of them for its resident CTAs
        per_warp = -(-regs * 32 // 256) * 256
        assert local == 0 and per_warp * (TC_THREADS // 32) <= 65536, (key, regs, local)


def test_sass_evidence_lists_the_tf32_kernels_with_wgmma_and_tma():
    if not shutil.which("cuobjdump"):
        pytest.skip("no cuobjdump here")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "sass_evidence.py")], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    ev = json.loads(r.stdout)
    tf32 = [k for k in ev["kernels"] if re.fullmatch(r"(void )?tc_scan_kernel<4, \d+, \d+>", k)]
    assert len(tf32) == 12, tf32
    assert all(k in ev["kernels_with_wgmma"] and k in ev["kernels_with_tma"] for k in tf32)
    assert not [k for k in ev["local_memory_spills"] if k in tf32]
    assert not ev["mma_sync_anywhere"]
