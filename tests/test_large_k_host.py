"""Large k (k > 256) without a GPU: the host slot replay keeps the slots' first argmax in a tournament tree above 256, and must
give the reference's answer bit for bit (rows, order, distances, max_index carry, INF trim); the built large-k kernels keep no
local memory and fit their planned blocks on an SM."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from oracle import pyoracle as po

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "sqlite_vector_b200", "lib", "libvsb200.so")


def _stream(rng, n, kind):
    """distances with heavy ties, +-INF, NaN and +-0 mixed in"""
    if kind == "ties":
        d = rng.integers(0, 7, n).astype(np.float32)
    elif kind == "falling":                                  # every row enters the slots
        d = np.arange(n, 0, -1).astype(np.float32) // 3
    else:
        d = rng.standard_normal(n).astype(np.float32)
    at = rng.random(n)
    d[at < 0.02] = np.inf
    d[(at >= 0.02) & (at < 0.03)] = -np.inf
    d[(at >= 0.03) & (at < 0.04)] = np.nan
    d[(at >= 0.04) & (at < 0.06)] = 0.0
    d[(at >= 0.06) & (at < 0.08)] = -0.0
    d[(at >= 0.08) & (at < 0.09)] = np.float32(1e-7)
    # the slots see distances after the scan's nearly-zero clamp (-0 and tiny values become +0), as the oracle applies it
    d[np.abs(d) <= 8 * np.finfo(np.float32).eps] = 0.0
    return d


def _cands(d, ids):
    import sqlite_vector_b200 as vs
    c = np.zeros(len(d), dtype=vs.api.CAND_DTYPE)
    c["dist"], c["rowid"], c["seq"] = d, ids, np.arange(len(d))
    return c


SMALL = [(257, 3000), (300, 301), (1000, 20_000), (4096, 4000), (5000, 30_000)]
# the exchange sort is O(k^2) on both sides (and the oracle's argmax O(k) per entry): one stream each for the largest k
CASES = [(k, n, kind) for k, n in SMALL for kind in ("ties", "falling", "normal")] + [(16_384, 20_000, "normal"), (65_536, 66_000, "ties")]


@pytest.mark.parametrize("k, n, kind", CASES)
def test_replay_equals_the_reference_slots(k, n, kind):
    import sqlite_vector_b200 as vs
    eng = vs.load_engine()
    oracle = po.Oracle()
    rng = np.random.Generator(np.random.PCG64(k + n + len(kind)))
    d = _stream(rng, n, kind)
    ids = rng.permutation(4 * n)[:n].astype(np.int64) + 1
    c = _cands(d, ids)
    starts = (0, 1, k // 2, k - 1) if k <= 5000 else (k - 1,)
    for mi in starts:
        got_ids, got_d, got_mi = eng.replay_topk(c, k, max_index=mi)
        want_ids, want_d = oracle.topk_from_distances(d, ids, k, start_max_index=mi)
        assert np.array_equal(got_ids, want_ids), (k, n, kind, mi)
        assert np.array_equal(got_d.view(np.uint64), np.asarray(want_d, np.float64).view(np.uint64)), (k, n, kind, mi)
        assert 0 <= got_mi < k


def test_replay_keeps_the_cursor_across_calls():
    """the max_index a call leaves is where the next one starts, as for a reference cursor that is never reset"""
    import sqlite_vector_b200 as vs
    eng = vs.load_engine()
    oracle = po.Oracle()
    rng = np.random.Generator(np.random.PCG64(7))
    mi = 0
    for k in (300, 1000, 257, 2000):
        d = _stream(rng, 5000, "ties")
        ids = np.arange(1, 5001, dtype=np.int64)
        got_ids, got_d, new_mi = eng.replay_topk(_cands(d, ids), k, max_index=mi)
        want_ids, want_d = oracle.topk_from_distances(d, ids, k, start_max_index=mi)
        assert np.array_equal(got_ids, want_ids) and np.array_equal(got_d, want_d), (k, mi)
        mi = new_mi


def test_large_k_kernels_spill_nothing_and_fit_their_blocks():
    """lk_hist / lk_count / lk_write (256 threads), lk_select (one warp per segment, 1024 threads) and lk_offsets (1024 threads):
    no local memory, registers for the planned block on one SM"""
    if not shutil.which("cuobjdump"):
        pytest.skip("no cuobjdump here")
    res = subprocess.run(["cuobjdump", "-res-usage", LIB], capture_output=True, text=True, check=True, timeout=300).stdout
    parts = re.split(r"Function (\S+):", res)
    names = parts[1::2]
    dem = subprocess.run(["c++filt"], input="\n".join(names), capture_output=True, text=True, check=True).stdout.splitlines()
    threads = {"lk_hist_kernel": 256, "lk_select_kernel": 1024, "lk_count_kernel": 256, "lk_offsets_kernel": 1024, "lk_write_kernel": 256}
    seen = {k: 0 for k in threads}
    for d, body in zip(dem, parts[2::2]):
        kind = next((k for k in threads if re.search(r"\b%s\b" % k, d)), None)
        if kind is None:
            continue
        seen[kind] += 1
        regs, local = int(re.search(r"REG:(\d+)", body).group(1)), int(re.search(r"LOCAL:(\d+)", body).group(1))
        per_warp = -(-regs * 32 // 256) * 256
        assert local == 0 and per_warp * (threads[kind] // 32) <= 65536, (d, regs, local)
        if kind == "lk_hist_kernel":                          # 32 segments x 256 bins of shared histogram, under the 48 KB static limit
            assert int(re.search(r"SHARED:(\d+)", body).group(1)) <= 48 * 1024, body
    assert seen == {k: 1 for k in threads}, seen
