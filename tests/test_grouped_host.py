"""Grouped top-k (vsb_scan_topk_grouped) without a GPU: its kernels keep no local memory and fit their blocks, the SQL
modules check their arguments before they touch a device, and the host restatement of its kernels (tests/groupedref.py) holds
on hand-worked cases and against a position-by-position walk."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from tests import groupedref as gr

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


# ------------------------------------------------------------------------------------------------ the host restatement
def _walk_one_by_one(d, k):
    """the walk of one piece, position by position: log when d < the running k-th value of the logged values (+INF until k)"""
    lst, pd = [], []
    for v in d:
        thr = sorted(lst)[k - 1] if len(lst) >= k else np.float32(np.inf)
        if v < thr:
            lst.append(v)
            pd.append(v)
        else:
            pd.append(np.float32(np.nan))
    return np.array(pd, np.float32), np.array((sorted(lst) + [np.inf] * k)[:k], np.float32)


def test_groupedref_hand_worked_walk():
    nan, inf = np.nan, np.inf
    lay = gr.layout([np.arange(6)])
    pd, lists = gr.walk(np.array([5, 3, 4, 1, 2, 6], np.float32), lay, 2)
    assert gr.same(pd, np.array([5, 3, 4, 1, 2, nan], np.float32)) and gr.same(lists, np.array([[1, 2]], np.float32))
    bound, kmin = gr.bounds(lists, lay, 2)
    assert gr.same(bound, np.array([inf], np.float32)) and gr.same(kmin, np.array([1], np.float32))
    assert gr.survivors(pd, bound, lay).tolist() == [[np.float32(v).view(np.uint32), p] for p, v in enumerate([5, 3, 4, 1, 2])]
    # NaN and +INF never log; ties with the running k-th value do not log; once k -INF are kept nothing logs
    d = np.array([nan, inf, 7, inf, nan, 7, 7, -inf, -inf, -5], np.float32)
    pd, lists = gr.walk(d, gr.layout([np.arange(10)]), 2)
    assert gr.same(pd, np.array([nan, nan, 7, nan, nan, 7, nan, -inf, -inf, nan], np.float32))
    assert gr.same(lists, np.array([[-inf, -inf]], np.float32))
    # a key shorter than k: its list is +INF padded and every finite value logs
    pd, lists = gr.walk(np.array([2, nan, 1], np.float32), gr.layout([[0, 1, 2]]), 5)
    assert gr.same(pd, np.array([2, nan, 1], np.float32)) and gr.same(lists, np.array([[1, 2, inf, inf, inf]], np.float32))


def test_groupedref_hand_worked_pieces_and_limit():
    inf = np.inf
    lay = gr.layout([[], np.arange(1030)[::-1], [7, 7, 3]])          # unsorted and duplicate rows: sorted, made unique
    assert lay["koff"].tolist() == [0, 0, 1030, 1032] and lay["pstart"].tolist() == [0, 1024, 1030, 1032]
    assert lay["pkey"].tolist() == [1, 1, 2] and lay["kpiece"].tolist() == [0, 0, 2, 3]
    assert lay["rows"][:3].tolist() == [0, 1, 2] and lay["rows"][-2:].tolist() == [3, 7]
    d = np.arange(1030, dtype=np.float32)                             # ascending: only the first k of each piece log
    pd, lists = gr.walk(d, lay, 3)
    assert np.flatnonzero(~np.isnan(pd)).tolist() == [0, 1, 2, 1024, 1025, 1026, 1030, 1031]
    bound, kmin = gr.bounds(lists, lay, 3)
    assert gr.same(bound, np.array([inf, 2, inf], np.float32)) and gr.same(kmin, np.array([inf, 0, 3], np.float32))
    assert gr.survivors(pd, bound, lay)[:, 1].tolist() == [0, 1, 2, 1030, 1031]    # piece 1's rows are not below 2
    assert gr.survivors(pd, bound, lay, np.array([0, 0, 1], np.uint8))[:, 1].tolist() == [1030, 1031]
    assert gr.shard_rows([[10, 11, 99], [12]], gr.RowMap([10, 3, 3, 3, 3, 11, 12]), 4, 7)[0].tolist() == [1]
    # the limit: the minimum over shards, the limit-th smallest as the bound, ties included
    kmins = [np.array([1, inf, 3, 2], np.float32), np.array([inf, 0.5, 3, inf], np.float32)]
    assert gr.limit_select(kmins, 2)[1].tolist() == [1, 1, 0, 0]
    assert gr.limit_select(kmins, 4)[1] is None and gr.limit_select(kmins, 0)[1] is None
    assert gr.limit_select([np.array([1, 1, 1, 2, inf], np.float32)], 1)[1].tolist() == [1, 1, 1, 0, 0]
    # signed zeros: bit for bit, or by value where the model leaves the sign open
    assert not gr.same(np.float32([-0.0]), np.float32([0.0])) and gr.same(np.float32([-0.0]), np.float32([0.0]), True)


def test_groupedref_walk_equals_one_by_one():
    rng = np.random.Generator(np.random.PCG64(71_000))
    for trial in range(12):
        lens = rng.integers(0, 2600, int(rng.integers(1, 6)))
        keys, at = [], 0
        for n in lens:
            keys.append(np.arange(at, at + n))
            at += n
        vals = np.array([0.0, -0.0, 1.0, 2.0, np.nan, np.inf, -np.inf], np.float32)
        d = rng.choice(vals, at) if trial % 2 else rng.standard_normal(at).astype(np.float32)
        for k in (1, 2, 31, 33, 256):
            lay = gr.layout(keys)
            pd, lists = gr.walk(d, lay, k)
            ps = lay["pstart"].astype(np.int64)
            for pc in range(len(ps) - 1):
                wpd, wl = _walk_one_by_one(d[lay["rows"][ps[pc]:ps[pc + 1]]], k)
                assert gr.same(pd[ps[pc]:ps[pc + 1]], wpd) and gr.same(lists[pc], wl, True), (trial, k, pc)
