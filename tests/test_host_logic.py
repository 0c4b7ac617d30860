"""CPU-only checks of the host side: C-ABI exports, loud failure without a GPU, slot replay, shard merge (gloo)."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest

from oracle import pyoracle as po
from tests.test_result_head import HEAD_BYTES, make_head

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    hdr = open(os.path.join(ROOT, "include", "vsb200.h")).read()
    return sorted(set(re.findall(r"VSB_API[^;(]*?\b(vsb_\w+)\s*\(", hdr)))


@pytest.mark.parametrize("lib", ["libvsb200.so", "vector.so"])
def test_library_exports_every_declared_symbol(lib):
    path = os.path.join(ROOT, "sqlite_vector_b200", "lib", lib)
    if lib == "vector.so" and not os.path.exists(path):
        pytest.skip("extension not built yet")
    out = subprocess.run(["nm", "-D", "--defined-only", path], capture_output=True, text=True, check=True).stdout
    exported = set(re.findall(r"\bT (\w+)", out))
    syms = declared_symbols()
    assert len(syms) >= 20
    missing = [s for s in syms if s not in exported]
    assert not missing, missing
    if lib == "vector.so":
        assert "sqlite3_vector_init" in exported


def test_python_mirror_matches_header():
    from sqlite_vector_b200 import api
    assert sorted(api._SIGNATURES) == declared_symbols()
    api.load_engine()  # binds every symbol; AttributeError if one is missing


def test_no_cpu_fallback():
    import sqlite_vector_b200 as vs
    eng = vs.load_engine()
    if eng.device_count() > 0:
        pytest.skip("a GPU is present")
    with pytest.raises(vs.VsbError, match="no CUDA device"):
        vs.Index(vs.api.I8, 16, 10)


def test_product_never_imports_oracle():
    for dp, _, files in os.walk(os.path.join(ROOT, "sqlite_vector_b200")):
        for f in files:
            if f.endswith((".py", ".c", ".cu", ".cuh", ".h")):
                src = open(os.path.join(dp, f), errors="ignore").read()
                assert "pyoracle" not in src and "vs_oracle" not in src and "libvs_oracle" not in src, f


def test_replay_matches_oracle_slots(oracle):
    """vsb_replay_topk (product, host) == the oracle's slot algorithm on arbitrary (distance,id) streams with ties."""
    import sqlite_vector_b200 as vs
    from sqlite_vector_b200 import api
    eng = vs.load_engine()
    rng = np.random.Generator(np.random.PCG64(3))
    for n, k, levels in [(500, 20, 4), (50, 100, 3), (2000, 7, 2), (300, 33, 50), (0, 5, 2), (5, 5, 1)]:
        d = rng.integers(0, levels, n).astype(np.float32)
        if n > 10:
            d[rng.integers(0, n, 3)] = np.inf
            d[rng.integers(0, n, 3)] = np.nan
            d[rng.integers(0, n, 2)] = 5e-7     # below the nearly-zero clamp? (the clamp is applied by the kernels, not by replay)
        ids = rng.permutation(n).astype(np.int64) + 100
        c = np.zeros(n, dtype=api.CAND_DTYPE)
        c["rowid"], c["seq"], c["dist"] = ids, np.arange(n), d
        for smi in (0, min(k - 1, 2)):
            got_ids, got_d, _ = eng.replay_topk(c, k, smi)
            # oracle.topk_from_distances clamps tiny values; feed it pre-clamped input so both see the same numbers
            dc = np.where(np.abs(d) <= 8 * np.finfo(np.float32).eps, 0, d).astype(np.float32)
            c2 = c.copy(); c2["dist"] = dc
            got_ids, got_d, _ = eng.replay_topk(c2, k, smi)
            want_ids, want_d = oracle.topk_from_distances(dc, ids, k, smi)
            assert np.array_equal(got_ids, want_ids) and np.array_equal(got_d, want_d), (n, k, levels)


def test_shard_pack_roundtrip():
    from sqlite_vector_b200 import api, shard
    rng = np.random.Generator(np.random.PCG64(1))
    blocks, parts = [], []
    for r in range(3):
        c = np.zeros(int(rng.integers(0, 40)), dtype=api.CAND_DTYPE)
        c["rowid"] = rng.integers(0, 1 << 40, c.shape[0]); c["seq"] = np.arange(c.shape[0]) + 1000 * r
        c["dist"] = rng.standard_normal(c.shape[0])
        parts.append(c); blocks.append(shard.pack_candidates(c, 64))
    got = shard.unpack_candidates(np.concatenate(blocks), 3, 64)
    assert np.array_equal(got, np.concatenate(parts))
    assert shard.shard_bounds(10, 4) == [0, 2, 5, 7, 10]
    with pytest.raises(ValueError):
        shard.pack_candidates(np.zeros(65, dtype=api.CAND_DTYPE), 64)


WORKER = r'''
import os, sys
import numpy as np
import torch.distributed as dist
sys.path.insert(0, sys.argv[1])
import sqlite_vector_b200 as vs
from sqlite_vector_b200 import api, shard
from oracle import pyoracle as po
rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
dist.init_process_group("gloo")
rng = np.random.Generator(np.random.PCG64(99))
n, dim, k = 4001, 16, 20
x = rng.integers(-3, 4, (n, dim)).astype(np.int8)          # tiny value range => heavy ties
q = rng.integers(-3, 4, dim).astype(np.int8)
rowids = np.arange(n, dtype=np.int64) * 5 + 3
b = shard.shard_bounds(n, world)
lo, hi = b[rank], b[rank + 1]
# stand-in for the GPU shard scan (no device here): every local row is a candidate, distances in exact integer math
diff = x[lo:hi].astype(np.int32) - q.astype(np.int32)
d = np.sqrt((diff * diff).sum(1).astype(np.float32))
c = np.zeros(hi - lo, dtype=api.CAND_DTYPE)
c["rowid"], c["seq"], c["dist"] = rowids[lo:hi], np.arange(lo, hi), d
ids, dd, _ = shard.sharded_topk(vs.load_engine(), c, k, cap=4096)
want_ids, want_d = po.Oracle().scan_dense(po.L2, po.I8, q, x, rowids, k)
assert np.array_equal(ids, want_ids) and np.array_equal(dd, want_d), (rank, ids, want_ids)
dist.barrier()
if rank == 0: print("SHARD_OK")
dist.destroy_process_group()
'''


def test_sharded_merge_gloo_world2(tmp_path):
    script = tmp_path / "worker.py"
    script.write_text(WORKER)
    env = dict(os.environ, MASTER_ADDR="127.0.0.1")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
                        "--master-port", "29613", str(script), ROOT], capture_output=True, text=True, timeout=300, env=env)
    assert r.returncode == 0 and "SHARD_OK" in r.stdout, r.stdout + r.stderr


QWORKER = r'''
import os, sys
import numpy as np
import torch.distributed as dist
sys.path.insert(0, sys.argv[1])
from sqlite_vector_b200 import shard
from oracle import pyoracle as po
rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
dist.init_process_group("gloo")
rng = np.random.Generator(np.random.PCG64(5))
n, dim, k, nq = 700, 12, 7, 11                                  # 11 queries over 2 ranks: ragged slices (5 + 6)
x = rng.integers(-3, 4, (n, dim)).astype(np.int8)
qs = rng.integers(-3, 4, (nq, dim)).astype(np.int8)
rowids = np.arange(n, dtype=np.int64) * 3 + 1
orc = po.Oracle()
class Replica:                                                   # stand-in for the full index on this rank's GPU (no device here)
    calls = 0
    def scan_topk(self, metric, q, kk, as_arrays=False):
        Replica.calls += q.shape[0]
        ids, dd, cnt = np.zeros((q.shape[0], kk), np.int64), np.zeros((q.shape[0], kk)), np.zeros(q.shape[0], np.int32)
        for i in range(q.shape[0]):
            ri, rd = orc.scan_dense(metric, po.I8, q[i], x, rowids, kk)
            cnt[i] = len(ri); ids[i, :cnt[i]] = ri; dd[i, :cnt[i]] = rd
        return ids, dd, cnt
ids, d, cnt = shard.query_sharded_batch_topk(Replica(), po.L2, qs, k)
b = shard.query_split(nq, world)
assert Replica.calls == b[rank + 1] - b[rank]
for i in range(nq):
    wi, wd = orc.scan_dense(po.L2, po.I8, qs[i], x, rowids, k)
    assert cnt[i] == len(wi) and np.array_equal(ids[i, :cnt[i]], wi) and np.array_equal(d[i, :cnt[i]], wd), (rank, i)
(li, ld, lc), (lo, hi) = shard.query_sharded_batch_topk(Replica(), po.L2, qs, k, gather=False)
assert (lo, hi) == (b[rank], b[rank + 1]) and np.array_equal(li, ids[lo:hi]) and np.array_equal(ld, d[lo:hi])
# fewer queries than ranks: the empty slice takes part in the gather without touching its replica
calls0 = Replica.calls
i1, d1, c1 = shard.query_sharded_batch_topk(Replica(), po.DOT, qs[:1], 3)
assert i1.shape == (1, 3) and Replica.calls - calls0 == (1 if rank == world - 1 else 0)
wi, wd = orc.scan_dense(po.DOT, po.I8, qs[0], x, rowids, 3)
assert np.array_equal(i1[0, :c1[0]], wi) and np.array_equal(d1[0, :c1[0]], wd)
assert shard.query_split(1, 2) == [0, 0, 1] and shard.query_split(10, 4) == [0, 2, 5, 7, 10]
dist.barrier()
if rank == 0: print("QSHARD_OK")
dist.destroy_process_group()
'''


def test_query_sharded_batch_gloo_world2(tmp_path):
    """replicas + query split: every rank answers its slice, one all-gather gives every rank all results"""
    script = tmp_path / "qworker.py"
    script.write_text(QWORKER)
    env = dict(os.environ, MASTER_ADDR="127.0.0.1")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
                        "--master-port", "29614", str(script), ROOT], capture_output=True, text=True, timeout=300, env=env)
    assert r.returncode == 0 and "QSHARD_OK" in r.stdout, r.stdout + r.stderr


def test_merge_result_blocks_matches_oracle(oracle):
    """vsb_merge_result_blocks (host) over hand-built shard result blocks == the oracle's scan of the whole column"""
    import sqlite_vector_b200 as vs
    eng = vs.load_engine()
    rng = np.random.Generator(np.random.PCG64(17))
    n, dim, k, world = 1500, 8, 20, 3
    x = rng.integers(-3, 4, (n, dim)).astype(np.int8)
    q = rng.integers(-3, 4, dim).astype(np.int8)
    bounds = [0, 400, 1100, n]
    heads = []
    for r in range(world):
        lo, hi = bounds[r], bounds[r + 1]
        diff = x[lo:hi].astype(np.int32) - q.astype(np.int32)
        d = np.sqrt((diff * diff).sum(1).astype(np.float32))
        half = (hi - lo) // 2
        heads.append(make_head(d, [(0, half), (half, hi - lo - half)]))   # two "filter blocks", contiguous in scan order
    ids, dist = eng.merge_result_blocks(np.concatenate(heads), world, HEAD_BYTES, np.array(bounds[:world]), k)
    want_ids, want_d = oracle.scan_dense(po.L2, po.I8, q, x, np.arange(1, n + 1, dtype=np.int64), k)
    assert np.array_equal(ids, want_ids) and np.array_equal(dist, want_d)


def test_merge_result_groups_matches_oracle(oracle):
    """vsb_merge_result_groups (host): a gathered GROUP of queries, rank-major like the NCCL all-gather lays it out
    (rank r's blocks of queries 0..G-1, then rank r+1's) == the oracle's scan of the whole column for every query"""
    import sqlite_vector_b200 as vs
    eng = vs.load_engine()
    rng = np.random.Generator(np.random.PCG64(23))
    n, dim, k, world, G = 900, 8, 20, 3, 4
    x = rng.integers(-3, 4, (n, dim)).astype(np.int8)
    qs = rng.integers(-3, 4, (G, dim)).astype(np.int8)
    bounds = [0, 250, 610, n]
    heads = []
    for r in range(world):
        lo, hi = bounds[r], bounds[r + 1]
        for j in range(G):
            diff = x[lo:hi].astype(np.int32) - qs[j].astype(np.int32)
            d = np.sqrt((diff * diff).sum(1).astype(np.float32))
            heads.append(make_head(d, [(0, hi - lo)]))
    res = eng.merge_result_groups(np.concatenate(heads), world, G * HEAD_BYTES, HEAD_BYTES, G, np.array(bounds[:world]), k)
    assert len(res) == G
    for j in range(G):
        want_ids, want_d = oracle.scan_dense(po.L2, po.I8, qs[j], x, np.arange(1, n + 1, dtype=np.int64), k)
        assert np.array_equal(res[j][0], want_ids) and np.array_equal(res[j][1], want_d), j


def test_built_kernels_use_wgmma_and_tma_not_mma_sync():
    """the library that travels to the GPU box: tensor-core kernels are Hopper warpgroup MMAs (HGMMA / IGMMA) fed by TMA tensor
    loads, the scan kernels use TMA bulk copies, nothing falls back to mma.sync (tools/sass_evidence.py over cuobjdump -sass)"""
    import shutil
    if not shutil.which("cuobjdump"):
        pytest.skip("no cuobjdump here")
    import json
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "sass_evidence.py")], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    ev = json.loads(r.stdout)
    ks = ev["kernels"]
    tc = [k for k in ks if "tc_scan_kernel" in k]
    assert len(tc) >= 24 and all(("IGMMA" in ks[k] or "HGMMA" in ks[k]) and "UTMALDG" in ks[k] and "WARPGROUP" in ks[k] for k in tc), tc
    staged = [k for k in ks if "scan_kernel<" in k and "tc_" not in k and k.rstrip(">").endswith("false")]
    assert len(staged) == 20 and all("UBLKCP" in ks[k] for k in staged), staged
    assert not ev["mma_sync_anywhere"]
    assert all("tc_scan_kernel" not in k and "scan_kernel<" not in k for k in ev["local_memory_spills"]), ev["local_memory_spills"]
