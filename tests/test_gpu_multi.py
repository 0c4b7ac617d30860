"""Row-sharded scans on >= 2 GPUs, one process per GPU over NCCL (torchrun): the grouped device exchange of the
single-query path and the sharded tensor-core batch path, both against a whole-column index on rank 0's GPU and
against the oracle.  Skipped on a 1-GPU box.  -m gpu."""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

WORKER = r'''
import os, sys
import numpy as np
import torch, torch.distributed as dist
sys.path.insert(0, sys.argv[1])
import sqlite_vector_b200 as vs
from sqlite_vector_b200 import api, shard
from oracle import pyoracle as po
rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
local = int(os.environ.get("LOCAL_RANK", rank))
torch.cuda.set_device(local)
device = torch.device("cuda", local)
dist.init_process_group("nccl", device_id=device)
eng = vs.load_engine()
rng = np.random.Generator(np.random.PCG64(4242))
n, dim, k = 300_000, 128, 20
x = rng.integers(-6, 7, (n, dim)).astype(np.int8)            # small value range => ties at the k-th place
nq = 37
q = rng.integers(-6, 7, (nq, dim)).astype(np.int8)
bounds = shard.shard_bounds(n, world)
lo, hi = bounds[rank], bounds[rank + 1]
ix = vs.Index(api.I8, dim, hi - lo, device=local, first_seq=lo)
ix.append_dense(x[lo:hi])
ix.finalize()
orc = po.Oracle()
rowids = np.arange(1, n + 1, dtype=np.int64)

# ---- single queries through the grouped, pipelined device exchange (host queries and device queries)
pitch = ix.query_pitch
qd = torch.zeros((nq, pitch), dtype=torch.uint8, device=device)
qd[:, :dim] = torch.from_numpy(q.view(np.uint8)).to(device)
torch.cuda.synchronize()
for group in (1, 3, 8):
    exch = shard.DeviceExchange(ix, eng, world, bounds, device, group=group)
    for on_device in (True, False):
        results, pending = [], None
        for g0 in range(0, nq, exch.group):
            idx = range(g0, min(nq, g0 + exch.group))
            if group == 3:      # list form
                qs = [qd[i].data_ptr() for i in idx] if on_device else [q[i] for i in idx]
                t = exch.submit(api.L2, qs, k, on_device=on_device)
            elif on_device:     # strided form: one engine call per group
                t = exch.submit_strided(api.L2, qd[g0].data_ptr(), pitch, len(idx), k, True)
            else:
                t = exch.submit_strided(api.L2, q[g0:g0 + len(idx)], q.strides[0], len(idx), k, False)
            if pending is not None:
                results += exch.finish(pending)
            pending = t
        results += exch.finish(pending)
        assert len(results) == nq
        for b in range(nq):
            want_ids, want_d = orc.scan_dense(po.L2, po.I8, q[b], x, rowids, k)
            assert np.array_equal(results[b][0], want_ids) and np.array_equal(results[b][1], want_d), (rank, group, on_device, b)

# ---- batched queries: tensor-core levels per shard, all-gather of the entry logs, GPU merge
for metric in (api.L2, api.COSINE, api.DOT):
    res = shard.sharded_batch_topk(ix, metric, q, k, bounds, device)
    assert res is not None, "the sharded batch path refused"
    for b in range(nq):
        want_ids, want_d = orc.scan_dense(metric, po.I8, q[b], x, rowids, k)
        assert np.array_equal(res[b][0], want_ids) and np.array_equal(res[b][1], want_d), (rank, metric, b)
# explicit rowids travel through lookup + all-reduce
ix2 = vs.Index(api.I8, dim, hi - lo, device=local, first_seq=lo)
rid = np.arange(n, dtype=np.int64) * 7 + 3
ix2.append_dense(x[lo:hi], rid[lo:hi])
ix2.finalize()
res = shard.sharded_batch_topk(ix2, api.L2, q, k, bounds, device, implicit_rowids=False)
for b in range(nq):
    want_ids, want_d = orc.scan_dense(po.L2, po.I8, q[b], x, rid, k)
    assert np.array_equal(res[b][0], want_ids) and np.array_equal(res[b][1], want_d), (rank, b)
# a shard that cannot take the batch path (f32 column) makes every rank fall back together
ixf = vs.Index(api.F32, 16, 1000, device=local, first_seq=rank * 1000)
ixf.append_dense(np.zeros((1000, 16), dtype=np.float32)); ixf.finalize()
assert shard.sharded_batch_topk(ixf, api.L2, np.zeros((32, 16), dtype=np.float32), 5, [r * 1000 for r in range(world + 1)], device) is None
dist.barrier()
if rank == 0: print("MULTI_GPU_OK")
dist.destroy_process_group()
'''


def test_sharded_paths_nccl(tmp_path):
    import torch
    ngpu = torch.cuda.device_count()
    if ngpu < 2:
        pytest.skip("needs >= 2 GPUs")
    world = 2 if ngpu < 4 else 4
    script = tmp_path / "worker.py"
    script.write_text(WORKER)
    env = dict(os.environ, MASTER_ADDR="127.0.0.1")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr", "127.0.0.1",
                        "--master-port", "29633", str(script), ROOT], capture_output=True, text=True, timeout=900, env=env)
    assert r.returncode == 0 and "MULTI_GPU_OK" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]
