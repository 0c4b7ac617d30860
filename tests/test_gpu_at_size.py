"""BASELINE.json configs at (or near) their stated shapes, CUDA path vs the oracle.  -m gpu.

  C3  vector_full_scan dot bf16 dim=768 k=20 batch=1024 (tensor-core path), n = 1M rows here (10M in the bench, where the
      same check runs on a query sample against the same oracle)
  C4  vector_quantize_scan cosine uint8 dim=1536 k=100 batch=256, row-sharded: n = 1M rows in 3 shards on this GPU
      (the 8-GPU run has 6.25M rows per shard; the exchange itself is covered by tests/test_gpu_multi.py)
  C5  all 5 metrics x 5 dtypes, dim in {128, 384, 768, 1536}, n = 1M, batch 1: recall@20 and distance tolerance

Inputs are generated on the GPU with torch (plumbing: numpy would take minutes for 1.5e9 normals), brought to the host for
the oracle, and appended to the index from device memory.  The oracle's C loops run on a thread pool (ctypes drops the GIL)."""
import os
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

from oracle import pyoracle as po
from tests.fpcheck import assert_fp_topk

pytestmark = pytest.mark.gpu
METRICS = [po.L2, po.L2SQ, po.COS, po.DOT, po.L1]
THREADS = max(4, min(64, (os.cpu_count() or 8)))


def _gen(n, dim, seed):
    import torch
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn((n, dim), generator=g, device="cuda", dtype=torch.float32)


def _to_type(xf, vtype):
    """torch f32 (cuda) -> storage of `vtype` (cuda tensor); same rules as oracle.pyoracle.convert"""
    import torch
    if vtype == po.F32:
        return xf
    if vtype == po.F16:
        return xf.to(torch.float16)
    if vtype == po.BF16:
        return xf.to(torch.bfloat16)
    if vtype == po.I8:
        return (xf * 24.0).round().clamp_(-128, 127).to(torch.int8)
    return (xf.abs() * 48.0).round().clamp_(0, 255).to(torch.uint8)


def _host(t, vtype):
    import torch
    if vtype in (po.F16, po.BF16):
        return t.view(torch.int16).cpu().numpy().view(np.uint16)
    return t.cpu().numpy()


def _index_from_device(vtype, t, first_seq=0):
    import torch

    import sqlite_vector_b200 as vs
    ix = vs.Index(vtype, t.shape[1], t.shape[0], first_seq=first_seq)
    torch.cuda.synchronize()
    ix.append_device(t.data_ptr(), t.shape[0])
    ix.finalize()
    return ix


def test_convert_rules_match_pyoracle():
    xf = _gen(1000, 64, 5)
    xh = xf.cpu().numpy()
    for vt in (po.F16, po.BF16, po.I8, po.U8):
        assert np.array_equal(_host(_to_type(xf, vt), vt), po.convert(xh, vt)), vt


@pytest.mark.parametrize("dim", [128, 384, 768, 1536])
def test_config5_at_size(oracle, dim):
    n, k = 1_000_000, 20
    xf, qf = _gen(n, dim, 1234), _gen(1, dim, 4321)
    rowids = np.arange(1, n + 1, dtype=np.int64)
    for vtype in (po.F32, po.F16, po.BF16, po.U8, po.I8):
        xt = _to_type(xf, vtype).contiguous()
        x, q = _host(xt, vtype), _host(_to_type(qf, vtype), vtype)[0]
        ix = _index_from_device(vtype, xt)
        del xt
        with ThreadPoolExecutor(len(METRICS)) as ex:
            wants = list(ex.map(lambda m: oracle.scan_dense(m, vtype, q, x, rowids, k), METRICS))
        for metric, (want_ids, want_d) in zip(METRICS, wants):
            (res,) = ix.scan_topk(metric, q, k)
            if vtype in (po.U8, po.I8):
                assert np.array_equal(res[0], want_ids) and np.array_equal(res[1], want_d), (vtype, metric, dim)
            else:
                assert_fp_topk(res[0], res[1], want_ids, want_d, metric, lambda r: oracle.distance(metric, vtype, q, x[r - 1]), (vtype, metric, dim))
                assert len(set(res[0].tolist()) & set(want_ids.tolist())) / k >= 0.95         # recall@20
        ix.close()


def test_config3_shape_bf16_dot_batch1024(oracle):
    """bf16 DOT dim 768 k=20 B=1024 on 1M rows: the batch (wgmma) result of every query against the oracle for a sample of
    128 queries, and against the single-query CUDA-core path for all 1024"""
    import sqlite_vector_b200 as vs
    n, dim, nq, k = 1_000_000, 768, 1024, 20
    xt = _to_type(_gen(n, dim, 7000), po.BF16).contiguous()
    x, q = _host(xt, po.BF16), _host(_to_type(_gen(nq, dim, 4322), po.BF16), po.BF16)
    ix = _index_from_device(po.BF16, xt)
    del xt
    b0 = ix.stat("batches")
    res = ix.scan_topk(po.DOT, q, k)
    assert ix.stat("batches") == b0 + 1, "the tensor-core batch path did not run"
    rowids = np.arange(1, n + 1, dtype=np.int64)
    sample = list(range(0, nq, 8))
    with ThreadPoolExecutor(THREADS) as ex:
        wants = list(ex.map(lambda b: oracle.scan_dense(po.DOT, po.BF16, q[b], x, rowids, k), sample))
    for b, (want_ids, want_d) in zip(sample, wants):
        assert_fp_topk(res[b][0], res[b][1], want_ids, want_d, po.DOT, lambda r, b=b: oracle.distance(po.DOT, po.BF16, q[b], x[r - 1]), ("c3", b))
    eng = vs.load_engine()
    eng.set_option("no_batch", 1)
    try:
        for b in range(nq):
            (one,) = ix.scan_topk(po.DOT, q[b], k)
            assert_fp_topk(res[b][0], res[b][1], one[0], one[1], po.DOT, lambda r, b=b: oracle.distance(po.DOT, po.BF16, q[b], x[r - 1]), ("c3-single", b))
    finally:
        eng.set_option("no_batch", 0)
    ix.close()


def test_config4_shape_u8_cosine_k100_batch256_sharded(oracle):
    """uint8 COSINE dim 1536 k=100 B=256 over 3 row shards (the config-4 pipeline: per-shard tensor-core levels with entry
    logs, gathered blocks, GPU merge replay) == the oracle's single scan, bit for bit, for every query"""
    import torch

    from sqlite_vector_b200.shard import _DevView
    n, dim, nq, k = 1_000_000, 1536, 256, 100
    xt = _to_type(_gen(n, dim, 1234), po.U8).contiguous()
    x, q = _host(xt, po.U8), _host(_to_type(_gen(nq, dim, 4321), po.U8), po.U8)
    bounds = [0, 333_333, 700_001, n]
    shards = [_index_from_device(po.U8, xt[a:b], first_seq=a) for a, b in zip(bounds[:-1], bounds[1:])]
    del xt
    parts = []
    for ix in shards:
        ptr, nbytes = ix.batch_shard_scan(po.COS, q, k)
        parts.append(torch.as_tensor(_DevView(ptr, nbytes), device="cuda").clone())
    gathered = torch.cat(parts)
    torch.cuda.synchronize()
    seq, d, counts = shards[0].batch_merge(gathered.data_ptr(), len(shards), nbytes, np.asarray(bounds[:-1], dtype=np.int64), nq, k)
    rowids = np.arange(1, n + 1, dtype=np.int64)
    with ThreadPoolExecutor(THREADS) as ex:
        wants = list(ex.map(lambda b: oracle.scan_dense(po.COS, po.U8, q[b], x, rowids, k), range(nq)))
    for b, (want_ids, want_d) in enumerate(wants):
        assert counts[b] == k
        assert np.array_equal(seq[b] + 1, want_ids) and np.array_equal(d[b], want_d), ("c4", b)
    for ix in shards:
        ix.close()
