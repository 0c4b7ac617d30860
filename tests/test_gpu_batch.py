"""Batched queries (wgmma tensor-core path) vs the oracle and vs the per-query CUDA-core path.  -m gpu."""
import numpy as np
import pytest

from oracle import pyoracle as po

pytestmark = pytest.mark.gpu
METRICS = [po.L2, po.L2SQ, po.COS, po.DOT]


def _index(vtype, x, rowids=None):
    import sqlite_vector_b200 as vs
    ix = vs.Index(vtype, x.shape[1], x.shape[0])
    ix.append_dense(x, rowids)
    ix.finalize()
    return ix


@pytest.mark.parametrize("epi_chunk", [1, 0])
@pytest.mark.parametrize("vtype", [po.I8, po.U8])
@pytest.mark.parametrize("metric", METRICS)
def test_batch_int_bit_exact(oracle, vtype, metric, epi_chunk):
    """epi_chunk = 1 (default): the epilogue tests 32-column chunks (max score vs the chunk's weakest bound) before any
    per-column work; 0: every score against its own bound.  Same candidate log, same results."""
    import sqlite_vector_b200 as vs
    eng = vs.load_engine()
    old_chunk = eng.set_option("epi_chunk", epi_chunk)
    try:
        _batch_int_bit_exact(oracle, eng, vtype, metric)
    finally:
        eng.set_option("epi_chunk", old_chunk)


def test_batch_chunk_test_with_very_different_query_norms(oracle):
    """queries whose bounds differ by orders of magnitude inside one 32-column chunk: the chunk test degrades to the
    per-column test (it may never lose a hit)"""
    import sqlite_vector_b200 as vs
    rng = np.random.Generator(np.random.PCG64(99))
    n, dim, nq, k = 40000, 128, 64, 20
    x = rng.integers(-100, 101, (n, dim)).astype(np.int8)
    q = rng.integers(-100, 101, (nq, dim)).astype(np.int8)
    q[::3] //= 50                     # tiny norms next to full-range ones
    q[1::7] = 0                       # zero vectors
    ix = _index(po.I8, x)
    rowids = np.arange(1, n + 1, dtype=np.int64)
    for metric in METRICS:
        res = ix.scan_topk(metric, q, k)
        for b in range(nq):
            want_ids, want_d = oracle.scan_dense(metric, po.I8, q[b], x, rowids, k)
            assert np.array_equal(res[b][0], want_ids) and np.array_equal(res[b][1], want_d), (metric, b)
    ix.close()


def _batch_int_bit_exact(oracle, eng, vtype, metric):
    rng = np.random.Generator(np.random.PCG64(500 + 10 * vtype + metric))
    for (n, dim, nq, k) in [(20000, 128, 16, 20), (50000, 384, 100, 20), (30000, 200, 300, 33)]:
        x = po.convert(rng.standard_normal((n, dim), dtype=np.float32), vtype)
        q = po.convert(rng.standard_normal((nq, dim), dtype=np.float32), vtype)
        rowids = np.arange(n, dtype=np.int64) * 2 + 5
        ix = _index(vtype, x, rowids)
        b0 = ix.stat("batches")
        res = ix.scan_topk(metric, q, k)
        assert ix.stat("batches") == b0 + 1, "the tensor-core batch path did not run"
        for b in list(range(0, nq, max(1, nq // 7)))[:8] + [nq - 1]:
            want_ids, want_d = oracle.scan_dense(metric, vtype, q[b], x, rowids, k)
            assert np.array_equal(res[b][0], want_ids), (vtype, metric, n, dim, nq, b)
            assert np.array_equal(res[b][1], want_d)
        eng.set_option("no_batch", 1)
        try:
            loop = ix.scan_topk(metric, q, k)
        finally:
            eng.set_option("no_batch", 0)
        for b in range(nq):
            assert np.array_equal(res[b][0], loop[b][0]) and np.array_equal(res[b][1], loop[b][1]), (vtype, metric, b)
        ix.close()


@pytest.mark.parametrize("vtype", [po.BF16, po.F16])
@pytest.mark.parametrize("metric", METRICS)
def test_batch_fp_matches_oracle_every_query(oracle, vtype, metric):
    """north_star tolerance (1e-5 relative) against the ORACLE for every query of the batch; rowids identical except where
    the oracle's own distances tie with the k-th one (tests/fpcheck.py).  dim 1536 = 24 K-slices per tile exercises the
    dim-derived slack of the tensor-core bound (tc_fp_eps)."""
    from concurrent.futures import ThreadPoolExecutor

    from tests.fpcheck import assert_fp_topk
    rng = np.random.Generator(np.random.PCG64(700 + 10 * vtype + metric))
    for (n, dim, nq, k) in [(20000, 128, 32, 20), (40000, 768, 130, 20), (30000, 1536, 64, 100)]:
        x = po.convert(rng.standard_normal((n, dim), dtype=np.float32), vtype)
        q = po.convert(rng.standard_normal((nq, dim), dtype=np.float32), vtype)
        ix = _index(vtype, x)
        b0 = ix.stat("batches")
        res = ix.scan_topk(metric, q, k)
        assert ix.stat("batches") == b0 + 1, "the tensor-core batch path did not run"
        rowids = np.arange(1, n + 1, dtype=np.int64)
        with ThreadPoolExecutor(16) as ex:       # the oracle's C loop releases the GIL
            wants = list(ex.map(lambda b: oracle.scan_dense(metric, vtype, q[b], x, rowids, k), range(nq)))
        for b in range(nq):
            want_ids, want_d = wants[b]
            assert_fp_topk(res[b][0], res[b][1], want_ids, want_d, metric,
                           lambda r, b=b: oracle.distance(metric, vtype, q[b], x[r - 1]), (vtype, metric, n, dim, b))
        ix.close()


def _sharded_batch(indexes, bounds, metric, q, k):
    """the row-sharded batch path with the shards on ONE GPU: vsb_batch_shard_scan per shard, the blocks concatenated on
    the device (what the NCCL all-gather does across GPUs), vsb_batch_merge, rowid lookup summed over the shards"""
    import torch

    from sqlite_vector_b200.shard import _DevView
    world = len(indexes)
    parts = []
    for ix in indexes:
        ptr, nbytes = ix.batch_shard_scan(metric, q, k)
        parts.append(torch.as_tensor(_DevView(ptr, nbytes), device="cuda").clone())
    gathered = torch.cat(parts)
    torch.cuda.synchronize()
    seq, d, counts = indexes[-1].batch_merge(gathered.data_ptr(), world, nbytes, np.asarray(bounds[:world], dtype=np.int64), q.shape[0], k)
    ids = sum(ix.lookup_rowids(seq) for ix in indexes)
    return [(ids[b, :counts[b]], d[b, :counts[b]]) for b in range(q.shape[0])]


@pytest.mark.parametrize("vtype", [po.I8, po.U8])
@pytest.mark.parametrize("metric", METRICS)
def test_batch_row_sharded_bit_exact(oracle, vtype, metric):
    """BASELINE config 4 in miniature: batched queries over 3 row shards == one scan over the whole column (heavy ties)"""
    import sqlite_vector_b200 as vs
    rng = np.random.Generator(np.random.PCG64(900 + 10 * vtype + metric))
    for (n, dim, nq, k, lo_v, hi_v) in [(60000, 128, 40, 20, -3, 4), (45000, 256, 64, 100, -20, 21)]:
        if vtype == po.U8:
            lo_v, hi_v = 0, hi_v - lo_v
        dt = np.int8 if vtype == po.I8 else np.uint8
        x = rng.integers(lo_v, hi_v, (n, dim)).astype(dt)
        q = rng.integers(lo_v, hi_v, (nq, dim)).astype(dt)
        rowids = np.arange(n, dtype=np.int64) * 3 + 7
        bounds = [0, n // 4 + 11, (2 * n) // 3, n]
        shards = []
        for a, b in zip(bounds[:-1], bounds[1:]):
            ix = vs.Index(vtype, dim, b - a, first_seq=a)
            ix.append_dense(x[a:b], rowids[a:b])
            ix.finalize()
            shards.append(ix)
        res = _sharded_batch(shards, bounds, metric, q, k)
        whole = _index(vtype, x, rowids)
        one = whole.scan_topk(metric, q, k)
        for b in range(nq):
            assert np.array_equal(res[b][0], one[b][0]) and np.array_equal(res[b][1], one[b][1]), (vtype, metric, n, b)
        for b in (0, nq // 2, nq - 1):
            want_ids, want_d = oracle.scan_dense(metric, vtype, q[b], x, rowids, k)
            assert np.array_equal(res[b][0], want_ids) and np.array_equal(res[b][1], want_d), (vtype, metric, n, b)
        for ix in shards + [whole]:
            ix.close()


def test_batch_row_sharded_fp_equals_single_shard():
    import sqlite_vector_b200 as vs
    rng = np.random.Generator(np.random.PCG64(77))
    n, dim, nq, k = 50000, 768, 48, 20
    x = po.convert(rng.standard_normal((n, dim), dtype=np.float32), po.BF16)
    q = po.convert(rng.standard_normal((nq, dim), dtype=np.float32), po.BF16)
    bounds = [0, 20000, n]
    shards = []
    for a, b in zip(bounds[:-1], bounds[1:]):
        ix = vs.Index(po.BF16, dim, b - a, first_seq=a)
        ix.append_dense(x[a:b])
        ix.finalize()
        shards.append(ix)
    whole = _index(po.BF16, x)
    for metric in (po.DOT, po.COS, po.L2):
        res = _sharded_batch(shards, bounds, metric, q, k)
        one = whole.scan_topk(metric, q, k)
        for b in range(nq):      # same refine arithmetic, same replay: identical, not merely close
            assert np.array_equal(res[b][0], one[b][0]) and np.array_equal(res[b][1], one[b][1]), (metric, b)
    for ix in shards + [whole]:
        ix.close()


def test_batch_shard_scan_refuses_what_the_batch_path_cannot_do():
    import sqlite_vector_b200 as vs
    x = np.zeros((20000, 16), dtype=np.float32)
    ix = _index(po.F32, x)
    with pytest.raises(vs.VsbError, match="no tensor-core batch path"):
        ix.batch_shard_scan(po.L2, np.zeros((32, 16), dtype=np.float32), 5)
    ix.close()


@pytest.mark.parametrize("m0,growth", [(128, 4), (256, 8), (2048, 64)])
def test_batch_level_schedule_does_not_change_results(oracle, m0, growth):
    """the level schedule (exhaustive prefix, geometric growth) is a performance knob: results stay bit-exact"""
    import sqlite_vector_b200 as vs
    eng = vs.load_engine()
    rng = np.random.Generator(np.random.PCG64(31337))
    n, dim, nq, k = 70000, 128, 50, 20
    x = rng.integers(-8, 9, (n, dim)).astype(np.int8)
    q = rng.integers(-8, 9, (nq, dim)).astype(np.int8)
    ix = _index(po.I8, x)
    old = eng.set_option("batch_m0", m0), eng.set_option("batch_growth", growth)
    try:
        b0 = ix.stat("batches")
        res = ix.scan_topk(po.L2, q, k)
        assert ix.stat("batches") == b0 + 1
    finally:
        eng.set_option("batch_m0", old[0]); eng.set_option("batch_growth", old[1])
    rowids = np.arange(1, n + 1, dtype=np.int64)
    for b in range(nq):
        want_ids, want_d = oracle.scan_dense(po.L2, po.I8, q[b], x, rowids, k)
        assert np.array_equal(res[b][0], want_ids) and np.array_equal(res[b][1], want_d), (m0, growth, b)
    ix.close()


def test_batch_bucket_overflow_falls_back(oracle):
    """descending distances: every row enters the slots, the per-level buckets overflow, the call falls back to the
    per-query path and still returns the exact result"""
    import sqlite_vector_b200 as vs
    n, dim, nq, k = 40000, 128, 16, 5
    x = np.zeros((n, dim), dtype=np.int8)
    x[:, 0] = np.clip((n - 1 - np.arange(n)) // 320, 0, 124).astype(np.int8)      # distance to q shrinks along the scan
    x[:, 1] = ((n - 1 - np.arange(n)) % 320 // 3).astype(np.int8)
    q = np.zeros((nq, dim), dtype=np.int8)
    ix = _index(po.I8, x)
    f0 = ix.stat("fallbacks")
    res = ix.scan_topk(po.L2, q, k)
    rowids = np.arange(1, n + 1, dtype=np.int64)
    for b in (0, nq - 1):
        want_ids, want_d = oracle.scan_dense(po.L2, po.I8, q[b], x, rowids, k)
        assert np.array_equal(res[b][0], want_ids) and np.array_equal(res[b][1], want_d)
    assert ix.stat("fallbacks") >= f0       # the fallback counter only moves when a capacity was exceeded
    ix.close()
