"""Every CUDA allocation, event, stream and IPC mapping the library takes is given back: each case builds an object, runs
every path of it that allocates, frees it, and checks that vsb_debug_live_handles is back where it started.  -m gpu."""
import gc

import numpy as np
import pytest

import sqlite_vector_b200 as vs
from sqlite_vector_b200 import api

pytestmark = pytest.mark.gpu
REPEATS = 3
QUANT_U8 = 1                                              # VSB_QUANT_U8


def _rows(rng, n, dim):
    return rng.integers(-20, 21, (n, dim)).astype(np.int8)


def _index(x, **kw):
    ix = vs.Index(api.I8, x.shape[1], x.shape[0], **kw)
    ix.append_dense(x)
    ix.finalize()
    return ix


def _check_returns(case):
    """runs case() REPEATS times; each run must hold handles while it works and give all of them back"""
    eng = vs.load_engine()
    gc.collect()
    base = eng.debug_live_handles()
    for _ in range(REPEATS):
        held = case()
        assert held > base, "the case took no handles"
        gc.collect()
        assert eng.debug_live_handles() == base


def test_resident_index_returns_every_handle():
    eng = vs.load_engine()
    rng = np.random.Generator(np.random.PCG64(1))
    n, dim = 20_000, 64
    x = _rows(rng, n, dim)
    qs = _rows(rng, 1024, dim)

    def case():
        ix = _index(x)
        for k in (10, 100, 300):                          # both filter kernels, then the all-distances path
            ix.scan_topk(api.L2, qs[0], k)
        ix.collect(ix.scan_submit(api.L2, qs[1], 10), 10)
        ix.scan_all(api.L2, qs[2])
        ix.scan_topk(api.L2, qs, 10)                      # tensor-core batch path
        ix.scan_topk(api.L1, qs, 10)                      # L1 batch kernel
        old = eng.set_option("time_kernels", 1)
        try:
            ix.scan_topk(api.L2, qs[3], 10)
            ix.profile_read()
        finally:
            eng.set_option("time_kernels", old)
        nq = 32
        U = np.full(nq, np.inf, np.float32)
        ix.debug_tc_level(api.L2, qs[:nq], U, 0, 128)
        ix.debug_tc_level(api.L2, qs[:nq], U, 0, 128, scores=True)
        pairs = np.stack([np.arange(64, dtype=np.uint32), np.arange(64, dtype=np.uint32) % nq], axis=1)
        ix.debug_refine(api.SQUARED_L2, qs[:nq], pairs, U)
        bucket = np.zeros((nq, api.BUCKET_CAP, 2), np.uint32)
        ix.debug_replay(api.SQUARED_L2, qs[:nq], 10, bucket, np.zeros(nq, np.uint32), acc_cap=512, final_sort=True)
        held = eng.debug_live_handles()
        ix.close()
        return held

    _check_returns(case)


def test_streamed_index_returns_every_handle():
    eng = vs.load_engine()
    rng = np.random.Generator(np.random.PCG64(2))
    x = _rows(rng, 10_000, 64)
    q = _rows(rng, 1, 64)[0]

    def case():
        ix = _index(x, window_rows=4096)
        ix.scan_topk(api.L2, q, 10)
        ix.scan_topk(api.L2, q, 300)
        ix.scan_all(api.L2, q)
        held = eng.debug_live_handles()
        ix.close()
        return held

    _check_returns(case)


def test_group_returns_every_handle(monkeypatch):
    monkeypatch.setenv("VSB_GROUP_ALIAS", "1")            # three shards on however many GPUs there are
    eng = vs.load_engine()
    rng = np.random.Generator(np.random.PCG64(3))
    n, dim = 30_000, 64
    x = _rows(rng, n, dim)
    qs = _rows(rng, 64, dim)

    def case():
        g = vs.Group(api.I8, dim, n, 3)
        g.append_dense(x)
        g.finalize()
        g.scan_topk(api.L2, qs, 10)                       # batch path: entry logs gathered on the leader
        g.scan_topk(api.L2, qs[:4], 10)                   # per-query path: heads pushed to the leader
        held = eng.debug_live_handles()
        g.close()
        return held

    _check_returns(case)


def test_exchange_returns_every_handle():
    eng = vs.load_engine()
    rng = np.random.Generator(np.random.PCG64(4))
    n, dim = 20_000, 64
    x = _rows(rng, n, dim)
    qs = _rows(rng, 1024, dim)
    first_seq = np.zeros(1, np.int64)

    def case():
        ix = _index(x)
        ix.exchange_attach(ix.exchange_export(1, 0))      # a world of one: the rank's own buffer, no IPC mapping
        ix.exchange_submit(api.L2, qs[:4], qs.strides[0], 4, 10, False, 0)
        ix.exchange_collect(0, 4, first_seq, 10)
        ix.exchange_batch_collect(ix.exchange_batch_submit(api.L2, qs, 10, first_seq), len(qs), 10)
        held = eng.debug_live_handles()
        ix.close()
        return held

    _check_returns(case)


@pytest.mark.parametrize("retain", [False, True])
def test_quantizer_returns_every_handle(retain):
    eng = vs.load_engine()
    rng = np.random.Generator(np.random.PCG64(5))
    n, dim = 5_000, 32
    rows = rng.standard_normal((n, dim), dtype=np.float32)
    rowids = np.arange(1, n + 1, dtype=np.int64)

    def case():
        qz = api.Quantizer(api.F32, dim, retain_rows=n if retain else 0)
        qz.minmax(rows)
        lo, hi, _ = qz.minmax_result()
        scale = 255.0 / (hi - lo)
        if retain:
            assert qz.retained_rows == n
            qz.encode(None, rowids, lo, scale, QUANT_U8)
        else:
            qz.encode(rows, rowids, lo, scale, QUANT_U8)
        held = eng.debug_live_handles()
        qz.close()
        return held

    _check_returns(case)


def test_failed_create_returns_every_handle():
    eng = vs.load_engine()
    gc.collect()
    base = eng.debug_live_handles()
    for _ in range(REPEATS):
        # 4e9 rows x 16 KB: far beyond any device, so the allocation fails at once and reserves nothing
        with pytest.raises(vs.VsbError) as err:
            vs.Index(api.F32, 4096, 4_000_000_000)
        assert err.value.rc == api.ENOMEM
        assert eng.debug_live_handles() == base            # the streams it had created are gone again
