"""Batched queries on streamed columns: the batch path's levels run window by window, one pass of the column per batch.
-m gpu.

(a) a streamed index gives the resident batch path's results bit for bit (rowids and distances, every element type and metric,
    f32 with f32_batch on and off, dims 8 / 128 / 771, k 1..256, nq 16..1500, windows of 128, 300, 5000 and >= n rows, a window 0
    shorter than batch_m0), and the oracle's (int8 / uint8 exact, fp within tests/fpcheck.py);
(b) one pass per batch: stream_bytes, batches, fallbacks, tc_rows and the device footprint of a batch over 32 windows; the fp DOT
    pass for the largest row norm once per column version;
(c) edges: NaN / Inf / norm-overflowing rows in later windows and on window boundaries, a bucket overflow that falls back to the
    per-query loop, windows below 128 rows;
(d) groups under a device budget, vsb_batch_shard_scan + vsb_batch_merge over streamed shards, the SQL batch functions, and the
    exchange's refusal of a streamed index."""
import contextlib
import os

import numpy as np
import pytest

from oracle import pyoracle as po
from tests.fpcheck import assert_fp_topk

pytestmark = pytest.mark.gpu
METRICS = [po.L2, po.L2SQ, po.COS, po.DOT, po.L1]
TYPES = [po.F32, po.F16, po.BF16, po.U8, po.I8]


def _vs():
    import sqlite_vector_b200 as vs
    return vs


@contextlib.contextmanager
def _options(**opts):
    eng = _vs().load_engine()
    old = {name: eng.set_option(name, v) for name, v in opts.items()}
    try:
        yield
    finally:
        for name, v in old.items():
            eng.set_option(name, v)


@contextlib.contextmanager
def _env(**kv):
    old = {k: os.environ.get(k) for k in kv}
    os.environ.update(kv)
    try:
        yield
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def _column(vtype, n, dim, rng):
    if vtype == po.I8:
        return rng.integers(-20, 21, (n, dim)).astype(np.int8)           # narrow range: ties at the k-th place
    if vtype == po.U8:
        return rng.integers(0, 40, (n, dim)).astype(np.uint8)
    return po.convert(rng.standard_normal((n, dim), dtype=np.float32), vtype)


def _pair(vtype, x, window, rowids=None, capacity=None):
    """a resident and a streamed index of the same rows"""
    vs = _vs()
    cap = capacity or x.shape[0]
    res = vs.Index(vtype, x.shape[1], cap)
    st = vs.Index(vtype, x.shape[1], cap, window_rows=window)
    for ix in (res, st):
        ix.append_dense(x, rowids)
        ix.finalize()
    return res, st


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint64)


def _assert_same(got, want, ctx):
    """as_arrays outputs of vsb_scan_topk, bit for bit"""
    assert np.array_equal(got[2], want[2]), ctx
    assert np.array_equal(got[0], want[0]), ctx
    assert np.array_equal(_bits(got[1]), _bits(want[1])), ctx


def _check_oracle(oracle, vtype, metric, x, q, k, out, rowids, queries):
    ids, dist, counts = out
    for b in queries:
        want_ids, want_d = oracle.scan_dense(metric, vtype, q[b], x, rowids, k)
        got_ids, got_d = ids[b, :counts[b]], dist[b, :counts[b]]
        if vtype in (po.I8, po.U8):
            assert np.array_equal(got_ids, want_ids) and np.array_equal(got_d, want_d), (vtype, metric, k, b)
        else:
            assert_fp_topk(got_ids, got_d, want_ids, want_d, metric,
                           lambda r, b=b: oracle.distance(metric, vtype, q[b], x[int(r) - 1]), (vtype, metric, k, b))


def _run_both(res, st, metric, q, k):
    """the same batch on both indexes; returns both outputs and the streamed index's stat deltas"""
    names = ("batches", "fallbacks", "stream_bytes", "tc_rows")
    before = {s: st.stat(s) for s in names}
    rb = res.stat("batches")
    want = res.scan_topk(metric, q, k, as_arrays=True)
    got = st.scan_topk(metric, q, k, as_arrays=True)
    delta = {s: st.stat(s) - before[s] for s in names}
    delta["resident_batches"] = res.stat("batches") - rb
    return got, want, delta


# ---------------------------------------------------------------------------------------------- (a) resident parity
@pytest.mark.parametrize("f32_batch", [0, 1])
@pytest.mark.parametrize("vtype", TYPES)
def test_every_type_and_metric_equals_resident_batch(oracle, vtype, f32_batch):
    """dim 128, 300 queries, k = 20, windows of 5000 rows (the last one ragged): identical to the resident batch path; the
    streamed index batches exactly where the resident one does (f32 L2 / cos / dot only with f32_batch on)"""
    if vtype != po.F32 and f32_batch == 0:
        pytest.skip("f32_batch only concerns f32 columns")
    rng = np.random.Generator(np.random.PCG64(7100 + vtype))
    n, dim, nq, k = 23_456, 128, 300, 20
    x = _column(vtype, n, dim, rng)
    q = _column(vtype, nq, dim, rng)
    rowids = np.arange(1, n + 1, dtype=np.int64)
    with _options(f32_batch=f32_batch):
        res, st = _pair(vtype, x, 5000)
        for metric in METRICS:
            got, want, d = _run_both(res, st, metric, q, k)
            _assert_same(got, want, (vtype, metric, f32_batch))
            batched = d["resident_batches"] == 1
            assert d["batches"] == d["resident_batches"], (vtype, metric, d)
            assert batched == (vtype != po.F32 or f32_batch == 1 or metric == po.L1), (vtype, metric, d)
            if batched:                                # the first fp DOT batch also streams the column for the largest row norm
                passes = 2 if (metric == po.DOT and vtype not in (po.I8, po.U8)) else 1
                assert d["fallbacks"] == 0 and d["stream_bytes"] == passes * n * st.query_pitch, (vtype, metric, d)
            _check_oracle(oracle, vtype, metric, x, q, k, got, rowids, range(0, nq, 1 if vtype in (po.I8, po.U8) else 37))
        res.close()
        st.close()


# (vtype, metric, dim, k, nq, window, batch_m0, f32_batch)
SHAPES = [
    (po.I8, po.L2, 8, 1, 16, 128, 128, 0),
    (po.I8, po.DOT, 771, 256, 17, 300, 128, 0),
    (po.U8, po.COS, 128, 100, 1500, 5000, 128, 0),
    (po.I8, po.L1, 128, 20, 300, 128, 256, 0),            # window 0 shorter than the exhaustive prefix
    (po.BF16, po.DOT, 771, 100, 16, 300, 128, 0),
    (po.F16, po.COS, 8, 256, 17, 1 << 20, 128, 0),        # one window
    (po.BF16, po.L2, 128, 1, 1500, 128, 256, 0),
    (po.F32, po.L1, 771, 20, 300, 300, 128, 0),
    (po.F16, po.L2SQ, 771, 256, 300, 5000, 128, 0),
    (po.U8, po.L1, 8, 100, 1500, 300, 128, 0),
    (po.I8, po.COS, 8, 20, 1500, 1 << 20, 128, 0),
    (po.F32, po.DOT, 128, 100, 17, 128, 256, 1),
    (po.F32, po.L2, 771, 1, 300, 300, 128, 1),
    (po.U8, po.DOT, 8, 256, 1500, 128, 128, 0),
]


@pytest.mark.parametrize("vtype,metric,dim,k,nq,window,m0,f32_batch", SHAPES)
def test_shapes_equal_resident_batch(oracle, vtype, metric, dim, k, nq, window, m0, f32_batch):
    rng = np.random.Generator(np.random.PCG64(7200 + dim + k + nq + window % 1000))
    n = 20_011
    x = _column(vtype, n, dim, rng)
    q = _column(vtype, nq, dim, rng)
    with _options(batch_m0=m0, f32_batch=f32_batch):
        res, st = _pair(vtype, x, window)
        got, want, d = _run_both(res, st, metric, q, k)
        _assert_same(got, want, (vtype, metric, dim, k, nq, window))
        assert d["batches"] == 1 and d["fallbacks"] == 0, d
        rows0 = min(window, n)
        assert d["tc_rows"] == n - min(m0, rows0), d
        _check_oracle(oracle, vtype, metric, x, q, k, got, np.arange(1, n + 1, dtype=np.int64),
                      range(0, nq, 1 if vtype in (po.I8, po.U8) else max(1, nq // 5)))
        res.close()
        st.close()


# ---------------------------------------------------------------------------------------------- (b) one pass per batch
def test_one_pass_of_the_windows_per_batch(oracle):
    """int8 L2 over 32 windows (the last one ragged): stream_bytes grows by one column, tc_rows by every row outside the
    prefix, one batch and no fallback; the device holds the two windows and their norms, not the column"""
    rng = np.random.Generator(np.random.PCG64(7300))
    n, dim, nq, k, win = 40_000, 128, 256, 20, 1280
    x = _column(po.I8, n, dim, rng)
    q = _column(po.I8, nq, dim, rng)
    res, st = _pair(po.I8, x, win)
    for rep in range(2):
        tc_us = st.stat("tc_us")
        got, want, d = _run_both(res, st, po.L2, q, k)
        _assert_same(got, want, rep)
        assert d["stream_bytes"] == n * st.query_pitch, d
        assert d["batches"] == 1 and d["fallbacks"] == 0, d
        assert d["tc_rows"] == n - 128, d
        assert st.stat("tc_us") > tc_us and st.stat("stream_us") > 0
    assert 0 < st.eng.lib.vsb_index_device_bytes(st.h) < n * st.query_pitch
    _check_oracle(oracle, po.I8, po.L2, x, q, k, got, np.arange(1, n + 1, dtype=np.int64), range(nq))
    res.close()
    st.close()


@pytest.mark.parametrize("vtype", [po.BF16, po.F16])
def test_fp_dot_row_norm_pass_once_per_column_version(oracle, vtype):
    """fp DOT reads the column's largest row norm: the first batch streams the column twice, later ones once; appending rows
    (one of them with a larger norm) makes the next batch take the extra pass again.  Other metrics never take it."""
    rng = np.random.Generator(np.random.PCG64(7400 + vtype))
    n, extra, dim, nq, k, win = 20_000, 3_001, 96, 64, 20, 3000
    x = _column(vtype, n + extra, dim, rng)
    x[n + 1500] = po.convert(np.full((1, dim), 9.0, np.float32), vtype)[0]       # the new largest norm
    q = _column(vtype, nq, dim, rng)
    res, st = _pair(vtype, x[:n], win, capacity=n + extra)
    pitch = st.query_pitch
    for want_bytes in (2 * n * pitch, n * pitch):
        got, want, d = _run_both(res, st, po.DOT, q, k)
        _assert_same(got, want, want_bytes)
        assert d["stream_bytes"] == want_bytes and d["batches"] == 1, d
    got, want, d = _run_both(res, st, po.L2, q, k)
    assert d["stream_bytes"] == n * pitch, d
    for ix in (res, st):
        ix.append_dense(x[n:])
    m = n + extra
    for want_bytes in (2 * m * pitch, m * pitch):
        got, want, d = _run_both(res, st, po.DOT, q, k)
        _assert_same(got, want, ("appended", want_bytes))
        assert d["stream_bytes"] == want_bytes and d["batches"] == 1, d
    _check_oracle(oracle, vtype, po.DOT, x, q, k, got, np.arange(1, m + 1, dtype=np.int64), range(0, nq, 7))
    res.close()
    st.close()


# ---------------------------------------------------------------------------------------------- (c) edges
@pytest.mark.parametrize("vtype,f32_batch", [(po.BF16, 0), (po.F16, 0), (po.F32, 1)])
def test_special_rows_in_later_windows(vtype, f32_batch):
    """NaN, +-Inf and rows whose fp32 sum of squares overflows, inside later windows and on both sides of window boundaries;
    one query whose norm overflows: identical to the resident batch path for every metric"""
    rng = np.random.Generator(np.random.PCG64(7500 + vtype))
    n, dim, nq, k, win = 12_000, 64, 33, 20, 1000
    x = rng.standard_normal((n, dim), dtype=np.float32)
    big = np.float32(3e38) if vtype != po.F16 else np.float32(6e4)
    for r, v in [(2999, np.nan), (3000, np.inf), (4000, -np.inf), (5999, big), (6000, big), (9500, np.nan), (10999, big)]:
        x[r, r % dim] = v
    x[7000, :] = big                                                   # every element large: the norm overflows (bf16, f32)
    qf = rng.standard_normal((nq, dim), dtype=np.float32)
    qf[5, :] = big                                                     # a query whose norm overflows
    xc, qc = po.convert(x, vtype), po.convert(qf, vtype)
    with _options(f32_batch=f32_batch):
        res, st = _pair(vtype, xc, win)
        batched = 0
        for metric in METRICS:
            got, want, d = _run_both(res, st, metric, qc, k)
            _assert_same(got, want, (vtype, metric))
            assert d["batches"] == d["resident_batches"], (metric, d)
            batched += d["batches"]
        assert batched >= 3, batched
        res.close()
        st.close()


def test_bucket_overflow_falls_back_to_single_queries(oracle):
    """window 1 holds 5000 rows that each come closer to the queries than every row before them: more than a query's bucket
    can keep in one level.  VSB_ERANGE inside, the per-query streamed loop answers exactly, fallbacks + 1, no batch counted."""
    n, dim, nq, k, win = 20_000, 16, 16, 20, 5000
    x = np.full((n, dim), 0, dtype=np.int8)
    x[:, 0] = 120
    x[5000:10000, 0] = 127 - np.arange(5000) // 40                      # 127 .. 3, descending in window 1
    q = np.zeros((nq, dim), dtype=np.int8)
    q[:, 1] = np.arange(nq) % 3
    res, st = _pair(po.I8, x, win)
    got, want, d = _run_both(res, st, po.L1, q, k)
    assert d["batches"] == 0 and d["fallbacks"] == 1, d
    _assert_same(got, want, "overflow")
    _check_oracle(oracle, po.I8, po.L1, x, q, k, got, np.arange(1, n + 1, dtype=np.int64), range(nq))
    res.close()
    st.close()


def test_windows_below_a_tile_keep_the_per_query_path(oracle):
    rng = np.random.Generator(np.random.PCG64(7600))
    n, dim, nq, k = 9_000, 32, 20, 10
    x = _column(po.I8, n, dim, rng)
    q = _column(po.I8, nq, dim, rng)
    res, st = _pair(po.I8, x, 64)
    got, want, d = _run_both(res, st, po.L2, q, k)
    assert d["batches"] == 0 and d["resident_batches"] == 1 and d["stream_bytes"] == nq * n * st.query_pitch, d
    _assert_same(got, want, "64-row windows")
    _check_oracle(oracle, po.I8, po.L2, x, q, k, got, np.arange(1, n + 1, dtype=np.int64), range(nq))
    res.close()
    st.close()


# ---------------------------------------------------------------------------------------------- (d) groups, shards, SQL
def _group(vtype, x, ngpus):
    g = _vs().Group(vtype, x.shape[1], x.shape[0], ngpus)
    for a in range(0, x.shape[0], 7919):
        g.append_dense(x[a:a + 7919])
    g.finalize()
    return g


@pytest.mark.parametrize("vtype,metric", [(po.I8, po.L2), (po.U8, po.L1), (po.BF16, po.DOT), (po.F16, po.COS)])
def test_streamed_groups_batch_like_resident_groups(oracle, vtype, metric):
    """VSB_DEVICE_BUDGET_MB below a shard's size streams the shards of 1- and 3-shard groups (VSB_GROUP_ALIAS=1: on one
    GPU): the batch equals the unbudgeted group's and every shard counts one batch"""
    vs = _vs()
    lib = vs.load_engine().lib
    rng = np.random.Generator(np.random.PCG64(7700 + vtype))
    n, dim, nq, k = 60_000, 64, 40, 20
    x = _column(vtype, n, dim, rng)
    q = _column(vtype, nq, dim, rng)
    with _env(VSB_GROUP_ALIAS="1"):
        for ngpus in (1, 3):
            plain = _group(vtype, x, ngpus)
            want = plain.scan_topk(metric, q, k)
            plain.close()
            with _env(VSB_DEVICE_BUDGET_MB="0.5"):
                g = _group(vtype, x, ngpus)
            shards = [lib.vsb_group_shard(g.h, s) for s in range(ngpus)]
            assert all(lib.vsb_index_is_streamed(s) == 1 for s in shards)
            b0 = [lib.vsb_index_stat(s, b"batches") for s in shards]
            got = g.scan_topk(metric, q, k)
            assert [lib.vsb_index_stat(s, b"batches") - b for s, b in zip(shards, b0)] == [1] * ngpus, ngpus
            for b in range(nq):
                assert np.array_equal(got[b][0], want[b][0]) and np.array_equal(_bits(got[b][1]), _bits(want[b][1])), (ngpus, b)
            g.close()
    ids = np.arange(1, n + 1, dtype=np.int64)
    for b in range(0, nq, 1 if vtype in (po.I8, po.U8) else 9):
        want_ids, want_d = oracle.scan_dense(metric, vtype, q[b], x, ids, k)
        if vtype in (po.I8, po.U8):
            assert np.array_equal(got[b][0], want_ids) and np.array_equal(got[b][1], want_d), b
        else:
            assert_fp_topk(got[b][0], got[b][1], want_ids, want_d, metric, lambda r, b=b: oracle.distance(metric, vtype, q[b], x[int(r) - 1]), b)


def test_batch_shard_scan_and_merge_over_streamed_shards():
    """vsb_batch_shard_scan on three streamed shards (entry-log blocks), gathered and replayed by vsb_batch_merge: the batch of
    one resident index over all rows"""
    import torch

    from sqlite_vector_b200.shard import _DevView
    vs = _vs()
    rng = np.random.Generator(np.random.PCG64(7800))
    n, dim, nq, k = 45_000, 96, 64, 33
    x = _column(po.I8, n, dim, rng)
    q = _column(po.I8, nq, dim, rng)
    bounds = [0, 14_000, 29_500, n]
    whole = vs.Index(po.I8, dim, n)
    whole.append_dense(x)
    whole.finalize()
    for metric in (po.L2, po.DOT, po.L1):
        want = whole.scan_topk(metric, q, k)
        shards, parts = [], []
        for s in range(3):
            ix = vs.Index(po.I8, dim, bounds[s + 1] - bounds[s], first_seq=bounds[s], window_rows=3000)
            ix.append_dense(x[bounds[s]:bounds[s + 1]])
            ix.finalize()
            ptr, nbytes = ix.batch_shard_scan(metric, q, k)
            parts.append(torch.as_tensor(_DevView(ptr, nbytes), device="cuda").clone())
            assert ix.stat("batches") == 1 and ix.stat("stream_bytes") == (bounds[s + 1] - bounds[s]) * ix.query_pitch
            shards.append(ix)
        gathered = torch.cat(parts)
        torch.cuda.synchronize()
        seq, d, counts = shards[0].batch_merge(gathered.data_ptr(), 3, nbytes, np.asarray(bounds[:3], dtype=np.int64), nq, k)
        ids = sum(ix.lookup_rowids(seq) for ix in shards)
        for b in range(nq):
            assert np.array_equal(ids[b, :counts[b]], want[b][0]) and np.array_equal(d[b, :counts[b]], want[b][1]), (metric, b)
        for ix in shards:
            ix.close()
    whole.close()


def test_sql_batch_functions_under_a_tiny_budget():
    """vector_quantize_scan_batch and vector_full_scan_batch over a 9000-row table streamed through small windows return
    the rows they return without the budget"""
    from tests.sqlrun import OURS, run_sql
    rng = np.random.Generator(np.random.PCG64(7900))
    n, dim, nq, k = 9_000, 16, 20, 7
    x = rng.integers(-20, 21, (n, dim)).astype(np.int8)
    q = rng.integers(-20, 21, (nq, dim)).astype(np.int8)
    s = ["CREATE TABLE t (id INTEGER PRIMARY KEY, e BLOB)", f"SELECT vector_init('t','e','type=INT8,dimension={dim}')"]
    for i in range(n):
        s.append(["INSERT INTO t(id, e) VALUES (?, ?)", [3 * i + 2, {"hex": x[i].tobytes().hex()}]])
    s.append(["SELECT query, id, distance FROM vector_full_scan_batch('t','e',?,?)", [{"hex": q.tobytes().hex()}, k]])
    s.append("SELECT vector_quantize('t','e')")
    s.append(["SELECT query, id, distance FROM vector_quantize_scan_batch('t','e',?,?)", [{"hex": q.tobytes().hex()}, k]])
    one = run_sql(OURS, s)[-3:]
    tiny = run_sql(OURS, s, env={"VSB_DEVICE_BUDGET_MB": "0.03"})[-3:]   # 144 KB of int8: windows of ~650 rows
    for a, b in ((one[0], tiny[0]), (one[2], tiny[2])):
        assert "rows" in a and len(a["rows"]) == nq * k, a
        assert a == b


def test_exchange_batch_refuses_a_streamed_index():
    vs = _vs()
    ix = vs.Index(po.I8, 16, 20_000, window_rows=4096)
    ix.append_dense(np.ones((20_000, 16), dtype=np.int8))
    ix.finalize()
    with pytest.raises(vs.VsbError) as e:
        ix.exchange_batch_submit(po.L2, np.ones((32, 16), dtype=np.int8), 5, np.zeros(1, dtype=np.int64))
    assert e.value.rc == -5      # VSB_ERANGE
    ix.close()
