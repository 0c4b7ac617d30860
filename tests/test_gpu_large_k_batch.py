"""Batched top-k for k > 256 (DESIGN §3.12): the batch levels find each query's candidates with per-query bounds, one pass of the
column per batch, and the host replays them.  -m gpu.

The yardstick is the single call on the same index (vsb_scan_topk with one query, the large-k path of §3.11): every query of a
batch must give the same rowids and the same distance bits, for every element type, metric, filter and scan path.  The bounds
and candidates are restated in numpy from the all-distances scan: a piece of level L >= 1 is refined against U = the k-th
smallest key (float order) of the query's kept entries of the levels before L (+INF when fewer than k), and a query keeps the
eligible rows of each piece with d < U (level 0: U = +INF)."""
import contextlib
import os

import numpy as np
import pytest

from oracle import pyoracle as po
from tests.sqlrun import OURS, run_sql

pytestmark = pytest.mark.gpu
TYPES = [po.F32, po.F16, po.BF16, po.U8, po.I8]


def _vs():
    import sqlite_vector_b200 as vs
    return vs


@contextlib.contextmanager
def _env(**kv):
    old = {k: os.environ.get(k) for k in kv}
    os.environ.update({k: str(v) for k, v in kv.items()})
    try:
        yield
    finally:
        for k, v in old.items():
            os.environ.pop(k, None) if v is None else os.environ.update({k: v})


@contextlib.contextmanager
def _option(name, value):
    eng = _vs().load_engine()
    old = eng.set_option(name, value)
    try:
        yield
    finally:
        eng.set_option(name, old)


def _column(vtype, n, dim, rng, spread=20):
    if vtype == po.I8:
        return rng.integers(-spread, spread + 1, (n, dim)).astype(np.int8)
    if vtype == po.U8:
        return rng.integers(0, 2 * spread, (n, dim)).astype(np.uint8)
    return po.convert(rng.standard_normal((n, dim), dtype=np.float32), vtype)


def _index(vtype, x, rowids=None, window=0):
    ix = _vs().Index(vtype, x.shape[1], x.shape[0], window_rows=window)
    ix.append_dense(x, rowids)
    ix.finalize()
    return ix


def _group(vtype, x, ngpus, rowids=None, chunk=7919):
    g = _vs().Group(vtype, x.shape[1], x.shape[0], ngpus)
    for a in range(0, x.shape[0], chunk):
        g.append_dense(x[a:a + chunk], None if rowids is None else rowids[a:a + chunk])
    g.finalize()
    return g


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint64 if np.asarray(a).dtype == np.float64 else np.uint32)


def _key(d):
    u = np.ascontiguousarray(d, dtype=np.float32).view(np.uint32)
    return np.where(u & np.uint32(0x80000000), ~u, u | np.uint32(0x80000000))


def _unkey(k):
    k = np.uint32(k)
    u = (k & np.uint32(0x7FFFFFFF)) if (k & np.uint32(0x80000000)) else ~k
    return np.array([u], np.uint32).view(np.float32)[0]


def same(got, want, ctx):
    assert np.array_equal(got[0], want[0]), (ctx, "rowids")
    assert np.array_equal(_bits(np.asarray(got[1], np.float64)), _bits(np.asarray(want[1], np.float64))), (ctx, "distances")


def counters(ix):
    return {s: ix.stat(s) for s in ("large_k_batches", "large_k_batch_fallbacks", "large_k_query_fallbacks", "large_k_queries", "large_k_cands")}


def batch_equals_singles(ix, metric, qs, k, allow=None, ctx=()):
    """the batch of qs against one single call per query; returns the counter deltas of the batch"""
    c0 = counters(ix)
    got = ix.scan_topk(metric, qs, k) if allow is None else ix.scan_topk_filtered(metric, qs, k, allow)
    c1 = counters(ix)
    assert len(got) == len(qs)
    for b in range(len(qs)):
        want = ix.scan_topk(metric, qs[b], k)[0] if allow is None else ix.scan_topk_filtered(metric, qs[b], k, allow)[0]
        same(got[b], want, ctx + (b,))
    return {s: c1[s] - c0[s] for s in c0}, got


def batch_bounds(ix):
    head = ix.debug_read("large_k_batch_bounds", np.int64, 2)
    P, Q = int(head[0]), int(head[1])
    raw = ix.debug_read("large_k_batch_bounds", np.uint8, 16 + 24 * P + 4 * P * Q)
    pieces = raw[16:16 + 24 * P].view(np.int64).reshape(P, 3)
    U = raw[16 + 24 * P:].view(np.float32).reshape(P, Q)
    return pieces, U


def batch_cands(ix):
    """each query's candidates of the last batch: None for a query answered alone, else (distance bits, shard rows) in order"""
    nq = int(ix.debug_read("large_k_batch_cands", np.int64, 1)[0])
    cnt = ix.debug_read("large_k_batch_cands", np.int64, 1 + nq)[1:]
    raw = ix.debug_read("large_k_batch_cands", np.uint32, 2 + 2 * nq + 2 * int(cnt[cnt > 0].sum()))[2 + 2 * nq:].reshape(-1, 2)
    out, at = [], 0
    for c in cnt:
        out.append(None if c < 0 else (raw[at:at + c, 0], raw[at:at + c, 1].astype(np.int64)))
        at += max(int(c), 0)
    return out


def restate(d, elig, pieces, k):
    """the bounds a query's pieces must carry and the rows it keeps, from its distances d (scan order)"""
    key = _key(d)
    kept = np.zeros(len(d), bool)
    want_u = []
    for lvl in sorted(set(pieces[:, 2].tolist())):
        if lvl == 0:
            u = np.float32(np.inf)
        else:
            kk = key[kept]
            if len(kk) < k:
                u = np.float32(np.inf)
            else:
                u = _unkey(np.partition(kk, k - 1)[k - 1])
        for p in np.nonzero(pieces[:, 2] == lvl)[0]:
            a, b = pieces[p, :2]
            with np.errstate(invalid="ignore"):
                kept[a:b] = elig[a:b] & (d[a:b] < u)
            want_u.append((p, u))
    return dict(want_u), kept


# ------------------------------------------------------------------------------------------------ every admitted pair
PAIRS = [(t, m) for t in (po.I8, po.U8, po.F16, po.BF16) for m in (po.L2, po.L2SQ, po.COS, po.DOT)] + [(t, po.L1) for t in TYPES] + \
        [(po.F32, m) for m in (po.L2, po.L2SQ, po.COS, po.DOT)]
NQS = (16, 40, 300)


@pytest.mark.parametrize("dim", [16, 128, 771])
@pytest.mark.parametrize("vtype, metric", PAIRS)
def test_admitted_pairs_equal_single_calls(vtype, metric, dim):
    rng = np.random.Generator(np.random.PCG64(1000 + 10 * vtype + metric + dim))
    n = 8192
    x = _column(vtype, n, dim, rng)
    ix = _index(vtype, x)
    at = PAIRS.index((vtype, metric)) + dim
    with _option("f32_batch", 1 if vtype == po.F32 else 0):
        for nq, k in ((NQS[at % 3], 257), (NQS[(at + 1) % 3], 1000), (16, n)):
            qs = _column(vtype, nq, dim, rng)
            dc, _ = batch_equals_singles(ix, metric, qs, k, ctx=(vtype, metric, dim, nq, k))
            assert dc["large_k_batches"] == 1 and dc["large_k_batch_fallbacks"] == 0 and dc["large_k_query_fallbacks"] == 0, dc
            assert dc["large_k_queries"] == nq, dc
    ix.close()


# ------------------------------------------------------------------------------------------------ bounds and candidates
@pytest.mark.parametrize("vtype, metric, window", [(po.I8, po.L2, 0), (po.BF16, po.DOT, 0), (po.F16, po.COS, 0), (po.U8, po.L1, 3000)])
def test_bounds_and_candidates_against_numpy(vtype, metric, window):
    rng = np.random.Generator(np.random.PCG64(2000 + vtype + metric + window))
    n, dim, k, nq = 20_000, 64, 300, 16
    x = _column(vtype, n, dim, rng)
    ix = _index(vtype, x, window=window)
    qs = _column(vtype, nq, dim, rng)
    for allow in (None, rng.random(n) < 0.4):
        elig = np.ones(n, bool) if allow is None else allow
        c0 = ix.stat("large_k_cands")
        ix.scan_topk(metric, qs, k) if allow is None else ix.scan_topk_filtered(metric, qs, k, allow)
        got_cands = ix.stat("large_k_cands") - c0
        pieces, U = batch_bounds(ix)
        cands = batch_cands(ix)
        assert len(cands) == nq
        assert pieces[0, 0] == 0 and pieces[-1, 1] == n and np.array_equal(pieces[1:, 0], pieces[:-1, 1])
        total = 0
        for q in range(nq):
            d = ix.scan_all(metric, qs[q])
            want_u, kept = restate(d, elig, pieces, k)
            for p, u in want_u.items():
                assert _bits(np.float32(U[p, q])) == _bits(np.float32(u)), (vtype, metric, q, p, U[p, q], u)
            rows = np.nonzero(kept)[0]
            assert cands[q] is not None and np.array_equal(cands[q][1], rows), (vtype, metric, q, "rows in scan order")
            assert np.array_equal(cands[q][0], _bits(d[rows])), (vtype, metric, q, "distance bits")
            total += int(kept.sum())
        assert got_cands == total, (got_cands, total)
    ix.close()


# ------------------------------------------------------------------------------------------------ edge data
def test_special_values_and_ties():
    rng = np.random.Generator(np.random.PCG64(3000))
    n, dim = 9000, 32
    for vtype in (po.F16, po.BF16, po.F32):
        x = rng.standard_normal((n, dim), dtype=np.float32)
        at = rng.random(n)
        x[at < 0.01, 3] = np.nan
        x[(at >= 0.01) & (at < 0.02), 5] = np.inf
        x[(at >= 0.02) & (at < 0.03), 7] = -np.inf
        x = po.convert(x, vtype)
        ix = _index(vtype, x)
        qs = po.convert(rng.standard_normal((20, dim), dtype=np.float32), vtype)
        qs[1, 2] = po.convert(np.array([np.nan], np.float32), vtype)[0] if vtype != po.F32 else np.nan
        qs[2, 4] = po.convert(np.array([np.inf], np.float32), vtype)[0] if vtype != po.F32 else np.inf
        metrics = (po.L2, po.L2SQ, po.COS, po.DOT, po.L1) if vtype != po.F32 else (po.L1,)
        for metric in metrics:
            for k in (257, 2000):
                dc, got = batch_equals_singles(ix, metric, qs, k, ctx=(vtype, metric, k))
                assert dc["large_k_batches"] == 1, dc
                if vtype != po.F32 and metric == po.DOT:
                    assert any(np.isneginf(np.asarray(g[1])).any() for g in got), "no -INF distance was exercised"
        ix.close()
    x = rng.integers(-1, 2, (n, 24)).astype(np.int8)                  # heavy ties at every bound
    ix = _index(po.I8, x)
    qs = rng.integers(-1, 2, (32, 24)).astype(np.int8)
    for metric in (po.L2, po.DOT, po.L1, po.COS):
        for k in (257, 1000, 4000):
            dc, _ = batch_equals_singles(ix, metric, qs, k, ctx=("ties", metric, k))
            assert dc["large_k_batches"] == 1 and dc["large_k_query_fallbacks"] == 0, dc
    ix.close()


# ------------------------------------------------------------------------------------------------ filters
def test_filters_equal_filtered_single_calls():
    rng = np.random.Generator(np.random.PCG64(4000))
    n, dim = 30_000, 48
    x = _column(po.I8, n, dim, rng)
    ix = _index(po.I8, x, np.arange(n, dtype=np.int64) * 3 + 7)
    qs = _column(po.I8, 24, dim, rng)
    block = np.zeros(n, bool)
    block[12_000:15_500] = True
    few = np.zeros(n, bool)
    few[rng.choice(n, 200, replace=False)] = True
    masks = {"10%": rng.random(n) < 0.10, "1%": rng.random(n) < 0.01, "block": block, "fewer than k": few, "none": np.zeros(n, bool)}
    for name, m in masks.items():
        for metric in (po.L2, po.DOT):
            for k in (257, 1000):
                dc, got = batch_equals_singles(ix, metric, qs, k, allow=m, ctx=(name, metric, k))
                assert dc["large_k_batches"] == 1, (name, dc)
                if name == "none":
                    assert all(len(g[0]) == 0 for g in got)
    ix.close()


# ------------------------------------------------------------------------------------------------ streamed windows
@pytest.mark.parametrize("window", [128, 700, 6001])
def test_streamed_windows_equal_resident_and_singles(window):
    rng = np.random.Generator(np.random.PCG64(5000 + window))
    n, dim = 20_000, 40
    x = _column(po.I8, n, dim, rng)
    st, res = _index(po.I8, x, window=window), _index(po.I8, x)
    qs = _column(po.I8, 20, dim, rng)
    m = (np.arange(n) // 900) % 3 != 0
    pitch = st.query_pitch
    for metric in (po.L2, po.COS):
        for k in (257, 1000):
            b0 = st.stat("stream_bytes")
            got = st.scan_topk(metric, qs, k)
            assert st.stat("stream_bytes") - b0 == n * pitch, window     # one pass of the column for the batch
            want = res.scan_topk(metric, qs, k)
            for b in range(len(qs)):
                same(got[b], want[b], (window, metric, k, b))
                same(got[b], st.scan_topk(metric, qs[b], k)[0], (window, metric, k, b, "single"))
            dc, _ = batch_equals_singles(st, metric, qs, k, allow=m, ctx=(window, metric, k, "filtered"))
            assert dc["large_k_batches"] == 1, dc
    st.close(); res.close()


# ------------------------------------------------------------------------------------------------ groups
@pytest.mark.parametrize("ngpus", [1, 3])
def test_groups_equal_one_index(ngpus, monkeypatch):
    monkeypatch.setenv("VSB_GROUP_ALIAS", "1")
    rng = np.random.Generator(np.random.PCG64(6000 + ngpus))
    n = 30_001
    x = _column(po.U8, n, 20, rng)
    ids = rng.permutation(3 * n)[:n].astype(np.int64) + 1
    ix = _index(po.U8, x, ids)
    qs = _column(po.U8, 20, 20, rng)
    m = np.zeros(n, bool)
    m[n // 3 - 500:n // 3 + 500] = True
    m |= rng.random(n) < 0.05
    for budget in (None, "0.2"):                                       # resident, then streamed shards
        with _env(**({"VSB_DEVICE_BUDGET_MB": budget} if budget else {})):
            g = _group(po.U8, x, ngpus, ids)
        shards = [g.eng.lib.vsb_group_shard(g.h, s) for s in range(ngpus)]
        assert all(bool(g.eng.lib.vsb_index_is_streamed(h)) == (budget is not None) for h in shards)
        for metric in (po.L2, po.L1):
            for k in (257, 2000):
                got, want = g.scan_topk(metric, qs, k), ix.scan_topk(metric, qs, k)
                for b in range(len(qs)):
                    same(got[b], want[b], (ngpus, budget, metric, k, b))
                got, want = g.scan_topk_filtered(metric, qs, k, m), ix.scan_topk_filtered(metric, qs, k, m)
                for b in range(len(qs)):
                    same(got[b], want[b], (ngpus, budget, metric, k, b, "filtered"))
        batches = sum(g.eng.lib.vsb_index_stat(h, b"large_k_batches") for h in shards)
        assert batches == 8 * ngpus, batches
        g.close()
    ix.close()


# ------------------------------------------------------------------------------------------------ fallbacks
def test_bucket_overflow_answers_the_query_alone():
    """rows whose distance to the all-ones query falls strictly with the row: every row enters the slots, so those queries'
    buckets overflow and they are answered alone; the other queries stay in the batch"""
    rng = np.random.Generator(np.random.PCG64(7000))
    n, dim = 8192, 128
    r = np.arange(n)[:, None]
    x = np.clip(r - 127 * np.arange(dim)[None, :], 0, 127).astype(np.int8)   # row sums 0, 1, ..., n - 1
    ix = _index(po.I8, x)
    qs = np.ones((16, dim), np.int8)
    qs[1::2] = -1                                                      # rising distances: these keep little more than level 0
    qs[1::2, :8] = rng.integers(-3, 1, (8, 8))
    dc, _ = batch_equals_singles(ix, po.DOT, qs, 257, ctx=("falling",))
    assert dc["large_k_batches"] == 1 and dc["large_k_query_fallbacks"] == 8 and dc["large_k_batch_fallbacks"] == 0, dc
    assert dc["large_k_queries"] == 16, dc                             # 8 in the batch, 8 alone: each counted once
    ix.close()


def test_candidate_log_overflow_answers_every_query_alone():
    """f32 L1 to the zero query falls strictly with the row: a level of 150k rows hits for every one of 300 queries, beyond the
    candidate log"""
    n, dim = 300_000, 16
    x = np.repeat((n - np.arange(n, dtype=np.float32))[:, None], dim, axis=1)
    ix = _index(po.F32, x)
    qs = np.zeros((300, dim), np.float32)
    qs[:, 0] = np.arange(300, dtype=np.float32) * 1e-3
    dc, _ = batch_equals_singles(ix, po.L1, qs, 257, ctx=("log",))
    assert dc["large_k_batch_fallbacks"] == 1 and dc["large_k_batches"] == 0 and dc["large_k_queries"] == 300, dc
    ix.close()


def test_more_queries_than_one_tile_of_pairs_fits_the_log():
    """131 072 queries x one 128-row tile of level 0 fill the candidate log exactly, and the scorer's per-query bounds fill its
    shared memory far earlier: a larger batch is split into sub-batches instead of writing a level-0 piece past the log"""
    rng = np.random.Generator(np.random.PCG64(7500))
    n, dim, nq = 8192, 16, 131_072 + 1000
    x = _column(po.I8, n, dim, rng)
    ix = _index(po.I8, x)
    qs = _column(po.I8, nq, dim, rng)
    c0 = counters(ix)
    got = ix.scan_topk(po.L2, qs, 257)
    dc = {s: ix.stat(s) - c0[s] for s in c0}
    assert dc["large_k_batches"] == 1 and dc["large_k_batch_fallbacks"] == 0 and dc["large_k_query_fallbacks"] == 0, dc
    assert dc["large_k_queries"] == nq, dc
    pieces, U = batch_bounds(ix)
    assert U.shape[1] < nq                                             # the bounds of the last sub-batch only
    for b in list(range(0, nq, 4999)) + [131_071, 131_072, nq - 1]:
        same(got[b], ix.scan_topk(po.L2, qs[b], 257)[0], ("sub-batches", b))
    ix.close()


# ------------------------------------------------------------------------------------------------ SQL and handles
def test_sql_batch_modules_equal_single_modules():
    rng = np.random.Generator(np.random.PCG64(8000))
    n, dim, nq = 9000, 16, 17
    x = rng.integers(-40, 41, (n, dim)).astype(np.int8)
    ids = np.arange(n, dtype=np.int64) * 2 + 1
    q = rng.integers(-40, 41, (nq, dim)).astype(np.int8)
    allq = {"hex": q.tobytes().hex()}
    s = ["CREATE TABLE t (id INTEGER PRIMARY KEY, e BLOB, tag INTEGER)", f"SELECT vector_init('t','e','type=INT8,dimension={dim}')"]
    s += [["INSERT INTO t(id, e, tag) VALUES (?, ?, ?)", [int(ids[i]), {"hex": x[i].tobytes().hex()}, int(i % 7)]] for i in range(n)]
    s.append("SELECT vector_quantize('t','e')")
    mark = len(s)
    sub = "(SELECT vector_rowid_set(id) FROM t WHERE tag < 3)"
    cases = []
    for k in (257, 1000):
        for mod in ("full", "quantize"):
            cases.append((mod, k, False))
            s.append(["SELECT query, id, distance FROM vector_%s_scan_batch('t','e',?,?)" % mod, [allq, k]])
            cases.append((mod, k, True))
            s.append(["SELECT query, id, distance FROM vector_%s_scan_batch_filtered('t','e',?,?,%s)" % (mod, sub), [allq, k]])
            for b in range(nq):
                qb = {"hex": q[b].tobytes().hex()}
                s.append(["SELECT id, distance FROM vector_%s_scan('t','e',?,?)" % mod, [qb, k]])
                s.append(["SELECT id, distance FROM vector_%s_scan_filtered('t','e',?,?,%s)" % (mod, sub), [qb, k]])
    r = run_sql(OURS, s)[mark:]
    assert all("error" not in e for e in r), [e for e in r if "error" in e][:2]
    at = 0
    for k in (257, 1000):
        for mod in ("full", "quantize"):
            batch, batch_f = r[at], r[at + 1]
            singles = r[at + 2:at + 2 + 2 * nq]
            at += 2 + 2 * nq
            for b in range(nq):
                assert [row[1:] for row in batch["rows"] if row[0] == b] == singles[2 * b]["rows"], (mod, k, b)
                assert [row[1:] for row in batch_f["rows"] if row[0] == b] == singles[2 * b + 1]["rows"], (mod, k, b, "filtered")
            assert len(singles[0]["rows"]) == k


def test_large_k_batches_leak_no_handles():
    eng = _vs().load_engine()
    rng = np.random.Generator(np.random.PCG64(9000))
    x = _column(po.I8, 40_000, 16, rng)
    q = _column(po.I8, 20, 16, rng)
    base = eng.debug_live_handles()
    for window in (0, 9000):
        ix = _index(po.I8, x, window=window)
        ix.scan_topk(po.L2, q, 1000)
        ix.scan_topk_filtered(po.L2, q, 500, rng.random(40_000) < 0.5)
        assert ix.stat("large_k_batches") == 2
        assert eng.debug_live_handles() > base
        ix.close()
        assert eng.debug_live_handles() == base, window
