"""Filtered top-k (vsb_scan_topk_filtered and its group / SQL doors): the k nearest among the eligible rows equal the unfiltered
scan of the sub-column x[mask], ids[mask].  -m gpu.

(1) every row eligible: bit for bit the unfiltered call (single query, max_index carry, batches of every kind, streamed windows,
    1- and 3-shard groups, SQL);
(2) the oracle on the sub-column for every (type, metric) pair, dims 5 / 128 / 771, k 1..300 and a family of masks;
(3) the batch path really runs for every mask family (batches +1, no fallback) and equals B filtered single calls; a forced
    bucket overflow falls back and stays exact;
(4) poisoned ineligible rows (copies of the queries) never appear and do not flood the candidate log;
(5) streamed windows and groups with clustered masks across window and (unaligned) shard boundaries; the rowid bitmaps;
(6) SQL: the four filtered modules and vector_rowid_set; (7) device handles return to their baseline."""
import contextlib
import os

import numpy as np
import pytest

from oracle import pyoracle as po
from tests.fpcheck import assert_fp_topk
from tests.sqlrun import OURS, run_sql

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


@pytest.fixture(scope="module", autouse=True)
def _alias():
    old = os.environ.get("VSB_GROUP_ALIAS")
    os.environ["VSB_GROUP_ALIAS"] = "1"
    yield
    if old is None:
        os.environ.pop("VSB_GROUP_ALIAS", None)
    else:
        os.environ["VSB_GROUP_ALIAS"] = old


def _column(vtype, n, dim, rng):
    if vtype == po.I8:
        return rng.integers(-20, 21, (n, dim)).astype(np.int8)
    if vtype == po.U8:
        return rng.integers(0, 40, (n, dim)).astype(np.uint8)
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


def masks(n, k, rng):
    """the mask families of the filtered tests"""
    m = {f"random{s}": rng.random(n) < s for s in (0.5, 0.1, 0.01, 0.001)}
    for name, a in (("block_start", 0), ("block_middle", n // 2 - n // 10), ("block_end", n - n // 5)):
        b = np.zeros(n, bool)
        b[a:a + n // 5] = True
        m[name] = b
    m["alternating"] = (np.arange(n) // 997) % 2 == 1
    m["every7"] = np.arange(n) % 7 == 0
    m["empty"] = np.zeros(n, bool)
    exact = np.zeros(n, bool)
    exact[rng.choice(n, size=min(k, n), replace=False)] = True
    m["exactly_k"] = exact
    few = np.zeros(n, bool)
    few[rng.choice(n, size=max(k // 2, 1) if k > 1 else 0, replace=False)] = True
    m["fewer_than_k"] = few
    return m


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint64)


def _assert_same(got, want, ctx):
    """as_arrays outputs, bit for bit"""
    assert np.array_equal(got[2], want[2]), ctx
    for b in range(len(got[2])):
        c = int(got[2][b])
        assert np.array_equal(got[0][b, :c], want[0][b, :c]), (ctx, b)
        assert np.array_equal(_bits(got[1][b, :c]), _bits(want[1][b, :c])), (ctx, b)


def _check_sub(oracle, vtype, metric, x, ids, mask, q, k, got_ids, got_d, ctx, smi=0):
    want_ids, want_d = oracle.scan_dense(metric, vtype, q, x[mask], ids[mask], k, start_max_index=smi)
    if vtype in (po.I8, po.U8):
        assert np.array_equal(got_ids, want_ids) and np.array_equal(got_d, want_d), ctx
    else:
        pos = {int(r): i for i, r in enumerate(ids)}
        assert_fp_topk(got_ids, got_d, want_ids, want_d, metric, lambda r: oracle.distance(metric, vtype, q, x[pos[int(r)]]), ctx)
    assert set(got_ids.tolist()) <= set(ids[mask].tolist()), ctx


# ------------------------------------------------------------------------------------------------ (1) all eligible == unfiltered
@pytest.mark.parametrize("vtype", TYPES)
def test_all_eligible_equals_unfiltered(vtype):
    rng = np.random.Generator(np.random.PCG64(9000 + vtype))
    n, dim = 20_000, 128
    x = _column(vtype, n, dim, rng)
    rowids = np.arange(n, dtype=np.int64) * 3 + 7
    ix = _index(vtype, x, rowids)
    full = np.ones(n, bool)
    q1 = _column(vtype, 1, dim, rng)
    qb = _column(vtype, 64, dim, rng)
    for metric in METRICS:
        for k in (1, 20, 256, 300):
            _assert_same(ix.scan_topk_filtered(metric, q1, k, full, as_arrays=True), ix.scan_topk(metric, q1, k, as_arrays=True), (metric, k))
        for f32_batch in ((0, 1) if vtype == po.F32 else (0,)):
            with _options(f32_batch=f32_batch):
                b0 = ix.stat("batches")
                want = ix.scan_topk(metric, qb, 20, as_arrays=True)
                b1 = ix.stat("batches")
                got = ix.scan_topk_filtered(metric, qb, 20, full, as_arrays=True)
                assert ix.stat("batches") - b1 == b1 - b0, (metric, f32_batch)       # the filtered call batches where the plain one does
                _assert_same(got, want, (metric, f32_batch))
    # the max_index cursor carries through a k = 100 -> 10 -> 33 sequence exactly as unfiltered
    mi_a = mi_b = 0
    for k in (100, 10, 33):
        ra, mi_a = ix.scan_topk(po.L2, q1, k, max_index=mi_a, as_arrays=True)
        rb, mi_b = ix.scan_topk_filtered(po.L2, q1, k, full, max_index=mi_b, as_arrays=True)
        _assert_same(rb, ra, k)
        assert mi_a == mi_b
    ix.close()


@pytest.mark.parametrize("window", [128, 300, 5000])
def test_all_eligible_streamed_equals_unfiltered(window):
    rng = np.random.Generator(np.random.PCG64(9100 + window))
    n, dim = 12_000, 64
    x = _column(po.I8, n, dim, rng)
    st = _index(po.I8, x, window=window)
    full = np.ones(n, bool)
    q = _column(po.I8, 40, dim, rng)
    for metric, k in ((po.L2, 20), (po.DOT, 256), (po.L1, 7)):
        rows0, b0 = st.stat("tc_rows"), st.stat("batches")
        want = st.scan_topk(metric, q, k, as_arrays=True)
        rows1, b1 = st.stat("tc_rows"), st.stat("batches")
        got = st.scan_topk_filtered(metric, q, k, full, as_arrays=True)
        _assert_same(got, want, (window, metric, k))
        assert (st.stat("tc_rows") - rows1, st.stat("batches") - b1) == (rows1 - rows0, b1 - b0), (window, metric)   # the same schedule
        _assert_same(st.scan_topk_filtered(metric, q[:1], k, full, as_arrays=True), st.scan_topk(metric, q[:1], k, as_arrays=True), (window, k))
    st.close()


@pytest.mark.parametrize("ngpus", [1, 3])
def test_all_eligible_group_equals_unfiltered(ngpus):
    rng = np.random.Generator(np.random.PCG64(9200 + ngpus))
    n, dim = 30_001, 32
    x = _column(po.I8, n, dim, rng)
    g = _group(po.I8, x, ngpus)
    full = np.ones(n, bool)
    q = _column(po.I8, 20, dim, rng)
    for metric in METRICS:
        for qq, k in ((q, 20), (q[:1], 20), (q[:1], 300)):
            got, want = g.scan_topk_filtered(metric, qq, k, full), g.scan_topk(metric, qq, k)
            assert len(got) == len(want) == len(qq)
            for (a_ids, a_d), (b_ids, b_d) in zip(got, want):
                assert np.array_equal(a_ids, b_ids) and np.array_equal(_bits(a_d), _bits(b_d)), (ngpus, metric, k)
    g.close()


# ------------------------------------------------------------------------------------------------ (2) the oracle on the sub-column
@pytest.mark.parametrize("dim", [5, 128, 771])
@pytest.mark.parametrize("vtype", TYPES)
def test_single_query_matches_oracle_on_sub_column(oracle, vtype, dim):
    rng = np.random.Generator(np.random.PCG64(9300 + 10 * vtype + dim))
    n = 4000
    x = _column(vtype, n, dim, rng)
    rowids = np.arange(n, dtype=np.int64) * 2 + 5
    ix = _index(vtype, x, rowids)
    for metric in METRICS:
        q = _column(vtype, 1, dim, rng)[0]
        for k in (1, 20, 100, 256, 300):
            for name, m in masks(n, k, rng).items():
                ((ids, d),) = ix.scan_topk_filtered(metric, q, k, m)
                _check_sub(oracle, vtype, metric, x, rowids, m, q, k, ids, d, (vtype, dim, metric, k, name))
    ix.close()


# ------------------------------------------------------------------------------------------------ (3) the batch path runs
@pytest.mark.parametrize("nq", [16, 1024])
def test_filtered_batch_runs_and_equals_single_calls(oracle, nq):
    rng = np.random.Generator(np.random.PCG64(9400 + nq))
    n, dim, k = 20_000, 64, 20
    x = _column(po.I8, n, dim, rng)
    rowids = np.arange(n, dtype=np.int64) + 1
    ix = _index(po.I8, x, rowids)
    q = _column(po.I8, nq, dim, rng)
    for name, m in masks(n, k, rng).items():
        for metric in (po.L2, po.L1):
            b0, f0 = ix.stat("batches"), ix.stat("fallbacks")
            got = ix.scan_topk_filtered(metric, q, k, m, as_arrays=True)
            assert ix.stat("batches") == b0 + 1 and ix.stat("fallbacks") == f0, (name, metric)
            for b in range(0, nq, max(1, nq // 32)):
                c = int(got[2][b])
                ((ids, d),) = ix.scan_topk_filtered(metric, q[b], k, m)
                assert np.array_equal(ids, got[0][b, :c]) and np.array_equal(d, got[1][b, :c]), (name, metric, b)
                if b % 8 == 0:
                    _check_sub(oracle, po.I8, metric, x, rowids, m, q[b], k, ids, d, (name, metric, b))
    ix.close()


def test_bucket_overflow_falls_back_and_stays_exact(oracle):
    """f32 L1 rows that each come closer to the queries than every row before them: a level's eligible rows all beat the
    bound, more than a bucket holds; the batch reports the overflow and the per-query filtered loop answers"""
    n, dim, nq, k = 40_000, 8, 16, 20
    x = np.zeros((n, dim), np.float32)
    x[:, 0] = np.arange(n, 0, -1, dtype=np.float32)
    q = np.zeros((nq, dim), np.float32)
    q[:, 1] = np.arange(nq, dtype=np.float32)
    rng = np.random.Generator(np.random.PCG64(9500))
    m = rng.random(n) < 0.5
    ix = _index(po.F32, x)
    f0, b0 = ix.stat("fallbacks"), ix.stat("batches")
    got = ix.scan_topk_filtered(po.L1, q, k, m, as_arrays=True)
    assert ix.stat("fallbacks") > f0 and ix.stat("batches") == b0
    ids = np.arange(1, n + 1, dtype=np.int64)
    for b in range(nq):
        c = int(got[2][b])
        _check_sub(oracle, po.F32, po.L1, x, ids, m, q[b], k, got[0][b, :c], got[1][b, :c], b)
    ix.close()


# ------------------------------------------------------------------------------------------------ (4) poisoned rows
@pytest.mark.parametrize("metric", [po.L2, po.COS, po.L1])
def test_poisoned_ineligible_rows_never_hit(oracle, metric):
    rng = np.random.Generator(np.random.PCG64(9600 + metric))
    n, dim, nq, k = 30_000, 64, 64, 20
    q = _column(po.I8, nq, dim, rng)
    clean = _column(po.I8, n, dim, rng)
    m = rng.random(n) < 0.1
    poisoned = clean.copy()
    bad = np.flatnonzero(~m)
    poisoned[bad] = q[bad % nq]                          # every ineligible row is a copy of a query: distance 0, far below U
    ids = np.arange(1, n + 1, dtype=np.int64)
    cands = {}
    for name, x in (("clean", clean), ("poisoned", poisoned)):
        ix = _index(po.I8, x)
        c0, f0 = ix.stat("batch_cands"), ix.stat("fallbacks")
        got = ix.scan_topk_filtered(metric, q, k, m, as_arrays=True)
        cands[name] = ix.stat("batch_cands") - c0
        assert ix.stat("fallbacks") == f0, name
        for b in range(nq):
            c = int(got[2][b])
            assert np.all(m[got[0][b, :c] - 1]), (name, b)
            if b % 8 == 0:
                _check_sub(oracle, po.I8, metric, x, ids, m, q[b], k, got[0][b, :c], got[1][b, :c], (name, b))
        ix.close()
    assert cands["poisoned"] <= 2 * cands["clean"] + 1000, cands


# ------------------------------------------------------------------------------------------------ (5) streamed and groups
def _clustered(n, rng):
    out = {}
    for name, blocks in (("cross", [(4990, 5300), (9990, 10020)]), ("late", [(n - 700, n - 600)]), ("sparse_late", [(n - 3, n)])):
        m = np.zeros(n, bool)
        for a, b in blocks:
            m[a:b] = True
        out[name] = m
    out["random0.01"] = rng.random(n) < 0.01
    return out


@pytest.mark.parametrize("window", [128, 300, 5000])
def test_streamed_clustered_masks_equal_resident(window):
    rng = np.random.Generator(np.random.PCG64(9700 + window))
    n, dim = 15_000, 32
    x = _column(po.I8, n, dim, rng)
    res, st = _index(po.I8, x), _index(po.I8, x, window=window)
    q = _column(po.I8, 24, dim, rng)
    for name, m in _clustered(n, rng).items():
        for metric, k in ((po.L2, 20), (po.L1, 100)):
            f0 = st.stat("fallbacks")
            _assert_same(st.scan_topk_filtered(metric, q, k, m, as_arrays=True), res.scan_topk_filtered(metric, q, k, m, as_arrays=True), (window, name, metric))
            assert st.stat("fallbacks") == f0, (window, name, metric)
            _assert_same(st.scan_topk_filtered(metric, q[:1], 300, m, as_arrays=True), res.scan_topk_filtered(metric, q[:1], 300, m, as_arrays=True), (window, name))
    res.close()
    st.close()


@pytest.mark.parametrize("ngpus", [2, 3])
def test_group_clustered_masks_equal_single_index(ngpus):
    rng = np.random.Generator(np.random.PCG64(9800 + ngpus))
    n, dim = 30_001, 32                                   # shard boundaries 10000 / 20000 (3 shards) or 15000 (2): not multiples of 32
    x = _column(po.I8, n, dim, rng)
    rowids = np.arange(n, dtype=np.int64) * 5 + 3
    ix, g = _index(po.I8, x, rowids), _group(po.I8, x, ngpus, rowids)
    q = _column(po.I8, 20, dim, rng)
    ms = _clustered(n, rng)
    for a in (9999, 14999, 19999):
        b = np.zeros(n, bool)
        b[a - 40:a + 41] = True
        ms[f"boundary{a}"] = b
    for name, m in ms.items():
        for metric, qq, k in ((po.L2, q, 20), (po.DOT, q[:1], 20), (po.L1, q[:1], 300)):
            want = ix.scan_topk_filtered(metric, qq, k, m)
            got = g.scan_topk_filtered(metric, qq, k, m)
            for (a_ids, a_d), (b_ids, b_d) in zip(got, want):
                assert np.array_equal(a_ids, b_ids) and np.array_equal(_bits(a_d), _bits(b_d)), (ngpus, name, metric)
    ix.close()
    g.close()


@pytest.mark.parametrize("ngpus", [1, 3])
def test_rowid_bitmaps_match_isin(ngpus):
    rng = np.random.Generator(np.random.PCG64(9900 + ngpus))
    n, dim = 9_001, 8
    x = _column(po.I8, n + 500, dim, rng)
    explicit = rng.permutation(100_000)[: n + 500].astype(np.int64)
    for rowids in (explicit, None):
        g = _vs().Group(po.I8, dim, n + 500, ngpus)
        ix = _vs().Index(po.I8, dim, n + 500)
        for obj in (g, ix):
            obj.append_dense(x[:n], None if rowids is None else rowids[:n])
        ids = np.arange(1, n + 501, dtype=np.int64) if rowids is None else rowids
        for step in range(2):
            rows = n + 500 * step
            ask = np.concatenate([rng.choice(ids[:rows], 700), rng.integers(-5, 200_000, 300), ids[:5], ids[:5]])   # absent ids, duplicates
            want = np.isin(ids[:rows], ask)
            for obj in (g, ix):
                bits, cnt = obj.rowid_bitmap(ask)
                got = np.array([(int(bits[i >> 5]) >> (i & 31)) & 1 for i in range(rows)], dtype=bool)
                assert np.array_equal(got, want) and cnt == int(want.sum()), (ngpus, rowids is None, step)
            if step == 0:
                for obj in (g, ix):                    # after an append the lookup covers the new rows
                    obj.append_dense(x[n:], None if rowids is None else rowids[n:])
        g.close()
        ix.close()


# ------------------------------------------------------------------------------------------------ (6) SQL
def test_sql_filtered_modules_match_oracle(oracle):
    rng = np.random.Generator(np.random.PCG64(10_000))
    n, dim, k = 9000, 16, 10
    x = rng.integers(-40, 41, (n, dim)).astype(np.int8)
    ids = np.arange(n, dtype=np.int64) * 2 + 1
    lang = np.where(rng.random(n) < 0.05, "en", "de")
    q = rng.integers(-40, 41, (20, dim)).astype(np.int8)
    qb, allq = {"hex": q[0].tobytes().hex()}, {"hex": q.tobytes().hex()}
    s = ["CREATE TABLE t (id INTEGER PRIMARY KEY, e BLOB, lang TEXT)", f"SELECT vector_init('t','e','type=INT8,dimension={dim}')"]
    s += [["INSERT INTO t(id, e, lang) VALUES (?, ?, ?)", [int(ids[i]), {"hex": x[i].tobytes().hex()}, str(lang[i])]] for i in range(n)]
    mark = len(s)
    sub = "(SELECT vector_rowid_set(id) FROM t WHERE lang = 'en')"
    extra = np.concatenate([ids[lang == "en"][:30], ids[lang == "en"][:30], [10**9, -4]]).astype("<i8")
    s += [["SELECT id, distance FROM vector_full_scan_filtered('t','e',?,?," + sub + ")", [qb, k]],                          # 0
          ["SELECT query, id, distance FROM vector_full_scan_batch_filtered('t','e',?,?," + sub + ")", [allq, k]],           # 1
          ["SELECT id, distance FROM vector_full_scan_filtered('t','e',?,?,?)", [qb, k, {"hex": extra.tobytes().hex()}]],   # 2 absent + duplicates
          ["SELECT id, distance FROM vector_full_scan_filtered('t','e',?,?,x'')", [qb, k]],                                 # 3 empty set
          ["SELECT id, distance FROM vector_full_scan_filtered('t','e',?,0," + sub + ")", [qb]],                             # 4 k = 0
          "BEGIN",                                                                                                           # 5
          ["INSERT INTO t(id, e, lang) VALUES (100001, ?, 'en')", [qb]],                                                     # 6
          ["SELECT id, distance FROM vector_full_scan_filtered('t','e',?,3," + sub + ")", [qb]],                             # 7 sees it
          "ROLLBACK",                                                                                                        # 8
          ["SELECT id, distance FROM vector_full_scan_filtered('t','e',?,3," + sub + ")", [qb]],                             # 9 must not
          "SELECT vector_quantize('t','e')",                                                                                 # 10
          ["SELECT id, distance FROM vector_quantize_scan_filtered('t','e',?,?," + sub + ")", [qb, k]],                      # 11
          ["SELECT query, id, distance FROM vector_quantize_scan_batch_filtered('t','e',?,?," + sub + ")", [allq, k]],       # 12
          ["SELECT id, distance FROM vector_quantize_scan('t','e',?,?)", [qb, k]]]                                           # 13
    r = run_sql(OURS, s)[mark:]
    en = lang == "en"

    def want(qv, kk, m):
        a, d = oracle.scan_dense(po.L2, po.I8, qv, x[m], ids[m], kk)
        return [[int(i), float(v)] for i, v in zip(a, d)]
    assert r[0]["rows"] == want(q[0], k, en)
    for b in range(20):
        assert [row[1:] for row in r[1]["rows"] if row[0] == b] == want(q[b], k, en), b
    assert r[2]["rows"] == want(q[0], k, np.isin(ids, extra))
    assert r[3]["rows"] == [] and r[4]["rows"] == []
    assert r[7]["rows"][0] == [100001, 0.0]
    assert r[9]["rows"] == want(q[0], 3, en)
    assert len(r[11]["rows"]) == k and {row[0] for row in r[11]["rows"]} <= set(ids[en].tolist())
    assert [row[1:] for row in r[12]["rows"] if row[0] == 0] == r[11]["rows"]
    assert r[13]["rows"] != r[11]["rows"]


# ------------------------------------------------------------------------------------------------ (7) handles
def test_filtered_calls_leave_no_handles():
    eng = _vs().load_engine()
    rng = np.random.Generator(np.random.PCG64(10_100))
    n, dim = 12_000, 32
    x = _column(po.I8, n, dim, rng)
    q = _column(po.I8, 20, dim, rng)
    m = rng.random(n) < 0.3
    base = eng.debug_live_handles()
    for make in (lambda: _index(po.I8, x), lambda: _index(po.I8, x, window=1000), lambda: _group(po.I8, x, 3)):
        obj = make()
        obj.scan_topk_filtered(po.L2, q, 20, m)
        obj.scan_topk_filtered(po.L2, q[:1], 300, m)
        obj.close()
        assert eng.debug_live_handles() == base
