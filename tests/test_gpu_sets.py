"""Per-query eligible sets (vsb_scan_topk_sets and its group door): each query's k nearest among its own set of rows, in one pass
of the column.  Query b's result equals vsb_scan_topk_filtered over the same queries with b's set, bit for bit.  -m gpu.

(1) every set = every row: the unfiltered batch; one shared set: the filtered batch;
(2) distinct random sets per query for every (type, metric) pair the batch path admits, dims 5 / 128 / 771: the filtered batch
    under each query's set bit for bit, the oracle on the sub-column; the one-pass path ran (sets_batches) and did not fall back;
(3) poisoned rows (copies of a query that only other queries may see) never reach it and do not flood the candidate log, for
    tc_scan_kernel with the chunk test on and off and for l1_batch_kernel;
(4) edge sets: empty, fewer than k, single rows, ties, no rows in the first levels, 16 tenants as blocks and as partitions;
(5) a forced bucket overflow answers set by set; (6) streamed windows equal resident; (7) groups of 1 / 2 / 3 shards;
(8) the set-by-set path (nq < 16, k > 256, f32 with f32_batch off, the max_index carry), the level budget and the memory limit;
(9) SQL: vector_*_scan_batch_sets against vector_*_scan_batch_filtered per query, sparse and unnamed set indexes, NULL
    query_sets; argument errors; handles."""
import contextlib
import os

import numpy as np
import pytest

from oracle import pyoracle as po
from tests.fpcheck import assert_fp_topk

pytestmark = pytest.mark.gpu
METRICS = [po.L2, po.L2SQ, po.COS, po.DOT, po.L1]
TYPES = [po.F32, po.F16, po.BF16, po.U8, po.I8]
EINVAL = -1


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


def _group(vtype, x, ngpus, chunk=7919):
    g = _vs().Group(vtype, x.shape[1], x.shape[0], ngpus)
    for a in range(0, x.shape[0], chunk):
        g.append_dense(x[a:a + chunk])
    g.finalize()
    return g


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint64)


def _same_row(got, want, b, wb, ctx):
    """query b of as_arrays output `got` equals query wb of `want`, bit for bit"""
    c = int(want[2][wb])
    assert int(got[2][b]) == c, ctx
    assert np.array_equal(got[0][b, :c], want[0][wb, :c]), ctx
    assert np.array_equal(_bits(got[1][b, :c]), _bits(want[1][wb, :c])), ctx


def _per_set_reference(ix, metric, q, k, sets, soq):
    """each query's answer from vsb_scan_topk_filtered over ALL the queries with that query's set (one call per distinct set)"""
    want = {}
    for s in sorted(set(int(v) for v in soq)):
        want[s] = ix.scan_topk_filtered(metric, q, k, sets[s], as_arrays=True)
    return want


def _check_against_filtered(ix, metric, q, k, sets, soq, got, ctx):
    want = _per_set_reference(ix, metric, q, k, sets, soq)
    for b in range(q.shape[0]):
        _same_row(got, want[int(soq[b])], b, b, (ctx, b))


def _check_sub(oracle, vtype, metric, x, ids, mask, q, k, got_ids, got_d, ctx):
    want_ids, want_d = oracle.scan_dense(metric, vtype, q, x[mask], ids[mask], k)
    if vtype in (po.I8, po.U8):
        assert np.array_equal(got_ids, want_ids) and np.array_equal(got_d, want_d), ctx
    else:
        pos = {int(r): i for i, r in enumerate(ids)}
        assert_fp_topk(got_ids, got_d, want_ids, want_d, metric, lambda r: oracle.distance(metric, vtype, q, x[pos[int(r)]]), ctx)
    assert set(got_ids.tolist()) <= set(ids[mask].tolist()), ctx


def _sets_call(ix, metric, q, k, sets, soq=None, expect_batch=True):
    b0, f0 = ix.stat("sets_batches"), ix.stat("sets_fallbacks")
    got = ix.scan_topk_sets(metric, q, k, sets, soq, as_arrays=True)
    if expect_batch:
        assert (ix.stat("sets_batches"), ix.stat("sets_fallbacks")) == (b0 + 1, f0), (metric, k)
    return got


def _admitted(vtype, metric):
    return not (vtype == po.F32 and metric != po.L1)   # f32 L2 / cosine / dot batch only with f32_batch on


# ------------------------------------------------------------------------------------------------ (1) trivial sets
@pytest.mark.parametrize("vtype", TYPES)
def test_every_row_equals_unfiltered_batch(vtype):
    rng = np.random.Generator(np.random.PCG64(12000 + vtype))
    n, dim = 20_000, 64
    x = _column(vtype, n, dim, rng)
    ix = _index(vtype, x, np.arange(n, dtype=np.int64) * 3 + 7)
    full = np.ones(n, bool)
    for nq in (16, 1024):
        q = _column(vtype, nq, dim, rng)
        for metric in METRICS:
            with _options(f32_batch=1 if vtype == po.F32 else 0):
                want = ix.scan_topk(metric, q, 20, as_arrays=True)
                got = _sets_call(ix, metric, q, 20, [full], np.zeros(nq, np.int32))
            for b in range(nq):
                _same_row(got, want, b, b, (vtype, nq, metric))
    ix.close()


def test_one_shared_set_equals_filtered_batch():
    rng = np.random.Generator(np.random.PCG64(12100))
    n, dim, nq = 30_000, 96, 64
    x = _column(po.I8, n, dim, rng)
    ix = _index(po.I8, x)
    q = _column(po.I8, nq, dim, rng)
    m = rng.random(n) < 0.1
    for metric in METRICS:
        got = _sets_call(ix, metric, q, 20, [m], np.zeros(nq, np.int32))
        want = ix.scan_topk_filtered(metric, q, 20, m, as_arrays=True)
        for b in range(nq):
            _same_row(got, want, b, b, metric)
    ix.close()


# ------------------------------------------------------------------------------------------------ (2) distinct random sets
@pytest.mark.parametrize("dim", [5, 128, 771])
@pytest.mark.parametrize("vtype", TYPES)
def test_distinct_random_sets(oracle, vtype, dim):
    rng = np.random.Generator(np.random.PCG64(12200 + 10 * vtype + dim))
    n, nq, k = 12_000, 24, 20
    x = _column(vtype, n, dim, rng)
    ids = np.arange(n, dtype=np.int64) * 2 + 5
    ix = _index(vtype, x, ids)
    q = _column(vtype, nq, dim, rng)
    fracs = [0.5, 0.1, 0.02, 0.005]
    sets = [rng.random(n) < fracs[i % len(fracs)] for i in range(nq)]
    for metric in METRICS:
        for f32_batch in ((0, 1) if vtype == po.F32 else (0,)):
            with _options(f32_batch=f32_batch):
                admitted = _admitted(vtype, metric) or f32_batch == 1
                got = _sets_call(ix, metric, q, k, sets, None, expect_batch=admitted)
                _check_against_filtered(ix, metric, q, k, sets, np.arange(nq), got, (vtype, dim, metric, f32_batch))
            for b in range(0, nq, 5):
                c = int(got[2][b])
                _check_sub(oracle, vtype, metric, x, ids, sets[b], q[b], k, got[0][b, :c], got[1][b, :c], (vtype, dim, metric, b))
    ix.close()


def test_1024_queries_with_shared_and_distinct_sets(oracle):
    rng = np.random.Generator(np.random.PCG64(12300))
    n, dim, nq, k = 40_000, 64, 1024, 20
    x = _column(po.I8, n, dim, rng)
    ids = np.arange(1, n + 1, dtype=np.int64)
    ix = _index(po.I8, x)
    q = _column(po.I8, nq, dim, rng)
    sets = [rng.random(n) < 0.1 for _ in range(300)]
    soq = rng.integers(0, 300, nq).astype(np.int32)
    for metric in (po.L2, po.DOT, po.L1):
        got = _sets_call(ix, metric, q, k, sets, soq)
        _check_against_filtered(ix, metric, q, k, sets, soq, got, metric)
        for b in range(0, nq, 97):
            c = int(got[2][b])
            _check_sub(oracle, po.I8, metric, x, ids, sets[soq[b]], q[b], k, got[0][b, :c], got[1][b, :c], (metric, b))
    ix.close()


# ------------------------------------------------------------------------------------------------ (3) poisoned rows
@pytest.mark.parametrize("metric,chunk", [(po.L2, 1), (po.L2, 0), (po.COS, 1), (po.DOT, 0), (po.L1, 0)])
def test_poisoned_rows_of_other_queries_never_hit(oracle, metric, chunk):
    """every query's set holds 10 % clean rows; every other row is an exact copy of some query and belongs only to the sets of
    the OTHER queries (the set of the query it copies excludes it)"""
    rng = np.random.Generator(np.random.PCG64(12400 + 10 * metric + chunk))
    n, dim, nq, k = 30_000, 64, 64, 20
    q = _column(po.I8, nq, dim, rng)
    x = _column(po.I8, n, dim, rng)
    base = rng.random(n) < 0.1
    copies = np.flatnonzero(~base)
    of = copies % nq
    x[copies] = q[of]
    sets = []
    for b in range(nq):
        m = base.copy()
        m[copies[(of != b) & (rng.random(copies.size) < 0.02)]] = True      # some copies of the other queries
        sets.append(m)
    ids = np.arange(1, n + 1, dtype=np.int64)
    cands = {}
    for name, col in (("clean", _column(po.I8, n, dim, rng)), ("poisoned", x)):
        ix = _index(po.I8, col)
        with _options(epi_chunk=chunk):
            c0 = ix.stat("batch_cands")
            got = _sets_call(ix, metric, q, k, sets)
            cands[name] = ix.stat("batch_cands") - c0
        for b in range(nq):
            c = int(got[2][b])
            assert np.all(sets[b][got[0][b, :c] - 1]), (name, b)
            if b % 8 == 0:
                _check_sub(oracle, po.I8, metric, col, ids, sets[b], q[b], k, got[0][b, :c], got[1][b, :c], (name, b))
        ix.close()
    assert cands["poisoned"] <= 2 * cands["clean"] + 1000, cands


# ------------------------------------------------------------------------------------------------ (4) edge sets
def test_edge_sets(oracle):
    rng = np.random.Generator(np.random.PCG64(12500))
    n, dim, nq, k = 20_000, 32, 32, 20
    x = rng.integers(-2, 3, (n, dim)).astype(np.int8)          # tie-heavy
    ids = np.arange(1, n + 1, dtype=np.int64)
    ix = _index(po.I8, x)
    q = rng.integers(-2, 3, (nq, dim)).astype(np.int8)
    late = np.zeros(n, bool)
    late[n - 3000:] = rng.random(3000) < 0.3                   # no rows in the first levels
    single = np.zeros(n, bool)
    single[12345] = True
    few = np.zeros(n, bool)
    few[rng.choice(n, k // 2, replace=False)] = True
    sets = [np.zeros(n, bool), few, single, late, rng.random(n) < 0.2, np.ones(n, bool)]
    soq = np.arange(nq, dtype=np.int32) % len(sets)
    for metric in METRICS:
        got = _sets_call(ix, metric, q, k, sets, soq)
        _check_against_filtered(ix, metric, q, k, sets, soq, got, metric)
        for b in range(nq):
            c = int(got[2][b])
            assert c == min(k, int(sets[soq[b]].sum())), (metric, b)
            _check_sub(oracle, po.I8, metric, x, ids, sets[soq[b]], q[b], k, got[0][b, :c], got[1][b, :c], (metric, b))
    ix.close()


@pytest.mark.parametrize("layout", ["blocks", "partitions"])
def test_tenants(layout):
    rng = np.random.Generator(np.random.PCG64(12600 + len(layout)))
    n, dim, nq, k, T = 200_000, 32, 256, 20, 16
    x = _column(po.I8, n, dim, rng)
    ix = _index(po.I8, x)
    q = _column(po.I8, nq, dim, rng)
    tenant = (np.arange(n) * T // n) if layout == "blocks" else rng.integers(0, T, n)
    sets = [tenant == t for t in range(T)]
    soq = (np.arange(nq) // (nq // T)).astype(np.int32)
    got = _sets_call(ix, po.L2, q, k, sets, soq)
    levels = ix.stat("sets_levels")
    assert 0 < levels <= 256, levels
    _check_against_filtered(ix, po.L2, q, k, sets, soq, got, layout)
    ix.close()


# ------------------------------------------------------------------------------------------------ (5) forced fallback
def test_bucket_overflow_answers_set_by_set(oracle):
    """f32 L1 rows that each come closer to the queries than every row before them overflow a bucket (as in the filtered
    tests): the call answers set by set and stays exact"""
    n, dim, nq, k = 40_000, 8, 16, 20
    x = np.zeros((n, dim), np.float32)
    x[:, 0] = np.arange(n, 0, -1, dtype=np.float32)
    q = np.zeros((nq, dim), np.float32)
    q[:, 1] = np.arange(nq, dtype=np.float32)
    rng = np.random.Generator(np.random.PCG64(12700))
    sets = [rng.random(n) < 0.5, rng.random(n) < 0.7]
    soq = (np.arange(nq) % 2).astype(np.int32)
    ix = _index(po.F32, x)
    b0, f0 = ix.stat("sets_batches"), ix.stat("sets_fallbacks")
    got = ix.scan_topk_sets(po.L1, q, k, sets, soq, as_arrays=True)
    assert (ix.stat("sets_batches"), ix.stat("sets_fallbacks")) == (b0, f0 + 1)
    ids = np.arange(1, n + 1, dtype=np.int64)
    for b in range(nq):
        c = int(got[2][b])
        _check_sub(oracle, po.F32, po.L1, x, ids, sets[soq[b]], q[b], k, got[0][b, :c], got[1][b, :c], b)
    ix.close()


def test_level_budget_and_memory_limit_answer_set_by_set(oracle):
    """256 tenants owning contiguous blocks need more than 256 levels in one view (each block restarts its set at m0 rows); a
    device memory limit below the call's buffers (option sets_mem_mb) refuses the upload.  Both answer set by set, exactly."""
    rng = np.random.Generator(np.random.PCG64(12750))
    n, dim, T, k = 200_000, 16, 256, 10
    x = _column(po.I8, n, dim, rng)
    ids = np.arange(1, n + 1, dtype=np.int64)
    ix = _index(po.I8, x)
    q = _column(po.I8, T, dim, rng)
    owner = np.arange(n) * T // n
    sets = [owner == t for t in range(T)]
    soq = np.arange(T, dtype=np.int32)
    for opts in ({}, {"sets_mem_mb": 1}):
        with _options(**opts):
            b0, f0 = ix.stat("sets_batches"), ix.stat("sets_fallbacks")
            got = ix.scan_topk_sets(po.L2, q, k, sets, soq, as_arrays=True)
            assert (ix.stat("sets_batches"), ix.stat("sets_fallbacks")) == (b0, f0 + 1), opts
        for b in range(0, T, 17):
            c = int(got[2][b])
            _check_sub(oracle, po.I8, po.L2, x, ids, sets[b], q[b], k, got[0][b, :c], got[1][b, :c], (opts, b))
    # 64 tenants fit the budget and the memory: one pass
    got = _sets_call(ix, po.L2, q[:64], k, [owner // 4 == t for t in range(64)], np.arange(64, dtype=np.int32))
    assert ix.stat("sets_levels") <= 256
    ix.close()


# ------------------------------------------------------------------------------------------------ (6) streamed windows
@pytest.mark.parametrize("window", [128, 300, 5000])
def test_streamed_equals_resident(window):
    rng = np.random.Generator(np.random.PCG64(12800 + window))
    n, dim, nq, k = 12_000, 64, 40, 20
    x = _column(po.I8, n, dim, rng)
    res, st = _index(po.I8, x), _index(po.I8, x, window=window)
    q = _column(po.I8, nq, dim, rng)
    blocks = np.zeros(n, bool)
    blocks[4990:5300] = True
    blocks[n - 700:n - 600] = True
    sets = [rng.random(n) < 0.1, blocks, rng.random(n) < 0.01, np.arange(n) % 7 == 0]
    soq = (np.arange(nq) % len(sets)).astype(np.int32)
    for metric in (po.L2, po.DOT, po.L1):
        want = _sets_call(res, metric, q, k, sets, soq)
        s0 = st.stat("stream_bytes")
        got = _sets_call(st, metric, q, k, sets, soq)
        assert st.stat("stream_bytes") - s0 == n * st.query_pitch, (window, metric)   # one pass of the column
        for b in range(nq):
            _same_row(got, want, b, b, (window, metric))
    res.close()
    st.close()


# ------------------------------------------------------------------------------------------------ (7) groups
def _shard0_stat(g, name):
    lib = g.eng.lib
    return int(lib.vsb_index_stat(lib.vsb_group_shard(g.h, 0), name.encode()))


def _group_sets_call(g, metric, q, k, sets, soq):
    """the group's call, which must take the one-pass path (its counters live on shard 0)"""
    b0, f0 = _shard0_stat(g, "sets_batches"), _shard0_stat(g, "sets_fallbacks")
    got = g.scan_topk_sets(metric, q, k, sets, soq, as_arrays=True)
    assert (_shard0_stat(g, "sets_batches"), _shard0_stat(g, "sets_fallbacks")) == (b0 + 1, f0), metric
    return got


@pytest.mark.parametrize("ngpus", [1, 2, 3])
def test_group_equals_single_index(ngpus):
    rng = np.random.Generator(np.random.PCG64(12900 + ngpus))
    n, dim, nq, k = 30_001, 32, 32, 20
    x = _column(po.I8, n, dim, rng)
    ix, g = _index(po.I8, x), _group(po.I8, x, ngpus)
    q = _column(po.I8, nq, dim, rng)
    sets = [rng.random(n) < f for f in (0.3, 0.05, 0.01)] + [np.arange(n) >= 20_000]
    soq = (np.arange(nq) % len(sets)).astype(np.int32)
    for metric in (po.L2, po.COS, po.L1):
        want = ix.scan_topk_sets(metric, q, k, sets, soq, as_arrays=True)
        got = _group_sets_call(g, metric, q, k, sets, soq)
        for b in range(nq):
            _same_row(got, want, b, b, (ngpus, metric))
    ix.close()
    g.close()


def test_group_with_a_streamed_shard_equals_single_index():
    rng = np.random.Generator(np.random.PCG64(12950))
    n, dim, nq, k = 30_000, 32, 32, 20
    x = _column(po.I8, n, dim, rng)
    ix = _index(po.I8, x)
    pitch = 32
    old = os.environ.get("VSB_DEVICE_BUDGET_MB")
    os.environ["VSB_DEVICE_BUDGET_MB"] = str(12_000 * pitch / 1048576.0)   # the 10 000-row shards fit, 15 000 do not
    try:
        g = _group(po.I8, x, 2)
    finally:
        if old is None:
            os.environ.pop("VSB_DEVICE_BUDGET_MB", None)
        else:
            os.environ["VSB_DEVICE_BUDGET_MB"] = old
    q = _column(po.I8, nq, dim, rng)
    sets = [rng.random(n) < f for f in (0.3, 0.05)]
    soq = (np.arange(nq) % 2).astype(np.int32)
    for metric in (po.L2, po.L1):
        want = ix.scan_topk_sets(metric, q, k, sets, soq, as_arrays=True)
        got = _group_sets_call(g, metric, q, k, sets, soq)
        for b in range(nq):
            _same_row(got, want, b, b, metric)
    ix.close()
    g.close()


# ------------------------------------------------------------------------------------------------ SQL
def test_sql_sets_modules_equal_filtered_batches():
    from tests.sqlrun import OURS, run_sql
    rng = np.random.Generator(np.random.PCG64(12980))
    n, dim, k, nq = 9000, 16, 10, 20
    x = rng.integers(-40, 41, (n, dim)).astype(np.int8)
    ids = np.arange(n, dtype=np.int64) * 2 + 1
    tenant = rng.integers(0, 5, n) * 7 + 3                    # sparse set indexes 3, 10, 17, 24, 31
    q = rng.integers(-40, 41, (nq, dim)).astype(np.int8)
    allq = {"hex": q.tobytes().hex()}
    qsets = (np.arange(nq) % 6 * 7 + 3).astype("<i8")        # 38: a set that no pair names (empty)
    s = ["CREATE TABLE t (id INTEGER PRIMARY KEY, e BLOB, tenant INTEGER)", f"SELECT vector_init('t','e','type=INT8,dimension={dim}')"]
    s += [["INSERT INTO t(id, e, tenant) VALUES (?, ?, ?)", [int(ids[i]), {"hex": x[i].tobytes().hex()}, int(tenant[i])]] for i in range(n)]
    s += ["SELECT vector_quantize('t','e')"]
    mark = len(s)
    sets = "(SELECT vector_rowid_sets(tenant, id) FROM t)"
    byset = lambda t: f"(SELECT vector_rowid_set(id) FROM t WHERE tenant = {t})"
    for mod in ("full", "quantize"):
        s += [["SELECT query, id, distance FROM vector_%s_scan_batch_sets('t','e',?,?,%s,?)" % (mod, sets), [allq, k, {"hex": qsets.tobytes().hex()}]]]
        s += [["SELECT query, id, distance FROM vector_%s_scan_batch_filtered('t','e',?,?,%s)" % (mod, byset(t)), [allq, k]] for t in (3, 10, 17, 24, 31, 38)]
    # NULL query_sets: query b uses set b (dense 0..4 over sets 0..4; here the first 5 queries, set b = tenant index b)
    s += [["SELECT query, id, distance FROM vector_full_scan_batch_sets('t','e',?,?,(SELECT vector_rowid_sets((tenant - 3) / 7, id) FROM t),NULL)",
           [{"hex": q[:5].tobytes().hex()}, k]]]
    s += [["SELECT query, id, distance FROM vector_full_scan_batch_filtered('t','e',?,?,%s)" % byset(3 + 7 * b), [{"hex": q[:5].tobytes().hex()}, k]]
          for b in range(5)]
    r = run_sql(OURS, s)[mark:]
    for m in range(2):
        got, want = r[7 * m], r[7 * m + 1:7 * m + 7]
        assert "rows" in got, got
        for b in range(nq):
            t = (int(qsets[b]) - 3) // 7
            assert [row[1:] for row in got["rows"] if row[0] == b] == [row[1:] for row in want[t]["rows"] if row[0] == b], (m, b)
        assert not any(row[0] % 6 == 5 for row in got["rows"])           # the empty set gives no rows
    got = r[14]
    for b in range(5):
        assert [row[1:] for row in got["rows"] if row[0] == b] == [row[1:] for row in r[15 + b]["rows"] if row[0] == b], b


# ------------------------------------------------------------------------------------------------ (8) set by set, errors, handles
def test_set_by_set_paths():
    rng = np.random.Generator(np.random.PCG64(13000))
    n, dim = 20_000, 48
    x8 = _column(po.I8, n, dim, rng)
    xf = _column(po.F32, n, dim, rng)
    i8, f32 = _index(po.I8, x8), _index(po.F32, xf)
    sets = [rng.random(n) < 0.2, rng.random(n) < 0.05]
    for ix, x, vtype, metric, nq, k in ((i8, x8, po.I8, po.L2, 8, 20), (i8, x8, po.I8, po.L2, 32, 300), (f32, xf, po.F32, po.L2, 32, 20)):
        q = _column(vtype, nq, dim, rng)
        soq = (np.arange(nq) % 2).astype(np.int32)
        b0, f0 = ix.stat("sets_batches"), ix.stat("sets_fallbacks")
        got = ix.scan_topk_sets(metric, q, k, sets, soq, as_arrays=True)
        assert (ix.stat("sets_batches"), ix.stat("sets_fallbacks")) == (b0, f0), (nq, k)   # not admitted: not a fallback
        _check_against_filtered(ix, metric, q, k, sets, soq, got, (vtype, nq, k))
    # the max_index carry of one query: the C ABI with a cursor equals the filtered call with the same cursor
    vs = _vs()
    lib = i8.eng.lib
    import ctypes as C
    q1 = np.ascontiguousarray(_column(po.I8, 1, dim, rng))
    flat = np.ascontiguousarray(np.stack([vs.api.row_bitmap(s) for s in sets]))
    soq1 = np.array([1], np.int32)
    mi_a = mi_b = 0
    for k in (100, 10, 33):
        ids = np.zeros(k, np.int64); d = np.zeros(k); cnt = np.zeros(1, np.int32); mi = C.c_int(mi_a)
        i8.eng.check(lib.vsb_scan_topk_sets(i8.h, po.L2, q1.ctypes.data, 1, k, flat.ctypes.data, 2, n, soq1.ctypes.data,
                                            ids.ctypes.data, d.ctypes.data, cnt.ctypes.data, C.byref(mi)))
        mi_a = mi.value
        ((want_ids, want_d),), mi_b = i8.scan_topk_filtered(po.L2, q1[0], k, sets[1], max_index=mi_b)
        assert np.array_equal(ids[:cnt[0]], want_ids) and np.array_equal(d[:cnt[0]], want_d) and mi_a == mi_b, k
    i8.close()
    f32.close()


def test_argument_errors():
    vs = _vs()
    rng = np.random.Generator(np.random.PCG64(13100))
    n, dim = 1000, 16
    ix = _index(po.I8, _column(po.I8, n, dim, rng))
    q = _column(po.I8, 4, dim, rng)
    lib = ix.eng.lib
    bits = np.ascontiguousarray(np.stack([vs.api.row_bitmap(np.ones(n, bool))] * 4))
    out_i = np.zeros(4 * 5, np.int64); out_d = np.zeros(4 * 5); cnt = np.zeros(4, np.int32)

    def call(sets_ptr, nsets, nbits, soq):
        return lib.vsb_scan_topk_sets(ix.h, po.L2, q.ctypes.data, 4, 5, sets_ptr, nsets, nbits,
                                      None if soq is None else soq.ctypes.data, out_i.ctypes.data, out_d.ctypes.data, cnt.ctypes.data, None)

    assert call(bits.ctypes.data, 4, n - 1, None) == EINVAL
    assert call(bits.ctypes.data, 4, n, np.array([0, 1, 2, 4], np.int32)) == EINVAL
    assert call(bits.ctypes.data, 4, n, np.array([0, -1, 2, 3], np.int32)) == EINVAL
    assert call(None, 4, n, None) == EINVAL
    assert call(bits.ctypes.data, 3, n, None) == EINVAL
    assert b"set" in lib.vsb_last_error()
    assert call(bits.ctypes.data, 4, n, None) == 0
    assert call(bits.ctypes.data, 1, n, np.zeros(4, np.int32)) == 0
    ix.close()


def test_sets_calls_leave_no_handles():
    eng = _vs().load_engine()
    rng = np.random.Generator(np.random.PCG64(13200))
    n, dim, nq = 20_000, 32, 32
    x = _column(po.I8, n, dim, rng)
    q = _column(po.I8, nq, dim, rng)
    sets = [rng.random(n) < 0.1 for _ in range(nq)]
    ix = _index(po.I8, x)
    ix.scan_topk_sets(po.L2, q, 20, sets)                     # workspaces of the batch and per-query paths exist from here on
    ix.scan_topk_sets(po.L2, q[:4], 20, sets, np.arange(4))
    h0 = eng.debug_live_handles()
    for _ in range(3):
        ix.scan_topk_sets(po.L2, q, 20, sets)
        ix.scan_topk_sets(po.L2, q[:4], 20, sets, np.arange(4))
    assert eng.debug_live_handles() == h0
    ix.close()
