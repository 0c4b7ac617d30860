"""Listed rows (vsb_scan_topk_rows and its group / SQL doors): the k nearest among a per-query list of rowids, reading only the
listed rows, equal bit for bit the filtered scan with the bitmap of each query's rowids.  -m gpu.

(1) every (type, metric) pair at dims 5 / 128 / 771, k from 1 to 1000 (the large-k path included), list sizes 0 .. 5000 with
    duplicates, absent and explicit non-contiguous rowids: rowids, order, distance bits and the returned max_index; the oracle on
    the sub-column (bit-exact for int8 / uint8); a max_index carried over k = 100 -> 10 -> 33;
(2) the shapes where the single-query plan switches between DIRECT and staged with k;
(3) NaN / +-Inf rows and queries, -INF dot distances, tie-heavy int8;
(4) batches of 16 and 1024 ragged lists equal single calls bit for bit, floating point included;
(5) streamed windows (128 rows, ragged): the filtered scan's results, the resident index's where the windows keep the warp tiles
    (int8, 128 rows), no window copy, rows_host_bytes = listed rows x pitch;
(6) groups of 1 and 3 shards, one of them streamed; (7) one kernel launch per shard, handles back to their baseline;
(8) SQL: vector_quantize_scan_rerank equals the composed filtered statement, the batch module the single one."""
import contextlib
import os

import numpy as np
import pytest

from oracle import pyoracle as po
from tests.sqlrun import OURS, run_sql

pytestmark = pytest.mark.gpu
METRICS = [po.L2, po.L2SQ, po.COS, po.DOT, po.L1]
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
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


@pytest.fixture(scope="module", autouse=True)
def _alias():
    with _env(VSB_GROUP_ALIAS="1"):
        yield


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


def _group(vtype, x, ngpus, rowids=None):
    g = _vs().Group(vtype, x.shape[1], x.shape[0], ngpus)
    g.append_dense(x, rowids)
    g.finalize()
    return g


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint64)


def _same(got, want, ctx):
    """two lists of (rowids, distances), bit for bit"""
    assert len(got) == len(want), ctx
    for b, ((gi, gd), (wi, wd)) in enumerate(zip(got, want)):
        assert np.array_equal(gi, wi), (ctx, b)
        assert np.array_equal(_bits(gd), _bits(wd)), (ctx, b)


def _filtered(obj, metric, q, k, rowids, mi=None):
    bits, _ = obj.rowid_bitmap(np.asarray(rowids, dtype=np.int64))
    return obj.scan_topk_filtered(metric, q, k, bits, max_index=mi)


def _check(obj, metric, q, k, rowids, ctx, mi=None):
    """one query: scan_topk_rows == scan_topk_filtered with the bitmap of its rowids, max_index included"""
    got = obj.scan_topk_rows(metric, q, k, [rowids], max_index=mi)
    want = _filtered(obj, metric, q, k, rowids, mi)
    if mi is None:
        _same(got, want, ctx)
        return got[0]
    _same(got[0], want[0], ctx)
    assert got[1] == want[1], ctx
    return got[0][0]


def _lists(ids, k, rng):
    """the list shapes: empty, one, k - 1, k, 4k and 5000 rowids, each with duplicates and rowids that are not in the column"""
    out = []
    for size in (0, 1, k - 1, k, 4 * k, 5000):
        size = max(0, min(size, len(ids)))
        r = rng.choice(ids, size, replace=False)
        if size:
            r = np.concatenate([r, r[: max(1, size // 3)], [-7, 10**12]])
        out.append(r.astype(np.int64))
    return out


# ------------------------------------------------------------------------------------------------ (1) every pair, k, list shape
@pytest.mark.parametrize("dim", [5, 128, 771])
@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("vtype", TYPES)
def test_rows_equal_filtered(oracle, vtype, metric, dim):
    rng = np.random.Generator(np.random.PCG64(31_000 + 100 * vtype + 10 * metric + dim))
    n = 6000
    x = _column(vtype, n, dim, rng)
    ids = (rng.permutation(n) * 3 + 7).astype(np.int64)                      # explicit, not contiguous, not in row order
    q = _column(vtype, 1, dim, rng)[0]
    ix = _index(vtype, x, ids)
    try:
        for k in (1, 20, 256, 257, 1000):
            for li, rows in enumerate(_lists(ids, k, rng)):
                got_ids, got_d = _check(ix, metric, q, k, rows, (k, li))
                assert len(got_ids) == min(k, len(set(rows.tolist()) & set(ids.tolist()))), (k, li)
                if vtype in (po.I8, po.U8):
                    m = np.isin(ids, rows)
                    want_ids, want_d = oracle.scan_dense(metric, vtype, q, x[m], ids[m], k)
                    assert np.array_equal(got_ids, want_ids) and np.array_equal(got_d, want_d), (k, li)
    finally:
        ix.close()


def test_rows_max_index_carry():
    rng = np.random.Generator(np.random.PCG64(31_500))
    n, dim = 5000, 48
    for vtype in (po.I8, po.BF16):
        x = _column(vtype, n, dim, rng)
        ix = _index(vtype, x)
        rows = rng.choice(np.arange(1, n + 1), 700, replace=False)
        q = _column(vtype, 1, dim, rng)[0]
        mi_r = mi_f = 0
        for k in (100, 10, 33):
            got, mi_r = ix.scan_topk_rows(po.L2, q, k, [rows], max_index=mi_r)
            want, mi_f = _filtered(ix, po.L2, q, k, rows, mi_f)
            _same(got, want, (vtype, k))
            assert mi_r == mi_f, (vtype, k)
        ix.close()


# ------------------------------------------------------------------------------------------------ (2) plan-switching shapes
@pytest.mark.parametrize("vtype,dim", [(po.F32, 110), (po.BF16, 220), (po.I8, 440)])
def test_rows_plan_switching_shapes(vtype, dim):
    rng = np.random.Generator(np.random.PCG64(32_000 + dim))
    n = 4000
    x = _column(vtype, n, dim, rng)
    ix = _index(vtype, x)
    try:
        for metric in METRICS:
            q = _column(vtype, 1, dim, rng)[0]
            for k in (20, 64, 300):
                rows = rng.choice(np.arange(1, n + 1), 4 * k, replace=False)
                _check(ix, metric, q, k, rows, (metric, k))
    finally:
        ix.close()


# ------------------------------------------------------------------------------------------------ (3) special values, ties
@pytest.mark.parametrize("vtype", [po.F32, po.F16, po.BF16])
def test_rows_special_values(vtype):
    rng = np.random.Generator(np.random.PCG64(33_000 + vtype))
    n, dim = 3000, 40
    x = rng.standard_normal((n, dim)).astype(np.float32)
    for r in range(0, n, 7):
        x[r, rng.integers(0, dim)] = rng.choice([np.nan, np.inf, -np.inf])
    x[::53] = np.inf
    x[1::53] = -np.inf
    xs = po.convert(x, vtype)
    ix = _index(vtype, xs)
    try:
        base = rng.standard_normal(dim).astype(np.float32)
        queries = [base]
        for v in (np.nan, np.inf, -np.inf):
            qq = base.copy()
            qq[3] = v
            queries.append(qq)
        for qi, qf in enumerate(queries):
            q = po.convert(qf[None, :], vtype)[0]
            for metric in METRICS:
                for k in (20, 300):
                    rows = rng.choice(np.arange(1, n + 1), 1200, replace=False)
                    _check(ix, metric, q, k, rows, (qi, metric, k))
    finally:
        ix.close()


def test_rows_ties_int8(oracle):
    rng = np.random.Generator(np.random.PCG64(33_500))
    n, dim = 5000, 16
    x = rng.integers(0, 2, (n, dim)).astype(np.int8)
    ids = np.arange(1, n + 1, dtype=np.int64)
    ix = _index(po.I8, x)
    try:
        for metric in METRICS:
            q = rng.integers(0, 2, dim).astype(np.int8)
            for k in (20, 300):
                rows = rng.choice(ids, 2000, replace=False)
                got_ids, got_d = _check(ix, metric, q, k, rows, (metric, k))
                m = np.isin(ids, rows)
                want_ids, want_d = oracle.scan_dense(metric, po.I8, q, x[m], ids[m], k)
                assert np.array_equal(got_ids, want_ids) and np.array_equal(got_d, want_d), (metric, k)
    finally:
        ix.close()


# ------------------------------------------------------------------------------------------------ (4) batches
@pytest.mark.parametrize("vtype", [po.F32, po.BF16, po.I8])
@pytest.mark.parametrize("nq", [16, 1024])
def test_rows_batch_equals_single_calls(vtype, nq):
    rng = np.random.Generator(np.random.PCG64(34_000 + vtype + nq))
    n, dim, k = 20_000, 64, 20
    x = _column(vtype, n, dim, rng)
    q = _column(vtype, nq, dim, rng)
    ix = _index(vtype, x)
    try:
        lists = [rng.choice(np.arange(1, n + 1), int(rng.integers(0, 400)), replace=True) for _ in range(nq)]
        for metric in (po.L2, po.COS, po.L1):
            for kk in (k, 300):
                got = ix.scan_topk_rows(metric, q, kk, lists)
                singles = [ix.scan_topk_rows(metric, q[b], kk, [lists[b]])[0] for b in range(nq)]
                _same(got, singles, (metric, kk))
                for b in range(0, nq, max(1, nq // 8)):
                    _same([got[b]], _filtered(ix, metric, q[b], kk, lists[b]), (metric, kk, b))
    finally:
        ix.close()


# ------------------------------------------------------------------------------------------------ (5) streamed windows
@pytest.mark.parametrize("window,n", [(128, 2048), (100, 1050)])
@pytest.mark.parametrize("vtype", [po.BF16, po.I8, po.F32])
def test_rows_streamed(vtype, window, n):
    rng = np.random.Generator(np.random.PCG64(35_000 + window + vtype))
    dim = 40
    x = _column(vtype, n, dim, rng)
    res, st = _index(vtype, x), _index(vtype, x, window=window)
    try:
        pitch = st.query_pitch
        for metric in METRICS:
            q = _column(vtype, 3, dim, rng)
            for k in (20, 300):
                lists = [rng.choice(np.arange(1, n + 1), int(s), replace=True) for s in (3 * k, 1, 700)]
                sb, hb = st.stat("stream_bytes"), st.stat("rows_host_bytes")
                got = st.scan_topk_rows(metric, q, k, lists)
                assert st.stat("stream_bytes") == sb, (metric, k)
                assert st.stat("rows_host_bytes") - hb == sum(len(set(r.tolist())) for r in lists) * pitch, (metric, k)
                if vtype == po.I8 or window % 32 == 0:
                    # fp: the chunk order rotates by the row's place in its warp tile, counted from the window's start, so a
                    # window that is not a multiple of 32 rows sums some rows in another order than the resident index (the
                    # streamed filtered scan does the same, checked below)
                    _same(got, res.scan_topk_rows(metric, q, k, lists), (metric, k))
                for b in range(3):
                    _same([got[b]], _filtered(st, metric, q[b], k, lists[b]), (metric, k, b))
    finally:
        res.close()
        st.close()


# ------------------------------------------------------------------------------------------------ (6) groups
@pytest.mark.parametrize("vtype", [po.I8, po.F16])
def test_rows_groups(vtype):
    rng = np.random.Generator(np.random.PCG64(36_000 + vtype))
    n, dim = 3001, 16
    x = _column(vtype, n, dim, rng)
    q = _column(vtype, 20, dim, rng)
    ix = _index(vtype, x)
    pitch = ix.query_pitch
    # shards of 1000, 1000 and 1001 rows: a budget of 1000.5 rows streams only the last one
    with _env(VSB_DEVICE_BUDGET_MB=repr(1000.5 * pitch / 1048576.0)):
        g3 = _group(vtype, x, 3)
    g1 = _group(vtype, x, 1)
    try:
        lib = g3.eng.lib
        assert [lib.vsb_index_is_streamed(lib.vsb_group_shard(g3.h, s)) for s in range(3)] == [0, 0, 1]
        lists = [rng.choice(np.arange(1, n + 1), int(rng.integers(0, 900)), replace=True) for _ in range(20)]
        for metric in METRICS:
            for k in (20, 300):
                want = ix.scan_topk_rows(metric, q, k, lists)
                for g in (g1, g3):
                    got = g.scan_topk_rows(metric, q, k, lists)
                    for b in (0, 7):
                        _same([got[b]], _filtered(g, metric, q[b], k, lists[b]), (g.gpus, metric, k, b))
                    if vtype == po.I8 or g is g1:                               # fp shards rotate chunks by shard-local rows
                        _same(got, want, (g.gpus, metric, k))
    finally:
        for o in (ix, g1, g3):
            o.close()


# ------------------------------------------------------------------------------------------------ (7) launches and handles
def test_rows_one_launch_per_shard_and_no_handles():
    eng = _vs().load_engine()
    rng = np.random.Generator(np.random.PCG64(37_000))
    n, dim = 6000, 32
    x = _column(po.I8, n, dim, rng)
    q = _column(po.I8, 20, dim, rng)
    lists = [rng.choice(np.arange(1, n + 1), 500) for _ in range(20)]
    base = eng.debug_live_handles()
    for make, shards in ((lambda: _index(po.I8, x), 1), (lambda: _index(po.I8, x, window=1000), 1), (lambda: _group(po.I8, x, 3), 3)):
        obj = make()
        for qq, ll in ((q, lists), (q[:1], lists[:1])):
            for k in (20, 300):
                before = eng.kernel_launches()
                obj.scan_topk_rows(po.L2, qq, k, ll)
                assert eng.kernel_launches() - before == shards, (shards, k, len(ll))
        obj.close()
        assert eng.debug_live_handles() == base


# ------------------------------------------------------------------------------------------------ (8) SQL
def _sql_script(vtype_name, metric, dim, x, ids, q, qtype, k, cands, gpus=1, insert=None):
    opts = f"type={vtype_name},dimension={dim},distance={metric}" + (f",gpus={gpus}" if gpus > 1 else "")
    s = ["CREATE TABLE t (id INTEGER PRIMARY KEY, e BLOB)", f"SELECT vector_init('t','e','{opts}')"]
    s += [["INSERT INTO t(id, e) VALUES (?, ?)", [int(ids[i]), {"hex": x[i].tobytes().hex()}]] for i in range(len(ids))]
    s += [f"SELECT vector_quantize('t','e','qtype={qtype}')"]
    if insert is not None:                                                   # the quantization is now stale
        s += [["INSERT INTO t(id, e) VALUES (?, ?)", [int(insert[0]), {"hex": insert[1].tobytes().hex()}]]]
    mark = len(s)
    allq = {"hex": q.tobytes().hex()}
    for c in cands:
        for b in range(len(q)):
            qb = {"hex": q[b].tobytes().hex()}
            s += [["SELECT id, distance FROM vector_quantize_scan_rerank('t','e',?,?,?)", [qb, k, c]],
                  ["SELECT id, distance FROM vector_full_scan_filtered('t','e',?,?,"
                   "(SELECT vector_rowid_set(id) FROM vector_quantize_scan('t','e',?,?)))", [qb, k, qb, c]]]
        s += [["SELECT query, id, distance FROM vector_quantize_scan_rerank_batch('t','e',?,?,?)", [allq, k, c]]]
    return s, mark


def _check_sql(r, nq, ncands, ctx):
    at = 0
    for c in range(ncands):
        singles = []
        for b in range(nq):
            mine, composed = r[at], r[at + 1]
            assert "error" not in mine, (ctx, c, b, mine)
            assert mine == composed, (ctx, c, b)
            singles.append(mine["rows"])
            at += 2
        batch = r[at]["rows"]
        at += 1
        for b in range(nq):
            assert [row[1:] for row in batch if row[0] == b] == singles[b], (ctx, c, b)


@pytest.mark.parametrize("vtype_name", ["FLOAT32", "FLOAT16", "FLOATB16"])
def test_sql_rerank_matches_composed(vtype_name):
    vtype = {"FLOAT32": po.F32, "FLOAT16": po.F16, "FLOATB16": po.BF16}[vtype_name]
    rng = np.random.Generator(np.random.PCG64(38_000 + vtype))
    n, dim, k, nq = 1500, 24, 10, 3
    x = po.convert(rng.standard_normal((n, dim), dtype=np.float32), vtype)
    ids = (np.arange(n) * 2 + 5).astype(np.int64)
    q = po.convert(rng.standard_normal((nq, dim), dtype=np.float32), vtype)
    cands = [0, 5, k, 4 * k, 300]
    for qtype in ("UINT8", "INT8"):
        for metric in ("L2", "SQUARED_L2", "COSINE", "DOT", "L1"):
            s, mark = _sql_script(vtype_name, metric, dim, x, ids, q, qtype, k, cands)
            _check_sql(run_sql(OURS, s)[mark:], nq, len(cands), (qtype, metric))


def test_sql_rerank_groups_streamed_and_stale():
    rng = np.random.Generator(np.random.PCG64(38_500))
    n, dim, k, nq = 1500, 24, 10, 3
    x = rng.standard_normal((n, dim), dtype=np.float32)
    ids = (np.arange(n) * 3 + 1).astype(np.int64)
    q = rng.standard_normal((nq, dim), dtype=np.float32)
    cands = [0, 5, k, 4 * k, 300]
    s, mark = _sql_script("FLOAT32", "L2", dim, x, ids, q, "INT8", k, cands, gpus=3)
    _check_sql(run_sql(OURS, s, env={"VSB_GROUP_ALIAS": "1"})[mark:], nq, len(cands), "gpus=3")
    s, mark = _sql_script("FLOAT32", "COSINE", dim, x, ids, q, "UINT8", k, cands)
    _check_sql(run_sql(OURS, s, env={"VSB_DEVICE_BUDGET_MB": "0.02"})[mark:], nq, len(cands), "streamed")
    s, mark = _sql_script("FLOAT32", "L2", dim, x, ids, q, "INT8", k, cands, insert=(10**6, q[0]))
    r = run_sql(OURS, s)[mark:]
    _check_sql(r, nq, len(cands), "stale")
    assert all(row[0] != 10**6 for e in r for row in e["rows"])      # the new row has no quantized copy, so it is never a candidate


def test_sql_rerank_errors():
    s = ["CREATE TABLE t (id INTEGER PRIMARY KEY, e BLOB)", "SELECT vector_init('t','e','type=FLOAT32,dimension=4')",
         "INSERT INTO t(id, e) VALUES (1, vector_as_f32('[1,2,3,4]'))",
         "SELECT id FROM vector_quantize_scan_rerank('t','e',vector_as_f32('[1,2,3,4]'),3,10)",      # 3 not quantized
         "SELECT vector_quantize('t','e')",
         "SELECT id, distance FROM vector_quantize_scan_rerank('t','e',vector_as_f32('[1,2,3,4]'),3,10)",
         "SELECT id, distance FROM vector_quantize_scan_rerank('t','e','[1,2,3,4]',3,0)"]
    r = run_sql(OURS, s)
    assert "Quantization table not found" in r[3]["error"]
    assert r[5]["rows"] == [[1, 0.0]] and r[6]["rows"] == []
