"""Grouped top-k (vsb_scan_topk_grouped, its group and SQL doors): each key's k nearest rows for the best keys, from one scan of
the column per query.  Every returned key equals scan_topk_filtered (nq = 1) with the bitmap of its rowids, bit for bit, and the
keys and their order equal a numpy ranking of every key's filtered answer.  -m gpu.

(1) every (type, metric) pair at dims 5 / 384 / 771 with empty keys, keys of absent rowids, singletons, duplicates, overlapping
    keys, keys shorter than k and a key of several pieces, k = 1 / 3 / 32 / 33 / 256, limits 0 / 1 / 3 / >= nkeys; int8 and
    uint8 also against the oracle;
(2) the shapes where the filtered call's plan changes lanes or turns DIRECT with k;
(3) one key of every row equals vsb_scan_topk from a fresh cursor; piece boundaries hit exactly beside tiny keys;
(4) ties in key minima at the limit; (5) NaN / +-Inf rows and -INF dot distances;
(6) falling distances force a regrow of the pair list without changing the result;
(7) streamed windows equal the resident index; (8) groups of 1 / 2 / 3 shards, one streamed, keys across shard boundaries and a
    key that makes the limit only through its rows on a shard where it is locally poor;
(9) argument errors, handles back to baseline; (10) SQL: each key of vector_*_scan_grouped equals vector_*_scan_filtered."""
import contextlib
import os

import numpy as np
import pytest

from oracle import pyoracle as po
from tests.sqlrun import OURS, run_sql

pytestmark = pytest.mark.gpu
METRICS = [po.L2, po.L2SQ, po.COS, po.DOT, po.L1]
TYPES = [po.F32, po.F16, po.BF16, po.U8, po.I8]
PIECE = 1024                                                                  # rows of a piece (kGroupedPiece)


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
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64)


def _filtered(obj, metric, q, k, rowids):
    bits, _ = obj.rowid_bitmap(np.asarray(rowids, dtype=np.int64))
    return obj.scan_topk_filtered(metric, q, k, bits)[0]


def _want(obj, metric, q, k, keys, limit, row_of):
    """every key's filtered answer, ranked by (first distance, scan row of the first row, key) and cut to limit"""
    ranked = []
    for g, rows in enumerate(keys):
        ids, d = _filtered(obj, metric, q, k, rows)
        if len(ids):
            ranked.append((float(d[0]), row_of[int(ids[0])], g, ids, d))
    ranked.sort(key=lambda t: t[:3])
    if limit:
        ranked = ranked[:limit]
    return [(t[2], t[3], t[4]) for t in ranked]


def _same(got, want, ctx):
    assert [g for g, _, _ in got] == [g for g, _, _ in want], ctx
    for (g, gi, gd), (_, wi, wd) in zip(got, want):
        assert np.array_equal(gi, wi), (ctx, g)
        assert np.array_equal(_bits(gd), _bits(wd)), (ctx, g)


def _check(obj, metric, q, k, keys, limit, row_of, ctx):
    (got,) = obj.scan_topk_grouped(metric, q, k, keys, limit)
    want = _want(obj, metric, q, k, keys, limit, row_of)
    _same(got, want, ctx)
    return got


def _keys(ids, k, rng):
    """the key shapes: empty, absent rowids only, one row, a row twice, k - 1 rows, k rows, overlapping keys, 1500 rows (two
    pieces), random sizes"""
    pick = lambda m: rng.choice(ids, min(m, len(ids)), replace=False)
    a = pick(300)
    keys = [np.zeros(0, np.int64), np.array([-5, 10**12], np.int64), pick(1), np.repeat(pick(1), 2), pick(max(k - 1, 0)), pick(k),
            a, np.concatenate([a[:150], pick(100)]), pick(1500)]
    keys += [pick(int(rng.integers(1, 200))) for _ in range(6)]
    return [np.concatenate([r, r[: len(r) // 4]]).astype(np.int64) for r in keys]


# ------------------------------------------------------------------------------------------------ (1) every pair
@pytest.mark.parametrize("dim", [5, 384, 771])
@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("vtype", TYPES)
def test_grouped_equals_filtered(oracle, vtype, metric, dim):
    rng = np.random.Generator(np.random.PCG64(61_000 + 100 * vtype + 10 * metric + dim))
    n = 3000
    x = _column(vtype, n, dim, rng)
    ids = (rng.permutation(n) * 3 + 7).astype(np.int64)                      # explicit, not contiguous, not in row order
    row_of = {int(r): i for i, r in enumerate(ids)}
    q = _column(vtype, 1, dim, rng)[0]
    ix = _index(vtype, x, ids)
    try:
        for k in (1, 3, 32, 33, 256):
            keys = _keys(ids, k, rng)
            for limit in ((0, 1, 3, 100) if k in (1, 33) else (0, 4)):
                got = _check(ix, metric, q, k, keys, limit, row_of, (k, limit))
                if vtype in (po.I8, po.U8) and limit == 0:
                    for g, gi, gd in got[:4]:
                        m = np.isin(ids, keys[g])
                        wi, wd = oracle.scan_dense(metric, vtype, q, x[m], ids[m], k)
                        assert np.array_equal(gi, wi) and np.array_equal(gd, wd), (k, g)
    finally:
        ix.close()


# ------------------------------------------------------------------------------------------------ (2) plan-switching shapes
@pytest.mark.parametrize("vtype,dim", [(po.F32, 110), (po.BF16, 220), (po.I8, 440)])
def test_grouped_plan_switching_shapes(vtype, dim):
    rng = np.random.Generator(np.random.PCG64(62_000 + dim))
    n = 4000
    x = _column(vtype, n, dim, rng)
    row_of = {i + 1: i for i in range(n)}
    ix = _index(vtype, x)
    try:
        for metric in METRICS:
            q = _column(vtype, 1, dim, rng)[0]
            for k in (1, 32, 33, 64, 256):
                keys = [rng.choice(np.arange(1, n + 1), int(s), replace=False) for s in (4 * k, 2000, 7)]
                _check(ix, metric, q, k, keys, 0, row_of, (metric, k))
    finally:
        ix.close()


# ------------------------------------------------------------------------------------------------ (3) one key of every row, pieces
def test_grouped_one_key_of_every_row_equals_topk():
    rng = np.random.Generator(np.random.PCG64(63_000))
    for vtype, n, dim in ((po.I8, 70_000, 64), (po.F32, 20_000, 40)):
        x = _column(vtype, n, dim, rng)
        ix = _index(vtype, x)
        try:
            for metric in (po.L2, po.DOT):
                q = _column(vtype, 2, dim, rng)
                for k in (1, 10, 256):
                    got = ix.scan_topk_grouped(metric, q, k, [np.arange(1, n + 1)])
                    for b in range(2):
                        (wi, wd), = ix.scan_topk(metric, q[b], k)
                        assert len(got[b]) == 1 and got[b][0][0] == 0, (metric, k, b)
                        assert np.array_equal(got[b][0][1], wi) and np.array_equal(_bits(got[b][0][2]), _bits(wd)), (metric, k, b)
        finally:
            ix.close()


def test_grouped_piece_boundaries_beside_tiny_keys():
    rng = np.random.Generator(np.random.PCG64(63_500))
    n, dim = 12_000, 24
    for vtype in (po.I8, po.BF16):
        x = _column(vtype, n, dim, rng)
        row_of = {i + 1: i for i in range(n)}
        ix = _index(vtype, x)
        try:
            ar = np.arange(1, n + 1)
            keys = [ar[:PIECE - 1], ar[:PIECE], ar[:PIECE + 1], rng.permutation(ar)[:2 * PIECE], ar[: 3 * PIECE + 5], ar,
                    ar[5:6], ar[-1:], ar[PIECE - 1:PIECE + 1]]
            keys += [rng.choice(ar, 3, replace=False) for _ in range(8)]
            for metric in (po.L2, po.COS, po.L1):
                q = _column(vtype, 1, dim, rng)[0]
                for k in (1, 3, 33, 256):
                    for limit in (0, 2):
                        _check(ix, metric, q, k, keys, limit, row_of, (vtype, metric, k, limit))
        finally:
            ix.close()


# ------------------------------------------------------------------------------------------------ (4) ties at the limit
def test_grouped_ties_at_the_limit():
    rng = np.random.Generator(np.random.PCG64(64_000))
    n, dim = 2000, 8
    base = rng.integers(-3, 4, (40, dim)).astype(np.int8)
    x = base[rng.integers(0, 40, n)]                                          # many equal rows: equal distances, equal key minima
    row_of = {i + 1: i for i in range(n)}
    ix = _index(po.I8, x)
    try:
        ar = np.arange(1, n + 1)
        keys = [rng.choice(ar, int(rng.integers(1, 30)), replace=False) for _ in range(60)]
        keys += [keys[3].copy(), keys[3][::-1].copy()]                        # identical keys: same minimum and first row
        q = x[17].copy()
        for metric in (po.L2, po.DOT, po.L1):
            for k in (1, 3, 10):
                for limit in (0, 1, 2, 5, 17, 62, 100):
                    got = _check(ix, metric, q, k, keys, limit, row_of, (metric, k, limit))
                    assert len(got) == (min(limit, 62) if limit else 62), (metric, k, limit)
    finally:
        ix.close()


# ------------------------------------------------------------------------------------------------ (5) special values
@pytest.mark.parametrize("vtype", [po.F32, po.F16, po.BF16])
def test_grouped_special_values(vtype):
    rng = np.random.Generator(np.random.PCG64(65_000 + vtype))
    n, dim = 3000, 40
    x = rng.standard_normal((n, dim)).astype(np.float32)
    for r in range(0, n, 7):
        x[r, rng.integers(0, dim)] = rng.choice([np.nan, np.inf, -np.inf])
    x[::53] = np.inf
    x[1::53] = -np.inf
    xs = po.convert(x, vtype)
    row_of = {i + 1: i for i in range(n)}
    ix = _index(vtype, xs)
    try:
        ar = np.arange(1, n + 1)
        keys = [ar[0::7][:30], ar[::53][:20], ar[1::53][:20], rng.choice(ar, 500, replace=False), ar[0:1], ar[53:54]]
        keys += [rng.choice(ar, 40, replace=False) for _ in range(10)]
        base = rng.standard_normal(dim).astype(np.float32)
        queries = [base]
        for v in (np.nan, np.inf, -np.inf):
            qq = base.copy()
            qq[3] = v
            queries.append(qq)
        for qi, qf in enumerate(queries):
            q = po.convert(qf[None, :], vtype)[0]
            for metric in METRICS:
                for k in (3, 33):
                    _check(ix, metric, q, k, keys, 0, row_of, (qi, metric, k))
                    _check(ix, metric, q, k, keys, 3, row_of, (qi, metric, k, 3))
    finally:
        ix.close()


# ------------------------------------------------------------------------------------------------ (6) regrow
def test_grouped_falling_distances_regrow():
    n, dim = 100_000, 4
    x = np.zeros((n, dim), np.float32)
    x[:, 0] = np.arange(n, 0, -1, dtype=np.float32)                           # L2 to the zero query falls in scan order
    row_of = {i + 1: i for i in range(n)}
    ix = _index(po.F32, x)
    try:
        q = np.zeros(dim, np.float32)
        keys = [np.arange(1, n + 1), np.arange(1, 50), np.arange(n - 10, n + 1)]
        r0 = ix.stat("grouped_regrows")
        got = _check(ix, po.L2, q, 5, keys, 0, row_of, "regrow")
        assert ix.stat("grouped_regrows") - r0 >= 1
        assert ix.stat("grouped_cands") >= n
        assert ix.stat("grouped_pairs") == n + 49 + 11
        (again,) = ix.scan_topk_grouped(po.L2, q, 5, keys)
        _same(again, got, "after the regrow")
    finally:
        ix.close()


# ------------------------------------------------------------------------------------------------ (7) streamed windows
@pytest.mark.parametrize("window,n", [(128, 4096), (100, 1050)])
@pytest.mark.parametrize("vtype", [po.I8, po.BF16])
def test_grouped_streamed(vtype, window, n):
    rng = np.random.Generator(np.random.PCG64(67_000 + window + vtype))
    dim = 40
    x = _column(vtype, n, dim, rng)
    row_of = {i + 1: i for i in range(n)}
    res, st = _index(vtype, x), _index(vtype, x, window=window)
    try:
        ar = np.arange(1, n + 1)
        keys = [ar[:window], ar[window - 1:window + 1], ar[: PIECE + 3], rng.permutation(ar)]
        keys += [rng.choice(ar, int(rng.integers(1, 300)), replace=False) for _ in range(12)]
        for metric in METRICS:
            q = _column(vtype, 2, dim, rng)
            for k in (3, 33):
                got = st.scan_topk_grouped(metric, q, k, keys, 5)
                if vtype == po.I8 or window % 32 == 0:                       # fp rows rotate by their window-local tile place
                    want = res.scan_topk_grouped(metric, q, k, keys, 5)
                    for b in range(2):
                        _same(got[b], want[b], (metric, k, b))
                _check(st, metric, q[0], k, keys, 5, row_of, (metric, k))
        assert st.stat("stream_bytes") > 0
    finally:
        res.close()
        st.close()


# ------------------------------------------------------------------------------------------------ (8) groups
@pytest.mark.parametrize("vtype", [po.I8, po.F16])
def test_grouped_groups(vtype):
    rng = np.random.Generator(np.random.PCG64(68_000 + vtype))
    n, dim = 3001, 16
    x = _column(vtype, n, dim, rng)
    q = _column(vtype, 1, dim, rng)[0]
    row_of = {i + 1: i for i in range(n)}
    ix = _index(vtype, x)
    pitch = ix.query_pitch
    with _env(VSB_DEVICE_BUDGET_MB=repr(1000.5 * pitch / 1048576.0)):       # shards of 1000, 1000, 1001 rows: the last one streams
        g3 = _group(vtype, x, 3)
    g1, g2 = _group(vtype, x, 1), _group(vtype, x, 2)
    try:
        lib = g3.eng.lib
        assert [lib.vsb_index_is_streamed(lib.vsb_group_shard(g3.h, s)) for s in range(3)] == [0, 0, 1]
        ar = np.arange(1, n + 1)
        keys = [ar[990:1010], ar[1995:2005], ar[::97], ar[1000:1001], ar[2999:], rng.permutation(ar)[:1200]]
        keys += [rng.choice(ar, int(rng.integers(1, 60)), replace=False) for _ in range(20)]
        for metric in METRICS:
            for k in (3, 33):
                for limit in (0, 4):
                    want = ix.scan_topk_grouped(metric, q, k, keys, limit)[0]
                    for g in (g1, g2, g3):
                        got = _check(g, metric, q, k, keys, limit, row_of, (g.gpus, metric, k, limit))
                        if vtype == po.I8 or g is g1:                        # fp shards rotate chunks by shard-local rows
                            _same(got, want, (g.gpus, metric, k, limit))
    finally:
        for o in (ix, g1, g2, g3):
            o.close()


def test_grouped_limit_uses_every_shards_minimum():
    """key 0's rows on shard 0 are far from the query and its only close row is on shard 2; the other keys live on shard 0
    and beat key 0 there.  With limit 1 key 0 must win, and its rows from shard 0 must still be in its answer."""
    n, dim = 3000, 4
    x = np.zeros((n, dim), np.float32)
    x[:, 0] = 50.0 + np.arange(n, dtype=np.float32) % 7
    x[:1000, 0] = 10.0 + np.arange(1000, dtype=np.float32) % 13               # shard 0: moderate distances
    x[:6, 0] = 40.0                                                            # key 0's shard-0 rows: poor there
    x[2500, 0] = 1.0                                                           # key 0's close row on shard 2
    q = np.zeros(dim, np.float32)
    row_of = {i + 1: i for i in range(n)}
    keys = [np.concatenate([np.arange(1, 7), [2501]])] + [np.arange(10 + 20 * i, 30 + 20 * i) for i in range(30)]
    for ngpus in (1, 2, 3):
        g = _group(po.F32, x, ngpus)
        try:
            got = _check(g, po.L2, q, 5, keys, 1, row_of, ngpus)
            assert got[0][0] == 0 and len(got[0][1]) == 5 and got[0][1][0] == 2501, ngpus
        finally:
            g.close()


# ------------------------------------------------------------------------------------------------ (9) arguments, handles
def test_grouped_arguments_and_handles():
    vs = _vs()
    eng = vs.load_engine()
    rng = np.random.Generator(np.random.PCG64(69_000))
    n, dim = 2000, 32
    x = _column(po.I8, n, dim, rng)
    q = _column(po.I8, 3, dim, rng)
    keys = [rng.choice(np.arange(1, n + 1), 100) for _ in range(30)]
    base = eng.debug_live_handles()
    for make in (lambda: _index(po.I8, x), lambda: _index(po.I8, x, window=500), lambda: _group(po.I8, x, 3)):
        obj = make()
        for k in (1, 33):
            obj.scan_topk_grouped(po.L2, q, k, keys, 3)
        assert obj.scan_topk_grouped(po.L2, q, 0, keys) == [[], [], []]
        assert obj.scan_topk_grouped(po.L2, q, 5, []) == [[], [], []]
        for bad in (dict(k=257), dict(k=-1), dict(limit=-1), dict(metric=99)):
            a = dict(metric=po.L2, k=5, limit=0) | bad
            with pytest.raises(vs.VsbError) as e:
                obj.scan_topk_grouped(a["metric"], q, a["k"], keys, a["limit"])
            assert e.value.rc == vs.api.EINVAL, bad
        fn = obj._fn("scan_topk_grouped")
        res = vs.api._vp()
        rid = np.arange(1, 5, dtype=np.int64)
        for offs, nk in ((np.array([1, 4], np.int64), 1), (np.array([0, 3, 2], np.int64), 2), (np.array([0, 4], np.int64), -1)):
            rc = fn(obj.h, po.L2, vs.api._ptr(q), 1, 5, vs.api._ptr(rid), vs.api._ptr(offs), nk, 0, vs.api.C.byref(res))
            assert rc == vs.api.EINVAL and not res.value, (offs, nk)
        rc = fn(obj.h, po.L2, vs.api._ptr(q), 1, 5, None, vs.api._ptr(np.array([0, 2], np.int64)), 1, 0, vs.api.C.byref(res))
        assert rc == vs.api.EINVAL
        obj.close()
        assert eng.debug_live_handles() == base


# ------------------------------------------------------------------------------------------------ (10) SQL
def _sql_script(vtype_name, metric, dim, x, ids, doc, q, k, limits, gpus=1):
    opts = f"type={vtype_name},dimension={dim},distance={metric}" + (f",gpus={gpus}" if gpus > 1 else "")
    s = ["CREATE TABLE t (id INTEGER PRIMARY KEY, e BLOB, doc INTEGER)", f"SELECT vector_init('t','e','{opts}')"]
    s += [["INSERT INTO t(id, e, doc) VALUES (?, ?, ?)", [int(ids[i]), {"hex": x[i].tobytes().hex()}, int(doc[i])]] for i in range(len(ids))]
    s += ["SELECT vector_quantize('t','e','qtype=INT8')"]
    mark = len(s)
    qb = {"hex": q.tobytes().hex()}
    docs = sorted(set(int(d) for d in doc))
    for mod in ("full", "quantize"):
        for limit in limits:
            s += [[f"SELECT key, id, distance FROM vector_{mod}_scan_grouped('t','e',?,?,(SELECT vector_rowid_sets(doc, id) FROM t),?)",
                   [qb, k, limit]]]
        for d in docs:
            s += [[f"SELECT id, distance FROM vector_{mod}_scan_filtered('t','e',?,?,(SELECT vector_rowid_set(id) FROM t WHERE doc = ?))",
                   [qb, k, d]]]
    return s, mark, docs


def _check_sql(r, docs, limits, id_row, ctx):
    at = 0
    for mod in ("full", "quantize"):
        grouped = r[at:at + len(limits)]
        at += len(limits)
        per = {}
        for d in docs:
            assert "error" not in r[at], (ctx, mod, r[at])
            per[d] = r[at]["rows"]
            at += 1
        rank = sorted((rows[0][1], id_row[rows[0][0]], d) for d, rows in per.items() if rows)
        for limit, g in zip(limits, grouped):
            assert "error" not in g, (ctx, mod, g)
            want_keys = [d for _, _, d in rank][: limit or None]
            got_keys = list(dict.fromkeys(row[0] for row in g["rows"]))
            assert got_keys == want_keys, (ctx, mod, limit)
            for d in got_keys:
                assert [row[1:] for row in g["rows"] if row[0] == d] == per[d], (ctx, mod, limit, d)


@pytest.mark.parametrize("vtype_name,metric", [("FLOAT32", "L2"), ("FLOAT16", "COSINE"), ("INT8", "DOT"), ("UINT8", "L1")])
def test_sql_grouped_matches_filtered(vtype_name, metric):
    vtype = {"FLOAT32": po.F32, "FLOAT16": po.F16, "INT8": po.I8, "UINT8": po.U8}[vtype_name]
    rng = np.random.Generator(np.random.PCG64(70_000 + vtype))
    n, dim, k = 1200, 24, 4
    x = _column(vtype, n, dim, rng)
    ids = (np.arange(n) * 2 + 5).astype(np.int64)
    doc = (rng.integers(0, 40, n) * 1000 - 7000).astype(np.int64)             # sparse, negative keys too
    q = _column(vtype, 1, dim, rng)[0]
    limits = [None, 0, 1, 5, 100]
    id_row = {int(r): i for i, r in enumerate(ids)}
    s, mark, docs = _sql_script(vtype_name, metric, dim, x, ids, doc, q, k, limits)
    _check_sql(run_sql(OURS, s)[mark:], docs, limits, id_row, (vtype_name, metric))


def test_sql_grouped_groups_and_streamed():
    rng = np.random.Generator(np.random.PCG64(70_500))
    n, dim, k = 1500, 24, 3
    x = rng.standard_normal((n, dim), dtype=np.float32)
    ids = (np.arange(n) * 3 + 1).astype(np.int64)
    doc = rng.integers(0, 25, n).astype(np.int64)
    q = rng.standard_normal(dim, dtype=np.float32)
    limits = [None, 2, 10]
    id_row = {int(r): i for i, r in enumerate(ids)}
    s, mark, docs = _sql_script("FLOAT32", "L2", dim, x, ids, doc, q, k, limits, gpus=3)
    _check_sql(run_sql(OURS, s, env={"VSB_GROUP_ALIAS": "1"})[mark:], docs, limits, id_row, "gpus=3")
    s, mark, docs = _sql_script("FLOAT32", "COSINE", dim, x, ids, doc, q, k, limits)
    _check_sql(run_sql(OURS, s, env={"VSB_DEVICE_BUDGET_MB": "0.02"})[mark:], docs, limits, id_row, "streamed")
