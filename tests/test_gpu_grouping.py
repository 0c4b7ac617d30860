"""Groupings and the device layout builder of grouped top-k (DESIGN §3.15).  -m gpu.

(1) The layout built on the device (vsb_debug_read "grouped" after a call) equals a numpy restatement byte for byte: implicit and
    explicit rowids (negative and very large ones), rowids absent from the column, duplicates inside a key, a rowid held by
    several rows, empty keys (runs of them at the start and the end), keys in random rowid order, key lengths 1023 / 1024 / 1025 /
    2048 / 2049, one key of every row, 10^6 keys of a few rows, a streamed index, and groups of 1 - 3 shards with one streamed.
(2) A grouping's answers equal scan_topk_grouped's bit for bit: every (type, metric) pair at two dimensions, k = 1 / 32 / 33 / 256,
    limits 0 / 1 / 3; many queries, metrics, k and limits on one grouping in any order, and after a per-call grouped call on the
    same index.  (3) "grouped_layout_reuses" counts the calls on a kept layout, and "grouped_layout_us" does not grow on them.
(4) Errors and lifetime: rows appended after the grouping was made, its column freed first, bad arguments, live handles.
(5) SQL: a repeated statement with the same groups BLOB launches no layout kernel and returns the same rows; a different BLOB, an
    INSERT and a ROLLBACK each lay the keys out anew, with every key's rows those of vector_full_scan_filtered."""
import contextlib
import os

import numpy as np
import pytest

from oracle import pyoracle as po
from tests.sqlrun import OURS, run_sql

pytestmark = pytest.mark.gpu
METRICS = [po.L2, po.L2SQ, po.COS, po.DOT, po.L1]
TYPES = [po.F32, po.F16, po.BF16, po.U8, po.I8]
PIECE = 1024


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


def _column(vtype, n, dim, rng):
    if vtype == po.I8:
        return rng.integers(-20, 21, (n, dim)).astype(np.int8)
    if vtype == po.U8:
        return rng.integers(0, 40, (n, dim)).astype(np.uint8)
    return po.convert(rng.standard_normal((n, dim), dtype=np.float32), vtype)


def _index(vtype, x, rowids=None, window=0, cap=None):
    ix = _vs().Index(vtype, x.shape[1], cap or x.shape[0], window_rows=window)
    ix.append_dense(x, rowids)
    ix.finalize()
    return ix


def _group(vtype, x, ngpus, rowids=None):
    g = _vs().Group(vtype, x.shape[1], x.shape[0], ngpus)
    g.append_dense(x, rowids)
    g.finalize()
    return g


class _Shard:
    """a group's shard (vsb_group_shard): the Index debug methods on its handle"""

    def __init__(self, g, s):
        self.eng, self.h = g.eng, g.eng.lib.vsb_group_shard(g.h, s)

    def debug_read(self, *a):
        return _vs().Index.debug_read(self, *a)

    def debug_grouped(self):
        return _vs().Index.debug_grouped(self)


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64)


def _same(got, want, ctx):
    assert len(got) == len(want), ctx
    for qa, qb in zip(got, want):
        assert [g for g, _, _ in qa] == [g for g, _, _ in qb], ctx
        for (g, gi, gd), (_, wi, wd) in zip(qa, qb):
            assert np.array_equal(gi, wi), (ctx, g)
            assert np.array_equal(_bits(gd), _bits(wd)), (ctx, g)


# ------------------------------------------------------------------------------------------------ (1) the layout
def _want_layout(keys, ids, lo, hi):
    """the layout of the keys on the shard of global scan rows [lo, hi) of a column whose row i has rowid ids[i]: every rowid
    becomes each row that holds it, each key's rows sorted and unique, cut every PIECE positions"""
    nkeys = len(keys)
    flat = np.concatenate([np.asarray(k, np.int64).reshape(-1) for k in keys]) if nkeys else np.zeros(0, np.int64)
    key_of = np.repeat(np.arange(nkeys, dtype=np.int64), [len(k) for k in keys])
    order = np.argsort(ids, kind="stable")
    sid = np.asarray(ids, np.int64)[order]
    a, b = np.searchsorted(sid, flat, "left"), np.searchsorted(sid, flat, "right")
    cnt = b - a
    total = int(cnt.sum())
    start = np.repeat(a - (np.cumsum(cnt) - cnt), cnt) + np.arange(total)
    rows, kk = order[start], np.repeat(key_of, cnt)
    keep = (rows >= lo) & (rows < hi)
    span = max(hi - lo, 1)
    comp = np.unique(kk[keep] * span + (rows[keep] - lo))
    kk, rows = comp // span, comp % span
    koff = np.searchsorted(kk, np.arange(nkeys + 1))
    npk = (np.diff(koff) + PIECE - 1) // PIECE
    kpiece = np.concatenate([[0], np.cumsum(npk)])
    pkey = np.repeat(np.arange(nkeys), npk)
    pstart = np.append(koff[pkey] + PIECE * (np.arange(len(pkey)) - kpiece[pkey]), koff[-1])
    u4 = lambda v: np.asarray(v, np.int64).astype(np.uint32)
    return {"rows": u4(rows), "koff": u4(koff), "pstart": u4(pstart), "pkey": u4(pkey), "kpiece": u4(kpiece)}


def _check_layout(shard, keys, ids, lo, hi, ctx):
    got, want = shard.debug_grouped(), _want_layout(keys, ids, lo, hi)
    for name, w in want.items():
        assert got[name].dtype == np.uint32 and np.array_equal(got[name], w), (ctx, name, got[name][:20], w[:20])


def _key_shapes(ids, rng):
    """empty keys (a run at the start and one at the end), absent rowids, duplicates, random order, the piece edges"""
    ids = np.asarray(ids, np.int64)
    pick = lambda m: rng.choice(ids, min(m, len(ids)), replace=False)
    absent = np.array([-(2 ** 63), -5, 0, 10 ** 18, 2 ** 63 - 1], np.int64)
    absent = absent[~np.isin(absent, ids)]
    keys = [np.zeros(0, np.int64)] * 3 + [absent, np.concatenate([absent, pick(3)]), np.repeat(pick(2), 3)]
    keys += [pick(m) for m in (1023, 1024, 1025, 2048, 2049)]
    keys += [np.sort(pick(1500)), np.sort(pick(1500))[::-1], np.concatenate([pick(700), pick(700)])]
    keys += [pick(int(rng.integers(1, 40))) for _ in range(30)] + [np.zeros(0, np.int64)] * 4
    return keys


def _layout_cases(ix, x, ids, keys, ctx):
    q = x[0]
    ix.scan_topk_grouped(po.L2, q, 1, keys)
    _check_layout(ix, keys, ids, 0, len(ids), (ctx, "per call"))
    with ix.grouping(keys) as g:
        g.scan_topk(po.L2, q, 5)
        _check_layout(ix, keys, ids, 0, len(ids), (ctx, "grouping"))


def test_layout_implicit_rowids():
    rng = np.random.Generator(np.random.PCG64(90_001))
    n = 5000
    x = _column(po.I8, n, 8, rng)
    ids = np.arange(1, n + 1, dtype=np.int64)
    ix = _index(po.I8, x)
    try:
        _layout_cases(ix, x, ids, _key_shapes(ids, rng), "implicit")
        _layout_cases(ix, x, ids, [rng.permutation(ids)], "one key of every row")
        _layout_cases(ix, x, ids, [np.zeros(0, np.int64), np.array([n + 1, -1], np.int64)], "nothing on the shard")
    finally:
        ix.close()


def test_layout_explicit_rowids():
    rng = np.random.Generator(np.random.PCG64(90_002))
    n = 5000
    x = _column(po.F16, n, 8, rng)
    ids = np.unique(np.concatenate([rng.integers(-(2 ** 62), 2 ** 62, n + 10), [-(2 ** 63) + 1, 2 ** 63 - 2, -1, 1]]))
    ids = rng.permutation(ids)[:n].astype(np.int64)
    ix = _index(po.F16, x, ids)
    try:
        _layout_cases(ix, x, ids, _key_shapes(ids, rng), "explicit")
        _layout_cases(ix, x, ids, [rng.permutation(ids)], "one key of every row")
    finally:
        ix.close()


def test_layout_rowid_held_by_several_rows():
    rng = np.random.Generator(np.random.PCG64(90_003))
    n = 3000
    x = _column(po.F32, n, 8, rng)
    ids = rng.integers(-50, 400, n).astype(np.int64)                     # every rowid held by several rows
    ix = _index(po.F32, x, ids)
    try:
        _layout_cases(ix, x, ids, _key_shapes(np.unique(ids), rng) + [ids[:2000]], "shared rowids")
    finally:
        ix.close()


def test_layout_a_million_keys_of_a_few_rows():
    rng = np.random.Generator(np.random.PCG64(90_004))
    n, nkeys = 200_000, 1_000_000
    x = _column(po.I8, n, 8, rng)
    ids = np.arange(1, n + 1, dtype=np.int64)
    lens = rng.integers(0, 4, nkeys)
    flat = rng.integers(1, n + 1, int(lens.sum())).astype(np.int64)
    keys = np.split(flat, np.cumsum(lens)[:-1])
    ix = _index(po.I8, x)
    try:
        ix.scan_topk_grouped(po.L2, x[0], 2, keys, 10)
        _check_layout(ix, keys, ids, 0, n, "1e6 keys")
    finally:
        ix.close()


def test_layout_streamed_and_groups():
    rng = np.random.Generator(np.random.PCG64(90_005))
    n, dim = 3001, 16
    x = _column(po.I8, n, dim, rng)
    ids = np.arange(1, n + 1, dtype=np.int64)
    keys = _key_shapes(ids, rng) + [ids[990:1010], ids[1995:2005]]
    ix = _index(po.I8, x, window=700)
    try:
        _layout_cases(ix, x, ids, keys, "streamed")
    finally:
        ix.close()
    pitch = ((dim + 15) // 16) * 16
    with _env(VSB_GROUP_ALIAS="1"):
        with _env(VSB_DEVICE_BUDGET_MB=repr(1000.5 * pitch / 1048576.0)):
            g3 = _group(po.I8, x, 3)
        groups = [_group(po.I8, x, 1), _group(po.I8, x, 2), g3]
        try:
            lib = g3.eng.lib
            assert [lib.vsb_index_is_streamed(lib.vsb_group_shard(g3.h, s)) for s in range(3)] == [0, 0, 1]
            for g in groups:
                bound = [n * s // g.gpus for s in range(g.gpus + 1)]
                for how in ("per call", "grouping"):
                    if how == "per call":
                        g.scan_topk_grouped(po.L2, x[0], 3, keys)
                    else:
                        gg = g.grouping(keys)
                        gg.scan_topk(po.L2, x[1], 3)
                    for s in range(g.gpus):
                        _check_layout(_Shard(g, s), keys, ids, bound[s], bound[s + 1], (g.gpus, s, how))
        finally:
            for g in groups:
                g.close()


# ------------------------------------------------------------------------------------------------ (2) kept layout = per call
@pytest.mark.parametrize("dim", [16, 384])
@pytest.mark.parametrize("vtype", TYPES)
def test_grouping_equals_per_call(vtype, dim):
    rng = np.random.Generator(np.random.PCG64(91_000 + 10 * vtype + dim))
    n = 3000
    x = _column(vtype, n, dim, rng)
    q = _column(vtype, 2, dim, rng)
    ids = np.arange(1, n + 1, dtype=np.int64)
    keys = _key_shapes(ids, rng)
    ix = _index(vtype, x)
    try:
        with ix.grouping(keys) as g:
            for metric in METRICS:
                for k in (1, 32, 33, 256):
                    for limit in (0, 1, 3):
                        _same(g.scan_topk(metric, q, k, limit), ix.scan_topk_grouped(metric, q, k, keys, limit), (vtype, dim, metric, k, limit))
    finally:
        ix.close()


def test_grouping_many_calls_any_order_and_groups():
    rng = np.random.Generator(np.random.PCG64(91_500))
    n, dim = 4000, 24
    x = _column(po.F32, n, dim, rng)
    ids = rng.permutation(np.arange(10, 10 + 3 * n, 3, dtype=np.int64))
    keys = _key_shapes(ids, rng)
    other = [rng.choice(ids, 50) for _ in range(40)]
    ix = _index(po.F32, x, ids)
    with _env(VSB_GROUP_ALIAS="1"):
        g2 = _group(po.F32, x, 2, ids)
    try:
        for obj in (ix, g2):
            gr = obj.grouping(keys)
            calls = [(m, k, lim, int(rng.integers(1, 4))) for m in METRICS for k in (1, 7, 33, 256) for lim in (0, 2)]
            for i in rng.permutation(len(calls)):
                m, k, lim, nq = calls[i]
                q = _column(po.F32, nq, dim, rng)
                want = obj.scan_topk_grouped(m, q, k, keys, lim)
                if i % 3 == 0:
                    obj.scan_topk_grouped(m, q, 5, other, 1)                 # a per-call grouped call in between
                _same(gr.scan_topk(m, q, k, lim), want, (obj, m, k, lim, nq))
            gr.close()
    finally:
        ix.close()
        g2.close()


# ------------------------------------------------------------------------------------------------ (3) counters
def test_grouping_counters():
    rng = np.random.Generator(np.random.PCG64(92_000))
    n = 6000
    x = _column(po.I8, n, 32, rng)
    keys = [rng.integers(1, n + 1, 400) for _ in range(100)]
    ix = _index(po.I8, x)
    try:
        l0 = ix.stat("grouped_layout_us")
        g = ix.grouping(keys)
        l1, r1 = ix.stat("grouped_layout_us"), ix.stat("grouped_layout_reuses")
        assert l1 > l0 and r1 == 0
        for i in range(5):
            g.scan_topk(po.L2, x[i], 10, 3)
        assert ix.stat("grouped_layout_us") == l1 and ix.stat("grouped_layout_reuses") == 5
        ix.scan_topk_grouped(po.L2, x[0], 10, keys, 3)
        assert ix.stat("grouped_layout_us") > l1 and ix.stat("grouped_layout_reuses") == 5
        g.scan_topk(po.L2, x[0], 0)                                          # k = 0: nothing runs
        assert ix.stat("grouped_layout_reuses") == 5
        g.close()
    finally:
        ix.close()


# ------------------------------------------------------------------------------------------------ (4) errors, lifetime
def test_grouping_errors_and_lifetime():
    vs = _vs()
    eng = vs.load_engine()
    rng = np.random.Generator(np.random.PCG64(93_000))
    n, dim = 2000, 16
    x = _column(po.I8, n, dim, rng)
    q = _column(po.I8, 2, dim, rng)
    keys = [rng.integers(1, n + 1, 50) for _ in range(20)]
    base = eng.debug_live_handles()
    for make in (lambda: _index(po.I8, x, cap=n + 10), lambda: _index(po.I8, x, window=500, cap=n + 10)):
        obj = make()
        g = obj.grouping(keys)
        assert eng.debug_live_handles() > base
        assert g.scan_topk(po.L2, q, 0) == [[], []]
        assert obj.grouping([]).scan_topk(po.L2, q, 5) == [[], []]
        for bad in (dict(k=257), dict(k=-1), dict(limit=-1), dict(metric=99)):
            a = dict(metric=po.L2, k=5, limit=0) | bad
            with pytest.raises(vs.VsbError) as e:
                g.scan_topk(a["metric"], q, a["k"], a["limit"])
            assert e.value.rc == vs.api.EINVAL, bad
        out = vs.api._vp()
        rid = np.arange(1, 5, dtype=np.int64)
        for offs, nk in ((np.array([1, 4], np.int64), 1), (np.array([0, 3, 2], np.int64), 2), (np.array([0, 4], np.int64), -1)):
            rc = eng.lib.vsb_grouping_create(obj.h, vs.api._ptr(rid), vs.api._ptr(offs), nk, vs.api.C.byref(out))
            assert rc == vs.api.EINVAL and not out.value, (offs, nk)
        assert eng.lib.vsb_grouping_create(obj.h, None, vs.api._ptr(np.array([0, 2], np.int64)), 1, vs.api.C.byref(out)) == vs.api.EINVAL
        assert eng.lib.vsb_scan_topk_grouping(None, po.L2, vs.api._ptr(q), 1, 5, 0, vs.api.C.byref(out)) == vs.api.EINVAL
        g.scan_topk(po.L2, q, 5)
        obj.append_dense(x[:3])                                              # the column changed
        with pytest.raises(vs.VsbError) as e:
            g.scan_topk(po.L2, q, 5)
        assert e.value.rc == vs.api.EINVAL and "changed" in str(e.value)
        g2 = obj.grouping(keys)
        g2.scan_topk(po.L2, q, 5)
        eng.lib.vsb_index_free(obj.h)                                        # the column first, behind Python's back
        obj.h = None
        for gr in (g, g2):
            with pytest.raises(vs.VsbError) as e:
                gr.scan_topk(po.L2, q, 5)
            assert e.value.rc == vs.api.EINVAL
            gr.close()
        assert eng.debug_live_handles() == base
    with _env(VSB_GROUP_ALIAS="1"):
        grp = _group(po.I8, x, 3)
    g = grp.grouping(keys)
    g.scan_topk(po.L2, q, 5)
    grp.close()                                                              # Python closes the column's groupings first
    assert g.h is None
    with pytest.raises(vs.VsbError):
        g.scan_topk(po.L2, q, 5)
    assert eng.debug_live_handles() == base


# ------------------------------------------------------------------------------------------------ (5) SQL
def _sql_setup(x, doc):
    s = ["CREATE TABLE t (id INTEGER PRIMARY KEY, e BLOB, doc INTEGER)", "SELECT vector_init('t','e','type=FLOAT32,dimension=16,distance=L2')"]
    s += [["INSERT INTO t(id, e, doc) VALUES (?, ?, ?)", [i + 1, {"hex": x[i].tobytes().hex()}, int(doc[i])]] for i in range(len(x))]
    return s


GROUPED = "SELECT key, id, distance FROM vector_full_scan_grouped('t','e',?,4,(SELECT vector_rowid_sets(doc, id) FROM t WHERE doc < ?),3)"
PER_KEY = "SELECT id, distance FROM vector_full_scan_filtered('t','e',?,4,(SELECT vector_rowid_set(id) FROM t WHERE doc = ?))"


def _grouped_ok(rows, per_key):
    keys = list(dict.fromkeys(r[0] for r in rows))
    assert 0 < len(keys) <= 3
    for d in keys:
        assert [r[1:] for r in rows if r[0] == d] == per_key[d], d


def test_sql_repeated_statement_reuses_the_grouping():
    rng = np.random.Generator(np.random.PCG64(94_000))
    x = rng.standard_normal((1500, 16), dtype=np.float32)
    doc = rng.integers(0, 30, 1500)
    qb = {"hex": x[7].tobytes().hex()}
    setup = _sql_setup(x, doc)
    stmt = [GROUPED, [qb, 20]]
    one = run_sql(OURS, setup + [stmt], want_launches=True)
    two = run_sql(OURS, setup + [stmt, stmt], want_launches=True)
    three = run_sql(OURS, setup + [stmt, stmt, stmt], want_launches=True)
    other = run_sql(OURS, setup + [stmt, [GROUPED, [qb, 25]]], want_launches=True)
    m = len(setup)
    assert "error" not in one[m] and one[m]["rows"]
    assert two[m + 1] == one[m] and three[m + 2] == one[m]
    reuse = two[-1]["kernel_launches"] - one[-1]["kernel_launches"]
    assert three[-1]["kernel_launches"] - two[-1]["kernel_launches"] == reuse
    assert other[-1]["kernel_launches"] - one[-1]["kernel_launches"] > reuse     # a different BLOB lays its keys out


def test_sql_changes_rebuild_the_grouping():
    rng = np.random.Generator(np.random.PCG64(94_500))
    x = rng.standard_normal((1200, 16), dtype=np.float32)
    doc = rng.integers(0, 25, 1200)
    close = {"hex": (x[3] + np.float32(1e-3)).tobytes().hex()}         # the query, and the rows inserted below
    qb = close
    s = _sql_setup(x, doc)
    m = len(s)
    per = lambda: [[PER_KEY, [qb, d]] for d in range(25)]
    plan = [("first", [[GROUPED, [qb, 20]]]), ("other blob", [[GROUPED, [qb, 12]]]),
            ("insert", ["INSERT INTO t(id, e, doc) VALUES (5000, ?, 2)"]), ("after insert", [[GROUPED, [qb, 12]]]),
            ("txn", ["BEGIN", "INSERT INTO t(id, e, doc) VALUES (5001, ?, 4)"]), ("in txn", [[GROUPED, [qb, 12]]]),
            ("rollback", ["ROLLBACK"]), ("after rollback", [[GROUPED, [qb, 12]]])]
    marks = {}
    for name, stmts in plan:
        stmts = [[st, [close]] if isinstance(st, str) and "?" in st else st for st in stmts]
        marks[name] = len(s)
        s += stmts
        if name in ("first", "other blob", "after insert", "in txn", "after rollback"):
            marks[name + " per"] = len(s)
            s += per()
    r = run_sql(OURS, s)
    assert all("error" not in x for x in r[m:]), [x for x in r[m:] if "error" in x]
    for name in ("first", "other blob", "after insert", "in txn", "after rollback"):
        per_key = {d: r[marks[name + " per"] + d]["rows"] for d in range(25)}
        rows = r[marks[name]]["rows"]
        _grouped_ok(rows, per_key)
        if name in ("after insert", "in txn"):
            assert rows[0][1] in (5000, 5001), name                        # the new row is the nearest
    assert 5001 not in [row[1] for row in r[marks["after rollback"]]["rows"]]
