"""Grouped top-k in passes of several queries (DESIGN §3.15, "Passes of several queries"): a call of nq queries returns, query
for query, bit for bit what nq single-query calls return, on a kept grouping and per call, for an index and a group.  -m gpu.

(1) every (type, metric) pair at dims 16 and 384 and a plan-switching shape (int8 dim 440, f32 dim 110 and their kin), k = 1 /
    3 / 32 / 33 / 256, limit 0 / 1 / 3 with ties at the limit, nq = 2 / 3 / 8 / 9 / 17; int types also equal the oracle for
    each returned key through its filtered scan; (2) the pass counters and one resident scan launch per pass; (3) each query's
    device state of a pass (vsb_debug_read "grouped_pass") against tests/groupedref.py on planted per-query distances (NaN, -INF,
    ties, key lengths around k and 1024, a 2M-row key) and on real distances, whose rows equal a single call's bit for bit;
    (4) a streamed index in ragged windows: resident answers, one column of stream bytes per pass; (5) groups of 1 - 3 shards,
    one streamed, with a key that makes the limit only through another shard; (6) a small grouped_mem_mb narrows the pass;
    (7) the grouped_dist hook at rows and nq x rows floats, a wrong size rejected; (8) nq = 0, k = 0, empty keys; (9) the SQL
    batch modules against the single module, BLOB and JSON queries, and the kept grouping shared between them."""
import contextlib
import json
import os

import numpy as np
import pytest

from oracle import pyoracle as po
from tests import groupedref as gr

pytestmark = pytest.mark.gpu
METRICS = [po.L2, po.L2SQ, po.COS, po.DOT, po.L1]
TYPES = [po.F32, po.F16, po.BF16, po.U8, po.I8]
NAN, INF = np.float32(np.nan), np.float32(np.inf)
# (1): a plan-switching shape per element type (the lanes per row or the ring change from dim 384)
SWITCH = {po.F32: 110, po.F16: 220, po.BF16: 220, po.U8: 440, po.I8: 440}


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
    with _env(VSB_GROUP_ALIAS="1"):
        yield


def _column(vtype, n, dim, rng):
    if vtype == po.I8:
        return rng.integers(-3, 4, (n, dim)).astype(np.int8)        # a small value set: ties between rows and keys
    if vtype == po.U8:
        return rng.integers(0, 5, (n, dim)).astype(np.uint8)
    return po.convert(rng.integers(-2, 3, (n, dim)).astype(np.float32) * np.float32(0.5) + rng.standard_normal((n, dim), dtype=np.float32)
                      * np.float32(rng.random() < 0.5), vtype)


def _index(vtype, x, rowids=None, window=0):
    ix = _vs().Index(vtype, x.shape[1], x.shape[0], window_rows=window)
    ix.append_dense(x, rowids)
    ix.finalize()
    return ix


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64)


def _same(got, want, ctx):
    """two grouped answers (per query: [(key, rowids, distances)]) equal bit for bit"""
    assert len(got) == len(want), ctx
    for b, (g, w) in enumerate(zip(got, want)):
        assert [t[0] for t in g] == [t[0] for t in w], (ctx, b)
        for (key, gi, gd), (_, wi, wd) in zip(g, w):
            assert np.array_equal(gi, wi) and np.array_equal(_bits(gd), _bits(wd)), (ctx, b, key)


def _singles(obj, metric, q, k, keys, limit):
    return [obj.scan_topk_grouped(metric, q[b], k, keys, limit)[0] for b in range(len(q))]


def _keys(ids, rng, k):
    """keys around k rows, a long one, ties-prone small ones, an empty one and an absent rowid"""
    n = len(ids)
    keys = [ids[:max(k - 1, 1)], ids[k:2 * k + 1], ids[n // 3: n // 3 + 1100], np.zeros(0, np.int64), np.array([-5], np.int64)]
    keys += [rng.choice(ids, int(rng.integers(1, 60)), replace=False) for _ in range(30)]
    return keys


# ------------------------------------------------------------------------------------------------ (1) every pair
CASES = [(1, 0, 2), (3, 1, 3), (32, 3, 8), (33, 1, 9), (256, 3, 17), (3, 0, 17), (33, 3, 2)]


@pytest.mark.parametrize("vtype", TYPES)
def test_every_pair_equals_single_calls(oracle, vtype):
    rng = np.random.Generator(np.random.PCG64(95_000 + vtype))
    n = 2500
    for dim in (16, 384, SWITCH[vtype]):
        x = _column(vtype, n, dim, rng)
        ids = (rng.permutation(n) * 3 + 1).astype(np.int64)
        row_of = gr.RowMap(ids)
        ix = _index(vtype, x, ids)
        try:
            for mi, metric in enumerate(METRICS):
                k, limit, nq = CASES[(mi + dim) % len(CASES)]
                keys = _keys(ids, rng, k)
                q = _column(vtype, nq, dim, rng)
                q[1] = x[5]                                             # a query on a row: ties at distance 0
                want = _singles(ix, metric, q, k, keys, limit)
                got = ix.scan_topk_grouped(metric, q, k, keys, limit)
                _same(got, want, (vtype, dim, metric, "per call"))
                with ix.grouping(keys) as g:
                    _same(g.scan_topk(metric, q, k, limit), want, (vtype, dim, metric, "kept"))
                    k2, limit2, nq2 = CASES[(mi + dim + 3) % len(CASES)]
                    q2 = _column(vtype, nq2, dim, rng)
                    _same(g.scan_topk(metric, q2, k2, limit2), _singles(ix, metric, q2, k2, keys, limit2), (vtype, dim, metric, k2))
                if vtype in (po.I8, po.U8):
                    for key, gi, gd in got[0][:6]:
                        rows = np.sort(row_of(keys[key]))
                        rows = rows[np.r_[True, rows[1:] != rows[:-1]]] if len(rows) else rows
                        wi, wd = oracle.scan_dense(metric, vtype, q[0], x[rows], ids[rows], k)
                        assert np.array_equal(gi, wi) and np.array_equal(_bits(gd), _bits(wd)), (dim, metric, key)
        finally:
            ix.close()


# ------------------------------------------------------------------------------------------------ (2) pass counters
def test_pass_counters_and_one_scan_per_pass():
    rng = np.random.Generator(np.random.PCG64(95_100))
    n, dim = 20_000, 64
    x = _column(po.I8, n, dim, rng)
    ids = np.arange(1, n + 1, dtype=np.int64)
    ix = _index(po.I8, x)
    eng = ix.eng
    try:
        keys = [ids[i::50] for i in range(50)]
        q = _column(po.I8, 8, dim, rng)
        with ix.grouping(keys) as g:
            g.scan_topk(po.L2, q[:1], 5, 3)                              # warm: the pass buffers exist
            l0, p0, w0 = eng.kernel_launches(), ix.stat("grouped_passes"), ix.stat("grouped_pass_queries")
            g.scan_topk(po.L2, q[:1], 5, 3)
            single = eng.kernel_launches() - l0
            assert (ix.stat("grouped_passes") - p0, ix.stat("grouped_pass_queries") - w0) == (1, 1)
            l0, p0, w0 = eng.kernel_launches(), ix.stat("grouped_passes"), ix.stat("grouped_pass_queries")
            g.scan_topk(po.L2, q, 5, 3)
            passes = ix.stat("grouped_passes") - p0
            assert ix.stat("grouped_pass_queries") - w0 == 8 and passes < 8       # several queries shared each pass
            assert eng.kernel_launches() - l0 == passes * single                    # one scan (and one of each step) per pass
    finally:
        ix.close()


# ------------------------------------------------------------------------------------------------ (3) device state
def _check_pass_state(ix, dists, key_rows, k, limit, ctx):
    st = ix.debug_grouped_pass()
    assert len(st["queries"]) == len(dists), ctx
    for j, qs in enumerate(st["queries"]):
        want = gr.state(dists[j], key_rows, k, limit=limit)
        got = dict({n: st[n] for n in ("rows", "koff", "pstart", "pkey", "kpiece")}, k=st["k"], **qs)
        assert gr.diff(got, want) == [], (ctx, j)
    return st


def test_planted_pass_state():
    rng = np.random.Generator(np.random.PCG64(95_200))
    n = 2_100_000
    ids = np.arange(1, n + 1, dtype=np.int64)
    row_of = gr.RowMap(ids)
    ix = _index(po.I8, np.zeros((n, 4), np.int8))
    try:
        for k, limit in ((3, 2), (33, 0), (256, 1)):
            keys = [ids[:2_000_000:1]] + [ids[2_000_000 + 1100 * i: 2_000_000 + 1100 * i + L]
                                          for i, L in enumerate((k - 1, k, k + 1, 1023, 1024, 1025))]
            keys += [rng.choice(ids[2_010_000:], int(rng.integers(1, 300)), replace=False) for _ in range(12)]
            kr = gr.shard_rows(keys, row_of, 0, n)
            nq = 3
            dists = rng.standard_normal((nq, n)).astype(np.float32)
            dists[0, 2_000_000:2_001_100] = NAN
            dists[1, 2_000_000:2_000_400] = -INF
            dists[2, :] = np.round(dists[2, :])                          # ties everywhere, at the limit too
            dists[1, 5:20] = NAN
            ix.debug_write("grouped_dist", dists.reshape(-1))
            got = ix.scan_topk_grouped(po.L2, np.zeros((nq, 4), np.int8), k, keys, limit)
            _check_pass_state(ix, dists, kr, k, limit, (k, limit))
            for j in range(nq):                                          # each query alone on its own row
                ix.debug_write("grouped_dist", dists[j])
                _same([got[j]], ix.scan_topk_grouped(po.L2, np.zeros(4, np.int8), k, keys, limit), (k, limit, j))
    finally:
        ix.close()


@pytest.mark.parametrize("vtype", TYPES)
def test_real_pass_state(vtype):
    rng = np.random.Generator(np.random.PCG64(95_300 + vtype))
    n, dim = 6000, 48
    x = _column(vtype, n, dim, rng)
    ids = (rng.permutation(n) + 10).astype(np.int64)
    row_of = gr.RowMap(ids)
    ix = _index(vtype, x, ids)
    try:
        keys = [ids[:1500]] + [rng.choice(ids, int(rng.integers(1, 200)), replace=False) for _ in range(20)]
        kr = gr.shard_rows(keys, row_of, 0, n)
        for metric in METRICS:
            for k, limit in ((1, 0), (33, 4)):
                q = _column(vtype, 3, dim, rng)
                ix.scan_topk_grouped(metric, q, k, keys, limit)
                st = ix.debug_grouped_pass()
                dists = [qs["dist"] for qs in st["queries"]]
                _check_pass_state(ix, dists, kr, k, limit, (metric, k))
                for j in range(3):
                    ix.scan_topk_grouped(metric, q[j], k, keys, limit)
                    assert np.array_equal(ix.debug_grouped()["dist"].view(np.uint32), dists[j].view(np.uint32)), (metric, k, j)
    finally:
        ix.close()


# ------------------------------------------------------------------------------------------------ (4) streamed
@pytest.mark.parametrize("window", [700, 4096])
def test_streamed_pass(window):
    rng = np.random.Generator(np.random.PCG64(95_400 + window))
    n, dim = 10_001, 32
    x = _column(po.I8, n, dim, rng)
    ids = np.arange(1, n + 1, dtype=np.int64)
    res, st = _index(po.I8, x), _index(po.I8, x, window=window)
    try:
        assert st.eng.lib.vsb_index_is_streamed(st.h) == 1
        keys = [ids[i::40] for i in range(40)]
        q = _column(po.I8, 8, dim, rng)
        for metric, k, limit in ((po.L2, 3, 5), (po.DOT, 33, 0), (po.L1, 256, 2)):
            want = res.scan_topk_grouped(metric, q, k, keys, limit)
            s0, p0 = st.stat("stream_bytes"), st.stat("grouped_passes")
            got = st.scan_topk_grouped(metric, q, k, keys, limit)
            passes = st.stat("grouped_passes") - p0
            assert passes < len(q)
            assert st.stat("stream_bytes") - s0 == passes * n * st.query_pitch, (window, metric)
            _same(got, want, (window, metric))
    finally:
        res.close()
        st.close()


# ------------------------------------------------------------------------------------------------ (5) groups
@pytest.mark.parametrize("ngpus", [1, 2, 3])
def test_group_passes(ngpus):
    rng = np.random.Generator(np.random.PCG64(95_500 + ngpus))
    n, dim = 6001, 16
    x = _column(po.F32, n, dim, rng)
    ids = np.arange(1, n + 1, dtype=np.int64)
    probe = _index(po.F32, x[:1])
    pitch = probe.query_pitch
    probe.close()
    with _env(**({"VSB_DEVICE_BUDGET_MB": repr(2000.5 * pitch / 1048576.0)} if ngpus == 3 else {})):
        g = _vs().Group(po.F32, dim, n, ngpus)
        g.append_dense(x)
        g.finalize()
    lone = _index(po.F32, x)
    try:
        bounds = np.linspace(0, n, ngpus + 1).astype(int)
        q = _column(po.F32, 5, dim, rng)
        # key 0: rows on every shard, but its only near row is on the last shard
        key0 = np.concatenate([ids[b:b + 5] for b in bounds[:-1]] + [ids[n - 3:n - 2]])
        keys = [key0] + [rng.choice(ids, int(rng.integers(1, 150)), replace=False) for _ in range(25)]
        q[:, :] = x[n - 3] + np.float32(1e-3)                             # every query nearest to key 0's last-shard row
        q[1:] += rng.standard_normal((4, dim), dtype=np.float32) * np.float32(0.01)
        for k, limit in ((1, 1), (33, 3), (3, 0)):
            want = _singles(g, po.L2, q, k, keys, limit)
            got = g.scan_topk_grouped(po.L2, q, k, keys, limit)
            if ngpus < 3:                                                 # resident shards: the lone index's bits too
                _same(got, _singles(lone, po.L2, q, k, keys, limit), (ngpus, k, limit, "lone"))
            _same(got, want, (ngpus, k, limit))
            if limit == 1:
                assert [t[0] for t in got[0]] == [0], (ngpus, k)
            with g.grouping(keys) as gg:
                _same(gg.scan_topk(po.L2, q, k, limit), want, (ngpus, k, limit, "kept"))
    finally:
        g.close()
        lone.close()


# ------------------------------------------------------------------------------------------------ (6) budget
def test_budget_narrows_the_pass():
    rng = np.random.Generator(np.random.PCG64(95_600))
    n, dim = 200_000, 16
    x = _column(po.I8, n, dim, rng)
    ids = np.arange(1, n + 1, dtype=np.int64)
    ix = _index(po.I8, x)
    try:
        keys = [ids[i::500] for i in range(500)]
        q = _column(po.I8, 8, dim, rng)
        p0 = ix.stat("grouped_passes")
        want = ix.scan_topk_grouped(po.L2, q, 3, keys, 10)
        wide = ix.stat("grouped_passes") - p0
        with _options(grouped_mem_mb=1):                                 # 0.8 MB of distances a query: one query a pass
            p0 = ix.stat("grouped_passes")
            got = ix.scan_topk_grouped(po.L2, q, 3, keys, 10)
            narrow = ix.stat("grouped_passes") - p0
        assert narrow == 8 and wide < narrow
        _same(got, want, "budget")
    finally:
        ix.close()


# ------------------------------------------------------------------------------------------------ (7) hooks, (8) edges
def test_plant_sizes_and_edges():
    vs = _vs()
    rng = np.random.Generator(np.random.PCG64(95_700))
    n = 5000
    ids = np.arange(1, n + 1, dtype=np.int64)
    ix = _index(po.I8, np.zeros((n, 4), np.int8))
    try:
        keys = [ids[i::30] for i in range(30)]
        q = np.zeros((3, 4), np.int8)
        d = rng.standard_normal(n).astype(np.float32)
        ix.debug_write("grouped_dist", d)                                # one row: every query uses it
        got = ix.scan_topk_grouped(po.L2, q, 3, keys, 4)
        _same(got[1:], got[:2], "one row")
        d3 = rng.standard_normal((3, n)).astype(np.float32)
        ix.debug_write("grouped_dist", d3.reshape(-1))                   # nq rows: query j uses row j
        got = ix.scan_topk_grouped(po.L2, q, 3, keys, 4)
        for j in range(3):
            ix.debug_write("grouped_dist", d3[j])
            _same([got[j]], ix.scan_topk_grouped(po.L2, q[0], 3, keys, 4), ("nq rows", j))
        with pytest.raises(vs.VsbError) as e:
            ix.debug_write("grouped_dist", np.zeros(n + 1, np.float32))   # not whole rows: at write time
        assert e.value.rc == vs.api.EINVAL
        ix.debug_write("grouped_dist", np.zeros(2 * n, np.float32))      # two rows for three queries: at the call
        with pytest.raises(vs.VsbError) as e:
            ix.scan_topk_grouped(po.L2, q, 3, keys, 4)
        assert e.value.rc == vs.api.EINVAL
        # edges: no queries, k = 0, no keys, keys without rows
        assert ix.scan_topk_grouped(po.L2, np.zeros((0, 4), np.int8), 3, keys, 4) == []
        assert ix.scan_topk_grouped(po.L2, q, 0, keys, 4) == [[], [], []]
        assert ix.scan_topk_grouped(po.L2, q, 3, [], 4) == [[], [], []]
        assert ix.scan_topk_grouped(po.L2, q, 3, [np.zeros(0, np.int64), np.array([-1], np.int64)], 0) == [[], [], []]
    finally:
        ix.close()


# ------------------------------------------------------------------------------------------------ (9) SQL
def test_sql_batch_modules():
    from tests.sqlrun import OURS, run_sql
    rng = np.random.Generator(np.random.PCG64(95_800))
    n, dim, B = 1500, 16, 5
    x = rng.standard_normal((n, dim), dtype=np.float32)
    doc = rng.integers(0, 30, n)
    q = rng.standard_normal((B, dim), dtype=np.float32)
    s = ["CREATE TABLE t (id INTEGER PRIMARY KEY, e BLOB, doc INTEGER)",
         "SELECT vector_init('t','e','type=FLOAT32,dimension=16,distance=L2')"]
    s += [["INSERT INTO t(id, e, doc) VALUES (?, ?, ?)", [i + 1, {"hex": x[i].tobytes().hex()}, int(doc[i])]] for i in range(n)]
    s += ["SELECT vector_quantize('t','e')"]
    groups = "(SELECT vector_rowid_sets(doc, id) FROM t WHERE doc < 25)"
    m = len(s)
    plan = []
    for mod in ("full", "quantize"):
        single = f"SELECT key, id, distance FROM vector_{mod}_scan_grouped('t','e',?,3,{groups},4)"
        batch = f"SELECT query, key, id, distance FROM vector_{mod}_scan_grouped_batch('t','e',?,3,{groups},4)"
        for b in range(B):
            plan.append(("single", mod, b, [single, [{"hex": q[b].tobytes().hex()}]]))
        plan.append(("blob", mod, None, [batch, [{"hex": q.tobytes().hex()}]]))
        plan.append(("json", mod, None, [batch, [json.dumps([float(v) for v in q.reshape(-1)])]]))
        plan.append(("k0", mod, None, [batch.replace(",3,", ",0,"), [{"hex": q.tobytes().hex()}]]))
    s += [p[3] for p in plan]
    r = run_sql(OURS, s)
    assert all("error" not in v for v in r[m:]), [v for v in r[m:] if "error" in v]
    for mod in ("full", "quantize"):
        want = []
        for i, (kind, md, b, _) in enumerate(plan):
            if kind == "single" and md == mod:
                rows = r[m + i]["rows"]
                assert rows
                want += [[b] + row for row in rows]
        for i, (kind, md, _, _) in enumerate(plan):
            if md == mod and kind in ("blob", "json"):
                assert r[m + i]["rows"] == want, (mod, kind)
            if md == mod and kind == "k0":
                assert r[m + i]["rows"] == [], mod


def test_sql_batch_shares_the_kept_grouping():
    from tests.sqlrun import OURS, run_sql
    rng = np.random.Generator(np.random.PCG64(95_900))
    n, dim = 1200, 16
    x = rng.standard_normal((n, dim), dtype=np.float32)
    doc = rng.integers(0, 20, n)
    q = rng.standard_normal((4, dim), dtype=np.float32)
    s = ["CREATE TABLE t (id INTEGER PRIMARY KEY, e BLOB, doc INTEGER)",
         "SELECT vector_init('t','e','type=FLOAT32,dimension=16,distance=L2')"]
    s += [["INSERT INTO t(id, e, doc) VALUES (?, ?, ?)", [i + 1, {"hex": x[i].tobytes().hex()}, int(doc[i])]] for i in range(n)]
    groups = "(SELECT vector_rowid_sets(doc, id) FROM t)"
    single = [f"SELECT key, id, distance FROM vector_full_scan_grouped('t','e',?,3,{groups},5)", [{"hex": q[0].tobytes().hex()}]]
    batch = [f"SELECT query, key, id, distance FROM vector_full_scan_grouped_batch('t','e',?,3,{groups},5)", [{"hex": q.tobytes().hex()}]]
    base = run_sql(OURS, s + [single], want_launches=True)
    after = run_sql(OURS, s + [single, batch], want_launches=True)
    lay = run_sql(OURS, s + [batch], want_launches=True)
    again = run_sql(OURS, s + [batch, single], want_launches=True)
    m = len(s)
    assert [[0] + row for row in base[m]["rows"]] == [row for row in after[m + 1]["rows"] if row[0] == 0]
    # a batch after a single statement with the same groups BLOB lays nothing out: it costs what a batch on a kept layout costs
    batch_kept = after[-1]["kernel_launches"] - base[-1]["kernel_launches"]
    batch_fresh = lay[-1]["kernel_launches"] - run_sql(OURS, s, want_launches=True)[-1]["kernel_launches"]
    assert batch_kept < batch_fresh
    single_kept = again[-1]["kernel_launches"] - lay[-1]["kernel_launches"]
    single_fresh = base[-1]["kernel_launches"] - run_sql(OURS, s, want_launches=True)[-1]["kernel_launches"]
    assert single_kept < single_fresh
    assert again[m + 1]["rows"] == base[m]["rows"]
