"""Large k (k > 256, DESIGN §3.11): the exact k nearest from a GPU-selected candidate set.  -m gpu.

The yardstick is the engine's own all-distances scan replayed over EVERY row (vsb_scan_all + vsb_replay_topk): the path k > 256
took before, reached through public calls, so the answers must match it bit for bit for every element type.  The candidate set
and the prefix bounds are restated in numpy from the same distances: segment ends k, 2k, 4k, ... below n, then n; the bound of
segment s >= 1 is the k-th smallest key (float order, -0 < +0) of the eligible non-NaN rows of [0, ends[s - 1]), +INF when there
are fewer than k; the candidates are the eligible rows with d < their segment's bound, in scan order."""
import base64
import contextlib
import json
import os
import struct

import numpy as np
import pytest

from oracle import pyoracle as po
from tests.fpcheck import assert_fp_topk
from tests.sqlrun import OURS, run_sql

pytestmark = pytest.mark.gpu
TYPES = [po.F32, po.F16, po.BF16, po.U8, po.I8]
METRICS = [po.L2, po.L2SQ, po.COS, po.DOT, po.L1]
INTS = (po.U8, po.I8)


def _vs():
    import sqlite_vector_b200 as vs
    return vs


@pytest.fixture(scope="module", autouse=True)
def _alias():
    old = os.environ.get("VSB_GROUP_ALIAS")
    os.environ["VSB_GROUP_ALIAS"] = "1"
    yield
    os.environ.pop("VSB_GROUP_ALIAS", None) if old is None else os.environ.update(VSB_GROUP_ALIAS=old)


@pytest.fixture(scope="module")
def oracle():
    return po.Oracle()


@contextlib.contextmanager
def _env(**kv):
    old = {k: os.environ.get(k) for k in kv}
    os.environ.update({k: str(v) for k, v in kv.items()})
    try:
        yield
    finally:
        for k, v in old.items():
            os.environ.pop(k, None) if v is None else os.environ.update({k: v})


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


def expect_candidates(d, k, allow=None):
    """(candidate rows in scan order, segment ends, segment bounds) of one view"""
    n = len(d)
    ends, e = [], k
    while e < n and len(ends) < 31:
        ends.append(e)
        e *= 2
    ends.append(n)
    elig = np.ones(n, bool) if allow is None else np.asarray(allow, bool)
    key = _key(d)
    bounds = [np.float32(np.inf)]
    for j in range(len(ends) - 1):
        kk = key[:ends[j]][(elig & ~np.isnan(d))[:ends[j]]]
        bounds.append(np.float32(np.inf) if len(kk) < k else _unkey(np.partition(kk, k - 1)[k - 1]))
    seg = np.searchsorted(np.asarray(ends), np.arange(n), side="right")
    with np.errstate(invalid="ignore"):
        cand = elig & (d < np.asarray(bounds, np.float32)[seg])
    return np.nonzero(cand)[0], np.asarray(ends, np.int64), np.asarray(bounds, np.float32)


def topk_bounds(ix):
    raw = ix.debug_read("topk_bounds", np.uint8, 8 + 8 * 32 + 4 * 32)
    nseg = int(raw[:8].view(np.int64)[0])
    return raw[8:264].view(np.int64)[:nseg].copy(), raw[264:392].view(np.float32)[:nseg].copy()


def old_path(eng, d_all, ids, k, mi=0):
    """the parent's k > 256 answer: every row through the slot replay"""
    c = np.zeros(len(d_all), dtype=_vs().api.CAND_DTYPE)
    c["dist"], c["rowid"], c["seq"] = d_all, ids, np.arange(len(d_all))
    return eng.replay_topk(c, k, max_index=mi)


def same(got, want, ctx):
    assert np.array_equal(got[0], want[0]), (ctx, "rowids")
    assert np.array_equal(_bits(np.asarray(got[1], np.float64)), _bits(np.asarray(want[1], np.float64))), (ctx, "distances")


# ------------------------------------------------------------------------------------------------ bit-identical to the old path
@pytest.mark.parametrize("dim", [5, 128, 771])
@pytest.mark.parametrize("vtype", TYPES)
def test_topk_equals_replay_over_every_row(oracle, vtype, dim):
    rng = np.random.Generator(np.random.PCG64(100 + dim + vtype))
    n = 3000
    x = _column(vtype, n, dim, rng)
    ids = np.arange(1, n + 1, dtype=np.int64)
    ix = _index(vtype, x)
    q = _column(vtype, 1, dim, rng)[0]
    eng = ix.eng
    for metric in METRICS:
        d_all = ix.scan_all(metric, q)
        for k in (257, 300, 1000, 4096, n - 1, n, 2 * n):
            q0, c0 = ix.stat("large_k_queries"), ix.stat("large_k_cands")
            (got,) = ix.scan_topk(metric, q, k)
            assert ix.stat("large_k_queries") == q0 + 1
            want = old_path(eng, d_all, ids, k)
            same(got, want, (vtype, dim, metric, k))
            assert ix.stat("large_k_cands") - c0 <= n
            o_ids, o_d = oracle.scan_dense(metric, vtype, q, x, ids, k, int_exact=vtype in INTS)
            if vtype in INTS:
                same(got, (o_ids, o_d), (vtype, dim, metric, k, "oracle"))
            else:
                dmap = dict(zip(ids.tolist(), oracle.distances_all(metric, vtype, q, x).tolist()))
                assert_fp_topk(got[0], got[1], o_ids, o_d, metric, lambda r: dmap[r], (vtype, dim, metric, k))
    ix.close()


# ------------------------------------------------------------------------------------------------ the candidate set and bounds
def _check_candidates(ix, metric, q, k, ctx):
    d_all = ix.scan_all(metric, q)
    (c,) = ix.scan_candidates(metric, q, k, cap=len(d_all) + 1)
    rows, ends, bounds = expect_candidates(d_all, k)
    assert np.array_equal(c["seq"], rows), (ctx, len(c), len(rows))
    assert np.array_equal(_bits(c["dist"]), _bits(d_all[rows])), ctx
    got_ends, got_bounds = topk_bounds(ix)
    assert np.array_equal(got_ends, ends) and np.array_equal(_bits(got_bounds), _bits(bounds)), (ctx, got_bounds, bounds)
    return d_all, c


def test_candidates_and_bounds_equal_numpy():
    eng = _vs().load_engine()
    rng = np.random.Generator(np.random.PCG64(200))
    n = 50_000
    x = _column(po.I8, n, 24, rng)
    x[rng.random(n) < 0.3] = 0                                        # heavy ties
    ix = _index(po.I8, x)
    q = _column(po.I8, 1, 24, rng)[0]
    for metric in METRICS:
        for k in (257, 1000, 4096, 30_000, n - 1, n, 2 * n):
            d_all, c = _check_candidates(ix, metric, q, k, ("i8", metric, k))
            if k <= 4096:                                              # (the O(k^2) exchange sort of larger k: the test above)
                same(eng.replay_topk(c, k)[:2], old_path(eng, d_all, np.arange(1, n + 1), k)[:2], ("replay", metric, k))
            if k == 1000 and metric == po.L2:
                assert len(c) < n // 4, len(c)                         # random order: about k (1 + log2(n / k)) rows
    ix.close()


def test_candidates_with_nan_inf_and_equal_rows():
    rng = np.random.Generator(np.random.PCG64(201))
    n, dim = 20_000, 16
    x = rng.standard_normal((n, dim), dtype=np.float32)
    x[rng.random(n) < 0.05, 3] = np.nan                               # NaN distances: never candidates, never counted
    ix = _index(po.F32, x)
    q = rng.standard_normal(dim, dtype=np.float32)
    for metric in (po.L2, po.DOT, po.COS):
        for k in (257, 3000, 19_000):
            _check_candidates(ix, metric, q, k, ("nan", metric, k))
    ix.close()
    # f16 DOT: rows holding +INF give -INF distances (and INF * 0 gives NaN)
    h = po.convert(rng.standard_normal((n, dim), dtype=np.float32), po.F16)
    hv = h.view(np.uint16)
    hv[rng.random(n) < 0.03, 0] = 0x7C00
    hq = po.convert(np.abs(rng.standard_normal(dim, dtype=np.float32)) + 0.1, po.F16)
    ix = _index(po.F16, h)
    for k in (257, 5000):
        _check_candidates(ix, po.DOT, hq, k, ("f16 -inf", k))
    ix.close()
    # every distance equal: the first k rows, then nothing beats the bound
    ix = _index(po.U8, np.full((n, 8), 7, np.uint8))
    d_all, c = _check_candidates(ix, po.L2, np.zeros(8, np.uint8), 300, "equal")
    assert len(c) == 300
    ix.close()


def test_filters_fewer_than_k_and_none():
    eng = _vs().load_engine()
    rng = np.random.Generator(np.random.PCG64(202))
    n = 40_000
    x = _column(po.I8, n, 32, rng)
    ids = np.arange(1, n + 1, dtype=np.int64) * 3
    ix = _index(po.I8, x, ids)
    q = _column(po.I8, 1, 32, rng)[0]
    masks = {"random": rng.random(n) < 0.2, "clustered": (np.arange(n) // 3000) % 3 == 1, "sparse": rng.random(n) < 0.004,
             "none": np.zeros(n, bool)}
    for name, m in masks.items():
        for metric in (po.L2, po.DOT, po.L1):
            d_all = ix.scan_all(metric, q)
            for k in (257, 1000, 5000):
                got = ix.scan_topk_filtered(metric, q, k, m)[0]
                want = old_path(eng, d_all[m], ids[m], k)
                same(got, want, (name, metric, k))
                ends, bounds = expect_candidates(d_all, k, m)[1:]
                got_ends, got_bounds = topk_bounds(ix)
                assert np.array_equal(got_ends, ends) and np.array_equal(_bits(got_bounds), _bits(bounds)), (name, metric, k)
    ix.close()


def test_descending_distances_regrow_and_stay_exact():
    """strictly falling distances: every row is a candidate; 100 000 pairs outgrow the first list (65 536 pairs)"""
    eng = _vs().load_engine()
    n = 100_000
    x = np.zeros((n, 5), np.float32)
    x[:, 0] = np.arange(n, 0, -1, dtype=np.float32)
    q = np.zeros(5, np.float32)
    ids = np.arange(1, n + 1, dtype=np.int64)
    for window in (0, 30_000):
        ix = _index(po.F32, x, window=window)
        r0 = ix.stat("large_k_regrows")
        (got,) = ix.scan_topk(po.L1, q, 300)
        assert ix.stat("large_k_regrows") == r0 + 1, window
        same(got, old_path(eng, ix.scan_all(po.L1, q), ids, 300), ("descending", window))
        (got,) = ix.scan_topk(po.L1, q, 300)                         # the list has grown: no second regrow
        assert ix.stat("large_k_regrows") == r0 + 1, window
        ix.close()


def test_max_index_carries_across_k(oracle):
    rng = np.random.Generator(np.random.PCG64(203))
    n = 6000
    x = rng.integers(0, 3, (n, 8)).astype(np.uint8)
    ids = np.arange(1, n + 1, dtype=np.int64)
    ix = _index(po.U8, x)
    mi = 0
    for k, seed in ((300, 1), (1000, 2), (257, 3), (20, 4)):
        q = rng.integers(0, 3, 8).astype(np.uint8)
        got, new_mi = ix.scan_topk(po.L2, q, k, max_index=mi)
        want = oracle.scan_dense(po.L2, po.U8, q, x, ids, k, start_max_index=mi, int_exact=True)
        same(got[0], want, (k, mi))
        mi_ref = old_path(ix.eng, ix.scan_all(po.L2, q), ids, k, mi)[2]
        assert new_mi == mi_ref, (k, new_mi, mi_ref)
        mi = new_mi
    ix.close()


# ------------------------------------------------------------------------------------------------ every other path == resident
@pytest.mark.parametrize("window", [128, 300, 5000, 100_000])
def test_streamed_windows_equal_resident(window):
    rng = np.random.Generator(np.random.PCG64(300 + window))
    n = 30_000
    x = _column(po.I8, n, 40, rng)
    ids = np.arange(1, n + 1, dtype=np.int64) * 2
    st, res = _index(po.I8, x, ids, window=window), _index(po.I8, x, ids)
    qs = _column(po.I8, 2, 40, rng)
    m = (np.arange(n) // 700) % 2 == 0
    for metric in (po.L2, po.DOT):
        for k in (257, 1000, 5000):
            same(st.scan_topk(metric, qs[0], k)[0], res.scan_topk(metric, qs[0], k)[0], (window, metric, k))
            same(st.scan_topk_filtered(metric, qs[1], k, m)[0], res.scan_topk_filtered(metric, qs[1], k, m)[0], (window, metric, k, "filtered"))
    if window < n:                                                    # the last window's own segments and bounds
        last = n - ((n - 1) // window) * window
        d_last = st.scan_all(po.L2, qs[0])[n - last:]
        st.scan_topk(po.L2, qs[0], 257)
        ends, bounds = expect_candidates(d_last, 257)[1:]
        got_ends, got_bounds = topk_bounds(st)
        assert np.array_equal(got_ends, ends) and np.array_equal(_bits(got_bounds), _bits(bounds)), window
    st.close(); res.close()


@pytest.mark.parametrize("ngpus", [1, 3])
def test_groups_equal_one_index(ngpus):
    rng = np.random.Generator(np.random.PCG64(400 + ngpus))
    n = 25_001
    x = _column(po.U8, n, 20, rng)
    ids = rng.permutation(3 * n)[:n].astype(np.int64) + 1
    g, ix = _group(po.U8, x, ngpus, ids), _index(po.U8, x, ids)
    qs = _column(po.U8, 20, 20, rng)
    m = np.zeros(n, bool)
    m[n // 3 - 500:n // 3 + 500] = True                               # across the first shard boundary
    m |= rng.random(n) < 0.05
    for metric in (po.L2, po.COS, po.L1):
        for k in (257, 2000):
            same(g.scan_topk(metric, qs[0], k)[0], ix.scan_topk(metric, qs[0], k)[0], (ngpus, metric, k))
            same(g.scan_topk_filtered(metric, qs[1], k, m)[0], ix.scan_topk_filtered(metric, qs[1], k, m)[0], (ngpus, metric, k, "filtered"))
    got = g.scan_topk(po.L2, qs, 300)                                 # 20 queries: one at a time, each on the large-k path
    for b in range(20):
        same(got[b], ix.scan_topk(po.L2, qs[b], 300)[0], (ngpus, "batch", b))
    g.close()
    with _env(VSB_DEVICE_BUDGET_MB="0.2"):                            # a streamed group
        gs = _group(po.U8, x, ngpus, ids)
    assert all(gs.eng.lib.vsb_index_is_streamed(gs.eng.lib.vsb_group_shard(gs.h, s)) for s in range(ngpus))
    for k in (257, 3000):
        same(gs.scan_topk(po.L1, qs[2], k)[0], ix.scan_topk(po.L1, qs[2], k)[0], (ngpus, "streamed", k))
        same(gs.scan_topk_filtered(po.L2, qs[3], k, m)[0], ix.scan_topk_filtered(po.L2, qs[3], k, m)[0], (ngpus, "streamed filtered", k))
    gs.close(); ix.close()


def test_batch_equals_single_calls():
    rng = np.random.Generator(np.random.PCG64(500))
    n = 40_000
    for vtype in (po.I8, po.BF16):
        x = _column(vtype, n, 64, rng)
        ix = _index(vtype, x)
        qs = _column(vtype, 20, 64, rng)
        q0 = ix.stat("large_k_queries")
        got = ix.scan_topk(po.L2, qs, 300)
        assert ix.stat("large_k_queries") == q0 + 20
        for b in range(20):
            same(got[b], ix.scan_topk(po.L2, qs[b], 300)[0], (vtype, b))
        ix.close()


# ------------------------------------------------------------------------------------------------ SQL and handles
def _rowid_blob(ids):
    return {"hex": struct.pack("<%dq" % len(ids), *ids).hex()}


def golden_setup(gold):
    """the SQL that builds the tables of tests/golden/sql_large_k.json (tools/large_k_golden.py records the reference with it):
    rowids 1..n, elements from the digit strings; <name>_sub holds the rows of `keep` only"""
    setup = []
    for t in gold["tables"]:
        x = np.array([int(c) for c in t["x"]], np.float32).reshape(-1, t["dim"])
        for name in (t["name"], t["name"] + "_sub"):
            setup += [f"CREATE TABLE {name} (id INTEGER PRIMARY KEY, e BLOB)", f"SELECT vector_init('{name}', 'e', '{t['opts']}')"]
        setup.append("INSERT INTO %s VALUES %s" % (t["name"], ", ".join(f"({i + 1}, x'{v.tobytes().hex()}')" for i, v in enumerate(x))))
        setup.append(f"INSERT INTO {t['name']}_sub SELECT id, e FROM {t['name']} WHERE id IN ({','.join(map(str, t['keep']))})")
        if t["qopts"]:
            setup += [f"SELECT vector_quantize('{n}', 'e', '{t['qopts']}')" for n in (t["name"], t["name"] + "_sub")]
    return setup


def golden_query(gold, e, filtered_module=False):
    """one case as SQL: a filtered case is the plain module over <name>_sub, or (filtered_module) the _filtered module over <name>
    with the rowids of `keep`"""
    t = next(t for t in gold["tables"] if t["name"] == e["table"])
    q = np.array([int(c) for c in t["query"]], np.float32).tobytes().hex()
    mod = "vector_quantize_scan" if e["quantized"] else "vector_full_scan"
    if e["filtered"] and filtered_module:
        return [f"SELECT id, distance FROM {mod}_filtered('{t['name']}', 'e', x'{q}', {e['k']}, ?)", [_rowid_blob(t["keep"])]]
    return f"SELECT id, distance FROM {mod}('{t['name']}{'_sub' if e['filtered'] else ''}', 'e', x'{q}', {e['k']})"


def test_sql_matches_reference_golden():
    """the reference's own top-k at k > 256 (tools/large_k_golden.py), through vector.so"""
    gold = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "sql_large_k.json")))
    setup = golden_setup(gold)
    res = run_sql(OURS, setup + [golden_query(gold, e, filtered_module=True) for e in gold["cases"]])
    assert all("error" not in r for r in res[:len(setup)]), [r for r in res if "error" in r][:2]
    for e, r in zip(gold["cases"], res[len(setup):]):
        ids = np.frombuffer(base64.b64decode(e["ids"]), "<u2").tolist()
        want = [[i, d] for i, d in zip(ids, [v for v, c in e["dist"] for _ in range(c)])]
        assert r.get("rows") == want, (e["table"], e["quantized"], e["k"], e["filtered"], r.get("error"))
    assert sum(c for e in gold["cases"] for _, c in e["dist"]) > 8_000


def test_large_k_calls_leak_no_handles():
    eng = _vs().load_engine()
    rng = np.random.Generator(np.random.PCG64(600))
    x = _column(po.I8, 70_000, 16, rng)
    q = _column(po.I8, 2, 16, rng)
    base = eng.debug_live_handles()
    for _ in range(2):
        for window in (0, 9000):
            ix = _index(po.I8, x, window=window)
            ix.scan_topk(po.L2, q[0], 1000)
            ix.scan_topk(po.L2, q, 300)
            ix.scan_topk_filtered(po.L2, q[1], 500, rng.random(70_000) < 0.5)
            assert eng.debug_live_handles() > base
            ix.close()
            assert eng.debug_live_handles() == base, window
        g = _group(po.I8, x, 3)
        g.scan_topk(po.L2, q[0], 1000)
        g.close()
        assert eng.debug_live_handles() == base, "group"
