"""The per-query sets kernels and the row filter of the batch scorers on their own, against tests/setsref.py.  -m gpu.

(a) The plan of a sets call (vsb_debug_read "sets_plan", option sets_debug): each shard's cut sets, their union, the prefix
    counts, the level ends, the levels per view, pairs0 and the budget flag equal the host restatement bit for bit: rows around
    word and tile edges, more than 1024 and 2048 tiles, 1 to several thousand sets, thousands of queries sharing sets, edge and
    random sets, garbage past the last row, several k and forced m0 / growth, streamed windows, tenant blocks at exactly 256
    and 257 levels, and groups of 2 and 3 shards whose bounds are not multiples of 32.
(b) Level 0 (vsb_debug_tc_level_filtered, level0): sets_pairs_kernel and the filtered all_pairs_kernel emit exactly the
    model's pairs, once each, and the count the plan's pairs0 predicts.
(c) The scorers' epilogues under a row filter and under sets: every tc_scan_kernel kind at every N it is built for and every
    l1_batch_kernel type log exactly the unfiltered log's admissible pairs; int8 / uint8 equal the host tc_hit on exact scores."""
import contextlib
import os

import numpy as np
import pytest

from oracle import pyoracle as po
from tests import fpfamilies as fam
from tests import setsref as sr
from tests.test_gpu_tc_kernel import _exact_distances, _int_hits

pytestmark = pytest.mark.gpu


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


def _i8(rng, n, dim):
    return rng.integers(-20, 21, (n, dim)).astype(np.int8)


def _index(vtype, x, window=0):
    ix = _vs().Index(vtype, x.shape[1], x.shape[0], window_rows=window)
    ix.append_dense(x)
    ix.finalize()
    return ix


class _Shard:
    """a group's shard (vsb_group_shard): the Index debug methods on its handle"""

    def __init__(self, g, s):
        self.eng, self.h = g.eng, g.eng.lib.vsb_group_shard(g.h, s)
        self.rows = int(self.eng.lib.vsb_index_rows(self.h))

    def debug_read(self, *a):
        return _vs().Index.debug_read(self, *a)

    def debug_sets_plan(self):
        return _vs().Index.debug_sets_plan(self)


def _words(masks, n, garbage=False, rng=None):
    """uint32 [nsets, words] bitmaps of boolean masks over n rows; garbage: random bits past row n in the last word"""
    w = np.stack([sr.to_words(m) for m in masks]) if len(masks) else np.zeros((0, sr.words_of(n)), np.uint32)
    if garbage and n % 32:
        junk = rng.integers(0, 2 ** 32, len(masks), dtype=np.uint64).astype(np.uint32)
        w[:, -1] |= junk & ~np.uint32((1 << (n % 32)) - 1)
    return np.ascontiguousarray(w)


def _sets_call(col, q, k, words, soq, fallback=False):
    ix0 = col if isinstance(col, _vs().Index) else _Shard(col, 0)
    lib = _vs().load_engine().lib
    stat = lambda name: int(lib.vsb_index_stat(ix0.h, name.encode()))
    b0, f0 = stat("sets_batches"), stat("sets_fallbacks")
    with _options(sets_debug=1):
        col.scan_topk_sets(po.L2, q, k, words, soq, as_arrays=True)
    assert (stat("sets_batches"), stat("sets_fallbacks")) == ((b0, f0 + 1) if fallback else (b0 + 1, f0))


def _check_plan(got, words, nbits, soq, k, win=0, m0=128, growth=8, ctx=""):
    """the device plan of one shard equals setsref's over the shard's sets (words: its cut of every set, uint32 [nsets, W])"""
    want = sr.shard_plan(list(words), nbits, soq, k, win, m0, growth)
    used = want["used"]
    assert np.array_equal(got["tb"], want["tb"]) and np.array_equal(got["vt"], want["vt"]), ctx
    assert (got["m0"], got["growth"], got["nsets"], got["words"]) == (want["m0"], want["growth"], len(used), sr.words_of(nbits)), ctx
    assert np.array_equal(got["sets"], words[used].reshape(len(used), -1)), (ctx, "cut sets")
    assert np.array_equal(got["union"], want["union"]), (ctx, "union")
    assert np.array_equal(got["prefix"].astype(np.int64), want["prefix"]), (ctx, "prefix", _first_diff(got["prefix"], want["prefix"]))
    assert got["over"] == want["over"], (ctx, "over")
    if want["over"]:
        return want
    assert [e.tolist() for e in got["ends"]] == want["ends"], (ctx, "ends")
    assert got["nlev"].tolist() == want["nlev"], ctx
    assert got["pairs0"] == want["pairs0"], (ctx, "pairs0", got["pairs0"], want["pairs0"])
    for v, e in enumerate(want["ends"]):                     # no level crosses a view
        assert e[-1] == want["vt"][v + 1], ctx
    return want


def _first_diff(a, b):
    bad = np.argwhere(np.asarray(a, np.int64) != np.asarray(b, np.int64))
    return bad[:3].tolist()


def _random_masks(rng, n, densities):
    return [rng.random(n) < d for d in densities]


def _edge_masks(n):
    full, zero, first, last = np.ones(n, bool), np.zeros(n, bool), np.zeros(n, bool), np.zeros(n, bool)
    first[0] = True
    last[n - 1] = True
    return [full, zero, first, last]


# ------------------------------------------------------------------------------------------------ (a) the plan
@pytest.mark.parametrize("n", [8192, 8193, 8223, 8225, 8192 + 127, 8192 + 129])
def test_plan_at_word_and_tile_edges(n):
    rng = np.random.Generator(np.random.PCG64(21000 + n))
    x = _i8(rng, n, 16)
    ix = _index(po.I8, x)
    masks = _edge_masks(n) + _random_masks(rng, n, [1e-3, 1e-2, 0.1, 0.5])
    words = _words(masks, n, garbage=True, rng=rng)
    nq = 40
    soq = rng.integers(0, len(masks), nq).astype(np.int32)
    soq[:len(masks)] = np.arange(len(masks))
    _sets_call(ix, _i8(rng, nq, 16), 10, words, soq)
    _check_plan(ix.debug_sets_plan(), words, n, soq, 10, ctx=n)
    ix.close()


@pytest.mark.parametrize("tiles", [1100, 2100])
def test_plan_past_1024_and_2048_tiles(tiles):
    """the prefix kernel's chunks of 1024 tiles carry their totals; sets with rows only after the first chunk, or only in it"""
    rng = np.random.Generator(np.random.PCG64(21100 + tiles))
    n = 128 * tiles + 77
    ix = _index(po.I8, _i8(rng, n, 16))
    late, early = np.zeros(n, bool), np.zeros(n, bool)
    late[128 * 1030:] = rng.random(n - 128 * 1030) < 0.05
    early[:128 * 1000] = rng.random(128 * 1000) < 0.01
    masks = [late, early] + _random_masks(rng, n, [1e-3, 0.02, 0.3])
    words = _words(masks, n, garbage=True, rng=rng)
    soq = np.arange(32, dtype=np.int32) % len(masks)
    _sets_call(ix, _i8(rng, 32, 16), 20, words, soq)
    _check_plan(ix.debug_sets_plan(), words, n, soq, 20, ctx=tiles)
    ix.close()


@pytest.mark.parametrize("nsets", [1, 1024, 1025, 4000])
def test_plan_with_many_sets(nsets):
    """sets past the plan block's 1024 threads (the set-stride loop) constrain the levels: the densest set comes last; thousands
    of queries, many sharing a set"""
    rng = np.random.Generator(np.random.PCG64(21200 + nsets))
    n = 20000
    ix = _index(po.I8, _i8(rng, n, 16))
    dens = 10.0 ** rng.uniform(-3, -2, nsets)                # too sparse to end a level before tile 100
    dens[-1] = 1.0
    masks = _random_masks(rng, n, dens)
    words = _words(masks, n)
    nq = max(2 * nsets, 3000) if nsets > 1 else 64
    rest = rng.integers(0, nsets, nq - nsets)
    soq = np.concatenate([np.arange(nsets), rest]).astype(np.int32)   # set s is the s-th used: the full one comes last
    _sets_call(ix, _i8(rng, nq, 16), 10, words, soq)
    want = _check_plan(ix.debug_sets_plan(), words, n, soq, 10, ctx=nsets)
    assert want["ends"] == [[1, 8, 64, len(want["tb"]) - 1]]  # the full set's levels
    ix.close()


@pytest.mark.parametrize("k,m0,growth", [(1, 128, 8), (10, 1000, 8), (100, 128, 3), (200, 2048, 8), (256, 128, 1000)])
def test_plan_for_k_and_forced_m0_growth(k, m0, growth):
    rng = np.random.Generator(np.random.PCG64(21300 + k))
    n = 60000
    ix = _index(po.I8, _i8(rng, n, 16))
    masks = _random_masks(rng, n, [0.5, 0.05, 0.003]) + _edge_masks(n)[2:]
    words = _words(masks, n, garbage=True, rng=rng)
    soq = np.arange(48, dtype=np.int32) % len(masks)
    with _options(batch_m0=m0, batch_growth=growth):
        _sets_call(ix, _i8(rng, 48, 16), k, words, soq)
    _check_plan(ix.debug_sets_plan(), words, n, soq, k, m0=m0, growth=growth, ctx=(k, m0, growth))
    ix.close()


@pytest.mark.parametrize("window", [100, 128, 129, 300])
def test_plan_of_streamed_windows(window):
    """every window is a view of its own, cut into levels that end on its last tile; a window below one 128-row tile never
    reaches the plan (the batch path needs a whole scoring tile per window) and is answered set by set, not as a fallback"""
    rng = np.random.Generator(np.random.PCG64(21400 + window))
    n = 9000 + window // 3
    ix = _index(po.I8, _i8(rng, n, 16), window=window)
    blocks = np.zeros(n, bool)
    blocks[4000:4700] = True
    masks = [blocks] + _random_masks(rng, n, [0.5, 0.02]) + _edge_masks(n)[2:]
    words = _words(masks, n, garbage=True, rng=rng)
    soq = np.arange(24, dtype=np.int32) % len(masks)
    if window < 128:
        b0, f0 = ix.stat("sets_batches"), ix.stat("sets_fallbacks")
        ix.scan_topk_sets(po.L2, _i8(rng, 24, 16), 10, words, soq)
        assert (ix.stat("sets_batches"), ix.stat("sets_fallbacks")) == (b0, f0)
        with pytest.raises(_vs().VsbError):
            ix.debug_sets_plan()
        ix.close()
        return
    _sets_call(ix, _i8(rng, 24, 16), 10, words, soq)
    want = _check_plan(ix.debug_sets_plan(), words, n, soq, 10, win=window, ctx=window)
    assert len(want["vt"]) - 1 == (n + window - 1) // window
    ix.close()


@pytest.mark.parametrize("levels", [256, 257])
def test_plan_at_the_level_budget(levels):
    """T tenants owning blocks of two tiles each need T + 1 levels (the model's count, checked): 256 levels fit the budget,
    257 make the call answer set by set once"""
    rng = np.random.Generator(np.random.PCG64(21500 + levels))
    T = levels - 1
    n = 256 * T
    masks = [np.arange(n) // 256 == t for t in range(T)]
    words = _words(masks, n)
    soq = np.arange(T, dtype=np.int32)
    tb, vt = sr.view_tiles(n)
    assert sr.plan(sr.prefixes(list(words), n, tb), vt, 128, 8, soq, budget=1 << 20)["nlev"] == [levels]
    ix = _index(po.I8, _i8(rng, n, 16))
    _sets_call(ix, _i8(rng, T, 16), 10, words, soq, fallback=levels > 256)
    got = ix.debug_sets_plan()
    _check_plan(got, words, n, soq, 10, ctx=levels)
    assert got["over"] == (levels > 256) and got["nlev"].tolist() == [0 if levels > 256 else 256]
    ix.close()


@pytest.mark.parametrize("ngpus", [2, 3])
def test_plan_of_group_shards(ngpus):
    """each shard's cut of every set equals the numpy slice (group_cut), and its plan the model over that cut"""
    rng = np.random.Generator(np.random.PCG64(21600 + ngpus))
    n = ngpus * 8300 + 37
    x = _i8(rng, n, 16)
    g = _vs().Group(po.I8, 16, n, ngpus)
    for a in range(0, n, 7919):
        g.append_dense(x[a:a + 7919])
    g.finalize()
    masks = _edge_masks(n) + _random_masks(rng, n, [0.002, 0.2])
    blocks = np.zeros(n, bool)
    blocks[8200:8400] = True                                 # across the first shard bound
    masks.append(blocks)
    words = _words(masks, n, garbage=True, rng=rng)
    soq = np.arange(20, dtype=np.int32) % len(masks)
    _sets_call(g, _i8(rng, 20, 16), 10, words, soq)
    base = 0
    bounds = []
    for s in range(ngpus):
        sh = _Shard(g, s)
        cut = np.stack([sr.group_cut(w, n, base, sh.rows) for w in words])
        for i, m in enumerate(masks):
            assert np.array_equal(sr.to_mask(cut[i], sh.rows), m[base:base + sh.rows]), (s, i)
        _check_plan(sh.debug_sets_plan(), cut, sh.rows, soq, 10, ctx=(ngpus, s))
        base += sh.rows
        bounds.append(base)
    assert base == n and any(b % 32 for b in bounds[:-1]), bounds
    g.close()


def test_plan_without_sets_debug_has_no_bitmaps():
    rng = np.random.Generator(np.random.PCG64(21700))
    n = 9000
    ix = _index(po.I8, _i8(rng, n, 16))
    words = _words(_random_masks(rng, n, [0.1, 0.5]), n)
    soq = np.arange(16, dtype=np.int32) % 2
    ix.scan_topk_sets(po.L2, _i8(rng, 16, 16), 10, words, soq)
    got = ix.debug_sets_plan()
    assert got["sets"] is None and got["union"] is None and got["prefix"] is None
    want = sr.shard_plan(list(words), n, soq, 10)
    assert [e.tolist() for e in got["ends"]] == want["ends"] and got["pairs0"] == want["pairs0"]
    ix.close()


# ------------------------------------------------------------------------------------------------ (b) level 0
def _keys(res, nq):
    log = res["log"].astype(np.int64)
    keys = log[:, 0] * nq + log[:, 1]
    assert len(np.unique(keys)) == len(keys), "duplicate pairs"
    assert np.all(log[:, 1] < nq), "a query past nq"
    return np.sort(keys)


@pytest.mark.parametrize("nq", [20, 33, 70, 300])
@pytest.mark.parametrize("allow_base", [0, 37])
def test_level0_pairs(nq, allow_base):
    rng = np.random.Generator(np.random.PCG64(22000 + nq + allow_base))
    n, dim = 9000, 16
    ix = _index(po.I8, _i8(rng, n, dim))
    q = _i8(rng, nq, dim)
    U = np.full(nq, np.inf, np.float32)
    nbits = n + allow_base
    masks = _edge_masks(nbits) + _random_masks(rng, nbits, [0.01, 0.3, 0.9])
    sets = _words(masks, nbits, garbage=True, rng=rng)
    soq = rng.integers(0, len(masks), nq).astype(np.int32)
    allow = sets[5]
    for hi in (128, 1000, 2043, 2048):
        res = ix.debug_tc_level(po.L2, q, U, 0, hi, sets=sets, set_of_query=soq, allow_base=allow_base, level0=True)
        want = sr.level0_pairs(hi, nq, allow_base=allow_base, sets=list(sets), soq=soq)
        assert res["count"] == len(want) and np.array_equal(_keys(res, nq), want), ("sets", hi)
        res = ix.debug_tc_level(po.L2, q, U, 0, hi, allow=allow, allow_base=allow_base, level0=True)
        want = sr.level0_pairs(hi, nq, allow=allow, allow_base=allow_base)
        assert res["count"] == len(want) and np.array_equal(_keys(res, nq), want), ("allow", hi)
    res = ix.debug_tc_level(po.L2, q, U, 0, 1000, level0=True)             # no filter: every pair
    assert res["count"] == 1000 * nq and np.array_equal(_keys(res, nq), sr.level0_pairs(1000, nq))
    ix.close()


def test_level0_count_equals_plan_pairs0():
    rng = np.random.Generator(np.random.PCG64(22100))
    n, dim, nq = 30000, 16, 100
    ix = _index(po.I8, _i8(rng, n, dim))
    masks = _random_masks(rng, n, [0.002, 0.05, 0.5]) + _edge_masks(n)
    words = _words(masks, n, garbage=True, rng=rng)
    soq = rng.integers(0, len(masks), nq).astype(np.int32)
    q = _i8(rng, nq, dim)
    _sets_call(ix, q, 10, words, soq)
    plan = ix.debug_sets_plan()
    used, dense = sr.used_sets(soq)
    hi = int(plan["tb"][plan["ends"][0][0]])
    res = ix.debug_tc_level(po.L2, q, np.full(nq, np.inf, np.float32), 0, hi, sets=words[used], set_of_query=dense.astype(np.int32),
                            level0=True)
    assert res["count"] == plan["pairs0"] > 0
    ix.close()


# ------------------------------------------------------------------------------------------------ (c) scorer epilogues
TC_METRICS = [po.L2, po.COS, po.DOT]
INSTANCES = ([(vt, m, N) for vt in (po.I8, po.U8) for m in TC_METRICS for N in (32, 64, 128, 256)]
             + [(vt, m, N) for vt in (po.F16, po.BF16, po.F32) for m in TC_METRICS for N in (32, 64, 128)]
             + [(vt, po.L1, N) for vt in (po.I8, po.U8, po.F16, po.BF16, po.F32) for N in (32, 64, 128)])


def _data(vtype, n, dim, rng):
    if vtype == po.I8:
        return rng.integers(-128, 128, (n, dim)).astype(np.int8)
    if vtype == po.U8:
        return rng.integers(0, 256, (n, dim)).astype(np.uint8)
    return po.convert(rng.standard_normal((n, dim)).astype(np.float32), vtype)


def _decode(vtype, a):
    if vtype in (po.I8, po.U8):
        return a.astype(np.float64)
    if vtype == po.F32:
        return a.astype(np.float64)
    return fam.decode(vtype, a)


def _distances(metric, x, q):
    if metric == po.L1:
        return np.stack([np.abs(x - q[j]).sum(1) for j in range(q.shape[0])], axis=1)
    return _exact_distances(metric, x @ q.T, (x ** 2).sum(1), (q ** 2).sum(1))


def _fixture(vtype, metric, N, rng, poison=True):
    """a column whose first rows are copies of queries (the poison: outside the sets of those queries), nq = 2N + 5 queries
    (NG = 3, the last group ragged) and bounds at a per-query quantile of the exact distances"""
    n, dim = 2048 + 77, 40
    x = _data(vtype, n, dim, rng)
    nq = 2 * N + 5
    q = _data(vtype, nq, dim, rng)
    x[300:300 + nq] = q                                      # row 300 + j: query j itself
    d = _distances(metric, _decode(vtype, x), _decode(vtype, q))
    U = np.array([np.quantile(d[:, j], 0.05 + 0.3 * (j % 3)) for j in range(nq)], np.float32)
    return x, q, U


def _admission_cases(n, nbits, nq, N, allow_base, rng):
    """(name, sets [nsets, words], set_of_query) of the epilogue tests: random sets, only column N - 1 of the first query group
    admitted, only the rows a thread holds second (tile rows 8 - 15 mod 16), nothing; and the poison rows outside their own
    query's set"""
    rows = np.arange(nbits) - allow_base
    cases = []
    masks = _random_masks(rng, nbits, [0.05, 0.3, 0.7, 1.0])
    soq = rng.integers(0, 4, nq).astype(np.int32)
    for j in range(nq):                                      # row 300 + j (query j's copy) is outside query j's set
        masks[soq[j]][allow_base + 300 + j] = False
    cases.append(("random", masks, soq))
    one = np.zeros(nq, np.int32)
    one[N - 1] = 1
    cases.append(("column N-1", [np.zeros(nbits, bool), np.ones(nbits, bool)], one))
    second = (rows >= 0) & (rows % 16 >= 8)
    cases.append(("second rows", [second, ~second & (rows >= 0)], (np.arange(nq) % 2).astype(np.int32)))
    cases.append(("nothing", [np.zeros(nbits, bool)], np.zeros(nq, np.int32)))
    return [(name, _words(m, nbits, garbage=True, rng=rng), s) for name, m, s in cases]


@pytest.mark.parametrize("vtype,metric,N", INSTANCES)
def test_epilogue_log_is_the_admissible_unfiltered_log(vtype, metric, N):
    rng = np.random.Generator(np.random.PCG64(23000 + 100 * vtype + 10 * metric + N))
    x, q, U = _fixture(vtype, metric, N, rng)
    n, nq = x.shape[0], q.shape[0]
    with _options(f32_batch=1):
        ix = _index(vtype, x)
        r0, r1 = 256, n - 37                                 # r0 > 0, r1 not a multiple of 128
        full = ix.debug_tc_level(metric, q, U, r0, r1, N=N)
        base = _keys(full, nq)
        assert full["count"] == len(base) and 0 < len(base) < (r1 - r0) * nq, (len(base), "the bounds should split the pairs")
        for allow_base in (0, 37):
            nbits = n + allow_base
            allow = _words([rng.random(nbits) < 0.6], nbits, garbage=True, rng=rng)[0]
            res = ix.debug_tc_level(metric, q, U, r0, r1, N=N, allow=allow, allow_base=allow_base)
            want = sr.admissible(base, nq, allow=allow, allow_base=allow_base)
            assert res["count"] == len(want) and np.array_equal(_keys(res, nq), want), ("allow", allow_base)
            for name, sets, soq in _admission_cases(n, nbits, nq, N, allow_base, rng):
                res = ix.debug_tc_level(metric, q, U, r0, r1, N=N, sets=sets, set_of_query=soq, allow_base=allow_base)
                got = _keys(res, nq)
                want = sr.admissible(base, nq, allow_base=allow_base, sets=list(sets), soq=soq)
                assert res["count"] == len(got) and np.array_equal(got, want), (name, allow_base, len(got), len(want))
                if name == "random":
                    poison = (300 + np.arange(nq)) * nq + np.arange(nq)
                    assert np.isin(poison, base).sum() > nq // 2, "the query copies should hit unfiltered"
                    assert not np.isin(poison, got).any(), "a query's copy outside its set was logged"
                if name == "column N-1":
                    assert np.all(got % nq == N - 1) and len(got) > 0
                if name == "second rows":
                    assert len(got) > 0 and np.all(((got // nq) % 16 >= 8) == (soq[got % nq] == 0))
                if name == "nothing":
                    assert res["count"] == 0
        # a cap below the hit count: every hit counted, the stored ones admissible
        sets, soq = _admission_cases(n, n, nq, N, 0, rng)[0][1:]
        want = sr.admissible(base, nq, sets=list(sets), soq=soq)
        cap = max(1, len(want) // 3)
        res = ix.debug_tc_level(metric, q, U, r0, r1, N=N, sets=sets, set_of_query=soq, cap=cap)
        assert res["count"] == len(want) and len(res["log"]) == cap and np.all(np.isin(_keys(res, nq), want))
        ix.close()


@pytest.mark.parametrize("epi_chunk", [1, 0])
@pytest.mark.parametrize("metric", TC_METRICS)
@pytest.mark.parametrize("vtype", [po.I8, po.U8])
def test_int_epilogue_equals_exact_hits_under_sets(vtype, metric, epi_chunk):
    """the sets log equals the host tc_hit on exact X @ Q.T restricted to the admissible pairs, with the chunk test on and off"""
    rng = np.random.Generator(np.random.PCG64(24000 + 10 * vtype + metric + 100 * epi_chunk))
    with _options(epi_chunk=epi_chunk):
        for N in (64, 256):
            x, q, U = _fixture(vtype, metric, N, rng)
            n, nq = x.shape[0], q.shape[0]
            ix = _index(vtype, x)
            r0, r1 = 128, n - 5
            x64 = x.astype(np.float64)
            for allow_base in (0, 37):
                nbits = n + allow_base
                for name, sets, soq in _admission_cases(n, nbits, nq, N, allow_base, rng):
                    res = ix.debug_tc_level(metric, q, U, r0, r1, N=N, sets=sets, set_of_query=soq, allow_base=allow_base)
                    s = (x64[r0:r1] @ q.astype(np.float64).T).astype(np.int64)
                    rr, qq = np.nonzero(_int_hits(vtype, metric, s, res["norms"], res["qc"], nq))
                    want = sr.admissible(np.sort((rr + r0) * nq + qq), nq, allow_base=allow_base, sets=list(sets), soq=soq)
                    got = _keys(res, nq)
                    assert res["count"] == len(got) and np.array_equal(got, want), (N, name, allow_base, len(got), len(want))
            ix.close()
