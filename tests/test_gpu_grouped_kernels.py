"""Grouped top-k's kernels directly (DESIGN §3.15): after each call, one shard's whole device state (vsb_debug_read "grouped":
the layout, the query's distances, pd, the pieces' k-lists, bounds, key minima, the limit's key selection and the survivor
pairs) equals the host restatement in tests/groupedref.py, and each key's answer equals eng.replay_topk over the key's rows in
global scan order.  -m gpu.

Planted distances (vsb_debug_write "grouped_dist") replace the scans, so every edge is exact and chosen:
(1) k = 1 / 2 / 31 / 32 / 33 / 63 / 64 / 200 / 255 / 256 over key lengths 0, 1, k - 1, k, k + 1, 1023 / 1024 / 1025, 2048 /
    2049 and about 5000 in ascending, descending, constant, sawtooth and small-value-set orders, keys of NaN / +INF / -INF and
    mixed +-0, absent and duplicate rowids, overlapping keys, a key count that is not a multiple of 8, and limits that select
    no subset, some keys and every key through a tie;
(2) one key of about 2M rows (about 2000 pieces); (3) 5000 keys of 1 - 3 rows (more than 1024 pieces: the offsets kernel
    carries across chunks); (4) more than 2^16 survivors on a fresh index with a limit that cuts (the pair list regrows);
(5) one index serving k = 256 with many keys, then k = 3 with few, then k = 33 (state reused across layouts);
(6) a streamed index, and groups of 2 and 3 shards (one streamed), planted per shard, with a key that is all +INF or NaN on
    one shard.
Real distances: (7) for every (type, metric) pair at k = 1 / 33 / 256 the survivors equal the restatement from the call's own
distance buffer, every distance scan_topk_filtered returns for a key equals that buffer bit for bit, int8 / uint8 buffers equal
the oracle's exact distances, and grouped_cands grows by the restated survivor count."""
import contextlib
import os

import numpy as np
import pytest

from oracle import pyoracle as po
from tests import groupedref as gr

pytestmark = pytest.mark.gpu
METRICS = [po.L2, po.L2SQ, po.COS, po.DOT, po.L1]
TYPES = [po.F32, po.F16, po.BF16, po.U8, po.I8]
NAN, INF = np.float32(np.nan), np.float32(np.inf)


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


class _Shard:
    """a group's shard (vsb_group_shard), borrowed from the group: the Index debug methods on its handle"""

    def __init__(self, g, s):
        self.eng, self.h = g.eng, g.eng.lib.vsb_group_shard(g.h, s)

    def debug_read(self, *a):
        return _vs().Index.debug_read(self, *a)

    def debug_write(self, *a):
        return _vs().Index.debug_write(self, *a)

    def debug_grouped(self):
        return _vs().Index.debug_grouped(self)


def _index(vtype, x, rowids=None, window=0):
    ix = _vs().Index(vtype, x.shape[1], x.shape[0], window_rows=window)
    ix.append_dense(x, rowids)
    ix.finalize()
    return ix


def _group(vtype, x, ngpus):
    g = _vs().Group(vtype, x.shape[1], x.shape[0], ngpus)
    g.append_dense(x)
    g.finalize()
    return g


def _shards(obj):
    """[(shard, first global scan row, end)] of an Index or a Group"""
    if isinstance(obj, _vs().Index):
        return [(obj, 0, obj.rows)]
    out, lo = [], 0
    for s in range(obj.gpus):
        sh = _Shard(obj, s)
        n = int(obj.eng.lib.vsb_index_rows(sh.h))
        out.append((sh, lo, lo + n))
        lo += n
    return out


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64)


def _expected_answers(eng, dist, keys, row_of, ids, k, limit):
    """each key's k nearest by eng.replay_topk over its rows in global scan order (NaN and +INF rows, which no scan logs, left
    out), ranked by (first distance, scan row of the first row, key) and cut to limit"""
    vs = _vs()
    ranked = []
    for g, r in enumerate(keys):
        rows = np.unique(row_of(r))
        d = dist[rows]
        rows = rows[~np.isnan(d) & (d < INF)]
        c = np.zeros(len(rows), vs.api.CAND_DTYPE)
        c["rowid"], c["seq"], c["dist"] = ids[rows], rows, dist[rows]
        wi, wd, _ = eng.replay_topk(c, k)
        if len(wi):
            ranked.append((float(wd[0]), int(row_of(wi[:1])[0]), g, wi, wd))
    ranked.sort(key=lambda t: t[:3])
    return [(t[2], t[3], t[4]) for t in (ranked[:limit] if limit else ranked)]


def _check_planted(obj, dist, keys, row_of, ids, k, limit, ctx, q=None):
    """plant dist on every shard of obj, run one grouped call and check every shard's state and every key's answer; returns
    the shards' states"""
    shards = _shards(obj)
    for sh, lo, hi in shards:
        sh.debug_write("grouped_dist", dist[lo:hi])
    q = np.zeros(obj.dim, np.int8 if obj.vtype == po.I8 else np.float32) if q is None else q
    (got,) = obj.scan_topk_grouped(po.L2, q, k, keys, limit)
    per = []
    for sh, lo, hi in shards:
        kr = gr.shard_rows(keys, row_of, lo, hi)
        lay = gr.layout(kr)
        pd, lists = gr.walk(dist[lo:hi], lay, k)
        bound, kmin = gr.bounds(lists, lay, k)
        per.append((lay, pd, lists, bound, kmin, dist[lo:hi]))
    states = []
    for i, (sh, lo, hi) in enumerate(shards):
        lay, pd, lists, bound, kmin, d = per[i]
        _, ksel = gr.limit_select([p[4] for p in per], limit)
        want = dict(lay, pd=pd, lists=lists, bound=bound, kmin=kmin, k=k, dist=d if len(lay["rows"]) else np.zeros(0, np.float32),
                    ksel=ksel if len(lay["rows"]) else None, pairs=gr.survivors(pd, bound, lay, ksel if len(lay["rows"]) else None))
        st = sh.debug_grouped()
        assert gr.diff(st, want) == [], (ctx, i)
        states.append(st)
    want = _expected_answers(obj.eng, dist, keys, row_of, ids, k, limit)
    assert [g for g, _, _ in got] == [g for g, _, _ in want], ctx
    for (g, gi, gd), (_, wi, wd) in zip(got, want):
        assert np.array_equal(gi, wi) and np.array_equal(_bits(gd), _bits(wd)), (ctx, g)
    return states


# ------------------------------------------------------------------------------------------------ planted orders
def _order(kind, n, rng):
    if kind == "ascending":                                   # only the first k log
        return np.arange(n, dtype=np.float32)
    if kind == "descending":                                  # every position logs
        return np.arange(n, 0, -1, dtype=np.float32)
    if kind == "constant":                                    # ties with the running k-th value: only the first k log
        return np.full(n, 3.5, np.float32)
    if kind == "sawtooth":
        return (np.arange(n) % 37)[::-1].astype(np.float32) + (np.arange(n) // 37).astype(np.float32) * 0.25
    return rng.choice(np.float32([0.5, 1.0, 1.5, 2.0]), n)    # a small value set: many ties


ORDERS = ("ascending", "descending", "constant", "sawtooth", "few")


def _special(n, k, rng):
    """keys of special values: NaN / +INF / -INF / +-0 draws, more than k -INF then falling values, mixed signed zeros, all +INF,
    all NaN"""
    return [rng.choice(np.float32([np.nan, np.inf, -np.inf, 0.0, -0.0, 1.0, -1.0]), n),
            np.concatenate([np.full(k + 5, -np.inf, np.float32), np.arange(n, 0, -1, dtype=np.float32)]),
            np.where(rng.random(n) < 0.5, np.float32(-0.0), np.float32(0.0)) - (rng.random(n) < 0.01).astype(np.float32),
            np.full(n // 4 + 1, np.inf, np.float32), np.full(n // 4 + 1, np.nan, np.float32)]


@pytest.fixture(scope="module")
def planted_column():
    """one int8 column of 120 000 rows with explicit rowids not in row order; the tests plant its distances"""
    rng = np.random.Generator(np.random.PCG64(72_000))
    n = 120_000
    ids = (rng.permutation(n) * 3 + 7).astype(np.int64)
    ix = _index(po.I8, np.zeros((n, 4), np.int8), ids)
    yield ix, ids, gr.RowMap(ids)
    ix.close()


def _planted_keys(k, n, ids, rng):
    """(dist [n], keys): every length of the module docstring in every order on rows of their own, the special keys, and keys of
    absent rowids, duplicates and overlaps; the key count is not a multiple of 8"""
    dist = rng.standard_normal(n).astype(np.float32) * 10
    keys, at = [], 0
    lens = sorted({0, 1, max(k - 1, 0), k, k + 1, 1023, 1024, 1025, 2048, 2049, 4999})
    for kind in ORDERS:
        for L in lens:
            dist[at:at + L] = _order(kind, L, rng)
            keys.append(ids[at:at + L][rng.permutation(L)])
            at += L
    for v in _special(1500, k, rng):
        dist[at:at + len(v)] = v
        keys.append(ids[at:at + len(v)])
        at += len(v)
    assert at <= n
    keys.append(np.array([-1, 10**12, 5], np.int64))                              # absent rowids only
    keys.append(np.concatenate([keys[len(lens) + 3], keys[len(lens) + 3][:7], [-3]]))   # duplicates and an absent rowid
    keys.append(np.concatenate([keys[5][::2], keys[len(lens) * 2 + 4]]))         # overlaps two keys
    keys += [rng.choice(ids, int(rng.integers(1, 300)), replace=False) for _ in range(7)]
    if len(keys) % 8 == 0:
        keys.append(ids[-3:])
    return dist, keys


@pytest.mark.parametrize("k", [1, 2, 31, 32, 33, 63, 64, 200, 255, 256])
def test_planted_state_every_k(planted_column, k):
    ix, ids, row_of = planted_column
    rng = np.random.Generator(np.random.PCG64(72_100 + k))
    dist, keys = _planted_keys(k, len(ids), ids, rng)
    assert len(keys) % 8 != 0
    for limit in (0, 3, 17):
        st = _check_planted(ix, dist, keys, row_of, ids, k, limit, (k, limit))[0]
        assert (st["ksel"] is None) == (limit == 0), (k, limit)
        if limit:
            assert 0 < int(st["ksel"].sum()) < len(keys), (k, limit)
    # every key with a row has the same minimum: a limit of 1 selects every one of them through the tie
    tie = np.maximum(dist, np.float32(-6.0))                                    # NaN stays NaN
    live = np.array([len(row_of(r)) > 0 for r in keys])
    tie[[int(row_of(r).min()) for r, a in zip(keys, live) if a]] = -7.0
    st = _check_planted(ix, tie, keys, row_of, ids, k, 1, (k, "tie"))[0]
    assert np.array_equal(st["ksel"].astype(bool), live), k


def test_planted_key_of_2m_rows():
    """one key of about 2M rows (about 2000 pieces: one warp merges every piece's list), falling by steps so that later pieces
    keep surviving, beside small keys"""
    rng = np.random.Generator(np.random.PCG64(72_200))
    n = 2_100_000
    ix = _index(po.I8, np.zeros((n, 4), np.int8))
    try:
        ids = np.arange(1, n + 1, dtype=np.int64)
        row_of = gr.RowMap(ids)
        big = np.arange(2_050_000)
        dist = rng.standard_normal(n).astype(np.float32)
        dist[big] = (np.float32(3000.0) - (big // 1024).astype(np.float32) * np.float32(1.5)
                     + rng.random(len(big)).astype(np.float32))
        keys = [ids[big], ids[2_050_000:2_050_100], ids[2_060_000:2_063_000], ids[::1000]]
        for k in (2, 33, 256):
            st = _check_planted(ix, dist, keys, row_of, ids, k, 0, ("2M", k))[0]
            assert len(st["pkey"]) > 2000 and np.count_nonzero(st["pkey"] == 0) > 2000
            assert np.count_nonzero(st["pairs"][:, 1] >= 1024 * 1500) > 0, k    # late pieces still have survivors
    finally:
        ix.close()


def test_planted_more_than_1024_pieces(planted_column):
    """5000 keys of 1 - 3 rows: 5000 pieces, so the offsets kernel carries its sums from one 1024-piece chunk to the next"""
    ix, ids, row_of = planted_column
    rng = np.random.Generator(np.random.PCG64(72_300))
    dist = rng.standard_normal(len(ids)).astype(np.float32)
    keys = [rng.choice(ids[:40_000], int(rng.integers(1, 4)), replace=False) for _ in range(5000)]
    for k, limit in ((1, 0), (3, 0), (33, 0), (3, 2500)):
        st = _check_planted(ix, dist, keys, row_of, ids, k, limit, ("pieces", k, limit))[0]
        assert len(st["pkey"]) == 5000 and int(st["pairs"][:, 1].max()) >= int(st["pstart"][4096]), (k, limit)


def test_planted_regrow_with_a_limit():
    """more than 2^16 survivors on a fresh index while the limit selects keys: the pair list grows and is written again"""
    n = 100_000
    ix = _index(po.I8, np.zeros((n, 4), np.int8))
    try:
        ids = np.arange(1, n + 1, dtype=np.int64)
        row_of = gr.RowMap(ids)
        dist = np.arange(n, 0, -1, dtype=np.float32)                            # falling: every row of key 0 survives
        dist[90_000:] = np.arange(10_000, dtype=np.float32) + 200_000.0
        keys = [ids[:90_000]] + [ids[90_000 + 100 * i:90_100 + 100 * i] for i in range(20)]
        r0 = ix.stat("grouped_regrows")
        st = _check_planted(ix, dist, keys, row_of, ids, 5, 1, "regrow")[0]
        assert ix.stat("grouped_regrows") - r0 >= 1 and len(st["pairs"]) > 1 << 16
        assert st["ksel"] is not None and st["ksel"].tolist() == [1] + [0] * 20
    finally:
        ix.close()


def test_planted_state_reused_across_calls(planted_column):
    """k = 256 with many keys, then k = 3 with few, then k = 33: every call's state is its own"""
    ix, ids, row_of = planted_column
    rng = np.random.Generator(np.random.PCG64(72_400))
    dist, many = _planted_keys(256, len(ids), ids, rng)
    _check_planted(ix, dist, many, row_of, ids, 256, 0, "many")
    few = [ids[:5], ids[100:2100], ids[50_000:50_003]]
    st = _check_planted(ix, dist[::-1].copy(), few, row_of, ids, 3, 2, "few")[0]
    assert len(st["rows"]) == 2008 and st["lists"].shape == (4, 3)
    _check_planted(ix, dist, many[::3], row_of, ids, 33, 4, "again")


@pytest.mark.parametrize("window", [128, 1000])
def test_planted_streamed(window):
    rng = np.random.Generator(np.random.PCG64(72_500 + window))
    n = 9000
    ids = (rng.permutation(n) + 1).astype(np.int64)
    row_of = gr.RowMap(ids)
    st_ix = _index(po.I8, np.zeros((n, 4), np.int8), ids, window=window)
    try:
        assert st_ix.eng.lib.vsb_index_is_streamed(st_ix.h) == 1
        dist = rng.standard_normal(n).astype(np.float32)
        dist[:3000] = _order("descending", 3000, rng)
        keys = [ids[:3000], ids[3000:3100]] + [rng.choice(ids, int(rng.integers(1, 400)), replace=False) for _ in range(11)]
        for k, limit in ((1, 0), (33, 3), (256, 0)):
            _check_planted(st_ix, dist, keys, row_of, ids, k, limit, (window, k, limit))
    finally:
        st_ix.close()


@pytest.mark.parametrize("ngpus", [2, 3])
def test_planted_groups(ngpus):
    """per-shard plants on groups of 2 and 3 shards (the last of 3 streamed); key 0 is all +INF or NaN on shard 0 (and NaN on
    shard 1 of 3) with its only finite row on the last shard, so it makes a limit of 1 through that shard alone"""
    rng = np.random.Generator(np.random.PCG64(72_600 + ngpus))
    n = 6001
    x = np.zeros((n, 4), np.int8)
    ids = np.arange(1, n + 1, dtype=np.int64)
    row_of = gr.RowMap(ids)
    ix = _index(po.I8, x)
    pitch = ix.query_pitch
    ix.close()
    with _env(**({"VSB_DEVICE_BUDGET_MB": repr(2000.5 * pitch / 1048576.0)} if ngpus == 3 else {})):
        g = _group(po.I8, x, ngpus)
    try:
        shards = _shards(g)
        lib = g.eng.lib
        assert [lib.vsb_index_is_streamed(s.h) for s, _, _ in shards] == ([0, 0, 1] if ngpus == 3 else [0, 0])
        dist = rng.standard_normal(n).astype(np.float32)
        lo0, lo1, last = shards[0][1], shards[1][1], shards[-1][1]
        dist[lo0:lo0 + 50] = np.where(np.arange(50) % 2, NAN, INF)
        dist[lo1:lo1 + 50] = NAN
        dist[last + 60] = -5.0
        k0 = np.concatenate([ids[lo0:lo0 + 50], ids[lo1:lo1 + 50], ids[last + 60:last + 61]])
        keys = [k0, ids[::7], ids[lo1 - 30:lo1 + 30]] + [rng.choice(ids, int(rng.integers(1, 200)), replace=False) for _ in range(20)]
        for k, limit in ((3, 0), (3, 1), (33, 5), (256, 0)):
            sts = _check_planted(g, dist, keys, row_of, ids, k, limit, (ngpus, k, limit))
            assert [float(s["kmin"][0]) for s in sts] == [np.inf] * (ngpus - 1) + [-5.0], (ngpus, k, limit)
    finally:
        g.close()


def test_plant_is_checked_and_dropped(planted_column):
    vs = _vs()
    ix, ids, row_of = planted_column
    with pytest.raises(vs.VsbError) as e:
        ix.debug_write("grouped_dist", np.zeros(len(ids) - 1, np.float32))
    assert e.value.rc == vs.api.EINVAL
    q = np.zeros(4, np.int8)
    keys = [ids[:10]]
    ix.debug_write("grouped_dist", np.full(len(ids), -1.0, np.float32))
    with pytest.raises(vs.VsbError):
        ix.scan_topk_grouped(po.L2, q, 300, keys)                               # a failing call drops the plant too
    (got,) = ix.scan_topk_grouped(po.L2, q, 3, keys)                            # scanned: the all-zero rows are at distance 0
    assert [float(d) for d in got[0][2]] == [0.0, 0.0, 0.0]
    assert float(ix.debug_grouped()["dist"][0]) == 0.0


# ------------------------------------------------------------------------------------------------ real distances
def _column(vtype, n, dim, rng):
    if vtype == po.I8:
        return rng.integers(-20, 21, (n, dim)).astype(np.int8)
    if vtype == po.U8:
        return rng.integers(0, 40, (n, dim)).astype(np.uint8)
    return po.convert(rng.standard_normal((n, dim), dtype=np.float32), vtype)


@pytest.mark.parametrize("vtype", TYPES)
def test_real_distances_state(oracle, vtype):
    rng = np.random.Generator(np.random.PCG64(72_700 + vtype))
    n, dim = 4000, 40
    x = _column(vtype, n, dim, rng)
    ids = (rng.permutation(n) * 2 + 3).astype(np.int64)
    row_of = gr.RowMap(ids)
    ix = _index(vtype, x, ids)
    try:
        keys = [ids[:1500], rng.choice(ids, 2500, replace=False)] + [rng.choice(ids, int(rng.integers(1, 120)), replace=False)
                                                                    for _ in range(13)]
        kr = gr.shard_rows(keys, row_of, 0, n)
        for metric in METRICS:
            q = _column(vtype, 1, dim, rng)[0]
            for k in (1, 33, 256):
                limit = 4 if k == 33 else 0
                c0 = ix.stat("grouped_cands")
                (got,) = ix.scan_topk_grouped(metric, q, k, keys, limit)
                st = ix.debug_grouped()
                want = gr.state(st["dist"], kr, k, limit=limit)
                assert gr.diff(st, want) == [], (metric, k)
                assert ix.stat("grouped_cands") - c0 == len(want["pairs"]), (metric, k)
                for g in range(len(keys)):
                    bits, _ = ix.rowid_bitmap(keys[g])
                    (fi, fd), = ix.scan_topk_filtered(metric, q, k, bits)
                    rows = row_of(fi)
                    assert np.array_equal(_bits(fd), _bits(st["dist"][rows].astype(np.float64))), (metric, k, g)
                if vtype in (po.I8, po.U8):
                    assert gr.same(st["dist"], oracle.distances_all(metric, vtype, q, x, int_exact=True)), metric
    finally:
        ix.close()
