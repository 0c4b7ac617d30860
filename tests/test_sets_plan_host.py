"""The host restatement of the per-query sets plan (tests/setsref.py) without a GPU: hand-worked tiles, prefixes, level ends,
pairs of level 0, the level budget, a group shard's cut and the admissible part of a log, and the plan against a row-by-row
walk of DESIGN §3.14's level rule."""
import numpy as np
import pytest

from tests import setsref as sr


def test_view_tiles_resident_and_streamed():
    tb, vt = sr.view_tiles(300)
    assert tb.tolist() == [0, 128, 256, 300] and vt.tolist() == [0, 3]
    tb, vt = sr.view_tiles(256)
    assert tb.tolist() == [0, 128, 256] and vt.tolist() == [0, 2]
    tb, vt = sr.view_tiles(300, win_rows=129)                # a window one row past a tile: a one-row tile per window
    assert tb.tolist() == [0, 128, 129, 257, 258, 300] and vt.tolist() == [0, 2, 4, 5]
    tb, vt = sr.view_tiles(300, win_rows=100)
    assert tb.tolist() == [0, 100, 200, 300] and vt.tolist() == [0, 1, 2, 3]


def test_bitmaps_and_prefix_ignore_bits_past_nbits():
    m = np.zeros(70, bool)
    m[[0, 31, 32, 69]] = True
    w = sr.to_words(m)
    assert w.tolist() == [0x80000001, 1, 0x20]
    assert np.array_equal(sr.to_mask(w, 70), m)
    w[2] |= np.uint32(0xFFFFFFC0)                            # garbage past row 69
    tb, _ = sr.view_tiles(70)
    assert sr.prefix(w, 70, tb).tolist() == [0, 4]
    assert sr.prefix(np.full(2, 0xFFFFFFFF, np.uint32), 40, np.array([0, 31, 32, 40])).tolist() == [0, 31, 32, 40]


def test_m0_and_growth():
    assert [sr.m0_of(v) for v in (0, 128, 200, 1000, 5000)] == [128, 128, 128, 896, 2048]
    assert sr.growth_of(10) == 8 and sr.growth_of(256) == 4 and sr.growth_of(200) == 5 and sr.growth_of(1) == 8
    assert sr.growth_of(10, batch_growth=3) == 3 and sr.growth_of(10, batch_growth=1) == 2 and sr.growth_of(10, 5000) == 82


def test_plan_of_one_full_set():
    """prefix(j) = 128 j: level 0 takes m0 = 128 rows, then each level ends where the rows reach 8x those before it"""
    n = 128 * 100
    tb, vt = sr.view_tiles(n)
    P = sr.prefixes([sr.to_words(np.ones(n, bool))], n, tb)
    p = sr.plan(P, vt, 128, 8, np.zeros(5, np.int64))
    assert p["ends"] == [[1, 8, 64, 100]] and p["pairs0"] == 5 * 128 and not p["over"]
    p = sr.plan(P, vt, 512, 8, np.zeros(3, np.int64))       # m0 = 512: four tiles exhaustively, then 8x
    assert p["ends"] == [[4, 32, 100]] and p["pairs0"] == 3 * 512


def test_plan_minimum_over_sets_and_empty_sets():
    n = 128 * 40
    tb, vt = sr.view_tiles(n)
    sparse = np.zeros(n, bool)
    sparse[::128] = True                                     # one row per tile
    dense = np.zeros(n, bool)
    dense[128 * 20:] = True                                  # nothing before tile 20
    empty = np.zeros(n, bool)
    sets = [sr.to_words(s) for s in (sparse, dense, empty)]
    P = sr.prefixes(sets, n, tb)
    # sparse alone: 128 rows fit in one level of 40 tiles
    assert sr.plan(P[:1], vt, 128, 8, [0])["ends"] == [[40]]
    # dense: level 0 to tile 21 (128 rows), then 8 x 128 = 1024 rows: tiles 21 .. 28
    assert sr.plan(P[1:2], vt, 128, 8, [0])["ends"] == [[21, 28, 40]]
    p = sr.plan(P, vt, 128, 8, [0, 1, 1, 2])
    assert p["ends"] == [[21, 28, 40]]
    assert p["pairs0"] == 21 + 2 * 128 + 0                   # the queries' sets' rows in tiles [0, 21)
    assert sr.plan(P[2:], vt, 128, 8, [0])["ends"] == [[40]]
    assert sr.plan(P[:0], vt, 128, 8, [])["ends"] == [[40]]


def test_plan_level_holds_at_least_one_tile():
    """a tile of 128 rows of a set that has already passed m0 with growth x before: the level still takes the tile"""
    n = 128 * 3
    tb, vt = sr.view_tiles(n)
    P = sr.prefixes([sr.to_words(np.ones(n, bool))], n, tb)
    assert sr.plan(P, vt, 128, 2, [0])["ends"] == [[1, 2, 3]]


def test_plan_views_and_budget():
    n = 1000
    tb, vt = sr.view_tiles(n, win_rows=300)                  # views of 300, 300, 300, 100 rows: 3 + 3 + 3 + 1 tiles
    P = sr.prefixes([sr.to_words(np.ones(n, bool))], n, tb)
    p = sr.plan(P, vt, 128, 8, [0, 0])
    assert p["ends"] == [[1, 3], [6], [9], [10]] and p["pairs0"] == 256
    assert all(e[-1] == vt[v + 1] for v, e in enumerate(p["ends"]))
    assert sr.plan(P, vt, 128, 8, [0], budget=1)["over"]
    assert not sr.plan(P, vt, 128, 8, [0], budget=2)["over"]


def _tenants(T, rows_each):
    n = T * rows_each
    return n, [sr.to_words(np.arange(n) // rows_each == t) for t in range(T)]


def test_contiguous_tenants_cut_a_level_inside_each_block():
    """blocks of 256 rows on tile bounds: a set reaches m0 = 128 rows after its block's first tile, so a level ends there; the
    earlier sets then allow 8x their rows, and the next block's first tile joins the level"""
    n, sets = _tenants(4, 256)
    tb, vt = sr.view_tiles(n)
    p = sr.plan(sr.prefixes(sets, n, tb), vt, 128, 8, [0, 1, 2, 3])
    assert p["ends"] == [[1, 3, 5, 7, 8]] and p["pairs0"] == 128
    n, sets = _tenants(300, 256)                             # one level per tenant, and the last tile's: over 256 levels
    tb, vt = sr.view_tiles(n)
    P = sr.prefixes(sets, n, tb)
    assert sr.plan(P, vt, 128, 8, np.arange(300))["over"]
    assert sr.plan(P[:255], vt[:1].tolist() + [510], 128, 8, np.arange(255))["nlev"] == [256]


def _walk(masks, n, win, m0, g):
    """the level rule row by row: per view, a level from tile t ends at the largest tile end u where no set has more than
    max(m0, g * rows before t) rows before u, and at least one tile later"""
    tb, vt = sr.view_tiles(n, win)
    ends = []
    for v in range(len(vt) - 1):
        t, ve = int(vt[v]), []
        while t < vt[v + 1]:
            best = int(vt[v + 1])
            for m in masks:
                cap = max(m0, g * int(m[:tb[t]].sum()))
                u = t
                while u < vt[v + 1] and int(m[:tb[u + 1]].sum()) <= cap:
                    u += 1
                best = min(best, u)
            t = max(t + 1, best)
            ve.append(t)
        ends.append(ve)
    return ends


@pytest.mark.parametrize("seed", range(6))
def test_plan_equals_row_walk(seed):
    rng = np.random.Generator(np.random.PCG64(seed))
    n = int(rng.integers(200, 4000))
    win = int(rng.choice([0, 100, 128, 129, 300, 1000]))
    masks = [rng.random(n) < d for d in rng.choice([0.0, 0.001, 0.05, 0.3, 1.0], size=int(rng.integers(1, 5)))]
    tb, vt = sr.view_tiles(n, win)
    m0, g = sr.m0_of(int(rng.choice([128, 256, 700]))), int(rng.integers(2, 9))
    p = sr.plan(sr.prefixes([sr.to_words(m) for m in masks], n, tb), vt, m0, g, np.arange(len(masks)))
    assert p["ends"] == _walk(masks, n, win, m0, g)
    assert p["pairs0"] == sum(int(m[:tb[p["ends"][0][0]]].sum()) for m in masks)


def test_used_sets_and_shard_plan():
    used, dense = sr.used_sets([4, 2, 4, 0, 2])
    assert used == [4, 2, 0] and dense.tolist() == [0, 1, 0, 2, 1]
    n = 128 * 10
    sets = [sr.to_words(np.ones(n, bool)), sr.to_words(np.zeros(n, bool)), sr.to_words(np.arange(n) < 5)]
    p = sr.shard_plan(sets, n, [2, 2, 0], k=10)
    assert p["used"] == [2, 0] and p["ends"] == [[1, 8, 10]] and p["pairs0"] == 5 + 5 + 128
    assert p["union"].tolist() == sets[0].tolist() and p["prefix"].shape == (2, 11)


def test_group_cut_takes_the_shard_bits_and_carries_the_next():
    rng = np.random.Generator(np.random.PCG64(9))
    total = 200
    m = rng.random(total) < 0.5
    w = sr.to_words(m)
    for base, rows in ((0, 37), (37, 100), (137, 63), (64, 64), (1, 199)):
        cut = sr.group_cut(w, total, base, rows)
        assert len(cut) == sr.words_of(rows)
        assert np.array_equal(sr.to_mask(cut, rows), m[base:base + rows]), (base, rows)
        tail = 32 * len(cut) - rows                          # the last word's extra bits: the next rows of the column, or 0 past it
        more = m[base + rows:base + rows + tail]
        want = np.concatenate([more, np.zeros(tail - len(more), bool)])
        assert np.array_equal(sr.to_mask(cut, 32 * len(cut))[rows:], want), (base, rows)


def test_level0_pairs_and_admissible_logs():
    nq = 3
    allow = sr.to_words(np.array([1, 0, 1, 1, 0, 0, 0, 1], bool))
    assert sr.level0_pairs(2, nq).tolist() == [0, 1, 2, 3, 4, 5]
    assert sr.level0_pairs(4, nq, allow=allow).tolist() == [0, 1, 2, 6, 7, 8, 9, 10, 11]
    assert sr.level0_pairs(3, nq, allow=allow, allow_base=2).tolist() == [0, 1, 2, 3, 4, 5]      # bits 2, 3 of rows 0, 1
    sets = [sr.to_words(np.array([1, 1, 0, 0, 0, 0, 0, 0], bool)), sr.to_words(np.array([0, 0, 0, 1, 0, 0, 0, 1], bool))]
    soq = [1, 0, 1]
    assert sr.level0_pairs(8, nq, sets=sets, soq=soq).tolist() == [1, 4, 9, 11, 21, 23]
    assert sr.level0_pairs(4, nq, allow_base=4, sets=sets, soq=soq).tolist() == [9, 11]
    keys = np.array([1, 4, 9, 10, 11, 21, 22, 23])
    assert sr.admissible(keys, nq, sets=sets, soq=soq).tolist() == [1, 4, 9, 11, 21, 23]
    assert sr.admissible(keys, nq, allow=allow).tolist() == [1, 9, 10, 11, 21, 22, 23]
    assert sr.admissible(keys, nq, allow=allow, sets=sets, soq=soq).tolist() == [1, 9, 11, 21, 23]
