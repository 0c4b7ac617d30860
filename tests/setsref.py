"""Host restatement of the per-query sets plan (DESIGN §3.14) and of what its kernels emit: the tiles of every view, each set's
prefix counts, the level ends, the pairs of level 0, the level-budget overflow, a group shard's cut of a set, the pairs of the
level-0 kernels and the admissible part of a scorer's candidate log.  vsb_debug_read "sets_plan" (Index.debug_sets_plan) and
vsb_debug_tc_level_filtered (Index.debug_tc_level with a filter) return the same things from the device.

Bitmaps are uint32 words, bit r & 31 of word r >> 5 for row r.  Bits at or past a bitmap's nbits are never counted."""
import numpy as np

TILE = 128                                        # rows of a scorer tile (kTcM)
BUDGET = 256                                      # levels per view (kSetsLevelBudget)
BUCKET_CAP = 2048                                 # kBucketCap


def words_of(nbits):
    return (int(nbits) + 31) // 32


def to_words(mask):
    """uint32 bitmap of a boolean mask"""
    m = np.asarray(mask, bool)
    out = np.zeros(max(words_of(len(m)), 1), np.uint32)
    if len(m):
        packed = np.packbits(m, bitorder="little")
        packed = np.concatenate([packed, np.zeros(4 * len(out) - len(packed), np.uint8)])
        out[:] = packed.view("<u4")
    return out[: words_of(len(m))] if len(m) else out[:0]


def to_mask(words, nbits):
    """the first nbits bits of a bitmap as booleans"""
    w = np.ascontiguousarray(words, dtype="<u4")
    return np.unpackbits(w.view(np.uint8), bitorder="little")[:nbits].astype(bool)


def m0_of(batch_m0=128):
    """batch_m0(): the option rounded down to whole tiles, in [128, BUCKET_CAP]"""
    return min(max(128, (batch_m0 // 128) * 128), BUCKET_CAP)


def growth_of(k, batch_growth=8):
    """batch_growth(k): the option, capped so that 2.5 k (g - 1) candidates fit a query's bucket, at least 2"""
    cap = int(BUCKET_CAP / (2.5 * max(k, 1))) + 1
    return max(2, min(min(batch_growth, 1024), cap))


def view_tiles(n, win_rows=0):
    """tile bounds tb (shard rows) and view tiles vt: view v holds tiles [vt[v], vt[v + 1]); a resident shard is one view, a
    streamed one a view per window of win_rows rows; every view's last tile may be partial"""
    vrows = win_rows if win_rows > 0 else max(n, 1)
    tb, vt = [0], [0]
    for r0 in range(0, n, vrows):
        rows = min(vrows, n - r0)
        tb.extend(range(r0 + TILE, r0 + rows, TILE))
        tb.append(r0 + rows)
        vt.append(len(tb) - 1)
    return np.array(tb, np.int64), np.array(vt, np.int64)


def prefix(words, nbits, tb):
    """prefix[j]: the set's rows in tile rows [tb[0], tb[j]), j = 0 .. T"""
    cs = np.concatenate([[0], np.cumsum(to_mask(words, nbits), dtype=np.int64)])
    return cs[tb] - cs[tb[0]]


def prefixes(sets, nbits, tb):
    """prefix of every set, [nsets, T + 1]"""
    return np.array([prefix(s, nbits, tb) for s in sets], np.int64).reshape(len(sets), len(tb))


def union(sets, nwords):
    """the sets OR-ed word by word (every word, bits past nbits included)"""
    out = np.zeros(nwords, np.uint32)
    for s in sets:
        out |= np.asarray(s, np.uint32)[:nwords]
    return out


def used_sets(soq):
    """sets_used: the sets the queries name in order of first use, and each query's position among them"""
    pos, used, dense = {}, [], []
    for s in (int(v) for v in soq):
        if s not in pos:
            pos[s] = len(used)
            used.append(s)
        dense.append(pos[s])
    return used, np.array(dense, np.int64)


def plan(P, vt, m0, growth, soq, budget=BUDGET):
    """the levels of every view.  A level from tile t ends at the minimum over the sets of the last u <= the view's end with
    P[s][u] <= max(m0, growth P[s][t]), and holds at least one tile.  Returns {"ends": [per view, tile indices], "nlev",
    "pairs0": sum over queries of P[soq[q]][first end of view 0], "over": a view needs more than `budget` levels}; with over,
    "ends", "nlev" and "pairs0" are None (the device stops there)."""
    P = np.asarray(P, np.int64)
    nsets = P.shape[0]
    soq = np.asarray(soq, np.int64)
    if nsets == 0:                                # no set: one level per view, no row eligible
        ends = [[int(vt[v + 1])] for v in range(len(vt) - 1)]
        return {"ends": ends, "nlev": [1] * len(ends), "pairs0": 0, "over": False}
    ends, pairs0 = [], None
    for v in range(len(vt) - 1):
        t, te = int(vt[v]), int(vt[v + 1])
        ve = []
        while t < te:
            if len(ve) == budget:
                return {"ends": None, "nlev": None, "pairs0": None, "over": True}
            cap = np.maximum(m0, growth * P[:, t])
            last = t + (P[:, t:te + 1] <= cap[:, None]).sum(axis=1) - 1      # prefixes never decrease
            u = max(t + 1, int(last.min()))
            if pairs0 is None:
                pairs0 = int(P[soq, u].sum())
            ve.append(u)
            t = u
        ends.append(ve)
    return {"ends": ends, "nlev": [len(e) for e in ends], "pairs0": int(pairs0 or 0), "over": False}


def shard_plan(sets, nbits, soq, k, win_rows=0, batch_m0=128, batch_growth=8):
    """the whole plan of one shard of nbits rows for the sets the queries name (set_of_query soq), as sets_begin makes it:
    {"tb", "vt", "m0", "growth", "used", "prefix", "union", and plan()'s keys}"""
    used, dense = used_sets(soq)
    cut = [np.asarray(sets[s], np.uint32) for s in used]
    tb, vt = view_tiles(nbits, win_rows)
    m0, g = m0_of(batch_m0), growth_of(k, batch_growth)
    P = prefixes(cut, nbits, tb)
    out = plan(P, vt, m0, g, dense)
    out.update(tb=tb, vt=vt, m0=m0, growth=g, used=used, prefix=P, union=union(cut, words_of(nbits)))
    return out


def group_cut(words, total_rows, base, rows):
    """shard rows [base, base + rows) of a bitmap over a column of total_rows rows (group_cut): words_of(rows) words; the last
    may carry the next shard's bits (never counted)"""
    src = np.asarray(words, np.uint64)
    gw = words_of(total_rows)
    w = np.arange(words_of(rows), dtype=np.int64)
    i = (base + 32 * w) >> 5
    sh = ((base + 32 * w) & 31).astype(np.uint64)
    v = src[i] >> sh
    nxt = (sh != 0) & (i + 1 < gw)
    hi = np.where(nxt, src[np.minimum(i + 1, gw - 1)] << ((np.uint64(32) - sh) & np.uint64(63)), 0)
    return ((v | hi) & np.uint64(0xFFFFFFFF)).astype(np.uint32)


def bit(words, r):
    """bit r of a bitmap, for an array of rows r"""
    w = np.asarray(words, np.uint32)
    r = np.asarray(r, np.int64)
    return ((w[r >> 5] >> (r & 31).astype(np.uint32)) & 1).astype(bool)


def level0_pairs(hi, nq, allow=None, allow_base=0, sets=None, soq=None):
    """keys row * nq + q of level 0 over rows [0, hi), sorted: every pair (all_pairs_kernel without a filter), the allowed rows'
    pairs (with `allow`), or the pairs with row in query q's set (sets_pairs_kernel: sets[soq[q]]); row r is bit allow_base + r"""
    rows = np.arange(hi, dtype=np.int64)
    if sets is not None:
        inset = np.stack([bit(sets[int(s)], allow_base + rows) for s in soq], axis=1) if nq else np.zeros((hi, 0), bool)
    else:
        ok = np.ones(hi, bool) if allow is None else bit(allow, allow_base + rows)
        inset = np.repeat(ok[:, None], nq, axis=1)
    r, q = np.nonzero(inset)
    return np.sort(r * nq + q)


def admissible(keys, nq, allow=None, allow_base=0, sets=None, soq=None):
    """the keys row * nq + q of a scorer log whose row a filtered level may report for q: row allowed, and in q's set"""
    keys = np.asarray(keys, np.int64)
    r, q = keys // nq, keys % nq
    ok = np.ones(len(keys), bool)
    if allow is not None:
        ok &= bit(allow, allow_base + r)
    if sets is not None:
        soq = np.asarray(soq, np.int64)
        for s in np.unique(soq[q]) if len(keys) else []:
            sel = soq[q] == s
            ok[sel] &= bit(sets[int(s)], allow_base + r[sel])
    return keys[ok]
