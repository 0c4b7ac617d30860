"""Host restatement of grouped top-k's device state (DESIGN §3.15) from one shard's distances and the keys' shard rows: the
layout, the walk (pd and each piece's k-list), the key bounds and minima, the survivors of the selected keys, and the host's
limit selection over shards.  vsb_debug_read "grouped" (Index.debug_grouped) returns the same arrays from the device.

Comparison rule: every array compares bit for bit, except that a zero may compare by value (-0 == +0) in lists, bound and kmin.
Those are merged with fminf and value comparisons on the device, so which signed zero a tie keeps is left open; pd, the
distances and the survivor pairs copy the distance itself, so their bits are fixed."""
import numpy as np

PIECE = 1024                                      # positions of a piece (kGroupedPiece)
INF = np.float32(np.inf)
NAN = np.float32(np.nan)                          # bits 0x7FC00000, as the walk writes for a position it did not log


class RowMap:
    """rowid -> global scan row of a column whose row i has rowid ids[i]"""

    def __init__(self, ids):
        self.ids = np.asarray(ids, np.int64)
        self.order = np.argsort(self.ids, kind="stable")
        self.sorted = self.ids[self.order]

    def __call__(self, rowids):
        """the scan rows of the rowids present in the column, in the order given (absent rowids dropped)"""
        r = np.asarray(rowids, np.int64).reshape(-1)
        at = np.minimum(np.searchsorted(self.sorted, r), max(len(self.sorted) - 1, 0))
        hit = self.sorted[at] == r if len(self.sorted) else np.zeros(len(r), bool)
        return self.order[at[hit]]


def shard_rows(keys, row_map, lo, hi):
    """each key's rowids mapped to shard rows of the shard holding global scan rows [lo, hi): rowids absent from the column or
    on other shards are dropped"""
    out = []
    for r in keys:
        g = row_map(r)
        out.append(g[(g >= lo) & (g < hi)] - lo)
    return out


def layout(key_rows):
    """rows (each key's shard rows sorted and unique, key after key), koff [G + 1], and the pieces: pstart [N + 1], pkey [N],
    kpiece [G + 1]; a key's run is cut every PIECE positions"""
    runs = [np.unique(np.asarray(r, np.int64)) for r in key_rows]
    lens = np.array([len(u) for u in runs], np.int64)
    koff = np.zeros(len(runs) + 1, np.int64)
    koff[1:] = np.cumsum(lens)
    npk = (lens + PIECE - 1) // PIECE
    kpiece = np.zeros(len(runs) + 1, np.int64)
    kpiece[1:] = np.cumsum(npk)
    pkey = np.repeat(np.arange(len(runs)), npk)
    pstart = np.append(koff[pkey] + PIECE * (np.arange(len(pkey)) - kpiece[pkey]), koff[-1])
    rows = np.concatenate(runs) if runs else np.zeros(0, np.int64)
    u4 = lambda a: np.asarray(a, np.int64).astype(np.uint32)
    return {"rows": u4(rows), "koff": u4(koff), "pstart": u4(pstart), "pkey": u4(pkey), "kpiece": u4(kpiece)}


def _pieces(d, pstart, width):
    """the positions' values as [N, width] (NaN past a piece's end)"""
    N = len(pstart) - 1
    m = np.full((N, width), NAN, np.float32)
    if N:
        lens = np.diff(pstart.astype(np.int64))
        col = np.arange(width)
        ok = col[None, :] < lens[:, None]
        m[ok] = d[(pstart[:-1].astype(np.int64)[:, None] + col[None, :])[ok]]
    return m


def earlier_le(m):
    """[N, W] (W a power of two): for each entry, how many earlier non-NaN entries of its row are <= it, by a bottom-up merge
    count over every row at once (at each level, a right run's entries count the left run's entries at or below them)"""
    N, W = m.shape
    nan = np.isnan(m)
    u = np.unique(m[~nan])                              # -0 and +0 are one value here
    R = len(u) + 2
    r = np.where(nan, len(u) + 1, np.searchsorted(u, np.where(nan, 0, m))).astype(np.int64).reshape(-1)
    cnt = np.zeros(N * W, np.int64)
    srt, s = r.copy(), 1                                # srt: sorted runs of s entries
    while s < W:
        runs = srt.reshape(-1, 2 * s)
        nb = runs.shape[0]
        base = np.arange(nb, dtype=np.int64)[:, None]
        keys = (base * R + runs[:, :s]).reshape(-1)     # increasing: run after run, each sorted
        q = (base * R + r.reshape(-1, 2 * s)[:, s:]).reshape(-1)
        c = np.searchsorted(keys, q, side="right").reshape(nb, s) - base * s
        cnt.reshape(-1, 2 * s)[:, s:] += c
        srt = np.sort(runs, axis=1).reshape(-1)
        s *= 2
    return cnt.reshape(N, W)


def walk(dist, lay, k):
    """(pd [P], lists [N, k]): position j of a piece logs when d_j < the k-th smallest of the piece's earlier non-NaN values
    (+INF while there are fewer than k), strict, so NaN and +INF never log; equivalently d_j < +INF and fewer than k earlier
    values are <= d_j.  pd is d where logged, NaN elsewhere; a list is the piece's k smallest values, ascending, +INF padded."""
    d = np.asarray(dist, np.float32)[lay["rows"].astype(np.int64)]
    lens = np.diff(lay["pstart"].astype(np.int64))
    width = 1 << int(max(int(lens.max()) if len(lens) else 1, 1) - 1).bit_length()
    m = _pieces(d, lay["pstart"], width)
    log = (m < INF) & (earlier_le(m) < k)
    ok = np.arange(width)[None, :] < lens[:, None]
    pd = np.full(len(d), NAN, np.float32)
    sel = log[ok]                                        # position order: pieces are consecutive runs of positions
    pd[sel] = d[sel]
    lists = np.sort(np.where(np.isnan(m), INF, m), axis=1)[:, :k]
    if lists.shape[1] < k:
        lists = np.concatenate([lists, np.full((m.shape[0], k - lists.shape[1]), INF, np.float32)], axis=1)
    return pd, np.ascontiguousarray(lists, np.float32)


def bounds(lists, lay, k):
    """(bound [N], kmin [G]): a piece's bound is the k-th smallest of its key's earlier pieces' lists (+INF for the key's first
    piece); a key's minimum is its smallest list value (+INF: no piece)"""
    N, G = lists.shape[0], len(lay["kpiece"]) - 1
    bound = np.full(N, INF, np.float32)
    kp = lay["kpiece"].astype(np.int64)
    for g in np.flatnonzero(np.diff(kp) > 1):
        run = np.full(k, INF, np.float32)
        for pc in range(kp[g], kp[g + 1]):
            bound[pc] = run[k - 1]
            run = np.sort(np.concatenate([run, lists[pc]]))[:k]
    kmin = np.full(G, INF, np.float32)
    has = np.diff(kp) > 0
    if has.any():
        kmin[has] = np.minimum.reduceat(lists[:, 0], kp[:-1][has])
    return bound, kmin


def survivors(pd, bound, lay, ksel=None):
    """uint32 [C, 2] (distance bits, position), in position order: the positions of the selected keys (ksel None: every key)
    with pd < their piece's bound"""
    pc = np.repeat(np.arange(len(lay["pkey"])), np.diff(lay["pstart"].astype(np.int64)))
    keep = pd < bound[pc]
    if ksel is not None:
        keep &= np.asarray(ksel, bool)[lay["pkey"][pc].astype(np.int64)]
    pos = np.flatnonzero(keep)
    return np.stack([pd[pos].view(np.uint32), pos.astype(np.uint32)], axis=1)


def limit_select(kmins, limit):
    """the host's limit cut over the shards' key minima: (every key's minimum over the shards, uint8 ksel or None when the limit
    does not cut).  Keys with a minimum below +INF compete; with limit > 0 below their count, the limit-th smallest minimum is
    the bound and every key at or below it is selected (ties included)"""
    gmin = np.min(np.stack(kmins), axis=0) if len(kmins) else np.zeros(0, np.float32)
    live = gmin < INF
    if not (0 < limit < int(live.sum())):
        return gmin, None
    b = np.sort(gmin[live])[limit - 1]
    return gmin, (gmin <= b).astype(np.uint8)


def state(dist, key_rows, k, kmins_other=(), limit=0):
    """one shard's whole expected state, as Index.debug_grouped names it; kmins_other: the other shards' key minima (the limit
    is taken over all shards)"""
    lay = layout(key_rows)
    pd, lists = walk(dist, lay, k)
    bound, kmin = bounds(lists, lay, k)
    _, ksel = limit_select([kmin, *kmins_other], limit)
    s = dict(lay, pd=pd, lists=lists, bound=bound, kmin=kmin, ksel=ksel, k=k)
    s["pairs"] = survivors(pd, bound, lay, ksel)
    s["dist"] = np.asarray(dist, np.float32) if len(lay["rows"]) else np.zeros(0, np.float32)
    if len(lay["rows"]) == 0:
        s["ksel"] = None                       # a shard without positions compacts nothing
    return s


def same(a, b, zero_by_value=False):
    """bit-for-bit equality of two float32 (or integer) arrays; zero_by_value: -0 and +0 also match"""
    a, b = np.asarray(a), np.asarray(b)
    if a.shape != b.shape:
        return False
    if a.dtype != np.float32 or b.dtype != np.float32:
        return np.array_equal(a, b)
    eq = a.view(np.uint32) == b.view(np.uint32)
    if zero_by_value:
        eq |= (a == 0) & (b == 0)
    return bool(eq.all())


OPEN_ZERO = ("lists", "bound", "kmin")


def diff(got, want):
    """the names whose arrays differ under the comparison rule (empty: the states agree)"""
    bad = []
    for name in ("rows", "koff", "pstart", "pkey", "kpiece", "dist", "pd", "lists", "bound", "kmin", "pairs", "ksel"):
        g, w = got[name], want[name]
        if g is None or w is None:
            if not (g is None and w is None):
                bad.append(name)
        elif not same(g, w, name in OPEN_ZERO):
            bad.append(name)
    if got["k"] != want["k"]:
        bad.append("k")
    return bad
