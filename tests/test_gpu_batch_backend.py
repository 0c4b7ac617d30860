"""The exact back end of the batch path on its own: refine_kernel (vsb_debug_refine), replay_kernel and final_sort_kernel
(vsb_debug_replay), merge_logs_kernel (hand-built entry-log blocks through vsb_batch_merge) and row_norm_kernel (the norms of
vsb_debug_tc_level).  References are numpy float64 / int64, the oracle, and a short restatement of the reference's slot rule
(src/sqlite-vector.c:2145-2152 strict '<', 2022-2049 first index of the maximum, 2057-2065 the exchange sort).  -m gpu.

(a) refine distances: int8 / uint8 bit-exact, f16 / bf16 within the bound of the refine's order of summation, NaN / Inf classes;
(b) the keep rule d < U[q]: ties dropped, bucket overflow, a candidate log longer than its capacity;
(c) replay: planted buckets of 0 .. 2049 entries, k = 1 .. 256, ties, rows past 2^31, every slot -Inf, chained levels, qc;
(d) the final exchange sort, tie order included;
(e) the shard-log merge: world 1 .. 40, every error status, 32-bit global rows, re-arm after a failure;
(f) the entry log of a real shard scan against the host replay of every row;
(g) k rows at -Inf for every query, end to end through the level loop (f16 / bf16 DOT);
(h) row norms: exact int64 sums (uint32 past 2^31), fp within the bound of a lane-strided FMA chain."""
import contextlib
import math

import numpy as np
import pytest

from oracle import pyoracle as po
from tests import fpfamilies as fam
from tests.test_gpu_parity import _special_matrix
from tests.test_gpu_scan_kernel import _assert_within, _fp_bound_and_exact, _int_expected

pytestmark = pytest.mark.gpu

CAP = 2048                              # kBucketCap
INF = math.inf
NAMES = {po.I8: "int8", po.U8: "uint8", po.F16: "f16", po.BF16: "bf16"}


def _vs():
    import sqlite_vector_b200 as vs
    return vs


def _index(vtype, x):
    ix = _vs().Index(vtype, x.shape[1], x.shape[0])
    ix.append_dense(x)
    ix.finalize()
    return ix


@contextlib.contextmanager
def _options(**kw):
    eng = _vs().load_engine()
    old = {k: eng.set_option(k, v) for k, v in kw.items()}
    try:
        yield
    finally:
        for k, v in old.items():
            eng.set_option(k, v)


def _f32(bits):
    return np.asarray(bits, dtype=np.uint32).view(np.float32)


def _fl(bits):
    return float(np.uint32(bits).view(np.float32))


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def _int_data(vtype, n, dim, rng):
    if vtype == po.I8:
        x = rng.integers(-128, 128, (n, dim)).astype(np.int8)
        x[1::17] = -128
    else:
        x = rng.integers(0, 256, (n, dim)).astype(np.uint8)
        x[1::17] = 255
    x[::23] = 0
    return x


# ---------------------------------------------------------------------------------------------- the reference's slot rule
class Slots:
    """one query's slots as the reference keeps them: k distances (+INF unused), rows, max_index; fillers k..kcap-1 are -INF"""

    def __init__(self, k, d=None, r=None, mi=0):
        self.k, self.kcap = k, (k + 31) & ~31
        self.d = [INF] * k if d is None else [float(v) for v in d[:k]]
        self.r = [0] * k if r is None else [int(v) for v in r[:k]]
        self.mi = mi
        self.log = []                                   # (distance, row) of every offer that entered

    def offer(self, d, row):
        if d < self.d[self.mi]:
            self.d[self.mi], self.r[self.mi] = d, row
            self.mi = int(np.argmax(self.d))            # first index of the maximum (vFullScanFindMaxIndex)
            self.log.append((d, row))
            return True
        return False

    @property
    def U(self):
        return self.d[self.mi]

    def sorted(self):
        """vFullScanSortSlots: for i, for j > i, swap on d[j] < d[i]"""
        d, r = list(self.d), list(self.r)
        for i in range(self.k - 1):
            for j in range(i + 1, self.k):
                if d[j] < d[i]:
                    d[i], d[j], r[i], r[j] = d[j], d[i], r[j], r[i]
        return d, r

    def full(self, d=None, r=None):
        d, r = (self.d, self.r) if d is None else (d, r)
        return (np.array(d + [-INF] * (self.kcap - self.k), dtype=np.float32),
                np.array(r + [0] * (self.kcap - self.k), dtype=np.uint32))


def _replay_host(slots, entries):
    """a level as replay_kernel runs it: entries (row, dist bits) ordered by the unsigned key (row << 32) | bits"""
    keys = sorted((int(r) << 32) | int(b) for r, b in entries)
    for key in keys:
        slots.offer(_fl(key & 0xFFFFFFFF), key >> 32)


# ---------------------------------------------------------------------------------------------- (a) refine distances
def _refine_pairs(rng, n, nq, per_query):
    """per query: the last row, row 0 and random others (unique rows); queries up to nq - 1"""
    pairs = []
    for q in range(nq):
        rows = np.unique(np.concatenate([[0, n - 1], rng.choice(n, min(n, per_query) - 2, replace=False)]))[:per_query]
        pairs.append(np.stack([rows, np.full(rows.size, q)], 1))
    p = np.concatenate(pairs).astype(np.uint32)
    return p[rng.permutation(len(p))]


def _bucket_dict(res, nq):
    """{(row, query): distance bits} of the stored entries; asserts the counts fit and unused entries stay all ones"""
    out = {}
    for q in range(nq):
        c = int(res["bcount"][q])
        assert c <= CAP, (q, c)
        b = res["bucket"][q]
        assert np.all(b[c:] == 0xFFFFFFFF), ("written past the count", q)
        for row, bits in b[:c]:
            assert (int(row), q) not in out, ("duplicate", int(row), q)
            out[int(row), q] = int(bits)
    return out


@pytest.mark.parametrize("vtype,dim", [(po.I8, 16), (po.I8, 100), (po.I8, 384), (po.I8, 4096), (po.U8, 16), (po.U8, 100),
                                       (po.U8, 384), (po.U8, 4096), (po.U8, 33040)])
def test_refine_int_distances_bit_exact(oracle, vtype, dim):
    """against the oracle's integer arithmetic bit for bit (NaN and +Inf are never kept, so their pairs must be missing).
    dim 16: one 16-byte chunk, 7 of the 8 lanes idle; 100: pitch tail; uint8 33040: an all-255 row's sum of squares
    (2.149e9) exceeds 2^31 (L2 and COSINE only there)"""
    rng = np.random.Generator(np.random.PCG64(11 * dim + vtype))
    n = 600 if dim > 4096 else 3000
    nq = 300 if dim <= 100 else (40 if dim <= 4096 else 16)
    x = _int_data(vtype, n, dim, rng)
    q = _int_data(vtype, nq, dim, rng)
    if dim > 4096:
        # the reference's integer kernels keep the sum of squared differences in int32 (the oracle's int_exact): no zero
        # vectors here, so that no pair's sum passes 2^31 while the all-255 rows' and queries' own norms do
        x[::23] = rng.integers(1, 256, (x[::23].shape))
        q[::23] = rng.integers(1, 256, (q[::23].shape))
    hi = -128 if vtype == po.I8 else 255
    x[n - 1] = hi
    q[nq - 1] = hi
    metrics = [po.L2, po.COS] if dim > 4096 else [po.L2, po.L2SQ, po.COS, po.DOT]
    ix = _index(vtype, x)
    pairs = _refine_pairs(rng, n, nq, 200 if nq > 100 else 600)
    for metric in metrics:
        res = ix.debug_refine(metric, q, pairs, np.full(nq, np.inf, np.float32))
        got = _bucket_dict(res, nq)
        assert res["stats"][0] == len(pairs) and res["stats"][2] == 0
        for qi in sorted({0, nq - 1} | set(rng.choice(nq, 6).tolist())):
            want = oracle.distances_all(metric, vtype, q[qi], x, int_exact=True)
            rows = pairs[pairs[:, 1] == qi, 0].astype(np.int64)
            kept = np.array([(int(r), qi) in got for r in rows])
            assert np.array_equal(kept, want[rows] < np.inf), (NAMES[vtype], dim, po.METRIC_NAMES[metric], qi, "kept set",
                                                               rows[kept != (want[rows] < np.inf)][:5].tolist())
            rows = rows[kept]
            g = np.array([got[int(r), qi] for r in rows], dtype=np.uint32)
            bad = np.flatnonzero(g != _bits(want[rows]))
            assert bad.size == 0, (NAMES[vtype], dim, po.METRIC_NAMES[metric], qi, rows[bad[:5]].tolist(),
                                   _f32(g[bad[:5]]).tolist(), want[rows[bad[:5]]].tolist())
    ix.close()


def _report(rec, path="VSB_REFINE_ERR_REPORT"):
    import json
    import os
    p = os.environ.get(path)
    if p:
        with open(p, "a") as f:
            f.write(json.dumps(rec) + "\n")


@pytest.mark.parametrize("family", fam.FAMILIES)
@pytest.mark.parametrize("vtype", [po.F16, po.BF16])
def test_refine_fp_within_bound(vtype, family):
    """the refine's order: 8 lanes per pair, chunks sub, sub + 8, ..., two FMA chains by element parity, three butterflies
    (the scan kernel's bound at P = 8); the query norm of COSINE is an 8-lane chain here"""
    rng = np.random.Generator(np.random.PCG64(300 + 10 * vtype + fam.FAMILIES.index(family)))
    for dim in (8, 100, 771):
        n, nq = 700, 20
        pitch = (dim * 2 + 15) // 16 * 16
        x = fam.make(family, vtype, n, dim, rng)
        q = fam.make(family, vtype, nq, dim, rng, queries=True)
        xr, qd = fam.decode(vtype, x), fam.decode(vtype, q)
        ix = _index(vtype, x)
        pairs = _refine_pairs(rng, n, nq, 400)
        for metric in (po.L2, po.L2SQ, po.COS, po.DOT):
            res = ix.debug_refine(metric, q, pairs, np.full(nq, np.inf, np.float32))
            got = _bucket_dict(res, nq)
            worst = 0.0
            for qi in range(nq):
                rows = np.sort(pairs[pairs[:, 1] == qi, 0].astype(np.int64))
                d, bound = _fp_bound_and_exact(metric, vtype, xr[rows], qd[qi], pitch // 16, 3, q_lanes=8)
                keep = d < np.inf                          # the bound is finite for these families: every pair is kept
                assert all((int(r), qi) in got for r in rows[keep]), (dim, metric, qi, "kept set")
                g = _f32(np.array([got[int(r), qi] for r in rows[keep]], dtype=np.uint32))
                worst = max(worst, _assert_within(g, d[keep], bound[keep], (NAMES[vtype], family, po.METRIC_NAMES[metric], dim, qi)))
            _report({"type": NAMES[vtype], "family": family, "metric": po.METRIC_NAMES[metric], "dim": dim, "ratio": worst})
        ix.close()


def _classes(a):
    a = np.asarray(a, dtype=np.float64)
    return np.where(np.isnan(a), 0, np.where(np.isposinf(a), 1, np.where(np.isneginf(a), 2, np.where(a == 1.0, 3, 4))))


@pytest.mark.parametrize("vtype,metrics", [(po.F16, (po.L2, po.L2SQ, po.COS, po.DOT)), (po.BF16, (po.L2,))])
def test_refine_special_classes(oracle, vtype, metrics):
    """rows holding NaN / +-Inf (f16, every metric) and bf16 "huge" rows (L2): the kept pairs are exactly the oracle's
    pairs below +INF (NaN and +Inf never kept), each with the oracle's class; finite values within 1e-5"""
    rng = np.random.Generator(np.random.PCG64(77 + vtype))
    dim = 40
    if vtype == po.F16:
        x, _ = _special_matrix(vtype, rng, 96, dim)
        q = np.concatenate([x[[0, 5, 11, 9, 13]], po.convert(rng.standard_normal((3, dim), dtype=np.float32), vtype)])
    else:
        x = fam.make("huge", vtype, 96, dim, rng)
        q = po.convert(rng.standard_normal((6, dim), dtype=np.float32), vtype)
    n, nq = x.shape[0], q.shape[0]
    ix = _index(vtype, x)
    pairs = np.array([(r, j) for j in range(nq) for r in range(n)], dtype=np.uint32)
    for metric in metrics:
        got = _bucket_dict(ix.debug_refine(metric, q, pairs, np.full(nq, np.inf, np.float32)), nq)
        for j in range(nq):
            want = oracle.distances_all(metric, vtype, q[j], x)
            kept = np.array([(r, j) in got for r in range(n)])
            assert np.array_equal(kept, want < np.inf), (NAMES[vtype], metric, j, np.flatnonzero(kept != (want < np.inf)))
            rows = np.flatnonzero(kept)
            g = _f32(np.array([got[int(r), j] for r in rows], dtype=np.uint32)).astype(np.float64)
            w = want[rows].astype(np.float64)
            assert np.array_equal(_classes(g), _classes(w)), (NAMES[vtype], metric, j, rows[_classes(g) != _classes(w)])
            fin = np.isfinite(w)
            scale = np.maximum(np.abs(w[fin]), 1.0 if metric in (po.COS, po.DOT) else 1e-30)
            assert np.all(np.abs(g[fin] - w[fin]) <= 1e-5 * scale), (NAMES[vtype], metric, j)
    ix.close()


# ---------------------------------------------------------------------------------------------- (b) refine keep rule
def test_refine_keep_rule_ties_and_capacities():
    """int8 L2SQ: integer distances, so U can sit exactly on a pair's distance (dropped: strict <), on its float successor
    (kept), at +INF (all) and -INF (none); a query with more than 2048 kept pairs; a pair list longer than cand_cap"""
    rng = np.random.Generator(np.random.PCG64(4))
    n, dim, nq = 3000, 16, 24
    x = rng.integers(-3, 4, (n, dim)).astype(np.int8)            # few distinct distances: many ties
    q = rng.integers(-3, 4, (nq, dim)).astype(np.int8)
    d = np.stack([_int_expected(po.I8, po.L2SQ, x, q[j]) for j in range(nq)], 1)   # [n, nq]
    ix = _index(po.I8, x)
    rows_of = [rng.choice(n - 1, 1500, replace=False) for _ in range(nq)]
    rows_of[0] = np.arange(n)                                     # query 0: 3000 pairs
    pairs = np.concatenate([np.stack([r, np.full(r.size, j)], 1) for j, r in enumerate(rows_of)]).astype(np.uint32)
    pairs = pairs[rng.permutation(len(pairs))]
    U = np.empty(nq, np.float32)
    for j in range(nq):
        pick = np.float32(d[rows_of[j][7], j])
        U[j] = [pick, np.nextafter(pick, np.float32(np.inf)), np.inf, -np.inf][j % 4]
    U[0] = np.inf
    U[1] = -np.inf                                                # right after the overflowing query: must stay empty
    for cap in (len(pairs), len(pairs) // 3):
        res = ix.debug_refine(po.L2SQ, q, pairs, U, cand_cap=cap)
        assert res["stats"][0] == cap and res["stats"][2] == (1 if cap < len(pairs) else 0), res["stats"]
        seen = pairs[:cap]
        for j in range(nq):
            rj = seen[seen[:, 1] == j, 0].astype(np.int64)
            want = set(rj[d[rj, j] < U[j]].tolist())
            c = int(res["bcount"][j])
            stored = res["bucket"][j][: min(c, CAP)]
            assert np.all(res["bucket"][j][min(c, CAP):] == 0xFFFFFFFF), ("written beyond the stored entries", j)
            assert c == len(want), (cap, j, c, len(want), float(U[j]))
            assert set(stored[:, 0].tolist()) <= want and len(set(stored[:, 0].tolist())) == min(c, CAP)
            assert np.array_equal(stored[:, 1], _bits(d[stored[:, 0].astype(np.int64), j])), j
        if cap == len(pairs):
            assert res["bcount"][0] == n > CAP
    # NaN / +Inf distances (f16 rows with specials) are never kept, not even under U = +INF: see test_refine_special_classes
    ix.close()


# ---------------------------------------------------------------------------------------------- (c) replay
def _plant(rng, nq, counts, row_pool, dist_fn):
    """buckets [nq, CAP, 2] in random order with counts[q] entries (only the first CAP stored), unique rows per query"""
    b = np.full((nq, CAP, 2), 0xFFFFFFFF, dtype=np.uint32)
    entries = []
    for j in range(nq):
        c = min(int(counts[j]), CAP)
        rows = rng.choice(row_pool, c, replace=False) if c else np.zeros(0, np.uint64)
        e = np.stack([rows.astype(np.uint32), _bits(dist_fn(c))], 1) if c else np.zeros((0, 2), np.uint32)
        b[j, :c] = e
        entries.append(e)
    return b, entries


def _ints(rng, lo, hi):
    return lambda c: rng.integers(lo, hi, c).astype(np.float32)


def _with_specials(rng):
    def f(c):
        v = rng.integers(0, 40, c).astype(np.float32)
        sp = rng.random(c)
        v[sp < 0.05] = -np.inf
        v[(sp >= 0.05) & (sp < 0.1)] = np.inf
        return v
    return f


def _replay_index(vtype=po.I8, dim=64, n=256, seed=1):
    rng = np.random.Generator(np.random.PCG64(seed))
    x = _int_data(vtype, n, dim, rng) if vtype in (po.I8, po.U8) else po.convert(rng.standard_normal((n, dim), dtype=np.float32), vtype)
    return _index(vtype, x), rng


def _queries(vtype, nq, dim, rng):
    if vtype in (po.I8, po.U8):
        return _int_data(vtype, nq, dim, rng)
    return po.convert(rng.standard_normal((nq, dim), dtype=np.float32), vtype)


def _check_replay(res, hosts, k, ctx, acc_cap=0):
    nq = len(hosts)
    for j, h in enumerate(hosts):
        wd, wr = h.full()
        assert np.array_equal(_bits(res["slot_d"][j]), _bits(wd)), (ctx, j, "slot distances", res["slot_d"][j][:k].tolist(), wd[:k].tolist())
        assert np.array_equal(res["slot_row"][j][:k], wr[:k]), (ctx, j, "slot rows")
        assert res["slot_mi"][j] == h.mi, (ctx, j, f"slot_mi {int(res['slot_mi'][j]):#x}, want {h.mi}")
        assert _bits(res["U"][j]) == _bits(np.float32(h.U)), (ctx, j, "U")
        if acc_cap:
            assert res["acc_count"][j] == len(h.log), (ctx, j, "log count", int(res["acc_count"][j]), len(h.log))
            m = min(len(h.log), acc_cap)
            want = np.array([(int(np.float32(dd).view(np.uint32)), r) for dd, r in h.log[:m]], dtype=np.uint32).reshape(-1, 2)
            assert np.array_equal(res["acc_log"][j][:m], want), (ctx, j, "log entries")
    assert np.all(res["bcount"][:nq] == 0), (ctx, "bcount not reset")


COUNTS = [0, 1, 31, 32, 33, 1023, 1024, 1025, 2047, 2048, 2049]


@pytest.mark.parametrize("k", [1, 20, 31, 32, 33, 200, 256])
def test_replay_planted_buckets(k):
    """every bucket size from empty to one past the capacity, in random order, small integer distances (ties with the
    current maximum must not enter), +-INF, rows at and above 2^31 up to 0xFFFFFFFF (the unsigned key order against the
    ~0 padding); one level from the initial state with the entry log on"""
    ix, rng = _replay_index(seed=k)
    nq = len(COUNTS) + 2
    counts = COUNTS + [5000, 300]
    q = _queries(po.I8, nq, 64, rng)
    pool = np.concatenate([np.arange(0, 3000), np.arange(2 ** 31 - 1000, 2 ** 31 + 1000), np.arange(2 ** 32 - 500, 2 ** 32)]).astype(np.uint64)
    b, entries = _plant(rng, nq, counts, pool, _with_specials(rng))
    acc_cap = 600
    res = ix.debug_replay(po.L2SQ, q, k, b, np.array(counts, np.uint32), acc_cap=acc_cap)
    hosts = []
    for j in range(nq):
        h = Slots(k)
        _replay_host(h, entries[j])
        hosts.append(h)
    _check_replay(res, hosts, k, ("k", k), acc_cap)
    assert res["stats"][1] == sum(min(c, CAP) for c in counts) and res["stats"][2] == 2, res["stats"]
    res2 = ix.debug_replay(po.L2SQ, q[:3], k, b[:3], np.array(counts[:3], np.uint32))
    assert res2["stats"][2] == 0
    ix.close()


@pytest.mark.parametrize("vtype", [po.I8, po.F16])
def test_replay_every_slot_neg_inf(vtype):
    """k or more -INF entries fill every real slot: the first index of the maximum is slot 0 (the reference's
    vFullScanFindMaxIndex), and the next level continues from there; an empty level keeps the state"""
    ix, rng = _replay_index(vtype, seed=5)
    nq = 16
    q = _queries(vtype, nq, 64, rng)
    for k in (1, 5, 32, 33):
        counts = np.array([k + (j % 3) for j in range(nq)], np.uint32)
        b = np.full((nq, CAP, 2), 0xFFFFFFFF, np.uint32)
        entries = []
        for j in range(nq):
            c = int(counts[j])
            e = np.stack([rng.choice(10000, c, replace=False).astype(np.uint32), _bits(np.full(c, -np.inf, np.float32))], 1)
            e[0, 1] = np.float32(3.0).view(np.uint32) if c > k else e[0, 1]
            b[j, :c] = e
            entries.append(e)
        res = ix.debug_replay(po.DOT, q, k, b, counts)
        hosts = []
        for j in range(nq):
            h = Slots(k)
            _replay_host(h, entries[j])
            hosts.append(h)
            assert h.mi == 0 and h.U == -INF
        _check_replay(res, hosts, k, ("all -inf", k))
        # the next level: an empty bucket, and one with more -INF / finite offers (none can enter)
        nxt = ix.debug_replay(po.DOT, q, k, b, np.array([0, 5] * (nq // 2), np.uint32), level0=False, slot_d=res["slot_d"],
                              slot_row=res["slot_row"], slot_mi=res["slot_mi"])
        assert np.array_equal(_bits(nxt["slot_d"]), _bits(res["slot_d"])) and np.array_equal(nxt["slot_mi"], res["slot_mi"])
    ix.close()


def test_replay_chained_levels_and_entry_log():
    """levels fed back into the hook: slot_mi, the slots and the entry log's count carry across; a log that fills exactly
    acc_cap is complete, one entry more shows as a count of acc_cap + 1 with acc_cap entries stored"""
    ix, rng = _replay_index(seed=9)
    nq, k = 24, 20
    q = _queries(po.I8, nq, 64, rng)
    hosts = [Slots(k) for _ in range(nq)]
    state = None
    row0 = 0
    # descending distance bands per level: nearly every offer enters, so the logs grow by about one level's entries
    for level, c in enumerate([40, 300, 700, 2048, 5]):
        counts = np.full(nq, c, np.uint32)
        b = np.full((nq, CAP, 2), 0xFFFFFFFF, np.uint32)
        for j in range(nq):
            rows = np.arange(row0, row0 + c, dtype=np.uint32)
            dist = (rng.integers(0, 1000, c) + 1000 * (10 - level)).astype(np.float32)
            e = np.stack([rows, _bits(dist)], 1)
            b[j, :c] = e[rng.permutation(c)]
            _replay_host(hosts[j], e)
        row0 += c
        kw = {} if state is None else dict(level0=False, slot_d=state["slot_d"], slot_row=state["slot_row"], slot_mi=state["slot_mi"],
                                           acc_log=state["acc_log"], acc_count=state["acc_count"])
        # acc_cap: for query 0 exactly the final count, for query 1 one below it (decided after the fact: rerun below)
        state = ix.debug_replay(po.L2SQ, q, k, b, counts, acc_cap=4096, **kw)
        _check_replay(state, hosts, k, ("level", level), 4096)
    total = [len(h.log) for h in hosts]
    assert min(total) > k
    ix.close()
    # the capacity edge: replay the concatenated levels as one planted level with acc_cap = count and count - 1
    ix, rng = _replay_index(seed=10)
    c = 1500
    e = np.stack([np.arange(c, dtype=np.uint32), _bits((3000 - np.arange(c)).astype(np.float32))], 1)   # every offer enters
    b = np.full((nq, CAP, 2), 0xFFFFFFFF, np.uint32)
    b[:, :c] = e[rng.permutation(c)]
    h = Slots(k)
    _replay_host(h, e)
    assert len(h.log) == c
    for acc_cap in (c, c - 1):
        res = ix.debug_replay(po.L2SQ, q, k, b, np.full(nq, c, np.uint32), acc_cap=acc_cap)
        assert np.all(res["acc_count"] == c), (acc_cap, res["acc_count"][:4])
        want = np.array([(int(np.float32(dd).view(np.uint32)), r) for dd, r in h.log[:acc_cap]], dtype=np.uint32)
        assert all(np.array_equal(res["acc_log"][j], want) for j in range(nq)), acc_cap
    ix.close()


def _qc_int(metric, U, qnorm):
    """conservative_qc (batch_kernels.cuh) for the integer kinds, restated in float64 / float32 like the device code; qnorm
    is the exact query sum of squares (uint8 past 2^31 included: the device reads it as uint32)"""
    lo, hi = -2147483647.0, 2147483646.0
    qq = float(qnorm)
    Ud = float(U)
    with np.errstate(invalid="ignore", over="ignore"):
        if metric == po.DOT:
            b = -Ud - 1.0 - 2e-7 * abs(Ud)
            if not (np.float32(U) < np.float32(3.0e38)):
                b = lo
            return int(np.fmin(np.fmax(np.floor(b), lo), hi))
        if metric in (po.L2, po.L2SQ):
            u2 = Ud * Ud if metric == po.L2 else Ud
            d2max = math.ceil(u2 * (1.0 + 1e-6)) + 1.0 if math.isfinite(u2) else u2 + 1.0
            if not (np.float32(U) < np.float32(3.0e38)) or not (d2max < 4.0e9):
                d2max = 4.0e9
            return int(np.fmin(np.fmax(qq - d2max, lo), hi))
        u = np.fmin(np.float32(U), np.float32(3.0e38))
        v = (np.float32(1.0) - u - np.float32(1e-5)) * np.sqrt(np.float32(qq))
        return int(np.float32(np.fmin(np.fmax(v, np.float32(-1e30)), np.float32(1e30))).view(np.int32))


@pytest.mark.parametrize("vtype", [po.I8, po.U8, po.F16, po.BF16])
def test_replay_qc(vtype):
    """the next level's constant: int kinds equal to a restatement of conservative_qc; fp kinds equal to the qc that
    vsb_debug_tc_level derives from the same U (the same device function)"""
    dim = 33040 if vtype == po.U8 else 64                 # uint8: query norms past 2^31 (all-255 queries)
    ix, rng = _replay_index(vtype, dim=dim, seed=20 + vtype)
    nq, k = 40, 3
    q = _queries(vtype, nq, dim, rng)
    if vtype == po.U8:
        q[::5] = 255
    counts = np.array([j % 7 for j in range(nq)], np.uint32)
    b, _ = _plant(rng, nq, counts, np.arange(5000, dtype=np.uint64), lambda c: (rng.random(c) * 10.0 ** rng.integers(-3, 9, c)).astype(np.float32))
    b[3, 0, 1] = np.float32(-np.inf).view(np.uint32)             # U = -INF for query 3 (k = 3 slots, three -INF when count 3)
    b[3, 1, 1] = np.float32(-np.inf).view(np.uint32)
    b[3, 2, 1] = np.float32(-np.inf).view(np.uint32)
    for metric in (po.L2, po.L2SQ, po.COS, po.DOT):
        res = ix.debug_replay(metric, q, k, b, counts)
        if vtype in (po.I8, po.U8):
            q64 = q.astype(np.int64)
            qn = (q64 * q64).sum(1)
            want = np.array([_qc_int(metric, res["U"][j], int(qn[j])) for j in range(nq)], dtype=np.int64).astype(np.int32).view(np.uint32)
        else:
            want = ix.debug_tc_level(metric, q, res["U"], 0, 128)["qc"]
        assert np.array_equal(res["qc"], want), (NAMES[vtype], metric, np.flatnonzero(res["qc"] != want)[:5],
                                                 res["U"][res["qc"] != want][:5])
    ix.close()


def test_replay_rejects_bad_state():
    vs = _vs()
    ix, rng = _replay_index(seed=30)
    q = _queries(po.I8, 16, 64, rng)
    b = np.full((16, CAP, 2), 0xFFFFFFFF, np.uint32)
    z = np.zeros(16, np.uint32)
    for k, mi in ((20, 20), (20, -1), (1, 1)):
        with pytest.raises(vs.VsbError) as e:
            ix.debug_replay(po.L2, q, k, b, z, level0=False, slot_mi=np.full(16, mi, np.int32))
        assert e.value.rc == vs.api.EINVAL
    for k in (0, 257):
        with pytest.raises(vs.VsbError) as e:
            ix.debug_replay(po.L2, q, k, b, z)
        assert e.value.rc == vs.api.EINVAL
    ix.close()


# ---------------------------------------------------------------------------------------------- (d) final sort
@pytest.mark.parametrize("k", [1, 33, 256])
def test_final_sort_exchange_order(k):
    """the exchange sort of vFullScanSortSlots, tie order included, +INF (unused) slots at the end; k = 256 takes more
    than 48 KB of dynamic shared memory"""
    ix, rng = _replay_index(seed=40 + k)
    nq = 40
    q = _queries(po.I8, nq, 64, rng)
    counts = np.array([rng.integers(0, 3 * k + 2) for _ in range(nq)], np.uint32)
    counts[0], counts[1] = 0, k
    b, entries = _plant(rng, nq, counts, np.arange(100000, dtype=np.uint64), _with_specials(rng))
    res = ix.debug_replay(po.L2SQ, q, k, b, counts, final_sort=True)
    for j in range(nq):
        h = Slots(k)
        _replay_host(h, entries[j])
        wd, wr = h.full(*h.sorted())
        assert np.array_equal(_bits(res["slot_d"][j]), _bits(wd)), (k, j, res["slot_d"][j][:8].tolist(), wd[:8].tolist())
        assert np.array_equal(res["slot_row"][j][:k], wr[:k]), (k, j, "rows (tie order)")
    ix.close()


# ---------------------------------------------------------------------------------------------- (e) merge
def _acc_cap(k):
    return max(512, 24 * k)


def _block(nq, k, counts, logs, hdr3=0, hdr=None):
    """one shard's entry-log block (acc_block_* in batch_kernels.cuh): 64-byte header, counts, nq x acc_cap (bits, row)"""
    cap = _acc_cap(k)
    off = 64 + 4 * ((nq + 15) & ~15)
    buf = np.zeros(off + 8 * nq * cap, np.uint8)
    h = buf[:64].view(np.int32)
    h[:4] = (nq, k, cap, hdr3) if hdr is None else hdr
    buf[64:64 + 4 * nq].view(np.int32)[:] = counts
    lg = buf[off:].view(np.uint32).reshape(nq, cap, 2)
    for j in range(nq):
        m = min(int(counts[j]), cap, len(logs[j]))
        lg[j, :m] = logs[j][:m]
    return buf


def _merge(ix, blocks, first_seq, nq, k, stride=None):
    import torch
    nbytes = blocks[0].size
    stride = stride or nbytes
    host = np.zeros(stride * len(blocks), np.uint8)
    for r, blk in enumerate(blocks):
        host[r * stride:r * stride + nbytes] = blk
    dev = torch.from_numpy(host).cuda()
    torch.cuda.synchronize()
    try:
        return ix.batch_merge(dev.data_ptr(), len(blocks), stride, np.asarray(first_seq, np.int64), nq, k)
    finally:
        torch.cuda.synchronize()
        del dev


def _random_logs(rng, nq, k, counts, nrows):
    logs = []
    for j in range(nq):
        c = int(counts[j])
        rows = np.sort(rng.choice(nrows, c, replace=False)).astype(np.uint32)
        d = rng.integers(0, 30, c).astype(np.float32)
        d[rng.random(c) < 0.05] = np.inf
        logs.append(np.stack([_bits(d), rows], 1))
    return logs


@pytest.mark.parametrize("world", [1, 2, 3, 16, 17, 40])
def test_merge_against_slot_rule(world):
    """world 17 and above take the pageable first_seq copy instead of store_ints_kernel; counts of 0 and exactly acc_cap,
    ties across shards, +INF entries, a block stride larger than a block"""
    ix, rng = _replay_index(seed=50 + world)
    nq = 18
    for k in (1, 20):
        cap = _acc_cap(k)
        first, blocks, all_logs = [], [], []
        base = 0
        for r in range(world):
            counts = rng.integers(0, 60, nq)
            counts[0] = 0
            counts[1] = cap if r % 3 == 0 else counts[1]
            nrows = 5000
            logs = _random_logs(rng, nq, k, counts, nrows)
            first.append(base)
            base += nrows
            blocks.append(_block(nq, k, counts, logs))
            all_logs.append(logs)
        for stride in (None, blocks[0].size + 4096):
            seq, dist, cnt = _merge(ix, blocks, first, nq, k, stride)
            for j in range(nq):
                h = Slots(k)
                for r in range(world):
                    for bits, row in all_logs[r][j]:
                        h.offer(_fl(bits), first[r] + int(row))
                wd, wr = h.sorted()
                used = [i for i in range(k) if wd[i] != INF]
                assert cnt[j] == len(used), (world, k, j)
                assert np.array_equal(dist[j][:len(used)], np.array(wd[:len(used)], np.float64)), (world, k, j)
                assert np.array_equal(seq[j][:len(used)], np.array(wr[:len(used)], np.int64)), (world, k, j)
    ix.close()


def test_merge_error_statuses_and_rearm():
    """a header that does not match (nq, k, acc_cap): VSB_EINVAL; hdr[3] != 0 (a shard's levels overflowed), a count above
    acc_cap, and a global row first_seq + local row >= 2^32: VSB_ERANGE; a clean merge right after each succeeds"""
    vs = _vs()
    ix, rng = _replay_index(seed=60)
    nq, k = 16, 5
    cap = _acc_cap(k)
    counts = rng.integers(1, 40, nq)
    logs = _random_logs(rng, nq, k, counts, 100)
    good = _block(nq, k, counts, logs)
    clean = _merge(ix, [good, good], [0, 100], nq, k)
    over = counts.copy()
    over[5] = cap + 1
    wrap_logs = [lg.copy() for lg in logs]
    wrap_logs[3][-1, 1] = 20
    cases = [
        ("header nq", [good, _block(nq, k, counts, logs, hdr=(nq + 1, k, cap, 0))], [0, 100], vs.api.EINVAL),
        ("header k", [_block(nq, k, counts, logs, hdr=(nq, k + 1, cap, 0)), good], [0, 100], vs.api.EINVAL),
        ("header acc_cap", [good, _block(nq, k, counts, logs, hdr=(nq, k, cap - 1, 0))], [0, 100], vs.api.EINVAL),
        ("hdr[3]", [good, _block(nq, k, counts, logs, hdr3=2)], [0, 100], vs.api.ERANGE),
        ("count > acc_cap", [good, _block(nq, k, over, logs)], [0, 100], vs.api.ERANGE),
        ("global row >= 2^32", [good, _block(nq, k, counts, wrap_logs)], [0, 2 ** 32 - 10], vs.api.ERANGE),
    ]
    for name, blocks, first, rc in cases:
        with pytest.raises(vs.VsbError) as e:
            _merge(ix, blocks, first, nq, k)
        assert e.value.rc == rc, (name, e.value.rc, str(e.value))
        again = _merge(ix, [good, good], [0, 100], nq, k)
        assert all(np.array_equal(a, b) for a, b in zip(again, clean)), ("not re-armed after", name)
    # the last row that fits: first_seq + local row = 2^32 - 1 is carried exactly
    edge = [lg.copy() for lg in logs]
    for lg in edge:
        lg[:, 1] = np.minimum(lg[:, 1], 8)
    edge[3][-1, 1] = 9
    edge[3][-1, 0] = np.float32(-1.0).view(np.uint32)
    seq, dist, _ = _merge(ix, [_block(nq, k, counts, edge)], [2 ** 32 - 10], nq, k)
    assert seq[3][0] == 2 ** 32 - 1 and dist[3][0] == -1.0
    ix.close()


# ---------------------------------------------------------------------------------------------- (f) composition
def _shard_block(ix, metric, q, k):
    import torch

    from sqlite_vector_b200.shard import _DevView
    ptr, nbytes = ix.batch_shard_scan(metric, q, k)
    blk = torch.as_tensor(_DevView(ptr, nbytes), device="cuda").cpu().numpy().copy()
    nq = q.shape[0]
    h = blk[:64].view(np.int32)
    cap = _acc_cap(k)
    assert tuple(h[:3]) == (nq, k, cap)
    counts = blk[64:64 + 4 * nq].view(np.int32)
    off = 64 + 4 * ((nq + 15) & ~15)
    lg = blk[off:off + 8 * nq * cap].view(np.uint32).reshape(nq, cap, 2)
    return counts, lg


@pytest.mark.parametrize("vtype", [po.I8, po.U8])
def test_entry_log_of_a_real_shard_scan(vtype):
    """the log a shard scan returns is exactly the host replay of every row in scan order: the rows whose distance is below
    the running k-th smallest over all earlier rows, with their distances; for several level schedules"""
    rng = np.random.Generator(np.random.PCG64(70 + vtype))
    n, dim, nq = 20000, 48, 16
    x = _int_data(vtype, n, dim, rng)
    q = _int_data(vtype, nq, dim, rng)
    ix = _index(vtype, x)
    metric = po.L2
    d = np.stack([_int_expected(vtype, metric, x, q[j]) for j in range(nq)])
    for k in (1, 20, 256):
        hosts = []
        for j in range(nq):
            h = Slots(k)
            dj = d[j].tolist()
            for r in range(n):
                if dj[r] < h.d[h.mi]:
                    h.offer(dj[r], r)
            hosts.append(h)
        for m0, g in ((None, None), (256, 8), (2048, 64)):
            opts = {} if m0 is None else dict(batch_m0=m0, batch_growth=g)
            with _options(**opts):
                counts, lg = _shard_block(ix, metric, q, k)
            for j in range(nq):
                log = hosts[j].log
                assert counts[j] == len(log), (NAMES[vtype], k, m0, j, int(counts[j]), len(log))
                want = np.array([(int(np.float32(dd).view(np.uint32)), r) for dd, r in log], dtype=np.uint32)
                assert np.array_equal(lg[j, :len(log)], want), (NAMES[vtype], k, m0, j)
    ix.close()


@pytest.mark.parametrize("vtype", [po.F16, po.BF16])
def test_entry_log_fp_replays_to_scan_topk(vtype):
    """fp: the log is strictly increasing in row, every entry enters when the log is replayed, and the replay gives exactly
    the scan_topk result of the same index"""
    rng = np.random.Generator(np.random.PCG64(80 + vtype))
    n, dim, nq = 20000, 64, 16
    x = po.convert(rng.standard_normal((n, dim), dtype=np.float32), vtype)
    q = po.convert(rng.standard_normal((nq, dim), dtype=np.float32), vtype)
    ix = _index(vtype, x)
    for metric in (po.L2, po.COS, po.DOT):
        for k in (1, 20):
            counts, lg = _shard_block(ix, metric, q, k)
            res = ix.scan_topk(metric, q, k)
            for j in range(nq):
                e = lg[j, :counts[j]]
                assert np.all(np.diff(e[:, 1].astype(np.int64)) > 0), (metric, k, j, "rows not increasing")
                h = Slots(k)
                for bits, row in e:
                    assert h.offer(_fl(bits), int(row)), (metric, k, j, "a logged entry does not enter")
                wd, wr = h.sorted()
                m = sum(1 for v in wd if v != INF)
                assert np.array_equal(res[j][0], np.array(wr[:m], np.int64) + 1), (metric, k, j)
                assert np.array_equal(res[j][1], np.array(wd[:m], np.float64)), (metric, k, j)
    ix.close()


# ---------------------------------------------------------------------------------------------- (g) -Inf slots end to end
@pytest.mark.parametrize("k", [1, 5])
@pytest.mark.parametrize("vtype", [po.F16, po.BF16])
def test_batch_all_slots_neg_inf_end_to_end(oracle, vtype, k):
    """k or more rows at -INF for every query (a +Inf element against a positive query element), placed in rows 0..127,
    in a middle level and in the last level: the batch path must give the oracle's result"""
    rng = np.random.Generator(np.random.PCG64(90 + vtype + k))
    n, dim, nq = 20000, 40, 32
    pinf = 0x7C00 if vtype == po.F16 else 0x7F80
    q = po.convert(np.abs(rng.standard_normal((nq, dim), dtype=np.float32)) + 0.5, vtype)
    rowids = np.arange(1, n + 1, dtype=np.int64)
    for where in ((3, 50, 127), (1500, 4000, 7000), (12000, 15000, 19999)):
        x = po.convert(rng.standard_normal((n, dim), dtype=np.float32), vtype)
        rows = np.unique(np.concatenate([np.array(where), rng.integers(where[0], where[-1] + 1, k)]))
        assert rows.size >= k
        x[rows, 0] = pinf
        ix = _index(vtype, x)
        b0 = ix.stat("batches")
        res = ix.scan_topk(po.DOT, q, k)
        assert ix.stat("batches") == b0 + 1, "the tensor-core batch path did not run"
        for b in range(nq):
            want_ids, want_d = oracle.scan_dense(po.DOT, vtype, q[b], x, rowids, k)
            got_ids, got_d = res[b]
            assert len(got_d) == len(want_d), (where, b)
            inf = np.isinf(want_d)
            assert np.array_equal(np.isinf(got_d), inf) and np.array_equal(np.sign(got_d[inf]), np.sign(want_d[inf])), (where, b, got_d, want_d)
            assert np.array_equal(got_ids[inf], want_ids[inf]), (where, b, got_ids, want_ids)
            fin = ~inf
            assert np.all(np.abs(got_d[fin] - want_d[fin]) <= 1e-5 * np.maximum(np.abs(want_d[fin]), 1.0)), (where, b)
        ix.close()


# ---------------------------------------------------------------------------------------------- tile widths of the scoring kernels
def test_tc_level_tile_widths():
    """vsb_debug_tc_level takes exactly the query tiles a scoring kernel exists for: N = 32 .. 256 for int8 / uint8 on the
    tensor cores, 32 .. 128 for f16 / bf16 and for L1 on every type, N = 0 (the production width) wherever a kernel exists;
    every other N, and f32 with a tensor-core metric, is VSB_EINVAL"""
    vs = _vs()
    rng = np.random.Generator(np.random.PCG64(120))
    n, dim, nq = 256, 64, 40
    for vtype in (po.F32, po.F16, po.BF16, po.U8, po.I8):
        make = (lambda m: _int_data(vtype, m, dim, rng)) if vtype in (po.I8, po.U8) else (lambda m: fam.make("normal", vtype, m, dim, rng))
        ix = _index(vtype, make(n))
        q = make(nq)
        for metric in (po.L2, po.DOT, po.COS, po.L1):
            if metric == po.L1:
                widths = {32, 64, 128}
            elif vtype == po.F32:
                widths = set()
            else:
                widths = {32, 64, 128, 256} if vtype in (po.I8, po.U8) else {32, 64, 128}
            for N in (0, 16, 32, 48, 64, 128, 256, 512):
                ok = N in widths or (N == 0 and bool(widths))
                try:
                    ix.debug_tc_level(metric, q, np.full(nq, np.inf, np.float32), 0, 128, N=N, cap=1 << 16)
                    rc = 0
                except vs.VsbError as e:
                    rc = e.rc
                assert rc == (0 if ok else vs.api.EINVAL), (vtype, metric, N, rc)
        ix.close()


# ---------------------------------------------------------------------------------------------- (h) row norms
@pytest.mark.parametrize("vtype,dim", [(po.I8, 16), (po.I8, 100), (po.I8, 4096), (po.U8, 16), (po.U8, 100), (po.U8, 4096), (po.U8, 33040)])
def test_row_norms_int_exact(vtype, dim):
    rng = np.random.Generator(np.random.PCG64(100 + dim + vtype))
    n = 512 if dim > 4096 else 2048
    x = _int_data(vtype, n, dim, rng)
    x[-1] = -128 if vtype == po.I8 else 255
    ix = _index(vtype, x)
    res = ix.debug_tc_level(po.DOT, _int_data(vtype, 16, dim, rng), np.full(16, -np.inf, np.float32), 0, n)
    got = res["norms"].view(np.uint32).astype(np.int64) if vtype == po.U8 else res["norms"].astype(np.int64)
    want = (x.astype(np.int64) ** 2).sum(1)
    if dim == 33040:
        assert want[1] > 2 ** 31
    bad = np.flatnonzero(got != want)
    assert bad.size == 0, (NAMES[vtype], dim, bad[:5].tolist(), got[bad[:5]].tolist(), want[bad[:5]].tolist())
    ix.close()


@pytest.mark.parametrize("family", fam.FAMILIES)
@pytest.mark.parametrize("vtype", [po.F16, po.BF16])
def test_row_norms_fp_within_bound(vtype, family):
    """row_norm_kernel: lane l sums chunks l, l + 32, ... (8 elements each) in one FMA chain, then five butterflies: a term
    passes through at most ceil(nc / 32) * 8 + 5 roundings"""
    rng = np.random.Generator(np.random.PCG64(110 + vtype + fam.FAMILIES.index(family)))
    for dim in (8, 100, 771, 4096):
        n = 1024
        x = fam.make(family, vtype, n, dim, rng)
        ix = _index(vtype, x)
        res = ix.debug_tc_level(po.DOT, fam.make(family, vtype, 16, dim, rng), np.full(16, -np.inf, np.float32), 0, n)
        xr = fam.decode(vtype, x)
        want = (xr * xr).sum(1)
        nc = (dim * 2 + 15) // 16
        bound = 1.001 * (-(-nc // 32) * 8 + 6) * 2.0 ** -24 * want
        got = res["norms"].astype(np.float64)
        bad = np.flatnonzero(np.abs(got - want) > bound)
        assert bad.size == 0, (NAMES[vtype], family, dim, bad[:5].tolist(), got[bad[:5]].tolist(), want[bad[:5]].tolist())
        ix.close()
