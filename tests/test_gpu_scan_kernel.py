"""The single-query scan pipeline on its own: scan_kernel (distances, per-stream candidate logs), filter_kernel (prefix
thresholds, adaptive row partition) and the host's slot replay.  References are numpy float64 / int64, and the oracle where the
reference's own arithmetic is the question.  -m gpu.

(1) integer distances are bit-exact for every plan shape (lanes per row P = 1..32, ring depth, DIRECT) that the options can
    force, at row counts around the stream and tile boundaries, and at dims whose sums pass 2^24 and 2^31;
(2) fp distances stay within the error bound of the kernel's order of summation, on every input family of tests/fpfamilies.py;
(3) scan_candidates returns exactly the survivors of a host restatement of the stream logs and the filter's thresholds;
(4) planted row partitions (vsb_debug_write) keep (3) and the top-k exact, and the filter's partition update is the damped rule;
(5) rows whose fp32 sum of squares overflows get the reference's (double) value on both the single-query and the batch path."""
import contextlib
import heapq
import json
import math
import os

import numpy as np
import pytest

from oracle import pyoracle as po
from tests import fpfamilies as fam

pytestmark = pytest.mark.gpu

WARPS = 8                      # scan streams per CTA (kWarps)
FILTER_SEGMENTS = 8            # kSegments
OUTCAP = 1 << 16               # survivor capacity per query (kOutCap)
FLT_EPS = float(np.finfo(np.float32).eps)
U = 2.0 ** -24
INF = math.inf
ALL_METRICS = [po.L2, po.L2SQ, po.COS, po.DOT, po.L1]


def _eng():
    import sqlite_vector_b200 as vs
    return vs.load_engine()


def _index(vtype, x):
    import sqlite_vector_b200 as vs
    ix = vs.Index(vtype, x.shape[1], x.shape[0])
    ix.append_dense(x)
    ix.finalize()
    return ix


@contextlib.contextmanager
def _options(**kw):
    eng = _eng()
    old = {k: eng.set_option(k, v) for k, v in kw.items()}
    try:
        yield
    finally:
        for k, v in old.items():
            eng.set_option(k, v)


def _plan_options(pitch, log2p=None, nsw=None, direct=False):
    """options that force a plan of make_plan (engine.cu) for a scan without top-k (no shared memory kept for the filter)"""
    if direct:
        return dict(direct=1, stage_bytes=16384, ring_bytes=0)
    wtile = (32 >> log2p) * pitch
    return dict(direct=0, stage_bytes=wtile, ring_bytes=WARPS * nsw * wtile if nsw else 0)


def _plan(ix):
    return ix.stat("plan_log2p"), ix.stat("plan_nsw"), ix.stat("plan_direct")


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def _clamp32(d):
    d = np.asarray(d, dtype=np.float32).copy()
    d[np.abs(d) <= np.float32(8 * FLT_EPS)] = np.float32(0)
    return d


# ---------------------------------------------------------------------------------------------- (1) integer distances
def _int_data(vtype, n, dim, rng):
    if vtype == po.I8:
        x = rng.integers(-128, 128, (n, dim)).astype(np.int8)
        x[1::17] = -128                                    # all -128 rows
    else:
        x = rng.integers(0, 256, (n, dim)).astype(np.uint8)
        x[1::17] = 255                                     # all 255 rows
    x[::23] = 0                                            # zero rows: the cosine's zero-norm branch
    return x


def _int_expected(vtype, metric, x, q):
    """what finalize() makes of the exact integer sums: float of the exact int, sqrt_rn; cosine in fp32 in the kernel's order"""
    x64, q64 = x.astype(np.int64), q.astype(np.int64)
    if metric == po.L1:
        d = np.abs(x64 - q64[None, :]).sum(1).astype(np.float32)
    elif metric == po.DOT:
        d = -((x64 @ q64).astype(np.float32))
    elif metric in (po.L2, po.L2SQ):
        s = ((x64 - q64[None, :]) ** 2).sum(1)
        d = s.astype(np.float32)
        if metric == po.L2:
            d = np.sqrt(d)
    else:
        dot, nr, nq = x64 @ q64, (x64 * x64).sum(1), int((q64 * q64).sum())
        fq = np.float32(nq)
        fr, fd = nr.astype(np.float32), dot.astype(np.float32)
        with np.errstate(divide="ignore", invalid="ignore"):
            c = np.float32(1.0) - fd / (np.sqrt(fq) * np.sqrt(fr))
        d = np.where((nr == 0) | (nq == 0), np.float32(1.0), c).astype(np.float32)
    return _clamp32(d)


def _int_references(oracle, vtype, x, queries):
    """{(query, metric): exact distances}, each also checked against the oracle's int_exact arithmetic bit for bit"""
    out = {}
    for i, q in enumerate(queries):
        for metric in ALL_METRICS:
            want = _int_expected(vtype, metric, x, q)
            ref = oracle.distances_all(metric, vtype, q, x, int_exact=True)
            assert np.array_equal(_bits(want), _bits(ref)), (po.METRIC_NAMES[metric], "host != oracle", np.flatnonzero(_bits(want) != _bits(ref))[:5])
            out[i, metric] = want
    return out


def _check_int(ix, queries, refs, n, ctx):
    for i, q in enumerate(queries):
        for metric in ALL_METRICS:
            got = ix.scan_all(metric, q)
            want = refs[i, metric][:n]
            bad = np.flatnonzero(_bits(got) != _bits(want))
            assert bad.size == 0, (ctx, po.METRIC_NAMES[metric], "rows", bad[:5].tolist(), got[bad[:5]].tolist(), want[bad[:5]].tolist())


def _sweep_plans(nc, pitch):
    """(log2P, nsw, direct) shapes that fit shared memory at this pitch: 2 .. 8 stages of (32 / P) rows per warp"""
    shapes = []
    for log2p in range(6):
        wtile = (32 >> log2p) * pitch
        if WARPS * 8 * wtile <= 200 * 1024:
            shapes.append((log2p, 8, False))
        elif WARPS * 2 * wtile <= 200 * 1024:
            shapes.append((log2p, 2, False))
    log2p = min(s[0] for s in shapes if s[1] == 8)          # ring depths 2 and 3 at the widest tile that takes 8
    shapes += [(log2p, 2, False), (log2p, 3, False), (5, 1, True)]
    return shapes


@pytest.mark.parametrize("dim", [100, 1000])
@pytest.mark.parametrize("vtype", [po.U8, po.I8])
def test_int_plan_sweep_bit_exact(oracle, vtype, dim):
    """dims 100 / 1000: 7 / 63 chunks per row, never a multiple of P > 1 (nc = 7 < P: lanes that own no chunk at all)."""
    rng = np.random.Generator(np.random.PCG64(70 + dim + vtype))
    import sqlite_vector_b200 as vs
    sms = vs.Index(vtype, dim, 1).stat("sms")
    pitch = (dim + 15) // 16 * 16
    nc = pitch // 16
    big = WARPS * sms * 32 * 2 + 77                         # every stream walks several 32-row tiles
    xs = _int_data(vtype, big, dim, rng)
    queries = [_int_data(vtype, 1, dim, rng)[0], np.full(dim, -128 if vtype == po.I8 else 255, dtype=xs.dtype)]
    refs = _int_references(oracle, vtype, xs, queries)
    for n in (1, WARPS * sms // 2 + 3, 3 * 32 + 5, big):    # one row; most streams empty; a ragged last tile; many tiles
        ix = _index(vtype, np.ascontiguousarray(xs[:n]))
        for log2p, nsw, direct in _sweep_plans(nc, pitch):
            with _options(**_plan_options(pitch, log2p, nsw, direct)):
                _check_int(ix, queries, refs, n, (n, log2p, nsw, direct))
                assert _plan(ix) == (log2p, nsw, int(direct)), ("forced plan did not run", (log2p, nsw, direct), _plan(ix))
        ix.close()


@pytest.mark.parametrize("vtype,dim", [(po.U8, 1536), (po.I8, 1536), (po.U8, 4096), (po.I8, 4096), (po.U8, 20000), (po.I8, 20000),
                                       (po.U8, 33000), (po.I8, 33000)])
def test_int_large_dims_bit_exact(oracle, vtype, dim):
    """sums beyond 2^24 (the GPU gives the exact integer converted once, like the reference's AVX2 kernels, not the scalar
    kernel's float accumulation); uint8 dim 33000: |q|^2 + |r|^2 passes 2^31, so finalize's L2 formula wraps in uint32 and
    must still give the exact difference (which stays below 2^31)."""
    rng = np.random.Generator(np.random.PCG64(dim * 7 + vtype))
    n = 3 * 1024 + 9 if dim <= 4096 else 700
    x = _int_data(vtype, n, dim, rng)
    hi = -128 if vtype == po.I8 else 255
    lo = 127 if vtype == po.I8 else 0
    queries = [np.full(dim, lo, dtype=x.dtype), np.full(dim, hi, dtype=x.dtype), _int_data(vtype, 1, dim, rng)[0]]
    x[2] = hi
    x[3] = lo
    ix = _index(vtype, x)
    _check_int(ix, queries, _int_references(oracle, vtype, x, queries), n, dim)
    log2p, nsw, direct = _plan(ix)
    assert (direct == 1) == (log2p == 5 and nsw == 1) and (direct == 1 or nsw >= 2), _plan(ix)
    ix.close()


# ---------------------------------------------------------------------------------------------- (2) fp error bound
def _chain_len(nc, log2p, esz):
    """roundings a term of the scan's sum passes through: ceil(nc / P) chunks of E = 16 / esz elements on a lane, split over two
    FFMA chains (E / 2 each per chunk), log2 P butterfly additions, and s0 + s1"""
    P = 1 << log2p
    E = 16 // esz
    return -(-nc // P) * E // 2 + log2p + 1


def _fp_bound_and_exact(metric, vtype, xr, qv, nc, log2p, q_lanes=32):
    """float64 exact distances and the bound |d_gpu - d| <= bound, from the kernel's order of summation.

    Sums S = sum t_i (DOT: x_i y_i; L2SQ: (x_i - y_i)^2; L1: |x_i - y_i|): every term passes through at most L roundings of
    the accumulation (_chain_len) and, for L2SQ / L1, up to 2 more of forming it (the difference, the square), so
        |S_gpu - S| <= (L + 2) 2^-24 sum |t_i|          (first order; the factor 1.001 below covers the rest).
    L2 = sqrt(S):  |sqrt(S') - sqrt(S)| <= min(sqrt(E_S), E_S / sqrt(S)), plus the sqrt's own rounding 2^-24 sqrt(S').
    COSINE = 1 - s / (sqrt(qq) sqrt(ny)): s has E_s as above; the row norm ny is ONE chain per lane (L_n = ceil(nc/P) E +
    log2 P + 1 roundings), the query norm is lane-strided over q_lanes lanes (L_q = ceil(nc/q_lanes) E + log2 q_lanes + 1:
    32 lanes in the scan kernel, the refine's 8); with c = s / (|q||r|)
        |c' - c| <= E_s / (|q||r|) + |c| (E_qq / 2qq + E_ny / 2ny + 4 * 2^-24),  then 1 - c' adds 2^-24 |d|."""
    esz = po.ELEM_SIZE[vtype]
    E = 16 // esz
    L = _chain_len(nc, log2p, esz)
    if metric == po.DOT:
        t = xr * qv[None, :]
        S = t.sum(1)
        return -S, 1.001 * (L + 2) * U * np.abs(t).sum(1)
    if metric in (po.L2, po.L2SQ, po.L1):
        diff = np.abs(xr - qv[None, :])
        t = diff if metric == po.L1 else diff * diff
        S = t.sum(1)
        ES = 1.001 * (L + 2) * U * t.sum(1)
        if metric != po.L2:
            return S, ES
        r = np.sqrt(S)
        with np.errstate(divide="ignore", invalid="ignore"):
            lin = np.where(r > 0, ES / np.where(r > 0, r, 1.0), np.inf)
        return r, np.minimum(np.sqrt(ES), lin) + 1.001 * U * (r + np.sqrt(ES))
    # cosine
    P = 1 << log2p
    s = xr @ qv
    Es = 1.001 * (L + 2) * U * np.abs(xr * qv[None, :]).sum(1)
    ny = (xr * xr).sum(1)
    qq = float(qv @ qv)
    Eny = 1.001 * (-(-nc // P) * E + log2p + 2) * U * ny
    Eqq = 1.001 * (-(-nc // q_lanes) * E + q_lanes.bit_length()) * U * qq
    den = np.sqrt(ny * qq)
    zero = (ny == 0) | (qq == 0)
    with np.errstate(divide="ignore", invalid="ignore"):
        c = np.where(zero, 0.0, s / np.where(zero, 1.0, den))
        if vtype == po.F16:
            c = np.clip(c, -1.0, 1.0)
        rq = Eqq / qq if qq > 0 else 0.0
        rn = np.where(ny > 0, Eny / np.where(ny > 0, ny, 1.0), 0.0)
        b = Es / np.where(zero, 1.0, den) + np.abs(c) * (rq / 2 + rn / 2 + 4 * U) + U * np.abs(1.0 - c) + 4 * U * np.abs(c) * (rq + rn)
    d = np.where(zero, 1.0, 1.0 - c)
    return d, np.where(zero, 0.0, 1.001 * b)


def _assert_within(got, d, bound, ctx):
    """the nearly-zero clamp applies to the exact value; where |d| lies within the bound of 8 FLT_EPSILON either side is fine"""
    got = got.astype(np.float64)
    thr = 8 * FLT_EPS
    near = np.abs(np.abs(d) - thr) <= bound
    want = np.where(np.abs(d) <= thr, 0.0, d)
    ok = np.abs(got - want) <= bound
    ok |= near & ((got == 0.0) | (np.abs(got - d) <= bound))
    bad = np.flatnonzero(~ok)
    assert bad.size == 0, (ctx, "rows", bad[:5].tolist(), got[bad[:5]].tolist(), d[bad[:5]].tolist(), bound[bad[:5]].tolist())
    nz = bound > 0
    return float(np.max(np.abs(got - want)[nz] / bound[nz])) if nz.any() else 0.0


def _report(rec):
    path = os.environ.get("VSB_SCAN_ERR_REPORT")
    if path:
        with open(path, "a") as f:
            f.write(json.dumps(rec) + "\n")


@pytest.mark.parametrize("family", fam.FAMILIES)
@pytest.mark.parametrize("vtype", [po.F32, po.F16, po.BF16])
def test_fp_error_bound_every_plan(vtype, family):
    """pitch 48 B (3 chunks: P = 1 .. 32 all stage) and 1552 B (97 chunks; P >= 4 stage, plus DIRECT), every metric"""
    rng = np.random.Generator(np.random.PCG64(900 + vtype * 10 + fam.FAMILIES.index(family)))
    esz = po.ELEM_SIZE[vtype]
    for pitch in (48, 1552):
        dim = pitch // esz
        nc = pitch // 16
        n = 2000
        x = fam.make(family, vtype, n, dim, rng)
        qs = fam.make(family, vtype, 3, dim, rng, queries=True)
        xr = fam.decode(vtype, x)
        ix = _index(vtype, x)
        shapes = [(l, 2, False) for l in range(6) if WARPS * 2 * (32 >> l) * pitch <= 200 * 1024] + [(5, 1, True)]
        for log2p, nsw, direct in shapes:
            with _options(**_plan_options(pitch, log2p, nsw, direct)):
                for qi in (1, 2):
                    qv = fam.decode(vtype, qs[qi][None, :])[0]
                    for metric in ALL_METRICS:
                        got = ix.scan_all(metric, qs[qi])
                        d, bound = _fp_bound_and_exact(metric, vtype, xr, qv, nc, log2p)
                        ctx = (po.TYPE_NAMES[vtype], family, po.METRIC_NAMES[metric], pitch, log2p, direct)
                        ratio = _assert_within(got, d, bound, ctx)
                        _report({"type": po.TYPE_NAMES[vtype], "family": family, "metric": po.METRIC_NAMES[metric], "pitch": pitch,
                                 "P": 1 << log2p, "direct": direct, "ratio": ratio})
                assert _plan(ix) == (log2p, nsw, int(direct))
        ix.close()


# ---------------------------------------------------------------------------------------------- (3) survivor sets
def _streams(n, rpw, sms, bounds=None):
    """row ranges of the 8 * sms streams (scan_kernel): CTA c owns tiles bounds[c] .. bounds[c+1] (equal shares without a
    partition), warp w the w-th eighth of them"""
    T = -(-n // rpw)
    b = bounds if bounds is not None else [(T * c) // sms for c in range(sms + 1)]
    out = []
    for c in range(sms):
        c0, c1 = int(b[c]), int(b[c + 1])
        for w in range(WARPS):
            t0, t1 = c0 + ((c1 - c0) * w) // WARPS, c0 + ((c1 - c0) * (w + 1)) // WARPS
            out.append((min(t0 * rpw, n), min(t1 * rpw, n)))
    return out


def _kth(vals, k):
    return vals[k - 1] if len(vals) >= k else INF


def _merge(a, b, k):
    return heapq.nsmallest(k, a + b)


def _host_survivors(d, k, streams, logcap):
    """(survivor rows in scan order, overflow): the stream logs (rows that beat the running k-th value of their stream,
    strict <), then the filter's threshold min(in-CTA prefix, in-segment prefix, earlier segments) (k <= 32) or min(in-segment
    prefix, earlier segments) over the streams (k > 32)"""
    dl = d.tolist()
    logs, lists, overflow = [], [], False
    for r0, r1 in streams:
        h, lg = [], []
        for r in range(r0, r1):
            v = dl[r]
            thr = -h[0] if len(h) == k else INF
            if v < thr:
                lg.append(r)
                if len(h) < k:
                    heapq.heappush(h, -v)
                else:
                    heapq.heapreplace(h, -v)
        overflow |= len(lg) > logcap
        logs.append(lg[:logcap])
        lists.append(sorted(-v for v in h))
    S = len(streams)
    T = [INF] * S
    if k <= 32:
        ncta = S // WARPS
        GC = -(-ncta // FILTER_SEGMENTS)
        cta_lists = []
        for c in range(ncta):
            acc = []
            for w in range(WARPS):
                T[c * WARPS + w] = _kth(acc, k)
                acc = _merge(acc, lists[c * WARPS + w], k)
            cta_lists.append(acc)
        tseg, acc = [], []
        for c in range(ncta):
            if c % GC == 0:
                tseg.append(_kth(acc, k))
                seg = []
            tcta = _kth(seg, k)
            for w in range(WARPS):
                T[c * WARPS + w] = min(T[c * WARPS + w], tcta, tseg[c // GC])
            seg = _merge(seg, cta_lists[c], k)
            acc = _merge(acc, cta_lists[c], k)
    else:
        G = -(-S // FILTER_SEGMENTS)
        acc = []
        for s in range(S):
            if s % G == 0:
                tseg = _kth(acc, k)
                seg = []
            T[s] = min(_kth(seg, k), tseg)
            seg = _merge(seg, lists[s], k)
            acc = _merge(acc, lists[s], k)
    surv = [r for s in range(S) for r in logs[s] if dl[r] < T[s]]
    return surv, overflow or len(surv) > OUTCAP


def _check_candidates(ix, metric, q, k, d_all, bounds=None, ctx=()):
    """scan_candidates == the host's survivors of the same distances (rows, distances, scan order); fallbacks move exactly
    when the host predicts a log or output overflow.  The workspace's log capacity is max(256, 12 k) of the largest k it
    was sized for: callers run their k in ascending order (vsb_debug_write sizes it for k = 32)."""
    sms = ix.stat("sms")
    plan_all = _plan(ix)
    fb0 = ix.stat("fallbacks")
    (c,) = ix.scan_candidates(metric, q, k, cap=max(len(d_all), OUTCAP) + 1)
    fell = ix.stat("fallbacks") - fb0
    if not fell:
        assert _plan(ix)[0] == plan_all[0] and _plan(ix)[2] == plan_all[2], (ctx, "top-k plan differs in P / DIRECT", plan_all, _plan(ix))
    rpw = 32 >> plan_all[0]
    surv, overflow = _host_survivors(d_all, k, _streams(len(d_all), rpw, sms, bounds), max(256, 12 * max(k, 32 if bounds is not None else k)))
    assert fell == int(overflow), (ctx, k, "fallbacks", fell, "host predicts overflow", overflow)
    rows = np.arange(len(d_all)) if overflow else np.asarray(surv, dtype=np.int64)
    assert np.array_equal(c["seq"], rows), (ctx, k, len(c), len(rows), c["seq"][:10].tolist(), rows[:10].tolist())
    assert np.array_equal(_bits(c["dist"]), _bits(d_all[rows])), (ctx, k)
    return c


def _tie_heavy(n, rng):
    x = rng.integers(0, 3, (n, 16)).astype(np.uint8)       # L1 to the zero query: 33 distinct distances
    return x


def _descending(n, rng):
    """random rows, with runs in which the distance to the zero query strictly falls: every row of such a run is logged, so a
    stream inside one logs more than max(256, 12 k) entries for small k"""
    x = rng.integers(0, 256, (n, 16)).astype(np.uint8)
    for start, length in ((n // 3, 700), (n // 2 + 11, 300), (n - 400, 390)):
        s = np.arange(length)[::-1] + 10                   # L1 sums length + 9 .. 10, descending
        x[start:start + length] = 0
        for j in range(16):                                # spread the sum over the bytes (<= 255 each)
            x[start:start + length, j] = np.minimum(255, np.maximum(0, s - 255 * j)).astype(np.uint8)
    return x


@pytest.mark.parametrize("data", ["ties", "descending"])
def test_candidates_equal_host_survivors(oracle, data):
    rng = np.random.Generator(np.random.PCG64(55 if data == "ties" else 56))
    import sqlite_vector_b200 as vs
    sms = vs.Index(po.U8, 16, 1).stat("sms")
    n = WARPS * sms * 280 + 123                             # ~280 rows per stream (> 256: a descending stream overflows at k <= 7)
    x = _tie_heavy(n, rng) if data == "ties" else _descending(n, rng)
    ix = _index(po.U8, x)
    q0 = np.zeros(16, dtype=np.uint8)
    q1 = rng.integers(0, 3, 16).astype(np.uint8)
    rowids = np.arange(1, n + 1, dtype=np.int64)
    cases = [(po.L1, q0), (po.L2SQ, q1), (po.DOT, q1)]
    with _options(balance=0):
        d_alls = [ix.scan_all(metric, q) for metric, q in cases]
        for k in (1, 7, 32, 33, 100, 256):                  # ascending: the log capacity max(256, 12 k) is this k's
            for (metric, q), d_all in zip(cases, d_alls):
                c = _check_candidates(ix, metric, q, k, d_all, ctx=(data, po.METRIC_NAMES[metric]))
                ids, dist, _ = _eng().replay_topk(c, k)
                want_ids, want_d = oracle.topk_from_distances(d_all, rowids, k)
                assert np.array_equal(ids, want_ids) and np.array_equal(dist, want_d), (data, metric, k)
    ix.close()


# ---------------------------------------------------------------------------------------------- (4) planted partitions
def _planted(kind, T, sms, rng):
    b = np.zeros(sms + 1, dtype=np.int64)
    if kind == "one_cta_90pct":
        sizes = np.full(sms, (T - T * 9 // 10) // (sms - 1), dtype=np.int64)
        sizes[5] = 0
        sizes[5] = T - sizes.sum()
    elif kind == "zero_front_middle_end":
        sizes = np.zeros(sms, dtype=np.int64)
        live = np.setdiff1d(np.arange(sms), [0, 1, sms // 2, sms // 2 + 1, sms // 2 + 7, sms - 2, sms - 1])
        sizes[live] = T // len(live)
        sizes[live[-1]] += T - sizes.sum()
    elif kind == "one_to_seven":
        sizes = (np.arange(sms) % 7 + 1).astype(np.int64)   # fewer tiles than warps: some warps own no rows
        sizes[sms // 3] += T - sizes.sum()
    else:                                                   # random sizes, mostly not multiples of 8
        w = rng.random(sms) + 0.05
        sizes = np.floor(w / w.sum() * T).astype(np.int64)
        sizes[-1] += T - sizes.sum()
    b[1:] = np.cumsum(sizes)
    assert b[-1] == T and np.all(np.diff(b) >= 0)
    return b


def _partition_index(rng):
    """uint8 dim 16 (one 16-byte chunk); stage_bytes 16 forces P = 32, one row per tile: the partition is used from 64 tiles
    per CTA, i.e. n >= 64 * #SMs rows"""
    import sqlite_vector_b200 as vs
    sms = vs.Index(po.U8, 16, 1).stat("sms")
    n = 64 * sms + 1000
    x = rng.integers(0, 4, (n, 16)).astype(np.uint8)
    x[n // 2:n // 2 + 300] = np.repeat(np.arange(300)[::-1, None] // 20, 16, 1).astype(np.uint8)   # descending, tied steps
    return _index(po.U8, x), x, n, sms


@pytest.mark.parametrize("kind", ["one_cta_90pct", "zero_front_middle_end", "one_to_seven", "ragged"])
def test_planted_partition_survivors_and_topk(oracle, kind):
    rng = np.random.Generator(np.random.PCG64(["one_cta_90pct", "zero_front_middle_end", "one_to_seven", "ragged"].index(kind)))
    ix, x, n, sms = _partition_index(rng)
    q = rng.integers(0, 4, 16).astype(np.uint8)
    rowids = np.arange(1, n + 1, dtype=np.int64)
    with _options(stage_bytes=16, ring_bytes=0, direct=0, balance=1):
        b = _planted(kind, n, sms, rng)
        for metric in (po.L1, po.L2, po.DOT):
            d_all = ix.scan_all(metric, q)
            assert _plan(ix)[0] == 5 and _plan(ix)[2] == 0
            for k, mi in ((1, 0), (7, 3), (32, 31)):
                ix.debug_write("bounds", b)
                _check_candidates(ix, metric, q, k, d_all, bounds=b.tolist(), ctx=(kind, po.METRIC_NAMES[metric]))
                ix.debug_write("bounds", b)
                (res, mi_out) = ix.scan_topk(metric, q, k, max_index=mi)
                assert np.array_equal(ix.debug_read("bounds", np.int64, sms + 1), _expected_update(b, ix.debug_read("cta_time", np.uint32, sms), n))
                want = oracle.scan_dense(metric, po.U8, q, x, rowids, k, start_max_index=mi, int_exact=True)
                assert np.array_equal(res[0][0], want[0]) and np.array_equal(res[0][1], want[1]), (kind, metric, k, mi)
    ix.close()


def _expected_update(b_old, cta_time, T):
    """filter_kernel's partition update, restated: fp32 speeds, double accumulation in CTA order, round half up, at least one
    tile per warp, clamped to T; unchanged when a CTA had no tiles or reported no time"""
    ncta = len(cta_time)
    tiles = np.diff(b_old).astype(np.float32)
    t = np.maximum(cta_time.astype(np.uint32), np.uint32(1)).astype(np.float32)
    if np.any(cta_time == 0) or np.any(~(tiles > 0)):
        return b_old.copy()
    spd = (tiles / t).astype(np.float32)
    total = 0.0
    for v in spd.tolist():                                  # sequential (sum() would compensate)
        total += v
    out = b_old.copy()
    acc, prev = 0.0, 0
    for c in range(ncta):
        cur = float(int(b_old[c + 1]) - prev)
        want = float(T) * float(spd[c]) / total
        prev = int(b_old[c + 1])
        acc += 0.5 * cur + 0.5 * want
        v = T if c == ncta - 1 else int(math.floor(acc + 0.5))
        v = max(v, int(out[c]) + WARPS)
        out[c + 1] = min(v, T)
    return out


def test_partition_update_rule():
    rng = np.random.Generator(np.random.PCG64(77))
    ix, x, n, sms = _partition_index(rng)
    q = rng.integers(0, 4, 16).astype(np.uint8)
    with _options(stage_bytes=16, ring_bytes=0, direct=0, balance=1):
        for kind in ("one_cta_90pct", "ragged", "one_to_seven", "zero_front_middle_end"):
            b0 = _planted(kind, n, sms, rng)
            ix.debug_write("bounds", b0)
            ix.scan_topk(po.L2, q, 10)
            t = ix.debug_read("cta_time", np.uint32, sms)
            got = ix.debug_read("bounds", np.int64, sms + 1)
            want = _expected_update(b0, t, n)
            assert np.array_equal(got, want), (kind, np.flatnonzero(got != want)[:5].tolist())
            if kind == "zero_front_middle_end":
                assert np.array_equal(got, b0)              # a CTA without tiles: the partition is left alone
            else:
                assert not np.array_equal(got, b0)
        with pytest.raises(Exception, match="non-decreasing"):
            bad = _planted("ragged", n, sms, rng)
            bad[3], bad[4] = bad[4] + 1, bad[3]
            ix.debug_write("bounds", bad)
        with pytest.raises(Exception, match="from 0"):
            ix.debug_write("bounds", _planted("ragged", n - 1, sms, rng))
    ix.close()


# ---------------------------------------------------------------------------------------------- (5) large magnitudes
def _huge_setup(vtype, n, dim, seed):
    rng = np.random.Generator(np.random.PCG64(seed))
    x = fam.make("huge", vtype, n, dim, rng)
    q = fam.make("normal", vtype, 2, dim, rng)[1]
    return x, q


def _lassq_float(vtype, x, q, root):
    """(float) sqrt(sum d^2) in float64 with d the reference's fp32 element difference: the oracle's LASSQ value"""
    xr, qv = fam.decode(vtype, x), fam.decode(vtype, q[None, :])[0]
    d = (xr.astype(np.float32) - qv.astype(np.float32)[None, :]).astype(np.float64)
    s = (d * d).sum(1)
    with np.errstate(over="ignore"):
        return (np.sqrt(s) if root else s).astype(np.float32), s


@pytest.mark.parametrize("vtype,metric", [(po.BF16, po.L2), (po.BF16, po.L2SQ), (po.BF16, po.L1), (po.F32, po.L1)])
def test_huge_values_scan_all_and_topk(oracle, vtype, metric):
    """bf16 L2: the reference's double LASSQ stays finite for rows whose fp32 sum of squares overflows; so must we"""
    n, dim = 200, 64
    x, q = _huge_setup(vtype, n, dim, 31 + vtype + metric)
    ix = _index(vtype, x)
    ref = oracle.distances_all(metric, vtype, q, x)
    exact_rows = np.zeros(n, dtype=bool)
    if metric in (po.L2, po.L2SQ):
        want, s = _lassq_float(vtype, x, q, metric == po.L2)
        assert np.array_equal(_bits(want), _bits(ref))
        exact_rows = s > np.finfo(np.float32).max               # the fp32 sum overflowed: these rows take the exact path
        assert exact_rows.sum() >= 20
    for direct in (0, 1):
        with _options(direct=direct):
            got = ix.scan_all(metric, q)
        assert np.array_equal(np.isinf(got), np.isinf(ref)), (direct, np.flatnonzero(np.isinf(got) != np.isinf(ref))[:5].tolist())
        if metric == po.L2:
            assert np.isfinite(got).all()
        assert np.array_equal(_bits(got[exact_rows]), _bits(ref[exact_rows])), direct
        fin = np.isfinite(ref)
        assert np.allclose(got[fin], ref[fin], rtol=1e-5, atol=0), direct
    k = 256                                                     # k >= n: every row with a finite distance comes back
    (res,) = ix.scan_topk(metric, q, k)
    want_ids, want_d = oracle.scan_dense(metric, vtype, q, x, np.arange(1, n + 1, dtype=np.int64), k)
    assert len(res[0]) == len(want_ids) == int(np.isfinite(ref).sum())
    assert set(res[0].tolist()) == set(want_ids.tolist())
    got_by_row = dict(zip(res[0].tolist(), res[1].tolist()))
    for r in np.flatnonzero(exact_rows & np.isfinite(ref)):                # (+Inf rows never enter the slots)
        assert got_by_row[r + 1] == float(ref[r]), r
    ix.close()


def test_huge_values_batch_path(oracle):
    """batch of 32 bf16 L2 queries: rows 0..127 (refined exhaustively) ordinary, every later row has an element of magnitude
    2^65 .. 2^124, so its fp32 norm overflows; the top-256 holds 128 of them.  Query 5 also carries a 2^70 element (its own norm
    overflows)."""
    from tests.fpcheck import assert_fp_topk
    rng = np.random.Generator(np.random.PCG64(404))
    n, dim, k, nq = 8192, 64, 256, 32
    xr = rng.standard_normal((n, dim))
    cols = rng.integers(0, dim, n)
    e = rng.integers(65, 125, n).astype(np.float64)
    xr[np.arange(n), cols] = np.where(rng.random(n) < 0.5, -1.0, 1.0) * (1.0 + rng.integers(0, 128, n) / 128.0) * np.exp2(e)
    xr[:128] = rng.standard_normal((128, dim))
    x = po.convert(xr.astype(np.float32), po.BF16)
    qr = rng.standard_normal((nq, dim))
    qr[5, 0] = 2.0 ** 70
    qs = po.convert(qr.astype(np.float32), po.BF16)
    ix = _index(po.BF16, x)
    b0, f0 = ix.stat("batches"), ix.stat("fallbacks")
    res = ix.scan_topk(po.L2, qs, k)
    assert ix.stat("batches") == b0 + 1 and ix.stat("fallbacks") == f0, "the batch path did not run to the end"
    rowids = np.arange(1, n + 1, dtype=np.int64)
    for j in range(nq):
        want_ids, want_d = oracle.scan_dense(po.L2, po.BF16, qs[j], x, rowids, k)
        ref = None

        def dist_of_row(r, j=j):
            nonlocal ref
            if ref is None:
                ref = oracle.distances_all(po.L2, po.BF16, qs[j], x)
            return ref[r - 1]
        assert_fp_topk(res[j][0], res[j][1], want_ids, want_d, po.L2, dist_of_row, ctx=("query", j))
    ix.close()
