"""Host restatement of the scan pipeline (scan_kernel / scan_pass_kernel, filter_kernel): the stream row ranges, each stream's
candidate log, the filter's thresholds, the adaptive partition's update rule, exact integer distances, and the options that
force a plan shape.  Shared by tests/test_gpu_scan_kernel.py and tests/test_gpu_pass_kernel.py."""
import contextlib
import heapq
import math

import numpy as np

from oracle import pyoracle as po

WARPS = 8                      # scan streams per CTA (kWarps)
FILTER_SEGMENTS = 8            # kSegments
OUTCAP = 1 << 16               # survivor capacity per query (kOutCap)
FLT_EPS = float(np.finfo(np.float32).eps)
INF = math.inf


def _eng():
    import sqlite_vector_b200 as vs
    return vs.load_engine()


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
