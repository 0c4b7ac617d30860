"""The multi-query pass on its own: scan_pass_kernel's per-query k-lists, logs, in-CTA bounds and overflow flags, the filter
launch of each query, and the checks of a submission.  Each slot's survivors are read with vsb_debug_survivors (the pairs
vsb_collect replays, in scan order) and compared with the same query run alone and with the host restatement of
tests/scanref.py.  -m gpu.

"Lone" is a one-query group (scan_kernel) read with the same hook: pass_max keeps the plan of a pass that of one query, so
lone and pass see identical streams (balance = 0 throughout, except for the planted partitions).  Passes go to slots >= 1,
which no synchronous call stages into, and are read before any synchronous call.  Within an index k only grows: the log
capacity max(256, 12 k) of the workspace never shrinks, and the restatement must use the same capacity.

(1) survivor sets per query equal the lone ones and the restatement, every type and metric, k = 1 .. 256, widths 2 .. 8,
    partly filled and uneven passes, a group at first_slot 5;
(2) every plan shape (P = 1 .. 32, ring depths 2 / 3 / 8, DIRECT) at every width plan_pass_max admits;
(3) NaN / +-Inf rows and an infinite query element at m >= 1, staged, P >= 8 and DIRECT;
(4) planted partitions: survivors over the planted streams, and the partition updated once per pass;
(5) a per-query log overflow predicted to the entry, wherever the query sits in its pass, and the slot re-armed afterwards;
(6) 32 queries in flight over the rotating workspaces;
(7) submissions rejected before they are held or launched."""

import numpy as np
import pytest

from oracle import pyoracle as po
from tests import fpcheck
from tests import fpfamilies as fam
from tests.scanref import (WARPS, _bits, _descending, _eng, _expected_update, _host_survivors, _int_expected, _options,
                           _plan, _plan_options, _planted, _streams, _tie_heavy)

pytestmark = pytest.mark.gpu

ALL_METRICS = [po.L2, po.L2SQ, po.COS, po.DOT, po.L1]
KS = (1, 7, 32, 33, 100, 256)
LONE_SLOT = 20                 # lone queries go to slots 20 .. 31, passes to 1 .. 18


def _index(vtype, x):
    import sqlite_vector_b200 as vs
    ix = vs.Index(vtype, x.shape[1], x.shape[0])
    ix.append_dense(x)
    ix.finalize()
    return ix


def _sms():
    import sqlite_vector_b200 as vs
    return vs.Index(po.U8, 16, 1).stat("sms")


def _logcap(k):
    return max(256, 12 * k)


def _group(ix, metric, q, k, first_slot):
    """q[0:nq] as one group into slots first_slot ..; returns (pairs, flags) of every slot and the passes it launched"""
    q = np.ascontiguousarray(q)
    p0, c0 = ix.stat("scan_passes"), ix.stat("pass_queries")
    ix.scan_submit_group(metric, q, q.strides[0], len(q), k, False, first_slot, fetch=True)
    got = [ix.debug_survivors(first_slot + j) for j in range(len(q))]
    assert ix.stat("pass_queries") - c0 == len(q)
    return got, ix.stat("scan_passes") - p0


def _lone(ix, metric, q, k):
    out = []
    for j in range(len(q)):
        got, passes = _group(ix, metric, q[j:j + 1], k, LONE_SLOT + j % 12)
        assert passes == 1
        out.append(got[0])
    return out


def _same_pairs(a, b):
    return a[1] == b[1] and np.array_equal(a[0], b[0])


def _check_pass(ix, metric, q, k, first_slot, lone, ctx):
    """q as one group: every query's survivors (rows, distance bits, order, flags) are its lone ones; the passes are those of
    the width that ran"""
    got, passes = _group(ix, metric, q, k, first_slot)
    width = ix.stat("plan_pass_max")
    assert passes == -(-len(q) // width), (ctx, len(q), width, passes)
    for j in range(len(q)):
        assert _same_pairs(got[j], lone[j]), (ctx, "query", j, "of", len(q), got[j][0].shape, lone[j][0].shape, got[j][1], lone[j][1])
    return width


def _check_host(pairs_flags, d, k, streams, logcap, ctx, host=None):
    """a slot's survivors == the restatement over these streams (host: its result, if already computed); flags exactly
    where it predicts an overflow"""
    pairs, flags = pairs_flags
    surv, overflow = host if host is not None else _host_survivors(d, k, streams, logcap)
    assert bool(flags) == overflow, (ctx, "flags", flags, "host predicts overflow", overflow)
    if not overflow:
        rows = np.asarray(surv, dtype=np.int64)
        assert np.array_equal(pairs[:, 1].astype(np.int64), rows), (ctx, len(pairs), len(rows), pairs[:8, 1].tolist(), rows[:8].tolist())
        assert np.array_equal(pairs[:, 0], _bits(d[rows])), ctx
    return overflow


# ---------------------------------------------------------------------------------------------- (1) survivor sets per query
def _data(kind, n, rng):
    """(vtype, column, 13 queries)"""
    if kind in ("ties", "descending"):
        x = _tie_heavy(n, rng) if kind == "ties" else _descending(n, rng)
        q = rng.integers(0, 3, (13, 16)).astype(np.uint8)
        q[0] = 0                                             # the zero query: the descending runs overflow its logs at small k
        q[5] = 0
        return po.U8, x, q
    if kind == "int8":
        return po.I8, rng.integers(-128, 128, (n, 24)).astype(np.int8), rng.integers(-128, 128, (13, 24)).astype(np.int8)
    vtype, dim = {"f32": (po.F32, 12), "f16": (po.F16, 20), "bf16": (po.BF16, 24)}[kind]
    return (vtype, po.convert(rng.standard_normal((n, dim), dtype=np.float32), vtype),
            po.convert(rng.standard_normal((13, dim), dtype=np.float32), vtype))


@pytest.mark.parametrize("kind", ["ties", "descending", "int8", "f32", "f16", "bf16"])
def test_pass_survivors_equal_lone_and_host(kind):
    rng = np.random.Generator(np.random.PCG64(["ties", "descending", "int8", "f32", "f16", "bf16"].index(kind) + 300))
    sms = _sms()
    n = WARPS * sms * 280 + 123                              # ~280 rows per stream: a descending stream overflows at k <= 7
    vtype, x, q = _data(kind, n, rng)
    ix = _index(vtype, x)
    widths = set()
    with _options(balance=0):
        d_alls = [[ix.scan_all(metric, q[j]) for j in range(13)] for metric in ALL_METRICS]
        for ki, k in enumerate(KS):                          # ascending: the log capacity max(256, 12 k) is this k's
            for mi, metric in enumerate(ALL_METRICS):
                d_all = d_alls[mi]
                ctx = (kind, po.METRIC_NAMES[metric], k)
                lone = _lone(ix, metric, q, k)
                rpw = 32 >> _plan(ix)[0]
                j = 1 + (mi + ki) % 7                        # one query at m >= 1 restated per (metric, k)
                _check_host(lone[j], d_all[j], k, _streams(n, rpw, sms), _logcap(k), ctx + (j,))
                if kind == "descending" and k == 1 and metric == po.L1:
                    assert lone[0][1] != 0, "the zero query's log did not overflow"
                    _check_host(lone[0], d_all[0], k, _streams(n, rpw, sms), _logcap(k), ctx + (0,))
                for nq in (2, 3, 4, 5, 7, 8):
                    widths.add(_check_pass(ix, metric, q[:nq], k, 1, lone[:nq], ctx + (nq,)))
                assert _check_pass(ix, metric, q, k, 5, lone, ctx + (13,)) == 8    # 13 = 8 + 5, slots 5 .. 17
    assert widths == {8}, widths
    ix.close()


# ---------------------------------------------------------------------------------------------- (2) every plan shape, every width
def _shapes(pitch):
    """(log2P, nsw, direct) the options can force at this pitch, as in test_fp_error_bound_every_plan, plus ring depths 3 and 8"""
    shapes = [(l, 2, False) for l in range(6) if WARPS * 2 * (32 >> l) * pitch <= 200 * 1024]
    l8 = [l for l in range(6) if WARPS * 8 * (32 >> l) * pitch <= 200 * 1024]
    if l8:
        shapes += [(l8[0], 3, False), (l8[0], 8, False)]
    return shapes + [(5, 1, True)]


def _all_rows_expected(vtype, metric, x, q, ix):
    """every row's distance as the pass must give it: int64 numpy for the integer types, the lone scan_all for fp"""
    if vtype in (po.U8, po.I8):
        return _int_expected(vtype, metric, x, q)
    return ix.scan_all(metric, q)


@pytest.mark.parametrize("vtype", [po.U8, po.I8, po.F32, po.F16, po.BF16])
def test_every_plan_every_width(vtype):
    """n = 200 <= k = 256: every row with a finite distance survives, so each slot holds every such row's distance in scan
    order.  At pitch 48 B every P takes passes of 2, 4 and 8; at 1552 B (k = 200) the wider passes that do not fit beside the
    forced ring are named."""
    rng = np.random.Generator(np.random.PCG64(500 + vtype))
    esz = po.ELEM_SIZE[vtype]
    not_admitted = []
    for pitch, k in ((48, 256), (1552, 200)):
        dim = pitch // esz
        n = 200
        if vtype in (po.U8, po.I8):
            lo, hi = (-128, 128) if vtype == po.I8 else (0, 256)
            dt = np.int8 if vtype == po.I8 else np.uint8
            x, q = rng.integers(lo, hi, (n, dim)).astype(dt), rng.integers(lo, hi, (8, dim)).astype(dt)
            x[::23] = 0
        else:
            x = fam.make("normal", vtype, n, dim, rng)
            q = fam.make("normal", vtype, 8, dim, rng, queries=True)
        ix = _index(vtype, x)
        for log2p, nsw, direct in _shapes(pitch):
            shape = (pitch, 1 << log2p, nsw, direct)
            with _options(balance=0, **_plan_options(pitch, log2p, nsw, direct)):
                for metric in ALL_METRICS:
                    want = [_all_rows_expected(vtype, metric, x, q[j], ix) for j in range(8)]
                    lone = _lone(ix, metric, q, k)
                    if _plan(ix) != (log2p, nsw, int(direct)):
                        not_admitted.append((shape, "k = %d: the lone plan is %s" % (k, _plan(ix))))
                        break
                    for j in range(8):
                        fin = np.flatnonzero(np.isfinite(want[j]))
                        pairs, flags = lone[j]
                        assert flags == 0 and np.array_equal(pairs[:, 1], fin), (shape, metric, j)
                        assert np.array_equal(pairs[:, 0], _bits(want[j][fin])), (shape, po.METRIC_NAMES[metric], j)
                    w = ix.stat("plan_pass_max")
                    if pitch == 48:
                        assert w == 8, (shape, "plan_pass_max", w)
                    elif w < 8 and metric == po.L2:
                        not_admitted.append((shape, "k = %d: widths above %d change the plan (pass_max)" % (k, w)))
                    for nq in sorted({2, 3, 4, 5, 8} & set(range(2, w + 1))):
                        _check_pass(ix, metric, q[:nq], k, 1, lone[:nq], (shape, po.METRIC_NAMES[metric]))
                        assert _plan(ix) == (log2p, nsw, int(direct)), (shape, nq, _plan(ix))
        ix.close()
    assert all(s[0] == 1552 for s, _ in not_admitted), not_admitted
    print("shapes not admitting every width:", not_admitted)


@pytest.mark.parametrize("vtype", [po.U8, po.F16])
def test_every_plan_multi_tile(vtype):
    """several tiles per stream and a ragged last tile, at every plan shape of pitch 48 B, widths 2 .. 8, k = 33 (k > 32
    keeps no filter reserve, so the forced ring holds)"""
    rng = np.random.Generator(np.random.PCG64(600 + vtype))
    sms = _sms()
    dim = 48 // po.ELEM_SIZE[vtype]
    n = WARPS * sms * 100 + 77
    if vtype == po.U8:
        x, q = rng.integers(0, 256, (n, dim)).astype(np.uint8), rng.integers(0, 256, (8, dim)).astype(np.uint8)
    else:
        x, q = fam.make("normal", vtype, n, dim, rng), fam.make("normal", vtype, 8, dim, rng, queries=True)
    ix = _index(vtype, x)
    k = 33
    for si, (log2p, nsw, direct) in enumerate(_shapes(48)):
        with _options(balance=0, **_plan_options(48, log2p, nsw, direct)):
            metric = ALL_METRICS[si % 5]
            lone = _lone(ix, metric, q, k)
            assert _plan(ix) == (log2p, nsw, int(direct)), (log2p, nsw, direct, _plan(ix))
            j = 1 + si % 7
            _check_host(lone[j], ix.scan_all(metric, q[j]), k, _streams(n, 32 >> log2p, sms), _logcap(k), (log2p, nsw, direct, j))
            for nq in (2, 3, 4, 6, 8):
                _check_pass(ix, metric, q[:nq], k, 1, lone[:nq], (log2p, nsw, direct))
    ix.close()


# ---------------------------------------------------------------------------------------------- (3) special values
def _lanes_options(pitch, log2p, direct):
    """P (or DIRECT) forced, the ring left to make_plan: k <= 32 keeps the filter reserve, which a forced ring would not fit"""
    return dict(direct=int(direct), stage_bytes=(32 >> log2p) * pitch, ring_bytes=0)


def _assert_topk(oracle, vtype, metric, x, q, ids, d, k, ctx):
    """the oracle's top-k: infinite distances (DOT against an infinite element) exactly, the finite ones by tests/fpcheck.py"""
    want_ids, want_d = oracle.scan_dense(metric, vtype, q, x, np.arange(1, len(x) + 1, dtype=np.int64), k)
    assert len(ids) == len(want_ids), ctx
    inf = ~np.isfinite(want_d)
    assert np.array_equal(d[inf], want_d[inf]) and np.array_equal(ids[inf], want_ids[inf]), ctx
    fpcheck.assert_fp_topk(ids[~inf], d[~inf], want_ids[~inf], want_d[~inf], metric,
                           lambda r: oracle.distance(metric, vtype, q, x[r - 1]), ctx)


def _special(vtype, family, n, dim, rng):
    x = fam.make(family, vtype, n, dim, rng)
    q = fam.make("normal", vtype, 8, dim, rng, queries=True)
    NAN, PINF, NINF = (0x7E00, 0x7C00, 0xFC00) if vtype == po.F16 else (0x7FC0, 0x7F80, 0xFF80)
    for r in range(0, n, 97):
        x[r, r % dim] = (NAN, PINF, NINF)[r % 3]
    x[11, 4] = PINF
    x[11, 9] = NINF
    q[1, 3] = PINF                                           # an infinite element in queries at m >= 1
    q[6, 0] = NINF
    return x, q


@pytest.mark.parametrize("vtype,family,metrics", [(po.F16, "normal", ALL_METRICS), (po.BF16, "huge", [po.L2])])
def test_special_values_every_path(oracle, vtype, family, metrics):
    """f16: NaN / Inf rows and queries take special_row_distance; bf16 "huge": rows whose fp32 sum of squares overflows do.
    Staged P = 1, staged P = 8 and DIRECT, passes of 2 and 8."""
    rng = np.random.Generator(np.random.PCG64(700 + vtype))
    n, dim = 3000, 24
    x, q = _special(vtype, family, n, dim, rng)
    ix = _index(vtype, x)
    for log2p, direct in ((0, False), (3, False), (5, True)):
        with _options(balance=0, **_lanes_options(48, log2p, direct)):
            for metric in metrics:
                for k in (5, 40):
                    lone = _lone(ix, metric, q, k)
                    assert _plan(ix)[0] == log2p and _plan(ix)[2] == int(direct), _plan(ix)
                    for nq in (2, 8):
                        ctx = (log2p, direct, po.METRIC_NAMES[metric], k, nq)
                        _check_pass(ix, metric, q[:nq], k, 1, lone[:nq], ctx)
                        for j in range(nq):
                            ids, d = ix.collect(1 + j, k)
                            _assert_topk(oracle, vtype, metric, x, q[j], ids, d, k, ctx + (j,))
    ix.close()


# ---------------------------------------------------------------------------------------------- (4) planted partitions
@pytest.mark.parametrize("kind", ["one_cta_90pct", "zero_front_middle_end", "one_to_seven", "ragged"])
def test_planted_partition_pass(kind):
    """uint8 dim 16 at P = 32 (one row per tile).  vsb_debug_write sizes the workspaces for one query; a wider pass would
    regrow them and drop the plant, so one pass of the full width runs first."""
    rng = np.random.Generator(np.random.PCG64(800 + ["one_cta_90pct", "zero_front_middle_end", "one_to_seven", "ragged"].index(kind)))
    sms = _sms()
    n = 64 * sms + 1000
    x = rng.integers(0, 4, (n, 16)).astype(np.uint8)
    x[n // 2:n // 2 + 300] = np.repeat(np.arange(300)[::-1, None] // 20, 16, 1).astype(np.uint8)
    q = rng.integers(0, 4, (8, 16)).astype(np.uint8)
    ix = _index(po.U8, x)
    equal = [(n * c) // sms for c in range(sms + 1)]
    with _options(stage_bytes=16, ring_bytes=0, direct=0, balance=1):
        for metric in (po.L1, po.L2, po.DOT):
            d_all = [ix.scan_all(metric, q[j]) for j in range(8)]
            for nq in (8, 3):
                _group(ix, metric, q[:nq], 32, 1)            # the workspaces at their full width for this pass
                for k in (1, 7, 32):
                    b = _planted(kind, n, sms, rng)
                    assert b.tolist() != equal
                    ix.debug_write("bounds", b)
                    got, passes = _group(ix, metric, q[:nq], k, 1)
                    assert passes == 1 and _plan(ix)[0] == 5
                    for j in range(nq):
                        _check_host(got[j], d_all[j], k, _streams(n, 1, sms, b.tolist()), _logcap(32), (kind, metric, nq, k, j))
                    t = ix.debug_read("cta_time", np.uint32, sms)
                    after = ix.debug_read("bounds", np.int64, sms + 1)
                    assert np.array_equal(after, _expected_update(b, t, n)), (kind, metric, nq, k, "partition not updated once")
    ix.close()


# ---------------------------------------------------------------------------------------------- (5) per-query log overflow
def _run_rows(sums):
    """uint8 dim-16 rows with these L1 sums to the zero query (each <= 16 * 255)"""
    s = np.asarray(sums, dtype=np.int64)
    base, rem = s // 16, s % 16
    return (base[:, None] + (np.arange(16)[None, :] < rem[:, None])).astype(np.uint8)


@pytest.mark.parametrize("delta", [-2, -1, 0, 1, 2])
def test_per_query_log_overflow(oracle, delta):
    """background rows at L1 sum 2048; stream A holds a falling run (for the zero query) and stream B a rising one (for the
    all-255 query), each of length logcap + delta - k after 16 background rows: the stream logs k + run = logcap + delta
    entries for that query and few for the other.  The flags, the asynchronous collect and the fallback follow exactly."""
    sms = _sms()
    k = 10
    logcap = _logcap(k)
    S = WARPS * sms
    n = S * 11 * 32 + 5
    streams = _streams(n, 32, sms)
    x = np.full((n, 16), 128, dtype=np.uint8)
    R = logcap + delta - k
    (a0, a1), (b0, b1) = streams[S // 3], streams[2 * S // 3]
    assert a1 - a0 >= 16 + R + 1 and b1 - b0 >= 16 + R + 1
    x[a0 + 16:a0 + 16 + R] = _run_rows(2000 - np.arange(R))                 # falls for the zero query, rises for all-255
    x[b0 + 16:b0 + 16 + R] = _run_rows(2100 + np.arange(R))                 # the opposite
    rng = np.random.Generator(np.random.PCG64(900 + delta))
    zero, full = np.zeros(16, np.uint8), np.full(16, 255, np.uint8)
    fill = rng.integers(110, 146, (8, 16)).astype(np.uint8)
    ix = _index(po.U8, x)
    rowids = np.arange(1, n + 1, dtype=np.int64)
    over = delta > 0
    with _options(balance=0, **_lanes_options(16, 0, False)):
        vec = {"zero": zero, "full": full, **{f"f{i}": fill[i] for i in range(8)}}
        d = {s: ix.scan_all(po.L1, v) for s, v in vec.items()}
        host = {s: _host_survivors(d[s], k, streams, logcap) for s in vec}
        want = {s: oracle.scan_dense(po.L1, po.U8, v, x, rowids, k, int_exact=True) for s, v in vec.items()}
        for s in ("zero", "full"):
            assert host[s][1] == over, (s, delta, "the restatement's count is not logcap + delta")
        passes = [["zero", "f0", "f1", "f2"],                              # first
                  ["f0", "f1", "zero", "f2", "f3"],                        # middle
                  ["f0", "f1", "f2", "full"],                              # last
                  ["f0", "f1", "full"],                                    # last of a partial pass (3 in M = 4)
                  ["zero", "f0", "full", "f1", "f2", "f3", "f4", "f5"],    # two in one pass
                  ["f2", "f3", "f4", "f5", "f6", "f7", "f0", "f1"]]        # clean, on the slots the overflows used
        for names in passes:
            qs = np.stack([vec[s] for s in names])
            got, _ = _group(ix, po.L1, qs, k, 1)
            assert _plan(ix)[0] == 0 and _plan(ix)[2] == 0
            for j, s in enumerate(names):
                o = _check_host(got[j], d[s], k, streams, logcap, (delta, names, j), host[s])
                assert o == (over and s in ("zero", "full")), (delta, names, j)
            for j, s in enumerate(names):
                want_ids, want_d = want[s]
                if got[j][1]:
                    with pytest.raises(Exception, match="overflow"):
                        ix.collect(1 + j, k)
                else:
                    ids, dist = ix.collect(1 + j, k)
                    assert np.array_equal(ids, want_ids) and np.array_equal(dist, want_d), (delta, names, j)
            for j, s in enumerate(names):                                  # synchronous calls only after the pass is read
                if got[j][1]:
                    f0 = ix.stat("fallbacks")
                    (res,) = ix.scan_topk(po.L1, vec[s], k)
                    assert ix.stat("fallbacks") - f0 == 1
                    want_ids, want_d = want[s]
                    assert np.array_equal(res[0], want_ids) and np.array_equal(res[1], want_d), (delta, s)
    ix.close()


# ---------------------------------------------------------------------------------------------- (6) many passes in flight
def _dim_for_width(want, k):
    """an int8 dim whose widest pass at this k is `want` (vsb_index_stat "plan_pass_max" before any query: k <= 32)"""
    import sqlite_vector_b200 as vs
    for dim in range(384, 8192, 16):
        ix = vs.Index(po.I8, dim, 1)
        if k <= 32:
            w = ix.stat("plan_pass_max")
        else:
            ix.append_dense(np.zeros((1, dim), np.int8))
            ix.finalize()
            ix.scan_topk(po.L2, np.zeros(dim, np.int8), k)
            w = ix.stat("plan_pass_max")
        ix.close()
        if w == want:
            return dim
    return None


@pytest.mark.parametrize("want", [2, 4, 8])
def test_many_passes_in_flight(want):
    """a 32-query group (every slot) with scan_streams = 2: 32 / w passes rotate over the four workspaces before anything is
    collected; one scan launch per pass and one filter per query"""
    k = 20
    dim = _dim_for_width(want, k)
    assert dim is not None, ("no int8 dim below 8192 has plan_pass_max", want)
    rng = np.random.Generator(np.random.PCG64(1000 + want))
    n = 40_000
    x, q = rng.integers(-128, 128, (n, dim)).astype(np.int8), rng.integers(-128, 128, (32, dim)).astype(np.int8)
    ix = _index(po.I8, x)
    eng = _eng()
    with _options(balance=0, scan_streams=2):
        for metric in (po.L2, po.DOT):
            lone = [ix.scan_topk(metric, q[j], k)[0] for j in range(32)]
            l0, p0 = eng.kernel_launches(), ix.stat("scan_passes")
            qc = np.ascontiguousarray(q)
            ix.scan_submit_group(metric, qc, qc.strides[0], 32, k, False, 0, fetch=True)
            assert ix.stat("plan_pass_max") == want
            assert ix.stat("scan_passes") - p0 == 32 // want
            assert eng.kernel_launches() - l0 == 32 // want + 32
            for j in range(32):
                ids, d = ix.collect(j, k)
                assert np.array_equal(ids, lone[j][0]) and np.array_equal(d.view(np.uint64), lone[j][1].view(np.uint64)), (want, metric, j)
    ix.close()


# ---------------------------------------------------------------------------------------------- (7) submission checks
def test_submissions_rejected_before_hold_or_launch():
    import torch

    import sqlite_vector_b200 as vs
    rng = np.random.Generator(np.random.PCG64(1100))
    n, dim, k = 20_000, 40, 10                                # pitch 48 > dim
    x, q = rng.integers(-128, 128, (n, dim)).astype(np.int8), rng.integers(-128, 128, (4, dim)).astype(np.int8)
    ix = _index(po.I8, x)
    eng = _eng()
    pitch = ix.query_pitch
    assert pitch == 48
    lone = [ix.scan_topk(po.L2, q[j], k)[0] for j in range(4)]

    def rejected(call):
        l0, p0 = eng.kernel_launches(), ix.stat("scan_passes")
        with pytest.raises(vs.VsbError) as e:
            call()
        assert e.value.rc == -1                                # VSB_EINVAL
        assert eng.kernel_launches() == l0 and ix.stat("scan_passes") == p0

    # one query outstanding: a held submission with an unknown metric takes no slot and launches nothing
    a = ix.scan_submit(po.L2, q[0], k)
    rejected(lambda: ix.scan_submit(99, q[1], k))
    rejected(lambda: ix.scan_submit(po.L2, q[1], 0))
    rejected(lambda: ix.scan_submit(po.L2, q[1], 257))
    b = ix.scan_submit(po.L2, q[1], k)                        # held behind a, in the slot the rejected ones did not take
    assert b == (a + 1) % ix.stat("slots")
    for slot, j in ((a, 0), (b, 1)):
        ids, d = ix.collect(slot, k)
        assert np.array_equal(ids, lone[j][0]) and np.array_equal(d, lone[j][1]), j

    qd = torch.zeros((4, 2 * pitch), dtype=torch.uint8, device="cuda")
    qd[:, :dim] = torch.from_numpy(q.view(np.uint8)).cuda()
    torch.cuda.synchronize()
    base = qd.data_ptr()
    assert base % 16 == 0
    a = ix.scan_submit(po.L2, base, k, on_device=True)        # outstanding again: later submissions would be held
    rejected(lambda: ix.scan_submit(po.L2, base + 8, k, on_device=True))
    rejected(lambda: ix.scan_submit_group(po.L2, base + 4, 2 * pitch, 2, k, True, 4, fetch=True))
    rejected(lambda: ix.scan_submit_group(po.L2, base, dim, 2, k, True, 4, fetch=True))          # stride below the pitch
    rejected(lambda: ix.scan_submit_group(po.L2, base, pitch + 8, 2, k, True, 4, fetch=True))    # not a multiple of 16
    rejected(lambda: ix.scan_submit_group(99, base, 2 * pitch, 2, k, True, 4, fetch=True))
    ids, d = ix.collect(a, k)
    assert np.array_equal(ids, lone[0][0]) and np.array_equal(d, lone[0][1])
    ix.scan_submit_group(po.L2, base, 2 * pitch, 4, k, True, 4, fetch=True)                       # a valid stride
    for j in range(4):
        ids, d = ix.collect(4 + j, k)
        assert np.array_equal(ids, lone[j][0]) and np.array_equal(d, lone[j][1]), j
    ix.close()
