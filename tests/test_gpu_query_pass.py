"""Passes of several queries over one read of the column (DESIGN §3.1, §3.2).  -m gpu.

(1) every query of a pass (vsb_scan_submit_group, nq = 2, 3, 4, 8) returns bit for bit what the same query scanned alone
    returns, for every element type and metric, at plan shapes P = 1, P > 1 and DIRECT, below the stream count and at 1M rows
    (adaptive partition); the lone results match the oracle (exact for integer types, tests/fpcheck.py for fp);
(2) NaN / Inf rows in a pass, and a pass in which only one query overflows its candidate log;
(3) the hold rule of vsb_scan_submit, seen through the counters scan_passes / pass_queries and kernel_launches."""
import numpy as np
import pytest

from oracle import pyoracle as po
from tests import fpcheck

pytestmark = pytest.mark.gpu

METRICS = [po.L2, po.L2SQ, po.COS, po.DOT, po.L1]
KS = [1, 20, 32, 33, 256]


@pytest.fixture(scope="module")
def eng():
    import sqlite_vector_b200 as vs
    e = vs.load_engine()
    assert e.device_count() >= 1, "no CUDA device: the GPU tests must not pass on a fallback"
    return e


def _index(vtype, x):
    import sqlite_vector_b200 as vs
    ix = vs.Index(vtype, x.shape[1], x.shape[0])
    ix.append_dense(x)
    ix.finalize()
    return ix


def _data(vtype, n, dim, nq, seed):
    rng = np.random.Generator(np.random.PCG64(seed))
    if vtype in (po.I8, po.U8):
        lo, hi = (-128, 128) if vtype == po.I8 else (0, 256)
        dt = np.int8 if vtype == po.I8 else np.uint8
        return rng.integers(lo, hi, (n, dim)).astype(dt), rng.integers(lo, hi, (nq, dim)).astype(dt)
    return (po.convert(rng.standard_normal((n, dim), dtype=np.float32), vtype),
            po.convert(rng.standard_normal((nq, dim), dtype=np.float32), vtype))


def _passes(ix, metric, q, k, nq):
    """q[0:nq] as one group: passes of up to plan_pass_max queries; results of slots 0 .. nq - 1"""
    q = np.ascontiguousarray(q[:nq])
    ix.scan_submit_group(metric, q, q.strides[0], nq, k, False, 0, fetch=True)
    return [ix.collect(j, k) for j in range(nq)]


def _same(a, b):
    return np.array_equal(a[0], b[0]) and np.array_equal(a[1].view(np.uint64), b[1].view(np.uint64))


# (type, dim): P = 1 staged (int8 384, the bench shape), staged with 4-query passes at most (int8 420), DIRECT (int8 449),
# fp staged (f32 110, bf16 220), P = 2 (f16 300), P = 4 (int8 1000), a one-chunk row (uint8 5)
SHAPES = [(po.I8, 384), (po.I8, 420), (po.I8, 449), (po.F32, 110), (po.BF16, 220), (po.F16, 300), (po.I8, 1000), (po.U8, 5)]


@pytest.mark.parametrize("n", [1000, 1_000_000])
@pytest.mark.parametrize("vtype,dim", SHAPES)
def test_pass_equals_lone_query(eng, oracle, vtype, dim, n):
    x, q = _data(vtype, n, dim, 8, 77 + dim)
    ix = _index(vtype, x)
    rowids = np.arange(1, n + 1, dtype=np.int64)
    integer = vtype in (po.I8, po.U8)
    widths = set()
    for metric in METRICS:
        for k in KS:
            lone = [ix.scan_topk(metric, q[b], k)[0] for b in range(8)]
            if n <= 1000:
                for b in range(8):
                    want_ids, want_d = oracle.scan_dense(metric, vtype, q[b], x, rowids, k)
                    if integer:
                        assert np.array_equal(lone[b][0], want_ids) and np.array_equal(lone[b][1], want_d), (metric, k, b)
                    else:
                        fpcheck.assert_fp_topk(lone[b][0], lone[b][1], want_ids, want_d, metric,
                                               lambda r, b=b: oracle.distance(metric, vtype, q[b], x[r - 1]), (metric, k, b))
            for nq in (2, 3, 4, 8):
                p0, q0 = ix.stat("scan_passes"), ix.stat("pass_queries")
                got = _passes(ix, metric, q, k, nq)
                width = ix.stat("plan_pass_max")
                widths.add(width)
                assert ix.stat("pass_queries") - q0 == nq
                assert ix.stat("scan_passes") - p0 == -(-nq // width), (nq, width)
                for b in range(nq):
                    assert _same(got[b], lone[b]), (metric, k, nq, b)
    assert max(widths) >= 2, "this shape never shared a pass"
    ix.close()


def test_plan_unchanged_by_pass_width(eng):
    """the bench shape keeps its one-query plan (P = 1, two stages, staged) at every pass width it launches"""
    x, q = _data(po.I8, 300_000, 384, 8, 5)
    ix = _index(po.I8, x)
    ix.scan_topk(po.L2, q[0], 20)
    one = [ix.stat(s) for s in ("plan_log2p", "plan_nsw", "plan_direct")]
    assert one == [0, 2, 0]
    assert ix.stat("plan_pass_max") == 8
    for nq in (2, 4, 8):
        _passes(ix, po.L2, q, 20, nq)
        assert [ix.stat(s) for s in ("plan_log2p", "plan_nsw", "plan_direct")] == one, nq
    ix.close()


@pytest.mark.parametrize("vtype", [po.F16, po.BF16, po.F32])
def test_special_values_in_a_pass(eng, oracle, vtype):
    rng = np.random.Generator(np.random.PCG64(9))
    n, dim = 5000, 40
    x = po.convert(rng.standard_normal((n, dim), dtype=np.float32), vtype)
    q = po.convert(rng.standard_normal((8, dim), dtype=np.float32), vtype)
    if vtype == po.F32:
        NAN, PINF, NINF = np.float32(np.nan), np.float32(np.inf), np.float32(-np.inf)
    elif vtype == po.F16:
        NAN, PINF, NINF = 0x7E00, 0x7C00, 0xFC00
    else:
        NAN, PINF, NINF = 0x7FC0, 0x7F80, 0xFF80
    for r in range(0, n, 97):
        x[r, r % dim] = (NAN, PINF, NINF)[r % 3]
    x[11, 4] = PINF; x[11, 9] = NINF
    q[2, 3] = PINF                                   # a query with an infinity in the pass
    ix = _index(vtype, x)
    for metric in METRICS:
        for k in (5, 40):
            lone = [ix.scan_topk(metric, q[b], k)[0] for b in range(8)]
            got = _passes(ix, metric, q, k, 8)
            for b in range(8):
                assert _same(got[b], lone[b]), (metric, k, b)
    ix.close()


def test_one_query_overflows_its_log(eng, oracle):
    """strictly falling distances along the scan order make every row of query 0 beat its running k-th value, which overflows
    its log (256 entries per stream at k = 10); the other queries of the pass keep their own logs and flags"""
    n, dim = 1_000_000, 32
    t = (n - 1 - np.arange(n)).astype(np.int64)              # the squared distance of row r to query 0, falling with r
    a = np.zeros((n, dim), dtype=np.int64)
    for j in range(dim):                                      # t as a sum of squares of terms <= 255
        a[:, j] = np.minimum(np.sqrt(t).astype(np.int64), 255)
        a[:, j] -= (a[:, j] * a[:, j] > t)
        t -= a[:, j] * a[:, j]
    assert not t.any()
    x = (127 - a).astype(np.int8)
    q = np.random.Generator(np.random.PCG64(8)).integers(-128, 128, (4, dim)).astype(np.int8)
    q[0] = 127
    ix = _index(po.I8, x)
    rowids = np.arange(1, n + 1, dtype=np.int64)
    k = 10
    f0 = ix.stat("fallbacks")
    q4 = np.ascontiguousarray(q)
    ix.scan_submit_group(po.L2, q4, q4.strides[0], 4, k, False, 0, fetch=True)
    with pytest.raises(Exception):
        ix.collect(0, k)                                     # query 0's log overflowed: the asynchronous collect reports it
    for b in range(1, 4):
        ids, d = ix.collect(b, k)
        want_ids, want_d = oracle.scan_dense(po.L2, po.I8, q[b], x, rowids, k)
        assert np.array_equal(ids, want_ids) and np.array_equal(d, want_d), b
    (res,) = ix.scan_topk(po.L2, q[0], k)                    # the synchronous call answers it through the all-distances path
    want_ids, want_d = oracle.scan_dense(po.L2, po.I8, q[0], x, rowids, k)
    assert np.array_equal(res[0], want_ids) and np.array_equal(res[1], want_d)
    assert ix.stat("fallbacks") - f0 == 1
    ix.close()


def _counts(ix):
    return ix.stat("scan_passes"), ix.stat("pass_queries")


def test_hold_rule(eng, oracle):
    import torch
    n, dim, k = 200_000, 384, 20
    x, q = _data(po.I8, n, dim, 16, 3)
    ix = _index(po.I8, x)
    lone = {(m, kk, b): ix.scan_topk(m, q[b], kk)[0] for m in (po.L2, po.DOT) for kk in (k, 7) for b in range(16)}
    pitch = ix.query_pitch
    qd = torch.zeros((16, pitch), dtype=torch.uint8, device="cuda")
    qd[:, :dim] = torch.from_numpy(q.view(np.uint8)).cuda()
    torch.cuda.synchronize()

    def check(slot, m, kk, b):
        assert _same(ix.collect(slot, kk), lone[(m, kk, b)]), (slot, m, kk, b)

    # a lone caller: each submission launches at once
    p, c = _counts(ix)
    for b in range(3):
        check(ix.scan_submit(po.L2, q[b], k), po.L2, k, b)
    assert _counts(ix) == (p + 3, c + 3)

    # submit i+1, collect i: the queries pair up, one launch of the scan kernel per pass
    p, c = _counts(ix)
    l0 = eng.kernel_launches()
    pend = (ix.scan_device_query(po.L2, qd[0].data_ptr(), k), 0)
    for b in range(1, 9):
        s = ix.scan_device_query(po.L2, qd[b].data_ptr(), k)
        check(pend[0], po.L2, k, pend[1])
        pend = (s, b)
    check(pend[0], po.L2, k, pend[1])
    # 9 queries: 0 alone, then (1, 2), (3, 4), (5, 6), (7, 8)
    assert _counts(ix) == (p + 5, c + 9)
    assert eng.kernel_launches() - l0 == 5 + 9               # one scan launch per pass, one filter per query

    # a held query waits for nothing else: each of these calls launches it
    def held_then(call, own_passes=0):
        a = ix.scan_submit(po.L2, q[0], k)
        b = ix.scan_submit(po.L2, q[1], k)                   # held (a is outstanding)
        p1, c1 = _counts(ix)
        call()
        assert _counts(ix) == (p1 + 1 + own_passes, c1 + 1 + own_passes), call
        check(a, po.L2, k, 0)
        check(b, po.L2, k, 1)

    held_then(lambda: ix.result_block(0))
    held_then(lambda: ix.scan_topk(po.L2, q[3], k), own_passes=1)
    held_then(lambda: ix.scan_range(po.L2, q[3:4], [1.0]))
    held_then(lambda: ix.profile_read())

    # collect_last launches the held pass and returns its query
    a = ix.scan_submit(po.L2, q[0], k)
    b = ix.scan_submit(po.L2, q[1], k)
    r = ix.collect_last(k)
    assert _same(r, lone[(po.L2, k, 1)])
    check(a, po.L2, k, 0)

    # collecting the held query launches its pass
    a = ix.scan_submit(po.L2, q[0], k)
    b = ix.scan_submit(po.L2, q[1], k)
    c_ = ix.scan_submit(po.L2, q[2], k)
    p1, c1 = _counts(ix)
    check(c_, po.L2, k, 2)
    assert _counts(ix) == (p1 + 1, c1 + 2)                   # b and c in one pass
    check(a, po.L2, k, 0)
    check(b, po.L2, k, 1)

    # another k, another metric: the held pass is launched first
    for m2, k2 in ((po.L2, 7), (po.DOT, k)):
        a = ix.scan_submit(po.L2, q[0], k)
        b = ix.scan_submit(po.L2, q[1], k)
        p1, c1 = _counts(ix)
        c_ = ix.scan_submit(m2, q[2], k2)                    # launches (b); c is held behind a, b
        assert _counts(ix) == (p1 + 1, c1 + 1)
        check(a, po.L2, k, 0)
        check(b, po.L2, k, 1)
        check(c_, m2, k2, 2)

    # reusing the slot of a held query launches it first
    a = ix.scan_submit(po.L2, q[0], k)
    b = ix.scan_submit(po.L2, q[1], k)
    p1, c1 = _counts(ix)
    b2 = ix.scan_submit(po.L2, q[2], k, slot=b)
    assert b2 == b and _counts(ix) == (p1 + 1, c1 + 1)
    check(a, po.L2, k, 0)
    check(b2, po.L2, k, 2)

    # a full pass launches by itself
    w = ix.stat("plan_pass_max")
    a = ix.scan_submit(po.L2, q[0], k)
    p1, c1 = _counts(ix)
    slots = [ix.scan_submit(po.L2, q[1 + j], k) for j in range(w)]
    assert _counts(ix) == (p1 + 1, c1 + w)
    check(a, po.L2, k, 0)
    for j, s in enumerate(slots):
        check(s, po.L2, k, 1 + j)

    # results read on the device (fetch = 0) are never held
    a = ix.scan_submit(po.L2, q[0], k)
    p1, c1 = _counts(ix)
    ix.scan_submit(po.L2, q[1], k, fetch=False)
    assert _counts(ix) == (p1 + 1, c1 + 1)
    check(a, po.L2, k, 0)

    # close launches what is held
    ix.scan_submit(po.L2, q[0], k)
    ix.scan_submit(po.L2, q[1], k)
    ix.close()
