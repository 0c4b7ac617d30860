"""CUDA path vs the oracle through the C ABI (include/vsb200.h).  Run on an H100: pytest -m gpu.

Bit-exact for int8/uint8 (rowids, order, distances); 1e-5 relative for fp distances
(tolerance relative to max(|d|, sum|a_i*b_i| scale) as documented in DESIGN.md §5)."""
import os

import numpy as np
import pytest

from oracle import pyoracle as po

pytestmark = pytest.mark.gpu

TYPES = [po.F32, po.F16, po.BF16, po.U8, po.I8]
METRICS = [po.L2, po.L2SQ, po.COS, po.DOT, po.L1]
G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.fixture(scope="module")
def eng():
    import sqlite_vector_b200 as vs
    e = vs.load_engine()
    assert e.device_count() >= 1, "no CUDA device: the GPU tests must not pass on a fallback"
    return e


def make_index(vtype, x, rowids=None, **kw):
    import sqlite_vector_b200 as vs
    ix = vs.Index(vtype, x.shape[1], x.shape[0], **kw)
    ix.append_dense(x, rowids)
    ix.finalize()
    return ix


def fp_tol(oracle, metric, vtype, q, x, ids_rows):
    """absolute tolerance per row: 1e-5 * max(|d|, magnitude of the terms being summed)"""
    return 1e-5


def check_fp(oracle, metric, vtype, q, x, got_ids, got_d, k, rowids):
    want_ids, want_d = oracle.scan_dense(metric, vtype, q, x, rowids, k)
    assert len(got_ids) == len(want_ids)
    # distances (sorted ascending on both sides) agree to 1e-5 relative (+ tiny abs for cancellation-prone metrics)
    xf = None
    scale = np.maximum(np.abs(want_d), 1e-30)
    if metric in (po.DOT, po.COS):
        scale = np.maximum(scale, 1.0 if metric == po.COS else float(np.abs(want_d).max()))
    assert np.all(np.abs(got_d - want_d) <= 1e-5 * scale + 1e-30), (metric, vtype, np.abs(got_d - want_d).max())
    # same rows except where the oracle's own distances are within tolerance of each other (near ties)
    if not np.array_equal(got_ids, want_ids):
        dall = oracle.distances_all(metric, vtype, q, x).astype(np.float64)
        pos = {int(r): i for i, r in enumerate(rowids)}
        kth = want_d[-1]
        for r in set(got_ids.tolist()) ^ set(want_ids.tolist()):
            assert abs(dall[pos[int(r)]] - kth) <= 2e-5 * max(abs(kth), 1e-30 if metric not in (po.DOT, po.COS) else scale.max()), (metric, vtype, r)


@pytest.mark.parametrize("vtype", TYPES)
@pytest.mark.parametrize("metric", METRICS)
def test_all_distances_match_oracle(eng, oracle, vtype, metric):
    rng = np.random.Generator(np.random.PCG64(1000 + 10 * vtype + metric))
    for (n, dim) in [(1000, 128), (777, 384), (300, 771), (64, 1536), (2050, 5)]:
        x = po.convert(rng.standard_normal((n, dim), dtype=np.float32), vtype)
        q = po.convert(rng.standard_normal((1, dim), dtype=np.float32), vtype)[0]
        ix = make_index(vtype, x)
        got = ix.scan_all(metric, q)
        want = oracle.distances_all(metric, vtype, q, x, int_exact=True)
        if vtype in (po.U8, po.I8):
            assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (vtype, metric, n, dim)
            want_scalar = oracle.distances_all(metric, vtype, q, x, int_exact=False)  # distance-cpu.c float accumulation
            assert np.array_equal(got.view(np.uint32), want_scalar.view(np.uint32)), "sums < 2^24 here: scalar == exact"
        else:
            scale = np.maximum(np.abs(want), 1e-30)
            if metric == po.COS:
                scale = np.maximum(scale, 1.0)
            if metric == po.DOT:
                xf = oracle.distances_all(po.L1, vtype, np.zeros_like(q), x)  # sum |x_i| as magnitude proxy
                scale = np.maximum(scale, 1e-2 * xf)
            assert np.all(np.abs(got - want) <= 1e-5 * scale), (vtype, metric, n, dim, np.max(np.abs(got - want) / scale))
        ix.close()


@pytest.mark.parametrize("vtype", [po.U8, po.I8])
@pytest.mark.parametrize("metric", METRICS)
def test_topk_int_bit_exact_with_ties(eng, oracle, vtype, metric):
    rng = np.random.Generator(np.random.PCG64(2000 + 10 * vtype + metric))
    for (n, dim, k, spread) in [(5000, 16, 20, 3), (20000, 32, 20, 30), (50, 8, 100, 2), (3000, 4, 7, 1), (40000, 384, 33, 60), (9, 16, 20, 5)]:
        lo, hi = (0, 2 * spread) if vtype == po.U8 else (-spread, spread)
        x = rng.integers(lo, hi + 1, (n, dim)).astype(po.NP_STORAGE[vtype])
        rowids = np.arange(n, dtype=np.int64) * 3 + 7
        q = rng.integers(lo, hi + 1, dim).astype(x.dtype)
        ix = make_index(vtype, x, rowids)
        for smi in (0, min(2, k - 1)):
            (res,), mi = ix.scan_topk(metric, q, k, max_index=smi)
            want_ids, want_d = oracle.scan_dense(metric, vtype, q, x, rowids, k, start_max_index=smi)
            assert np.array_equal(res[0], want_ids), (vtype, metric, n, dim, k)
            assert np.array_equal(res[1], want_d)
        ix.close()


@pytest.mark.parametrize("vtype", [po.F32, po.F16, po.BF16])
@pytest.mark.parametrize("metric", METRICS)
def test_topk_fp(eng, oracle, vtype, metric):
    rng = np.random.Generator(np.random.PCG64(3000 + 10 * vtype + metric))
    for (n, dim, k) in [(20000, 128, 20), (5000, 384, 20), (3000, 768, 50), (100, 24, 200)]:
        x = po.convert(rng.standard_normal((n, dim), dtype=np.float32), vtype)
        q = po.convert(rng.standard_normal((1, dim), dtype=np.float32), vtype)[0]
        rowids = np.arange(1, n + 1, dtype=np.int64)
        ix = make_index(vtype, x, rowids)
        (res,) = ix.scan_topk(metric, q, k)
        check_fp(oracle, metric, vtype, q, x, res[0], res[1], k, rowids)
        ix.close()


def test_quant_chunk_preload_layout(eng, oracle):
    """vsb_index_append_quant_chunk consumes the reference's shadow-table blob format."""
    rng = np.random.Generator(np.random.PCG64(42))
    n, dim, k = 30000, 384, 20
    xf = rng.standard_normal((n, dim), dtype=np.float32)
    scale, offset, qt = oracle.quant_params(po.F32, xf)
    assert qt == po.Q_S8
    rowids = np.arange(n, dtype=np.int64) * 2 + 1
    buf = oracle.build_quant_buffer(po.F32, xf, rowids, offset, scale, qt)
    import sqlite_vector_b200 as vs
    ix = vs.Index(po.I8, dim, n)
    third = (n // 3) * (8 + dim)
    ix.append_quant_chunk(buf[:third], n // 3)            # chunked like the 30 MB shadow-table rows
    ix.append_quant_chunk(buf[third:], n - n // 3)
    ix.finalize()
    qf = rng.standard_normal(dim).astype(np.float32)
    qq = oracle.quantize(po.F32, qf, offset, scale, qt)
    for metric in METRICS:
        (res,) = ix.scan_topk(metric, qq, k)
        want_ids, want_d = oracle.scan_quant_buffer(metric, qt, qq, buf, n, dim, k)
        assert np.array_equal(res[0], want_ids) and np.array_equal(res[1], want_d), metric
    ix.close()


def test_golden_topk(eng):
    """CUDA vs the committed reference outputs (no oracle in the loop)."""
    g = np.load(os.path.join(G, "topk.npz"))
    for c in range(int(g["ncases"][0])):
        qt, n, dim, k = (int(v) for v in g[f"c{c}_meta"])
        vt = po.U8 if qt == po.Q_U8 else po.I8
        ix = make_index(vt, g[f"c{c}_vec"], g[f"c{c}_rowids"])
        for m in METRICS:
            (res,) = ix.scan_topk(m, g[f"c{c}_q"], k)
            assert np.array_equal(res[0], g[f"c{c}_ids_{m}"]) and np.array_equal(res[1], g[f"c{c}_dist_{m}"]), (c, m)
        ix.close()


def test_edge_cases(eng, oracle):
    rng = np.random.Generator(np.random.PCG64(9))
    x = rng.integers(-5, 6, (100, 16)).astype(np.int8)
    ix = make_index(po.I8, x)
    q = x[3].copy()
    (res,) = ix.scan_topk(po.L2, q, 0)                     # k = 0 -> empty (sqlite-vector.c:1796)
    assert len(res[0]) == 0
    (res,) = ix.scan_topk(po.L2, q, 150)                   # k > n -> n rows, INF slots trimmed
    want_ids, want_d = oracle.scan_dense(po.L2, po.I8, q, x, np.arange(1, 101, dtype=np.int64), 150)
    assert np.array_equal(res[0], want_ids) and np.array_equal(res[1], want_d)
    (res,) = ix.scan_topk(po.L2, q, 300)                   # k above the candidate path -> all-distances path
    want_ids, want_d = oracle.scan_dense(po.L2, po.I8, q, x, np.arange(1, 101, dtype=np.int64), 300)
    assert np.array_equal(res[0], want_ids) and np.array_equal(res[1], want_d)
    ix.close()
    # descending distances: every row enters the slots -> candidate log overflows -> exact fallback
    n = 200000
    x = np.zeros((n, 16), dtype=np.int8)
    x[:, 0] = np.clip(np.arange(n)[::-1] // 1600, 0, 127)
    ix = make_index(po.I8, x)
    q = np.zeros(16, dtype=np.int8)
    (res,) = ix.scan_topk(po.L1, q, 20)
    want_ids, want_d = oracle.scan_dense(po.L1, po.I8, q, x, np.arange(1, n + 1, dtype=np.int64), 20)
    assert np.array_equal(res[0], want_ids) and np.array_equal(res[1], want_d)
    ix.close()
    # empty index
    import sqlite_vector_b200 as vs
    ix = vs.Index(po.F32, 8, 0)
    ix.finalize()
    (res,) = ix.scan_topk(po.L2, np.zeros(8, np.float32), 5)
    assert len(res[0]) == 0
    ix.close()


def test_special_values_f16(eng, oracle):
    """NaN lanes are skipped and a single infinity propagates like the reference (distance-cpu.c:318-466)."""
    x = po.convert(np.random.Generator(np.random.PCG64(5)).standard_normal((64, 8), dtype=np.float32), po.F16)
    x[3, 2] = 0x7E00   # NaN
    x[5, 1] = 0x7C00   # +Inf
    x[9, :] = 0        # zero vector
    q = x[0].copy()
    ix = make_index(po.F16, x)
    for metric in METRICS:
        got = ix.scan_all(metric, q)
        want = oracle.distances_all(metric, po.F16, q, x)
        both_nan = np.isnan(got) & np.isnan(want)
        ok = both_nan | (np.abs(got - want) <= 1e-5 * np.maximum(np.abs(want), 1.0)) | (got == want)
        assert ok.all(), (metric, got[~ok], want[~ok])
    ix.close()


def test_multi_shard_candidates_replay(eng, oracle):
    """row-sharded scan: per-shard candidates concatenated in scan order + vsb_replay_topk == one-shard result."""
    rng = np.random.Generator(np.random.PCG64(77))
    n, dim, k = 60000, 64, 20
    x = rng.integers(-20, 21, (n, dim)).astype(np.int8)
    q = rng.integers(-20, 21, dim).astype(np.int8)
    rowids = np.arange(1, n + 1, dtype=np.int64)
    import sqlite_vector_b200 as vs
    bounds = [0, 15000, 15001, 40000, n]
    parts = []
    for a, b in zip(bounds[:-1], bounds[1:]):
        ix = vs.Index(po.I8, dim, b - a, first_seq=a)
        ix.append_dense(x[a:b], rowids[a:b])
        ix.finalize()
        parts.append(ix.scan_candidates(po.L2, q, k)[0])
        ix.close()
    cands = np.concatenate(parts)
    assert np.all(np.diff(cands["seq"]) > 0)
    ids, d, _ = eng.replay_topk(cands, k)
    want_ids, want_d = oracle.scan_dense(po.L2, po.I8, q, x, rowids, k)
    assert np.array_equal(ids, want_ids) and np.array_equal(d, want_d)


@pytest.mark.parametrize("vtype,dim,n", [(po.I8, 384, 150_000), (po.U8, 100, 40_000), (po.F32, 64, 30_000), (po.BF16, 1536, 9_000), (po.I8, 20000, 700)])
def test_group_launch_equals_single_queries(eng, oracle, vtype, dim, n):
    """vsb_scan_submit_group (one scan launch per query, a full group and a partial one) must give exactly what single
    queries give, host queries and device-side staging alike; the last case is the no-staging (DIRECT) kernel."""
    import sqlite_vector_b200 as vs
    rng = np.random.Generator(np.random.PCG64(2024 + dim))
    x = po.convert(rng.standard_normal((n, dim), dtype=np.float32), vtype)
    nq = 13
    q = po.convert(rng.standard_normal((nq, dim), dtype=np.float32), vtype)
    ix = make_index(vtype, x)
    for metric, k in [(po.L2, 20), (po.COS, 7), (po.DOT, 32), (po.L1, 40)]:
        want = ix.scan_topk(metric, q[0], k)            # warms the workspace for this k
        want = [ix.scan_topk(metric, q[b], k)[0] for b in range(nq)]
        got = []
        for g0, m, first in [(0, 8, 0), (8, 5, 8)]:     # a full group and a partial one
            ix.scan_submit_group(metric, np.ascontiguousarray(q[g0:g0 + m]), q.strides[0], m, k, False, first, fetch=True)
            got += [ix.collect(first + j, k) for j in range(m)]
        for b in range(nq):
            assert np.array_equal(got[b][0], want[b][0]) and np.array_equal(got[b][1], want[b][1]), (vtype, metric, k, b)
    ix.close()


def test_k_sequence_on_one_index(eng, oracle):
    """ADVICE r1 (high): the scan workspace never shrinks, so a k <= 32 query after a 33 <= k <= 256 one used to run the
    generic list layout against the k <= 32 filter.  Every k of the sequence must match the oracle on ONE index, through
    the synchronous call and through submit/collect."""
    rng = np.random.Generator(np.random.PCG64(4242))
    n, dim = 60000, 64
    x = rng.integers(-30, 31, (n, dim)).astype(np.int8)
    rowids = np.arange(n, dtype=np.int64) * 2 + 3
    ix = make_index(po.I8, x, rowids)
    for i, k in enumerate([100, 10, 33, 20, 256, 5, 32, 64, 1, 300, 7]):
        q = rng.integers(-30, 31, dim).astype(np.int8)
        metric = METRICS[i % len(METRICS)]
        want_ids, want_d = oracle.scan_dense(metric, po.I8, q, x, rowids, k)
        (res,) = ix.scan_topk(metric, q, k)
        assert np.array_equal(res[0], want_ids) and np.array_equal(res[1], want_d), ("sync", k)
        if k <= 256:
            slot = ix.scan_submit(metric, q, k, on_device=False, fetch=True)
            ids, d = ix.collect(slot, k)
            assert np.array_equal(ids, want_ids) and np.array_equal(d, want_d), ("submit", k)
    ix.close()


def _special_matrix(vtype, rng, n=96, dim=40):
    """rows with NaN / +-Inf / zero vectors / mixed-sign infinities at assorted positions (storage bits of `vtype`)"""
    x = po.convert(rng.standard_normal((n, dim), dtype=np.float32), vtype)
    if vtype == po.F32:
        NAN, PINF, NINF = np.float32(np.nan), np.float32(np.inf), np.float32(-np.inf)
    elif vtype == po.F16:
        NAN, PINF, NINF = 0x7E00, 0x7C00, 0xFC00
    else:
        NAN, PINF, NINF = 0x7FC0, 0x7F80, 0xFF80
    x[3, 2] = NAN
    x[5, 1] = PINF
    x[6, 7] = NINF
    x[9, :] = 0
    x[11, 4] = PINF; x[11, dim - 10] = NINF      # mixed-sign infinities in one row (round-1 deviation 6)
    x[12, dim - 10] = PINF; x[12, 4] = NINF
    x[13, 0] = NAN; x[13, 5] = PINF
    x[14, 3] = PINF; x[14, 9] = NAN; x[14, 20] = NINF
    x[15, dim - 1] = NINF                         # last element (tail loop of the reference)
    x[16, 8] = PINF; x[16, 9] = PINF
    return x, (NAN, PINF, NINF)


@pytest.mark.parametrize("vtype", [po.F32, po.F16, po.BF16])
def test_special_values_all_fp_types(eng, oracle, vtype):
    """NaN / Inf policies of the reference's fp kernels (distance-cpu.c:39-159 f32, :164-314 bf16, :318-466 f16), including
    rows that mix infinities of both signs and queries that carry specials themselves: bit pattern of the result class
    (NaN / +Inf / -Inf) identical, finite values within 1e-5."""
    rng = np.random.Generator(np.random.PCG64(50 + vtype))
    x, (NAN, PINF, NINF) = _special_matrix(vtype, rng)
    dim = x.shape[1]
    queries = [x[0].copy(), x[5].copy(), x[11].copy(), x[9].copy()]
    qz = x[1].copy(); qz[4] = 0; qz[dim - 10] = 0  # zeros where rows 11/12 hold infinities: Inf * 0
    queries.append(qz)
    qn = x[2].copy(); qn[8] = NAN; qn[3] = NINF
    queries.append(qn)
    ix = make_index(vtype, x)
    for qi, q in enumerate(queries):
        for metric in METRICS:
            got = ix.scan_all(metric, q)
            want = oracle.distances_all(metric, vtype, q, x)
            same_class = (np.isnan(got) == np.isnan(want)) & (np.isposinf(got) == np.isposinf(want)) & (np.isneginf(got) == np.isneginf(want))
            assert same_class.all(), (vtype, metric, qi, np.nonzero(~same_class)[0], got[~same_class], want[~same_class])
            fin = np.isfinite(want)
            assert np.all(np.abs(got[fin] - want[fin]) <= 1e-5 * np.maximum(np.abs(want[fin]), 1.0)), (vtype, metric, qi)
            # and the top-k built from them (NaN never enters, -Inf sorts first)
            (res,) = ix.scan_topk(metric, q, 10)
            want_ids, want_d = oracle.scan_dense(metric, vtype, q, x, np.arange(1, x.shape[0] + 1, dtype=np.int64), 10)
            assert len(res[0]) == len(want_ids)
            assert np.array_equal(np.isinf(res[1]), np.isinf(want_d)) and np.array_equal(np.sign(res[1][np.isinf(res[1])]), np.sign(want_d[np.isinf(want_d)]))
    ix.close()


@pytest.mark.parametrize("vtype", [po.F16, po.BF16])
def test_special_values_through_the_batch_path(eng, oracle, vtype):
    """the tensor-core path must hand rows with NaN / Inf scores to the exact refinement: same result classes as the oracle"""
    rng = np.random.Generator(np.random.PCG64(150 + vtype))
    n, dim, nq, k = 20000, 40, 32, 12
    x = po.convert(rng.standard_normal((n, dim), dtype=np.float32), vtype)
    xs, _ = _special_matrix(vtype, rng, 96, dim)
    x[5000:5096] = xs
    q = po.convert(rng.standard_normal((nq, dim), dtype=np.float32), vtype)
    q[3] = xs[11]; q[4] = xs[5]
    ix = make_index(vtype, x)
    rowids = np.arange(1, n + 1, dtype=np.int64)
    for metric in (po.L2, po.COS, po.DOT):
        b0, f0 = ix.stat("batches"), ix.stat("fallbacks")
        res = ix.scan_topk(metric, q, k)
        # a query that holds an infinity makes every row a candidate: the batch call may then hit a capacity and fall back to the
        # per-query path (counted); either way the tensor-core entry point was taken and the results must be the oracle's
        assert ix.stat("batches") == b0 + 1 or ix.stat("fallbacks") > f0
        for b in range(nq):
            want_ids, want_d = oracle.scan_dense(metric, vtype, q[b], x, rowids, k)
            got_ids, got_d = res[b]
            assert len(got_d) == len(want_d), (vtype, metric, b)
            inf = np.isinf(want_d)
            assert np.array_equal(np.isinf(got_d), inf) and np.array_equal(np.sign(got_d[inf]), np.sign(want_d[inf])), (vtype, metric, b, got_d, want_d)
            assert set(got_ids[inf].tolist()) == set(want_ids[inf].tolist())
            fin = ~inf
            scale = np.maximum(np.abs(want_d[fin]), 1.0 if metric in (po.COS, po.DOT) else 1e-30)
            assert np.all(np.abs(got_d[fin] - want_d[fin]) <= 1e-5 * scale), (vtype, metric, b)
    ix.close()


@pytest.mark.parametrize("vtype", [po.F32, po.F16, po.BF16])
def test_golden_special_value_distances(eng, vtype):
    """CUDA vs the committed outputs of the UNMODIFIED reference on NaN / Inf / signed-zero / 65504 inputs (tests/golden/
    distances.npz, keys spa/spb/spd; no oracle in the loop): same NaN / +-Inf classes, finite values within 1e-5."""
    g = np.load(os.path.join(G, "distances.npz"))
    a, b = g[f"spa_{vtype}"], g[f"spb_{vtype}"]
    ix = make_index(vtype, np.ascontiguousarray(b))
    for m in METRICS:
        want = g[f"spd_{vtype}_{m}"]
        got = np.array([ix.scan_all(m, np.ascontiguousarray(a[i]))[i] for i in range(a.shape[0])], dtype=np.float32)
        # the golden values are raw kernel results; the scan applies the nearly-zero clamp on top (sqlite-vector.c:2099)
        want = np.where(np.abs(want) <= 8 * np.finfo(np.float32).eps, np.float32(0), want)
        same = (np.isnan(got) == np.isnan(want)) & (np.isposinf(got) == np.isposinf(want)) & (np.isneginf(got) == np.isneginf(want))
        assert same.all(), (vtype, m, np.nonzero(~same)[0], got[~same], want[~same])
        fin = np.isfinite(want)
        assert np.all(np.abs(got[fin] - want[fin]) <= 1e-5 * np.maximum(np.abs(want[fin]), 1.0)), (vtype, m)
    ix.close()


@pytest.mark.parametrize("vtype", TYPES)
def test_quantizer_bytes_match_oracle(eng, oracle, vtype):
    """vsb_quantizer_* (the GPU loops of vector_quantize, sqlite-vector.c:1224-1320) against the oracle's quantize /
    build_quant_buffer (pinned to the reference): min / max / qtype decision and every output byte, both qtypes, retained and
    streamed, including NaN / Inf / huge inputs and values that land exactly on .5"""
    import sqlite_vector_b200 as vs
    rng = np.random.Generator(np.random.PCG64(600 + vtype))
    n, dim = 20_000, 37
    xf = rng.standard_normal((n, dim), dtype=np.float32) * 3
    xf[::97, 3] = np.round(xf[::97, 3] * 2) / 2                  # exact halves
    x = po.convert(xf, vtype)
    if vtype in (po.F32, po.F16, po.BF16):
        sp, _ = _special_matrix(vtype, rng, 96, dim)
        x[500:596] = sp
        if vtype == po.F32:
            x[700, 0] = np.float32(3e38); x[701, 1] = np.float32(-3e38); x[702, 2] = np.float32(1e10)
    rowids = np.arange(n, dtype=np.int64) * 5 - 1000              # negative and positive rowids
    scale0, offset0, qt0 = oracle.quant_params(vtype, x)
    for retain in (n, 0):
        qz = vs.api.Quantizer(vtype, dim, retain_rows=retain)
        for a in range(0, n, 6000):
            qz.minmax(x[a:a + 6000])
        lo, hi, neg = qz.minmax_result()
        assert qz.retained_rows == (n if retain else -1)
        qt = po.Q_S8 if neg else po.Q_U8
        assert qt == qt0
        abs_max = max(abs(np.float32(lo)), abs(np.float32(hi)))
        scale = np.float32(255.0) / (np.float32(hi) - np.float32(lo)) if qt == po.Q_U8 else np.float32(127.0) / np.float32(abs_max)
        offset = np.float32(lo) if qt == po.Q_U8 else np.float32(0)
        assert (np.float32(scale) == np.float32(scale0) or (np.isnan(scale) and np.isnan(scale0))) and (np.float32(offset) == np.float32(offset0) or (np.isnan(offset) and np.isnan(offset0))), (scale, scale0, offset, offset0)
        for q, sc, off in ((po.Q_U8, np.float32(37.5), np.float32(-2.0)), (po.Q_S8, np.float32(31.0), np.float32(0.0)), (qt, np.float32(scale), np.float32(offset))):
            if not np.isfinite(sc):
                continue
            want = oracle.build_quant_buffer(vtype, x, rowids, off, sc, q)
            got = qz.encode(None if retain else x, rowids, float(off), float(sc), q)
            assert np.array_equal(got, want), (vtype, retain, q, np.nonzero(got != want)[0][:10])
        qz.close()
