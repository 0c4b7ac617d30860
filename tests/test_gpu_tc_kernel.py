"""The wgmma scoring kernel (tc_scan_kernel) on its own, through vsb_debug_tc_level: one tensor-core level of the batch path
with given per-query bounds.  References are numpy float64 only.  -m gpu.

(a) integer scores equal X @ Q.T exactly (every N, ragged query groups, rows under one 128-byte block, many K blocks);
(b) integer candidate logs equal the host evaluation of tc_hit on the exact scores, with the kernel's own constants and norms;
(c) f16 / bf16 scores stay within the error model of tc_fp_eps, |s_tc - s| <= dim * 2^-21 * sum |q_i r_i|, on adversarial
    input families (tests/fpfamilies.py);
(d) f16 / bf16 logs hold every pair whose exact distance is below the bound by more than the refine's own error."""
import numpy as np
import pytest

from oracle import pyoracle as po
from tests import fpfamilies as fam

pytestmark = pytest.mark.gpu

TC_METRICS = [po.L2, po.COS, po.DOT]
KIND_NAMES = {po.I8: "int8", po.U8: "uint8", po.F16: "f16", po.BF16: "bf16"}


def _index(vtype, x):
    import sqlite_vector_b200 as vs
    ix = vs.Index(vtype, x.shape[1], x.shape[0])
    ix.append_dense(x)
    ix.finalize()
    return ix


def _epi_chunk(value):
    import sqlite_vector_b200 as vs
    return vs.load_engine().set_option("epi_chunk", value)


def _int_data(vtype, n, dim, rng):
    if vtype == po.I8:
        return rng.integers(-128, 128, (n, dim)).astype(np.int8)
    return rng.integers(0, 256, (n, dim)).astype(np.uint8)


# ---------------------------------------------------------------------------------------------- (a) integer scores
def _rows_for(dim):
    # enough 128-row tiles that each of the 132 CTAs walks several, and (small dim: one K block per tile) the stage ring
    # wraps its phase many times; about 3e7 bytes of corpus
    return int(min(200_000, max(10_000, 30_000_000 // dim)))


def _check_scores(ix, x64, q, r0, r1, N):
    res = ix.debug_tc_level(po.DOT, q, np.full(q.shape[0], np.inf, np.float32), r0, r1, N=N, scores=True)
    want = x64[r0:r1] @ q.astype(np.float64).T
    got = res["scores"].astype(np.int64)
    bad = np.argwhere(got != want.astype(np.int64))
    assert bad.size == 0, (N, q.shape[0], r0, r1, "first wrong (row - r0, query):", bad[:5].tolist(), len(bad))


@pytest.mark.parametrize("dim", [16, 100, 128, 200, 1000, 1536, 4096])
@pytest.mark.parametrize("vtype", [po.I8, po.U8])
def test_int_scores_exact(vtype, dim):
    rng = np.random.Generator(np.random.PCG64(1000 + dim + vtype))
    n = _rows_for(dim)
    x = _int_data(vtype, n, dim, rng)
    x64 = x.astype(np.float64)
    ix = _index(vtype, x)
    r0, r1 = 256, n - 37                                    # r0 > 0, r1 not a multiple of 128
    for N in (32, 64, 128, 256):
        # NG = 1 full, NG > 1 ragged; and one group with fewer queries than N
        for nq in (N, 2 * N + 5) + ((20,) if N == 32 else ()):
            q = _int_data(vtype, nq, dim, rng)
            _check_scores(ix, x64, q, r0, r1, N)
    ix.close()


@pytest.mark.parametrize("vtype,value,dim", [(po.I8, -128, 4096), (po.U8, 255, 4096), (po.U8, 255, 20000)])
def test_int_scores_extreme_values(vtype, value, dim):
    """all -128 int8 / all 255 uint8; uint8 dim 20000: s = 1.3e9, so 2 s exceeds 2^31 (see test_int_log_when_2s_exceeds_int32)"""
    dt = np.int8 if vtype == po.I8 else np.uint8
    rng = np.random.Generator(np.random.PCG64(dim))
    n = 4000 if dim > 4096 else 20000
    x = np.full((n, dim), value, dtype=dt)
    x[1::2, : dim // 3] = _int_data(vtype, 1, dim // 3, rng)          # some rows not constant
    q = np.full((40, dim), value, dtype=dt)
    q[1] = _int_data(vtype, 1, dim, rng)
    ix = _index(vtype, x)
    for N in (32, 256):
        _check_scores(ix, x.astype(np.float64), q, 128, n - 5, N)
    ix.close()


# ---------------------------------------------------------------------------------------------- (b) integer candidate logs
def _int_hits(vtype, metric, s, norms, qc_bits, valid_q):
    """host tc_hit (batch_kernels.cuh) on exact scores s [rows, nq] (int64), the kernel's norms [rows] and qc bits [nq]"""
    if metric == po.DOT:
        return s > qc_bits.view(np.int32)[None, :].astype(np.int64)
    nn = norms.view(np.uint32).astype(np.int64) if vtype == po.U8 else norms.astype(np.int64)
    if metric in (po.L2, po.L2SQ):
        return (2 * s - nn[:, None]) >= qc_bits.view(np.int32)[None, :].astype(np.int64)
    # cosine: !(fmaf(-qc, rowf, (float)s) < 0) with rowf = __fsqrt_rn((float)nn); the fma is exact before its one rounding,
    # and rounding keeps the sign, so the test is exact in float64 (a product of two floats is exact there)
    rowf = np.sqrt(nn.astype(np.float32)).astype(np.float64)
    qcf = qc_bits.view(np.float32).astype(np.float64)
    s32 = s.astype(np.float32).astype(np.float64)
    return (s32 - qcf[None, :] * rowf[:, None]) >= 0.0


def _exact_distances(metric, s, nn, qq):
    """exact (float64) distances from exact scores and squared norms; cosine of a zero vector is taken as 1"""
    if metric == po.DOT:
        return -s
    if metric in (po.L2, po.L2SQ):
        d2 = np.maximum(qq[None, :] + nn[:, None] - 2.0 * s, 0.0)
        return np.sqrt(d2) if metric == po.L2 else d2
    den = np.sqrt(nn[:, None] * qq[None, :])
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.where(den > 0, 1.0 - s / np.where(den > 0, den, 1.0), 1.0)


def _bounds_at_quantiles(d, rng):
    """per query a bound at one of several quantiles of its exact distances, +INF for some"""
    levels = [1e-3, 1e-2, 0.1, 0.5, np.inf]
    U = np.empty(d.shape[1], dtype=np.float32)
    for j in range(d.shape[1]):
        lv = levels[(j + int(rng.integers(0, 5))) % len(levels)]
        U[j] = np.inf if lv == np.inf else np.float32(np.quantile(d[:, j], lv))
    return U


def _log_set(res, nq, r0, r1):
    log = res["log"]
    rows, qs = log[:, 0].astype(np.int64), log[:, 1].astype(np.int64)
    assert np.all(qs < nq), "a padded query column was logged"
    assert np.all((rows >= r0) & (rows < r1)), "a row outside the level was logged"
    keys = rows * nq + qs
    assert len(np.unique(keys)) == len(keys), "duplicate (row, query) pairs"
    return keys


def _check_int_log(ix, vtype, metric, x64, q, U, r0, r1, N):
    nq = q.shape[0]
    res = ix.debug_tc_level(metric, q, U, r0, r1, N=N)
    s = (x64[r0:r1] @ q.astype(np.float64).T).astype(np.int64)
    hits = _int_hits(vtype, metric, s, res["norms"], res["qc"], nq)
    rr, qq = np.nonzero(hits)
    want = np.sort((rr + r0) * nq + qq)
    got = np.sort(_log_set(res, nq, r0, r1))
    assert res["count"] == len(got)
    if not np.array_equal(got, want):
        missing, extra = np.setdiff1d(want, got), np.setdiff1d(got, want)
        raise AssertionError(f"log != exact hit set ({KIND_NAMES[vtype]}, metric {metric}, N {N}): {len(missing)} missing "
                             f"{[(int(k // nq), int(k % nq)) for k in missing[:4]]}, {len(extra)} extra "
                             f"{[(int(k // nq), int(k % nq)) for k in extra[:4]]}")
    return len(want)


@pytest.mark.parametrize("epi_chunk", [1, 0])
@pytest.mark.parametrize("metric", TC_METRICS)
@pytest.mark.parametrize("vtype", [po.I8, po.U8])
def test_int_log_equals_exact_hits(vtype, metric, epi_chunk):
    rng = np.random.Generator(np.random.PCG64(2000 + 10 * vtype + metric))
    n, dim, nq = 60000, 200, 70
    x = _int_data(vtype, n, dim, rng)
    x[::997] = 0                                             # zero rows: with cosine a padded (+INF) column would hit them
    q = _int_data(vtype, nq, dim, rng)
    q[::3] //= 50                                            # bounds orders of magnitude apart inside one 32-column chunk
    q[1::11] = 0
    x64 = x.astype(np.float64)
    r0, r1 = 256, n - 77
    s = x64[r0:r1] @ q.astype(np.float64).T
    d = _exact_distances(metric, s, (x64[r0:r1] ** 2).sum(1), (q.astype(np.float64) ** 2).sum(1))
    U = _bounds_at_quantiles(d, rng)
    old = _epi_chunk(epi_chunk)
    try:
        ix = _index(vtype, x)
        for N in (0, 32, 64):                                # 0: the production N (128 for 70 queries, 58 padded columns)
            total = _check_int_log(ix, vtype, metric, x64, q, U, r0, r1, N)
        # a cap below the hit count: the raw count still counts every hit, the stored pairs are hits
        cap = max(1, total // 3)
        res = ix.debug_tc_level(metric, q, U, r0, r1, cap=cap)
        assert res["count"] == total and len(res["log"]) == cap
        full = ix.debug_tc_level(metric, q, U, r0, r1)
        assert np.all(np.isin(_log_set(res, nq, r0, r1), _log_set(full, nq, r0, r1)))
        ix.close()
    finally:
        _epi_chunk(old)


@pytest.mark.parametrize("epi_chunk", [1, 0])
def test_int_log_when_2s_exceeds_int32(epi_chunk):
    """uint8 L2 at dim 20000: 2 s ~ 2.6e9 overflows int32 while 2 s - |r|^2 fits; tc_hit's int32 arithmetic must still
    give the exact answer"""
    rng = np.random.Generator(np.random.PCG64(4242))
    n, dim, nq = 3000, 20000, 24
    x = (255 - rng.integers(0, 4, (n, dim))).astype(np.uint8)
    q = (255 - rng.integers(0, 4, (nq, dim))).astype(np.uint8)
    x64 = x.astype(np.float64)
    s = x64[128:] @ q.astype(np.float64).T
    assert s.min() * 2 > 2 ** 31
    d = _exact_distances(po.L2, s, (x64[128:] ** 2).sum(1), (q.astype(np.float64) ** 2).sum(1))
    U = _bounds_at_quantiles(d, rng)
    old = _epi_chunk(epi_chunk)
    try:
        ix = _index(po.U8, x)
        for N in (32, 0):
            assert _check_int_log(ix, po.U8, po.L2, x64, q, U, 128, n, N) > 0
        ix.close()
    finally:
        _epi_chunk(old)


# ---------------------------------------------------------------------------------------------- (c) fp error model
FP_DIMS = [8, 40, 100, 771, 1536, 4096]


def _fp_scores(vtype, family, dim, rng, n=2048, nq=72):
    x = fam.make(family, vtype, n, dim, rng)
    q = fam.make(family, vtype, nq, dim, rng, queries=True)
    ix = _index(vtype, x)
    res = ix.debug_tc_level(po.DOT, q, np.full(nq, np.inf, np.float32), 128, n, scores=True)
    ix.close()
    xd, qd = fam.decode(vtype, x)[128:], fam.decode(vtype, q)
    return res["scores"].astype(np.float64), xd @ qd.T, np.abs(xd) @ np.abs(qd).T


@pytest.mark.parametrize("family", fam.FAMILIES)
@pytest.mark.parametrize("vtype", [po.BF16, po.F16])
def test_fp_scores_within_error_model(vtype, family):
    """|s_tc - s| <= dim * 2^-21 * sum |q_i r_i| for every pair (s and the sum exact in float64: the products are).  Prints
    the largest ratio err / bound per dim: the margin the model leaves on this hardware."""
    rng = np.random.Generator(np.random.PCG64(3000 + 10 * vtype + fam.FAMILIES.index(family)))
    worst = {}
    for dim in FP_DIMS:
        got, s, mag = _fp_scores(vtype, family, dim, rng)
        assert np.all(np.isfinite(got)), (dim, "non-finite score")
        err = np.abs(got - s)
        bound = dim * 2.0 ** -21 * mag
        zero = bound == 0
        assert np.all(err[zero] == 0), (dim, "an all-zero row or query scored non-zero")
        ratio = np.where(zero, 0.0, err / np.where(zero, 1.0, bound))
        worst[dim] = float(ratio.max())
        i, j = np.unravel_index(int(ratio.argmax()), ratio.shape)
        assert worst[dim] <= 1.0, (dim, "row", i + 128, "query", j, "s_tc", got[i, j], "s", s[i, j], "sum|t|", mag[i, j])
    print(f"\ntc_fp_error {KIND_NAMES[vtype]} {family}: max err / (dim 2^-21 sum|q_i r_i|) by dim "
          + " ".join(f"{d}:{r:.3e}" for d, r in worst.items()) + f"  overall {max(worst.values()):.3e}")


# ---------------------------------------------------------------------------------------------- (d) fp logs are supersets
def _near_duplicates(vtype, n, dim, rng):
    """three quarters of the rows are one base row with about 16 elements moved by 1 - 4 units in the last place, so that
    many pairs sit within the tensor-core slack of a bound placed at one of their distances; the rest are unrelated.
    Returns the column and the mask of the near-duplicates."""
    base = po.convert(rng.standard_normal((1, dim)).astype(np.float32), vtype)[0]
    nudge = rng.random((n, dim)) < 16.0 / dim
    step = rng.integers(1, 5, (n, dim)) * np.where(rng.random((n, dim)) < 0.5, -1, 1)
    x = np.where(nudge, base.astype(np.int32)[None, :] + step, base.astype(np.int32)[None, :]).astype(np.uint16)
    dup = rng.random(n) >= 0.25
    x[~dup] = po.convert(rng.standard_normal((int((~dup).sum()), dim)).astype(np.float32), vtype)
    return np.ascontiguousarray(x), dup


def _refine_delta(metric, dim, d, mag):
    """the refine's own documented error (tc_fp_eps): an fp32 FMA chain over dim terms is within dim 2^-24 of the sum of
    their magnitudes.  DOT: dim 2^-24 sum|q_i r_i|.  L2: the sum of squares is within (dim + 1) 2^-24 relative (one more
    rounding per squared difference), the root halves it; dim 2^-24 d bounds both.  COSINE: the score's error relative to
    |q||r| (>= sum|q_i r_i|) plus the two norms' (halved by the root) plus the final divide / subtract: (2 dim + 8) 2^-24."""
    eps = dim * 2.0 ** -24
    if metric == po.DOT:
        return eps * mag
    if metric == po.L2:
        return (dim + 1) * 2.0 ** -24 * d
    return np.full_like(d, (2 * dim + 8) * 2.0 ** -24)


@pytest.mark.parametrize("metric", TC_METRICS)
@pytest.mark.parametrize("vtype", [po.BF16, po.F16])
def test_fp_log_is_superset_at_the_bound(vtype, metric):
    rng = np.random.Generator(np.random.PCG64(5000 + 10 * vtype + metric))
    n, dim, nq = 20000, 771, 40
    x, dup = _near_duplicates(vtype, n, dim, rng)
    q = po.convert(rng.standard_normal((nq, dim)).astype(np.float32), vtype)
    r0, r1 = 128, n
    dup = dup[r0:r1]
    xd, qd = fam.decode(vtype, x)[r0:r1], fam.decode(vtype, q)
    s = xd @ qd.T
    mag = np.abs(xd) @ np.abs(qd).T
    rn, qn = (xd ** 2).sum(1), (qd ** 2).sum(1)
    if metric == po.L2:
        d = np.sqrt(np.maximum(rn[:, None] + qn[None, :] - 2 * s, 0.0))
    else:
        d = _exact_distances(metric, s, rn, qn)
    # U just above the exact distance of a chosen near-duplicate: at rank 10 %, 30 % or 50 % among them
    U = np.empty(nq, dtype=np.float32)
    for j in range(nq):
        dd = np.sort(d[dup, j])
        pick = float(dd[int(len(dd) * [0.1, 0.3, 0.5][j % 3])])
        u = np.float32(pick)
        U[j] = np.nextafter(u, np.float32(np.inf)) if float(u) <= pick else u
    ix = _index(vtype, x)
    res = ix.debug_tc_level(metric, q, U, r0, r1)
    ix.close()
    assert res["count"] == len(res["log"])
    keys = _log_set(res, nq, r0, r1)
    logged = np.zeros((r1 - r0, nq), dtype=bool)
    logged.flat[(keys // nq - r0) * nq + keys % nq] = True
    delta = _refine_delta(metric, dim, d, mag)
    must = d < U.astype(np.float64)[None, :] - delta
    near = (d < U.astype(np.float64)[None, :] + delta) & ~must
    missing = np.argwhere(must & ~logged)
    assert missing.size == 0, (f"{len(missing)} pairs below U - delta not logged", [(int(a) + r0, int(b)) for a, b in missing[:5]])
    assert near.sum() > nq, "the corpus puts too few pairs within the slack of U to test the boundary"
    # no gross false positives: a logged pair passes tc_hit on the EXACT score once the bound is relaxed by twice the modelled
    # tensor-core slack (dim 2^-21 sum|q_i r_i|), plus one rounding of the epilogue's fp32 arithmetic
    slack = 2 * dim * 2.0 ** -21 * mag
    qc = res["qc"].view(np.float32).astype(np.float64)[None, :]
    nn = res["norms"].astype(np.float64)[:, None]
    ulp = 2.0 ** -23
    if metric == po.DOT:
        ok = s + slack + ulp * np.abs(qc) > qc
    elif metric == po.L2:
        eps = np.float64(np.float32(dim * 9.5367431640625e-7))
        rowf = np.float32(-nn * (1 - eps)).astype(np.float64)
        ok = 2 * (s + slack) + rowf + ulp * (np.abs(qc) + np.abs(rowf)) > qc
    else:
        rowf = np.sqrt(nn.astype(np.float32)).astype(np.float64)
        ok = s + slack + ulp * np.abs(qc * rowf) >= qc * rowf
    bad = np.argwhere(logged & ~ok)
    assert bad.size == 0, (f"{len(bad)} logged pairs fail the relaxed test", [(int(a) + r0, int(b)) for a, b in bad[:5]])
