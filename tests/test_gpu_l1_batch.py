"""Batched L1 queries: l1_batch_kernel (CUDA-core scoring on the tensor-core path's tiles) and the batch path's refine / replay
behind it.  -m gpu.

(a) int8 / uint8 batches bit-exact against the oracle and against the per-query path (no_batch);
(b) f32 / f16 / bf16 batches against the oracle under tests/fpcheck.py, plain and adversarial data (tests/fpfamilies.py);
(c) the kernel alone through vsb_debug_tc_level(L1): exact integer scores, fp scores within gamma S of the exact sums, integer
    logs equal to {(r, q) : (float)S < U_q}, fp logs holding every pair any fp32 summation order could put below U;
(d) NaN / Inf rows and queries, rows whose fp32 sum overflows, a bucket overflow that falls back;
(e) 3 row shards on one GPU (batch_shard_scan + batch_merge) and a 3-shard Group;
(f) the SQL batch functions on L1 columns against their per-query counterparts."""
import os
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

from oracle import pyoracle as po
from tests import fpfamilies as fam
from tests.fpcheck import assert_fp_topk

pytestmark = pytest.mark.gpu
FP_TYPES = [po.F32, po.F16, po.BF16]


def _index(vtype, x, rowids=None, first_seq=0):
    import sqlite_vector_b200 as vs
    ix = vs.Index(vtype, x.shape[1], x.shape[0], first_seq=first_seq)
    ix.append_dense(x, rowids)
    ix.finalize()
    return ix


def _ints(vtype, lo, hi, shape, rng):
    if vtype == po.U8:
        lo, hi = 0, hi - lo
    return rng.integers(lo, hi, shape).astype(np.int8 if vtype == po.I8 else np.uint8)


def _batched(ix, q, k):
    """scan_topk of the whole batch; asserts that the batch path ran to the end"""
    b0, f0 = ix.stat("batches"), ix.stat("fallbacks")
    res = ix.scan_topk(po.L1, q, k)
    assert ix.stat("batches") == b0 + 1 and ix.stat("fallbacks") == f0, "the L1 batch path did not run"
    return res


def _no_batch(ix, q, k):
    import sqlite_vector_b200 as vs
    eng = vs.load_engine()
    old = eng.set_option("no_batch", 1)
    try:
        return ix.scan_topk(po.L1, q, k)
    finally:
        eng.set_option("no_batch", old)


def _gamma(dim):
    mu = (dim + 1) * 2.0 ** -24
    return mu / (1 - mu)


def _l1_exact(xd, qd):
    """float64 sums |x - q| [rows, nq] (exact up to float64 rounding, far below the fp32 error under test)"""
    return np.stack([np.abs(xd - qd[j]).sum(1) for j in range(qd.shape[0])], axis=1)


# ---------------------------------------------------------------------------------------------- (a) integer batches
# (n, dim, nq, k, value range): dims 16 / 48 are shorter than one 128-byte K slice; k = 200 / 256 exceed the 128 rows refined
# exhaustively, so the first L1 level runs with U = +INF; narrow ranges make ties at the k-th place
INT_CASES = [(20000, 16, 16, 20, (-128, 128)), (30000, 48, 33, 200, (-2, 3)), (20000, 771, 100, 1, (-2, 3)),
             (10000, 1536, 300, 256, (-20, 21)), (24000, 771, 16, 33, (-128, 128))]


@pytest.mark.parametrize("case", range(len(INT_CASES)))
@pytest.mark.parametrize("vtype", [po.I8, po.U8])
def test_int_batch_bit_exact(oracle, vtype, case):
    n, dim, nq, k, (lo, hi) = INT_CASES[case]
    rng = np.random.Generator(np.random.PCG64(100 * case + vtype))
    x = _ints(vtype, lo, hi, (n, dim), rng)
    q = _ints(vtype, lo, hi, (nq, dim), rng)
    rowids = np.arange(n, dtype=np.int64) * 3 + 7
    ix = _index(vtype, x, rowids)
    res = _batched(ix, q, k)
    loop = _no_batch(ix, q, k)
    for b in range(nq):
        assert np.array_equal(res[b][0], loop[b][0]) and np.array_equal(res[b][1], loop[b][1]), (n, dim, nq, k, b)
    for b in sorted({0, nq // 3, nq // 2, nq - 1}):
        want_ids, want_d = oracle.scan_dense(po.L1, vtype, q[b], x, rowids, k)
        assert np.array_equal(res[b][0], want_ids) and np.array_equal(res[b][1], want_d), (n, dim, nq, k, b)
    ix.close()


# ---------------------------------------------------------------------------------------------- (b) fp batches
FP_CASES = [(20000, 128, 40, 20, None), (30000, 771, 70, 20, None), (20000, 771, 33, 20, "dominant"), (20000, 24, 17, 20, "wide"),
            (20000, 200, 130, 20, "cancel"), (20000, 24, 20, 33, "tiny"), (20000, 100, 16, 20, "huge")]


def _fp_check(oracle, vtype, x, q, k, res, ctx):
    rowids = np.arange(1, x.shape[0] + 1, dtype=np.int64)
    with ThreadPoolExecutor(16) as ex:                       # the oracle's C loop releases the GIL
        wants = list(ex.map(lambda b: oracle.scan_dense(po.L1, vtype, q[b], x, rowids, k), range(q.shape[0])))
    for b in range(q.shape[0]):
        want_ids, want_d = wants[b]
        assert_fp_topk(res[b][0], res[b][1], want_ids, want_d, po.L1,
                       lambda r, b=b: oracle.distance(po.L1, vtype, q[b], x[r - 1]), ctx + (b,))


@pytest.mark.parametrize("case", range(len(FP_CASES)))
@pytest.mark.parametrize("vtype", FP_TYPES)
def test_fp_batch_matches_oracle_every_query(oracle, vtype, case):
    n, dim, nq, k, family = FP_CASES[case]
    if (family == "tiny" and vtype != po.F16) or (family == "huge" and vtype == po.F16):
        pytest.skip("family not defined for this type")
    rng = np.random.Generator(np.random.PCG64(300 + 10 * case + vtype))
    if family is None:
        x = po.convert(rng.standard_normal((n, dim), dtype=np.float32), vtype)
        q = po.convert(rng.standard_normal((nq, dim), dtype=np.float32), vtype)
    else:
        x = fam.make(family, vtype, n, dim, rng)
        q = fam.make(family, vtype, nq, dim, rng, queries=True)
    ix = _index(vtype, x)
    res = _batched(ix, q, k)
    ix.close()
    _fp_check(oracle, vtype, x, q, k, res, (vtype, n, dim, family))


# ---------------------------------------------------------------------------------------------- (c) the kernel alone
@pytest.mark.parametrize("vtype", [po.I8, po.U8])
def test_kernel_int_scores_exact(vtype):
    rng = np.random.Generator(np.random.PCG64(40 + vtype))
    for n, dim in [(20000, 16), (12000, 200), (9000, 771)]:
        x = _ints(vtype, -128, 128, (n, dim), rng)
        ix = _index(vtype, x)
        r0, r1 = 256, n - 37
        xd = x[r0:r1].astype(np.float64)
        for N in (32, 64, 128):
            for nq in (N, 2 * N + 5) + ((20,) if N == 32 else ()):
                q = _ints(vtype, -128, 128, (nq, dim), rng)
                res = ix.debug_tc_level(po.L1, q, np.full(nq, np.inf, np.float32), r0, r1, N=N, scores=True)
                want = _l1_exact(xd, q.astype(np.float64)).astype(np.int64)
                bad = np.argwhere(res["scores"].astype(np.int64) != want)
                assert bad.size == 0, (dim, N, nq, "first wrong (row - r0, query):", bad[:5].tolist(), len(bad))
        ix.close()


@pytest.mark.parametrize("family", ("normal", "wide", "dominant", "tiny", "huge"))
@pytest.mark.parametrize("vtype", FP_TYPES)
def test_kernel_fp_scores_within_gamma(vtype, family):
    """|s - S| <= gamma S, gamma = m 2^-24 / (1 - m 2^-24), m = dim + 1: the bound conservative_qc builds on"""
    if (family == "tiny" and vtype != po.F16) or (family == "huge" and vtype == po.F16):
        pytest.skip("family not defined for this type")
    rng = np.random.Generator(np.random.PCG64(50 + 10 * vtype + len(family)))
    worst = {}
    for dim in (8, 40, 771, 1536):
        n, nq = 2048, 72
        x = fam.make(family, vtype, n, dim, rng)
        q = fam.make(family, vtype, nq, dim, rng, queries=True)
        ix = _index(vtype, x)
        res = ix.debug_tc_level(po.L1, q, np.full(nq, np.inf, np.float32), 128, n, scores=True)
        ix.close()
        S = _l1_exact(fam.decode(vtype, x)[128:], fam.decode(vtype, q))
        got = res["scores"].astype(np.float64)
        assert np.all(np.isfinite(got)), (dim, "non-finite score")
        err = np.abs(got - S)
        bound = _gamma(dim) * S
        assert np.all(err <= bound), (dim, float((err / np.maximum(bound, 1e-300)).max()))
        worst[dim] = float((err / np.maximum(bound, 1e-300)).max())
    print(f"\nl1_fp_error type {vtype} {family}: max err / (gamma S) by dim " + " ".join(f"{d}:{r:.3e}" for d, r in worst.items()))


def _log_set(res, nq, r0, r1):
    log = res["log"]
    rows, qs = log[:, 0].astype(np.int64), log[:, 1].astype(np.int64)
    assert np.all(qs < nq), "a padded query column was logged"
    assert np.all((rows >= r0) & (rows < r1)), "a row outside the level was logged"
    keys = rows * nq + qs
    assert len(np.unique(keys)) == len(keys), "duplicate (row, query) pairs"
    assert res["count"] == len(keys)
    return keys


def _bounds_at_quantiles(S, rng):
    levels = [0.0, 1e-3, 1e-2, 0.1, 0.5, np.inf]
    U = np.empty(S.shape[1], dtype=np.float32)
    for j in range(S.shape[1]):
        lv = levels[(j + int(rng.integers(0, len(levels)))) % len(levels)]
        U[j] = np.inf if lv == np.inf else np.float32(np.quantile(S[:, j], lv))
    return U


@pytest.mark.parametrize("vtype", [po.I8, po.U8])
def test_kernel_int_log_equals_exact_hits(vtype):
    rng = np.random.Generator(np.random.PCG64(60 + vtype))
    n, dim, nq = 40000, 200, 70
    x = _ints(vtype, -10, 11, (n, dim), rng)
    q = _ints(vtype, -10, 11, (nq, dim), rng)
    r0, r1 = 256, n - 77
    S = _l1_exact(x[r0:r1].astype(np.float64), q.astype(np.float64))
    U = _bounds_at_quantiles(S, rng)
    ix = _index(vtype, x)
    for N in (0, 32, 64, 128):                               # 0: the production N (128 for 70 queries: 58 padded columns)
        res = ix.debug_tc_level(po.L1, q, U, r0, r1, N=N)
        got = np.sort(_log_set(res, nq, r0, r1))
        rr, qq = np.nonzero(S.astype(np.float32) < U[None, :])
        want = np.sort((rr + r0) * nq + qq)
        assert np.array_equal(got, want), (N, len(got), len(want))
    ix.close()


@pytest.mark.parametrize("vtype", FP_TYPES)
def test_kernel_fp_log_holds_every_pair_below_the_bound(vtype):
    """every pair that ANY fp32 order of the sum could put below U (S < U / (1 - gamma)) is logged, in particular every pair
    whose single-query distance is below U; and no logged pair lies beyond qc / (1 - gamma)"""
    rng = np.random.Generator(np.random.PCG64(70 + vtype))
    n, dim, nq = 20000, 771, 40
    base = rng.standard_normal((1, dim)).astype(np.float32)
    x = base + (rng.random((n, dim)) < 16.0 / dim) * rng.standard_normal((n, dim)).astype(np.float32) * 1e-3
    x[rng.random(n) < 0.25] = rng.standard_normal((1, dim)).astype(np.float32)
    x = po.convert(x.astype(np.float32), vtype)
    q = po.convert((base + 1e-2 * rng.standard_normal((nq, dim))).astype(np.float32), vtype)
    r0, r1 = 128, n
    S = _l1_exact(fam.decode(vtype, x)[r0:r1], fam.decode(vtype, q))
    U = np.empty(nq, dtype=np.float32)
    for j in range(nq):                                      # just above an exact sum at rank 0.1 / 1 / 10 %
        pick = float(np.sort(S[:, j])[int(len(S) * [0.001, 0.01, 0.1][j % 3])])
        u = np.float32(pick)
        U[j] = np.nextafter(u, np.float32(np.inf)) if float(u) <= pick else u
    ix = _index(vtype, x)
    res = ix.debug_tc_level(po.L1, q, U, r0, r1)
    keys = _log_set(res, nq, r0, r1)
    logged = np.zeros((r1 - r0, nq), dtype=bool)
    logged.flat[(keys // nq - r0) * nq + keys % nq] = True
    g = _gamma(dim)
    must = S < U.astype(np.float64)[None, :] / (1 - g)
    missing = np.argwhere(must & ~logged)
    assert missing.size == 0, (len(missing), [(int(a) + r0, int(b)) for a, b in missing[:5]])
    for j in range(0, nq, 7):
        d = ix.scan_all(po.L1, q[j])[r0:r1]
        assert np.all(logged[d < U[j], j]), j
    qc = res["qc"].view(np.float32).astype(np.float64)
    assert np.all(S[logged] < np.broadcast_to(qc[None, :], S.shape)[logged] / (1 - g))
    ix.close()


# ---------------------------------------------------------------------------------------------- (d) edge data
@pytest.mark.parametrize("vtype", FP_TYPES)
def test_nan_inf_rows_and_queries(oracle, vtype):
    """NaN / +-Inf elements in rows (in the exhaustive prefix and in later levels) and in queries: the oracle's result
    classes (f16 skips NaN lanes, so such a row keeps a finite distance; f32 / bf16 rows become NaN and never enter)"""
    rng = np.random.Generator(np.random.PCG64(80 + vtype))
    n, dim, nq, k = 20000, 64, 24, 20
    xf = rng.standard_normal((n, dim)).astype(np.float32)
    qf = rng.standard_normal((nq, dim)).astype(np.float32)
    rows = rng.choice(n, 300, replace=False)
    rows[:6] = [0, 5, 100, 127, 128, 3000]
    for i, r in enumerate(rows):
        xf[r, rng.integers(0, dim, 1 + i % 3)] = [np.nan, np.inf, -np.inf][i % 3]
    qf[1, 3] = np.nan
    qf[2, 7] = np.inf
    qf[3, 0] = -np.inf
    qf[4, :2] = [np.inf, np.nan]
    x, q = po.convert(xf, vtype), po.convert(qf, vtype)
    ix = _index(vtype, x)
    b0, f0 = ix.stat("batches"), ix.stat("fallbacks")
    res = ix.scan_topk(po.L1, q, k)
    assert ix.stat("batches") + ix.stat("fallbacks") == b0 + f0 + 1
    ix.close()
    _fp_check(oracle, vtype, x, q, k, res, (vtype, "nan/inf"))


@pytest.mark.parametrize("vtype", [po.F32, po.BF16])
def test_rows_whose_sum_overflows(oracle, vtype):
    """rows whose fp32 L1 sum overflows (one term, or only the sum) have distance +INF and never enter the slots"""
    rng = np.random.Generator(np.random.PCG64(90 + vtype))
    n, dim, nq, k = 20000, 32, 16, 20
    xf = rng.standard_normal((n, dim)).astype(np.float32)
    qf = rng.standard_normal((nq, dim)).astype(np.float32)
    big = np.float32(2.5e38)
    xf[::97, 0] = big                                        # |big - (-big)| overflows in one term
    qf[:, 0] = np.where(np.arange(nq) % 2 == 0, -big, qf[:, 0])
    xf[50::131] = big / 8                                    # every term finite, the sum of 32 of them is not
    x, q = po.convert(xf, vtype), po.convert(qf, vtype)
    ix = _index(vtype, x)
    res = _batched(ix, q, k)
    ix.close()
    _fp_check(oracle, vtype, x, q, k, res, (vtype, "overflow"))


def test_bucket_overflow_falls_back_exactly(oracle):
    """descending L1 distances along the scan: every row enters the slots, a level's bucket overflows, the call falls back
    to the per-query path and the result stays exact"""
    n, dim, nq, k = 40000, 64, 16, 5
    x = np.zeros((n, dim), dtype=np.int8)
    x[:, 0] = np.clip((n - 1 - np.arange(n)) // 320, 0, 124).astype(np.int8)
    x[:, 1] = ((n - 1 - np.arange(n)) % 320 // 3).astype(np.int8)
    q = np.zeros((nq, dim), dtype=np.int8)
    ix = _index(po.I8, x)
    f0 = ix.stat("fallbacks")
    res = ix.scan_topk(po.L1, q, k)
    assert ix.stat("fallbacks") == f0 + 1
    rowids = np.arange(1, n + 1, dtype=np.int64)
    for b in (0, nq - 1):
        want_ids, want_d = oracle.scan_dense(po.L1, po.I8, q[b], x, rowids, k)
        assert np.array_equal(res[b][0], want_ids) and np.array_equal(res[b][1], want_d)
    ix.close()


# ---------------------------------------------------------------------------------------------- (e) shards and groups
def test_row_shards_bit_exact(oracle):
    from tests.test_gpu_batch import _sharded_batch
    rng = np.random.Generator(np.random.PCG64(95))
    n, dim, nq, k = 60000, 128, 40, 20
    x = rng.integers(-3, 4, (n, dim)).astype(np.int8)
    q = rng.integers(-3, 4, (nq, dim)).astype(np.int8)
    rowids = np.arange(n, dtype=np.int64) * 3 + 7
    bounds = [0, n // 4 + 11, (2 * n) // 3, n]
    shards = [_index(po.I8, x[a:b], rowids[a:b], first_seq=a) for a, b in zip(bounds[:-1], bounds[1:])]
    b0 = [s.stat("batches") for s in shards]
    res = _sharded_batch(shards, bounds, po.L1, q, k)
    assert [s.stat("batches") for s in shards] == [v + 1 for v in b0]
    whole = _index(po.I8, x, rowids)
    one = _batched(whole, q, k)
    for b in range(nq):
        assert np.array_equal(res[b][0], one[b][0]) and np.array_equal(res[b][1], one[b][1]), b
    for b in (0, nq // 2, nq - 1):
        want_ids, want_d = oracle.scan_dense(po.L1, po.I8, q[b], x, rowids, k)
        assert np.array_equal(res[b][0], want_ids) and np.array_equal(res[b][1], want_d), b
    for s in shards + [whole]:
        s.close()


def test_group_of_three_bit_exact(oracle, monkeypatch):
    """a 3-shard Group (shards wrap around the visible GPUs): batched L1 through the gathered entry logs"""
    import sqlite_vector_b200 as vs
    monkeypatch.setenv("VSB_GROUP_ALIAS", "1")
    rng = np.random.Generator(np.random.PCG64(96))
    n, dim, nq, k = 50000, 64, 32, 20
    x = rng.integers(-5, 6, (n, dim)).astype(np.int8)
    q = rng.integers(-5, 6, (nq, dim)).astype(np.int8)
    g = vs.Group(po.I8, dim, n, 3)
    g.append_dense(x)
    g.finalize()
    lib = g.eng.lib
    shard0 = lib.vsb_group_shard(g.h, 0)
    b0 = lib.vsb_index_stat(shard0, b"batches")
    res = g.scan_topk(po.L1, q, k)
    assert lib.vsb_index_stat(shard0, b"batches") == b0 + 1, "the group's batch path did not run"
    rowids = np.arange(1, n + 1, dtype=np.int64)
    for b in range(nq):
        want_ids, want_d = oracle.scan_dense(po.L1, po.I8, q[b], x, rowids, k)
        assert np.array_equal(res[b][0], want_ids) and np.array_equal(res[b][1], want_d), b
    g.close()


# ---------------------------------------------------------------------------------------------- (f) SQL
def _sql_table(vtype_name, x):
    s = ["CREATE TABLE t (id INTEGER PRIMARY KEY, e BLOB)", f"SELECT vector_init('t','e','type={vtype_name},dimension={x.shape[1]},distance=L1')"]
    for i in range(x.shape[0]):
        s.append(["INSERT INTO t(id, e) VALUES (?, ?)", [3 * i + 2, {"hex": x[i].tobytes().hex()}]])
    return s


def test_sql_quantize_scan_batch_int8_l1():
    from tests.sqlrun import OURS, run_sql
    rng = np.random.Generator(np.random.PCG64(97))
    n, dim, nq, k = 9000, 16, 20, 7
    x = rng.integers(-20, 21, (n, dim)).astype(np.int8)
    q = rng.integers(-20, 21, (nq, dim)).astype(np.int8)
    s = _sql_table("INT8", x) + ["SELECT vector_quantize('t','e')"]
    s.append(["SELECT query, id, distance FROM vector_quantize_scan_batch('t','e',?,?)", [{"hex": q.tobytes().hex()}, k]])
    for b in range(nq):
        s.append(["SELECT id, distance FROM vector_quantize_scan('t','e',?,?)", [{"hex": q[b].tobytes().hex()}, k]])
    r = run_sql(OURS, s)
    off = len(s) - (nq + 1)
    batch = r[off]["rows"]
    assert len(batch) == nq * k, r[off]
    for b in range(nq):
        assert [row[1:] for row in batch if row[0] == b] == r[off + 1 + b]["rows"], b


def test_sql_full_scan_batch_f32_l1():
    from tests.sqlrun import OURS, run_sql
    rng = np.random.Generator(np.random.PCG64(98))
    n, dim, nq, k = 9000, 16, 20, 7
    x = rng.standard_normal((n, dim)).astype(np.float32)
    q = rng.standard_normal((nq, dim)).astype(np.float32)
    s = _sql_table("FLOAT32", x)
    s.append(["SELECT query, id, distance FROM vector_full_scan_batch('t','e',?,?)", [{"hex": q.tobytes().hex()}, k]])
    for b in range(nq):
        s.append(["SELECT id, distance FROM vector_full_scan('t','e',?,?)", [{"hex": q[b].tobytes().hex()}, k]])
    r = run_sql(OURS, s)
    off = len(s) - (nq + 1)
    batch = r[off]["rows"]
    assert len(batch) == nq * k, r[off]
    for b in range(nq):
        got = [row[1:] for row in batch if row[0] == b]
        want = r[off + 1 + b]["rows"]
        gi, gd = np.array([v[0] for v in got]), np.array([v[1] for v in got])
        wi, wd = np.array([v[0] for v in want]), np.array([v[1] for v in want])
        assert_fp_topk(gi, gd, wi, wd, po.L1, lambda rid, b=b: float(np.abs(x[(rid - 2) // 3].astype(np.float64) - q[b]).sum()), (b,))
