"""Batched f32 L2 / squared L2 / cosine / dot queries on the tensor cores (option f32_batch): tc_scan_kernel<TK_TF32, ...>
scores the levels in TF32, the batch path's exact refine and replay stand behind it.  -m gpu.

(a) TF32 scores stay within the error model of tc_tf32_eps on every input family, and whether the hardware truncates or rounds;
(b) the candidate log holds every pair below the bound when the rows differ only below tf32 resolution;
(c) results against the oracle for every query (tests/fpcheck.py), every tile width, k = 20 and 100; the option off leaves f32
    batches on the per-query path;
(d) NaN / Inf rows and queries, rows and queries whose fp32 norm overflows, zero vectors, subnormals;
(e) row shards, 2- and 3-shard groups, vector_full_scan_batch, a bucket overflow that falls back, the tile widths."""
import contextlib
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

from oracle import pyoracle as po
from tests import fpfamilies as fam
from tests.fpcheck import assert_fp_topk

pytestmark = pytest.mark.gpu
METRICS = [po.L2, po.L2SQ, po.COS, po.DOT]
TC_METRICS = [po.L2, po.COS, po.DOT]


def _vs():
    import sqlite_vector_b200 as vs
    return vs


@contextlib.contextmanager
def _f32_batch(value):
    eng = _vs().load_engine()
    old = eng.set_option("f32_batch", value)
    try:
        yield
    finally:
        eng.set_option("f32_batch", old)


@pytest.fixture(autouse=True)
def f32_batch_on():
    with _f32_batch(1):
        yield


def _index(x, rowids=None, first_seq=0):
    ix = _vs().Index(po.F32, x.shape[1], x.shape[0], first_seq=first_seq)
    ix.append_dense(x, rowids)
    ix.finalize()
    return ix


def _normal(rng, n, dim):
    return rng.standard_normal((n, dim), dtype=np.float32)


def _model(dim):
    """the TF32 error model relative to sum |q_i r_i|: both operands within 2^-10 (truncated), products exact, the
    accumulation within dim 2^-21 of the (slightly larger) products' magnitudes"""
    op = 2.0 ** -9 + 2.0 ** -20
    return op + dim * 2.0 ** -21 * (1 + op)


def _tf32(a, rounding):
    b = np.ascontiguousarray(a, dtype=np.float32).view(np.uint32).astype(np.uint64)
    if rounding:
        b = b + 0xFFF + ((b >> 13) & 1)
    return (b & 0xFFFFE000).astype(np.uint32).view(np.float32).astype(np.float64)


# ---------------------------------------------------------------------------------------------- (a) error model
FP_DIMS = [8, 40, 100, 384, 771, 1536, 4096]


def _lowbits(rng, n, dim):
    """positive values whose 13 mantissa bits below tf32 resolution are all set: truncation loses the most, and every
    product's error has the same sign; rows 0 and every 61st are zero like the other families"""
    v = np.abs(rng.standard_normal((n, dim))).astype(np.float32) + np.float32(2.0 ** -20)
    x = (v.view(np.uint32) | np.uint32(0x1FFF)).view(np.float32)
    x[0] = 0
    x[::61] = 0
    return x


@pytest.mark.parametrize("family", fam.FAMILIES + ("huge", "lowbits"))
def test_tf32_scores_within_error_model(family):
    """|s_tc - s| <= ((2^-9 + 2^-20) + dim 2^-21 (1 + 2^-9 + 2^-20)) sum |q_i r_i| for every pair, s and the sum exact in
    float64; all-zero rows and queries score exactly 0.  Prints the largest ratio err / bound per dim; the "lowbits" family
    also prints whether the scores follow truncated or rounded operands."""
    rng = np.random.Generator(np.random.PCG64(6000 + len(family)))
    worst, verdict = {}, {}
    n, nq = 2048, 72
    for dim in FP_DIMS:
        if family == "lowbits":
            x, q = _lowbits(rng, n, dim), _lowbits(rng, nq, dim)
        else:
            x, q = fam.make(family, po.F32, n, dim, rng), fam.make(family, po.F32, nq, dim, rng, queries=True)
        if family == "huge":
            q[:, :] = rng.standard_normal((nq, dim)).astype(np.float32) * np.float32(2.0 ** -70)   # products stay finite
        ix = _index(x)
        res = ix.debug_tc_level(po.DOT, q, np.full(nq, np.inf, np.float32), 128, n, scores=True)
        ix.close()
        xd, qd = x[128:].astype(np.float64), q.astype(np.float64)
        got, s, mag = res["scores"].astype(np.float64), xd @ qd.T, np.abs(xd) @ np.abs(qd).T
        assert np.all(np.isfinite(got)), (family, dim, "non-finite score")
        err = np.abs(got - s)
        bound = _model(dim) * mag
        zero = bound == 0
        assert np.all(err[zero] == 0), (family, dim, "an all-zero row or query scored non-zero")
        ratio = np.where(zero, 0.0, err / np.where(zero, 1.0, bound))
        worst[dim] = float(ratio.max())
        i, j = np.unravel_index(int(ratio.argmax()), ratio.shape)
        assert worst[dim] <= 1.0, (family, dim, "row", i + 128, "query", j, "s_tc", got[i, j], "s", s[i, j], "sum|t|", mag[i, j])
        if family == "lowbits":
            e_trunc = np.abs(got - _tf32(x[128:], False) @ _tf32(q, False).T).mean()
            e_round = np.abs(got - _tf32(x[128:], True) @ _tf32(q, True).T).mean()
            verdict[dim] = "truncates" if e_trunc < e_round else "rounds"
    print(f"\ntc_tf32_error {family}: max err / model by dim " + " ".join(f"{d}:{r:.3e}" for d, r in worst.items())
          + f"  overall {max(worst.values()):.3e}" + (f"  operands: {sorted(set(verdict.values()))}" if verdict else ""))
    if verdict:
        assert len(set(verdict.values())) == 1, verdict


# ---------------------------------------------------------------------------------------------- (b) superset at the bound
def _near_duplicates(rng, n, dim):
    """three quarters of the rows are one base row with the 13 mantissa bits below tf32 resolution of every element redrawn
    (identical in tf32, different in f32); the rest are unrelated.  Returns the column and the mask of the near-duplicates."""
    base = rng.standard_normal(dim).astype(np.float32)
    low = rng.integers(0, 1 << 13, (n, dim)).astype(np.uint32)
    x = ((base.view(np.uint32) & np.uint32(0xFFFFE000))[None, :] | low).view(np.float32)
    dup = rng.random(n) >= 0.25
    x[~dup] = rng.standard_normal((int((~dup).sum()), dim)).astype(np.float32)
    return np.ascontiguousarray(x), dup


def _refine_delta(metric, dim, d, mag):
    """the refine's own error, generously: an fp32 chain over dim terms each formed with up to three roundings (difference,
    square or product, add) is within (3 dim + 8) 2^-24 of the sum of their magnitudes; the root halves it for L2"""
    eps = (3 * dim + 8) * 2.0 ** -24
    if metric == po.DOT:
        return eps * mag
    if metric == po.L2:
        return eps * d
    return np.full_like(d, 2 * eps)


@pytest.mark.parametrize("metric", TC_METRICS)
def test_tf32_log_is_superset_at_the_bound(metric):
    rng = np.random.Generator(np.random.PCG64(7000 + metric))
    n, dim, nq = 20000, 771, 40
    x, dup = _near_duplicates(rng, n, dim)
    q = _normal(rng, nq, dim)
    r0, r1 = 128, n
    dup = dup[r0:r1]
    xd, qd = x[r0:r1].astype(np.float64), q.astype(np.float64)
    s = xd @ qd.T
    mag = np.abs(xd) @ np.abs(qd).T
    rn, qn = (xd ** 2).sum(1), (qd ** 2).sum(1)
    if metric == po.L2:
        d = np.sqrt(np.maximum(rn[:, None] + qn[None, :] - 2 * s, 0.0))
    elif metric == po.DOT:
        d = -s
    else:
        d = 1.0 - s / np.sqrt(rn[:, None] * qn[None, :])
    # U just above the exact distance of a chosen near-duplicate: at rank 10 %, 30 % or 50 % among them
    U = np.empty(nq, dtype=np.float32)
    for j in range(nq):
        dd = np.sort(d[dup, j])
        pick = float(dd[int(len(dd) * [0.1, 0.3, 0.5][j % 3])])
        u = np.float32(pick)
        U[j] = np.nextafter(u, np.float32(np.inf)) if float(u) <= pick else u
    ix = _index(x)
    res = ix.debug_tc_level(metric, q, U, r0, r1)
    ix.close()
    log = res["log"].astype(np.int64)
    assert res["count"] == len(log)
    assert np.all((log[:, 0] >= r0) & (log[:, 0] < r1) & (log[:, 1] < nq))
    logged = np.zeros((r1 - r0, nq), dtype=bool)
    logged[log[:, 0] - r0, log[:, 1]] = True
    assert logged.sum() == len(log), "duplicate (row, query) pairs"
    delta = _refine_delta(metric, dim, d, mag)
    must = d < U.astype(np.float64)[None, :] - delta
    near = (d < U.astype(np.float64)[None, :] + delta) & ~must
    missing = np.argwhere(must & ~logged)
    assert missing.size == 0, (f"{len(missing)} pairs below U - delta not logged", [(int(a) + r0, int(b)) for a, b in missing[:5]])
    assert near.sum() > nq, "the corpus puts too few pairs within the slack of U to test the boundary"
    # no gross false positives: a logged pair passes tc_hit on the EXACT score once the bound is relaxed by twice the modelled
    # TF32 slack, plus one rounding of the epilogue's fp32 arithmetic
    slack = 2 * _model(dim) * mag
    qc = res["qc"].view(np.float32).astype(np.float64)[None, :]
    nn = res["norms"].astype(np.float64)[:, None]
    ulp = 2.0 ** -23
    if metric == po.DOT:
        ok = s + slack + ulp * np.abs(qc) > qc
    elif metric == po.L2:
        eps = np.float64(np.float32(2.0 ** -8 + dim * 2.0 ** -20))
        rowf = np.float32(-nn * (1 - eps)).astype(np.float64)
        ok = 2 * (s + slack) + rowf + ulp * (np.abs(qc) + np.abs(rowf)) > qc
    else:
        rowf = np.sqrt(nn.astype(np.float32)).astype(np.float64)
        ok = s + slack + ulp * np.abs(qc * rowf) >= qc * rowf
    bad = np.argwhere(logged & ~ok)
    assert bad.size == 0, (f"{len(bad)} logged pairs fail the relaxed test", [(int(a) + r0, int(b)) for a, b in bad[:5]])
    print(f"\ntf32 log {po.METRIC_NAMES[metric]}: {len(log)} pairs logged, {int(must.sum())} below U - delta")


# ---------------------------------------------------------------------------------------------- (c) against the oracle
def _batched(ix, metric, q, k):
    b0, f0, us0 = ix.stat("batches"), ix.stat("fallbacks"), ix.stat("tc_us")
    res = ix.scan_topk(metric, q, k)
    assert ix.stat("batches") == b0 + 1 and ix.stat("fallbacks") == f0, "the f32 batch path did not run to the end"
    assert ix.stat("tc_us") > us0, "no tensor-core level ran"
    return res


def _oracle_check(oracle, metric, x, q, k, res, ctx):
    rowids = np.arange(1, x.shape[0] + 1, dtype=np.int64)
    with ThreadPoolExecutor(16) as ex:                       # the oracle's C loop releases the GIL
        wants = list(ex.map(lambda b: oracle.scan_dense(metric, po.F32, q[b], x, rowids, k), range(q.shape[0])))
    for b in range(q.shape[0]):
        want_ids, want_d = wants[b]
        got_ids, got_d = res[b]
        assert len(got_d) == len(want_d), ctx + (b,)
        inf = np.isinf(want_d)                               # -INF distances (DOT against an Inf element) lead the list
        assert np.array_equal(got_d[inf], want_d[inf]) and np.array_equal(got_ids[inf], want_ids[inf]), ctx + (b, "infinite part")
        fin = ~inf
        assert_fp_topk(got_ids[fin], got_d[fin], want_ids[fin], want_d[fin], metric,
                       lambda r, b=b: oracle.distance(metric, po.F32, q[b], x[r - 1]), ctx + (b,))


# (dim, k, B): every tile width (B 16 / 40 -> N 32 / 64, 300 / 1024 -> N 128 with 3 and 8 query groups)
CASES = [(128, 20, 16), (384, 20, 1024), (771, 100, 300), (1536, 100, 40)]


@pytest.mark.parametrize("case", range(len(CASES)))
@pytest.mark.parametrize("metric", METRICS)
def test_f32_batch_matches_oracle_every_query(oracle, metric, case):
    dim, k, nq = CASES[case]
    rng = np.random.Generator(np.random.PCG64(8000 + 10 * case + metric))
    n = 12000
    x, q = _normal(rng, n, dim), _normal(rng, nq, dim)
    ix = _index(x)
    res = _batched(ix, metric, q, k)
    with _f32_batch(0):                                      # the default: f32 batches of these metrics run per query
        b0 = ix.stat("batches")
        off = ix.scan_topk(metric, q[:16], k)
        assert ix.stat("batches") == b0
    ix.close()
    _oracle_check(oracle, metric, x, q, k, res, (po.METRIC_NAMES[metric], dim, k, nq))
    for b in range(16):                                      # the per-query path agrees within the same tolerance
        assert_fp_topk(res[b][0], res[b][1], off[b][0], off[b][1], metric, lambda r, b=b: oracle.distance(metric, po.F32, q[b], x[r - 1]), (b,))


@pytest.mark.parametrize("family", ("dominant", "wide"))
def test_f32_batch_adversarial_families(oracle, family):
    """families whose results the oracle's tolerance can judge ("cancel" sums to a small residue of large f32 products, so
    any two fp32 orders of the sum already differ beyond it; tests (a) and (b) cover it)"""
    rng = np.random.Generator(np.random.PCG64(8500 + len(family)))
    n, dim, nq, k = 20000, 771, 40, 20
    x = fam.make(family, po.F32, n, dim, rng, span=20)
    q = fam.make(family, po.F32, nq, dim, rng, queries=True, span=20)
    ix = _index(x)
    for metric in METRICS:
        res = _batched(ix, metric, q, k)
        _oracle_check(oracle, metric, x, q, k, res, (family, po.METRIC_NAMES[metric]))
    ix.close()


# ---------------------------------------------------------------------------------------------- (d) special values
@pytest.mark.parametrize("metric", METRICS)
def test_f32_batch_special_values(oracle, metric):
    """NaN / +-Inf elements in rows (in the exhaustive prefix and in later levels) and in queries; rows and queries whose
    fp32 sum of squares overflows (one query a copy of such a row: a finite L2 distance); zero rows and a zero query;
    subnormal elements in rows and queries"""
    rng = np.random.Generator(np.random.PCG64(9000 + metric))
    n, dim, nq, k = 20000, 64, 24, 20
    x, q = _normal(rng, n, dim), _normal(rng, nq, dim)
    rows = rng.choice(np.arange(200, n), 300, replace=False)
    rows[:6] = [0, 5, 100, 127, 128, 3000]
    for i, r in enumerate(rows):
        x[r, rng.integers(0, dim, 1 + i % 3)] = [np.nan, np.inf, -np.inf][i % 3]
    huge = rng.choice(np.setdiff1d(np.arange(n), rows), 40, replace=False)
    x[huge, rng.integers(0, dim, huge.size)] = np.float32(2.0 ** 100) * np.where(rng.random(huge.size) < 0.5, -1, 1).astype(np.float32)
    sub = rng.choice(np.arange(n), 500, replace=False)
    x[sub[:, None], rng.integers(0, dim, (sub.size, 8))] = rng.standard_normal((sub.size, 8)).astype(np.float32) * np.float32(1e-40)
    x[7777] = 0
    x[64] = 0
    q[1, 3] = np.nan
    q[2, 7] = np.inf
    q[3, 0] = -np.inf
    q[4, :2] = [np.inf, np.nan]
    q[5] = x[huge[3]]                                        # its own norm overflows; distance 0 to that row
    q[6] = x[huge[7]] + rng.standard_normal(dim).astype(np.float32) * np.float32(1e-3)
    q[7] = 0
    q[8, ::3] = rng.standard_normal(len(range(0, dim, 3))).astype(np.float32) * np.float32(1e-39)
    q[9] = np.float32(1e-41)                                 # an all-subnormal query
    ix = _index(x)
    b0, f0 = ix.stat("batches"), ix.stat("fallbacks")
    res = ix.scan_topk(metric, q, k)
    assert ix.stat("batches") + ix.stat("fallbacks") == b0 + f0 + 1
    ix.close()
    _oracle_check(oracle, metric, x, q, k, res, ("special", po.METRIC_NAMES[metric]))


# ---------------------------------------------------------------------------------------------- (e) shards, groups, SQL, fallback
def test_row_shards_equal_one_shard_bit_for_bit():
    from tests.test_gpu_batch import _sharded_batch
    rng = np.random.Generator(np.random.PCG64(9100))
    n, dim, nq = 50000, 384, 48
    x, q = _normal(rng, n, dim), _normal(rng, nq, dim)
    bounds = [0, 20000, 33001, n]
    shards = [_index(x[a:b], first_seq=a) for a, b in zip(bounds[:-1], bounds[1:])]
    whole = _index(x)
    for metric in METRICS:
        for k in (1, 20):
            b0 = [s.stat("batches") for s in shards]
            res = _sharded_batch(shards, bounds, metric, q, k)
            assert [s.stat("batches") for s in shards] == [v + 1 for v in b0]
            one = _batched(whole, metric, q, k)
            for b in range(nq):                              # same refine arithmetic, same replay: identical, not merely close
                assert np.array_equal(res[b][0], one[b][0]) and np.array_equal(res[b][1], one[b][1]), (metric, k, b)
    for ix in shards + [whole]:
        ix.close()


@pytest.mark.parametrize("shards", [2, 3])
def test_group_batches(oracle, monkeypatch, shards):
    """a Group of 2 or 3 shards (wrapping around the visible GPUs): f32 batches through the gathered entry logs"""
    vs = _vs()
    monkeypatch.setenv("VSB_GROUP_ALIAS", "1")
    rng = np.random.Generator(np.random.PCG64(9200 + shards))
    n, dim, nq, k = 50000, 128, 32, 20
    x, q = _normal(rng, n, dim), _normal(rng, nq, dim)
    g = vs.Group(po.F32, dim, n, shards)
    g.append_dense(x)
    g.finalize()
    lib = g.eng.lib
    shard0 = lib.vsb_group_shard(g.h, 0)
    for metric in (po.L2, po.COS, po.DOT):
        b0 = lib.vsb_index_stat(shard0, b"batches")
        res = g.scan_topk(metric, q, k)
        assert lib.vsb_index_stat(shard0, b"batches") == b0 + 1, "the group's batch path did not run"
        _oracle_check(oracle, metric, x, q, k, res, ("group", shards, po.METRIC_NAMES[metric]))
    g.close()


def test_sql_full_scan_batch_f32():
    """vector_full_scan_batch on a FLOAT32 column with VSB_F32_BATCH=1 in the environment of the process that loads the
    extension: the per-query function's results, and a different launch count than with the variable unset"""
    from tests.sqlrun import OURS, run_sql
    rng = np.random.Generator(np.random.PCG64(9300))
    n, dim, nq, k = 9000, 32, 20, 7
    x, q = _normal(rng, n, dim), _normal(rng, nq, dim)
    s = ["CREATE TABLE t (id INTEGER PRIMARY KEY, e BLOB)", f"SELECT vector_init('t','e','type=FLOAT32,dimension={dim},distance=L2')"]
    for i in range(n):
        s.append(["INSERT INTO t(id, e) VALUES (?, ?)", [3 * i + 2, {"hex": x[i].tobytes().hex()}]])
    s.append(["SELECT query, id, distance FROM vector_full_scan_batch('t','e',?,?)", [{"hex": q.tobytes().hex()}, k]])
    batch_only = list(s)
    for b in range(nq):
        s.append(["SELECT id, distance FROM vector_full_scan('t','e',?,?)", [{"hex": q[b].tobytes().hex()}, k]])
    r = run_sql(OURS, s, env={"VSB_F32_BATCH": "1"})
    off = len(s) - (nq + 1)
    batch = r[off]["rows"]
    assert len(batch) == nq * k, r[off]
    for b in range(nq):
        got = [row[1:] for row in batch if row[0] == b]
        want = r[off + 1 + b]["rows"]
        gi, gd = np.array([v[0] for v in got]), np.array([v[1] for v in got])
        wi, wd = np.array([v[0] for v in want]), np.array([v[1] for v in want])
        assert_fp_topk(gi, gd, wi, wd, po.L2, lambda rid, b=b: float(np.sqrt(((x[(rid - 2) // 3].astype(np.float64) - q[b]) ** 2).sum())), (b,))
    on = run_sql(OURS, batch_only, env={"VSB_F32_BATCH": "1"}, want_launches=True)
    plain = run_sql(OURS, batch_only, env={"VSB_F32_BATCH": "0"}, want_launches=True)
    assert on[-2]["rows"] == batch
    assert on[-1]["kernel_launches"] != plain[-1]["kernel_launches"], "the variable did not change the path"


def test_bucket_overflow_falls_back_exactly(oracle):
    """distances that shrink along the scan: every row enters the slots, a level's bucket overflows, the call falls back to
    the per-query path and the result stays exact"""
    n, dim, nq, k = 40000, 64, 16, 5
    x = np.zeros((n, dim), dtype=np.float32)
    x[:, 0] = (n - np.arange(n)).astype(np.float32)
    q = np.zeros((nq, dim), dtype=np.float32)
    ix = _index(x)
    f0 = ix.stat("fallbacks")
    res = ix.scan_topk(po.L2, q, k)
    assert ix.stat("fallbacks") == f0 + 1
    rowids = np.arange(1, n + 1, dtype=np.int64)
    for b in (0, nq - 1):
        want_ids, want_d = oracle.scan_dense(po.L2, po.F32, q[b], x, rowids, k)
        assert np.array_equal(res[b][0], want_ids) and np.array_equal(res[b][1], want_d)
    ix.close()


def test_tc_level_tile_widths():
    """with the option on, vsb_debug_tc_level takes N = 32, 64, 128 and 0 for f32 L2 / dot / cosine, every other N is
    VSB_EINVAL; with it off, every N is"""
    vs = _vs()
    rng = np.random.Generator(np.random.PCG64(9400))
    n, dim, nq = 256, 64, 40
    ix = _index(_normal(rng, n, dim))
    q = _normal(rng, nq, dim)
    for on in (1, 0):
        with _f32_batch(on):
            for metric in (po.L2, po.DOT, po.COS):
                for N in (0, 16, 32, 48, 64, 128, 256, 512):
                    ok = on and N in (0, 32, 64, 128)
                    try:
                        ix.debug_tc_level(metric, q, np.full(nq, np.inf, np.float32), 0, 128, N=N, cap=1 << 16)
                        rc = 0
                    except vs.VsbError as e:
                        rc = e.rc
                    assert rc == (0 if ok else vs.api.EINVAL), (on, metric, N, rc)
    ix.close()
