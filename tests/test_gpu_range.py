"""Range search (vsb_scan_range and its group / SQL doors): every row with distance < r, by (distance, scan order).  -m gpu.

The expected answer is built from distances: keep (double)d < r (and the row filter), stable-sort by d.  From the engine's own
all-distances scan of the same column (same arithmetic, same row positions) that is bit-exact for every element type; from the
oracle it is bit-exact for int8 / uint8 and within the tests/fpcheck.py tolerance for fp."""
import contextlib
import json
import os
import struct

import numpy as np
import pytest

from oracle import pyoracle as po
from tests.sqlrun import OURS, blob, run_sql

pytestmark = pytest.mark.gpu
METRICS = [po.L2, po.L2SQ, po.COS, po.DOT, po.L1]
STATS = ("range_batches", "range_batch_fallbacks", "range_query_fallbacks")


def _vs():
    import sqlite_vector_b200 as vs
    return vs


@pytest.fixture(scope="module", autouse=True)
def _alias():
    old = os.environ.get("VSB_GROUP_ALIAS")
    os.environ["VSB_GROUP_ALIAS"] = "1"
    yield
    os.environ.pop("VSB_GROUP_ALIAS", None) if old is None else os.environ.update(VSB_GROUP_ALIAS=old)


@pytest.fixture(scope="module")
def oracle():
    return po.Oracle()


@contextlib.contextmanager
def _options(**opts):
    eng = _vs().load_engine()
    old = {name: eng.set_option(name, v) for name, v in opts.items()}
    yield
    for name, v in old.items():
        eng.set_option(name, v)


def _column(vtype, n, dim, rng, spread=20):
    if vtype == po.I8:
        return rng.integers(-spread, spread + 1, (n, dim)).astype(np.int8)
    if vtype == po.U8:
        return rng.integers(0, 2 * spread, (n, dim)).astype(np.uint8)
    return po.convert(rng.standard_normal((n, dim), dtype=np.float32), vtype)


def _index(vtype, x, rowids=None, window=0):
    ix = _vs().Index(vtype, x.shape[1], x.shape[0], window_rows=window)
    ix.append_dense(x, rowids)
    ix.finalize()
    return ix


def _group(vtype, x, ngpus, rowids=None, chunk=7919):
    g = _vs().Group(vtype, x.shape[1], x.shape[0], ngpus)
    for a in range(0, x.shape[0], chunk):
        g.append_dense(x[a:a + chunk], None if rowids is None else rowids[a:a + chunk])
    g.finalize()
    return g


def expect(dist, ids, r, mask=None):
    keep = dist.astype(np.float64) < r
    idx = np.nonzero(keep if mask is None else keep & mask)[0]
    sel = idx[np.argsort(dist[idx], kind="stable")]
    return ids[sel], dist[sel].astype(np.float64)


def same(got, want, ctx):
    assert np.array_equal(got[0], want[0]), (ctx, len(got[0]), len(want[0]))
    assert np.array_equal(np.ascontiguousarray(got[1]).view(np.uint64), np.ascontiguousarray(want[1]).view(np.uint64)), ctx


def _radii(d):
    """a row's exact distance (excluded), the next double above it (included), the 30th percentile, none and all"""
    f = np.sort(d[np.isfinite(d)]).astype(np.float64)
    at = float(f[len(f) // 50])
    return [at, float(np.nextafter(at, np.inf)), float(f[int(len(f) * 0.3)]), float(f[0]), float(f[-1]) + 1.0]


def _batch_radii(dist_of, nq, pattern=(0, 5, 100, 3000, 0, 40)):
    """per-query radii from 0 rows to thousands: query b's pattern[b % len]-th smallest distance (strict: that many rows)"""
    return np.array([float(np.sort(dist_of(b))[pattern[b % len(pattern)]]) for b in range(nq)])


def _delta(ix, before):
    return {k: ix.stat(k) - before.get(k, 0) for k in STATS}


def _fp_parity(got, want_all, ids, metric, r, ctx):
    """fp: rows whose oracle distance is outside the tolerance of r agree; distances within tolerance; order up to near ties"""
    w64 = want_all.astype(np.float64)
    scale = np.maximum(np.abs(w64), 1e-30)
    scale = np.maximum(scale, 1.0) if metric == po.COS else (np.maximum(scale, np.abs(w64).max()) if metric == po.DOT else scale)
    tol = 1e-5 * scale
    pos = {int(v): i for i, v in enumerate(ids)}
    diff = set(got[0].tolist()) ^ set(ids[w64 < r].tolist())
    assert all(abs(w64[pos[int(v)]] - r) <= 2 * tol[pos[int(v)]] for v in diff), (ctx, sorted(diff)[:5])
    rows = np.array([pos[int(v)] for v in got[0]], dtype=np.int64)
    if len(rows):
        assert np.all(np.abs(got[1] - w64[rows]) <= tol[rows] + 1e-30), ctx
        assert np.all(w64[rows][1:] >= w64[rows][:-1] - 2 * np.maximum(tol[rows][1:], tol[rows][:-1])), (ctx, "order")


# ------------------------------------------------------------------------------------------------ single queries
@pytest.mark.parametrize("vtype", [po.F32, po.F16, po.BF16, po.U8, po.I8])
@pytest.mark.parametrize("dim", [5, 128, 771])
def test_range_matches_oracle(oracle, vtype, dim):
    rng = np.random.Generator(np.random.PCG64(1000 + 7 * vtype + dim))
    x = _column(vtype, 3000, dim, rng)
    ids = np.arange(1, 3001, dtype=np.int64) * 3 + 1
    ix = _index(vtype, x, ids)
    q = _column(vtype, 1, dim, rng)[0]
    for metric in METRICS:
        want_all = oracle.distances_all(metric, vtype, q, x, int_exact=True)
        mine = ix.scan_all(metric, q)
        for r in _radii(want_all):
            got = ix.scan_range(metric, q, r)[0]
            same(got, expect(mine, ids, r), (vtype, dim, metric, r))
            if vtype in (po.I8, po.U8):
                same(got, expect(want_all, ids, r), (vtype, dim, metric, r))
            else:
                _fp_parity(got, want_all, ids, metric, r, (vtype, dim, metric, r))


def test_special_radii_and_heavy_ties(oracle):
    rng = np.random.Generator(np.random.PCG64(11))
    x = rng.integers(-1, 2, (5000, 4)).astype(np.int8)                # 81 distinct rows: every distance is shared by many rows
    ids = np.arange(1, 5001, dtype=np.int64)
    ix = _index(po.I8, x)
    q = np.array([1, 0, -1, 1], dtype=np.int8)
    for metric in METRICS:
        want_all = oracle.distances_all(metric, po.I8, q, x, int_exact=True)
        for r in (np.nan, np.inf, -np.inf, 0.0, -0.0, float(np.median(want_all)), -1.5, -2.0, 1e300, -1e300):
            got = ix.scan_range(metric, q, r)[0]
            same(got, expect(want_all, ids, r), (metric, r))
            if r != r or abs(r) == np.inf:
                assert len(got[0]) == (5000 if r == np.inf else 0), (metric, r)
        if metric == po.DOT:
            got = ix.scan_range(metric, q, -1.5)[0]                    # a negative radius keeps dot products above 1.5
            assert len(got[0]) > 0 and np.all(got[1] <= -2.0)


@pytest.mark.parametrize("vtype", [po.F16, po.BF16])
def test_nan_and_inf_rows(oracle, vtype):
    rng = np.random.Generator(np.random.PCG64(12 + vtype))
    xf = rng.standard_normal((2000, 16), dtype=np.float32)
    for i in rng.choice(2000, 300, replace=False):
        xf[i, rng.integers(0, 16, rng.integers(1, 3))] = rng.choice(np.array([np.nan, np.inf, -np.inf], dtype=np.float32))
    x = po.convert(xf, vtype)
    ids = np.arange(1, 2001, dtype=np.int64)
    ix = _index(vtype, x)
    q = po.convert(rng.standard_normal((1, 16), dtype=np.float32), vtype)[0]
    for metric in METRICS:
        want_all, mine = oracle.distances_all(metric, vtype, q, x), ix.scan_all(metric, q)
        for r in (np.inf, float(np.median(want_all[np.isfinite(want_all)])), -np.inf, np.nan):
            same(ix.scan_range(metric, q, r)[0], expect(mine, ids, r), (vtype, metric, r))
        got = ix.scan_range(metric, q, np.inf)[0]
        assert set(got[0].tolist()) == set(ids[want_all < np.inf].tolist()), (vtype, metric)   # NaN and +INF rows never qualify
        assert np.all(np.isneginf(got[1][:int(np.isneginf(want_all).sum())])) and not np.any(np.isnan(got[1]))


def test_radius_rounds_toward_plus_infinity():
    """r between two floats, closer to the lower one d: nearest rounding gives d, but (double)d < r keeps the rows at d; r just
    below d (nearest rounding again d) keeps none of them"""
    rng = np.random.Generator(np.random.PCG64(13))
    x = rng.standard_normal((4000, 32), dtype=np.float32)
    ids = np.arange(1, 4001, dtype=np.int64)
    ix = _index(po.F32, x)
    q = rng.standard_normal(32, dtype=np.float32)
    for metric in (po.L2, po.DOT, po.COS):
        dist = ix.scan_all(metric, q)
        for d in np.sort(dist)[[5, 100, 2500]]:
            ulp = float(np.spacing(np.float32(abs(d))))
            up, down = float(d) + 0.25 * ulp, float(d) - 0.25 * ulp
            assert np.float32(up) == d and np.float32(down) == d
            got_up, got_down = ix.scan_range(metric, q, up)[0], ix.scan_range(metric, q, down)[0]
            same(got_up, expect(dist, ids, up), (metric, "up"))
            same(got_down, expect(dist, ids, down), (metric, "down"))
            at = set(ids[dist == d].tolist())
            assert at <= set(got_up[0].tolist()) and not (at & set(got_down[0].tolist()))


def test_capacities_on_a_million_rows():
    """beyond the first pass's list: a second pass; beyond the GPU sort: the host orders; a batch whose candidate log overflows
    (17 L1 queries with every row within r: 2^20 rows x 17 > 2^24 pairs) is answered query by query"""
    rng = np.random.Generator(np.random.PCG64(14))
    n = 1_100_000
    x = rng.standard_normal((n, 8), dtype=np.float32)
    ids = np.arange(1, n + 1, dtype=np.int64)
    ix = _index(po.F32, x)
    q = rng.standard_normal((17, 8), dtype=np.float32)
    dist = ix.scan_all(po.L2, q[0])
    srt = np.sort(dist)
    # the list grows to the largest result so far: ascending sizes, so that each of the last two needs its second pass
    for r, passes, host in [(srt[3000], 0, 0), (srt[16_384], 0, 0), (srt[40_000], 0, 1), (srt[200_000], 1, 1), (np.inf, 1, 1)]:
        p0, h0 = ix.stat("range_passes"), ix.stat("range_host_sorts")
        same(ix.scan_range(po.L2, q[0], float(r))[0], expect(dist, ids, float(r)), r)
        assert (ix.stat("range_passes") - p0, ix.stat("range_host_sorts") - h0) == (passes, host), r
    s0 = {k: ix.stat(k) for k in STATS}
    got = ix.scan_range(po.L1, q, 1e9)
    assert _delta(ix, s0) == {"range_batches": 0, "range_batch_fallbacks": 1, "range_query_fallbacks": 0}
    for b in (0, 16):
        same(got[b], expect(ix.scan_all(po.L1, q[b]), ids, 1e9), b)


@pytest.mark.parametrize("vtype", [po.F32, po.BF16, po.I8])
def test_filters(vtype):
    rng = np.random.Generator(np.random.PCG64(15 + vtype))
    n = 30_000
    x = _column(vtype, n, 24, rng)
    ids = rng.permutation(n * 4)[:n].astype(np.int64) + 1
    ix = _index(vtype, x, ids)
    q = _column(vtype, 1, 24, rng)[0]
    masks = {"all": np.ones(n, bool), "r50": rng.random(n) < 0.5, "r1": rng.random(n) < 0.01, "block": (np.arange(n) // 4000) == 3}
    for metric in METRICS:
        dist = ix.scan_all(metric, q)
        for r in _radii(dist)[1:3] + [np.inf]:
            plain = ix.scan_range(metric, q, r)[0]
            for name, m in masks.items():
                got = ix.scan_range(metric, q, r, allow=m)[0]
                same(got, plain if name == "all" else expect(dist, ids, r, m), (metric, r, name))
                if vtype == po.I8 and name == "block":
                    sub = _index(vtype, x[m], ids[m])
                    same(got, sub.scan_range(metric, q, r)[0], (metric, r, name, "sub-column"))


# ------------------------------------------------------------------------------------------------ batches
@pytest.mark.parametrize("nq", [16, 1024])
@pytest.mark.parametrize("vtype", [po.I8, po.U8])
def test_integer_batch_equals_single_calls(vtype, nq):
    """the batch path (tensor cores; L1: the CUDA-core kernel) is bit for bit B single range calls for int8 / uint8"""
    rng = np.random.Generator(np.random.PCG64(16 + nq + vtype))
    x = _column(vtype, 20_000, 64, rng)
    ix = _index(vtype, x, np.arange(1, 20_001, dtype=np.int64) * 7)
    qs = _column(vtype, nq, 64, rng)
    for metric in METRICS:
        radii = _batch_radii(lambda b: ix.scan_all(metric, qs[b]), nq)
        s0 = {k: ix.stat(k) for k in STATS}
        got = ix.scan_range(metric, qs, radii)
        assert _delta(ix, s0) == {"range_batches": 1, "range_batch_fallbacks": 0, "range_query_fallbacks": 0}, metric
        assert sum(len(g[0]) == 0 for g in got) >= nq // 3
        for b in range(nq):
            same(got[b], ix.scan_range(metric, qs[b], radii[b])[0], (metric, b))


@pytest.mark.parametrize("vtype,f32_batch", [(po.F32, 1), (po.F32, 0), (po.F16, 0), (po.BF16, 0)])
def test_fp_batch_matches_oracle(oracle, vtype, f32_batch):
    """fp batches agree with the oracle within the fp rules; f32 takes the batch path only with f32_batch on (L1 always)"""
    rng = np.random.Generator(np.random.PCG64(21 + vtype + f32_batch))
    x = _column(vtype, 12_000, 48, rng)
    ids = np.arange(1, 12_001, dtype=np.int64)
    qs = _column(vtype, 24, 48, rng)
    with _options(f32_batch=f32_batch):
        ix = _index(vtype, x, ids)
        for metric in METRICS:
            radii = _batch_radii(lambda b: ix.scan_all(metric, qs[b]), 24)
            s0 = {k: ix.stat(k) for k in STATS}
            got = ix.scan_range(metric, qs, radii)
            assert _delta(ix, s0)["range_batches"] == int(vtype != po.F32 or f32_batch or metric == po.L1), metric
            for b in range(24):
                _fp_parity(got[b], oracle.distances_all(metric, vtype, qs[b], x), ids, metric, radii[b], (vtype, metric, b))


def test_batch_radii_filters_and_bucket_overflow():
    """special radii and row filters in one batch; a query keeping more rows than its bucket holds is answered alone"""
    rng = np.random.Generator(np.random.PCG64(24))
    n, nq = 40_000, 20
    x = _column(po.I8, n, 40, rng)
    ids = rng.permutation(2 * n)[:n].astype(np.int64) + 1
    ix = _index(po.I8, x, ids)
    qs = _column(po.I8, nq, 40, rng)
    masks = {None: None, "r30": rng.random(n) < 0.3, "block": (np.arange(n) // 1500) % 4 == 1}
    for metric in (po.L2, po.DOT, po.COS, po.L1):
        radii = _batch_radii(lambda b: ix.scan_all(metric, qs[b]), nq)
        radii[:7] = [np.nan, -np.inf, 0.0, -0.0, -1e30, -50.0, float(np.sort(ix.scan_all(metric, qs[6]))[30_000])]
        for name, m in masks.items():
            want = [expect(ix.scan_all(metric, qs[b]), ids, radii[b], m) for b in range(nq)]
            s0 = {k: ix.stat(k) for k in STATS}
            got = ix.scan_range(metric, qs, radii, allow=m)
            over = sum(len(w[0]) > 16_384 for w in want)                # more rows than a query's bucket: answered alone
            assert _delta(ix, s0) == {"range_batches": 1, "range_batch_fallbacks": 0, "range_query_fallbacks": over}, (metric, name)
            assert over >= int(name is None)
            for b in range(nq):
                same(got[b], want[b], (metric, name, b))
            assert len(got[0][0]) == len(got[1][0]) == 0


# ------------------------------------------------------------------------------------------------ streamed windows, groups
@pytest.mark.parametrize("window", [128, 300, 5000])
@pytest.mark.parametrize("vtype", [po.F16, po.I8])
def test_streamed_windows(vtype, window):
    rng = np.random.Generator(np.random.PCG64(17 + window + vtype))
    n = 70_000 if window == 5000 else 12_000
    x = _column(vtype, n, 40, rng)
    ids = np.arange(1, n + 1, dtype=np.int64) * 2
    ix, res = _index(vtype, x, ids, window=window), _index(vtype, x, ids)
    qs = _column(vtype, 16, 40, rng)
    m = rng.random(n) < 0.3
    for metric in (po.L2, po.COS, po.DOT):
        dist = ix.scan_all(metric, qs[0])
        for r in _radii(dist)[:3] + [np.inf]:
            got = ix.scan_range(metric, qs[0], r)[0]
            same(got, expect(dist, ids, r), (window, metric, r))
            same(ix.scan_range(metric, qs[0], r, allow=m)[0], expect(dist, ids, r, m), (window, metric, r, "filtered"))
            if vtype == po.I8:
                same(got, res.scan_range(metric, qs[0], r)[0], (window, metric, r, "resident"))
        if vtype == po.I8:                                             # the batch path, window by window
            radii = _batch_radii(lambda b: ix.scan_all(metric, qs[b]), 16)
            s0 = {k: ix.stat(k) for k in STATS}
            got = ix.scan_range(metric, qs, radii, allow=m)
            assert _delta(ix, s0)["range_batches"] == 1
            for b in range(16):
                same(got[b], expect(ix.scan_all(metric, qs[b]), ids, radii[b], m), (window, metric, b))
    if window == 5000:
        assert ix.stat("range_passes") >= 1                            # 70 000 rows within +INF: the second pass over the windows


@pytest.mark.parametrize("ngpus", [1, 2, 3])
@pytest.mark.parametrize("vtype", [po.F32, po.U8])
def test_groups_equal_one_index(vtype, ngpus):
    rng = np.random.Generator(np.random.PCG64(18 + ngpus + vtype))
    n = 25_001
    x = _column(vtype, n, 20, rng)
    ids = rng.permutation(3 * n)[:n].astype(np.int64) + 1
    g, ix = _group(vtype, x, ngpus, ids), _index(vtype, x, ids)
    qs = _column(vtype, 20, 20, rng)
    m = np.zeros(n, bool)
    m[n // 3 - 500:n // 3 + 500] = True                                # across the first shard boundary
    m |= rng.random(n) < 0.05
    for metric in (po.L2, po.DOT, po.L1):
        dist, gids = g.scan_all(metric, qs[0], want_rowids=True)
        assert np.array_equal(gids, ids)
        for r in _radii(dist)[:3] + [np.inf]:
            got = g.scan_range(metric, qs[0], r)[0]
            same(got, expect(dist, ids, r), (ngpus, metric, r))
            same(g.scan_range(metric, qs[0], r, allow=m)[0], expect(dist, ids, r, m), (ngpus, metric, r, "filtered"))
            if vtype == po.U8:
                same(got, ix.scan_range(metric, qs[0], r)[0], (ngpus, metric, r, "one index"))
        if vtype == po.U8:                                             # every shard runs the batch path on its rows
            radii = _batch_radii(lambda b: g.scan_all(metric, qs[b]), 20, (0, 50, 2000, 9000))
            got = g.scan_range(metric, qs, radii, allow=m)
            for b in range(20):
                same(got[b], expect(g.scan_all(metric, qs[b]), ids, radii[b], m), (ngpus, metric, b))


# ------------------------------------------------------------------------------------------------ SQL
def _rowid_blob(ids):
    return {"hex": struct.pack("<%dq" % len(ids), *ids).hex()}


def test_sql_matches_reference_golden():
    """the reference's own range answers (its stream modules with WHERE distance < r, tools/range_golden.py)"""
    gold = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "sql_range.json")))
    script = list(gold["setup"])
    for e in gold["cases"]:
        mod = "vector_%s_scan_range%s" % ("quantize" if e["quantized"] else "full", "" if e["filter"] is None else "_filtered")
        args = [{"hex": e["vector"]}, e["radius"]] + ([] if e["filter"] is None else [_rowid_blob(e["filter"])])
        script.append([f"SELECT id, distance FROM {mod}('{e['table']}', 'e', {', '.join('?' * len(args))})", args])
    res = run_sql(OURS, script)
    assert all("error" not in r for r in res[:len(gold["setup"])])
    for e, r in zip(gold["cases"], res[len(gold["setup"]):]):
        assert r.get("rows") == e["rows"], (e["table"], e["radius"], e["filter"] is not None, r.get("error"))
    assert sum(len(e["rows"]) for e in gold["cases"]) > 200


def test_sql_equals_our_stream_module_and_transactions():
    rng = np.random.Generator(np.random.PCG64(19))
    n, dim = 3000, 24
    x = rng.standard_normal((n, dim), dtype=np.float32)
    s = ["CREATE TABLE t (id INTEGER PRIMARY KEY, e BLOB)", f"SELECT vector_init('t', 'e', 'type=FLOAT32,dimension={dim},distance=COSINE')"]
    s += [["INSERT INTO t VALUES (?, ?)", [5 * i + 2, blob(x[i])]] for i in range(n)] + ["SELECT vector_quantize('t', 'e', 'qtype=INT8')"]
    keep = (np.arange(n)[rng.random(n) < 0.3] * 5 + 2).tolist()
    pairs = []
    for b in range(3):
        q = blob(rng.standard_normal(dim, dtype=np.float32))
        for r in (0.5, 0.9, 1.0, 2.5):
            for kind in ("full", "quantize"):
                stream = f"SELECT id, distance FROM vector_{kind}_scan_stream('t', 'e', ?) WHERE distance < ? AND id > 0"
                s += [[stream + " ORDER BY distance, id", [q, r]], [f"SELECT id, distance FROM vector_{kind}_scan_range('t', 'e', ?, ?)", [q, r]],
                      [stream + f" AND id IN ({','.join(map(str, keep))}) ORDER BY distance, id", [q, r]],
                      [f"SELECT id, distance FROM vector_{kind}_scan_range_filtered('t', 'e', ?, ?, ?)", [q, r, _rowid_blob(keep)]]]
                pairs.append((kind, r))
    # a transaction and its ROLLBACK behave like vector_full_scan
    rng_q = "x'0000803f0000803f'"                                          # [1, 1]
    t = ["CREATE TABLE u (id INTEGER PRIMARY KEY, e BLOB)", "SELECT vector_init('u', 'e', 'type=FLOAT32,dimension=2')",
         "INSERT INTO u VALUES (1, x'0000803f00000000'), (2, x'0000000000000040')"]
    look = [f"SELECT id FROM vector_full_scan_range('u', 'e', {rng_q}, 10)", f"SELECT id FROM vector_full_scan('u', 'e', {rng_q}, 10)"]
    t += look + ["BEGIN", "INSERT INTO u VALUES (3, x'0000803f0000803f')"] + look + ["ROLLBACK"] + look
    t += [f"SELECT id, distance FROM vector_full_scan_range('u', 'e', {rng_q}, 1.2)"]
    res = run_sql(OURS, s + t)
    assert all("error" not in r for r in res), [r for r in res if "error" in r][:2]
    out, tr = res[n + 3:len(s)], res[len(s):]
    for i, ctx in enumerate(pairs):
        assert out[4 * i]["rows"] == out[4 * i + 1]["rows"] and out[4 * i + 2]["rows"] == out[4 * i + 3]["rows"], ctx
    assert sum(bool(out[4 * i]["rows"]) for i in range(len(pairs))) >= len(pairs) // 2
    assert tr[3]["rows"] == tr[4]["rows"] == [[1], [2]] and tr[10]["rows"] == tr[11]["rows"] == [[1], [2]]
    assert tr[7]["rows"] == tr[8]["rows"] == [[3], [1], [2]] and tr[12]["rows"] == [[1, 1.0]]


def test_range_calls_leak_no_handles():
    eng = _vs().load_engine()
    rng = np.random.Generator(np.random.PCG64(20))
    x = _column(po.I8, 70_000, 16, rng)
    q = _column(po.I8, 2, 16, rng)
    base = eng.debug_live_handles()
    for _ in range(2):
        ix = _index(po.I8, x)
        ix.scan_range(po.L2, q[0], np.inf)                             # 70 000 rows: the list grows for a second pass
        assert ix.stat("range_passes") == 1
        ix.scan_range(po.L2, q, [np.inf, 300.0], allow=rng.random(len(x)) < 0.5)
        ix.close()
        st = _index(po.I8, x, window=9000)
        st.scan_range(po.DOT, q[0], -10.0)
        st.close()
        g = _group(po.I8, x, 3)
        g.scan_range(po.L1, q, 500.0, allow=rng.random(len(x)) < 0.5)
        g.close()
        assert eng.debug_live_handles() == base
