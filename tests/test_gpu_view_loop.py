"""Every scan path over views: a resident column is one view of all its rows, a streamed column one view per window.  -m gpu.

For a resident and a streamed index of the same rows (ragged windows: 20 000 rows in windows of 3 000), int8 and bf16, each of
scan_topk with k = 20 and k = 300, scan_topk_filtered, scan_all, scan_range (one query, a batch of 32) and a batch of 32 top-k
queries:
  - the exact kernel launches of the call, restated below from where each path launches;
  - stream_bytes: one pass of the column per call when streamed, nothing when resident; stream_us: nothing when resident;
  - the streamed results equal the resident ones bit for bit."""
import numpy as np
import pytest

from oracle import pyoracle as po

pytestmark = pytest.mark.gpu

N, WINDOW, DIM, NQ = 20000, 3000, 64, 32
M0, GROWTH = 128, 8              # the batch path's exhaustive prefix and level growth at k = 20 (batch_m0, batch_growth)
RANGE_LEVEL_ROWS = 1 << 20       # rows per level of a range batch


def _vs():
    import sqlite_vector_b200 as vs
    return vs


def _column(vtype, n, rng):
    if vtype == po.I8:
        return rng.integers(-60, 61, (n, DIM)).astype(np.int8)
    return po.convert(rng.standard_normal((n, DIM), dtype=np.float32), vtype)


def _views(streamed):
    """the rows of each view"""
    return [min(WINDOW, N - r0) for r0 in range(0, N, WINDOW)] if streamed else [N]


def _grow_levels(rows):
    """levels of the batch path's schedule over the first rows of a column: [0, M0), then each level GROWTH times the rows before it"""
    levels, lo = 0, 0
    while lo < rows:
        lo = min(rows, M0 if lo == 0 else lo * GROWTH)
        levels += 1
    return levels


def _expected_launches(call, vtype, streamed):
    views = _views(streamed)
    fp = vtype != po.I8
    if call in ("topk20", "filtered"):              # per view: scan_kernel + filter_kernel
        return 2 * len(views)
    if call == "topk300":                           # per view: the all-distances scan, 4 radix digits (histogram + select; select
        return sum(1 + 4 * (2 if 300 < r else 1) + 3 for r in views)   # alone without a prefix), count, offsets, write
    if call == "all":                               # per view: the all-distances scan
        return len(views)
    if call == "range1":                            # per view: the range scan; then range_sort_kernel
        return len(views) + 1
    # batches: resident row norms (+ the largest norm, fp) once per column; query norms + 2 fills of the upload
    prep = 0 if streamed else 1 + fp
    upload = 3
    if call == "range32":                           # conservative_qc; per view: its row norms when streamed, (scorer + refine) per
        per_view = sum((1 if streamed else 0) + 2 * -(-r // RANGE_LEVEL_ROWS) for r in views)   # level; range_sort_kernel
        return prep + upload + 1 + per_view + 1
    assert call == "topk32"                         # view 0 takes the grown schedule, every later window one level; each level
    levels = _grow_levels(views[0]) + len(views) - 1   # scorer (all_pairs at level 0) + refine + replay; then final_sort_kernel
    return prep + upload + (len(views) if streamed else 0) + 3 * levels + 1


CALLS = ["topk20", "topk300", "filtered", "all", "range1", "range32", "topk32"]


@pytest.mark.parametrize("vtype", [po.I8, po.BF16])
@pytest.mark.parametrize("call", CALLS)
def test_view_loop(vtype, call):
    vs = _vs()
    eng = vs.load_engine()
    rng = np.random.Generator(np.random.PCG64(7))
    x = _column(vtype, N, rng)
    q = _column(vtype, NQ, rng)
    res = vs.Index(vtype, DIM, N)
    st = vs.Index(vtype, DIM, N, window_rows=WINDOW)
    for ix in (res, st):
        ix.append_dense(x)
        ix.finalize()
    assert st.stat("stream_bytes") == 0
    # radii: each query's 60th smallest distance (about 60 rows each, well inside one range_sort_kernel)
    radius = np.array([float(np.sort(res.scan_all(po.L2, q[b]))[60]) for b in range(NQ)])
    allow = rng.random(N) < 0.5
    pitch = st.query_pitch

    def run(ix):
        if call == "topk20":
            return ix.scan_topk(po.L2, q[0], 20)
        if call == "topk300":
            return ix.scan_topk(po.L2, q[0], 300)
        if call == "filtered":
            return ix.scan_topk_filtered(po.L2, q[0], 20, allow)
        if call == "all":
            return [(ix.scan_all(po.L2, q[0]).astype(np.float64),)]
        if call == "range1":
            return ix.scan_range(po.L2, q[0], radius[0])
        if call == "range32":
            return ix.scan_range(po.L2, q, radius)
        return ix.scan_topk(po.L2, q, 20)

    out, got, want = {}, {}, {}
    for name, ix in (("resident", res), ("streamed", st)):
        l0, b0, u0 = eng.kernel_launches(), ix.stat("stream_bytes"), ix.stat("stream_us")
        out[name] = run(ix)
        got[name] = (eng.kernel_launches() - l0, ix.stat("stream_bytes") - b0)
        want[name] = (_expected_launches(call, vtype, ix is st), N * pitch if ix is st else 0)
        if ix is res:
            assert ix.stat("stream_us") == u0
    assert got == want
    if call == "range1":
        assert 2 <= len(out["resident"][0][0]) <= 16384
    assert len(out["resident"]) == len(out["streamed"]) == (NQ if call in ("range32", "topk32") else 1)
    for a, b in zip(out["resident"], out["streamed"]):
        for u, v in zip(a, b):
            assert u.dtype == v.dtype and u.shape == v.shape and len(u) > 0
            assert np.array_equal(np.ascontiguousarray(u).view(np.uint64), np.ascontiguousarray(v).view(np.uint64))
    res.close()
    st.close()
