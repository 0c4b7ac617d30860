"""A lone index and a one-shard group are the same column: every query kind takes the same path on both.  -m gpu.

For a resident and a streamed column of the same rows, int8 and bf16, each of the seven query kinds (top-k, filtered top-k,
per-query sets, listed rows, range, all distances, rowid bitmap) runs on an Index and on a one-shard Group: a single query and
a batch of 32, k = 20 and k = 300, with and without a row filter.  Both must return the same bits, make the same number of
kernel launches and move every counter of vsb_index_stat by the same amount (the host-clock counters, *_us, aside).  Each
call's launch counts are recorded as the test's `launches` property (pytest --junitxml)."""
import numpy as np
import pytest

from oracle import pyoracle as po

pytestmark = pytest.mark.gpu

N, DIM = 24000, 64
WINDOW = 4096            # rows per window of the streamed columns
KINDS = ["topk", "filtered", "sets", "rows", "range", "all", "bitmap"]
COUNTERS = ["queries", "survivors", "last_survivors", "fallbacks", "batches", "batch_cands", "batch_kept", "tc_rows", "stream_bytes",
            "plan_log2p", "plan_nsw", "plan_direct", "range_pairs", "range_passes", "range_host_sorts", "range_batches",
            "range_batch_fallbacks", "range_query_fallbacks", "large_k_queries", "large_k_cands", "large_k_regrows", "large_k_batches",
            "large_k_batch_fallbacks", "large_k_query_fallbacks", "large_k_replay_threads", "rows_queries", "rows_pairs",
            "rows_host_bytes", "sets_batches", "sets_fallbacks", "sets_levels"]


def _vs():
    import sqlite_vector_b200 as vs
    return vs


def _column(vtype, rng):
    if vtype == po.I8:
        return rng.integers(-20, 21, (N, DIM)).astype(np.int8)
    return po.convert(rng.standard_normal((N, DIM), dtype=np.float32), vtype)


def _pair(vtype, x, streamed, monkeypatch):
    """(Index, one-shard Group, the group's shard) over the rows x; streamed: both stream through WINDOW-row windows"""
    vs = _vs()
    ix = vs.Index(vtype, DIM, N, window_rows=WINDOW if streamed else 0)
    ix.append_dense(x)
    ix.finalize()
    if streamed:   # the group streams a shard that does not fit its budget, in windows of budget / 3 / pitch rows
        pitch = (DIM * x.itemsize + 15) // 16 * 16
        monkeypatch.setenv("VSB_DEVICE_BUDGET_MB", repr(WINDOW * 3 * pitch / 1048576.0))
    g = vs.Group(vtype, DIM, N, 1)
    monkeypatch.delenv("VSB_DEVICE_BUDGET_MB", raising=False)
    g.append_dense(x)
    g.finalize()
    lib = vs.load_engine().lib
    shard = lib.vsb_group_shard(g.h, 0)
    assert g.gpus == 1 and g.rows == ix.rows == N
    assert lib.vsb_index_is_streamed(ix.h) == lib.vsb_index_is_streamed(shard) == int(streamed)
    return ix, g, shard


def _stats(ptr):
    lib = _vs().load_engine().lib
    return {name: int(lib.vsb_index_stat(ptr, name.encode())) for name in COUNTERS}


def _run(kind, col, q, k, mask, rng_seed):
    """one call of `kind` on col (Index or Group); the arguments depend only on rng_seed, so both columns get the same call"""
    rng = np.random.default_rng(rng_seed)
    nq = q.shape[0]
    one = q[0] if nq == 1 else q
    mi = 0 if nq == 1 else None
    if kind == "topk":
        return col.scan_topk(po.L2, one, k, max_index=mi)
    if kind == "filtered":
        return col.scan_topk_filtered(po.L2, one, k, mask, max_index=mi)
    if kind == "sets":
        sets = [mask, rng.random(N) < 0.3, np.ones(N, bool)]
        return col.scan_topk_sets(po.L2, one, k, sets, set_of_query=np.arange(nq) % 3)
    if kind == "rows":
        lists = [rng.choice(np.nonzero(mask)[0], size=min(2 * k, int(mask.sum())), replace=False) + 1 for _ in range(nq)]
        return col.scan_topk_rows(po.L2, one, k, lists, max_index=mi)
    if kind == "range":
        d = col.scan_all(po.L2, q[0])
        radius = float(np.sort(d)[k])
        return col.scan_range(po.L2, one, radius, allow=None if mask.all() else mask)
    if kind == "all":
        return col.scan_all(po.L2, q[0], want_rowids=True)
    return col.rowid_bitmap(rng.integers(0, N + 50, size=5 * k))


def _same(a, b):
    if isinstance(a, (tuple, list)):
        assert type(a) is type(b) and len(a) == len(b)
        for u, v in zip(a, b):
            _same(u, v)
    elif isinstance(a, np.ndarray):
        assert a.dtype == b.dtype and a.shape == b.shape
        assert np.array_equal(a.view(np.uint8), b.view(np.uint8))
    else:
        assert a == b


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("vtype", [po.I8, po.BF16], ids=["int8", "bf16"])
@pytest.mark.parametrize("streamed", [False, True], ids=["resident", "streamed"])
def test_index_and_one_shard_group_take_the_same_path(streamed, vtype, kind, monkeypatch, record_property):
    eng = _vs().load_engine()
    rng = np.random.default_rng(1000 + 10 * vtype + streamed)
    x = _column(vtype, rng)
    queries = _column(vtype, rng)[:32]
    ix, g, shard = _pair(vtype, x, streamed, monkeypatch)
    launches = {}
    try:
        for nq in (1, 32):
            for k in (20, 300):
                for filtered in (False, True):
                    mask = rng.random(N) < 0.4 if filtered else np.ones(N, bool)
                    seed = int(rng.integers(1 << 31))
                    got, moved, calls = [], [], []
                    for col, ptr in ((ix, ix.h), (g, shard)):
                        s0, l0 = _stats(ptr), eng.kernel_launches()
                        got.append(_run(kind, col, queries[:nq], k, mask, seed))
                        calls.append(eng.kernel_launches() - l0)
                        s1 = _stats(ptr)
                        moved.append({c: s1[c] - s0[c] for c in COUNTERS})
                    case = f"nq={nq} k={k} filter={int(filtered)}"
                    launches[case] = calls
                    _same(got[0], got[1])
                    assert calls[0] == calls[1], (case, calls)
                    assert moved[0] == moved[1], (case, {c: (moved[0][c], moved[1][c]) for c in COUNTERS if moved[0][c] != moved[1][c]})
                    assert calls[0] > 0 or kind == "bitmap", case
    finally:
        record_property("launches", launches)
        ix.close()
        g.close()
