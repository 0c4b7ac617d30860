"""Row shards behind ONE process (vsb_group: what vector.so uses with gpus=N) and the peer-memory exchange between
processes (vsb_exchange_*: what bench.py uses under torchrun), on whatever GPUs the box has:

  * with VSB_GROUP_ALIAS=1 the shards of a group wrap around the visible devices, so a 1-GPU box runs the complete
    multi-shard machinery (push into the leader's gather buffer, flag wait, host replay, batched merge);
  * two PROCESSES can share one GPU: cudaIpc mappings, pushes and flags work exactly as between two GPUs (the handles
    are all-gathered over gloo, NCCL refuses two ranks per device).
On a multi-GPU box the same tests use distinct devices (real NVLink peer stores).  -m gpu."""
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import pyoracle as po

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
METRICS = [po.L2, po.L2SQ, po.COS, po.DOT, po.L1]


@pytest.fixture(scope="module", autouse=True)
def _alias():
    old = os.environ.get("VSB_GROUP_ALIAS")
    os.environ["VSB_GROUP_ALIAS"] = "1"
    yield
    if old is None:
        os.environ.pop("VSB_GROUP_ALIAS", None)
    else:
        os.environ["VSB_GROUP_ALIAS"] = old


def _group(vtype, x, ngpus, rowids=None, chunk=7919):
    import sqlite_vector_b200 as vs
    g = vs.Group(vtype, x.shape[1], x.shape[0], ngpus)
    for a in range(0, x.shape[0], chunk):                   # appended in pieces that straddle shard boundaries
        g.append_dense(x[a:a + chunk], None if rowids is None else rowids[a:a + chunk])
    g.finalize()
    return g


@pytest.mark.parametrize("ngpus", [2, 3, 8])
def test_group_int8_bit_exact(oracle, ngpus):
    rng = np.random.Generator(np.random.PCG64(100 + ngpus))
    n, dim = 50_000, 64
    x = rng.integers(-5, 6, (n, dim)).astype(np.int8)        # narrow value range: ties at the k-th place
    rowids = np.arange(n, dtype=np.int64) * 3 + 11
    g = _group(po.I8, x, ngpus, rowids)
    assert g.gpus == ngpus and g.rows == n
    for i, k in enumerate([20, 100, 10, 33, 1, 256, 300, 7]):
        q = rng.integers(-5, 6, dim).astype(np.int8)
        metric = METRICS[i % 5]
        for smi in (0, min(2, k - 1)):
            (res,), mi = g.scan_topk(metric, q, k, max_index=smi)
            want_ids, want_d = oracle.scan_dense(metric, po.I8, q, x, rowids, k, start_max_index=smi)
            assert np.array_equal(res[0], want_ids) and np.array_equal(res[1], want_d), (ngpus, metric, k, smi)
    # several queries in one call (pipelined window), implicit rowids, all-distances
    g2 = _group(po.I8, x, ngpus)
    qs = rng.integers(-5, 6, (40, dim)).astype(np.int8)
    import sqlite_vector_b200 as vs
    eng = vs.load_engine()
    eng.set_option("no_batch", 1)
    try:
        res = g2.scan_topk(po.L2, qs, 20)
    finally:
        eng.set_option("no_batch", 0)
    imp = np.arange(1, n + 1, dtype=np.int64)
    for b in range(40):
        want_ids, want_d = oracle.scan_dense(po.L2, po.I8, qs[b], x, imp, 20)
        assert np.array_equal(res[b][0], want_ids) and np.array_equal(res[b][1], want_d), (ngpus, b)
    d, ids = g2.scan_all(po.L1, qs[0], want_rowids=True)
    assert np.array_equal(ids, imp) and np.array_equal(d, oracle.distances_all(po.L1, po.I8, qs[0], x, int_exact=True))
    # batched queries: per-shard tensor-core levels, entry logs copied to the leader, merge replay
    res = g2.scan_topk(po.COS, qs, 20)
    for b in range(40):
        want_ids, want_d = oracle.scan_dense(po.COS, po.I8, qs[b], x, imp, 20)
        assert np.array_equal(res[b][0], want_ids) and np.array_equal(res[b][1], want_d), ("batch", ngpus, b)
    g.close(); g2.close()


def test_group_overflow_and_empty_shards(oracle):
    # descending distances: every row enters the slots, each shard's candidate log overflows -> all-distances fallback
    n = 120_000
    x = np.zeros((n, 16), dtype=np.int8)
    x[:, 0] = np.clip(np.arange(n)[::-1] // 960, 0, 127)
    g = _group(po.I8, x, 3)
    q = np.zeros(16, dtype=np.int8)
    (res,) = g.scan_topk(po.L1, q, 20)
    want_ids, want_d = oracle.scan_dense(po.L1, po.I8, q, x, np.arange(1, n + 1, dtype=np.int64), 20)
    assert np.array_equal(res[0], want_ids) and np.array_equal(res[1], want_d)
    g.close()
    # fewer rows than capacity (NULL rows skipped by the SQL layer): trailing shards are short or empty
    import sqlite_vector_b200 as vs
    rng = np.random.Generator(np.random.PCG64(8))
    y = rng.integers(-9, 10, (1000, 8)).astype(np.int8)
    g = vs.Group(po.I8, 8, 4000, 4)
    g.append_dense(y)
    g.finalize()
    (res,) = g.scan_topk(po.L2, y[5], 12)
    want_ids, want_d = oracle.scan_dense(po.L2, po.I8, y[5], y, np.arange(1, 1001, dtype=np.int64), 12)
    assert np.array_equal(res[0], want_ids) and np.array_equal(res[1], want_d)
    g.close()


@pytest.mark.parametrize("vtype", [po.F32, po.BF16])
def test_group_fp(oracle, vtype):
    from tests.fpcheck import assert_fp_topk
    rng = np.random.Generator(np.random.PCG64(300 + vtype))
    n, dim, k = 40_000, 96, 20
    x = po.convert(rng.standard_normal((n, dim), dtype=np.float32), vtype)
    q = po.convert(rng.standard_normal((24, dim), dtype=np.float32), vtype)
    rowids = np.arange(1, n + 1, dtype=np.int64)
    g = _group(vtype, x, 3)
    for metric in (po.L2, po.DOT, po.COS):
        res = g.scan_topk(metric, q, k)                       # bf16: batch path over the shards; f32: pipelined single queries
        for b in range(q.shape[0]):
            want_ids, want_d = oracle.scan_dense(metric, vtype, q[b], x, rowids, k)
            assert_fp_topk(res[b][0], res[b][1], want_ids, want_d, metric, lambda r, b=b: oracle.distance(metric, vtype, q[b], x[r - 1]), (vtype, metric, b))
    g.close()


def test_group_quant_chunks(oracle):
    """the reference's shadow-table chunk format appended across shard boundaries"""
    import sqlite_vector_b200 as vs
    rng = np.random.Generator(np.random.PCG64(42))
    n, dim, k = 30_000, 48, 20
    xf = rng.standard_normal((n, dim), dtype=np.float32)
    scale, offset, qt = oracle.quant_params(po.F32, xf)
    rowids = np.arange(n, dtype=np.int64) * 2 + 1
    buf = oracle.build_quant_buffer(po.F32, xf, rowids, offset, scale, qt)
    g = vs.Group(po.I8, dim, n, 3)
    cut = (n // 7) * (8 + dim)
    g.append_quant_chunk(buf[:cut], n // 7)
    g.append_quant_chunk(buf[cut:], n - n // 7)
    g.finalize()
    qq = oracle.quantize(po.F32, rng.standard_normal(dim).astype(np.float32), offset, scale, qt)
    for metric in METRICS:
        (res,) = g.scan_topk(metric, qq, k)
        want_ids, want_d = oracle.scan_quant_buffer(metric, qt, qq, buf, n, dim, k)
        assert np.array_equal(res[0], want_ids) and np.array_equal(res[1], want_d), metric
    g.close()


def test_sql_surface_with_gpus_option():
    """vector_init(..., 'gpus=3'): preload + scans through SQL on three shards == the single-shard golden output"""
    import json

    from tests import sql_cases
    from tests.sqlrun import OURS, run_sql
    script = sql_cases.scan_script()
    sharded = [s.replace("dimension=24')", "dimension=24,gpus=3')").replace("dimension=16,distance=", "dimension=16,gpus=2,distance=") if isinstance(s, str) else s for s in script]
    assert sharded != script
    one, many = run_sql(OURS, script), run_sql(OURS, sharded)
    assert len(one) == len(many)
    for s, a, b in zip(script, one, many):
        st = s if isinstance(s, str) else s[0]
        if "rows" not in a or "rows" not in b:
            assert a == b, (st, a, b)
            continue
        assert len(a["rows"]) == len(b["rows"]), st
        for x, y in zip(a["rows"], b["rows"]):
            for u, v in zip(x, y):
                # fp columns: a row's position inside its warp tile decides the order of the fp32 partial sums, and that position
                # depends on where its shard starts: last-ulp differences (both within 1e-5 of the reference); ints are exact
                if isinstance(u, float) and isinstance(v, float):
                    assert abs(u - v) <= 2e-6 * max(abs(v), 1.0), (st, x, y)
                else:
                    assert u == v, (st, x, y)
    want = json.load(open(os.path.join(ROOT, "tests", "golden", "sql_scan.json")))
    assert sum("rows" in r for r in many) == sum("rows" in r for r in want)


PEER_WORKER = r'''
import os, sys
import numpy as np
import torch, torch.distributed as dist
sys.path.insert(0, sys.argv[1])
import sqlite_vector_b200 as vs
from sqlite_vector_b200 import api, shard
from oracle import pyoracle as po
rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
ndev = torch.cuda.device_count()
local = rank % ndev                                   # two ranks may share one GPU
torch.cuda.set_device(local)
device = torch.device("cuda", local)
dist.init_process_group("gloo")                       # handles + barriers only; the data path is peer memory
eng = vs.load_engine()
rng = np.random.Generator(np.random.PCG64(4242))
n, dim, k, nq = 200_000, 128, 20, 45
x = rng.integers(-6, 7, (n, dim)).astype(np.int8)
q = rng.integers(-6, 7, (nq, dim)).astype(np.int8)
bounds = shard.shard_bounds(n, world)
lo, hi = bounds[rank], bounds[rank + 1]
ix = vs.Index(api.I8, dim, hi - lo, device=local, first_seq=lo)
ix.append_dense(x[lo:hi]); ix.finalize()
orc = po.Oracle()
rowids = np.arange(1, n + 1, dtype=np.int64)
pitch = ix.query_pitch
qd = torch.zeros((nq, pitch), dtype=torch.uint8, device=device)
qd[:, :dim] = torch.from_numpy(q.view(np.uint8)).to(device)
torch.cuda.synchronize()
exch = shard.PeerExchange(ix, eng, world, rank, bounds, group=8)
for on_device in (True, False):
    for metric in (api.L2, api.DOT):
        results, pending = [], []
        for g0 in range(0, nq, exch.group):
            m = min(exch.group, nq - g0)
            t = exch.submit_strided(metric, qd[g0].data_ptr(), pitch, m, k, True) if on_device else exch.submit_strided(metric, q[g0:g0 + m], q.strides[0], m, k, False)
            pending.append(t)
            if len(pending) == exch.max_in_flight:
                results += exch.finish(pending.pop(0))
        while pending:
            results += exch.finish(pending.pop(0))
        assert len(results) == nq
        for b in range(nq):
            want_ids, want_d = orc.scan_dense(metric, po.I8, q[b], x, rowids, k)
            assert np.array_equal(results[b][0], want_ids) and np.array_equal(results[b][1], want_d), (rank, on_device, metric, b)
r1 = exch.query(api.L1, q[3], 7, on_device=False)
want_ids, want_d = orc.scan_dense(po.L1, po.I8, q[3], x, rowids, 7)
assert np.array_equal(r1[0], want_ids) and np.array_equal(r1[1], want_d)
# k = 256: more than 1024 survivors per shard -> the tails travel too; and a group of 8
for kk in (256, 20):
    for b in (0, 7):
        rr = exch.query(api.L2, q[b], kk, on_device=False)
        want_ids, want_d = orc.scan_dense(po.L2, po.I8, q[b], x, rowids, kk)
        assert np.array_equal(rr[0], want_ids) and np.array_equal(rr[1], want_d), (rank, "tail", kk, b)
t = exch.submit_strided(api.DOT, q[8:16], q.strides[0], 8, 20, False)
for j, rr in enumerate(exch.finish(t)):
    want_ids, want_d = orc.scan_dense(po.DOT, po.I8, q[8 + j], x, rowids, 20)
    assert np.array_equal(rr[0], want_ids) and np.array_equal(rr[1], want_d), (rank, "group", j)
# ---- batched queries: entry logs pushed over peer memory, device-side wait, GPU merge; two batches in flight
qb = rng.integers(-6, 7, (70, dim)).astype(np.int8)
for metric, kk in ((api.L2, 20), (api.COSINE, 100), (api.DOT, 7)):
    t1 = exch.batch_submit(metric, qb[:40], kk)
    t2 = exch.batch_submit(metric, qb[40:], kk)
    res = exch.batch_finish(t1) + exch.batch_finish(t2)
    for b in range(70):
        want_ids, want_d = orc.scan_dense(metric, po.I8, qb[b], x, rowids, kk)
        assert np.array_equal(res[b][0], want_ids) and np.array_equal(res[b][1], want_d), (rank, "batch", metric, b)
# a longer pipeline (the buffers are reused, the merge of batch j overlaps the levels of batch j + 1)
qp = rng.integers(-6, 7, (7, 24, dim)).astype(np.int8)
want_p = [[orc.scan_dense(po.L2, po.I8, qp[j, b], x, rowids, 10) for b in range(24)] for j in range(7)]
got, pend = [], None
for j in range(7):
    t = exch.batch_submit(api.L2, qp[j], 10)
    if pend is not None:
        got.append(exch.batch_finish(pend))
    pend = t
got.append(exch.batch_finish(pend))
for j in range(7):
    for b in range(24):
        assert np.array_equal(got[j][b][0], want_p[j][b][0]) and np.array_equal(got[j][b][1], want_p[j][b][1]), (rank, "pipeline", j, b)
# a shard-local capacity overflow (descending distances: every row enters the slots) must reach EVERY rank as ERANGE
xo = np.zeros((n, 16), dtype=np.int8)
xo[:, 0] = np.clip((n - 1 - np.arange(n)) // 1600, 0, 124).astype(np.int8)
xo[:, 1] = ((n - 1 - np.arange(n)) % 1600 // 13).astype(np.int8)
ixo = vs.Index(api.I8, 16, hi - lo, device=local, first_seq=lo)
ixo.append_dense(xo[lo:hi]); ixo.finalize()
exo = shard.PeerExchange(ixo, eng, world, rank, bounds, group=8)
overflowed = 0
try:
    exo.batch_finish(exo.batch_submit(api.L2, np.zeros((16, 16), dtype=np.int8), 5))
except vs.VsbError as ex:
    assert ex.rc == api.ERANGE, ex
    overflowed = 1
flags = [None] * world
dist.all_gather_object(flags, overflowed)
assert flags == [1] * world, flags            # the verdict travels inside the pushed blocks: the same on every rank
# the first exchange is unaffected
r2 = exch.query(api.L2, q[5], 9, on_device=False)
want_ids, want_d = orc.scan_dense(po.L2, po.I8, q[5], x, rowids, 9)
assert np.array_equal(r2[0], want_ids) and np.array_equal(r2[1], want_d)
dist.barrier()
if rank == 0: print("PEER_EXCHANGE_OK", world, "ranks on", min(world, ndev), "GPU(s)")
dist.destroy_process_group()
'''


@pytest.mark.parametrize("world", [2, 3])
def test_peer_exchange_between_processes(tmp_path, world):
    script = tmp_path / "peer_worker.py"
    script.write_text(PEER_WORKER)
    env = dict(os.environ, MASTER_ADDR="127.0.0.1")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr", "127.0.0.1",
                        "--master-port", str(29640 + world), str(script), ROOT], capture_output=True, text=True, timeout=900, env=env)
    assert r.returncode == 0 and "PEER_EXCHANGE_OK" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]


# ---------------------------------------------------------------- f3: corpora larger than the device budget (streamed windows)
def test_streamed_index_matches_oracle(oracle):
    """vsb_index_create_streamed: the column stays in pinned host memory and passes through two device windows; every window is
    scanned like a shard.  Same results as a resident index: bit-exact for int8 (ties, k sequence, k > 256, overflow fallback,
    all-distances), 1e-5 for fp."""
    import sqlite_vector_b200 as vs
    from tests.fpcheck import assert_fp_topk
    rng = np.random.Generator(np.random.PCG64(2027))
    n, dim = 61_234, 64                                      # 13 windows of 5000 rows, the last one ragged
    x = rng.integers(-5, 6, (n, dim)).astype(np.int8)
    rowids = np.arange(n, dtype=np.int64) * 3 + 2
    ix = vs.Index(po.I8, dim, n, window_rows=5000)
    for a in range(0, n, 7000):
        ix.append_dense(x[a:a + 7000], rowids[a:a + 7000])
    ix.finalize()
    for i, k in enumerate([20, 100, 10, 33, 300, 1]):
        q = rng.integers(-5, 6, dim).astype(np.int8)
        metric = METRICS[i % 5]
        (res,), mi = ix.scan_topk(metric, q, k, max_index=min(1, k - 1))
        want_ids, want_d = oracle.scan_dense(metric, po.I8, q, x, rowids, k, start_max_index=min(1, k - 1))
        assert np.array_equal(res[0], want_ids) and np.array_equal(res[1], want_d), (metric, k)
    d = ix.scan_all(po.L2, x[17])
    assert np.array_equal(d, oracle.distances_all(po.L2, po.I8, x[17], x, int_exact=True))
    res = ix.scan_topk(po.DOT, x[:20].copy(), 5)             # 20 queries: no tensor-core path on a streamed index, per-query loop
    for b in range(20):
        want_ids, want_d = oracle.scan_dense(po.DOT, po.I8, x[b], x, rowids, 5)
        assert np.array_equal(res[b][0], want_ids) and np.array_equal(res[b][1], want_d), b
    assert ix.stat("stream_bytes") > 0
    ix.close()
    # overflow inside windows (descending distances) -> all-distances fallback, streamed as well
    n2 = 90_000
    y = np.zeros((n2, 16), dtype=np.int8)
    y[:, 0] = np.clip(np.arange(n2)[::-1] // 720, 0, 127)
    ix = vs.Index(po.I8, 16, n2, window_rows=40_000)
    ix.append_dense(y)
    ix.finalize()
    (res,) = ix.scan_topk(po.L1, np.zeros(16, dtype=np.int8), 20)
    want_ids, want_d = oracle.scan_dense(po.L1, po.I8, np.zeros(16, dtype=np.int8), y, np.arange(1, n2 + 1, dtype=np.int64), 20)
    assert np.array_equal(res[0], want_ids) and np.array_equal(res[1], want_d)
    ix.close()
    # fp
    xf = po.convert(rng.standard_normal((30_000, 96), dtype=np.float32), po.BF16)
    ix = vs.Index(po.BF16, 96, 30_000, window_rows=4096)
    ix.append_dense(xf)
    ix.finalize()
    ids = np.arange(1, 30_001, dtype=np.int64)
    for metric in (po.L2, po.COS, po.DOT):
        (res,) = ix.scan_topk(metric, xf[5], 20)
        want_ids, want_d = oracle.scan_dense(metric, po.BF16, xf[5], xf, ids, 20)
        assert_fp_topk(res[0], res[1], want_ids, want_d, metric, lambda r: oracle.distance(metric, po.BF16, xf[5], xf[r - 1]), ("bf16", metric))
    ix.close()


def test_group_and_sql_under_a_device_budget(oracle):
    """VSB_DEVICE_BUDGET_MB smaller than the column: the group's shards are streamed; the SQL scan script must still give the
    single-resident-shard output"""
    import sqlite_vector_b200 as vs
    from tests import sql_cases
    from tests.sqlrun import OURS, run_sql
    rng = np.random.Generator(np.random.PCG64(31))
    n, dim, k = 200_000, 128, 20                              # 25.6 MB of int8 against a 4 MB budget
    x = rng.integers(-6, 7, (n, dim)).astype(np.int8)
    old = os.environ.get("VSB_DEVICE_BUDGET_MB")
    os.environ["VSB_DEVICE_BUDGET_MB"] = "4"
    try:
        for ngpus in (1, 3):
            g = _group(po.I8, x, ngpus)
            assert vs.load_engine().lib.vsb_index_is_streamed(vs.load_engine().lib.vsb_group_shard(g.h, 0)) == 1
            q = rng.integers(-6, 7, dim).astype(np.int8)
            (res,) = g.scan_topk(po.L2, q, k)
            want_ids, want_d = oracle.scan_dense(po.L2, po.I8, q, x, np.arange(1, n + 1, dtype=np.int64), k)
            assert np.array_equal(res[0], want_ids) and np.array_equal(res[1], want_d), ngpus
            g.close()
    finally:
        if old is None:
            os.environ.pop("VSB_DEVICE_BUDGET_MB", None)
        else:
            os.environ["VSB_DEVICE_BUDGET_MB"] = old
    script = sql_cases.scan_script()
    one = run_sql(OURS, script)
    tiny = run_sql(OURS, script, env={"VSB_DEVICE_BUDGET_MB": "0.01"})     # 10 KB: the 600 x 24 f32 table streams through 64-row windows
    for s, a, b in zip(script, one, tiny):
        st = s if isinstance(s, str) else s[0]
        if "rows" not in a or "rows" not in b:
            assert a == b, (st, a, b)
            continue
        assert len(a["rows"]) == len(b["rows"]), st
        for u, v in zip(a["rows"], b["rows"]):
            for p, w in zip(u, v):
                assert (abs(p - w) <= 2e-6 * max(abs(w), 1.0)) if isinstance(p, float) and isinstance(w, float) else p == w, (st, u, v)
