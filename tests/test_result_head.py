"""CPU checks of the result-head format through vsb_merge_result_blocks / vsb_merge_result_groups.

A head is what filter_kernel writes for one query on one shard: a 64-byte header (total, flags, seq, nblocks, xseq, src,
headcap as int32), a table of (base, count) per filter block, then the first 1024 survivors as (distance bits, local row).
The merge walks each shard's survivors in block-table order and replays them through the reference's slot algorithm."""
import numpy as np
import pytest

HDR_BYTES, TABLE_CAP, HEAD_CAP = 64, 512, 1024
SURV_OFF = HDR_BYTES + 8 * TABLE_CAP
HEAD_BYTES = SURV_OFF + 8 * HEAD_CAP
FLAG_OVERFLOW, FLAG_PEER_LATE = 1, 8


@pytest.fixture(scope="module")
def eng():
    import sqlite_vector_b200 as vs
    return vs.load_engine()


def make_head(dists, table, total=None, flags=0, headcap=0, nblocks=None):
    """one head: survivor i is stored at position i with local row i; table = [(base, count)] in block order"""
    blk = np.zeros(HEAD_BYTES, dtype=np.uint8)
    d = np.asarray(dists, dtype=np.float32)
    hdr = blk[:HDR_BYTES].view(np.int32)
    hdr[0] = len(d) if total is None else total
    hdr[1], hdr[2] = flags, 1
    hdr[3] = len(table) if nblocks is None else nblocks
    hdr[6] = headcap
    blk[HDR_BYTES:SURV_OFF].view(np.int32).reshape(-1, 2)[:len(table)] = np.asarray(table, dtype=np.int32).reshape(-1, 2)
    out = blk[SURV_OFF:].view(np.uint32).reshape(-1, 2)
    out[:len(d), 0] = d.view(np.uint32)
    out[:len(d), 1] = np.arange(len(d), dtype=np.uint32)
    return blk


def table_order(dists, table, first_seq):
    """(distances, rowids) in block-table order, rowid = first_seq + local row + 1"""
    rows = np.array([b + i for b, c in table for i in range(c)], dtype=np.int64)
    return np.asarray(dists, dtype=np.float32)[rows], first_seq + rows + 1


def replay(eng, dists, ids, k):
    from sqlite_vector_b200 import api
    c = np.zeros(len(dists), dtype=api.CAND_DTYPE)
    c["dist"], c["rowid"] = dists, ids
    got_ids, got_d, _ = eng.replay_topk(c, k)
    return got_ids, got_d


def merge(eng, heads, first_seq, k):
    return eng.merge_result_blocks(np.concatenate(heads), len(heads), HEAD_BYTES, np.asarray(first_seq), k)


def test_block_table_order_decides_replay_order(eng):
    rng = np.random.Generator(np.random.PCG64(41))
    d = rng.integers(0, 3, 60).astype(np.float32)           # three values: every slot decision is a tie break
    table = [(45, 15), (0, 20), (35, 10), (20, 15)]           # blocks stored out of table order
    k = 7
    ids, dist = merge(eng, [make_head(d, table)], [1000], k)
    want = replay(eng, *table_order(d, table, 1000), k)
    stored = replay(eng, d, 1000 + np.arange(60) + 1, k)
    assert not np.array_equal(want[0], stored[0])             # the data tells the two orders apart
    assert np.array_equal(ids, want[0]) and np.array_equal(dist, want[1])


def test_shards_replay_in_shard_order_with_empty_blocks(eng):
    rng = np.random.Generator(np.random.PCG64(43))
    d0 = rng.integers(0, 4, 12).astype(np.float32)
    d2 = rng.integers(0, 4, 9).astype(np.float32)
    t0 = [(0, 0), (0, 5), (5, 0), (5, 7), (12, 0)]
    t2 = [(4, 5), (4, 0), (0, 4)]
    first_seq = [0, 100, 200]
    heads = [make_head(d0, t0), make_head([], []), make_head(d2, t2)]
    parts = [table_order(d0, t0, 0), table_order(d2, t2, 200)]
    for k in (1, 5, 30):
        ids, dist = merge(eng, heads, first_seq, k)
        want = replay(eng, np.concatenate([p[0] for p in parts]), np.concatenate([p[1] for p in parts]), k)
        assert np.array_equal(ids, want[0]) and np.array_equal(dist, want[1]), k


def test_all_empty_shards(eng):
    ids, dist = merge(eng, [make_head([], []), make_head([], [(0, 0), (0, 0)])], [0, 5], 4)
    assert len(ids) == 0 and len(dist) == 0


@pytest.mark.parametrize("headcap", [1, 7, 1024])
def test_headcap_in_range_is_honoured(eng, headcap):
    from sqlite_vector_b200 import api
    d = np.arange(headcap, 0, -1).astype(np.float32)
    ids, dist = merge(eng, [make_head(d, [(0, headcap)], headcap=headcap)], [0], 3)
    want = replay(eng, *table_order(d, [(0, headcap)], 0), 3)
    assert np.array_equal(ids, want[0]) and np.array_equal(dist, want[1])
    with pytest.raises(api.VsbError, match=rf"has {headcap + 1} candidates \(> {headcap} ") as e:
        merge(eng, [make_head(d, [(0, headcap)], total=headcap + 1, headcap=headcap)], [0], 3)
    assert e.value.rc == api.ERANGE


@pytest.mark.parametrize("headcap", [0, -1, 1025, 4096])
def test_headcap_out_of_range_falls_back_to_head_capacity(eng, headcap):
    from sqlite_vector_b200 import api
    d = np.arange(HEAD_CAP, 0, -1).astype(np.float32)
    ids, dist = merge(eng, [make_head(d, [(0, HEAD_CAP)], headcap=headcap)], [0], 3)
    assert np.array_equal(ids, [HEAD_CAP, HEAD_CAP - 1, HEAD_CAP - 2]) and np.array_equal(dist, [1, 2, 3])
    with pytest.raises(api.VsbError, match=rf"has {HEAD_CAP + 1} candidates \(> {HEAD_CAP} ") as e:
        merge(eng, [make_head(d, [(0, HEAD_CAP)], total=HEAD_CAP + 1, headcap=headcap)], [0], 3)
    assert e.value.rc == api.ERANGE


def test_overflow_flag_is_erange(eng):
    from sqlite_vector_b200 import api
    with pytest.raises(api.VsbError, match="shard 1 reported a candidate overflow") as e:
        merge(eng, [make_head([1, 2], [(0, 2)]), make_head([3], [(0, 1)], flags=FLAG_OVERFLOW)], [0, 10], 2)
    assert e.value.rc == api.ERANGE


@pytest.mark.parametrize("flags", [FLAG_PEER_LATE, FLAG_PEER_LATE | FLAG_OVERFLOW])
def test_peer_late_flag_is_ecuda(eng, flags):
    from sqlite_vector_b200 import api
    with pytest.raises(api.VsbError, match="shard 1 did not deliver its result head") as e:
        merge(eng, [make_head([1, 2], [(0, 2)]), make_head([3], [(0, 1)], flags=flags)], [0, 10], 2)
    assert e.value.rc == api.ECUDA


@pytest.mark.parametrize("nblocks", [-1, TABLE_CAP + 1])
def test_malformed_block_count_is_ecuda(eng, nblocks):
    from sqlite_vector_b200 import api
    with pytest.raises(api.VsbError, match="malformed result head from shard 0") as e:
        merge(eng, [make_head([1, 2], [(0, 2)], nblocks=nblocks)], [0], 2)
    assert e.value.rc == api.ECUDA


def test_full_block_table_is_accepted(eng):
    d = np.arange(TABLE_CAP, dtype=np.float32)[::-1].copy()
    table = [(i, 1) for i in range(TABLE_CAP)][::-1]
    ids, dist = merge(eng, [make_head(d, table)], [0], 4)
    want = replay(eng, *table_order(d, table, 0), 4)
    assert np.array_equal(ids, want[0]) and np.array_equal(dist, want[1])


def test_group_merge_checks_every_query(eng):
    from sqlite_vector_b200 import api
    rng = np.random.Generator(np.random.PCG64(47))
    world, G, k = 2, 3, 4
    first_seq = [0, 50]
    ds = [[rng.integers(0, 3, 20).astype(np.float32) for _ in range(G)] for _ in range(world)]
    tables = [[(10, 10), (0, 10)], [(0, 0), (0, 20)]]
    # rank-major: rank r's heads of queries 0..G-1, then rank r + 1's
    blocks = np.concatenate([make_head(ds[r][j], tables[r]) for r in range(world) for j in range(G)])
    res = eng.merge_result_groups(blocks, world, G * HEAD_BYTES, HEAD_BYTES, G, np.asarray(first_seq), k)
    for j in range(G):
        parts = [table_order(ds[r][j], tables[r], first_seq[r]) for r in range(world)]
        want = replay(eng, np.concatenate([p[0] for p in parts]), np.concatenate([p[1] for p in parts]), k)
        assert np.array_equal(res[j][0], want[0]) and np.array_equal(res[j][1], want[1]), j
    bad = blocks.copy()
    bad[(G + 1) * HEAD_BYTES:].view(np.int32)[1] = FLAG_OVERFLOW      # rank 1, query 1
    with pytest.raises(api.VsbError, match="shard 1 reported a candidate overflow") as e:
        eng.merge_result_groups(bad, world, G * HEAD_BYTES, HEAD_BYTES, G, np.asarray(first_seq), k)
    assert e.value.rc == api.ERANGE
