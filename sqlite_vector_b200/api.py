"""ctypes mirror of include/vsb200.h.  Fails loudly when the CUDA library is missing."""
from __future__ import annotations

import ctypes as C
import os
import weakref

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "lib", "libvsb200.so")

F32, F16, BF16, U8, I8 = 1, 2, 3, 4, 5
L2, SQUARED_L2, COSINE, DOT, L1 = 1, 2, 3, 4, 5
ELEM_SIZE = {F32: 4, F16: 2, BF16: 2, U8: 1, I8: 1}


class VsbError(RuntimeError):
    """rc: the VSB_E* code (callers fall back on VSB_ERANGE only; everything else is a real failure)"""

    def __init__(self, msg, rc: int = -1):
        super().__init__(msg)
        self.rc = rc


EINVAL, ENODEV, ENOMEM, ECUDA, ERANGE = -1, -2, -3, -4, -5


class Candidate(C.Structure):
    _fields_ = [("rowid", C.c_int64), ("seq", C.c_int64), ("dist", C.c_float), ("reserved", C.c_int32)]


CAND_DTYPE = np.dtype([("rowid", "<i8"), ("seq", "<i8"), ("dist", "<f4"), ("reserved", "<i4")])

_vp, _i, _i64 = C.c_void_p, C.c_int, C.c_int64

_SIGNATURES = {
    "vsb_device_count": (_i, []),
    "vsb_last_error": (C.c_char_p, []),
    "vsb_backend_name": (C.c_char_p, []),
    "vsb_index_create": (_i, [C.POINTER(_vp), _i, _i, _i, _i64, _i64]),
    "vsb_index_create_streamed": (_i, [C.POINTER(_vp), _i, _i, _i, _i64, _i64, _i64]),
    "vsb_index_is_streamed": (_i, [_vp]),
    "vsb_index_append_dense": (_i, [_vp, _vp, _vp, _i64]),
    "vsb_index_append_quant_chunk": (_i, [_vp, _vp, _i64]),
    "vsb_index_append_device": (_i, [_vp, _vp, _vp, _i64]),
    "vsb_index_finalize": (_i, [_vp]),
    "vsb_index_rows": (_i64, [_vp]),
    "vsb_index_device_bytes": (_i64, [_vp]),
    "vsb_index_free": (None, [_vp]),
    "vsb_scan_topk": (_i, [_vp, _i, _vp, _i, _i, _vp, _vp, _vp, _vp]),
    "vsb_scan_topk_filtered": (_i, [_vp, _i, _vp, _i, _i, _vp, _i64, _vp, _vp, _vp, _vp]),
    "vsb_index_rowid_bitmap": (_i64, [_vp, _vp, _i64, _vp]),
    "vsb_scan_topk_rows": (_i, [_vp, _i, _vp, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp]),
    "vsb_scan_topk_sets": (_i, [_vp, _i, _vp, _i, _i, _vp, _i, _i64, _vp, _vp, _vp, _vp, _vp]),
    "vsb_scan_topk_grouped": (_i, [_vp, _i, _vp, _i, _i, _vp, _vp, _i, _i, C.POINTER(_vp)]),
    "vsb_grouped_get": (_i, [_vp, _i, C.POINTER(_i), C.POINTER(_vp), C.POINTER(_vp), C.POINTER(_vp), C.POINTER(_vp)]),
    "vsb_grouped_free": (None, [_vp]),
    "vsb_grouping_create": (_i, [_vp, _vp, _vp, _i, C.POINTER(_vp)]),
    "vsb_scan_topk_grouping": (_i, [_vp, _i, _vp, _i, _i, _i, C.POINTER(_vp)]),
    "vsb_grouping_free": (None, [_vp]),
    "vsb_scan_range": (_i, [_vp, _i, _vp, _i, _vp, _vp, _i64, C.POINTER(_vp)]),
    "vsb_range_get": (_i, [_vp, _i, C.POINTER(_vp), C.POINTER(_vp), C.POINTER(_i64)]),
    "vsb_range_free": (None, [_vp]),
    "vsb_scan_all": (_i, [_vp, _i, _vp, _vp, _vp]),
    "vsb_scan_candidates": (_i, [_vp, _i, _vp, _i, _i, _vp, _i, _vp]),
    "vsb_replay_topk": (_i, [_vp, _i, _i, _vp, _vp, _vp]),
    "vsb_scan_device_query": (_i, [_vp, _i, _vp, _i]),
    "vsb_scan_submit": (_i, [_vp, _i, _vp, _i, _i, _i, _i]),
    "vsb_scan_submit_group": (_i, [_vp, _i, _vp, _i64, _i, _i, _i, _i, _i]),
    "vsb_merge_result_groups": (_i, [_vp, _i, _i64, _i64, _i, _vp, _i, _vp, _vp, _vp]),
    "vsb_collect_last": (_i, [_vp, _i, _vp, _vp, _vp]),
    "vsb_collect": (_i, [_vp, _i, _i, _vp, _vp, _vp]),
    "vsb_result_block": (_i, [_vp, _i, C.POINTER(_vp), C.POINTER(_i64)]),
    "vsb_merge_result_blocks": (_i, [_vp, _i, _i64, _vp, _i, _vp, _vp]),
    "vsb_batch_shard_scan": (_i, [_vp, _i, _vp, _i, _i, C.POINTER(_vp), C.POINTER(_i64)]),
    "vsb_batch_merge": (_i, [_vp, _vp, _i, _i64, _vp, _i, _i, _vp, _vp, _vp]),
    "vsb_index_lookup_rowids": (_i, [_vp, _vp, _i64, _vp]),
    "vsb_exchange_export": (_i, [_vp, _i, _i, _vp]),
    "vsb_exchange_attach": (_i, [_vp, _vp]),
    "vsb_exchange_submit": (_i, [_vp, _i, _vp, _i64, _i, _i, _i, _i]),
    "vsb_exchange_collect": (_i, [_vp, _i, _i, _vp, _i, _vp, _vp, _vp]),
    "vsb_exchange_batch_submit": (_i, [_vp, _i, _vp, _i, _i, _vp]),
    "vsb_exchange_batch_collect": (_i, [_vp, _i, _i, _i, _vp, _vp, _vp]),
    "vsb_group_create": (_i, [C.POINTER(_vp), _i, _i, _i, _i, _i64]),
    "vsb_group_append_dense": (_i, [_vp, _vp, _vp, _i64]),
    "vsb_group_append_quant_chunk": (_i, [_vp, _vp, _i64]),
    "vsb_group_finalize": (_i, [_vp]),
    "vsb_group_scan_topk": (_i, [_vp, _i, _vp, _i, _i, _vp, _vp, _vp, _vp]),
    "vsb_group_scan_all": (_i, [_vp, _i, _vp, _vp, _vp]),
    "vsb_group_scan_topk_filtered": (_i, [_vp, _i, _vp, _i, _i, _vp, _i64, _vp, _vp, _vp, _vp]),
    "vsb_group_rowid_bitmap": (_i64, [_vp, _vp, _i64, _vp]),
    "vsb_group_scan_topk_rows": (_i, [_vp, _i, _vp, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp]),
    "vsb_group_scan_topk_sets": (_i, [_vp, _i, _vp, _i, _i, _vp, _i, _i64, _vp, _vp, _vp, _vp, _vp]),
    "vsb_group_scan_topk_grouped": (_i, [_vp, _i, _vp, _i, _i, _vp, _vp, _i, _i, C.POINTER(_vp)]),
    "vsb_group_grouping_create": (_i, [_vp, _vp, _vp, _i, C.POINTER(_vp)]),
    "vsb_group_scan_range": (_i, [_vp, _i, _vp, _i, _vp, _vp, _i64, C.POINTER(_vp)]),
    "vsb_group_gpus": (_i, [_vp]),
    "vsb_group_rows": (_i64, [_vp]),
    "vsb_group_shard": (_vp, [_vp, _i]),
    "vsb_group_free": (None, [_vp]),
    "vsb_quantizer_create": (_i, [C.POINTER(_vp), _i, _i, _i, _i64]),
    "vsb_quantizer_minmax": (_i, [_vp, _vp, _i64]),
    "vsb_quantizer_minmax_result": (_i, [_vp, _vp, _vp, _vp]),
    "vsb_quantizer_retained_rows": (_i64, [_vp]),
    "vsb_quantizer_encode": (_i, [_vp, _vp, _i64, _vp, _i64, C.c_float, C.c_float, _i, _vp]),
    "vsb_quantizer_free": (None, [_vp]),
    "vsb_index_query_pitch": (_i, [_vp]),
    "vsb_index_stream": (_vp, [_vp]),
    "vsb_index_stat": (_i64, [_vp, C.c_char_p]),
    "vsb_kernel_launches": (_i64, []),
    "vsb_debug_live_handles": (_i64, []),
    "vsb_set_option": (_i, [C.c_char_p, _i]),
    "vsb_profile_read": (_i, [_vp, _vp, _vp, _vp, _vp]),
    "vsb_debug_read": (_i, [_vp, C.c_char_p, _vp, _i64]),
    "vsb_debug_write": (_i, [_vp, C.c_char_p, _vp, _i64]),
    "vsb_debug_survivors": (_i64, [_vp, _i, _vp, _i64, C.POINTER(_i)]),
    "vsb_debug_tc_level": (_i, [_vp, _i, _vp, _i, _vp, _i64, _i64, _i, _i, _vp, _i64, _vp, _vp, C.POINTER(_i64)]),
    "vsb_debug_tc_level_filtered": (_i, [_vp, _i, _vp, _i, _vp, _i64, _i64, _i, _i, _vp, _i64, _i64, _vp, _i, _vp, _vp, _i64, _vp, _vp,
                                         C.POINTER(_i64)]),
    "vsb_debug_refine": (_i, [_vp, _i, _vp, _i, _vp, _i64, _vp, _i64, _vp, _vp, _vp]),
    "vsb_debug_replay": (_i, [_vp, _i, _vp, _i, _i, _i, _vp, _vp, _vp, _vp, _vp, _i, _vp, _vp, _i, _vp, _vp, _vp, _vp]),
}

BUCKET_CAP = 2048              # kept candidates per query and level of the batch path (kBucketCap)


def _ptr(a):
    if a is None:
        return None
    if not a.flags["C_CONTIGUOUS"]:
        raise ValueError("array must be C-contiguous")
    return a.ctypes.data_as(C.c_void_p)


class Engine:
    def __init__(self, path: str = LIB_PATH):
        if not os.path.exists(path):
            raise VsbError(f"{path} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                           "(there is no CPU fallback)")
        self.path = path
        self.lib = C.CDLL(path)
        for name, (res, args) in _SIGNATURES.items():
            fn = getattr(self.lib, name)  # AttributeError => header and library disagree
            fn.restype = res
            fn.argtypes = args

    def check(self, rc: int):
        if rc != 0:
            raise VsbError(f"vsb error {rc}: {self.lib.vsb_last_error().decode()}", rc)

    def device_count(self) -> int:
        return self.lib.vsb_device_count()

    def backend_name(self) -> str:
        return self.lib.vsb_backend_name().decode()

    def kernel_launches(self) -> int:
        return int(self.lib.vsb_kernel_launches())

    def debug_live_handles(self) -> int:
        return int(self.lib.vsb_debug_live_handles())

    def set_option(self, name: str, value: int) -> int:
        return self.lib.vsb_set_option(name.encode(), int(value))

    def merge_result_blocks(self, blocks: np.ndarray, world: int, stride: int, first_seq: np.ndarray, k: int):
        ids = np.zeros(max(k, 1), dtype=np.int64)
        dist = np.zeros(max(k, 1), dtype=np.float64)
        fs = np.ascontiguousarray(first_seq, dtype=np.int64)
        cnt = self.lib.vsb_merge_result_blocks(_ptr(blocks), world, stride, _ptr(fs), k, _ptr(ids), _ptr(dist))
        if cnt < 0:
            self.check(cnt)
        return ids[:cnt], dist[:cnt]

    def merge_result_groups(self, blocks: np.ndarray, world: int, rank_stride: int, block_stride: int, nq: int, first_seq: np.ndarray, k: int):
        """merge a gathered group of nq queries in one call; returns a list of (rowids, distances)"""
        ids = np.zeros((nq, max(k, 1)), dtype=np.int64)
        dist = np.zeros((nq, max(k, 1)), dtype=np.float64)
        counts = np.zeros(nq, dtype=np.int32)
        fs = np.ascontiguousarray(first_seq, dtype=np.int64)
        self.check(self.lib.vsb_merge_result_groups(_ptr(blocks), world, rank_stride, block_stride, nq, _ptr(fs), k, _ptr(ids), _ptr(dist), _ptr(counts)))
        return [(ids[j, :counts[j]], dist[j, :counts[j]]) for j in range(nq)]

    def replay_topk(self, cands: np.ndarray, k: int, max_index: int = 0):
        cands = np.ascontiguousarray(cands, dtype=CAND_DTYPE)
        ids = np.zeros(max(k, 1), dtype=np.int64)
        dist = np.zeros(max(k, 1), dtype=np.float64)
        mi = C.c_int(max_index)
        cnt = self.lib.vsb_replay_topk(_ptr(cands), cands.shape[0], k, C.byref(mi), _ptr(ids), _ptr(dist))
        if cnt < 0:
            self.check(cnt)
        return ids[:cnt].copy(), dist[:cnt].copy(), mi.value


def row_bitmap(mask) -> np.ndarray:
    """boolean mask over scan-order rows -> the row bitmap of the filtered scans (uint32 words, row i: bit i & 31 of word i >> 5)"""
    b = np.packbits(np.ascontiguousarray(mask, dtype=bool), bitorder="little")
    return np.concatenate([b, np.zeros((-len(b)) % 4, np.uint8)]).view("<u4").copy()


def _allow_words(allow, rows: int) -> np.ndarray:
    """a bitmap of the filtered scans from a boolean mask of `rows` rows or from uint32 words"""
    a = np.asarray(allow)
    if a.dtype == bool:
        if a.shape != (rows,):
            raise ValueError(f"the mask has {a.shape} entries, the column {rows} rows")
        return row_bitmap(a)
    w = np.ascontiguousarray(a, dtype=np.uint32)
    if w.size < (rows + 31) // 32:
        raise ValueError(f"the bitmap has {w.size} words, {rows} rows need {(rows + 31) // 32}")
    return w


def _topk(eng: "Engine", call, queries: np.ndarray, k: int, max_index: int | None, as_arrays: bool):
    """the output handling of the scan_topk entry points: call(queries, nq, ids, dist, counts, max_index pointer) -> rc"""
    q = np.ascontiguousarray(queries)
    q2 = q.reshape(-1, q.shape[-1]) if q.ndim > 1 else q.reshape(1, -1)
    nq = q2.shape[0]
    ids = np.zeros((nq, max(k, 1)), dtype=np.int64)
    dist = np.zeros((nq, max(k, 1)), dtype=np.float64)
    counts = np.zeros(nq, dtype=np.int32)
    mi = C.c_int(0 if max_index is None else max_index)
    eng.check(call(_ptr(q2), nq, _ptr(ids), _ptr(dist), _ptr(counts), C.byref(mi) if max_index is not None else None))
    if as_arrays:
        return ((ids, dist, counts), mi.value) if max_index is not None else (ids, dist, counts)
    out = [(ids[b, :counts[b]].copy(), dist[b, :counts[b]].copy()) for b in range(nq)]
    return (out, mi.value) if max_index is not None else out


def _rows_topk(eng: "Engine", fn, h, metric: int, queries: np.ndarray, k: int, rowid_lists, max_index: int | None, as_arrays: bool):
    """the listed-rows entry points: fn(handle, metric, queries, nq, k, rowids, offsets, ids, dist, counts, max_index) -> rc;
    rowid_lists holds one sequence of rowids per query"""
    q = np.ascontiguousarray(queries)
    nq = 1 if q.ndim == 1 else int(np.prod(q.shape[:-1]))
    lists = [np.asarray(r, dtype=np.int64).reshape(-1) for r in rowid_lists]
    if len(lists) != nq:
        raise ValueError(f"{len(lists)} rowid lists for {nq} queries")
    offsets = np.zeros(nq + 1, dtype=np.int64)
    offsets[1:] = np.cumsum([len(r) for r in lists])
    flat = np.ascontiguousarray(np.concatenate(lists) if lists else np.zeros(0, np.int64))
    return _topk(eng, lambda qp, n, ids, dist, counts, mi: fn(h, metric, qp, n, k, _ptr(flat), _ptr(offsets), ids, dist, counts, mi),
                 q, k, max_index, as_arrays)


def _sets_topk(eng: "Engine", fn, h, rows: int, metric: int, queries: np.ndarray, k: int, sets, set_of_query, as_arrays: bool):
    """the per-query sets entry points: fn(handle, metric, queries, nq, k, sets, nsets, nbits, set_of_query, ids, dist, counts,
    max_index) -> rc; sets holds boolean masks or row bitmaps (or is one uint32 array [nsets, words]), set_of_query one set index per query (None: query b uses set b)"""
    words = (rows + 31) // 32
    if isinstance(sets, np.ndarray) and sets.dtype == np.uint32 and sets.ndim == 2 and sets.shape[1] == words and words > 0:
        flat = np.ascontiguousarray(sets)                      # already nsets bitmaps back to back
    else:
        bits = np.zeros((len(sets), max(words, 1)), dtype=np.uint32)
        for i, a in enumerate(sets):
            bits[i, :words] = _allow_words(a, rows)[:words]
        flat = np.ascontiguousarray(bits[:, :words]) if words > 0 else np.zeros(1, np.uint32)
    soq = None if set_of_query is None else np.ascontiguousarray(set_of_query, dtype=np.int32).reshape(-1)
    return _topk(eng, lambda qp, n, ids, dist, counts, mi: fn(h, metric, qp, n, k, _ptr(flat), len(sets), rows, _ptr(soq), ids, dist,
                                                            counts, mi),
                 queries, k, None, as_arrays)


def _range(eng: "Engine", fn, h, rows: int, metric: int, queries: np.ndarray, radius, allow):
    """the range entry points: fn(handle, metric, queries, nq, radius, allow, nbits, &result) -> rc; one (rowids, distances) pair
    per query, rows ordered by ascending distance (equal distances in scan order)"""
    q = np.ascontiguousarray(queries)
    q2 = q.reshape(-1, q.shape[-1]) if q.ndim > 1 else q.reshape(1, -1)
    nq = q2.shape[0]
    r = np.ascontiguousarray(np.broadcast_to(np.asarray(radius, dtype=np.float64), (nq,)))
    bits = None if allow is None else _allow_words(allow, rows)
    res = _vp()
    eng.check(fn(h, metric, _ptr(q2), nq, _ptr(r), _ptr(bits), rows if bits is not None else 0, C.byref(res)))
    out = []
    try:
        for b in range(nq):
            ids, dist, cnt = _vp(), _vp(), _i64()
            eng.check(eng.lib.vsb_range_get(res, b, C.byref(ids), C.byref(dist), C.byref(cnt)))
            n = int(cnt.value)
            if n == 0:
                out.append((np.zeros(0, np.int64), np.zeros(0, np.float64)))
                continue
            out.append((np.ctypeslib.as_array(C.cast(ids, C.POINTER(C.c_int64)), (n,)).copy(),
                        np.ctypeslib.as_array(C.cast(dist, C.POINTER(C.c_double)), (n,)).copy()))
    finally:
        eng.lib.vsb_range_free(res)
    return out


def _key_csr(key_lists):
    """one sequence of rowids per key -> (rowids, offsets) of the grouped entry points"""
    lists = [np.asarray(r, dtype=np.int64).reshape(-1) for r in key_lists]
    offsets = np.zeros(len(lists) + 1, dtype=np.int64)
    offsets[1:] = np.cumsum([len(r) for r in lists])
    return np.ascontiguousarray(np.concatenate(lists) if lists else np.zeros(0, np.int64)), offsets


def _grouped(eng: "Engine", fn, h, metric: int, queries: np.ndarray, k: int, key_lists, limit: int):
    """the grouped entry points: fn(handle, metric, queries, nq, k, rowids, offsets, nkeys, limit, &result) -> rc; per query a list
    of (key index, rowids, distances), keys in rank order"""
    flat, offsets = _key_csr(key_lists)
    return _grouped_call(eng, lambda qp, nq, res: fn(h, metric, qp, nq, k, _ptr(flat), _ptr(offsets), len(offsets) - 1, limit, res),
                         queries)


def _grouped_call(eng: "Engine", call, queries: np.ndarray):
    """call(queries, nq, &result) -> rc, and the result as _grouped returns it"""
    q = np.ascontiguousarray(queries)
    q2 = q.reshape(-1, q.shape[-1]) if q.ndim > 1 else q.reshape(1, -1)
    nq = q2.shape[0]
    res = _vp()
    eng.check(call(_ptr(q2), nq, C.byref(res)))
    out = []
    try:
        for b in range(nq):
            n, keys, offs, ids, dist = _i(), _vp(), _vp(), _vp(), _vp()
            eng.check(eng.lib.vsb_grouped_get(res, b, C.byref(n), C.byref(keys), C.byref(offs), C.byref(ids), C.byref(dist)))
            nk = n.value
            if nk == 0:
                out.append([])
                continue
            o = np.ctypeslib.as_array(C.cast(offs, C.POINTER(C.c_int64)), (nk + 1,))
            kk = np.ctypeslib.as_array(C.cast(keys, C.POINTER(C.c_int32)), (nk,))
            rid = np.ctypeslib.as_array(C.cast(ids, C.POINTER(C.c_int64)), (int(o[-1]),))
            dd = np.ctypeslib.as_array(C.cast(dist, C.POINTER(C.c_double)), (int(o[-1]),))
            out.append([(int(kk[i]), rid[o[i]:o[i + 1]].copy(), dd[o[i]:o[i + 1]].copy()) for i in range(nk)])
    finally:
        eng.lib.vsb_grouped_free(res)
    return out


def _rowid_bitmap(eng: "Engine", fn, h, rows: int, rowids) -> tuple[np.ndarray, int]:
    rid = np.ascontiguousarray(rowids, dtype=np.int64).reshape(-1)
    bits = np.zeros(max((rows + 31) // 32, 1), dtype=np.uint32)
    n = fn(h, _ptr(rid), rid.size, _ptr(bits))
    if n < 0:
        eng.check(int(n))
    return bits, int(n)


_ENGINE = None


def load_engine() -> Engine:
    global _ENGINE
    if _ENGINE is None:
        _ENGINE = Engine()
    return _ENGINE


class _Column:
    """The query methods of a column's shards, shared by Index and Group: each calls the C entry point `_prefix` + its name
    (vsb_scan_topk or vsb_group_scan_topk, ...); rows are in the column's scan order"""

    _prefix = ""
    _rowid_bitmap = ""

    def _fn(self, name: str):
        return getattr(self.eng.lib, self._prefix + name)

    def scan_topk(self, metric: int, queries: np.ndarray, k: int, max_index: int | None = None, as_arrays: bool = False):
        """top-k of one query or a batch.  Returns one (rowids, distances) pair per query, or with as_arrays the C-ABI's own
        output (rowids[nq, k], distances[nq, k], counts[nq]) without the per-query Python objects."""
        fn = self._fn("scan_topk")
        return _topk(self.eng, lambda q, nq, ids, dist, counts, mi: fn(self.h, metric, q, nq, k, ids, dist, counts, mi),
                     queries, k, max_index, as_arrays)

    def scan_topk_filtered(self, metric: int, queries: np.ndarray, k: int, allow, max_index: int | None = None, as_arrays: bool = False):
        """scan_topk among the eligible rows only (vsb_scan_topk_filtered): `allow` is a boolean mask over the scan-order rows or
        a uint32 row bitmap (row_bitmap, rowid_bitmap)"""
        bits, rows, fn = _allow_words(allow, self.rows), self.rows, self._fn("scan_topk_filtered")
        return _topk(self.eng, lambda q, nq, ids, dist, counts, mi: fn(self.h, metric, q, nq, k, _ptr(bits), rows, ids, dist, counts, mi),
                     queries, k, max_index, as_arrays)

    def scan_topk_rows(self, metric: int, queries: np.ndarray, k: int, rowid_lists, max_index: int | None = None, as_arrays: bool = False):
        """scan_topk among per-query lists of rowids, reading only the listed rows (vsb_scan_topk_rows): rowid_lists holds one
        sequence of rowids per query; each query's result equals scan_topk_filtered with the bitmap of its rowids"""
        return _rows_topk(self.eng, self._fn("scan_topk_rows"), self.h, metric, queries, k, rowid_lists, max_index, as_arrays)

    def scan_topk_sets(self, metric: int, queries: np.ndarray, k: int, sets, set_of_query=None, as_arrays: bool = False):
        """scan_topk of each query among its own set of rows (vsb_scan_topk_sets), one pass of the column for the whole batch:
        `sets` is a list of boolean masks over the scan-order rows or of uint32 row bitmaps, set_of_query[b] the index of query
        b's set (None: query b uses set b); each query's result equals scan_topk_filtered with its set"""
        return _sets_topk(self.eng, self._fn("scan_topk_sets"), self.h, self.rows, metric, queries, k, sets, set_of_query, as_arrays)

    def scan_topk_grouped(self, metric: int, queries: np.ndarray, k: int, key_lists, limit: int = 0):
        """each key's k nearest rows for the best keys (vsb_scan_topk_grouped): key_lists holds one sequence of rowids per key.
        Returns per query a list of (key index, rowids, distances), keys ranked by their first distance (then its scan row, then
        the key index) and cut to `limit` (0: every key with a row); each key's rows equal scan_topk_filtered with its rowids"""
        return _grouped(self.eng, self._fn("scan_topk_grouped"), self.h, metric, queries, k, key_lists, limit)

    def grouping(self, key_lists) -> "Grouping":
        """the keys laid out once for many grouped calls (vsb_grouping_create): Grouping.scan_topk answers as scan_topk_grouped
        with these key_lists.  The column's close() closes its groupings first"""
        return Grouping(self, key_lists)

    def _close_groupings(self):
        for g in list(getattr(self, "_groupings", ())):
            g.close()

    def scan_range(self, metric: int, queries: np.ndarray, radius, allow=None):
        """every row with distance < radius (vsb_scan_range), for one query or a batch; radius: one value or one per query, allow:
        None, a boolean mask over the scan-order rows or a uint32 row bitmap.  Returns one (rowids, distances) pair per query"""
        return _range(self.eng, self._fn("scan_range"), self.h, self.rows, metric, queries, radius, allow)

    def rowid_bitmap(self, rowids) -> tuple[np.ndarray, int]:
        """(row bitmap of the rows whose rowid is in `rowids`, number of such rows) (vsb_index_rowid_bitmap)"""
        return _rowid_bitmap(self.eng, getattr(self.eng.lib, self._rowid_bitmap), self.h, self.rows, rowids)

    def scan_all(self, metric: int, query: np.ndarray, want_rowids: bool = False):
        n = self.rows
        dist = np.zeros(n, dtype=np.float32)
        ids = np.zeros(n, dtype=np.int64) if want_rowids else None
        self.eng.check(self._fn("scan_all")(self.h, metric, _ptr(np.ascontiguousarray(query)), _ptr(dist), _ptr(ids)))
        return (dist, ids) if want_rowids else dist


class Index(_Column):
    """A resident shard of one column on one GPU (table_context.preloaded on the device)."""

    _prefix = "vsb_"
    _rowid_bitmap = "vsb_index_rowid_bitmap"

    def __init__(self, vtype: int, dim: int, capacity: int, device: int = 0, first_seq: int = 0, engine: Engine | None = None,
                 window_rows: int = 0):
        """window_rows > 0: streamed index (column in pinned host memory, two device windows of that many rows)"""
        self.eng = engine or load_engine()
        self.vtype, self.dim, self.device = vtype, dim, device
        h = _vp()
        if window_rows > 0:
            self.eng.check(self.eng.lib.vsb_index_create_streamed(C.byref(h), device, vtype, dim, capacity, first_seq, window_rows))
        else:
            self.eng.check(self.eng.lib.vsb_index_create(C.byref(h), device, vtype, dim, capacity, first_seq))
        self.h = h

    def close(self):
        if getattr(self, "h", None):
            self._close_groupings()
            self.eng.lib.vsb_index_free(self.h)
            self.h = None

    __del__ = close

    @property
    def rows(self) -> int:
        return int(self.eng.lib.vsb_index_rows(self.h))

    @property
    def query_pitch(self) -> int:
        return int(self.eng.lib.vsb_index_query_pitch(self.h))

    @property
    def stream(self) -> int:
        return int(self.eng.lib.vsb_index_stream(self.h) or 0)

    def append_dense(self, vectors: np.ndarray, rowids: np.ndarray | None = None):
        assert vectors.ndim == 2 and vectors.shape[1] * vectors.itemsize == self.dim * ELEM_SIZE[self.vtype]
        rid = None if rowids is None else np.ascontiguousarray(rowids, dtype=np.int64)
        self.eng.check(self.eng.lib.vsb_index_append_dense(self.h, _ptr(vectors), _ptr(rid), vectors.shape[0]))

    def append_quant_chunk(self, chunk: np.ndarray, nrows: int):
        self.eng.check(self.eng.lib.vsb_index_append_quant_chunk(self.h, _ptr(chunk), nrows))

    def append_device(self, d_ptr: int, nrows: int, d_rowids: int | None = None):
        self.eng.check(self.eng.lib.vsb_index_append_device(self.h, d_ptr, d_rowids, nrows))

    def finalize(self):
        self.eng.check(self.eng.lib.vsb_index_finalize(self.h))

    def scan_candidates(self, metric: int, queries: np.ndarray, k: int, cap: int = 8192):
        q2 = np.ascontiguousarray(queries).reshape(-1, queries.shape[-1])
        nq = q2.shape[0]
        out = np.zeros((nq, cap), dtype=CAND_DTYPE)
        counts = np.zeros(nq, dtype=np.int32)
        self.eng.check(self.eng.lib.vsb_scan_candidates(self.h, metric, _ptr(q2), nq, k, _ptr(out), cap, _ptr(counts)))
        return [out[b, :counts[b]].copy() for b in range(nq)]

    def scan_device_query(self, metric: int, d_query_ptr: int, k: int) -> int:
        slot = self.eng.lib.vsb_scan_device_query(self.h, metric, d_query_ptr, k)
        if slot < 0:
            self.eng.check(slot)
        return slot

    def scan_submit(self, metric: int, query, k: int, on_device: bool = False, fetch: bool = True, slot: int = -1) -> int:
        """asynchronous single-query scan; `query` is a device pointer (int) or a host array.  Returns the result slot."""
        if on_device:
            slot = self.eng.lib.vsb_scan_submit(self.h, metric, int(query), 1, k, int(fetch), slot)
        else:
            q = np.ascontiguousarray(query)
            slot = self.eng.lib.vsb_scan_submit(self.h, metric, _ptr(q), 0, k, int(fetch), slot)
        if slot < 0:
            self.eng.check(slot)
        return slot

    def scan_submit_group(self, metric: int, queries, stride: int, nq: int, k: int, on_device: bool, first_slot: int, fetch: bool = False):
        """nq independent queries in one call: `queries` is a device pointer (int) or a C-contiguous host array, query j at
        byte offset j * stride; result slots first_slot .. first_slot + nq - 1"""
        ptr = int(queries) if on_device else _ptr(queries)
        self.eng.check(self.eng.lib.vsb_scan_submit_group(self.h, metric, ptr, stride, nq, int(on_device), k, int(fetch), first_slot))

    def result_block(self, slot: int):
        """(device pointer, bytes) of the slot's result block"""
        ptr, nbytes = _vp(), _i64()
        self.eng.check(self.eng.lib.vsb_result_block(self.h, slot, C.byref(ptr), C.byref(nbytes)))
        return int(ptr.value), int(nbytes.value)

    def batch_shard_scan(self, metric: int, queries: np.ndarray, k: int):
        """tensor-core batch path over this shard; returns (device pointer, bytes) of the shard's entry-log block"""
        q2 = np.ascontiguousarray(queries).reshape(-1, queries.shape[-1])
        ptr, nbytes = _vp(), _i64()
        self.eng.check(self.eng.lib.vsb_batch_shard_scan(self.h, metric, _ptr(q2), q2.shape[0], k, C.byref(ptr), C.byref(nbytes)))
        return int(ptr.value), int(nbytes.value)

    def batch_merge(self, d_blocks: int, world: int, stride: int, first_seq, nq: int, k: int):
        """replay `world` gathered entry-log blocks (device memory) on the GPU; returns (seq[nq,k], dist[nq,k], counts[nq])"""
        seq = np.zeros((nq, k), dtype=np.int64)
        dist = np.zeros((nq, k), dtype=np.float64)
        counts = np.zeros(nq, dtype=np.int32)
        fs = np.ascontiguousarray(first_seq, dtype=np.int64)
        self.eng.check(self.eng.lib.vsb_batch_merge(self.h, d_blocks, world, stride, _ptr(fs), nq, k, _ptr(seq), _ptr(dist), _ptr(counts)))
        return seq, dist, counts

    def lookup_rowids(self, seq: np.ndarray) -> np.ndarray:
        sq = np.ascontiguousarray(seq, dtype=np.int64)
        out = np.zeros(sq.shape, dtype=np.int64)
        self.eng.check(self.eng.lib.vsb_index_lookup_rowids(self.h, _ptr(sq), sq.size, _ptr(out)))
        return out

    # ---- exchange over NVLink peer memory (one process per GPU)
    def exchange_export(self, world: int, rank: int) -> bytes:
        h = (C.c_ubyte * 64)()
        self.eng.check(self.eng.lib.vsb_exchange_export(self.h, world, rank, C.cast(h, C.c_void_p)))
        return bytes(h)

    def exchange_attach(self, handles: bytes):
        buf = (C.c_ubyte * len(handles)).from_buffer_copy(handles)
        self.eng.check(self.eng.lib.vsb_exchange_attach(self.h, C.cast(buf, C.c_void_p)))

    def exchange_submit(self, metric: int, queries, stride: int, nq: int, k: int, on_device: bool, first_slot: int):
        ptr = int(queries) if on_device else _ptr(queries)
        self.eng.check(self.eng.lib.vsb_exchange_submit(self.h, metric, ptr, stride, nq, int(on_device), k, first_slot))

    def exchange_collect(self, first_slot: int, nq: int, first_seq: np.ndarray, k: int):
        ids = np.zeros((nq, max(k, 1)), dtype=np.int64)
        dist = np.zeros((nq, max(k, 1)), dtype=np.float64)
        counts = np.zeros(nq, dtype=np.int32)
        fs = np.ascontiguousarray(first_seq, dtype=np.int64)
        self.eng.check(self.eng.lib.vsb_exchange_collect(self.h, first_slot, nq, _ptr(fs), k, _ptr(ids), _ptr(dist), _ptr(counts)))
        return [(ids[j, :counts[j]], dist[j, :counts[j]]) for j in range(nq)]

    def exchange_batch_submit(self, metric: int, queries: np.ndarray, k: int, first_seq: np.ndarray) -> int:
        q2 = np.ascontiguousarray(queries).reshape(-1, queries.shape[-1])
        fs = np.ascontiguousarray(first_seq, dtype=np.int64)
        t = self.eng.lib.vsb_exchange_batch_submit(self.h, metric, _ptr(q2), q2.shape[0], k, _ptr(fs))
        if t < 0:
            self.eng.check(t)
        return t

    def exchange_batch_collect(self, ticket: int, nq: int, k: int):
        seq = np.zeros((nq, k), dtype=np.int64)
        dist = np.zeros((nq, k), dtype=np.float64)
        counts = np.zeros(nq, dtype=np.int32)
        self.eng.check(self.eng.lib.vsb_exchange_batch_collect(self.h, ticket, nq, k, _ptr(seq), _ptr(dist), _ptr(counts)))
        return seq, dist, counts

    def collect(self, slot: int, k: int):
        ids = np.zeros(max(k, 1), dtype=np.int64)
        dist = np.zeros(max(k, 1), dtype=np.float64)
        cnt = C.c_int(0)
        self.eng.check(self.eng.lib.vsb_collect(self.h, slot, k, _ptr(ids), _ptr(dist), C.byref(cnt)))
        return ids[:cnt.value].copy(), dist[:cnt.value].copy()

    def stat(self, name: str) -> int:
        return int(self.eng.lib.vsb_index_stat(self.h, name.encode()))

    def debug_read(self, name: str, dtype, count: int) -> np.ndarray:
        out = np.zeros(count, dtype=dtype)
        got = self.eng.lib.vsb_debug_read(self.h, name.encode(), _ptr(out), out.nbytes)
        if got < 0:
            self.eng.check(got)
        return out[: got // out.itemsize]

    def debug_write(self, name: str, data: np.ndarray):
        """plant an internal buffer (vsb_debug_write); "bounds": int64 [stat("sms") + 1] tile boundaries; "grouped_dist":
        float32 [rows] (every query) or [nq * rows] (query j: row j), the distances of the next grouped call instead of its scans"""
        a = np.ascontiguousarray(data, dtype=np.float32 if name == "grouped_dist" else np.int64)
        self.eng.check(self.eng.lib.vsb_debug_write(self.h, name.encode(), _ptr(a), a.nbytes))

    def debug_grouped(self) -> dict:
        """this shard's state after the last grouped call, for its last query (vsb_debug_read "grouped"): numpy arrays "rows",
        "koff", "pstart", "pkey", "kpiece" (uint32 layout), "dist", "pd", "lists" [npieces, k], "bound", "kmin" (float32),
        "pairs" (uint32 [n, 2] of (distance bits, position)), "ksel" (uint8 per key, None when every key was compacted), and "k" """
        head = self.debug_read("grouped", np.int64, 7)
        P, N, G, k, D, S, Cn = (int(v) for v in head)
        sizes = [("rows", "<u4", P), ("koff", "<u4", G + 1), ("pstart", "<u4", N + 1), ("pkey", "<u4", N), ("kpiece", "<u4", G + 1),
                 ("dist", "<f4", D), ("pd", "<f4", P), ("lists", "<f4", N * k), ("bound", "<f4", N), ("kmin", "<f4", G),
                 ("pairs", "<u4", 2 * Cn), ("ksel", "u1", G if S else 0)]
        raw = self.debug_read("grouped", np.uint8, 56 + sum(np.dtype(t).itemsize * c for _, t, c in sizes))
        out, at = {"k": k}, 56
        for name, t, c in sizes:
            nb = np.dtype(t).itemsize * c
            out[name] = raw[at:at + nb].view(t).copy()
            at += nb
        out["lists"] = out["lists"].reshape(N, k)
        out["pairs"] = out["pairs"].reshape(Cn, 2)
        if not S:
            out["ksel"] = None
        return out

    def debug_grouped_pass(self) -> dict:
        """this shard's state after the last grouped call, for every query of its last pass (vsb_debug_read "grouped_pass"): the
        layout arrays of debug_grouped, "k", and "queries", one dict per query of the pass with "dist", "pd", "lists", "bound",
        "kmin", "pairs" and "ksel" as debug_grouped returns them"""
        head = self.debug_read("grouped_pass", np.int64, 6)
        P, N, G, k, D, W = (int(v) for v in head)
        lay = [("rows", "<u4", P), ("koff", "<u4", G + 1), ("pstart", "<u4", N + 1), ("pkey", "<u4", N), ("kpiece", "<u4", G + 1)]
        fixed = 48 + sum(np.dtype(t).itemsize * c for _, t, c in lay)
        per = 16 + 4 * (D + P + N * k + N + G)
        raw = self.debug_read("grouped_pass", np.uint8, fixed + W * (per + 8 * P + G))   # at most every position survives
        out, at = {"k": k}, 48
        for name, t, c in lay:
            nb = np.dtype(t).itemsize * c
            out[name] = raw[at:at + nb].view(t).copy()
            at += nb
        out["queries"] = []
        for _ in range(W):
            S, Cn = (int(v) for v in raw[at:at + 16].view("<i8"))
            at += 16
            q = {}
            for name, t, c in (("dist", "<f4", D), ("pd", "<f4", P), ("lists", "<f4", N * k), ("bound", "<f4", N), ("kmin", "<f4", G),
                               ("pairs", "<u4", 2 * Cn), ("ksel", "u1", G if S else 0)):
                nb = np.dtype(t).itemsize * c
                q[name] = raw[at:at + nb].view(t).copy()
                at += nb
            q["lists"] = q["lists"].reshape(N, k)
            q["pairs"] = q["pairs"].reshape(Cn, 2)
            if not S:
                q["ksel"] = None
            out["queries"].append(q)
        return out

    def debug_survivors(self, slot: int, cap: int = 1 << 16):
        """(pairs uint32 [n, 2] of (distance bits, local row) in scan order, head flags) of a result slot: what collect(slot)
        replays (vsb_debug_survivors); no pairs when the flags report an overflow"""
        pairs = np.zeros((cap, 2), dtype=np.uint32)
        flags = _i(0)
        n = self.eng.lib.vsb_debug_survivors(self.h, slot, _ptr(pairs), cap, C.byref(flags))
        if n < 0:
            self.eng.check(n)
        if n > cap:
            raise VsbError(f"slot {slot} holds {n} survivors, more than cap = {cap}")
        return pairs[:n].copy(), flags.value

    def debug_tc_level(self, metric: int, queries: np.ndarray, U: np.ndarray, r0: int, r1: int, N: int = 0, scores: bool = False,
                       cap: int = 1 << 22, allow=None, allow_base: int = 0, sets=None, set_of_query=None, level0: bool = False):
        """one tensor-core level of the batch path over rows [r0, r1) with the per-query bounds U (vsb_debug_tc_level; metric
        L1: one level of the CUDA-core L1 batch kernel, any column type).
        scores=False: {"log": (row, query) uint32 pairs, "count": hits counted (> len(log) when truncated at cap),
        "qc": uint32 bits [nq], "norms": row sums of squares [r1 - r0] (zeros for L1)}; scores=True: the same with "scores"
        [r1 - r0, nq] (int32 for int8 / uint8, float32 for f32 / f16 / bf16) instead of the log.
        allow / sets / level0 (vsb_debug_tc_level_filtered, the log only): the level as a filtered or sets batch runs it, row r
        being bit allow_base + r.  allow: a boolean mask or uint32 bitmap; sets: boolean masks of one length or a uint32 array
        [nsets, words], set_of_query[q] query q's set (their union is the row filter); level0: level 0 over rows [0, r1) (r0 = 0,
        U unused) instead of a scorer level"""
        q2 = np.ascontiguousarray(queries).reshape(-1, queries.shape[-1])
        nq = q2.shape[0]
        u = np.ascontiguousarray(U, dtype=np.float32)
        assert u.shape == (nq,)
        if allow is not None or sets is not None or level0:
            assert not scores, "a filtered level returns its log"
            return self._debug_tc_level_filtered(metric, q2, u, r0, r1, N, cap, allow, allow_base, sets, set_of_query, level0)
        integer = self.vtype in (U8, I8)
        qc = np.zeros(nq, dtype=np.uint32)
        norms = np.zeros(r1 - r0, dtype=np.int32 if integer else np.float32)
        count = _i64()
        if scores:
            out = np.zeros((r1 - r0, nq), dtype=np.int32 if integer else np.float32)
            cap = out.size
        else:
            out = np.zeros((cap, 2), dtype=np.uint32)
        self.eng.check(self.eng.lib.vsb_debug_tc_level(self.h, metric, _ptr(q2), nq, _ptr(u), r0, r1, N, int(scores), _ptr(out), cap,
                                                       _ptr(qc), _ptr(norms), C.byref(count)))
        res = {"count": int(count.value), "qc": qc, "norms": norms}
        if scores:
            res["scores"] = out
        else:
            res["log"] = out[: min(int(count.value), cap)].copy()
        return res

    def _debug_tc_level_filtered(self, metric, q2, u, r0, r1, N, cap, allow, allow_base, sets, set_of_query, level0):
        nq = q2.shape[0]
        bits, nbits, flat, nsets, soq = None, 0, None, 0, None
        if allow is not None:
            a = np.asarray(allow)
            bits = row_bitmap(a) if a.dtype == bool else np.ascontiguousarray(a, dtype=np.uint32)
            nbits = len(a) if a.dtype == bool else 32 * bits.size
        if sets is not None:
            if isinstance(sets, np.ndarray) and sets.dtype == np.uint32 and sets.ndim == 2:
                flat, nbits = np.ascontiguousarray(sets), 32 * sets.shape[1]
            else:
                nbits = len(sets[0])
                flat = np.stack([row_bitmap(np.asarray(m, bool)) for m in sets])
            nsets = flat.shape[0]
            soq = np.ascontiguousarray(set_of_query, dtype=np.int32)
            assert soq.shape == (nq,)
        if allow is None and sets is None:
            nbits = allow_base + r1
        integer = self.vtype in (U8, I8)
        qc = np.zeros(nq, dtype=np.uint32)
        norms = np.zeros(r1 - r0, dtype=np.int32 if integer else np.float32)
        count = _i64()
        out = np.zeros((cap, 2), dtype=np.uint32)
        self.eng.check(self.eng.lib.vsb_debug_tc_level_filtered(self.h, metric, _ptr(q2), nq, _ptr(u), r0, r1, N, int(level0), _ptr(bits),
                                                                allow_base, nbits, _ptr(flat), nsets, _ptr(soq), _ptr(out), cap, _ptr(qc),
                                                                _ptr(norms), C.byref(count)))
        return {"count": int(count.value), "qc": qc, "norms": norms, "log": out[: min(int(count.value), cap)].copy()}

    def debug_sets_plan(self) -> dict:
        """the level plan of this shard's most recent sets call (vsb_debug_read "sets_plan"): "tb", "vt", "nlev" and "ends" (one
        int64 array of level end tiles per view), "m0", "growth", "over", "pairs0", "nsets", "words"; with option sets_debug on
        during the call also "sets" (uint32 [nsets, words], this shard's cut of each set the queries name, in order of first use),
        "union" [words] and "prefix" (uint32 [nsets, T + 1]), else None"""
        head = self.debug_read("sets_plan", np.int64, 10)
        T, V, m0, growth, over, pairs0, S, W, L, D = (int(v) for v in head)
        n64 = 10 + (T + 1) + (V + 1) + V + L
        raw = self.debug_read("sets_plan", np.uint8, 8 * n64 + (4 * (S * W + W + S * (T + 1)) if D else 0))
        i64 = raw[: 8 * n64].view("<i8")
        at = 10
        tb, vt, nlev = i64[at:at + T + 1].copy(), i64[at + T + 1:at + T + V + 2].copy(), i64[at + T + V + 2:at + T + 2 * V + 2].copy()
        flat = i64[at + T + 2 * V + 2:].copy()
        cut = np.concatenate([[0], np.cumsum(nlev)]).astype(np.int64)
        out = {"tb": tb, "vt": vt, "nlev": nlev, "ends": [flat[cut[v]:cut[v + 1]] for v in range(V)], "m0": m0, "growth": growth,
               "over": bool(over), "pairs0": pairs0, "nsets": S, "words": W, "sets": None, "union": None, "prefix": None}
        if D:
            u4 = raw[8 * n64:].view("<u4")
            out["sets"] = u4[:S * W].reshape(S, W).copy()
            out["union"] = u4[S * W:S * W + W].copy()
            out["prefix"] = u4[S * W + W:].reshape(S, T + 1).copy()
        return out

    def debug_refine(self, metric: int, queries: np.ndarray, pairs: np.ndarray, U: np.ndarray, cand_cap: int | None = None):
        """one launch of the batch path's exact refinement over (row, query) pairs [npairs, 2] with the bounds U
        (vsb_debug_refine).  Returns {"bucket": uint32 [nq, BUCKET_CAP, 2] (row, distance bits; unused entries all ones),
        "bcount": uint32 [nq] entries appended, "stats": uint32 [3]}"""
        q2 = np.ascontiguousarray(queries).reshape(-1, queries.shape[-1])
        nq = q2.shape[0]
        p = np.ascontiguousarray(pairs, dtype=np.uint32).reshape(-1, 2)
        u = np.ascontiguousarray(U, dtype=np.float32)
        assert u.shape == (nq,)
        bucket = np.zeros((nq, BUCKET_CAP, 2), dtype=np.uint32)
        bcount = np.zeros(nq, dtype=np.uint32)
        stats = np.zeros(3, dtype=np.uint32)
        cap = p.shape[0] if cand_cap is None else cand_cap
        self.eng.check(self.eng.lib.vsb_debug_refine(self.h, metric, _ptr(q2), nq, _ptr(p), p.shape[0], _ptr(u), cap, _ptr(bucket),
                                                     _ptr(bcount), _ptr(stats)))
        return {"bucket": bucket, "bcount": bcount, "stats": stats}

    def debug_replay(self, metric: int, queries: np.ndarray, k: int, bucket: np.ndarray, bcount: np.ndarray, level0: bool = True,
                     slot_d=None, slot_row=None, slot_mi=None, acc_cap: int = 0, acc_log=None, acc_count=None, final_sort: bool = False):
        """one launch of the batch path's slot replay (vsb_debug_replay) on planted buckets [nq, BUCKET_CAP, 2] (row, distance
        bits) with bcount [nq] entries each.  level0=False continues from slot_d / slot_row [nq, kcap] and slot_mi [nq];
        acc_cap > 0 carries the entry log (acc_log [nq, acc_cap, 2] (distance bits, row), acc_count [nq]; zeros by default).
        Returns {"slot_d", "slot_row" [nq, kcap], "slot_mi", "U", "qc" (uint32 bits), "bcount", "stats" [3], and with a log
        "acc_log", "acc_count"}"""
        q2 = np.ascontiguousarray(queries).reshape(-1, queries.shape[-1])
        nq = q2.shape[0]
        kcap = (k + 31) & ~31
        b = np.ascontiguousarray(bucket, dtype=np.uint32)
        assert b.shape == (nq, BUCKET_CAP, 2)
        bc = np.ascontiguousarray(bcount, dtype=np.uint32)
        sd = np.zeros((nq, kcap), np.float32) if slot_d is None else np.array(slot_d, dtype=np.float32, order="C")
        sr = np.zeros((nq, kcap), np.uint32) if slot_row is None else np.array(slot_row, dtype=np.uint32, order="C")
        mi = np.zeros(nq, np.int32) if slot_mi is None else np.array(slot_mi, dtype=np.int32)
        assert sd.shape == (nq, kcap) and sr.shape == (nq, kcap) and mi.shape == (nq,)
        log = cnt = None
        if acc_cap > 0:
            log = np.zeros((nq, acc_cap, 2), np.uint32) if acc_log is None else np.array(acc_log, dtype=np.uint32, order="C")
            cnt = np.zeros(nq, np.int32) if acc_count is None else np.array(acc_count, dtype=np.int32)
        U = np.zeros(nq, np.float32)
        qc = np.zeros(nq, np.uint32)
        bout = np.zeros(nq, np.uint32)
        stats = np.zeros(3, np.uint32)
        self.eng.check(self.eng.lib.vsb_debug_replay(self.h, metric, _ptr(q2), nq, k, int(level0), _ptr(b), _ptr(bc), _ptr(sd), _ptr(sr),
                                                     _ptr(mi), acc_cap, _ptr(log), _ptr(cnt), int(final_sort), _ptr(U), _ptr(qc),
                                                     _ptr(bout), _ptr(stats)))
        res = {"slot_d": sd, "slot_row": sr, "slot_mi": mi, "U": U, "qc": qc, "bcount": bout, "stats": stats}
        if log is not None:
            res["acc_log"], res["acc_count"] = log, cnt
        return res

    def profile_read(self):
        a, b = C.c_double(), C.c_double()
        na, nb = C.c_int(), C.c_int()
        self.eng.check(self.eng.lib.vsb_profile_read(self.h, C.byref(a), C.byref(na), C.byref(b), C.byref(nb)))
        return {"scan_ms": a.value, "scan_launches": na.value, "filter_ms": b.value, "filter_launches": nb.value}

    def collect_last(self, k: int):
        ids = np.zeros(max(k, 1), dtype=np.int64)
        dist = np.zeros(max(k, 1), dtype=np.float64)
        cnt = C.c_int(0)
        self.eng.check(self.eng.lib.vsb_collect_last(self.h, k, _ptr(ids), _ptr(dist), C.byref(cnt)))
        return ids[:cnt.value].copy(), dist[:cnt.value].copy()


class Group(_Column):
    """One column row-sharded over several GPUs inside ONE process (what the SQLite extension uses with gpus=N)."""

    _prefix = "vsb_group_"
    _rowid_bitmap = "vsb_group_rowid_bitmap"

    def __init__(self, vtype: int, dim: int, capacity: int, ngpus: int, first_device: int = 0, engine: Engine | None = None):
        self.eng = engine or load_engine()
        self.vtype, self.dim = vtype, dim
        h = _vp()
        self.eng.check(self.eng.lib.vsb_group_create(C.byref(h), first_device, ngpus, vtype, dim, capacity))
        self.h = h

    def close(self):
        if getattr(self, "h", None):
            self._close_groupings()
            self.eng.lib.vsb_group_free(self.h)
            self.h = None

    __del__ = close

    @property
    def gpus(self) -> int:
        return int(self.eng.lib.vsb_group_gpus(self.h))

    @property
    def rows(self) -> int:
        return int(self.eng.lib.vsb_group_rows(self.h))

    def append_dense(self, vectors: np.ndarray, rowids: np.ndarray | None = None):
        rid = None if rowids is None else np.ascontiguousarray(rowids, dtype=np.int64)
        self.eng.check(self.eng.lib.vsb_group_append_dense(self.h, _ptr(np.ascontiguousarray(vectors)), _ptr(rid), vectors.shape[0]))

    def append_quant_chunk(self, chunk: np.ndarray, nrows: int):
        self.eng.check(self.eng.lib.vsb_group_append_quant_chunk(self.h, _ptr(chunk), nrows))

    def finalize(self):
        self.eng.check(self.eng.lib.vsb_group_finalize(self.h))


class Grouping:
    """A layout of keys on every shard of a column, kept across grouped calls (vsb_grouping_create): Index.grouping or
    Group.grouping make one.  It holds its column; a call after the column gained rows or was closed raises VsbError (EINVAL)."""

    def __init__(self, column: _Column, key_lists):
        self.eng, self.column = column.eng, column
        flat, offsets = _key_csr(key_lists)
        h = _vp()
        self.eng.check(column._fn("grouping_create")(column.h, _ptr(flat), _ptr(offsets), len(offsets) - 1, C.byref(h)))
        self.h = h
        if not hasattr(column, "_groupings"):
            column._groupings = weakref.WeakSet()
        column._groupings.add(self)

    def scan_topk(self, metric: int, queries: np.ndarray, k: int, limit: int = 0):
        """the column's scan_topk_grouped(metric, queries, k, key_lists, limit) on the kept layout (vsb_scan_topk_grouping)"""
        return _grouped_call(self.eng, lambda qp, nq, res: self.eng.lib.vsb_scan_topk_grouping(self.h, metric, qp, nq, k, limit, res),
                             queries)

    def close(self):
        if getattr(self, "h", None):
            self.eng.lib.vsb_grouping_free(self.h)
            self.h = None

    __del__ = close

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()


class Quantizer:
    """GPU side of vector_quantize (vsb_quantizer_*): min / max pass and chunk encoding, byte-identical to the reference."""

    def __init__(self, src_vtype: int, dim: int, retain_rows: int = 0, device: int = 0, engine: Engine | None = None):
        self.eng = engine or load_engine()
        self.vtype, self.dim = src_vtype, dim
        h = _vp()
        self.eng.check(self.eng.lib.vsb_quantizer_create(C.byref(h), device, src_vtype, dim, retain_rows))
        self.h = h

    def close(self):
        if getattr(self, "h", None):
            self.eng.lib.vsb_quantizer_free(self.h)
            self.h = None

    __del__ = close

    def minmax(self, rows: np.ndarray):
        self.eng.check(self.eng.lib.vsb_quantizer_minmax(self.h, _ptr(np.ascontiguousarray(rows)), rows.shape[0]))

    def minmax_result(self):
        lo, hi, neg = C.c_float(), C.c_float(), C.c_int()
        self.eng.check(self.eng.lib.vsb_quantizer_minmax_result(self.h, C.byref(lo), C.byref(hi), C.byref(neg)))
        return lo.value, hi.value, bool(neg.value)

    @property
    def retained_rows(self) -> int:
        return int(self.eng.lib.vsb_quantizer_retained_rows(self.h))

    def encode(self, rows, rowids: np.ndarray, offset: float, scale: float, qtype: int, retained_first_row: int = 0) -> np.ndarray:
        """rows: host array, or None to encode rows [retained_first_row, +len(rowids)) kept in HBM by minmax"""
        rid = np.ascontiguousarray(rowids, dtype=np.int64)
        n = rid.shape[0]
        out = np.zeros(n * (8 + self.dim), dtype=np.uint8)
        ptr = None if rows is None else _ptr(np.ascontiguousarray(rows))
        self.eng.check(self.eng.lib.vsb_quantizer_encode(self.h, ptr, retained_first_row, _ptr(rid), n, C.c_float(offset), C.c_float(scale), qtype, _ptr(out)))
        return out
