/*
 * vsb200.h — C ABI of the H100 scan engine (libvsb200.so / vector.so).
 *
 * This is the drop-in boundary for sqlite-vector's brute-force scan path.  Every entry point
 * names the reference interface it replaces (file:line relative to sqliteai/sqlite-vector 0.9.23).
 * Plain pointers and sizes only; no C++ or torch types.  All functions return VSB_OK (0) or a
 * negative VSB_E* code; vsb_last_error() gives the message for the calling thread.
 *
 * There is NO CPU fallback: without a CUDA device every scan entry point fails with VSB_ENODEV.
 */
#ifndef VSB200_H
#define VSB200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define VSB_API __attribute__((visibility("default")))
#else
#define VSB_API
#endif

/* element types and metrics: same numbering as the reference enums vector_type / vector_distance /
 * vector_qtype (src/distance-cpu.h:36-58) so values can be passed through unchanged. */
enum { VSB_F32 = 1, VSB_F16 = 2, VSB_BF16 = 3, VSB_U8 = 4, VSB_I8 = 5 };
enum { VSB_L2 = 1, VSB_SQUARED_L2 = 2, VSB_COSINE = 3, VSB_DOT = 4, VSB_L1 = 5 };
enum { VSB_QUANT_AUTO = 0, VSB_QUANT_U8 = 1, VSB_QUANT_S8 = 2 };

enum {
    VSB_OK = 0,
    VSB_EINVAL = -1,  /* bad argument */
    VSB_ENODEV = -2,  /* no CUDA device / CUDA runtime failure at start-up */
    VSB_ENOMEM = -3,  /* host or device allocation failed */
    VSB_ECUDA = -4,   /* a CUDA call or kernel failed */
    VSB_ERANGE = -5   /* capacity exceeded */
};

typedef struct vsb_index vsb_index; /* one resident shard of one column on one GPU */

/* A row that may enter the reference's k slots: distance (already clamped like
 * nearly_zero_float32, src/sqlite-vector.c:994-996), its rowid and its position in scan order. */
typedef struct vsb_candidate {
    int64_t rowid;
    int64_t seq;   /* global scan-order index = first_seq of the shard + local row */
    float dist;
    int32_t reserved;
} vsb_candidate;

/* ---- process-wide ------------------------------------------------------------------------- */
VSB_API int vsb_device_count(void);
VSB_API const char *vsb_last_error(void);
/* replaces distance_backend_name (src/distance-cpu.c:20, reported by vector_backend(), :2549) */
VSB_API const char *vsb_backend_name(void);

/* ---- residency: replaces table_context.preloaded / precounter (src/sqlite-vector.c:135-136)
 * and the staging loop of vector_quantize_preload (src/sqlite-vector.c:1338-1404) ------------- */
/* capacity_rows is an upper bound on rows appended later; first_seq is the global scan-order index
 * of this shard's first row (0 on a single GPU). */
VSB_API int vsb_index_create(vsb_index **out, int device, int vtype, int dim, int64_t capacity_rows, int64_t first_seq);
/* corpora larger than the device budget (the role of the reference's not-preloaded path, src/sqlite-vector.c:2186-2227, which
 * re-reads the chunks from the shadow table for every query): the column is kept in PINNED HOST memory and streamed through two
 * device windows of window_rows rows each — the copy of window w+1 (cudaMemcpyAsync on its own stream) overlaps the scan of
 * window w; every window is scanned like a shard and the survivors are replayed in scan order, so results are those of a
 * resident index.  vsb_scan_topk / vsb_scan_all / vsb_scan_candidates work.  A batch that the tensor-core path takes (see
 * vsb_scan_topk) runs its levels window by window, one pass of the column per batch, with the results of the resident batch path;
 * this needs windows of at least 128 rows (smaller windows: one pass per query), and vsb_batch_shard_scan works the same way.
 * fp DOT batches add one more pass, once per column version, for the largest row norm.  The asynchronous entry points
 * (vsb_scan_submit / vsb_collect) and the exchange need a resident index.  Counters: vsb_index_stat "stream_bytes" / "stream_us"
 * (a batch: device time from its first window copy to its last level). */
VSB_API int vsb_index_create_streamed(vsb_index **out, int device, int vtype, int dim, int64_t capacity_rows, int64_t first_seq,
                                      int64_t window_rows);
VSB_API int vsb_index_is_streamed(const vsb_index *ix);
/* rows x dim elements, row-major, HOST memory; rowids NULL => rowid = first_seq + row + 1.
 * Staged through pinned memory and copied with cudaMemcpyAsync. */
VSB_API int vsb_index_append_dense(vsb_index *ix, const void *vectors, const int64_t *rowids, int64_t nrows);
/* one shadow-table chunk blob: nrows x [int64 LE rowid][dim x 8-bit], the format written by
 * vector_rebuild_quantization (src/sqlite-vector.c:1295-1311) and read back at :1382-1394.
 * Only valid for VSB_U8 / VSB_I8 indexes. */
VSB_API int vsb_index_append_quant_chunk(vsb_index *ix, const void *chunk, int64_t nrows);
/* rows already in DEVICE memory of ix's GPU (dense, row pitch = dim*elem bytes); d_rowids may be NULL. */
VSB_API int vsb_index_append_device(vsb_index *ix, const void *d_vectors, const int64_t *d_rowids, int64_t nrows);
VSB_API int vsb_index_finalize(vsb_index *ix); /* waits for all staged copies */
VSB_API int64_t vsb_index_rows(const vsb_index *ix);
VSB_API int64_t vsb_index_device_bytes(const vsb_index *ix);
VSB_API void vsb_index_free(vsb_index *ix);

/* ---- the scan: replaces vFullScanRun (src/sqlite-vector.c:2071-2113) / vQuantRunMemory
 * (:2121-2157) followed by vFullScanSortSlots (:2051-2069) ------------------------------------
 * queries: nq x dim elements of the index's type in HOST memory (for a quantized column the caller
 * has already quantized the query, as vQuantRun does at :2162-2177).
 * For query b the results are out_rowids[b*k .. b*k+out_counts[b]) / out_dist[...] in the
 * reference's output order (distance ascending, reference tie order), distances widened to
 * double exactly like the cursor's distance[] array (:1804, :2011).
 * max_index (in/out, may be NULL, nq == 1 only): the cursor's slot index quirk (:1808-1813 never resets it).
 * nq > 1 has no counterpart in the reference (one vector per xFilter); each query then behaves like a fresh cursor.
 * For nq >= 16 on f16/bf16/int8/uint8 columns with L2/SQUARED_L2/COSINE/DOT the scores are computed on the tensor
 * cores (wgmma), and with L1 on any column type by a CUDA-core batch kernel over the same tiles; either way they are
 * refined exactly and results are the same as nq single calls.
 * k > 256 (any nq, one query at a time): the all-distances scan, then on the device the exact k-th distance of every prefix
 * [0, k 2^j) of the column and the rows below their segment's bound in scan order (DESIGN §3.11); the host replays only those.
 * Results are the same bits as a replay over every row ("large_k_queries", "large_k_cands", "large_k_regrows").
 * k > 256 with nq >= 16 where the batch path above runs: the batch levels find every query's candidates with per-query bounds,
 * one pass of the column per batch (DESIGN §3.12), and the host replays each query's; the same bits as nq single calls
 * ("large_k_batches", "large_k_batch_fallbacks", "large_k_query_fallbacks"). */
VSB_API int vsb_scan_topk(vsb_index *ix, int metric, const void *queries, int nq, int k, int64_t *out_rowids,
                          double *out_dist, int *out_counts, int *max_index);

/* ---- filtered top-k: the k nearest among a given set of rows (no counterpart in the reference) ------------------------------
 * allow: HOST bitmap over the index's scan-order rows, row i eligible when bit i & 31 of word i >> 5 is set; nbits must equal
 * vsb_index_rows(ix) (else VSB_EINVAL).  The result is exactly what vsb_scan_topk returns for a column holding only the eligible
 * rows, in this column's scan order: the same max_index carry, exchange sort and INF trim (fewer than k eligible rows give fewer
 * than k results, none give zero rows), bit-exact for int8/uint8.  With every row eligible it equals vsb_scan_topk bit for bit.
 * Otherwise the contract is vsb_scan_topk's: the same batch conditions and fallbacks.  The bitmap is copied to the device once per
 * call.  A filtered scan still reads the whole column. */
VSB_API int vsb_scan_topk_filtered(vsb_index *ix, int metric, const void *queries, int nq, int k, const uint32_t *allow, int64_t nbits,
                                   int64_t *out_rowids, double *out_dist, int *out_counts, int *max_index);
/* rowids -> eligibility bitmap of ix (out_bits: (vsb_index_rows + 31) / 32 words, overwritten).  Rowids not in the column are
 * ignored, duplicates are harmless.  Returns the number of eligible rows, or < 0.  Explicit rowids use a rowid -> row table built
 * on first use and rebuilt after an append. */
VSB_API int64_t vsb_index_rowid_bitmap(vsb_index *ix, const int64_t *rowids, int64_t n, uint32_t *out_bits);

/* ---- per-query eligible sets: each query's k nearest among its own set of rows, in one pass of the column (no counterpart in
 * the reference) -------------------------------------------------------------------------------------------------------------------
 * sets: nsets HOST bitmaps over the scan-order rows, each (nbits + 31) / 32 words, back to back, in the layout of
 * vsb_scan_topk_filtered; nbits == vsb_index_rows.  set_of_query[b] in [0, nsets) names query b's set (NULL: query b uses set b,
 * nsets == nq).  Query b's result is exactly what vsb_scan_topk_filtered returns for b under bitmap sets[set_of_query[b]]: the
 * same rowids, order and distances, exchange sort and INF trim (an empty set gives zero rows, a set of fewer than k rows fewer
 * than k rows), bit for bit for every element type.  max_index is carried for nq == 1 only; every query of a larger batch starts
 * from a fresh cursor.  A batch that vsb_scan_topk's batch path admits (nq >= 16, k <= 256) runs as ONE batch: the union of the
 * sets is the row filter, each scored pair is also tested against its query's set, and the levels are planned so that every set
 * keeps the bucket bound of the batch path (DESIGN §3.14).  A capacity overflow, a plan of more than 256 levels in a view, set
 * bitmaps and plan larger than 1/8 of free device memory (option "sets_mem_mb": that many MB), and every call outside those conditions answer set by set: one
 * vsb_scan_topk_filtered per distinct set over its queries in call order.  The bitmaps live on the device for the call only.
 * Counters: "sets_batches" (one-pass calls), "sets_fallbacks" (admitted calls answered set by set), "sets_levels" (levels of
 * the most recent one-pass call), "sets_plan_us" (time of its level plans).  SQL: vector_*_scan_batch_sets, vector_rowid_sets. */
VSB_API int vsb_scan_topk_sets(vsb_index *ix, int metric, const void *queries, int nq, int k, const uint32_t *sets, int nsets,
                               int64_t nbits, const int32_t *set_of_query, int64_t *out_rowids, double *out_dist, int *out_counts,
                               int *max_index);

/* ---- listed rows: the k nearest among a per-query list of rowids, reading only the listed rows (no counterpart in the
 * reference; the rerank step of vector_quantize_scan_rerank) -------------------------------------------------------------------
 * Query q's rowids are rowids[offsets[q], offsets[q + 1]) (offsets: nq + 1 non-decreasing values from 0).  For each query the
 * result is bit for bit what vsb_scan_topk_filtered returns for that one query with the bitmap of its rowids: the same rowids,
 * order and distances, for every element type, metric and k (k > 256 included), the same max_index carry (nq == 1 only), exchange
 * sort and INF trim.  Rowids not in the column are ignored, duplicates are harmless, an empty list gives zero rows and a list
 * shorter than k fewer than k rows.  A batch of nq queries equals nq single calls bit for bit, floating-point types included, and
 * each query starts from a fresh cursor.  Only the listed rows are read: one kernel computes the distance of every (query, row)
 * pair with the single-query scan's arithmetic (DESIGN §3.13); a streamed index reads those rows from its pinned host memory in
 * place, with no window copy.  Counters: "rows_queries", "rows_pairs", "rows_host_bytes". */
VSB_API int vsb_scan_topk_rows(vsb_index *ix, int metric, const void *queries, int nq, int k, const int64_t *rowids,
                               const int64_t *offsets, int64_t *out_rowids, double *out_dist, int *out_counts, int *max_index);

/* ---- grouped top-k: each key's k nearest rows for the best keys, from one scan of the column per query (no counterpart in the
 * reference, whose stream modules answer it with row_number() OVER (PARTITION BY key ORDER BY distance)) ---------------------------
 * Key g's rowids are rowids[offsets[g], offsets[g + 1]) (offsets: nkeys + 1 non-decreasing values from 0; rowids may be NULL when
 * there are none).  Rowids not in the column are ignored, a duplicate inside one key counts once, and keys may share rows.  For
 * query q and key g the rows are bit for bit what vsb_scan_topk_filtered returns for that one query (nq = 1, max_index NULL) under
 * the bitmap of g's rows: the same rowids, order and distances, exchange sort and INF trim, for every element type and metric.
 * Keys with at least one row are ranked by their first row's distance (ascending, -INF first), then that row's scan position,
 * then the key index; limit > 0 keeps the first limit keys, limit 0 every key with a row.  0 <= k <= 256 (k = 0: no keys; larger
 * k is VSB_EINVAL); nkeys >= 0; limit >= 0.  Queries are answered one after another, each from a fresh cursor.  Each shard lays
 * out its rows of every key once per call on the device (more than 2^32 - 1 (key, row) pairs on one shard: VSB_ERANGE); this is
 * the one-call case of a grouping (vsb_grouping_create, which keeps the layout across calls).  Then per query each shard scans
 * every distance, walks every key in pieces of 1024 rows on the device, and copies to the host only the candidates of the keys
 * whose smallest distance over all shards is at or below the limit-th smallest (DESIGN §3.15).  A streamed index keeps the
 * distances of all its windows on the device (4 bytes per row, in vsb_index_device_bytes).  Counters: "grouped_queries",
 * "grouped_pairs" (the (key, row) pairs of the last layout), "grouped_cands" (candidates replayed), "grouped_keys_replayed" (on a
 * group's first shard), "grouped_regrows", "grouped_layout_us" (layouts built), "grouped_layout_reuses" (calls that ran on a
 * grouping's kept layout), "grouped_passes" and "grouped_pass_queries" (passes of the column and the queries they scored), and
 * the device times "grouped_scan_us" (scans) and "grouped_walk_us" (walk, bounds and compaction), timed per pass, and the host
 * time "grouped_replay_us" (on a group's first shard).  Several queries share each pass of the column (at most the scan's
 * pass_max width, and as many per-query areas of distances and device arrays as fit option "grouped_mem_mb", default 1/8 of the
 * free device memory); each query's answer is bit for bit what a call of that query alone returns.  *out receives
 * a result owned by the caller (vsb_grouped_free); vsb_grouped_get borrows query q's arrays from it: nkeys_out keys in rank
 * order, key i's rows at [row_offsets[i], row_offsets[i + 1]) of rowids and dist. */
typedef struct vsb_grouped vsb_grouped;
VSB_API int vsb_scan_topk_grouped(vsb_index *ix, int metric, const void *queries, int nq, int k, const int64_t *rowids,
                                  const int64_t *offsets, int nkeys, int limit, vsb_grouped **out);
VSB_API int vsb_grouped_get(const vsb_grouped *r, int q, int *nkeys_out, const int32_t **keys, const int64_t **row_offsets /* nkeys_out + 1 */,
                            const int64_t **rowids, const double **dist); /* borrowed until free */
VSB_API void vsb_grouped_free(vsb_grouped *r);

/* ---- groupings: a layout of keys kept across grouped calls ------------------------------------------------------------------
 * vsb_grouping_create lays out the keys (rowids, offsets, nkeys as for vsb_scan_topk_grouped, same checks and codes) on every
 * shard of the column once; vsb_scan_topk_grouping then answers (metric, queries, nq, k, limit) on that layout and returns bit for
 * bit what vsb_scan_topk_grouped returns with the same keys, arguments checked as there.  The layout does not depend on k; the
 * per-call arrays are sized by the call's k and grown, never shrunk.  A call on a grouping whose column gained rows since it was
 * made is VSB_EINVAL ("the column changed since the grouping was made").  Freeing the index or group detaches its groupings: every
 * later call on one is VSB_EINVAL, and vsb_grouping_free still frees it.  A grouping is an owned handle (vsb_debug_live_handles);
 * the planted "grouped_dist" and vsb_debug_read "grouped" apply to its calls as to vsb_scan_topk_grouped. */
typedef struct vsb_grouping vsb_grouping;
VSB_API int vsb_grouping_create(vsb_index *ix, const int64_t *rowids, const int64_t *offsets, int nkeys, vsb_grouping **out);
VSB_API int vsb_scan_topk_grouping(vsb_grouping *gr, int metric, const void *queries, int nq, int k, int limit, vsb_grouped **out);
VSB_API void vsb_grouping_free(vsb_grouping *gr);

/* ---- range search: every row closer than a radius (no counterpart in the reference, whose stream modules answer it as
 * SELECT id, distance FROM vector_*_scan_stream(...) WHERE distance < r ORDER BY distance) --------------------------------------
 * For query b (nq HOST queries, as for vsb_scan_topk) the result is every row with (double)d < radius[b], d being the distance
 * vsb_scan_topk reports for that row (after the nearly-zero clamp); strict, so a NaN radius or distance never qualifies and
 * radius +INF selects every row with a finite (or -INF) distance.  Rows come ordered by ascending distance, equal distances in
 * scan order; distances are widened to double.  allow (may be NULL: every row) is the row bitmap of vsb_scan_topk_filtered,
 * nbits = vsb_index_rows.  A single query is one range scan into a list of the index (65536 pairs at first); a larger result is
 * counted exactly, the list grows to that count and a second pass collects it (vsb_index_stat "range_passes"): nothing is ever
 * truncated.  nq >= 16 queries under the conditions of vsb_scan_topk's batch path (k aside) run as one batch on the tensor cores
 * (L1: the CUDA-core batch kernel) with the exact refine: int8 / uint8 results equal nq single calls bit for bit, fp results
 * agree within the refine's rounding.  A query that keeps more than 16384 rows in a batch is answered alone ("range_query_fallbacks"),
 * and a batch whose candidate log overflows is answered query by query ("range_batch_fallbacks"; "range_batches" counts the
 * others).  Streamed indexes scan window by window.  *out receives a result owned by the caller (vsb_range_free); vsb_range_get
 * borrows query q's arrays from it. */
typedef struct vsb_range vsb_range;
VSB_API int vsb_scan_range(vsb_index *ix, int metric, const void *queries, int nq, const double *radius /* [nq] */,
                           const uint32_t *allow /* NULL: every row */, int64_t nbits, vsb_range **out);
VSB_API int vsb_range_get(const vsb_range *r, int q, const int64_t **rowids, const double **dist, int64_t *count); /* borrowed until free */
VSB_API void vsb_range_free(vsb_range *r);

/* every row's distance for one query, in scan order (what the *_stream modules compute one row per
 * xNext, src/sqlite-vector.c:1901-1998).  out_dist has vsb_index_rows() floats; out_rowids may be NULL. */
VSB_API int vsb_scan_all(vsb_index *ix, int metric, const void *query, float *out_dist, int64_t *out_rowids);

/* ---- multi-GPU plumbing: each shard emits a small superset of the rows that can enter the
 * reference's slots; the caller concatenates shards in scan order (e.g. after an NCCL all-gather)
 * and finishes with vsb_replay_topk.  k <= 256: the scan's survivors, or every row when its candidate log
 * overflowed; k > 256: the rows below their prefix bound (vsb_scan_topk, DESIGN §3.11), about
 * k (1 + log2(n / k)) rows for rows in random order, every row for strictly falling distances. ------------ */
VSB_API int vsb_scan_candidates(vsb_index *ix, int metric, const void *queries, int nq, int k, vsb_candidate *out,
                                int cap_per_query, int *out_counts);
/* the reference's slot algorithm over candidates in scan order: init (src/sqlite-vector.c:1808-1813),
 * replace-the-max with first-argmax (:2022-2049, :2145-2152), exchange sort and INF trim (:2051-2069,
 * :1816-1817).  Pure host code; for k > 256 the first argmax is kept in a tournament tree, O(log k) per
 * replaced slot, with the same result.  Returns the number of valid rows. */
VSB_API int vsb_replay_topk(const vsb_candidate *cands, int n, int k, int *max_index, int64_t *out_rowids,
                            double *out_dist);

/* ---- device-resident variants used by bench.py (inputs already in HBM) --------------------- */
/* runs the scan kernels for ONE query that is already in device memory (pitch-padded, see
 * vsb_index_query_pitch) and leaves the candidates in the engine's output buffer; no host copies. */
VSB_API int vsb_scan_device_query(vsb_index *ix, int metric, const void *d_query, int k); /* returns the result slot or <0 */
/* general form: submits scan + filter for ONE query and returns immediately with the result slot (>= 0).  The query is
 * either in device memory (query_on_device != 0, pitch-padded; read when its pass runs) or in HOST memory (dim elements;
 * staged through the slot's pinned buffer with cudaMemcpyAsync at submission, the xFilter argument of the reference,
 * src/sqlite-vector.c:1774-1776).  fetch != 0 also copies the slot's result block to pinned host memory for vsb_collect;
 * pass 0 when the block is exchanged on the device (vsb_result_block + all-gather).  Up to vsb_index_stat("slots") queries
 * may be in flight: slot < 0 hands slots out round-robin, slot >= 0 names the slot (a launcher that gathers groups of
 * consecutive slots manages them itself); either way a slot must be collected/merged before it is used again.
 * Queries share passes of the column (DESIGN §3.2): while the caller has an uncollected query (fetch != 0) on this index, a
 * new submission is held, and the held queries run as ONE pass, which reads the column once for all of them, at the first
 * of: the pass is full (vsb_index_stat "plan_pass_max"), a held query is collected, a submission with another metric or k
 * (or for a held query's slot) arrives, any other call on the index (vsb_collect_last, vsb_result_block, vsb_scan_topk*,
 * range, batch, profile or debug calls, close).  A submission with nothing outstanding, or with fetch == 0, launches at
 * once.  So "submit i+1, collect i" pairs the queries; a caller who submits a second query and then does host work before
 * collecting the first leaves the second waiting until it does.  Sharing a pass never changes a result.
 * A submission is checked before it is held or launched: VSB_EINVAL, with no slot taken and nothing launched, for an
 * unknown metric, k outside 1..256, a null query, or a device query that is not 16-byte aligned. */
VSB_API int vsb_scan_submit(vsb_index *ix, int metric, const void *query, int query_on_device, int k, int fetch, int slot);
/* blocks until the engine stream is idle and converts the last device-side result into top-k. */
VSB_API int vsb_collect_last(vsb_index *ix, int k, int64_t *out_rowids, double *out_dist, int *out_count);
/* same for a given result slot: several launches may be in flight (slots rotate), so query i+1 can be scanning while
 * the host finishes query i */
VSB_API int vsb_collect(vsb_index *ix, int slot, int k, int64_t *out_rowids, double *out_dist, int *out_count);
/* device address and size of a slot's result block (header + block table + first candidates) so that a launcher
 * can all-gather the shards' blocks on the device (NCCL) without a host round trip.  The blocks of all slots are
 * contiguous (slot s at block(0) + s * bytes): one collective can move a group of consecutive slots. */
VSB_API int vsb_result_block(vsb_index *ix, int slot, void **d_block, int64_t *bytes);
/* host-side merge of `world` gathered result blocks (block r starts at blocks + r*block_stride) into the reference's
 * top-k; rows are numbered first_seq[r] + local and rowids are implicit (global row + 1).  Returns the row count. */
VSB_API int vsb_merge_result_blocks(const void *blocks, int world, int64_t block_stride, const int64_t *first_seq, int k,
                                    int64_t *out_rowids, double *out_dist);
/* the same for a GROUP of nq independent queries in one call (query j at queries + j * query_stride; slots first_slot ..
 * first_slot + nq - 1): what the sharded launcher uses so that its per-query host cost stays far below one shard scan.
 * The queries are launched at once, as passes of up to vsb_index_stat("plan_pass_max") queries (one read of the column per
 * pass, one filter launch per query); each query's result is what it gets alone.  Device queries (query_on_device != 0) are
 * read as 16-byte vectors over the pitch: `queries` must be 16-byte aligned and, for nq > 1, query_stride a multiple of 16
 * and at least vsb_index_query_pitch, each query zero-padded to the pitch; else VSB_EINVAL before anything is launched. */
VSB_API int vsb_scan_submit_group(vsb_index *ix, int metric, const void *queries, int64_t query_stride, int nq, int query_on_device,
                                  int k, int fetch, int first_slot);
/* vsb_merge_result_blocks for a gathered group: query j's block of shard r is at blocks + r * rank_stride + j * block_stride;
 * results of query j at out_rowids/out_dist + j * k, out_counts[j] rows */
VSB_API int vsb_merge_result_groups(const void *blocks, int world, int64_t rank_stride, int64_t block_stride, int nq,
                                    const int64_t *first_seq, int k, int64_t *out_rowids, double *out_dist, int *out_counts);

/* ---- batched queries on a row-sharded column (BASELINE config 4: one shard per GPU) ----------------------------
 * step 1, on every shard: the batch path of vsb_scan_topk (same conditions: nq >= 16; f16/bf16/int8/uint8, or L1 on any
 * type) over this shard, leaving in DEVICE memory one block with, per query, the rows that entered the shard-local
 * slots in scan order (distance bits, local row).  *d_block / *bytes describe it (the same size on every shard for the
 * same nq and k) so that a launcher can all-gather the blocks (NCCL).  Returns VSB_ERANGE when the batch path does not
 * apply or a capacity was exceeded: use the per-query path (vsb_scan_candidates / vsb_scan_submit) then. */
VSB_API int vsb_batch_shard_scan(vsb_index *ix, int metric, const void *queries, int nq, int k, void **d_block, int64_t *bytes);
/* step 2, on any shard's GPU: `world` gathered blocks in shard (= scan) order, block r at d_blocks + r * block_stride in
 * DEVICE memory of ix's GPU (complete before the call).  Replays them through the reference's slot algorithm
 * (src/sqlite-vector.c:2145-2152, 2022-2069) on the GPU: exactly the result of one scan over the concatenated shards.
 * out_seq[b*k + j] is the GLOBAL scan-order row index (first_seq[r] + local row) of result j of query b; map it to a
 * rowid with vsb_index_lookup_rowids on the owning shard (implicit rowids: seq + 1). */
VSB_API int vsb_batch_merge(vsb_index *ix, const void *d_blocks, int world, int64_t block_stride, const int64_t *first_seq, int nq,
                            int k, int64_t *out_seq, double *out_dist, int *out_counts);
/* out[i] = rowid of global row seq[i] when this shard owns it, else 0 (so shards can be summed) */
VSB_API int vsb_index_lookup_rowids(const vsb_index *ix, const int64_t *seq, int64_t n, int64_t *out);
/* ---- exchange over NVLink peer memory: one process per GPU (torchrun), no collective library on the data path -----------
 * The final all-gather of the shards' per-query result heads (SURVEY §8e; north_star "final allgather of per-shard top-k over
 * NVLink") is a store kernel: after a group's filters, push_heads_kernel stores each head into row `rank` of EVERY peer's
 * gather buffer (cudaIpc-mapped peer memory) and raises an arrival flag; the receiver waits on the flags on its own stream and
 * copies the gathered heads to pinned host memory once per group.
 * setup (once): every rank calls vsb_exchange_export (allocates its gather buffer, returns a 64-byte cudaIpc handle), the
 * launcher all-gathers the handles (any transport: they are 64 bytes), every rank calls vsb_exchange_attach with all of them.
 * per group of 1..8 independent queries (the same call sequence on every rank): vsb_exchange_submit launches scan + filter
 * (+ push) and the receive; vsb_exchange_collect waits for the group and replays the reference's slot algorithm
 * (src/sqlite-vector.c:2145-2152, 2022-2069) over the shards in scan order — every rank gets the same complete result.
 * Slots are first_slot .. first_slot + nq - 1 of vsb_index_stat("slots"); a rank may have at most slots/2 queries in flight. */
VSB_API int vsb_exchange_export(vsb_index *ix, int world, int rank, void *handle64);
VSB_API int vsb_exchange_attach(vsb_index *ix, const void *handles /* world x 64 bytes, in rank order */);
VSB_API int vsb_exchange_submit(vsb_index *ix, int metric, const void *queries, int64_t query_stride, int nq, int query_on_device,
                                int k, int first_slot);
VSB_API int vsb_exchange_collect(vsb_index *ix, int first_slot, int nq, const int64_t *first_seq /* [world] */, int k,
                                 int64_t *out_rowids, double *out_dist, int *out_counts);

/* batched queries over the same exchange (BASELINE config 4 between processes): every rank runs the batch levels (tensor cores;
 * L1: the CUDA-core batch kernel, any column type) with entry logs over its shard, pushes its log block into every peer's log area over NVLink (push_logs_kernel), waits for the peers'
 * flags on the device and replays all logs in shard order on its GPU — the result of one scan over the whole column on every
 * rank, no collective library, ONE host wait per batch.  submit returns a ticket (0 / 1: two batches may be in flight) or a
 * negative code (VSB_ERANGE: the batch path does not apply — use vsb_exchange_submit per query); collect returns VSB_ERANGE on
 * EVERY rank when any shard exceeded a capacity.  out_seq holds GLOBAL scan-order rows (vsb_index_lookup_rowids / + 1). */
VSB_API int vsb_exchange_batch_submit(vsb_index *ix, int metric, const void *queries, int nq, int k, const int64_t *first_seq);
VSB_API int vsb_exchange_batch_collect(vsb_index *ix, int ticket, int nq, int k, int64_t *out_seq, double *out_dist, int *out_counts);

/* ---- shard group: ONE column row-sharded over several GPUs inside one process (the SQLite extension, option gpus=N) --------
 * Replaces table_context.preloaded (src/sqlite-vector.c:135-136) by `ngpus` resident shards of contiguous row ranges in scan
 * order: shard s holds rows [capacity*s/ngpus, capacity*(s+1)/ngpus).  Rows are appended in scan order exactly like the
 * single-index calls; scans have the contract of vsb_scan_topk / vsb_scan_all.  Every shard's filter pushes its head to the
 * leader GPU over NVLink peer memory (cudaDeviceEnablePeerAccess); batched queries gather the shards' entry logs with
 * cudaMemcpyPeerAsync and merge on the leader.  Every query kind runs the same code for an index and a group, chosen by the
 * shard count: ngpus == 1 takes exactly the paths of a vsb_index. */
typedef struct vsb_group vsb_group;
VSB_API int vsb_group_create(vsb_group **out, int first_device, int ngpus, int vtype, int dim, int64_t capacity_rows);
VSB_API int vsb_group_append_dense(vsb_group *g, const void *vectors, const int64_t *rowids, int64_t nrows);
VSB_API int vsb_group_append_quant_chunk(vsb_group *g, const void *chunk, int64_t nrows);
VSB_API int vsb_group_finalize(vsb_group *g);
VSB_API int vsb_group_scan_topk(vsb_group *g, int metric, const void *queries, int nq, int k, int64_t *out_rowids, double *out_dist,
                                int *out_counts, int *max_index);
VSB_API int vsb_group_scan_all(vsb_group *g, int metric, const void *query, float *out_dist, int64_t *out_rowids);
/* vsb_scan_topk_filtered / vsb_index_rowid_bitmap over the group's global scan order (nbits = vsb_group_rows) */
VSB_API int vsb_group_scan_topk_filtered(vsb_group *g, int metric, const void *queries, int nq, int k, const uint32_t *allow, int64_t nbits,
                                         int64_t *out_rowids, double *out_dist, int *out_counts, int *max_index);
VSB_API int64_t vsb_group_rowid_bitmap(vsb_group *g, const int64_t *rowids, int64_t n, uint32_t *out_bits);
/* vsb_scan_topk_sets over the group's global scan order: every set is cut per shard, each shard runs the one-pass batch and the
 * shards' entry logs merge as in vsb_group_scan_topk (counters on shard 0) */
VSB_API int vsb_group_scan_topk_sets(vsb_group *g, int metric, const void *queries, int nq, int k, const uint32_t *sets, int nsets,
                                     int64_t nbits, const int32_t *set_of_query, int64_t *out_rowids, double *out_dist,
                                     int *out_counts, int *max_index);
/* vsb_scan_topk_rows over the group's global scan order: every shard computes the distances of its own listed rows */
VSB_API int vsb_group_scan_topk_rows(vsb_group *g, int metric, const void *queries, int nq, int k, const int64_t *rowids,
                                     const int64_t *offsets, int64_t *out_rowids, double *out_dist, int *out_counts, int *max_index);
/* vsb_scan_topk_grouped over the group's global scan order: every shard lays out and walks its own rows of every key; the limit's
 * bound is taken from each key's minimum over all shards, and each key replays the shards' candidates in shard order */
VSB_API int vsb_group_scan_topk_grouped(vsb_group *g, int metric, const void *queries, int nq, int k, const int64_t *rowids,
                                        const int64_t *offsets, int nkeys, int limit, vsb_grouped **out);
/* vsb_grouping_create over the group's shards: one layout per shard (vsb_scan_topk_grouping answers on all of them) */
VSB_API int vsb_group_grouping_create(vsb_group *g, const int64_t *rowids, const int64_t *offsets, int nkeys, vsb_grouping **out);
/* vsb_scan_range over the group's global scan order (nbits = vsb_group_rows): every shard scans its rows, the shards' lists are
 * merged by (distance, global scan row) */
VSB_API int vsb_group_scan_range(vsb_group *g, int metric, const void *queries, int nq, const double *radius, const uint32_t *allow,
                                 int64_t nbits, vsb_range **out);
VSB_API int vsb_group_gpus(const vsb_group *g);
VSB_API int64_t vsb_group_rows(const vsb_group *g);
VSB_API vsb_index *vsb_group_shard(vsb_group *g, int shard); /* borrowed; for statistics */
VSB_API void vsb_group_free(vsb_group *g);

/* ---- GPU side of vector_quantize: replaces the two arithmetic loops of vector_rebuild_quantization (src/sqlite-vector.c:1224-1256
 * min / max / "negative seen"; :1281-1320 quantize into chunks) with kernels; stepping through the table and writing the
 * shadow-table rows stay with the extension.  Output bytes are identical to quantize_* / q_round_* (:495-757) and to the chunk
 * layout [int64 LE rowid][dim x 8-bit] (:1295-1311).
 * pass 1: vsb_quantizer_minmax for every block of rows (dense, source element type), then vsb_quantizer_minmax_result.
 * pass 2: vsb_quantizer_encode per chunk.  With retain_rows > 0 pass 1 keeps the raw column in HBM when it fits (check
 * vsb_quantizer_retained_rows() == rows fed), and pass 2 can encode rows [retained_first_row, +nrows) from there (rows == NULL):
 * the table is then stepped once instead of twice. */
typedef struct vsb_quantizer vsb_quantizer;
VSB_API int vsb_quantizer_create(vsb_quantizer **out, int device, int src_vtype, int dim, int64_t retain_rows);
VSB_API int vsb_quantizer_minmax(vsb_quantizer *qz, const void *rows, int64_t nrows);
VSB_API int vsb_quantizer_minmax_result(vsb_quantizer *qz, float *lo, float *hi, int *negative);
VSB_API int64_t vsb_quantizer_retained_rows(const vsb_quantizer *qz); /* rows kept in HBM by pass 1, or -1 when nothing is retained */
VSB_API int vsb_quantizer_encode(vsb_quantizer *qz, const void *rows, int64_t retained_first_row, const int64_t *rowids, int64_t nrows,
                                 float offset, float scale, int qtype, void *out_chunk /* nrows * (8 + dim) bytes, host */);
VSB_API void vsb_quantizer_free(vsb_quantizer *qz);

VSB_API int vsb_index_query_pitch(const vsb_index *ix); /* bytes per query row on the device (multiple of 16) */
/* counters since creation; name in {"queries","survivors","last_survivors","fallbacks","filter_blocks","fetch_bytes","slots","batches","batch_cands","batch_kept","tc_us","tc_rows","batch_us","stream_bytes","stream_us",
 * "sms" (scan CTAs per launch), "range_pairs" (rows returned by range queries), "range_passes" (range queries that took a second
 * pass), "range_host_sorts" (range results too long for the GPU sort, ordered on the host), "range_batches",
 * "range_batch_fallbacks", "range_query_fallbacks" (see vsb_scan_range), "large_k_queries" (queries with k > 256),
 * "large_k_cands" (their candidates replayed on the host), "large_k_regrows" (large-k queries whose candidates outgrew the pair
 * list, which then grew to the exact count), "large_k_batches" (calls whose k > 256 queries took the batch levels),
 * "large_k_batch_fallbacks" (such calls answered query by query: a candidate log overflowed), "large_k_query_fallbacks" (queries
 * of such a batch answered alone: their bucket or a sort segment overflowed), "large_k_levels_us" (host clock around the batch
 * levels, sort and candidate copy, which end in a stream synchronise), "large_k_replay_us" (host clock around the threaded slot
 * replay of such batches; a group counts it on its first shard), "large_k_replay_threads" (host threads of the last replay),
 * "rows_queries" (queries answered by vsb_scan_topk_rows), "rows_pairs" (their listed (query, row) pairs, each row counted once
 * per query), "rows_host_bytes" (bytes a streamed index's listed-rows kernel read from pinned host memory: pitch bytes per pair),
 * "sets_batches", "sets_fallbacks", "sets_levels", "sets_plan_us" (see vsb_scan_topk_sets), "scan_passes" (top-k passes of
 * the single-query scan kernel), "pass_queries" (the queries they scored: pass_queries / scan_passes queries per read of the
 * column), "grouped_*" (see vsb_scan_topk_grouped)}, and the plan of the most recent single-query scan launch: "plan_log2p" (log2 of the lanes per
 * row), "plan_nsw" (ring stages per warp), "plan_direct" (1: no staging), "plan_pass_max" (the widest pass of the shape at the k
 * of the most recent top-k pass, k <= 32 before any); -1 if unknown (or, for plan_*, before any scan) */
VSB_API int64_t vsb_index_stat(const vsb_index *ix, const char *name);
VSB_API void *vsb_index_stream(vsb_index *ix);           /* cudaStream_t of the engine, for event timing */
/* kernel launch counter (all kernels launched by this library since load) */
VSB_API int64_t vsb_kernel_launches(void);
/* diagnostics: CUDA allocations, events, streams and IPC mappings the library holds right now, over every index, group and
 * quantizer of the process; freeing an object returns the count to what it was before the object was created */
VSB_API int64_t vsb_debug_live_handles(void);
/* with option "time_kernels"=N (N >= 1) every N-th query's kernels are bracketed by CUDA events on their streams; this returns
 * (and resets) the summed device time and launch count of the scan kernel and of the filter kernel. */
VSB_API int vsb_profile_read(vsb_index *ix, double *scan_ms, int *scan_launches, double *filter_ms, int *filter_launches);
/* diagnostics: copies an internal device buffer of the most recent single-query scan to `out`; name in {"cta_time" (unsigned
 * cycles per scan CTA), "bounds" (int64 tile boundaries of the adaptive row partition), "topk_bounds" (the most recent k > 256
 * view, a resident column or one streamed window: int64 segment count S, int64 segment ends[32] (the first S used), float
 * bounds[32] (segment 0: +INF, segment s: the k-th distance of rows [0, ends[s - 1]))), "large_k_batch_bounds" (the most recent
 * large-k batch on this index: int64 piece count P, int64 query count Q, int64 [P][3] each piece's shard rows [first, end) and
 * level, float [P][Q] the bound each piece was refined against, +INF for level 0), "large_k_batch_cands" (the same batch's
 * candidates: int64 query count Q, int64 [Q] each query's count (-1: answered alone), then the queries' (uint32 distance bits,
 * uint32 shard row) pairs in scan order, query after query), "grouped" (this shard's state after the most recent
 * vsb_scan_topk_grouped, vsb_scan_topk_grouping or group call with k > 0, keys and queries, for its last query (DESIGN §3.15): int64 [7] {P positions,
 * N pieces, G keys, k, D distances (the shard's rows; 0 without positions), S (1: the limit selected keys), C survivor pairs},
 * then uint32 rows [P] (shard row of each position), koff [G + 1], pstart [N + 1], pkey [N], kpiece [G + 1], float dist [D] (the
 * query's distances), pd [P] (d where the walk logged, NaN otherwise), lists [N][k], bound [N], kmin [G], uint32 [C][2]
 * survivors (distance bits, position) in position order, and with S = 1 uint8 ksel [G] (1: the key was compacted))},
 * "grouped_pass" (the same shard's state for every query of the last pass of that call: int64 [6] {P, N, G, k, D, W queries},
 * the layout arrays rows, koff, pstart, pkey, kpiece as for "grouped", then per query int64 [2] {S, C} and dist [D], pd [P],
 * lists [N][k], bound [N], kmin [G], the C survivor pairs and with S = 1 ksel [G]), "sets_plan" (the level plan of the most
 * recent vsb_scan_topk_sets or group sets call on this shard that reached its plan, kept also when the call then answered set by
 * set (DESIGN §3.14): int64 [10] {T tiles, V views, m0, growth, over (1: a view needed more than 256 levels; no levels and
 * pairs0 0 then), pairs0, S sets (the distinct sets the queries name, in order of first use), W words per set, L levels in
 * all, D (1: the bitmaps follow)}, then int64 tb [T + 1] (tile bounds in shard rows), vt [V + 1] (view v: tiles [vt[v],
 * vt[v + 1])), nlev [V], ends [L] (each level's end tile, view after view), and with D = 1 (option "sets_debug" was 1 during
 * the call) uint32 sets [S][W] (the shard's cut of each set), union [W], prefix [S][T + 1] (each set's rows before each
 * tile)).  Returns the bytes copied or < 0. */
VSB_API int vsb_debug_read(vsb_index *ix, const char *name, void *out, int64_t bytes);
/* diagnostics: the counterpart of vsb_debug_read for name "bounds": plants a row partition (int64 tile boundaries, one per scan
 * CTA plus one, non-decreasing from 0 to the tile count of the k <= 32 plan; vsb_index_stat "sms" CTAs) into every scan
 * workspace of a resident index, so that the next single-query scans with k <= 32 use it instead of equal shares (the filter
 * then rewrites it as usual).  Rejects an index too small for the adaptive partition.  Name "grouped_dist": float32 [shard
 * rows], the distances every query of the next grouped call on this index (resident or streamed, or a shard of a group through
 * vsb_group_shard) uses instead of its scans, or float32 [nq][shard rows], row j for query j of a call of nq queries (a size
 * that is not whole rows is rejected here, a row count other than 1 or the call's nq by the call); everything after the scans runs as usual, and the call drops the plant when it
 * ends, however it ends.  Returns 0 or < 0. */
VSB_API int vsb_debug_write(vsb_index *ix, const char *name, const void *data, int64_t bytes);
/* diagnostics: the survivors of a result slot (fetch != 0) exactly as vsb_collect replays them: (uint32 distance bits, uint32
 * local row) pairs in block-table order, the head's then the tail's, which is scan order.  Waits for the slot's query; a
 * held query's pass is launched first, as vsb_collect does.  Writes the first `cap` pairs to out_pairs and the head's flags
 * to *flags (non-zero: the candidates overflowed, and no pair is returned).  Returns the survivor count or < 0. */
VSB_API int64_t vsb_debug_survivors(vsb_index *ix, int slot, uint32_t *out_pairs, int64_t cap, int *flags);
/* diagnostics: ONE tensor-core level of the batch path (tc_scan_kernel; metric VSB_L1: l1_batch_kernel, any column type) over
 * rows [r0, r1) of a finalized resident index (r0 a multiple of 128), for nq HOST queries whose exact distance bounds U[nq] are
 * given instead of found by earlier levels; the per-query constants are the batch path's own (conservative_qc).  N: queries
 * per tile, 32 / 64 / 128 (/ 256 for int8 and uint8, not L1), 0 = the batch path's choice for nq.
 *   mode 0 (candidate log, the production kernel): out receives up to out_cap (row, query) pairs of uint32, *out_count the
 *   number of hits the kernel counted (more than out_cap when the log was truncated).
 *   mode 1 (scores): out[(row - r0) * nq + q] = <row, query q> as the tensor cores computed it (L1: sum |row - query q|),
 *   int32 (int8 / uint8) or float (f32 / f16 / bf16); out_cap >= (r1 - r0) * nq.
 * out_qc (nq x 32 bits: float, or int for the integer kinds; L1: float) and out_norms (r1 - r0 row sums of squares, float /
 * int; left untouched for L1) may be NULL.  Synchronous. */
VSB_API int vsb_debug_tc_level(vsb_index *ix, int metric, const void *queries, int nq, const float *U, int64_t r0, int64_t r1,
                               int N, int mode, void *out, int64_t out_cap, void *out_qc, void *out_norms, int64_t *out_count);
/* diagnostics: vsb_debug_tc_level (mode 0) under a row filter or per-query sets, as a level of a filtered or sets batch runs:
 * row r of the index is bit allow_base + r of bitmaps of nbits bits (allow_base >= 0, allow_base + r1 <= nbits).  allow: one
 * row bitmap (the filter of vsb_scan_topk_filtered), or NULL; sets (with allow NULL): nsets bitmaps of words_of(nbits) words
 * back to back and set_of_query[nq], query q seeing only the rows of set set_of_query[q], their union the row filter (as
 * vsb_scan_topk_sets).  level0 != 0: level 0 instead of a scorer level, rows [0, r1) with r0 = 0: every (row, query) pair of
 * the eligible rows (all_pairs_kernel), or with sets each row's pairs with the queries whose set holds it (sets_pairs_kernel);
 * U is then unused, and a level of more than 16 Mi pairs returns VSB_ERANGE.  Synchronous. */
VSB_API int vsb_debug_tc_level_filtered(vsb_index *ix, int metric, const void *queries, int nq, const float *U, int64_t r0, int64_t r1,
                                        int N, int level0, const uint32_t *allow, int64_t allow_base, int64_t nbits, const uint32_t *sets,
                                        int nsets, const int32_t *set_of_query, void *out, int64_t out_cap, void *out_qc, void *out_norms,
                                        int64_t *out_count);
/* diagnostics: ONE launch of the batch path's exact refinement (refine_kernel, production grid) over npairs (row, query) uint32
 * pairs given by the caller (at most 16 Mi; only the first cand_cap are refined, like a truncated candidate log), with the
 * per-query bounds U[nq] (kept when distance < U).  out_bucket: nq x 2048 (row, distance bits) uint32 pairs, each query's
 * kept entries unordered, the rest all ones; out_bcount[nq]: entries appended (more than 2048 when the bucket overflowed);
 * out_stats[3]: candidates refined, 0, flags (1: pairs beyond cand_cap).  Synchronous. */
VSB_API int vsb_debug_refine(vsb_index *ix, int metric, const void *queries, int nq, const uint32_t *pairs, int64_t npairs, const float *U,
                             int64_t cand_cap, uint32_t *out_bucket, uint32_t *out_bcount, uint32_t *out_stats);
/* diagnostics: ONE launch of the batch path's slot replay (replay_kernel) for k in 1..256 on planted buckets (nq x 2048 (row,
 * distance bits); bcount[q] entries, more than 2048 flags an overflow).  Slots are kcap = round_up(k, 32) per query:
 * slot_d / slot_row / slot_mi are read when level0 == 0 (slot_mi in [0, k), else VSB_EINVAL) and always written back.
 * acc_log (nq x acc_cap (distance bits, row) uint32 pairs) and acc_count[nq] may both be NULL, or carry the entry log in
 * and out (acc_count is taken as 0 at level0).  final_sort != 0 then runs the final exchange sort on the slots.  Out: U and
 * qc bits per query (the next level's bound and tensor-core constant), bcount after the call, stats[3]: 0, entries
 * replayed, flags (2: a bucket overflowed).  Synchronous. */
VSB_API int vsb_debug_replay(vsb_index *ix, int metric, const void *queries, int nq, int k, int level0, const uint32_t *bucket,
                             const uint32_t *bcount, float *slot_d, uint32_t *slot_row, int *slot_mi, int acc_cap, uint32_t *acc_log,
                             int *acc_count, int final_sort, float *out_U, uint32_t *out_qc, uint32_t *out_bcount, uint32_t *out_stats);
/* tuning knobs for experiments: name in {"stage_bytes","direct","ring_bytes","time_kernels","no_batch","batch_debug","batch_m0","batch_growth","balance","scan_streams","xwait_ms","epi_chunk","f32_batch","sets_mem_mb","grouped_mem_mb","sets_debug"};
 * "sets_debug" = 1: sets calls also keep their bitmaps, union and prefix counts for vsb_debug_read "sets_plan" (default 0);
 * "f32_batch" = 1: f32 columns batch L2 / cosine / dot queries on the tensor cores in TF32 (default 0, or VSB_F32_BATCH=1 in the
 * environment when the library loads; per process).  Values are non-negative; returns the previous value, or a negative VSB_E* code (unknown name, negative value) */
VSB_API int vsb_set_option(const char *name, int value);

#ifdef __cplusplus
}
#endif
#endif /* VSB200_H */
