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
 * resident index.  vsb_scan_topk / vsb_scan_all / vsb_scan_candidates work; the asynchronous, exchange and tensor-core batch entry
 * points need a resident index.  Counters: vsb_index_stat "stream_bytes" / "stream_us". */
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
 * cores (wgmma) and refined exactly; results are the same as nq single calls. */
VSB_API int vsb_scan_topk(vsb_index *ix, int metric, const void *queries, int nq, int k, int64_t *out_rowids,
                          double *out_dist, int *out_counts, int *max_index);

/* every row's distance for one query, in scan order (what the *_stream modules compute one row per
 * xNext, src/sqlite-vector.c:1901-1998).  out_dist has vsb_index_rows() floats; out_rowids may be NULL. */
VSB_API int vsb_scan_all(vsb_index *ix, int metric, const void *query, float *out_dist, int64_t *out_rowids);

/* ---- multi-GPU plumbing: each shard emits a small superset of the rows that can enter the
 * reference's slots; the caller concatenates shards in scan order (e.g. after an NCCL all-gather)
 * and finishes with vsb_replay_topk. -------------------------------------------------------- */
VSB_API int vsb_scan_candidates(vsb_index *ix, int metric, const void *queries, int nq, int k, vsb_candidate *out,
                                int cap_per_query, int *out_counts);
/* the reference's slot algorithm over candidates in scan order: init (src/sqlite-vector.c:1808-1813),
 * replace-the-max with first-argmax (:2022-2049, :2145-2152), exchange sort and INF trim (:2051-2069,
 * :1816-1817).  Pure host code.  Returns the number of valid rows. */
VSB_API int vsb_replay_topk(const vsb_candidate *cands, int n, int k, int *max_index, int64_t *out_rowids,
                            double *out_dist);

/* ---- device-resident variants used by bench.py (inputs already in HBM) --------------------- */
/* runs the scan kernels for ONE query that is already in device memory (pitch-padded, see
 * vsb_index_query_pitch) and leaves the candidates in the engine's output buffer; no host copies. */
VSB_API int vsb_scan_device_query(vsb_index *ix, int metric, const void *d_query, int k); /* returns the result slot or <0 */
/* general form: launches scan + filter for ONE query and returns immediately with the result slot (>= 0).  The query is
 * either in device memory (query_on_device != 0, pitch-padded) or in HOST memory (dim elements; staged through the
 * slot's pinned buffer with cudaMemcpyAsync, the xFilter argument of the reference, src/sqlite-vector.c:1774-1776).
 * fetch != 0 also copies the slot's result block to pinned host memory for vsb_collect; pass 0 when the block is
 * exchanged on the device (vsb_result_block + all-gather).  Up to vsb_index_stat("slots") queries may be in flight:
 * slot < 0 hands slots out round-robin, slot >= 0 names the slot (a launcher that gathers groups of consecutive
 * slots manages them itself); either way a slot must be collected/merged before it is used again. */
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
 * With option "fuse_mb" > 0 (off by default) and one query reading fewer MB than that, up to 8 queries share ONE scan
 * launch: every CTA starts the next query as soon as its streams are done (no launch gap, the TMA ring runs across the
 * boundary); results are unchanged. */
VSB_API int vsb_scan_submit_group(vsb_index *ix, int metric, const void *queries, int64_t query_stride, int nq, int query_on_device,
                                  int k, int fetch, int first_slot);
/* vsb_merge_result_blocks for a gathered group: query j's block of shard r is at blocks + r * rank_stride + j * block_stride;
 * results of query j at out_rowids/out_dist + j * k, out_counts[j] rows */
VSB_API int vsb_merge_result_groups(const void *blocks, int world, int64_t rank_stride, int64_t block_stride, int nq,
                                    const int64_t *first_seq, int k, int64_t *out_rowids, double *out_dist, int *out_counts);

/* ---- batched queries on a row-sharded column (BASELINE config 4: one shard per GPU) ----------------------------
 * step 1, on every shard: the tensor-core batch path of vsb_scan_topk (same conditions: nq >= 16, f16/bf16/int8/uint8,
 * not L1) over this shard, leaving in DEVICE memory one block with, per query, the rows that entered the shard-local
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
 * NVLink") is a store kernel: after a group's filters, push_heads_kernel (the default; option push_mode = 0: the filter block that
 * completes a head) stores each head into row `rank` of EVERY peer's gather buffer (cudaIpc-mapped peer memory) and raises an
 * arrival flag; the receiver waits on the flags on its own stream and copies the gathered heads to pinned host memory once per
 * group.
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

/* batched queries over the same exchange (BASELINE config 4 between processes): every rank runs the tensor-core levels with entry
 * logs over its shard, pushes its log block into every peer's log area over NVLink (push_logs_kernel), waits for the peers'
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
 * cudaMemcpyPeerAsync and merge on the leader.  ngpus == 1 is exactly a vsb_index. */
typedef struct vsb_group vsb_group;
VSB_API int vsb_group_create(vsb_group **out, int first_device, int ngpus, int vtype, int dim, int64_t capacity_rows);
VSB_API int vsb_group_append_dense(vsb_group *g, const void *vectors, const int64_t *rowids, int64_t nrows);
VSB_API int vsb_group_append_quant_chunk(vsb_group *g, const void *chunk, int64_t nrows);
VSB_API int vsb_group_finalize(vsb_group *g);
VSB_API int vsb_group_scan_topk(vsb_group *g, int metric, const void *queries, int nq, int k, int64_t *out_rowids, double *out_dist,
                                int *out_counts, int *max_index);
VSB_API int vsb_group_scan_all(vsb_group *g, int metric, const void *query, float *out_dist, int64_t *out_rowids);
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
 * "sms" (scan CTAs per launch)}, and the plan of the most recent single-query scan launch: "plan_log2p" (log2 of the lanes per
 * row), "plan_nsw" (ring stages per warp), "plan_direct" (1: no staging); -1 if unknown (or, for plan_*, before any scan) */
VSB_API int64_t vsb_index_stat(const vsb_index *ix, const char *name);
VSB_API void *vsb_index_stream(vsb_index *ix);           /* cudaStream_t of the engine, for event timing */
/* kernel launch counter (all kernels launched by this library since load) */
VSB_API int64_t vsb_kernel_launches(void);
/* with option "time_kernels"=N (N >= 1) every N-th query's kernels are bracketed by CUDA events on their streams; this returns
 * (and resets) the summed device time and launch count of the scan kernel and of the filter kernel. */
VSB_API int vsb_profile_read(vsb_index *ix, double *scan_ms, int *scan_launches, double *filter_ms, int *filter_launches);
/* diagnostics: copies an internal device buffer of the most recent single-query scan to `out`; name in {"cta_time" (unsigned
 * cycles per scan CTA), "bounds" (int64 tile boundaries of the adaptive row partition)}.  Returns the bytes copied or < 0. */
VSB_API int vsb_debug_read(vsb_index *ix, const char *name, void *out, int64_t bytes);
/* diagnostics: the counterpart of vsb_debug_read for name "bounds": plants a row partition (int64 tile boundaries, one per scan
 * CTA plus one, non-decreasing from 0 to the tile count of the k <= 32 plan; vsb_index_stat "sms" CTAs) into every scan
 * workspace of a resident index, so that the next single-query scans with k <= 32 use it instead of equal shares (the filter
 * then rewrites it as usual).  Rejects an index too small for the adaptive partition.  Returns 0 or < 0. */
VSB_API int vsb_debug_write(vsb_index *ix, const char *name, const void *data, int64_t bytes);
/* diagnostics: ONE tensor-core level of the batch path (tc_scan_kernel) over rows [r0, r1) of a finalized resident index
 * (r0 a multiple of 128), for nq HOST queries whose exact distance bounds U[nq] are given instead of found by earlier levels;
 * the per-query constants are the batch path's own (conservative_qc).  N: queries per tile, 32 / 64 / 128 (/ 256 for
 * int8 and uint8), 0 = the batch path's choice for nq.
 *   mode 0 (candidate log, the production kernel): out receives up to out_cap (row, query) pairs of uint32, *out_count the
 *   number of hits the kernel counted (more than out_cap when the log was truncated).
 *   mode 1 (scores): out[(row - r0) * nq + q] = <row, query q> as the tensor cores computed it, int32 (int8 / uint8) or
 *   float (f16 / bf16); out_cap >= (r1 - r0) * nq.
 * out_qc (nq x 32 bits: float, or int for the integer kinds) and out_norms (r1 - r0 row sums of squares, float / int) may be
 * NULL.  Synchronous. */
VSB_API int vsb_debug_tc_level(vsb_index *ix, int metric, const void *queries, int nq, const float *U, int64_t r0, int64_t r1,
                               int N, int mode, void *out, int64_t out_cap, void *out_qc, void *out_norms, int64_t *out_count);
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
/* tuning knobs for experiments: name in {"stage_bytes","direct","ring_bytes","time_kernels","no_batch","batch_debug","batch_m0","batch_growth","balance","fuse_mb","scan_streams","xwait_ms","epi_chunk","push_mode","merge_stream" (experiment)};
 * values are non-negative; returns the previous value, or a negative VSB_E* code (unknown name, negative value) */
VSB_API int vsb_set_option(const char *name, int value);

#ifdef __cplusplus
}
#endif
#endif /* VSB200_H */
