// engine.cu — host side of the H100 scan engine behind include/vsb200.h.
//
// Owns device residency of a column shard (the GPU counterpart of table_context.preloaded,
// /root/reference/src/sqlite-vector.c:126-137, filled by vector_quantize_preload :1338-1404),
// launches the sm_90a kernels in scan_kernels.cuh and finishes each query with the reference's
// k-slot algorithm (:1808-1817, :2022-2069, :2145-2152) over the few hundred surviving candidates.
// No CPU fallback: if CUDA is unavailable every entry point returns VSB_ENODEV.
#include "../../include/vsb200.h"

#include <cuda_runtime.h>

#include <algorithm>
#include <atomic>
#include <chrono>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <limits>
#include <map>
#include <memory>
#include <mutex>
#include <new>
#include <string>
#include <thread>
#include <vector>

#include "scan_kernels.cuh"
#include "batch_kernels.cuh"
#include "quant_kernels.cuh"
#include "owners.cuh"

using namespace vsb;

namespace {

thread_local std::string g_err;
std::atomic<long long> g_launches{0};
int g_opt_stage_bytes = 16384; // upper bound of one warp tile (ring stage); int8 dim 384: 12 KB tiles x 2 stages (chosen on earlier hardware)
int g_opt_direct = 0;          // 1: force the no-staging kernel
int g_opt_ring_bytes = 0;      // 0: use all shared memory left
int g_opt_no_batch = 0;        // 1: never take the tensor-core batch path
int g_opt_batch_debug = 0;     // 1: print per-stage timings of the batch path to stderr (serialises the stages)
int g_opt_batch_m0 = 128;      // batch path: rows refined exhaustively before the first tensor-core level
int g_opt_batch_growth = 8;    // batch path: each tensor-core level covers rows [m, growth*m) (capped by k, see batch_growth)
int g_opt_balance = 1;         // 1: adaptive row partition of the single-query scan (per-CTA speeds feed the next partition)
int g_opt_epi_chunk = 1;       // 1: integer tensor-core epilogue tests 32-column chunks (max score vs weakest bound) before any per-column work
int g_opt_time_kernels = 0;    // 1: bracket every kernel launch with CUDA events (bench.py roofline leg)
int g_opt_scan_streams = 2;    // 2: consecutive scan launches alternate between two streams, so the CTAs of launch i+1 take over each SM
                               // as soon as the CTA of launch i on it exits (one scan CTA fits per SM): no grid-wide drain between
                               // launches, per-SM speed differences turn into an earlier start of the next query.  1: one stream.
// 1: f32 columns batch L2 / cosine / dot queries on the tensor cores in TF32 (tc_kind_of); 0: per query.  Set at load from
// VSB_F32_BATCH, so that users of the SQLite extension can turn it on; per process
int g_opt_f32_batch = [] {
    const char *e = getenv("VSB_F32_BATCH");
    return (e && atoi(e) > 0) ? 1 : 0;
}();
int g_opt_sets_mem_mb = 0;     // vsb_scan_topk_sets: device memory its one-pass buffers may take, in MB (0: 1/8 of the free memory)
int g_opt_xwait_ms = 10000;    // exchange: how long the receiving side waits for a peer's head before it reports an error (a dead
                               // peer, not a slow one: ranks sharing one GPU or a busy host can start a batch seconds apart)

// cudaFuncSetAttribute costs ~1 us per call; the dynamic shared memory limit of a kernel only ever needs to grow
int set_smem_limit(const void *fn, size_t bytes) {
    static std::mutex mu;
    static std::vector<std::pair<const void *, size_t>> seen;     // per process; devices are identical H100s
    std::lock_guard<std::mutex> lk(mu);
    int dev = 0;
    cudaGetDevice(&dev);
    const void *key = (const void *)((uintptr_t)fn ^ ((uintptr_t)dev << 56));
    for (auto &e : seen)
        if (e.first == key) {
            if (e.second >= bytes) return 0;
            cudaError_t r = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
            if (r == cudaSuccess) e.second = bytes;
            return (int)r;
        }
    cudaError_t r = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
    if (r == cudaSuccess) r = cudaFuncSetAttribute(fn, cudaFuncAttributePreferredSharedMemoryCarveout, (int)cudaSharedmemCarveoutMaxShared);
    if (r == cudaSuccess) seen.emplace_back(key, bytes);
    return (int)r;
}

int fail(int code, const char *fmt, ...) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    g_err = buf;
    return code;
}

#define CU(call)                                                                                           \
    do {                                                                                                   \
        cudaError_t e_ = (call);                                                                           \
        if (e_ != cudaSuccess)                                                                             \
            return fail(e_ == cudaErrorMemoryAllocation ? VSB_ENOMEM : VSB_ECUDA, "%s failed: %s (%s:%d)", \
                        #call, cudaGetErrorString(e_), __FILE__, __LINE__);                                \
    } while (0)

int elem_size(int vtype) {
    switch (vtype) {
    case VSB_F32: return 4;
    case VSB_F16: case VSB_BF16: return 2;
    case VSB_U8: case VSB_I8: return 1;
    }
    return 0;
}

// grows buf, which holds cap elements, to need elements (never shrinks).  The old contents are dropped: every caller is a
// synchronous call, so no launch still reads the old buffer.  counted: the byte count that the growth is added to, or null
template <template <class> class Buf, class T>
int grow_buf(Buf<T> &buf, long long &cap, long long need, size_t *counted) {
    if (need <= cap) return VSB_OK;
    Buf<T> b;
    CU(b.alloc(sizeof(T) * (size_t)need));
    if (counted) *counted += sizeof(T) * (size_t)(need - cap);
    buf = std::move(b);
    cap = need;
    return VSB_OK;
}

constexpr size_t kStageBuf = 32u << 20;  // pinned staging buffers for preload (two of them)
constexpr int kOutCap = 1 << 16;         // survivor capacity per query (mapped pinned)
constexpr int kMaxK = 256;               // candidate path; larger k takes the large-k path (large_k_candidates)
constexpr int kSlots = 32;               // result slots: queries in flight (the sharded exchange moves groups of them; a rank may have at most
                                         // kSlots / 2 queries in flight so that a peer never overwrites a gather row that is still being read)

// Scan workspace of one pass (per query of the pass: per-stream k-lists / CTA lists, in-CTA bounds, candidate logs, at the
// offsets pass_lists / pass_logs / pass_streams): written by scan_kernel, read by filter_kernel.  The Works rotate so that the
// filters of launch i (filter stream) overlap the scan of launch i+1.
struct Work {
    DeviceBuf<float> d_lists, d_tlocal;
    DeviceBuf<uint2> d_logs;
    DeviceBuf<int> d_counts;
    DeviceBuf<long long> d_bounds;   // [CTAs + 1] adaptive tile partition used by the NEXT scan on this workspace
    DeviceBuf<unsigned> d_cta_time;  // [CTAs] cycles each scan CTA took (written by scan_kernel, read by filter_kernel)
    long long bounds_tiles = -1;     // total tiles the bounds were laid out for (-1: not initialised)
    Event scanned;                   // scan stream: the scan that filled this workspace has finished
    Event drained;                   // filter stream: the filters that read this workspace have finished
    bool in_use = false;
};
constexpr int kWorks = 4;

// A query's result head (ResultHead, scan_kernels.cuh) is written by filter_kernel into DEVICE memory and fetched with one
// async copy; the (rare) survivors beyond kFirstFetch go to the slot's tail and are fetched by a second copy.  The heads of
// all slots are ONE contiguous allocation (slot s at s * kHeadBytes), so a launcher can all-gather the heads of a group of
// consecutive slots with a single collective.  (Zero-copy writes of ~300 scattered 8-byte records over PCIe made the filter
// kernel 5x slower than writing to HBM and copying once.)
struct Slot {
    ResultHead *d_head = nullptr, *h_head = nullptr; // this slot's head inside vsb_index::d_heads / h_heads
    uint2 *h_tail = nullptr, *d_tail = nullptr;      // survivors kFirstFetch.. (inside vsb_index::d_tails / h_tails)
    uint8_t *h_query = nullptr, *d_query = nullptr;  // pinned staging + device copy of the query (inside vsb_index::h_queries / d_queries)
    int *d_ctrl = nullptr;                           // inside vsb_index::d_ctrl
    Event done;   // recorded after the result block of this slot has been copied to the host
    int seq = 0;
};

// The pair list of range search and large k (pair_list_run): the (row, distance bits) pairs the kernels append, their counter,
// which keeps counting past cap, and the counter's host copy.  Large k reads the list back through the pinned h_pairs.
struct PairList {
    DeviceBuf<uint2> d_pairs;
    long long cap = 0;
    DeviceBuf<unsigned> d_count;
    HostBuf<unsigned> h_count;
    HostBuf<uint2> h_pairs;
    long long h_cap = 0;
};

// Single-query submissions held to share one pass of the column (vsb_scan_submit, DESIGN §3.2): one metric and k; query[j] is
// what the pass reads (a host query was staged into its slot's buffer on ss when it was submitted)
struct HeldPass {
    int nq = 0, metric = 0, k = 0;
    cudaStream_t ss = nullptr;
    const uint8_t *query[kMaxPass] = {};
    int slot[kMaxPass] = {};
};

struct BatchWs;   // batch_host.inc
struct SetsState;   // batch_host.inc
struct GroupedShard;   // batch_host.inc
void groupings_detach(std::vector<vsb_grouping *> &list);   // column.inc

}  // namespace

struct Exchange;    // exchange.inc

// Destroyed only with its streams drained and its device current (vsb_index_free); see owners.cuh
struct vsb_index {
    Stream stream;    // staging, scans and the batch path
    Stream fstream;   // filter + result copy of a query
    Stream stream2;   // second scan stream (option scan_streams = 2): single-query scans alternate between the two
    Stream xstream;   // exchange: flag wait + copy of the gathered heads to the host
    Stream cstream;   // streamed index: window copies
    int device = 0, vtype = 0, dim = 0, esize = 0, pitch = 0;
    long long cap = 0, n = 0, first_seq = 0;
    DeviceBuf<uint8_t> d_vec;
    bool implicit_ids = true;
    std::vector<int64_t> h_rowids;
    HostBuf<uint8_t> stage[2];
    Event stage_ev[2];
    int stage_next = 0;
    int num_sms = 0, max_smem = 0;
    // streamed mode (corpus larger than the device budget, SURVEY §8 f3): the column lives in pinned host memory and passes
    // through two device windows of win_rows rows; every window is scanned like a shard while the next one is copied
    bool streamed = false;
    HostBuf<uint8_t> h_arena;         // [cap][pitch] pinned
    DeviceBuf<uint8_t> d_win[2];
    long long win_rows = 0;
    Event win_copied[2], win_scanned[2];
    long long st_stream_bytes = 0, st_stream_us = 0;
    int snext = 0;
    std::unique_ptr<Exchange> xch;    // peer-memory exchange (multi-GPU), see exchange.inc
    // scan workspaces, for passes of up to ws_width queries (grown to the widest pass launched so far)
    int ws_kcap = 0, ws_logcap = 0, ws_streams = 0, ws_width = 0, ws_next = 0;
    Work work[kWorks];
    Slot slot[kSlots];
    // the allocations behind the result slots (a Slot holds views into them)
    DeviceBuf<uint8_t> d_heads;       // kSlots x kHeadBytes
    HostBuf<uint8_t> h_heads;
    DeviceBuf<uint8_t> d_tails;       // kSlots x (kOutCap - kFirstFetch) x uint2
    HostBuf<uint8_t> h_tails;
    HostBuf<uint8_t> h_queries;       // kSlots x pitch
    DeviceBuf<uint8_t> d_queries;
    DeviceBuf<int> d_ctrl;            // kSlots x 4
    bool slots_ready = false;
    DeviceBuf<float> d_dist_all;
    int last_slot = -1, last_metric = 0;
    HeldPass held;                    // vsb_scan_submit's queries waiting for a pass
    uint32_t uncollected = 0;         // slots of vsb_scan_submit (fetch != 0) not collected yet: bit s = slot s
    long long st_scan_passes = 0, st_pass_queries = 0;   // top-k passes and the queries they scored
    int last_kcap = 0;                // kcap of the most recent top-k pass (vsb_index_stat "plan_pass_max")
    // optional per-kernel event timing (vsb_profile_read)
    std::vector<Event> prof_ev;         // quadruples: before scan, after scan (scan stream), before filter, after filter (filter stream)
    std::vector<int> prof_kind;         // 1 = scan only, 2 = scan + filter
    size_t prof_used = 0;
    unsigned prof_tick = 0;
    size_t dev_bytes = 0;
    long long st_queries = 0, st_survivors = 0, st_fallbacks = 0, st_last_survivors = 0;
    long long st_batches = 0, st_batch_cands = 0, st_batch_kept = 0, st_tc_us = 0, st_tc_rows = 0, st_batch_us = 0;
    int last_log2p = -1, last_nsw = -1, last_direct = -1;   // plan of the most recent scan launch (vsb_index_stat "plan_*")
    std::unique_ptr<BatchWs> batch;   // tensor-core batch path workspace
    // row filter of the filtered scan in progress (vsb_scan_topk_filtered, FilterScope): bitmaps over this shard's rows (row i:
    // bit i & 31 of word i >> 5) on the host and in d_allow; both null outside such a call, when every row is eligible
    const uint32_t *flt_h = nullptr, *flt_d = nullptr;
    DeviceBuf<uint32_t> d_allow;      // rows / 32 words + 1: a warp's read past the last row stays inside
    long long allow_words = 0;
    // rowid -> row lookup of explicit rowids (vsb_index_rowid_bitmap): (rowid, row) sorted, built for rowid_rows rows on first
    // need; an append changes n and so rebuilds it
    std::vector<std::pair<int64_t, long long>> rowid_sorted;
    long long rowid_rows = -1;
    // range search (vsb_scan_range) and large k: the pair list, which starts at kRangeCap0 pairs or more and grows to the exact
    // count of a query that needed more
    PairList plist;
    long long st_range_pairs = 0, st_range_passes = 0, st_range_host_sorts = 0;
    long long st_range_batches = 0, st_range_batch_fallbacks = 0, st_range_query_fallbacks = 0;
    // large k (k > kMaxK, DESIGN §3.11): the prefix select's histograms and state and the compaction's per-block offsets (for
    // lk_boff_cap blocks); the candidates themselves go to the pair list
    DeviceBuf<unsigned> d_lk_hist, d_lk_boff;
    DeviceBuf<LkState> d_lk_state;
    long long lk_boff_cap = 0;
    long long st_large_k_queries = 0, st_large_k_cands = 0, st_large_k_regrows = 0;
    long long st_large_k_batches = 0, st_large_k_batch_fallbacks = 0, st_large_k_query_fallbacks = 0;   // DESIGN §3.12
    long long st_large_k_levels_us = 0, st_large_k_replay_us = 0, st_large_k_replay_threads = 0;
    // listed rows (vsb_scan_topk_rows, DESIGN §3.13): one staging area on each side for the queries, their norms, the (row,
    // query) pairs and the distances, grown never shrunk; a streamed index's kernel reads its rows at arena_dev, h_arena's
    // device address, checked on first use
    DeviceBuf<uint8_t> d_rows;
    HostBuf<uint8_t> h_rows;
    long long rows_cap = 0, rows_hcap = 0;
    const uint8_t *arena_dev = nullptr;
    long long st_rows_queries = 0, st_rows_pairs = 0, st_rows_host_bytes = 0;
    // per-query sets of the sets call in progress (vsb_scan_topk_sets, SetsScope): their device bitmaps, whose union is flt_d;
    // null outside such a call
    const SetsState *sets = nullptr;
    long long st_sets_batches = 0, st_sets_fallbacks = 0, st_sets_levels = 0, st_sets_plan_us = 0;
    // grouped top-k (vsb_scan_topk_grouped, DESIGN §3.15): one device area for the per-query arrays of a call, and a streamed
    // index's distances of every window (4 bytes per row), both grown never shrunk
    DeviceBuf<uint8_t> d_grouped;
    DeviceBuf<float> d_grouped_dist;
    long long grouped_cap = 0, grouped_dist_cap = 0;
    // the device's (rowid ^ 2^63, row) table of explicit rowids sorted by rowid, which the layout builder searches; built for
    // rowid_tab_rows rows on first need, so an append rebuilds it
    DeviceBuf<unsigned long long> d_rowid_tab;
    DeviceBuf<uint32_t> d_rowid_tab_row;
    long long rowid_tab_cap = 0, rowid_tab_row_cap = 0, rowid_tab_rows = -1;
    // the layout builder's pinned staging of the caller's keys (two buffers, allocated on first need)
    HostBuf<uint8_t> lay_stage[2];
    Event lay_stage_ev[2];
    int lay_next = 0;
    // this shard's state of the most recent grouped call (vsb_debug_read "grouped"), kept until the next one; and the distances
    // planted by vsb_debug_write "grouped_dist" for the next call (empty: scan them)
    std::unique_ptr<GroupedShard> grouped;
    std::vector<float> grouped_plant;
    // the groupings made on this index (vsb_grouping_create), detached when it is freed
    std::vector<vsb_grouping *> groupings;
    long long st_grouped_queries = 0, st_grouped_pairs = 0, st_grouped_cands = 0, st_grouped_keys_replayed = 0;
    long long st_grouped_regrows = 0, st_grouped_layout_us = 0, st_grouped_scan_us = 0, st_grouped_walk_us = 0, st_grouped_replay_us = 0;
    long long st_grouped_layout_reuses = 0;
};

// result of a range call (vsb_scan_range): per query, rowids and distances in result order
struct vsb_range {
    std::vector<std::vector<int64_t>> ids;
    std::vector<std::vector<double>> dist;
};

// result of a grouped call (vsb_scan_topk_grouped): per query, the keys in rank order and each key's rows in result order
struct vsb_grouped {
    struct Query {
        std::vector<int32_t> keys;
        std::vector<int64_t> offsets{0};
        std::vector<int64_t> ids;
        std::vector<double> dist;
    };
    std::vector<Query> q;
};

namespace {

// ------------------------------------------------------------------ kernel dispatch
using ScanFn = void (*)(const ScanParams);
// R: range mode; M: pass width (top-k and all distances)
template <int VT, int MC, bool D, bool R, int M>
ScanFn fn_of() {
    if constexpr (R) return scan_range_kernel<VT, MC, D>;
    else if constexpr (M == 1) return scan_kernel<VT, MC, D>;
    else return scan_pass_kernel<VT, MC, D, M>;
}

template <bool R, int M>
ScanFn pick_kernel_of(int vtype, int mc, bool direct) {
#define ROW(VT)                                                                                                   \
    case VT:                                                                                                      \
        switch (mc) {                                                                                             \
        case MC_L2: return direct ? fn_of<VT, MC_L2, true, R, M>() : fn_of<VT, MC_L2, false, R, M>();             \
        case MC_COS: return direct ? fn_of<VT, MC_COS, true, R, M>() : fn_of<VT, MC_COS, false, R, M>();          \
        case MC_DOT: return direct ? fn_of<VT, MC_DOT, true, R, M>() : fn_of<VT, MC_DOT, false, R, M>();          \
        case MC_L1: return direct ? fn_of<VT, MC_L1, true, R, M>() : fn_of<VT, MC_L1, false, R, M>();             \
        }                                                                                                         \
        break;
    switch (vtype) {
        ROW(T_F32) ROW(T_F16) ROW(T_BF16) ROW(T_U8) ROW(T_I8)
    }
#undef ROW
    return nullptr;
}
// range: the range-mode instantiation (vsb_scan_range); nq: the queries of a top-k pass, which runs the narrowest width that
// holds them
ScanFn pick_kernel(int vtype, int mc, bool direct, bool range = false, int nq = 1) {
    if (range) return pick_kernel_of<true, 1>(vtype, mc, direct);
    if (nq <= 1) return pick_kernel_of<false, 1>(vtype, mc, direct);
    if (nq <= 2) return pick_kernel_of<false, 2>(vtype, mc, direct);
    if (nq <= 4) return pick_kernel_of<false, 4>(vtype, mc, direct);
    return pick_kernel_of<false, 8>(vtype, mc, direct);
}

int metric_class(int metric, int *root) {
    *root = 0;
    switch (metric) {
    case VSB_L2: *root = 1; return MC_L2;
    case VSB_SQUARED_L2: return MC_L2;
    case VSB_COSINE: return MC_COS;
    case VSB_DOT: return MC_DOT;
    case VSB_L1: return MC_L1;
    }
    return -1;
}

struct Plan {
    bool direct;
    int log2P, wtile_bytes, nsw;
    bool reserved;      // the filter reserve was left free
    size_t smem;
};

// choose lanes-per-row, ring depth and shared-memory size for (pitch, kcap) and a pass of nq queries
Plan make_plan(const vsb_index *ix, int kcap, int nq = 1) {
    Plan pl{};
    const int pitch = ix->pitch;
    int log2P = 0;
    while (log2P < 5 && (32 >> log2P) * (long long)pitch > g_opt_stage_bytes) ++log2P;
    // Room for max(2, nq) query + list buffers.  A one-query pass uses one of each: the room of the second is what lets a
    // pass of two keep the plan of one (pass_max); giving it to the ring instead would change the plan at many shapes.
    const size_t nbuf = (size_t)std::max(2, nq);
    const size_t fixed = kBarrierBytes + ((nbuf * pitch + nbuf * kWarps * kcap * 4 + 127) & ~(size_t)127);
    size_t avail = (size_t)ix->max_smem > fixed ? (size_t)ix->max_smem - fixed : 0;
    if (g_opt_ring_bytes > 0 && (size_t)g_opt_ring_bytes < avail) avail = (size_t)g_opt_ring_bytes;
    const size_t wtile = (size_t)(32 >> log2P) * pitch;
    // leave room on the SM for one filter block of the previous query (it runs beside the scan CTA, see launch_scan)
    const size_t reserve = filter_fast_smem(ix->num_sms) + 3072;
    pl.reserved = kcap > 0 && kcap <= 32 && avail > reserve && (avail - reserve) / kWarps / (wtile ? wtile : 1) >= 2;
    if (pl.reserved) avail -= reserve;
    int nsw = (int)(avail / kWarps / (wtile ? wtile : 1));
    if (nsw > kMaxStages) nsw = kMaxStages;
    pl.direct = g_opt_direct || nsw < 2;
    if (pl.direct) {
        pl.log2P = 5;  // a whole warp per row, coalesced 16-byte loads straight from HBM
        pl.wtile_bytes = pitch;
        pl.nsw = 1;
        pl.smem = fixed;
    } else {
        pl.log2P = log2P;
        pl.wtile_bytes = (int)wtile;
        pl.nsw = nsw;
        pl.smem = fixed + (size_t)kWarps * nsw * wtile;
    }
    return pl;
}

// the widest pass of a shape: the largest width whose query and list buffers fit beside the one-query plan left as it is
// (the same lanes per row, ring depth, DIRECT and filter reserve), so that sharing a pass never slows the scan of a row
int pass_max(const vsb_index *ix, int kcap) {
    const Plan one = make_plan(ix, kcap);
    int w = 1;
    for (int m = 2; m <= kMaxPass; m *= 2) {
        const Plan pl = make_plan(ix, kcap, m);
        if (pl.direct != one.direct || pl.log2P != one.log2P || pl.nsw != one.nsw || pl.reserved != one.reserved ||
            pl.smem > (size_t)ix->max_smem)
            break;
        w = m;
    }
    return w;
}

// the result slots, built on first need
int ensure_slots(vsb_index *ix) {
    if (ix->slots_ready) return VSB_OK;
    const size_t tail_bytes = sizeof(uint2) * (size_t)(kOutCap - kFirstFetch);
    DeviceBuf<uint8_t> d_heads, d_tails, d_queries;
    HostBuf<uint8_t> h_heads, h_tails, h_queries;
    DeviceBuf<int> d_ctrl;
    Event done[kSlots];
    CU(d_heads.alloc(kHeadBytes * kSlots));
    CU(cudaMemset(d_heads, 0, kHeadBytes * kSlots));
    CU(h_heads.alloc(kHeadBytes * kSlots));
    memset(h_heads, 0, kHeadBytes * kSlots);
    CU(d_tails.alloc(tail_bytes * kSlots));
    CU(h_tails.alloc(tail_bytes * kSlots));
    CU(h_queries.alloc((size_t)ix->pitch * kSlots));        // query staging of all slots: one pinned + one device allocation
    CU(d_queries.alloc((size_t)ix->pitch * kSlots));
    CU(d_ctrl.alloc(sizeof(int) * 4 * kSlots));
    CU(cudaMemset(d_ctrl, 0, sizeof(int) * 4 * kSlots));
    for (Event &e : done) CU(e.create(cudaEventDisableTiming));
    for (int i = 0; i < kSlots; ++i) {
        Slot &s = ix->slot[i];
        s.d_head = (ResultHead *)(d_heads + kHeadBytes * i);
        s.h_head = (ResultHead *)(h_heads + kHeadBytes * i);
        s.d_tail = (uint2 *)(d_tails + tail_bytes * i);
        s.h_tail = (uint2 *)(h_tails + tail_bytes * i);
        s.h_query = h_queries + (size_t)ix->pitch * i;
        s.d_query = d_queries + (size_t)ix->pitch * i;
        s.d_ctrl = d_ctrl + 4 * i;
        s.done = std::move(done[i]);
    }
    ix->d_heads = std::move(d_heads); ix->h_heads = std::move(h_heads);
    ix->d_tails = std::move(d_tails); ix->h_tails = std::move(h_tails);
    ix->h_queries = std::move(h_queries); ix->d_queries = std::move(d_queries);
    ix->d_ctrl = std::move(d_ctrl);
    ix->slots_ready = true;
    return VSB_OK;
}

int flush_held(vsb_index *ix);

// waits for the scan streams and the filter stream of ix (after launching the held pass)
int drain(vsb_index *ix) {
    const int rc = flush_held(ix);
    if (rc) return rc;
    CU(cudaStreamSynchronize(ix->stream));
    CU(cudaStreamSynchronize(ix->stream2));
    CU(cudaStreamSynchronize(ix->fstream));
    return VSB_OK;
}

// the workspaces hold passes of `width` queries with this k (never shrunk: a caller who never shares a pass keeps width 1)
int ensure_workspace(vsb_index *ix, int k, int width = 1) {
    const int kcap = std::max((k + 31) & ~31, ix->ws_kcap);
    const int logcap = std::max(std::max(256, 12 * k), ix->ws_logcap);
    width = std::max(width, ix->ws_width);
    const int streams = ix->num_sms * kWarps;
    if (ix->ws_kcap >= kcap && ix->ws_logcap >= logcap && ix->ws_width >= width && ix->ws_streams == streams) return VSB_OK;
    const int rc = drain(ix);       // queries in flight still use the old workspaces
    if (rc) return rc;
    Work fresh[kWorks];
    for (int i = 0; i < kWorks; ++i) {
        Work &w = fresh[i], &old = ix->work[i];
        CU(w.d_lists.alloc(sizeof(float) * (size_t)width * streams * kcap));
        CU(w.d_logs.alloc(sizeof(uint2) * (size_t)width * streams * logcap));
        CU(w.d_counts.alloc(sizeof(int) * (size_t)width * streams));
        CU(w.d_tlocal.alloc(sizeof(float) * (size_t)width * streams));
        CU(w.d_bounds.alloc(sizeof(long long) * (size_t)(ix->num_sms + 1)));
        CU(w.d_cta_time.alloc(sizeof(unsigned) * (size_t)ix->num_sms));
        if (!old.scanned) CU(old.scanned.create(cudaEventDisableTiming));
        if (!old.drained) CU(old.drained.create(cudaEventDisableTiming));
    }
    for (int i = 0; i < kWorks; ++i) {   // the events stay across regrowth
        fresh[i].scanned = std::move(ix->work[i].scanned);
        fresh[i].drained = std::move(ix->work[i].drained);
        ix->work[i] = std::move(fresh[i]);
    }
    ix->ws_kcap = kcap; ix->ws_logcap = logcap; ix->ws_width = width; ix->ws_streams = streams;
    return VSB_OK;
}

// the ScanParams of a top-k and a range launch alike: rows [0, n) of vec, whose first row is shard row r0 (the row filter is
// indexed by shard rows), scanned with plan pl for the query at d_query (the first of a pass's queries)
ScanParams scan_params(const vsb_index *ix, const Plan &pl, int root, const uint8_t *d_query, const uint8_t *vec, long long n, long long r0) {
    ScanParams p{};
    p.vec = vec;
    p.n = n;
    p.pitch = ix->pitch;
    p.nc = ix->pitch / 16;
    p.log2P = pl.log2P;
    p.wtile_bytes = pl.wtile_bytes;
    p.nsw = pl.nsw;
    p.root = root;
    p.nq = 1;
    p.query[0] = d_query;
    p.allow = ix->flt_d;
    p.allow_base = r0;
    return p;
}

// the plan of the most recent scan launch (vsb_index_stat "plan_*")
void note_plan(vsb_index *ix, const Plan &pl) {
    ix->last_log2p = pl.log2P;
    ix->last_nsw = pl.nsw;
    ix->last_direct = pl.direct ? 1 : 0;
}

unsigned exchange_next_seq(vsb_index *ix, int slot);
int merge_blocks_strided(const uint8_t *blocks, int world, size_t stride, const int64_t *first_seq, int k, int64_t *out_rowids, double *out_dist);
int exchange_fill_push(vsb_index *ix, PushParams *pp);

// launches one pass of the scan kernel for nq <= pass_max queries (device pointers queries[j], pitch bytes each) on ss and, when
// k > 0, one filter per query on ix->fstream; slots[j] receives query j's result.  nq > 1 needs k > 0.
// fetch: copy each slot's head to pinned host memory afterwards (false when the heads are all-gathered on the device)
// ss: the scan stream of this launch (next_scan_stream); push: the heads are labelled for the exchange (shard index and
// exchange sequence number); push_heads_kernel moves them (exchange_push)
// view_vec / view_n: scan these rows instead of the resident column (the windows of a streamed index)
// view_r0: the shard row of view_vec's first row (the row filter is indexed by shard rows)
// plan_kcap >= 0 (k == 0 only): scan with the plan of that kcap instead of k's, for all-distances scans whose distances must have
// the bits of a top-k scan at that k (grouped top-k)
int launch_scan(vsb_index *ix, int metric, const uint8_t *const *queries, Slot *const *slots, int nq, int k, float *d_dist_all, bool fetch,
                cudaStream_t ss, bool push = false, const uint8_t *view_vec = nullptr, long long view_n = -1, long long view_r0 = 0,
                int plan_kcap = -1) {
    const uint8_t *scan_vec = view_vec ? view_vec : ix->d_vec;
    const long long scan_n = view_vec ? view_n : ix->n;
    if (!scan_vec) return fail(VSB_EINVAL, "this entry point needs a resident (not streamed) index");
    int root = 0;
    const int mc = metric_class(metric, &root);
    if (mc < 0) return fail(VSB_EINVAL, "unknown distance metric %d", metric);
    // per-launch list stride: the workspace may have been sized by an earlier, larger k (ensure_workspace never shrinks), but
    // the scan's list layout, the filter's FAST/generic choice and its shared-memory layout all follow THIS query's k
    const int kcap = k > 0 ? ((k + 31) & ~31) : 0;
    if (kcap > ix->ws_kcap) return fail(VSB_EINVAL, "scan workspace too small for k = %d", k);
    if (nq < 1 || (nq > 1 && (k <= 0 || nq > ix->ws_width || nq > pass_max(ix, kcap))))
        return fail(VSB_EINVAL, "bad pass of %d queries", nq);
    const Plan pl = make_plan(ix, k == 0 && plan_kcap >= 0 ? plan_kcap : kcap, nq);
    ScanFn fn = pick_kernel(ix->vtype, mc, pl.direct, false, nq);
    if (!fn) return fail(VSB_EINVAL, "unsupported vector type %d", ix->vtype);
    // max-shared carve-out for the scan AND the filter kernel: kernels that want different L1/shared splits cannot share
    // an SM, and the filter blocks of launch i are meant to run beside the scan CTAs of launch i+1
    CU((cudaError_t)set_smem_limit((const void *)fn, pl.smem));

    // the scan runs on its scan stream (ss), the filters (+ result copies) on ix->fstream: while the filters of this launch walk
    // the k-lists and compact the candidate logs, the scan of the next launch is already streaming the shard (the filter
    // blocks are small enough to sit on the SMs beside the scan CTAs).  The workspaces rotate.
    Work *wk = nullptr;
    if (k > 0) {
        wk = &ix->work[ix->ws_next];
        ix->ws_next = (ix->ws_next + 1) % kWorks;
        if (wk->in_use) CU(cudaStreamWaitEvent(ss, wk->drained, 0));   // its previous filters must have read it
    }
    // adaptive partition (k <= 32 path only: that filter kernel maintains it): equal shares to start with
    const long long rpw = 32 >> pl.log2P;
    const long long total_tiles = (scan_n + rpw - 1) / rpw;
    const bool balance = wk != nullptr && g_opt_balance && kcap == 32 && total_tiles >= 64ll * ix->num_sms;
    if (balance && wk->bounds_tiles != total_tiles) {
        std::vector<long long> b((size_t)ix->num_sms + 1);
        for (int c = 0; c <= ix->num_sms; ++c) b[(size_t)c] = (total_tiles * c) / ix->num_sms;
        CU(cudaMemcpyAsync(wk->d_bounds, b.data(), sizeof(long long) * b.size(), cudaMemcpyHostToDevice, ss));   // pageable: staged before return
        CU(cudaMemsetAsync(wk->d_cta_time, 0, sizeof(unsigned) * (size_t)ix->num_sms, ss));
        wk->bounds_tiles = total_tiles;
    }
    ScanParams p = scan_params(ix, pl, root, queries[0], scan_vec, scan_n, view_r0);
    p.nq = nq;
    for (int j = 0; j < nq; ++j) {
        p.query[j] = queries[j];
        p.ctrl[j] = slots[j] ? slots[j]->d_ctrl : nullptr;
    }
    p.k = k;
    p.kcap = kcap;
    p.logcap = ix->ws_logcap;
    p.lists = wk ? wk->d_lists.get() : nullptr;
    p.tlocal = wk ? wk->d_tlocal.get() : nullptr;
    p.logs = wk ? wk->d_logs.get() : nullptr;
    p.counts = wk ? wk->d_counts.get() : nullptr;
    p.dist_all = d_dist_all;
    p.bounds = balance ? wk->d_bounds.get() : nullptr;
    p.cta_time = balance ? wk->d_cta_time.get() : nullptr;
    Event *pev = nullptr;
    if (g_opt_time_kernels > 0 && (ix->prof_tick++ % g_opt_time_kernels) == 0) {   // time_kernels = N: every N-th launch
        if (ix->prof_used + 4 > ix->prof_ev.size()) {
            for (int i = 0; i < 4; ++i) {
                Event e;
                CU(e.create(cudaEventDefault));
                ix->prof_ev.push_back(std::move(e));
            }
        }
        pev = &ix->prof_ev[ix->prof_used];
        ix->prof_used += 4;
        ix->prof_kind.push_back(k > 0 ? 2 : 1);
        CU(cudaEventRecord(pev[0], ss));
    }
    fn<<<ix->num_sms, kThreads, pl.smem, ss>>>(p);
    CU(cudaGetLastError());
    ++g_launches;
    note_plan(ix, pl);
    if (k > 0) {
        ix->st_scan_passes++;
        ix->st_pass_queries += nq;
        ix->last_kcap = kcap;
    }
    if (pev) CU(cudaEventRecord(pev[1], ss));
    if (k > 0) {
        CU(cudaEventRecord(wk->scanned, ss));
        CU(cudaStreamWaitEvent(ix->fstream, wk->scanned, 0));
        PushParams pp{};
        if (push) {
            const int rc = exchange_fill_push(ix, &pp);
            if (rc) return rc;
        }
        const int S = ix->ws_streams;
        const bool fast = (kcap == 32) && filter_fast_smem(S / kWarps) + 2048 <= (size_t)ix->max_smem;
        const int fw = filter_warps(fast);
        const int nblocks = (S + fw - 1) / fw;
        if (nblocks > kTableCap) return fail(VSB_ERANGE, "too many filter blocks (%d)", nblocks);
        if (pev) CU(cudaEventRecord(pev[2], ix->fstream));
        for (int j = 0; j < nq; ++j) {
            Slot *slot = slots[j];
            FilterParams f{};
            f.src = pp.src;
            f.S = S;
            f.k = k;
            f.kcap = kcap;
            f.logcap = ix->ws_logcap;
            f.headcap = kFirstFetch;
            f.outcap = kOutCap;
            f.lists = wk->d_lists + pass_lists(j, S, kcap);
            f.tlocal = wk->d_tlocal + pass_streams(j, S);
            f.logs = wk->d_logs + pass_logs(j, S, ix->ws_logcap);
            f.counts = wk->d_counts + pass_streams(j, S);
            f.out = head_survivors(slot->d_head);
            f.out_tail = slot->d_tail;
            f.table = head_table(slot->d_head);
            f.hdr = slot->d_head;
            f.ctrl = slot->d_ctrl;
            f.seqno = ++slot->seq;
            f.xseq = push ? exchange_next_seq(ix, (int)(slot - ix->slot)) : 0u;
            f.bounds = (balance && j == 0) ? wk->d_bounds.get() : nullptr;   // the partition follows the CTA times once per pass
            f.cta_time = wk->d_cta_time;
            f.total_tiles = total_tiles;
            if (fast) {
                const size_t fsm = filter_fast_smem(S / kWarps);
                CU((cudaError_t)set_smem_limit((const void *)filter_kernel<true>, fsm));
                filter_kernel<true><<<nblocks, fw * 32, fsm, ix->fstream>>>(f);
            } else {
                const size_t fsm = sizeof(float) * ((size_t)2 * kFilterWarps * kcap + (size_t)S + 32);
                CU((cudaError_t)set_smem_limit((const void *)filter_kernel<false>, fsm));
                filter_kernel<false><<<nblocks, fw * 32, fsm, ix->fstream>>>(f);
            }
            CU(cudaGetLastError());
            ++g_launches;
            if (j == nq - 1) {                       // the pass's filters are the last readers of the workspace
                if (pev) CU(cudaEventRecord(pev[3], ix->fstream));
                CU(cudaEventRecord(wk->drained, ix->fstream));
                wk->in_use = true;
            }
            if (fetch) CU(cudaMemcpyAsync(slot->h_head, slot->d_head, kHeadBytes, cudaMemcpyDeviceToHost, ix->fstream));
            CU(cudaEventRecord(slot->done, ix->fstream));
        }
    }
    return VSB_OK;
}

// single-query scans alternate between two streams (option scan_streams, see g_opt_scan_streams)
cudaStream_t next_scan_stream(vsb_index *ix) {
    if (g_opt_scan_streams < 2) return ix->stream;
    ix->snext ^= 1;
    return ix->snext ? ix->stream2 : ix->stream;
}

inline int64_t rowid_of(const vsb_index *ix, uint32_t local) {
    return ix->implicit_ids ? (int64_t)(ix->first_seq + (long long)local + 1) : ix->h_rowids[local];
}

// ------------------------------------------------------------------ the reference's k-slot algorithm
inline int first_max(const double *v, int n) {  // first index of the maximum, strict '>' (:2022-2049)
    int b = 0;
    for (int i = 1; i < n; ++i)
        if (v[i] > v[b]) b = i;
    return b;
}
// k > kMaxK: first_max in O(log k) per slot change.  A tournament tree over the slots: node i (children 2i, 2i + 1, leaf j at
// node m + j) holds the first index of the maximum of its leaves.  A right child wins only when strictly greater, so equal
// values go to the lower index, as in first_max (the slots never hold NaN).  Leaves past k hold -1 and never win.
struct MaxTree {
    int m = 1;
    std::vector<int> node;
    static int better(const double *v, int a, int b) { return b < 0 ? a : a < 0 ? b : v[b] > v[a] ? b : a; }
    void build(const double *v, int k) {
        while (m < k) m <<= 1;
        node.assign((size_t)2 * m, -1);
        for (int j = 0; j < k; ++j) node[(size_t)(m + j)] = j;
        for (int i = m - 1; i >= 1; --i) node[(size_t)i] = better(v, node[(size_t)(2 * i)], node[(size_t)(2 * i + 1)]);
    }
    int update(const double *v, int j) {   // after slot j changed: the new first index of the maximum
        for (int i = (m + j) >> 1; i >= 1; i >>= 1) node[(size_t)i] = better(v, node[(size_t)(2 * i)], node[(size_t)(2 * i + 1)]);
        return node[1];
    }
};
struct SlotState {
    int k, mi;
    double *dist;
    int64_t *ids;
    MaxTree *tree = nullptr;   // k > kMaxK (slots_replay), else first_max
};
inline void slots_begin(SlotState &s) {  // :1808-1813 (max_index is carried over, not reset)
    for (int i = 0; i < s.k; ++i) { s.dist[i] = std::numeric_limits<double>::infinity(); s.ids[i] = 0; }
    if (s.mi < 0 || s.mi >= s.k) s.mi = 0;
}
inline void slots_offer(SlotState &s, float d, int64_t id) {  // :2102-2106 / :2145-2152
    if ((double)d < s.dist[s.mi]) {
        s.dist[s.mi] = (double)d;
        s.ids[s.mi] = id;
        s.mi = s.tree ? s.tree->update(s.dist, s.mi) : first_max(s.dist, s.k);
    }
}
inline int slots_finish(SlotState &s) {  // exchange sort + INF trim (:2051-2069, :1816-1817)
    const double inf = std::numeric_limits<double>::infinity();
    int unused = 0;
    for (int i = 0; i + 1 < s.k; ++i) {
        if (s.dist[i] == inf) ++unused;
        for (int j = i + 1; j < s.k; ++j)
            if (s.dist[j] < s.dist[i]) { std::swap(s.dist[i], s.dist[j]); std::swap(s.ids[i], s.ids[j]); }
    }
    if (s.dist[s.k - 1] == inf) ++unused;
    return s.k - unused;
}
// offers candidates as the kernels write them, (distance bits, local row), in order; row -> rowid through to_id
template <class ToId>
void slots_offer_cands(SlotState &s, const uint2 *c, size_t n, ToId to_id) {
    for (size_t i = 0; i < n; ++i) {
        float d;
        memcpy(&d, &c[i].x, 4);
        slots_offer(s, d, to_id(c[i].y));
    }
}
// one query through the k slots: feed(s) offers its candidates in scan order and returns VSB_OK or an error code.  *mi (null:
// 0) is the max_index cursor the slots start from; it is updated only when feed succeeds.  Returns the row count or the error.
template <class Feed>
int slots_replay(int k, int *mi, double *dist, int64_t *ids, Feed feed) {
    SlotState s{k, mi ? *mi : 0, dist, ids};
    slots_begin(s);
    MaxTree tree;
    if (k > kMaxK) {
        tree.build(dist, k);
        s.tree = &tree;
    }
    const int rc = feed(s);
    if (rc) return rc;
    if (mi) *mi = s.mi;
    return slots_finish(s);
}
// the max_index cursor of a scan of nq queries: a single query continues the caller's cursor and hands it back; the queries of
// a batch are independent, like nq separate cursors that each start at 0, and leave the caller's cursor alone
struct QueryCursor {
    int *caller;
    int nq, mi;
    QueryCursor(int *max_index, int nq) : caller(max_index), nq(nq), mi(max_index ? *max_index : 0) {}
    int *next() {   // the cursor of the next query
        if (nq > 1) mi = 0;
        return &mi;
    }
    void finish() const {
        if (caller && nq == 1) *caller = mi;
    }
};

// survivors a head holds itself: its headcap field when that is in (0, kFirstFetch], else kFirstFetch
int head_capacity(const ResultHead *h) { return (h->headcap > 0 && h->headcap <= kFirstFetch) ? h->headcap : kFirstFetch; }

// visits the survivors of one head in block-table order (= scan order): survivor i sits in the head below head_capacity(h),
// else at tail[i - head_capacity(h)].  VSB_ECUDA when the block count does not fit the table (`shard` names the head).
template <class Visit>
int for_each_survivor(const ResultHead *h, const uint2 *tail, int shard, Visit visit) {
    const int nblocks = h->nblocks;
    if (nblocks < 0 || nblocks > kTableCap) return fail(VSB_ECUDA, "malformed result head from shard %d", shard);
    const int headcap = head_capacity(h);
    const int2 *table = head_table(h);
    const uint2 *out = head_survivors(h);
    for (int b = 0; b < nblocks; ++b)
        for (int i = 0; i < table[b].y; ++i) {
            const int at = table[b].x + i;
            visit(at < headcap ? out[at] : tail[at - headcap]);
        }
    return VSB_OK;
}

// waits for the query of a slot and visits its survivors in scan order; *overflow: its candidates overflowed, nothing is visited
template <class Visit>
int visit_survivors(vsb_index *ix, Slot *slot, bool *overflow, Visit visit) {
    CU(cudaEventSynchronize(slot->done));
    *overflow = false;
    const ResultHead *h = slot->h_head;
    if (h->seq != slot->seq) return fail(VSB_ECUDA, "scan result header not published (seq %d != %d)", h->seq, slot->seq);
    if (h->flags) { *overflow = true; return VSB_OK; }
    const int total = h->total, headcap = head_capacity(h);
    if (total > headcap) {  // rare: fetch the tail of the survivor list
        if (cudaMemcpyAsync(slot->h_tail, slot->d_tail, sizeof(uint2) * (size_t)(total - headcap),
                            cudaMemcpyDeviceToHost, ix->fstream) != cudaSuccess ||
            cudaStreamSynchronize(ix->fstream) != cudaSuccess)
            return fail(VSB_ECUDA, "fetching %d survivors failed: %s", total, cudaGetErrorString(cudaGetLastError()));
    }
    long long n = 0;
    const int rc = for_each_survivor(h, slot->h_tail, 0, [&](uint2 c) { ++n; visit(c); });
    if (rc) return rc;
    ix->st_queries++;
    ix->st_survivors += n;
    ix->st_last_survivors = n;
    return VSB_OK;
}

// the all-distances buffer, allocated on first use: capacity floats for a resident index, two window halves for a streamed one
int ensure_dist_all(vsb_index *ix) {
    if (ix->d_dist_all) return VSB_OK;
    if (ix->streamed) {
        CU(ix->d_dist_all.alloc(sizeof(float) * 2 * (size_t)ix->win_rows));
        ix->dev_bytes += sizeof(float) * 2 * (size_t)ix->win_rows;
    } else {
        CU(ix->d_dist_all.alloc(sizeof(float) * (size_t)std::max<long long>(ix->cap, 1)));
        ix->dev_bytes += sizeof(float) * (size_t)ix->cap;
    }
    return VSB_OK;
}

int stage_query(vsb_index *ix, Slot *slot, const void *query, cudaStream_t ss) {
    const int qbytes = ix->dim * ix->esize;
    memcpy(slot->h_query, query, (size_t)qbytes);
    if (ix->pitch > qbytes) memset(slot->h_query + qbytes, 0, (size_t)(ix->pitch - qbytes));
    CU(cudaMemcpyAsync(slot->d_query, slot->h_query, (size_t)ix->pitch, cudaMemcpyHostToDevice, ss));
    return VSB_OK;
}

// ---- the view loop.  A view is rows [r0, r0 + rows) of the column in device memory at vec.  A resident index is one view, its
// whole column in d_vec.  A streamed index is one view per window: window w (rows [w * win_rows, ...)) is copied into
// d_win[w & 1] on the copy stream while window w-1 is being scanned, and its scan reads the window buffer with window-local rows.
struct View {
    long long index;      // window number
    long long r0, rows;   // shard row of the view's first row, and its rows
    const uint8_t *vec;
    int buf;              // window buffer, 0 or 1
    int slot;             // index % depth
};

// launch(view) enqueues the work of each view; visit(view) is called in view order, for a streamed index once `depth` later
// views are enqueued or the loop ends (a visit that waits for its view's result frees the slot that view index + depth uses).
// host_clock: add the loop's host time to stream_us, which measures the stream only when the visits wait for the windows (the
// batch path waits for nothing here and times its windows with events, batch_account).  A resident view copies nothing and
// counts no stream time or bytes.
template <class Launch, class Visit>
int for_each_view(vsb_index *ix, int depth, Launch launch, Visit visit, bool host_clock = true) {
    if (!ix->streamed) {
        const View v{0, 0, ix->n, ix->d_vec, 0, 0};
        const int rc = launch(v);
        return rc ? rc : visit(v);
    }
    const auto view_of = [&](long long w) {
        const long long r0 = w * ix->win_rows;
        return View{w, r0, std::min(ix->win_rows, ix->n - r0), ix->d_win[w & 1].get(), (int)(w & 1), (int)(w % depth)};
    };
    const long long W = (ix->n + ix->win_rows - 1) / ix->win_rows;
    const auto t0 = std::chrono::steady_clock::now();
    long long next_visit = 0;
    for (long long w = 0; w < W; ++w) {
        const View v = view_of(w);
        if (w >= 2) CU(cudaStreamWaitEvent(ix->cstream, ix->win_scanned[v.buf], 0));   // the scan of window w-2 has read this buffer
        CU(cudaMemcpyAsync(ix->d_win[v.buf], ix->h_arena + (size_t)v.r0 * ix->pitch, (size_t)v.rows * ix->pitch, cudaMemcpyHostToDevice, ix->cstream));
        CU(cudaEventRecord(ix->win_copied[v.buf], ix->cstream));
        CU(cudaStreamWaitEvent(ix->stream, ix->win_copied[v.buf], 0));
        for (; w - next_visit >= depth; ++next_visit) {                                  // free the slot this window will use
            const int rc = visit(view_of(next_visit));
            if (rc) return rc;
        }
        const int rc = launch(v);
        if (rc) return rc;
        CU(cudaEventRecord(ix->win_scanned[v.buf], ix->stream));
        ix->st_stream_bytes += v.rows * ix->pitch;
    }
    for (; next_visit < W; ++next_visit) {
        const int rc = visit(view_of(next_visit));
        if (rc) return rc;
    }
    if (host_clock) ix->st_stream_us += std::chrono::duration_cast<std::chrono::microseconds>(std::chrono::steady_clock::now() - t0).count();
    return VSB_OK;
}

// the visit of a view loop that waits for nothing: its work stays enqueued, the caller waits for the stream once
int no_visit(const View &) { return VSB_OK; }

// all distances of the column (stream modules, overflow fallback).  The distances of a view sit in half buf of d_dist_all
// (resident: win_rows is 0, the whole buffer); each copy is ordered behind its view's scan on the same stream.
int scan_all_into(vsb_index *ix, int metric, const uint8_t *d_query, std::vector<float> &dist) {
    const int rc = ensure_dist_all(ix);
    if (rc) return rc;
    dist.resize((size_t)ix->n);
    return for_each_view(ix, 2,
        [&](const View &v) {
            Slot *none = nullptr;
            return launch_scan(ix, metric, &d_query, &none, 1, 0, ix->d_dist_all + (size_t)v.buf * ix->win_rows, false, ix->stream, false, v.vec, v.rows, v.r0);
        },
        [&](const View &v) {
            CU(cudaMemcpyAsync(dist.data() + v.r0, ix->d_dist_all + (size_t)v.buf * ix->win_rows, sizeof(float) * (size_t)v.rows, cudaMemcpyDeviceToHost, ix->stream));
            CU(cudaStreamSynchronize(ix->stream));
            return (int)VSB_OK;
        });
}

inline bool row_eligible(const uint32_t *bits, long long row) { return ((bits[row >> 5] >> (row & 31)) & 1u) != 0u; }

// eligible rows among [a, b) of a row bitmap
long long count_bits(const uint32_t *bits, long long a, long long b) {
    long long c = 0;
    for (; a < b && (a & 31); ++a) c += row_eligible(bits, a);
    for (; a + 32 <= b; a += 32) c += __builtin_popcount(bits[a >> 5]);
    for (; a < b; ++a) c += row_eligible(bits, a);
    return c;
}

// the all-distances fallback (candidate overflow): every (eligible) row is a candidate, in scan order
int all_candidates(vsb_index *ix, int metric, const uint8_t *d_query, std::vector<uint2> &cands) {
    ix->st_fallbacks++;
    std::vector<float> dist;
    const int rc = scan_all_into(ix, metric, d_query, dist);
    if (rc) return rc;
    cands.clear();
    cands.reserve((size_t)ix->n);
    for (long long i = 0; i < ix->n; ++i) {
        if (ix->flt_h && !row_eligible(ix->flt_h, i)) continue;
        uint32_t bits;
        memcpy(&bits, &dist[(size_t)i], 4);
        cands.push_back(make_uint2(bits, (uint32_t)i));
    }
    return VSB_OK;
}

// Sets the row filter of one filtered call on ix (host bitmap `bits` over ix->n rows, uploaded once into ix->d_allow); the
// scope's destructor clears it, so that every other entry point sees an unfiltered index
struct FilterScope {
    vsb_index *ix = nullptr;
    FilterScope() = default;
    FilterScope(const FilterScope &) = delete;
    FilterScope &operator=(const FilterScope &) = delete;
    ~FilterScope() {
        if (ix) { ix->flt_h = nullptr; ix->flt_d = nullptr; }
    }
};

int filter_begin(vsb_index *ix, const uint32_t *bits, FilterScope *scope) {
    CU(cudaSetDevice(ix->device));
    const long long words = (ix->n + 31) / 32 + 1;
    const int rc = grow_buf(ix->d_allow, ix->allow_words, words, &ix->dev_bytes);
    if (rc) return rc;
    if (words > 1) CU(cudaMemcpyAsync(ix->d_allow, bits, 4 * (words - 1), cudaMemcpyHostToDevice, ix->stream));
    CU(cudaMemsetAsync(ix->d_allow + (words - 1), 0, 4, ix->stream));
    CU(cudaStreamSynchronize(ix->stream));   // the scans of a group may run on the second scan stream
    ix->flt_h = bits;
    ix->flt_d = ix->d_allow;
    scope->ix = ix;
    return VSB_OK;
}

// calls mark(row) for every row of ix whose rowid is in rowids[0, n); rowids not in the column are skipped
template <class Mark>
void rows_of_rowids(vsb_index *ix, const int64_t *rowids, int64_t n, Mark mark) {
    if (ix->implicit_ids) {                                   // rowid = first_seq + row + 1
        for (int64_t i = 0; i < n; ++i)
            if (rowids[i] > ix->first_seq && rowids[i] - ix->first_seq <= ix->n) mark((long long)(rowids[i] - ix->first_seq - 1));
        return;
    }
    if (ix->rowid_rows != ix->n) {
        ix->rowid_sorted.resize((size_t)ix->n);
        for (long long r = 0; r < ix->n; ++r) ix->rowid_sorted[(size_t)r] = {ix->h_rowids[(size_t)r], r};
        std::sort(ix->rowid_sorted.begin(), ix->rowid_sorted.end());
        ix->rowid_rows = ix->n;
    }
    const auto &s = ix->rowid_sorted;
    for (int64_t i = 0; i < n; ++i)
        for (auto it = std::lower_bound(s.begin(), s.end(), std::make_pair(rowids[i], (long long)INT64_MIN)); it != s.end() && it->first == rowids[i]; ++it)
            mark(it->second);
}

// stages one host query on ix->stream into the slot of the synchronous calls (streamed: slots 0..3 rotate over the windows,
// the query is parked in the last one)
int stage_host_query(vsb_index *ix, const void *query, Slot **slot) {
    CU(cudaSetDevice(ix->device));
    int rc = flush_held(ix);                       // a held query may sit in this slot
    if (rc) return rc;
    rc = ensure_slots(ix);
    if (rc) return rc;
    *slot = &ix->slot[ix->streamed ? kSlots - 1 : 0];
    return stage_query(ix, *slot, query, ix->stream);
}

int large_k_candidates(vsb_index *ix, int metric, const uint8_t *d_query, int k, std::vector<uint2> &cands);

// one query, host in / candidates out (sorted by scan order).  k > kMaxK takes the large-k path (DESIGN §3.11).  Falls back to
// the all-distances kernel when the candidate log overflowed (still GPU-computed distances).
int query_candidates(vsb_index *ix, int metric, const void *query, int k, std::vector<uint2> &cands) {
    Slot *slot = nullptr;
    int rc = stage_host_query(ix, query, &slot);   // synchronous call: one stream (a possible all-distances fallback reads d_query on it)
    if (rc) return rc;
    if (k > kMaxK) return large_k_candidates(ix, metric, slot->d_query, k, cands);
    cands.clear();
    cands.reserve(kFirstFetch);                    // one allocation for the usual few hundred survivors
    bool overflow = false;
    rc = ensure_workspace(ix, k);
    if (rc) return rc;
    // every view's survivors in scan order, rows made column-global; a streamed index rotates result slots 0..3 over its windows
    rc = for_each_view(ix, ix->streamed ? 4 : 1,
        [&](const View &v) {
            const uint8_t *q = slot->d_query;
            Slot *vs = &ix->slot[v.slot];
            return launch_scan(ix, metric, &q, &vs, 1, k, nullptr, true, ix->stream, false, v.vec, v.rows, v.r0);
        },
        [&](const View &v) {
            bool ovf = false;
            const int r = visit_survivors(ix, &ix->slot[v.slot], &ovf, [&](uint2 c) { cands.push_back(make_uint2(c.x, c.y + (uint32_t)v.r0)); });
            if (ovf) overflow = true;
            return r;
        });
    if (rc) return rc;
    return overflow ? all_candidates(ix, metric, slot->d_query, cands) : VSB_OK;
}

// launches the held pass (vsb_scan_submit), if any
int flush_held(vsb_index *ix) {
    if (ix->held.nq == 0) return VSB_OK;
    const HeldPass h = ix->held;
    ix->held.nq = 0;
    CU(cudaSetDevice(ix->device));
    Slot *slots[kMaxPass];
    for (int j = 0; j < h.nq; ++j) slots[j] = &ix->slot[h.slot[j]];
    const int rc = ensure_workspace(ix, h.k, h.nq);
    return rc ? rc : launch_scan(ix, h.metric, h.query, slots, h.nq, h.k, nullptr, true, h.ss);
}

// every entry point on an index but vsb_scan_submit and vsb_collect: launches the held pass first, so that no other call
// waits behind a query the caller has already submitted
int check_index(vsb_index *ix) {
    if (!ix) return fail(VSB_EINVAL, "null index");
    return flush_held(ix);
}

// what launch_scan would reject, checked before a submission stages, holds or launches anything.  A device query is read as
// 16-byte vectors over its pitch: query j of a group at queries + j * query_stride must be 16-byte aligned and hold the
// zero-padded pitch bytes before the next query begins.
int check_submission(const vsb_index *ix, int metric, const void *queries, int64_t query_stride, int nq, int query_on_device, int k) {
    int root = 0;
    if (!queries || k <= 0 || k > kMaxK) return fail(VSB_EINVAL, "bad scan arguments (k must be 1..%d)", kMaxK);
    if (metric_class(metric, &root) < 0) return fail(VSB_EINVAL, "unknown distance metric %d", metric);
    if (!query_on_device) return VSB_OK;
    if ((uintptr_t)queries % 16 != 0) return fail(VSB_EINVAL, "device queries must be 16-byte aligned");
    if (nq > 1 && (query_stride % 16 != 0 || query_stride < ix->pitch))
        return fail(VSB_EINVAL, "device query stride %lld: a multiple of 16 and at least the pitch (%d) expected", (long long)query_stride, ix->pitch);
    return VSB_OK;
}

// one pass of the column per pass_max queries of a group of independent queries (query j at queries + j * query_stride; slots
// first_slot ..).  push: the heads are labelled for the exchange targets (peer memory), see exchange.inc
int submit_group(vsb_index *ix, int metric, const void *queries, int64_t query_stride, int nq, int query_on_device, int k, int fetch,
                 int first_slot, bool push) {
    if (check_index(ix)) return VSB_EINVAL;
    if (nq <= 0 || first_slot < 0 || first_slot + nq > kSlots) return fail(VSB_EINVAL, "bad slot group [%d, %d)", first_slot, first_slot + nq);
    int rc = check_submission(ix, metric, queries, query_stride, nq, query_on_device, k);
    if (rc) return rc;
    CU(cudaSetDevice(ix->device));
    rc = ensure_slots(ix);
    if (rc) return rc;
    const int width = std::min(nq, pass_max(ix, (k + 31) & ~31));
    rc = ensure_workspace(ix, k, width);
    if (rc) return rc;
    for (int j0 = 0; j0 < nq; j0 += width) {
        const int m = std::min(width, nq - j0);
        cudaStream_t ss = next_scan_stream(ix);
        const uint8_t *q[kMaxPass];
        Slot *slots[kMaxPass];
        for (int j = 0; j < m; ++j) {
            Slot *slot = slots[j] = &ix->slot[first_slot + j0 + j];
            ix->uncollected &= ~(1u << (first_slot + j0 + j));     // a query left in this slot is given up
            q[j] = (const uint8_t *)queries + (size_t)(j0 + j) * (size_t)query_stride;
            if (!query_on_device) {
                if (slot->seq > 0) CU(cudaEventSynchronize(slot->done));   // the slot's pinned staging buffer is free again
                rc = stage_query(ix, slot, q[j], ss);
                if (rc) return rc;
                q[j] = slot->d_query;
            }
        }
        rc = launch_scan(ix, metric, q, slots, m, k, nullptr, fetch != 0, ss, push);
        if (rc) return rc;
        ix->last_slot = first_slot + j0 + m - 1;
        ix->last_metric = metric;
    }
    return VSB_OK;
}

// ------------------------------------------------------------------ range search (vsb_scan_range, DESIGN §3.10)
constexpr long long kRangeCap0 = 1 << 16;   // pairs of the first pass of a range query (512 KB); a larger result takes a second pass

// the float threshold of a double radius: the smallest float t with (double)t >= r, so that for every float d, d < t iff
// (double)d < r (the comparison `distance < r` of SQL over the float widened to double).  NaN: no float qualifies (-INF).
float range_threshold(double r) {
    if (r != r) return -INFINITY;
    float t = (float)r;
    if ((double)t < r) t = std::nextafter(t, INFINITY);
    return t;
}

// the pair list holds at least cap pairs (grow_buf)
int pair_list_reserve(vsb_index *ix, long long cap) {
    PairList &pl = ix->plist;
    if (!pl.d_count) {
        DeviceBuf<unsigned> d;
        HostBuf<unsigned> h;
        CU(d.alloc(sizeof(unsigned)));
        CU(h.alloc(sizeof(unsigned)));
        pl.d_count = std::move(d);
        pl.h_count = std::move(h);
        ix->dev_bytes += sizeof(unsigned);
    }
    return grow_buf(pl.d_pairs, pl.cap, cap, &ix->dev_bytes);
}

int pair_list_reset(vsb_index *ix) {
    CU(cudaMemsetAsync(ix->plist.d_count, 0, sizeof(unsigned), ix->stream));
    return VSB_OK;
}

// One query into the pair list, which first grows to first_cap pairs: the counter is reset, fill() appends on ix->stream and the
// count comes back in *count.  A count above the list's capacity grows the list to exactly that count, adds one to *regrows
// and calls refill() once, which writes the list again (resetting the counter itself if it appends everything again).  A count
// that still does not fit is an error; `what` names the caller in its message.
template <class Fill, class Refill>
int pair_list_run(vsb_index *ix, long long first_cap, const char *what, long long *regrows, Fill fill, Refill refill, long long *count) {
    PairList &pl = ix->plist;
    const auto read_count = [&]() -> int {
        CU(cudaMemcpyAsync(pl.h_count, pl.d_count, sizeof(unsigned), cudaMemcpyDeviceToHost, ix->stream));
        CU(cudaStreamSynchronize(ix->stream));
        *count = *pl.h_count;
        return VSB_OK;
    };
    int rc = pair_list_reserve(ix, first_cap);
    if (rc == VSB_OK) rc = pair_list_reset(ix);
    if (rc == VSB_OK) rc = fill();
    if (rc == VSB_OK) rc = read_count();
    if (rc || *count <= pl.cap) return rc;
    ++*regrows;
    rc = pair_list_reserve(ix, *count);
    if (rc == VSB_OK) rc = refill();
    if (rc == VSB_OK) rc = read_count();
    if (rc == VSB_OK && *count > pl.cap) return fail(VSB_ECUDA, "%s: %lld pairs after growing the list to %lld", what, *count, pl.cap);
    return rc;
}

// one range-mode scan over rows [0, n) of vec, whose first row is shard row r0, appending to the pair list on ix->stream
int launch_range(vsb_index *ix, int metric, const uint8_t *d_query, float t, const uint8_t *vec, long long n, long long r0) {
    int root = 0;
    const int mc = metric_class(metric, &root);
    if (mc < 0) return fail(VSB_EINVAL, "unknown distance metric %d", metric);
    const Plan pl = make_plan(ix, 0);
    ScanFn fn = pick_kernel(ix->vtype, mc, pl.direct, true);
    if (!fn) return fail(VSB_EINVAL, "unsupported vector type %d", ix->vtype);
    CU((cudaError_t)set_smem_limit((const void *)fn, pl.smem));
    ScanParams p = scan_params(ix, pl, root, d_query, vec, n, r0);
    p.range_t = t;
    p.range_pairs = ix->plist.d_pairs;
    p.range_count = ix->plist.d_count;
    p.range_cap = ix->plist.cap;
    p.range_row_base = (unsigned)r0;
    fn<<<ix->num_sms, kThreads, pl.smem, ix->stream>>>(p);
    CU(cudaGetLastError());
    ++g_launches;
    note_plan(ix, pl);
    return VSB_OK;
}

// the float order of distance bits as an unsigned order (fkey of scan_kernels.cuh, on the host)
inline uint32_t dist_order_key(uint32_t bits) { return (bits & 0x80000000u) ? ~bits : (bits | 0x80000000u); }

// orders `count` pairs (row, distance bits) by (distance, row) on the host: the lists longer than range_sort_kernel takes
void range_sort_host(uint2 *pairs, size_t count) {
    std::sort(pairs, pairs + count, [](const uint2 &a, const uint2 &b) {
        const uint32_t ka = dist_order_key(a.y), kb = dist_order_key(b.y);
        return ka != kb ? ka < kb : a.x < b.x;
    });
}

// one query staged at d_query: every eligible row of ix with distance < r, as (shard row, distance bits) ordered by (distance,
// row).  The first pass appends into kRangeCap0 pairs; when the counter says more, the list grows to the exact count and the
// scan runs once more.  A streamed index scans window by window into the same list.
int range_query(vsb_index *ix, int metric, const uint8_t *d_query, double r, std::vector<uint2> &out) {
    out.clear();
    const float t = range_threshold(r);
    if (ix->n == 0 || t == -INFINITY) return VSB_OK;            // nothing is below -INF (and NaN radii select nothing)
    const auto scan = [&]() {
        return for_each_view(ix, 2, [&](const View &v) { return launch_range(ix, metric, d_query, t, v.vec, v.rows, v.r0); }, no_visit);
    };
    long long cnt = 0;
    const int rc = pair_list_run(ix, kRangeCap0, "range scan", &ix->st_range_passes, scan,
        [&]() {
            const int r = pair_list_reset(ix);
            return r ? r : scan();
        }, &cnt);
    if (rc) return rc;
    if (cnt >= 2 && cnt <= kRangeSortCap) {
        size_t n2 = 2;
        while (n2 < cnt) n2 <<= 1;
        const size_t smem = sizeof(unsigned long long) * n2;
        CU((cudaError_t)set_smem_limit((const void *)range_sort_kernel, smem));
        RangeSortParams sp{ix->plist.d_pairs, ix->plist.d_count, 0, nullptr, nullptr};
        range_sort_kernel<<<1, kRangeSortThreads, smem, ix->stream>>>(sp);
        CU(cudaGetLastError());
        ++g_launches;
    }
    out.resize((size_t)cnt);
    if (cnt > 0) CU(cudaMemcpyAsync(out.data(), ix->plist.d_pairs, sizeof(uint2) * (size_t)cnt, cudaMemcpyDeviceToHost, ix->stream));
    CU(cudaStreamSynchronize(ix->stream));
    if (cnt > kRangeSortCap) {
        ix->st_range_host_sorts++;
        range_sort_host(out.data(), out.size());
    }
    ix->st_range_pairs += cnt;
    return VSB_OK;
}

// checks the arguments of a range call and allocates its result
int range_begin(int metric, const void *queries, int nq, const double *radius, vsb_range **out) {
    if (!out) return fail(VSB_EINVAL, "out is null");
    *out = nullptr;
    if (nq < 0 || (nq > 0 && (!queries || !radius))) return fail(VSB_EINVAL, "bad range arguments");
    int root = 0;
    if (metric_class(metric, &root) < 0) return fail(VSB_EINVAL, "unknown distance metric %d", metric);
    vsb_range *r = new (std::nothrow) vsb_range();
    if (!r) return fail(VSB_ENOMEM, "out of host memory");
    r->ids.resize((size_t)nq);
    r->dist.resize((size_t)nq);
    *out = r;
    return VSB_OK;
}

// query q's n result rows into r: at(i) -> (rowid, distance bits) of row i in result order
template <class At>
void range_put(vsb_range *r, int q, size_t n, At at) {
    r->ids[(size_t)q].resize(n);
    r->dist[(size_t)q].resize(n);
    for (size_t i = 0; i < n; ++i) {
        const std::pair<int64_t, uint32_t> e = at(i);
        float d;
        memcpy(&d, &e.second, 4);
        r->ids[(size_t)q][i] = e.first;
        r->dist[(size_t)q][i] = (double)d;
    }
}

// ------------------------------------------------------------------ large k (k > kMaxK, DESIGN §3.11)
constexpr size_t kLkHistBytes = sizeof(unsigned) * kLkPasses * kLkMaxSeg * 256;

// the select's histograms and state, and the compaction's offsets for views of up to `rows` rows (grown, never shrunk;
// large-k calls are synchronous, no launch reads the old buffers)
int ensure_large_k(vsb_index *ix, long long rows) {
    if (!ix->d_lk_state) {
        DeviceBuf<unsigned> hist;
        DeviceBuf<LkState> st;
        CU(hist.alloc(kLkHistBytes));
        CU(st.alloc(sizeof(LkState)));
        CU(cudaMemset(st, 0, sizeof(LkState)));
        ix->d_lk_hist = std::move(hist);
        ix->d_lk_state = std::move(st);
        ix->dev_bytes += kLkHistBytes + sizeof(LkState);
    }
    const long long blocks = std::max<long long>(1, (rows + kLkRows - 1) / kLkRows);
    return grow_buf(ix->d_lk_boff, ix->lk_boff_cap, blocks, &ix->dev_bytes);
}

// the candidates of one view (its n distances at dist, its first row shard row r0) appended to the pair list on ix->stream:
// segment ends k, 2k, 4k, ... below n, then n; the prefix bounds digit by digit; the ordered compaction.  write_only: only
// the compaction's write, again (the list grew to the count the offsets kernel left)
int large_k_view(vsb_index *ix, const float *dist, long long n, long long r0, int k, bool write_only = false) {
    if (n <= 0) return VSB_OK;
    LkParams p{};
    p.dist = dist;
    p.n = n;
    p.k = k;
    for (long long e = k; e < n && p.nseg < kLkMaxSeg - 1; e *= 2) p.ends[p.nseg++] = e;
    p.ends[p.nseg++] = n;
    p.allow = ix->flt_d;
    p.allow_base = r0;
    p.hist = ix->d_lk_hist;
    p.st = ix->d_lk_state;
    p.boff = ix->d_lk_boff;
    p.total = ix->plist.d_count;
    p.out = ix->plist.d_pairs;
    p.cap = ix->plist.cap;
    p.row_base = (unsigned)r0;
    p.nblocks = (int)((n + kLkRows - 1) / kLkRows);
    if (!write_only) {
        const int prefixes = p.nseg - 1;
        if (prefixes > 0) CU(cudaMemsetAsync(ix->d_lk_hist, 0, kLkHistBytes, ix->stream));
        for (p.pass = 0; p.pass < kLkPasses; ++p.pass) {
            if (prefixes > 0) {
                lk_hist_kernel<<<(unsigned)((p.ends[prefixes - 1] + kLkRows - 1) / kLkRows), kLkThreads, 0, ix->stream>>>(p);
                CU(cudaGetLastError());
                ++g_launches;
            }
            lk_select_kernel<<<1, kLkMaxSeg * 32, 0, ix->stream>>>(p);   // the last digit also records the segments and bounds
            CU(cudaGetLastError());
            ++g_launches;
        }
        lk_count_kernel<<<p.nblocks, kLkThreads, 0, ix->stream>>>(p);
        CU(cudaGetLastError());
        lk_offsets_kernel<<<1, kLkScanThreads, 0, ix->stream>>>(p);
        CU(cudaGetLastError());
        g_launches += 2;
    }
    lk_write_kernel<<<p.nblocks, kLkThreads, 0, ix->stream>>>(p);
    CU(cudaGetLastError());
    ++g_launches;
    return VSB_OK;
}

// the candidates of one query with k > kMaxK staged at d_query: the all-distances scan, then the bounds and the compaction of
// each view on the device (the resident column, or every window behind its scan), (distance bits, shard row) in scan order.  The
// first pair list holds kRangeCap0 pairs or twice what rows in random order give; a larger count grows the list to the exact
// count and, resident, writes again from the distances still in HBM, streamed, runs the windows once more.
int large_k_candidates(vsb_index *ix, int metric, const uint8_t *d_query, int k, std::vector<uint2> &cands) {
    cands.clear();
    ix->st_large_k_queries++;
    if (ix->n == 0) return VSB_OK;
    const long long view = ix->streamed ? std::min(ix->win_rows, ix->n) : ix->n, views = (ix->n + view - 1) / view;
    const long long expect = views * k * (2 + (long long)std::log2(std::max(1.0, (double)view / k)));
    int rc = ensure_dist_all(ix);
    if (rc == VSB_OK) rc = ensure_large_k(ix, view);
    if (rc) return rc;
    // the distances of a view sit in half buf of d_dist_all (resident: win_rows is 0, the whole buffer)
    const auto scan = [&]() {
        return for_each_view(ix, 2,
            [&](const View &v) {
                float *dist = ix->d_dist_all + (size_t)v.buf * ix->win_rows;
                Slot *none = nullptr;
                const int r = launch_scan(ix, metric, &d_query, &none, 1, 0, dist, false, ix->stream, false, v.vec, v.rows, v.r0);
                return r ? r : large_k_view(ix, dist, v.rows, v.r0, k);
            },
            no_visit);
    };
    long long cnt = 0;
    rc = pair_list_run(ix, std::max(kRangeCap0, std::min(ix->n, 2 * expect)), "large-k candidates", &ix->st_large_k_regrows, scan,
        [&]() {
            // a resident column's distances are still in HBM: only the compaction's write runs again.  A streamed column's
            // windows have been overwritten and run again.
            if (!ix->streamed) return large_k_view(ix, ix->d_dist_all, ix->n, 0, k, true);
            const int r = pair_list_reset(ix);
            return r ? r : scan();
        }, &cnt);
    if (rc == VSB_OK) rc = grow_buf(ix->plist.h_pairs, ix->plist.h_cap, cnt, nullptr);
    if (rc) return rc;
    if (cnt > 0) CU(cudaMemcpyAsync(ix->plist.h_pairs, ix->plist.d_pairs, sizeof(uint2) * (size_t)cnt, cudaMemcpyDeviceToHost, ix->stream));
    CU(cudaStreamSynchronize(ix->stream));
    cands.assign(ix->plist.h_pairs.get(), ix->plist.h_pairs.get() + cnt);
    ix->st_large_k_cands += cnt;
    return VSB_OK;
}

}  // namespace

#include "batch_host.inc"
#include "exchange.inc"
#include "column.inc"
#include "quantize.inc"

// ====================================================================== C ABI
extern "C" {

int vsb_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
    return n;
}

const char *vsb_last_error(void) { return g_err.c_str(); }

const char *vsb_backend_name(void) {
    static std::once_flag once;
    static char name[160];
    std::call_once(once, [] {
        int n = vsb_device_count();
        if (n <= 0) { snprintf(name, sizeof name, "CUDA sm_90a (no device)"); return; }
        cudaDeviceProp pr{};
        cudaGetDeviceProperties(&pr, 0);
        snprintf(name, sizeof name, "CUDA sm_90a (%s x%d, cc %d.%d)", pr.name, n, pr.major, pr.minor);
    });
    return name;
}

int64_t vsb_kernel_launches(void) { return g_launches.load(); }

int64_t vsb_debug_live_handles(void) { return g_live_handles.load(); }

int vsb_set_option(const char *name, int value) {
    int *p = nullptr;
    if (!strcmp(name, "stage_bytes")) p = &g_opt_stage_bytes;
    else if (!strcmp(name, "direct")) p = &g_opt_direct;
    else if (!strcmp(name, "ring_bytes")) p = &g_opt_ring_bytes;
    else if (!strcmp(name, "time_kernels")) p = &g_opt_time_kernels;
    else if (!strcmp(name, "no_batch")) p = &g_opt_no_batch;
    else if (!strcmp(name, "epi_chunk")) p = &g_opt_epi_chunk;
    else if (!strcmp(name, "balance")) p = &g_opt_balance;
    else if (!strcmp(name, "batch_m0")) p = &g_opt_batch_m0;
    else if (!strcmp(name, "batch_growth")) p = &g_opt_batch_growth;
    else if (!strcmp(name, "batch_debug")) p = &g_opt_batch_debug;
    else if (!strcmp(name, "scan_streams")) p = &g_opt_scan_streams;
    else if (!strcmp(name, "xwait_ms")) p = &g_opt_xwait_ms;
    else if (!strcmp(name, "f32_batch")) p = &g_opt_f32_batch;
    else if (!strcmp(name, "sets_mem_mb")) p = &g_opt_sets_mem_mb;
    if (!p) return fail(VSB_EINVAL, "unknown option %s", name);
    if (value < 0) return fail(VSB_EINVAL, "option %s: values are non-negative", name);   // so that a negative return is always an error
    int old = *p;
    *p = value;
    return old;
}

static int index_create(vsb_index **out, int device, int vtype, int dim, int64_t capacity_rows, int64_t first_seq, int64_t window_rows);

int vsb_index_create(vsb_index **out, int device, int vtype, int dim, int64_t capacity_rows, int64_t first_seq) {
    return index_create(out, device, vtype, dim, capacity_rows, first_seq, 0);
}

int vsb_index_create_streamed(vsb_index **out, int device, int vtype, int dim, int64_t capacity_rows, int64_t first_seq, int64_t window_rows) {
    if (window_rows <= 0) return fail(VSB_EINVAL, "window_rows must be positive");
    return index_create(out, device, vtype, dim, capacity_rows, first_seq, window_rows);
}

int vsb_index_is_streamed(const vsb_index *ix) { return ix && ix->streamed ? 1 : 0; }

static int index_create(vsb_index **out, int device, int vtype, int dim, int64_t capacity_rows, int64_t first_seq, int64_t window_rows) {
    if (!out) return fail(VSB_EINVAL, "out is null");
    *out = nullptr;
    const int es = elem_size(vtype);
    if (!es) return fail(VSB_EINVAL, "unknown vector type %d", vtype);
    if (dim <= 0) return fail(VSB_EINVAL, "dimension must be positive");
    if (capacity_rows < 0 || capacity_rows > 0xFFFFFFF0ll) return fail(VSB_EINVAL, "capacity_rows out of range");
    int ndev = vsb_device_count();
    if (ndev <= 0) return fail(VSB_ENODEV, "no CUDA device available (this build has no CPU fallback)");
    if (device < 0 || device >= ndev) return fail(VSB_EINVAL, "device %d out of range (have %d)", device, ndev);
    CU(cudaSetDevice(device));
    cudaDeviceProp pr{};
    CU(cudaGetDeviceProperties(&pr, device));
    if (pr.major != 9 || pr.minor != 0)   // sm_90a code (wgmma, TMA) runs on compute capability 9.0 only
        return fail(VSB_ENODEV, "device %s (cc %d.%d): this build holds sm_90a (H100) code only", pr.name, pr.major, pr.minor);
    std::unique_ptr<vsb_index> ix(new (std::nothrow) vsb_index());
    if (!ix) return fail(VSB_ENOMEM, "out of host memory");
    ix->device = device; ix->vtype = vtype; ix->dim = dim; ix->esize = es;
    ix->pitch = (dim * es + 15) & ~15;
    ix->cap = capacity_rows; ix->first_seq = first_seq;
    ix->num_sms = pr.multiProcessorCount;
    ix->max_smem = (int)pr.sharedMemPerBlockOptin;
    cudaError_t e = ix->stream.create();
    if (e == cudaSuccess) e = ix->stream2.create();
    if (e == cudaSuccess) e = ix->fstream.create();
    if (e == cudaSuccess) e = ix->xstream.create();
    if (e != cudaSuccess) return fail(VSB_ECUDA, "cudaStreamCreate: %s", cudaGetErrorString(e));
    size_t bytes = (size_t)std::max<long long>(capacity_rows, 1) * ix->pitch + 1024;
    if (window_rows > 0) {
        // streamed: the column stays in pinned host memory, two windows on the device
        ix->streamed = true;
        ix->win_rows = std::min<long long>(std::max<long long>(window_rows, 32), std::max<long long>(capacity_rows, 32));
        e = ix->h_arena.alloc(bytes);
        const size_t wb = (size_t)ix->win_rows * ix->pitch + 1024;
        for (int b = 0; b < 2 && e == cudaSuccess; ++b) {
            e = ix->d_win[b].alloc(wb);
            if (e == cudaSuccess) e = ix->win_copied[b].create(cudaEventDisableTiming);
            if (e == cudaSuccess) e = ix->win_scanned[b].create(cudaEventDisableTiming);
        }
        if (e == cudaSuccess) e = ix->cstream.create();
        bytes = 2 * wb;
    } else {
        e = ix->d_vec.alloc(bytes);
    }
    if (e != cudaSuccess) {
        cudaGetLastError();
        return fail(VSB_ENOMEM, "allocating %zu bytes for the %s column failed: %s", bytes, window_rows > 0 ? "streamed" : "resident", cudaGetErrorString(e));
    }
    ix->dev_bytes = bytes;
    *out = ix.release();
    return VSB_OK;
}

static int stage_acquire(vsb_index *ix, int *which) {
    const int b = ix->stage_next;
    if (!ix->stage[b]) {
        HostBuf<uint8_t> buf;
        Event ev;
        CU(buf.alloc(kStageBuf));
        CU(ev.create(cudaEventDisableTiming));
        ix->stage[b] = std::move(buf);
        ix->stage_ev[b] = std::move(ev);
    } else {
        CU(cudaEventSynchronize(ix->stage_ev[b]));  // previous copy out of this buffer finished
    }
    ix->stage_next ^= 1;
    *which = b;
    return VSB_OK;
}

// explicit rowids from now on: the implicit ids of the rows appended so far become a list
static void materialise_rowids(vsb_index *ix) {
    if (!ix->implicit_ids) return;
    ix->h_rowids.resize((size_t)ix->n);
    for (long long i = 0; i < ix->n; ++i) ix->h_rowids[(size_t)i] = ix->first_seq + i + 1;
    ix->implicit_ids = false;
}

// the little-endian int64 rowid in front of a preloaded vector (INT64_FROM_INT8PTR, :86-94)
static int64_t inline_rowid(const uint8_t *row) {
    uint64_t v = 0;
    for (int i = 7; i >= 0; --i) v = (v << 8) | row[i];
    return (int64_t)v;
}

// src_stride: bytes between rows in host memory; src_off: offset of the vector inside a row
static int append_rows(vsb_index *ix, const uint8_t *src, size_t src_stride, size_t src_off, const int64_t *rowids,
                       bool ids_inline, int64_t nrows) {
    if (nrows < 0) return fail(VSB_EINVAL, "negative row count");
    if (ix->n + nrows > ix->cap) return fail(VSB_ERANGE, "index capacity exceeded (%lld + %lld > %lld)", ix->n, (long long)nrows, ix->cap);
    CU(cudaSetDevice(ix->device));
    const size_t rowbytes = (size_t)ix->dim * ix->esize;
    const size_t pitch = (size_t)ix->pitch;
    if (ids_inline || rowids != nullptr) materialise_rowids(ix);
    if (pitch > kStageBuf) return fail(VSB_ERANGE, "row pitch %zu exceeds the %zu-byte staging buffer", pitch, (size_t)kStageBuf);
    const int64_t per_buf = (int64_t)(kStageBuf / pitch);
    int64_t done = 0;
    if (ix->streamed) {                      // the pinned arena IS the staging area
        for (int64_t r = 0; r < nrows; ++r) {
            const uint8_t *row = src + (size_t)r * src_stride;
            uint8_t *dst = ix->h_arena + (size_t)(ix->n + r) * pitch;
            memcpy(dst, row + src_off, rowbytes);
            if (pitch > rowbytes) memset(dst + rowbytes, 0, pitch - rowbytes);
            if (ids_inline) ix->h_rowids.push_back(inline_rowid(row));
        }
        done = nrows;
    }
    while (done < nrows) {
        const int64_t m = std::min<int64_t>(per_buf, nrows - done);
        int b;
        int rc = stage_acquire(ix, &b);
        if (rc) return rc;
        uint8_t *dst = ix->stage[b];
        for (int64_t r = 0; r < m; ++r) {
            const uint8_t *row = src + (size_t)(done + r) * src_stride;
            memcpy(dst + (size_t)r * pitch, row + src_off, rowbytes);
            if (pitch > rowbytes) memset(dst + (size_t)r * pitch + rowbytes, 0, pitch - rowbytes);
            if (ids_inline) ix->h_rowids.push_back(inline_rowid(row));
        }
        CU(cudaMemcpyAsync(ix->d_vec + (size_t)(ix->n + done) * pitch, dst, (size_t)m * pitch, cudaMemcpyHostToDevice, ix->stream));
        CU(cudaEventRecord(ix->stage_ev[b], ix->stream));
        done += m;
    }
    if (!ids_inline) {
        if (rowids) ix->h_rowids.insert(ix->h_rowids.end(), rowids, rowids + nrows);
        else if (!ix->implicit_ids)
            for (int64_t r = 0; r < nrows; ++r) ix->h_rowids.push_back(ix->first_seq + ix->n + r + 1);
    }
    ix->n += nrows;
    return VSB_OK;
}

int vsb_index_append_dense(vsb_index *ix, const void *vectors, const int64_t *rowids, int64_t nrows) {
    if (check_index(ix)) return VSB_EINVAL;
    if (!vectors && nrows > 0) return fail(VSB_EINVAL, "vectors is null");
    return append_rows(ix, (const uint8_t *)vectors, (size_t)ix->dim * ix->esize, 0, rowids, false, nrows);
}

int vsb_index_append_quant_chunk(vsb_index *ix, const void *chunk, int64_t nrows) {
    if (check_index(ix)) return VSB_EINVAL;
    if (ix->esize != 1) return fail(VSB_EINVAL, "quantized chunks need a UINT8/INT8 index");
    if (!chunk && nrows > 0) return fail(VSB_EINVAL, "chunk is null");
    return append_rows(ix, (const uint8_t *)chunk, (size_t)ix->dim + 8, 8, nullptr, true, nrows);
}

int vsb_index_append_device(vsb_index *ix, const void *d_vectors, const int64_t *d_rowids, int64_t nrows) {
    if (check_index(ix)) return VSB_EINVAL;
    if (nrows < 0 || ix->n + nrows > ix->cap) return fail(VSB_ERANGE, "index capacity exceeded");
    if (ix->streamed) return fail(VSB_EINVAL, "a streamed index takes host rows (vsb_index_append_dense / _quant_chunk)");
    CU(cudaSetDevice(ix->device));
    const size_t rowbytes = (size_t)ix->dim * ix->esize;
    if ((size_t)ix->pitch != rowbytes)
        CU(cudaMemsetAsync(ix->d_vec + (size_t)ix->n * ix->pitch, 0, (size_t)nrows * ix->pitch, ix->stream));
    CU(cudaMemcpy2DAsync(ix->d_vec + (size_t)ix->n * ix->pitch, (size_t)ix->pitch, d_vectors, rowbytes, rowbytes, (size_t)nrows,
                         cudaMemcpyDeviceToDevice, ix->stream));
    if (d_rowids) {
        materialise_rowids(ix);
        ix->h_rowids.resize((size_t)(ix->n + nrows));
        CU(cudaMemcpyAsync(ix->h_rowids.data() + ix->n, d_rowids, sizeof(int64_t) * (size_t)nrows, cudaMemcpyDeviceToHost, ix->stream));
    } else if (!ix->implicit_ids) {
        for (int64_t r = 0; r < nrows; ++r) ix->h_rowids.push_back(ix->first_seq + ix->n + r + 1);
    }
    CU(cudaStreamSynchronize(ix->stream));
    ix->n += nrows;
    return VSB_OK;
}

int vsb_index_finalize(vsb_index *ix) {
    if (check_index(ix)) return VSB_EINVAL;
    CU(cudaSetDevice(ix->device));
    CU(cudaStreamSynchronize(ix->stream));
    for (int b = 0; b < 2; ++b) {  // the staging buffers are only needed while loading
        ix->stage[b].reset();
        ix->stage_ev[b].reset();
    }
    return VSB_OK;
}

int64_t vsb_index_rows(const vsb_index *ix) { return ix ? ix->n : 0; }
int64_t vsb_index_device_bytes(const vsb_index *ix) { return ix ? (int64_t)ix->dev_bytes : 0; }
int vsb_index_query_pitch(const vsb_index *ix) { return ix ? ix->pitch : 0; }
int64_t vsb_index_stat(const vsb_index *ix, const char *name) {
    if (!ix || !name) return -1;
    if (!strcmp(name, "queries")) return ix->st_queries;
    if (!strcmp(name, "survivors")) return ix->st_survivors;
    if (!strcmp(name, "last_survivors")) return ix->st_last_survivors;
    if (!strcmp(name, "fallbacks")) return ix->st_fallbacks;
    if (!strcmp(name, "batches")) return ix->st_batches;
    if (!strcmp(name, "batch_cands")) return ix->st_batch_cands;
    if (!strcmp(name, "batch_kept")) return ix->st_batch_kept;
    if (!strcmp(name, "tc_us")) return ix->st_tc_us;
    if (!strcmp(name, "batch_us")) return ix->st_batch_us;
    if (!strcmp(name, "tc_rows")) return ix->st_tc_rows;
    if (!strcmp(name, "stream_bytes")) return ix->st_stream_bytes;
    if (!strcmp(name, "stream_us")) return ix->st_stream_us;
    if (!strcmp(name, "fetch_bytes")) return (long long)kHeadBytes;
    if (!strcmp(name, "slots")) return kSlots;
    if (!strcmp(name, "filter_blocks")) return (ix->num_sms * kWarps + kFilterWarpsFast - 1) / kFilterWarpsFast;
    if (!strcmp(name, "sms")) return ix->num_sms;
    if (!strcmp(name, "plan_log2p")) return ix->last_log2p;
    if (!strcmp(name, "plan_pass_max")) return pass_max(ix, ix->last_kcap > 0 ? ix->last_kcap : 32);   // for the k of the last top-k pass
    if (!strcmp(name, "scan_passes")) return ix->st_scan_passes;
    if (!strcmp(name, "pass_queries")) return ix->st_pass_queries;
    if (!strcmp(name, "plan_nsw")) return ix->last_nsw;
    if (!strcmp(name, "plan_direct")) return ix->last_direct;
    if (!strcmp(name, "range_pairs")) return ix->st_range_pairs;
    if (!strcmp(name, "range_passes")) return ix->st_range_passes;
    if (!strcmp(name, "range_host_sorts")) return ix->st_range_host_sorts;
    if (!strcmp(name, "range_batches")) return ix->st_range_batches;
    if (!strcmp(name, "range_batch_fallbacks")) return ix->st_range_batch_fallbacks;
    if (!strcmp(name, "range_query_fallbacks")) return ix->st_range_query_fallbacks;
    if (!strcmp(name, "large_k_queries")) return ix->st_large_k_queries;
    if (!strcmp(name, "large_k_cands")) return ix->st_large_k_cands;
    if (!strcmp(name, "large_k_regrows")) return ix->st_large_k_regrows;
    if (!strcmp(name, "large_k_batches")) return ix->st_large_k_batches;
    if (!strcmp(name, "large_k_batch_fallbacks")) return ix->st_large_k_batch_fallbacks;
    if (!strcmp(name, "large_k_query_fallbacks")) return ix->st_large_k_query_fallbacks;
    if (!strcmp(name, "large_k_levels_us")) return ix->st_large_k_levels_us;
    if (!strcmp(name, "large_k_replay_us")) return ix->st_large_k_replay_us;
    if (!strcmp(name, "large_k_replay_threads")) return ix->st_large_k_replay_threads;
    if (!strcmp(name, "rows_queries")) return ix->st_rows_queries;
    if (!strcmp(name, "rows_pairs")) return ix->st_rows_pairs;
    if (!strcmp(name, "rows_host_bytes")) return ix->st_rows_host_bytes;
    if (!strcmp(name, "grouped_queries")) return ix->st_grouped_queries;
    if (!strcmp(name, "grouped_pairs")) return ix->st_grouped_pairs;
    if (!strcmp(name, "grouped_cands")) return ix->st_grouped_cands;
    if (!strcmp(name, "grouped_keys_replayed")) return ix->st_grouped_keys_replayed;
    if (!strcmp(name, "grouped_regrows")) return ix->st_grouped_regrows;
    if (!strcmp(name, "grouped_layout_us")) return ix->st_grouped_layout_us;
    if (!strcmp(name, "grouped_layout_reuses")) return ix->st_grouped_layout_reuses;
    if (!strcmp(name, "grouped_scan_us")) return ix->st_grouped_scan_us;
    if (!strcmp(name, "grouped_walk_us")) return ix->st_grouped_walk_us;
    if (!strcmp(name, "grouped_replay_us")) return ix->st_grouped_replay_us;
    if (!strcmp(name, "sets_batches")) return ix->st_sets_batches;
    if (!strcmp(name, "sets_fallbacks")) return ix->st_sets_fallbacks;
    if (!strcmp(name, "sets_levels")) return ix->st_sets_levels;
    if (!strcmp(name, "sets_plan_us")) return ix->st_sets_plan_us;
    return -1;
}
void *vsb_index_stream(vsb_index *ix) { return ix ? (void *)ix->fstream : nullptr; }

void vsb_index_free(vsb_index *ix) {
    if (!ix) return;
    cudaSetDevice(ix->device);
    drain(ix);
    cudaStreamSynchronize(ix->xstream);
    groupings_detach(ix->groupings);
    delete ix;
}

int vsb_range_get(const vsb_range *r, int q, const int64_t **rowids, const double **dist, int64_t *count) {
    if (!r || q < 0 || (size_t)q >= r->ids.size()) return fail(VSB_EINVAL, "bad range result or query %d", q);
    if (rowids) *rowids = r->ids[(size_t)q].data();
    if (dist) *dist = r->dist[(size_t)q].data();
    if (count) *count = (int64_t)r->ids[(size_t)q].size();
    return VSB_OK;
}

void vsb_range_free(vsb_range *r) { delete r; }

int vsb_scan_candidates(vsb_index *ix, int metric, const void *queries, int nq, int k, vsb_candidate *out, int cap_per_query,
                        int *out_counts) {
    if (check_index(ix)) return VSB_EINVAL;
    if (!queries || !out || !out_counts || nq < 0 || k <= 0 || cap_per_query <= 0) return fail(VSB_EINVAL, "bad scan arguments");
    const size_t qbytes = (size_t)ix->dim * ix->esize;
    std::vector<uint2> cands;
    for (int b = 0; b < nq; ++b) {
        int rc = query_candidates(ix, metric, (const uint8_t *)queries + (size_t)b * qbytes, k, cands);
        if (rc) return rc;
        if ((int)cands.size() > cap_per_query) {
            // too many to ship: reduce on this shard first (the shard-local replay keeps exactly the rows
            // that survive locally; a superset of what can survive globally is NOT guaranteed by truncation,
            // so instead we report the condition)
            return fail(VSB_ERANGE, "query %d produced %zu candidates (> cap %d)", b, cands.size(), cap_per_query);
        }
        vsb_candidate *o = out + (size_t)b * cap_per_query;
        for (size_t i = 0; i < cands.size(); ++i) {
            memcpy(&o[i].dist, &cands[i].x, 4);
            o[i].rowid = rowid_of(ix, cands[i].y);
            o[i].seq = ix->first_seq + (long long)cands[i].y;
            o[i].reserved = 0;
        }
        out_counts[b] = (int)cands.size();
    }
    return VSB_OK;
}

int vsb_replay_topk(const vsb_candidate *cands, int n, int k, int *max_index, int64_t *out_rowids, double *out_dist) {
    if (k <= 0) return 0;
    if ((!cands && n > 0) || !out_rowids || !out_dist) return fail(VSB_EINVAL, "bad replay arguments");
    return slots_replay(k, max_index, out_dist, out_rowids, [&](SlotState &s) {
        for (int i = 0; i < n; ++i) slots_offer(s, cands[i].dist, cands[i].rowid);
        return (int)VSB_OK;
    });
}

int vsb_debug_read(vsb_index *ix, const char *name, void *out, int64_t bytes) {
    if (check_index(ix)) return VSB_EINVAL;
    if (!name || !out || bytes <= 0) return fail(VSB_EINVAL, "bad debug read arguments");
    CU(cudaSetDevice(ix->device));
    const int rc = drain(ix);
    if (rc) return rc;
    const Work &w = ix->work[(ix->ws_next + kWorks - 1) % kWorks];     // the workspace of the most recent query
    const void *src = nullptr;
    size_t have = 0;
    if (!strcmp(name, "cta_time")) { src = w.d_cta_time; have = sizeof(unsigned) * (size_t)ix->num_sms; }
    else if (!strcmp(name, "bounds")) { src = w.d_bounds; have = sizeof(long long) * (size_t)(ix->num_sms + 1); }
    else if (!strcmp(name, "topk_bounds")) { src = ix->d_lk_state; have = offsetof(LkState, sel); }   // segments and bounds of the last large-k view
    else if (!strcmp(name, "large_k_batch_bounds")) {                   // host copy: pieces and bounds of the last large-k batch
        if (!ix->batch || ix->batch->lkb_debug.empty()) return fail(VSB_EINVAL, "no large-k batch has run yet");
        const std::vector<uint8_t> &d = ix->batch->lkb_debug;
        memcpy(out, d.data(), std::min<size_t>(d.size(), (size_t)bytes));
        return (int)std::min<size_t>(d.size(), (size_t)bytes);
    }
    else if (!strcmp(name, "large_k_batch_cands")) {                    // host copy: every query's candidates of the last large-k batch
        if (!ix->batch || ix->batch->lkb_cnt.empty()) return fail(VSB_EINVAL, "no large-k batch has run yet");
        const BatchWs &b = *ix->batch;
        std::vector<uint8_t> d(8 + 8 * b.lkb_cnt.size());
        const long long nq = (long long)b.lkb_cnt.size();
        memcpy(d.data(), &nq, 8);
        memcpy(d.data() + 8, b.lkb_cnt.data(), 8 * b.lkb_cnt.size());
        for (size_t q = 0; q < b.lkb_cnt.size(); ++q)
            if (b.lkb_cnt[q] > 0) {
                const uint8_t *src = reinterpret_cast<const uint8_t *>(b.h_kout.get() + b.lkb_off[q]);
                d.insert(d.end(), src, src + sizeof(uint2) * (size_t)b.lkb_cnt[q]);
            }
        const size_t n = std::min<size_t>({d.size(), (size_t)bytes, (size_t)INT32_MAX});
        memcpy(out, d.data(), n);
        return (int)n;
    }
    else if (!strcmp(name, "grouped")) {                                // the layout and last query of the last grouped call
        if (!ix->grouped || !ix->grouped->lay) return fail(VSB_EINVAL, "no grouped call has run yet");
        const GroupedShard &gs = *ix->grouped;
        const GroupedLayout &L = *gs.lay;
        const GroupedParams &p = gs.p;
        const size_t npos = (size_t)L.npos, np = (size_t)L.npieces, nk = gs.kmin.size(), kk = (size_t)p.k;
        const size_t ndist = npos ? (size_t)ix->n : 0;
        const long long head[7] = {(long long)npos, (long long)np, (long long)nk, (long long)kk, (long long)ndist, gs.ksel_used ? 1 : 0,
                                   (long long)gs.pairs.size()};
        std::vector<uint8_t> d(sizeof head);
        memcpy(d.data(), head, sizeof head);
        const auto host = [&](const void *src, size_t n) {
            d.insert(d.end(), (const uint8_t *)src, (const uint8_t *)src + n);
        };
        const auto dev = [&](const void *src, size_t n) {
            const size_t at = d.size();
            d.resize(at + n);
            if (n) CU(cudaMemcpy(d.data() + at, src, n, cudaMemcpyDeviceToHost));
            return (int)VSB_OK;
        };
        host(L.h_rows.data(), 4 * npos);
        host(L.koff.data(), 4 * (nk + 1));
        int rc2 = dev(L.pstart, 4 * (np + 1));
        if (rc2 == VSB_OK) rc2 = dev(L.pkey, 4 * np);
        if (rc2 == VSB_OK) rc2 = dev(L.kpiece, 4 * (nk + 1));
        if (rc2 == VSB_OK) rc2 = dev(gs.d_dist, 4 * ndist);
        if (rc2 == VSB_OK) rc2 = dev(p.pd, 4 * npos);
        if (rc2 == VSB_OK) rc2 = dev(p.lists, 4 * np * kk);
        if (rc2 == VSB_OK) rc2 = dev(p.bound, 4 * np);
        if (rc2) return rc2;
        host(gs.kmin.data(), 4 * nk);
        host(gs.pairs.data(), sizeof(uint2) * gs.pairs.size());
        if (gs.ksel_used && (rc2 = dev(gs.d_ksel, nk))) return rc2;
        const size_t n = std::min<size_t>({d.size(), (size_t)bytes, (size_t)INT32_MAX});
        memcpy(out, d.data(), n);
        return (int)n;
    }
    else return fail(VSB_EINVAL, "unknown debug buffer %s", name);
    if (!src) return fail(VSB_EINVAL, "no %s has run yet", strcmp(name, "topk_bounds") ? "scan" : "large-k query");
    CU(cudaMemcpy(out, src, std::min<size_t>(have, (size_t)bytes), cudaMemcpyDeviceToHost));
    return (int)std::min<size_t>(have, (size_t)bytes);
}

int vsb_debug_write(vsb_index *ix, const char *name, const void *data, int64_t bytes) {
    if (check_index(ix)) return VSB_EINVAL;
    if (!name || !data) return fail(VSB_EINVAL, "bad debug write arguments");
    if (!strcmp(name, "grouped_dist")) {       // the distances of every shard row for the next grouped call, instead of its scans
        if (bytes != (int64_t)sizeof(float) * ix->n || ix->n == 0)
            return fail(VSB_EINVAL, "grouped_dist: %lld bytes expected (float32 x %lld)", (long long)sizeof(float) * ix->n, ix->n);
        ix->grouped_plant.assign((const float *)data, (const float *)data + ix->n);
        return VSB_OK;
    }
    if (strcmp(name, "bounds") != 0) return fail(VSB_EINVAL, "unknown debug buffer %s", name);
    if (ix->streamed || !ix->d_vec) return fail(VSB_EINVAL, "the row partition belongs to a resident index");
    const size_t want = sizeof(long long) * (size_t)(ix->num_sms + 1);
    if (bytes != (int64_t)want) return fail(VSB_EINVAL, "bounds: %zu bytes expected (int64 x %d)", want, ix->num_sms + 1);
    CU(cudaSetDevice(ix->device));
    int rc = ensure_workspace(ix, 32);       // the k <= 32 workspaces: a later query with k <= 32 keeps them (and the plant)
    if (rc) return rc;
    const long long rpw = 32 >> make_plan(ix, 32).log2P;
    const long long total_tiles = (ix->n + rpw - 1) / rpw;
    if (total_tiles < 64ll * ix->num_sms)
        return fail(VSB_EINVAL, "bounds: %lld tiles, the partition is used from %lld", total_tiles, 64ll * ix->num_sms);
    const long long *b = (const long long *)data;
    if (b[0] != 0 || b[ix->num_sms] != total_tiles) return fail(VSB_EINVAL, "bounds must run from 0 to %lld tiles", total_tiles);
    for (int c = 0; c < ix->num_sms; ++c)
        if (b[c + 1] < b[c]) return fail(VSB_EINVAL, "bounds must be non-decreasing (CTA %d)", c);
    rc = drain(ix);
    if (rc) return rc;
    for (int i = 0; i < kWorks; ++i) {
        Work &w = ix->work[i];
        CU(cudaMemcpy(w.d_bounds, b, want, cudaMemcpyHostToDevice));
        w.bounds_tiles = total_tiles;         // the next launch on this workspace uses the plant instead of equal shares
    }
    return VSB_OK;
}

int64_t vsb_debug_survivors(vsb_index *ix, int slot_id, uint32_t *out_pairs, int64_t cap, int *flags) {
    if (!ix) return fail(VSB_EINVAL, "null index");
    if (slot_id < 0 || slot_id >= kSlots || !ix->slots_ready || (!out_pairs && cap > 0) || cap < 0 || !flags)
        return fail(VSB_EINVAL, "bad debug survivors arguments");
    for (int j = 0; j < ix->held.nq; ++j)            // as vsb_collect: reading a held query launches its pass
        if (ix->held.slot[j] == slot_id) {
            const int rc = flush_held(ix);
            if (rc) return rc;
        }
    CU(cudaSetDevice(ix->device));
    Slot *slot = &ix->slot[slot_id];
    bool overflow = false;
    int64_t n = 0;
    const int rc = visit_survivors(ix, slot, &overflow, [&](uint2 c) {
        if (n < cap) { out_pairs[2 * n] = c.x; out_pairs[2 * n + 1] = c.y; }
        ++n;
    });
    if (rc) return rc;
    *flags = slot->h_head->flags;
    return n;
}

int vsb_debug_tc_level(vsb_index *ix, int metric, const void *queries, int nq, const float *U, int64_t r0, int64_t r1, int N, int mode,
                       void *out, int64_t out_cap, void *out_qc, void *out_norms, int64_t *out_count) {
    if (check_index(ix)) return VSB_EINVAL;
    long long cnt = 0;
    const int rc = batch_tc_level(ix, metric, queries, nq, U, r0, r1, N, mode, out, out_cap, out_qc, out_norms, &cnt);
    if (rc == VSB_OK && out_count) *out_count = cnt;
    return rc;
}

int vsb_debug_refine(vsb_index *ix, int metric, const void *queries, int nq, const uint32_t *pairs, int64_t npairs, const float *U,
                     int64_t cand_cap, uint32_t *out_bucket, uint32_t *out_bcount, uint32_t *out_stats) {
    if (check_index(ix)) return VSB_EINVAL;
    return batch_debug_refine(ix, metric, queries, nq, pairs, npairs, U, cand_cap, out_bucket, out_bcount, out_stats);
}

int vsb_debug_replay(vsb_index *ix, int metric, const void *queries, int nq, int k, int level0, const uint32_t *bucket, const uint32_t *bcount,
                     float *slot_d, uint32_t *slot_row, int *slot_mi, int acc_cap, uint32_t *acc_log, int *acc_count, int final_sort,
                     float *out_U, uint32_t *out_qc, uint32_t *out_bcount, uint32_t *out_stats) {
    if (check_index(ix)) return VSB_EINVAL;
    return batch_debug_replay(ix, metric, queries, nq, k, level0, bucket, bcount, slot_d, slot_row, slot_mi, acc_cap, acc_log, acc_count,
                              final_sort, out_U, out_qc, out_bcount, out_stats);
}

int vsb_profile_read(vsb_index *ix, double *scan_ms, int *scan_launches, double *filter_ms, int *filter_launches) {
    if (check_index(ix)) return VSB_EINVAL;
    CU(cudaSetDevice(ix->device));
    const int rc = drain(ix);
    if (rc) return rc;
    double a = 0, b = 0;
    int na = 0, nb = 0;
    for (size_t i = 0; i < ix->prof_kind.size(); ++i) {
        float ms = 0;
        CU(cudaEventElapsedTime(&ms, ix->prof_ev[4 * i], ix->prof_ev[4 * i + 1]));
        a += ms; ++na;
        if (ix->prof_kind[i] == 2) {
            CU(cudaEventElapsedTime(&ms, ix->prof_ev[4 * i + 2], ix->prof_ev[4 * i + 3]));
            b += ms; ++nb;
        }
    }
    ix->prof_kind.clear();
    ix->prof_used = 0;
    if (scan_ms) *scan_ms = a;
    if (scan_launches) *scan_launches = na;
    if (filter_ms) *filter_ms = b;
    if (filter_launches) *filter_launches = nb;
    return VSB_OK;
}

// The hold rule (DESIGN §3.2): while the caller has an uncollected query on this index, a new submission waits to share a pass
// with the next ones; the held pass is launched when it is full, when one of its queries is collected, when a submission with
// another metric or k (or for one of its slots) arrives, and by any other call on the index (check_index).  A submission with
// nothing outstanding launches at once.  fetch == 0 submissions are read on the device, where their collection cannot be seen:
// they launch at once and never count as outstanding.
int vsb_scan_submit(vsb_index *ix, int metric, const void *query, int query_on_device, int k, int fetch, int want_slot) {
    if (!ix) return fail(VSB_EINVAL, "null index");
    if (want_slot >= kSlots) return fail(VSB_EINVAL, "slot %d out of range (have %d)", want_slot, kSlots);
    int rc = check_submission(ix, metric, query, 0, 1, query_on_device, k);   // before a held query could take a slot
    if (rc) return rc;
    const int si = want_slot >= 0 ? want_slot : (ix->last_slot + 1) % kSlots;
    HeldPass &h = ix->held;
    bool in_pass = false;
    for (int j = 0; j < h.nq; ++j) in_pass |= h.slot[j] == si;
    if (h.nq > 0 && (in_pass || h.metric != metric || h.k != k)) rc = flush_held(ix);
    if (rc) return rc;
    ix->uncollected &= ~(1u << si);                 // a query left uncollected in this slot is given up
    if (fetch == 0 || ix->uncollected == 0) {
        rc = submit_group(ix, metric, query, 0, 1, query_on_device, k, fetch, si, false);
    } else {
        CU(cudaSetDevice(ix->device));
        rc = ensure_slots(ix);
        if (rc) return rc;
        if (h.nq == 0) {
            h.metric = metric;
            h.k = k;
            h.ss = next_scan_stream(ix);
        }
        Slot *slot = &ix->slot[si];
        const uint8_t *q = (const uint8_t *)query;
        if (!query_on_device) {
            if (slot->seq > 0) CU(cudaEventSynchronize(slot->done));   // the slot's pinned staging buffer is free again
            rc = stage_query(ix, slot, q, h.ss);
            if (rc) return rc;
            q = slot->d_query;
        }
        h.query[h.nq] = q;
        h.slot[h.nq] = si;
        ++h.nq;
        ix->last_slot = si;
        ix->last_metric = metric;
        if (h.nq >= pass_max(ix, (k + 31) & ~31)) rc = flush_held(ix);
    }
    if (rc) return rc;
    if (fetch != 0) ix->uncollected |= 1u << si;
    return si;   // slot id (>= 0) for vsb_collect / vsb_result_block
}

int vsb_scan_submit_group(vsb_index *ix, int metric, const void *queries, int64_t query_stride, int nq, int query_on_device, int k,
                          int fetch, int first_slot) {
    return submit_group(ix, metric, queries, query_stride, nq, query_on_device, k, fetch, first_slot, false);
}

int vsb_scan_device_query(vsb_index *ix, int metric, const void *d_query, int k) {
    return vsb_scan_submit(ix, metric, d_query, 1, k, 1, -1);
}

int vsb_result_block(vsb_index *ix, int slot_id, void **d_block, int64_t *bytes) {
    if (check_index(ix)) return VSB_EINVAL;
    if (slot_id < 0 || slot_id >= kSlots) return fail(VSB_EINVAL, "bad slot");
    CU(cudaSetDevice(ix->device));
    int rc = ensure_slots(ix);
    if (rc) return rc;
    if (d_block) *d_block = ix->slot[slot_id].d_head;
    if (bytes) *bytes = (int64_t)kHeadBytes;
    return VSB_OK;
}

int vsb_merge_result_blocks(const void *blocks, int world, int64_t block_stride, const int64_t *first_seq, int k, int64_t *out_rowids,
                            double *out_dist) {
    if (!blocks || world <= 0 || !first_seq || k <= 0 || !out_rowids || !out_dist) return fail(VSB_EINVAL, "bad merge arguments");
    return merge_blocks_strided((const uint8_t *)blocks, world, (size_t)block_stride, first_seq, k, out_rowids, out_dist);
}

int vsb_merge_result_groups(const void *blocks, int world, int64_t rank_stride, int64_t block_stride, int nq, const int64_t *first_seq,
                            int k, int64_t *out_rowids, double *out_dist, int *out_counts) {
    if (!blocks || nq <= 0 || !out_counts) return fail(VSB_EINVAL, "bad merge arguments");
    for (int j = 0; j < nq; ++j) {
        const int cnt = vsb_merge_result_blocks((const uint8_t *)blocks + (size_t)j * (size_t)block_stride, world, rank_stride, first_seq, k,
                                                out_rowids + (size_t)j * k, out_dist + (size_t)j * k);
        if (cnt < 0) return cnt;
        out_counts[j] = cnt;
    }
    return VSB_OK;
}

int vsb_batch_shard_scan(vsb_index *ix, int metric, const void *queries, int nq, int k, void **d_block, int64_t *bytes) {
    if (check_index(ix)) return VSB_EINVAL;
    if (!queries || nq <= 0 || k <= 0 || !d_block || !bytes) return fail(VSB_EINVAL, "bad batch scan arguments");
    if (!batch_supported(ix, metric, nq, k))
        return fail(VSB_ERANGE, "no tensor-core batch path for this shard (type %d, metric %d, %d queries, k %d, %lld rows)", ix->vtype, metric,
                    nq, k, ix->n);
    const auto t0 = std::chrono::steady_clock::now();
    int rc = batch_levels(ix, metric, queries, nq, k, true);
    if (rc) return rc;
    CU(cudaStreamSynchronize(ix->stream));
    rc = batch_check(ix, ix->batch.get());
    if (rc) return rc;
    ix->st_batch_us += std::chrono::duration_cast<std::chrono::microseconds>(std::chrono::steady_clock::now() - t0).count();
    *d_block = ix->batch->d_acc;
    *bytes = (int64_t)acc_block_bytes(nq, acc_cap_of(k));
    return VSB_OK;
}

int vsb_batch_merge(vsb_index *ix, const void *d_blocks, int world, int64_t block_stride, const int64_t *first_seq, int nq, int k,
                    int64_t *out_seq, double *out_dist, int *out_counts) {
    if (check_index(ix)) return VSB_EINVAL;
    if (!d_blocks || world <= 0 || !first_seq || nq <= 0 || k <= 0 || k > kMaxK || !out_seq || !out_dist)
        return fail(VSB_EINVAL, "bad batch merge arguments");
    if (block_stride < (int64_t)acc_block_bytes(nq, acc_cap_of(k))) return fail(VSB_EINVAL, "block stride smaller than a block");
    const auto t0 = std::chrono::steady_clock::now();
    int rc = batch_merge(ix, d_blocks, world, block_stride, first_seq, nq, k, out_seq, out_dist, out_counts);
    ix->st_batch_us += std::chrono::duration_cast<std::chrono::microseconds>(std::chrono::steady_clock::now() - t0).count();
    return rc;
}

int vsb_index_lookup_rowids(const vsb_index *ix, const int64_t *seq, int64_t n, int64_t *out) {
    if (!ix || (!seq && n > 0) || (!out && n > 0) || n < 0) return fail(VSB_EINVAL, "bad lookup arguments");
    for (int64_t i = 0; i < n; ++i) {
        const long long local = (long long)seq[i] - ix->first_seq;
        out[i] = (local >= 0 && local < ix->n) ? rowid_of(ix, (uint32_t)local) : 0;
    }
    return VSB_OK;
}

int vsb_collect_last(vsb_index *ix, int k, int64_t *out_rowids, double *out_dist, int *out_count) {
    if (check_index(ix)) return VSB_EINVAL;
    if (ix->last_slot < 0) return fail(VSB_EINVAL, "no device scan was launched");
    return vsb_collect(ix, ix->last_slot, k, out_rowids, out_dist, out_count);
}

int vsb_collect(vsb_index *ix, int slot_id, int k, int64_t *out_rowids, double *out_dist, int *out_count) {
    if (!ix) return fail(VSB_EINVAL, "null index");
    if (slot_id < 0 || slot_id >= kSlots || !ix->slots_ready) return fail(VSB_EINVAL, "bad slot");
    for (int j = 0; j < ix->held.nq; ++j)            // collecting a held query launches its pass; collecting another does not
        if (ix->held.slot[j] == slot_id) {
            const int rc = flush_held(ix);
            if (rc) return rc;
        }
    ix->uncollected &= ~(1u << slot_id);
    CU(cudaSetDevice(ix->device));
    bool overflow = false;
    const int cnt = slots_replay(k, nullptr, out_dist, out_rowids, [&](SlotState &s) {   // waits for this query only; a later launch may still run
        return visit_survivors(ix, &ix->slot[slot_id], &overflow, [&](uint2 c) { slots_offer_cands(s, &c, 1, [&](uint32_t row) { return rowid_of(ix, row); }); });
    });
    if (cnt < 0) return cnt;
    if (overflow) return fail(VSB_ERANGE, "candidate log overflowed; use vsb_scan_topk (host query) for this input");
    if (out_count) *out_count = cnt;
    return VSB_OK;
}

}  // extern "C"
