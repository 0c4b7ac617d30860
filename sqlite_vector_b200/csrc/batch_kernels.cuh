// batch_kernels.cuh — batched-query path: wgmma tensor-core scoring + exact candidate refinement.
//
// For B queries against the resident shard the scores  S[row][q] = <row, query_q>  are a dense GEMM
// (rows x dim) x (dim x B): this is the one place where the scan IS tensor-core work (north_star).
// tc_scan_kernel computes S tile by tile with Hopper warpgroup MMAs (A = 128 corpus rows, B = up to 256 queries, both K-major
// in 128B-swizzled shared memory filled by TMA, accumulators in registers) and NEVER materialises S: each consumer warpgroup
// tests its 64 x N accumulators against a per-query bound straight from registers, appending the rare hits (row, query) to a
// candidate log.  The bound is conservative (it absorbs the tensor-core rounding), so the log
// is a superset of the rows whose EXACT reference distance beats the query's running k-th distance; the refinement
// kernels below recompute those distances with exactly the arithmetic of the single-query kernel (accum16/finalize)
// and replay the reference's slot algorithm (src/sqlite-vector.c:2022-2069, 2145-2152) per query, level by level.
#pragma once
#include <cuda.h>

#include <type_traits>

#include "scan_kernels.cuh"
#include "wgmma.cuh"

namespace vsb {

enum { TK_BF16 = 0, TK_F16 = 1, TK_I8 = 2, TK_U8 = 3 };
// warps 0-7: two consumer warpgroups (rows 0-63 and 64-127 of the corpus tile), warp 8: TMA producer
constexpr int kTcConsumers = 2;
constexpr int kTcThreads = kTcConsumers * 128 + 32;
constexpr int kTcMaxStages = 8;
constexpr int kTcM = 128;           // corpus rows per tile
constexpr int kTcKBytes = 128;      // one swizzle atom of K per stage
// tc_scan_kernel<KIND, MC_TC_SCORES, N>: the same tile walk and MMAs, but every score of rows [r0, r1) x queries [0, nq) is
// stored to TcParams::scores instead of being tested (vsb_debug_tc_level checks the scores against an exact GEMM)
constexpr int MC_TC_SCORES = 4;

struct TcParams {
    long long r0, r1;       // row range of this level (r0 multiple of 128)
    long long n;            // rows in the shard
    int nq;                 // queries
    int N;                  // MMA N: 32, 64, 128 or 256 queries per tile
    int NG;                 // query groups = ceil(nq / N)
    int KB;                 // 128-byte K blocks per row
    int nstages;            // ring depth (2..kTcMaxStages)
    int mc;                 // MC_L2 / MC_COS / MC_DOT (l1_batch_kernel: MC_L1), or MC_TC_SCORES
    int chunk_test;         // integer kinds: test 32-column chunks before single scores (see tc_scan_kernel)
    float eps;              // fp kinds: relative slack of the tensor-core score, see tc_fp_eps
    const float *qc;        // [NG*N] per-query constant (float, or int bit pattern for the integer kinds)
    const void *norms;      // [n] float (fp kinds) or int (integer kinds): sum of squares of each row
    uint2 *cand;            // (row, query)
    unsigned *cand_count;
    unsigned cand_cap;
    uint32_t *scores;       // MC_TC_SCORES only: [r1 - r0][nq] int32 / float bits
};

// ------------------------------------------------------------------ PTX wrappers (TMA / wgmma)
__device__ __forceinline__ void tma_load_2d(void *dst, const CUtensorMap *map, int c0, int c1, uint64_t *bar) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(
                     smem_u32(dst)),
                 "l"(map), "r"(c0), "r"(c1), "r"(smem_u32(bar))
                 : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t *bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int PENDING>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(PENDING) : "memory"); }

// K-major operand tile in 128B-swizzled shared memory (rows of 128 bytes, 8-row groups 1024 B apart):
// start address >> 4 | LBO = 1 (unused with this swizzle) | SBO = 1024 >> 4 | layout SWIZZLE_128B (1 << 62)
__device__ __forceinline__ uint64_t gmma_desc_sw128(const void *smem) {
    const uint64_t addr = (uint64_t)((smem_u32(smem) & 0x3FFFFu) >> 4);
    return addr | (uint64_t(1) << 16) | (uint64_t(1024 >> 4) << 32) | (uint64_t(1) << 62);
}

template <int KIND, int N, class Acc>
__device__ __forceinline__ void tc_mma(Acc (&d)[N / 2], uint64_t a, uint64_t b, uint32_t scale_d) {
    if constexpr (KIND == TK_BF16) Wgmma<N>::bf16(d, a, b, scale_d);
    else if constexpr (KIND == TK_F16) Wgmma<N>::f16(d, a, b, scale_d);
    else if constexpr (KIND == TK_I8) Wgmma<N>::s8(d, a, b, scale_d);
    else Wgmma<N>::u8(d, a, b, scale_d);
}

// the per-element candidate test.  fp kinds use negated comparisons so that NaN scores count as hits.
template <bool INT8, int MC>
__device__ __forceinline__ bool tc_hit(uint32_t sbits, uint32_t qcbits, float rowf, int rowi) {
    if constexpr (INT8) {
        const int s = (int)sbits;
        if constexpr (MC == MC_DOT) return s > (int)qcbits;
        else if constexpr (MC == MC_L2) return (2 * s + rowi) >= (int)qcbits;           // rowi = -|row|^2
        else return !(fmaf(-__uint_as_float(qcbits), rowf, (float)s) < 0.0f);            // cosine: rowf = |row|
    } else {
        const float s = __uint_as_float(sbits), qc = __uint_as_float(qcbits);
        if constexpr (MC == MC_DOT) return !(s <= qc);
        else if constexpr (MC == MC_L2) return !(fmaf(2.0f, s, rowf) <= qc);             // rowf = -|row|^2 (1 - e)
        else return !(fmaf(-qc, rowf, s) < 0.0f);                                        // cosine: rowf = |row|
    }
}

// one lane of the calling (converged) warp; keeps the producer warp in warp-uniform control flow around the TMA issue
__device__ __forceinline__ bool elect_one() {
    uint32_t pred;
    asm volatile("{\n\t.reg .pred p;\n\telect.sync _|p, 0xFFFFFFFF;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(pred));
    return pred != 0;
}

// Tile order: tile t = corpus-tile * NG + query-group, t = blockIdx.x, + gridDim.x, ...  (both operands streamed through the
// stage ring; the query groups of one corpus tile run on different CTAs at about the same time, so the corpus tile is read
// from HBM once and from L2 by the others).  Walked incrementally: no division per tile.
struct TileWalk {
    long long mt0;        // first corpus tile of the level
    uint32_t count;       // tiles this CTA processes
    uint32_t q, r;        // current tile: corpus tile mt0 + q, query group r
    uint32_t gq, gr, NG;  // gridDim.x = gq * NG + gr
    __device__ __forceinline__ void init(const TcParams &p) {
        mt0 = p.r0 / kTcM;
        const long long ntm = (p.r1 + kTcM - 1) / kTcM - mt0;
        const long long total = ntm * p.NG;
        NG = (uint32_t)p.NG;
        count = (total > (long long)blockIdx.x) ? (uint32_t)((total - blockIdx.x + gridDim.x - 1) / gridDim.x) : 0u;
        q = blockIdx.x / NG; r = blockIdx.x % NG;
        gq = gridDim.x / NG; gr = gridDim.x % NG;
    }
    __device__ __forceinline__ long long mt() const { return mt0 + q; }
    __device__ __forceinline__ int ng() const { return (int)r; }
    __device__ __forceinline__ void next() {
        q += gq; r += gr;
        if (r >= NG) { r -= NG; ++q; }
    }
};

// The stage ring of both scoring kernels: NS stages [A | B] of one 128-byte K slice each (A = the 128 corpus rows of a tile,
// B = its N queries; 128B-swizzled, 1024-aligned, filled by TMA), then the full / empty mbarriers of kTcMaxStages stages.
// full[s] completes on the producer's arrival plus the stage's bytes, empty[s] on `consumers` arrivals of the consumers that
// have read stage s.  end() is the first byte after the barriers.
template <int N>
struct StageRing {
    static constexpr uint32_t a_bytes = kTcM * kTcKBytes, b_bytes = (uint32_t)N * kTcKBytes;
    static constexpr uint32_t stage_bytes = a_bytes + b_bytes;
    uint8_t *stages;
    uint64_t *full, *empty;
    __device__ __forceinline__ StageRing(uint8_t *smem, int NS)
        : stages(smem), full(reinterpret_cast<uint64_t *>(smem + (size_t)NS * stage_bytes)), empty(full + kTcMaxStages) {}
    __device__ __forceinline__ uint8_t *stage(int s) const { return stages + (size_t)s * stage_bytes; }
    __device__ __forceinline__ uint8_t *end() const { return reinterpret_cast<uint8_t *>(empty + kTcMaxStages); }
    __device__ __forceinline__ void init(int consumers) const {   // thread 0; the caller syncs the block before any use
        if (threadIdx.x == 0) {
            for (int i = 0; i < kTcMaxStages; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], consumers); }
            fence_barrier_init();
        }
    }
    // the TMA producer: the whole warp walks the tiles, one lane issues each stage's two loads
    __device__ __forceinline__ void produce(TileWalk tw, int KB, int NS, const CUtensorMap *tmA, const CUtensorMap *tmB) const {
        int s = 0;
        uint32_t ph = 1;                                                       // parity to wait for on empty[s]: the first pass is free
        for (uint32_t tl = 0; tl < tw.count; ++tl, tw.next()) {
            const int row0 = (int)(tw.mt() * kTcM), col0 = tw.ng() * N;
            for (int kb = 0; kb < KB; ++kb) {
                mbar_wait(&empty[s], ph);
                if (elect_one()) {
                    mbar_expect_tx(&full[s], stage_bytes);
                    uint8_t *st = stage(s);
                    tma_load_2d(st, tmA, kb * kTcKBytes, row0, &full[s]);
                    tma_load_2d(st + a_bytes, tmB, kb * kTcKBytes, col0, &full[s]);
                }
                __syncwarp();
                if (++s == NS) { s = 0; ph ^= 1u; }
            }
        }
    }
};

// Appends the calling lane's `mine` hits to the candidate log with one atomic per warp (call it from the whole warp, inside
// the warp's ballot that some lane may have hits): an inclusive scan of the counts, one atomicAdd by lane 31, then every lane
// writes its hits from its offset on; positions at or past cand_cap are counted but not stored.  visit(emit) calls
// emit(row, query) once for each of the lane's hits.
template <class Visit>
__device__ __forceinline__ void append_hits(const TcParams &prm, int lane, int mine, Visit visit) {
    int incl = mine;
    for (int off = 1; off < 32; off <<= 1) {
        const int o = __shfl_up_sync(0xFFFFFFFFu, incl, off);
        if (lane >= off) incl += o;
    }
    const int total = __shfl_sync(0xFFFFFFFFu, incl, 31);
    unsigned base = 0;
    if (lane == 31) base = atomicAdd(prm.cand_count, (unsigned)total);
    base = __shfl_sync(0xFFFFFFFFu, base, 31);
    unsigned w = base + (unsigned)(incl - mine);
    if (mine) {
        visit([&](long long row, int query) {
            if (w < prm.cand_cap) prm.cand[w] = make_uint2((uint32_t)row, (uint32_t)query);
            ++w;
        });
    }
}

// Accumulator layout of one consumer warpgroup (m64nN, PTX ISA "wgmma register fragments"): thread t of the warpgroup holds
// rows  ra = 16 * (t / 32) + (t % 32) / 4  and  ra + 8  of its 64 rows; d[4j + 0/1] are row ra, columns 8j + 2 (t % 4) + 0/1,
// d[4j + 2/3] row ra + 8, the same columns.
// chunk_test (integer kinds): the hit condition is monotone in the score, so the 8 scores a thread holds of one row in a
// 32-column chunk can only contain a hit if their maximum passes against the chunk's WEAKEST bound (min over its 32 columns,
// precomputed in shared memory).  Only chunks that pass run the per-column test; the log is the same set of (row, query)
// pairs either way.
template <int KIND, int MC, int N>
__global__ void __launch_bounds__(kTcThreads, 1) tc_scan_kernel(const __grid_constant__ CUtensorMap tmA,
                                                                const __grid_constant__ CUtensorMap tmB, const TcParams prm) {
    constexpr bool INT8 = (KIND == TK_I8 || KIND == TK_U8);
    using Acc = typename std::conditional<INT8, uint32_t, float>::type;
    extern __shared__ __align__(1024) uint8_t tsm[];
    const int NS = prm.nstages;
    const StageRing<N> ring(tsm, NS);
    uint32_t *qc_s = reinterpret_cast<uint32_t *>(ring.end());                // [NG*N]
    uint32_t *qcm_s = qc_s + prm.NG * N;                                       // [NG*N/32] weakest bound of each 32-column chunk

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    ring.init(kTcConsumers);                                                   // one arrival per consumer warpgroup
    for (int i = threadIdx.x; i < prm.NG * N; i += kTcThreads) qc_s[i] = __float_as_uint(prm.qc[i]);
    __syncthreads();
    const bool chunk = INT8 && prm.chunk_test;
    if (chunk) {
        for (int c = threadIdx.x; c < prm.NG * N / 32; c += kTcThreads) {
            if constexpr (MC == MC_COS) {
                float m = __uint_as_float(qc_s[c * 32]);
                for (int j = 1; j < 32; ++j) m = fminf(m, __uint_as_float(qc_s[c * 32 + j]));
                qcm_s[c] = __float_as_uint(m);
            } else {
                int m = (int)qc_s[c * 32];
                for (int j = 1; j < 32; ++j) m = min(m, (int)qc_s[c * 32 + j]);
                qcm_s[c] = (uint32_t)m;
            }
        }
        __syncthreads();
    }

    TileWalk tw;
    tw.init(prm);
    const int KB = prm.KB;

    if (warp == kTcConsumers * 4) {                                            // ===== TMA producer
        ring.produce(tw, KB, NS, &tmA, &tmB);
        return;
    }

    // ===== consumer warpgroup wg: MMAs of its 64 rows, then the threshold test from registers
    const int wg = warp >> 2, t = threadIdx.x & 127;
    const int ra = wg * 64 + 16 * (t >> 5) + (lane >> 2);                     // tile rows ra and ra + 8
    const int cq = 2 * (lane & 3);                                             // first of the thread's two columns in each group of 8
    Acc d[N / 2];
    int s = 0;
    uint32_t ph = 0;                                                           // parity to wait for on full[s]
    for (uint32_t tl = 0; tl < tw.count; ++tl, tw.next()) {
        const long long mt = tw.mt();
        const int ng = tw.ng();
        const long long row[2] = {mt * kTcM + ra, mt * kTcM + ra + 8};
        bool rowvalid[2];
        uint32_t nbits[2];
#pragma unroll
        for (int h = 0; h < 2; ++h) {                                          // issued before the MMAs: the load latency hides behind them
            rowvalid[h] = row[h] >= prm.r0 && row[h] < prm.r1;
            nbits[h] = rowvalid[h] ? reinterpret_cast<const uint32_t *>(prm.norms)[row[h]] : 0u;
        }
        int prev = -1;
        for (int kb = 0; kb < KB; ++kb) {
            mbar_wait(&ring.full[s], ph);
            const uint8_t *st = ring.stage(s);
            const uint64_t ad = gmma_desc_sw128(st + wg * 64 * kTcKBytes), bd = gmma_desc_sw128(st + ring.a_bytes);
            wgmma_fence();
#pragma unroll
            for (int k4 = 0; k4 < kTcKBytes / 32; ++k4)                        // K = 32 bytes per MMA: advance the start address by 2 (x16 B)
                tc_mma<KIND, N>(d, ad + (uint64_t)(2 * k4), bd + (uint64_t)(2 * k4), (uint32_t)((kb | k4) != 0));
            wgmma_commit();
            wgmma_wait<1>();                                                   // the previous K block's MMAs have read their stage
            if (prev >= 0 && t == 0) mbar_arrive(&ring.empty[prev]);
            prev = s;
            if (++s == NS) { s = 0; ph ^= 1u; }
        }
        wgmma_wait<0>();
        if (t == 0) mbar_arrive(&ring.empty[prev]);                                // the producer refills it while the scores are tested
        if constexpr (MC == MC_TC_SCORES) {
            const int ncol = prm.nq - ng * N;
#pragma unroll
            for (int i = 0; i < N / 2; ++i) {                                  // accumulator i: row ra + 8 * ((i >> 1) & 1), column 8 (i >> 2) + cq + (i & 1)
                const int h = (i >> 1) & 1, col = 8 * (i >> 2) + cq + (i & 1);
                uint32_t v;
                if constexpr (INT8) v = d[i];
                else v = __float_as_uint(d[i]);
                if (rowvalid[h] && col < ncol) prm.scores[(size_t)(row[h] - prm.r0) * prm.nq + ng * N + col] = v;
            }
            continue;
        }

        float rowf[2] = {0.0f, 0.0f};
        int rowi[2] = {0, 0};
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            if (!rowvalid[h]) continue;
            if constexpr (INT8) {
                const int nn = (int)nbits[h];
                rowi[h] = -nn;
                rowf[h] = (KIND == TK_U8) ? __fsqrt_rn((float)(uint32_t)nn) : __fsqrt_rn((float)nn);
            } else {
                const float nn = __uint_as_float(nbits[h]);
                // L2: a row whose fp32 sum of squares overflowed (bf16 elements beyond ~2^64) can still have a finite distance;
                // NaN makes it a hit, and the refine computes it exactly (special_row_distance)
                if constexpr (MC == MC_L2) rowf[h] = (nn <= FLT_MAX) ? -nn * (1.0f - prm.eps) : __int_as_float(0x7FC00000);
                else rowf[h] = __fsqrt_rn(nn);
            }
        }
        const uint32_t *qc = qc_s + ng * N;
        auto bits = [&](int i) -> uint32_t {
            if constexpr (INT8) return d[i];
            else return __float_as_uint(d[i]);
        };
        auto hit = [&](int i) -> bool {                                       // accumulator i: row ra + 8 * ((i >> 1) & 1), column 8 (i >> 2) + cq + (i & 1)
            const int h = (i >> 1) & 1, col = 8 * (i >> 2) + cq + (i & 1);
            return rowvalid[h] && tc_hit<INT8, MC>(bits(i), qc[col], rowf[h], rowi[h]);
        };
        bool any = false;
        if (chunk) {
#pragma unroll
            for (int c = 0; c < N / 32; ++c) {
                const uint32_t qm = qcm_s[(ng * N >> 5) + c];
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    int m = INT_MIN;
#pragma unroll
                    for (int j = 4 * c; j < 4 * c + 4; ++j) m = max(m, max((int)bits(4 * j + 2 * h), (int)bits(4 * j + 2 * h + 1)));
                    bool a;
                    if constexpr (MC == MC_DOT) a = m > (int)qm;
                    else if constexpr (MC == MC_L2) a = (2 * m + rowi[h]) >= (int)qm;
                    else a = !(fmaf(-__uint_as_float(qm), rowf[h], (float)m) < 0.0f);   // rowf >= 0: monotone in both m and the bound
                    any |= a && rowvalid[h];
                }
            }
        } else {
#pragma unroll
            for (int j = 0; j < N / 8; ++j) {
                const uint2 c = *reinterpret_cast<const uint2 *>(qc + 8 * j + cq);
                any |= (rowvalid[0] && (tc_hit<INT8, MC>(bits(4 * j + 0), c.x, rowf[0], rowi[0]) | tc_hit<INT8, MC>(bits(4 * j + 1), c.y, rowf[0], rowi[0]))) ||
                       (rowvalid[1] && (tc_hit<INT8, MC>(bits(4 * j + 2), c.x, rowf[1], rowi[1]) | tc_hit<INT8, MC>(bits(4 * j + 3), c.y, rowf[1], rowi[1])));
            }
        }
        if (__ballot_sync(0xFFFFFFFFu, any)) {                                 // rare: append (row, query) hits
            const int ncol = prm.nq - ng * N;                                  // padded query columns are never reported
            int mine = 0;
            if (any) {
#pragma unroll
                for (int i = 0; i < N / 2; ++i) mine += (hit(i) && 8 * (i >> 2) + cq + (i & 1) < ncol) ? 1 : 0;
            }
            append_hits(prm, lane, mine, [&](auto emit) {
#pragma unroll
                for (int i = 0; i < N / 2; ++i) {
                    const int col = 8 * (i >> 2) + cq + (i & 1);
                    if (hit(i) && col < ncol) emit(row[(i >> 1) & 1], ng * N + col);
                }
            });
        }
    }
}

// ------------------------------------------------------------------ L1 scores on the CUDA cores
// sum |row_i - q_i| has no GEMM form, but over a batch it is the same dense all-pairs work, compute-bound once the corpus is
// read once per level.  l1_batch_kernel walks the tiles of tc_scan_kernel (TileWalk, and StageRing's TMA producer warp and
// stage ring: 128 corpus rows and N queries per 128-byte K slice, 128B swizzle, full / empty mbarriers) and adds the sums on
// the CUDA cores.  Consumer warp w owns queries [w N/8, (w + 1) N/8) of the tile and lane l the rows l + 32 i, i < 4: a thread keeps
// 4 x N/8 sums in registers.  Every 16-byte chunk is one LDS.128; the query chunks a warp reads are broadcasts, and chunk c of
// row r sits at c ^ (r & 7), so the 8 lanes of one LDS.128 phase hit 8 different 16-byte bank groups.
//   int8 / uint8: VABSDIFF4 + IDP.4A per 4 element pairs, exact int32 (the same instructions as accum16).
//   f32 / f16 / bf16: s += |x - y| in fp32, every term formed with one rounding, like accum16 (only the order of the sum differs).
// The epilogue tests every (row, query) against qc[query] from registers and appends hits to the candidate log with one atomic
// per warp (append_hits): integer types (float)S < qc with qc = U, exactly the refine's keep condition; fp types
// !(s >= qc) with the conservative constant of conservative_qc (NaN scores are hits).  Padded query columns are never
// reported.  prm.mc == MC_TC_SCORES stores every score of rows [r0, r1) instead (vsb_debug_tc_level mode 1).
constexpr int kL1Warps = 8;
constexpr int kL1Threads = kL1Warps * 32 + 32;   // warps 0-7: consumers, warp 8: TMA producer

template <int VT, int N>
__global__ void __launch_bounds__(kL1Threads, 1) l1_batch_kernel(const __grid_constant__ CUtensorMap tmA,
                                                                 const __grid_constant__ CUtensorMap tmB, const TcParams prm) {
    constexpr bool INT8 = (VT == T_I8 || VT == T_U8);
    constexpr int C = N / kL1Warps;                                            // queries per warp
    constexpr int R = kTcM / 32;                                               // rows per lane
    constexpr int NE = (VT == T_F32) ? 4 : 8;                                  // elements per 16-byte chunk (fp types)
    using Acc = typename std::conditional<INT8, uint32_t, float>::type;
    extern __shared__ __align__(1024) uint8_t lsm[];
    const int NS = prm.nstages;
    const StageRing<N> ring(lsm, NS);

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    ring.init(kL1Warps);                                                       // one arrival per consumer warp
    __syncthreads();

    TileWalk tw;
    tw.init(prm);
    const int KB = prm.KB;

    if (warp == kL1Warps) {                                                    // ===== TMA producer
        ring.produce(tw, KB, NS, &tmA, &tmB);
        return;
    }

    // ===== consumer warp: queries q0 .. q0 + C - 1 of the tile, rows lane + 32 i
    const int q0 = warp * C;
    const uint32_t rsw = (uint32_t)(lane & 7);                                 // swizzle of all this lane's rows
    int s = 0;
    uint32_t ph = 0;
    for (uint32_t tl = 0; tl < tw.count; ++tl, tw.next()) {
        const long long mt = tw.mt();
        const int ng = tw.ng();
        const int ncol = prm.nq - ng * N - q0;                                 // real queries of this warp (C or fewer, maybe none)
        Acc acc[R][C];
#pragma unroll
        for (int i = 0; i < R; ++i)
#pragma unroll
            for (int j = 0; j < C; ++j) acc[i][j] = 0;
        for (int kb = 0; kb < KB; ++kb) {
            mbar_wait(&ring.full[s], ph);
            if (ncol > 0) {                                                    // warp-uniform: padding-only warps just pass the stage on
                const uint8_t *A = ring.stage(s) + lane * kTcKBytes;
                const uint8_t *B = ring.stage(s) + ring.a_bytes + q0 * kTcKBytes;
#pragma unroll 2
                for (uint32_t c = 0; c < kTcKBytes / 16; ++c) {
                    uint4 rv[R];
#pragma unroll
                    for (int i = 0; i < R; ++i) rv[i] = *reinterpret_cast<const uint4 *>(A + i * 32 * kTcKBytes + ((c ^ rsw) << 4));
                    if constexpr (INT8) {
#pragma unroll
                        for (int j = 0; j < C; ++j) {
                            const uint4 qv = *reinterpret_cast<const uint4 *>(B + j * kTcKBytes + ((c ^ (uint32_t)((q0 + j) & 7)) << 4));
                            const uint32_t qw[4] = {qv.x, qv.y, qv.z, qv.w};
#pragma unroll
                            for (int i = 0; i < R; ++i) {
                                const uint32_t rw[4] = {rv[i].x, rv[i].y, rv[i].z, rv[i].w};
#pragma unroll
                                for (int e = 0; e < 4; ++e) {
                                    const uint32_t ad = (VT == T_U8) ? __vabsdiffu4(rw[e], qw[e]) : __vabsdiffs4(rw[e], qw[e]);
                                    acc[i][j] = __dp4a(ad, 0x01010101u, acc[i][j]);
                                }
                            }
                        }
                    } else {
                        float y[R][8];
#pragma unroll
                        for (int i = 0; i < R; ++i) unpack8<VT>(rv[i], y[i]);
#pragma unroll
                        for (int j = 0; j < C; ++j) {
                            const uint4 qv = *reinterpret_cast<const uint4 *>(B + j * kTcKBytes + ((c ^ (uint32_t)((q0 + j) & 7)) << 4));
                            float x[8];
                            unpack8<VT>(qv, x);
#pragma unroll
                            for (int i = 0; i < R; ++i)
#pragma unroll
                                for (int e = 0; e < NE; ++e) acc[i][j] += fabsf(x[e] - y[i][e]);
                        }
                    }
                }
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(&ring.empty[s]);                        // this warp has read the stage
            if (++s == NS) { s = 0; ph ^= 1u; }
        }
        if (ncol <= 0) continue;
        long long row[R];
        bool rowvalid[R];
#pragma unroll
        for (int i = 0; i < R; ++i) {
            row[i] = mt * kTcM + lane + 32 * i;
            rowvalid[i] = row[i] >= prm.r0 && row[i] < prm.r1;
        }
        const int qbase = ng * N + q0;
        if (prm.mc == MC_TC_SCORES) {
#pragma unroll
            for (int i = 0; i < R; ++i)
#pragma unroll
                for (int j = 0; j < C; ++j) {
                    uint32_t v;
                    if constexpr (INT8) v = acc[i][j];
                    else v = __float_as_uint(acc[i][j]);
                    if (rowvalid[i] && j < ncol) prm.scores[(size_t)(row[i] - prm.r0) * prm.nq + qbase + j] = v;
                }
            continue;
        }
        float qc[C];
#pragma unroll
        for (int j = 0; j < C; ++j) qc[j] = __ldg(prm.qc + qbase + j);         // padded columns: +INF from the upload
        auto hit = [&](int i, int j) -> bool {
            bool h;
            if constexpr (INT8) h = (float)acc[i][j] < qc[j];
            else h = !(acc[i][j] >= qc[j]);
            return h && rowvalid[i] && j < ncol;
        };
        int mine = 0;
#pragma unroll
        for (int i = 0; i < R; ++i)
#pragma unroll
            for (int j = 0; j < C; ++j) mine += hit(i, j) ? 1 : 0;
        if (__ballot_sync(0xFFFFFFFFu, mine != 0)) {                           // rare: append (row, query) hits
            append_hits(prm, lane, mine, [&](auto emit) {
#pragma unroll
                for (int i = 0; i < R; ++i)
#pragma unroll
                    for (int j = 0; j < C; ++j)
                        if (hit(i, j)) emit(row[i], qbase + j);
            });
        }
    }
}


// ------------------------------------------------------------------ row norms (once per resident shard)
template <int VT>
__global__ void row_norm_kernel(const uint8_t *vec, long long n, int pitch, void *out) {
    const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (row >= n) return;
    const uint4 *p = reinterpret_cast<const uint4 *>(vec + (size_t)row * pitch);
    float f = 0.0f;
    int iq = 0;
    for (int c = lane; c < pitch / 16; c += 32) {
        const uint4 q = ldg_stream(p + c);
        if constexpr (VT == T_U8) {
            iq = (int)__dp4a(q.x, q.x, (uint32_t)iq); iq = (int)__dp4a(q.y, q.y, (uint32_t)iq);
            iq = (int)__dp4a(q.z, q.z, (uint32_t)iq); iq = (int)__dp4a(q.w, q.w, (uint32_t)iq);
        } else if constexpr (VT == T_I8) {
            iq = __dp4a((int)q.x, (int)q.x, iq); iq = __dp4a((int)q.y, (int)q.y, iq);
            iq = __dp4a((int)q.z, (int)q.z, iq); iq = __dp4a((int)q.w, (int)q.w, iq);
        } else {
            constexpr int NE = (VT == T_F32) ? 4 : 8;                           // unpack8 writes 4 floats for f32
            float x[8];
            unpack8<VT>(q, x);
#pragma unroll
            for (int j = 0; j < NE; ++j) f = fmaf(x[j], x[j], f);
        }
    }
    for (int off = 16; off >= 1; off >>= 1) {
        f += __shfl_xor_sync(0xFFFFFFFFu, f, off);
        iq += __shfl_xor_sync(0xFFFFFFFFu, iq, off);
    }
    if (lane == 0) {
        if constexpr (VT == T_U8 || VT == T_I8) reinterpret_cast<int *>(out)[row] = iq;
        else reinterpret_cast<float *>(out)[row] = f;
    }
}

// ------------------------------------------------------------------ exact refinement
// level 0: every (row, query) pair of the first m0 rows is a candidate
__global__ void all_pairs_kernel(uint2 *cand, unsigned *count, long long m0, int nq) {
    const long long total = m0 * nq;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x)
        cand[i] = make_uint2((uint32_t)(i % m0), (uint32_t)(i / m0));
    if (blockIdx.x == 0 && threadIdx.x == 0) *count = (unsigned)total;
}

struct RefineParams {
    const uint8_t *vec;      // [n][pitch]
    const uint8_t *queries;  // [nq][pitch] zero padded
    int pitch, root;
    const uint2 *cand;
    const unsigned *cand_count;
    unsigned cand_cap;
    const float *U;          // [nq] exact distance bound of this level (strict <)
    uint2 *bucket;           // [nq][bucket_cap] (row, distance bits) kept for each query, unordered
    unsigned *bcount;        // [nq] entries appended this level (may exceed bucket_cap => overflow, seen by replay_kernel)
    unsigned bucket_cap;
    unsigned *stats;         // [0] += candidates refined, [2] |= 1 when the candidate log overflowed
};

constexpr unsigned kBucketCap = 2048;   // kept candidates per query and level (replay_kernel sorts them in shared memory)

// f16 L1 rows of refine_kernel: a copy of special_row_distance of its own.  A noinline function shared with
// scan_kernel<T_F16, MC_L1> is register-allocated for every caller, so sharing it would change the single-query kernel's code.
template <int VT, int MC>
__device__ __noinline__ float refine_special_row_distance(const uint8_t *row, const uint8_t *query, int nelem, int root) {
    return special_row_distance_body<VT, MC>(row, query, nelem, root);
}

// eight lanes per candidate (four candidates per warp step): the reference distance with the arithmetic of the
// single-query kernel; survivors go to their query's bucket (one atomic each on nq different counters; no global sort
// and no host round trip per level: replay_kernel orders each bucket by row itself).
template <int VT, int MC>
__global__ void refine_kernel(const RefineParams rp) {
    constexpr int G = 8;
    const unsigned ncand_raw = *rp.cand_count;
    const unsigned ncand = min(ncand_raw, rp.cand_cap);
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        atomicAdd(&rp.stats[0], ncand);
        if (ncand_raw > rp.cand_cap) atomicOr(&rp.stats[2], 1u);
    }
    const int lane = threadIdx.x & 31, sub = lane & (G - 1), grp = lane / G;
    const unsigned wpb = blockDim.x >> 5, per_step = 32 / G;
    const int nc = rp.pitch / 16;
    const unsigned steps = (ncand + per_step - 1) / per_step;
    for (unsigned st = blockIdx.x * wpb + (threadIdx.x >> 5); st < steps; st += gridDim.x * wpb) {
        const unsigned c = st * per_step + grp;
        const bool live = c < ncand;
        uint2 cq = make_uint2(0, 0);
        if (live) cq = rp.cand[c];
        const uint4 *rowp = reinterpret_cast<const uint4 *>(rp.vec + (size_t)cq.x * rp.pitch);
        const uint4 *qp = reinterpret_cast<const uint4 *>(rp.queries + (size_t)cq.y * rp.pitch);
        Accum A = {0.f, 0.f, 0.f, 0, 0};
        QueryNorm qn = {0.f, 0};
        if (live) {
            for (int i = sub; i < nc; i += G) {
                const uint4 rv = __ldg(rowp + i), qv = __ldg(qp + i);
                accum16<VT, MC>(A, rv, qv);
                if constexpr (VT == T_U8) {
                    qn.i = (int)__dp4a(qv.x, qv.x, (uint32_t)qn.i); qn.i = (int)__dp4a(qv.y, qv.y, (uint32_t)qn.i);
                    qn.i = (int)__dp4a(qv.z, qv.z, (uint32_t)qn.i); qn.i = (int)__dp4a(qv.w, qv.w, (uint32_t)qn.i);
                } else if constexpr (VT == T_I8) {
                    qn.i = __dp4a((int)qv.x, (int)qv.x, qn.i); qn.i = __dp4a((int)qv.y, (int)qv.y, qn.i);
                    qn.i = __dp4a((int)qv.z, (int)qv.z, qn.i); qn.i = __dp4a((int)qv.w, (int)qv.w, qn.i);
                } else if constexpr (MC == MC_COS) {
                    constexpr int NE = (VT == T_F32) ? 4 : 8;                   // unpack8 writes 4 floats for f32
                    float x[8];
                    unpack8<VT>(qv, x);
#pragma unroll
                    for (int j = 0; j < NE; ++j) qn.f = fmaf(x[j], x[j], qn.f);
                }
            }
        }
        accum_reduce(A, G);
        for (int off = G / 2; off >= 1; off >>= 1) {
            qn.f += __shfl_xor_sync(0xFFFFFFFFu, qn.f, off);
            qn.i += __shfl_xor_sync(0xFFFFFFFFu, qn.i, off);
        }
        float d = finalize<VT, MC>(A, qn, rp.root);
        if constexpr (has_special_policy<VT, MC>()) {       // rows (or queries) holding NaN / Inf: the reference's own element loop
            if (live && sub == 0 && row_needs_exact<VT, MC>(A, qn)) {
                const uint8_t *r8 = reinterpret_cast<const uint8_t *>(rowp), *q8 = reinterpret_cast<const uint8_t *>(qp);
                if constexpr (MC == MC_L1) d = refine_special_row_distance<VT, MC>(r8, q8, rp.pitch / 2, rp.root);
                else d = special_row_distance<VT, MC>(r8, q8, rp.pitch / 2, rp.root);
            }
        }
        const bool keep = live && sub == 0 && d < rp.U[cq.y];
        if (keep) {
            const unsigned w = atomicAdd(&rp.bcount[cq.y], 1u);
            if (w < rp.bucket_cap) rp.bucket[(size_t)cq.y * rp.bucket_cap + w] = make_uint2(cq.x, __float_as_uint(d));
        }
    }
}

// final exchange sort of each query's slots, literally the loop of vFullScanSortSlots (src/sqlite-vector.c:2057-2065):
// one thread per query, its k slots staged in shared memory.  Unused slots stay +INF and sort to the end.
__global__ void final_sort_kernel(float *slot_d, unsigned *slot_row, int nq, int k, int kcap) {
    extern __shared__ __align__(16) uint8_t fsm2[];
    const int stride = k | 1;                                        // odd stride: conflict-free per-thread rows
    float *sd = reinterpret_cast<float *>(fsm2) + (size_t)threadIdx.x * stride;
    unsigned *sr = reinterpret_cast<unsigned *>(reinterpret_cast<float *>(fsm2) + (size_t)blockDim.x * stride) + (size_t)threadIdx.x * stride;
    const int q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= nq) return;
    float *gd = slot_d + (size_t)q * kcap;
    unsigned *gr = slot_row + (size_t)q * kcap;
    for (int j = 0; j < k; ++j) { sd[j] = gd[j]; sr[j] = gr[j]; }
    for (int i = 0; i + 1 < k; ++i) {
        float di = sd[i];
        unsigned ri = sr[i];
        for (int j = i + 1; j < k; ++j) {
            const float dj = sd[j];
            if (dj < di) {
                const unsigned rj = sr[j];
                sd[j] = di; sr[j] = ri;
                di = dj; ri = rj;
            }
        }
        sd[i] = di; sr[i] = ri;
    }
    for (int j = 0; j < k; ++j) { gd[j] = sd[j]; gr[j] = sr[j]; }
}

// per-query slot state carried across levels (the reference's cursor arrays, src/sqlite-vector.c:1808-1813)
struct ReplayParams {
    const uint2 *bucket;    // [nq][bucket_cap] (row, distance bits) of this level, unordered
    unsigned *bcount;       // [nq] in: entries of this level; reset to 0 for the next level
    unsigned bucket_cap;
    unsigned *stats;        // [1] += entries replayed, [2] |= 2 when a bucket overflowed
    int nq, k, kcap;
    float *slot_d;          // [nq][kcap]
    unsigned *slot_row;     // [nq][kcap]
    int *slot_mi;           // [nq] max_index
    float *U;               // [nq] out: running k-th distance after this level
    float *qc;              // [NGN] out: conservative constant for the next level
    int mc, vt, root;       // vt: element type (T_*)
    const void *qnorm;      // [nq] float / int sum of squares of each query
    float rnmax;            // max row norm (fp kinds, DOT slack)
    int dim;                // elements per row (fp kinds: slack of the tensor-core score)
    int level0;             // 1: initialise the slots first
    // optional (row-sharded batches): log of the rows that entered the slots, in scan order.  A row that does not
    // enter the slots of its own shard scanned alone cannot enter them in the full scan either (the bound there is
    // tighter), so the concatenation of the shards' logs replayed in shard order reproduces the full scan exactly.
    uint2 *acc_log;         // [nq][acc_cap] (dist bits, local row) or nullptr
    int *acc_count;         // [nq] entries logged so far (may exceed acc_cap => overflow, detected by the merge)
    int acc_cap;
};

// The reference's slot update for up to 32 (distance, row) offers held one per lane, in lane order:
// strict '<' against the slot at max_index (src/sqlite-vector.c:2145), then vFullScanFindMaxIndex (:2022-2049, first
// index of the maximum).  sd/sr: this query's slots (kcap entries, a multiple of 32; entries >= k hold -INF); on_accept(dist,
// row) is called by the whole warp for every offer that enters.  Each lane starts from its own first slot, so when every
// slot is -INF the maximum is slot 0, as in the reference (a lane starting from -INF would never update and leave no index).
template <class F>
__device__ __forceinline__ void warp_offer32(float *sd, unsigned *sr, int kcap, int lane, float d, unsigned row, int &mi, float &cur,
                                             F on_accept) {
    unsigned m = __ballot_sync(0xFFFFFFFFu, d < cur);
    while (m) {
        const int sl = __ffs(m) - 1;
        m &= m - 1;
        const float dv = __shfl_sync(0xFFFFFFFFu, d, sl);
        const unsigned rv = __shfl_sync(0xFFFFFFFFu, row, sl);
        if (dv < cur) {
            if (lane == 0) { sd[mi] = dv; sr[mi] = rv; }
            __syncwarp();
            float best = sd[lane];
            int bi = lane;
            for (int j = lane + 32; j < kcap; j += 32) {
                const float v = sd[j];
                if (v > best) { best = v; bi = j; }
            }
            const uint32_t key = fkey(best);
            const uint32_t mx = __reduce_max_sync(0xFFFFFFFFu, key);
            const int cand = (key == mx) ? bi : 0x7FFFFFFF;
            mi = __reduce_min_sync(0xFFFFFFFFu, cand);
            cur = funkey(mx);
            __syncwarp();                      // every lane has read the slots before lane 0 writes the next accepted offer (racecheck: WAR)
            on_accept(dv, rv);
        }
    }
}

__device__ __forceinline__ float clampf(float x, float lo, float hi) { return fminf(fmaxf(x, lo), hi); }

// Slack of the fp tensor-core score, relative to |q||r| (>= sum |q_i r_i|).  bf16 x bf16 and f16 x f16 products are exact in
// fp32; what is not specified is how the tensor core adds them (block order, alignment to the largest exponent, truncation).  Any
// scheme that keeps 24 bits relative to the largest addend of a block loses < 2^-22 * sum|terms| per addend it aligns, i.e.
// |s_tc - s| <= dim * 2^-21 * sum|q_i r_i| over a row of `dim` products (accumulator re-aligned once per block included).  The
// exact refine adds its own fp32 FMA-chain error (<= dim * 2^-24 * sum|terms|) and the norms carry the same relative error.
// eps = dim * 2^-20 covers the sum of all three with a factor ~1.8 to spare.  (Round 1 used a fixed 1e-4, which is below
// dim * 2^-24 * ... only up to dim ~ 1600: the verdict's weak item 1.)
__host__ __device__ inline float tc_fp_eps(int dim) { return (float)dim * 9.5367431640625e-7f; }

// Bound of the fp L1 score.  l1_batch_kernel and the refine both add the same dim non-negative terms t_i = fl(|x_i - y_i|)
// (one rounding each; padding terms are exact zeros), in different orders.  With u = 2^-24, every term is within u of
// |x_i - y_i| and any summation order of dim terms within gamma_(dim-1) of their sum, so for ANY order the computed sum s
// obeys |s - S| <= gamma S, S = sum |x_i - y_i| exact, gamma = m u / (1 - m u), m = dim + 1 (one to spare).  The refine's
// distance d is s clamped by nearly_zero_float32 (sums <= 8 FLT_EPSILON become 0), so d < U  =>  s_refine <= B = max(U,
// 8 FLT_EPSILON)  =>  S <= B / (1 - gamma)  =>  s_kernel <= B (1 + gamma) / (1 - gamma).  The constant is that bound computed
// in double, widened by 2^-40 for the double arithmetic and rounded up to float, so the kernel's test !(s >= qc) keeps every
// such pair.  A bound beyond FLT_MAX (or U = +INF) returns NaN: every pair is a hit then, also a sum that overflowed to +INF.
__device__ inline float l1_fp_qc(float U, int dim) {
    if (!(U <= FLT_MAX)) return __int_as_float(0x7FC00000);
    const double mu = (double)(dim + 1) * 0x1p-24, gamma = mu / (1.0 - mu);
    const double b = fmax((double)U, 8.0 * (double)FLT_EPSILON) * (1.0 + gamma) / (1.0 - gamma) * (1.0 + 0x1p-40);
    return (b < (double)FLT_MAX) ? __double2float_ru(b) : __int_as_float(0x7FC00000);
}

// conservative per-query constant for tc_hit (or the L1 test of l1_batch_kernel) from the exact bound U (see DESIGN.md §3.4):
// every row whose exact (refine) distance is < U passes the kernel's test with this constant.  vt: element type (T_*).
__device__ inline float conservative_qc(int vt, int mc, int root, float U, const void *qnorm, int q, float rnmax, int dim) {
    const bool INT8 = (vt == T_I8 || vt == T_U8);
    if (mc == MC_L1) return INT8 ? U : l1_fp_qc(U, dim);   // integer sums are exact: the kernel tests (float)S < U like the refine
    if (INT8) {
        const int qi = reinterpret_cast<const int *>(qnorm)[q];
        const double qq = (vt == T_U8) ? (double)(uint32_t)qi : (double)qi;
        if (mc == MC_DOT) {          // d = -(float)s < U  <=  s > -U - 1 - 2e-7|U|
            double b = -(double)U - 1.0 - 2e-7 * fabs((double)U);
            if (!(U < 3.0e38f)) b = -2147483647.0;
            b = fmin(fmax(floor(b), -2147483647.0), 2147483646.0);
            return __int_as_float((int)b);
        }
        if (mc == MC_L2) {           // d2 = qq + nn - 2s <= d2max  <=>  2s - nn >= qq - d2max
            double u2 = root ? (double)U * (double)U : (double)U;
            double d2max = ceil(u2 * (1.0 + 1e-6)) + 1.0;
            if (!(U < 3.0e38f) || !(d2max < 4.0e9)) d2max = 4.0e9;
            double b = fmin(fmax(qq - d2max, -2147483647.0), 2147483646.0);
            return __int_as_float((int)b);
        }
        const float u = fminf(U, 3.0e38f);                                       // cosine
        return clampf((1.0f - u - 1e-5f) * sqrtf((float)qq), -1e30f, 1e30f);
    }
    const float qq = reinterpret_cast<const float *>(qnorm)[q];
    if (!(U < 3.0e38f)) return (mc == MC_COS) ? -1e30f : -INFINITY;
    const float eps = tc_fp_eps(dim);
    // DOT: d = -s < U.  |s_tc - s_refine| <= eps |q||r| <= eps |q| rnmax (rnmax = largest row norm, 1.0001 for its own rounding)
    if (mc == MC_DOT) return -U - (eps * sqrtf(qq) * rnmax * 1.0001f + 4e-7f * fabsf(U)) - 1e-30f;
    if (mc == MC_L2) {
        // a query whose fp32 sum of squares overflowed: NaN makes every row a hit (the refine's distances are exact)
        if (!(qq <= FLT_MAX)) return __int_as_float(0x7FC00000);
        // |q-r|^2 = qq + nn - 2 s: the score error is <= 2 eps_tc |q||r| <= eps_tc (qq + nn), so shrinking both norms by
        // (1 - eps) absorbs it (tc_scan_kernel shrinks nn the same way); the refine's own sum of squares is within
        // dim * 2^-23 relative of the true one, hence the factor on U^2
        const float u2 = root ? U * U : U;
        return qq * (1.0f - eps) - u2 * (1.0f + 0.25f * eps + 1e-6f) - 1e-30f;
    }
    return clampf((1.0f - U - eps - 2e-6f) * sqrtf(qq), -1e30f, 1e30f);             // cosine: s > (1 - U - slack) |q||r|
}

// the constants replay_kernel would derive from the bounds U[nq] (vsb_debug_tc_level: one tensor-core level in isolation)
__global__ void conservative_qc_kernel(float *qc, const float *U, int nq, int vt, int mc, int root, const void *qnorm, float rnmax, int dim) {
    const int q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q < nq) qc[q] = conservative_qc(vt, mc, root, U[q], qnorm, q, rnmax, dim);
}

constexpr int kReplayThreads = 128;

// one block per query: order this level's kept candidates by row (bitonic sort in shared memory), then one warp feeds them
// through the reference's slot update.  The slots live in shared memory while the block works on them.
__global__ void __launch_bounds__(kReplayThreads) replay_kernel(const ReplayParams rp) {
    __shared__ unsigned long long keys[kBucketCap];          // (row << 32) | distance bits
    __shared__ float sd[256];
    __shared__ unsigned sr[256];
    const int q = blockIdx.x;
    const int tid = threadIdx.x, lane = tid & 31;
    float *gd = rp.slot_d + (size_t)q * rp.kcap;
    unsigned *gr = rp.slot_row + (size_t)q * rp.kcap;
    const unsigned c_raw = rp.bcount[q];
    const unsigned c = min(c_raw, rp.bucket_cap);
    unsigned n = 32;
    while (n < c) n <<= 1;
    const uint2 *bk = rp.bucket + (size_t)q * rp.bucket_cap;
    for (unsigned i = tid; i < n; i += kReplayThreads) {
        unsigned long long key = ~0ull;
        if (i < c) { const uint2 e = bk[i]; key = ((unsigned long long)e.x << 32) | e.y; }
        keys[i] = key;
    }
    for (int j = tid; j < rp.kcap; j += kReplayThreads) {
        if (rp.level0) { sd[j] = (j < rp.k) ? INFINITY : -INFINITY; sr[j] = 0; }
        else { sd[j] = gd[j]; sr[j] = gr[j]; }
    }
    __syncthreads();
    for (unsigned size = 2; size <= n; size <<= 1) {
        for (unsigned stride = size >> 1; stride > 0; stride >>= 1) {
            for (unsigned t = tid; t < (n >> 1); t += kReplayThreads) {
                const unsigned i = ((t & ~(stride - 1)) << 1) | (t & (stride - 1)), j = i + stride;
                const unsigned long long a = keys[i], b = keys[j];
                const bool up = (i & size) == 0;
                if ((a > b) == up) { keys[i] = b; keys[j] = a; }
            }
            __syncthreads();
        }
    }
    if (tid < 32) {
        int mi = rp.level0 ? 0 : rp.slot_mi[q];
        float cur = sd[mi];
        int acc_n = (rp.acc_log != nullptr && !rp.level0) ? rp.acc_count[q] : 0;
        uint2 *alog = rp.acc_log ? rp.acc_log + (size_t)q * rp.acc_cap : nullptr;
        for (unsigned base = 0; base < c; base += 32) {
            const unsigned i = base + lane;
            const unsigned long long key = (i < c) ? keys[i] : 0ull;
            const float d = (i < c) ? __uint_as_float((unsigned)(key & 0xFFFFFFFFu)) : INFINITY;
            const unsigned row = (unsigned)(key >> 32);
            warp_offer32(sd, sr, rp.kcap, lane, d, row, mi, cur, [&](float dv, unsigned rv) {
                if (alog != nullptr && lane == 0 && acc_n < rp.acc_cap) alog[acc_n] = make_uint2(__float_as_uint(dv), rv);
                ++acc_n;
            });
        }
        if (lane == 0) {
            rp.slot_mi[q] = mi;
            rp.U[q] = cur;
            rp.qc[q] = conservative_qc(rp.vt, rp.mc, rp.root, cur, rp.qnorm, q, rp.rnmax, rp.dim);
            if (rp.acc_log != nullptr) rp.acc_count[q] = acc_n;
            rp.bcount[q] = 0;
            atomicAdd(&rp.stats[1], c);
            if (c_raw > rp.bucket_cap) atomicOr(&rp.stats[2], 2u);
        }
    }
    __syncthreads();
    for (int j = tid; j < rp.kcap; j += kReplayThreads) { gd[j] = sd[j]; gr[j] = sr[j]; }
}

// ------------------------------------------------------------------ row-sharded batches: merge of the shards' entry logs
// block of one shard: [hdr 64 B: nq, k, acc_cap, 0...][counts: int x round_up(nq,16)][log: nq x acc_cap x uint2]
__host__ __device__ inline size_t acc_block_counts_off() { return 64; }
__host__ __device__ inline size_t acc_block_log_off(int nq) { return 64 + 4 * (size_t)((nq + 15) & ~15); }
__host__ __device__ inline size_t acc_block_bytes(int nq, int acc_cap) { return acc_block_log_off(nq) + 8 * (size_t)nq * acc_cap; }

struct MergeParams {
    const uint8_t *blocks;      // world blocks, block r at blocks + r * block_stride (device memory)
    long long block_stride;
    int world, nq, k, kcap, acc_cap;
    const long long *first_seq; // [world] global scan-order index of each shard's first row (device)
    float *slot_d;              // [nq][kcap] out
    unsigned *slot_row;         // [nq][kcap] out: GLOBAL row index
    int *status;                // [0] |= 1 when a shard's log overflowed, |= 2 on a malformed block, |= 8 when a global row
                                // (first_seq + local row) does not fit 32 bits
};

// one warp per query: the shards' logs, in shard (= scan) order, through the reference's slot update
__global__ void merge_logs_kernel(const MergeParams mp) {
    const int q = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (q >= mp.nq) return;
    float *sd = mp.slot_d + (size_t)q * mp.kcap;
    unsigned *sr = mp.slot_row + (size_t)q * mp.kcap;
    for (int j = lane; j < mp.kcap; j += 32) { sd[j] = (j < mp.k) ? INFINITY : -INFINITY; sr[j] = 0; }
    __syncwarp();
    int mi = 0;
    float cur = INFINITY;
    for (int r = 0; r < mp.world; ++r) {
        const uint8_t *blk = mp.blocks + (size_t)r * (size_t)mp.block_stride;
        const int *hdr = reinterpret_cast<const int *>(blk);
        if (hdr[0] != mp.nq || hdr[1] != mp.k || hdr[2] != mp.acc_cap) {
            if (lane == 0) atomicOr(mp.status, 2);
            return;
        }
        if (hdr[3] != 0) {                      // the shard's levels exceeded a capacity (pushed blocks carry the flag, see push_logs_kernel)
            if (lane == 0) atomicOr(mp.status, 1);
            return;
        }
        const int cnt = reinterpret_cast<const int *>(blk + acc_block_counts_off())[q];
        if (cnt > mp.acc_cap) {
            if (lane == 0) atomicOr(mp.status, 1);
            return;
        }
        const uint2 *lg = reinterpret_cast<const uint2 *>(blk + acc_block_log_off(mp.nq)) + (size_t)q * mp.acc_cap;
        const unsigned long long base_row = (unsigned long long)mp.first_seq[r];
        for (int base = 0; base < cnt; base += 32) {
            const int i = base + lane;
            const uint2 e = (i < cnt) ? lg[i] : make_uint2(0x7F800000u, 0u);
            if (__any_sync(0xFFFFFFFFu, i < cnt && base_row + e.y > 0xFFFFFFFFull)) {   // the slots carry 32-bit global rows
                if (lane == 0) atomicOr(mp.status, 8);
                return;
            }
            warp_offer32(sd, sr, mp.kcap, lane, __uint_as_float(e.x), (unsigned)(base_row + e.y), mi, cur, [](float, unsigned) {});
        }
    }
}

// ------------------------------------------------------------------ row-sharded batches: entry logs over NVLink peer memory
// The counterpart of the head push in filter_kernel for the batched path: after the last level every shard stores the USED
// part of its entry-log block (header, counts, `count` entries per query) into row `src` of every target's log area and raises
// the target's flag when all of its blocks have fenced.  grid = (targets, slices); the header travels with the shard's overflow
// flags (stats[2]) in hdr[3], so every rank reaches the same verdict without a host round trip.
// a few integers passed by value to device memory (headers, shard offsets): keeps pageable host copies, which can make the
// host wait for the stream, out of the pipelined paths
struct SmallInts { int n; long long v[16]; };
__global__ void store_ints_kernel(long long *out64, int *out32, const SmallInts s) {
    const int i = threadIdx.x;
    if (i < s.n) {
        if (out64) out64[i] = s.v[i];
        if (out32) out32[i] = (int)s.v[i];
    }
}

struct LogPushParams {
    const uint8_t *block;        // local entry-log block (acc_block layout)
    const unsigned *stats;       // [2] = overflow flags of this batch's levels
    int nq, acc_cap;
    int ntargets, src, world, buf;
    unsigned bseq;
    unsigned long long slot_stride;   // bytes between the rows of a target's log area
    uint8_t *xlog[kMaxPeers];    // target t: base of its log area [2][world][slot_stride]
    unsigned *lflags[kMaxPeers]; // target t: [2][world] arrival flags
    unsigned *done;              // [targets] local block counters (zero before the launch, re-armed by the last block)
};
__global__ void push_logs_kernel(const LogPushParams lp) {
    const int t = blockIdx.x, S = gridDim.y, j = blockIdx.y;
    uint8_t *dst = lp.xlog[t] + ((size_t)lp.buf * lp.world + lp.src) * lp.slot_stride;
    const size_t log_off = acc_block_log_off(lp.nq);
    if (j == 0) {                                                   // header + counts
        const uint32_t *src32 = reinterpret_cast<const uint32_t *>(lp.block);
        uint32_t *d32 = reinterpret_cast<uint32_t *>(dst);
        for (size_t i = threadIdx.x; i < log_off / 4; i += blockDim.x) d32[i] = (i == 3) ? lp.stats[2] : src32[i];
    }
    const int *counts = reinterpret_cast<const int *>(lp.block + acc_block_counts_off());
    for (int q = j; q < lp.nq; q += S) {
        const int cnt = min(max(counts[q], 0), lp.acc_cap);
        const uint2 *s2 = reinterpret_cast<const uint2 *>(lp.block + log_off) + (size_t)q * lp.acc_cap;
        uint2 *d2 = reinterpret_cast<uint2 *>(dst + log_off) + (size_t)q * lp.acc_cap;
        for (int i = threadIdx.x; i < cnt; i += blockDim.x) d2[i] = s2[i];
    }
    __threadfence_system();
    __syncthreads();
    if (threadIdx.x == 0) {
        const unsigned prev = atomicAdd(&lp.done[t], 1u);
        if (prev == (unsigned)S - 1u) {                              // every block of this target has fenced its stores
            lp.done[t] = 0u;
            st_release_sys(lp.lflags[t] + (size_t)lp.buf * lp.world + lp.src, lp.bseq);
        }
    }
}
// receiving side: wait until the `n` flags carry `expect`; bounded (status |= 4 on timeout)
__global__ void log_wait_kernel(const unsigned *flags, int n, unsigned expect, long long timeout, int *status) {
    const int t = threadIdx.x;
    if (t >= n) return;
    const long long t0 = clock64();
    while (ld_acquire_sys(flags + t) != expect) {
        if (clock64() - t0 > timeout) { atomicOr(status, 4); break; }
        __nanosleep(200);
    }
}

__global__ void fill_kernel(float *p, float v, int n) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) p[i] = v;
}

__global__ void max_norm_kernel(const float *norms, long long n, float *out) {   // out must be zeroed; norms >= 0
    float m = 0.0f;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) m = fmaxf(m, norms[i]);
    for (int off = 16; off >= 1; off >>= 1) m = fmaxf(m, __shfl_xor_sync(0xFFFFFFFFu, m, off));
    if ((threadIdx.x & 31) == 0) atomicMax(reinterpret_cast<int *>(out), __float_as_int(m));
}

}  // namespace vsb
