// scan_kernels.cuh — sm_90a kernels of the single-query (HBM-bound) distance scan.
//
// Replaces, for a whole resident shard at once, the per-row loop of the reference:
//   fn = dispatch_distance_table[metric][type]; d = fn(q,row,dim); clamp; slot update
//   (/root/reference/src/sqlite-vector.c:2089-2107 and :2138-2153, kernels in src/distance-cpu.c:39-693).
//
// Design (see DESIGN.md §3):
//   * corpus rows are dense in HBM ([n][pitch], pitch = dim*elt rounded up to 16 B, zero padded);
//   * every WARP owns a contiguous range of rows ("stream") and pulls it through its own ring of
//     shared-memory stages with TMA bulk copies (cp.async.bulk + mbarrier complete_tx) that it issues
//     itself — no block-level barrier anywhere in the steady state;
//   * P = 1..32 lanes cooperate on a row; 16-byte LDS with a per-row rotation keeps the shared-memory
//     reads conflict-free; integer types use dp4a / vabsdiff4 (exact int32), fp types FFMA;
//   * top-k: each warp keeps the k smallest distances of its own stream in shared memory and logs every
//     row that beats the running k-th value (strict <).  That log is a superset of the rows that can
//     ever enter the reference's k slots; filter_kernel tightens it with prefix thresholds and the
//     host replays the reference's slot algorithm over the few hundred survivors, which reproduces
//     the reference's history-dependent tie handling exactly.
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <float.h>
#include <stddef.h>
#include <stdint.h>

namespace vsb {

constexpr int kWarps = 8;             // consumer warps per CTA (each one is a stream)
constexpr int kThreads = kWarps * 32;
constexpr int kMaxStages = 8;         // ring stages per warp
constexpr int kBarrierBytes = 1024;   // reserved at the start of dynamic smem for mbarriers + scalars

enum { T_F32 = 1, T_F16 = 2, T_BF16 = 3, T_U8 = 4, T_I8 = 5 };
enum { MC_L2 = 0, MC_COS = 1, MC_DOT = 2, MC_L1 = 3 };  // L2 and SQUARED_L2 share a kernel (root flag)

constexpr int kMaxGroup = 8;          // queries of one exchange group (vsb_exchange_submit): heads waited for and pushed together
constexpr int kMaxPass = 8;           // queries scored in one pass of the column (scan_pass_kernel's widest compile-time width)

// One scan launch is a pass: it reads every row of the column once and scores it against nq <= M queries.  Query j
// has its own k-lists, logs, counts and in-CTA bounds at j times the per-query stride of each workspace array (pass_lists
// and friends), and its own overflow flag ctrl[j][1].
struct ScanParams {
    const uint8_t *vec;   // [n][pitch]
    long long n;
    int pitch;            // bytes per row (multiple of 16)
    int nc;               // 16-byte chunks per row
    int log2P;            // lanes per row = 1 << log2P
    int wtile_bytes;      // (32 >> log2P) * pitch
    int nsw;              // ring stages per warp
    int root;             // metric L2: take the square root
    int k;                // 0 => no top-k (dist_all only)
    int kcap;             // k rounded up to 32
    int logcap;
    int nq;               // queries of the pass (1 .. the kernel's M)
    const uint8_t *query[kMaxPass]; // device, pitch bytes each, zero padded
    float *lists;         // k <= 32: [CTAs][32] the k smallest distances of each CTA's rows, sorted ascending, +INF padded;
                          // k > 32:  [streams][kcap] k smallest distances of each stream (unsorted)
    float *tlocal;        // k <= 32: [streams] k-th smallest distance over the EARLIER streams of the same CTA (+INF if < k rows)
    uint2 *logs;          // [streams][logcap] (dist bits, local row)
    int *counts;          // [streams] log entries written (may exceed logcap => overflow)
    int *ctrl[kMaxPass];  // ctrl[j][1] = overflow flag of query j
    float *dist_all;      // optional [n]
    // adaptive row partition (optional): bounds[c] .. bounds[c+1] are the warp-tiles of CTA c (contiguous, ascending, any
    // sizes: the exactness argument only needs streams to be contiguous row ranges in scan order).  Each CTA reports the
    // cycles it took; filter_kernel turns speeds into the partition of the query after next (SMs do not all pull from
    // HBM at the same rate, and with equal shares the slowest one sets the kernel time).
    const long long *bounds;   // [gridDim.x + 1] or nullptr (equal shares)
    unsigned *cta_time;        // [gridDim.x] or nullptr
    // row filter (vsb_scan_topk_filtered): row r of vec is eligible when bit allow_base + r of the shard bitmap `allow` is set;
    // nullptr: every row is.  An ineligible row never enters a k-list or a log (dist_all is written for every row)
    const uint32_t *allow;
    long long allow_base;      // shard row of vec's first row (a window of a streamed index), else 0
    // range mode (scan_range_kernel, vsb_scan_range): every eligible row with d < range_t is appended to range_pairs
    // as (row_base + local row, distance bits) at the position one atomicAdd on *range_count reserves for the warp's ballot; the
    // counter keeps counting past range_cap, so the host sees the exact size of an overflowed list
    float range_t;
    uint2 *range_pairs;        // [range_cap]
    unsigned *range_count;
    long long range_cap;
    unsigned range_row_base;   // shard row of vec's first row, added to the rows written (the windows of a streamed index)
};

// query j's part of the pass workspaces (streams = scan CTAs x kWarps; the filter of query j gets the same offsets)
__host__ __device__ inline size_t pass_lists(int j, long long streams, int kcap) { return (size_t)j * streams * kcap; }
__host__ __device__ inline size_t pass_logs(int j, long long streams, int logcap) { return (size_t)j * streams * logcap; }
__host__ __device__ inline size_t pass_streams(int j, long long streams) { return (size_t)j * streams; }

// bit `row` of a row bitmap (bit row & 31 of word row >> 5); nullptr: every row is eligible
__device__ __forceinline__ bool row_allowed(const uint32_t *allow, long long row) {
    return allow == nullptr || ((__ldg(allow + (row >> 5)) >> (row & 31)) & 1u) != 0u;
}

// ------------------------------------------------------------------ PTX helpers
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t *bar, int count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "WAIT_%=:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra DONE_%=;\n\t"
        "bra WAIT_%=;\n\t"
        "DONE_%=:\n\t}" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
// TMA bulk copy global -> shared, completion signalled on an mbarrier (SASS: UBLKCP)
__device__ __forceinline__ void bulk_g2s(void *dst, const void *src, uint32_t bytes, uint64_t *bar, uint64_t policy) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;" ::"r"(smem_u32(dst)),
        "l"(src), "r"(bytes), "r"(smem_u32(bar)), "l"(policy)
        : "memory");
}
__device__ __forceinline__ uint64_t policy_evict_first() {
    uint64_t p;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
    return p;
}
__device__ __forceinline__ void fence_barrier_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ uint4 ldg_stream(const uint4 *p) {
    uint4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
    return r;
}

// monotone float -> uint32 key (total order, -0 < +0), used for warp-wide max via REDUX
__device__ __forceinline__ uint32_t fkey(float f) {
    uint32_t u = __float_as_uint(f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

// ------------------------------------------------------------------ accumulation
struct Accum {
    float s0, s1;   // fp: primary sum split in two chains (dot / sum of squares / sum of |d|)
    float ny;       // fp cosine: row norm (the query norm is computed once per query, QueryNorm)
    int ia, ib;     // int: dot or sad, row norm
};

template <int VT>
__device__ __forceinline__ void unpack8(const uint4 v, float (&o)[8]) {
    if constexpr (VT == T_F32) {
        o[0] = __uint_as_float(v.x); o[1] = __uint_as_float(v.y); o[2] = __uint_as_float(v.z); o[3] = __uint_as_float(v.w);
    } else if constexpr (VT == T_F16) {
        const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            __half2 h = *reinterpret_cast<const __half2 *>(&w[j]);
            float2 f = __half22float2(h);
            o[2 * j] = f.x; o[2 * j + 1] = f.y;
        }
    } else {  // bf16: value = bits << 16 (src/distance-cpu.h:100-102)
        const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            o[2 * j] = __uint_as_float(w[j] << 16);
            o[2 * j + 1] = __uint_as_float(w[j] & 0xFFFF0000u);
        }
    }
}

// one 16-byte chunk of the row (r) against the same chunk of the query (q).  NORM = false leaves out the row's own terms (its
// norm, A.ib / A.ny), which a pass accumulates once for all its queries
template <int VT, int MC, bool NORM = true>
__device__ __forceinline__ void accum16(Accum &A, const uint4 r, const uint4 q) {
    if constexpr (VT == T_U8 || VT == T_I8) {
        const uint32_t rw[4] = {r.x, r.y, r.z, r.w}, qw[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            if constexpr (MC == MC_L1) {
                // sum |a-b|: per-byte absolute difference, then dot with 1s (exact)
                uint32_t ad = (VT == T_U8) ? __vabsdiffu4(rw[j], qw[j]) : __vabsdiffs4(rw[j], qw[j]);
                A.ia = (int)__dp4a(ad, 0x01010101u, (uint32_t)A.ia);
            } else {
                if constexpr (VT == T_U8) {
                    A.ia = (int)__dp4a(rw[j], qw[j], (uint32_t)A.ia);
                    if constexpr (MC != MC_DOT && NORM) A.ib = (int)__dp4a(rw[j], rw[j], (uint32_t)A.ib);
                } else {
                    A.ia = __dp4a((int)rw[j], (int)qw[j], A.ia);
                    if constexpr (MC != MC_DOT && NORM) A.ib = __dp4a((int)rw[j], (int)rw[j], A.ib);
                }
            }
        }
    } else {
        constexpr int NE = (VT == T_F32) ? 4 : 8;
        float y[8], x[8];
        unpack8<VT>(r, y);
        unpack8<VT>(q, x);
        // Plain IEEE accumulation, no per-element special-value tests: the reference's NaN-lane / infinity policies (f16: all
        // metrics, src/distance-cpu.c:318-466; bf16 L2: :164-197) only matter for rows (or queries) that actually hold a NaN or
        // an infinity, and any such element leaves a non-finite accumulator behind.  Those rows are recomputed with the
        // reference's exact policy by special_row_distance (row_needs_exact below).
#pragma unroll
        for (int j = 0; j < NE; ++j) {
            float &s = (j & 1) ? A.s1 : A.s0;
            if constexpr (MC == MC_L2) {
                const float d = x[j] - y[j];
                s = fmaf(d, d, s);
            } else if constexpr (MC == MC_L1) {
                s += fabsf(x[j] - y[j]);
            } else if constexpr (MC == MC_DOT) {
                s = fmaf(x[j], y[j], s);
            } else {  // cosine
                s = fmaf(x[j], y[j], s);
                if constexpr (NORM) A.ny = fmaf(y[j], y[j], A.ny);
            }
        }
    }
}

// one 16-byte chunk of the row against the same chunk of each of the pass's nq queries (query m's chunk at q + m * qstride).
// The row's norm goes to A[0] only; every accumulator sees its terms in the order of a lone query, so each query's distance
// is bit for bit the one a pass of its own computes.
template <int VT, int MC, int M>
__device__ __forceinline__ void accum16_pass(Accum (&A)[M], const uint4 r, const uint8_t *q, int qstride, int nq) {
    accum16<VT, MC>(A[0], r, *reinterpret_cast<const uint4 *>(q));
#pragma unroll
    for (int m = 1; m < M; ++m)
        if (m < nq) accum16<VT, MC, false>(A[m], r, *reinterpret_cast<const uint4 *>(q + (size_t)m * qstride));
}

struct QueryNorm {
    float f;     // fp: sum x^2 of the query
    int i;       // int: sum q^2 (bit pattern; unsigned for u8)
};

// accumulators -> the float the reference kernel returns, then the nearly-zero clamp
template <int VT, int MC>
__device__ __forceinline__ float finalize(const Accum &A, const QueryNorm qn, int root) {
    float d;
    if constexpr (VT == T_U8 || VT == T_I8) {
        if constexpr (MC == MC_L2) {
            // sum (a-b)^2 = |q|^2 + |row|^2 - 2 q.row, exact in 32-bit (src/distance-avx2.c int32 path;
            // equals the float-accumulating scalar kernel, src/distance-cpu.c:470-502, while sums < 2^24)
            float f;
            if constexpr (VT == T_U8) f = (float)((uint32_t)qn.i + (uint32_t)A.ib - 2u * (uint32_t)A.ia);
            else f = (float)(qn.i + A.ib - 2 * A.ia);
            d = root ? __fsqrt_rn(f) : f;
        } else if constexpr (MC == MC_COS) {
            // src/distance-cpu.c:533-538, 645-650
            if (qn.i == 0 || A.ib == 0) d = 1.0f;
            else {
                float fq = (VT == T_U8) ? (float)(uint32_t)qn.i : (float)qn.i;
                float fr = (VT == T_U8) ? (float)(uint32_t)A.ib : (float)A.ib;
                float fd = (VT == T_U8) ? (float)(uint32_t)A.ia : (float)A.ia;
                float den = __fmul_rn(__fsqrt_rn(fq), __fsqrt_rn(fr));
                d = __fsub_rn(1.0f, __fdiv_rn(fd, den));
            }
        } else if constexpr (MC == MC_DOT) {
            d = (VT == T_U8) ? -(float)(uint32_t)A.ia : -(float)A.ia;
        } else {
            d = (float)(uint32_t)A.ia;
        }
    } else {
        const float s = A.s0 + A.s1;
        if constexpr (MC == MC_L2) d = root ? __fsqrt_rn(s) : s;
        else if constexpr (MC == MC_DOT) d = -s;
        else if constexpr (MC == MC_L1) d = s;
        else {
            if constexpr (VT == T_F16) {
                // src/distance-cpu.c:457-465 (finite inputs; rows with NaN / Inf go through special_row_distance): bad
                // denominator -> 1; clamp cos to [-1,1]
                float den = __fmul_rn(__fsqrt_rn(qn.f), __fsqrt_rn(A.ny));
                if (!(den > 0.0f) || isinf(den) || den != den || isinf(s) || s != s) d = 1.0f;
                else {
                    float c = __fdiv_rn(s, den);
                    c = fminf(1.0f, fmaxf(-1.0f, c));
                    d = 1.0f - c;
                }
            } else {
                // src/distance-cpu.c:105-109, 248-252
                if (qn.f == 0.0f || A.ny == 0.0f) d = 1.0f;
                else d = __fsub_rn(1.0f, __fdiv_rn(s, __fmul_rn(__fsqrt_rn(qn.f), __fsqrt_rn(A.ny))));
            }
        }
    }
    // nearly_zero_float32: |d| <= 8*FLT_EPSILON -> +0.0 (src/sqlite-vector.c:994-996, 2099, 2143)
    return (fabsf(d) <= 8.0f * FLT_EPSILON) ? 0.0f : d;
}

// ------------------------------------------------------------------ rows with NaN / Inf elements (rare path)
// kinds whose reference kernel treats special values differently from IEEE propagation
template <int VT, int MC>
__host__ __device__ constexpr bool has_special_policy() { return VT == T_F16 || (VT == T_BF16 && MC == MC_L2); }

// after accum_reduce: does this row (or the query) hold a NaN / Inf, or did its fp32 sum overflow?  f16 sums of finite inputs
// cannot overflow (values <= 65504), but a bf16 L2 sum of squares does once a difference exceeds 2^64 (or the sum FLT_MAX),
// while the reference's double LASSQ stays finite as long as the root does: special_row_distance recomputes those rows in double.
template <int VT, int MC>
__device__ __forceinline__ bool row_needs_exact(const Accum &A, const QueryNorm qn) {
    if constexpr (!has_special_policy<VT, MC>()) return false;
    else if constexpr (MC == MC_COS) return !(fabsf(A.s0 + A.s1) <= FLT_MAX) || !(A.ny <= FLT_MAX) || !(qn.f <= FLT_MAX);
    else return !(fabsf(A.s0 + A.s1) <= FLT_MAX);
}

// The reference's own element loop for one row, one thread, element order (f16: fp32 accumulation instead of double: the result
// classes — NaN, +Inf, -Inf, 1.0 — are exact, finite values agree to ~dim * 2^-24; bf16 L2 accumulates in double, because a
// finite LASSQ value can lie beyond the fp32 range of the sum of squares, up to (float)sqrt(sum) <= FLT_MAX):
//   f16 L2 / L1 (:318-400): a lane with an infinity that is not paired with an equal-signed infinity -> +INF at once (checked
//       BEFORE the NaN test); NaN lanes skipped; Inf - Inf poisons the sum (LASSQ: NaN unless every other difference is 0)
//   f16 DOT (:402-432): NaN lanes skipped; the FIRST infinite product decides: -INF if positive, +INF if negative; Inf * 0 poisons
//   f16 COSINE (:434-466): NaN lanes skipped; any infinity -> 1; bad denominator / non-finite dot -> 1; clamp to [-1, 1]
//   bf16 L2 (:164-197): float difference; infinite difference -> +INF; NaN difference skipped
template <int VT, int MC>
__device__ __forceinline__ float special_row_distance_body(const uint8_t *row, const uint8_t *query, int nelem, int root) {
    const uint16_t *yb = reinterpret_cast<const uint16_t *>(row), *xb = reinterpret_cast<const uint16_t *>(query);
    float s = 0.0f, nx = 0.0f, ny = 0.0f;
    double sd = 0.0;                                                            // bf16 L2
    bool poisoned = false, anynz = false;
    for (int e = 0; e < nelem; ++e) {
        float xf, yf;
        if constexpr (VT == T_F16) {
            xf = __half2float(__ushort_as_half(xb[e]));
            yf = __half2float(__ushort_as_half(yb[e]));
        } else {
            xf = __uint_as_float((uint32_t)xb[e] << 16);
            yf = __uint_as_float((uint32_t)yb[e] << 16);
        }
        if constexpr (VT == T_BF16) {                                           // bf16 L2
            const float d = xf - yf;
            if (isinf(d)) return INFINITY;
            if (d == d) sd = fma((double)d, (double)d, sd);                     // exact square: |d| < 2^128 fits double's range
        } else if constexpr (MC == MC_L2 || MC == MC_L1) {
            const bool xi = isinf(xf), yi = isinf(yf);
            if ((xi || yi) && !(xi && yi && (xf > 0.0f) == (yf > 0.0f))) return INFINITY;
            if (xf != xf || yf != yf) continue;
            const float d = xf - yf;                                            // NaN for an equal-signed pair of infinities
            if (d != d) poisoned = true;
            else {
                if (d != 0.0f) anynz = true;
                s = (MC == MC_L2) ? fmaf(d, d, s) : s + fabsf(d);
            }
        } else {
            if (xf != xf || yf != yf) continue;
            if constexpr (MC == MC_DOT) {
                const float p = xf * yf;                                        // exact for f16 inputs; infinite iff an input is
                if (isinf(p)) return p > 0.0f ? -INFINITY : INFINITY;
                s += p;                                                         // Inf * 0 = NaN poisons, like `dot += p`
            } else {
                if (isinf(xf) || isinf(yf)) return 1.0f;
                s = fmaf(xf, yf, s); nx = fmaf(xf, xf, nx); ny = fmaf(yf, yf, ny);
            }
        }
    }
    float d;
    if constexpr (VT == T_BF16) {
        d = (float)(root ? sqrt(sd) : sd);                                     // rounded once, like lassq_result (+Inf beyond FLT_MAX)
    } else if constexpr (MC == MC_L2) {
        if (poisoned) d = anynz ? __int_as_float(0x7FC00000) : 0.0f;           // LASSQ: scale == 0 -> 0 (:346 / :194)
        else d = root ? __fsqrt_rn(s) : s;
    } else if constexpr (MC == MC_L1) {
        d = poisoned ? __int_as_float(0x7FC00000) : s;
    } else if constexpr (MC == MC_DOT) {
        d = -s;
    } else {
        const float den = __fmul_rn(__fsqrt_rn(nx), __fsqrt_rn(ny));
        if (!(den > 0.0f) || isinf(den) || den != den || isinf(s) || s != s) d = 1.0f;
        else d = 1.0f - fminf(1.0f, fmaxf(-1.0f, __fdiv_rn(s, den)));
    }
    return (fabsf(d) <= 8.0f * FLT_EPSILON) ? 0.0f : d;
}
// out of line: the rare path stays out of the hot loop's registers
template <int VT, int MC>
__device__ __noinline__ float special_row_distance(const uint8_t *row, const uint8_t *query, int nelem, int root) {
    return special_row_distance_body<VT, MC>(row, query, nelem, root);
}

template <bool NORM = true>
__device__ __forceinline__ void accum_reduce(Accum &A, int P) {
    for (int off = P >> 1; off >= 1; off >>= 1) {
        A.s0 += __shfl_xor_sync(0xFFFFFFFFu, A.s0, off);
        A.s1 += __shfl_xor_sync(0xFFFFFFFFu, A.s1, off);
        if constexpr (NORM) A.ny += __shfl_xor_sync(0xFFFFFFFFu, A.ny, off);
        A.ia += __shfl_xor_sync(0xFFFFFFFFu, A.ia, off);
        if constexpr (NORM) A.ib += __shfl_xor_sync(0xFFFFFFFFu, A.ib, off);
    }
}

// ------------------------------------------------------------------ warp-private k-smallest list
// list[0..kcap) in shared memory: entries < k start at +INF, entries >= k at -INF (never the max).
// Returns the current maximum (= running k-th smallest, +INF until k rows were seen) and its position.
__device__ __forceinline__ void list_argmax(const float *list, int kcap, int lane, float &thr, int &pos) {
    float best = list[lane];
    int bi = lane;
    for (int j = lane + 32; j < kcap; j += 32) {
        float v = list[j];
        if (v > best) { best = v; bi = j; }
    }
    uint32_t key = fkey(best);
    uint32_t mx = __reduce_max_sync(0xFFFFFFFFu, key);
    int src = __ffs(__ballot_sync(0xFFFFFFFFu, key == mx)) - 1;
    thr = __shfl_sync(0xFFFFFFFFu, best, src);
    pos = __shfl_sync(0xFFFFFFFFu, bi, src);
}

// bitonic sort of one value per lane, ascending by lane
__device__ __forceinline__ float warp_sort_asc(float v, int lane) {
#pragma unroll
    for (int size = 2; size <= 32; size <<= 1) {
#pragma unroll
        for (int stride = size >> 1; stride >= 1; stride >>= 1) {
            const float o = __shfl_xor_sync(0xFFFFFFFFu, v, stride);
            const bool up = ((lane & size) == 0);            // ascending block?
            const bool lower = ((lane & stride) == 0);
            v = (lower == up) ? fminf(v, o) : fmaxf(v, o);
        }
    }
    return v;
}
// v is a bitonic sequence across the lanes -> ascending
__device__ __forceinline__ float warp_bitonic_merge_asc(float v, int lane) {
#pragma unroll
    for (int stride = 16; stride >= 1; stride >>= 1) {
        const float o = __shfl_xor_sync(0xFFFFFFFFu, v, stride);
        v = ((lane & stride) == 0) ? fminf(v, o) : fmaxf(v, o);
    }
    return v;
}

__device__ __forceinline__ float funkey(uint32_t k) {  // inverse of fkey
    return __uint_as_float((k & 0x80000000u) ? (k & 0x7FFFFFFFu) : ~k);
}

// k <= 32: the warp's k-list lives in one register per lane, SORTED ascending (lanes >= k hold +INF); the running
// k-th value is lane k-1.  Incoming lists are sorted too (scan_kernel publishes them that way), so an offer is either
// a couple of shift-inserts or one bitonic merge — no serial chain of k inserts for the first streams of a segment.
struct SortedList {
    float v, thr;
    int k;
    __device__ __forceinline__ void init(int lane, int k_) { k = k_; v = INFINITY; thr = INFINITY; }
    __device__ __forceinline__ void insert(int lane, float dv) {           // dv < thr
        const int pos = __popc(__ballot_sync(0xFFFFFFFFu, v <= dv));       // elements that stay in front of dv
        const float up = __shfl_up_sync(0xFFFFFFFFu, v, 1);
        v = (lane < pos) ? v : (lane == pos ? dv : up);
        if (lane >= k) v = INFINITY;
        thr = __shfl_sync(0xFFFFFFFFu, v, k - 1);
    }
    // val: a sorted ascending list, one value per lane, +INF padded
    __device__ __forceinline__ void offer_sorted(int lane, float val) {
        const int cnt = __popc(__ballot_sync(0xFFFFFFFFu, val < thr));     // these are the first cnt lanes
        if (cnt == 0) return;
        if (cnt <= 2) {
            const float a = __shfl_sync(0xFFFFFFFFu, val, 0);
            insert(lane, a);
            if (cnt == 2) {
                const float b = __shfl_sync(0xFFFFFFFFu, val, 1);
                if (b < thr) insert(lane, b);
            }
            return;
        }
        // 32 smallest of the 64 values: min(L[i], R[31-i]) is bitonic; one merge network sorts it
        const float rev = __shfl_sync(0xFFFFFFFFu, val, 31 - lane);
        v = warp_bitonic_merge_asc(fminf(v, rev), lane);
        if (lane >= k) v = INFINITY;
        thr = __shfl_sync(0xFFFFFFFFu, v, k - 1);
    }
};

// ------------------------------------------------------------------ the scan kernel
// One launch is one pass over the shard: scan_kernel (one query: top-k, all distances), scan_pass_kernel (top-k for nq <= M
// queries scored against every staged row) and scan_range_kernel (range search, one query) share this body.  Each query keeps its own running k-th value, k-list, log and counts; the streams are the same contiguous
// row ranges for every query, so the exactness argument of a lone query (DESIGN §3.1) holds for each one unchanged.
// RANGE: the fixed threshold prm.range_t instead of the k-lists, hits appended to prm.range_pairs (no log, no lists, no
// filter_kernel afterwards).
template <int VT, int MC, bool DIRECT, bool RANGE, int M>
__device__ __forceinline__ void scan_body(const ScanParams &prm) {
    static_assert(M >= 1 && M <= kMaxPass && (!RANGE || M == 1), "range search scans one query per pass");
    extern __shared__ __align__(1024) uint8_t smem[];
    const int nq = (M == 1) ? 1 : prm.nq;
    uint64_t *bars = reinterpret_cast<uint64_t *>(smem);                    // [kWarps][kMaxStages]
    uint8_t *qs = smem + kBarrierBytes;                                      // [nq][pitch] the queries
    float *lists_s = reinterpret_cast<float *>(qs + nq * prm.pitch);         // [kWarps][nq][kcap]
    uint8_t *ring = qs + ((nq * (prm.pitch + kWarps * prm.kcap * 4) + 127) & ~127); // [kWarps][nsw][wtile_bytes]

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int P = 1 << prm.log2P, rpw = 32 >> prm.log2P;
    const int nsw = prm.nsw;
    const long long clk0 = clock64();

    // ---- prologue: barriers, queries
    if (tid == 0) {
        for (int i = 0; i < kWarps * kMaxStages; ++i) mbar_init(&bars[i], 1);
        fence_barrier_init();
    }
#pragma unroll
    for (int m = 0; m < M; ++m)
        if (m < nq)
            for (int i = tid; i < prm.nc; i += kThreads)
                reinterpret_cast<uint4 *>(qs + m * prm.pitch)[i] = reinterpret_cast<const uint4 *>(prm.query[m])[i];
    __syncthreads();

    // ---- this warp's stream: a contiguous range of warp-tiles (rpw rows each)
    const long long S = (long long)gridDim.x * kWarps;
    const long long sidx = (long long)blockIdx.x * kWarps + warp;
    const long long T = (prm.n + rpw - 1) / rpw;
    long long c0, c1;                                                        // this CTA's warp-tiles
    if (prm.bounds != nullptr) { c0 = prm.bounds[blockIdx.x]; c1 = prm.bounds[blockIdx.x + 1]; }
    else { c0 = (T * blockIdx.x) / gridDim.x; c1 = (T * (blockIdx.x + 1)) / gridDim.x; }
    const long long t0 = c0 + ((c1 - c0) * warp) / kWarps, t1 = c0 + ((c1 - c0) * (warp + 1)) / kWarps;
    const int ntiles = (int)(t1 - t0);

    uint64_t *mybars = bars + warp * kMaxStages;
    uint8_t *myring = ring + (size_t)warp * nsw * prm.wtile_bytes;
    const uint64_t pol = policy_evict_first();

    // the tile fetched into the stage just freed is always the one nsw positions ahead
    int pf_it = 0;                                                           // stream tile index of the next fetch (lane 0)
    auto issue = [&](int s) {  // lane 0 only: next tile of the stream into stage s
        const long long row0 = (t0 + pf_it) * rpw;
        long long rows = prm.n - row0;
        if (rows > rpw) rows = rpw;
        const uint32_t bytes = (uint32_t)rows * (uint32_t)prm.pitch;
        mbar_expect_tx(&mybars[s], bytes);
        bulk_g2s(myring + (size_t)s * prm.wtile_bytes, prm.vec + (size_t)row0 * prm.pitch, bytes, &mybars[s], pol);
        ++pf_it;
    };
    if constexpr (!DIRECT) {
        if (lane == 0)
            for (int s = 0; s < nsw && pf_it < ntiles; ++s) issue(s);
    }
    int stage = 0;                                                           // ring position of the next tile to consume
    uint32_t parity = 0;

    const int r = lane >> prm.log2P, p = lane & (P - 1);
    const int cnt = (prm.nc > p) ? (prm.nc - p + P - 1) >> prm.log2P : 0;  // chunks owned by this lane
    const int i0 = cnt ? (r % cnt) : 0;                                       // rotation: conflict-free LDS.128
    const bool topk = !RANGE && prm.k > 0;
    constexpr bool kFix16 = has_special_policy<VT, MC>();   // rows with NaN / Inf are recomputed from the staged tile: see special_row_distance
    const uint8_t *fix_row = nullptr;
    int fix_stage = 0;

    // query norms (every warp computes them the same way: lane-strided chunks, butterfly sum)
    QueryNorm qn[M];
#pragma unroll
    for (int m = 0; m < M; ++m) {
        float f = 0.0f;
        int iq = 0;
        const uint8_t *qm = qs + m * prm.pitch;
        for (int c = lane; c < prm.nc && m < nq; c += 32) {
            const uint4 q = reinterpret_cast<const uint4 *>(qm)[c];
            if constexpr (VT == T_U8) {
                iq = (int)__dp4a(q.x, q.x, (uint32_t)iq); iq = (int)__dp4a(q.y, q.y, (uint32_t)iq);
                iq = (int)__dp4a(q.z, q.z, (uint32_t)iq); iq = (int)__dp4a(q.w, q.w, (uint32_t)iq);
            } else if constexpr (VT == T_I8) {
                iq = __dp4a((int)q.x, (int)q.x, iq); iq = __dp4a((int)q.y, (int)q.y, iq);
                iq = __dp4a((int)q.z, (int)q.z, iq); iq = __dp4a((int)q.w, (int)q.w, iq);
            } else {
                float x[8];
                unpack8<VT>(q, x);
                constexpr int NE = (VT == T_F32) ? 4 : 8;
#pragma unroll
                for (int j = 0; j < NE; ++j) f = fmaf(x[j], x[j], f);
            }
        }
        for (int off = 16; off >= 1; off >>= 1) {
            f += __shfl_xor_sync(0xFFFFFFFFu, f, off);
            iq += __shfl_xor_sync(0xFFFFFFFFu, iq, off);
        }
        qn[m].f = f; qn[m].i = iq;
    }
    // query m's k-list of this warp, its log
    auto mylist = [&](int m) { return lists_s + ((size_t)warp * nq + m) * prm.kcap; };
    for (int m = 0; m < nq; ++m)
        for (int j = lane; j < prm.kcap; j += 32) mylist(m)[j] = (j < prm.k) ? INFINITY : -INFINITY;
    __syncwarp();

    float thr[M];
    int pos[M], logged[M];
#pragma unroll
    for (int m = 0; m < M; ++m) { thr[m] = INFINITY; pos[m] = 0; logged[m] = 0; }
    uint2 *mylog = prm.logs + (size_t)sidx * prm.logcap;

    for (int it = 0; it < ntiles; ++it) {
        const long long row0 = (t0 + it) * rpw;
        const bool valid = (row0 + r) < prm.n;
        Accum A[M];
#pragma unroll
        for (int m = 0; m < M; ++m) A[m] = {0.f, 0.f, 0.f, 0, 0};
        if constexpr (!DIRECT) {
            const int s = stage;
            mbar_wait(&mybars[s], parity);
            if (++stage == nsw) { stage = 0; parity ^= 1u; }
            const uint8_t *rowp = myring + (size_t)s * prm.wtile_bytes + (size_t)r * prm.pitch;
            if (valid) {
#pragma unroll 4
                for (int i = 0; i < cnt; ++i) {
                    int ii = i0 + i;
                    if (ii >= cnt) ii -= cnt;
                    const int c = p + (ii << prm.log2P);
                    const uint4 rv = *reinterpret_cast<const uint4 *>(rowp + (size_t)c * 16);
                    accum16_pass<VT, MC, M>(A, rv, qs + (size_t)c * 16, prm.pitch, nq);
                }
            }
            __syncwarp();
            if constexpr (!kFix16) {
                if (lane == 0 && pf_it < ntiles) issue(s);
            } else {
                fix_row = rowp;                                           // the stage stays valid until the fix-up below has run
                fix_stage = s;
            }
        } else {
            const uint8_t *rowp = prm.vec + (size_t)(row0 + r) * prm.pitch;
            if (valid) {
#pragma unroll 4
                for (int i = 0; i < cnt; ++i) {
                    const int c = p + (i << prm.log2P);
                    const uint4 rv = ldg_stream(reinterpret_cast<const uint4 *>(rowp) + c);
                    accum16_pass<VT, MC, M>(A, rv, qs + (size_t)c * 16, prm.pitch, nq);
                }
            }
        }
        accum_reduce(A[0], P);
        float d[M];
#pragma unroll
        for (int m = 0; m < M; ++m) {
            if (m >= nq) break;
            if (m > 0) {
                accum_reduce<false>(A[m], P);
                A[m].ny = A[0].ny;
                A[m].ib = A[0].ib;
            }
            d[m] = finalize<VT, MC>(A[m], qn[m], prm.root);
        }
        if constexpr (kFix16) {
#pragma unroll
            for (int m = 0; m < M; ++m) {
                if (m >= nq) break;
                if (valid && p == 0 && row_needs_exact<VT, MC>(A[m], qn[m])) {
                    if constexpr (DIRECT) fix_row = prm.vec + (size_t)(row0 + r) * prm.pitch;
                    d[m] = special_row_distance<VT, MC>(fix_row, qs + m * prm.pitch, prm.pitch / 2, prm.root);
                }
            }
            if constexpr (!DIRECT) {
                __syncwarp();
                if (lane == 0 && pf_it < ntiles) issue(fix_stage);
            }
        }
        if constexpr (RANGE) {
            // one reservation per ballot; hit lanes write at their rank among the hits (slots are ordered later, range_sort_kernel)
            const bool hit = valid && p == 0 && d[0] < prm.range_t && row_allowed(prm.allow, prm.allow_base + row0 + r);
            const unsigned msk = __ballot_sync(0xFFFFFFFFu, hit);
            if (msk != 0u) {
                unsigned base = 0;
                if (lane == 0) base = atomicAdd(prm.range_count, (unsigned)__popc(msk));
                base = __shfl_sync(0xFFFFFFFFu, base, 0);
                const unsigned at = base + (unsigned)__popc(msk & ((1u << lane) - 1u));
                if (hit && (long long)at < prm.range_cap)
                    prm.range_pairs[at] = make_uint2(prm.range_row_base + (unsigned)(row0 + r), __float_as_uint(d[0]));
            }
            continue;
        }
        if (prm.dist_all != nullptr && valid && p == 0) prm.dist_all[row0 + r] = d[0];
        if (topk) {
#pragma unroll
            for (int m = 0; m < M; ++m) {
                if (m >= nq) break;
                // rows are visited in scan order (lane order); strict '<' like the reference (:2102, :2145)
                unsigned msk = __ballot_sync(0xFFFFFFFFu, valid && p == 0 && d[m] < thr[m] && row_allowed(prm.allow, prm.allow_base + row0 + r));
                while (msk) {
                    const int src = __ffs(msk) - 1;
                    msk &= msk - 1;
                    const float dv = __shfl_sync(0xFFFFFFFFu, d[m], src);
                    if (dv < thr[m]) {
                        if (lane == 0) {
                            if (logged[m] < prm.logcap)
                                mylog[pass_logs(m, S, prm.logcap) + logged[m]] = make_uint2(__float_as_uint(dv), (uint32_t)(row0 + (src >> prm.log2P)));
                            mylist(m)[pos[m]] = dv;
                        }
                        ++logged[m];
                        __syncwarp();
                        list_argmax(mylist(m), prm.kcap, lane, thr[m], pos[m]);
                    }
                }
            }
        }
    }
    if (topk) {
        __syncwarp();
#pragma unroll
        for (int m = 0; m < M; ++m) {
            if (m >= nq) break;
            if (lane == 0) {
                prm.counts[pass_streams(m, S) + sidx] = logged[m];
                if (logged[m] > prm.logcap) atomicExch(&prm.ctrl[m][1], 1);
            }
            if (prm.kcap == 32) {
                // k <= 32: the CTA's 8 streams are consecutive in scan order.  Sort each stream's list, then one warp per query
                // merges them in stream order, recording the running k-th value BEFORE each stream (its in-CTA prefix bound), and
                // publishes ONE sorted list per CTA: filter_kernel then walks one list per CTA instead of one per stream.
                float v = (lane < prm.k) ? mylist(m)[lane] : INFINITY;
                v = warp_sort_asc(v, lane);
                mylist(m)[lane] = v;
            } else {
                float *gl = prm.lists + pass_lists(m, S, prm.kcap) + (size_t)sidx * prm.kcap;
                for (int j = lane; j < prm.kcap; j += 32) gl[j] = mylist(m)[j];
            }
        }
    }
    if (topk && prm.kcap == 32) __syncthreads();                             // every stream's sorted lists are in lists_s
    if (tid == 0 && prm.cta_time != nullptr)
        prm.cta_time[blockIdx.x] = (unsigned)min((long long)0xFFFFFFFFll, (clock64() - clk0) >> 6);   // units of 64 cycles
    if (topk && prm.kcap == 32 && warp < nq) {                               // warp m merges query m's lists (nq <= kWarps)
        const int m = warp;
        SortedList Lm;
        Lm.init(lane, prm.k);
        for (int w = 0; w < kWarps; ++w) {
            if (lane == 0) prm.tlocal[pass_streams(m, S) + (size_t)blockIdx.x * kWarps + w] = Lm.thr;
            Lm.offer_sorted(lane, lists_s[((size_t)w * nq + m) * 32 + lane]);
        }
        prm.lists[pass_lists(m, S, 32) + (size_t)blockIdx.x * 32 + lane] = Lm.v;
    }
}

template <int VT, int MC, bool DIRECT>
__global__ void __launch_bounds__(kThreads, 1) scan_kernel(const ScanParams prm) { scan_body<VT, MC, DIRECT, false, 1>(prm); }
// a pass of 2 <= nq <= M queries
template <int VT, int MC, bool DIRECT, int M>
__global__ void __launch_bounds__(kThreads, 1) scan_pass_kernel(const ScanParams prm) { scan_body<VT, MC, DIRECT, false, M>(prm); }
template <int VT, int MC, bool DIRECT>
__global__ void __launch_bounds__(kThreads, 1) scan_range_kernel(const ScanParams prm) { scan_body<VT, MC, DIRECT, true, 1>(prm); }

// ------------------------------------------------------------------ range search: result order
// One block per query orders that query's (row, distance bits) pairs by (distance, row), in place: a bitonic sort of 64-bit keys
// (fkey(distance) << 32 | row) in shared memory.  fkey preserves the float order, so negative DOT distances and -INF come first;
// equal distances keep scan order (the row).  A query with more than kRangeSortCap pairs is left as it is (the host orders it
// or, in a batch, answers the query alone).
constexpr int kRangeSortCap = 16384;     // 128 KB of keys
constexpr int kRangeSortThreads = 1024;
struct RangeSortParams {
    uint2 *pairs;             // query q: pairs + q * stride, count[q] entries (row, distance bits)
    const unsigned *count;    // [gridDim.x]
    long long stride;
    uint2 *out;               // nullptr: in place; else query q's ordered pairs go to out + out_off[q] (the batch's compaction)
    const long long *out_off;
};
// The block's bitonic sort of n >= 2 pairs from pr into dst (may be pr) by the 64-bit key to_key(pair); from_key(key) restores the
// pair.  rkeys: shared memory for the next power of two >= n keys.
template <class ToKey, class FromKey>
__device__ __forceinline__ void block_sort_pairs(const uint2 *pr, uint2 *dst, int n, unsigned long long *rkeys, ToKey to_key, FromKey from_key) {
    int n2 = 2;
    while (n2 < n) n2 <<= 1;
    for (int i = threadIdx.x; i < n2; i += blockDim.x) {
        if (i < n) {
            rkeys[i] = to_key(pr[i]);
        } else {
            rkeys[i] = ~0ull;
        }
    }
    __syncthreads();
    for (int size = 2; size <= n2; size <<= 1) {
        for (int stride = size >> 1; stride > 0; stride >>= 1) {
            for (int i = threadIdx.x; i < n2; i += blockDim.x) {
                const int j = i ^ stride;
                if (j > i) {
                    const unsigned long long a = rkeys[i], b = rkeys[j];
                    if ((a > b) == ((i & size) == 0)) { rkeys[i] = b; rkeys[j] = a; }
                }
            }
            __syncthreads();
        }
    }
    for (int i = threadIdx.x; i < n; i += blockDim.x) dst[i] = from_key(rkeys[i]);
}

__global__ void __launch_bounds__(kRangeSortThreads, 1) range_sort_kernel(const RangeSortParams sp) {
    extern __shared__ __align__(16) unsigned long long rkeys[];
    const unsigned cnt = sp.count[blockIdx.x];
    if (cnt > (unsigned)kRangeSortCap) return;
    uint2 *pr = sp.pairs + (size_t)blockIdx.x * (size_t)sp.stride;
    uint2 *dst = sp.out ? sp.out + sp.out_off[blockIdx.x] : pr;
    if (cnt < 2u) {
        if (cnt == 1u && threadIdx.x == 0 && dst != pr) dst[0] = pr[0];
        return;
    }
    block_sort_pairs(pr, dst, (int)cnt, rkeys,
        [](const uint2 e) { return ((unsigned long long)fkey(__uint_as_float(e.y)) << 32) | e.x; },
        [](const unsigned long long key) { return make_uint2((unsigned)key, __float_as_uint(funkey((uint32_t)(key >> 32)))); });
}

// ---- large-k batches (batch_large_k, DESIGN §3.12): each query's bucket holds its kept (distance bits, shard row) pairs of every
// piece back to back, each piece's entries unordered (the refine appends with atomics).  One block per (query, piece) orders that
// segment by row and writes it to out + out_off[query] + the segment's start, so that every query's candidates come out in scan
// order.  A query with out_off < 0 is skipped (it is answered alone); no segment is longer than kRangeSortCap (the host checks).
struct LkbSortParams {
    const uint2 *bucket;      // query q: bucket + q * stride
    long long stride;
    const unsigned *pcount;   // [pieces][nq] the query's bucket count after each piece
    int nq;
    uint2 *out;
    const long long *out_off; // [nq]
};
constexpr int kLkbSortThreads = 512;
__global__ void __launch_bounds__(kLkbSortThreads) lkb_sort_kernel(const LkbSortParams sp) {
    extern __shared__ __align__(16) unsigned long long lkeys[];
    const int q = blockIdx.x, piece = blockIdx.y;
    const long long off = sp.out_off[q];
    if (off < 0) return;
    const unsigned a = piece ? sp.pcount[(size_t)(piece - 1) * sp.nq + q] : 0u, b = sp.pcount[(size_t)piece * sp.nq + q];
    if (b <= a || b - a > (unsigned)kRangeSortCap) return;
    const uint2 *pr = sp.bucket + (size_t)q * (size_t)sp.stride + a;
    uint2 *dst = sp.out + off + a;
    if (b - a == 1u) {
        if (threadIdx.x == 0) dst[0] = make_uint2(pr[0].y, pr[0].x);
        return;
    }
    block_sort_pairs(pr, dst, (int)(b - a), lkeys,
        [](const uint2 e) { return ((unsigned long long)e.x << 32) | e.y; },
        [](const unsigned long long key) { return make_uint2((unsigned)key, (unsigned)(key >> 32)); });
}

// ------------------------------------------------------------------ large k (k > 256): prefix bounds and ordered candidates
// One scanned view (a resident shard, one streamed window) whose distances scan_kernel wrote to dist_all.  Its rows are cut into
// segments [0, k), [k, 2k), [2k, 4k), ..., [.., n).  Segment s >= 1 is tested against B_{s-1}, the k-th smallest distance (fkey
// order) of the eligible, non-NaN rows of the prefix [0, ends[s-1]), +INF when that prefix has fewer than k such rows; segment 0
// against +INF.  A row that can enter the k slots has d < its segment's bound (DESIGN §3.11), so the eligible rows with
// d < bound, in scan order, are a superset of the rows the host replay needs.
//   lk_hist_kernel + lk_select_kernel, once per digit: a radix select of every prefix's k-th key at once, 4 digits of 8 bits,
//   most significant first, on the device (no host round trip between digits);
//   lk_count_kernel, lk_offsets_kernel, lk_write_kernel: the ordered compaction of the candidates into the pair list.
constexpr int kLkMaxSeg = 32;        // segments of a view: n < 2^32 and k > 256 need at most 25
constexpr int kLkThreads = 256;
constexpr int kLkRows = 8192;        // rows of one block of the histogram and compaction kernels (32 per thread)
constexpr int kLkPasses = 4;         // radix digits of 8 bits
constexpr int kLkScanThreads = 1024; // lk_offsets_kernel; lk_select_kernel runs one warp per prefix (kLkMaxSeg warps)

// the most recent view's segments and bounds (vsb_debug_read "topk_bounds" returns the first three fields) and the select's state
struct LkState {
    long long nseg;
    long long ends[kLkMaxSeg];       // segment s = rows [s ? ends[s - 1] : 0, ends[s]); ends[nseg - 1] = n
    float bound[kLkMaxSeg];          // bound[0] = +INF, bound[s] = B_{s-1}
    unsigned sel[kLkMaxSeg];         // prefix j = rows [0, ends[j]): the key digits chosen so far
    unsigned rank[kLkMaxSeg];        // prefix j: rank (from 1) of the k-th key among the keys that start with sel[j]
    int live[kLkMaxSeg];             // prefix j holds at least k keys (else its bound is +INF)
};

struct LkParams {
    const float *dist;               // [n] distances of the view
    long long n;
    int k, nseg;                     // prefixes: nseg - 1
    long long ends[kLkMaxSeg];
    const uint32_t *allow;           // row filter as in ScanParams: row r is eligible at bit allow_base + r (nullptr: every row)
    long long allow_base;
    unsigned *hist;                  // [kLkPasses][kLkMaxSeg][256], zero before the first digit
    LkState *st;
    unsigned *boff;                  // [blocks]: candidates per compaction block (count), then where they start (offsets)
    unsigned *total;                 // pairs of the views so far (the pair list's counter); the offsets kernel adds this view's
    uint2 *out;                      // pair list: (distance bits, row_base + row); positions at or past cap are not written
    long long cap;
    unsigned row_base;
    int pass;                        // lk_hist_kernel / lk_select_kernel: the digit (0 = most significant)
    int nblocks;                     // lk_offsets_kernel: compaction blocks
};

// the segment ends into shared memory (compile-time parameter offsets only: no local copy of the parameter block)
__device__ __forceinline__ void lk_load_ends(const LkParams &p, long long *ends) {
#pragma unroll
    for (int i = 0; i < kLkMaxSeg; ++i)
        if ((int)threadIdx.x == i) ends[i] = i < p.nseg ? p.ends[i] : 0x7FFFFFFFFFFFFFFFll;
}

// histogram of digit p.pass: every eligible, non-NaN row of a prefix whose higher digits match the prefix's chosen ones (all of
// them at digit 0) adds to that prefix's bin.  Row r lies in the prefixes j >= its segment; rows of the last segment in none.
__global__ void __launch_bounds__(kLkThreads) lk_hist_kernel(const LkParams p) {
    __shared__ unsigned h[kLkMaxSeg * 256];
    __shared__ long long ends[kLkMaxSeg];
    __shared__ unsigned sel[kLkMaxSeg];
    __shared__ int live[kLkMaxSeg];
    const int J = p.nseg - 1;
    lk_load_ends(p, ends);
    if ((int)threadIdx.x < J) {
        sel[threadIdx.x] = p.pass ? p.st->sel[threadIdx.x] : 0u;
        live[threadIdx.x] = p.pass ? p.st->live[threadIdx.x] : 1;
    }
    __syncthreads();
    const long long c0 = (long long)blockIdx.x * kLkRows, c1 = min(c0 + (long long)kLkRows, ends[J - 1]);
    int s0 = 0;
    while (c0 >= ends[s0]) ++s0;
    for (int i = s0 * 256 + threadIdx.x; i < J * 256; i += kLkThreads) h[i] = 0u;
    __syncthreads();
    const int shift = 24 - 8 * p.pass;
    int s = s0;
    for (long long r = c0 + threadIdx.x; r < c1; r += kLkThreads) {
        while (r >= ends[s]) ++s;
        const float d = p.dist[r];
        if (d != d || !row_allowed(p.allow, p.allow_base + r)) continue;
        const uint32_t key = fkey(d), dig = (key >> shift) & 255u;
        const uint32_t hi = p.pass ? key >> (shift + 8) : 0u;
        for (int j = s; j < J; ++j)
            if (live[j] && hi == sel[j]) atomicAdd(&h[j * 256 + dig], 1u);
    }
    __syncthreads();
    unsigned *g = p.hist + (size_t)p.pass * kLkMaxSeg * 256;
    for (int i = s0 * 256 + threadIdx.x; i < J * 256; i += kLkThreads)
        if (h[i]) atomicAdd(g + i, h[i]);
}

// one warp per prefix: the bin of digit p.pass that holds the prefix's k-th key.  At digit 0 a prefix with fewer than k keys
// is done (bound +INF).  After the last digit the chosen digits are the k-th key; the view's segments and bounds are written.
__global__ void __launch_bounds__(kLkMaxSeg * 32, 1) lk_select_kernel(const LkParams p) {
    const int j = threadIdx.x >> 5, lane = threadIdx.x & 31, J = p.nseg - 1;
    LkState *st = p.st;
    if (j < J) {
        unsigned sel = p.pass ? st->sel[j] : 0u, rank = p.pass ? st->rank[j] : (unsigned)p.k;
        int live = p.pass ? st->live[j] : 1;
        if (live) {
            const unsigned *hj = p.hist + ((size_t)p.pass * kLkMaxSeg + j) * 256 + lane * 8;
            unsigned c[8], sum = 0;
#pragma unroll
            for (int i = 0; i < 8; ++i) { c[i] = hj[i]; sum += c[i]; }
            unsigned incl = sum;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const unsigned v = __shfl_up_sync(0xFFFFFFFFu, incl, o);
                if (lane >= o) incl += v;
            }
            if (__shfl_sync(0xFFFFFFFFu, incl, 31) < rank) {
                live = 0;
            } else {
                const int src = __ffs(__ballot_sync(0xFFFFFFFFu, incl >= rank)) - 1;
                unsigned dig = 0, nr = 0, cum = incl - sum;
                bool found = false;
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                    if (!found && cum + c[i] >= rank) { dig = (unsigned)(lane * 8 + i); nr = rank - cum; found = true; }
                    cum += c[i];
                }
                sel = (sel << 8) | __shfl_sync(0xFFFFFFFFu, dig, src);
                rank = __shfl_sync(0xFFFFFFFFu, nr, src);
            }
        }
        if (lane == 0) {
            st->sel[j] = sel;
            st->rank[j] = rank;
            st->live[j] = live;
            if (p.pass == kLkPasses - 1) st->bound[j + 1] = live ? funkey(sel) : INFINITY;
        }
    }
    if (p.pass == kLkPasses - 1) {
#pragma unroll
        for (int i = 0; i < kLkMaxSeg; ++i)
            if ((int)threadIdx.x == i) st->ends[i] = i < p.nseg ? p.ends[i] : 0;
        if (threadIdx.x == 0) {
            st->nseg = p.nseg;
            st->bound[0] = INFINITY;
        }
    }
}

// the segment ends and bounds of a compaction block, and the segment of its first row
__device__ __forceinline__ int lk_load_bounds(const LkParams &p, long long *ends, float *bound, long long c0) {
    lk_load_ends(p, ends);
    if ((int)threadIdx.x < p.nseg) bound[threadIdx.x] = p.st->bound[threadIdx.x];
    __syncthreads();
    int s = 0;
    while (c0 >= ends[s]) ++s;
    return s;
}

__device__ __forceinline__ bool lk_candidate(const LkParams &p, long long r, float d, float bound) {
    return d < bound && row_allowed(p.allow, p.allow_base + r);
}

// candidates of each block of kLkRows rows
__global__ void __launch_bounds__(kLkThreads) lk_count_kernel(const LkParams p) {
    __shared__ long long ends[kLkMaxSeg];
    __shared__ float bound[kLkMaxSeg];
    __shared__ unsigned wsum[kLkThreads / 32];
    const long long c0 = (long long)blockIdx.x * kLkRows, c1 = min(c0 + (long long)kLkRows, p.n);
    int s = lk_load_bounds(p, ends, bound, c0);
    unsigned c = 0;
    for (long long r = c0 + threadIdx.x; r < c1; r += kLkThreads) {
        while (r >= ends[s]) ++s;
        c += lk_candidate(p, r, p.dist[r], bound[s]) ? 1u : 0u;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xFFFFFFFFu, c, o);
    if ((threadIdx.x & 31) == 0) wsum[threadIdx.x >> 5] = c;
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned t = 0;
        for (int w = 0; w < kLkThreads / 32; ++w) t += wsum[w];
        p.boff[blockIdx.x] = t;
    }
}

// one block: the block counts become the positions their candidates start at, after the pairs of the earlier views (*total);
// *total grows by this view's candidates
__global__ void __launch_bounds__(kLkScanThreads, 1) lk_offsets_kernel(const LkParams p) {
    __shared__ unsigned wsum[kLkScanThreads / 32];
    __shared__ unsigned carry;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) carry = *p.total;
    __syncthreads();
    for (int b0 = 0; b0 < p.nblocks; b0 += kLkScanThreads) {
        const int i = b0 + (int)threadIdx.x;
        const unsigned v = i < p.nblocks ? p.boff[i] : 0u;
        unsigned incl = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const unsigned t = __shfl_up_sync(0xFFFFFFFFu, incl, o);
            if (lane >= o) incl += t;
        }
        if (lane == 31) wsum[warp] = incl;
        __syncthreads();
        if (warp == 0) {
            unsigned w = wsum[lane];
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const unsigned t = __shfl_up_sync(0xFFFFFFFFu, w, o);
                if (lane >= o) w += t;
            }
            wsum[lane] = w;
        }
        __syncthreads();
        const unsigned base = carry;
        if (i < p.nblocks) p.boff[i] = base + (warp ? wsum[warp - 1] : 0u) + incl - v;
        __syncthreads();
        if (threadIdx.x == 0) carry = base + wsum[kLkScanThreads / 32 - 1];
        __syncthreads();
    }
    if (threadIdx.x == 0) *p.total = carry;
}

// writes each block's candidates in scan order from its offset on (pairs at or past cap are dropped; the host grows the list to
// the count and runs this kernel again)
__global__ void __launch_bounds__(kLkThreads) lk_write_kernel(const LkParams p) {
    __shared__ long long ends[kLkMaxSeg];
    __shared__ float bound[kLkMaxSeg];
    __shared__ unsigned wcnt[kLkThreads / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const long long c0 = (long long)blockIdx.x * kLkRows, c1 = min(c0 + (long long)kLkRows, p.n);
    int s = lk_load_bounds(p, ends, bound, c0);
    unsigned pos = p.boff[blockIdx.x];
    for (long long r0 = c0; r0 < c1; r0 += kLkThreads) {
        const long long r = r0 + threadIdx.x;
        bool hit = false;
        float d = 0.f;
        if (r < c1) {
            while (r >= ends[s]) ++s;
            d = p.dist[r];
            hit = lk_candidate(p, r, d, bound[s]);
        }
        const unsigned m = __ballot_sync(0xFFFFFFFFu, hit);
        if (lane == 0) wcnt[warp] = (unsigned)__popc(m);
        __syncthreads();
        unsigned before = 0, tot = 0;
#pragma unroll
        for (int w = 0; w < kLkThreads / 32; ++w) {
            before += w < warp ? wcnt[w] : 0u;
            tot += wcnt[w];
        }
        if (hit) {
            const unsigned at = pos + before + (unsigned)__popc(m & ((1u << lane) - 1u));
            if ((long long)at < p.cap) p.out[at] = make_uint2(__float_as_uint(d), p.row_base + (unsigned)r);
        }
        pos += tot;
        __syncthreads();
    }
}

// ------------------------------------------------------------------ grouped top-k (DESIGN §3.15)
// The keys' rows of one shard are laid out as positions in (key, scan order) order; every key's run is cut into pieces of at
// most kGroupedPiece positions, and no piece crosses a key.  The distances of one query are already in dist (the all-distances
// scan with the plan of the filtered call at this k).
//   grouped_walk_kernel: one warp per piece reads d[row] in piece order and keeps the piece's k smallest.  A position is logged
//   when d < the piece's running k-th value (+INF until k rows were seen, strict, as scan_kernel's ballot: NaN and +INF never
//   log); pd[pos] is d for a logged position and NaN otherwise.  The piece publishes its k smallest, ascending, +INF padded.
//   grouped_bounds_kernel: one warp per key merges its pieces' lists in piece order; a piece's bound is the k-th smallest of the
//   earlier pieces of its key (+INF for the first), the key's minimum the smallest value of all of them (+INF: empty key).
//   grouped_count_kernel, lk_offsets_kernel, grouped_write_kernel: the ordered compaction of the positions with pd < their
//   piece's bound, of the selected keys only, into the pair list as (distance bits, position).
constexpr int kGroupedPiece = 1024;  // positions of a piece
constexpr int kGroupedWarps = 8;     // warps of a block: one piece or key each

struct GroupedParams {
    const float *dist;               // [shard rows] the query's distances
    const uint32_t *rows;            // [positions] shard row of each position
    const uint32_t *pstart;          // [npieces + 1] first position of each piece
    const uint32_t *pkey;            // [npieces] key of each piece
    const uint32_t *kpiece;          // [nkeys + 1] first piece of each key
    float *pd;                       // [positions] d of a logged position, NaN otherwise
    float *lists;                    // [npieces][k] each piece's k smallest, ascending, +INF padded
    float *bound;                    // [npieces]
    float *kmin;                     // [nkeys]
    const uint8_t *ksel;             // [nkeys] keys to compact (nullptr: every key)
    unsigned *pcount;                // [npieces] survivors of each piece, then where they start (lk_offsets_kernel)
    uint2 *out;                      // pair list; positions at or past cap are not written
    long long cap;
    long long npieces;
    int nkeys, k;
};

// the k smallest values (k <= kcap, entries >= k of list hold -INF) of a warp's shared list, ascending, into out[0, k)
__device__ __forceinline__ void grouped_sorted_out(const float *list, int k, int lane, float *out) {
    for (int j = lane; j < k; j += 32) {
        const float v = list[j];
        int rank = 0;
        for (int i = 0; i < k; ++i) {
            const float u = list[i];
            rank += (u < v || (u == v && i < j)) ? 1 : 0;
        }
        out[rank] = v;
    }
}

// SMALL: k <= 32, the running list in registers (SortedList); otherwise a shared list of kMaxK entries per warp (list_argmax)
template <bool SMALL>
__global__ void __launch_bounds__(kGroupedWarps * 32) grouped_walk_kernel(const GroupedParams p) {
    __shared__ float sl[SMALL ? 1 : kGroupedWarps * 256];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const long long pc = (long long)blockIdx.x * kGroupedWarps + warp;
    if (pc >= p.npieces) return;
    const uint32_t a = p.pstart[pc], b = p.pstart[pc + 1];
    const int k = p.k, kcap = (k + 31) & ~31;
    SortedList L;
    float *list = sl + (SMALL ? 0 : warp * 256);
    float thr = INFINITY;
    int pos = 0;
    if constexpr (SMALL) {
        L.init(lane, k);
    } else {
        for (int j = lane; j < kcap; j += 32) list[j] = (j < k) ? INFINITY : -INFINITY;
        __syncwarp();
        list_argmax(list, kcap, lane, thr, pos);
    }
    for (uint32_t c0 = a; c0 < b; c0 += 32) {
        const uint32_t at = c0 + (uint32_t)lane;
        const bool valid = at < b;
        const float d = valid ? p.dist[p.rows[at]] : __int_as_float(0x7FC00000);
        unsigned msk = __ballot_sync(0xFFFFFFFFu, valid && d < (SMALL ? L.thr : thr));
        unsigned logged = 0u;
        while (msk) {
            const int src = __ffs(msk) - 1;
            msk &= msk - 1;
            const float dv = __shfl_sync(0xFFFFFFFFu, d, src);
            if constexpr (SMALL) {
                if (dv < L.thr) {
                    L.insert(lane, dv);
                    logged |= 1u << src;
                }
            } else if (dv < thr) {
                if (lane == 0) list[pos] = dv;
                __syncwarp();
                list_argmax(list, kcap, lane, thr, pos);
                logged |= 1u << src;
            }
        }
        if (valid) p.pd[at] = ((logged >> lane) & 1u) ? d : __int_as_float(0x7FC00000);
    }
    float *out = p.lists + (size_t)pc * k;
    if constexpr (SMALL) {
        if (lane < k) out[lane] = L.v;
    } else {
        __syncwarp();
        grouped_sorted_out(list, k, lane, out);
    }
}

// one warp per key: its pieces' bounds and its minimum
template <bool SMALL>
__global__ void __launch_bounds__(kGroupedWarps * 32) grouped_bounds_kernel(const GroupedParams p) {
    __shared__ float sl[SMALL ? 1 : kGroupedWarps * 256];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int g = blockIdx.x * kGroupedWarps + warp;
    if (g >= p.nkeys) return;
    const int k = p.k, kcap = (k + 31) & ~31;
    const uint32_t q0 = p.kpiece[g], q1 = p.kpiece[g + 1];
    SortedList L;
    float *list = sl + (SMALL ? 0 : warp * 256);
    float thr = INFINITY, mn = INFINITY;
    int pos = 0;
    if constexpr (SMALL) {
        L.init(lane, k);
    } else {
        for (int j = lane; j < kcap; j += 32) list[j] = (j < k) ? INFINITY : -INFINITY;
        __syncwarp();
        list_argmax(list, kcap, lane, thr, pos);
    }
    for (uint32_t pc = q0; pc < q1; ++pc) {
        const float *src = p.lists + (size_t)pc * k;
        if (lane == 0) p.bound[pc] = SMALL ? L.thr : thr;
        mn = fminf(mn, src[0]);
        if constexpr (SMALL) {
            L.offer_sorted(lane, lane < k ? src[lane] : INFINITY);
        } else {
            // the list is ascending: once a value is not below the running k-th value, none after it is
            for (int j0 = 0; j0 < k; j0 += 32) {
                const float v = j0 + lane < k ? src[j0 + lane] : INFINITY;
                unsigned msk = __ballot_sync(0xFFFFFFFFu, v < thr);
                if (!msk) break;
                while (msk) {
                    const int s = __ffs(msk) - 1;
                    msk &= msk - 1;
                    const float dv = __shfl_sync(0xFFFFFFFFu, v, s);
                    if (dv < thr) {
                        if (lane == 0) list[pos] = dv;
                        __syncwarp();
                        list_argmax(list, kcap, lane, thr, pos);
                    }
                }
            }
        }
    }
    if (lane == 0) p.kmin[g] = mn;
}

__device__ __forceinline__ bool grouped_selected(const GroupedParams &p, long long pc) {
    return p.ksel == nullptr || p.ksel[p.pkey[pc]] != 0;
}

// one warp per piece: its survivors
__global__ void __launch_bounds__(kGroupedWarps * 32) grouped_count_kernel(const GroupedParams p) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const long long pc = (long long)blockIdx.x * kGroupedWarps + warp;
    if (pc >= p.npieces) return;
    unsigned c = 0;
    if (grouped_selected(p, pc)) {
        const uint32_t a = p.pstart[pc], b = p.pstart[pc + 1];
        const float bd = p.bound[pc];
        for (uint32_t at = a + (uint32_t)lane; at < b; at += 32) c += p.pd[at] < bd ? 1u : 0u;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xFFFFFFFFu, c, o);
    }
    if (lane == 0) p.pcount[pc] = c;
}

// one warp per piece: its survivors in position order from the piece's offset on
__global__ void __launch_bounds__(kGroupedWarps * 32) grouped_write_kernel(const GroupedParams p) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const long long pc = (long long)blockIdx.x * kGroupedWarps + warp;
    if (pc >= p.npieces || !grouped_selected(p, pc)) return;
    const uint32_t a = p.pstart[pc], b = p.pstart[pc + 1];
    const float bd = p.bound[pc];
    unsigned w = p.pcount[pc];
    for (uint32_t c0 = a; c0 < b; c0 += 32) {
        const uint32_t at = c0 + (uint32_t)lane;
        const float d = at < b ? p.pd[at] : __int_as_float(0x7FC00000);
        const bool hit = d < bd;
        const unsigned m = __ballot_sync(0xFFFFFFFFu, hit);
        const unsigned o = w + (unsigned)__popc(m & ((1u << lane) - 1u));
        if (hit && (long long)o < p.cap) p.out[o] = make_uint2(__float_as_uint(d), at);
        w += (unsigned)__popc(m);
    }
}

// ------------------------------------------------------------------ grouped layout (DESIGN §3.15)
// One shard's layout of a set of keys, built on the device from the caller's CSR keys (rowids, offsets):
//   grouped_map_count_kernel, grouped_scan64_kernel, grouped_map_write_kernel: every (key, rowid) pair becomes the shard rows that
//   hold the rowid (implicit rowids by arithmetic, explicit ones by a binary search of the index's (rowid, row) table sorted by
//   rowid; a rowid held by several rows yields each of them), counted, placed and written as the composite key << rbits | row;
//   grouped_sort_hist_kernel, grouped_sort_scan_kernel, grouped_sort_scatter_kernel: one pass of a stable LSD radix sort of 64-bit
//   keys (and optional 32-bit values) by an 8-bit digit; a sort runs only the passes its keys' bits need;
//   grouped_uniq_count_kernel, lk_offsets_kernel, grouped_uniq_write_kernel: the sorted composites without adjacent repeats;
//   grouped_koff_kernel: each key's first position (a binary search of its smallest composite);
//   grouped_piece_count_kernel, lk_offsets_kernel, grouped_piece_write_kernel, grouped_rows_kernel: each key cut into pieces of at
//   most kGroupedPiece positions (kpiece, pstart, pkey) and the shard row of every position.
constexpr int kLayoutThreads = 256;
constexpr int kLayoutItems = 8;                                  // entries per thread of the map, unique and piece kernels
constexpr int kLayoutTile = kLayoutThreads * kLayoutItems;       // entries per block of those kernels
constexpr int kSortTile = kLayoutThreads * 16;                   // keys per block of a sort pass

struct LayoutParams {
    const int64_t *rowids;           // [m] the keys' rowids, back to back
    const int64_t *offsets;          // [nkeys + 1] key g's rowids are [offsets[g], offsets[g + 1])
    long long m0, m;                 // map kernels: the pairs [m0, m) (m0 a multiple of kLayoutTile)
    int nkeys, rbits;                // rbits: bits of a shard row in a composite
    int implicit;                    // rowid = first_seq + row + 1
    long long first_seq, n;          // n: shard rows
    const unsigned long long *tab;   // explicit rowids: [n] rowid ^ 2^63, ascending
    const uint32_t *tab_row;         // [n] the row of each
    unsigned long long *bcount;      // [map blocks] rows of each block's pairs, then where they start
    unsigned long long *comp;        // composites (map: written; unique: read, sorted)
    unsigned long long *uniq;        // the unique composites
    const unsigned *npos;            // device: the unique composites' count
    unsigned *boff;                  // [blocks] per-block counts, then offsets (lk_offsets_kernel)
    uint32_t *koff;                  // [nkeys + 1]
    uint32_t *rows, *pstart, *pkey, *kpiece;
};

struct SortParams {
    const unsigned long long *kin;
    unsigned long long *kout;
    const uint32_t *vin;             // values (nullptr: keys only)
    uint32_t *vout;
    long long m;
    int shift, nblocks;
    unsigned *hist;                  // [256][nblocks]: the digit counts of each block, then where they start within the digit
    unsigned *dtot;                  // [256] keys of each digit
};

// exclusive prefix of v over the kLayoutThreads threads of a block (in thread order) and the block's total; wsum: shared [8],
// free again after the next __syncthreads
template <class T>
__device__ __forceinline__ T layout_block_scan(T v, T *wsum, T &total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    T incl = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const T t = __shfl_up_sync(0xFFFFFFFFu, incl, o);
        if (lane >= o) incl += t;
    }
    if (lane == 31) wsum[warp] = incl;
    __syncthreads();
    T before = 0, tot = 0;
#pragma unroll
    for (int w = 0; w < kLayoutThreads / 32; ++w) {
        before += w < warp ? wsum[w] : T(0);
        tot += wsum[w];
    }
    total = tot;
    return before + incl - v;
}

// the shard rows of rowid r: rows lo .. hi - 1 (implicit), or tab_row[lo .. hi) (explicit)
__device__ __forceinline__ void layout_rows_of(const LayoutParams &p, int64_t r, long long &lo, long long &hi) {
    if (p.implicit) {
        const bool in = r > p.first_seq && r - p.first_seq <= p.n;
        lo = in ? r - p.first_seq - 1 : 0;
        hi = in ? lo + 1 : 0;
        return;
    }
    const unsigned long long key = (unsigned long long)r ^ (1ull << 63);
    long long a = 0, b = p.n;
    while (a < b) {
        const long long mid = (a + b) >> 1;
        if (p.tab[mid] < key) a = mid + 1; else b = mid;
    }
    lo = a;
    b = p.n;
    while (a < b) {
        const long long mid = (a + b) >> 1;
        if (p.tab[mid] <= key) a = mid + 1; else b = mid;
    }
    hi = a;
}

// rows of each block's pairs
__global__ void __launch_bounds__(kLayoutThreads) grouped_map_count_kernel(const LayoutParams p) {
    __shared__ unsigned long long wsum[kLayoutThreads / 32];
    const long long i0 = p.m0 + (long long)blockIdx.x * kLayoutTile;
    unsigned long long c = 0;
#pragma unroll
    for (int j = 0; j < kLayoutItems; ++j) {
        const long long i = i0 + j * kLayoutThreads + threadIdx.x;
        if (i < p.m) {
            long long lo, hi;
            layout_rows_of(p, p.rowids[i], lo, hi);
            c += (unsigned long long)(hi - lo);
        }
    }
    unsigned long long total;
    layout_block_scan(c, wsum, total);
    if (threadIdx.x == 0) p.bcount[i0 / kLayoutTile] = total;
}

// one block: the block counts v[0, n) become where each block's entries start; *total = their sum
__global__ void __launch_bounds__(1024, 1) grouped_scan64_kernel(unsigned long long *v, long long n, unsigned long long *total) {
    __shared__ unsigned long long wsum[32];
    __shared__ unsigned long long carry;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    for (long long b0 = 0; b0 < n; b0 += 1024) {
        const long long i = b0 + threadIdx.x;
        const unsigned long long x = i < n ? v[i] : 0ull;
        unsigned long long incl = x;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const unsigned long long t = __shfl_up_sync(0xFFFFFFFFu, incl, o);
            if (lane >= o) incl += t;
        }
        if (lane == 31) wsum[warp] = incl;
        __syncthreads();
        if (warp == 0) {
            unsigned long long w = wsum[lane];
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const unsigned long long t = __shfl_up_sync(0xFFFFFFFFu, w, o);
                if (lane >= o) w += t;
            }
            wsum[lane] = w;
        }
        __syncthreads();
        const unsigned long long base = carry;
        if (i < n) v[i] = base + (warp ? wsum[warp - 1] : 0ull) + incl - x;
        __syncthreads();
        if (threadIdx.x == 0) carry = base + wsum[31];
        __syncthreads();
    }
    if (threadIdx.x == 0) *total = carry;
}

// each pair's rows as composites from its block's offset on (the order inside a block is free: the sort follows)
__global__ void __launch_bounds__(kLayoutThreads) grouped_map_write_kernel(const LayoutParams p) {
    __shared__ unsigned long long wsum[kLayoutThreads / 32];
    const long long i0 = (long long)blockIdx.x * kLayoutTile;
    long long lo[kLayoutItems], hi[kLayoutItems];
    unsigned long long c = 0;
#pragma unroll
    for (int j = 0; j < kLayoutItems; ++j) {
        const long long i = i0 + j * kLayoutThreads + threadIdx.x;
        lo[j] = hi[j] = 0;
        if (i < p.m) layout_rows_of(p, p.rowids[i], lo[j], hi[j]);
        c += (unsigned long long)(hi[j] - lo[j]);
    }
    unsigned long long total;
    unsigned long long at = p.bcount[blockIdx.x] + layout_block_scan(c, wsum, total);
#pragma unroll
    for (int j = 0; j < kLayoutItems; ++j) {
        if (hi[j] == lo[j]) continue;
        const long long i = i0 + j * kLayoutThreads + threadIdx.x;
        int a = 0, b = p.nkeys + 1;                                  // the key: the last g with offsets[g] <= i
        while (a < b) {
            const int mid = (a + b) >> 1;
            if (p.offsets[mid] <= i) a = mid + 1; else b = mid;
        }
        const unsigned long long key = (unsigned long long)(a - 1) << p.rbits;
        for (long long r = lo[j]; r < hi[j]; ++r) p.comp[at++] = key | (p.implicit ? (unsigned long long)r : (unsigned long long)p.tab_row[r]);
    }
}

__device__ __forceinline__ unsigned sort_digit(unsigned long long key, int shift) { return (unsigned)(key >> shift) & 255u; }

// the digit counts of each block's keys
__global__ void __launch_bounds__(kLayoutThreads) grouped_sort_hist_kernel(const SortParams p) {
    __shared__ unsigned h[256];
    h[threadIdx.x] = 0u;
    __syncthreads();
    const long long i0 = (long long)blockIdx.x * kSortTile, i1 = min(i0 + (long long)kSortTile, p.m);
    for (long long i = i0 + threadIdx.x; i < i1; i += kLayoutThreads) atomicAdd(&h[sort_digit(p.kin[i], p.shift)], 1u);
    __syncthreads();
    p.hist[(size_t)threadIdx.x * p.nblocks + blockIdx.x] = h[threadIdx.x];
}

// block d: digit d's block counts become where each block's keys of digit d start inside the digit; dtot[d] = the digit's keys
__global__ void __launch_bounds__(kLayoutThreads) grouped_sort_scan_kernel(const SortParams p) {
    __shared__ unsigned wsum[kLayoutThreads / 32];
    unsigned *h = p.hist + (size_t)blockIdx.x * p.nblocks;
    unsigned carry = 0;
    for (int b0 = 0; b0 < p.nblocks; b0 += kLayoutThreads) {
        const int i = b0 + (int)threadIdx.x;
        const unsigned v = i < p.nblocks ? h[i] : 0u;
        unsigned total;
        const unsigned ex = layout_block_scan(v, wsum, total);
        if (i < p.nblocks) h[i] = carry + ex;
        carry += total;
        __syncthreads();
    }
    if (threadIdx.x == 0) p.dtot[blockIdx.x] = carry;
}

// each block's keys to their places, stably: in index order inside the block (warp by warp through __match_any_sync), after the
// same digit's keys of earlier blocks, after the keys of smaller digits
__global__ void __launch_bounds__(kLayoutThreads) grouped_sort_scatter_kernel(const SortParams p) {
    __shared__ unsigned base[256];
    __shared__ unsigned wc[kLayoutThreads / 32][256];
    __shared__ unsigned wsum[kLayoutThreads / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, t = threadIdx.x;
    unsigned total;
    const unsigned ex = layout_block_scan(p.dtot[t], wsum, total);
    base[t] = ex + p.hist[(size_t)t * p.nblocks + blockIdx.x];
#pragma unroll
    for (int w = 0; w < kLayoutThreads / 32; ++w) wc[w][t] = 0u;
    __syncthreads();
    const long long i0 = (long long)blockIdx.x * kSortTile;
    for (int it = 0; it < kSortTile / kLayoutThreads; ++it) {
        const long long i = i0 + (long long)it * kLayoutThreads + t;
        if (i0 + (long long)it * kLayoutThreads >= p.m) break;              // uniform across the block
        const bool valid = i < p.m;
        const unsigned long long key = valid ? p.kin[i] : 0ull;
        const unsigned d = valid ? sort_digit(key, p.shift) : 256u;
        const unsigned peers = __match_any_sync(0xFFFFFFFFu, d);
        const unsigned rank = (unsigned)__popc(peers & ((1u << lane) - 1u));
        if (valid && rank == 0) wc[warp][d] = (unsigned)__popc(peers);
        __syncthreads();
        unsigned run = base[t];
#pragma unroll
        for (int w = 0; w < kLayoutThreads / 32; ++w) {
            const unsigned c = wc[w][t];
            wc[w][t] = run;
            run += c;
        }
        base[t] = run;
        __syncthreads();
        if (valid) {
            const unsigned at = wc[warp][d] + rank;
            p.kout[at] = key;
            if (p.vin) p.vout[at] = p.vin[i];
        }
        __syncthreads();
#pragma unroll
        for (int w = 0; w < kLayoutThreads / 32; ++w) wc[w][t] = 0u;
        __syncthreads();
    }
}

// explicit rowids: the table's keys (rowid ^ 2^63, so that unsigned order is signed order) and rows before the sort
__global__ void __launch_bounds__(kLayoutThreads) grouped_table_keys_kernel(const int64_t *rowids, long long n, unsigned long long *keys,
                                                                            uint32_t *rows) {
    for (long long i = (long long)blockIdx.x * kLayoutThreads + threadIdx.x; i < n; i += (long long)gridDim.x * kLayoutThreads) {
        keys[i] = (unsigned long long)rowids[i] ^ (1ull << 63);
        rows[i] = (uint32_t)i;
    }
}

// the sorted composites' first occurrences, thread by thread in index order
__device__ __forceinline__ unsigned layout_firsts(const LayoutParams &p, long long i0, bool *first) {
    unsigned c = 0;
#pragma unroll
    for (int j = 0; j < kLayoutItems; ++j) {
        const long long i = i0 + j;
        first[j] = i < p.m && (i == 0 || p.comp[i] != p.comp[i - 1]);
        c += first[j] ? 1u : 0u;
    }
    return c;
}

__global__ void __launch_bounds__(kLayoutThreads) grouped_uniq_count_kernel(const LayoutParams p) {
    __shared__ unsigned wsum[kLayoutThreads / 32];
    bool first[kLayoutItems];
    const unsigned c = layout_firsts(p, (long long)blockIdx.x * kLayoutTile + (long long)threadIdx.x * kLayoutItems, first);
    unsigned total;
    layout_block_scan(c, wsum, total);
    if (threadIdx.x == 0) p.boff[blockIdx.x] = total;
}

__global__ void __launch_bounds__(kLayoutThreads) grouped_uniq_write_kernel(const LayoutParams p) {
    __shared__ unsigned wsum[kLayoutThreads / 32];
    bool first[kLayoutItems];
    const long long i0 = (long long)blockIdx.x * kLayoutTile + (long long)threadIdx.x * kLayoutItems;
    const unsigned c = layout_firsts(p, i0, first);
    unsigned total;
    unsigned at = p.boff[blockIdx.x] + layout_block_scan(c, wsum, total);
#pragma unroll
    for (int j = 0; j < kLayoutItems; ++j)
        if (first[j]) p.uniq[at++] = p.comp[i0 + j];
}

// koff[g] for g in [0, nkeys]: the first unique composite of key g or later
__global__ void __launch_bounds__(kLayoutThreads) grouped_koff_kernel(const LayoutParams p) {
    const long long g = (long long)blockIdx.x * kLayoutThreads + threadIdx.x;
    if (g > p.nkeys) return;
    const unsigned long long key = (unsigned long long)g << p.rbits;
    unsigned a = 0, b = *p.npos;
    while (a < b) {
        const unsigned mid = a + ((b - a) >> 1);
        if (p.uniq[mid] < key) a = mid + 1; else b = mid;
    }
    p.koff[g] = a;
}

// the pieces of keys [g0, g0 + kLayoutItems), thread by thread in key order
__device__ __forceinline__ unsigned layout_pieces(const LayoutParams &p, long long g0, unsigned *np) {
    unsigned c = 0;
#pragma unroll
    for (int j = 0; j < kLayoutItems; ++j) {
        const long long g = g0 + j;
        np[j] = g < p.nkeys ? (p.koff[g + 1] - p.koff[g] + (unsigned)kGroupedPiece - 1u) / (unsigned)kGroupedPiece : 0u;
        c += np[j];
    }
    return c;
}

__global__ void __launch_bounds__(kLayoutThreads) grouped_piece_count_kernel(const LayoutParams p) {
    __shared__ unsigned wsum[kLayoutThreads / 32];
    unsigned np[kLayoutItems];
    const unsigned c = layout_pieces(p, (long long)blockIdx.x * kLayoutTile + (long long)threadIdx.x * kLayoutItems, np);
    unsigned total;
    layout_block_scan(c, wsum, total);
    if (threadIdx.x == 0) p.boff[blockIdx.x] = total;
}

__global__ void __launch_bounds__(kLayoutThreads) grouped_piece_write_kernel(const LayoutParams p) {
    __shared__ unsigned wsum[kLayoutThreads / 32];
    unsigned np[kLayoutItems];
    const long long g0 = (long long)blockIdx.x * kLayoutTile + (long long)threadIdx.x * kLayoutItems;
    const unsigned c = layout_pieces(p, g0, np);
    unsigned total;
    unsigned at = p.boff[blockIdx.x] + layout_block_scan(c, wsum, total);
#pragma unroll
    for (int j = 0; j < kLayoutItems; ++j) {
        const long long g = g0 + j;
        if (g >= p.nkeys) break;
        p.kpiece[g] = at;
        for (unsigned q = 0; q < np[j]; ++q, ++at) {
            p.pstart[at] = p.koff[g] + q * (unsigned)kGroupedPiece;
            p.pkey[at] = (uint32_t)g;
        }
        if (g == p.nkeys - 1) {
            p.kpiece[p.nkeys] = at;
            p.pstart[at] = p.koff[p.nkeys];
        }
    }
}

// the shard row of every position
__global__ void __launch_bounds__(kLayoutThreads) grouped_rows_kernel(const LayoutParams p) {
    const unsigned long long mask = (1ull << p.rbits) - 1ull;
    for (long long i = (long long)blockIdx.x * kLayoutThreads + threadIdx.x; i < (long long)*p.npos; i += (long long)gridDim.x * kLayoutThreads)
        p.rows[i] = (uint32_t)(p.uniq[i] & mask);
}

// ------------------------------------------------------------------ candidate filter
// One warp per stream.  thresholds: a row of stream s can only enter the reference's slots if its distance
// is below the k-th smallest distance among ALL earlier rows; any subset of earlier rows gives a valid upper
// bound.  We use  min( k-th smallest over all streams of earlier segments,
//                      k-th smallest over the earlier streams of the same segment ),
// both built from the streams' final k-lists (each contains the k smallest values of its stream).
// Result head of one query, written by filter_kernel; this is what a host copy or a peer push moves:
//   [ResultHead, 64 B][block table: kTableCap x int2 (base, count)][first kFirstFetch survivors x uint2 (dist bits, local row)]
// The survivors of block b are base .. base + count - 1 of the survivor list, and the blocks in table order are the scan order.
// Survivors beyond the head's capacity go to a separate tail area.
constexpr int kTableCap = 512;
constexpr int kFirstFetch = 1024;
constexpr int kHeadOverflow = 1;    // flags: the candidate log or the survivor list overflowed (all-distances fallback)
constexpr int kHeadPeerLate = 8;    // flags: exchange_wait_kernel gave up waiting for this head (set with a plain store)
struct ResultHead {
    int total;          // survivors
    int flags;          // kHeadOverflow, kHeadPeerLate
    int seq;            // the slot's query sequence number
    int nblocks;        // filter blocks = entries of the block table
    int xseq;           // exchange sequence number (pushed heads)
    int src;            // shard that wrote the head (pushed heads)
    int headcap;        // survivors stored in the head itself
    int pad[9];
};
static_assert(sizeof(ResultHead) == 64, "the header is 8 uint2 words (push_heads_kernel)");
static_assert(offsetof(ResultHead, total) == 0 && offsetof(ResultHead, flags) == 4 && offsetof(ResultHead, seq) == 8 &&
                  offsetof(ResultHead, nblocks) == 12 && offsetof(ResultHead, xseq) == 16 && offsetof(ResultHead, src) == 20 &&
                  offsetof(ResultHead, headcap) == 24,
              "tests/test_result_head.py builds heads with these offsets");
constexpr size_t kResHdrBytes = sizeof(ResultHead) + sizeof(int2) * kTableCap;
constexpr size_t kHeadBytes = kResHdrBytes + sizeof(uint2) * kFirstFetch;
inline int2 *head_table(ResultHead *h) { return reinterpret_cast<int2 *>(h + 1); }
inline const int2 *head_table(const ResultHead *h) { return reinterpret_cast<const int2 *>(h + 1); }
inline uint2 *head_survivors(ResultHead *h) { return reinterpret_cast<uint2 *>(reinterpret_cast<uint8_t *>(h) + kResHdrBytes); }
inline const uint2 *head_survivors(const ResultHead *h) { return reinterpret_cast<const uint2 *>(reinterpret_cast<const uint8_t *>(h) + kResHdrBytes); }

// NVLink peer-memory all-gather: push_heads_kernel, after a group's filters, copies the used part of each head (header, block
// table, survivors) straight into the gather buffer of every target GPU — peer memory mapped through cudaIpc (one process per
// GPU) or cudaDeviceEnablePeerAccess (one process, several GPUs) — and then raises that target's arrival flag with a
// system-scope release store.  No NCCL kernel, no host synchronisation: the receiving side waits on the flags with exchange_wait_kernel on
// ITS stream and copies the gathered heads to the host.
constexpr int kMaxPeers = 16;
struct PushParams {
    int ntargets;                 // 0: nothing is pushed (single shard)
    int src;                      // this shard's index inside a slot's gather row
    int world;                    // shards per slot in the gather layout [slots][world][kHeadBytes]
    int tailcap;                 // survivors beyond the head's headcap travel to a separate tail row of this many entries
    uint8_t *gather[kMaxPeers];   // target t: base of its gather buffer
    unsigned *flags[kMaxPeers];   // target t: [slots][world] arrival flags (the exchange sequence number of the slot)
    uint2 *tails[kMaxPeers];      // target t: [slots][world][tailcap] tail rows (k > 32 on large shards: > headcap survivors)
};

__device__ __forceinline__ void st_release_sys(unsigned *p, unsigned v) {
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned ld_acquire_sys(const unsigned *p) {
    unsigned v;
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}

// receiving side: one thread per (slot of the group, source shard) spins until that shard's flag carries the expected
// sequence number.  Bounded: after `timeout` clock cycles the missing head's flags are set to kHeadPeerLate (a plain store:
// whatever else the head holds is stale) so that the merge reports an error instead of the GPU hanging on a peer that died.
struct WaitParams {
    const unsigned *flags;        // [slots][world]
    uint8_t *gather;              // [slots][world][kHeadBytes] (local)
    int world, first_slot, nq;
    unsigned xseq[kMaxGroup];
    long long timeout;
};
__global__ void exchange_wait_kernel(const WaitParams wp) {
    const int t = threadIdx.x;
    if (t >= wp.nq * wp.world) return;
    const int j = t / wp.world, r = t % wp.world;
    const size_t at = (size_t)(wp.first_slot + j) * wp.world + r;
    const long long t0 = clock64();
    while (ld_acquire_sys(wp.flags + at) != wp.xseq[j]) {
        if (clock64() - t0 > wp.timeout) {
            reinterpret_cast<ResultHead *>(wp.gather + at * kHeadBytes)->flags = kHeadPeerLate;
            break;
        }
        __nanosleep(200);
    }
}

// The heads of a finished group are pushed by their own small kernel on the exchange stream, so the filter stream never waits
// for NVLink acknowledgements.  Block j stores the used part of query j's head (header, block table, survivors; the survivors
// beyond headcap from the slot's tail area) into row (xslot, src) of every target and raises the targets' flags.  The heads
// are complete and visible: the kernel runs in stream order after the filters.
struct PushGroupParams {
    PushParams push;
    int nq, headcap;
    const ResultHead *hdr[kMaxGroup];
    const uint2 *out[kMaxGroup];
    const uint2 *out_tail[kMaxGroup];
    int xslot[kMaxGroup];
    unsigned xseq[kMaxGroup];
};
__global__ void push_heads_kernel(const PushGroupParams gp) {
    const int j = blockIdx.x;
    if (j >= gp.nq) return;
    const PushParams &pp = gp.push;
    const ResultHead *hdr = gp.hdr[j];
    const int total = max(__ldcg(&hdr->total), 0), nblocks = __ldcg(&hdr->nblocks);
    const int nhead = (int)(sizeof(ResultHead) / sizeof(uint2)) + nblocks;   // uint2 words of header + block table
    const int nsurv = min(total, gp.headcap);
    const int ntail = min(max(total - gp.headcap, 0), pp.tailcap);
    const uint2 *src_head = reinterpret_cast<const uint2 *>(hdr);
    const size_t row = (size_t)gp.xslot[j] * pp.world + pp.src;
    for (int t = 0; t < pp.ntargets; ++t) {
        uint8_t *dst = pp.gather[t] + row * kHeadBytes;
        uint2 *dh = reinterpret_cast<uint2 *>(dst);
        uint2 *ds = reinterpret_cast<uint2 *>(dst + kResHdrBytes);
        for (int i = (int)threadIdx.x; i < nhead; i += (int)blockDim.x) dh[i] = __ldcg(src_head + i);
        for (int i = (int)threadIdx.x; i < nsurv; i += (int)blockDim.x) ds[i] = __ldcg(gp.out[j] + i);
        if (ntail > 0) {
            uint2 *dt = pp.tails[t] + row * (size_t)pp.tailcap;
            for (int i = (int)threadIdx.x; i < ntail; i += (int)blockDim.x) dt[i] = __ldcg(gp.out_tail[j] + i);
        }
    }
    __threadfence_system();
    __syncthreads();
    if ((int)threadIdx.x < pp.ntargets) st_release_sys(pp.flags[threadIdx.x] + row, gp.xseq[j]);
}

struct FilterParams {
    const float *lists; // k <= 32: [S / kWarps][32] sorted CTA lists; else [S][kcap] stream lists
    const float *tlocal;// k <= 32: [S] in-CTA prefix bound of each stream (from scan_kernel)
    const uint2 *logs;  // [S][logcap]
    const int *counts;  // [S]
    uint2 *out;         // survivors (dist bits, local row), grouped by block in stream order: the first headcap of them
    uint2 *out_tail;    //   go to out (inside the slot's head, the part that travels), the rest to out_tail
    int2 *table;        // [gridDim.x] (base, count) of each block's survivors in out
    ResultHead *hdr;
    int *ctrl;          // device: [0] cursor, [1] overflow from scan_kernel, [2] blocks done
    int seqno;
    int src;            // this shard's index inside a gather row (ResultHead::src)
    unsigned xseq;      // exchange sequence number published with the head (ResultHead::xseq)
    int S;              // streams
    int k, kcap;
    int logcap;
    int headcap;
    int outcap;         // total capacity (head + tail)
    // adaptive partition (k <= 32 path): the last block turns the scan's per-CTA cycles into new tile bounds, in place
    long long *bounds;          // [ncta + 1] or nullptr
    const unsigned *cta_time;   // [ncta]
    long long total_tiles;
};

constexpr int kFilterWarps = 32;      // generic path: streams (warps) per block
constexpr int kFilterWarpsFast = 8;   // k <= 32 path: small blocks (8 warps, ~21 KB smem) that fit on an SM NEXT TO a scan CTA, so
                                      // that the filter of query i runs while the scan of query i+1 streams (engine: two streams)
__host__ __device__ constexpr int filter_warps(bool fast) { return fast ? kFilterWarpsFast : kFilterWarps; }
// shared memory of the k <= 32 path: [kSegments][32] segment lists | [ncta4] per-CTA bound | [32] segment bounds | [ncta][32] CTA lists
__host__ __device__ constexpr size_t filter_fast_smem(int ncta) {
    return sizeof(float) * ((size_t)8 * 32 + (size_t)((ncta + 3) & ~3) + 32 + (size_t)ncta * 32);
}
constexpr int kSegments = 8;  // threshold segments: few long serial walks beat many short ones (issue-bound otherwise)
constexpr int kLogRegs = 8;   // log entries per lane prefetched into registers (256 per stream)

// FAST: k <= 32: scan_kernel published one sorted list per CTA plus each stream's in-CTA prefix bound; the lists are
// merged in registers (one L2 round trip for 19 KB of lists).
template <bool FAST>
__global__ void __launch_bounds__(filter_warps(FAST) * 32, 1) filter_kernel(const FilterParams fp) {
    constexpr int FW = filter_warps(FAST);
    static_assert(FW >= kSegments, "the segment walks use the first kSegments warps");
    extern __shared__ __align__(16) uint8_t fsm[];
    const int k = fp.k, kcap = fp.kcap;
    const int ncta = fp.S / kWarps;                                         // scan CTAs (FAST: each published one sorted list)
    // generic: [32][kcap] segment lists | [32][kcap] scratch | [S] in-segment prefix bound | [32] segment bounds
    // FAST:    see filter_fast_smem (kcap == 32)
    float *seglist = reinterpret_cast<float *>(fsm);
    float *work = seglist + kFilterWarps * kcap;                            // generic only
    float *tlocal = FAST ? seglist + kSegments * 32 : work + kFilterWarps * kcap;   // FAST: per-CTA bound
    float *tseg = tlocal + (FAST ? ((ncta + 3) & ~3) : fp.S);               // [32]
    float *slists = tseg + 32;                                              // FAST: [ncta][32] copy of the CTA lists
    __shared__ int wcount[FW], woff[FW];
    __shared__ int blk_base;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int G = (fp.S + kSegments - 1) / kSegments;                       // streams per segment (generic)

    // ---- issue this warp's log loads first: they do not depend on the thresholds
    const int s = blockIdx.x * FW + warp;
    int n_log = 0;
    uint2 ereg[kLogRegs];
    const uint2 *lg = fp.logs + (size_t)s * fp.logcap;
    if (s < fp.S) n_log = min(fp.counts[s], fp.logcap);
#pragma unroll
    for (int i = 0; i < kLogRegs; ++i) {
        const int j = i * 32 + lane;
        ereg[i] = (j < n_log) ? lg[j] : make_uint2(0x7FC00000u, 0u);       // NaN never survives
    }

    if constexpr (FAST) {
        const int GC = (ncta + kSegments - 1) / kSegments;                  // CTAs per segment
        {   // all CTA lists (ncta x 32 floats, ~19 KB) -> shared memory in one coalesced pass
            const float4 *src = reinterpret_cast<const float4 *>(fp.lists);
            float4 *dst = reinterpret_cast<float4 *>(slists);
            const int tot4 = ncta * 8;
            for (int i = (int)threadIdx.x; i < tot4; i += FW * 32) dst[i] = __ldg(src + i);
        }
        __syncthreads();
        if (warp < kSegments) {   // phase 1: warp g walks the CTAs of segment g in order, recording the running k-th value before each CTA
            SortedList L;
            L.init(lane, k);
            const int c0 = warp * GC, c1 = min(ncta, c0 + GC);
            for (int c = c0; c < c1; ++c) {
                if (lane == 0) tlocal[c] = L.thr;
                L.offer_sorted(lane, slists[c * 32 + lane]);
            }
            seglist[warp * kcap + lane] = L.v;
        }
        __syncthreads();
        if (warp < kSegments) {   // phase 2: warp g merges the lists of segments 0..g-1
            SortedList L;
            L.init(lane, k);
            for (int g = 0; g < warp; ++g) L.offer_sorted(lane, seglist[g * kcap + lane]);
            if (lane == 0) tseg[warp] = L.thr;
        }
        __syncthreads();
    } else {
        // generic path (any k): lists stay in global memory / L2, k-lists in shared memory
        if (warp < kSegments) {
            float *L = seglist + warp * kcap;
            for (int j = lane; j < kcap; j += 32) L[j] = (j < k) ? INFINITY : -INFINITY;
            __syncwarp();
            float thr = INFINITY;
            int pos = 0;
            const int s0 = warp * G, s1 = min(fp.S, s0 + G);
            for (int st = s0; st < s1; ++st) {
                if (lane == 0) tlocal[st] = thr;
                const float *src = fp.lists + (size_t)st * kcap;
                for (int base = 0; base < k; base += 32) {
                    const int j = base + lane;
                    const float v = (j < k) ? src[j] : INFINITY;
                    unsigned m = __ballot_sync(0xFFFFFFFFu, v < thr);
                    while (m) {
                        const int sl = __ffs(m) - 1;
                        m &= m - 1;
                        const float dv = __shfl_sync(0xFFFFFFFFu, v, sl);
                        if (dv < thr) {
                            if (lane == 0) L[pos] = dv;
                            __syncwarp();
                            list_argmax(L, kcap, lane, thr, pos);
                        }
                    }
                }
            }
        }
        __syncthreads();
        if (warp < kSegments) {
            float *L = work + warp * kcap;
            for (int j = lane; j < kcap; j += 32) L[j] = (j < k) ? INFINITY : -INFINITY;
            __syncwarp();
            float thr = INFINITY;
            int pos = 0;
            for (int g = 0; g < warp; ++g) {
                const float *src = seglist + g * kcap;
                for (int base = 0; base < k; base += 32) {
                    const int j = base + lane;
                    const float v = (j < k) ? src[j] : INFINITY;
                    unsigned m = __ballot_sync(0xFFFFFFFFu, v < thr);
                    while (m) {
                        const int sl = __ffs(m) - 1;
                        m &= m - 1;
                        const float dv = __shfl_sync(0xFFFFFFFFu, v, sl);
                        if (dv < thr) {
                            if (lane == 0) L[pos] = dv;
                            __syncwarp();
                            list_argmax(L, kcap, lane, thr, pos);
                        }
                    }
                }
            }
            if (lane == 0) tseg[warp] = thr;
        }
        __syncthreads();
    }

    // ---- phase 3: count, reserve, write — survivors of this block's 32 streams in stream order
    float T = INFINITY;
    if (s < fp.S) {
        if constexpr (FAST) {
            const int c = s / kWarps, GC = (ncta + kSegments - 1) / kSegments;
            T = fminf(fminf(__ldg(fp.tlocal + s), tlocal[c]), tseg[c / GC]);
        } else {
            T = fminf(tlocal[s], tseg[s / G]);
        }
    }
    int mine = 0;
#pragma unroll
    for (int i = 0; i < kLogRegs; ++i) mine += __popc(__ballot_sync(0xFFFFFFFFu, __uint_as_float(ereg[i].x) < T));
    for (int base = kLogRegs * 32; base < n_log; base += 32) {
        const int j = base + lane;
        const bool keep = (j < n_log) && (__uint_as_float(lg[j].x) < T);
        mine += __popc(__ballot_sync(0xFFFFFFFFu, keep));
    }
    if (lane == 0) wcount[warp] = mine;
    __syncthreads();
    if (threadIdx.x == 0) {
        int tot = 0;
        for (int w = 0; w < FW; ++w) { woff[w] = tot; tot += wcount[w]; }
        const int base = atomicAdd(&fp.ctrl[0], tot);
        blk_base = base;
        fp.table[blockIdx.x] = make_int2(base, tot);
    }
    __syncthreads();
    int wr = blk_base + woff[warp];
#pragma unroll
    for (int i = 0; i < kLogRegs; ++i) {
        const bool keep = __uint_as_float(ereg[i].x) < T;
        const unsigned m = __ballot_sync(0xFFFFFFFFu, keep);
        const int off = wr + __popc(m & ((1u << lane) - 1u));
        if (keep && off < fp.outcap) *(off < fp.headcap ? fp.out + off : fp.out_tail + (off - fp.headcap)) = ereg[i];
        wr += __popc(m);
    }
    for (int base = kLogRegs * 32; base < n_log; base += 32) {
        const int j = base + lane;
        uint2 e = make_uint2(0, 0);
        bool keep = false;
        if (j < n_log) { e = lg[j]; keep = __uint_as_float(e.x) < T; }
        const unsigned m = __ballot_sync(0xFFFFFFFFu, keep);
        const int off = wr + __popc(m & ((1u << lane) - 1u));
        if (keep && off < fp.outcap) *(off < fp.headcap ? fp.out + off : fp.out_tail + (off - fp.headcap)) = e;
        wr += __popc(m);
    }
    if constexpr (FAST) {
        // ---- adaptive partition: share of CTA c for the query after next  ∝  its measured speed (tiles per cycle), damped
        if (fp.bounds != nullptr && blockIdx.x == gridDim.x - 1 && fp.total_tiles >= 64ll * ncta && ncta <= 1024) {
            __shared__ float spd[1024];
            __shared__ int bad;
            if (threadIdx.x == 0) bad = 0;
            __syncthreads();
            for (int c = threadIdx.x; c < ncta; c += FW * 32) {
                const float tiles = (float)(fp.bounds[c + 1] - fp.bounds[c]);
                const unsigned t = fp.cta_time[c];
                if (t == 0u || !(tiles > 0.0f)) bad = 1;
                spd[c] = tiles / (float)max(t, 1u);
            }
            __syncthreads();
            if (threadIdx.x == 0 && !bad) {
                double sum = 0.0;
                for (int c = 0; c < ncta; ++c) sum += (double)spd[c];
                double acc = 0.0;                       // running boundary in tiles
                long long prev = 0;
                for (int c = 0; c < ncta; ++c) {
                    const double cur = (double)(fp.bounds[c + 1] - prev);            // old share (prev = old bounds[c])
                    const double want = (double)fp.total_tiles * (double)spd[c] / sum;
                    prev = fp.bounds[c + 1];
                    acc += 0.5 * cur + 0.5 * want;
                    long long b = (c == ncta - 1) ? fp.total_tiles : (long long)(acc + 0.5);
                    const long long lo = fp.bounds[c] + kWarps;                       // every CTA keeps at least one tile per warp
                    if (b < lo) b = lo;
                    if (b > fp.total_tiles) b = fp.total_tiles;
                    fp.bounds[c + 1] = b;
                }
            }
            __syncthreads();
        }
    }
    // last block publishes the header and re-arms the control words for the next query.  The host only reads the
    // mapped buffers after the stream has drained, so device-scope ordering between blocks is all that is needed.
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) {
        const int done = atomicAdd(&fp.ctrl[2], 1);
        if (done == (int)gridDim.x - 1) {
            __threadfence();
            const int total = atomicAdd(&fp.ctrl[0], 0);
            const int ovf = atomicAdd(&fp.ctrl[1], 0);
            fp.hdr->total = total;
            fp.hdr->flags = (ovf != 0 || total > fp.outcap) ? kHeadOverflow : 0;
            fp.hdr->seq = fp.seqno;
            fp.hdr->nblocks = (int)gridDim.x;
            fp.hdr->xseq = (int)fp.xseq;
            fp.hdr->src = fp.src;
            fp.hdr->headcap = fp.headcap;
            fp.ctrl[0] = 0; fp.ctrl[1] = 0; fp.ctrl[2] = 0;
        }
    }
}

}  // namespace vsb
