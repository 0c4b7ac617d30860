// quant_kernels.cuh — GPU side of vector_quantize (/root/reference/src/sqlite-vector.c:1147-1336).
//
// Pass 1 reduces min / max / "a negative value exists" over the column (:1224-1256), pass 2 encodes every row into the
// shadow-table chunk format [int64 LE rowid][dim x 8-bit] (:1295-1311) with the arithmetic of quantize_* / q_round_* (:495-757):
//   s = (v - offset) * scale       two separately rounded fp32 operations
//   r = s + (s < 0 ? -0.5 : +0.5)  round half away from zero
//   f32 sources: (int) cast, then clamp (the x86 cast yields INT_MIN for NaN and for |r| >= 2^31: reproduced here);
//   other sources: the NaN / Inf-safe q_round_u8 / q_round_s8.
// Byte-identical output is the bar (tests/golden/sql_surface.json holds the reference's chunk hex dumps).
#pragma once
#include "scan_kernels.cuh"

namespace vsb {

template <int VT>
__device__ __forceinline__ float quant_src(const uint8_t *row, int i) {       // elem as fp32, like the reference's per-type loops
    if constexpr (VT == T_F32) return reinterpret_cast<const float *>(row)[i];
    else if constexpr (VT == T_F16) return __half2float(__ushort_as_half(reinterpret_cast<const uint16_t *>(row)[i]));
    else if constexpr (VT == T_BF16) return __uint_as_float((uint32_t)reinterpret_cast<const uint16_t *>(row)[i] << 16);
    else if constexpr (VT == T_U8) return (float)row[i];
    else return (float)reinterpret_cast<const int8_t *>(row)[i];
}

// acc[0] = key of the minimum, acc[1] = key of the maximum (fkey order; NaN never enters, like `x < lo` / `x > hi`),
// acc[2] = 1 when a value < 0 exists.  Initialise with {0xFFFFFFFF, 0, 0}.
template <int VT>
__global__ void quant_minmax_kernel(const uint8_t *rows, long long nelem, unsigned *acc) {
    unsigned lo = 0xFFFFFFFFu, hi = 0u, neg = 0u;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nelem; i += (long long)gridDim.x * blockDim.x) {
        float x;
        if constexpr (VT == T_F32) x = reinterpret_cast<const float *>(rows)[i];
        else if constexpr (VT == T_F16) x = __half2float(__ushort_as_half(reinterpret_cast<const uint16_t *>(rows)[i]));
        else if constexpr (VT == T_BF16) x = __uint_as_float((uint32_t)reinterpret_cast<const uint16_t *>(rows)[i] << 16);
        else if constexpr (VT == T_U8) x = (float)rows[i];
        else x = (float)reinterpret_cast<const int8_t *>(rows)[i];
        if (x == x) {
            const unsigned kx = fkey(x);
            lo = min(lo, kx);
            hi = max(hi, kx);
            neg |= (x < 0.0f) ? 1u : 0u;
        }
    }
    lo = __reduce_min_sync(0xFFFFFFFFu, lo);
    hi = __reduce_max_sync(0xFFFFFFFFu, hi);
    neg = __reduce_or_sync(0xFFFFFFFFu, neg);
    if ((threadIdx.x & 31) == 0) {
        atomicMin(&acc[0], lo);
        atomicMax(&acc[1], hi);
        if (neg) atomicOr(&acc[2], 1u);
    }
}

__device__ __forceinline__ int x86_float_to_int(float r) {       // cvttss2si: "integer indefinite" for NaN and out-of-range values
    return (r != r || !(fabsf(r) < 2147483648.0f)) ? (int)0x80000000 : __float2int_rz(r);
}

// one thread per element; out row r = [rowid LE 8 B][dim bytes] at out + r * (8 + dim)
template <int VT>
__global__ void quant_encode_kernel(const uint8_t *rows, const long long *rowids, long long nrows, int dim, float offset, float scale, int qtype_u8,
                                    uint8_t *out) {
    const long long total = nrows * dim;
    const size_t es = (VT == T_F32) ? 4 : ((VT == T_F16 || VT == T_BF16) ? 2 : 1);
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const long long r = i / dim;
        const int c = (int)(i - r * dim);
        const float x = quant_src<VT>(rows + (size_t)r * dim * es, c);
        const float s = __fmul_rn(__fsub_rn(x, offset), scale);
        const float adj = (s < 0.0f) ? -0.5f : 0.5f;
        uint8_t q;
        if constexpr (VT == T_F32) {
            const int v = x86_float_to_int(__fadd_rn(s, adj));
            q = qtype_u8 ? (uint8_t)(v > 255 ? 255 : (v < 0 ? 0 : v)) : (uint8_t)(int8_t)(v > 127 ? 127 : (v < -128 ? -128 : v));
        } else if (qtype_u8) {
            if (!(fabsf(s) <= FLT_MAX)) q = (s > 0.0f) ? 255u : 0u;                    // q_round_u8: NaN -> 0, +Inf -> 255, -Inf -> 0
            else {
                const float rr = __fadd_rn(s, adj);
                q = rr >= 255.0f ? 255u : (rr <= 0.0f ? 0u : (uint8_t)__float2int_rz(rr));
            }
        } else {
            if (!(fabsf(s) <= FLT_MAX)) q = (uint8_t)(int8_t)((s > 0.0f) ? 127 : (s < 0.0f ? -128 : 0));
            else {
                const float rr = __fadd_rn(s, adj);
                q = (uint8_t)(int8_t)(rr >= 127.0f ? 127 : (rr <= -128.0f ? -128 : __float2int_rz(rr)));
            }
        }
        uint8_t *o = out + (size_t)r * (8 + (size_t)dim);
        o[8 + c] = q;
        // little-endian rowid (INT64_TO_INT8PTR, :75-85): the row's threads cover bytes c, c + dim, ... < 8, so all 8 are written
        // even when dim < 8
        for (int b = c; b < 8; b += dim) o[b] = (uint8_t)((unsigned long long)rowids[r] >> (8 * b));
    }
}

}  // namespace vsb
