// FP8 quantisation for the FP8 linear layers (ops/fp8.py): per-tensor "current" scaling of a bf16 matrix t [R, C].
//
//   amax(t) = max |t|;  s = 2^floor(log2(max_f / amax)) (max_e4m3 = 448, max_e5m2 = 57344);  amax = 0 -> s = 1;  amax not finite -> NaN
//   q(t)    = t * s rounded to nearest even in the format (cvt.rn.satfinite: never saturates, every |t * s| <= max_f)
//
// fp8_amax_kernel : per-CTA maxima of |t| as bf16 bit patterns (an unsigned max over the sign-cleared bits orders finite values,
//                   puts Inf above them and NaN above Inf, so a NaN or Inf anywhere reaches the scale).  Max is order-independent: the
//                   result does not depend on the grid.
// fp8_cast_kernel : every CTA reduces those maxima (at most kMaxAmaxCtas), derives s exactly from the exponent of amax, and CTA 0
//                   writes {s, 1/s, amax} for the GEMM epilogues.  Each CTA quantises a 64 x 64 tile read once: row-major q [R, C]
//                   (8-byte stores) and / or the transpose qT [C, R] through shared memory (16-byte stores, four threads per 64-byte run).
// No host round trip: the chain amax -> cast -> GEMM reads the scale from device memory, so it can be captured in a CUDA graph.
#include <stdint.h>

#include "common.cuh"

namespace acco_fp8 {

constexpr int kMaxAmaxCtas = 1024;
constexpr int kTile = 64;
constexpr int kPitch = kTile + 4;     // bytes per shared-memory row of the quantised tile

__device__ __forceinline__ uint32_t warp_umax(uint32_t v) { return __reduce_max_sync(0xffffffffu, v); }

// 256 threads: max over the block, every thread gets it
__device__ __forceinline__ uint32_t block_umax(uint32_t v, uint32_t* red) {
    v = warp_umax(v);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    v = red[threadIdx.x & 7];
    return warp_umax(v);
}

__global__ void __launch_bounds__(256) fp8_amax_kernel(const uint4* __restrict__ t, long long n8, uint32_t* __restrict__ partial) {
    __shared__ uint32_t red[8];
    uint32_t m = 0;
    for (long long i = blockIdx.x * 256ll + threadIdx.x; i < n8; i += (long long)gridDim.x * 256) {
        const uint4 v = __ldg(t + i);
        const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) m = max(m, max(w[j] & 0x7FFFu, (w[j] >> 16) & 0x7FFFu));
    }
    m = block_umax(m, red);
    if (threadIdx.x == 0) partial[blockIdx.x] = m;
}

// s = 2^k with k the largest integer such that amax * 2^k <= max_f = 1.75 * 2^e_max, computed from the exponent and mantissa of amax
// (exact, no rounding).  k is capped at 127 so that s stays a finite fp32; 1/s is then the subnormal 2^-127.
__device__ __forceinline__ void scale_from_amax(uint32_t amax_bits, int e_max, float& s, float& inv_s) {
    if (amax_bits == 0) { s = 1.f; inv_s = 1.f; return; }
    if (amax_bits >= 0x7F80u) { s = __int_as_float(0x7FC00000); inv_s = s; return; }
    const uint32_t exp_f = amax_bits >> 7, man = amax_bits & 0x7Fu;
    int e;                        // amax = (1 + m) * 2^e, m in [0, 1)
    uint32_t mant7;               // 7-bit mantissa after normalisation
    if (exp_f == 0) {             // subnormal bf16: man * 2^-133
        const int lead = 31 - __clz(man);
        e = -133 + lead;
        mant7 = (man << (7 - lead)) & 0x7Fu;
    } else {
        e = (int)exp_f - 127;
        mant7 = man;
    }
    int k = e_max - e - (mant7 > 0x60u ? 1 : 0);     // 1.75 = 1 + 0x60 / 128
    if (k > 127) k = 127;
    s = __int_as_float((k + 127) << 23);
    inv_s = k <= 126 ? __int_as_float((127 - k) << 23) : __int_as_float(0x00400000);
}

__device__ __forceinline__ float mul_exact(float a, float b) {      // no flush-to-zero of subnormal inputs (this file builds with fast math)
    float r;
    asm("mul.rn.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
    return r;
}

template <int E5M2>
__device__ __forceinline__ uint16_t cvt2(float lo, float hi) {
    uint16_t r;
    if constexpr (E5M2) asm("cvt.rn.satfinite.e5m2x2.f32 %0, %1, %2;" : "=h"(r) : "f"(hi), "f"(lo));
    else asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(r) : "f"(hi), "f"(lo));
    return r;
}

// t [R, C] bf16 (row stride C) -> q [R, C] and / or qT [C, R] (either may be null); R % 16 == 0, C % 16 == 0.
// scale_out: {s, 1/s, amax}.
template <int E5M2>
__global__ void __launch_bounds__(256) fp8_cast_kernel(const __nv_bfloat16* __restrict__ t, const uint32_t* __restrict__ partial, int n_partial,
                                                       uint8_t* __restrict__ q, uint8_t* __restrict__ qT, float* __restrict__ scale_out, int R,
                                                       int C) {
    __shared__ uint32_t red[8];
    __shared__ __align__(16) uint8_t tile[kTile * kPitch];
    uint32_t m = 0;
    for (int i = threadIdx.x; i < n_partial; i += 256) m = max(m, partial[i]);
    m = block_umax(m, red);
    float s, inv_s;
    scale_from_amax(m, E5M2 ? 15 : 8, s, inv_s);
    if (blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0) {
        scale_out[0] = s;
        scale_out[1] = inv_s;
        scale_out[2] = __uint_as_float(m << 16);
    }
    const int r0 = blockIdx.y * kTile, c0 = blockIdx.x * kTile;
    const int cc = (threadIdx.x & 7) * 8;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        const int rr = (threadIdx.x >> 3) + 32 * i, r = r0 + rr, c = c0 + cc;
        uint2 packed = make_uint2(0u, 0u);
        if (r < R && c < C) {
            float f[8];
            acco::unpack8(acco::ld_stream(t + (size_t)r * C + c), f);
            uint16_t h[4];
#pragma unroll
            for (int j = 0; j < 4; ++j) h[j] = cvt2<E5M2>(mul_exact(f[2 * j], s), mul_exact(f[2 * j + 1], s));
            packed.x = (uint32_t)h[0] | ((uint32_t)h[1] << 16);
            packed.y = (uint32_t)h[2] | ((uint32_t)h[3] << 16);
            if (q != nullptr) *reinterpret_cast<uint2*>(q + (size_t)r * C + c) = packed;
        }
        if (qT != nullptr) {
            uint32_t* row = reinterpret_cast<uint32_t*>(tile + rr * kPitch + cc);
            row[0] = packed.x;
            row[1] = packed.y;
        }
    }
    if (qT == nullptr) return;
    __syncthreads();
    // transposed: thread -> column c0 + tc, rows [r0 + tr, r0 + tr + 16): one 16-byte store
    const int tc = threadIdx.x >> 2, tr = (threadIdx.x & 3) * 16;
    if (c0 + tc >= C || r0 + tr >= R) return;
    uint32_t w[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const uint8_t* p = tile + (tr + 4 * j) * kPitch + tc;
        w[j] = (uint32_t)p[0] | ((uint32_t)p[kPitch] << 8) | ((uint32_t)p[2 * kPitch] << 16) | ((uint32_t)p[3 * kPitch] << 24);
    }
    *reinterpret_cast<uint4*>(qT + (size_t)(c0 + tc) * R + r0 + tr) = make_uint4(w[0], w[1], w[2], w[3]);
}

}  // namespace acco_fp8

extern "C" int acco_fp8_amax_ctas(long long n, int sms) {
    long long g = (n / 8 + 256 * 4 - 1) / (256 * 4);       // >= 4 vectors per thread
    if (g > 2ll * sms) g = 2ll * sms;
    if (g > acco_fp8::kMaxAmaxCtas) g = acco_fp8::kMaxAmaxCtas;
    return g < 1 ? 1 : (int)g;
}

// t [R, C] bf16 -> q [R, C] (or null), qT [C, R] (or null) in e4m3 (e5m2 = 0) or e5m2; scale_out float[3 + ctas] (its tail holds the
// per-CTA maxima); ctas from acco_fp8_amax_ctas.
extern "C" int acco_fp8_quantize(const void* t, int R, int C, int e5m2, void* q, void* qT, float* scale_out, int ctas, cudaStream_t st) {
    if (R <= 0 || C <= 0 || (R % 16) || (C % 16) || ((uintptr_t)t % 16) || ((uintptr_t)q % 16) || ((uintptr_t)qT % 16)) return -1;
    if (ctas < 1 || ctas > acco_fp8::kMaxAmaxCtas) return -1;
    uint32_t* partial = reinterpret_cast<uint32_t*>(scale_out + 3);
    acco_fp8::fp8_amax_kernel<<<ctas, 256, 0, st>>>((const uint4*)t, (long long)R * C / 8, partial);
    const dim3 grid((C + acco_fp8::kTile - 1) / acco_fp8::kTile, (R + acco_fp8::kTile - 1) / acco_fp8::kTile);
    if (e5m2)
        acco_fp8::fp8_cast_kernel<1><<<grid, 256, 0, st>>>((const __nv_bfloat16*)t, partial, ctas, (uint8_t*)q, (uint8_t*)qT, scale_out, R, C);
    else
        acco_fp8::fp8_cast_kernel<0><<<grid, 256, 0, st>>>((const __nv_bfloat16*)t, partial, ctas, (uint8_t*)q, (uint8_t*)qT, scale_out, R, C);
    return (int)cudaGetLastError();
}
