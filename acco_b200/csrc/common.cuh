// Shared device helpers for the acco_b200 sm_90a kernels.
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#define ACCO_DEVINL __device__ __forceinline__

namespace acco {

constexpr int kWarp = 32;

// ---- 16-byte vectors of 8 bf16 -------------------------------------------------------------
struct alignas(16) bf16x8 {
    __nv_bfloat162 v[4];
};

ACCO_DEVINL void unpack8(const bf16x8& p, float (&f)[8]) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        float2 t = __bfloat1622float2(p.v[i]);
        f[2 * i] = t.x;
        f[2 * i + 1] = t.y;
    }
}

ACCO_DEVINL bf16x8 pack8(const float (&f)[8]) {
    bf16x8 p;
#pragma unroll
    for (int i = 0; i < 4; ++i) p.v[i] = __floats2bfloat162_rn(f[2 * i], f[2 * i + 1]);
    return p;
}

// streaming (read-once / write-once) 16-byte global accesses: keep them out of L1
ACCO_DEVINL bf16x8 ld_stream(const void* ptr) {
    uint4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
                 : "l"(ptr));
    return *reinterpret_cast<bf16x8*>(&r);
}
// same, for buffers that this kernel also writes (no .nc)
ACCO_DEVINL bf16x8 ld_stream_rw(const void* ptr) {
    uint4 r;
    asm volatile("ld.global.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
                 : "l"(ptr)
                 : "memory");
    return *reinterpret_cast<bf16x8*>(&r);
}
ACCO_DEVINL bf16x8 ld_vec(const void* ptr) { return *reinterpret_cast<const bf16x8*>(ptr); }
ACCO_DEVINL void st_vec(void* ptr, const bf16x8& v) { *reinterpret_cast<bf16x8*>(ptr) = v; }
ACCO_DEVINL void st_stream(void* ptr, const bf16x8& v) {
    const uint4& r = *reinterpret_cast<const uint4*>(&v);
    asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(ptr), "r"(r.x), "r"(r.y), "r"(r.z),
                 "r"(r.w)
                 : "memory");
}

ACCO_DEVINL float4 ld_f4_stream(const float* ptr) {
    float4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
                 : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w)
                 : "l"(ptr));
    return r;
}

// ---- reductions ----------------------------------------------------------------------------
ACCO_DEVINL float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
ACCO_DEVINL float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// block-wide sum over up to 32 warps; `smem` must hold 32 floats. All threads get the result.
ACCO_DEVINL float block_sum(float v, float* smem) {
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
    v = warp_sum(v);
    __syncthreads();
    if (lane == 0) smem[wid] = v;
    __syncthreads();
    v = (lane < nw) ? smem[lane] : 0.f;
    return warp_sum(v);
}
ACCO_DEVINL float block_max(float v, float* smem) {
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
    v = warp_max(v);
    __syncthreads();
    if (lane == 0) smem[wid] = v;
    __syncthreads();
    v = (lane < nw) ? smem[lane] : -INFINITY;
    return warp_max(v);
}

}  // namespace acco
