// RoPE (in place on the fused QKV buffer) and SwiGLU forward/backward.  Pure streaming kernels:
// 16-byte vector accesses, one pass, grid sized by the caller's element count.
#include <stdlib.h>

#include "common.cuh"

namespace acco {

// RoPE kernels: ONE WARP PER TOKEN.  lane = (head group, 8-pair vector): the cos/sin values of the token are
// loaded once per lane and reused for every head the lane visits; no integer divisions in the inner loop; the
// warp consumes the token's whole QKV row (contiguous 2*(Hq+Hk)*D bytes).
//   out1 = x1*cos - x2*sin ; out2 = x2*cos + x1*sin      (inverse: sin -> -sin)
ACCO_DEVINL void load_cs(const float* __restrict__ cos_t, const float* __restrict__ sin_t, int pos, int half, int v, float (&c)[8],
                         float (&s)[8]) {
    const float4* cp = reinterpret_cast<const float4*>(cos_t + (size_t)pos * half + 8 * v);
    const float4* sp = reinterpret_cast<const float4*>(sin_t + (size_t)pos * half + 8 * v);
    const float4 c0 = __ldg(cp), c1 = __ldg(cp + 1), s0 = __ldg(sp), s1 = __ldg(sp + 1);
    c[0] = c0.x; c[1] = c0.y; c[2] = c0.z; c[3] = c0.w; c[4] = c1.x; c[5] = c1.y; c[6] = c1.z; c[7] = c1.w;
    s[0] = s0.x; s[1] = s0.y; s[2] = s0.z; s[3] = s0.w; s[4] = s1.x; s[5] = s1.y; s[6] = s1.z; s[7] = s1.w;
}

// qkv: [T, n_total, D] bf16 (T = B*S, position = t % S).  Rotates heads [0, n_rot) in place (HF rotate_half pairing).
__global__ void __launch_bounds__(256) rope_qkv_kernel(__nv_bfloat16* __restrict__ qkv, const float* __restrict__ cos_t,
                                                       const float* __restrict__ sin_t, int T, int S, int n_rot,
                                                       int n_total, int D, float sign) {
    const int half = D >> 1;
    const int vph = half >> 3;                  // 8-pair vectors per head (power of two, <= 32)
    const int lane = threadIdx.x & 31;
    const int v = lane % vph, hg = lane / vph, hstep = 32 / vph;
    const int warps = (gridDim.x * blockDim.x) >> 5;
    for (int t = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; t < T; t += warps) {
        float c[8], s[8];
        load_cs(cos_t, sin_t, t % S, half, v, c, s);
        __nv_bfloat16* row = qkv + (size_t)t * n_total * D + 8 * v;
        for (int h = hg; h < n_rot; h += hstep) {
            __nv_bfloat16* p1 = row + (size_t)h * D;
            float x1[8], x2[8], o1[8], o2[8];
            unpack8(ld_vec(p1), x1);
            unpack8(ld_vec(p1 + half), x2);
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const float sj = sign * s[j];
                o1[j] = x1[j] * c[j] - x2[j] * sj;
                o2[j] = x2[j] * c[j] + x1[j] * sj;
            }
            st_vec(p1, pack8(o1));
            st_vec(p1 + half, pack8(o2));
        }
    }
}

// Backward companion: gather the three attention gradients dq [B,S,Hq,D], dk/dv [B,S,Hk,D] (arbitrary
// b/s/h strides, d contiguous) into ONE fused d(qkv) buffer [T, Hq+2Hk, D], applying the inverse rotation
// to the q and k heads on the way.  One pass instead of autograd's zero-fill + slice-copy + add chain.
struct PackSrc {
    const __nv_bfloat16* ptr[3];
    long long sb[3], ss[3], sh[3];   // element strides of (batch, seq, head)
};
__global__ void __launch_bounds__(256) rope_pack_bwd_kernel(PackSrc src, __nv_bfloat16* __restrict__ dqkv,
                                                            const float* __restrict__ cos_t, const float* __restrict__ sin_t,
                                                            int B, int S, int Hq, int Hk, int D) {
    const int half = D >> 1;
    const int vph = half >> 3;
    const int n_total = Hq + 2 * Hk;
    const int lane = threadIdx.x & 31;
    const int v = lane % vph, hg = lane / vph, hstep = 32 / vph;
    const int warps = (gridDim.x * blockDim.x) >> 5;
    const int T = B * S;
    for (int t = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; t < T; t += warps) {
        const int s = t % S, b = t / S;
        float c[8], sn[8];
        load_cs(cos_t, sin_t, s, half, v, c, sn);
        __nv_bfloat16* orow = dqkv + (size_t)t * n_total * D + 8 * v;
        for (int head = hg; head < n_total; head += hstep) {
            int which, h;
            if (head < Hq) { which = 0; h = head; }
            else if (head < Hq + Hk) { which = 1; h = head - Hq; }
            else { which = 2; h = head - Hq - Hk; }
            const __nv_bfloat16* p1 = src.ptr[which] + b * src.sb[which] + s * src.ss[which] + h * src.sh[which] + 8 * v;
            float x1[8], x2[8];
            unpack8(ld_stream(p1), x1);
            unpack8(ld_stream(p1 + half), x2);
            __nv_bfloat16* o1 = orow + (size_t)head * D;
            if (which == 2) {
                st_vec(o1, pack8(x1));
                st_vec(o1 + half, pack8(x2));
            } else {
                float r1[8], r2[8];
#pragma unroll
                for (int j = 0; j < 8; ++j) {      // inverse rotation: sin -> -sin
                    r1[j] = x1[j] * c[j] + x2[j] * sn[j];
                    r2[j] = x2[j] * c[j] - x1[j] * sn[j];
                }
                st_vec(o1, pack8(r1));
                st_vec(o1 + half, pack8(r2));
            }
        }
    }
}

// gu: [T, 2I] (gate | up) -> out [T, I] = silu(gate) * up
__global__ void __launch_bounds__(256) swiglu_fwd_kernel(const __nv_bfloat16* __restrict__ gu, __nv_bfloat16* __restrict__ out,
                                                         long long T, int I) {
    const int vpr = I >> 3;
    const long long total = T * vpr;
    for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
         idx += (long long)gridDim.x * blockDim.x) {
        const long long t = idx / vpr;
        const int v = (int)(idx % vpr);
        const __nv_bfloat16* g = gu + t * 2 * I + 8 * v;
        float fg[8], fu[8], o[8];
        unpack8(ld_stream(g), fg);
        unpack8(ld_stream(g + I), fu);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const float sg = 1.f / (1.f + __expf(-fg[j]));
            o[j] = fg[j] * sg * fu[j];
        }
        st_stream(out + t * I + 8 * v, pack8(o));
    }
}

// dgu [T, 2I]:  dgate = dout * up * sig(g) * (1 + g*(1-sig(g)));  dup = dout * silu(g)
__global__ void __launch_bounds__(256) swiglu_bwd_kernel(const __nv_bfloat16* __restrict__ dout,
                                                         const __nv_bfloat16* __restrict__ gu, __nv_bfloat16* __restrict__ dgu,
                                                         long long T, int I) {
    const int vpr = I >> 3;
    const long long total = T * vpr;
    for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
         idx += (long long)gridDim.x * blockDim.x) {
        const long long t = idx / vpr;
        const int v = (int)(idx % vpr);
        const __nv_bfloat16* g = gu + t * 2 * I + 8 * v;
        float fg[8], fu[8], fd[8], dg[8], du[8];
        unpack8(ld_stream(g), fg);
        unpack8(ld_stream(g + I), fu);
        unpack8(ld_stream(dout + t * I + 8 * v), fd);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const float sg = 1.f / (1.f + __expf(-fg[j]));
            const float silu = fg[j] * sg;
            dg[j] = fd[j] * fu[j] * sg * (1.f + fg[j] * (1.f - sg));
            du[j] = fd[j] * silu;
        }
        __nv_bfloat16* o = dgu + t * 2 * I + 8 * v;
        st_stream(o, pack8(dg));
        st_stream(o + I, pack8(du));
    }
}

static int grid_for(long long work_items, int threads, int sms) {
    long long want = (work_items + threads - 1) / threads;
    long long cap = (long long)sms * (2048 / threads) * 4;  // a few waves; kernels are grid-stride
    if (want < 1) want = 1;
    return (int)(want < cap ? want : cap);
}

}  // namespace acco

extern "C" int acco_rope_qkv(void* qkv, const float* cos_t, const float* sin_t, int T, int S, int n_rot, int n_total, int D,
                             int inverse, int sms, cudaStream_t st) {
    if (D % 16 != 0 || (32 % (D / 16)) != 0) return -1;
    const long long work = (long long)T * 32;   // one warp per token
    acco::rope_qkv_kernel<<<acco::grid_for(work, 256, sms), 256, 0, st>>>((__nv_bfloat16*)qkv, cos_t, sin_t, T, S, n_rot,
                                                                          n_total, D, inverse ? -1.f : 1.f);
    return 0;
}

extern "C" int acco_rope_pack_bwd(const void* dq, const void* dk, const void* dv, const long long* strides /* 9: (sb,ss,sh) x (q,k,v) */,
                                  void* dqkv, const float* cos_t, const float* sin_t, int B, int S, int Hq, int Hk, int D, int sms,
                                  cudaStream_t st) {
    if (D % 16 != 0 || (32 % (D / 16)) != 0) return -1;
    acco::PackSrc src;
    src.ptr[0] = (const __nv_bfloat16*)dq; src.ptr[1] = (const __nv_bfloat16*)dk; src.ptr[2] = (const __nv_bfloat16*)dv;
    for (int i = 0; i < 3; ++i) { src.sb[i] = strides[3 * i]; src.ss[i] = strides[3 * i + 1]; src.sh[i] = strides[3 * i + 2]; }
    const long long work = (long long)B * S * 32;   // one warp per token
    acco::rope_pack_bwd_kernel<<<acco::grid_for(work, 256, sms), 256, 0, st>>>(src, (__nv_bfloat16*)dqkv, cos_t, sin_t, B, S, Hq, Hk, D);
    return 0;
}

extern "C" int acco_swiglu_fwd(const void* gu, void* out, long long T, int I, int sms, cudaStream_t st) {
    if (I % 8 != 0) return -1;
    acco::swiglu_fwd_kernel<<<acco::grid_for(T * (I / 8), 256, sms), 256, 0, st>>>((const __nv_bfloat16*)gu,
                                                                                    (__nv_bfloat16*)out, T, I);
    return 0;
}

extern "C" int acco_swiglu_bwd(const void* dout, const void* gu, void* dgu, long long T, int I, int sms, cudaStream_t st) {
    if (I % 8 != 0) return -1;
    acco::swiglu_bwd_kernel<<<acco::grid_for(T * (I / 8), 256, sms), 256, 0, st>>>(
        (const __nv_bfloat16*)dout, (const __nv_bfloat16*)gu, (__nv_bfloat16*)dgu, T, I);
    return 0;
}

// ---- debug: an SM "occupier" with the resource footprint of the NVLS round kernel (256 threads x 64 registers, no dynamic smem),
// one CTA per SM, spinning for `ns` nanoseconds.  tools/coresidency_check.py launches it next to the wgmma GEMMs to see whether
// the two kinds of CTA share an SM (ACCO's overlap depends on it).
namespace acco {
__global__ void __launch_bounds__(256, 4) occupy_kernel(unsigned long long ns, float* sink) {
    float v[56];
#pragma unroll
    for (int i = 0; i < 56; ++i) v[i] = (float)(threadIdx.x + i);
    unsigned long long t0, t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
    do {
#pragma unroll
        for (int i = 0; i < 56; ++i) v[i] = v[i] * 1.0001f + v[(i + 7) % 56];      // keeps 56 values live -> 64 registers
        __nanosleep(200);
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    } while (t - t0 < ns);
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < 56; ++i) s += v[i];
    if (s == 123.456f) sink[0] = s;
}
}  // namespace acco

extern "C" int acco_debug_occupy(unsigned long long ns, int ctas, float* sink, cudaStream_t st) {
    // same SM shared-memory configuration as the GEMMs (max carve-out): an SM is only re-partitioned between L1 and shared memory
    // when it is idle, so kernels that prefer different carve-outs cannot share it (ACCO_OCCUPY_DEFAULT_CARVEOUT=1: leave the default)
    static bool once = false;
    if (!once) {
        const char* e = getenv("ACCO_OCCUPY_DEFAULT_CARVEOUT");
        if (!(e && e[0] == '1')) cudaFuncSetAttribute(acco::occupy_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
        once = true;
    }
    acco::occupy_kernel<<<ctas, 256, 0, st>>>(ns, sink);
    return (int)cudaGetLastError();
}
