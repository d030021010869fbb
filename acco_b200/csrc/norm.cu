// RMSNorm / fused residual-add + RMSNorm, forward and backward, bf16 I/O with fp32 statistics.
//
// Replaces HF Llama's ~7 eager kernels per norm (modeling_llama.py:53-70).
// Layout: x [T, H] row-major bf16.  A row is owned by `tpr` consecutive threads (a multiple of
// 32), each holding VPT 16-byte vectors of the row in registers as packed bf16, so every element
// is read from HBM exactly once per pass; a CTA of 256..512 threads processes several rows at a
// time and walks the rows grid-stride (persistent).
//   fwd :  h = a (+ r);  rstd = rsqrt(mean(h^2) + eps);  y = h * rstd * w
//   bwd :  xh = h*rstd;  wdy = dy*w;  c = mean(wdy * xh);  dh = rstd*(wdy - xh*c) (+ dh_extra)
//          dw = sum_rows dy * xh  -> per-CTA fp32 partials, reduced by a second tiny kernel
//          (deterministic, no atomics)
#include "common.cuh"

namespace acco {

// sum `v` over the `tpr` threads that own one row.  `red` has one float per warp of the CTA.
ACCO_DEVINL float row_sum(float v, float* red, int tpr) {
    v = warp_sum(v);
    if (tpr == 32) return v;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    __syncthreads();
    if (lane == 0) red[warp] = v;
    __syncthreads();
    const int wpr = tpr >> 5;
    const int w0 = (warp / wpr) * wpr;
    float s = 0.f;
    for (int k = 0; k < wpr; ++k) s += red[w0 + k];
    return s;
}

template <int VPT, bool HAS_RES>
__global__ void __launch_bounds__(512) rmsnorm_fwd_kernel(
    const __nv_bfloat16* __restrict__ a, const __nv_bfloat16* __restrict__ r, const __nv_bfloat16* __restrict__ w,
    __nv_bfloat16* __restrict__ y, __nv_bfloat16* __restrict__ h_out, float* __restrict__ rstd_out, int T, int H,
    float eps, int tpr) {
    __shared__ float red[32];
    const int rpc = blockDim.x / tpr;           // rows per CTA iteration
    const int lrow = threadIdx.x / tpr, t = threadIdx.x % tpr;
    const int nvec = H >> 3;
    bf16x8 wv[VPT];
#pragma unroll
    for (int i = 0; i < VPT; ++i) {
        const int v = t + tpr * i;
        if (v < nvec) wv[i] = ld_vec(w + 8 * v);
    }
    for (int row0 = blockIdx.x * rpc; row0 < T; row0 += gridDim.x * rpc) {
        const int row = row0 + lrow;
        const bool rv_ok = row < T;
        const size_t base = (size_t)row * H;
        bf16x8 hv[VPT];
        float ss = 0.f;
#pragma unroll
        for (int i = 0; i < VPT; ++i) {
            const int v = t + tpr * i;
            if (rv_ok && v < nvec) {
                bf16x8 av = ld_stream(a + base + 8 * v);
                if (HAS_RES) {
                    bf16x8 rv = ld_stream(r + base + 8 * v);
                    float fa[8], fr[8];
                    unpack8(av, fa);
                    unpack8(rv, fr);
#pragma unroll
                    for (int j = 0; j < 8; ++j) fa[j] += fr[j];
                    av = pack8(fa);  // h is *stored* in bf16: normalise exactly what is stored
                    st_vec(h_out + base + 8 * v, av);
                }
                hv[i] = av;
                float f[8];
                unpack8(av, f);
#pragma unroll
                for (int j = 0; j < 8; ++j) ss += f[j] * f[j];
            }
        }
        ss = row_sum(ss, red, tpr);
        const float rstd = rsqrtf(ss / (float)H + eps);
        if (rv_ok && t == 0) rstd_out[row] = rstd;
#pragma unroll
        for (int i = 0; i < VPT; ++i) {
            const int v = t + tpr * i;
            if (rv_ok && v < nvec) {
                float f[8], fw[8];
                unpack8(hv[i], f);
                unpack8(wv[i], fw);
#pragma unroll
                for (int j = 0; j < 8; ++j) f[j] = f[j] * rstd * fw[j];
                st_stream(y + base + 8 * v, pack8(f));
            }
        }
    }
}

template <int VPT, bool HAS_EXTRA>
__global__ void __launch_bounds__(512) rmsnorm_bwd_kernel(
    const __nv_bfloat16* __restrict__ dy, const __nv_bfloat16* __restrict__ dh_extra,
    const __nv_bfloat16* __restrict__ h, const __nv_bfloat16* __restrict__ w, const float* __restrict__ rstd_in,
    __nv_bfloat16* __restrict__ dh, float* __restrict__ dw_partial, int T, int H, int tpr) {
    extern __shared__ float dyn[];              // [blockDim.x * 8] staging for the CTA-level dw reduction
    __shared__ float red[32];
    const int rpc = blockDim.x / tpr;
    const int lrow = threadIdx.x / tpr, t = threadIdx.x % tpr;
    const int nvec = H >> 3;
    bf16x8 wv[VPT];
    float dw[VPT][8];
#pragma unroll
    for (int i = 0; i < VPT; ++i) {
        const int v = t + tpr * i;
        if (v < nvec) wv[i] = ld_vec(w + 8 * v);
#pragma unroll
        for (int j = 0; j < 8; ++j) dw[i][j] = 0.f;
    }
    for (int row0 = blockIdx.x * rpc; row0 < T; row0 += gridDim.x * rpc) {
        const int row = row0 + lrow;
        const bool rv_ok = row < T;
        const size_t base = (size_t)row * H;
        const float rstd = rv_ok ? rstd_in[row] : 0.f;
        bf16x8 dyv[VPT], hv[VPT];
        float c = 0.f;
#pragma unroll
        for (int i = 0; i < VPT; ++i) {
            const int v = t + tpr * i;
            if (rv_ok && v < nvec) {
                dyv[i] = ld_stream(dy + base + 8 * v);
                hv[i] = ld_stream(h + base + 8 * v);
                float fd[8], fh[8], fw[8];
                unpack8(dyv[i], fd);
                unpack8(hv[i], fh);
                unpack8(wv[i], fw);
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const float xh = fh[j] * rstd;
                    c += fd[j] * fw[j] * xh;
                    dw[i][j] += fd[j] * xh;
                }
            }
        }
        c = row_sum(c, red, tpr) / (float)H;
#pragma unroll
        for (int i = 0; i < VPT; ++i) {
            const int v = t + tpr * i;
            if (rv_ok && v < nvec) {
                float fd[8], fh[8], fw[8], o[8];
                unpack8(dyv[i], fd);
                unpack8(hv[i], fh);
                unpack8(wv[i], fw);
                if (HAS_EXTRA) {
                    float fe[8];
                    unpack8(ld_stream(dh_extra + base + 8 * v), fe);
#pragma unroll
                    for (int j = 0; j < 8; ++j) o[j] = fe[j] + rstd * (fd[j] * fw[j] - fh[j] * rstd * c);
                } else {
#pragma unroll
                    for (int j = 0; j < 8; ++j) o[j] = rstd * (fd[j] * fw[j] - fh[j] * rstd * c);
                }
                st_stream(dh + base + 8 * v, pack8(o));
            }
        }
    }
    // reduce dw over the rpc row-groups of the CTA, then emit this CTA's partial
#pragma unroll
    for (int i = 0; i < VPT; ++i) {
        __syncthreads();
#pragma unroll
        for (int j = 0; j < 8; ++j) dyn[(lrow * tpr + t) * 8 + j] = dw[i][j];
        __syncthreads();
        if (lrow == 0) {
            const int v = t + tpr * i;
            if (v < nvec) {
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    float s = 0.f;
                    for (int k = 0; k < rpc; ++k) s += dyn[(k * tpr + t) * 8 + j];
                    dw_partial[(size_t)blockIdx.x * H + 8 * v + j] = s;
                }
            }
        }
    }
}

// out[col] = sum_p partial[p][col]   (deterministic).  Block (32, 32): 32 columns x 32 partial-groups.
// If `accum` is given the sum is ADDED to the bf16 gradient there (fused AccumulateGrad), else it
// is written to fp32 `out`.
__global__ void __launch_bounds__(1024) reduce_partials_kernel(const float* __restrict__ partial, float* __restrict__ out,
                                                               __nv_bfloat16* __restrict__ accum, int nparts, int H, int pitch) {
    __shared__ float sm[32][33];
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    const int col = blockIdx.x * 32 + tx;
    float s0 = 0.f, s1 = 0.f;
    if (col < H) {
        int p = ty;
        for (; p + 32 < nparts; p += 64) {
            s0 += partial[(size_t)p * pitch + col];
            s1 += partial[(size_t)(p + 32) * pitch + col];
        }
        if (p < nparts) s0 += partial[(size_t)p * pitch + col];
    }
    sm[ty][tx] = s0 + s1;
    __syncthreads();
    if (ty == 0 && col < H) {
        float s = 0.f;
#pragma unroll
        for (int k = 0; k < 32; ++k) s += sm[k][tx];
        if (accum) accum[col] = __float2bfloat16(__bfloat162float(accum[col]) + s);
        else out[col] = s;
    }
}

// ------------------------------------------------------------------------------------------------------------
// Warp-per-row variants for H <= 1024 (VPT <= 4 vectors per lane): no __syncthreads in the row loop, the whole row
// of every tensor is in flight per warp (Little's law: ~35 KB/SM must be outstanding to saturate HBM3e).
// ------------------------------------------------------------------------------------------------------------
constexpr int kWarpsPerCta = 8;

template <int VPT, bool HAS_RES>
__global__ void __launch_bounds__(kWarpsPerCta * 32) rmsnorm_fwd_warp_kernel(
    const __nv_bfloat16* __restrict__ a, const __nv_bfloat16* __restrict__ r, const __nv_bfloat16* __restrict__ w,
    __nv_bfloat16* __restrict__ y, __nv_bfloat16* __restrict__ h_out, float* __restrict__ rstd_out, int T, int H, float eps) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int nvec = H >> 3;
    bf16x8 wv[VPT];
#pragma unroll
    for (int i = 0; i < VPT; ++i) {
        const int v = lane + 32 * i;
        if (v < nvec) wv[i] = ld_vec(w + 8 * v);
    }
    for (int row = blockIdx.x * kWarpsPerCta + warp; row < T; row += gridDim.x * kWarpsPerCta) {
        const size_t base = (size_t)row * H;
        bf16x8 av[VPT], rv[VPT];
#pragma unroll
        for (int i = 0; i < VPT; ++i) {            // issue every load of the row before touching any
            const int v = lane + 32 * i;
            if (v < nvec) {
                av[i] = ld_stream(a + base + 8 * v);
                if (HAS_RES) rv[i] = ld_stream(r + base + 8 * v);
            }
        }
        float ss = 0.f;
#pragma unroll
        for (int i = 0; i < VPT; ++i) {
            const int v = lane + 32 * i;
            if (v < nvec) {
                float fa[8];
                unpack8(av[i], fa);
                if (HAS_RES) {
                    float fr[8];
                    unpack8(rv[i], fr);
#pragma unroll
                    for (int j = 0; j < 8; ++j) fa[j] += fr[j];
                    av[i] = pack8(fa);
                    st_vec(h_out + base + 8 * v, av[i]);
                    unpack8(av[i], fa);            // normalise exactly what was stored (bf16)
                }
#pragma unroll
                for (int j = 0; j < 8; ++j) ss += fa[j] * fa[j];
            }
        }
        ss = warp_sum(ss);
        const float rstd = rsqrtf(ss / (float)H + eps);
        if (lane == 0) rstd_out[row] = rstd;
#pragma unroll
        for (int i = 0; i < VPT; ++i) {
            const int v = lane + 32 * i;
            if (v < nvec) {
                float f[8], fw[8];
                unpack8(av[i], f);
                unpack8(wv[i], fw);
#pragma unroll
                for (int j = 0; j < 8; ++j) f[j] = f[j] * rstd * fw[j];
                st_stream(y + base + 8 * v, pack8(f));
            }
        }
    }
}

template <int VPT, bool HAS_EXTRA>
__global__ void __launch_bounds__(kWarpsPerCta * 32) rmsnorm_bwd_warp_kernel(
    const __nv_bfloat16* __restrict__ dy, const __nv_bfloat16* __restrict__ dh_extra, const __nv_bfloat16* __restrict__ h,
    const __nv_bfloat16* __restrict__ w, const float* __restrict__ rstd_in, __nv_bfloat16* __restrict__ dh,
    float* __restrict__ dw_partial, int T, int H) {
    extern __shared__ float dyn[];                 // [kWarpsPerCta][32*8] staging for the CTA-level dw reduction
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int nvec = H >> 3;
    bf16x8 wv[VPT];
    float dw[VPT][8];
#pragma unroll
    for (int i = 0; i < VPT; ++i) {
        const int v = lane + 32 * i;
        if (v < nvec) wv[i] = ld_vec(w + 8 * v);
#pragma unroll
        for (int j = 0; j < 8; ++j) dw[i][j] = 0.f;
    }
    for (int row = blockIdx.x * kWarpsPerCta + warp; row < T; row += gridDim.x * kWarpsPerCta) {
        const size_t base = (size_t)row * H;
        bf16x8 dyv[VPT], hv[VPT], ev[VPT];
#pragma unroll
        for (int i = 0; i < VPT; ++i) {
            const int v = lane + 32 * i;
            if (v < nvec) {
                dyv[i] = ld_stream(dy + base + 8 * v);
                hv[i] = ld_stream(h + base + 8 * v);
                if (HAS_EXTRA) ev[i] = ld_stream(dh_extra + base + 8 * v);
            }
        }
        const float rstd = rstd_in[row];
        float c = 0.f;
#pragma unroll
        for (int i = 0; i < VPT; ++i) {
            const int v = lane + 32 * i;
            if (v < nvec) {
                float fd[8], fh[8], fw[8];
                unpack8(dyv[i], fd);
                unpack8(hv[i], fh);
                unpack8(wv[i], fw);
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const float xh = fh[j] * rstd;
                    c += fd[j] * fw[j] * xh;
                    dw[i][j] += fd[j] * xh;
                }
            }
        }
        c = warp_sum(c) / (float)H;
#pragma unroll
        for (int i = 0; i < VPT; ++i) {
            const int v = lane + 32 * i;
            if (v < nvec) {
                float fd[8], fh[8], fw[8], o[8];
                unpack8(dyv[i], fd);
                unpack8(hv[i], fh);
                unpack8(wv[i], fw);
#pragma unroll
                for (int j = 0; j < 8; ++j) o[j] = rstd * (fd[j] * fw[j] - fh[j] * rstd * c);
                if (HAS_EXTRA) {
                    float fe[8];
                    unpack8(ev[i], fe);
#pragma unroll
                    for (int j = 0; j < 8; ++j) o[j] += fe[j];
                }
                st_stream(dh + base + 8 * v, pack8(o));
            }
        }
    }
#pragma unroll
    for (int i = 0; i < VPT; ++i) {
        __syncthreads();
#pragma unroll
        for (int j = 0; j < 8; ++j) dyn[warp * 256 + lane * 8 + j] = dw[i][j];
        __syncthreads();
        const int col = threadIdx.x;               // 256 threads <-> the 256 columns of chunk i
        float s = 0.f;
#pragma unroll
        for (int k = 0; k < kWarpsPerCta; ++k) s += dyn[k * 256 + col];
        const int gcol = 256 * i + col;
        if (gcol < H) dw_partial[(size_t)blockIdx.x * H + gcol] = s;
    }
}

struct NormGeom {
    int vpt, tpr, threads;
};

static NormGeom geom(int H) {
    const int nvec = H / 8;
    int vpt = 1;
    while ((nvec + vpt - 1) / vpt > 512) vpt *= 2;
    int tpr = (((nvec + vpt - 1) / vpt) + 31) / 32 * 32;
    int rows = tpr >= 256 ? 1 : 256 / tpr;
    return {vpt, tpr, tpr * rows};
}

}  // namespace acco

#define ACCO_DISPATCH_WVPT(H, ...)                                    \
    do {                                                              \
        const int _v = ((H) / 8 + 31) / 32;                           \
        if (_v <= 1) { constexpr int VPT = 1; __VA_ARGS__; }          \
        else if (_v <= 2) { constexpr int VPT = 2; __VA_ARGS__; }     \
        else if (_v <= 3) { constexpr int VPT = 3; __VA_ARGS__; }     \
        else if (_v <= 4) { constexpr int VPT = 4; __VA_ARGS__; }     \
        else { constexpr int VPT = 8; __VA_ARGS__; }                  \
    } while (0)

#define ACCO_DISPATCH_VPT(vpt, ...)                                  \
    do {                                                             \
        if ((vpt) == 1) { constexpr int VPT = 1; __VA_ARGS__; }      \
        else if ((vpt) == 2) { constexpr int VPT = 2; __VA_ARGS__; } \
        else if ((vpt) == 4) { constexpr int VPT = 4; __VA_ARGS__; } \
        else return -1;                                              \
    } while (0)

// Number of CTAs to launch for T rows of width H on a device with `sms` SMs (also the number of
// dw partials the backward needs room for).
extern "C" int acco_norm_grid(int T, int H, int sms, int backward) {
    if (H <= 1024) {   // warp-per-row kernels: 8 rows per CTA per iteration
        int want = (T + acco::kWarpsPerCta - 1) / acco::kWarpsPerCta;
        int cap = sms * (backward ? 2 : 8);
        if (want < 1) want = 1;
        return want < cap ? want : cap;
    }
    acco::NormGeom g = acco::geom(H);
    const int rpc = g.threads / g.tpr;
    int want = (T + rpc - 1) / rpc;
    // forward: fill the machine; backward: every CTA emits one dw partial, so stay at ~4 CTAs per SM
    int per_sm = 2048 / g.threads;
    if (backward && per_sm > 4) per_sm = 4;
    int cap = sms * per_sm;
    if (want < 1) want = 1;
    return want < cap ? want : cap;
}

// r == nullptr: plain rmsnorm (h is not written).  Returns 0 on success, -1 if H is unsupported.
extern "C" int acco_rmsnorm_fwd(const void* a, const void* r, const void* w, void* y, void* h, float* rstd, int T, int H,
                                float eps, int grid, cudaStream_t st) {
    using namespace acco;
    if (H % 8 != 0 || H > 8 * 512 * 4) return -1;
    NormGeom g = geom(H);
    auto A = (const __nv_bfloat16*)a;
    auto R = (const __nv_bfloat16*)r;
    auto W = (const __nv_bfloat16*)w;
    auto Y = (__nv_bfloat16*)y;
    auto Ho = (__nv_bfloat16*)h;
    if (H <= 1024) {
        ACCO_DISPATCH_WVPT(H, {
            if (r) rmsnorm_fwd_warp_kernel<VPT, true><<<grid, kWarpsPerCta * 32, 0, st>>>(A, R, W, Y, Ho, rstd, T, H, eps);
            else rmsnorm_fwd_warp_kernel<VPT, false><<<grid, kWarpsPerCta * 32, 0, st>>>(A, R, W, Y, nullptr, rstd, T, H, eps);
        });
        return 0;
    }
    ACCO_DISPATCH_VPT(g.vpt, {
        if (r) rmsnorm_fwd_kernel<VPT, true><<<grid, g.threads, 0, st>>>(A, R, W, Y, Ho, rstd, T, H, eps, g.tpr);
        else rmsnorm_fwd_kernel<VPT, false><<<grid, g.threads, 0, st>>>(A, R, W, Y, nullptr, rstd, T, H, eps, g.tpr);
    });
    return 0;
}

// dw_partial must hold grid*H floats; dw_out H floats (ignored when dw_accum_bf16 != nullptr: the
// reduced dw is then added to that bf16 gradient in place).
extern "C" int acco_rmsnorm_bwd(const void* dy, const void* dh_extra, const void* h, const void* w, const float* rstd,
                                void* dh, float* dw_partial, float* dw_out, void* dw_accum_bf16, int T, int H, int grid,
                                cudaStream_t st) {
    using namespace acco;
    if (H % 8 != 0 || H > 8 * 512 * 4) return -1;
    NormGeom g = geom(H);
    auto DY = (const __nv_bfloat16*)dy;
    auto DE = (const __nv_bfloat16*)dh_extra;
    auto Hh = (const __nv_bfloat16*)h;
    auto W = (const __nv_bfloat16*)w;
    auto DH = (__nv_bfloat16*)dh;
    if (H <= 1024) {
        const size_t wsmem = (size_t)kWarpsPerCta * 256 * sizeof(float);
        ACCO_DISPATCH_WVPT(H, {
            if (dh_extra) rmsnorm_bwd_warp_kernel<VPT, true><<<grid, kWarpsPerCta * 32, wsmem, st>>>(DY, DE, Hh, W, rstd, DH, dw_partial, T, H);
            else rmsnorm_bwd_warp_kernel<VPT, false><<<grid, kWarpsPerCta * 32, wsmem, st>>>(DY, DE, Hh, W, rstd, DH, dw_partial, T, H);
        });
        reduce_partials_kernel<<<(H + 31) / 32, 1024, 0, st>>>(dw_partial, dw_out, (__nv_bfloat16*)dw_accum_bf16, grid, H, H);
        return 0;
    }
    const size_t smem = (size_t)g.threads * 8 * sizeof(float);
    ACCO_DISPATCH_VPT(g.vpt, {
        if (dh_extra) rmsnorm_bwd_kernel<VPT, true><<<grid, g.threads, smem, st>>>(DY, DE, Hh, W, rstd, DH, dw_partial, T, H, g.tpr);
        else rmsnorm_bwd_kernel<VPT, false><<<grid, g.threads, smem, st>>>(DY, DE, Hh, W, rstd, DH, dw_partial, T, H, g.tpr);
    });
    reduce_partials_kernel<<<(H + 31) / 32, 1024, 0, st>>>(dw_partial, dw_out, (__nv_bfloat16*)dw_accum_bf16, grid, H, H);
    return 0;
}

// out[col] (fp32) = or accum[col] (bf16) += sum_p partial[p * pitch + col], col < width  (shared with layernorm.cu)
extern "C" int acco_reduce_partials(const float* partial, float* out, void* accum_bf16, int nparts, int width, int pitch, cudaStream_t st) {
    acco::reduce_partials_kernel<<<(width + 31) / 32, 1024, 0, st>>>(partial, out, (__nv_bfloat16*)accum_bf16, nparts, width, pitch);
    return (int)cudaGetLastError();
}
