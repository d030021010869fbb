// RMSNorm and LayerNorm (weight + bias), each with an optional fused residual add: forward and backward, bf16 I/O with
// fp32 statistics.  One kernel pair serves both norms; LAYER = false is RMSNorm, whose mean, bias and db disappear at
// compile time.
//
//   fwd :  h = a (+ r);  RMSNorm:   rstd = rsqrt(mean(h^2) + eps);                       y = h * rstd * w
//                        LayerNorm: mu = mean(h);  rstd = rsqrt(mean((h-mu)^2) + eps);   y = (h-mu) * rstd * w + b
//   bwd :  xh = (h-mu)*rstd (mu = 0 for RMSNorm);  g = dy*w;  c1 = mean(g*xh);  c2 = mean(g) (LayerNorm only)
//          dh = rstd*(g - c2 - xh*c1) (+ dh_extra)
//          dw = sum_rows dy*xh,  db = sum_rows dy  -> per-CTA fp32 partials [grid][NP*H] (NP = 1: dw; NP = 2: dw | db),
//          reduced by a second tiny kernel (deterministic, no atomics)
//
// One WARP per row for H <= 1024 (every 16-byte vector of the row in flight at once, no block barrier in the row loop);
// one CTA per row above that, up to H = 16384.  Both walk the rows grid-stride (persistent).
#include "common.cuh"
#include <type_traits>

namespace acco {

constexpr int kWarpsPerCta = 8;        // warp-per-row CTAs: 8 rows per CTA per iteration
constexpr int kMaxCtaThreads = 512;    // CTA-per-row CTAs: up to 512 threads, each holding VPT vectors of the row
constexpr int kMaxH = 16384;

// sum over the owners of one row: a warp (CTA_ROW = false) or the whole CTA (CTA_ROW = true)
template <bool CTA_ROW>
ACCO_DEVINL float row_sum(float v, float* red) {
    if constexpr (CTA_ROW) return block_sum(v, red);
    else return warp_sum(v);
}

template <int VPT, bool HAS_RES, bool CTA_ROW, bool LAYER>
__global__ void __launch_bounds__(CTA_ROW ? kMaxCtaThreads : kWarpsPerCta * 32) norm_fwd_kernel(
    const __nv_bfloat16* __restrict__ a, const __nv_bfloat16* __restrict__ r, const __nv_bfloat16* __restrict__ w,
    const __nv_bfloat16* __restrict__ b, __nv_bfloat16* __restrict__ y, __nv_bfloat16* __restrict__ h_out,
    float* __restrict__ mean_out, float* __restrict__ rstd_out, int T, int H, float eps) {
    __shared__ float red[32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int tid = CTA_ROW ? threadIdx.x : lane;               // index among the owners of a row
    const int stride = CTA_ROW ? blockDim.x : 32;
    const int nvec = H >> 3;
    const int row_step = CTA_ROW ? gridDim.x : gridDim.x * kWarpsPerCta;
    for (int row = CTA_ROW ? blockIdx.x : blockIdx.x * kWarpsPerCta + warp; row < T; row += row_step) {
        const size_t base = (size_t)row * H;
        bf16x8 av[VPT], rv[VPT];
#pragma unroll
        for (int i = 0; i < VPT; ++i) {            // issue every load of the row before touching any
            const int v = tid + stride * i;
            if (v < nvec) {
                av[i] = ld_stream(a + base + 8 * v);
                if (HAS_RES) rv[i] = ld_stream(r + base + 8 * v);
            }
        }
        float s = 0.f;                             // sum(h) for LayerNorm, sum(h^2) for RMSNorm
#pragma unroll
        for (int i = 0; i < VPT; ++i) {
            const int v = tid + stride * i;
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
                for (int j = 0; j < 8; ++j) s += LAYER ? fa[j] : fa[j] * fa[j];
            }
        }
        float mu = 0.f, rstd;
        if constexpr (LAYER) {
            mu = row_sum<CTA_ROW>(s, red) / (float)H;
            float ss = 0.f;
#pragma unroll
            for (int i = 0; i < VPT; ++i) {
                const int v = tid + stride * i;
                if (v < nvec) {
                    float fa[8];
                    unpack8(av[i], fa);
#pragma unroll
                    for (int j = 0; j < 8; ++j) ss += (fa[j] - mu) * (fa[j] - mu);
                }
            }
            rstd = rsqrtf(row_sum<CTA_ROW>(ss, red) / (float)H + eps);
        } else {
            rstd = rsqrtf(row_sum<CTA_ROW>(s, red) / (float)H + eps);
        }
        if (tid == 0) {
            if constexpr (LAYER) mean_out[row] = mu;
            rstd_out[row] = rstd;
        }
#pragma unroll
        for (int i = 0; i < VPT; ++i) {
            const int v = tid + stride * i;
            if (v < nvec) {
                float f[8], fw[8];
                unpack8(av[i], f);
                unpack8(ld_vec(w + 8 * v), fw);
                if constexpr (LAYER) {
                    float fb[8];
                    unpack8(ld_vec(b + 8 * v), fb);
#pragma unroll
                    for (int j = 0; j < 8; ++j) f[j] = (f[j] - mu) * rstd * fw[j] + fb[j];
                } else {
#pragma unroll
                    for (int j = 0; j < 8; ++j) f[j] = f[j] * rstd * fw[j];
                }
                st_stream(y + base + 8 * v, pack8(f));
            }
        }
    }
}

// partial layout: [grid][NP][H] (dw, then db for LayerNorm)
template <int VPT, bool HAS_EXTRA, bool CTA_ROW, bool LAYER>
__global__ void __launch_bounds__(CTA_ROW ? kMaxCtaThreads : kWarpsPerCta * 32) norm_bwd_kernel(
    const __nv_bfloat16* __restrict__ dy, const __nv_bfloat16* __restrict__ dh_extra, const __nv_bfloat16* __restrict__ h,
    const __nv_bfloat16* __restrict__ w, const float* __restrict__ mean_in, const float* __restrict__ rstd_in,
    __nv_bfloat16* __restrict__ dh, float* __restrict__ partial, int T, int H) {
    constexpr int NP = LAYER ? 2 : 1;
    extern __shared__ float dyn[];                 // warp rows: [kWarpsPerCta][256] staging for the CTA-level reduction
    __shared__ float red[32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int tid = CTA_ROW ? threadIdx.x : lane;
    const int stride = CTA_ROW ? blockDim.x : 32;
    const int nvec = H >> 3;
    const int row_step = CTA_ROW ? gridDim.x : gridDim.x * kWarpsPerCta;
    float acc[NP][VPT][8];                         // acc[0] = dw, acc[1] = db
#pragma unroll
    for (int p = 0; p < NP; ++p)
#pragma unroll
        for (int i = 0; i < VPT; ++i)
#pragma unroll
            for (int j = 0; j < 8; ++j) acc[p][i][j] = 0.f;
    for (int row = CTA_ROW ? blockIdx.x : blockIdx.x * kWarpsPerCta + warp; row < T; row += row_step) {
        const size_t base = (size_t)row * H;
        bf16x8 dyv[VPT], hv[VPT], ev[VPT];
#pragma unroll
        for (int i = 0; i < VPT; ++i) {
            const int v = tid + stride * i;
            if (v < nvec) {
                dyv[i] = ld_stream(dy + base + 8 * v);
                hv[i] = ld_stream(h + base + 8 * v);
                if (HAS_EXTRA && !CTA_ROW) ev[i] = ld_stream(dh_extra + base + 8 * v);
            }
        }
        const float mu = LAYER ? mean_in[row] : 0.f, rstd = rstd_in[row];
        float c1 = 0.f, c2 = 0.f;
#pragma unroll
        for (int i = 0; i < VPT; ++i) {
            const int v = tid + stride * i;
            if (v < nvec) {
                float fd[8], fh[8], fw[8];
                unpack8(dyv[i], fd);
                unpack8(hv[i], fh);
                unpack8(ld_vec(w + 8 * v), fw);
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const float xh = (LAYER ? fh[j] - mu : fh[j]) * rstd, g = fd[j] * fw[j];
                    c1 += g * xh;
                    acc[0][i][j] += fd[j] * xh;
                    if constexpr (LAYER) {
                        c2 += g;
                        acc[1][i][j] += fd[j];
                    }
                }
            }
        }
        c1 = row_sum<CTA_ROW>(c1, red) / (float)H;
        if constexpr (LAYER) c2 = row_sum<CTA_ROW>(c2, red) / (float)H;
#pragma unroll
        for (int i = 0; i < VPT; ++i) {
            const int v = tid + stride * i;
            if (v < nvec) {
                float fd[8], fh[8], fw[8], o[8];
                unpack8(dyv[i], fd);
                unpack8(hv[i], fh);
                unpack8(ld_vec(w + 8 * v), fw);
                if constexpr (LAYER) {
#pragma unroll
                    for (int j = 0; j < 8; ++j) o[j] = rstd * (fd[j] * fw[j] - c2 - (fh[j] - mu) * rstd * c1);
                } else {
#pragma unroll
                    for (int j = 0; j < 8; ++j) o[j] = rstd * (fd[j] * fw[j] - fh[j] * rstd * c1);
                }
                if (HAS_EXTRA) {
                    // a CTA row reads dh_extra only here: held from the start it would make the LayerNorm VPT = 4 kernel spill
                    float fe[8];
                    unpack8(CTA_ROW ? ld_stream(dh_extra + base + 8 * v) : ev[i], fe);
#pragma unroll
                    for (int j = 0; j < 8; ++j) o[j] += fe[j];
                }
                st_stream(dh + base + 8 * v, pack8(o));
            }
        }
    }
    float* my = partial + (size_t)blockIdx.x * NP * H;
    if constexpr (CTA_ROW) {
        // every thread owns distinct columns: write its sums directly
#pragma unroll
        for (int i = 0; i < VPT; ++i) {
            const int v = tid + stride * i;
            if (v < nvec) {
#pragma unroll
                for (int p = 0; p < NP; ++p)
#pragma unroll
                    for (int j = 0; j < 8; ++j) my[p * H + 8 * v + j] = acc[p][i][j];
            }
        }
    } else {
        // the warps of the CTA own the same columns of different rows: reduce over warps through smem
#pragma unroll
        for (int p = 0; p < NP; ++p) {
#pragma unroll
            for (int i = 0; i < VPT; ++i) {
                __syncthreads();
#pragma unroll
                for (int j = 0; j < 8; ++j) dyn[warp * 256 + lane * 8 + j] = acc[p][i][j];
                __syncthreads();
                const int col = threadIdx.x;               // 256 threads <-> the 256 columns of chunk i
                float s = 0.f;
#pragma unroll
                for (int k = 0; k < kWarpsPerCta; ++k) s += dyn[k * 256 + col];
                const int gcol = 256 * i + col;
                if (gcol < H) my[p * H + gcol] = s;
            }
        }
    }
}

// out[col] = sum_p partial[p][col]   (deterministic).  Block (32, 32): 32 columns x 32 partial-groups.
// If `accum` is given the sum is ADDED to the gradient there (fused AccumulateGrad; G = bf16: one rounding, G = float: an fp32
// gradient accumulator), else it is written to fp32 `out`.
template <typename G>
__global__ void __launch_bounds__(1024) reduce_partials_kernel(const float* __restrict__ partial, float* __restrict__ out,
                                                               G* __restrict__ accum, int nparts, int H, int pitch) {
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
        if (accum) {
            if constexpr (std::is_same<G, float>::value) accum[col] += s;
            else accum[col] = __float2bfloat16(__bfloat162float(accum[col]) + s);
        } else {
            out[col] = s;
        }
    }
}

// out[col] (fp32) = or accum[col] (bf16, or fp32 when accum_f32) += sum_p partial[p * pitch + col], col < width
static void reduce_partials(const float* partial, float* out, void* accum, int accum_f32, int nparts, int width, int pitch, cudaStream_t st) {
    if (accum_f32) reduce_partials_kernel<float><<<(width + 31) / 32, 1024, 0, st>>>(partial, out, (float*)accum, nparts, width, pitch);
    else reduce_partials_kernel<__nv_bfloat16><<<(width + 31) / 32, 1024, 0, st>>>(partial, out, (__nv_bfloat16*)accum, nparts, width, pitch);
}

// CTA-per-row geometry (H > 1024): the fewest 16-byte vectors per thread (a power of two) that keep the row within
// kMaxCtaThreads threads, and the thread count (a multiple of 32) that covers the row with them.
struct CtaGeom {
    int vpt, threads;
};
static CtaGeom cta_geom(int H) {
    const int nvec = H / 8;
    int vpt = 1;
    while ((nvec + vpt - 1) / vpt > kMaxCtaThreads) vpt *= 2;
    return {vpt, ((nvec + vpt - 1) / vpt + 31) / 32 * 32};
}

static bool supported(int H) { return H % 8 == 0 && H > 0 && H <= kMaxH; }

template <int VPT, bool CTA_ROW>
static void launch_fwd(const void* a, const void* r, const void* w, const void* b, void* y, void* h, float* mean, float* rstd, int T,
                       int H, float eps, int grid, cudaStream_t st) {
    const int threads = CTA_ROW ? cta_geom(H).threads : kWarpsPerCta * 32;
    auto A = (const __nv_bfloat16*)a;
    auto R = (const __nv_bfloat16*)r;
    auto W = (const __nv_bfloat16*)w;
    auto B = (const __nv_bfloat16*)b;
    auto Y = (__nv_bfloat16*)y;
    auto Ho = (__nv_bfloat16*)h;
    if (b) {
        if (r) norm_fwd_kernel<VPT, true, CTA_ROW, true><<<grid, threads, 0, st>>>(A, R, W, B, Y, Ho, mean, rstd, T, H, eps);
        else norm_fwd_kernel<VPT, false, CTA_ROW, true><<<grid, threads, 0, st>>>(A, R, W, B, Y, Ho, mean, rstd, T, H, eps);
    } else {
        if (r) norm_fwd_kernel<VPT, true, CTA_ROW, false><<<grid, threads, 0, st>>>(A, R, W, B, Y, Ho, mean, rstd, T, H, eps);
        else norm_fwd_kernel<VPT, false, CTA_ROW, false><<<grid, threads, 0, st>>>(A, R, W, B, Y, Ho, mean, rstd, T, H, eps);
    }
}

template <int VPT, bool CTA_ROW>
static void launch_bwd(const void* dy, const void* dh_extra, const void* h, const void* w, const float* mean, const float* rstd, void* dh,
                       float* partial, int T, int H, int grid, cudaStream_t st) {
    const int threads = CTA_ROW ? cta_geom(H).threads : kWarpsPerCta * 32;
    auto DY = (const __nv_bfloat16*)dy;
    auto DE = (const __nv_bfloat16*)dh_extra;
    auto Hh = (const __nv_bfloat16*)h;
    auto W = (const __nv_bfloat16*)w;
    auto DH = (__nv_bfloat16*)dh;
    const size_t smem = CTA_ROW ? 0 : (size_t)kWarpsPerCta * 256 * sizeof(float);
    if (mean) {
        if (dh_extra) norm_bwd_kernel<VPT, true, CTA_ROW, true><<<grid, threads, smem, st>>>(DY, DE, Hh, W, mean, rstd, DH, partial, T, H);
        else norm_bwd_kernel<VPT, false, CTA_ROW, true><<<grid, threads, smem, st>>>(DY, DE, Hh, W, mean, rstd, DH, partial, T, H);
    } else {
        if (dh_extra) norm_bwd_kernel<VPT, true, CTA_ROW, false><<<grid, threads, smem, st>>>(DY, DE, Hh, W, mean, rstd, DH, partial, T, H);
        else norm_bwd_kernel<VPT, false, CTA_ROW, false><<<grid, threads, smem, st>>>(DY, DE, Hh, W, mean, rstd, DH, partial, T, H);
    }
}

}  // namespace acco

// Runs `launch<VPT, CTA_ROW>(...)` for width H: one warp per row with VPT = ceil(H / 256) for H <= 1024, else one CTA
// per row with cta_geom(H).vpt.
#define ACCO_NORM_DISPATCH(H, launch, ...)                                                           \
    do {                                                                                             \
        if ((H) <= 1024) {                                                                           \
            const int _v = ((H) / 8 + 31) / 32;                                                      \
            if (_v <= 1) launch<1, false>(__VA_ARGS__);                                              \
            else if (_v == 2) launch<2, false>(__VA_ARGS__);                                         \
            else if (_v == 3) launch<3, false>(__VA_ARGS__);                                         \
            else launch<4, false>(__VA_ARGS__);                                                      \
        } else {                                                                                     \
            const int _v = acco::cta_geom(H).vpt;                                                    \
            if (_v == 1) launch<1, true>(__VA_ARGS__);                                               \
            else if (_v == 2) launch<2, true>(__VA_ARGS__);                                          \
            else launch<4, true>(__VA_ARGS__);                                                       \
        }                                                                                            \
    } while (0)

// Number of CTAs to launch for T rows of width H on a device with `sms` SMs (also the number of dw / db partials the
// backward needs room for).
extern "C" int acco_norm_grid(int T, int H, int sms, int backward) {
    int want, per_sm;
    if (H <= 1024) {   // warp-per-row: 8 rows per CTA per iteration
        want = (T + acco::kWarpsPerCta - 1) / acco::kWarpsPerCta;
        per_sm = backward ? 2 : 8;
    } else {           // CTA-per-row.  forward: fill the machine; backward: every CTA emits one partial, so stay at 4 CTAs per SM
        want = T;
        per_sm = 2048 / acco::cta_geom(H).threads;
        if (backward && per_sm > 4) per_sm = 4;
    }
    const int cap = sms * per_sm;
    if (want < 1) want = 1;
    return want < cap ? want : cap;
}

// RMSNorm when b == nullptr (mean is then not written), LayerNorm otherwise.  r == nullptr: no residual (h is not
// written).  Returns cudaSuccess, or -1 if H is not supported.
extern "C" int acco_norm_fwd(const void* a, const void* r, const void* w, const void* b, void* y, void* h, float* mean, float* rstd, int T,
                             int H, float eps, int grid, cudaStream_t st) {
    if (!acco::supported(H)) return -1;
    ACCO_NORM_DISPATCH(H, acco::launch_fwd, a, r, w, b, y, h, mean, rstd, T, H, eps, grid, st);
    return (int)cudaGetLastError();
}

static int norm_bwd(const void* dy, const void* dh_extra, const void* h, const void* w, const float* mean, const float* rstd, void* dh,
                    float* partial, float* dwdb_out, void* dw_accum, void* db_accum, int accum_f32, int T, int H, int grid, cudaStream_t st) {
    if (!acco::supported(H)) return -1;
    ACCO_NORM_DISPATCH(H, acco::launch_bwd, dy, dh_extra, h, w, mean, rstd, dh, partial, T, H, grid, st);
    const int width = (mean ? 2 : 1) * H;
    // one reduction over the whole partial row when it lands in fp32, one per parameter when accumulated into the arena
    if (dw_accum) {
        acco::reduce_partials(partial, nullptr, dw_accum, accum_f32, grid, H, width, st);
        if (mean) acco::reduce_partials(partial + H, nullptr, db_accum, accum_f32, grid, H, width, st);
    } else {
        acco::reduce_partials(partial, dwdb_out, nullptr, 0, grid, width, width, st);
    }
    return (int)cudaGetLastError();
}

// RMSNorm when mean == nullptr, LayerNorm otherwise.  partial: grid * NP * H floats.  dw (| db) are written to fp32
// `dwdb_out` [NP * H], or, when `dw_accum` is given (and `db_accum` for LayerNorm), added in place to those bf16 gradients.
extern "C" int acco_norm_bwd(const void* dy, const void* dh_extra, const void* h, const void* w, const float* mean, const float* rstd,
                             void* dh, float* partial, float* dwdb_out, void* dw_accum, void* db_accum, int T, int H, int grid,
                             cudaStream_t st) {
    return norm_bwd(dy, dh_extra, h, w, mean, rstd, dh, partial, dwdb_out, dw_accum, db_accum, 0, T, H, grid, st);
}

// As acco_norm_bwd with the sums added to fp32 gradients dw_accum [H] (and db_accum [H] for LayerNorm), both required.
extern "C" int acco_norm_bwd_acc_f32(const void* dy, const void* dh_extra, const void* h, const void* w, const float* mean, const float* rstd,
                                     void* dh, float* partial, float* dw_accum, float* db_accum, int T, int H, int grid, cudaStream_t st) {
    if (!dw_accum || (mean && !db_accum)) return -1;
    return norm_bwd(dy, dh_extra, h, w, mean, rstd, dh, partial, nullptr, dw_accum, db_accum, 1, T, H, grid, st);
}
