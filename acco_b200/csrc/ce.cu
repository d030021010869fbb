// Softmax cross-entropy over bf16 logits [T, Vp] with `V <= Vp` valid columns (the rest is LM-head
// alignment padding), HF semantics: rows whose label == ignore_index contribute nothing, loss is
// the mean over the remaining rows (loss_utils.py:45-67).  No fp32 copy of the logits is ever made
// (the reference up-casts all 8x1024x50257 logits to fp32 = 1.5 GiB).
//
//   ce_fwd : one CTA per row, ONE streaming pass (online max/sum in fp32) -> lse[row], row_loss[row]
//   ce_reduce : deterministic tree over rows -> loss (mean) and inv_n = 1 / #valid rows
//   ce_bwd : in place  logits <- (softmax - onehot) * scale   (scale = dloss * inv_n, device scalar);
//            ignored rows and padded columns are written as 0.
//
// Label smoothing (kSmooth, eps > 0; HF LabelSmoother / F.cross_entropy(label_smoothing=eps) over the V valid columns):
//   row_loss = lse - (1 - eps) x[label] - (eps / V) sum_{c<V} x_c,   d = (softmax - (1 - eps) onehot - eps / V) * scale.
// The forward adds the row sum of x to the same streaming pass and one more block reduction; `one_m_eps` = 1 - eps and
// `eps_v` = eps / V are fp32 values computed on the host.  eps = 0 launches the kSmooth = false instantiations, which ignore
// both arguments and compile to the same code as before smoothing existed.
//
// Z-loss (kZ, z > 0; PaLM's auxiliary term, keeps the softmax normaliser near 0):
//   row_loss += z lse^2,   d = (softmax (1 + 2 z lse) - (1 - eps) onehot - eps / V) * scale.
// The forward adds the term at the row end from the lse it already has; ce_reduce also writes the mean z-term over the
// non-ignored rows to `z_out`; the backward forms 1 + 2 z lse once per row.  z = 0 launches the kZ = false instantiations,
// which ignore `z` and `z_out` and compile to the same code as before the z-loss existed.
#include "common.cuh"

namespace acco {

constexpr int kCEThreads = 512;

template <bool kSmooth, bool kZ>
__global__ void __launch_bounds__(kCEThreads) ce_fwd_kernel(const __nv_bfloat16* __restrict__ logits,
                                                            const long long* __restrict__ labels, float* __restrict__ lse_out,
                                                            float* __restrict__ row_loss, int V, int Vp, long long ignore_index,
                                                            float one_m_eps, float eps_v, float z) {
    __shared__ float red[32];
    const long long row = blockIdx.x;
    const __nv_bfloat16* x = logits + row * (size_t)Vp;
    const long long label = labels[row];
    if (label == ignore_index) {           // uniform per CTA: skip the row entirely
        if (threadIdx.x == 0) {
            lse_out[row] = 0.f;
            row_loss[row] = 0.f;
        }
        return;
    }
    const int nvec_full = V >> 3;          // vectors entirely inside the valid range
    float m = -INFINITY, s = 0.f;
    float sx = 0.f;                        // kSmooth: running sum of the valid logits
    for (int v = threadIdx.x; v < nvec_full; v += kCEThreads) {
        float f[8];
        unpack8(ld_stream(x + 8 * v), f);
        float lm = f[0];
#pragma unroll
        for (int j = 1; j < 8; ++j) lm = fmaxf(lm, f[j]);
        const float nm = fmaxf(m, lm);
        float acc = 0.f;
#pragma unroll
        for (int j = 0; j < 8; ++j) acc += __expf(f[j] - nm);
        s = s * __expf(m - nm) + acc;
        m = nm;
        if constexpr (kSmooth) {
            float ax = f[0];
#pragma unroll
            for (int j = 1; j < 8; ++j) ax += f[j];
            sx += ax;
        }
    }
    // ragged tail (V not a multiple of 8): scalar, handled by the first few threads
    for (int c = (nvec_full << 3) + threadIdx.x; c < V; c += kCEThreads) {
        const float f = __bfloat162float(x[c]);
        const float nm = fmaxf(m, f);
        s = s * __expf(m - nm) + __expf(f - nm);
        m = nm;
        if constexpr (kSmooth) sx += f;
    }
    const float gm = block_max(m, red);
    const float part = (m == -INFINITY) ? 0.f : s * __expf(m - gm);
    const float gs = block_sum(part, red);
    if constexpr (kSmooth) {
        const float gsx = block_sum(sx, red);
        if (threadIdx.x == 0) {
            const float lse = gm + __logf(gs);
            lse_out[row] = lse;
            const float ce = lse - one_m_eps * __bfloat162float(x[label]) - eps_v * gsx;
            if constexpr (kZ) row_loss[row] = ce + z * lse * lse;
            else row_loss[row] = ce;
        }
    } else {
        if (threadIdx.x == 0) {
            const float lse = gm + __logf(gs);
            lse_out[row] = lse;
            const float ce = lse - __bfloat162float(x[label]);
            if constexpr (kZ) row_loss[row] = ce + z * lse * lse;
            else row_loss[row] = ce;
        }
    }
}

// kZ: also `*z_out` = mean over the non-ignored rows of z lse^2, summed in the same order as the row losses.
template <bool kZ>
__global__ void __launch_bounds__(1024) ce_reduce_kernel(const float* __restrict__ row_loss, const long long* __restrict__ labels,
                                                         float* __restrict__ loss, float* __restrict__ inv_n, long long T,
                                                         long long ignore_index, const float* __restrict__ lse, float* __restrict__ z_out,
                                                         float z) {
    __shared__ float red[32];
    float s = 0.f, n = 0.f, sz = 0.f;
    for (long long i = threadIdx.x; i < T; i += blockDim.x) {
        if (labels[i] != ignore_index) {
            s += row_loss[i];
            n += 1.f;
            if constexpr (kZ) {
                const float l = lse[i];
                sz += z * l * l;
            }
        }
    }
    s = block_sum(s, red);
    n = block_sum(n, red);
    if constexpr (kZ) sz = block_sum(sz, red);
    if (threadIdx.x == 0) {
        const float inv = n > 0.f ? 1.f / n : 0.f;
        *loss = s * inv;
        *inv_n = inv;
        if constexpr (kZ) *z_out = sz * inv;
    }
}

template <bool kSmooth, bool kZ>
__global__ void __launch_bounds__(kCEThreads) ce_bwd_kernel(__nv_bfloat16* __restrict__ logits, const long long* __restrict__ labels,
                                                            const float* __restrict__ lse_in, const float* __restrict__ scale_ptr,
                                                            int V, int Vp, long long ignore_index, float one_m_eps, float eps_v, float z) {
    const long long row = blockIdx.x;
    __nv_bfloat16* x = logits + row * (size_t)Vp;
    const long long label = labels[row];
    const int nvec = Vp >> 3;
    if (label == ignore_index) {
        bf16x8 z;
#pragma unroll
        for (int i = 0; i < 4; ++i) z.v[i] = __floats2bfloat162_rn(0.f, 0.f);
        for (int v = threadIdx.x; v < nvec; v += kCEThreads) st_stream(x + 8 * v, z);
        return;
    }
    const float lse = lse_in[row];
    const float scale = *scale_ptr;
    float zf = 1.f;                        // kZ: d(z lse^2) / dx_c = 2 z lse softmax_c folds into the softmax's factor
    if constexpr (kZ) zf = 1.f + 2.f * z * lse;
    for (int v = threadIdx.x; v < nvec; v += kCEThreads) {
        float f[8];
        unpack8(ld_stream_rw(x + 8 * v), f);
        const int c0 = 8 * v;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int c = c0 + j;
            if constexpr (kZ) {
                float p = (c < V) ? __expf(f[j] - lse) * zf - eps_v : 0.f;   // eps_v = 0 unless kSmooth
                if (c == label) p -= one_m_eps;                               // one_m_eps = 1 unless kSmooth
                f[j] = p * scale;
            } else if constexpr (kSmooth) {
                float p = (c < V) ? __expf(f[j] - lse) - eps_v : 0.f;
                if (c == label) p -= one_m_eps;
                f[j] = p * scale;
            } else {
                float p = (c < V) ? __expf(f[j] - lse) : 0.f;
                if (c == label) p -= 1.f;
                f[j] = p * scale;
            }
        }
        st_stream(x + 8 * v, pack8(f));
    }
}

template <bool kSmooth, bool kZ>
void launch_ce_fwd(const void* logits, const long long* labels, float* lse, float* row_loss, float* loss, float* inv_n, long long T, int V,
                   int Vp, long long ignore_index, float one_m_eps, float eps_v, float z, float* z_out, cudaStream_t st) {
    ce_fwd_kernel<kSmooth, kZ><<<(unsigned)T, kCEThreads, 0, st>>>((const __nv_bfloat16*)logits, labels, lse, row_loss, V, Vp, ignore_index,
                                                                   one_m_eps, eps_v, z);
    ce_reduce_kernel<kZ><<<1, 1024, 0, st>>>(row_loss, labels, loss, inv_n, T, ignore_index, lse, z_out, z);
}

template <bool kSmooth, bool kZ>
void launch_ce_bwd(void* logits, const long long* labels, const float* lse, const float* scale, long long T, int V, int Vp,
                   long long ignore_index, float one_m_eps, float eps_v, float z, cudaStream_t st) {
    ce_bwd_kernel<kSmooth, kZ><<<(unsigned)T, kCEThreads, 0, st>>>((__nv_bfloat16*)logits, labels, lse, scale, V, Vp, ignore_index,
                                                                   one_m_eps, eps_v, z);
}

}  // namespace acco

// `label_smoothing` in [0, 1] and `z_loss` >= 0 (checked by the binding); 0 runs the instantiation without the term.  With
// z_loss > 0, `z_out` (one fp32) receives the mean z-term.
extern "C" int acco_ce_fwd(const void* logits, const long long* labels, float* lse, float* row_loss, float* loss, float* inv_n,
                           long long T, int V, int Vp, long long ignore_index, float label_smoothing, float z_loss, float* z_out,
                           cudaStream_t st) {
    if (Vp % 8 != 0 || V > Vp || (z_loss != 0.f && z_out == nullptr)) return -1;
    const float one_m_eps = 1.f - label_smoothing, eps_v = label_smoothing / (float)V;
    const bool smooth = label_smoothing != 0.f, zl = z_loss != 0.f;
    auto f = smooth ? (zl ? acco::launch_ce_fwd<true, true> : acco::launch_ce_fwd<true, false>)
                    : (zl ? acco::launch_ce_fwd<false, true> : acco::launch_ce_fwd<false, false>);
    f(logits, labels, lse, row_loss, loss, inv_n, T, V, Vp, ignore_index, one_m_eps, eps_v, z_loss, z_out, st);
    return 0;
}

extern "C" int acco_ce_bwd(void* logits, const long long* labels, const float* lse, const float* scale, long long T, int V, int Vp,
                           long long ignore_index, float label_smoothing, float z_loss, cudaStream_t st) {
    if (Vp % 8 != 0 || V > Vp) return -1;
    const float one_m_eps = 1.f - label_smoothing, eps_v = label_smoothing / (float)V;
    const bool smooth = label_smoothing != 0.f, zl = z_loss != 0.f;
    auto f = smooth ? (zl ? acco::launch_ce_bwd<true, true> : acco::launch_ce_bwd<true, false>)
                    : (zl ? acco::launch_ce_bwd<false, true> : acco::launch_ce_bwd<false, false>);
    f(logits, labels, lse, scale, T, V, Vp, ignore_index, one_m_eps, eps_v, z_loss, st);
    return 0;
}
