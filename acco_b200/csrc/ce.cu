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
#include "common.cuh"

namespace acco {

constexpr int kCEThreads = 512;

template <bool kSmooth>
__global__ void __launch_bounds__(kCEThreads) ce_fwd_kernel(const __nv_bfloat16* __restrict__ logits,
                                                            const long long* __restrict__ labels, float* __restrict__ lse_out,
                                                            float* __restrict__ row_loss, int V, int Vp, long long ignore_index,
                                                            float one_m_eps, float eps_v) {
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
            row_loss[row] = lse - one_m_eps * __bfloat162float(x[label]) - eps_v * gsx;
        }
    } else {
        if (threadIdx.x == 0) {
            const float lse = gm + __logf(gs);
            lse_out[row] = lse;
            row_loss[row] = lse - __bfloat162float(x[label]);
        }
    }
}

__global__ void __launch_bounds__(1024) ce_reduce_kernel(const float* __restrict__ row_loss, const long long* __restrict__ labels,
                                                         float* __restrict__ loss, float* __restrict__ inv_n, long long T,
                                                         long long ignore_index) {
    __shared__ float red[32];
    float s = 0.f, n = 0.f;
    for (long long i = threadIdx.x; i < T; i += blockDim.x) {
        if (labels[i] != ignore_index) {
            s += row_loss[i];
            n += 1.f;
        }
    }
    s = block_sum(s, red);
    n = block_sum(n, red);
    if (threadIdx.x == 0) {
        const float inv = n > 0.f ? 1.f / n : 0.f;
        *loss = s * inv;
        *inv_n = inv;
    }
}

template <bool kSmooth>
__global__ void __launch_bounds__(kCEThreads) ce_bwd_kernel(__nv_bfloat16* __restrict__ logits, const long long* __restrict__ labels,
                                                            const float* __restrict__ lse_in, const float* __restrict__ scale_ptr,
                                                            int V, int Vp, long long ignore_index, float one_m_eps, float eps_v) {
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
    for (int v = threadIdx.x; v < nvec; v += kCEThreads) {
        float f[8];
        unpack8(ld_stream_rw(x + 8 * v), f);
        const int c0 = 8 * v;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int c = c0 + j;
            if constexpr (kSmooth) {
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

}  // namespace acco

// `label_smoothing` in [0, 1] (checked by the binding); 0 runs the unsmoothed instantiation.
extern "C" int acco_ce_fwd(const void* logits, const long long* labels, float* lse, float* row_loss, float* loss, float* inv_n,
                           long long T, int V, int Vp, long long ignore_index, float label_smoothing, cudaStream_t st) {
    if (Vp % 8 != 0 || V > Vp) return -1;
    const float one_m_eps = 1.f - label_smoothing, eps_v = label_smoothing / (float)V;
    if (label_smoothing != 0.f)
        acco::ce_fwd_kernel<true><<<(unsigned)T, acco::kCEThreads, 0, st>>>((const __nv_bfloat16*)logits, labels, lse, row_loss, V, Vp,
                                                                            ignore_index, one_m_eps, eps_v);
    else
        acco::ce_fwd_kernel<false><<<(unsigned)T, acco::kCEThreads, 0, st>>>((const __nv_bfloat16*)logits, labels, lse, row_loss, V, Vp,
                                                                             ignore_index, one_m_eps, eps_v);
    acco::ce_reduce_kernel<<<1, 1024, 0, st>>>(row_loss, labels, loss, inv_n, T, ignore_index);
    return 0;
}

extern "C" int acco_ce_bwd(void* logits, const long long* labels, const float* lse, const float* scale, long long T, int V, int Vp,
                           long long ignore_index, float label_smoothing, cudaStream_t st) {
    if (Vp % 8 != 0 || V > Vp) return -1;
    const float one_m_eps = 1.f - label_smoothing, eps_v = label_smoothing / (float)V;
    if (label_smoothing != 0.f)
        acco::ce_bwd_kernel<true><<<(unsigned)T, acco::kCEThreads, 0, st>>>((__nv_bfloat16*)logits, labels, lse, scale, V, Vp, ignore_index,
                                                                            one_m_eps, eps_v);
    else
        acco::ce_bwd_kernel<false><<<(unsigned)T, acco::kCEThreads, 0, st>>>((__nv_bfloat16*)logits, labels, lse, scale, V, Vp,
                                                                             ignore_index, one_m_eps, eps_v);
    return 0;
}
