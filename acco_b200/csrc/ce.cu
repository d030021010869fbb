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
//
// Knowledge distillation (kd_*, separate kernels; the ce_* instantiations above are untouched).  Student logits s and frozen
// teacher logits t, both bf16 [T, Vp], temperature T > 0 and weight a in (0, 1]; per non-ignored row
//   row = (1 - a) (lse(s) - s[y])  +  a T^2 KL(softmax(t/T) || softmax(s/T)),
//   KL  = sum_c q_c (t_c/T - s_c/T) - lse(t/T) + lse(s/T),   q = softmax(t/T),
//   d s_c = scale ((1 - a) (softmax(s)_c - [c = y]) + a T (softmax(s/T)_c - q_c))      (c < V; padding, ignored rows: 0).
//   kd_fwd : one CTA per row, ONE streaming pass over both rows: online max/sum of s, of s/T and of t/T, plus the running sum
//            K = sum e^{t/T - m} (t/T - s/T) rescaled with the t/T sum, so sum_c q_c (t/T - s/T) = K / S at the row end.
//            Stores lse(s), lse(s/T), lse(t/T) [3, T] and the row's CE and KL [2, T].  kT1 (T == 1) shares the first two.
//   kd_reduce : ce_reduce's order -> objective, inv_n, and out[2] = (mean CE, mean KL) over the non-ignored rows.
//   kd_bwd : in place on s, reading t once more.
//
// DPO (dpo_*, separate kernels).  Policy logits s and frozen reference logits r, both bf16 [2P S, Vp]: rows [0, P) of the
// [2P, S] token layout are the chosen responses, rows [P, 2P) the rejected ones, pair i = (i, P + i); R(row) = its non-ignored
// positions.  l(row) = sum_{t in R(row)} (s_t[y_t] - lse(s_t)), l_ref the same over r;
//   z_i = beta [(l(c_i) - l_ref(c_i)) - (l(r_i) - l_ref(r_i))],  loss = mean over valid pairs (both rows non-empty) of softplus(-z_i),
//   d s_tc = dloss (+-beta sigma(-z_i) / n) (softmax(s_t)_c - [c = y_t])   (+ chosen, - rejected; padding, ignored, invalid: 0).
//   dpo_fwd : one CTA per token row, ONE streaming pass over both rows -> lse(s_t) and d_t = (s_t[y] - lse(s_t)) - (r_t[y] - lse(r_t)).
//             Subtracting per token keeps the cancellation out of the long fp32 sums and makes d == 0 exact for s == r.
//   dpo_reduce : one CTA, fixed order: row sums of d, z, the loss, the per-row weight w and three logged means.
//   dpo_bwd : in place on s, like ce_bwd with the scale dloss * w[row].
//
// Reference-free preference objectives (pref_reduce<kSimPO | kORPO>; no reference logits).  Same [2P, S] pair layout;
// l(row) = sum_{t in R(row)} (s_t[y_t] - lse(s_t)), a(row) = l(row) / |row|, valid pair = both rows non-empty, n = #valid.
//   SimPO: z_i = beta (a(c_i) - a(r_i)) - gamma,  loss = mean_valid softplus(-z_i),
//          w(c_i) = beta sigma(-z_i) / (n |c_i|),  w(r_i) = -beta sigma(-z_i) / (n |r_i|).
//   ORPO:  nll = -sum_valid l(c_i) / N_c (N_c = sum_valid |c_i|),  lo_i = (a - log(1 - e^a'))(c_i) - (a - log(1 - e^a'))(r_i),
//          a' = min(a, -2^-20) (the clamp also enters the gradient),  loss = nll + lambda mean_valid softplus(-lo_i),
//          w(c_i) = 1 / N_c + lambda sigma(-lo_i) / (n |c_i| (1 - e^a'(c_i))),  w(r_i) = -lambda sigma(-lo_i) / (n |r_i| (1 - e^a'(r_i))).
//   Forward: ce_fwd<false, false> (lse and -log p per token) and pref_reduce; backward: dpo_bwd with the weights w.
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

// ---------------------------------------------------------------- knowledge distillation
// Online update of (m, sum) with 8 values already in the softmax's scale.
ACCO_DEVINL void online8(const float (&f)[8], float& m, float& s) {
    float lm = f[0];
#pragma unroll
    for (int j = 1; j < 8; ++j) lm = fmaxf(lm, f[j]);
    const float nm = fmaxf(m, lm);
    float acc = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) acc += __expf(f[j] - nm);
    s = s * __expf(m - nm) + acc;
    m = nm;
}

// lse of the CTA from each thread's (m, s); every thread gets it.
ACCO_DEVINL float block_lse(float m, float s, float* red) {
    const float gm = block_max(m, red);
    const float part = (m == -INFINITY) ? 0.f : s * __expf(m - gm);
    return gm + __logf(block_sum(part, red));
}

// lse3 [3, T]: lse(s), lse(s/T), lse(t/T); rows [2, T]: CE and KL of the row (all 0 on ignored rows).  inv_t = 1/T (fp32, host).
template <bool kT1>
__global__ void __launch_bounds__(kCEThreads) kd_fwd_kernel(const __nv_bfloat16* __restrict__ student, const __nv_bfloat16* __restrict__ teacher,
                                                            const long long* __restrict__ labels, float* __restrict__ lse3,
                                                            float* __restrict__ rows, long long T, int V, int Vp, long long ignore_index,
                                                            float inv_t) {
    __shared__ float red[32];
    const long long row = blockIdx.x;
    const __nv_bfloat16* x = student + row * (size_t)Vp;
    const __nv_bfloat16* y = teacher + row * (size_t)Vp;
    const long long label = labels[row];
    if (label == ignore_index) {
        if (threadIdx.x == 0) {
            lse3[row] = lse3[T + row] = lse3[2 * T + row] = 0.f;
            rows[row] = rows[T + row] = 0.f;
        }
        return;
    }
    const int nvec_full = V >> 3;
    float m1 = -INFINITY, s1 = 0.f;        // s
    float m2 = -INFINITY, s2 = 0.f;        // s / T  (!kT1)
    float m3 = -INFINITY, s3 = 0.f;        // t / T
    float k3 = 0.f;                        // sum e^{t/T - m3} (t/T - s/T), rescaled with s3
    for (int v = threadIdx.x; v < nvec_full; v += kCEThreads) {
        float f[8], g[8];
        unpack8(ld_stream(x + 8 * v), f);
        unpack8(ld_stream(y + 8 * v), g);
        online8(f, m1, s1);
        if constexpr (!kT1) {
#pragma unroll
            for (int j = 0; j < 8; ++j) { f[j] *= inv_t; g[j] *= inv_t; }
            online8(f, m2, s2);
        }
        float lm = g[0];
#pragma unroll
        for (int j = 1; j < 8; ++j) lm = fmaxf(lm, g[j]);
        const float nm = fmaxf(m3, lm);
        float acc = 0.f, acck = 0.f;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const float e = __expf(g[j] - nm);
            acc += e;
            acck += e * (g[j] - f[j]);
        }
        const float r = __expf(m3 - nm);
        s3 = s3 * r + acc;
        k3 = k3 * r + acck;
        m3 = nm;
    }
    for (int c = (nvec_full << 3) + threadIdx.x; c < V; c += kCEThreads) {
        float f = __bfloat162float(x[c]), g = __bfloat162float(y[c]);
        float nm = fmaxf(m1, f);
        s1 = s1 * __expf(m1 - nm) + __expf(f - nm);
        m1 = nm;
        if constexpr (!kT1) {
            f *= inv_t;
            g *= inv_t;
            nm = fmaxf(m2, f);
            s2 = s2 * __expf(m2 - nm) + __expf(f - nm);
            m2 = nm;
        }
        nm = fmaxf(m3, g);
        const float r = __expf(m3 - nm), e = __expf(g - nm);
        s3 = s3 * r + e;
        k3 = k3 * r + e * (g - f);
        m3 = nm;
    }
    const float lse1 = block_lse(m1, s1, red);
    float lse2 = lse1;
    if constexpr (!kT1) lse2 = block_lse(m2, s2, red);
    const float gm3 = block_max(m3, red);
    const float w = (m3 == -INFINITY) ? 0.f : __expf(m3 - gm3);
    const float gs3 = block_sum(s3 * w, red);
    const float gk3 = block_sum(k3 * w, red);
    if (threadIdx.x == 0) {
        const float lse_t = gm3 + __logf(gs3);
        lse3[row] = lse1;
        lse3[T + row] = lse2;
        lse3[2 * T + row] = lse_t;
        rows[row] = lse1 - __bfloat162float(x[label]);
        rows[T + row] = (gk3 / gs3 - lse_t) + lse2;
    }
}

// loss = (one_m_a sum CE + a_t2 sum KL) / n; out = (sum CE / n, sum KL / n); the sums in ce_reduce_kernel's order.
__global__ void __launch_bounds__(1024) kd_reduce_kernel(const float* __restrict__ rows, const long long* __restrict__ labels,
                                                         float* __restrict__ loss, float* __restrict__ inv_n, float* __restrict__ out,
                                                         long long T, long long ignore_index, float one_m_a, float a_t2) {
    __shared__ float red[32];
    float sc = 0.f, sk = 0.f, n = 0.f;
    for (long long i = threadIdx.x; i < T; i += blockDim.x) {
        if (labels[i] != ignore_index) {
            sc += rows[i];
            sk += rows[T + i];
            n += 1.f;
        }
    }
    sc = block_sum(sc, red);
    sk = block_sum(sk, red);
    n = block_sum(n, red);
    if (threadIdx.x == 0) {
        const float inv = n > 0.f ? 1.f / n : 0.f;
        const float ce = sc * inv, kl = sk * inv;
        *loss = one_m_a * ce + a_t2 * kl;
        *inv_n = inv;
        out[0] = ce;
        out[1] = kl;
    }
}

// s <- scale ((1 - a)(softmax(s) - onehot) + a T (softmax(s/T) - softmax(t/T))); kT1: scale (softmax(s) - (1 - a) onehot - a q).
template <bool kT1>
__global__ void __launch_bounds__(kCEThreads) kd_bwd_kernel(__nv_bfloat16* __restrict__ student, const __nv_bfloat16* __restrict__ teacher,
                                                            const long long* __restrict__ labels, const float* __restrict__ lse3,
                                                            const float* __restrict__ scale_ptr, long long T, int V, int Vp,
                                                            long long ignore_index, float one_m_a, float a_t, float inv_t) {
    const long long row = blockIdx.x;
    __nv_bfloat16* x = student + row * (size_t)Vp;
    const __nv_bfloat16* y = teacher + row * (size_t)Vp;
    const long long label = labels[row];
    const int nvec = Vp >> 3;
    if (label == ignore_index) {
        bf16x8 z;
#pragma unroll
        for (int i = 0; i < 4; ++i) z.v[i] = __floats2bfloat162_rn(0.f, 0.f);
        for (int v = threadIdx.x; v < nvec; v += kCEThreads) st_stream(x + 8 * v, z);
        return;
    }
    const float lse1 = lse3[row], lse2 = lse3[T + row], lse_t = lse3[2 * T + row];
    const float scale = *scale_ptr;
    for (int v = threadIdx.x; v < nvec; v += kCEThreads) {
        float f[8], g[8];
        unpack8(ld_stream_rw(x + 8 * v), f);
        unpack8(ld_stream(y + 8 * v), g);
        const int c0 = 8 * v;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int c = c0 + j;
            float d = 0.f;
            if (c < V) {
                const float p = __expf(f[j] - lse1);
                if constexpr (kT1) {
                    d = p - a_t * __expf(g[j] - lse_t);                  // a_t = a when T == 1
                } else {
                    d = one_m_a * p + a_t * (__expf(f[j] * inv_t - lse2) - __expf(g[j] * inv_t - lse_t));
                }
                if (c == label) d -= one_m_a;
            }
            f[j] = d * scale;
        }
        st_stream(x + 8 * v, pack8(f));
    }
}

template <bool kT1>
void launch_kd(const void* s, const void* t, const long long* labels, float* lse3, float* rows, float* loss, float* inv_n, float* out,
               long long T, int V, int Vp, long long ignore_index, float one_m_a, float a_t2, float inv_t, cudaStream_t st) {
    kd_fwd_kernel<kT1><<<(unsigned)T, kCEThreads, 0, st>>>((const __nv_bfloat16*)s, (const __nv_bfloat16*)t, labels, lse3, rows, T, V, Vp,
                                                           ignore_index, inv_t);
    kd_reduce_kernel<<<1, 1024, 0, st>>>(rows, labels, loss, inv_n, out, T, ignore_index, one_m_a, a_t2);
}

bool kd_args_ok(int V, int Vp, float alpha, float temperature) {
    return Vp % 8 == 0 && V > 0 && V <= Vp && alpha > 0.f && alpha <= 1.f && temperature > 0.f && temperature < INFINITY;
}

// ---------------------------------------------------------------- DPO
// d [T]: per token (s[y] - lse(s)) - (r[y] - lse(r)), lse [T]: lse(s); both 0 on ignored rows.  The two log-probabilities are
// formed by the same instructions, so d == 0 exactly when s and r are bitwise equal.
__global__ void __launch_bounds__(kCEThreads) dpo_fwd_kernel(const __nv_bfloat16* __restrict__ policy, const __nv_bfloat16* __restrict__ ref,
                                                             const long long* __restrict__ labels, float* __restrict__ lse_out,
                                                             float* __restrict__ d_out, int V, int Vp, long long ignore_index) {
    __shared__ float red[32];
    const long long row = blockIdx.x;
    const __nv_bfloat16* x = policy + row * (size_t)Vp;
    const __nv_bfloat16* y = ref + row * (size_t)Vp;
    const long long label = labels[row];
    if (label == ignore_index) {
        if (threadIdx.x == 0) lse_out[row] = d_out[row] = 0.f;
        return;
    }
    const int nvec_full = V >> 3;
    float m1 = -INFINITY, s1 = 0.f, m2 = -INFINITY, s2 = 0.f;
    for (int v = threadIdx.x; v < nvec_full; v += kCEThreads) {
        float f[8], g[8];
        unpack8(ld_stream(x + 8 * v), f);
        unpack8(ld_stream(y + 8 * v), g);
        online8(f, m1, s1);
        online8(g, m2, s2);
    }
    for (int c = (nvec_full << 3) + threadIdx.x; c < V; c += kCEThreads) {
        const float f = __bfloat162float(x[c]), g = __bfloat162float(y[c]);
        float nm = fmaxf(m1, f);
        s1 = s1 * __expf(m1 - nm) + __expf(f - nm);
        m1 = nm;
        nm = fmaxf(m2, g);
        s2 = s2 * __expf(m2 - nm) + __expf(g - nm);
        m2 = nm;
    }
    const float lse1 = block_lse(m1, s1, red);
    const float lse2 = block_lse(m2, s2, red);
    if (threadIdx.x == 0) {
        lse_out[row] = lse1;
        d_out[row] = (__bfloat162float(x[label]) - lse1) - (__bfloat162float(y[label]) - lse2);
    }
}

// One CTA of 1024 threads, fixed order (two launches are bitwise equal).  Rows are [2P, S] token rows: pair i is (i, P + i).
//   rowbuf [2, 2P]: per row sum of d and count of non-ignored tokens (warp w sums rows w, w + 32, ...).
//   z_i = beta (D[i] - D[P + i]); a pair is valid when both rows have a token; n = #valid.
//   loss = sum_valid softplus(-z_i) / n;  w[i] = beta sigma(-z_i) / n = -w[P + i] (0 for invalid pairs);
//   out = (mean beta D[i], mean beta D[P + i], mean [z_i > 0]) over the valid pairs.  n = 0: all 0.
__global__ void __launch_bounds__(1024) dpo_reduce_kernel(const float* __restrict__ d, const long long* __restrict__ labels,
                                                          float* __restrict__ rowbuf, float* __restrict__ w, float* __restrict__ loss,
                                                          float* __restrict__ out, int P, int S, long long ignore_index, float beta) {
    __shared__ float red[32];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
    const int R = 2 * P;
    for (int r = wid; r < R; r += nw) {
        float sd = 0.f, cnt = 0.f;
        for (int t = lane; t < S; t += 32) {
            const long long i = (long long)r * S + t;
            if (labels[i] != ignore_index) {
                sd += d[i];
                cnt += 1.f;
            }
        }
        sd = warp_sum(sd);
        cnt = warp_sum(cnt);
        if (lane == 0) {
            rowbuf[r] = sd;
            rowbuf[R + r] = cnt;
        }
    }
    __syncthreads();
    float n = 0.f, sl = 0.f, sc = 0.f, sr = 0.f, sa = 0.f;
    for (int i = threadIdx.x; i < P; i += blockDim.x) {
        if (rowbuf[R + i] > 0.f && rowbuf[R + P + i] > 0.f) {
            const float rc = __fmul_rn(beta, rowbuf[i]), rr = __fmul_rn(beta, rowbuf[P + i]), z = __fsub_rn(rc, rr);
            n += 1.f;
            sl += fmaxf(-z, 0.f) + log1pf(__expf(-fabsf(z)));      // softplus(-z), stable for any |z|
            sc += rc;
            sr += rr;
            sa += z > 0.f ? 1.f : 0.f;
        }
    }
    n = block_sum(n, red);
    sl = block_sum(sl, red);
    sc = block_sum(sc, red);
    sr = block_sum(sr, red);
    sa = block_sum(sa, red);
    const float inv = n > 0.f ? 1.f / n : 0.f;
    for (int i = threadIdx.x; i < P; i += blockDim.x) {
        float c = 0.f;
        if (rowbuf[R + i] > 0.f && rowbuf[R + P + i] > 0.f) {
            const float z = __fsub_rn(__fmul_rn(beta, rowbuf[i]), __fmul_rn(beta, rowbuf[P + i]));   // as above
            const float e = __expf(-fabsf(z));
            c = beta * (z >= 0.f ? e / (1.f + e) : 1.f / (1.f + e)) * inv;    // beta sigma(-z) / n
        }
        w[i] = c;
        w[P + i] = -c;
    }
    if (threadIdx.x == 0) {
        *loss = sl * inv;
        out[0] = sc * inv;
        out[1] = sr * inv;
        out[2] = sa * inv;
    }
}

// In place on the policy logits: dloss w[row / S] (softmax - onehot) on non-ignored rows and valid columns, else 0.
__global__ void __launch_bounds__(kCEThreads) dpo_bwd_kernel(__nv_bfloat16* __restrict__ logits, const long long* __restrict__ labels,
                                                             const float* __restrict__ lse_in, const float* __restrict__ w,
                                                             const float* __restrict__ dloss, int S, int V, int Vp, long long ignore_index) {
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
    const float scale = *dloss * w[row / S];
    for (int v = threadIdx.x; v < nvec; v += kCEThreads) {
        float f[8];
        unpack8(ld_stream_rw(x + 8 * v), f);
        const int c0 = 8 * v;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int c = c0 + j;
            float p = (c < V) ? __expf(f[j] - lse) : 0.f;
            if (c == label) p -= 1.f;
            f[j] = p * scale;
        }
        st_stream(x + 8 * v, pack8(f));
    }
}

// ---------------------------------------------------------------- SimPO / ORPO
constexpr int kSimPO = 0, kORPO = 1;
constexpr float kORPOMaxA = -9.5367431640625e-07f;      // -2^-20: a is clamped below 0 so that log(1 - e^a) stays finite

ACCO_DEVINL float softplus_neg(float z) { return fmaxf(-z, 0.f) + log1pf(__expf(-fabsf(z))); }     // softplus(-z), any |z|

ACCO_DEVINL float sigmoid_neg(float z) {                // sigma(-z), any |z|
    const float e = __expf(-fabsf(z));
    return z >= 0.f ? e / (1.f + e) : 1.f / (1.f + e);
}

ACCO_DEVINL float log1m_exp(float a) {                  // log(1 - e^a) for a < 0, without cancellation on either side of -ln 2
    return a > -0.693147182f ? __logf(-expm1f(a)) : log1pf(-__expf(a));
}

// One CTA of 1024 threads, fixed order (two launches are bitwise equal), over ce_fwd's per-token -log p (0 on ignored tokens).
//   rowbuf [2, 2P]: per row l = -sum row_loss and the count of non-ignored tokens (warp w sums rows w, w + 32, ...).
//   coef: SimPO's beta or ORPO's lambda; gamma: SimPO's margin (ORPO ignores it).
//   out: SimPO (mean beta a(c), mean beta a(r), mean [a(c) > a(r)]), ORPO (nll, mean lo, mean [lo > 0]).  n = 0: loss, w, out 0.
template <int kObj>
__global__ void __launch_bounds__(1024) pref_reduce_kernel(const float* __restrict__ row_loss, const long long* __restrict__ labels,
                                                           float* __restrict__ rowbuf, float* __restrict__ w, float* __restrict__ loss,
                                                           float* __restrict__ out, int P, int S, long long ignore_index, float coef,
                                                           float gamma) {
    __shared__ float red[32];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
    const int R = 2 * P;
    for (int r = wid; r < R; r += nw) {
        float sl = 0.f, cnt = 0.f;
        for (int t = lane; t < S; t += 32) {
            const long long i = (long long)r * S + t;
            if (labels[i] != ignore_index) {
                sl -= row_loss[i];
                cnt += 1.f;
            }
        }
        sl = warp_sum(sl);
        cnt = warp_sum(cnt);
        if (lane == 0) {
            rowbuf[r] = sl;
            rowbuf[R + r] = cnt;
        }
    }
    __syncthreads();
    // SimPO: s1, s2 = sums of beta a(c), beta a(r).  ORPO: s1 = sum l(c), s2 = sum lo, sn = N_c.
    float n = 0.f, sl = 0.f, s1 = 0.f, s2 = 0.f, sa = 0.f, sn = 0.f;
    for (int i = threadIdx.x; i < P; i += blockDim.x) {
        const float nc = rowbuf[R + i], nr = rowbuf[R + P + i];
        if (nc > 0.f && nr > 0.f) {
            const float ac = rowbuf[i] / nc, ar = rowbuf[P + i] / nr;
            n += 1.f;
            if constexpr (kObj == kSimPO) {
                const float rc = __fmul_rn(coef, ac), rr = __fmul_rn(coef, ar);
                sl += softplus_neg(__fsub_rn(__fsub_rn(rc, rr), gamma));
                s1 += rc;
                s2 += rr;
                sa += ac > ar ? 1.f : 0.f;
            } else {
                const float lo = (ac - log1m_exp(fminf(ac, kORPOMaxA))) - (ar - log1m_exp(fminf(ar, kORPOMaxA)));
                sl += softplus_neg(lo);
                s1 += rowbuf[i];
                s2 += lo;
                sa += lo > 0.f ? 1.f : 0.f;
                sn += nc;
            }
        }
    }
    n = block_sum(n, red);
    sl = block_sum(sl, red);
    s1 = block_sum(s1, red);
    s2 = block_sum(s2, red);
    sa = block_sum(sa, red);
    if constexpr (kObj == kORPO) sn = block_sum(sn, red);
    const float inv = n > 0.f ? 1.f / n : 0.f;
    const float inv_nc = sn > 0.f ? 1.f / sn : 0.f;
    for (int i = threadIdx.x; i < P; i += blockDim.x) {
        const float nc = rowbuf[R + i], nr = rowbuf[R + P + i];
        float wc = 0.f, wr = 0.f;
        if (nc > 0.f && nr > 0.f) {
            const float ac = rowbuf[i] / nc, ar = rowbuf[P + i] / nr;                                   // as above
            if constexpr (kObj == kSimPO) {
                const float z = __fsub_rn(__fsub_rn(__fmul_rn(coef, ac), __fmul_rn(coef, ar)), gamma);
                const float g = coef * sigmoid_neg(z) * inv;
                wc = g / nc;
                wr = -g / nr;
            } else {
                const float cc = fminf(ac, kORPOMaxA), cr = fminf(ar, kORPOMaxA);
                const float g = coef * sigmoid_neg((ac - log1m_exp(cc)) - (ar - log1m_exp(cr))) * inv;
                wc = inv_nc + g / (nc * -expm1f(cc));
                wr = -g / (nr * -expm1f(cr));
            }
        }
        w[i] = wc;
        w[P + i] = wr;
    }
    if (threadIdx.x == 0) {
        if constexpr (kObj == kSimPO) {
            *loss = sl * inv;
            out[0] = s1 * inv;
        } else {
            const float nll = (0.f - s1) * inv_nc;
            *loss = nll + coef * (sl * inv);
            out[0] = nll;
        }
        out[1] = s2 * inv;
        out[2] = sa * inv;
    }
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

// Knowledge distillation: `alpha` in (0, 1], finite `temperature` > 0, Vp % 8 == 0 and V <= Vp, else -1 (nothing launched).
// `out` (two fp32) receives the mean CE and the mean KL over the non-ignored rows.
extern "C" int acco_kd_fwd(const void* student, const void* teacher, const long long* labels, float* lse3, float* rows, float* loss,
                           float* inv_n, float* out, long long T, int V, int Vp, long long ignore_index, float alpha, float temperature,
                           cudaStream_t st) {
    if (!acco::kd_args_ok(V, Vp, alpha, temperature) || out == nullptr) return -1;
    const float one_m_a = 1.f - alpha, a_t2 = alpha * temperature * temperature, inv_t = 1.f / temperature;
    auto f = temperature == 1.f ? acco::launch_kd<true> : acco::launch_kd<false>;
    f(student, teacher, labels, lse3, rows, loss, inv_n, out, T, V, Vp, ignore_index, one_m_a, a_t2, inv_t, st);
    return 0;
}

extern "C" int acco_kd_bwd(void* student, const void* teacher, const long long* labels, const float* lse3, const float* scale, long long T,
                           int V, int Vp, long long ignore_index, float alpha, float temperature, cudaStream_t st) {
    if (!acco::kd_args_ok(V, Vp, alpha, temperature)) return -1;
    const float one_m_a = 1.f - alpha, a_t = alpha * temperature, inv_t = 1.f / temperature;
    auto k = temperature == 1.f ? acco::kd_bwd_kernel<true> : acco::kd_bwd_kernel<false>;
    k<<<(unsigned)T, acco::kCEThreads, 0, st>>>((__nv_bfloat16*)student, (const __nv_bfloat16*)teacher, labels, lse3, scale, T, V, Vp,
                                                ignore_index, one_m_a, a_t, inv_t);
    return 0;
}

// DPO over T = 2 P S token rows (pair i = rows [i S, (i+1) S) and [(P+i) S, (P+i+1) S)): finite beta > 0, P, S > 0, Vp % 8 == 0 and
// V <= Vp, else -1 (nothing launched).  Writes lse, d [T], rowbuf [4P], w [2P], the loss and `out` (three fp32).
extern "C" int acco_dpo_fwd(const void* policy, const void* ref, const long long* labels, float* lse, float* d, float* rowbuf, float* w,
                            float* loss, float* out, int P, int S, int V, int Vp, long long ignore_index, float beta, cudaStream_t st) {
    if (Vp % 8 != 0 || V <= 0 || V > Vp || P <= 0 || S <= 0 || !(beta > 0.f && beta < INFINITY) || out == nullptr) return -1;
    const long long T = 2LL * P * S;
    acco::dpo_fwd_kernel<<<(unsigned)T, acco::kCEThreads, 0, st>>>((const __nv_bfloat16*)policy, (const __nv_bfloat16*)ref, labels, lse, d, V,
                                                                   Vp, ignore_index);
    acco::dpo_reduce_kernel<<<1, 1024, 0, st>>>(d, labels, rowbuf, w, loss, out, P, S, ignore_index, beta);
    return 0;
}

extern "C" int acco_dpo_bwd(void* policy, const long long* labels, const float* lse, const float* w, const float* dloss, int P, int S, int V,
                            int Vp, long long ignore_index, cudaStream_t st) {
    if (Vp % 8 != 0 || V <= 0 || V > Vp || P <= 0 || S <= 0) return -1;
    acco::dpo_bwd_kernel<<<(unsigned)(2LL * P * S), acco::kCEThreads, 0, st>>>((__nv_bfloat16*)policy, labels, lse, w, dloss, S, V, Vp,
                                                                               ignore_index);
    return 0;
}

// SimPO (orpo == 0: coef = beta, gamma >= 0) or ORPO (orpo != 0: coef = lambda) over T = 2 P S token rows: finite coef > 0, finite
// gamma >= 0, P, S > 0, Vp % 8 == 0 and V <= Vp, else -1 (nothing launched).  Writes lse, row_loss [T], rowbuf [4P], w [2P], the
// loss and `out` (three fp32).  The backward is acco_dpo_bwd with these w.
extern "C" int acco_pref_fwd(const void* logits, const long long* labels, float* lse, float* row_loss, float* rowbuf, float* w, float* loss,
                             float* out, int P, int S, int V, int Vp, long long ignore_index, int orpo, float coef, float gamma,
                             cudaStream_t st) {
    if (Vp % 8 != 0 || V <= 0 || V > Vp || P <= 0 || S <= 0 || !(coef > 0.f && coef < INFINITY) || !(gamma >= 0.f && gamma < INFINITY) ||
        out == nullptr)
        return -1;
    const long long T = 2LL * P * S;
    acco::ce_fwd_kernel<false, false><<<(unsigned)T, acco::kCEThreads, 0, st>>>((const __nv_bfloat16*)logits, labels, lse, row_loss, V, Vp,
                                                                                ignore_index, 1.f, 0.f, 0.f);
    auto k = orpo ? acco::pref_reduce_kernel<acco::kORPO> : acco::pref_reduce_kernel<acco::kSimPO>;
    k<<<1, 1024, 0, st>>>(row_loss, labels, rowbuf, w, loss, out, P, S, ignore_index, coef, gamma);
    return 0;
}
