// Python bindings (torch extension) for the acco_b200 sm_90a kernels.  Kernels live in plain .cu
// files with C launchers (no torch headers there, so they compile in seconds); this file only
// validates tensors, allocates outputs and forwards raw pointers on the current CUDA stream.
#include <torch/extension.h>
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <cuda_runtime.h>

#include <cmath>
#include <cstdlib>
#include <vector>

extern "C" {
int acco_norm_grid(int T, int H, int sms, int backward);
int acco_norm_fwd(const void* a, const void* r, const void* w, const void* b, void* y, void* h, float* mean, float* rstd, int T, int H,
                  float eps, int grid, cudaStream_t st);
int acco_norm_bwd(const void* dy, const void* dh_extra, const void* h, const void* w, const float* mean, const float* rstd, void* dh,
                  float* partial, float* dwdb_out, void* dw_accum, void* db_accum, int T, int H, int grid, cudaStream_t st);
int acco_rope_pack_bwd(const void* dq, const void* dk, const void* dv, const long long* strides, void* dqkv, const float* cos_t,
                       const float* sin_t, int B, int S, int Hq, int Hk, int D, int sms, cudaStream_t st);
int acco_rope_qkv(void* qkv, const float* cos_t, const float* sin_t, int T, int S, int n_rot, int n_total, int D, int inverse,
                  int sms, cudaStream_t st);
int acco_swiglu_fwd(const void* gu, void* out, long long T, int I, int sms, cudaStream_t st);
int acco_swiglu_bwd(const void* dout, const void* gu, void* dgu, long long T, int I, int sms, cudaStream_t st);
int acco_ce_fwd(const void* logits, const long long* labels, float* lse, float* row_loss, float* loss, float* inv_n, long long T,
                int V, int Vp, long long ignore_index, float label_smoothing, float z_loss, float* z_out, cudaStream_t st);
int acco_ce_bwd(void* logits, const long long* labels, const float* lse, const float* scale, long long T, int V, int Vp,
                long long ignore_index, float label_smoothing, float z_loss, cudaStream_t st);
int acco_kd_fwd(const void* student, const void* teacher, const long long* labels, float* lse3, float* rows, float* loss, float* inv_n,
                float* out, long long T, int V, int Vp, long long ignore_index, float alpha, float temperature, cudaStream_t st);
int acco_kd_bwd(void* student, const void* teacher, const long long* labels, const float* lse3, const float* scale, long long T, int V, int Vp,
                long long ignore_index, float alpha, float temperature, cudaStream_t st);
int acco_dpo_fwd(const void* policy, const void* ref, const long long* labels, float* lse, float* d, float* rowbuf, float* w, float* loss,
                 float* out, int P, int S, int V, int Vp, long long ignore_index, float beta, cudaStream_t st);
int acco_pref_fwd(const void* logits, const long long* labels, float* lse, float* row_loss, float* rowbuf, float* w, float* loss, float* out,
                  int P, int S, int V, int Vp, long long ignore_index, int orpo, float coef, float gamma, cudaStream_t st);
int acco_dpo_bwd(void* policy, const long long* labels, const float* lse, const float* w, const float* dloss, int P, int S, int V, int Vp,
                 long long ignore_index, cudaStream_t st);
int acco_norm_bwd_acc_f32(const void* dy, const void* dh_extra, const void* h, const void* w, const float* mean, const float* rstd, void* dh,
                          float* partial, float* dw_accum, float* db_accum, int T, int H, int grid, cudaStream_t st);
int acco_embedding_bwd(void* grad, const long long* sorted, const long long* perm, const void* dy, int T, int H, int sms, cudaStream_t st);
int acco_embedding_bwd_f32(float* grad, const long long* sorted, const long long* perm, const void* dy, int T, int H, int sms, cudaStream_t st);
int acco_gelu_fwd(const void* x, void* y, long long n, int sms, cudaStream_t st);
int acco_gelu_bwd(const void* dy, const void* x, void* dx, long long n, int sms, cudaStream_t st);
int acco_debug_occupy(unsigned long long ns, int ctas, float* sink, cudaStream_t st);
int acco_round_params_size();
int acco_gemm_run(const void* a, long long lda, int a_mn, const void* b, long long ldb, int b_mn, void* d, long long ldd, const void* bias,
                  int M, int N, int K, int accumulate, int bn_req, int splits_req, int pm_req, int pn_req, int msub_req, int sms, cudaStream_t st);
int acco_gemm_tn_gather(const void* x, const void* w_local, void* y, int M, int N, int K, const void* const* peers, int n_peers,
                        const int* tile_owner, uint32_t* flags, uint32_t* epoch, uint32_t* done, int sms, cudaStream_t st);
long long acco_gemm_map_encodes();
int acco_gemm_max_clusters(int cl, int sms);
void acco_gemm_set_debug(unsigned long long* buf);
void acco_gemm_choose(int M, int N, int K, int a_mn, int b_mn, int accumulate, int sms, int* out5);
int acco_gemm_fp8_run(const void* a, long long lda, const void* b, long long ldb, void* d, long long ldd, const void* bias, int M, int N, int K,
                      int accumulate, int a_e5m2, const float* inv_a, const float* inv_b, int bn_req, int splits_req, int sms, cudaStream_t st);
int acco_gemm_wgrad_f32(const void* a, long long lda, const void* b, long long ldb, float* d, long long ldd, int M, int N, int K, int bn_req,
                        int splits_req, int sms, cudaStream_t st);
int acco_gemm_fp8_acc_f32(const void* a, long long lda, const void* b, long long ldb, float* d, long long ldd, int M, int N, int K, int a_e5m2,
                          const float* inv_a, const float* inv_b, int bn_req, int splits_req, int sms, cudaStream_t st);
int acco_fp8_amax_ctas(long long n, int sms);
int acco_fp8_quantize(const void* t, int R, int C, int e5m2, void* q, void* qT, float* scale_out, int ctas, cudaStream_t st);
int acco_gemm_tile_n();
int acco_gemm_tile_k();
int acco_attn_supported(int B, int S, int Hq, int Hk, int D, float scale);
int acco_attn_fwd(const void* q, const void* k, const void* v, long long ld, void* o, long long ld_o, float* lse, int B, int S, int Hq, int Hk,
                  int D, float scale, int window, const int* seg, cudaStream_t st);
int acco_attn_bwd(const void* q, const void* k, const void* v, long long ld, const void* o, long long ld_o, const void* d_o, long long ld_do,
                  const float* lse, float* delta, float* dq_acc, void* dk, void* dv, int B, int S, int Hq, int Hk, int D, float scale, int window,
                  const int* seg, cudaStream_t st);
}

namespace {

constexpr int kMaxWorld = 16;
struct RoundParams {   // must mirror acco::RoundParams in rs_adam_ag.cu
    const void* acc_peer[kMaxWorld];
    void* theta_peer[kMaxWorld];
    uint32_t* pad_peer[kMaxWorld];
    const void* acc_mc;
    void* theta_mc;
    float* master;
    float* exp_avg;
    float* exp_avg_sq;
    float* stash;
    int* stash_count;
    int* total_out;
    uint32_t* epoch;
    uint32_t* done_ctas;
    const float* inv_count_in;
    const long long* skip;
    int n_skip;
    const long long* nodecay;
    int n_nodecay;
    long long nodecay_base;
    int watchdog_s;
    int gated;
    long long slice;
    int rank, world, local_count;
    float lr, beta1, beta2, eps, weight_decay, bc1, bc2_rsqrt;
    int commit, add_stash, write_stash;
};
extern "C" int acco_rs_adam_ag(const RoundParams* P, int grad_bf16, int out_bf16, int mode, int grid, cudaStream_t st);
extern "C" int acco_round_norm(const RoundParams* P, int grad_bf16, int mode, int grid, float max_norm, float* out, cudaStream_t st);

int sm_count() {
    static int n = 0;
    if (!n) n = at::cuda::getCurrentDeviceProperties()->multiProcessorCount;
    return n;
}
cudaStream_t stream() { return at::cuda::getCurrentCUDAStream().stream(); }

void check_bf16(const torch::Tensor& t, const char* name) {
    TORCH_CHECK(t.is_cuda() && t.scalar_type() == torch::kBFloat16 && t.is_contiguous(), name, " must be a contiguous CUDA bf16 tensor");
}
void check_f32(const torch::Tensor& t, const char* name) {
    TORCH_CHECK(t.is_cuda() && t.scalar_type() == torch::kFloat32 && t.is_contiguous(), name, " must be a contiguous CUDA fp32 tensor");
}

// ---------------------------------------------------------------- norms
// RMSNorm when b is undefined, LayerNorm otherwise; r defined: fused residual add.  Returns {y, h = a + r, mean, rstd};
// h is None without r and mean is None for RMSNorm.
std::vector<torch::Tensor> norm_fwd(torch::Tensor a, c10::optional<torch::Tensor> r, torch::Tensor w, c10::optional<torch::Tensor> b,
                                    double eps) {
    check_bf16(a, "a"); check_bf16(w, "weight");
    const bool has_r = r.has_value() && r->defined(), layer = b.has_value() && b->defined();
    if (has_r) check_bf16(*r, "r");
    if (layer) check_bf16(*b, "bias");
    const c10::cuda::CUDAGuard guard(a.device());
    const int T = a.size(0), H = a.size(1);
    TORCH_CHECK(w.numel() == H && (!layer || b->numel() == H), "norm: weight/bias size");
    auto y = torch::empty_like(a);
    auto f32 = a.options().dtype(torch::kFloat32);
    auto rstd = torch::empty({T}, f32);
    torch::Tensor mean = layer ? torch::empty({T}, f32) : torch::Tensor();
    torch::Tensor h = has_r ? torch::empty_like(a) : torch::Tensor();
    const int grid = acco_norm_grid(T, H, sm_count(), 0);
    TORCH_CHECK(acco_norm_fwd(a.data_ptr(), has_r ? r->data_ptr() : nullptr, w.data_ptr(), layer ? b->data_ptr() : nullptr, y.data_ptr(),
                              has_r ? h.data_ptr() : nullptr, layer ? mean.data_ptr<float>() : nullptr, rstd.data_ptr<float>(), T, H,
                              (float)eps, grid, stream()) == 0,
                "norm_fwd: unsupported hidden size ", H);
    return {y, h, mean, rstd};
}

// RMSNorm when mean is undefined, LayerNorm otherwise.  Returns {dh, dwdb}: dwdb is fp32 [H] (dw) or [2H] (dw | db), or
// empty when the parameters' existing bf16 .grad (wgrad, and bgrad for LayerNorm) are given: the sums are then added to them.
std::vector<torch::Tensor> norm_bwd(torch::Tensor dy, c10::optional<torch::Tensor> dh_extra, torch::Tensor h, torch::Tensor w,
                                    c10::optional<torch::Tensor> mean, torch::Tensor rstd, c10::optional<torch::Tensor> wgrad,
                                    c10::optional<torch::Tensor> bgrad) {
    check_bf16(dy, "dy"); check_bf16(h, "h"); check_bf16(w, "weight"); check_f32(rstd, "rstd");
    const bool has_e = dh_extra.has_value() && dh_extra->defined(), layer = mean.has_value() && mean->defined();
    if (has_e) check_bf16(*dh_extra, "dh_extra");
    if (layer) check_f32(*mean, "mean");
    const c10::cuda::CUDAGuard guard(dy.device());
    const int T = dy.size(0), H = dy.size(1), np = layer ? 2 : 1;
    auto dh = torch::empty_like(dy);
    const int grid = acco_norm_grid(T, H, sm_count(), 1);
    auto f32 = dy.options().dtype(torch::kFloat32);
    auto partial = torch::empty({grid, np * H}, f32);
    const bool accum = wgrad.has_value() && wgrad->defined() && (!layer || (bgrad.has_value() && bgrad->defined()));
    torch::Tensor dwdb;
    if (accum) {
        check_bf16(*wgrad, "weight.grad");
        TORCH_CHECK(wgrad->numel() == H, "weight.grad has the wrong size");
        if (layer) {
            check_bf16(*bgrad, "bias.grad");
            TORCH_CHECK(bgrad->numel() == H, "bias.grad has the wrong size");
        }
        dwdb = torch::empty({0}, f32);
    } else {
        dwdb = torch::empty({np * H}, f32);
    }
    TORCH_CHECK(acco_norm_bwd(dy.data_ptr(), has_e ? dh_extra->data_ptr() : nullptr, h.data_ptr(), w.data_ptr(),
                              layer ? mean->data_ptr<float>() : nullptr, rstd.data_ptr<float>(), dh.data_ptr(), partial.data_ptr<float>(),
                              accum ? nullptr : dwdb.data_ptr<float>(), accum ? wgrad->data_ptr() : nullptr,
                              accum && layer ? bgrad->data_ptr() : nullptr, T, H, grid, stream()) == 0,
                "norm_bwd: unsupported hidden size ", H);
    return {dh, dwdb};
}

// As norm_bwd with the dw (| db) sums added to fp32 gradients (fp32 gradient accumulators under bf16 weights): wgrad, and bgrad for
// LayerNorm, are required.  Returns dh.
torch::Tensor norm_bwd_acc_f32(torch::Tensor dy, c10::optional<torch::Tensor> dh_extra, torch::Tensor h, torch::Tensor w,
                               c10::optional<torch::Tensor> mean, torch::Tensor rstd, torch::Tensor wgrad, c10::optional<torch::Tensor> bgrad) {
    check_bf16(dy, "dy"); check_bf16(h, "h"); check_bf16(w, "weight"); check_f32(rstd, "rstd"); check_f32(wgrad, "weight.grad");
    const bool has_e = dh_extra.has_value() && dh_extra->defined(), layer = mean.has_value() && mean->defined();
    if (has_e) check_bf16(*dh_extra, "dh_extra");
    const c10::cuda::CUDAGuard guard(dy.device());
    const int T = dy.size(0), H = dy.size(1), np = layer ? 2 : 1;
    TORCH_CHECK(wgrad.numel() == H, "weight.grad has the wrong size");
    if (layer) {
        check_f32(*mean, "mean");
        TORCH_CHECK(bgrad.has_value() && bgrad->defined(), "norm_bwd_acc_f32: LayerNorm needs bias.grad");
        check_f32(*bgrad, "bias.grad");
        TORCH_CHECK(bgrad->numel() == H, "bias.grad has the wrong size");
    }
    auto dh = torch::empty_like(dy);
    const int grid = acco_norm_grid(T, H, sm_count(), 1);
    auto partial = torch::empty({grid, np * H}, dy.options().dtype(torch::kFloat32));
    TORCH_CHECK(acco_norm_bwd_acc_f32(dy.data_ptr(), has_e ? dh_extra->data_ptr() : nullptr, h.data_ptr(), w.data_ptr(),
                                      layer ? mean->data_ptr<float>() : nullptr, rstd.data_ptr<float>(), dh.data_ptr(), partial.data_ptr<float>(),
                                      wgrad.data_ptr<float>(), layer ? bgrad->data_ptr<float>() : nullptr, T, H, grid, stream()) == 0,
                "norm_bwd_acc_f32: unsupported hidden size ", H);
    return dh;
}

// ---------------------------------------------------------------- gelu (GPT family)
torch::Tensor gelu_fwd(torch::Tensor x) {
    check_bf16(x, "x");
    const c10::cuda::CUDAGuard guard(x.device());
    auto y = torch::empty_like(x);
    TORCH_CHECK(acco_gelu_fwd(x.data_ptr(), y.data_ptr(), x.numel(), sm_count(), stream()) == 0, "gelu: numel must be a multiple of 8");
    return y;
}
torch::Tensor gelu_bwd(torch::Tensor dy, torch::Tensor x) {
    check_bf16(x, "x"); check_bf16(dy, "dy");
    const c10::cuda::CUDAGuard guard(x.device());
    auto dx = torch::empty_like(x);
    TORCH_CHECK(acco_gelu_bwd(dy.data_ptr(), x.data_ptr(), dx.data_ptr(), x.numel(), sm_count(), stream()) == 0, "gelu: numel must be a multiple of 8");
    return dx;
}

// ---------------------------------------------------------------- rope / swiglu
void rope_qkv_inplace(torch::Tensor qkv, torch::Tensor cos_t, torch::Tensor sin_t, int64_t B, int64_t S, int64_t n_rot,
                      int64_t n_total, int64_t D, bool inverse) {
    check_bf16(qkv, "qkv"); check_f32(cos_t, "cos"); check_f32(sin_t, "sin");
    const c10::cuda::CUDAGuard guard(qkv.device());
    TORCH_CHECK(qkv.numel() == B * S * n_total * D, "qkv has the wrong number of elements");
    TORCH_CHECK(cos_t.size(0) >= S && cos_t.size(1) == D / 2, "cos/sin tables must be [>=S, D/2]");
    TORCH_CHECK(acco_rope_qkv(qkv.data_ptr(), cos_t.data_ptr<float>(), sin_t.data_ptr<float>(), (int)(B * S), (int)S, (int)n_rot,
                              (int)n_total, (int)D, inverse ? 1 : 0, sm_count(), stream()) == 0,
                "rope: head_dim must be a multiple of 16");
}

// d(qkv) [B*S, (Hq+2Hk)*D] from the three SDPA gradients (any b/s/h strides, contiguous head dim), inverse RoPE applied.
torch::Tensor rope_pack_bwd(torch::Tensor dq, torch::Tensor dk, torch::Tensor dv, torch::Tensor cos_t, torch::Tensor sin_t) {
    // dq: [B,S,Hq,D] view ; dk, dv: [B,S,Hk,D] views
    TORCH_CHECK(dq.is_cuda() && dq.scalar_type() == torch::kBFloat16 && dk.scalar_type() == torch::kBFloat16 && dv.scalar_type() == torch::kBFloat16, "bf16 CUDA grads expected");
    TORCH_CHECK(dq.stride(3) == 1 && dk.stride(3) == 1 && dv.stride(3) == 1, "head dim must be contiguous");
    check_f32(cos_t, "cos"); check_f32(sin_t, "sin");
    const c10::cuda::CUDAGuard guard(dq.device());
    const int64_t B = dq.size(0), S = dq.size(1), Hq = dq.size(2), D = dq.size(3), Hk = dk.size(2);
    for (auto* t : {&dq, &dk, &dv}) TORCH_CHECK((t->stride(0) % 8 == 0) && (t->stride(1) % 8 == 0) && (t->stride(2) % 8 == 0) && ((uintptr_t)t->data_ptr() % 16 == 0), "16-byte aligned strides required");
    auto out = torch::empty({B * S, (Hq + 2 * Hk) * D}, dq.options());
    long long st[9] = {dq.stride(0), dq.stride(1), dq.stride(2), dk.stride(0), dk.stride(1), dk.stride(2), dv.stride(0), dv.stride(1), dv.stride(2)};
    TORCH_CHECK(acco_rope_pack_bwd(dq.data_ptr(), dk.data_ptr(), dv.data_ptr(), st, out.data_ptr(), cos_t.data_ptr<float>(), sin_t.data_ptr<float>(),
                                   (int)B, (int)S, (int)Hq, (int)Hk, (int)D, sm_count(), stream()) == 0, "rope_pack_bwd: head_dim must be a multiple of 16");
    return out;
}

torch::Tensor swiglu_fwd(torch::Tensor gu) {
    check_bf16(gu, "gate_up");
    const c10::cuda::CUDAGuard guard(gu.device());
    const int64_t T = gu.size(0), I = gu.size(1) / 2;
    auto out = torch::empty({T, I}, gu.options());
    TORCH_CHECK(acco_swiglu_fwd(gu.data_ptr(), out.data_ptr(), T, (int)I, sm_count(), stream()) == 0, "swiglu: I must be a multiple of 8");
    return out;
}

torch::Tensor swiglu_bwd(torch::Tensor dout, torch::Tensor gu) {
    check_bf16(dout, "dout"); check_bf16(gu, "gate_up");
    const c10::cuda::CUDAGuard guard(gu.device());
    const int64_t T = gu.size(0), I = gu.size(1) / 2;
    auto dgu = torch::empty_like(gu);
    TORCH_CHECK(acco_swiglu_bwd(dout.data_ptr(), gu.data_ptr(), dgu.data_ptr(), T, (int)I, sm_count(), stream()) == 0, "swiglu: I must be a multiple of 8");
    return dgu;
}

// ---------------------------------------------------------------- embedding backward
// grad [R, H] += the rows of dy [T, H] scattered by the ids, in place: `sorted` is the stably sorted ids (int64 [T]) and `perm`
// the dy row of each sorted position.  Each row an id hits is read and written once, from an fp32 sum in a fixed order.
void embedding_bwd(torch::Tensor grad, torch::Tensor sorted, torch::Tensor perm, torch::Tensor dy) {
    check_bf16(grad, "grad"); check_bf16(dy, "dy");
    for (auto* t : {&sorted, &perm})
        TORCH_CHECK(t->is_cuda() && t->scalar_type() == torch::kInt64 && t->is_contiguous() && t->numel() == dy.size(0),
                    "sorted ids / permutation must be contiguous CUDA int64 with one entry per dy row");
    TORCH_CHECK(grad.dim() == 2 && dy.dim() == 2 && grad.size(1) == dy.size(1), "grad and dy must be [R, H] and [T, H]");
    TORCH_CHECK(grad.device() == dy.device() && sorted.device() == dy.device() && perm.device() == dy.device(), "tensors on different devices");
    TORCH_CHECK((uintptr_t)grad.data_ptr() % 16 == 0 && (uintptr_t)dy.data_ptr() % 16 == 0, "grad and dy must be 16-byte aligned");
    const c10::cuda::CUDAGuard guard(dy.device());
    TORCH_CHECK(acco_embedding_bwd(grad.data_ptr(), (const long long*)sorted.data_ptr<int64_t>(), (const long long*)perm.data_ptr<int64_t>(),
                                   dy.data_ptr(), (int)dy.size(0), (int)dy.size(1), sm_count(), stream()) == 0,
                "embedding_bwd: hidden size must be a multiple of 8");
}

// As embedding_bwd into fp32 rows: grad [R, H] fp32 (an fp32 gradient accumulator) += the bf16 rows of dy, one fp32 sum per row hit.
void embedding_bwd_f32(torch::Tensor grad, torch::Tensor sorted, torch::Tensor perm, torch::Tensor dy) {
    check_f32(grad, "grad"); check_bf16(dy, "dy");
    for (auto* t : {&sorted, &perm})
        TORCH_CHECK(t->is_cuda() && t->scalar_type() == torch::kInt64 && t->is_contiguous() && t->numel() == dy.size(0),
                    "sorted ids / permutation must be contiguous CUDA int64 with one entry per dy row");
    TORCH_CHECK(grad.dim() == 2 && dy.dim() == 2 && grad.size(1) == dy.size(1), "grad and dy must be [R, H] and [T, H]");
    TORCH_CHECK(grad.device() == dy.device() && sorted.device() == dy.device() && perm.device() == dy.device(), "tensors on different devices");
    TORCH_CHECK((uintptr_t)grad.data_ptr() % 16 == 0 && (uintptr_t)dy.data_ptr() % 16 == 0, "grad and dy must be 16-byte aligned");
    const c10::cuda::CUDAGuard guard(dy.device());
    TORCH_CHECK(acco_embedding_bwd_f32(grad.data_ptr<float>(), (const long long*)sorted.data_ptr<int64_t>(), (const long long*)perm.data_ptr<int64_t>(),
                                       dy.data_ptr(), (int)dy.size(0), (int)dy.size(1), sm_count(), stream()) == 0,
                "embedding_bwd_f32: hidden size must be a multiple of 8");
}

// ---------------------------------------------------------------- cross entropy
void check_label_smoothing(double eps) {
    TORCH_CHECK(std::isfinite(eps) && eps >= 0.0 && eps <= 1.0, "label_smoothing must be finite and in [0, 1], got ", eps);
}

void check_z_loss(double z) {
    TORCH_CHECK(std::isfinite(z) && z >= 0.0 && std::isfinite((float)z), "z_loss must be finite and >= 0, got ", z);
}

// `z_out`: with z_loss > 0, a one-element fp32 tensor on the logits' device that receives the mean z-term (z lse^2 over the
// non-ignored rows); the return value stays (loss, inv_n, lse), with loss = mean CE + that term.
std::vector<torch::Tensor> ce_fwd(torch::Tensor logits, torch::Tensor labels, int64_t V, int64_t ignore_index, double label_smoothing,
                                  double z_loss, c10::optional<torch::Tensor> z_out) {
    check_bf16(logits, "logits");
    check_label_smoothing(label_smoothing);
    check_z_loss(z_loss);
    TORCH_CHECK(labels.is_cuda() && labels.scalar_type() == torch::kInt64 && labels.is_contiguous(), "labels must be contiguous CUDA int64");
    float* z_ptr = nullptr;
    if (z_loss != 0.0) {
        TORCH_CHECK(z_out.has_value(), "ce_fwd: z_loss > 0 needs z_out");
        TORCH_CHECK(z_out->is_cuda() && z_out->device() == logits.device() && z_out->scalar_type() == torch::kFloat32 && z_out->numel() == 1,
                    "z_out must be a one-element fp32 tensor on the logits' device");
        z_ptr = z_out->data_ptr<float>();
    }
    const c10::cuda::CUDAGuard guard(logits.device());
    const int64_t T = logits.size(0), Vp = logits.size(1);
    TORCH_CHECK(labels.numel() == T, "labels/logits row mismatch");
    auto f32 = logits.options().dtype(torch::kFloat32);
    auto lse = torch::empty({T}, f32);
    auto row_loss = torch::empty({T}, f32);
    auto loss = torch::empty({}, f32);
    auto inv_n = torch::empty({1}, f32);
    TORCH_CHECK(acco_ce_fwd(logits.data_ptr(), (const long long*)labels.data_ptr<int64_t>(), lse.data_ptr<float>(), row_loss.data_ptr<float>(),
                            loss.data_ptr<float>(), inv_n.data_ptr<float>(), T, (int)V, (int)Vp, ignore_index, (float)label_smoothing,
                            (float)z_loss, z_ptr, stream()) == 0,
                "ce_fwd: padded vocab must be a multiple of 8 and >= V");
    return {loss, inv_n, lse};
}

void ce_bwd_inplace(torch::Tensor logits, torch::Tensor labels, torch::Tensor lse, torch::Tensor scale, int64_t V, int64_t ignore_index,
                    double label_smoothing, double z_loss) {
    check_bf16(logits, "logits"); check_f32(lse, "lse"); check_f32(scale, "scale");
    check_label_smoothing(label_smoothing);
    check_z_loss(z_loss);
    const c10::cuda::CUDAGuard guard(logits.device());
    const int64_t T = logits.size(0), Vp = logits.size(1);
    TORCH_CHECK(acco_ce_bwd(logits.data_ptr(), (const long long*)labels.data_ptr<int64_t>(), lse.data_ptr<float>(), scale.data_ptr<float>(), T,
                            (int)V, (int)Vp, ignore_index, (float)label_smoothing, (float)z_loss, stream()) == 0, "ce_bwd: bad shapes");
}

// ---------------------------------------------------------------- knowledge distillation
void check_distill(const torch::Tensor& s, const torch::Tensor& t, const torch::Tensor& labels, int64_t V, double alpha, double temperature) {
    check_bf16(s, "logits"); check_bf16(t, "teacher_logits");
    TORCH_CHECK(s.dim() == 2 && t.sizes() == s.sizes() && t.device() == s.device(), "teacher_logits must match the student logits' [T, Vp] shape "
                "and device, got ", t.sizes(), " vs ", s.sizes());
    TORCH_CHECK(labels.is_cuda() && labels.scalar_type() == torch::kInt64 && labels.is_contiguous() && labels.numel() == s.size(0),
                "labels must be contiguous CUDA int64 with one entry per row");
    TORCH_CHECK(s.size(1) % 8 == 0 && V > 0 && V <= s.size(1), "distillation: padded vocab must be a multiple of 8 and >= V, got V=", V,
                " Vp=", s.size(1));
    TORCH_CHECK(std::isfinite(alpha) && alpha > 0.0 && alpha <= 1.0 && (float)alpha > 0.f, "alpha must be in (0, 1], got ", alpha);
    TORCH_CHECK(std::isfinite(temperature) && temperature > 0.0 && std::isfinite((float)temperature) && (float)temperature > 0.f,
                "temperature must be finite and > 0, got ", temperature);
}

// Returns (loss, inv_n, lse3 [3, T]); `out` (two fp32 on the logits' device) receives the mean CE and the mean KL.
std::vector<torch::Tensor> kd_fwd(torch::Tensor logits, torch::Tensor teacher_logits, torch::Tensor labels, int64_t V, int64_t ignore_index,
                                  double alpha, double temperature, torch::Tensor out) {
    check_distill(logits, teacher_logits, labels, V, alpha, temperature);
    TORCH_CHECK(out.is_cuda() && out.device() == logits.device() && out.scalar_type() == torch::kFloat32 && out.numel() == 2 && out.is_contiguous(),
                "out must be a contiguous two-element fp32 tensor on the logits' device");
    const c10::cuda::CUDAGuard guard(logits.device());
    const int64_t T = logits.size(0), Vp = logits.size(1);
    auto f32 = logits.options().dtype(torch::kFloat32);
    auto lse3 = torch::empty({3, T}, f32);
    auto rows = torch::empty({2, T}, f32);
    auto loss = torch::empty({}, f32);
    auto inv_n = torch::empty({1}, f32);
    TORCH_CHECK(acco_kd_fwd(logits.data_ptr(), teacher_logits.data_ptr(), (const long long*)labels.data_ptr<int64_t>(), lse3.data_ptr<float>(),
                            rows.data_ptr<float>(), loss.data_ptr<float>(), inv_n.data_ptr<float>(), out.data_ptr<float>(), T, (int)V, (int)Vp,
                            ignore_index, (float)alpha, (float)temperature, stream()) == 0, "kd_fwd: bad arguments");
    return {loss, inv_n, lse3};
}

void kd_bwd_inplace(torch::Tensor logits, torch::Tensor teacher_logits, torch::Tensor labels, torch::Tensor lse3, torch::Tensor scale, int64_t V,
                    int64_t ignore_index, double alpha, double temperature) {
    check_distill(logits, teacher_logits, labels, V, alpha, temperature);
    check_f32(lse3, "lse3"); check_f32(scale, "scale");
    TORCH_CHECK(lse3.numel() == 3 * logits.size(0), "lse3 must hold 3 x T values");
    const c10::cuda::CUDAGuard guard(logits.device());
    const int64_t T = logits.size(0), Vp = logits.size(1);
    TORCH_CHECK(acco_kd_bwd(logits.data_ptr(), teacher_logits.data_ptr(), (const long long*)labels.data_ptr<int64_t>(), lse3.data_ptr<float>(),
                            scale.data_ptr<float>(), T, (int)V, (int)Vp, ignore_index, (float)alpha, (float)temperature, stream()) == 0,
                "kd_bwd: bad arguments");
}

// ---------------------------------------------------------------- DPO
// logits / ref_logits [2 P S, Vp] bf16, labels [2 P S] int64 (shifted, -100 = not a response token); returns S.
int64_t check_dpo(const torch::Tensor& s, const torch::Tensor& labels, int64_t P, int64_t V) {
    check_bf16(s, "logits");
    TORCH_CHECK(s.dim() == 2 && s.size(1) % 8 == 0 && V > 0 && V <= s.size(1), "dpo: logits must be [T, Vp] with Vp a multiple of 8 and >= V, "
                "got ", s.sizes(), " and V=", V);
    TORCH_CHECK(labels.is_cuda() && labels.device() == s.device() && labels.scalar_type() == torch::kInt64 && labels.is_contiguous() &&
                labels.numel() == s.size(0), "labels must be contiguous CUDA int64 with one entry per row");
    TORCH_CHECK(P > 0 && s.size(0) % (2 * P) == 0 && s.size(0) / (2 * P) <= INT32_MAX && P <= INT32_MAX,
                "dpo: the rows must be 2 P S token rows, got ", s.size(0), " for P=", P);
    return s.size(0) / (2 * P);
}

// Returns (loss, lse [T], w [2P]); `out` (three fp32 on the logits' device) receives the mean chosen reward, the mean rejected reward
// and the accuracy over the valid pairs.
std::vector<torch::Tensor> dpo_fwd(torch::Tensor logits, torch::Tensor ref_logits, torch::Tensor labels, int64_t P, int64_t V,
                                   int64_t ignore_index, double beta, torch::Tensor out) {
    const int64_t S = check_dpo(logits, labels, P, V);
    check_bf16(ref_logits, "ref_logits");
    TORCH_CHECK(ref_logits.sizes() == logits.sizes() && ref_logits.device() == logits.device(), "ref_logits must match the policy logits' "
                "[T, Vp] shape and device, got ", ref_logits.sizes(), " vs ", logits.sizes());
    TORCH_CHECK(std::isfinite(beta) && beta > 0.0 && std::isfinite((float)beta) && (float)beta > 0.f, "beta must be finite and > 0, got ", beta);
    TORCH_CHECK(out.is_cuda() && out.device() == logits.device() && out.scalar_type() == torch::kFloat32 && out.numel() == 3 && out.is_contiguous(),
                "out must be a contiguous three-element fp32 tensor on the logits' device");
    const c10::cuda::CUDAGuard guard(logits.device());
    const int64_t T = logits.size(0), Vp = logits.size(1);
    auto f32 = logits.options().dtype(torch::kFloat32);
    auto lse = torch::empty({T}, f32);
    auto d = torch::empty({T}, f32);
    auto rowbuf = torch::empty({4 * P}, f32);
    auto w = torch::empty({2 * P}, f32);
    auto loss = torch::empty({}, f32);
    TORCH_CHECK(acco_dpo_fwd(logits.data_ptr(), ref_logits.data_ptr(), (const long long*)labels.data_ptr<int64_t>(), lse.data_ptr<float>(),
                             d.data_ptr<float>(), rowbuf.data_ptr<float>(), w.data_ptr<float>(), loss.data_ptr<float>(), out.data_ptr<float>(),
                             (int)P, (int)S, (int)V, (int)Vp, ignore_index, (float)beta, stream()) == 0, "dpo_fwd: bad arguments");
    return {loss, lse, w};
}

// SimPO (orpo false: coef = beta, gamma the margin) or ORPO (orpo true: coef = lambda, gamma unused and 0) over the same pair
// layout as DPO, without reference logits.  Returns (loss, lse [T], w [2P]); `out` (three fp32 on the logits' device) receives SimPO's
// mean chosen reward, mean rejected reward and accuracy, or ORPO's NLL, mean log odds ratio and accuracy.  The backward is
// dpo_bwd_inplace with these w.
std::vector<torch::Tensor> pref_fwd(torch::Tensor logits, torch::Tensor labels, int64_t P, int64_t V, int64_t ignore_index, bool orpo,
                                    double coef, double gamma, torch::Tensor out) {
    const int64_t S = check_dpo(logits, labels, P, V);
    const char* name = orpo ? "lambda" : "beta";
    TORCH_CHECK(std::isfinite(coef) && coef > 0.0 && std::isfinite((float)coef) && (float)coef > 0.f, name, " must be finite and > 0, got ",
                coef);
    TORCH_CHECK(std::isfinite(gamma) && gamma >= 0.0 && std::isfinite((float)gamma) && (!orpo || gamma == 0.0),
                "gamma must be finite and >= 0 (and 0 for ORPO), got ", gamma);
    TORCH_CHECK(out.is_cuda() && out.device() == logits.device() && out.scalar_type() == torch::kFloat32 && out.numel() == 3 && out.is_contiguous(),
                "out must be a contiguous three-element fp32 tensor on the logits' device");
    const c10::cuda::CUDAGuard guard(logits.device());
    const int64_t T = logits.size(0), Vp = logits.size(1);
    auto f32 = logits.options().dtype(torch::kFloat32);
    auto lse = torch::empty({T}, f32);
    auto row_loss = torch::empty({T}, f32);
    auto rowbuf = torch::empty({4 * P}, f32);
    auto w = torch::empty({2 * P}, f32);
    auto loss = torch::empty({}, f32);
    TORCH_CHECK(acco_pref_fwd(logits.data_ptr(), (const long long*)labels.data_ptr<int64_t>(), lse.data_ptr<float>(), row_loss.data_ptr<float>(),
                              rowbuf.data_ptr<float>(), w.data_ptr<float>(), loss.data_ptr<float>(), out.data_ptr<float>(), (int)P, (int)S,
                              (int)V, (int)Vp, ignore_index, orpo ? 1 : 0, (float)coef, (float)gamma, stream()) == 0,
                "pref_fwd: bad arguments");
    return {loss, lse, w};
}

// In place: logits <- dloss w[row] (softmax - onehot) on the response tokens' valid columns, 0 elsewhere.
void dpo_bwd_inplace(torch::Tensor logits, torch::Tensor labels, torch::Tensor lse, torch::Tensor w, torch::Tensor dloss, int64_t P, int64_t V,
                     int64_t ignore_index) {
    const int64_t S = check_dpo(logits, labels, P, V);
    check_f32(lse, "lse"); check_f32(w, "w"); check_f32(dloss, "dloss");
    TORCH_CHECK(lse.numel() == logits.size(0) && w.numel() == 2 * P && dloss.numel() == 1, "lse must hold T values, w 2P and dloss one");
    const c10::cuda::CUDAGuard guard(logits.device());
    TORCH_CHECK(acco_dpo_bwd(logits.data_ptr(), (const long long*)labels.data_ptr<int64_t>(), lse.data_ptr<float>(), w.data_ptr<float>(),
                             dloss.data_ptr<float>(), (int)P, (int)S, (int)V, (int)logits.size(1), ignore_index, stream()) == 0,
                "dpo_bwd: bad arguments");
}

// ---------------------------------------------------------------- fused round kernel
int default_grid(int mode, long long slice) {
    const long long vec = slice / 8;
    long long want = (vec + 255) / 256;
    // comm round: ONE CTA per SM (256 threads x 64 registers).  A GEMM CTA fills its SM's register file, so round CTAs run on the SMs
    // no GEMM CTA holds; more than one per SM would not add bandwidth on the NVLS path.
    long long cap = mode == 0 ? (long long)sm_count() * 4 : (long long)sm_count();
    if (want < 1) want = 1;
    return (int)std::min(want, cap);
}

void fill_hyper(RoundParams& P, double lr, double b1, double b2, double eps, double wd, int64_t step, int64_t commit, bool add_stash, bool write_stash) {
    P.lr = (float)lr; P.beta1 = (float)b1; P.beta2 = (float)b2; P.eps = (float)eps; P.weight_decay = (float)wd;
    P.bc1 = (float)(1.0 - std::pow(b1, (double)step));
    P.bc2_rsqrt = (float)(1.0 / std::sqrt(1.0 - std::pow(b2, (double)step)));
    P.commit = (int)commit; P.add_stash = add_stash ? 1 : 0; P.write_stash = write_stash ? 1 : 0;
}

// No-decay table of a round: sorted, disjoint [lo, hi) ranges of flat parameter indices updated without weight decay, and the flat
// index of the shard's element 0.  The caller guarantees the order (ShardedAdamW.set_no_decay checks it where the table is built):
// checking it here would copy the table to the host on every round.
void set_nodecay(RoundParams& P, const c10::optional<torch::Tensor>& ranges, int64_t base) {
    if (!ranges.has_value() || !ranges->defined() || ranges->numel() == 0) return;
    TORCH_CHECK(ranges->is_cuda() && ranges->scalar_type() == torch::kInt64 && ranges->is_contiguous() && ranges->dim() == 2 && ranges->size(1) == 2,
                "no_decay_ranges must be a contiguous CUDA int64 [n, 2] tensor");
    TORCH_CHECK(base >= 0, "shard_base must not be negative");
    P.nodecay = (const long long*)ranges->data_ptr<int64_t>();
    P.n_nodecay = (int)ranges->size(0);
    P.nodecay_base = base;
}

// The round kernel moves every shard tensor in 16-byte vectors and takes its scalars and counters from device memory.
// The address is taken from the storage: data_ptr() is null for an empty view, wherever it lies.
void check_round_vec(const torch::Tensor& t, const torch::Tensor& master, const char* name) {
    TORCH_CHECK(t.device() == master.device(), name, " must be on the device of master (", master.device(), "), got ", t.device());
    const uintptr_t addr = (uintptr_t)t.storage().data() + (uintptr_t)t.storage_offset() * (uintptr_t)t.element_size();
    TORCH_CHECK(addr % 16 == 0, name, " must be 16-byte aligned");
}
void check_same_device(const torch::Tensor& t, const torch::Tensor& master, const char* name) {
    TORCH_CHECK(t.device() == master.device(), name, " must be on the device of master (", master.device(), "), got ", t.device());
}
void check_moments(const torch::Tensor& exp_avg, const torch::Tensor& exp_avg_sq, int64_t S) {
    TORCH_CHECK(exp_avg.numel() == S && exp_avg_sq.numel() == S, "exp_avg and exp_avg_sq must hold the shard's ", S, " elements, got ",
                exp_avg.numel(), " and ", exp_avg_sq.numel());
}

// Local (single GPU / post-NCCL) sharded AdamW: grad_sum [S] (bf16|fp32) -> out [S] (bf16|fp32)
void adamw_shard(torch::Tensor grad_sum, torch::Tensor master, torch::Tensor exp_avg, torch::Tensor exp_avg_sq, torch::Tensor stash,
                 torch::Tensor out, torch::Tensor inv_count, torch::Tensor scratch /* int32[4]: stash_count,total,epoch,done */,
                 double lr, double b1, double b2, double eps, double wd, int64_t step, int64_t commit, bool add_stash, bool write_stash,
                 c10::optional<torch::Tensor> no_decay_ranges, int64_t shard_base) {
    check_f32(master, "master"); check_f32(exp_avg, "exp_avg"); check_f32(exp_avg_sq, "exp_avg_sq"); check_f32(stash, "stash"); check_f32(inv_count, "inv_count");
    const c10::cuda::CUDAGuard guard(master.device());
    const int64_t S = master.numel();
    TORCH_CHECK(S % 8 == 0, "shard size must be a multiple of 8 (use slice alignment >= 8)");
    TORCH_CHECK(grad_sum.numel() >= S && out.numel() >= S && grad_sum.is_contiguous() && out.is_contiguous(), "bad grad/out");
    check_moments(exp_avg, exp_avg_sq, S);
    TORCH_CHECK(stash.numel() == S, "stash must hold the shard's ", S, " elements, got ", stash.numel());
    check_round_vec(grad_sum, master, "grad_sum"); check_round_vec(master, master, "master"); check_round_vec(exp_avg, master, "exp_avg");
    check_round_vec(exp_avg_sq, master, "exp_avg_sq"); check_round_vec(stash, master, "stash"); check_round_vec(out, master, "out");
    check_same_device(inv_count, master, "inv_count"); check_same_device(scratch, master, "scratch");
    TORCH_CHECK(scratch.scalar_type() == torch::kInt32 && scratch.numel() >= 4, "scratch must be int32[4]");
    const bool gb = grad_sum.scalar_type() == torch::kBFloat16, ob = out.scalar_type() == torch::kBFloat16;
    TORCH_CHECK(gb || grad_sum.scalar_type() == torch::kFloat32, "grad dtype");
    TORCH_CHECK(ob || out.scalar_type() == torch::kFloat32, "out dtype");
    RoundParams P{};
    P.acc_peer[0] = grad_sum.data_ptr();
    P.theta_peer[0] = out.data_ptr();
    P.master = master.data_ptr<float>(); P.exp_avg = exp_avg.data_ptr<float>(); P.exp_avg_sq = exp_avg_sq.data_ptr<float>(); P.stash = stash.data_ptr<float>();
    int* sc = scratch.data_ptr<int>();
    P.stash_count = sc; P.total_out = sc + 1; P.epoch = (uint32_t*)(sc + 2); P.done_ctas = (uint32_t*)(sc + 3);
    P.inv_count_in = inv_count.data_ptr<float>();
    P.slice = S; P.rank = 0; P.world = 1; P.local_count = 0;
    fill_hyper(P, lr, b1, b2, eps, wd, step, commit, add_stash, write_stash);
    set_nodecay(P, no_decay_ranges, shard_base);
    TORCH_CHECK(acco_rs_adam_ag(&P, gb, ob, 0, default_grid(0, S), stream()) == 0, "adamw_shard launch failed");
}

// Transport, counts and barrier state of one round (shared by rs_adam_ag and round_norm).
RoundParams round_params(const std::vector<int64_t>& acc_ptrs, const std::vector<int64_t>& theta_ptrs, const std::vector<int64_t>& pad_ptrs,
                         int64_t acc_mc, int64_t theta_mc, const torch::Tensor& stash, const torch::Tensor& scratch, int64_t slice, int64_t rank,
                         int64_t world, int64_t local_count, int64_t mode) {
    check_f32(stash, "stash");
    TORCH_CHECK(world >= 1 && world <= kMaxWorld, "world size out of range");
    TORCH_CHECK(mode >= 0 && mode <= 2, "mode must be 0 (local), 1 (p2p) or 2 (multimem)");
    TORCH_CHECK((int64_t)acc_ptrs.size() >= (mode == 0 ? 1 : world), "peer pointer table too short");
    TORCH_CHECK(mode == 0 || (int64_t)pad_ptrs.size() >= world, "signal pad table too short");
    TORCH_CHECK(slice % 8 == 0 && stash.numel() == slice, "slice must be a multiple of 8 and match the shard state");
    TORCH_CHECK(mode != 2 || acc_mc != 0, "multicast mode needs multicast pointers");
    TORCH_CHECK(scratch.scalar_type() == torch::kInt32 && scratch.numel() >= 4, "scratch must be int32[4]");
    for (int64_t p : acc_ptrs) TORCH_CHECK(p % 16 == 0, "acc_ptrs must be 16-byte aligned addresses");
    RoundParams P{};
    for (size_t i = 0; i < acc_ptrs.size() && i < (size_t)kMaxWorld; ++i) P.acc_peer[i] = (const void*)acc_ptrs[i];
    for (size_t i = 0; i < theta_ptrs.size() && i < (size_t)kMaxWorld; ++i) P.theta_peer[i] = (void*)theta_ptrs[i];
    for (size_t i = 0; i < pad_ptrs.size() && i < (size_t)kMaxWorld; ++i) P.pad_peer[i] = (uint32_t*)pad_ptrs[i];
    P.acc_mc = (const void*)acc_mc; P.theta_mc = (void*)theta_mc;
    P.stash = stash.data_ptr<float>();
    int* sc = scratch.data_ptr<int>();
    P.stash_count = sc; P.total_out = sc + 1; P.epoch = (uint32_t*)(sc + 2); P.done_ctas = (uint32_t*)(sc + 3);
    P.inv_count_in = nullptr;
    P.slice = slice; P.rank = (int)rank; P.world = (int)world; P.local_count = (int)local_count;
    static int watchdog = -1;
    if (watchdog < 0) { const char* e = std::getenv("ACCO_ROUND_WATCHDOG_S"); watchdog = e ? std::atoi(e) : 1800; }
    P.watchdog_s = watchdog;
    static int gated = -1;
    // default ON: the start barrier runs as a one-warp kernel, so a rank that is ahead of its peers waits with 32 threads instead
    // of a resident grid and its next micro-batches keep the SMs (ACCO_ROUND_GATE=0: barrier inside the round kernel)
    if (gated < 0) { const char* e = std::getenv("ACCO_ROUND_GATE"); gated = (e && e[0] == '0') ? 0 : 1; }
    P.gated = mode != 0 ? gated : 0;
    return P;
}

// Multi-GPU fused round (also valid for world == 1 with mode 0, counts handled in-kernel).
// inv_count: None, or the fp32 scratch of a round_norm launched just before on this stream for the same round.  The update then
// scales the gradient sum by its inv_eff (1/count * clip coefficient), and the start barrier, which round_norm ran, is not repeated.
void rs_adam_ag(std::vector<int64_t> acc_ptrs, std::vector<int64_t> theta_ptrs, std::vector<int64_t> pad_ptrs, int64_t acc_mc, int64_t theta_mc,
                torch::Tensor master, torch::Tensor exp_avg, torch::Tensor exp_avg_sq, torch::Tensor stash,
                torch::Tensor scratch /* int32[4] */, int64_t slice, int64_t rank, int64_t world, int64_t local_count,
                double lr, double b1, double b2, double eps, double wd, int64_t step, int64_t commit, bool add_stash, bool write_stash,
                bool grad_bf16, bool out_bf16, int64_t mode, int64_t grid, c10::optional<torch::Tensor> skip_ranges,
                c10::optional<torch::Tensor> inv_count, c10::optional<torch::Tensor> no_decay_ranges) {
    check_f32(master, "master"); check_f32(exp_avg, "exp_avg"); check_f32(exp_avg_sq, "exp_avg_sq");
    const c10::cuda::CUDAGuard guard(master.device());
    TORCH_CHECK(master.numel() == slice, "slice must match the shard state");
    check_moments(exp_avg, exp_avg_sq, slice);
    check_round_vec(master, master, "master"); check_round_vec(exp_avg, master, "exp_avg"); check_round_vec(exp_avg_sq, master, "exp_avg_sq");
    check_round_vec(stash, master, "stash"); check_same_device(scratch, master, "scratch");
    for (int64_t p : theta_ptrs) TORCH_CHECK(p % 16 == 0, "theta_ptrs must be 16-byte aligned addresses");
    TORCH_CHECK((int64_t)theta_ptrs.size() >= (mode == 0 ? 1 : world), "peer pointer tables too short");
    TORCH_CHECK(mode != 2 || theta_mc != 0, "multicast mode needs multicast pointers");
    RoundParams P = round_params(acc_ptrs, theta_ptrs, pad_ptrs, acc_mc, theta_mc, stash, scratch, slice, rank, world, local_count, mode);
    P.master = master.data_ptr<float>(); P.exp_avg = exp_avg.data_ptr<float>(); P.exp_avg_sq = exp_avg_sq.data_ptr<float>();
    if (skip_ranges.has_value() && skip_ranges->defined() && skip_ranges->numel() > 0) {
        TORCH_CHECK(skip_ranges->is_cuda() && skip_ranges->scalar_type() == torch::kInt64 && skip_ranges->is_contiguous() && skip_ranges->numel() % 2 == 0,
                    "skip_ranges must be a contiguous CUDA int64 [n, 2] tensor");
        P.skip = (const long long*)skip_ranges->data_ptr<int64_t>();
        P.n_skip = (int)(skip_ranges->numel() / 2);
    }
    if (inv_count.has_value() && inv_count->defined()) {
        check_f32(*inv_count, "inv_count");
        check_same_device(*inv_count, master, "inv_count");
        TORCH_CHECK(inv_count->numel() >= 2, "inv_count must be the scratch of round_norm (inv_eff at index 1)");
        P.inv_count_in = inv_count->data_ptr<float>() + 1;
        if (mode != 0) P.gated = 2;
    }
    fill_hyper(P, lr, b1, b2, eps, wd, step, commit, add_stash, write_stash);
    set_nodecay(P, no_decay_ranges, rank * slice);
    const int g = grid > 0 ? (int)grid : default_grid((int)mode, slice);
    TORCH_CHECK(acco_rs_adam_ag(&P, grad_bf16, out_bf16, (int)mode, g, stream()) == 0, "rs_adam_ag launch failed");
}

// Norm pass of a clipped round: reads the round's reduced gradient (+ stash) like rs_adam_ag, runs the start barrier (round gate or
// in-kernel, as rs_adam_ag would) and writes out = {norm, inv_eff, sum of squares, per-CTA partials...} (fp32, >= 3 + grid).  Pass
// `out` to the round's rs_adam_ag as `inv_count`.
void round_norm(std::vector<int64_t> acc_ptrs, std::vector<int64_t> pad_ptrs, int64_t acc_mc, torch::Tensor stash, torch::Tensor scratch,
                torch::Tensor out, int64_t slice, int64_t rank, int64_t world, int64_t local_count, bool add_stash, bool grad_bf16, int64_t mode,
                int64_t grid, double max_norm) {
    check_f32(out, "out");
    const c10::cuda::CUDAGuard guard(stash.device());
    TORCH_CHECK(max_norm > 0, "max_norm must be positive");
    RoundParams P = round_params(acc_ptrs, std::vector<int64_t>(), pad_ptrs, acc_mc, 0, stash, scratch, slice, rank, world, local_count, mode);
    P.add_stash = add_stash ? 1 : 0;
    const int g = grid > 0 ? (int)grid : default_grid((int)mode, slice);
    TORCH_CHECK(out.numel() >= 3 + g, "out must hold 3 + grid floats (", 3 + g, ")");
    TORCH_CHECK(acco_round_norm(&P, grad_bf16, (int)mode, g, (float)max_norm, out.data_ptr<float>(), stream()) == 0, "round_norm launch failed");
}

// ---------------------------------------------------------------- wgmma GEMM (+ fused weight all-gather)
// y[M,N] = x[M,K] @ w[N,K]^T.  With `peer_ptrs` (address of W on every rank), `tile_owner` (int32 [ceil(N/256)]: -1 local,
// r = pull from rank r), `flags` (uint32 [ceil(N/256)*ceil(K/64)*2]) and `state` (int32[2]: epoch, done counter) the weight
// tiles owned by other ranks are gathered over NVLink inside the GEMM and written through to `w`.
torch::Tensor gemm_tn(torch::Tensor x, torch::Tensor w, std::vector<int64_t> peer_ptrs, c10::optional<torch::Tensor> tile_owner,
                      c10::optional<torch::Tensor> flags, c10::optional<torch::Tensor> state, int64_t max_ctas) {
    check_bf16(x, "x"); check_bf16(w, "w");
    TORCH_CHECK(x.dim() == 2 && w.dim() == 2 && x.size(1) == w.size(1), "gemm_tn: x [M,K], w [N,K]");
    const c10::cuda::CUDAGuard guard(x.device());
    const int64_t M = x.size(0), K = x.size(1), N = w.size(0);
    TORCH_CHECK(K % 8 == 0 && N % 8 == 0, "gemm_tn: K and N must be multiples of 8");
    TORCH_CHECK((uintptr_t)x.data_ptr() % 16 == 0 && (uintptr_t)w.data_ptr() % 16 == 0, "gemm_tn: 16-byte aligned operands required");
    auto y = torch::empty({M, N}, x.options());
    const void* peers[8] = {nullptr};
    const int n_peers = (int)peer_ptrs.size();
    TORCH_CHECK(n_peers <= 8, "gemm_tn: at most 8 peers");
    const int* owner = nullptr; uint32_t* fl = nullptr; uint32_t* ep = nullptr; uint32_t* dn = nullptr;
    if (n_peers > 0) {
        TORCH_CHECK(tile_owner.has_value() && flags.has_value() && state.has_value(), "gather mode needs tile_owner, flags and state");
        const int64_t num_n = (N + acco_gemm_tile_n() - 1) / acco_gemm_tile_n(), num_k = (K + acco_gemm_tile_k() - 1) / acco_gemm_tile_k();
        TORCH_CHECK(tile_owner->scalar_type() == torch::kInt32 && tile_owner->numel() >= num_n && tile_owner->is_cuda(), "tile_owner: int32 CUDA [num_n]");
        TORCH_CHECK(flags->scalar_type() == torch::kInt32 && flags->numel() >= num_n * num_k * 2 && flags->is_cuda(), "flags: int32 CUDA [num_n*num_k*2]");
        TORCH_CHECK(state->scalar_type() == torch::kInt32 && state->numel() >= 2 && state->is_cuda(), "state: int32 CUDA [2]");
        for (int i = 0; i < n_peers; ++i) peers[i] = (const void*)peer_ptrs[i];
        owner = tile_owner->data_ptr<int>();
        fl = (uint32_t*)flags->data_ptr<int>();
        ep = (uint32_t*)state->data_ptr<int>();
        dn = ep + 1;
    }
    int sms = sm_count();
    if (max_ctas > 0 && max_ctas < sms) sms = (int)max_ctas;
    int rc;
    if (n_peers > 0)
        rc = acco_gemm_tn_gather(x.data_ptr(), w.data_ptr(), y.data_ptr(), (int)M, (int)N, (int)K, peers, n_peers, owner, fl, ep, dn, sms, stream());
    else
        rc = acco_gemm_run(x.data_ptr(), K, 0, w.data_ptr(), K, 0, y.data_ptr(), N, nullptr, (int)M, (int)N, (int)K, 0, 0, 0, 0, 0, 0, sms, stream());
    TORCH_CHECK(rc == 0, "gemm_tn launch failed, code ", rc);
    return y;
}

// General wgmma GEMM:  out[M,N] (+)= A * B^T (+ bias).
//   a: [M,K] (a_mn = false, K contiguous) or [K,M] (a_mn = true);   b: [N,K] (b_mn = false) or [K,N] (b_mn = true)
//   rows may be strided (stride(0) % 8 == 0, stride(1) == 1).  accumulate: out += (adding epilogue, split-K allowed).
torch::Tensor gemm(torch::Tensor a, torch::Tensor b, c10::optional<torch::Tensor> out, c10::optional<torch::Tensor> bias, bool a_mn, bool b_mn,
                   bool accumulate, int64_t bn, int64_t splits, int64_t pm, int64_t pn, int64_t msub, int64_t max_ctas) {
    auto ok2d = [](const torch::Tensor& t) {
        return t.is_cuda() && t.scalar_type() == torch::kBFloat16 && t.dim() == 2 && t.stride(1) == 1 && t.stride(0) % 8 == 0 && t.stride(0) >= t.size(1) &&
               (uintptr_t)t.data_ptr() % 16 == 0;
    };
    TORCH_CHECK(ok2d(a) && ok2d(b), "gemm: operands must be 2-D CUDA bf16, unit inner stride, 16-byte aligned rows");
    const c10::cuda::CUDAGuard guard(a.device());
    const int64_t M = a_mn ? a.size(1) : a.size(0), K = a_mn ? a.size(0) : a.size(1);
    const int64_t N = b_mn ? b.size(1) : b.size(0), Kb = b_mn ? b.size(0) : b.size(1);
    TORCH_CHECK(K == Kb, "gemm: contraction sizes differ (", K, " vs ", Kb, ")");
    TORCH_CHECK(N % 8 == 0, "gemm: N must be a multiple of 8");
    torch::Tensor y;
    if (out.has_value() && out->defined()) {
        y = *out;
        TORCH_CHECK(ok2d(y) && y.size(0) == M && y.size(1) == N, "gemm: out must be a [M,N] CUDA bf16 matrix");
    } else {
        TORCH_CHECK(!accumulate, "gemm: accumulate needs `out`");
        y = torch::empty({M, N}, a.options());
    }
    const void* bias_p = nullptr;
    if (bias.has_value() && bias->defined()) {
        TORCH_CHECK(bias->is_cuda() && bias->scalar_type() == torch::kBFloat16 && bias->is_contiguous() && bias->numel() == N &&
                    (uintptr_t)bias->data_ptr() % 16 == 0, "gemm: bias must be a contiguous, 16-byte aligned CUDA bf16 [N] vector");
        bias_p = bias->data_ptr();
    }
    int sms = sm_count();
    if (max_ctas > 0 && max_ctas < sms) sms = (int)max_ctas;
    const int rc = acco_gemm_run(a.data_ptr(), a.stride(0), a_mn ? 1 : 0, b.data_ptr(), b.stride(0), b_mn ? 1 : 0, y.data_ptr(), y.stride(0), bias_p,
                             (int)M, (int)N, (int)K, accumulate ? 1 : 0, (int)bn, (int)splits, (int)pm, (int)pn, (int)msub, sms, stream());
    TORCH_CHECK(rc == 0, "gemm launch failed, code ", rc, " (M=", M, " N=", N, " K=", K, ")");
    return y;
}

// wgrad into an fp32 gradient:  out[M,N] += A * B^T with a [K,M] and b [K,N] (both MN-major bf16, rows may be strided as in gemm) and
// out a [M,N] fp32 matrix (unit inner stride, rows 16-byte aligned).  One K split adds exactly; split-K adds fp32 partials through TMA.
void gemm_wgrad_f32(torch::Tensor a, torch::Tensor b, torch::Tensor out, int64_t bn, int64_t splits, int64_t max_ctas) {
    auto ok2d = [](const torch::Tensor& t) {
        return t.is_cuda() && t.scalar_type() == torch::kBFloat16 && t.dim() == 2 && t.stride(1) == 1 && t.stride(0) % 8 == 0 && t.stride(0) >= t.size(1) &&
               (uintptr_t)t.data_ptr() % 16 == 0;
    };
    TORCH_CHECK(ok2d(a) && ok2d(b), "gemm_wgrad_f32: operands must be 2-D CUDA bf16, unit inner stride, 16-byte aligned rows");
    const c10::cuda::CUDAGuard guard(a.device());
    const int64_t M = a.size(1), K = a.size(0), N = b.size(1);
    TORCH_CHECK(b.size(0) == K, "gemm_wgrad_f32: contraction sizes differ (", K, " vs ", b.size(0), ")");
    TORCH_CHECK(N % 8 == 0, "gemm_wgrad_f32: N must be a multiple of 8");
    TORCH_CHECK(out.is_cuda() && out.scalar_type() == torch::kFloat32 && out.dim() == 2 && out.size(0) == M && out.size(1) == N && out.stride(1) == 1 &&
                out.stride(0) % 8 == 0 && out.stride(0) >= N && (uintptr_t)out.data_ptr() % 16 == 0,
                "gemm_wgrad_f32: out must be a [M,N] CUDA fp32 matrix with 16-byte aligned rows");
    int sms = sm_count();
    if (max_ctas > 0 && max_ctas < sms) sms = (int)max_ctas;
    const int rc = acco_gemm_wgrad_f32(a.data_ptr(), a.stride(0), b.data_ptr(), b.stride(0), out.data_ptr<float>(), out.stride(0), (int)M, (int)N,
                                       (int)K, (int)bn, (int)splits, sms, stream());
    TORCH_CHECK(rc == 0, "gemm_wgrad_f32 launch failed, code ", rc, " (M=", M, " N=", N, " K=", K, ")");
}

// ---------------------------------------------------------------- FP8 (per-tensor current scaling)
// t [R, C] bf16 -> {q [R, C] or None, qT [C, R] or None, scale fp32 [3 + ctas] = {s, 1/s, amax, per-CTA maxima...}}; e4m3 or (e5m2) e5m2.
std::vector<torch::Tensor> fp8_quantize(torch::Tensor t, bool e5m2, bool rowmajor, bool transposed) {
    check_bf16(t, "t");
    TORCH_CHECK(t.dim() == 2 && t.size(0) % 16 == 0 && t.size(1) % 16 == 0 && t.numel() > 0, "fp8_quantize: t must be [R, C] with R, C multiples of 16");
    TORCH_CHECK((uintptr_t)t.data_ptr() % 16 == 0, "fp8_quantize: 16-byte aligned input required");
    const c10::cuda::CUDAGuard guard(t.device());
    const int64_t R = t.size(0), C = t.size(1);
    const auto f8 = t.options().dtype(e5m2 ? torch::kFloat8_e5m2 : torch::kFloat8_e4m3fn);
    torch::Tensor q = rowmajor ? torch::empty({R, C}, f8) : torch::Tensor();
    torch::Tensor qT = transposed ? torch::empty({C, R}, f8) : torch::Tensor();
    const int ctas = acco_fp8_amax_ctas(t.numel(), sm_count());
    auto scale = torch::empty({3 + ctas}, t.options().dtype(torch::kFloat32));
    TORCH_CHECK(acco_fp8_quantize(t.data_ptr(), (int)R, (int)C, e5m2 ? 1 : 0, rowmajor ? q.data_ptr() : nullptr, transposed ? qT.data_ptr() : nullptr,
                                  scale.data_ptr<float>(), ctas, stream()) == 0,
                "fp8_quantize launch failed");
    return {q, qT, scale};
}

// out[M,N] (+)= a[M,K] * b[N,K]^T / (s_a s_b) (+ bias).  a: e4m3 or e5m2, b: e4m3, both K-major with 16-byte aligned rows; scale_a / scale_b:
// the scale tensors of fp8_quantize (1/s read on the device).  accumulate: out += (bf16 reduce-add epilogue, split-K allowed).
// max_ctas > 0 caps the persistent grid, as in gemm.
torch::Tensor gemm_fp8(torch::Tensor a, torch::Tensor b, torch::Tensor scale_a, torch::Tensor scale_b, c10::optional<torch::Tensor> out,
                       c10::optional<torch::Tensor> bias, bool accumulate, int64_t bn, int64_t splits, int64_t max_ctas) {
    auto ok2d = [](const torch::Tensor& t) {
        return t.is_cuda() && t.dim() == 2 && t.stride(1) == 1 && t.stride(0) % 16 == 0 && t.stride(0) >= t.size(1) && (uintptr_t)t.data_ptr() % 16 == 0;
    };
    TORCH_CHECK(ok2d(a) && ok2d(b), "gemm_fp8: operands must be 2-D CUDA, unit inner stride, 16-byte aligned rows");
    TORCH_CHECK(a.scalar_type() == torch::kFloat8_e4m3fn || a.scalar_type() == torch::kFloat8_e5m2, "gemm_fp8: a must be e4m3 or e5m2");
    TORCH_CHECK(b.scalar_type() == torch::kFloat8_e4m3fn, "gemm_fp8: b must be e4m3");
    check_f32(scale_a, "scale_a"); check_f32(scale_b, "scale_b");
    TORCH_CHECK(scale_a.numel() >= 2 && scale_b.numel() >= 2, "gemm_fp8: scales must be {s, 1/s, ...}");
    const c10::cuda::CUDAGuard guard(a.device());
    const int64_t M = a.size(0), K = a.size(1), N = b.size(0);
    TORCH_CHECK(b.size(1) == K, "gemm_fp8: contraction sizes differ (", K, " vs ", b.size(1), ")");
    TORCH_CHECK(K % 16 == 0 && N % 8 == 0, "gemm_fp8: K must be a multiple of 16 and N of 8");
    torch::Tensor y;
    if (out.has_value() && out->defined()) {
        y = *out;
        TORCH_CHECK(y.is_cuda() && y.scalar_type() == torch::kBFloat16 && y.dim() == 2 && y.size(0) == M && y.size(1) == N && y.stride(1) == 1 &&
                    y.stride(0) % 8 == 0 && (uintptr_t)y.data_ptr() % 16 == 0, "gemm_fp8: out must be a [M,N] CUDA bf16 matrix with 16-byte aligned rows");
    } else {
        TORCH_CHECK(!accumulate, "gemm_fp8: accumulate needs `out`");
        y = torch::empty({M, N}, a.options().dtype(torch::kBFloat16));
    }
    const void* bias_p = nullptr;
    if (bias.has_value() && bias->defined()) {
        TORCH_CHECK(bias->is_cuda() && bias->scalar_type() == torch::kBFloat16 && bias->is_contiguous() && bias->numel() == N &&
                    (uintptr_t)bias->data_ptr() % 16 == 0, "gemm_fp8: bias must be a contiguous, 16-byte aligned CUDA bf16 [N] vector");
        bias_p = bias->data_ptr();
    }
    int sms = sm_count();
    if (max_ctas > 0 && max_ctas < sms) sms = (int)max_ctas;
    const int rc = acco_gemm_fp8_run(a.data_ptr(), a.stride(0), b.data_ptr(), b.stride(0), y.data_ptr(), y.stride(0), bias_p, (int)M, (int)N, (int)K,
                                     accumulate ? 1 : 0, a.scalar_type() == torch::kFloat8_e5m2 ? 1 : 0, scale_a.data_ptr<float>() + 1,
                                     scale_b.data_ptr<float>() + 1, (int)bn, (int)splits, sms, stream());
    TORCH_CHECK(rc == 0, "gemm_fp8 launch failed, code ", rc, " (M=", M, " N=", N, " K=", K, ")");
    return y;
}

// As gemm_fp8 with accumulate, into an fp32 out [M,N] (an fp32 gradient accumulator): out += a * b^T / (s_a s_b); no bias.
void gemm_fp8_acc_f32(torch::Tensor a, torch::Tensor b, torch::Tensor scale_a, torch::Tensor scale_b, torch::Tensor out, int64_t bn, int64_t splits,
                      int64_t max_ctas) {
    auto ok2d = [](const torch::Tensor& t) {
        return t.is_cuda() && t.dim() == 2 && t.stride(1) == 1 && t.stride(0) % 16 == 0 && t.stride(0) >= t.size(1) && (uintptr_t)t.data_ptr() % 16 == 0;
    };
    TORCH_CHECK(ok2d(a) && ok2d(b), "gemm_fp8_acc_f32: operands must be 2-D CUDA, unit inner stride, 16-byte aligned rows");
    TORCH_CHECK(a.scalar_type() == torch::kFloat8_e4m3fn || a.scalar_type() == torch::kFloat8_e5m2, "gemm_fp8_acc_f32: a must be e4m3 or e5m2");
    TORCH_CHECK(b.scalar_type() == torch::kFloat8_e4m3fn, "gemm_fp8_acc_f32: b must be e4m3");
    check_f32(scale_a, "scale_a"); check_f32(scale_b, "scale_b");
    TORCH_CHECK(scale_a.numel() >= 2 && scale_b.numel() >= 2, "gemm_fp8_acc_f32: scales must be {s, 1/s, ...}");
    const c10::cuda::CUDAGuard guard(a.device());
    const int64_t M = a.size(0), K = a.size(1), N = b.size(0);
    TORCH_CHECK(b.size(1) == K, "gemm_fp8_acc_f32: contraction sizes differ (", K, " vs ", b.size(1), ")");
    TORCH_CHECK(K % 16 == 0 && N % 8 == 0, "gemm_fp8_acc_f32: K must be a multiple of 16 and N of 8");
    TORCH_CHECK(out.is_cuda() && out.scalar_type() == torch::kFloat32 && out.dim() == 2 && out.size(0) == M && out.size(1) == N && out.stride(1) == 1 &&
                out.stride(0) % 8 == 0 && out.stride(0) >= N && (uintptr_t)out.data_ptr() % 16 == 0,
                "gemm_fp8_acc_f32: out must be a [M,N] CUDA fp32 matrix with 16-byte aligned rows");
    int sms = sm_count();
    if (max_ctas > 0 && max_ctas < sms) sms = (int)max_ctas;
    const int rc = acco_gemm_fp8_acc_f32(a.data_ptr(), a.stride(0), b.data_ptr(), b.stride(0), out.data_ptr<float>(), out.stride(0), (int)M, (int)N,
                                         (int)K, a.scalar_type() == torch::kFloat8_e5m2 ? 1 : 0, scale_a.data_ptr<float>() + 1,
                                         scale_b.data_ptr<float>() + 1, (int)bn, (int)splits, sms, stream());
    TORCH_CHECK(rc == 0, "gemm_fp8_acc_f32 launch failed, code ", rc, " (M=", M, " N=", N, " K=", K, ")");
}

// heuristic's pick for a shape: {bn, splits, pm, pn, rows per CTA / 128}
std::vector<int64_t> gemm_choose(int64_t M, int64_t N, int64_t K, bool a_mn, bool b_mn, bool accumulate) {
    int o[5] = {0, 0, 0, 0, 0};
    acco_gemm_choose((int)M, (int)N, (int)K, a_mn ? 1 : 0, b_mn ? 1 : 0, accumulate ? 1 : 0, sm_count(), o);
    return {o[0], o[1], o[2], o[3], o[4]};
}
int64_t gemm_map_encodes() { return acco_gemm_map_encodes(); }
// int64 CUDA tensor of >= 16 elements (or None): CTA 0 of every following GEMM writes %globaltimer stamps of its phases into it
void gemm_set_debug(c10::optional<torch::Tensor> buf) {
    if (buf.has_value() && buf->defined()) {
        TORCH_CHECK(buf->is_cuda() && buf->scalar_type() == torch::kInt64 && buf->numel() >= 16 && buf->is_contiguous(), "int64 CUDA [16] expected");
        acco_gemm_set_debug((unsigned long long*)buf->data_ptr<int64_t>());
    } else {
        acco_gemm_set_debug(nullptr);
    }
}
int64_t gemm_max_clusters(int64_t cl) { return acco_gemm_max_clusters((int)cl, sm_count()); }

int64_t num_sms() { return sm_count(); }

// Experimental (ACCO_CARVEOUT_ALL=1): make "large shared memory" the device-wide default L1 / shared split, so that kernels without an
// explicit preference (elementwise, norms, CE, ATen, cuDNN) use the same carve-out as the wgmma GEMMs and the round kernel and can
// share an SM with them (an SM is only re-partitioned when idle: tools/coresidency_check.py).  Returns the CUDA error code.
int64_t prefer_shared_carveout() { return (int64_t)cudaDeviceSetCacheConfig(cudaFuncCachePreferShared); }

// ---------------------------------------------------------------- flash attention (opt-in: ACCO_ATTN=own)
bool attn_supported(int64_t B, int64_t S, int64_t Hq, int64_t Hk, int64_t D, double scale) {
    return acco_attn_supported((int)B, (int)S, (int)Hq, (int)Hk, (int)D, (float)scale) != 0;
}
static void check_rows(const torch::Tensor& t, int64_t rows, int64_t cols, const char* name) {
    TORCH_CHECK(t.is_cuda() && t.scalar_type() == torch::kBFloat16 && t.dim() == 2 && t.size(0) == rows && t.size(1) == cols && t.stride(1) == 1 &&
                t.stride(0) % 8 == 0 && (uintptr_t)t.data_ptr() % 16 == 0, name, " must be a [", rows, ", ", cols, "] CUDA bf16 matrix with 16-byte aligned rows");
}
// seg: None, or int32 [B*S] per-token segment starts (document masking of packed rows: key kv is visible from query s iff
// seg[s] <= kv <= s; non-decreasing within a row)
static const int* seg_ptr(const c10::optional<torch::Tensor>& seg, int64_t B, int64_t S) {
    if (!seg.has_value() || !seg->defined()) return nullptr;
    TORCH_CHECK(seg->is_cuda() && seg->scalar_type() == torch::kInt32 && seg->is_contiguous() && seg->numel() == B * S,
                "seg must be a contiguous CUDA int32 tensor of B*S segment starts");
    return seg->data_ptr<int>();
}
// qkv [B*S, (Hq + 2 Hk) * D] (rotary embedding already applied) -> {o [B*S, Hq*D] bf16, lse [B, Hq, S] fp32}.  window <= 0: plain causal.
std::vector<torch::Tensor> attn_fwd(torch::Tensor qkv, int64_t B, int64_t S, int64_t Hq, int64_t Hk, int64_t D, double scale, int64_t window,
                                    c10::optional<torch::Tensor> seg) {
    check_rows(qkv, B * S, (Hq + 2 * Hk) * D, "qkv");
    const c10::cuda::CUDAGuard guard(qkv.device());
    auto o = torch::empty({B * S, Hq * D}, qkv.options());
    auto lse = torch::empty({B, Hq, S}, qkv.options().dtype(torch::kFloat32));
    const auto* base = (const char*)qkv.data_ptr();      // bf16: 2 bytes per element
    const int rc = acco_attn_fwd(base, base + 2 * Hq * D, base + 2 * (Hq + Hk) * D, qkv.stride(0), o.data_ptr(), o.stride(0), lse.data_ptr<float>(), (int)B, (int)S,
                                 (int)Hq, (int)Hk, (int)D, (float)scale, (int)window, seg_ptr(seg, B, S), stream());
    TORCH_CHECK(rc == 0, "attn_fwd launch failed, code ", rc, " (B=", B, " S=", S, " Hq=", Hq, " Hk=", Hk, " D=", D, ")");
    return {o, lse};
}
// -> {dq fp32 [B*S, Hq*D], dk bf16 [B*S, Hk*D], dv bf16 [B*S, Hk*D]}
std::vector<torch::Tensor> attn_bwd(torch::Tensor qkv, torch::Tensor o, torch::Tensor d_o, torch::Tensor lse, int64_t B, int64_t S, int64_t Hq, int64_t Hk,
                                    int64_t D, double scale, int64_t window, c10::optional<torch::Tensor> seg) {
    check_rows(qkv, B * S, (Hq + 2 * Hk) * D, "qkv");
    check_rows(o, B * S, Hq * D, "o");
    check_rows(d_o, B * S, Hq * D, "d_o");
    check_f32(lse, "lse");
    TORCH_CHECK(lse.numel() == B * Hq * S, "lse must be [B, Hq, S]");
    const c10::cuda::CUDAGuard guard(qkv.device());
    auto f32 = qkv.options().dtype(torch::kFloat32);
    auto delta = torch::empty({B, Hq, S}, f32);
    auto dq = torch::empty({B * S, Hq * D}, f32);
    auto dk = torch::empty({B * S, Hk * D}, qkv.options());
    auto dv = torch::empty({B * S, Hk * D}, qkv.options());
    const auto* base = (const char*)qkv.data_ptr();
    const int rc = acco_attn_bwd(base, base + 2 * Hq * D, base + 2 * (Hq + Hk) * D, qkv.stride(0), o.data_ptr(), o.stride(0), d_o.data_ptr(), d_o.stride(0),
                                 lse.data_ptr<float>(), delta.data_ptr<float>(), dq.data_ptr<float>(), dk.data_ptr(), dv.data_ptr(), (int)B, (int)S, (int)Hq,
                                 (int)Hk, (int)D, (float)scale, (int)window, seg_ptr(seg, B, S), stream());
    TORCH_CHECK(rc == 0, "attn_bwd launch failed, code ", rc);
    return {dq, dk, dv};
}

// debug: park one 256-thread x ~64-register CTA on `ctas` SMs for `us` microseconds on the current stream
void debug_occupy(double us, int64_t ctas, torch::Tensor sink) {
    check_f32(sink, "sink");
    const c10::cuda::CUDAGuard guard(sink.device());
    TORCH_CHECK(acco_debug_occupy((unsigned long long)(us * 1e3), (int)ctas, sink.data_ptr<float>(), stream()) == 0, "occupy launch failed");
}

}  // namespace

torch::Tensor pack_const_len_native(torch::Tensor flat_tokens, torch::Tensor doc_lens, int64_t max_length, int64_t eos);   // host_data.cpp

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m) {
    TORCH_CHECK(acco_round_params_size() == (int)sizeof(RoundParams), "RoundParams layout mismatch between bindings.cpp and rs_adam_ag.cu");
    m.def("norm_fwd", &norm_fwd);
    m.def("norm_bwd", &norm_bwd);
    m.def("norm_bwd_acc_f32", &norm_bwd_acc_f32);
    m.def("gelu_fwd", &gelu_fwd);
    m.def("gelu_bwd", &gelu_bwd);
    m.def("rope_qkv_inplace", &rope_qkv_inplace);
    m.def("rope_pack_bwd", &rope_pack_bwd);
    m.def("swiglu_fwd", &swiglu_fwd);
    m.def("swiglu_bwd", &swiglu_bwd);
    m.def("embedding_bwd", &embedding_bwd);
    m.def("embedding_bwd_f32", &embedding_bwd_f32);
    m.def("ce_fwd", &ce_fwd, py::arg("logits"), py::arg("labels"), py::arg("V"), py::arg("ignore_index"), py::arg("label_smoothing") = 0.0,
          py::arg("z_loss") = 0.0, py::arg("z_out") = py::none());
    m.def("ce_bwd_inplace", &ce_bwd_inplace, py::arg("logits"), py::arg("labels"), py::arg("lse"), py::arg("scale"), py::arg("V"),
          py::arg("ignore_index"), py::arg("label_smoothing") = 0.0, py::arg("z_loss") = 0.0);
    m.def("kd_fwd", &kd_fwd, py::arg("logits"), py::arg("teacher_logits"), py::arg("labels"), py::arg("V"), py::arg("ignore_index"),
          py::arg("alpha"), py::arg("temperature"), py::arg("out"));
    m.def("dpo_fwd", &dpo_fwd, py::arg("logits"), py::arg("ref_logits"), py::arg("labels"), py::arg("P"), py::arg("V"), py::arg("ignore_index"),
          py::arg("beta"), py::arg("out"));
    m.def("pref_fwd", &pref_fwd, py::arg("logits"), py::arg("labels"), py::arg("P"), py::arg("V"), py::arg("ignore_index"), py::arg("orpo"),
          py::arg("coef"), py::arg("gamma"), py::arg("out"));
    m.def("dpo_bwd_inplace", &dpo_bwd_inplace, py::arg("logits"), py::arg("labels"), py::arg("lse"), py::arg("w"), py::arg("dloss"), py::arg("P"),
          py::arg("V"), py::arg("ignore_index"));
    m.def("kd_bwd_inplace", &kd_bwd_inplace, py::arg("logits"), py::arg("teacher_logits"), py::arg("labels"), py::arg("lse3"), py::arg("scale"),
          py::arg("V"), py::arg("ignore_index"), py::arg("alpha"), py::arg("temperature"));
    m.def("adamw_shard", &adamw_shard, py::arg("grad_sum"), py::arg("master"), py::arg("exp_avg"), py::arg("exp_avg_sq"), py::arg("stash"),
          py::arg("out"), py::arg("inv_count"), py::arg("scratch"), py::arg("lr"), py::arg("b1"), py::arg("b2"), py::arg("eps"), py::arg("wd"),
          py::arg("step"), py::arg("commit"), py::arg("add_stash"), py::arg("write_stash"), py::arg("no_decay_ranges") = py::none(),
          py::arg("shard_base") = 0);
    m.def("rs_adam_ag", &rs_adam_ag, py::arg("acc_ptrs"), py::arg("theta_ptrs"), py::arg("pad_ptrs"), py::arg("acc_mc"), py::arg("theta_mc"),
          py::arg("master"), py::arg("exp_avg"), py::arg("exp_avg_sq"), py::arg("stash"), py::arg("scratch"), py::arg("slice"), py::arg("rank"),
          py::arg("world"), py::arg("local_count"), py::arg("lr"), py::arg("b1"), py::arg("b2"), py::arg("eps"), py::arg("wd"), py::arg("step"),
          py::arg("commit"), py::arg("add_stash"), py::arg("write_stash"), py::arg("grad_bf16"), py::arg("out_bf16"), py::arg("mode"),
          py::arg("grid"), py::arg("skip_ranges"), py::arg("inv_count") = py::none(), py::arg("no_decay_ranges") = py::none());
    m.def("round_norm", &round_norm, py::arg("acc_ptrs"), py::arg("pad_ptrs"), py::arg("acc_mc"), py::arg("stash"), py::arg("scratch"),
          py::arg("out"), py::arg("slice"), py::arg("rank"), py::arg("world"), py::arg("local_count"), py::arg("add_stash"), py::arg("grad_bf16"),
          py::arg("mode"), py::arg("grid"), py::arg("max_norm"));
    m.def("gemm_tn", &gemm_tn);
    m.def("gemm", &gemm);
    m.def("gemm_wgrad_f32", &gemm_wgrad_f32, py::arg("a"), py::arg("b"), py::arg("out"), py::arg("bn") = 0, py::arg("splits") = 0,
          py::arg("max_ctas") = 0);
    m.def("gemm_choose", &gemm_choose);
    m.def("fp8_quantize", &fp8_quantize);
    m.def("gemm_fp8", &gemm_fp8);
    m.def("gemm_fp8_acc_f32", &gemm_fp8_acc_f32, py::arg("a"), py::arg("b"), py::arg("scale_a"), py::arg("scale_b"), py::arg("out"), py::arg("bn") = 0,
          py::arg("splits") = 0, py::arg("max_ctas") = 0);
    m.def("gemm_map_encodes", &gemm_map_encodes);
    m.def("gemm_max_clusters", &gemm_max_clusters);
    m.def("gemm_set_debug", &gemm_set_debug);
    m.def("num_sms", &num_sms);
    m.def("prefer_shared_carveout", &prefer_shared_carveout);
    m.def("attn_supported", &attn_supported);
    m.def("attn_fwd", &attn_fwd, py::arg("qkv"), py::arg("B"), py::arg("S"), py::arg("Hq"), py::arg("Hk"), py::arg("D"), py::arg("scale"),
          py::arg("window"), py::arg("seg") = py::none());
    m.def("attn_bwd", &attn_bwd, py::arg("qkv"), py::arg("o"), py::arg("d_o"), py::arg("lse"), py::arg("B"), py::arg("S"), py::arg("Hq"),
          py::arg("Hk"), py::arg("D"), py::arg("scale"), py::arg("window"), py::arg("seg") = py::none());
    m.def("debug_occupy", &debug_occupy);
    m.def("pack_const_len", &pack_const_len_native);
}
