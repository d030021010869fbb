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
int acco_rmsnorm_fwd(const void* a, const void* r, const void* w, void* y, void* h, float* rstd, int T, int H, float eps,
                     int grid, cudaStream_t st);
int acco_rmsnorm_bwd(const void* dy, const void* dh_extra, const void* h, const void* w, const float* rstd, void* dh,
                     float* dw_partial, float* dw_out, void* dw_accum_bf16, int T, int H, int grid, cudaStream_t st);
int acco_rope_pack_bwd(const void* dq, const void* dk, const void* dv, const long long* strides, void* dqkv, const float* cos_t,
                       const float* sin_t, int B, int S, int Hq, int Hk, int D, int sms, cudaStream_t st);
int acco_rope_qkv(void* qkv, const float* cos_t, const float* sin_t, int T, int S, int n_rot, int n_total, int D, int inverse,
                  int sms, cudaStream_t st);
int acco_swiglu_fwd(const void* gu, void* out, long long T, int I, int sms, cudaStream_t st);
int acco_swiglu_bwd(const void* dout, const void* gu, void* dgu, long long T, int I, int sms, cudaStream_t st);
int acco_ce_fwd(const void* logits, const long long* labels, float* lse, float* row_loss, float* loss, float* inv_n, long long T,
                int V, int Vp, long long ignore_index, cudaStream_t st);
int acco_ce_bwd(void* logits, const long long* labels, const float* lse, const float* scale, long long T, int V, int Vp,
                long long ignore_index, cudaStream_t st);
int acco_layernorm_grid(int T, int H, int sms, int backward);
int acco_layernorm_fwd(const void* a, const void* r, const void* w, const void* b, void* y, void* h, float* mean, float* rstd, int T, int H,
                       float eps, int grid, cudaStream_t st);
int acco_layernorm_bwd(const void* dy, const void* dh_extra, const void* h, const void* w, const float* mean, const float* rstd, void* dh,
                       float* partial, float* dwdb_out, void* dw_accum_bf16, void* db_accum_bf16, int T, int H, int grid, cudaStream_t st);
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
int acco_gemm_tile_n();
int acco_gemm_tile_k();
int acco_attn_supported(int B, int S, int Hq, int Hk, int D, float scale);
int acco_attn_fwd(const void* q, const void* k, const void* v, long long ld, void* o, long long ld_o, float* lse, int B, int S, int Hq, int Hk,
                  int D, float scale, int window, cudaStream_t st);
int acco_attn_bwd(const void* q, const void* k, const void* v, long long ld, const void* o, long long ld_o, const void* d_o, long long ld_do,
                  const float* lse, float* delta, float* dq_acc, void* dk, void* dv, int B, int S, int Hq, int Hk, int D, float scale, int window,
                  cudaStream_t st);
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
    int watchdog_s;
    int gated;
    long long slice;
    int rank, world, local_count;
    float lr, beta1, beta2, eps, weight_decay, bc1, bc2_rsqrt;
    int commit, add_stash, write_stash;
};
extern "C" int acco_rs_adam_ag(const RoundParams* P, int grad_bf16, int out_bf16, int mode, int grid, cudaStream_t st);

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
std::vector<torch::Tensor> rmsnorm_fwd(torch::Tensor x, torch::Tensor w, double eps) {
    check_bf16(x, "x"); check_bf16(w, "weight");
    const c10::cuda::CUDAGuard guard(x.device());
    const int T = x.size(0), H = x.size(1);
    auto y = torch::empty_like(x);
    auto rstd = torch::empty({T}, x.options().dtype(torch::kFloat32));
    const int grid = acco_norm_grid(T, H, sm_count(), 0);
    TORCH_CHECK(acco_rmsnorm_fwd(x.data_ptr(), nullptr, w.data_ptr(), y.data_ptr(), nullptr, rstd.data_ptr<float>(), T, H, (float)eps, grid, stream()) == 0,
                "rmsnorm_fwd: unsupported hidden size ", H);
    return {y, rstd};
}

std::vector<torch::Tensor> add_rmsnorm_fwd(torch::Tensor a, torch::Tensor r, torch::Tensor w, double eps) {
    check_bf16(a, "a"); check_bf16(r, "r"); check_bf16(w, "weight");
    const c10::cuda::CUDAGuard guard(a.device());
    const int T = a.size(0), H = a.size(1);
    auto y = torch::empty_like(a);
    auto h = torch::empty_like(a);
    auto rstd = torch::empty({T}, a.options().dtype(torch::kFloat32));
    const int grid = acco_norm_grid(T, H, sm_count(), 0);
    TORCH_CHECK(acco_rmsnorm_fwd(a.data_ptr(), r.data_ptr(), w.data_ptr(), y.data_ptr(), h.data_ptr(), rstd.data_ptr<float>(), T, H, (float)eps, grid, stream()) == 0,
                "add_rmsnorm_fwd: unsupported hidden size ", H);
    return {y, h, rstd};
}

// If `wgrad` (the weight's existing bf16 .grad) is defined, dw is accumulated into it and the returned dw is empty.
std::vector<torch::Tensor> norm_bwd_impl(torch::Tensor dy, const torch::Tensor* de, torch::Tensor h, torch::Tensor w, torch::Tensor rstd,
                                         c10::optional<torch::Tensor> wgrad) {
    check_bf16(dy, "dy"); check_bf16(h, "h"); check_bf16(w, "weight"); check_f32(rstd, "rstd");
    const c10::cuda::CUDAGuard guard(dy.device());
    const int T = dy.size(0), H = dy.size(1);
    auto dh = torch::empty_like(dy);
    const int grid = acco_norm_grid(T, H, sm_count(), 1);
    auto partial = torch::empty({grid, H}, dy.options().dtype(torch::kFloat32));
    torch::Tensor dw;
    void* accum = nullptr;
    if (wgrad.has_value() && wgrad->defined()) {
        check_bf16(*wgrad, "weight.grad");
        TORCH_CHECK(wgrad->numel() == H, "weight.grad has the wrong size");
        accum = wgrad->data_ptr();
        dw = torch::empty({0}, dy.options().dtype(torch::kFloat32));
    } else {
        dw = torch::empty({H}, dy.options().dtype(torch::kFloat32));
    }
    TORCH_CHECK(acco_rmsnorm_bwd(dy.data_ptr(), de ? de->data_ptr() : nullptr, h.data_ptr(), w.data_ptr(), rstd.data_ptr<float>(), dh.data_ptr(),
                                 partial.data_ptr<float>(), accum ? nullptr : dw.data_ptr<float>(), accum, T, H, grid, stream()) == 0,
                "rmsnorm_bwd: unsupported hidden size ", H);
    return {dh, dw};
}
std::vector<torch::Tensor> rmsnorm_bwd(torch::Tensor dy, torch::Tensor x, torch::Tensor w, torch::Tensor rstd, c10::optional<torch::Tensor> wgrad) {
    return norm_bwd_impl(dy, nullptr, x, w, rstd, wgrad);
}
std::vector<torch::Tensor> add_rmsnorm_bwd(torch::Tensor dy, torch::Tensor dh_extra, torch::Tensor h, torch::Tensor w, torch::Tensor rstd,
                                           c10::optional<torch::Tensor> wgrad) {
    check_bf16(dh_extra, "dh_extra");
    return norm_bwd_impl(dy, &dh_extra, h, w, rstd, wgrad);
}

// ---------------------------------------------------------------- layernorm / gelu (GPT family)
// r undefined: plain LayerNorm (returns {y, mean, rstd}); else {y, h = a + r, mean, rstd}
std::vector<torch::Tensor> layernorm_fwd(torch::Tensor a, c10::optional<torch::Tensor> r, torch::Tensor w, torch::Tensor b, double eps) {
    check_bf16(a, "a"); check_bf16(w, "weight"); check_bf16(b, "bias");
    const bool has_r = r.has_value() && r->defined();
    if (has_r) check_bf16(*r, "r");
    const c10::cuda::CUDAGuard guard(a.device());
    const int T = a.size(0), H = a.size(1);
    TORCH_CHECK(w.numel() == H && b.numel() == H, "layernorm: weight/bias size");
    auto y = torch::empty_like(a);
    auto f32 = a.options().dtype(torch::kFloat32);
    auto mean = torch::empty({T}, f32), rstd = torch::empty({T}, f32);
    torch::Tensor h = has_r ? torch::empty_like(a) : torch::Tensor();
    const int grid = acco_layernorm_grid(T, H, sm_count(), 0);
    TORCH_CHECK(acco_layernorm_fwd(a.data_ptr(), has_r ? r->data_ptr() : nullptr, w.data_ptr(), b.data_ptr(), y.data_ptr(), has_r ? h.data_ptr() : nullptr,
                                   mean.data_ptr<float>(), rstd.data_ptr<float>(), T, H, (float)eps, grid, stream()) == 0,
                "layernorm_fwd: unsupported hidden size ", H);
    if (has_r) return {y, h, mean, rstd};
    return {y, mean, rstd};
}

// Returns {dh, dwdb}: dwdb is fp32 [2H] (dw | db), or empty when both bf16 accumulation targets (the parameters' .grad views) are given.
std::vector<torch::Tensor> layernorm_bwd(torch::Tensor dy, c10::optional<torch::Tensor> dh_extra, torch::Tensor h, torch::Tensor w, torch::Tensor mean,
                                         torch::Tensor rstd, c10::optional<torch::Tensor> wgrad, c10::optional<torch::Tensor> bgrad) {
    check_bf16(dy, "dy"); check_bf16(h, "h"); check_bf16(w, "weight"); check_f32(mean, "mean"); check_f32(rstd, "rstd");
    const bool has_e = dh_extra.has_value() && dh_extra->defined();
    if (has_e) check_bf16(*dh_extra, "dh_extra");
    const c10::cuda::CUDAGuard guard(dy.device());
    const int T = dy.size(0), H = dy.size(1);
    auto dh = torch::empty_like(dy);
    const int grid = acco_layernorm_grid(T, H, sm_count(), 1);
    auto f32 = dy.options().dtype(torch::kFloat32);
    auto partial = torch::empty({grid, 2 * H}, f32);
    const bool accum = wgrad.has_value() && wgrad->defined() && bgrad.has_value() && bgrad->defined();
    torch::Tensor dwdb;
    if (accum) {
        check_bf16(*wgrad, "weight.grad"); check_bf16(*bgrad, "bias.grad");
        TORCH_CHECK(wgrad->numel() == H && bgrad->numel() == H, "grad sizes");
        dwdb = torch::empty({0}, f32);
    } else {
        dwdb = torch::empty({2 * H}, f32);
    }
    TORCH_CHECK(acco_layernorm_bwd(dy.data_ptr(), has_e ? dh_extra->data_ptr() : nullptr, h.data_ptr(), w.data_ptr(), mean.data_ptr<float>(),
                                   rstd.data_ptr<float>(), dh.data_ptr(), partial.data_ptr<float>(), accum ? nullptr : dwdb.data_ptr<float>(),
                                   accum ? wgrad->data_ptr() : nullptr, accum ? bgrad->data_ptr() : nullptr, T, H, grid, stream()) == 0,
                "layernorm_bwd: unsupported hidden size ", H);
    return {dh, dwdb};
}

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

// ---------------------------------------------------------------- cross entropy
std::vector<torch::Tensor> ce_fwd(torch::Tensor logits, torch::Tensor labels, int64_t V, int64_t ignore_index) {
    check_bf16(logits, "logits");
    TORCH_CHECK(labels.is_cuda() && labels.scalar_type() == torch::kInt64 && labels.is_contiguous(), "labels must be contiguous CUDA int64");
    const c10::cuda::CUDAGuard guard(logits.device());
    const int64_t T = logits.size(0), Vp = logits.size(1);
    TORCH_CHECK(labels.numel() == T, "labels/logits row mismatch");
    auto f32 = logits.options().dtype(torch::kFloat32);
    auto lse = torch::empty({T}, f32);
    auto row_loss = torch::empty({T}, f32);
    auto loss = torch::empty({}, f32);
    auto inv_n = torch::empty({1}, f32);
    TORCH_CHECK(acco_ce_fwd(logits.data_ptr(), (const long long*)labels.data_ptr<int64_t>(), lse.data_ptr<float>(), row_loss.data_ptr<float>(),
                            loss.data_ptr<float>(), inv_n.data_ptr<float>(), T, (int)V, (int)Vp, ignore_index, stream()) == 0,
                "ce_fwd: padded vocab must be a multiple of 8 and >= V");
    return {loss, inv_n, lse};
}

void ce_bwd_inplace(torch::Tensor logits, torch::Tensor labels, torch::Tensor lse, torch::Tensor scale, int64_t V, int64_t ignore_index) {
    check_bf16(logits, "logits"); check_f32(lse, "lse"); check_f32(scale, "scale");
    const c10::cuda::CUDAGuard guard(logits.device());
    const int64_t T = logits.size(0), Vp = logits.size(1);
    TORCH_CHECK(acco_ce_bwd(logits.data_ptr(), (const long long*)labels.data_ptr<int64_t>(), lse.data_ptr<float>(), scale.data_ptr<float>(), T,
                            (int)V, (int)Vp, ignore_index, stream()) == 0, "ce_bwd: bad shapes");
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

// Local (single GPU / post-NCCL) sharded AdamW: grad_sum [S] (bf16|fp32) -> out [S] (bf16|fp32)
void adamw_shard(torch::Tensor grad_sum, torch::Tensor master, torch::Tensor exp_avg, torch::Tensor exp_avg_sq, torch::Tensor stash,
                 torch::Tensor out, torch::Tensor inv_count, torch::Tensor scratch /* int32[4]: stash_count,total,epoch,done */,
                 double lr, double b1, double b2, double eps, double wd, int64_t step, int64_t commit, bool add_stash, bool write_stash) {
    check_f32(master, "master"); check_f32(exp_avg, "exp_avg"); check_f32(exp_avg_sq, "exp_avg_sq"); check_f32(stash, "stash"); check_f32(inv_count, "inv_count");
    const c10::cuda::CUDAGuard guard(master.device());
    const int64_t S = master.numel();
    TORCH_CHECK(S % 8 == 0, "shard size must be a multiple of 8 (use slice alignment >= 8)");
    TORCH_CHECK(grad_sum.numel() >= S && out.numel() >= S && grad_sum.is_contiguous() && out.is_contiguous(), "bad grad/out");
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
    TORCH_CHECK(acco_rs_adam_ag(&P, gb, ob, 0, default_grid(0, S), stream()) == 0, "adamw_shard launch failed");
}

// Multi-GPU fused round (also valid for world == 1 with mode 0, counts handled in-kernel).
void rs_adam_ag(std::vector<int64_t> acc_ptrs, std::vector<int64_t> theta_ptrs, std::vector<int64_t> pad_ptrs, int64_t acc_mc, int64_t theta_mc,
                torch::Tensor master, torch::Tensor exp_avg, torch::Tensor exp_avg_sq, torch::Tensor stash,
                torch::Tensor scratch /* int32[4] */, int64_t slice, int64_t rank, int64_t world, int64_t local_count,
                double lr, double b1, double b2, double eps, double wd, int64_t step, int64_t commit, bool add_stash, bool write_stash,
                bool grad_bf16, bool out_bf16, int64_t mode, int64_t grid, c10::optional<torch::Tensor> skip_ranges) {
    check_f32(master, "master"); check_f32(exp_avg, "exp_avg"); check_f32(exp_avg_sq, "exp_avg_sq"); check_f32(stash, "stash");
    const c10::cuda::CUDAGuard guard(master.device());
    TORCH_CHECK(world >= 1 && world <= kMaxWorld, "world size out of range");
    TORCH_CHECK((int64_t)acc_ptrs.size() >= (mode == 0 ? 1 : world) && (int64_t)theta_ptrs.size() >= (mode == 0 ? 1 : world), "peer pointer tables too short");
    TORCH_CHECK(mode == 0 || (int64_t)pad_ptrs.size() >= world, "signal pad table too short");
    TORCH_CHECK(slice % 8 == 0 && master.numel() == slice, "slice must be a multiple of 8 and match the shard state");
    TORCH_CHECK(mode != 2 || (acc_mc != 0 && theta_mc != 0), "multicast mode needs multicast pointers");
    TORCH_CHECK(scratch.scalar_type() == torch::kInt32 && scratch.numel() >= 4, "scratch must be int32[4]");
    RoundParams P{};
    for (size_t i = 0; i < acc_ptrs.size() && i < (size_t)kMaxWorld; ++i) P.acc_peer[i] = (const void*)acc_ptrs[i];
    for (size_t i = 0; i < theta_ptrs.size() && i < (size_t)kMaxWorld; ++i) P.theta_peer[i] = (void*)theta_ptrs[i];
    for (size_t i = 0; i < pad_ptrs.size() && i < (size_t)kMaxWorld; ++i) P.pad_peer[i] = (uint32_t*)pad_ptrs[i];
    P.acc_mc = (const void*)acc_mc; P.theta_mc = (void*)theta_mc;
    P.master = master.data_ptr<float>(); P.exp_avg = exp_avg.data_ptr<float>(); P.exp_avg_sq = exp_avg_sq.data_ptr<float>(); P.stash = stash.data_ptr<float>();
    int* sc = scratch.data_ptr<int>();
    P.stash_count = sc; P.total_out = sc + 1; P.epoch = (uint32_t*)(sc + 2); P.done_ctas = (uint32_t*)(sc + 3);
    P.inv_count_in = nullptr;
    if (skip_ranges.has_value() && skip_ranges->defined() && skip_ranges->numel() > 0) {
        TORCH_CHECK(skip_ranges->is_cuda() && skip_ranges->scalar_type() == torch::kInt64 && skip_ranges->is_contiguous() && skip_ranges->numel() % 2 == 0,
                    "skip_ranges must be a contiguous CUDA int64 [n, 2] tensor");
        P.skip = (const long long*)skip_ranges->data_ptr<int64_t>();
        P.n_skip = (int)(skip_ranges->numel() / 2);
    }
    P.slice = slice; P.rank = (int)rank; P.world = (int)world; P.local_count = (int)local_count;
    {
        static int watchdog = -1;
        if (watchdog < 0) { const char* e = std::getenv("ACCO_ROUND_WATCHDOG_S"); watchdog = e ? std::atoi(e) : 1800; }
        P.watchdog_s = watchdog;
        static int gated = -1;
        // default ON: the start barrier runs as a one-warp kernel, so a rank that is ahead of its peers waits with 32 threads instead
        // of a resident grid and its next micro-batches keep the SMs (ACCO_ROUND_GATE=0: barrier inside the round kernel)
        if (gated < 0) { const char* e = std::getenv("ACCO_ROUND_GATE"); gated = (e && e[0] == '0') ? 0 : 1; }
        P.gated = mode != 0 ? gated : 0;
    }
    fill_hyper(P, lr, b1, b2, eps, wd, step, commit, add_stash, write_stash);
    const int g = grid > 0 ? (int)grid : default_grid((int)mode, slice);
    TORCH_CHECK(acco_rs_adam_ag(&P, grad_bf16, out_bf16, (int)mode, g, stream()) == 0, "rs_adam_ag launch failed");
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
// qkv [B*S, (Hq + 2 Hk) * D] (rotary embedding already applied) -> {o [B*S, Hq*D] bf16, lse [B, Hq, S] fp32}.  window <= 0: plain causal.
std::vector<torch::Tensor> attn_fwd(torch::Tensor qkv, int64_t B, int64_t S, int64_t Hq, int64_t Hk, int64_t D, double scale, int64_t window) {
    check_rows(qkv, B * S, (Hq + 2 * Hk) * D, "qkv");
    const c10::cuda::CUDAGuard guard(qkv.device());
    auto o = torch::empty({B * S, Hq * D}, qkv.options());
    auto lse = torch::empty({B, Hq, S}, qkv.options().dtype(torch::kFloat32));
    const auto* base = (const char*)qkv.data_ptr();      // bf16: 2 bytes per element
    const int rc = acco_attn_fwd(base, base + 2 * Hq * D, base + 2 * (Hq + Hk) * D, qkv.stride(0), o.data_ptr(), o.stride(0), lse.data_ptr<float>(), (int)B, (int)S,
                                 (int)Hq, (int)Hk, (int)D, (float)scale, (int)window, stream());
    TORCH_CHECK(rc == 0, "attn_fwd launch failed, code ", rc, " (B=", B, " S=", S, " Hq=", Hq, " Hk=", Hk, " D=", D, ")");
    return {o, lse};
}
// -> {dq fp32 [B*S, Hq*D], dk bf16 [B*S, Hk*D], dv bf16 [B*S, Hk*D]}
std::vector<torch::Tensor> attn_bwd(torch::Tensor qkv, torch::Tensor o, torch::Tensor d_o, torch::Tensor lse, int64_t B, int64_t S, int64_t Hq, int64_t Hk,
                                    int64_t D, double scale, int64_t window) {
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
                                 (int)Hk, (int)D, (float)scale, (int)window, stream());
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
    m.def("rmsnorm_fwd", &rmsnorm_fwd);
    m.def("rmsnorm_bwd", &rmsnorm_bwd);
    m.def("add_rmsnorm_fwd", &add_rmsnorm_fwd);
    m.def("add_rmsnorm_bwd", &add_rmsnorm_bwd);
    m.def("layernorm_fwd", &layernorm_fwd);
    m.def("layernorm_bwd", &layernorm_bwd);
    m.def("gelu_fwd", &gelu_fwd);
    m.def("gelu_bwd", &gelu_bwd);
    m.def("rope_qkv_inplace", &rope_qkv_inplace);
    m.def("rope_pack_bwd", &rope_pack_bwd);
    m.def("swiglu_fwd", &swiglu_fwd);
    m.def("swiglu_bwd", &swiglu_bwd);
    m.def("ce_fwd", &ce_fwd);
    m.def("ce_bwd_inplace", &ce_bwd_inplace);
    m.def("adamw_shard", &adamw_shard);
    m.def("rs_adam_ag", &rs_adam_ag);
    m.def("gemm_tn", &gemm_tn);
    m.def("gemm", &gemm);
    m.def("gemm_choose", &gemm_choose);
    m.def("gemm_map_encodes", &gemm_map_encodes);
    m.def("gemm_max_clusters", &gemm_max_clusters);
    m.def("gemm_set_debug", &gemm_set_debug);
    m.def("num_sms", &num_sms);
    m.def("prefer_shared_carveout", &prefer_shared_carveout);
    m.def("attn_supported", &attn_supported);
    m.def("attn_fwd", &attn_fwd);
    m.def("attn_bwd", &attn_bwd);
    m.def("debug_occupy", &debug_occupy);
    m.def("pack_const_len", &pack_const_len_native);
}
