"""T3: every sm_90a kernel against a plain PyTorch fp32 reference of the same op (run on an H100: `pytest -m gpu`)."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

from acco_b200 import ops
from acco_b200.optim import AdamHyper, ShardedAdamW, adamw_shard_update_
from acco_b200.parallel.schedule import COMMIT_ALL, COMMIT_NONE, COMMIT_STATE

DEV = "cuda"


def bf(*shape, scale=1.0, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(DEV, torch.bfloat16)


def test_extension_is_loaded_and_native():
    C = ops.load_ext(required=True)
    assert C.num_sms() >= 100
    assert ops.ext_path().endswith("_C.so")


@pytest.mark.parametrize("T,H", [(64, 64), (1000, 768), (257, 2048), (33, 4096), (16, 8192), (8, 12288), (64, 100)])
def test_rmsnorm_fwd_bwd(T, H):
    x = bf(T, H, seed=1).requires_grad_(True)
    w = (1 + 0.1 * torch.randn(H)).to(DEV, torch.bfloat16).requires_grad_(True)
    y = ops.rmsnorm(x, w, 1e-5)
    dy = bf(T, H, seed=2)
    y.backward(dy)
    xr = x.detach().float().requires_grad_(True)
    wr = w.detach().float().requires_grad_(True)
    yr = (xr * torch.rsqrt(xr.pow(2).mean(-1, keepdim=True) + 1e-5)) * wr
    yr.backward(dy.float())
    torch.testing.assert_close(y.float(), yr, rtol=2e-2, atol=2e-2)
    torch.testing.assert_close(x.grad.float(), xr.grad, rtol=2e-2, atol=2e-2)
    torch.testing.assert_close(w.grad.float(), wr.grad, rtol=2e-2, atol=0.05 * math.sqrt(T))


@pytest.mark.parametrize("T,H", [(512, 768), (100, 2048)])
def test_add_rmsnorm_fwd_bwd(T, H):
    a = bf(T, H, seed=1).requires_grad_(True)
    r = bf(T, H, seed=2).requires_grad_(True)
    w = (1 + 0.1 * torch.randn(H)).to(DEV, torch.bfloat16).requires_grad_(True)
    y, h = ops.add_rmsnorm(a, r, w, 1e-5)
    dy, dh = bf(T, H, seed=3), bf(T, H, seed=4)
    torch.autograd.backward([y, h], [dy, dh])
    ar, rr, wr = (t.detach().float().requires_grad_(True) for t in (a, r, w))
    hr = (ar + rr).to(torch.bfloat16).float() + 0 * (ar + rr)   # stored-in-bf16 semantics, keep graph
    hr = ar + rr
    yr = hr * torch.rsqrt(hr.pow(2).mean(-1, keepdim=True) + 1e-5) * wr
    torch.autograd.backward([yr, hr], [dy.float(), dh.float()])
    torch.testing.assert_close(h.float(), (ar + rr).detach(), rtol=1e-2, atol=2e-2)
    torch.testing.assert_close(y.float(), yr.detach(), rtol=3e-2, atol=3e-2)
    torch.testing.assert_close(a.grad.float(), ar.grad, rtol=3e-2, atol=3e-2)
    assert torch.equal(a.grad, r.grad)
    torch.testing.assert_close(w.grad.float(), wr.grad, rtol=3e-2, atol=0.05 * math.sqrt(T))


@pytest.mark.parametrize("B,S,Hq,Hk,D", [(2, 128, 12, 12, 64), (1, 77, 8, 2, 128), (3, 16, 4, 2, 16)])
def test_rope_qkv_inplace_and_inverse(B, S, Hq, Hk, D):
    qkv = bf(B * S, (Hq + 2 * Hk) * D, seed=5)
    cos, sin = ops.rope_tables(S, D, 10000.0, DEV)
    ref = ops.rope_qkv_ref(qkv.clone(), cos, sin, B, S, Hq, Hk, D)
    x = qkv.clone().requires_grad_(True)
    out = ops.rope_qkv(x * 1.0, cos, sin, B, S, Hq, Hk, D)
    torch.testing.assert_close(out.float(), ref.float(), rtol=2e-2, atol=2e-2)
    # V heads untouched
    v0 = qkv.view(B, S, Hq + 2 * Hk, D)[:, :, Hq + Hk:]
    assert torch.equal(out.view(B, S, Hq + 2 * Hk, D)[:, :, Hq + Hk:], v0)
    # backward == inverse rotation (orthogonal map): <R x, g> = <x, R^T g>
    g = bf(B * S, (Hq + 2 * Hk) * D, seed=6)
    out.backward(g)
    xr = qkv.float().requires_grad_(True)
    ops.rope_qkv_ref(xr, cos, sin, B, S, Hq, Hk, D).backward(g.float())
    torch.testing.assert_close(x.grad.float(), xr.grad, rtol=2e-2, atol=2e-2)


@pytest.mark.parametrize("B,S,Hq,Hk,D", [(2, 128, 12, 12, 64), (2, 64, 8, 2, 128)])
def test_fused_rope_attention_fwd_bwd(B, S, Hq, Hk, D):
    T = B * S
    qkv0 = bf(T, (Hq + 2 * Hk) * D, seed=11)
    cos, sin = ops.rope_tables(S, D, 10000.0, DEV)
    x = qkv0.clone().requires_grad_(True)
    out = ops.rope_causal_attention(x * 1.0, cos, sin, B, S, Hq, Hk, D)
    g = bf(T, Hq * D, seed=12)
    out.backward(g)
    xr = qkv0.float().requires_grad_(True)
    r = ops.rope_qkv_ref(xr, cos, sin, B, S, Hq, Hk, D).view(B, S, Hq + 2 * Hk, D)
    ref = ops.causal_attention_ref(r[:, :, :Hq], r[:, :, Hq:Hq + Hk], r[:, :, Hq + Hk:]).reshape(T, Hq * D)
    ref.backward(g.float())
    torch.testing.assert_close(out.float(), ref.detach(), rtol=3e-2, atol=3e-2)
    cosim = torch.nn.functional.cosine_similarity(x.grad.float().flatten(), xr.grad.flatten(), dim=0)
    assert cosim > 0.995, float(cosim)
    torch.testing.assert_close(x.grad.float(), xr.grad, rtol=5e-2, atol=5e-2)


def test_norm_weight_grad_accumulates_into_existing_grad():
    T, H = 300, 768
    x = bf(T, H, seed=1).requires_grad_(True)
    w = torch.ones(H, device=DEV, dtype=torch.bfloat16).requires_grad_(True)
    w.grad = torch.full((H,), 2.0, device=DEV, dtype=torch.bfloat16)
    keep = w.grad
    dy = bf(T, H, seed=2)
    ops.rmsnorm(x, w, 1e-5).backward(dy)
    assert w.grad is keep                                    # accumulated in place (fused AccumulateGrad)
    xr = x.detach().float()
    ref = (dy.float() * xr * torch.rsqrt(xr.pow(2).mean(-1, keepdim=True) + 1e-5)).sum(0) + 2.0
    torch.testing.assert_close(w.grad.float(), ref, rtol=2e-2, atol=0.15)


@pytest.mark.parametrize("T,I", [(1000, 2048), (17, 8192), (64, 128)])
def test_swiglu(T, I):
    gu = bf(T, 2 * I, seed=7).requires_grad_(True)
    out = ops.swiglu(gu)
    d = bf(T, I, seed=8)
    out.backward(d)
    gr = gu.detach().float().requires_grad_(True)
    g, u = gr.chunk(2, -1)
    outr = torch.nn.functional.silu(g) * u
    outr.backward(d.float())
    torch.testing.assert_close(out.float(), outr.detach(), rtol=2e-2, atol=2e-2)
    torch.testing.assert_close(gu.grad.float(), gr.grad, rtol=2e-2, atol=2e-2)


@pytest.mark.parametrize("T,V,Vp", [(512, 50257, 50304), (64, 1000, 1000), (33, 131, 136)])
def test_cross_entropy(T, V, Vp):
    logits = bf(T, Vp, scale=2.0, seed=9)
    labels = torch.randint(0, V, (T,), device=DEV)
    labels[::7] = -100
    ref_in = logits.float()[:, :V].clone().requires_grad_(True)
    ref = torch.nn.functional.cross_entropy(ref_in, labels, ignore_index=-100)
    (ref * 3.0).backward()
    x = logits.clone().requires_grad_(True)
    lg = x * 1.0
    loss = ops.softmax_cross_entropy(lg, labels, V, -100)
    (loss * 3.0).backward()
    torch.testing.assert_close(loss, ref.detach(), rtol=2e-3, atol=2e-3)
    torch.testing.assert_close(x.grad.float()[:, :V], ref_in.grad, rtol=3e-2, atol=2e-4)
    assert x.grad[:, V:].abs().sum() == 0 and x.grad[::7].abs().sum() == 0


@pytest.mark.parametrize("gdtype,odtype", [(torch.bfloat16, torch.bfloat16), (torch.float32, torch.float32), (torch.float32, torch.bfloat16)])
@pytest.mark.parametrize("commit,add,write", [(COMMIT_ALL, False, False), (COMMIT_NONE, False, True), (COMMIT_ALL, True, False), (COMMIT_STATE, False, False)])
def test_fused_adamw_matches_reference(gdtype, odtype, commit, add, write):
    S = 8 * 4099
    torch.manual_seed(3)
    p0 = torch.randn(S, device=DEV)
    a, b = ShardedAdamW(p0, 1e-3), ShardedAdamW(p0, 1e-3)
    m0, v0, s0 = torch.randn(S, device=DEV) * 0.1, torch.rand(S, device=DEV) * 0.01, torch.randn(S, device=DEV)
    for o in (a, b):
        o.exp_avg.copy_(m0)
        o.exp_avg_sq.copy_(v0)
        o.stash.copy_(s0)
    g = torch.randn(S, device=DEV).to(gdtype)
    oa, ob = torch.zeros(S, device=DEV, dtype=odtype), torch.zeros(S, device=DEV, dtype=odtype)
    hp = AdamHyper(lr=1e-2, beta1=0.9, beta2=0.95, eps=1e-8, weight_decay=0.1, step=3,
                   inv_count=torch.tensor([0.25], device=DEV), commit=commit, add_stash=add, write_stash=write)
    adamw_shard_update_(g, a.master, a.exp_avg, a.exp_avg_sq, a.stash, oa, hp)
    ops.fused_adamw_shard(g, b.master, b.exp_avg, b.exp_avg_sq, b.stash, ob, hp)
    for x, y in ((a.master, b.master), (a.exp_avg, b.exp_avg), (a.exp_avg_sq, b.exp_avg_sq), (a.stash, b.stash)):
        torch.testing.assert_close(y, x, rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(ob.float(), oa.float(), rtol=1e-2 if odtype == torch.bfloat16 else 1e-5, atol=1e-2 if odtype == torch.bfloat16 else 1e-6)


def test_native_llama_kernels_vs_eager_fp32(monkeypatch):
    """Whole-model check: bf16 kernel path vs the fp32 PyTorch path of the same weights."""
    from acco_b200.models import LlamaConfig, LlamaForCausalLM
    torch.manual_seed(0)
    cfg = LlamaConfig(vocab_size=1000, hidden_size=256, intermediate_size=512, num_hidden_layers=2, num_attention_heads=4,
                      num_key_value_heads=2, max_position_embeddings=128)
    m32 = LlamaForCausalLM(cfg).to(DEV).float()
    m16 = LlamaForCausalLM(cfg).to(DEV)
    m16.load_state_dict(m32.state_dict())
    m16 = m16.to(torch.bfloat16)
    ids = torch.randint(0, 1000, (4, 128), device=DEV)
    before = ops.total_launches()
    l16 = m16(input_ids=ids, labels=ids)[0]
    l16.backward()
    assert ops.total_launches() - before >= 10          # the native kernels really ran
    l32 = m32(input_ids=ids, labels=ids)[0]
    l32.backward()
    assert abs(float(l16) - float(l32)) < 3e-2
    g16 = m16.model.layers[0].mlp.down_proj.grad.float()
    g32 = m32.model.layers[0].mlp.down_proj.grad
    cos = torch.nn.functional.cosine_similarity(g16.flatten(), g32.flatten(), dim=0)
    assert cos > 0.99, float(cos)


def test_trainer_single_gpu_acco_with_graphs(tmp_path, monkeypatch):
    import logging
    from acco_b200 import AttrDict, DecoupledTrainer
    from acco_b200.data import synthetic_pretrain_dataset
    from acco_b200.launch import DistEnv
    from acco_b200.models import LlamaConfig, LlamaForCausalLM
    monkeypatch.chdir(tmp_path)
    torch.manual_seed(0)
    cfg = LlamaConfig(vocab_size=1000, hidden_size=256, intermediate_size=512, num_hidden_layers=2, num_attention_heads=4,
                      num_key_value_heads=4, max_position_embeddings=64)
    ds = synthetic_pretrain_dataset(600, 50, 1000, 64, seed=1)
    losses = {}
    for graphs in (True, False):
        torch.manual_seed(0)
        t = DecoupledTrainer(model=LlamaForCausalLM(cfg), train_dataset=ds,
                             args=AttrDict(method_name="acco", batch_size=8, max_length=64, nb_steps_tot=60, warmup=5, learning_rate=2e-3,
                                           save=False, tensorboard=False, cuda_graphs=graphs, seed=1),
                             log=logging.getLogger("t"), env=DistEnv(id_run="g"))
        ls = []
        while not t.finished():
            t.step()
            ls.append(float(t.loss_host))
        t._drain()
        t._finish("")
        assert t.backend.name == "symm-local"
        assert sum(ls[-5:]) / 5 < sum(ls[:5]) / 5 - 0.3, ls
        losses[graphs] = ls
    # graph replay and eager execution are the same computation
    assert abs(losses[True][-1] - losses[False][-1]) < 0.15


def test_sft_padded_batches_use_one_graph_per_padded_length(tmp_path, monkeypatch):
    import logging
    from acco_b200 import AttrDict, DecoupledTrainer
    from acco_b200.data import ByteTokenizer, synthetic_sft_dataset
    from acco_b200.launch import DistEnv
    from acco_b200.models import LlamaConfig, LlamaForCausalLM
    monkeypatch.chdir(tmp_path)
    torch.manual_seed(0)
    cfg = LlamaConfig(vocab_size=1000, hidden_size=256, intermediate_size=512, num_hidden_layers=2, num_attention_heads=4,
                      num_key_value_heads=4, max_position_embeddings=256)
    tok = ByteTokenizer()
    tok.pad_token_id = tok.eos_token_id = 999
    ds = synthetic_sft_dataset(400, 90, 999, 256, seed=1)
    t = DecoupledTrainer(model=LlamaForCausalLM(cfg), tokenizer=tok, train_dataset=ds,
                         args=AttrDict(method_name="acco", batch_size=4, n_grad_accumulation=2, max_length=256, nb_steps_tot=40, warmup=0,
                                       learning_rate=1e-3, save=False, tensorboard=False, const_len_batch=False, seed=1),
                         log=logging.getLogger("t"), env=DistEnv(id_run="sft"))
    ls = []
    while not t.finished():
        t.step()
        ls.append(float(t.loss_host))
    t._drain()
    t._finish("")
    assert t._graphs is not None and 1 <= len(t._graphs._graphs) <= 2 * 2 * 4      # (theta,acc) pairs x padded lengths {64,128,192,256}
    assert all(l == l for l in ls) and ls[-1] < ls[0]


@pytest.mark.parametrize("M,N,K", [(128, 256, 64), (256, 512, 128), (1000, 776, 200), (2048, 2304, 768), (4096, 768, 2048), (300, 50304, 768)])
def test_tcgen05_gemm_matches_fp32_reference(M, N, K):
    """KERNEL B (wgmma/TMA GEMM) as a plain GEMM: ragged M/N/K edges are zero-filled by TMA and clipped by the epilogue."""
    from acco_b200.ops.gemm import gemm_tn
    x, w = bf(M, K, seed=21), bf(N, K, seed=22)
    before = ops.launch_counts().get("gemm", 0)
    y = gemm_tn(x, w)
    assert ops.launch_counts().get("gemm", 0) == before + 1
    ref = x.float() @ w.float().t()
    rel = ((y.float() - ref).abs() / (ref.abs() + 1.0)).max()
    assert float(rel) < 1.5e-2, float(rel)
    # deterministic: same inputs -> bit-identical output
    assert torch.equal(y, gemm_tn(x, w))


def test_linear_gather_path_is_plain_gemm_without_remote_tiles():
    """GatherLinearFn with an all-local ownership table == ordinary linear (single GPU sanity of the fused-AG plumbing)."""
    from acco_b200.ops.gemm import GatheredWeight
    N, K, T = 512, 256, 384
    flat = bf(N * K + 4096, seed=30)
    w = flat[1024:1024 + N * K].view(N, K).detach().requires_grad_(True)
    w.grad = torch.zeros_like(w)
    gw = GatheredWeight(N, K, 1024, [flat.data_ptr()], size_slice=flat.numel(), rank=0, device=DEV)
    assert all(o == -1 for o in gw.owners)
    x = bf(T, K, seed=31).requires_grad_(True)
    y = ops.linear(x, w, gathered=gw)
    dy = bf(T, N, seed=32)
    y.backward(dy)
    ref = x.detach().float() @ w.detach().float().t()
    torch.testing.assert_close(y.float(), ref, rtol=2e-2, atol=5e-2)
    torch.testing.assert_close(w.grad.float(), dy.float().t() @ x.detach().float(), rtol=2e-2, atol=0.3)
    torch.testing.assert_close(x.grad.float(), dy.float() @ w.detach().float(), rtol=2e-2, atol=0.3)


def test_gptneo_family_trains_on_gpu_bf16(tmp_path, monkeypatch):
    """The reference's default model family (GPT-Neo: LayerNorm, learned positions, global + 256-window local attention)
    through the trainer on the GPU path."""
    import logging
    from acco_b200 import AttrDict, DecoupledTrainer
    from acco_b200.data import synthetic_pretrain_dataset
    from acco_b200.launch import DistEnv
    from acco_b200.models import GPTConfig, GPTForCausalLM
    monkeypatch.chdir(tmp_path)
    torch.manual_seed(0)
    cfg = GPTConfig(vocab_size=1000, hidden_size=256, num_hidden_layers=4, num_attention_heads=4, max_position_embeddings=128,
                    attention_layers="alternating", window_size=32)
    ds = synthetic_pretrain_dataset(600, 60, 1000, 128, seed=1)
    t = DecoupledTrainer(model=GPTForCausalLM(cfg), train_dataset=ds,
                         args=AttrDict(method_name="acco", batch_size=4, max_length=128, nb_steps_tot=40, warmup=2, learning_rate=2e-3,
                                       save=False, tensorboard=False, seed=1),
                         log=logging.getLogger("t"), env=DistEnv(id_run="neo"))
    ls = []
    while not t.finished():
        t.step()
        ls.append(float(t.loss_host))
    t._drain()
    t._finish("")
    assert all(l == l for l in ls) and sum(ls[-4:]) / 4 < sum(ls[:4]) / 4 - 0.2, ls


def test_graph_capture_failure_falls_back_to_eager(tmp_path, monkeypatch):
    """A model whose forward syncs with the host cannot be captured; the trainer must keep training eagerly."""
    import logging
    from acco_b200 import AttrDict, DecoupledTrainer
    from acco_b200.data import synthetic_pretrain_dataset
    from acco_b200.launch import DistEnv
    from acco_b200.models import LlamaConfig, LlamaForCausalLM
    monkeypatch.chdir(tmp_path)

    class Syncing(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.m = LlamaForCausalLM(LlamaConfig(vocab_size=512, hidden_size=128, intermediate_size=256, num_hidden_layers=1,
                                                  num_attention_heads=2, max_position_embeddings=64))

        def forward(self, input_ids=None, labels=None, **kw):
            out = self.m(input_ids=input_ids, labels=labels)
            _ = float(out[0].detach())          # host sync: illegal during stream capture
            return out

    ds = synthetic_pretrain_dataset(300, 40, 512, 64, seed=1)
    t = DecoupledTrainer(model=Syncing(), train_dataset=ds,
                         args=AttrDict(method_name="acco", batch_size=4, max_length=64, nb_steps_tot=16, warmup=0, learning_rate=1e-3,
                                       save=False, tensorboard=False, seed=1),
                         log=logging.getLogger("t"), env=DistEnv(id_run="nog"))
    t.train()
    assert t._graphs_disabled and t.sched.count_grad_tot >= 16 and float(t.loss_host) == float(t.loss_host)


# ------------------------------------------------------------------------------------------------------------------
# wgmma GEMM: every layout of the training step (forward TN, dgrad NN, wgrad TT + accumulate / split-K), all tile shapes
# ------------------------------------------------------------------------------------------------------------------
def _gemm_operands(layout, M, N, K, seed):
    if layout == "tn":
        return bf(M, K, scale=0.5, seed=seed), bf(N, K, scale=0.5, seed=seed + 1), dict()
    if layout == "nn":
        return bf(M, K, scale=0.5, seed=seed), bf(K, N, scale=0.5, seed=seed + 1), dict(b_mn=True)
    return bf(K, M, scale=0.5, seed=seed), bf(K, N, scale=0.5, seed=seed + 1), dict(a_mn=True, b_mn=True)


def _gemm_ref(layout, a, b):
    af = (a.t() if layout == "tt" else a).float()
    return af @ (b.float() if layout in ("nn", "tt") else b.float().t())


@pytest.mark.parametrize("layout", ["tn", "nn", "tt"])
@pytest.mark.parametrize("M,N,K", [(128, 256, 64), (1000, 776, 200), (520, 136, 72), (2304, 768, 1024), (8192, 768, 768)])
def test_tcgen05_gemm_layouts_vs_fp32(layout, M, N, K):
    """forward (K-major x K-major), dgrad (MN-major B) and wgrad (both operands MN-major) incl. ragged edges, vs fp32 matmul."""
    from acco_b200.ops.gemm import gemm
    a, b, kw = _gemm_operands(layout, M, N, K, seed=40)
    y = gemm(a, b, **kw)
    ref = _gemm_ref(layout, a, b)
    err = float((y.float() - ref).abs().max()) / (float(ref.abs().max()) + 1e-6)
    assert err < 8e-3, err


@pytest.mark.parametrize("layout", ["tn", "nn", "tt"])
@pytest.mark.parametrize("cfg", [dict(bn=64), dict(bn=128), dict(bn=256), dict(bn=128, pm=2), dict(bn=256, pm=2, pn=2),
                                 dict(bn=256, pm=1, pn=2)])
def test_tcgen05_gemm_every_tile_shape(layout, cfg):
    """128 x {64, 128, 256} CTA tiles, clusters with TMA multicast of A along a row / B along a column (odd tile counts -> phantom
    tiles)."""
    from acco_b200.ops.gemm import gemm
    a, b, kw = _gemm_operands(layout, 1304, 776, 328, seed=50)
    y = gemm(a, b, **kw, **cfg)
    ref = _gemm_ref(layout, a, b)
    err = float((y.float() - ref).abs().max()) / (float(ref.abs().max()) + 1e-6)
    assert err < 8e-3, (cfg, err)


@pytest.mark.parametrize("splits", [1, 3, 8])
def test_tcgen05_wgrad_accumulates_into_existing_grad(splits):
    """beta = 1 epilogue (read-modify-write, or atomic adds with split-K) straight into a strided view of a larger buffer."""
    from acco_b200.ops.gemm import gemm
    O, I, T = 768, 520, 2048
    dy, x = bf(T, O, scale=0.5, seed=60), bf(T, I, scale=0.5, seed=61)
    arena = bf(O * I + 64, scale=4.0, seed=62)
    g = arena[32:32 + O * I].view(O, I)
    before = g.float().clone()
    guard = (arena[:32].clone(), arena[32 + O * I:].clone())
    gemm(dy, x, out=g, a_mn=True, b_mn=True, accumulate=True, splits=splits)
    ref = before + dy.float().t() @ x.float()
    err = float((g.float() - ref).abs().max()) / float(ref.abs().max())
    assert err < 2.5e-2, err
    assert torch.equal(arena[:32], guard[0]) and torch.equal(arena[32 + O * I:], guard[1])      # nothing written outside the view


def test_tcgen05_gemm_bias_epilogue_and_linear_autograd():
    """ops.linear on CUDA bf16 = three wgmma GEMM launches (fwd with bias epilogue, dgrad, wgrad accumulate) and matches fp32 autograd."""
    T, I, O = 640, 264, 520
    x = bf(T, I, scale=0.5, seed=70).requires_grad_(True)
    w = bf(O, I, scale=0.5, seed=71).requires_grad_(True)
    b = bf(O, seed=72).requires_grad_(True)
    w.grad = torch.zeros_like(w)
    b.grad = torch.zeros_like(b)
    before = ops.launch_counts().get("gemm", 0)
    y = ops.linear(x, w, b)
    dy = bf(T, O, scale=0.5, seed=73)
    y.backward(dy)
    assert ops.launch_counts().get("gemm", 0) == before + 3
    xr, wr, br = (t.detach().float().requires_grad_(True) for t in (x, w, b))
    yr = torch.nn.functional.linear(xr, wr, br)
    yr.backward(dy.float())
    for got, want in ((y, yr), (x.grad, xr.grad), (w.grad, wr.grad), (b.grad, br.grad)):
        err = float((got.float() - want).abs().max()) / (float(want.abs().max()) + 1e-6)
        assert err < 1e-2, err


def test_tcgen05_tensor_maps_are_cached():
    from acco_b200.ops.gemm import gemm_tn
    C = ops.load_ext(required=True)
    x, w = bf(512, 256, seed=80), bf(384, 256, seed=81)
    out = gemm_tn(x, w)
    n0 = C.gemm_map_encodes()
    for _ in range(5):
        gemm_tn(x, w)
    # the operand maps are reused; only the freshly allocated outputs may need new ones (the caching allocator recycles them)
    assert C.gemm_map_encodes() - n0 <= 5


# ------------------------------------------------------------------------------------------------------------------
# GPT family kernels
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("T,H", [(64, 64), (1000, 768), (257, 1024), (100, 2048), (33, 4096), (16, 8192), (64, 100)])
@pytest.mark.parametrize("residual", [False, True])
def test_layernorm_fwd_bwd(T, H, residual):
    a = bf(T, H, seed=1).requires_grad_(True)
    r = bf(T, H, seed=2).requires_grad_(True) if residual else None
    w = (1 + 0.1 * torch.randn(H)).to(DEV, torch.bfloat16).requires_grad_(True)
    b = (0.1 * torch.randn(H)).to(DEV, torch.bfloat16).requires_grad_(True)
    dy, dh = bf(T, H, seed=3), bf(T, H, seed=4)
    if residual:
        y, h = ops.add_layernorm(a, r, w, b, 1e-5)
        torch.autograd.backward([y, h], [dy, dh])
    else:
        y = ops.layernorm(a, w, b, 1e-5)
        y.backward(dy)
    ar, wr, br = (t.detach().float().requires_grad_(True) for t in (a, w, b))
    if residual:
        rr = r.detach().float().requires_grad_(True)
        hr = ar + rr
        yr = torch.nn.functional.layer_norm(hr, (H,), wr, br, 1e-5)
        torch.autograd.backward([yr, hr], [dy.float(), dh.float()])
        assert torch.equal(a.grad, r.grad)
    else:
        yr = torch.nn.functional.layer_norm(ar, (H,), wr, br, 1e-5)
        yr.backward(dy.float())
    torch.testing.assert_close(y.float(), yr.detach(), rtol=3e-2, atol=3e-2)
    torch.testing.assert_close(a.grad.float(), ar.grad, rtol=3e-2, atol=4e-2)
    torch.testing.assert_close(w.grad.float(), wr.grad, rtol=3e-2, atol=0.06 * math.sqrt(T))
    torch.testing.assert_close(b.grad.float(), br.grad, rtol=3e-2, atol=0.06 * math.sqrt(T))


def test_layernorm_param_grads_accumulate_into_arena_views():
    T, H = 512, 768
    x = bf(T, H, seed=5).requires_grad_(True)
    w = torch.ones(H, device=DEV, dtype=torch.bfloat16, requires_grad=True)
    b = torch.zeros(H, device=DEV, dtype=torch.bfloat16, requires_grad=True)
    w.grad = torch.full_like(w, 2.0)
    b.grad = torch.full_like(b, -1.0)
    dy = bf(T, H, seed=6)
    ops.layernorm(x, w, b, 1e-5).backward(dy)
    xr = x.detach().float()
    xh = (xr - xr.mean(-1, keepdim=True)) * torch.rsqrt(xr.var(-1, unbiased=False, keepdim=True) + 1e-5)
    torch.testing.assert_close(w.grad.float(), 2.0 + (dy.float() * xh).sum(0), rtol=3e-2, atol=1.5)
    torch.testing.assert_close(b.grad.float(), -1.0 + dy.float().sum(0), rtol=3e-2, atol=1.5)


def test_gelu_new_fwd_bwd():
    x = bf(1000, 3072, seed=7).requires_grad_(True)
    dy = bf(1000, 3072, seed=8)
    y = ops.gelu_new(x)
    y.backward(dy)
    xr = x.detach().float().requires_grad_(True)
    yr = torch.nn.functional.gelu(xr, approximate="tanh")
    yr.backward(dy.float())
    torch.testing.assert_close(y.float(), yr.detach(), rtol=2e-2, atol=2e-2)
    torch.testing.assert_close(x.grad.float(), xr.grad, rtol=2e-2, atol=2e-2)


def test_gptneo_shipped_vocab_50257_kernel_path_vs_fp32():
    """The reference's default model with its real vocabulary (50257, not a multiple of 8): the LM head is padded to 50304 rows,
    the CE kernel masks the padding, and the bf16 kernel path tracks the fp32 PyTorch path of the same weights."""
    from acco_b200.models import GPTConfig, GPTForCausalLM
    torch.manual_seed(0)
    cfg = GPTConfig(vocab_size=50257, hidden_size=256, num_hidden_layers=2, num_attention_heads=4, max_position_embeddings=128,
                    attention_layers="alternating", window_size=32)
    m32 = GPTForCausalLM(cfg).to(DEV).float()
    m16 = GPTForCausalLM(cfg).to(DEV)
    m16.load_state_dict(m32.state_dict())
    m16 = m16.to(torch.bfloat16)
    assert m16.transformer.wte.shape[0] == 50304 and m16.state_dict()["transformer.wte.weight"].shape[0] == 50257
    ids = torch.randint(0, 50257, (4, 128), device=DEV)
    before = ops.total_launches()
    l16 = m16(input_ids=ids, labels=ids)[0]
    l16.backward()
    assert ops.total_launches() - before >= 20
    l32 = m32(input_ids=ids, labels=ids)[0]
    l32.backward()
    assert abs(float(l16.detach()) - float(l32.detach())) < 5e-2
    for p16, p32 in ((m16.transformer.h[0].mlp.c_proj.weight, m32.transformer.h[0].mlp.c_proj.weight),
                     (m16.transformer.h[1].attn.attention.qkv_proj, m32.transformer.h[1].attn.attention.qkv_proj),
                     (m16.transformer.h[0].ln_1.bias, m32.transformer.h[0].ln_1.bias)):
        cos = torch.nn.functional.cosine_similarity(p16.grad.float().flatten(), p32.grad.flatten(), dim=0)
        assert cos > 0.98, float(cos)
    assert float(m16.transformer.wte.grad[50257:].abs().max()) == 0.0      # vocabulary padding gets no gradient


_ORACLE_SCRIPT = r"""
import logging, sys, torch
sys.path.insert(0, {root!r})
from acco_b200 import AttrDict, DecoupledTrainer
from acco_b200.data import synthetic_pretrain_dataset
from acco_b200.launch import DistEnv
from acco_b200.models import LlamaConfig, LlamaForCausalLM
cuda = sys.argv[1] == "cuda"
cfg = LlamaConfig(vocab_size=512, hidden_size=128, intermediate_size=256, num_hidden_layers=2, num_attention_heads=4,
                  num_key_value_heads=2, max_position_embeddings=64)
torch.manual_seed(0)
m = LlamaForCausalLM(cfg)
init = {{k: v.detach().float().clone() for k, v in m.state_dict().items()}}
ds = synthetic_pretrain_dataset(400, 80, 512, 64, seed=3)
args = AttrDict(method_name="acco", batch_size=4, max_length=64, nb_steps_tot=24, warmup=2, learning_rate=1e-3, save=False, tensorboard=False,
                seed=1, weight_decay=0.0, use_mixed_precision=cuda)
from acco_b200.launch import discover_env
env = discover_env()
env.id_run = "o"
t = DecoupledTrainer(model=m, train_dataset=ds, args=args, log=logging.getLogger("o"), env=env)
t.train()
torch.save({{"init": init, "final": {{k: v.detach().float().cpu().clone() for k, v in t.model.state_dict().items()}},
            "counts": (t.sched.count_grad_tot, t.sched.opt_steps), "cuda": t.is_cuda}}, sys.argv[2])
"""


def test_trainer_gpu_parameters_track_fp32_cpu_trainer(tmp_path):
    """System-level oracle: N ACCO rounds on the GPU kernel path (bf16, CUDA graphs) vs the same trainer on the CPU in fp32 -
    same init, same data order, same schedule; the PARAMETERS (not just the loss) must agree within bf16 training noise."""
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    script = tmp_path / "oracle.py"
    script.write_text(_ORACLE_SCRIPT.format(root=root))
    outs = {}
    for dev in ("cuda", "cpu"):
        from acco_b200.launch import free_port
        env = {k: v for k, v in os.environ.items() if k not in ("RANK", "WORLD_SIZE", "LOCAL_RANK", "MASTER_ADDR")}
        env["MASTER_PORT"] = str(free_port())          # this pytest process already holds a process group on the default port
        if dev == "cpu":
            env["CUDA_VISIBLE_DEVICES"] = ""
        out = tmp_path / f"{dev}.pt"
        p = subprocess.run([sys.executable, str(script), dev, str(out)], cwd=tmp_path, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                           text=True, timeout=600)
        assert p.returncode == 0, p.stdout[-3000:]
        outs[dev] = torch.load(out, weights_only=False)
    gpu, cpu = outs["cuda"], outs["cpu"]
    assert gpu["cuda"] and not cpu["cuda"]
    assert gpu["counts"] == cpu["counts"]
    for k, ref in cpu["final"].items():
        moved = (ref - cpu["init"][k]).norm()                 # how far training moved this tensor
        err = (gpu["final"][k] - ref).norm()
        assert float(err) <= 0.35 * float(moved) + 2e-2 * float(ref.norm()) + 1e-3, (k, float(err), float(moved))


@pytest.mark.skipif(__import__("os").environ.get("ACCO_ATTN", "").lower() != "own",
                    reason="own flash attention is opt-in: run with ACCO_ATTN=own")
def test_tcgen05_attention_bringup_in_subprocess():
    """Own flash-attention forward / backward vs the fp32 reference (tools/attn_check.py), in a subprocess of its own."""
    import os, subprocess, sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    p = subprocess.run([sys.executable, os.path.join(root, "tools", "attn_check.py"), "--quick"], stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                       text=True, timeout=300)
    assert p.returncode == 0, p.stdout[-3000:]


@pytest.mark.skipif(__import__("os").environ.get("ACCO_ATTN", "").lower() != "own",
                    reason="own flash attention is opt-in: run with ACCO_ATTN=own")
def test_llama_with_own_attention_vs_fp32():
    """Whole model with the own attention kernels on the path (S = 256 = two key blocks, GQA, head_dim 64) vs the fp32 PyTorch
    path of the same weights: loss, and the gradient of the fused QKV weight (which sees dQ, dK, dV through the packed d(qkv))."""
    from acco_b200.models import LlamaConfig, LlamaForCausalLM
    torch.manual_seed(0)
    cfg = LlamaConfig(vocab_size=1000, hidden_size=256, intermediate_size=512, num_hidden_layers=2, num_attention_heads=4,
                      num_key_value_heads=2, max_position_embeddings=256)
    assert cfg.head_dim == 64
    m32 = LlamaForCausalLM(cfg).to(DEV).float()
    m16 = LlamaForCausalLM(cfg).to(DEV)
    m16.load_state_dict(m32.state_dict())
    m16 = m16.to(torch.bfloat16)
    ids = torch.randint(0, 1000, (2, 256), device=DEV)
    ops.reset_launch_counts()
    l16 = m16(input_ids=ids, labels=ids)[0]
    l16.backward()
    counts = ops.launch_counts()
    assert counts.get("attn_fwd", 0) == 2 and counts.get("attn_bwd", 0) == 4, counts      # the own kernels really ran (2 layers)
    l32 = m32(input_ids=ids, labels=ids)[0]
    l32.backward()
    assert abs(float(l16) - float(l32)) < 3e-2
    for name in ("qkv_proj", "o_proj"):
        g16 = getattr(m16.model.layers[0].self_attn, name).grad.float()
        g32 = getattr(m32.model.layers[0].self_attn, name).grad
        cos = torch.nn.functional.cosine_similarity(g16.flatten(), g32.flatten(), dim=0)
        assert cos > 0.99, (name, float(cos))
