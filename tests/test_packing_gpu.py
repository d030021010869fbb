"""Sample packing on the H100: the document-masked (segmented) flash-attention kernels against the fp32 reference, against the
unsegmented kernels on single-sample rows and against ``flash_attn_varlen_func``; a whole model on packed rows against its fp32 CPU
path; the trainer with ``packing=True`` and CUDA graphs."""
import logging
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

from acco_b200 import ops
from acco_b200.ops.attention import causal_attention_ref

from test_packing import random_seg

DEV = "cuda"
D = 64


def _inputs(B, S, Hq, Hk, seed):
    g = torch.Generator().manual_seed(seed)
    qkv = (torch.randn(B * S, (Hq + 2 * Hk) * D, generator=g) * 0.7).to(DEV, torch.bfloat16)
    d_o = (torch.randn(B * S, Hq * D, generator=g) * 0.5).to(DEV, torch.bfloat16)
    return qkv, d_o


@pytest.mark.parametrize("S", [512, 1024])
@pytest.mark.parametrize("Hq,Hk", [(12, 12), (32, 8)])
@pytest.mark.parametrize("window", [0, 256])
def test_segmented_kernels_vs_fp32_reference(S, Hq, Hk, window):
    """Tolerances of tools/attn_check.py: O max abs error 2e-2, dQ / dK / dV max error relative to the largest gradient 3e-2."""
    C = ops.load_ext(required=True)
    B = 2
    qkv, d_o = _inputs(B, S, Hq, Hk, S + Hq + window)
    seg = random_seg(B, S, seed=S + Hq + window).to(DEV)
    sc = 1.0 / math.sqrt(D)
    x = qkv.view(B, S, Hq + 2 * Hk, D)
    q, k, v = (t.float().requires_grad_() for t in (x[:, :, :Hq], x[:, :, Hq:Hq + Hk], x[:, :, Hq + Hk:]))
    ref = causal_attention_ref(q, k, v, scale=sc, window=window or None, seg=seg)
    gq, gk, gv = torch.autograd.grad(ref, (q, k, v), d_o.view(B, S, Hq, D).float())
    o, lse = C.attn_fwd(qkv, B, S, Hq, Hk, D, sc, window, seg)
    dq, dk, dv = C.attn_bwd(qkv, o, d_o, lse, B, S, Hq, Hk, D, sc, window, seg)
    torch.cuda.synchronize()
    assert float((o.view(B, S, Hq, D).float() - ref.detach()).abs().max()) < 2e-2
    assert bool(torch.isfinite(lse).all())
    for name, got, want in (("dq", dq.view(B, S, Hq, D), gq), ("dk", dk.view(B, S, Hk, D).float(), gk), ("dv", dv.view(B, S, Hk, D).float(), gv)):
        rel = float((got - want).abs().max() / want.abs().max())
        assert rel < 3e-2, (name, rel)


@pytest.mark.parametrize("Hq,Hk,window", [(12, 12, 0), (32, 8, 256)])
def test_single_sample_rows_match_the_unsegmented_kernels(Hq, Hk, window):
    """One sample per row (seg = 0): the bound never binds, so the segmented kernels do the unsegmented kernels' work in the same
    order.  dQ is summed with fp32 atomics whose order varies from run to run: equal within reassociation error."""
    C = ops.load_ext(required=True)
    B, S = 2, 1024
    qkv, d_o = _inputs(B, S, Hq, Hk, 7)
    seg = torch.zeros(B * S, dtype=torch.int32, device=DEV)
    sc = 1.0 / math.sqrt(D)
    o0, lse0 = C.attn_fwd(qkv, B, S, Hq, Hk, D, sc, window)
    o1, lse1 = C.attn_fwd(qkv, B, S, Hq, Hk, D, sc, window, seg)
    dq0, dk0, dv0 = C.attn_bwd(qkv, o0, d_o, lse0, B, S, Hq, Hk, D, sc, window)
    dq1, dk1, dv1 = C.attn_bwd(qkv, o1, d_o, lse1, B, S, Hq, Hk, D, sc, window, seg)
    torch.cuda.synchronize()
    assert torch.equal(o0, o1) and torch.equal(lse0, lse1) and torch.equal(dk0, dk1) and torch.equal(dv0, dv1)
    torch.testing.assert_close(dq1, dq0, rtol=1e-5, atol=1e-5 * float(dq0.abs().max()))


@pytest.mark.parametrize("Hq,Hk,window", [(12, 12, 0), (32, 8, 0), (12, 12, 256)])
def test_segmented_kernels_vs_flash_attn_varlen(Hq, Hk, window):
    try:
        from flash_attn import flash_attn_varlen_func
    except Exception as e:  # noqa: BLE001 - any import failure: the cross-check is not available here
        pytest.skip(f"flash_attn does not import: {e}")
    C = ops.load_ext(required=True)
    B, S = 2, 1024
    qkv, d_o = _inputs(B, S, Hq, Hk, 11)
    seg = random_seg(B, S, seed=11)
    starts = [b * S + s for b in range(B) for s in range(S) if s == int(seg[b * S + s])]
    cu = torch.tensor(starts + [B * S], dtype=torch.int32, device=DEV)
    max_len = int((cu[1:] - cu[:-1]).max())
    seg = seg.to(DEV)
    sc = 1.0 / math.sqrt(D)
    o, lse = C.attn_fwd(qkv, B, S, Hq, Hk, D, sc, window, seg)
    dq, dk, dv = C.attn_bwd(qkv, o, d_o, lse, B, S, Hq, Hk, D, sc, window, seg)
    x = qkv.view(B * S, Hq + 2 * Hk, D)
    q, k, v = (t.contiguous().requires_grad_() for t in (x[:, :Hq], x[:, Hq:Hq + Hk], x[:, Hq + Hk:]))
    fo = flash_attn_varlen_func(q, k, v, cu, cu, max_len, max_len, softmax_scale=sc, causal=True,
                                window_size=(window - 1, 0) if window else (-1, -1))
    fq, fk, fv = torch.autograd.grad(fo, (q, k, v), d_o.view(B * S, Hq, D))
    torch.cuda.synchronize()
    assert float((o.view(B * S, Hq, D).float() - fo.float()).abs().max()) < 2e-2
    for name, got, want in (("dq", dq.view(B * S, Hq, D), fq), ("dk", dk.view(B * S, Hk, D), fk), ("dv", dv.view(B * S, Hk, D), fv)):
        rel = float((got.float() - want.float()).abs().max() / want.float().abs().max())
        assert rel < 3e-2, (name, rel)


def _packed_rows(B, S, vocab, seed):
    import numpy as np
    from acco_b200.data import PackedCollator, pack_sft
    rng = np.random.default_rng(seed)
    docs = [rng.integers(0, vocab - 1, size=int(n)).tolist() for n in rng.choice([1, 63, 64, 65, 127, 128, 129, 30, 200], size=4 * B)]
    packed = pack_sft(docs, S)
    rows = [{"input_ids": r, "doc_lens": l} for r, l in zip(packed["input_ids"], packed["doc_lens"])][:B]
    return PackedCollator(vocab - 1, S)(rows)


@pytest.mark.parametrize("family", ["llama", "gptneo"])
def test_whole_model_on_packed_rows_vs_fp32_cpu(family):
    """bf16 kernel path (segmented attention) vs the fp32 CPU path of the same weights and rows: loss within 3e-2, gradients of the
    attention weights with cosine similarity > 0.99 (the tolerances of the whole-model test of the own kernels)."""
    from acco_b200.models import GPTConfig, GPTForCausalLM, LlamaConfig, LlamaForCausalLM
    torch.manual_seed(0)
    if family == "llama":
        cfg = LlamaConfig(vocab_size=1000, hidden_size=256, intermediate_size=512, num_hidden_layers=2, num_attention_heads=4,
                          num_key_value_heads=2, max_position_embeddings=256)
        m32 = LlamaForCausalLM(cfg)
        m16 = LlamaForCausalLM(cfg)
        attn = lambda m: m.model.layers[0].self_attn
        names = ("qkv_proj", "o_proj")
    else:
        cfg = GPTConfig(vocab_size=1000, hidden_size=256, num_hidden_layers=2, num_attention_heads=4, max_position_embeddings=256,
                        attention_layers="alternating", window_size=100)
        m32 = GPTForCausalLM(cfg)
        m16 = GPTForCausalLM(cfg)
        attn = lambda m: m.transformer.h[1].attn.attention                      # the local layer
        names = ("qkv_proj",)
    m16.load_state_dict(m32.state_dict())
    m16 = m16.to(DEV, torch.bfloat16)
    batch = _packed_rows(2, 256, 1000, seed=3)
    ops.reset_launch_counts()
    l16 = m16(**{k: v.to(DEV) for k, v in batch.items()}).loss
    l16.backward()
    counts = ops.launch_counts()
    assert counts.get("attn_fwd_seg", 0) == 2 and counts.get("attn_bwd_seg", 0) == 4, counts
    l32 = m32(**batch).loss
    l32.backward()
    assert abs(float(l16) - float(l32)) < 3e-2, (float(l16), float(l32))
    for name in names:
        g16 = getattr(attn(m16), name).grad.float().cpu()
        g32 = getattr(attn(m32), name).grad
        cos = torch.nn.functional.cosine_similarity(g16.flatten(), g32.flatten(), dim=0)
        assert cos > 0.99, (name, float(cos))


def test_trainer_packing_with_cuda_graphs(tmp_path, monkeypatch):
    from acco_b200 import AttrDict, DecoupledTrainer
    from acco_b200.data import ByteTokenizer, synthetic_sft_dataset
    from acco_b200.launch import DistEnv
    from acco_b200.models import LlamaConfig, LlamaForCausalLM
    monkeypatch.chdir(tmp_path)
    monkeypatch.delenv("ACCO_ATTN", raising=False)
    torch.manual_seed(0)
    cfg = LlamaConfig(vocab_size=1000, hidden_size=256, intermediate_size=512, num_hidden_layers=2, num_attention_heads=4,
                      num_key_value_heads=4, max_position_embeddings=256)
    tok = ByteTokenizer()
    tok.pad_token_id = tok.eos_token_id = 999
    ds = synthetic_sft_dataset(1200, 90, 999, 256, seed=1)
    ops.reset_launch_counts()
    t = DecoupledTrainer(model=LlamaForCausalLM(cfg), tokenizer=tok, train_dataset=ds,
                         args=AttrDict(method_name="acco", batch_size=4, n_grad_accumulation=2, max_length=256, nb_steps_tot=32, warmup=0,
                                       learning_rate=1e-3, save=False, tensorboard=False, const_len_batch=False, packing=True, seed=1),
                         log=logging.getLogger("t"), env=DistEnv(id_run="pack"))
    ls = []
    while not t.finished():
        t.step()
        ls.append(float(t.loss_host))
    t._drain()
    t._finish("")
    keys = list(t._graphs._graphs) if t._graphs is not None else []
    assert keys and not getattr(t, "_graphs_disabled", None)
    assert len({k[:3] for k in keys}) == len(keys) <= 4, keys     # one graph per (parameter, accumulator) buffer pair: one shape
    counts = ops.launch_counts()
    assert counts.get("attn_fwd_seg", 0) > 0 and counts.get("attn_bwd_seg", 0) > 0, counts
    assert t.sched.count_grad_tot >= 30 and all(math.isfinite(x) for x in ls)
    assert sum(ls[-5:]) / 5 < sum(ls[:5]) / 5, ls
