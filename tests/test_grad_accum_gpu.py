"""fp32 gradient accumulators under bf16 weights (train key ``grad_accum_dtype``) on the GPU.

* fp32-D wgrad GEMM (``gemm_f32acc_kernel``): with one K split, bit for bit against ``fp32_rn(C + A B^T)`` on exact operands at every tile
  width and at ragged M / N / K, the output a strided view whose guard cells must not change; split-K on exact operands (every order of
  the fp32 reduce-adds gives the same bits) and on random operands within an fp64 bound.  The FP8 instantiation
  (``gemm_fp8_f32acc_kernel``) at both A formats, both tile widths and the scale edges.
* Norm and embedding backward into fp32: the fp64 oracle, an fp32 emulator bit for bit, the same bits on a second call and under
  CUDA-graph replay.
* Whole step: ``run_step`` / ``step_ratios`` of ``test_step_oracle.py`` at ``n_acc`` 1, 4 and 16; with fp32 accumulators the worst ratio
  at 16 micro-batches is no worse than at 1, with bf16 ones it grows (both printed with ``-s``).
* Trainer: one-GPU ACCO with CUDA graphs and ``grad_accum_dtype=fp32`` (also with ``fp8``, ``packing`` and ``max_grad_norm``) against
  the fp32 CPU trainer, with no parameter holding a ``.grad`` after a micro-batch."""
import logging
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

from test_gemm_oracle import dense_exact, ints  # noqa: E402
from test_step_oracle import (emb_inputs, emb_ref, emulate_embedding_bwd, hf_from_native, hf_grads, native_grads, rel_err,  # noqa: E402
                              run_step, step_ratios, zipf_ids)

DEV = "cuda"


def ext():
    from acco_b200.ops import load_ext
    return load_ext(required=True)


def f32_in(t: torch.Tensor, seed: int):
    """(big, view): fp32 ``t`` inside a larger buffer of random guard values, rows 16-byte aligned."""
    r, c = t.shape
    width = -(-c // 8) * 8 + 16
    g = torch.Generator(device=DEV).manual_seed(seed)
    big = torch.randn(r + 3, width, generator=g, device=DEV)
    view = big[1:r + 1, 4:c + 4]
    view.copy_(t)
    assert view.data_ptr() % 16 == 0
    return big, view


def guards(big, r, c):
    m = torch.ones_like(big, dtype=torch.bool)
    m[1:r + 1, 4:c + 4] = False
    return big[m].clone(), m


# ---------------------------------------------------------------------------------------------- wgrad GEMM into fp32
# (M = output rows = the weight's rows, N = its columns, K = tokens)
ONE_SPLIT = [(bn, M, N, K) for bn in (64, 128, 256) for (M, N, K) in [(256, 512, 1024), (200, 72, 1000), (768, 2304, 4096)]]


@pytest.mark.parametrize("bn,M,N,K", ONE_SPLIT)
def test_wgrad_f32_one_split_is_exact(bn, M, N, K):
    dy = dense_exact(K, M, seed=M + K, device=DEV)            # A stored [K, M]
    x = dense_exact(K, N, seed=N + 3 * K, device=DEV)         # B stored [K, N]
    c0 = torch.randn(M, N, device=DEV) * 64                   # a prior accumulator with full fp32 mantissas
    big, out = f32_in(c0, seed=bn)
    g0, m = guards(big, M, N)
    ext().gemm_wgrad_f32(dy, x, out, bn, 1, 0)
    want = (c0.double() + dy.double().t() @ x.double()).float()   # the product is exact; one fp32 rounding of C + it
    assert torch.equal(out.view(torch.int32), want.view(torch.int32)), (bn, M, N, K)
    assert torch.equal(big[m], g0)


@pytest.mark.parametrize("splits", [2, 4, 16])
@pytest.mark.parametrize("bn", [64, 128, 256])
def test_wgrad_f32_split_k(bn, splits):
    M, N, K = 200, 136, 8192
    # exact tier: integer partials and an integer prior, every order of the fp32 reduce-adds is exact
    dy, x = ints((K, M), 2, seed=1, device=DEV), ints((K, N), 2, seed=2, device=DEV)
    c0 = ints((M, N), 1000, seed=3, device=DEV).float()
    big, out = f32_in(c0, seed=splits)
    g0, m = guards(big, M, N)
    ext().gemm_wgrad_f32(dy, x, out, bn, splits, 0)
    assert torch.equal(out, (c0.double() + dy.double().t() @ x.double()).float())
    assert torch.equal(big[m], g0)
    # random tier: within fp32 accumulation of K products plus one add per split
    g = torch.Generator(device=DEV).manual_seed(bn + splits)
    dy = torch.randn(K, M, generator=g, device=DEV).to(torch.bfloat16)
    x = torch.randn(K, N, generator=g, device=DEV).to(torch.bfloat16)
    c0 = torch.randn(M, N, generator=g, device=DEV) * math.sqrt(K)
    out = c0.clone()
    ext().gemm_wgrad_f32(dy, x, out, bn, splits, 0)
    y64 = c0.double() + dy.double().t() @ x.double()
    mag = c0.double().abs() + dy.double().abs().t() @ x.double().abs()
    ratio = ((out.double() - y64).abs() / ((K / 16 + splits + 2) * 2.0 ** -24 * mag)).max().item()
    print(f"split-K bn {bn} splits {splits}: worst error / bound {ratio:.3g}")
    assert ratio <= 1.0


def test_wgrad_f32_heuristic_and_rejections():
    from acco_b200.ops.gemm import gemm_tt_acc
    dy = dense_exact(8192, 768, seed=5, device=DEV)
    x = dense_exact(8192, 2048, seed=6, device=DEV)
    out = torch.zeros(768, 2048, device=DEV)
    gemm_tt_acc(dy, x, out)                                   # the fp32 path of the wgrad the linear layer calls
    assert torch.equal(out, (dy.double().t() @ x.double()).float())
    C = ext()
    with pytest.raises(RuntimeError, match="fp32"):
        C.gemm_wgrad_f32(dy, x, torch.zeros(768, 2048, dtype=torch.bfloat16, device=DEV))
    with pytest.raises(RuntimeError, match="bf16 matrix"):         # the bf16 GEMM keeps its contract
        C.gemm(dy, x, out, None, True, True, True, 0, 0, 0, 0, 0, 0)
    assert torch.equal(out, (dy.double().t() @ x.double()).float())


SCALE_EDGES = [(1.0, 1.0), (2.0 ** -20, 2.0 ** -20), (2.0 ** -127, 2.0 ** 10), (2.0 ** 120, 2.0 ** -100), (2.0 ** -127, 2.0 ** -127)]


@pytest.mark.parametrize("inv_a,inv_b", SCALE_EDGES)
@pytest.mark.parametrize("bn", [64, 128])
@pytest.mark.parametrize("fmt", ["e4m3", "e5m2"])
def test_fp8_f32acc_exact(fmt, bn, inv_a, inv_b):
    M, N, K = 200, 136, 1024
    fa = torch.float8_e5m2 if fmt == "e5m2" else torch.float8_e4m3fn
    a = ints((M, K), 2, seed=11, device=DEV).float().to(fa)
    b = ints((N, K), 2, seed=12, device=DEV).float().to(torch.float8_e4m3fn)
    sa = torch.tensor([1.0 / inv_a, inv_a, 0.0], dtype=torch.float32, device=DEV)
    sb = torch.tensor([1.0 / inv_b, inv_b, 0.0], dtype=torch.float32, device=DEV)
    c0 = torch.randn(M, N, device=DEV)
    big, out = f32_in(c0, seed=bn)
    g0, m = guards(big, M, N)
    ext().gemm_fp8_acc_f32(a, b, sa, sb, out, bn, 1, 0)
    y = (a.double() @ b.double().t()) * (float(sa[1]) * float(sb[1]))
    want = (c0.double() + y).float()
    assert torch.equal(out.view(torch.int32), want.view(torch.int32)), (fmt, bn, inv_a, inv_b)
    assert torch.equal(big[m], g0)
    out2 = c0.clone()
    ext().gemm_fp8_acc_f32(a, b, sa, sb, out2, bn, 4, 0)     # split-K: fp32 partials added by the TMA unit, in any order
    mag = c0.double().abs() + (a.double().abs() @ b.double().abs().t()) * abs(float(sa[1]) * float(sb[1]))
    assert ((out2.double() - (c0.double() + y)).abs() <= 8 * 2.0 ** -24 * mag + 1e-30).all()


# ---------------------------------------------------------------------------------------------- norm and embedding into fp32
@pytest.mark.parametrize("H,T", [(768, 8192), (2048, 4096), (64, 1000)])
@pytest.mark.parametrize("layer", [False, True], ids=["rmsnorm", "layernorm"])
def test_norm_bwd_into_fp32(layer, H, T):
    C = ext()
    g = torch.Generator(device=DEV).manual_seed(H + T)
    x = torch.randn(T, H, generator=g, device=DEV).to(torch.bfloat16)
    w = (1 + 0.1 * torch.randn(H, generator=g, device=DEV)).to(torch.bfloat16)
    b = (0.1 * torch.randn(H, generator=g, device=DEV)).to(torch.bfloat16) if layer else None
    dy = torch.randn(T, H, generator=g, device=DEV).to(torch.bfloat16)
    y, _, mean, rstd = C.norm_fwd(x, None, w, b, 1e-5)
    wg0 = torch.randn(H, generator=g, device=DEV) * 0.01
    bg0 = torch.randn(H, generator=g, device=DEV) * 0.01 if layer else None
    dh_ref, dwdb = C.norm_bwd(dy, None, x, w, mean, rstd, None, None)           # the same reduction into a fresh fp32 vector
    wg, bg = wg0.clone(), (bg0.clone() if layer else None)
    dh = C.norm_bwd_acc_f32(dy, None, x, w, mean, rstd, wg, bg)
    assert torch.equal(dh, dh_ref)
    assert torch.equal(wg, wg0 + dwdb[:H])                                         # fp32 emulator: the prior plus the kernel's sums
    if layer:
        assert torch.equal(bg, bg0 + dwdb[H:])
    # fp64 oracle
    xf = x.double()
    if layer:
        xh = (xf - xf.mean(-1, keepdim=True)) / torch.sqrt(xf.var(-1, unbiased=False, keepdim=True) + 1e-5)
    else:
        xh = xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + 1e-5)
    dw64 = wg0.double() + (dy.double() * xh).sum(0)
    e = rel_err(wg, dw64).item()
    assert e < 1e-5, e
    # a second call and a CUDA-graph replay give the same bits
    again = wg0.clone()
    bg2 = bg0.clone() if layer else None
    C.norm_bwd_acc_f32(dy, None, x, w, mean, rstd, again, bg2)
    assert torch.equal(again, wg)
    gw = wg0.clone()
    gb = bg0.clone() if layer else None
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        C.norm_bwd_acc_f32(dy, None, x, w, mean, rstd, gw, gb)        # warm-up (allocations), then reset the accumulator
        gw.copy_(wg0)
        if layer:
            gb.copy_(bg0)
        with torch.cuda.graph(graph, stream=s):
            C.norm_bwd_acc_f32(dy, None, x, w, mean, rstd, gw, gb)
    torch.cuda.current_stream().wait_stream(s)
    gw.copy_(wg0)
    if layer:
        gb.copy_(bg0)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(gw, wg) and (not layer or torch.equal(gb, bg))


EMB_CASES = [("llama1b-zipf", 128256, 128256, 2048, 4096, "zipf"), ("gptneo-zipf", 50257, 50304, 768, 8192, "zipf"),
             ("one-id-8192", 50257, 50304, 768, 8192, "one"), ("h776-edges", 50257, 50304, 776, 4096, "edges")]


@pytest.mark.parametrize("case", EMB_CASES, ids=[c[0] for c in EMB_CASES])
def test_embedding_bwd_into_fp32(case):
    from acco_b200 import ops
    from acco_b200.ops.embedding import embedding_bwd_f32
    name, V, Vp, H, T, kind = case
    grad0, ids, dy = (t.to(DEV) for t in emb_inputs(V, Vp, H, T, kind, seed=V + T, prior="small"))
    prior = grad0.float() + torch.randn(grad0.shape, device=DEV) * 1e-4     # an fp32 prior with bits below bf16's
    got = prior.clone()
    before = ops.launch_counts().get("embedding_bwd_f32", 0)
    embedding_bwd_f32(got, ids, dy)
    assert ops.launch_counts().get("embedding_bwd_f32", 0) == before + 1
    emu = emulate_embedding_bwd(prior, ids, dy)                               # fp32 rows: the emulator's last step rounds to fp32
    assert torch.equal(got.view(torch.int32), emu.view(torch.int32)), name
    hit = torch.zeros(grad0.shape[0], dtype=torch.bool, device=DEV)
    hit[ids] = True
    assert torch.equal(got[~hit], prior[~hit])                                # rows no id hits (the padding among them) keep their bits
    # fp64 oracle: no term passes through more than min(n, ceil(n / 8) + 8) fp32 roundings, plus the final one (test_step_oracle.py)
    o = emb_ref(prior, ids, dy)
    n = o["n"].unsqueeze(1).double()
    bnd = (torch.minimum(n, torch.ceil(n / 8) + 8) + 1) * 2.0 ** -24 * o["abs_terms"] + (n + 1) * 2.0 ** -125
    assert ((got.double() - o["y64"]).abs() <= bnd).all(), name
    again = prior.clone()
    embedding_bwd_f32(again, ids, dy)
    assert torch.equal(again, got)
    # CUDA graph: sort + kernel, replayed on the same prior
    gg = prior.clone()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        embedding_bwd_f32(gg, ids, dy)
        gg.copy_(prior)
        with torch.cuda.graph(graph, stream=s):
            embedding_bwd_f32(gg, ids, dy)
    torch.cuda.current_stream().wait_stream(s)
    gg.copy_(prior)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(gg, got)


def test_embedding_bwd_f32_rejections():
    C = ext()
    ids = torch.zeros(4, dtype=torch.long, device=DEV)
    with pytest.raises(RuntimeError):
        C.embedding_bwd_f32(torch.zeros(8, 16, dtype=torch.bfloat16, device=DEV), ids, ids, torch.zeros(4, 16, dtype=torch.bfloat16, device=DEV))
    with pytest.raises(RuntimeError, match="multiple of 8"):
        C.embedding_bwd_f32(torch.zeros(8, 12, device=DEV), ids, ids, torch.zeros(4, 12, dtype=torch.bfloat16, device=DEV))


# ---------------------------------------------------------------------------------------------- whole step
LLAMA125 = dict(vocab_size=50257, hidden_size=768, intermediate_size=2048, num_hidden_layers=2, num_attention_heads=12,
                num_key_value_heads=12, max_position_embeddings=1024)
GPTNEO125 = dict(vocab_size=50257, hidden_size=768, num_hidden_layers=2, num_attention_heads=12, max_position_embeddings=1024,
                 attention_layers="alternating", window_size=256)


def main_grads(native):
    """``native_grads`` over the fp32 ``main_grad`` views."""
    params = list(native.parameters())
    out = {}
    for key, view in native._hf_tensors():
        if key == "lm_head.weight" and native.config.tie_word_embeddings:
            continue
        p = next(p for p in params if p.untyped_storage().data_ptr() == view.untyped_storage().data_ptr())
        g = p.main_grad
        out[key] = g.as_strided(view.shape, view.stride(), g.storage_offset() + view.storage_offset() - p.storage_offset())
    return out


@pytest.mark.parametrize("arch", ["llama", "gptneo"])
def test_whole_step_fp32_accumulators_do_not_drift(arch):
    from acco_b200.models import GPTConfig, GPTForCausalLM, LlamaConfig, LlamaForCausalLM
    from acco_b200.parallel.arena import FlatArena
    B, S = 4, 1024
    worst = {}
    for n_acc in (1, 4, 16):
        torch.manual_seed(0)
        mk = (lambda: GPTForCausalLM(GPTConfig(**GPTNEO125))) if arch == "gptneo" else (lambda: LlamaForCausalLM(LlamaConfig(**LLAMA125)))
        base = mk().to(DEV).to(torch.bfloat16)
        V = base.config.vocab_size
        batches = [zipf_ids(B * S, V, seed=100 + i).view(B, S).to(DEV) for i in range(n_acc)]
        hf16 = hf_from_native(base, torch.bfloat16, DEV, attn="sdpa")
        hf64 = hf_from_native(base, torch.float64, DEV, attn="eager")
        run_step(hf16, batches, hf_V=V)
        run_step(hf64, batches, hf_V=V)
        g64, g16 = hf_grads(hf64), hf_grads(hf16)
        del hf64
        embed = "transformer.wte.weight" if arch == "gptneo" else "model.embed_tokens.weight"
        run_step(base, batches)                                               # bf16 accumulators (.grad)
        ours16 = native_grads(base)
        r_bf16 = max(step_ratios(ours16, g64, g16, embed, torch.cat(batches)).values())
        e_bf16 = max(float(rel_err(ours16[k], g64[k])) for k in g64)
        fp = mk().to(DEV).to(torch.bfloat16)
        fp.load_state_dict(base.state_dict())
        FlatArena(fp, 1, 0, torch.bfloat16, DEV, grad_dtype=torch.float32)
        for ids in batches:
            fp(input_ids=ids, labels=ids).loss.backward()
        assert all(p.grad is None for p in fp.parameters())
        ours32 = main_grads(fp)
        r_fp32 = max(step_ratios(ours32, g64, g16, embed, torch.cat(batches)).values())
        e_fp32 = max(float(rel_err(ours32[k], g64[k])) for k in g64)
        worst[n_acc] = (r_fp32, r_bf16, e_fp32, e_bf16)
        print(f"{arch} n_acc {n_acc}: worst ratio fp32 accumulators {r_fp32:.3f}, bf16 accumulators {r_bf16:.3f}; "
              f"worst relative error vs fp64 {e_fp32:.3g} / {e_bf16:.3g}")
        del base, fp, hf16, g64, g16, ours16, ours32
        torch.cuda.empty_cache()
    assert all(w[0] <= 1.0 for w in worst.values()), worst
    assert worst[16][0] <= worst[1][0] * 1.1, worst                           # fp32: no drift with the micro-batch count
    # bf16: the error the accumulator adds grows with the count, measured against the fp32 accumulators' on the same batches
    assert worst[16][3] / worst[16][2] > worst[1][3] / worst[1][2], worst


# ---------------------------------------------------------------------------------------------- trainer
def _make(tmp_path, monkeypatch, mixed=True, steps=16, **kw):
    from acco_b200 import AttrDict, DecoupledTrainer
    from acco_b200.data import ByteTokenizer, synthetic_pretrain_dataset, synthetic_sft_dataset
    from acco_b200.launch import DistEnv
    from acco_b200.models import LlamaConfig, LlamaForCausalLM
    monkeypatch.chdir(tmp_path)
    torch.manual_seed(0)
    cfg = LlamaConfig(vocab_size=1000, hidden_size=256, intermediate_size=512, num_hidden_layers=2, num_attention_heads=4,
                      num_key_value_heads=4, max_position_embeddings=256)
    tok = None
    if kw.get("packing"):
        tok = ByteTokenizer()
        tok.pad_token_id = tok.eos_token_id = 999
        ds = synthetic_sft_dataset(1200, 90, 999, 256, seed=1)
        kw.update(const_len_batch=False)
    else:
        ds = synthetic_pretrain_dataset(512, 100, 1000, 128, seed=0)
    args = AttrDict(method_name="acco", batch_size=4, n_grad_accumulation=4, max_length=128 if not kw.get("packing") else 256,
                    nb_steps_tot=steps, warmup=0, learning_rate=1e-3, save=False, tensorboard=False, use_mixed_precision=mixed,
                    static_accumulation=True, seed=1, **kw)
    return DecoupledTrainer(model=LlamaForCausalLM(cfg), tokenizer=tok, train_dataset=ds, args=args, log=logging.getLogger("ga"),
                            env=DistEnv(id_run="ga"))


def _train(t, check_grads=False):
    losses = []
    if check_grads:
        step = t.gradient_step

        def gradient_step(*a, **k):
            step(*a, **k)
            assert all(p.grad is None for p in t.model.parameters())      # nothing slipped past the arena
        t.gradient_step = gradient_step
    while not t.finished():
        t.step()
        losses.append(float(t.loss_host))
    t._drain()
    return losses


TRAINER_CASES = {"plain": {}, "fp8": dict(fp8=True), "max_grad_norm": dict(max_grad_norm=0.5), "packing": dict(packing=True)}


@pytest.mark.parametrize("case", list(TRAINER_CASES))
def test_trainer_fp32_accumulators_with_cuda_graphs(tmp_path, monkeypatch, case):
    from acco_b200 import ops
    kw = TRAINER_CASES[case]
    ops.reset_launch_counts()
    t = _make(tmp_path, monkeypatch, grad_accum_dtype="fp32", **kw)
    assert t.arena.grad_dtype == torch.float32 and t.arena.dtype == torch.bfloat16
    got = _train(t, check_grads=True)
    counts = ops.launch_counts()
    assert t._graphs is not None and not getattr(t, "_graphs_disabled", None)
    assert counts.get("gemm_fp8_f32acc" if case == "fp8" else "gemm_f32acc", 0) > 0, counts
    assert all(math.isfinite(x) for x in got)
    # the fp32 CPU trainer on the same data and initial weights
    with monkeypatch.context() as mp:
        mp.setattr(torch.cuda, "is_available", lambda: False)
        ref_t = _make(tmp_path, mp, mixed=False, **{k: v for k, v in kw.items() if k != "fp8"})
        ref = _train(ref_t)
    print(f"{case}: losses fp32 accumulators {got[:3]} ... {got[-3:]}, fp32 CPU {ref[:3]} ... {ref[-3:]}")
    assert len(got) == len(ref)
    tol = 0.06 if case == "fp8" else 0.03
    torch.testing.assert_close(torch.tensor(got), torch.tensor(ref), rtol=tol, atol=0)
