"""The embedding backward on the GPU (``ops.embedding`` -> ``embedding_bwd_kernel``) against the oracle of ``test_step_oracle.py``.

* Every case of ``GPU_CASES`` (Llama-3.2-1B and GPT-Neo widths, H = 64 and 776 where the last 256-column slice is partial, Zipf, uniform, ids 0 and V - 1 planted, one id over all 8192 tokens,
  a prior row 64x the addends as the tied LM-head wgrad leaves it) on both branches of ``EmbeddingFn.backward``: into an existing
  ``.grad`` and into a fresh ``dw``.  Every row hit is within the bound, every other row (the vocabulary padding included) keeps its
  bits, the result equals the fp32 emulator bit for bit, and a second call gives the same bits.
* Packed ``position_ids`` into GPT-Neo's ``wpe``.
* A CUDA graph of the forward and backward, replayed once, gives the bits of the eager call; the path without the kernels
  (``ACCO_FORCE_EAGER=1``) is capturable too and meets the bound.
* Rejected requests raise.
* Whole step: the gradients of a native training step (bf16 kernel path, ``n_acc`` micro-batches accumulated into ``.grad``), tensor by
  tensor under HF keys and embedding row by row, against HF in fp64 built from the same bf16 weights, with HF's own bf16 model as the
  yardstick (``step_ratios``; the worst ratio of each case is printed).  Cases: 2 layers at Llama-125M widths (tied, V = 50257,
  8 x 1024, ``n_acc`` 1 and 4, and with label smoothing 0.1), Llama-3.2-1B widths (GQA 32 / 8, llama3 ``rope_scaling``, tied,
  V = 128256), an untied Llama at V = 128256, and GPT-Neo-125M widths (alternating 256-token windows, ``wpe``)."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from test_step_oracle import (GPU_CASES, emb_bound, emb_checks, emb_inputs, emb_ref, emulate_embedding_bwd,  # noqa: E402
                              hf_from_native, hf_grads, native_grads, packed_positions, row_occurrences, run_step, step_ratios,
                              zipf_ids)

DEV = "cuda"


def run_op(grad0: torch.Tensor, ids: torch.Tensor, dy: torch.Tensor, fresh: bool) -> torch.Tensor:
    """``ops.embedding`` forward + backward into ``weight.grad`` (a copy of ``grad0``), or into a fresh ``dw`` (``grad0`` all zero)."""
    from acco_b200 import ops
    w = torch.nn.Parameter(torch.randn(grad0.shape, device=DEV).to(torch.bfloat16))
    if not fresh:
        w.grad = grad0.clone()
    before = ops.launch_counts().get("embedding_bwd", 0)
    ops.embedding(ids, w).backward(dy)
    assert ops.launch_counts().get("embedding_bwd", 0) == before + 1
    return w.grad


def check(grad0, ids, dy, got, name):
    o = emb_ref(grad0, ids, dy)
    c = emb_checks(got, grad0, o, emb_bound(o))
    n = row_occurrences(ids, grad0.shape[0])
    print(f"{name}: worst error/bound {c['rows']:.3f} over {int((n > 0).sum())} rows, max n_r {int(n.max())}")
    assert c["rows"] <= 0.5 and c["untouched"] == 0.0, (name, c)
    emu = emulate_embedding_bwd(grad0, ids, dy)
    assert torch.equal(got.view(torch.int16), emu.view(torch.int16)), name


@pytest.mark.parametrize("case", GPU_CASES, ids=[c[0] for c in GPU_CASES])
def test_embedding_bwd(case):
    name, V, Vp, H, T, kind, prior = case
    fresh = prior == "zero"
    grad0, ids, dy = (t.to(DEV) for t in emb_inputs(V, Vp, H, T, kind, seed=V + T, prior=prior))
    if fresh:
        grad0.zero_()                       # a fresh dw starts at zero, padding rows included
    got = run_op(grad0, ids, dy, fresh)
    check(grad0, ids, dy, got, name)
    again = run_op(grad0, ids, dy, fresh)
    assert torch.equal(got.view(torch.int16), again.view(torch.int16))


def test_packed_wpe():
    """GPT-Neo's position table under packed rows: 8 rows of 1024, documents of random length starting on and off 128-row blocks."""
    P, H, B, S = 2048, 768, 8, 1024
    g = torch.Generator().manual_seed(5)
    lens = []
    while sum(lens) < B * S:
        lens.append(int(torch.randint(1, 700, (1,), generator=g)))
    pos = torch.cat([packed_positions(S, lens[i::B] + [S]) for i in range(B)])      # per row: its documents, then fill to S
    grad0, _, dy = emb_inputs(P, P, H, B * S, "uniform", seed=11)
    grad0, pos, dy = grad0.to(DEV), pos.to(DEV), dy.to(DEV)
    got = run_op(grad0, pos, dy, fresh=False)
    check(grad0, pos, dy, got, "wpe-packed")


def test_cuda_graph_replay_matches_eager():
    """The trainer captures the whole step; the backward must have no host sync and a fixed output size."""
    from acco_b200 import ops
    name, V, Vp, H, T, kind, prior = GPU_CASES[0]
    grad0, ids, dy = (t.to(DEV) for t in emb_inputs(V, Vp, H, T, kind, seed=V + T, prior=prior))
    eager = run_op(grad0, ids, dy, fresh=False)
    w = torch.nn.Parameter(torch.randn(grad0.shape, device=DEV).to(torch.bfloat16))
    w.grad = grad0.clone()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):                       # warm-up outside the capture, as torch.cuda.graphs asks
        ops.embedding(ids, w).backward(dy)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ops.embedding(ids, w).backward(dy)
    w.grad.copy_(grad0)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(w.grad.view(torch.int16), eager.view(torch.int16))


def test_eager_path_is_capturable(monkeypatch):
    """Without the kernels (``ACCO_FORCE_EAGER=1``) the backward is ``embedding_bwd_ref``: capturable as well, and within the bound
    (its fp32 ``index_add_`` is atomic, so its bits may vary with the order of the adds)."""
    from acco_b200 import ops
    monkeypatch.setenv("ACCO_FORCE_EAGER", "1")
    name, V, Vp, H, T, kind, prior = GPU_CASES[-1]
    grad0, ids, dy = (t.to(DEV) for t in emb_inputs(V, Vp, H, T, kind, seed=V + T, prior=prior))
    w = torch.nn.Parameter(torch.randn(grad0.shape, device=DEV).to(torch.bfloat16))
    w.grad = grad0.clone()
    before = ops.launch_counts().get("embedding_bwd", 0)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ops.embedding(ids, w).backward(dy)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ops.embedding(ids, w).backward(dy)
    w.grad.copy_(grad0)
    graph.replay()
    torch.cuda.synchronize()
    assert ops.launch_counts().get("embedding_bwd", 0) == before
    o = emb_ref(grad0, ids, dy)
    c = emb_checks(w.grad, grad0, o, emb_bound(o))
    assert c["rows"] <= 0.5 and c["untouched"] == 0.0, c


def test_rejected_requests():
    from acco_b200.ops import load_ext
    C = load_ext(required=True)
    ids = torch.zeros(4, dtype=torch.long, device=DEV)
    grad = torch.zeros(8, 12, dtype=torch.bfloat16, device=DEV)
    with pytest.raises(RuntimeError, match="multiple of 8"):
        C.embedding_bwd(grad, ids, ids, torch.zeros(4, 12, dtype=torch.bfloat16, device=DEV))
    grad = torch.zeros(8, 16, dtype=torch.bfloat16, device=DEV)
    with pytest.raises(RuntimeError, match="one entry per dy row"):
        C.embedding_bwd(grad, ids[:3], ids[:3], torch.zeros(4, 16, dtype=torch.bfloat16, device=DEV))
    with pytest.raises(RuntimeError):
        C.embedding_bwd(grad.float(), ids, ids, torch.zeros(4, 16, dtype=torch.bfloat16, device=DEV))
    assert not grad.any()


LLAMA125 = dict(vocab_size=50257, hidden_size=768, intermediate_size=2048, num_hidden_layers=2, num_attention_heads=12,
                num_key_value_heads=12, max_position_embeddings=1024)
LLAMA1B = dict(vocab_size=128256, hidden_size=2048, intermediate_size=8192, num_hidden_layers=2, num_attention_heads=32,
               num_key_value_heads=8, max_position_embeddings=8192, rope_theta=500000.0,
               rope_scaling=dict(rope_type="llama3", factor=32.0, low_freq_factor=1.0, high_freq_factor=4.0,
                                 original_max_position_embeddings=8192))
GPTNEO125 = dict(vocab_size=50257, hidden_size=768, num_hidden_layers=2, num_attention_heads=12, max_position_embeddings=1024,
                 attention_layers="alternating", window_size=256)
STEP_CASES = [
    # (name, arch, config, B, S, n_acc, label smoothing)
    ("llama125m", "llama", LLAMA125, 8, 1024, 1, 0.0),
    ("llama125m-nacc4", "llama", LLAMA125, 8, 1024, 4, 0.0),
    ("llama125m-smooth0.1", "llama", LLAMA125, 8, 1024, 1, 0.1),
    ("llama1b-gqa-rope-llama3", "llama", LLAMA1B, 2, 2048, 1, 0.0),
    ("llama-untied-128256", "llama", dict(LLAMA1B, tie_word_embeddings=False), 2, 2048, 1, 0.0),
    ("gptneo125m", "gptneo", GPTNEO125, 4, 1024, 1, 0.0),
]


@pytest.mark.parametrize("case", STEP_CASES, ids=[c[0] for c in STEP_CASES])
def test_whole_step_gradients_vs_fp64(case):
    from acco_b200.models import GPTConfig, GPTForCausalLM, LlamaConfig, LlamaForCausalLM
    name, arch, cfg, B, S, n_acc, smoothing = case
    torch.manual_seed(0)
    native = (GPTForCausalLM(GPTConfig(**cfg)) if arch == "gptneo" else LlamaForCausalLM(LlamaConfig(**cfg))).to(DEV).to(torch.bfloat16)
    native.label_smoothing = smoothing
    V = native.config.vocab_size
    hf16 = hf_from_native(native, torch.bfloat16, DEV, attn="sdpa")
    hf64 = hf_from_native(native, torch.float64, DEV, attn="eager")
    batches = [zipf_ids(B * S, V, seed=100 + i).view(B, S).to(DEV) for i in range(n_acc)]
    run_step(native, batches)
    run_step(hf16, batches, smoothing, hf_V=V)
    run_step(hf64, batches, smoothing, hf_V=V)
    embed = "transformer.wte.weight" if arch == "gptneo" else "model.embed_tokens.weight"
    r = step_ratios(native_grads(native), hf_grads(hf64), hf_grads(hf16), embed, torch.cat(batches))
    worst = max(r.items(), key=lambda kv: kv[1])
    print(f"{name}: worst e(ours) / (2 e(HF bf16) + floor) = {worst[1]:.3f} ({worst[0]})")
    assert not native.embed_weight.grad[V:].any()                     # vocabulary padding rows get no gradient
    assert worst[1] <= 1.0, r
