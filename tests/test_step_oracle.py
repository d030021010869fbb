"""fp64 oracle of the embedding backward (``ops.embedding``, ``embedding_bwd_kernel``), the per-element bound of its GPU test
(``test_step_oracle_gpu.py``), and the margin table that shows the bound is the right size.  Runs on the CPU without the extension.

Contract.  For every row ``r`` of the gradient (``weight.grad`` in the arena, or the fresh ``dw`` when there is none):

    grad'[r] = bf16_rn(grad[r] + sum_{i: ids[i] = r} dy[i])

Rows no id hits - the vocabulary padding rows ``[V, Vp)`` among them - stay bit for bit unchanged.

Bound.  ``n_r`` (``row_occurrences``) is the number of ids equal to ``r``.  The kernel forms the sum of the ``n_r + 1`` terms (the prior
row and the addends) in fp32: 8 partial sums take the occurrences round-robin, then the partials are added in order and the prior
last.  No term passes through more than ``sum_depth(n_r) = min(n_r, ceil(n_r / 8) + 8)`` roundings, so before the final rounding the
sum errs by at most ``sum_depth(n_r) U sum|terms|`` (``U = 2^-24``; first order, as that depth times ``U`` is below ``2^-13`` here),
plus ``2^-125`` per term for the flush to zero.  With ``E`` twice that, every element gets ``|grad' - y64| <= 2^-7 (|y64| + E) + E``: one bf16 ulp, twice the half ulp of rounding to
nearest, so a kernel that rounds once stays within half, as the bounds of ``test_rowwise_oracle.py`` do.

The margin table (``test_margin_table``) runs ``emulate_embedding_bwd``, an fp32 emulator in the kernel's order (ids sorted stably, each
run of equal ids split round-robin over 8 partial sums, the partials added in order, then the prior row), and asserts it stays within
half of the bound, and that each mutant lands more than 3x out (or breaks an exact check, shown as ``inf``):

* ``per_occurrence``: the row rounded to bf16 after every occurrence, in a random order (a bf16 ``index_add_`` on CUDA);
* ``ids_plus_one``: every id off by one;
* ``prior_dropped`` / ``prior_twice``: the existing ``.grad`` ignored, or added twice;
* ``padding_written``: the padding rows ``[V, Vp)`` cleared, as a dense zero-fill would;
* ``wpe_token_ids``: the position table indexed by the token ids instead of the positions.

The whole-step part (``hf_from_native``, ``native_grads``, ``step_ratios``) compares a native training step's gradients with HF's;
its CPU checks are below and its GPU cases in ``test_step_oracle_gpu.py``.

Print the margin table with ``python tests/test_step_oracle.py``; ``test_per_occurrence_onset`` (``-s``) prints the smallest ``n_r`` from which the
per-occurrence rounding is 3x out on the ids of the GPU test's Llama-3.2-1B case."""
from __future__ import annotations

import math
from typing import Dict, Optional

import pytest
import torch

U = 2.0 ** -24                 # fp32 unit roundoff
B7 = 2.0 ** -7                 # one bf16 ulp, relative
FTZ = 2.0 ** -125              # twice the flush-to-zero threshold, per term
WARPS = 8                      # partial sums per run in embedding_bwd_kernel
DY_SCALE = 2.0 ** -10          # addends of the size of a per-token embedding gradient
LARGE_PRIOR = 64.0             # a prior row of LARGE_PRIOR * DY_SCALE, as the tied LM-head wgrad leaves it


def row_occurrences(ids: torch.Tensor, rows: int) -> torch.Tensor:
    """``n_r``: how many ids hit each row."""
    return torch.bincount(ids.reshape(-1).cpu(), minlength=rows)


def zipf_ids(T: int, V: int, seed: int, a: float = 1.0) -> torch.Tensor:
    """``T`` ids with a Zipf(``a``) marginal over a random ranking of ``[0, V)``: a few rows are hit hundreds of times, most once or not
    at all, as in text."""
    g = torch.Generator().manual_seed(seed)
    p = 1.0 / torch.arange(1, V + 1, dtype=torch.float64) ** a
    rank = torch.multinomial(p, T, replacement=True, generator=g)
    return torch.randperm(V, generator=g)[rank]


def packed_positions(T: int, doc_lens) -> torch.Tensor:
    """``position_ids`` of a packed row: each document counts from 0."""
    pos = torch.cat([torch.arange(n) for n in doc_lens])
    assert pos.numel() >= T
    return pos[:T]


def emb_inputs(V: int, Vp: int, H: int, T: int, ids: str, seed: int, prior: str = "small", pad_sentinel: float = 1.5):
    """(grad0, ids, dy).  ``ids``: ``zipf``, ``uniform``, ``one`` (one id repeated over all T), ``edges`` (Zipf with ids 0 and V - 1
    planted many times).  ``prior``: ``zero`` (a fresh ``dw``), ``small`` (an accumulated micro-batch of the same size as the
    addends), ``large`` (``LARGE_PRIOR`` times the addends).  The padding rows hold ``pad_sentinel``, which no valid update changes."""
    x, dy, g = emb_ids_dy(V, H, T, ids, seed)
    scale = {"zero": 0.0, "small": DY_SCALE, "large": LARGE_PRIOR * DY_SCALE}[prior]
    grad = (torch.randn(Vp, H, generator=g) * scale).to(torch.bfloat16)
    grad[V:] = pad_sentinel
    return grad, x, dy


def emb_ids_dy(V: int, H: int, T: int, ids: str, seed: int):
    """The ids and ``dy`` of ``emb_inputs``, and the generator that goes on to draw the prior."""
    g = torch.Generator().manual_seed(seed)
    if ids == "zipf":
        x = zipf_ids(T, V, seed)
    elif ids == "uniform":
        x = torch.randint(0, V, (T,), generator=g)
    elif ids == "one":
        x = torch.full((T,), V // 3, dtype=torch.long)
    elif ids == "edges":
        x = zipf_ids(T, V, seed)
        x[torch.randperm(T, generator=g)[: T // 8]] = 0
        x[torch.randperm(T, generator=g)[: T // 16]] = V - 1
    else:
        raise ValueError(ids)
    dy = (torch.randn(T, H, generator=g) * DY_SCALE).to(torch.bfloat16)
    return x, dy, g


def emb_ref(grad: torch.Tensor, ids: torch.Tensor, dy: torch.Tensor) -> Dict[str, torch.Tensor]:
    """fp64 oracle: ``y64`` (the exact new rows), ``abs_terms`` (``|grad| + sum |dy|`` per element), ``n`` (``n_r``), ``hit``."""
    ids = ids.reshape(-1)
    y = grad.double().index_add(0, ids, dy.double())
    a = grad.double().abs().index_add(0, ids, dy.double().abs())
    n = torch.bincount(ids, minlength=grad.shape[0]).to(grad.device)
    return {"y64": y, "abs_terms": a, "n": n, "hit": n > 0}


def sum_depth(n: torch.Tensor) -> torch.Tensor:
    """Most fp32 roundings any term of a row with ``n`` occurrences passes through in ``embedding_bwd_kernel``."""
    return torch.minimum(n, torch.div(n + WARPS - 1, WARPS, rounding_mode="floor") + WARPS)


def emb_bound(o: Dict[str, torch.Tensor]) -> torch.Tensor:
    n = o["n"].double().unsqueeze(1)
    E = 2 * (sum_depth(n) * U * o["abs_terms"] + FTZ * (n + 1))
    return B7 * (o["y64"].abs() + E) + E


def emb_checks(got: torch.Tensor, grad0: torch.Tensor, o: Dict[str, torch.Tensor], bnd: torch.Tensor) -> Dict[str, float]:
    """``rows``: the largest error / bound over the rows hit; ``untouched``: 0 if every other row (padding included) kept its bits,
    else inf."""
    hit = o["hit"]
    err = (got.double() - o["y64"]).abs()
    err = torch.where(torch.isfinite(got.double()), err, torch.full_like(err, math.inf))
    rows = float((err[hit] / bnd[hit]).max()) if bool(hit.any()) else 0.0
    same = torch.equal(got[~hit].view(torch.int16), grad0[~hit].view(torch.int16))
    return {"rows": rows, "untouched": 0.0 if same else math.inf}


def row_ratios(got: torch.Tensor, o: Dict[str, torch.Tensor], bnd: torch.Tensor) -> torch.Tensor:
    """Largest error / bound of each row (0 for rows no id hits)."""
    r = ((got.double() - o["y64"]).abs() / bnd).amax(dim=1)
    return torch.where(o["hit"], r, torch.zeros_like(r))


def _runs(ids: torch.Tensor):
    """Stable sort of the ids -> (perm, run index, rank in run, row of each run)."""
    s, perm = torch.sort(ids.reshape(-1), stable=True)
    start = torch.ones_like(s, dtype=torch.bool)
    start[1:] = s[1:] != s[:-1]
    run = torch.cumsum(start, 0) - 1
    first = torch.nonzero(start).squeeze(1)
    rank = torch.arange(s.numel(), device=s.device) - first[run]
    return perm, run, rank, s[first]


def emulate_embedding_bwd(grad: torch.Tensor, ids: torch.Tensor, dy: torch.Tensor, mutant: Optional[str] = None, V: int = 0,
                          positions: Optional[torch.Tensor] = None, seed: int = 0) -> torch.Tensor:
    """fp32 emulator of ``embedding_bwd_kernel`` (its exact summation order), or of one of the mutants of the module docstring.
    ``V``: where the padding rows start (``padding_written``).  ``positions``: the ``wpe_token_ids`` mutant indexes with ``ids`` where
    ``positions`` is the right index."""
    if mutant == "ids_plus_one":
        ids = (ids + 1) % grad.shape[0]
    if mutant == "wpe_token_ids":
        assert positions is not None
        ids = positions % grad.shape[0]
    out = grad.clone()
    if mutant == "per_occurrence":
        g = torch.Generator().manual_seed(seed)
        order = torch.randperm(ids.numel(), generator=g).to(ids.device)
        perm, run, rank, rows = _runs(ids.reshape(-1)[order])
        perm = order[perm]
        for k in range(int(rank.max()) + 1):
            sel = rank == k
            r = rows[run[sel]]
            out[r] = (out[r].float() + dy[perm[sel]].float()).to(out.dtype)
        return out
    perm, run, rank, rows = _runs(ids)
    acc = torch.zeros(rows.numel(), WARPS, dy.shape[1], dtype=torch.float32, device=dy.device)
    for k in range(int(rank.max()) // WARPS + 1):
        sel = (rank // WARPS) == k
        acc[run[sel], rank[sel] % WARPS] += dy[perm[sel]].float()
    t = acc[:, 0]
    for q in range(1, WARPS):
        t = t + acc[:, q]
    prior = out[rows].float()
    if mutant == "prior_dropped":
        prior = torch.zeros_like(prior)
    elif mutant == "prior_twice":
        prior = prior + prior
    out[rows] = (prior + t).to(out.dtype)
    if mutant == "padding_written":
        assert 0 < V < out.shape[0]
        out[V:] = 0
    return out


# GPU cases (test_step_oracle_gpu.py): (name, V, Vp, H, T, ids, prior)
GPU_CASES = [
    ("llama1b-zipf", 128256, 128256, 2048, 4096, "zipf", "small"),
    ("llama1b-zipf-large-prior", 128256, 128256, 2048, 4096, "zipf", "large"),
    ("llama1b-zipf-fresh", 128256, 128256, 2048, 4096, "zipf", "zero"),
    ("gptneo-zipf", 50257, 50304, 768, 8192, "zipf", "small"),
    ("gptneo-uniform", 50257, 50304, 768, 8192, "uniform", "small"),
    ("gptneo-edges", 50257, 50304, 768, 8192, "edges", "large"),
    ("one-id-8192", 50257, 50304, 768, 8192, "one", "large"),
    ("h64-zipf", 131, 144, 64, 4096, "zipf", "small"),              # the 64-wide preset: 8 of 32 lanes live
    ("h776-edges", 50257, 50304, 776, 4096, "edges", "large"),      # a ragged last 256-column slice
]


def test_per_occurrence_onset():
    """On the ids and ``dy`` of the GPU test's Llama-3.2-1B case, a row rounded once per occurrence is more than 3x out from its
    second rounded add on: every row with ``n_r >= 2`` when the row holds a prior, ``n_r >= 3`` for a fresh ``dw`` (whose first add is
    exact).  Rows hit once are one rounding either way.  Only the rows hit are formed (a full ``[V, H]`` fp64 table is GPU-sized)."""
    name, V, _, H, T, ids, _ = GPU_CASES[0]
    x, dy, g = emb_ids_dy(V, H, T, ids, seed=V + T)
    rows, inv = torch.unique(x, return_inverse=True)
    onset = {}
    for prior, scale in (("zero", 0.0), ("small", DY_SCALE)):
        g0 = (torch.randn(rows.numel(), H, generator=g) * scale).to(torch.bfloat16)
        o = emb_ref(g0, inv, dy)
        bnd = emb_bound(o)
        n = o["n"]
        r_mut = row_ratios(emulate_embedding_bwd(g0, inv, dy, mutant="per_occurrence"), o, bnd)
        r_emu = row_ratios(emulate_embedding_bwd(g0, inv, dy), o, bnd)
        assert float(r_emu.max()) <= 0.5
        onset[prior] = int(n[r_mut > 3].min())
        assert bool((r_mut[n >= onset[prior]] > 3).all()) and float(r_mut[n < onset[prior]].max()) <= 0.5, prior
        print(f"{name} prior={prior}: per-occurrence rounding > 3x out for every row from n_r = {onset[prior]} "
              f"(max n_r {int(n.max())}, worst {float(r_mut.max()):.3g})")
    assert onset == {"zero": 3, "small": 2}


@pytest.mark.parametrize("fresh", [False, True], ids=["accumulate", "fresh"])
def test_eager_path_meets_contract(fresh):
    """``ops.embedding``'s backward off the kernel path (``embedding_bwd_ref``: the CPU, and CUDA without the kernels) on both
    branches: within half the bound, untouched and padding rows bit for bit, empty ids a no-op."""
    from acco_b200 import ops
    grad0, ids, dy = emb_inputs(131, 144, 64, 2048, "edges", seed=2, prior="zero" if fresh else "large")
    w = torch.nn.Parameter(torch.randn(grad0.shape).to(torch.bfloat16))
    if fresh:
        grad0.zero_()
    else:
        w.grad = grad0.clone()
    ops.embedding(ids, w).backward(dy)
    o = emb_ref(grad0, ids, dy)
    c = emb_checks(w.grad, grad0, o, emb_bound(o))
    assert c["rows"] <= 0.5 and c["untouched"] == 0.0, c
    g = grad0.clone()
    from acco_b200.ops.embedding import embedding_bwd_ref
    embedding_bwd_ref(g, ids[:0], dy[:0])
    assert torch.equal(g.view(torch.int16), grad0.view(torch.int16))


# ================================================================================================= whole step
# A native training step's gradients against HF in fp64, built from the same bf16 weights (``hf_from_native``).  The comparator is
# HF's own bf16 model on the same weights and batch (cuBLAS, SDPA / eager attention, PyTorch's sorted embedding backward; no code shared
# with ours).  For each tensor ``t``, ``e_t(X) = ||g_X - g64||_F / ||g64||_F``; the native path must meet
# ``e_t(ours) <= K_STEP e_t(HF bf16) + FLOOR``, and so must every embedding row hit at least ``MIN_ROW_OCC`` times.  ``FLOOR`` is the
# rms relative error of rounding an fp64 gradient to bf16 once (``2^-9``): storing the gradient in the bf16 arena costs that much
# whatever the kernels do.
K_STEP = 2.0
FLOOR = 2.0 ** -9
MIN_ROW_OCC = 16


def hf_from_native(native, dtype, device, attn: str = "eager"):
    """The HF ``LlamaForCausalLM`` / ``GPTNeoForCausalLM`` of ``native``'s config, holding ``native.state_dict()`` cast to ``dtype``."""
    import transformers
    from acco_b200.models import GPTForCausalLM
    c = native.config
    if isinstance(native, GPTForCausalLM):
        layers = list(c.attention_layers)
        cfg = transformers.GPTNeoConfig(vocab_size=c.vocab_size, hidden_size=c.hidden_size, num_layers=c.num_hidden_layers,
                                        num_heads=c.num_attention_heads, max_position_embeddings=c.max_position_embeddings,
                                        attention_types=[[layers, 1]], window_size=c.window_size, intermediate_size=c.intermediate_size,
                                        layer_norm_epsilon=c.layer_norm_epsilon, attention_dropout=0, embed_dropout=0, resid_dropout=0,
                                        tie_word_embeddings=c.tie_word_embeddings, attn_implementation="eager")
        model = transformers.GPTNeoForCausalLM(cfg)
    else:
        cfg = transformers.LlamaConfig(vocab_size=c.vocab_size, hidden_size=c.hidden_size, intermediate_size=c.intermediate_size,
                                       num_hidden_layers=c.num_hidden_layers, num_attention_heads=c.num_attention_heads,
                                       num_key_value_heads=c.num_key_value_heads, max_position_embeddings=c.max_position_embeddings,
                                       rms_norm_eps=c.rms_norm_eps, rope_theta=c.rope_theta, rope_scaling=c.rope_scaling,
                                       tie_word_embeddings=c.tie_word_embeddings, attention_bias=False, mlp_bias=False,
                                       attn_implementation=attn)
        model = transformers.LlamaForCausalLM(cfg)
    model = model.to(device=device, dtype=dtype).eval()
    missing, unexpected = model.load_state_dict({k: v.to(dtype) for k, v in native.state_dict().items()}, strict=False)
    assert not unexpected and all(k.endswith(("rotary_emb.inv_freq", "attn.attention.bias", "masked_bias")) for k in missing), \
        (missing, unexpected)
    return model


def native_grads(native) -> Dict[str, torch.Tensor]:
    """The native gradients under HF keys: the model's own ``_hf_tensors`` table applied to the ``.grad`` views (the fused QKV and
    gate|up gradients split as the checkpoint splits the weights).  A tied head is the embedding: its key is dropped, so it counts once."""
    params = [p for p in native.parameters()]
    out = {}
    for key, view in native._hf_tensors():
        if key == "lm_head.weight" and native.config.tie_word_embeddings:
            continue
        p = next(p for p in params if p.untyped_storage().data_ptr() == view.untyped_storage().data_ptr())
        out[key] = p.grad.as_strided(view.shape, view.stride(), p.grad.storage_offset() + view.storage_offset() - p.storage_offset())
    return out


def hf_grads(hf) -> Dict[str, torch.Tensor]:
    return {k: p.grad for k, p in hf.named_parameters()}


def hf_loss(hf, ids: torch.Tensor, labels: torch.Tensor, V: int, smoothing: float = 0.0) -> torch.Tensor:
    """Mean next-token loss of an HF model, with label smoothing over the first ``V`` columns as ``F.cross_entropy`` defines it."""
    logits = hf(input_ids=ids).logits[:, :-1, :V]
    return torch.nn.functional.cross_entropy(logits.reshape(-1, V).float() if logits.dtype == torch.bfloat16 else logits.reshape(-1, V),
                                             labels[:, 1:].reshape(-1), ignore_index=-100, label_smoothing=smoothing)


def rel_err(g: torch.Tensor, g64: torch.Tensor, dim=None) -> torch.Tensor:
    d = (g.double() - g64).pow(2).sum(dim=dim).sqrt()
    return d / g64.pow(2).sum(dim=dim).sqrt().clamp_min(1e-300)


def step_ratios(ours: Dict[str, torch.Tensor], g64: Dict[str, torch.Tensor], hf16: Dict[str, torch.Tensor], embed_key: str,
                ids: torch.Tensor) -> Dict[str, float]:
    """Per tensor ``e_t(ours) / (K_STEP e_t(HF bf16) + FLOOR)``, plus ``embed rows``: the worst such ratio over the embedding rows hit
    at least ``MIN_ROW_OCC`` times.  A value above 1 fails the criterion."""
    assert set(ours) == set(g64) == set(hf16), (set(ours) ^ set(g64), set(g64) ^ set(hf16))
    out = {k: float(rel_err(ours[k], g64[k]) / (K_STEP * rel_err(hf16[k], g64[k]) + FLOOR)) for k in g64}
    n = torch.bincount(ids.reshape(-1).cpu(), minlength=g64[embed_key].shape[0])
    rows = torch.nonzero(n >= MIN_ROW_OCC).squeeze(1).to(g64[embed_key].device)
    if rows.numel():
        e_o = rel_err(ours[embed_key][rows], g64[embed_key][rows], dim=1)
        e_h = rel_err(hf16[embed_key][rows], g64[embed_key][rows], dim=1)
        out["embed rows"] = float((e_o / (K_STEP * e_h + FLOOR)).max())
    return out


def run_step(model, batches, smoothing: float = 0.0, hf_V: Optional[int] = None):
    """Forward + backward of every micro-batch, accumulating into ``.grad`` (the native model's own loss, or ``hf_loss``)."""
    for p in model.parameters():
        p.grad = None
    for ids in batches:
        if hf_V is None:
            model(input_ids=ids, labels=ids).loss.backward()
        else:
            hf_loss(model, ids, ids, hf_V, smoothing).backward()


def tiny_native(arch: str, tied: bool = True):
    from acco_b200.models import GPTConfig, GPTForCausalLM, LlamaConfig, LlamaForCausalLM
    torch.manual_seed(0)
    if arch == "gptneo":
        return GPTForCausalLM(GPTConfig(vocab_size=131, hidden_size=32, num_hidden_layers=2, num_attention_heads=4,
                                        max_position_embeddings=64, window_size=8, tie_word_embeddings=tied, pad_vocab_multiple=16))
    return LlamaForCausalLM(LlamaConfig(vocab_size=131, hidden_size=32, intermediate_size=64, num_hidden_layers=2, num_attention_heads=4,
                                        num_key_value_heads=2, max_position_embeddings=64, tie_word_embeddings=tied, pad_vocab_multiple=16))


@pytest.mark.parametrize("arch,tied", [("llama", True), ("llama", False), ("gptneo", True), ("gptneo", False)])
def test_key_mapping_and_microbatch_sum(arch, tied):
    """At V = 131 padded to 144 on the CPU (the native path in fp32, HF in fp64): every native gradient mapped through ``_hf_tensors``
    matches HF's to fp32 accuracy (a swapped or shifted split of the fused QKV / gate|up gradient is O(1) off), the tied head counts
    once (the embedding gradient holds both uses), the padding rows get nothing, and two micro-batches sum."""
    pytest.importorskip("transformers")
    native = tiny_native(arch, tied).float()
    hf = hf_from_native(native, torch.float64, "cpu")
    batches = [zipf_ids(2 * 24, 131, seed=s).view(2, 24) for s in (1, 2)]
    run_step(native, batches)
    run_step(hf, batches, hf_V=131)
    ours, ref = native_grads(native), hf_grads(hf)
    assert set(ours) == set(ref)
    assert ("lm_head.weight" in ref) == (not tied)
    for k in ref:
        assert float(rel_err(ours[k], ref[k])) < 1e-5, k
    assert not native.embed_weight.grad[131:].any()
    one = tiny_native(arch, tied).float()
    sums = {}
    for b in batches:
        run_step(one, [b])
        for k, g in native_grads(one).items():
            sums[k] = sums.get(k, 0) + g.clone()
    for k in ref:
        assert float(rel_err(ours[k], sums[k].double())) < 1e-6, k


def test_label_smoothing_formula():
    """The native loss with ``label_smoothing`` equals ``F.cross_entropy(label_smoothing=)`` over the first V columns of HF's logits
    (the padding columns take no share of the smoothing mass)."""
    pytest.importorskip("transformers")
    native = tiny_native("llama").float()
    native.label_smoothing = 0.1
    hf = hf_from_native(native, torch.float64, "cpu")
    ids = zipf_ids(48, 131, seed=3).view(2, 24)
    want = hf_loss(hf, ids, ids, 131, 0.1)
    assert abs(float(native(input_ids=ids, labels=ids).loss) - float(want)) < 1e-5 * float(want)
    native.label_smoothing = 0.0
    assert abs(float(native(input_ids=ids, labels=ids).loss) - float(want)) > 1e-3 * float(want)


@pytest.mark.parametrize("arch", ["llama", "gptneo"])
def test_native_cpu_bf16_within_half_the_step_criterion(arch):
    """The native CPU path in bf16 against HF bf16 on the CPU, both measured against HF fp64: within ``K_STEP / 2`` on every tensor."""
    pytest.importorskip("transformers")
    native = tiny_native(arch).to(torch.bfloat16)
    hf16 = hf_from_native(native, torch.bfloat16, "cpu")
    hf64 = hf_from_native(native, torch.float64, "cpu")
    batches = [zipf_ids(4 * 32, 131, seed=s).view(4, 32) for s in (4, 5)]
    for m, v in ((native, None), (hf16, 131), (hf64, 131)):
        run_step(m, batches, hf_V=v)
    embed = "transformer.wte.weight" if arch == "gptneo" else "model.embed_tokens.weight"
    r = step_ratios(native_grads(native), hf_grads(hf64), hf_grads(hf16), embed, torch.cat(batches))
    worst = max(r.items(), key=lambda kv: kv[1])
    print(f"{arch}: worst e(ours) / (K e(HF bf16) + floor) = {worst[1]:.3f} ({worst[0]})")
    assert worst[1] <= 0.5, worst


# ================================================================================================= margin table
CASES = [
    # (name, V, Vp, H, T, ids, prior)
    ("zipf-accumulate", 1000, 1024, 64, 4096, "zipf", "small"),
    ("zipf-large-prior", 1000, 1024, 64, 4096, "zipf", "large"),
    ("zipf-fresh", 1000, 1024, 64, 4096, "zipf", "zero"),
    ("edges", 131, 144, 64, 2048, "edges", "small"),
    ("one-id", 131, 144, 32, 8192, "one", "large"),
    ("uniform", 50257, 50304, 16, 2048, "uniform", "small"),
]
MUTANTS = ["per_occurrence", "ids_plus_one", "prior_dropped", "prior_twice", "padding_written"]


def margin_row(name, V, Vp, H, T, ids, prior):
    grad, x, dy = emb_inputs(V, Vp, H, T, ids, seed=V + T, prior=prior)
    o = emb_ref(grad, x, dy)
    bnd = emb_bound(o)
    emu = emb_checks(emulate_embedding_bwd(grad, x, dy), grad, o, bnd)
    caught = {}
    for m in MUTANTS:
        if m == "prior_dropped" and prior == "zero" or m == "prior_twice" and prior == "zero":
            continue                 # a zero prior: dropping or doubling it changes nothing
        c = emb_checks(emulate_embedding_bwd(grad, x, dy, mutant=m, V=V), grad, o, bnd)
        caught[m] = max(c.items(), key=lambda kv: kv[1])
    return emu, caught


def wpe_row():
    """Packed ``position_ids`` into a 1024-row position table: documents of 300, 700, 1024, 24 and 1000 tokens."""
    P, H, T = 1024, 64, 3072
    pos = packed_positions(T, [300, 700, 1024, 24, 1024])
    tok = zipf_ids(T, 50257, seed=3)
    grad, _, dy = emb_inputs(P, P, H, T, "uniform", seed=7)
    o = emb_ref(grad, pos, dy)
    bnd = emb_bound(o)
    emu = emb_checks(emulate_embedding_bwd(grad, pos, dy), grad, o, bnd)
    c = emb_checks(emulate_embedding_bwd(grad, pos, dy, mutant="wpe_token_ids", positions=tok), grad, o, bnd)
    return emu, {"wpe_token_ids": max(c.items(), key=lambda kv: kv[1])}


ROWS = {**{c[0]: (lambda c=c: margin_row(*c)) for c in CASES}, "wpe-packed": wpe_row}


@pytest.mark.parametrize("name", list(ROWS))
def test_margin_table(name):
    emu, caught = ROWS[name]()
    for k, r in emu.items():
        assert r <= 0.5, (name, "emulator", k, r)
    for m, (k, r) in caught.items():
        assert r > 3.0, (name, m, k, r)


def test_every_mutant_has_a_case():
    caught = set()
    for name, row in ROWS.items():
        caught |= set(row()[1])
    assert caught == set(MUTANTS) | {"wpe_token_ids"}


if __name__ == "__main__":               # print the margin table: python tests/test_step_oracle.py
    for name, row in ROWS.items():
        emu, caught = row()
        print(f"{name:18s} emulator/bound " + " ".join(f"{k}={v:.3f}" for k, v in emu.items()))
        print(" " * 19 + "mutants " + "  ".join(f"{m}: {k}={r:.3g}" for m, (k, r) in caught.items()))
