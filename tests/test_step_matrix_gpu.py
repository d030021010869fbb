"""A native training step at training widths (2 layers) on the H100 against HF in fp64, for every attention route, row layout and
training objective: the harness and criterion of ``test_step_matrix.py`` (``K_STEP``, ``FLOOR``, ``MIN_ROW_OCC`` of
``test_step_oracle.py``), on the kernels.

* Full rows with plain / smoothed cross-entropy, the six cases of ``test_step_oracle_gpu.py``, on the own flash-attention kernels
  (``ACCO_ATTN=own``; the default route is covered there).
* Document-masked pre-training rows (``DocumentCollator``: one row with starts at 127 / 128 / 129 and beside later 128-block edges,
  the others of Zipf-length documents, several GPT-Neo documents longer than its 256 window) at Llama-125M (S = 1024), Llama-3.2-1B
  (GQA 32 / 8, S = 2048) and GPT-Neo-125M widths, and packed SFT rows (``PackedCollator``: prompts masked, a pad tail) at Llama-125M
  and GPT-Neo-125M widths, each on the default and the own route (both run the segmented kernels).
* Right-padded SFT rows (``PadCollator``: prompts masked, one row fully ignored) at S = 1000 on the own route, which falls back to
  SDPA there (S % 128 != 0).
* Full rows with the z-loss (1e-4 and 1e-2, alone and with label smoothing 0.1; GPT-Neo at 1e-2), distillation from a wider native
  Llama (``a, T`` = (0.5, 1), (0.5, 2), (1, 2)), DPO against the policy itself and against a perturbed copy (Llama and GPT-Neo),
  SimPO (beta 2, gamma 0.5) and ORPO (lambda 0.1) on preference pairs (P = 4, S = 1024, prompts masked, one invalid pair).
* Document-masked CE, z-loss and DPO at ``n_acc = 4``.

Each case asserts the gradient, loss and logged-scalar criterion, the vocabulary padding rows, and the route it claims from
``ops.launch_counts()``: the plain or segmented attention kernels, or none, and the loss kernel (``ce_fwd`` / ``kd_fwd`` /
``dpo_fwd`` / ``pref_reduce``).  Each control (``CONTROLS`` of ``test_step_matrix.py``: document rows without ``position_ids``,
packed rows that keep labels at sample starts, the z weight doubled, distillation at T = 1 against an oracle at T = 2, DPO beta
doubled, SimPO gamma 0 against 0.5, ORPO lambda doubled) runs against the unchanged oracle and must land out of the criterion.
Run with ``-s`` to see every case's ratios, route, controls and peak memory."""
import time
from dataclasses import replace

import pytest
import torch

pytestmark = pytest.mark.gpu

from acco_b200 import ops  # noqa: E402

from test_step_matrix import (CONTROLS, Objective, assert_meets, embed_key, frozen_logits, judge, make_batches, oracle_step,  # noqa: E402
                              perturbed, report, with_start_labels)
from test_step_oracle import hf_from_native, zipf_ids  # noqa: E402
from test_step_oracle_gpu import GPTNEO125, LLAMA1B, LLAMA125, STEP_CASES  # noqa: E402

DEV = "cuda"
TEACHER = dict(LLAMA125, hidden_size=1024, intermediate_size=2816, num_attention_heads=16, num_key_value_heads=16)
MODELS = {"llama125m": ("llama", LLAMA125), "llama1b": ("llama", LLAMA1B), "gptneo125m": ("gptneo", GPTNEO125)}
ATTN = ("attn_fwd", "attn_bwd", "attn_fwd_seg", "attn_bwd_seg")
LOSS = ("ce_fwd", "kd_fwd", "dpo_fwd", "pref_reduce")

CE = Objective()
MATRIX = {
    # name: (model, layout, B (P for pairs), S, n_acc, objective, frozen model, routes, controls)
    "llama125m-doc": ("llama125m", "doc", 4, 1024, 1, CE, None, ("default", "own"), ("doc-without-position-ids",)),
    "llama1b-doc": ("llama1b", "doc", 2, 2048, 1, CE, None, ("default", "own"), ()),
    "gptneo125m-doc": ("gptneo125m", "doc", 4, 1024, 1, CE, None, ("default", "own"), ()),
    "llama125m-packed": ("llama125m", "packed", 4, 1024, 1, CE, None, ("default", "own"), ("packed-start-labels-kept",)),
    "gptneo125m-packed": ("gptneo125m", "packed", 4, 1024, 1, CE, None, ("default", "own"), ()),
    "llama125m-pad-s1000": ("llama125m", "pad", 4, 1000, 1, CE, None, ("own",), ()),
    "llama125m-z1e-4": ("llama125m", "full", 4, 1024, 1, Objective(z=1e-4), None, ("default",), ()),
    "llama125m-z1e-4-smooth0.1": ("llama125m", "full", 4, 1024, 1, Objective(z=1e-4, smoothing=0.1), None, ("default",), ()),
    "llama125m-z1e-2": ("llama125m", "full", 4, 1024, 1, Objective(z=1e-2), None, ("default",), ()),
    "llama125m-z1e-2-smooth0.1": ("llama125m", "full", 4, 1024, 1, Objective(z=1e-2, smoothing=0.1), None, ("default",),
                                  ("z-loss-doubled",)),
    "gptneo125m-z1e-2": ("gptneo125m", "full", 4, 1024, 1, Objective(z=1e-2), None, ("default",), ()),
    "llama125m-kd-a0.5-T1": ("llama125m", "full", 4, 1024, 1, Objective("kd", alpha=0.5, T=1.0), "teacher", ("default",), ()),
    "llama125m-kd-a0.5-T2": ("llama125m", "full", 4, 1024, 1, Objective("kd", alpha=0.5, T=2.0), "teacher", ("default",), ()),
    "llama125m-kd-a1-T2": ("llama125m", "full", 4, 1024, 1, Objective("kd", alpha=1.0, T=2.0), "teacher", ("default",),
                           ("distill-T1-vs-T2",)),
    "llama125m-dpo-self": ("llama125m", "pairs", 4, 1024, 1, Objective("dpo"), "self", ("default",), ()),
    "llama125m-dpo-perturbed": ("llama125m", "pairs", 4, 1024, 1, Objective("dpo"), "perturbed", ("default",), ("dpo-beta-doubled",)),
    "gptneo125m-dpo-self": ("gptneo125m", "pairs", 4, 1024, 1, Objective("dpo"), "self", ("default",), ()),
    "gptneo125m-dpo-perturbed": ("gptneo125m", "pairs", 4, 1024, 1, Objective("dpo"), "perturbed", ("default",), ()),
    "llama125m-simpo": ("llama125m", "pairs", 4, 1024, 1, Objective("simpo", beta=2.0, gamma=0.5), None, ("default",),
                        ("simpo-gamma-0-vs-0.5",)),
    "llama125m-orpo": ("llama125m", "pairs", 4, 1024, 1, Objective("orpo", lam=0.1), None, ("default",), ("orpo-lambda-doubled",)),
    "llama125m-doc-nacc4": ("llama125m", "doc", 2, 1024, 4, CE, None, ("default",), ()),
    "llama125m-z1e-2-smooth0.1-nacc4": ("llama125m", "full", 2, 1024, 4, Objective(z=1e-2, smoothing=0.1), None, ("default",), ()),
    "llama125m-dpo-perturbed-nacc4": ("llama125m", "pairs", 4, 1024, 4, Objective("dpo"), "perturbed", ("default",), ()),
}

_CACHE = {}


def models(key: str, arch: str, cfg: dict):
    """The native bf16 model and its HF bf16 / fp64 twins; one set is kept between tests (the cases are grouped by model)."""
    if key not in _CACHE:
        _CACHE.clear()
        torch.cuda.empty_cache()
        from acco_b200.models import GPTConfig, GPTForCausalLM, LlamaConfig, LlamaForCausalLM
        torch.manual_seed(0)
        native = (GPTForCausalLM(GPTConfig(**cfg)) if arch == "gptneo" else LlamaForCausalLM(LlamaConfig(**cfg))).to(DEV).to(torch.bfloat16)
        _CACHE[key] = (native, hf_from_native(native, torch.bfloat16, DEV, attn="sdpa"), hf_from_native(native, torch.float64, DEV))
    return _CACHE[key]


def teacher():
    from acco_b200.models import LlamaConfig, LlamaForCausalLM
    torch.manual_seed(1)
    return LlamaForCausalLM(LlamaConfig(**TEACHER)).to(DEV).to(torch.bfloat16)


def expected_route(layout: str, route: str, S: int) -> str:
    if layout in ("doc", "packed"):
        return "segmented"                              # packed rows take the segmented kernels on either route
    return "own" if route == "own" and S % 128 == 0 else "none"


def check_route(counts: dict, want: str, obj: Objective, layers: int, n_acc: int) -> str:
    """Assert the attention kernels and the loss kernel the launch counts show; returns them as text."""
    attn = {k: counts.get(k, 0) for k in ATTN}
    n = layers * n_acc
    expect = {"own": {"attn_fwd": n, "attn_bwd": 2 * n}, "segmented": {"attn_fwd_seg": n, "attn_bwd_seg": 2 * n}, "none": {}}[want]
    assert attn == {k: expect.get(k, 0) for k in ATTN}, (want, counts)
    loss = {"ce": "ce_fwd", "kd": "kd_fwd", "dpo": "dpo_fwd", "simpo": "pref_reduce", "orpo": "pref_reduce"}[obj.kind]
    others = [k for k in LOSS if k != loss and not (k == "ce_fwd" and loss == "pref_reduce")]
    assert counts.get(loss, 0) > 0 and all(counts.get(k, 0) == 0 for k in others), (obj, counts)
    return f"attention {want} {({k: v for k, v in attn.items() if v})}, loss kernel {loss}"


def run_routes(name, native, batches, obj, oracle, ekey, frozen, routes, layout, S, n_acc, monkeypatch, self_reference=False):
    for route in routes:
        if route == "own":
            monkeypatch.setenv("ACCO_ATTN", "own")
        else:
            monkeypatch.delenv("ACCO_ATTN", raising=False)
        ops.reset_launch_counts()
        j = judge(native, batches, obj, oracle, ekey, frozen, self_reference=self_reference)
        torch.cuda.synchronize()
        route_text = check_route(ops.launch_counts(), expected_route(layout, route, S), obj, native.config.num_hidden_layers, n_acc)
        print(f"[step matrix] {report(f'{name} ({obj.label()}, route {route})', j)}; {route_text}")
        assert_meets(name, j)
    monkeypatch.delenv("ACCO_ATTN", raising=False)


@pytest.mark.parametrize("case", STEP_CASES, ids=[c[0] for c in STEP_CASES])
def test_full_rows_on_the_own_attention_kernels(case, monkeypatch):
    name, arch, cfg, B, S, n_acc, smoothing = case
    t0 = time.time()
    torch.cuda.reset_peak_memory_stats()
    native, hf16, hf64 = models(name, arch, cfg)
    V = native.config.vocab_size
    batches = [{"ids": ids, "labels": ids} for ids in (zipf_ids(B * S, V, seed=100 + i).view(B, S).to(DEV) for i in range(n_acc))]
    obj = Objective(smoothing=smoothing)
    oracle = oracle_step(hf64, hf16, batches, obj, V)
    run_routes(name, native, batches, obj, oracle, embed_key(arch), None, ("own",), "full", S, n_acc, monkeypatch)
    print(f"[step matrix] {name}: {time.time() - t0:.1f} s, peak memory {torch.cuda.max_memory_allocated() / 2**30:.1f} GiB")


@pytest.mark.parametrize("name", list(MATRIX))
def test_step_matrix(name, monkeypatch):
    key, layout, B, S, n_acc, obj, fr, routes, controls = MATRIX[name]
    arch, cfg = MODELS[key]
    t0 = time.time()
    torch.cuda.reset_peak_memory_stats()
    native, hf16, hf64 = models(key, arch, cfg)
    V = native.config.vocab_size
    monkeypatch.delenv("ACCO_ATTN", raising=False)
    batches = make_batches(layout, V, S, B, n_acc, seed=100, device=DEV)
    if arch == "gptneo" and layout == "doc":
        starts = [torch.nonzero(row == 0).flatten().tolist() for mb in batches for row in mb["pos"]]
        lens = [e - a for st in starts for a, e in zip(st, st[1:] + [S])]
        assert sum(n > 256 for n in lens) >= 2, lens                  # documents that outgrow the local window
    frozen = None
    if fr == "teacher":
        frozen = frozen_logits(teacher(), batches)
    elif fr == "self":
        frozen = frozen_logits(native, batches)
    elif fr == "perturbed":
        frozen = frozen_logits(perturbed(native), batches)
    oracle = oracle_step(hf64, hf16, batches, obj, V, frozen)
    run_routes(name, native, batches, obj, oracle, embed_key(arch), frozen, routes, layout, S, n_acc, monkeypatch,
               self_reference=fr == "self")
    for c in controls:
        change = CONTROLS[c][1]
        with_start_labels(batches)
        j = judge(native, batches, replace(obj, **change.get("obj", {})), oracle, embed_key(arch), frozen,
                  use_pos=change.get("use_pos", True), labels_key=change.get("labels_key", "labels"))
        print(f"[step matrix] control {c}: worst ratio {j['worst']:.3g} ({report(name, j)})")
        assert j["worst"] > 1.0, (c, j)
    print(f"[step matrix] {name}: {time.time() - t0:.1f} s, peak memory {torch.cuda.max_memory_allocated() / 2**30:.1f} GiB")
