"""A native training step against HF in fp64 for every row layout and training objective: the harness, checked on the CPU.

``test_step_oracle.py`` compares a native step's gradients with HF's on full rows with ``labels = input_ids`` and plain (or
label-smoothed) cross-entropy.  This file extends that comparison, with the same criterion (``K_STEP``, ``FLOOR``, ``MIN_ROW_OCC``),
to the other row layouts and objectives a native step can train:

* layouts: full rows; document-masked pre-training rows (``DocumentCollator``); packed SFT rows (``PackedCollator``, prompts masked,
  a pad tail); right-padded SFT rows (``PadCollator``, prompts masked, one row fully ignored); preference pairs
  (``PreferenceCollator``, prompts masked, one invalid pair);
* objectives: cross-entropy with z-loss and label smoothing, distillation from a frozen teacher, DPO against a frozen reference,
  SimPO and ORPO.

The native side is the model's own loss (``model(input_ids, labels=, position_ids=, teacher_logits= | reference_logits= |
preference_pairs=True)``), one ``.backward()`` per micro-batch.  HF in fp64 is the oracle and HF in bf16 the yardstick; both take the
objective from their logits ``[..., :V]`` with the formulas the CPU oracles state (``test_z_loss.formula``, ``test_distill.formula``,
``test_dpo.trl_loss``, ``test_pref_free.trl_simpo`` / ``trl_orpo``), in fp64 on the oracle and in fp32 on the yardstick's logits.
HF has no document mask, so on document-masked and packed rows both HF sides run every document alone (positions from 0, which
also index GPT-Neo's ``wpe``), and the loss is the sum over all documents' targets divided by the micro-batch's number of targets:
the native mean.  The teacher's or reference's logits are computed once, from a frozen native model (``padded_logits``), and the
same tensor goes to all three sides.

Per case (``judge``): every gradient tensor and every embedding row hit ``MIN_ROW_OCC`` times within ``step_ratios``; the loss of
every micro-batch within ``|L - L64| <= K_STEP |L16 - L64| + FLOOR |L64|``; every logged device scalar (``z_loss_out``,
``distill_out``, ``dpo_out``, ``pref_out``) within the same criterion in the norms of ``step_ratios``, over the vector of its values
across the step's micro-batches (the chosen and rejected rewards as one vector): a reward is one small difference of two large
log-probability sums, and one number's yardstick error can be arbitrarily small by chance; the logged accuracies equal to fp64's except on pairs whose fp64 margin is
within ``K_STEP`` times the yardstick's error of it; the vocabulary padding rows of the embedding gradient exactly zero.  With the
reference equal to the policy (the first DPO step) the native rewards and accuracy are exactly 0: the policy's and the reference's
log-probabilities are the same numbers, so the fp64 reward (which sees the reference through its bf16 logits) measures the rounding
of that input, not the step; those three scalars are checked for exact zeros instead.

Here, on tiny models (V = 131 padded to 144), every layout and objective: the native path in fp32 within 1e-5 of fp64 (the
per-document split, the label shift, the normalisation and the teacher / reference plumbing of the harness), the native path in
bf16 near half the criterion, and every control (a native-side variant run against the unchanged oracle) out of it.  The same
cases at training widths, with the attention route and loss kernels proven from the launch counts, are in
``test_step_matrix_gpu.py``."""
from __future__ import annotations

import copy
import math
from dataclasses import dataclass, replace
from typing import Dict, List, Optional

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from test_distill import formula as kd_formula  # noqa: E402
from test_dpo import trl_loss as dpo_formula  # noqa: E402
from test_pref_free import _avg_logps, trl_orpo, trl_simpo  # noqa: E402
from test_step_oracle import (FLOOR, K_STEP, MIN_ROW_OCC, hf_from_native, hf_grads, native_grads, rel_err, step_ratios,  # noqa: E402
                              zipf_ids)
from test_z_loss import formula as z_formula  # noqa: E402

assert MIN_ROW_OCC == 16           # the row criterion of step_ratios, unchanged


# ================================================================================================= objectives
@dataclass(frozen=True)
class Objective:
    """``kind``: ``ce`` (with ``smoothing`` and ``z``), ``kd`` (``alpha``, ``T``), ``dpo`` (``beta``), ``simpo`` (``beta``, ``gamma``),
    ``orpo`` (``lam``)."""
    kind: str = "ce"
    smoothing: float = 0.0
    z: float = 0.0
    alpha: float = 0.5
    T: float = 1.0
    beta: float = 0.1
    gamma: float = 0.5
    lam: float = 0.1

    @property
    def pairs(self) -> bool:
        return self.kind in ("dpo", "simpo", "orpo")

    @property
    def scalars(self) -> List[str]:
        """The logged device scalars, in the order of the model's ``*_out`` tensor."""
        return {"ce": ["z_term"] if self.z else [], "kd": ["ce", "kl"], "dpo": ["chosen", "rejected", "acc"],
                "simpo": ["chosen", "rejected", "acc"], "orpo": ["nll", "log_odds", "acc"]}[self.kind]

    def label(self) -> str:
        return {"ce": f"ce(eps={self.smoothing}, z={self.z})", "kd": f"kd(a={self.alpha}, T={self.T})", "dpo": f"dpo(beta={self.beta})",
                "simpo": f"simpo(beta={self.beta}, gamma={self.gamma})", "orpo": f"orpo(lambda={self.lam})"}[self.kind]


def configure(model, obj: Objective) -> Optional[str]:
    """Set ``obj`` on a native model; returns the name of the ``*_out`` attribute that logs its scalars (None when none)."""
    model.label_smoothing = obj.smoothing if obj.kind == "ce" else 0.0
    model.z_loss_weight = obj.z if obj.kind == "ce" else 0.0
    model.distill_alpha, model.distill_temperature = obj.alpha, obj.T
    model.dpo_beta = obj.beta
    model.simpo_beta, model.simpo_gamma = (obj.beta, obj.gamma) if obj.kind == "simpo" else (None, 0.5)
    model.orpo_lambda = obj.lam if obj.kind == "orpo" else None
    return {"ce": "z_loss_out" if obj.z else None, "kd": "distill_out", "dpo": "dpo_out", "simpo": "pref_out",
            "orpo": "pref_out"}[obj.kind]


# ================================================================================================= row layouts
# A micro-batch is a dict of [B, S] int64 tensors: ``ids``, ``labels`` and, on document-masked and packed rows, ``pos``.

_RANKINGS: Dict[int, tuple] = {}


def _doc_tokens(n: int, V: int, rng) -> List[int]:
    """``n`` tokens with a Zipf(1) marginal over one fixed ranking of ``[0, V - 1)`` (never the EOS / pad id V - 1)."""
    if V not in _RANKINGS:
        p = 1.0 / np.arange(1, V, dtype=np.float64)
        _RANKINGS[V] = (p / p.sum(), np.random.default_rng(V).permutation(V - 1))
    p, perm = _RANKINGS[V]
    return perm[rng.choice(V - 1, size=n, p=p)].tolist()


def edge_starts(S: int, blk: int) -> List[int]:
    """Document starts one before, on and one after the first block edge (two one-token documents), then on or either side of the
    later edges."""
    return [blk - 1, blk, blk + 1] + [k * blk + d for k in range(2, S // blk) for d in ((0,) if k % 2 else (-1, 1))]


def zipf_lengths(S: int, rng) -> List[int]:
    """Document lengths ``0.6 S / r`` with ``r`` Zipf(1.3): a few long documents, many short ones, down to one token."""
    lens = []
    while sum(lens) < S:
        lens.append(max(1, int(0.6 * S / min(int(rng.zipf(1.3)), S))))
    return lens


def doc_batch(V: int, S: int, B: int, seed: int, blk: int) -> Dict[str, torch.Tensor]:
    """``DocumentCollator`` rows (EOS = V - 1): row 0 with ``edge_starts``, the others of ``zipf_lengths`` documents."""
    from acco_b200.data import DocumentCollator
    rng = np.random.default_rng(seed)
    rows = []
    for b in range(B):
        if b == 0:
            row = _doc_tokens(S, V, rng)
            for s in edge_starts(S, blk):
                row[s - 1] = V - 1
        else:
            row = []
            for n in zipf_lengths(S, rng):
                row += _doc_tokens(n - 1, V, rng) + [V - 1]
            row = row[:S]
        rows.append(np.asarray(row, dtype=np.int64))
    out = DocumentCollator(V - 1)([{"input_ids": r} for r in rows])
    return {"ids": out["input_ids"], "labels": out["labels"], "pos": out["position_ids"]}


def packed_batch(V: int, S: int, B: int, seed: int) -> Dict[str, torch.Tensor]:
    """``PackedCollator`` rows (pad = V - 1) of SFT samples with a pad tail; each sample's prompt (none on every second sample, so
    some segment starts carry only the collator's -100) masked to -100.  ``starts``: per row, the starts of the samples without a
    prompt (the ``packed_start_labels`` control)."""
    from acco_b200.data import PackedCollator
    rng = np.random.default_rng(seed)
    samples, prompts = [], []
    for b in range(B):
        lens = []
        while True:
            n = int(rng.integers(max(2, S // 32), S // 6))
            if sum(lens) + n > S - S // 8:
                break
            lens.append(n)
        toks = sum((_doc_tokens(n, V, rng) for n in lens), [])
        samples.append({"input_ids": toks, "doc_lens": lens})
        prompts.append([0 if i % 2 == 1 else int(rng.integers(1, n // 2 + 1)) for i, n in enumerate(lens)])
    out = PackedCollator(V - 1, S)(samples)
    labels = out["labels"].clone()
    bare = torch.zeros_like(labels, dtype=torch.bool)
    for b, (s, ks) in enumerate(zip(samples, prompts)):
        a = 0
        for n, k in zip(s["doc_lens"], ks):
            labels[b, a:a + k] = -100
            bare[b, a] = k == 0 and a > 0
            a += n
    return {"ids": out["input_ids"], "labels": labels, "pos": out["position_ids"], "bare_starts": bare}


def pad_batch(V: int, S: int, B: int, seed: int) -> Dict[str, torch.Tensor]:
    """``PadCollator`` rows (pad = V - 1, right padding to the longest row, which is S long): prompts masked, the last row fully
    ignored (its whole sequence is prompt)."""
    from acco_b200.data import PadCollator
    rng = np.random.default_rng(seed)
    lens = [S] + [int(rng.integers(S // 4, S)) for _ in range(B - 1)]
    rows = [_doc_tokens(n, V, rng) for n in lens]
    out = PadCollator(V - 1, max_length=S)([{"input_ids": r} for r in rows])
    labels = out["labels"].clone()
    for b, n in enumerate(lens):
        labels[b, :n if b == B - 1 else int(rng.integers(1, n // 2))] = -100
    assert out["input_ids"].shape == (B, S) and not bool((labels[-1] != -100).any())
    return {"ids": out["input_ids"], "labels": labels}


def pair_batch(V: int, S: int, P: int, seed: int) -> Dict[str, torch.Tensor]:
    """``PreferenceCollator`` rows (pad = V - 1): ``P`` pairs, the first filling S, the last with an empty rejected response (an
    invalid pair)."""
    from acco_b200.data import PreferenceCollator
    rng = np.random.default_rng(seed)
    pairs = []
    for i in range(P):
        k = int(rng.integers(S // 8, S // 4))
        c = S - k if i == 0 else int(rng.integers(S // 8, S - k))
        r = 0 if i == P - 1 else int(rng.integers(S // 8, S - k))
        pairs.append({"prompt_ids": _doc_tokens(k, V, rng), "chosen_ids": _doc_tokens(c, V, rng), "rejected_ids": _doc_tokens(r, V, rng)})
    out = PreferenceCollator(V - 1, max_length=S)(pairs)
    assert out["input_ids"].shape == (2 * P, S)
    return {"ids": out["input_ids"], "labels": out["labels"]}


def full_batch(V: int, S: int, B: int, seed: int) -> Dict[str, torch.Tensor]:
    ids = zipf_ids(B * S, V, seed=seed).view(B, S)
    return {"ids": ids, "labels": ids.clone()}


def make_batches(layout: str, V: int, S: int, B: int, n_acc: int, seed: int, device, blk: int = 128) -> List[Dict[str, torch.Tensor]]:
    """``n_acc`` micro-batches of ``layout`` (``full``, ``doc``, ``packed``, ``pad``, ``pairs``; ``B`` is ``P`` for pairs)."""
    out = []
    for i in range(n_acc):
        s = seed + 7919 * i
        mb = {"full": lambda: full_batch(V, S, B, s), "doc": lambda: doc_batch(V, S, B, s, blk), "packed": lambda: packed_batch(V, S, B, s),
              "pad": lambda: pad_batch(V, S, B, s), "pairs": lambda: pair_batch(V, S, B, s)}[layout]()
        out.append({k: v.to(device) for k, v in mb.items()})
    return out


# ================================================================================================= frozen models
def frozen_logits(model, batches) -> List[torch.Tensor]:
    """A frozen model's ``padded_logits`` of every micro-batch, computed once and fed to all three sides.  Taken with autograd on, as
    the training forward is, so a policy that is its own reference reproduces its training logits bit for bit."""
    with torch.enable_grad():
        return [model.padded_logits(mb["ids"], mb.get("pos")).detach() for mb in batches]


@torch.no_grad()
def perturbed(model, rel: float = 0.05, seed: int = 1):
    """A copy of ``model`` with every weight scaled by ``1 + rel N(0, 1)`` (vocabulary padding rows stay zero)."""
    m = copy.deepcopy(model)
    g = torch.Generator().manual_seed(seed)
    for p in m.parameters():
        p.mul_(1 + rel * torch.randn(p.shape, generator=g).to(p.device, p.dtype))
    return m


# ================================================================================================= the three sides
def native_step(model, batches, obj: Objective, frozen: Optional[List[torch.Tensor]] = None, use_pos: bool = True,
                labels_key: str = "labels"):
    """Forward + backward of every micro-batch through the native model's own loss, accumulating into ``.grad`` -> (loss per
    micro-batch, logged scalars per micro-batch)."""
    out_attr = configure(model, obj)
    for p in model.parameters():
        p.grad = None
    losses, scalars = [], []
    dev = next(model.parameters()).device
    for i, mb in enumerate(batches):
        kw = {}
        if obj.kind == "kd":
            kw["teacher_logits"] = frozen[i]
        elif obj.kind == "dpo":
            kw["reference_logits"] = frozen[i]
        elif obj.pairs:
            kw["preference_pairs"] = True
        if out_attr is not None:
            setattr(model, out_attr, torch.full((len(obj.scalars),), math.nan, device=dev, dtype=torch.float32))
        loss = model(mb["ids"], labels=mb[labels_key], position_ids=mb.get("pos") if use_pos else None, **kw).loss
        loss.backward()
        losses.append(float(loss.detach()))
        scalars.append({} if out_attr is None else dict(zip(obj.scalars, getattr(model, out_attr).tolist())))
        if out_attr is not None:
            setattr(model, out_attr, None)
    return losses, scalars


def target_rows(hf, mb, V: int, dtype, frozen: Optional[torch.Tensor] = None):
    """The logits ``[N, V]`` (``dtype``), targets ``[N]`` and frozen logits ``[N, V]`` of every position with a next token: whole
    rows, or with ``pos`` every document alone (documents with no target are not run)."""
    ids, lab = mb["ids"], mb["labels"]
    B, S = ids.shape
    fr = None if frozen is None else frozen.view(B, S, -1)[..., :V]
    xs, ys, ts = [], [], []
    if mb.get("pos") is None:
        xs.append(hf(input_ids=ids).logits[:, :-1, :V].reshape(-1, V))
        ys.append(lab[:, 1:].reshape(-1))
        if fr is not None:
            ts.append(fr[:, :-1].reshape(-1, V))
    else:
        pos = mb["pos"]
        for b in range(B):
            starts = torch.nonzero(pos[b] == 0).flatten().tolist() + [S]
            for a, e in zip(starts[:-1], starts[1:]):
                if not bool((lab[b, a + 1:e] != -100).any()):
                    continue                           # a one-token document, a pad tail or a prompt: nothing to learn
                xs.append(hf(input_ids=ids[b:b + 1, a:e]).logits[0, :-1, :V])
                ys.append(lab[b, a + 1:e])
                if fr is not None:
                    ts.append(fr[b, a:e - 1])
    x, y = torch.cat(xs).to(dtype), torch.cat(ys)
    return x, y, (torch.cat(ts).to(dtype) if ts else None)


def pair_terms(x3, labels, P: int, obj: Objective, r3=None):
    """The objective and its logged scalars on ``[2P, S, V]`` logits (TRL's formulas), and each pair's margin (the quantity whose
    sign is the logged accuracy) with the valid-pair mask."""
    l, cnt, a, mask = _avg_logps(x3, labels)
    valid = mask[:P].any(1) & mask[P:].any(1)
    if obj.kind == "dpo":
        loss = dpo_formula(x3, r3, labels, P, obj.beta)
        lr = _avg_logps(r3, labels)[0]
        rc, rr = obj.beta * (l[:P] - lr[:P]), obj.beta * (l[P:] - lr[P:])
        margin, logged = rc - rr, (rc, rr)
    elif obj.kind == "simpo":
        loss = trl_simpo(x3, labels, P, obj.beta, obj.gamma)
        margin, logged = a[:P] - a[P:], (obj.beta * a[:P], obj.beta * a[P:])
    else:
        loss = trl_orpo(x3, labels, P, obj.lam, clamp=True)
        lo = (a[:P] - a[P:]) - (torch.log1p(-torch.exp(a[:P])) - torch.log1p(-torch.exp(a[P:])))
        n_c = torch.where(valid, cnt[:P], torch.zeros_like(cnt[:P])).sum()
        nll = -torch.where(valid, l[:P], torch.zeros_like(l[:P])).sum() / n_c
        margin, logged = lo, (nll.expand(P), lo)
    n = valid.sum().clamp(min=1)
    vals = [float(torch.where(valid, v.detach(), torch.zeros_like(v)).sum() / n) for v in logged]
    vals.append(float((valid & (margin.detach() > 0)).sum() / n))
    return loss, dict(zip(obj.scalars, vals)), margin.detach(), valid


def hf_step(hf, batches, obj: Objective, V: int, frozen: Optional[List[torch.Tensor]] = None):
    """The oracle / yardstick step: the objective on HF's logits (fp64 on an fp64 model, fp32 on bf16 logits), one backward per
    micro-batch -> (losses, scalars, per micro-batch (margins, valid) of the pair objectives)."""
    dtype = torch.float64 if next(hf.parameters()).dtype == torch.float64 else torch.float32
    for p in hf.parameters():
        p.grad = None
    losses, scalars, margins = [], [], []
    for i, mb in enumerate(batches):
        fr = None if frozen is None else frozen[i]
        if obj.pairs:
            P = mb["ids"].shape[0] // 2
            x3 = hf(input_ids=mb["ids"]).logits[..., :V].to(dtype)
            r3 = None if fr is None else fr.view(2 * P, -1, fr.shape[-1])[..., :V].to(dtype)
            loss, sc, m, valid = pair_terms(x3, mb["labels"], P, obj, r3)
            margins.append((m, valid))
        else:
            x, y, t = target_rows(hf, mb, V, dtype, fr)
            valid = y != -100
            if obj.kind == "kd":
                loss = kd_formula(x, t, y, obj.alpha, obj.T)
                kl = F.kl_div(torch.log_softmax(x[valid] / obj.T, -1), torch.log_softmax(t[valid] / obj.T, -1), reduction="batchmean",
                              log_target=True)
                sc = {"ce": float(F.cross_entropy(x.detach(), y)), "kl": float(kl.detach())}
            else:
                loss = z_formula(x, y, obj.smoothing, obj.z)
                sc = {"z_term": float(obj.z * torch.logsumexp(x[valid].detach(), -1).square().mean())} if obj.z else {}
        loss.backward()
        losses.append(float(loss.detach()))
        scalars.append(sc)
    return losses, scalars, margins


def oracle_step(hf64, hf16, batches, obj: Objective, V: int, frozen=None) -> Dict:
    """Both HF sides of a case, computed once and judged against any number of native runs."""
    L64, s64, m64 = hf_step(hf64, batches, obj, V, frozen)
    L16, s16, m16 = hf_step(hf16, batches, obj, V, frozen)
    return {"g64": hf_grads(hf64), "g16": hf_grads(hf16), "L64": L64, "L16": L16, "s64": s64, "s16": s16, "m64": m64, "m16": m16}


def vector_ratio(x, x64, x16) -> float:
    """``scalar_ratio`` of the vectors of a logged quantity over a step's micro-batches, in the norms of ``step_ratios``: a single
    number's yardstick error can be arbitrarily small by chance, a vector's much less so."""
    x, x64, x16 = (torch.tensor(v, dtype=torch.float64) for v in (x, x64, x16))
    if not bool(torch.isfinite(x).all()):
        return math.inf
    num, den = float((x - x64).norm()), K_STEP * float((x16 - x64).norm()) + FLOOR * float(x64.norm())
    return num / den if den > 0 else (0.0 if num == 0 else math.inf)


def scalar_ratio(x: float, x64: float, x16: float) -> float:
    """``|x - x64| / (K_STEP |x16 - x64| + FLOOR |x64|)``: above 1 fails the criterion."""
    num, den = abs(x - x64), K_STEP * abs(x16 - x64) + FLOOR * abs(x64)
    if not math.isfinite(x):
        return math.inf
    return num / den if den > 0 else (0.0 if num == 0 else math.inf)


def judge(native, batches, obj: Objective, oracle: Dict, embed_key: str, frozen=None, use_pos: bool = True,
          labels_key: str = "labels", self_reference: bool = False) -> Dict:
    """Run the native step and measure it against ``oracle`` -> ``grad`` (the worst ``step_ratios`` entry), ``loss`` (worst over the
    micro-batches), ``scalars`` (name -> ``vector_ratio``), ``acc_off`` (accuracy miscounts beyond the ambiguous pairs), ``pad`` (largest
    |gradient| on the vocabulary padding rows), ``ratios`` (all of ``step_ratios``), ``worst`` (the largest of grad, loss, scalars)."""
    losses, scalars = native_step(native, batches, obj, frozen, use_pos, labels_key)
    ids = torch.cat([mb["ids"].reshape(-1) for mb in batches])
    r = step_ratios(native_grads(native), oracle["g64"], oracle["g16"], embed_key, ids)
    grad = max(r.items(), key=lambda kv: kv[1])
    loss = max(scalar_ratio(L, L64, L16) for L, L64, L16 in zip(losses, oracle["L64"], oracle["L16"]))
    acc_off, exact = 0.0, True
    pooled: Dict[str, List[tuple]] = {}
    for i, sc in enumerate(scalars):
        for k, v in sc.items():
            if self_reference and obj.kind == "dpo":
                exact = exact and v == 0.0               # policy = reference: the native rewards and accuracy are exactly 0
            elif k == "acc":
                (m64, valid), (m16, _) = oracle["m64"][i], oracle["m16"][i]
                n = int(valid.sum())
                ambiguous = int((valid & (m64.abs() <= K_STEP * (m16 - m64).abs())).sum())
                off = abs(v * n - float((valid & (m64 > 0)).sum()))
                acc_off = max(acc_off, max(0.0, off - ambiguous - 1e-3))
            else:
                name = "rewards" if k in ("chosen", "rejected") else k
                pooled.setdefault(name, []).append((v, oracle["s64"][i][k], oracle["s16"][i][k]))
    sr = {k: vector_ratio(*zip(*vals)) for k, vals in pooled.items()}
    pads = [native.embed_weight.grad[native.config.vocab_size:]]
    if native.lm_head is not None:
        pads.append(native.lm_head.grad[native.config.vocab_size:])
    pad = max(float(t.abs().max()) if t.numel() else 0.0 for t in pads)
    worst = max([grad[1], loss] + list(sr.values()))
    return {"grad": grad, "loss": loss, "scalars": sr, "acc_off": acc_off, "exact_zero": exact, "pad": pad, "ratios": r, "worst": worst,
            "losses": losses, "logged": scalars}


def report(name: str, j: Dict) -> str:
    s = " ".join(f"{k}={v:.3f}" for k, v in j["scalars"].items())
    return (f"{name}: worst grad ratio {j['grad'][1]:.3f} ({j['grad'][0]}), loss ratio {j['loss']:.3f}"
            + (f", scalar ratios {s}" if s else "") + (f", accuracy miscounts {j['acc_off']:g}" if j["acc_off"] else ""))


def assert_meets(name: str, j: Dict, bound: float = 1.0) -> None:
    assert j["grad"][1] <= bound, (name, j["ratios"])
    assert j["loss"] <= bound, (name, j["losses"])
    assert all(v <= bound for v in j["scalars"].values()), (name, j["scalars"], j["logged"])
    assert j["acc_off"] == 0.0 and j["exact_zero"], (name, j["logged"])
    assert j["pad"] == 0.0, (name, "vocabulary padding rows", j["pad"])


# ================================================================================================= CPU cases (tiny models)
def tiny(arch: str, dtype, hidden: int = 64):
    from acco_b200.models import GPTConfig, GPTForCausalLM, LlamaConfig, LlamaForCausalLM
    torch.manual_seed(0)
    if arch == "gptneo":
        m = GPTForCausalLM(GPTConfig(vocab_size=131, hidden_size=hidden, num_hidden_layers=2, num_attention_heads=4,
                                     max_position_embeddings=64, window_size=8, pad_vocab_multiple=16))
    else:
        m = LlamaForCausalLM(LlamaConfig(vocab_size=131, hidden_size=hidden, intermediate_size=2 * hidden, num_hidden_layers=2,
                                         num_attention_heads=4, num_key_value_heads=2, max_position_embeddings=64, pad_vocab_multiple=16))
    return m.to(dtype)


def embed_key(arch: str) -> str:
    return "transformer.wte.weight" if arch == "gptneo" else "model.embed_tokens.weight"


Z = Objective(z=1e-2)
CPU_CASES = {
    # name: (arch, layout, B (P for pairs), S, n_acc, objective, frozen model: None | teacher | self | perturbed)
    "llama-doc": ("llama", "doc", 3, 64, 1, Objective(), None),
    "gptneo-doc": ("gptneo", "doc", 3, 64, 1, Objective(), None),
    "llama-packed": ("llama", "packed", 3, 64, 1, Objective(), None),
    "gptneo-packed": ("gptneo", "packed", 3, 64, 1, Objective(), None),
    "llama-pad": ("llama", "pad", 4, 60, 1, Objective(), None),
    "llama-z1e-4": ("llama", "full", 4, 32, 1, Objective(z=1e-4), None),
    "llama-z1e-2-smooth": ("llama", "full", 4, 32, 1, Objective(z=1e-2, smoothing=0.1), None),
    "gptneo-z1e-2": ("gptneo", "full", 4, 32, 1, Z, None),
    "llama-kd-a0.5-T2": ("llama", "full", 4, 32, 1, Objective("kd", alpha=0.5, T=2.0), "teacher"),
    "llama-kd-a1-T2": ("llama", "full", 4, 32, 1, Objective("kd", alpha=1.0, T=2.0), "teacher"),
    "llama-dpo-self": ("llama", "pairs", 4, 32, 1, Objective("dpo"), "self"),
    "llama-dpo-perturbed": ("llama", "pairs", 4, 32, 1, Objective("dpo"), "perturbed"),
    "gptneo-dpo-perturbed": ("gptneo", "pairs", 4, 32, 1, Objective("dpo"), "perturbed"),
    "llama-simpo": ("llama", "pairs", 4, 32, 1, Objective("simpo", beta=2.0, gamma=0.5), None),
    "llama-orpo": ("llama", "pairs", 4, 32, 1, Objective("orpo", lam=0.1), None),
    "llama-doc-nacc4": ("llama", "doc", 2, 64, 4, Objective(), None),
    "llama-z-nacc4": ("llama", "full", 2, 32, 4, Objective(z=1e-2, smoothing=0.1), None),
    "llama-dpo-nacc4": ("llama", "pairs", 2, 32, 4, Objective("dpo"), "perturbed"),
}

# name: (case, native-side change: {"obj": Objective fields} | {"use_pos": False} | {"labels_key": ...})
CONTROLS = {
    "doc-without-position-ids": ("llama-doc", {"use_pos": False}),
    "packed-start-labels-kept": ("llama-packed", {"labels_key": "start_labels"}),
    "z-loss-doubled": ("llama-z1e-2-smooth", {"obj": dict(z=2e-2)}),
    "distill-T1-vs-T2": ("llama-kd-a1-T2", {"obj": dict(T=1.0)}),
    "dpo-beta-doubled": ("llama-dpo-perturbed", {"obj": dict(beta=0.2)}),
    "simpo-gamma-0-vs-0.5": ("llama-simpo", {"obj": dict(gamma=0.0)}),
    "orpo-lambda-doubled": ("llama-orpo", {"obj": dict(lam=0.2)}),
}


def with_start_labels(batches) -> None:
    """The ``packed-start-labels-kept`` control's labels: every prompt-less sample's start keeps its token as label."""
    for mb in batches:
        if "bare_starts" in mb:
            mb["start_labels"] = torch.where(mb["bare_starts"], mb["ids"], mb["labels"])


def frozen_for(kind: Optional[str], native, batches, arch: str, make) -> Optional[List[torch.Tensor]]:
    """The frozen logits of a case: ``teacher`` a wider model of the same vocabulary, ``self`` the policy, ``perturbed`` a perturbed
    copy of it.  ``make(arch, hidden)`` builds the teacher."""
    if kind is None:
        return None
    model = {"teacher": lambda: make(arch, 2 * native.config.hidden_size), "self": lambda: native, "perturbed": lambda: perturbed(native)}[kind]()
    return frozen_logits(model, batches)


def cpu_case(name: str, dtype):
    arch, layout, B, S, n_acc, obj, fr = CPU_CASES[name]
    native = tiny(arch, dtype)
    batches = make_batches(layout, 131, S, B, n_acc, seed=11, device="cpu", blk=16)
    frozen = frozen_for(fr, native, batches, arch, lambda a, h: tiny(a, dtype, hidden=h))
    return native, batches, obj, frozen, arch, fr


def test_layouts_have_their_edges():
    """The rows the cases run: document starts on and beside block edges with one-token documents, GPT-Neo documents longer than
    its window, prompt-less packed samples and a pad tail, a fully ignored padded row, an invalid preference pair."""
    d = doc_batch(131, 64, 3, 11, 16)
    starts = [torch.nonzero(d["pos"][b] == 0).flatten().tolist() for b in range(3)]
    assert {15, 16, 17} <= set(starts[0]) and len(starts[1]) >= 2
    lens = [e - a for st in starts for a, e in zip(st, st[1:] + [64])]
    assert 1 in lens and sum(n > 8 for n in lens) >= 3
    p = packed_batch(131, 64, 3, 11)
    assert bool(p["bare_starts"].any()) and bool((p["ids"][:, -1] == 130).all()) and bool((p["labels"][:, -1] == -100).all())
    assert not bool((pad_batch(131, 60, 4, 11)["labels"][-1] != -100).any())
    q = pair_batch(131, 32, 4, 11)["labels"]
    assert not bool((q[-1] != -100).any()) and all(bool((q[i] != -100).any()) for i in range(7))
    big = doc_batch(50257, 1024, 4, 100, 128)
    starts = [torch.nonzero(big["pos"][b] == 0).flatten().tolist() for b in range(4)]
    assert {127, 128, 129} <= set(starts[0])
    assert sum(e - a > 256 for st in starts for a, e in zip(st, st[1:] + [1024])) >= 3


@pytest.mark.parametrize("name", list(CPU_CASES))
def test_native_fp32_matches_fp64(name):
    """The native path in fp32 against HF fp64: every gradient, every micro-batch's loss and every logged scalar within 1e-5."""
    pytest.importorskip("transformers")
    native, batches, obj, frozen, arch, fr = cpu_case(name, torch.float32)
    hf64 = hf_from_native(native, torch.float64, "cpu")
    L64, s64, m64 = hf_step(hf64, batches, obj, 131, frozen)
    losses, scalars = native_step(native, batches, obj, frozen)
    ours, ref = native_grads(native), hf_grads(hf64)
    for k in ref:
        assert float(rel_err(ours[k], ref[k])) < 1e-5, (name, k, float(rel_err(ours[k], ref[k])))
    for L, want in zip(losses, L64):
        assert abs(L - want) <= 1e-5 * abs(want), (name, L, want)
    for sc, want in zip(scalars, s64):
        assert set(sc) == set(obj.scalars)
        for k, v in sc.items():
            if fr == "self":
                assert v == 0.0, (name, k, v)
            else:
                assert abs(v - want[k]) <= 1e-5 * max(abs(want[k]), 1.0), (name, k, v, want[k])   # rewards are differences
    assert not native.embed_weight.grad[131:].any()


@pytest.mark.parametrize("name", list(CPU_CASES))
def test_native_bf16_within_the_criterion(name):
    """The native CPU path in bf16 against HF bf16, both measured against HF fp64: an honest bf16 step, of the yardstick's accuracy,
    lands near half the criterion (worst tensor 0.39 - 0.51 over these cases); asserted with a margin, at 0.6.  The loss within half
    the criterion, the logged scalars within it."""
    pytest.importorskip("transformers")
    native, batches, obj, frozen, arch, fr = cpu_case(name, torch.bfloat16)
    o = oracle_step(hf_from_native(native, torch.float64, "cpu"), hf_from_native(native, torch.bfloat16, "cpu"), batches, obj, 131, frozen)
    j = judge(native, batches, obj, o, embed_key(arch), frozen, self_reference=fr == "self")
    print(report(name, j))
    assert j["grad"][1] <= 0.6 and j["loss"] <= 0.5, (name, j["ratios"], j["losses"])
    assert_meets(name, j)


@pytest.mark.parametrize("name", list(CONTROLS))
def test_control_fails(name):
    """Each control, on the native bf16 CPU path against the unchanged oracle, is out of the criterion."""
    pytest.importorskip("transformers")
    case, change = CONTROLS[name]
    native, batches, obj, frozen, arch, fr = cpu_case(case, torch.bfloat16)
    o = oracle_step(hf_from_native(native, torch.float64, "cpu"), hf_from_native(native, torch.bfloat16, "cpu"), batches, obj, 131, frozen)
    with_start_labels(batches)
    j = judge(native, batches, replace(obj, **change.get("obj", {})), o, embed_key(arch), frozen, use_pos=change.get("use_pos", True),
              labels_key=change.get("labels_key", "labels"))
    print(f"control {name}: " + report(case, j))
    assert j["worst"] > 1.0, (name, j["worst"])
