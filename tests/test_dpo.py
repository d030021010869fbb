"""DPO against a frozen reference (``train.dpo_beta`` / ``DecoupledTrainer(reference=...)``): the fp64 oracle of the ``dpo_*`` kernels
and its per-element bounds, the margin table of a blockwise fp32 emulator and its mutants, the collator, and the op, model and
trainer routes.  Runs on the CPU without the extension; ``test_dpo_gpu.py`` runs the kernels against the same oracle.

Semantics (``P`` pairs as ``[2P, S]`` rows, chosen rows first; policy logits ``s``, reference logits ``r``; ``R(row)`` the positions
whose shifted label is not -100)::

    d_t    = (s_t[y_t] - lse(s_t)) - (r_t[y_t] - lse(r_t))             (t in R; else 0)
    D(row) = sum_t d_t,   z_i = beta (D(i) - D(P + i)),   valid_i = both rows non-empty,   n = #valid
    loss   = sum_valid softplus(-z_i) / n,   w(i) = beta sigma(-z_i) / n = -w(P + i)    (invalid: 0)
    ds_tc  = dloss w(row) (softmax(s_t)_c - [c = y_t])                  (c < V, t in R; else 0)
    out    = (mean beta D(chosen), mean beta D(rejected), mean [z > 0]) over the valid pairs

Bounds: each ``lse`` as in the CE oracle; ``d_t`` adds both log-probabilities' roundings; a row sum of ``S`` terms is
``ceil(S / 32) + 5`` fp32 adds deep; ``z`` adds three roundings; ``softplus`` and ``sigma`` get ``sigma(-z) E_z`` (resp.
``sigma(1 - sigma) E_z``) plus the error of ``__expf`` and a few roundings; the pair means are a ``block_sum`` over at most 1024
values (10 adds deep).  The gradient is ``|dloss| (|w| E_p + |p - oh| E_w)`` plus three roundings, and one bf16 ulp.  Everything is
doubled, as elsewhere.

The margin table asserts the emulator stays within half of every bound and that each mutant (beta missing, chosen and rejected
swapped, reference ignored, prompt tokens counted, mean instead of sum, an invalid pair counted) lands far outside on some case.
Print it with ``python tests/test_dpo.py``."""
from __future__ import annotations

import functools
import json
import math
import os
import sys
from typing import Dict, Optional

import pytest
import torch
import torch.nn.functional as F

from test_distill import _lse_bound, _logged, _tensors, _write_hf_dir, emulate_kd  # noqa: E402
from test_gemm_oracle import bf16_rn  # noqa: E402
from test_rowwise_oracle import FTZ, U, e_exp, f32, out_bound, ratio  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LN2 = math.log(2.0)


# ================================================================================================= TRL's formulation
def trl_loss(s: torch.Tensor, r: torch.Tensor, labels: torch.Tensor, P: int, beta: float) -> torch.Tensor:
    """TRL ``DPOTrainer``'s sigmoid loss on ``[2P, S, V]`` logits and unshifted ``[2P, S]`` labels: ``log_softmax``, gather over the
    response tokens, ``-F.logsigmoid``; the mean is over the pairs whose two rows both have a response token."""
    lb = labels[:, 1:]
    mask = lb != -100
    idx = torch.where(mask, lb, torch.zeros_like(lb))[..., None]

    def logps(x):
        return (torch.log_softmax(x[:, :-1], -1).gather(-1, idx)[..., 0] * mask).sum(-1)

    lp, lr = logps(s), logps(r.detach())
    z = beta * ((lp[:P] - lr[:P]) - (lp[P:] - lr[P:]))
    valid = mask[:P].any(1) & mask[P:].any(1)
    return torch.where(valid, -F.logsigmoid(z), torch.zeros_like(z)).sum() / valid.sum().clamp(min=1)


def shift(labels: torch.Tensor) -> torch.Tensor:
    """The models' HF shift: position t predicts token t + 1; the last position has no target."""
    out = torch.full_like(labels, -100)
    out[:, :-1] = labels[:, 1:]
    return out.reshape(-1)


# ================================================================================================= fp64 oracle
def dpo_token_terms(s, r, labels, V: int, ignore_index: int = -100) -> Dict:
    """Per token row of ``[T, Vp]`` logits (on their device, fp64): ``lse(s)`` and its bound, ``d`` and its bound (0 off ``R``)."""
    x, y = s[:, :V].double(), r[:, :V].double()
    vt = labels != ignore_index
    lab = torch.where(vt, labels, torch.zeros_like(labels))
    lse1, lse2 = torch.logsumexp(x, 1), torch.logsumexp(y, 1)
    lp1, lp2 = x.gather(1, lab[:, None])[:, 0] - lse1, y.gather(1, lab[:, None])[:, 0] - lse2
    z0 = torch.zeros_like(lse1)
    d = torch.where(vt, lp1 - lp2, z0)
    E1, _ = _lse_bound(x, lse1, V, False)
    E2, _ = _lse_bound(y, lse2, V, False)
    E_d = torch.where(vt, E1 + E2 + 2 * U * (lp1.abs() + lp2.abs()) + U * d.abs(), z0)
    return {"lse": lse1, "E_lse": E1, "d": d, "E_d": E_d, "vt": vt}


def dpo_grad_ref(s, labels, lse1, E1, w_t, E_w_t, V: int, dloss: float, ignore_index: int = -100):
    """d-logits of token rows ``s`` (fp64) and their bounds, given each row's weight ``w_t`` and its bound."""
    Tn, Vp = s.shape
    x = s[:, :V].double()
    vt = labels != ignore_index
    lab = torch.where(vt, labels, torch.zeros_like(labels))
    p = torch.exp(x - lse1[:, None])
    oh = torch.zeros_like(p)
    oh.scatter_(1, lab[:, None], 1.0)
    g = dloss * w_t[:, None] * (p - oh)
    E_p = p * (E1[:, None] + U * (x - lse1[:, None]).abs() + e_exp(x - lse1[:, None]))
    E = 2 * (abs(dloss) * (w_t.abs()[:, None] * E_p + (p - oh).abs() * E_w_t[:, None]) + 3 * U * g.abs())
    grad = torch.zeros(Tn, Vp, dtype=torch.float64, device=x.device)
    bnd = torch.full((Tn, Vp), FTZ, dtype=torch.float64, device=x.device)
    grad[:, :V] = torch.where(vt[:, None], g, torch.zeros_like(g))
    bnd[:, :V] = torch.where(vt[:, None], out_bound(g, E), torch.full_like(g, FTZ))
    return grad, bnd


def dpo_ref(s, r, labels, P: int, V: int, beta: float, dloss: Optional[float] = None, ignore_index: int = -100,
            terms: Optional[Dict] = None) -> Dict:
    """fp64 oracle of the ``dpo_*`` kernels on ``[2P S, Vp]`` logits and shifted labels ``[2P S]``, bounds included (``terms``: the
    :func:`dpo_token_terms` of all rows, computed elsewhere)."""
    tt = dpo_token_terms(s, r, labels, V, ignore_index) if terms is None else terms
    tt = {k: v.cpu() for k, v in tt.items()}
    Tn = tt["d"].numel()
    S = Tn // (2 * P)
    d, E_d, vt = tt["d"], tt["E_d"], tt["vt"]
    D = d.view(2 * P, S).sum(1)
    cnt = vt.view(2 * P, S).sum(1)
    E_D = E_d.view(2 * P, S).sum(1) + (-(-S // 32) + 5) * U * d.abs().view(2 * P, S).sum(1)
    valid = (cnt[:P] > 0) & (cnt[P:] > 0)
    n = int(valid.sum())
    inv = 1.0 / n if n else 0.0
    rc, rr = beta * D[:P], beta * D[P:]
    z = rc - rr
    E_rc, E_rr = beta * E_D[:P] + U * rc.abs(), beta * E_D[P:] + U * rr.abs()
    E_z = E_rc + E_rr + U * z.abs()
    sp = torch.logaddexp(torch.zeros_like(z), -z)
    sig = torch.sigmoid(-z)
    e = torch.exp(-z.abs())
    E_sp = sig * E_z + e * e_exp(z.abs()) + 4 * U * (sp + z.abs())
    pair = torch.zeros_like(z)
    vsum = lambda v: float(torch.where(valid, v, pair).sum())
    mean_b = lambda sv, sa: 2 * ((sv + 12 * U * sa) * inv + 4 * U * sa * inv) + FTZ
    loss = vsum(sp) * inv
    acc = vsum((z > 0).double()) * inv
    amb = vsum((z.abs() <= 2 * E_z).double())          # pairs whose sign the fp32 z may flip
    z0 = torch.zeros_like(tt["lse"])
    res = {"lse": torch.where(vt, tt["lse"], z0), "b_lse": 2 * torch.where(vt, tt["E_lse"], z0) + FTZ, "loss": loss,
           "b_loss": mean_b(vsum(E_sp), vsum(sp)), "reward_chosen": vsum(rc) * inv, "b_reward_chosen": mean_b(vsum(E_rc), vsum(rc.abs())),
           "reward_rejected": vsum(rr) * inv, "b_reward_rejected": mean_b(vsum(E_rr), vsum(rr.abs())), "accuracy": acc,
           "b_accuracy": (amb * inv + 16 * U) * 2 + FTZ, "z": z, "valid": valid, "n": n}
    c = torch.where(valid, beta * sig * inv, pair)
    E_c = torch.where(valid, (beta * sig * (1 - sig) * E_z + 8 * U * beta * sig) * inv, pair)
    wv, E_w = torch.cat([c, -c]), torch.cat([E_c, E_c])
    res.update(w=wv, b_w=2 * E_w + FTZ)
    if dloss is not None and terms is None:
        row = torch.arange(Tn) // S
        res["grad"], res["b_grad"] = dpo_grad_ref(s, labels, tt["lse"], tt["E_lse"], wv[row], E_w[row], V, dloss, ignore_index)
    return res


def dpo_checks(got, o) -> Dict[str, float]:
    out = {k: abs(float(got[k]) - o[k]) / o[f"b_{k}"] for k in ("loss", "reward_chosen", "reward_rejected", "accuracy")}
    for k in ("lse", "w", "grad"):
        if k in got:
            out[k] = ratio(got[k], o[k], o[f"b_{k}"])
    return out


# ================================================================================================= emulator
DPO_MUTANTS = ("beta_missing", "swapped", "reference_ignored", "prompt_counted", "mean_not_sum", "invalid_counted")


def _bfly(v: torch.Tensor) -> torch.Tensor:
    """``warp_sum``'s xor butterfly over the last dimension (32 lanes), fp32 adds."""
    for o in (16, 8, 4, 2, 1):
        v = f32(v + v[..., torch.arange(32) ^ o])
    return v[..., 0]


def _block_sum1024(vals: torch.Tensor) -> torch.Tensor:
    """``block_sum`` over 1024 threads, thread i holding ``vals[i]`` (0 past the end)."""
    v = torch.zeros(1024, dtype=torch.float64)
    v[: vals.numel()] = vals
    return _bfly(_bfly(v.view(32, 32)))


def emulate_dpo(s, r, labels, P: int, V: int, beta: float, dloss: float = 1.0, mutant=None, prompt_labels=None) -> Dict:
    """fp32 emulator of ``dpo_fwd_kernel`` (the online max / sum of ``kd_fwd_kernel``'s ``T == 1`` path for both rows),
    ``dpo_reduce_kernel`` (warp-per-row sums, one pair per thread, ``block_sum``) and ``dpo_bwd_kernel``."""
    Tn, Vp = s.shape
    S = Tn // (2 * P)
    lb = prompt_labels if mutant == "prompt_counted" else labels
    vt = lb != -100
    lses = emulate_kd(s, r, lb, V, 1.0, 1.0)["lse"]
    lse1, lse2 = lses[0], lses[2]
    lab = torch.where(vt, lb, torch.zeros_like(lb))
    x, y = s.double(), r.double()
    lp1 = f32(x.gather(1, lab[:, None])[:, 0] - lse1)
    lp2 = f32(y.gather(1, lab[:, None])[:, 0] - lse2)
    d = lp1 if mutant == "reference_ignored" else f32(lp1 - lp2)
    d = torch.where(vt, d, torch.zeros_like(d))
    S32 = -(-S // 32) * 32
    terms = torch.zeros(2 * P, S32, dtype=torch.float64)
    terms[:, :S] = d.view(2 * P, S)
    acc = torch.zeros(2 * P, 32, dtype=torch.float64)
    for k in range(S32 // 32):
        acc = f32(acc + terms[:, 32 * k: 32 * (k + 1)])
    D = _bfly(acc)
    cnt = vt.view(2 * P, S).sum(1).double()
    if mutant == "mean_not_sum":
        D = torch.where(cnt > 0, f32(D / cnt.clamp(min=1)), D)
    Dc, Dr = (D[P:], D[:P]) if mutant == "swapped" else (D[:P], D[P:])
    b = 1.0 if mutant == "beta_missing" else beta
    bf = float(f32(torch.tensor(b)))
    valid = (cnt[:P] > 0) & (cnt[P:] > 0)
    if mutant == "invalid_counted":
        valid = torch.ones_like(valid)
    rc, rr = f32(bf * Dc), f32(bf * Dr)
    z = f32(rc - rr)
    e = f32(torch.exp(-z.abs()))
    sp = f32(f32(torch.clamp(-z, min=0)) + f32(torch.log1p(e)))
    zero = torch.zeros_like(z)
    sums = [_block_sum1024(torch.where(valid, v, zero)) for v in (valid.double(), sp, rc, rr, (z > 0).double())]
    n = float(sums[0])
    inv = float(f32(torch.tensor(1.0 / n))) if n else 0.0
    sig = torch.where(z >= 0, f32(e / f32(1 + e)), f32(1 / f32(1 + e)))
    c = torch.where(valid, f32(f32(bf * sig) * inv), zero)
    w = torch.cat([c, -c])
    if mutant == "swapped":
        w = -w
    row = torch.arange(Tn) // S
    scale = f32(dloss * w[row])
    cols = torch.arange(Vp)
    p = torch.where(cols[None, :] < V, f32(torch.exp(f32(x - lse1[:, None]))), torch.zeros_like(x))
    p = torch.where(cols[None, :] == lab[:, None], f32(p - 1), p)
    grad = bf16_rn(f32(p * scale[:, None])).double()
    grad = torch.where(vt[:, None], grad, torch.zeros_like(grad))
    if mutant == "prompt_counted":                       # the lse of the real response rows is what the kernel would keep
        lse1 = torch.where(labels != -100, lse1, torch.zeros_like(lse1))
    return {"lse": lse1, "loss": float(f32(sums[1] * inv)), "reward_chosen": float(f32(sums[2] * inv)),
            "reward_rejected": float(f32(sums[3] * inv)), "accuracy": float(f32(sums[4] * inv)), "w": w, "grad": grad, "d": d, "z": z}


def dpo_inputs(P: int, S: int, V: int, Vp: int, seed: int, noise: float = 0.5, pad_fill: Optional[float] = None, invalid: bool = True):
    """``[2P S, Vp]`` policy logits and a reference ``noise`` away, shifted labels with a random prompt / response / padding split per
    row, and the labels a model counting prompt tokens would use.  Pair 0's rejected row has its response cut away (``invalid``); the
    reference equals the policy on chosen row 1 (when ``P > 1``)."""
    g = torch.Generator().manual_seed(seed)
    Tn = 2 * P * S
    s = (3 * torch.randn(Tn, Vp, generator=g)).to(torch.bfloat16)
    r = (s.float() + noise * torch.randn(Tn, Vp, generator=g)).to(torch.bfloat16)
    if P > 1:
        r.view(2 * P, S, Vp)[1] = s.view(2 * P, S, Vp)[1]
    if pad_fill is not None and Vp > V:
        s[:, V:] = pad_fill
        r[:, V:] = pad_fill
    tok = torch.randint(0, V, (2 * P, S), generator=g)
    lab = torch.full((2 * P, S), -100)
    plab = torch.full((2 * P, S), -100)
    for i in range(2 * P):
        a = int(torch.randint(1, max(S // 2, 2), (1,), generator=g))
        e = int(torch.randint(a + 1, S + 1, (1,), generator=g))
        if invalid and P > 1 and i == P:
            e = a
        lab[i, a:e] = tok[i, a:e]
        plab[i, 1:e] = tok[i, 1:e]
    return s, r, shift(lab), shift(plab), lab


# ================================================================================================= oracle vs TRL autograd
@pytest.mark.parametrize("beta", [0.1, 1.0])
@pytest.mark.parametrize("V,Vp", [(37, 40), (40, 40), (1003, 1008)], ids=["ragged-padded", "exact", "ragged-1003"])
@pytest.mark.parametrize("noise", [0.5, 8.0], ids=["small-z", "large-z"])
def test_oracle_matches_trl_autograd(beta, V, Vp, noise):
    """Prompt masks, padding rows and columns, ragged V, an invalid pair, large |z| - against autograd of TRL's formulation in fp64."""
    P, S = 3, 12
    s, r, lb, _, lab2d = dpo_inputs(P, S, V, Vp, seed=V + int(noise), noise=noise, pad_fill=30.0)
    o = dpo_ref(s, r, lb, P, V, beta, dloss=1.5)
    x = s[:, :V].double().view(2 * P, S, V).requires_grad_(True)
    loss = trl_loss(x, r[:, :V].double().view(2 * P, S, V), lab2d, P, beta)
    (1.5 * loss).backward()
    assert o["n"] == P - 1 and not bool(o["valid"][0])
    assert abs(o["loss"] - float(loss)) <= 1e-12 * max(1.0, abs(float(loss)))
    torch.testing.assert_close(o["grad"][:, :V], x.grad.reshape(-1, V), rtol=1e-10, atol=1e-14)
    assert bool((o["grad"][:, V:] == 0).all()) and bool((o["grad"][lb == -100] == 0).all())
    if noise > 1 and beta == 1.0:
        assert float(o["z"].abs().max()) > 30                   # large |z|: the stable forms are exercised


def test_all_invalid_batch_has_zero_loss_and_gradient():
    P, S, V = 2, 8, 50
    s, r, lb, _, _ = dpo_inputs(P, S, V, 56, seed=4)
    lb.view(2 * P, S)[P:] = -100                                # every rejected response cut away
    o = dpo_ref(s, r, lb, P, V, 0.1, dloss=1.0)
    assert o["n"] == 0 and o["loss"] == 0.0 and o["accuracy"] == 0.0 and bool((o["grad"] == 0).all())
    e = emulate_dpo(s, r, lb, P, V, 0.1)
    assert e["loss"] == 0.0 and bool((e["grad"] == 0).all())
    from acco_b200 import ops
    xs = s.float().requires_grad_(True)
    out = torch.full((3,), -1.0)
    loss = ops.dpo_loss(xs, r.float(), lb, P, V, 0.1, out=out)
    loss.backward()
    assert float(loss) == 0.0 and bool((xs.grad == 0).all()) and bool((out == 0).all())


@pytest.mark.parametrize("beta", [0.1, 1.0])
def test_policy_equal_to_reference_gives_ln2_and_the_scaled_ce_gradient(beta):
    P, S, V = 3, 10, 131
    s, _, lb, _, _ = dpo_inputs(P, S, V, 136, seed=3)
    o = dpo_ref(s, s, lb, P, V, beta, dloss=1.0)
    n = o["n"]
    assert bool((o["z"] == 0).all()) and o["loss"] == pytest.approx(LN2, abs=1e-15)
    ce = torch.zeros_like(o["grad"])                        # the un-normalised CE gradient direction of each response token
    x = s[:, :V].double()
    vt = lb != -100
    p = torch.softmax(x, 1)
    p[torch.arange(len(lb)), torch.where(vt, lb, 0)] -= 1
    ce[:, :V] = torch.where(vt[:, None], p, torch.zeros_like(p))
    sign = torch.ones(2 * P, 1, dtype=torch.float64)
    sign[P:] = -1
    sign[[0, P]] = 0                                          # the invalid pair
    want = (beta / (2 * n)) * ce * sign.repeat_interleave(S, 0)
    torch.testing.assert_close(o["grad"], want, rtol=1e-12, atol=1e-15)
    e = emulate_dpo(s, s, lb, P, V, beta)
    assert bool((e["d"] == 0).all()) and bool((e["z"] == 0).all())     # the kernel forms both log-probabilities identically
    assert e["loss"] == float(f32(torch.tensor(LN2)))
    from acco_b200 import ops
    out = torch.zeros(3)
    assert float(ops.dpo_loss(s.float(), s.float(), lb, P, V, beta, out=out)) == pytest.approx(LN2, rel=1e-6)
    assert out.tolist() == [0.0, 0.0, 0.0]


# ================================================================================================= margin table
DPO_CASES = [
    # (name, P, S, V, Vp, beta, noise, padding fill)
    ("P3-S16-V1003-b0.1-pad", 3, 16, 1003, 1008, 0.1, 0.5, 20.0),
    ("P4-S24-V131-b1", 4, 24, 131, 136, 1.0, 0.5, None),
    ("P2-S40-V40-b1-large-z", 2, 40, 40, 40, 1.0, 8.0, None),
    ("P2-S8-V50257-b0.1", 2, 8, 50257, 50304, 0.1, 0.5, 30.0),
    ("P2-S4-V128256-b0.1", 2, 4, 128256, 128256, 0.1, 0.5, None),
]


def dpo_row(name, P, S, V, Vp, beta, noise, pad_fill):
    s, r, lb, plb, _ = dpo_inputs(P, S, V, Vp, seed=V + S, noise=noise, pad_fill=pad_fill)
    o = dpo_ref(s, r, lb, P, V, beta, dloss=0.75)
    emu = dpo_checks(emulate_dpo(s, r, lb, P, V, beta, dloss=0.75), o)
    caught = {}
    for m in DPO_MUTANTS:
        if m == "beta_missing" and beta == 1.0:
            continue
        c = dpo_checks(emulate_dpo(s, r, lb, P, V, beta, dloss=0.75, mutant=m, prompt_labels=plb), o)
        caught[m] = max(c.items(), key=lambda kv: kv[1])
    return emu, caught


ROWS = {c[0]: functools.lru_cache(maxsize=None)(lambda c=c: dpo_row(*c)) for c in DPO_CASES}


@pytest.mark.parametrize("name", list(ROWS))
def test_margin_table_emulator_within_half(name):
    emu, _ = ROWS[name]()
    for k, v in emu.items():
        assert v < 0.5, (name, "emulator", k, v)


def test_every_mutant_lands_far_outside_on_some_case():
    best = {m: 0.0 for m in DPO_MUTANTS}
    for name, row in ROWS.items():
        _, caught = row()
        for m, (k, v) in caught.items():
            best[m] = max(best[m], v)
    assert all(v > 100.0 for v in best.values()), best


# ================================================================================================= op reference path
def test_op_reference_path_matches_trl_and_writes_out():
    from acco_b200 import ops
    P, S, V = 3, 9, 37
    s, r, lb, _, lab2d = dpo_inputs(P, S, V, 40, seed=6, noise=2.0, pad_fill=5.0)
    out = torch.full((3,), -1.0)
    x = s.float().requires_grad_(True)
    rf = r.float()
    got = ops.dpo_loss(x, rf, lb, P, V, 0.5, out=out)
    got.backward()
    xr = s[:, :V].float().view(2 * P, S, V).requires_grad_(True)
    ref = trl_loss(xr, r[:, :V].float().view(2 * P, S, V), lab2d, P, 0.5)
    ref.backward()
    assert float(got) == pytest.approx(float(ref), rel=1e-5)
    torch.testing.assert_close(x.grad[:, :V], xr.grad.reshape(-1, V), rtol=1e-4, atol=1e-7)
    assert bool((x.grad[:, V:] == 0).all())
    o = dpo_ref(s, r, lb, P, V, 0.5)
    assert out.tolist() == pytest.approx([o["reward_chosen"], o["reward_rejected"], o["accuracy"]], rel=1e-5, abs=1e-6)
    assert torch.equal(rf, r.float())                        # the reference logits are never written
    for bad in (0.0, -0.1, math.inf, math.nan, True):
        with pytest.raises(ValueError, match="beta"):
            ops.dpo_loss(x, rf, lb, P, V, bad)
    with pytest.raises(ValueError, match="ref_logits"):
        ops.dpo_loss(x, rf[:, :36], lb, P, V, 0.1)
    with pytest.raises(ValueError, match="2 P S rows"):
        ops.dpo_loss(x, rf, lb, 4, V, 0.1)


# ================================================================================================= collator
def test_collator_against_a_per_token_oracle():
    from acco_b200.data import PreferenceCollator
    g = torch.Generator().manual_seed(0)
    pairs = []
    for _ in range(5):
        lp, lc, lr = (int(v) for v in torch.randint(0, 14, (3,), generator=g))
        mk = lambda n: torch.randint(0, 50, (n,), generator=g).tolist()
        pairs.append({"prompt_ids": mk(lp), "chosen_ids": mk(lc), "rejected_ids": mk(lr)})
    pairs.append({"prompt_ids": list(range(20)), "chosen_ids": [1, 2], "rejected_ids": [3]})     # response cut away: invalid
    L, mult, pad = 16, 8, 99
    b = PreferenceCollator(pad_token_id=pad, max_length=L, pad_to_multiple_of=mult)(pairs)
    P = len(pairs)
    assert b["input_ids"].shape[0] == 2 * P and b["input_ids"].shape[1] % mult == 0
    S = b["input_ids"].shape[1]
    for i in range(2 * P):
        pr = pairs[i % P]
        resp = pr["chosen_ids"] if i < P else pr["rejected_ids"]
        full = pr["prompt_ids"] + resp
        for t in range(S):
            in_row = t < min(len(full), L)
            assert int(b["input_ids"][i, t]) == (full[t] if in_row else pad)
            assert int(b["attention_mask"][i, t]) == int(in_row)
            assert int(b["labels"][i, t]) == (full[t] if in_row and t >= len(pr["prompt_ids"]) else -100)
    lb = shift(b["labels"]).view(2 * P, S)
    assert not bool((lb[P - 1] != -100).any()) and not bool((lb[2 * P - 1] != -100).any())


def test_synthetic_pairs_and_tokenised_text_pairs():
    from acco_b200.data import ByteTokenizer, TokenDataset, make_preference_tokenize_fn, synthetic_preference_dataset
    ds = synthetic_preference_dataset(64, 40, 96, seed=1)
    assert set(ds.column_names) == {"prompt_ids", "chosen_ids", "rejected_ids"}
    succ = lambda a, b: b == (31 * a + 7) % 95                # the Markov source's successor map
    follows = sum(succ(row["prompt_ids"][-1], row["chosen_ids"][0]) for row in ds) + \
        sum(succ(a, b) for row in ds for a, b in zip(row["chosen_ids"], row["chosen_ids"][1:]))
    follows_rej = sum(succ(a, b) for row in ds for a, b in zip(row["rejected_ids"], row["rejected_ids"][1:]))
    assert follows > 10 * max(follows_rej, 1)
    tok = ByteTokenizer(eos_token_id=256)
    text = TokenDataset({"prompt": ["ab", "x"], "chosen": ["c", "yz"], "rejected": ["d", ""]})
    out = text.map(make_preference_tokenize_fn(tok), batched=True, remove_columns=text.column_names)
    assert out[0] == {"prompt_ids": [97, 98], "chosen_ids": [99, 256], "rejected_ids": [100, 256]}
    assert out[1]["rejected_ids"] == [256]


# ================================================================================================= models
def _tiny_llama(seed=0, layers=2):
    from acco_b200.models import LlamaConfig, LlamaForCausalLM
    torch.manual_seed(seed)
    return LlamaForCausalLM(LlamaConfig(vocab_size=90, hidden_size=32, intermediate_size=48, num_hidden_layers=layers, num_attention_heads=4,
                                        num_key_value_heads=2, max_position_embeddings=32, pad_vocab_multiple=8))


def _tiny_gpt(seed=0):
    from acco_b200.models import GPTConfig, GPTForCausalLM
    torch.manual_seed(seed)
    return GPTForCausalLM(GPTConfig(vocab_size=90, hidden_size=32, num_hidden_layers=2, num_attention_heads=4, max_position_embeddings=32,
                                    attention_layers=["global", "local"], window_size=8, pad_vocab_multiple=8))


def _pair_batch(P, S, V, seed):
    from acco_b200.data import PreferenceCollator
    g = torch.Generator().manual_seed(seed)
    pairs = [{k: torch.randint(0, V, (int(torch.randint(2, S // 2, (1,), generator=g)),), generator=g).tolist()
              for k in ("prompt_ids", "chosen_ids", "rejected_ids")} for _ in range(P)]
    return PreferenceCollator(pad_token_id=V - 1, max_length=S)(pairs)


@pytest.mark.parametrize("make", [_tiny_llama, _tiny_gpt], ids=["llama-gqa", "gptneo"])
@pytest.mark.parametrize("beta", [0.1, 1.0])
def test_native_model_matches_the_formula(make, beta):
    """``reference_logits`` with labels gives the loss and gradients of TRL's formula on the model's own logits (fp32); the
    reference gets no gradient."""
    m, ref = make(0).float(), make(5).float()
    ref.requires_grad_(False)
    b = _pair_batch(3, 16, 90, seed=1)
    m.dpo_beta, m.dpo_out = beta, torch.zeros(3)
    with torch.no_grad():
        rl = ref.padded_logits(b["input_ids"])
    loss = m(input_ids=b["input_ids"], labels=b["labels"], reference_logits=rl)[0]
    loss.backward()
    got = {k: p.grad.clone() for k, p in m.named_parameters()}
    m.zero_grad()
    logits = m(input_ids=b["input_ids"]).logits
    want = trl_loss(logits, ref(input_ids=b["input_ids"]).logits, b["labels"], 3, beta)
    want.backward()
    assert float(loss.detach()) == pytest.approx(float(want.detach()), rel=2e-6)
    for k, p in m.named_parameters():
        torch.testing.assert_close(got[k], p.grad, rtol=1e-4, atol=1e-5 * float(p.grad.abs().max()), msg=k)
    assert all(p.grad is None for p in ref.parameters())
    with pytest.raises(ValueError, match="labels"):
        m(input_ids=b["input_ids"], reference_logits=rl)
    with pytest.raises(ValueError, match="even number of rows"):
        m(input_ids=b["input_ids"][:3], labels=b["labels"][:3], reference_logits=rl[: 3 * 16])


# ================================================================================================= trainer
class _DPORef(torch.nn.Module):
    """A non-native model around the policy's weights whose loss is TRL's formula in plain torch, with the reference outside its
    parameters: the plain PyTorch loop the trainer is checked against."""

    def __init__(self, m, reference, beta):
        super().__init__()
        self.m, self._r, self.beta = m, [reference], beta

    def forward(self, input_ids=None, labels=None, **kw):
        logits = self.m(input_ids=input_ids).logits
        with torch.no_grad():
            rl = self._r[0](input_ids=input_ids).logits
        return (trl_loss(logits.float(), rl.float(), labels, input_ids.shape[0] // 2, self.beta),)


def _pairs(n=96, seed=3):
    from acco_b200.data import synthetic_preference_dataset
    return synthetic_preference_dataset(n, 14, 95, seed=seed)


def _trainer(model, reference=None, method="acco", ds="pairs", **kw):
    from acco_b200 import DecoupledTrainer
    from acco_b200.launch import DistEnv
    from helpers import LOG, base_args
    kw = {"nb_steps_tot": 8, "const_len_batch": False, "dpo_beta": 0.1, **kw}
    data = _pairs() if ds == "pairs" else ds
    return DecoupledTrainer(model=model, train_dataset=data, eval_dataset=_pairs(16, seed=8) if data is not None else None,
                            args=base_args(method_name=method, **kw), log=LOG, env=DistEnv(id_run="dpo"),
                            reference=reference)


def _ref(seed=9):
    from helpers import tiny_model
    return tiny_model(seed=seed, layers=1)


@pytest.mark.parametrize("method,impl", [("acco", "native"), ("dpu", "native"), ("ddp", "native"), ("ddp", "torch")])
def test_trainers_track_a_plain_pytorch_loop(workdir, method, impl):
    from helpers import tiny_model
    kw = dict(ddp_impl=impl, log_every=1, nb_steps_tot=16, dpo_beta=0.5)
    t = _trainer(tiny_model(), _ref(), method, **kw)
    assert t.model.dpo_out is t.dpo_static and t.model.dpo_beta == 0.5
    t.is_cuda = True                                       # graphs need a GPU; everything else about the route allows them
    assert t._use_graphs()
    t.is_cuda = False
    ref = _trainer(_DPORef(tiny_model(), _ref(), 0.5), None, method, ds=None, **{**kw, "dpo_beta": None})
    ref.train_dataloader = t.get_train_dataloader()        # the same pairs in the same order, through the same collator
    a, b = _logged(t), _logged(ref)
    assert len(a) == len(b) >= 4
    for x, y in zip(a, b):
        assert abs(x["loss"] - y["loss"]) <= 1e-5 * abs(y["loss"]), (a, b)
        assert "dpo_accuracy" in x and "dpo_accuracy" not in y
    assert all(not p.requires_grad for p in t.reference.parameters())


def test_eval_reports_the_objective_and_the_accuracy(workdir):
    from helpers import tiny_model
    t = _trainer(tiny_model(), _ref(), max_eval_batches=3)
    t.dpo_static.fill_(7.0)
    loss = float(t.eval_loop())
    assert t.dpo_static.tolist() == [7.0, 7.0, 7.0]        # the logged training scalars are not overwritten
    batches = [b for _, b in zip(range(3), t.eval_dataloader)]
    want = []
    with torch.no_grad():
        for b in batches:
            want.append(float(trl_loss(t.model(input_ids=b["input_ids"]).logits, t.reference(input_ids=b["input_ids"]).logits,
                                       b["labels"], b["input_ids"].shape[0] // 2, 0.1)))
    assert loss == pytest.approx(sum(want) / len(want), rel=1e-5)
    assert 0.0 <= t.eval_dpo_accuracy <= 1.0


def _worker(rank, world, port, tmp, q):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    os.environ.update(CUDA_VISIBLE_DEVICES="", MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank))
    os.chdir(tmp)
    torch.set_num_threads(2)
    from acco_b200 import DecoupledTrainer
    from acco_b200.data import synthetic_preference_dataset
    from acco_b200.launch import shutdown_distributed
    from helpers import LOG, base_args, tiny_model
    args = base_args(method_name="acco", nb_steps_tot=16, batch_size=2, const_len_batch=False, dpo_beta=0.1)
    t = DecoupledTrainer(model=tiny_model(seed=rank), train_dataset=synthetic_preference_dataset(64, 14, 95, seed=7), args=args, log=LOG,
                         reference=tiny_model(seed=9, layers=1))
    accs = []
    while not t.finished():
        t.step()
        accs.append(float(t.dpo_host[2]))
    t._drain()
    t._finish("")
    q.put((rank, float(t.params.double().sum()), accs, t.len_params))
    shutdown_distributed()


def test_two_gloo_ranks_train_with_a_reference(workdir):
    import tempfile
    import torch.multiprocessing as mp
    from acco_b200.launch import free_port
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = free_port()
    with tempfile.TemporaryDirectory() as tmp:
        procs = [ctx.Process(target=_worker, args=(r, 2, port, tmp, q)) for r in range(2)]
        for p in procs:
            p.start()
        out = sorted(q.get(timeout=240) for _ in procs)
        for p in procs:
            p.join(timeout=60)
            assert p.exitcode == 0
    (_, w0, a0, n0), (_, w1, a1, _) = out
    assert w0 == w1                                        # the ranks end on the same weights
    assert all(0.0 <= a <= 1.0 for a in a0 + a1)
    from helpers import tiny_model
    assert n0 == sum(p.numel() for p in tiny_model().parameters())      # the arena holds the policy only


def test_the_rejections(workdir):
    from helpers import tiny_model
    from acco_b200.data import synthetic_sft_dataset
    with pytest.raises(ValueError, match="not both"):
        _trainer(tiny_model(), _ref(), dpo_reference="/nonexistent")
    with pytest.raises(ValueError, match="needs a frozen reference"):
        _trainer(tiny_model(), None)
    with pytest.raises(ValueError, match="without dpo_beta"):
        _trainer(tiny_model(), _ref(), dpo_beta=None)
    for bad in (0, 0.0, -0.1, math.nan, math.inf, True, "0.1"):
        with pytest.raises(ValueError, match="dpo_beta"):
            _trainer(tiny_model(), _ref(), dpo_beta=bad)
    with pytest.raises(ValueError, match="native policy"):
        _trainer(_DPORef(tiny_model(), _ref(), 0.1), _ref())
    with pytest.raises(ValueError, match="native model"):
        _trainer(tiny_model(), _DPORef(_ref(), _ref(), 0.1))
    with pytest.raises(ValueError, match="vocabularies differ"):
        _trainer(tiny_model(), tiny_model(vocab=90))
    with pytest.raises(ValueError, match="distill_teacher"):
        _trainer(tiny_model(), _ref(), distill_teacher="/nonexistent")
    from acco_b200 import DecoupledTrainer
    from acco_b200.launch import DistEnv
    from helpers import LOG, base_args
    with pytest.raises(ValueError, match="distill_teacher"):
        DecoupledTrainer(model=tiny_model(), train_dataset=_pairs(), args=base_args(const_len_batch=False, dpo_beta=0.1), log=LOG,
                         env=DistEnv(id_run="dpo"), teacher=_ref(), reference=_ref(3))
    for key, val in (("label_smoothing_factor", 0.1), ("z_loss_weight", 1e-4), ("packing", True), ("document_mask", True),
                     ("const_len_batch", True)):
        with pytest.raises(ValueError, match=key):
            _trainer(tiny_model(), _ref(), **{key: val})
    m = tiny_model()
    with pytest.raises(ValueError, match="separate model"):
        _trainer(m, m)
    with pytest.raises(ValueError, match="preference pairs"):
        _trainer(tiny_model(), _ref(), ds=synthetic_sft_dataset(32, 10, 95, 16))
    assert _trainer(tiny_model(), None, ds=synthetic_sft_dataset(32, 10, 95, 16), dpo_beta=None).reference is None     # off


def test_reference_stays_out_of_the_arena_and_checkpoint_and_a_resume_reloads_it(workdir):
    from helpers import tiny_model
    ref = _ref()
    rdir = os.path.join(os.getcwd(), "reference")
    _write_hf_dir(ref, rdir)
    t = _trainer(tiny_model(), None, dpo_reference=rdir, save_optimizer=True)
    assert t.len_params == sum(p.numel() for p in t.model.parameters())
    assert not any(t.reference is mod for mod in t.model.modules())
    t.train()
    ck = os.path.join(os.getcwd(), "ck", "policy.pt")
    t.save_checkpoint(ck)
    saved = torch.load(ck, map_location="cpu", weights_only=False)
    assert set(saved) == set(t.model.state_dict())
    assert sum(v.numel() for v in _tensors(saved)) == sum(v.numel() for v in t.model.state_dict().values())     # the policy alone
    r2 = _trainer(tiny_model(seed=4), None, dpo_reference=rdir, resume_from=ck)
    for (k, a), b in zip(r2.reference.state_dict().items(), ref.state_dict().values()):
        assert torch.equal(a, b), k                                   # the reference again, not a copy of the resumed policy
    for k, v in r2.model.state_dict().items():
        assert torch.equal(v, saved[k]), k


@pytest.mark.parametrize("on", [False, True])
def test_dpo_scalars_are_logged_only_with_dpo(workdir, on):
    from helpers import tiny_model
    from acco_b200.data import synthetic_sft_dataset
    if on:
        t = _trainer(tiny_model(), _ref(), tensorboard=True, log_every=2, nb_steps_tot=10, eval=True, eval_step=4, max_eval_batches=2)
    else:
        t = _trainer(tiny_model(), None, ds=synthetic_sft_dataset(64, 10, 95, 16), dpo_beta=None, tensorboard=True, log_every=2,
                     nb_steps_tot=10)
    logs = _logged(t)
    t.writer.flush()
    rows = [json.loads(line) for line in open(os.path.join(t.writer.logdir, "scalars.jsonl"))]
    tags = {r["tag"] for r in rows}
    names = ("dpo_reward_chosen", "dpo_reward_rejected", "dpo_accuracy")
    assert logs
    if not on:
        assert all(k not in d for d in logs for k in names) and not (set(names) & tags)
        return
    for d in logs:
        assert 0.0 <= d["dpo_accuracy"] <= 1.0 and d["loss"] > 0
    assert set(names) <= tags and sum(r["tag"] == "dpo_accuracy" for r in rows) == len(logs)
    assert any("eval_dpo_accuracy" in d for d in logs)


def test_cli_preference_data_with_the_pretrained_policy_as_reference(workdir, monkeypatch):
    sys.path.insert(0, ROOT)
    import main as cli
    from acco_b200 import DecoupledTrainer, ops
    from acco_b200.models import LlamaConfig, LlamaForCausalLM
    seen, srcs = [], []
    orig, orig_setup = ops.dpo_loss, DecoupledTrainer._setup_frozen

    def dpo(*a, **kw):
        seen.append((a[3], a[5]))
        return orig(*a, **kw)

    def setup(self, src, *a):
        srcs.append(src)
        return orig_setup(self, src, *a)
    monkeypatch.setattr(ops, "dpo_loss", dpo)
    monkeypatch.setattr(DecoupledTrainer, "_setup_frozen", setup)
    torch.manual_seed(2)
    pol = LlamaForCausalLM(LlamaConfig(vocab_size=512, hidden_size=32, intermediate_size=48, num_hidden_layers=1, num_attention_heads=4,
                                       max_position_embeddings=64))      # config/model/tiny.yaml's vocabulary
    pdir = os.path.join(os.getcwd(), "pretrained")
    _write_hf_dir(pol, pdir)
    stats = cli.main(["train=acco-ft", "data=preference", "model=tiny", f"model.pretrained={pdir}", "train.dpo_beta=0.1",
                      "train.nb_steps_tot=6", "train.batch_size=2", "train.max_length=32", "train.use_mixed_precision=False",
                      "data.synthetic_docs=64", "data.synthetic_mean_len=12", "train.eval=False", "run_name=dpo", "train.save=False",
                      "train.dataloader_num_workers=0"])
    assert stats["count_grad_tot"] >= 6
    assert seen and set(seen) == {(2, 0.1)}
    assert pdir in [str(s) for s in srcs]


if __name__ == "__main__":               # print the margin table: python tests/test_dpo.py
    for name, row in ROWS.items():
        emu, caught = row()
        print(f"{name:24s} emulator/bound " + " ".join(f"{k}={v:.3f}" for k, v in emu.items()))
        for m, (k, v) in caught.items():
            print(f"{'':24s}   mutant {m:18s} worst {k}: {v:.3g}x")
