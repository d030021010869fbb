"""Reference-free preference tuning (``train.simpo_beta`` / ``train.orpo_lambda``): the fp64 oracle of ``ce_fwd`` + ``pref_reduce``
+ ``dpo_bwd`` and its per-element bounds, checked against autograd of TRL's formulations; the margin table of a blockwise fp32
emulator and its mutants; the identities; and the op, model and trainer routes.  Runs on the CPU without the extension;
``test_pref_free_gpu.py`` runs the kernels against the same oracle.

Semantics (``P`` pairs as ``[2P, S]`` rows, chosen rows first; ``R(row)`` the positions whose shifted label is not -100)::

    lp_t = s_t[y_t] - lse(s_t),   l(row) = sum_{t in R} lp_t,   a(row) = l(row) / |row|,   valid_i = both rows non-empty,  n = #valid
    SimPO: z_i = beta (a(c_i) - a(r_i)) - gamma,   loss = sum_valid softplus(-z_i) / n,
           w(c_i) = beta sigma(-z_i) / (n |c_i|),   w(r_i) = -beta sigma(-z_i) / (n |r_i|)
    ORPO:  nll = -sum_valid l(c_i) / N_c,   lo_i = (a - log(1 - e^a'))(c_i) - (a - log(1 - e^a'))(r_i),   a' = min(a, -2^-20),
           loss = nll + lambda sum_valid softplus(-lo_i) / n,
           w(c_i) = 1 / N_c + lambda sigma(-lo_i) / (n |c_i| (1 - e^a'(c_i))),   w(r_i) = -lambda sigma(-lo_i) / (n |r_i| (1 - e^a'(r_i)))
    ds_tc = dloss w(row) (softmax(s_t)_c - [c = y_t])                   (c < V, t in R; else 0)

Bounds: ``lse`` as in the CE oracle; ``l`` is a warp sum of ``S`` terms (``ceil(S / 32) + 5`` fp32 adds deep); the division by the
count is the fast-math one (4 u); ``log(1 - e^a')`` carries the error of ``a'`` times its slope ``e^a / (1 - e^a)`` at the worst
point of the interval, plus the ``__logf`` / ``log1pf`` / ``__expf`` errors; ``softplus`` and ``sigma`` as in the DPO oracle; the
pair sums are a ``block_sum`` over 1024 values.  The gradient reuses the DPO oracle's.  Everything is doubled, as elsewhere.

The margin table asserts the emulator stays within half of every bound and that each mutant lands more than 3x outside on some case.
Print it with ``python tests/test_pref_free.py``."""
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
from test_dpo import _block_sum1024, _bfly, _pair_batch, _pairs, _tiny_gpt, _tiny_llama, dpo_grad_ref, shift  # noqa: E402
from test_gemm_oracle import bf16_rn  # noqa: E402
from test_rowwise_oracle import FTZ, U, e_exp, f32, ratio  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LN2 = math.log(2.0)
A_MAX = -(2.0 ** -20)


# ================================================================================================= TRL's formulations
def _avg_logps(s: torch.Tensor, labels: torch.Tensor):
    """TRL's ``average_log_prob``: ``[2P, S, V]`` logits and unshifted ``[2P, S]`` labels -> per row (sum, count, mean)."""
    lb = labels[:, 1:]
    mask = lb != -100
    idx = torch.where(mask, lb, torch.zeros_like(lb))[..., None]
    tok = torch.log_softmax(s[:, :-1], -1).gather(-1, idx)[..., 0] * mask
    cnt = mask.sum(-1)
    return tok.sum(-1), cnt, tok.sum(-1) / cnt.clamp(min=1), mask


def trl_simpo(s, labels, P: int, beta: float, gamma: float) -> torch.Tensor:
    """TRL ``CPOTrainer(loss_type="simpo", cpo_alpha=0)``: ``-logsigmoid(beta ((a_c - a_r) - gamma / beta))``, mean over the pairs
    whose two rows have a response token."""
    _, _, a, mask = _avg_logps(s, labels)
    logits = (a[:P] - a[P:]) - gamma / beta
    valid = mask[:P].any(1) & mask[P:].any(1)
    return torch.where(valid, -F.logsigmoid(beta * logits), torch.zeros_like(logits)).sum() / valid.sum().clamp(min=1)


def trl_orpo_from_rows(l, cnt, P: int, lam: float, clamp: bool = False) -> torch.Tensor:
    """TRL ``ORPOTrainer`` from per-row log-probability sums and counts: the chosen responses' token-mean NLL minus ``lam`` times the
    mean ``logsigmoid`` of the log odds ratio ``(a_c - a_r) - (log1p(-e^a_c) - log1p(-e^a_r))``.  ``clamp``: ``a`` in the two log1p
    terms is clamped at -2^-20 straight through (TRL returns inf / NaN once a reaches 0)."""
    a = torch.where(cnt > 0, l / cnt.clamp(min=1), -torch.ones_like(l))      # an empty row (invalid pair) stays out of the log terms
    valid = (cnt[:P] > 0) & (cnt[P:] > 0)
    ac = a + (a.clamp(max=A_MAX) - a).detach() if clamp else a
    log_odds = (a[:P] - a[P:]) - (torch.log1p(-torch.exp(ac[:P])) - torch.log1p(-torch.exp(ac[P:])))
    zero = torch.zeros_like(log_odds)
    nll = -torch.where(valid, l[:P], zero).sum() / torch.where(valid, cnt[:P], torch.zeros_like(cnt[:P])).sum().clamp(min=1)
    return nll - lam * torch.where(valid, F.logsigmoid(log_odds), zero).sum() / valid.sum().clamp(min=1)


def trl_orpo(s, labels, P: int, lam: float, clamp: bool = False) -> torch.Tensor:
    l, cnt, _, _ = _avg_logps(s, labels)
    return trl_orpo_from_rows(l, cnt, P, lam, clamp)


# ================================================================================================= fp64 oracle
def token_terms(s, labels, V: int, ignore_index: int = -100) -> Dict:
    """Per token row of ``[T, Vp]`` logits (on their device, fp64): ``lse`` and its bound, ``lp`` and its bound (0 off ``R``)."""
    x = s[:, :V].double()
    vt = labels != ignore_index
    lab = torch.where(vt, labels, torch.zeros_like(labels))
    lse = torch.logsumexp(x, 1)
    lp = x.gather(1, lab[:, None])[:, 0] - lse
    z0 = torch.zeros_like(lse)
    E1, _ = _lse_bound(x, lse, V, False)
    return {"lse": lse, "E_lse": E1, "lp": torch.where(vt, lp, z0), "E_lp": torch.where(vt, E1 + U * lp.abs(), z0), "vt": vt}


def log1m_exp(a: torch.Tensor) -> torch.Tensor:
    return torch.where(a > -LN2, torch.log(-torch.expm1(a)), torch.log1p(-torch.exp(a)))


def _sp_sig(z, E_z):
    """softplus(-z), sigma(-z) and their bounds (the stable forms of ``dpo_reduce_kernel``)."""
    sp = torch.logaddexp(torch.zeros_like(z), -z)
    sig = torch.sigmoid(-z)
    e = torch.exp(-z.abs())
    return sp, sig, sig * E_z + e * e_exp(z.abs()) + 4 * U * (sp + z.abs()), sig * (1 - sig) * E_z + 8 * U * sig


def pair_stage(l, E_l, cnt, P: int, obj: str, coef: float, gamma: float = 0.0, l_abs=None) -> Dict:
    """fp64 oracle of ``pref_reduce`` from per-row ``l`` (fp64), its bound and the counts; ``l_abs`` = per-row sum of ``|lp|``."""
    l, E_l, cnt = l.double(), E_l.double(), cnt.double()
    l_abs = l.abs() if l_abs is None else l_abs.double()
    valid = (cnt[:P] > 0) & (cnt[P:] > 0)
    n = int(valid.sum())
    inv = 1.0 / n if n else 0.0
    c1 = cnt.clamp(min=1)
    a = l / c1
    E_a = E_l / c1 + 4 * U * a.abs()
    pair = torch.zeros(P, dtype=torch.float64)
    vsum = lambda v: float(torch.where(valid, v, pair).sum())
    mean_b = lambda sv, sa: 2 * ((sv + 12 * U * sa) * inv + 4 * U * sa * inv) + FTZ
    res = {"valid": valid, "n": n, "a": a}
    if obj == "simpo":
        rc, rr = coef * a[:P], coef * a[P:]
        E_rc, E_rr = coef * E_a[:P] + 2 * U * rc.abs(), coef * E_a[P:] + 2 * U * rr.abs()
        z = rc - rr - gamma
        E_z = E_rc + E_rr + U * (rc - rr).abs() + U * z.abs() + U * gamma
        sp, sig, E_sp, E_sig = _sp_sig(z, E_z)
        amb = vsum(((a[:P] - a[P:]).abs() <= 2 * (E_a[:P] + E_a[P:])).double())
        res.update(loss=vsum(sp) * inv, b_loss=mean_b(vsum(E_sp), vsum(sp)), out0=vsum(rc) * inv, b_out0=mean_b(vsum(E_rc), vsum(rc.abs())),
                   out1=vsum(rr) * inv, b_out1=mean_b(vsum(E_rr), vsum(rr.abs())), z=z)
        res.update(out2=vsum((a[:P] > a[P:]).double()) * inv, b_out2=(amb * inv + 16 * U) * 2 + FTZ)
        g = coef * sig * inv
        E_g = (coef * E_sig + 2 * U * coef * sig) * inv
        wc, wr = g / c1[:P], -g / c1[P:]
        E_wc, E_wr = E_g / c1[:P] + 4 * U * wc.abs(), E_g / c1[P:] + 4 * U * wr.abs()
    else:
        ap = a.clamp(max=A_MAX)
        L = log1m_exp(ap)
        hi = (ap + E_a).clamp(max=A_MAX)                      # the slope e^a / (1 - e^a) grows towards 0: take it at the interval's top
        slope = torch.exp(hi) / -torch.expm1(hi)
        E_L = slope * E_a + 2.0 ** -20 + 8 * U * L.abs() + 4 * e_exp(ap) * torch.exp(ap)
        h = a - L
        E_h = E_a + E_L + U * h.abs()
        lo = h[:P] - h[P:]
        E_lo = E_h[:P] + E_h[P:] + U * lo.abs()
        sp, sig, E_sp, E_sig = _sp_sig(lo, E_lo)
        n_c = vsum(cnt[:P])
        inv_nc = 1.0 / n_c if n_c else 0.0
        nll = -vsum(l[:P]) * inv_nc
        E_nll = (vsum(E_l[:P]) + 12 * U * vsum(l_abs[:P])) * inv_nc + 4 * U * abs(nll)
        m_sp, E_msp = vsum(sp) * inv, ((vsum(E_sp) + 12 * U * vsum(sp)) * inv + 4 * U * vsum(sp) * inv)
        loss = nll + coef * m_sp
        amb = vsum((lo.abs() <= 2 * E_lo).double())
        res.update(loss=loss, b_loss=2 * (E_nll + coef * E_msp + 2 * U * (abs(nll) + coef * m_sp)) + FTZ, out0=nll, b_out0=2 * E_nll + FTZ,
                   out1=vsum(lo) * inv, b_out1=mean_b(vsum(E_lo), vsum(lo.abs())), out2=vsum((lo > 0).double()) * inv,
                   b_out2=(amb * inv + 16 * U) * 2 + FTZ, lo=lo, ap=ap)
        q = -torch.expm1(ap)
        E_q = torch.exp(ap) * E_a + 2 * U * q
        g = coef * sig * inv
        E_g = (coef * E_sig + 2 * U * coef * sig) * inv
        t = g[None, :] / (c1.view(2, P) * q.view(2, P))
        E_t = t.abs() * ((E_g / g.clamp(min=1e-300))[None, :] + E_q.view(2, P) / q.view(2, P) + 8 * U)
        wc, wr = inv_nc + t[0], -t[1]
        E_wc, E_wr = E_t[0] + 4 * U * inv_nc + U * wc.abs(), E_t[1] + U * wr.abs()
    wc, wr = torch.where(valid, wc, pair), torch.where(valid, wr, pair)
    E_wc, E_wr = torch.where(valid, E_wc, pair), torch.where(valid, E_wr, pair)
    res.update(w=torch.cat([wc, wr]), E_w=torch.cat([E_wc, E_wr]))
    res["b_w"] = 2 * res["E_w"] + FTZ
    return res


def pref_ref(s, labels, P: int, V: int, obj: str, coef: float, gamma: float = 0.0, dloss: Optional[float] = None,
             terms: Optional[Dict] = None) -> Dict:
    """fp64 oracle of the SimPO / ORPO kernels on ``[2P S, Vp]`` logits and shifted labels ``[2P S]``, bounds included (``terms``:
    the :func:`token_terms` of all rows, computed elsewhere)."""
    tt = token_terms(s, labels, V) if terms is None else terms
    tt = {k: v.cpu() for k, v in tt.items()}
    Tn = tt["lp"].numel()
    S = Tn // (2 * P)
    lp, E_lp, vt = tt["lp"].view(2 * P, S), tt["E_lp"].view(2 * P, S), tt["vt"].view(2 * P, S)
    l, l_abs = lp.sum(1), lp.abs().sum(1)
    E_l = E_lp.sum(1) + (-(-S // 32) + 5) * U * l_abs
    res = pair_stage(l, E_l, vt.sum(1), P, obj, coef, gamma, l_abs)
    z0 = torch.zeros_like(tt["lse"])
    res.update(lse=torch.where(tt["vt"], tt["lse"], z0), b_lse=2 * torch.where(tt["vt"], tt["E_lse"], z0) + FTZ, l=l)
    if dloss is not None and terms is None:
        row = torch.arange(Tn) // S
        res["grad"], res["b_grad"] = dpo_grad_ref(s, labels, tt["lse"], tt["E_lse"], res["w"][row], res["E_w"][row], V, dloss)
    return res


def pref_checks(got, o) -> Dict[str, float]:
    out = {k: abs(float(got[k]) - o[k]) / o[f"b_{k}"] for k in ("loss", "out0", "out1", "out2")}
    for k in ("lse", "w", "grad"):
        if k in got:
            out[k] = ratio(got[k], o[k], o[f"b_{k}"])
    return out


# ================================================================================================= emulator
SIMPO_MUTANTS = ("sum_not_mean", "gamma_dropped", "gamma_sign", "beta_missing", "swapped", "prompt_counted", "invalid_counted")
ORPO_MUTANTS = ("nll_dropped", "nll_rejected_too", "log1m_dropped", "mean_prob_odds", "lambda_missing", "sum_not_mean",
                "invalid_counted")


def _f(v: float) -> float:
    return float(f32(torch.tensor(v)))


def emulate_pref(s, labels, P: int, V: int, obj: str, coef: float, gamma: float = 0.0, dloss: float = 1.0, mutant=None,
                 prompt_labels=None) -> Dict:
    """fp32 emulator of ``ce_fwd_kernel<false, false>`` (``kd_fwd_kernel``'s ``T == 1`` online max / sum), ``pref_reduce_kernel``
    (warp-per-row sums, one pair per thread, ``block_sum``) and ``dpo_bwd_kernel``."""
    Tn, Vp = s.shape
    S = Tn // (2 * P)
    lb = prompt_labels if mutant == "prompt_counted" else labels
    vt = lb != -100
    lse = emulate_kd(s, s, lb, V, 1.0, 1.0)["lse"][0]
    lab = torch.where(vt, lb, torch.zeros_like(lb))
    x = s.double()
    row_loss = torch.where(vt, f32(lse - x.gather(1, lab[:, None])[:, 0]), torch.zeros_like(lse))
    S32 = -(-S // 32) * 32
    terms = torch.zeros(2 * P, S32, dtype=torch.float64)
    terms[:, :S] = row_loss.view(2 * P, S)
    acc = torch.zeros(2 * P, 32, dtype=torch.float64)
    for k in range(S32 // 32):
        acc = f32(acc - terms[:, 32 * k: 32 * (k + 1)])
    l = _bfly(acc)
    cnt = vt.view(2 * P, S).sum(1).double()
    c1 = cnt.clamp(min=1)
    a = l if mutant == "sum_not_mean" else f32(l / c1)
    if mutant == "mean_prob_odds":                              # log of the mean token probability instead of the mean log-probability
        p = torch.where(vt, torch.exp(-row_loss), torch.zeros_like(row_loss)).view(2 * P, S).sum(1)
        a = f32(torch.log((p / c1).clamp(min=1e-300)))
    if mutant == "swapped":
        a, l, cnt = torch.cat([a[P:], a[:P]]), torch.cat([l[P:], l[:P]]), torch.cat([cnt[P:], cnt[:P]])
        c1 = cnt.clamp(min=1)
    valid = (cnt[:P] > 0) & (cnt[P:] > 0)
    if mutant == "invalid_counted":
        valid = torch.ones_like(valid)
    zero = torch.zeros(P, dtype=torch.float64)
    ac, ar = a[:P], a[P:]
    cf = _f(1.0 if mutant in ("beta_missing", "lambda_missing") else coef)
    gm = 0.0 if mutant == "gamma_dropped" else (-_f(gamma) if mutant == "gamma_sign" else _f(gamma))

    def sp_sig(z):
        e = f32(torch.exp(-z.abs()))
        sp = f32(f32(torch.clamp(-z, min=0)) + f32(torch.log1p(e)))
        sig = torch.where(z >= 0, f32(e / f32(1 + e)), f32(1 / f32(1 + e)))
        return sp, sig

    if obj == "simpo":
        rc, rr = f32(cf * ac), f32(cf * ar)
        z = f32(f32(rc - rr) - gm)
        sp, sig = sp_sig(z)
        sums = [_block_sum1024(torch.where(valid, v, zero)) for v in (valid.double(), sp, rc, rr, (ac > ar).double())]
        n = float(sums[0])
        inv = _f(1.0 / n) if n else 0.0
        g = torch.where(valid, f32(f32(cf * sig) * inv), zero)
        w = torch.cat([f32(g / c1[:P]), f32(-g / c1[P:])])
        loss, out = float(f32(sums[1] * inv)), [float(f32(sums[2] * inv)), float(f32(sums[3] * inv)), float(f32(sums[4] * inv))]
    else:
        def h(v):
            vp = torch.clamp(v, max=A_MAX)
            if mutant == "log1m_dropped":
                return v, vp
            L = torch.where(vp > -LN2, f32(torch.log(f32(-torch.expm1(vp)))), f32(torch.log1p(f32(-f32(torch.exp(vp))))))
            return f32(v - L), vp
        (hc, cc), (hr, cr) = h(ac), h(ar)
        lo = f32(hc - hr)
        sp, sig = sp_sig(lo)
        nl_terms = f32(l[:P] + l[P:]) if mutant == "nll_rejected_too" else l[:P]
        nc_terms = cnt[:P] + cnt[P:] if mutant == "nll_rejected_too" else cnt[:P]
        sums = [_block_sum1024(torch.where(valid, v, zero)) for v in (valid.double(), sp, nl_terms, lo, (lo > 0).double(), nc_terms)]
        n, sn = float(sums[0]), float(sums[5])
        inv = _f(1.0 / n) if n else 0.0
        inv_nc = _f(1.0 / sn) if sn else 0.0
        nll = 0.0 if mutant == "nll_dropped" else float(f32(-sums[2] * inv_nc))
        loss = float(f32(nll + f32(cf * f32(sums[1] * inv))))
        g = f32(f32(cf * sig) * inv)
        qc, qr = f32(-torch.expm1(cc)), f32(-torch.expm1(cr))
        if mutant == "log1m_dropped":
            qc, qr = torch.ones_like(qc), torch.ones_like(qr)
        base = 0.0 if mutant == "nll_dropped" else inv_nc
        wc = torch.where(valid, f32(base + f32(g / f32(c1[:P] * qc))), zero)
        wr = torch.where(valid, f32(-g / f32(c1[P:] * qr)), zero)
        w = torch.cat([wc, wr])
        out = [nll, float(f32(sums[3] * inv)), float(f32(sums[4] * inv))]
    if mutant == "swapped":
        w = torch.cat([w[P:], w[:P]])
    row = torch.arange(Tn) // S
    scale = f32(dloss * w[row])
    cols = torch.arange(Vp)
    p = torch.where(cols[None, :] < V, f32(torch.exp(f32(x - lse[:, None]))), torch.zeros_like(x))
    p = torch.where(cols[None, :] == lab[:, None], f32(p - 1), p)
    grad = bf16_rn(f32(p * scale[:, None])).double()
    grad = torch.where(vt[:, None], grad, torch.zeros_like(grad))
    if mutant == "prompt_counted":                       # the lse of the real response rows is what the kernel would keep
        lse = torch.where(labels != -100, lse, torch.zeros_like(lse))
    else:
        lse = torch.where(vt, lse, torch.zeros_like(lse))
    return {"lse": lse, "loss": loss, "out0": out[0], "out1": out[1], "out2": out[2], "w": w, "grad": grad, "a": a}


def pref_inputs(P: int, S: int, V: int, Vp: int, seed: int, scale: float = 3.0, sharp: float = 0.0, pad_fill: Optional[float] = None,
                invalid: bool = True):
    """``[2P S, Vp]`` bf16 logits, shifted labels with a random prompt / response / padding split per row, the labels a model counting
    prompt tokens would use, and the unshifted ``[2P, S]`` labels.  ``sharp`` is added to the label's logit on the response tokens
    (chosen rows get ``sharp``, rejected rows ``-sharp / 2``), so the chosen rows' mean log-probabilities approach 0 and the log odds
    ratios grow.  Pair 0's rejected row has its
    response cut away (``invalid``)."""
    g = torch.Generator().manual_seed(seed)
    Tn = 2 * P * S
    s = scale * torch.randn(Tn, Vp, generator=g)
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
    lb, plb = shift(lab), shift(plab)
    if sharp:
        rows = torch.arange(Tn) // S
        boost = torch.where(rows < P, sharp, -sharp / 2).float()
        m = lb != -100
        s[m, lb[m]] += boost[m]
    s = s.to(torch.bfloat16)
    if pad_fill is not None and Vp > V:
        s[:, V:] = pad_fill
    return s, lb, plb, lab


def _autograd(fn, s, V, P, S, lab2d, dloss):
    x = s[:, :V].double().view(2 * P, S, V).requires_grad_(True)
    loss = fn(x, lab2d)
    (dloss * loss).backward()
    return float(loss.detach()), x.grad.reshape(-1, V)


# ================================================================================================= oracle vs TRL autograd
@pytest.mark.parametrize("beta,gamma", [(0.5, 0.0), (2.5, 0.5), (2.5, 1.4), (0.5, 1.4)])
@pytest.mark.parametrize("V,Vp", [(37, 40), (40, 40), (1003, 1008)], ids=["ragged-padded", "exact", "ragged-1003"])
@pytest.mark.parametrize("scale", [3.0, 40.0], ids=["small-z", "large-z"])
def test_simpo_oracle_matches_trl_autograd(beta, gamma, V, Vp, scale):
    """Prompt masks, padding rows and columns, ragged V, an invalid pair, large |z| - against autograd of TRL's SimPO in fp64."""
    P, S = 3, 12
    s, lb, _, lab2d = pref_inputs(P, S, V, Vp, seed=V + int(scale), scale=scale, pad_fill=30.0)
    o = pref_ref(s, lb, P, V, "simpo", beta, gamma, dloss=1.5)
    want, grad = _autograd(lambda x, lab: trl_simpo(x, lab, P, beta, gamma), s, V, P, S, lab2d, 1.5)
    assert o["n"] == P - 1 and not bool(o["valid"][0])
    assert abs(o["loss"] - want) <= 1e-12 * max(1.0, abs(want))
    torch.testing.assert_close(o["grad"][:, :V], grad, rtol=1e-10, atol=1e-14)
    assert bool((o["grad"][:, V:] == 0).all()) and bool((o["grad"][lb == -100] == 0).all())
    if scale > 10 and beta > 1:
        assert float(o["z"].abs().max()) > 30                   # large |z|: the stable forms are exercised


@pytest.mark.parametrize("lam", [0.1, 1.0])
@pytest.mark.parametrize("V,Vp", [(37, 40), (40, 40), (1003, 1008)], ids=["ragged-padded", "exact", "ragged-1003"])
@pytest.mark.parametrize("sharp", [0.0, 12.0, 60.0], ids=["plain", "confident", "large-lo"])
def test_orpo_oracle_matches_trl_autograd(lam, V, Vp, sharp):
    """The same cases for ORPO, with confident rows (``a`` near 0, where ``log(1 - e^a)`` matters) and large ``|lo|``."""
    P, S = 3, 12
    s, lb, _, lab2d = pref_inputs(P, S, V, Vp, seed=V + int(sharp), sharp=sharp, pad_fill=30.0)
    o = pref_ref(s, lb, P, V, "orpo", lam, dloss=1.5)
    assert bool((o["a"][o["valid"].repeat(2)] < A_MAX).all()) or sharp == 60.0      # TRL's own formula is finite on these rows
    want, grad = _autograd(lambda x, lab: trl_orpo(x, lab, P, lam, clamp=True), s, V, P, S, lab2d, 1.5)
    assert o["n"] == P - 1
    assert abs(o["loss"] - want) <= 1e-12 * max(1.0, abs(want))
    torch.testing.assert_close(o["grad"][:, :V], grad, rtol=1e-9, atol=1e-9 * float(grad.abs().max()))
    assert bool((o["grad"][:, V:] == 0).all()) and bool((o["grad"][lb == -100] == 0).all())
    if sharp == 60.0:
        assert float(o["lo"].abs().max()) > 20


@pytest.mark.parametrize("a_c", [0.0, 3e-6, -1e-7], ids=["a-zero", "a-positive", "a-inside-clamp"])
def test_orpo_clamp_matches_trl_with_the_clamp_in_loss_and_gradient(a_c):
    """Rows whose mean log-probability is 0 exactly, above 0 (as fp32 fast-math can give) or between the clamp and 0: TRL's formula
    is inf / NaN there; with the clamp taken straight through it is finite, and the oracle is that, loss and gradient in l."""
    P, lam = 2, 0.1
    cnt = torch.tensor([4, 6, 5, 3], dtype=torch.float64)
    l = torch.tensor([a_c * 4, -1.2, -2.5, -0.9], dtype=torch.float64, requires_grad=True)
    o = pair_stage(l.detach(), torch.zeros(4, dtype=torch.float64), cnt, P, "orpo", lam)
    loss = trl_orpo_from_rows(l, cnt, P, lam, clamp=True)
    loss.backward()
    assert math.isfinite(float(loss.detach())) and o["loss"] == pytest.approx(float(loss.detach()), rel=1e-12)
    assert float(o["ap"][0]) == A_MAX
    # d loss / d l(row) = -w(row): the weight multiplies (softmax - onehot) = -d lp / d s
    torch.testing.assert_close(-o["w"], l.grad, rtol=1e-10, atol=0)
    if a_c >= 0.0:
        l2 = l.detach().clone().requires_grad_(True)
        plain = trl_orpo_from_rows(l2, cnt, P, lam, clamp=False)
        plain.backward()
        assert not (math.isfinite(float(plain.detach())) and bool(torch.isfinite(l2.grad).all()))      # what the clamp is for


def test_all_invalid_batch_has_zero_loss_and_gradient():
    from acco_b200 import ops
    P, S, V = 2, 8, 50
    s, lb, _, _ = pref_inputs(P, S, V, 56, seed=4)
    lb.view(2 * P, S)[P:] = -100                                # every rejected response cut away
    for obj, coef, gamma in (("simpo", 2.0, 0.5), ("orpo", 0.1, 0.0)):
        o = pref_ref(s, lb, P, V, obj, coef, gamma, dloss=1.0)
        assert o["n"] == 0 and o["loss"] == 0.0 and o["out2"] == 0.0 and bool((o["grad"] == 0).all())
        e = emulate_pref(s, lb, P, V, obj, coef, gamma)
        assert e["loss"] == 0.0 and bool((e["grad"] == 0).all())
        xs = s.float().requires_grad_(True)
        out = torch.full((3,), -1.0)
        loss = ops.simpo_loss(xs, lb, P, V, coef, gamma, out=out) if obj == "simpo" else ops.orpo_loss(xs, lb, P, V, coef, out=out)
        loss.backward()
        assert float(loss) == 0.0 and bool((xs.grad == 0).all()) and bool((out == 0).all())


# ================================================================================================= identities
def _identical_pairs(P, S, V, Vp, seed):
    s, lb, _, _ = pref_inputs(P, S, V, Vp, seed=seed, invalid=False)
    s.view(2 * P, S, Vp)[P:] = s.view(2 * P, S, Vp)[:P]
    lb.view(2 * P, S)[P:] = lb.view(2 * P, S)[:P]
    return s, lb


@pytest.mark.parametrize("gamma", [0.0, 0.5, 1.4])
def test_identical_pair_gives_softplus_gamma_for_simpo(gamma):
    P, S, V = 3, 10, 131
    s, lb = _identical_pairs(P, S, V, 136, seed=3)
    o = pref_ref(s, lb, P, V, "simpo", 2.5, gamma, dloss=1.0)
    assert o["loss"] == pytest.approx(math.log1p(math.exp(gamma)), abs=1e-14)
    assert torch.equal(o["w"][:P], -o["w"][P:]) and bool((o["w"][:P] > 0).all())
    e = emulate_pref(s, lb, P, V, "simpo", 2.5, gamma)
    assert e["loss"] == pytest.approx(math.log1p(math.exp(gamma)), rel=1e-6) and torch.equal(e["w"][:P], -e["w"][P:])
    from acco_b200 import ops
    assert float(ops.simpo_loss(s.float(), lb, P, V, 2.5, gamma)) == pytest.approx(math.log1p(math.exp(gamma)), rel=1e-6)


@pytest.mark.parametrize("lam", [0.1, 1.0])
def test_identical_pair_gives_nll_plus_lambda_ln2_for_orpo(lam):
    P, S, V = 3, 10, 131
    s, lb = _identical_pairs(P, S, V, 136, seed=5)
    o = pref_ref(s, lb, P, V, "orpo", lam, dloss=1.0)
    assert o["loss"] == pytest.approx(o["out0"] + lam * LN2, abs=1e-14) and o["out1"] == 0.0
    n_c = float(torch.where(lb != -100, 1.0, 0.0).view(2 * P, S)[:P].sum())
    assert o["out0"] == pytest.approx(-float(o["l"][:P].sum()) / n_c, rel=1e-14)
    torch.testing.assert_close(o["w"][:P] - 1.0 / n_c, -o["w"][P:], rtol=1e-12, atol=0)       # opposite odds-ratio weights
    from acco_b200 import ops
    out = torch.zeros(3)
    got = float(ops.orpo_loss(s.float(), lb, P, V, lam, out=out))
    assert got == pytest.approx(o["loss"], rel=1e-5) and out[1] == 0.0 and out[2] == 0.0


@pytest.mark.parametrize("obj", ["simpo", "orpo"])
def test_duplicated_positions_leave_the_mean_and_the_loss_unchanged(obj):
    """Length normalisation at the op level: every row's scored (logit row, label) positions written twice give the same ``a``."""
    from acco_b200 import ops
    P, S, V = 3, 8, 61
    s, lb, _, _ = pref_inputs(P, S, V, 64, seed=9)
    s2 = torch.cat([s.view(2 * P, S, -1)] * 2, 1).reshape(2 * P * 2 * S, -1)
    lb2 = torch.cat([lb.view(2 * P, S)] * 2, 1).reshape(-1)
    o1, o2 = pref_ref(s, lb, P, V, obj, 2.0, 0.5), pref_ref(s2, lb2, P, V, obj, 2.0, 0.5)
    torch.testing.assert_close(o1["a"], o2["a"], rtol=1e-14, atol=0)
    assert o1["loss"] == pytest.approx(o2["loss"], rel=1e-13)
    f = (lambda x, l: ops.simpo_loss(x, l, P, V, 2.0, 0.5)) if obj == "simpo" else (lambda x, l: ops.orpo_loss(x, l, P, V, 2.0))
    assert float(f(s.float(), lb)) == pytest.approx(float(f(s2.float(), lb2)), rel=1e-5)


# ================================================================================================= margin table
PREF_CASES = [
    # (name, objective, P, S, V, Vp, coef, gamma, logit scale, sharp, padding fill)
    ("simpo-P3-S16-V1003-b2.5-g0.5-pad", "simpo", 3, 16, 1003, 1008, 2.5, 0.5, 3.0, 0.0, 20.0),
    ("simpo-P4-S24-V131-b0.5-g1.4", "simpo", 4, 24, 131, 136, 0.5, 1.4, 3.0, 4.0, None),
    ("simpo-P2-S40-V40-b2.5-g0-large-z", "simpo", 2, 40, 40, 40, 2.5, 0.0, 40.0, 0.0, None),
    ("simpo-P2-S8-V50257-b2.5-g1.4", "simpo", 2, 8, 50257, 50304, 2.5, 1.4, 3.0, 0.0, 30.0),
    ("orpo-P3-S16-V1003-l0.1-pad", "orpo", 3, 16, 1003, 1008, 0.1, 0.0, 3.0, 0.0, 20.0),
    ("orpo-P4-S24-V131-l1-confident", "orpo", 4, 24, 131, 136, 1.0, 0.0, 3.0, 12.0, None),
    ("orpo-P2-S40-V40-l0.1-large-lo", "orpo", 2, 40, 40, 40, 0.1, 0.0, 3.0, 60.0, None),
    ("orpo-P2-S8-V50257-l1", "orpo", 2, 8, 50257, 50304, 1.0, 0.0, 3.0, 14.0, 30.0),
]


def pref_row(name, obj, P, S, V, Vp, coef, gamma, scale, sharp, pad_fill):
    s, lb, plb, _ = pref_inputs(P, S, V, Vp, seed=V + S, scale=scale, sharp=sharp, pad_fill=pad_fill)
    o = pref_ref(s, lb, P, V, obj, coef, gamma, dloss=0.75)
    emu = pref_checks(emulate_pref(s, lb, P, V, obj, coef, gamma, dloss=0.75), o)
    caught = {}
    for m in SIMPO_MUTANTS if obj == "simpo" else ORPO_MUTANTS:
        c = pref_checks(emulate_pref(s, lb, P, V, obj, coef, gamma, dloss=0.75, mutant=m, prompt_labels=plb), o)
        caught[m] = max(c.items(), key=lambda kv: kv[1])
    return emu, caught


ROWS = {c[0]: functools.lru_cache(maxsize=None)(lambda c=c: pref_row(*c)) for c in PREF_CASES}


@pytest.mark.parametrize("name", list(ROWS))
def test_margin_table_emulator_within_half(name):
    emu, _ = ROWS[name]()
    for k, v in emu.items():
        assert v < 0.5, (name, "emulator", k, v)


@pytest.mark.parametrize("obj,mutants", [("simpo", SIMPO_MUTANTS), ("orpo", ORPO_MUTANTS)])
def test_every_mutant_lands_far_outside_on_some_case(obj, mutants):
    best = {m: 0.0 for m in mutants}
    for name, row in ROWS.items():
        if not name.startswith(obj):
            continue
        _, caught = row()
        for m, (k, v) in caught.items():
            best[m] = max(best[m], v)
    assert all(v > 3.0 for v in best.values()), best


# ================================================================================================= op reference path
def test_op_reference_paths_match_trl_and_write_out():
    from acco_b200 import ops
    P, S, V = 3, 9, 37
    s, lb, _, lab2d = pref_inputs(P, S, V, 40, seed=6, sharp=5.0, pad_fill=5.0)
    for obj in ("simpo", "orpo"):
        out = torch.full((3,), -1.0)
        x = s.float().requires_grad_(True)
        got = ops.simpo_loss(x, lb, P, V, 2.0, 0.5, out=out) if obj == "simpo" else ops.orpo_loss(x, lb, P, V, 0.1, out=out)
        got.backward()
        xr = s[:, :V].float().view(2 * P, S, V).requires_grad_(True)
        ref = trl_simpo(xr, lab2d, P, 2.0, 0.5) if obj == "simpo" else trl_orpo(xr, lab2d, P, 0.1)
        ref.backward()
        assert float(got) == pytest.approx(float(ref), rel=1e-5)
        torch.testing.assert_close(x.grad[:, :V], xr.grad.reshape(-1, V), rtol=1e-4, atol=1e-7)
        assert bool((x.grad[:, V:] == 0).all())
        o = pref_ref(s, lb, P, V, obj, 2.0 if obj == "simpo" else 0.1, 0.5 if obj == "simpo" else 0.0)
        assert out.tolist() == pytest.approx([o["out0"], o["out1"], o["out2"]], rel=1e-5, abs=1e-6)
    x = s.float()
    for bad in (0.0, -0.1, math.inf, math.nan, True):
        with pytest.raises(ValueError, match="beta"):
            ops.simpo_loss(x, lb, P, V, bad, 0.5)
        with pytest.raises(ValueError, match="lambda"):
            ops.orpo_loss(x, lb, P, V, bad)
    for bad in (-0.1, math.inf, math.nan, True):
        with pytest.raises(ValueError, match="gamma"):
            ops.simpo_loss(x, lb, P, V, 2.0, bad)
    with pytest.raises(ValueError, match="2 P S rows"):
        ops.simpo_loss(x, lb, 4, V, 2.0, 0.5)
    with pytest.raises(ValueError, match="three-element"):
        ops.orpo_loss(x, lb, P, V, 0.1, out=torch.zeros(2))


# ================================================================================================= models
@pytest.mark.parametrize("make", [_tiny_llama, _tiny_gpt], ids=["llama-gqa", "gptneo"])
@pytest.mark.parametrize("obj", ["simpo", "orpo"])
def test_native_model_matches_the_formula(make, obj):
    """``preference_pairs=True`` with labels gives the loss and gradients of TRL's formula on the model's own logits (fp32)."""
    m = make(0).float()
    b = _pair_batch(3, 16, 90, seed=1)
    if obj == "simpo":
        m.simpo_beta, m.simpo_gamma = 2.0, 0.5
    else:
        m.orpo_lambda = 0.1
    m.pref_out = torch.zeros(3)
    loss = m(input_ids=b["input_ids"], labels=b["labels"], preference_pairs=True)[0]
    loss.backward()
    got = {k: p.grad.clone() for k, p in m.named_parameters()}
    m.zero_grad()
    logits = m(input_ids=b["input_ids"]).logits
    want = trl_simpo(logits, b["labels"], 3, 2.0, 0.5) if obj == "simpo" else trl_orpo(logits, b["labels"], 3, 0.1)
    want.backward()
    assert float(loss.detach()) == pytest.approx(float(want.detach()), rel=2e-6)
    for k, p in m.named_parameters():
        torch.testing.assert_close(got[k], p.grad, rtol=1e-4, atol=1e-5 * float(p.grad.abs().max()), msg=k)
    assert m(input_ids=b["input_ids"], labels=b["labels"])[0] is not None       # without the keyword: the cross-entropy, as before
    with pytest.raises(ValueError, match="labels"):
        m(input_ids=b["input_ids"], preference_pairs=True)
    with pytest.raises(ValueError, match="even number of rows"):
        m(input_ids=b["input_ids"][:3], labels=b["labels"][:3], preference_pairs=True)
    with pytest.raises(ValueError, match="no frozen model"):
        m(input_ids=b["input_ids"], labels=b["labels"], preference_pairs=True, reference_logits=m.padded_logits(b["input_ids"]).detach())
    with pytest.raises(ValueError, match="no frozen model"):
        m(input_ids=b["input_ids"], labels=b["labels"], preference_pairs=True, teacher_logits=m.padded_logits(b["input_ids"]).detach())
    m.simpo_beta = m.orpo_lambda = None
    with pytest.raises(ValueError, match="exactly one objective"):
        m(input_ids=b["input_ids"], labels=b["labels"], preference_pairs=True)


def test_labelled_forward_without_the_keyword_is_the_cross_entropy():
    m = _tiny_llama(0).float()
    b = _pair_batch(2, 16, 90, seed=2)
    want = float(m(input_ids=b["input_ids"], labels=b["labels"])[0])
    m.simpo_beta, m.pref_out = 2.0, torch.zeros(3)
    assert float(m(input_ids=b["input_ids"], labels=b["labels"])[0]) == want
    assert m.pref_out.tolist() == [0.0, 0.0, 0.0]


# ================================================================================================= trainer
class _PrefRef(torch.nn.Module):
    """A non-native model around the policy's weights whose loss is TRL's formula in plain torch: the plain PyTorch loop the trainer
    is checked against."""

    def __init__(self, m, obj, coef, gamma=0.5):
        super().__init__()
        self.m, self.obj, self.coef, self.gamma = m, obj, coef, gamma

    def forward(self, input_ids=None, labels=None, **kw):
        logits = self.m(input_ids=input_ids).logits.float()
        P = input_ids.shape[0] // 2
        if self.obj == "simpo":
            return (trl_simpo(logits, labels, P, self.coef, self.gamma),)
        return (trl_orpo(logits, labels, P, self.coef),)


KEYS = {"simpo": {"simpo_beta": 2.0, "simpo_gamma": 0.5}, "orpo": {"orpo_lambda": 0.1}}


def _trainer(model, obj="simpo", method="acco", ds="pairs", **kw):
    from acco_b200 import DecoupledTrainer
    from acco_b200.launch import DistEnv
    from helpers import LOG, base_args
    reference = kw.pop("reference", None)
    kw = {"nb_steps_tot": 8, "const_len_batch": False, **(KEYS[obj] if obj else {}), **kw}
    data = _pairs() if ds == "pairs" else ds
    return DecoupledTrainer(model=model, train_dataset=data, eval_dataset=_pairs(16, seed=8) if data is not None else None,
                            args=base_args(method_name=method, **kw), log=LOG, env=DistEnv(id_run="pref"), reference=reference)


@pytest.mark.parametrize("obj", ["simpo", "orpo"])
@pytest.mark.parametrize("method,impl", [("acco", "native"), ("dpu", "native"), ("ddp", "native"), ("ddp", "torch")])
def test_trainers_track_a_plain_pytorch_loop(workdir, obj, method, impl):
    from helpers import tiny_model
    kw = dict(ddp_impl=impl, log_every=1, nb_steps_tot=16)
    t = _trainer(tiny_model(), obj, method, **kw)
    assert t.model.pref_out is t.pref_static and t.pref_objective == obj and t.reference is None and t.teacher is None
    t.is_cuda = True                                       # graphs need a GPU; everything else about the route allows them
    assert t._use_graphs()
    t.is_cuda = False
    coef = 2.0 if obj == "simpo" else 0.1
    ref = _trainer(_PrefRef(tiny_model(), obj, coef), None, method, ds=None, **kw)
    ref.train_dataloader = t.get_train_dataloader()        # the same pairs in the same order, through the same collator
    a, b = _logged(t), _logged(ref)
    assert len(a) == len(b) >= 4
    acc = f"{obj}_accuracy"
    for x, y in zip(a, b):
        assert abs(x["loss"] - y["loss"]) <= 1e-5 * abs(y["loss"]), (a, b)
        assert acc in x and acc not in y and 0.0 <= x[acc] <= 1.0


@pytest.mark.parametrize("obj", ["simpo", "orpo"])
def test_eval_reports_the_objective_and_the_accuracy(workdir, obj):
    from acco_b200 import ops
    from helpers import tiny_model
    t = _trainer(tiny_model(), obj, max_eval_batches=3)
    t.pref_static.fill_(7.0)
    loss = float(t.eval_loop())
    assert t.pref_static.tolist() == [7.0, 7.0, 7.0]       # the logged training scalars are not overwritten
    batches = [b for _, b in zip(range(3), t.eval_dataloader)]
    want, accs = [], []
    with torch.no_grad():
        for b in batches:
            logits, P = t.model(input_ids=b["input_ids"]).logits, b["input_ids"].shape[0] // 2
            want.append(float(trl_simpo(logits, b["labels"], P, 2.0, 0.5) if obj == "simpo" else trl_orpo(logits, b["labels"], P, 0.1)))
            out, flat = torch.zeros(3), logits.reshape(-1, logits.shape[-1])
            if obj == "simpo":
                ops.simpo_loss(flat, shift(b["labels"]), P, flat.shape[1], 2.0, 0.5, out=out)
            else:
                ops.orpo_loss(flat, shift(b["labels"]), P, flat.shape[1], 0.1, out=out)
            accs.append(float(out[2]))
    assert loss == pytest.approx(sum(want) / len(want), rel=1e-5)
    assert t.eval_pref_accuracy == pytest.approx(sum(accs) / len(accs), abs=1e-6)


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
    args = base_args(method_name="acco", nb_steps_tot=16, batch_size=2, const_len_batch=False, orpo_lambda=0.1)
    t = DecoupledTrainer(model=tiny_model(seed=rank), train_dataset=synthetic_preference_dataset(64, 14, 95, seed=7), args=args, log=LOG)
    accs = []
    while not t.finished():
        t.step()
        accs.append(float(t.pref_host[2]))
    t._drain()
    t._finish("")
    q.put((rank, float(t.params.double().sum()), accs, t.len_params))
    shutdown_distributed()


def test_two_gloo_ranks_train_with_orpo(workdir):
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
    for bad in (0, 0.0, -0.1, math.nan, math.inf, True, "2"):
        with pytest.raises(ValueError, match="simpo_beta"):
            _trainer(tiny_model(), "simpo", simpo_beta=bad)
        with pytest.raises(ValueError, match="orpo_lambda"):
            _trainer(tiny_model(), "orpo", orpo_lambda=bad)
    for bad in (-0.1, math.nan, math.inf, True, "0.5"):
        with pytest.raises(ValueError, match="simpo_gamma"):
            _trainer(tiny_model(), "simpo", simpo_gamma=bad)
    for extra in ({"orpo_lambda": 0.1}, {"dpo_beta": 0.1}, {"distill_teacher": "/nonexistent"}):
        with pytest.raises(ValueError, match="at most one"):
            _trainer(tiny_model(), "simpo", **extra)
    with pytest.raises(ValueError, match="at most one"):
        _trainer(tiny_model(), "orpo", dpo_beta=0.1, reference=tiny_model(seed=9, layers=1))
    from acco_b200 import DecoupledTrainer
    from acco_b200.launch import DistEnv
    from helpers import LOG, base_args
    with pytest.raises(ValueError, match="at most one"):
        DecoupledTrainer(model=tiny_model(), train_dataset=_pairs(), args=base_args(const_len_batch=False, orpo_lambda=0.1), log=LOG,
                         env=DistEnv(id_run="pref"), teacher=tiny_model(seed=9, layers=1))
    with pytest.raises(ValueError, match="reference-free"):
        _trainer(tiny_model(), "simpo", reference=tiny_model(seed=9, layers=1))
    with pytest.raises(ValueError, match="reference-free"):
        _trainer(tiny_model(), "orpo", dpo_reference="/nonexistent")
    with pytest.raises(ValueError, match="native policy"):
        _trainer(_PrefRef(tiny_model(), "simpo", 2.0), "simpo")
    for key, val in (("label_smoothing_factor", 0.1), ("z_loss_weight", 1e-4), ("packing", True), ("document_mask", True),
                     ("const_len_batch", True)):
        for obj in ("simpo", "orpo"):
            with pytest.raises(ValueError, match=key):
                _trainer(tiny_model(), obj, **{key: val})
    for obj, key in (("simpo", "simpo_beta"), ("orpo", "orpo_lambda")):
        with pytest.raises(ValueError, match=f"{key} needs preference pairs"):
            _trainer(tiny_model(), obj, ds=synthetic_sft_dataset(32, 10, 95, 16))
    t = _trainer(tiny_model(), None, ds=synthetic_sft_dataset(32, 10, 95, 16))       # off
    assert t.pref_objective is None and t.model.pref_out is None


@pytest.mark.parametrize("obj", ["simpo", "orpo"])
def test_arena_and_checkpoint_hold_the_policy_only(workdir, obj):
    from helpers import tiny_model
    t = _trainer(tiny_model(), obj, save_optimizer=True)
    assert t.len_params == sum(p.numel() for p in t.model.parameters())
    t.train()
    ck = os.path.join(os.getcwd(), "ck", "policy.pt")
    t.save_checkpoint(ck)
    saved = torch.load(ck, map_location="cpu", weights_only=False)
    assert set(saved) == set(t.model.state_dict())
    assert sum(v.numel() for v in _tensors(saved)) == sum(v.numel() for v in t.model.state_dict().values())
    r2 = _trainer(tiny_model(seed=4), obj, resume_from=ck)
    for k, v in r2.model.state_dict().items():
        assert torch.equal(v, saved[k]), k


@pytest.mark.parametrize("obj", [None, "simpo", "orpo"])
def test_scalars_are_logged_only_with_their_objective(workdir, obj):
    from helpers import tiny_model
    from acco_b200.data import synthetic_sft_dataset
    from acco_b200.trainer import PREF_SCALARS
    if obj:
        t = _trainer(tiny_model(), obj, tensorboard=True, log_every=2, nb_steps_tot=10, eval=True, eval_step=4, max_eval_batches=2)
    else:
        t = _trainer(tiny_model(), None, ds=synthetic_sft_dataset(64, 10, 95, 16), tensorboard=True, log_every=2, nb_steps_tot=10)
    logs = _logged(t)
    t.writer.flush()
    rows = [json.loads(line) for line in open(os.path.join(t.writer.logdir, "scalars.jsonl"))]
    tags = {r["tag"] for r in rows}
    assert logs
    for o, names in PREF_SCALARS.items():
        if o != obj:
            assert all(k not in d for d in logs for k in names) and not (set(names) & tags)
    if not obj:
        return
    names = PREF_SCALARS[obj]
    for d in logs:
        assert 0.0 <= d[names[2]] <= 1.0 and d["loss"] > 0
    assert set(names) <= tags and sum(r["tag"] == names[2] for r in rows) == len(logs)
    assert any(f"eval_{names[2]}" in d for d in logs)


@pytest.mark.parametrize("key,val", [("simpo_beta", 2.0), ("orpo_lambda", 0.1)])
def test_cli_preference_data_without_a_reference(workdir, monkeypatch, key, val):
    sys.path.insert(0, ROOT)
    import main as cli
    from acco_b200 import DecoupledTrainer, ops
    from acco_b200.models import LlamaConfig, LlamaForCausalLM
    seen, srcs = [], []
    name = "simpo_loss" if key == "simpo_beta" else "orpo_loss"
    orig, orig_setup = getattr(ops, name), DecoupledTrainer._setup_frozen

    def loss(*a, **kw):
        seen.append((a[2], a[4]))
        return orig(*a, **kw)

    def setup(self, src, *a):
        srcs.append(src)
        return orig_setup(self, src, *a)
    monkeypatch.setattr(ops, name, loss)
    monkeypatch.setattr(DecoupledTrainer, "_setup_frozen", setup)
    torch.manual_seed(2)
    pol = LlamaForCausalLM(LlamaConfig(vocab_size=512, hidden_size=32, intermediate_size=48, num_hidden_layers=1, num_attention_heads=4,
                                       max_position_embeddings=64))      # config/model/tiny.yaml's vocabulary
    pdir = os.path.join(os.getcwd(), "pretrained")
    _write_hf_dir(pol, pdir)
    stats = cli.main(["train=acco-ft", "data=preference", "model=tiny", f"model.pretrained={pdir}", f"train.{key}={val}",
                      "train.nb_steps_tot=6", "train.batch_size=2", "train.max_length=32", "train.use_mixed_precision=False",
                      "data.synthetic_docs=64", "data.synthetic_mean_len=12", "train.eval=False", "run_name=pref", "train.save=False",
                      "train.dataloader_num_workers=0"])
    assert stats["count_grad_tot"] >= 6
    assert seen and set(seen) == {(2, val)}
    assert srcs and all(s is None for s in srcs)             # no reference (and no teacher) is loaded


if __name__ == "__main__":               # print the margin table: python tests/test_pref_free.py
    for name, row in ROWS.items():
        emu, caught = row()
        print(f"{name:36s} emulator/bound " + " ".join(f"{k}={v:.3f}" for k, v in emu.items()))
        for m, (k, v) in caught.items():
            print(f"{'':36s}   mutant {m:18s} worst {k}: {v:.3g}x")
