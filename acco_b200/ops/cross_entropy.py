"""Softmax cross-entropy over (possibly vocab-padded) bf16 logits.

HF up-casts the whole ``[B*S, V]`` logits tensor to fp32, shifts and runs log_softmax + nll
(`transformers/loss/loss_utils.py:45-67`: 1.5 GiB of fp32 at 8x1024x50257).  Here
forward is one streaming pass that keeps only ``lse[T]`` (online max/sum in fp32) and backward
overwrites the logits buffer in place with ``(softmax - onehot) * scale`` (``csrc/ce.cu``).
Columns ``>= valid_vocab`` (alignment padding of the LM head) are excluded from the softmax and
receive zero gradient.  Labels equal to ``ignore_index`` contribute neither loss nor gradient;
the loss is the mean over the remaining rows (HF semantics).

``label_smoothing = eps > 0`` gives HF ``LabelSmoother`` / ``F.cross_entropy(label_smoothing=eps)`` over the valid vocabulary:
row loss ``lse - (1 - eps) x[label] - (eps / V) sum_c x_c``, gradient ``softmax - (1 - eps) onehot - eps / V`` on valid columns.
The kernels take the row sum of the logits in the same streaming pass; ``eps = 0`` runs the unsmoothed kernels.

``z_loss = z > 0`` adds PaLM's auxiliary z-loss, which keeps the softmax normaliser ``lse = log sum_{c<V} exp(x_c)`` near 0::

    loss = mean over rows r with label != ignore_index of [ ce_r + z lse_r^2 ]
    d x_rc = scale (softmax_rc (1 + 2 z lse_r) - (1 - eps) [c = y_r] - eps / V)      (c < V; padding and ignored rows: 0)

with ``ce_r`` the (smoothed) row loss above.  The forward adds the term from the ``lse`` it already computes, the backward forms
``1 + 2 z lse`` once per row; ``z = 0`` runs the kernels without the term.  ``z_loss_out`` (a one-element fp32 tensor) receives the
mean z-term, so the cross-entropy alone is ``loss - z_loss_out``; it is written on the device, without a host sync.

:func:`distill_cross_entropy` is knowledge distillation from a frozen teacher's logits ``t`` (same padded ``[T, Vp]`` layout),
temperature ``T > 0`` and weight ``a`` in (0, 1] (Hinton's forward KL, teacher entropy included, so >= 0 and 0 for ``t == s``)::

    loss = mean over rows r with label != -100 of  (1 - a) (lse(s_r) - s_r[y_r])  +  a T^2 KL(softmax(t_r / T) || softmax(s_r / T))
    d s_rc = scale ((1 - a) (softmax(s_r)_c - [c = y_r]) + a T (softmax(s_r / T)_c - softmax(t_r / T)_c))      (c < V; else 0)

The kernels make one streaming pass over both rows forward and one more backward (in place on ``s``), with no fp32 copy of
either; ``out`` (two fp32) receives the mean CE and the mean KL on the device.  The teacher logits are read, never written.

:func:`dpo_loss` is DPO (Rafailov et al. 2023) against a frozen reference's logits ``r`` (same padded layout).  The ``2P S`` rows are
``[2P, S]`` token rows: rows ``0..P-1`` the chosen responses, ``P..2P-1`` the rejected ones, pair ``i`` = rows ``(i, P+i)``; ``R(row)``
its positions whose (shifted) label is not -100::

    l(row) = sum_{t in R(row)} (s_t[y_t] - lse(s_t)),   l_ref(row) the same over r
    z_i    = beta ((l(c_i) - l_ref(c_i)) - (l(r_i) - l_ref(r_i)))
    loss   = (1/n) sum over valid pairs (both rows have a response token) of softplus(-z_i)        (n = 0: loss 0, gradient 0)
    d s_tc = +-(beta sigma(-z_i) / n) (softmax(s_t)_c - [c = y_t])       (+ chosen, - rejected; c < V; else 0)

The forward makes one streaming pass over both rows and takes the per-token difference of the two log-probabilities before any
sum, so equal policy and reference logits give ``z = 0`` exactly; a one-CTA reduction forms the loss and the per-row weights, and
the backward writes the gradient in place over ``s``.  ``out`` (three fp32) receives the mean chosen reward ``beta (l - l_ref)(c)``,
the mean rejected reward and the accuracy (fraction of valid pairs with ``z > 0``) on the device.

:func:`simpo_loss` (SimPO, Meng et al. 2024; TRL ``CPOTrainer(loss_type="simpo")`` without the NLL term) and :func:`orpo_loss` (ORPO,
Hong et al. 2024; TRL ``ORPOTrainer``) take the same pair layout and need no reference.  With ``a(row) = l(row) / |row|`` the mean
log-probability of the row's response tokens and ``n`` the number of valid pairs::

    SimPO:  z_i  = beta (a(c_i) - a(r_i)) - gamma,    loss = (1/n) sum_valid softplus(-z_i)
            d s_tc = +-(beta sigma(-z_i) / (n |row|)) (softmax(s_t)_c - [c = y_t])
    ORPO:   nll  = -(1/N_c) sum_valid l(c_i)    (N_c = sum_valid |c_i|)
            lo_i = (a(c_i) - log(1 - e^a'(c_i))) - (a(r_i) - log(1 - e^a'(r_i))),   a' = min(a, -2^-20)
            loss = nll + lambda (1/n) sum_valid softplus(-lo_i)
            d s_tc = (1/N_c + lambda sigma(-lo_i) / (n |c_i| (1 - e^a'(c_i)))) (softmax - onehot)          (chosen)
                     -(lambda sigma(-lo_i) / (n |r_i| (1 - e^a'(r_i)))) (softmax - onehot)                  (rejected)

The clamp ``a'`` keeps ``log(1 - e^a)`` finite once the policy is certain of every response token (``a`` can reach 0, and in fp32
even pass it); it is applied in the loss and, straight through, in the gradient.  No valid pair: loss 0 and gradient 0.  The forward
is the cross-entropy's streaming pass (``lse`` and ``-log p`` per token) and one one-CTA reduction to the loss and a weight per row;
the backward is DPO's, in place over ``s``.  ``out`` (three fp32) receives, on the device, SimPO's mean chosen reward ``beta a(c)``,
mean rejected reward and accuracy (fraction of valid pairs with ``a(c) > a(r)``; gamma is not part of it), or ORPO's ``nll``, mean
``lo`` and accuracy (fraction with ``lo > 0``)."""
from __future__ import annotations

import math
from typing import Optional

import torch
import torch.nn.functional as F

from . import count_launch, load_ext, use_kernels


def softmax_cross_entropy_ref(logits: torch.Tensor, labels: torch.Tensor, valid_vocab: int, ignore_index: int = -100,
                              label_smoothing: float = 0.0, z_loss: float = 0.0,
                              z_loss_out: Optional[torch.Tensor] = None) -> torch.Tensor:
    lg = logits[..., :valid_vocab].float().reshape(-1, valid_vocab)
    lb = labels.reshape(-1)
    loss = F.cross_entropy(lg, lb, ignore_index=ignore_index, reduction="mean", label_smoothing=float(label_smoothing))
    if not z_loss:
        return loss
    valid = lb != ignore_index
    zterm = (float(z_loss) * torch.logsumexp(lg[valid], -1).square()).sum() / valid.sum().clamp(min=1)
    if z_loss_out is not None:
        z_loss_out.copy_(zterm.detach().reshape(z_loss_out.shape))
    return loss + zterm


def _check_z_loss(z_loss: float, z_loss_out: Optional[torch.Tensor]) -> None:
    if not (math.isfinite(z_loss) and z_loss >= 0.0):
        raise ValueError(f"z_loss must be finite and >= 0, got {z_loss!r}")
    if z_loss_out is not None and (z_loss_out.numel() != 1 or z_loss_out.dtype != torch.float32):
        raise ValueError("z_loss_out must be a one-element fp32 tensor")


class _CEFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, logits, labels, valid_vocab, ignore_index, label_smoothing, z_loss, z_loss_out):
        C = load_ext(required=True)
        lg = logits.reshape(-1, logits.shape[-1])
        assert lg.is_contiguous()
        lb = labels.reshape(-1).contiguous()
        if z_loss and z_loss_out is None:
            z_loss_out = torch.empty(1, device=lg.device, dtype=torch.float32)
        loss, inv_n, lse = C.ce_fwd(lg, lb, int(valid_vocab), int(ignore_index), float(label_smoothing), float(z_loss), z_loss_out)
        count_launch("ce_fwd", 2)
        ctx.save_for_backward(lg, lb, lse, inv_n)
        ctx.valid_vocab, ctx.ignore_index, ctx.shape = int(valid_vocab), int(ignore_index), logits.shape
        ctx.label_smoothing, ctx.z_loss = float(label_smoothing), float(z_loss)
        return loss

    @staticmethod
    def backward(ctx, dloss):
        C = load_ext(required=True)
        lg, lb, lse, inv_n = ctx.saved_tensors
        scale = (dloss.float().reshape(1) * inv_n)
        C.ce_bwd_inplace(lg, lb, lse, scale, ctx.valid_vocab, ctx.ignore_index, ctx.label_smoothing, ctx.z_loss)
        count_launch("ce_bwd")
        return lg.view(ctx.shape), None, None, None, None, None, None


def softmax_cross_entropy(logits: torch.Tensor, labels: torch.Tensor, valid_vocab: int = None, ignore_index: int = -100,
                          label_smoothing: float = 0.0, z_loss: float = 0.0, z_loss_out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Mean CE, smoothed by ``label_smoothing`` in [0, 1], plus ``z_loss`` times the mean ``lse^2`` (written to ``z_loss_out`` when
    given and ``z_loss > 0``).  NOTE (kernel path): ``logits`` is consumed - its storage is reused for the gradient during backward,
    so it must not be read after this call."""
    V = int(valid_vocab) if valid_vocab is not None else logits.shape[-1]
    z_loss = float(z_loss)
    _check_z_loss(z_loss, z_loss_out)
    if use_kernels(logits) and logits.dtype == torch.bfloat16:
        return _CEFn.apply(logits, labels, V, ignore_index, label_smoothing, z_loss, z_loss_out)
    return softmax_cross_entropy_ref(logits, labels, V, ignore_index, label_smoothing, z_loss, z_loss_out)


# ------------------------------------------------------------------------------------------------ knowledge distillation
def distill_cross_entropy_ref(logits: torch.Tensor, teacher_logits: torch.Tensor, labels: torch.Tensor, valid_vocab: int, alpha: float,
                              temperature: float, out: Optional[torch.Tensor] = None, ignore_index: int = -100) -> torch.Tensor:
    """fp32 reference of :func:`distill_cross_entropy` (the CPU and non-bf16 path)."""
    V, T, a = int(valid_vocab), float(temperature), float(alpha)
    x = logits[..., :V].float().reshape(-1, V)
    t = teacher_logits[..., :V].detach().float().reshape(-1, V)
    lb = labels.reshape(-1)
    valid = lb != ignore_index
    n = valid.sum().clamp(min=1)
    ce = F.cross_entropy(x, lb, ignore_index=ignore_index, reduction="sum") / n
    lq = torch.log_softmax(t[valid] / T, -1)
    kl = (lq.exp() * (lq - torch.log_softmax(x[valid] / T, -1))).sum() / n
    if out is not None:
        out.copy_(torch.stack([ce.detach(), kl.detach()]).reshape(out.shape))
    return (1.0 - a) * ce + a * T * T * kl


def _check_distill(alpha: float, temperature: float, out: Optional[torch.Tensor]) -> None:
    if isinstance(alpha, bool) or not (math.isfinite(alpha) and 0.0 < alpha <= 1.0):
        raise ValueError(f"alpha must be in (0, 1], got {alpha!r}")
    if isinstance(temperature, bool) or not (math.isfinite(temperature) and temperature > 0.0):
        raise ValueError(f"temperature must be finite and > 0, got {temperature!r}")
    if out is not None and (out.numel() != 2 or out.dtype != torch.float32):
        raise ValueError("out must be a two-element fp32 tensor")


class _KDFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, logits, teacher_logits, labels, valid_vocab, alpha, temperature, out):
        C = load_ext(required=True)
        lg = logits.reshape(-1, logits.shape[-1])
        tl = teacher_logits.reshape(-1, teacher_logits.shape[-1])
        assert lg.is_contiguous() and tl.is_contiguous()
        lb = labels.reshape(-1).contiguous()
        if out is None:
            out = torch.empty(2, device=lg.device, dtype=torch.float32)
        loss, inv_n, lse3 = C.kd_fwd(lg, tl, lb, int(valid_vocab), -100, float(alpha), float(temperature), out)
        count_launch("kd_fwd", 2)
        ctx.save_for_backward(lg, tl, lb, lse3, inv_n)
        ctx.valid_vocab, ctx.shape, ctx.alpha, ctx.temperature = int(valid_vocab), logits.shape, float(alpha), float(temperature)
        return loss

    @staticmethod
    def backward(ctx, dloss):
        C = load_ext(required=True)
        lg, tl, lb, lse3, inv_n = ctx.saved_tensors
        scale = dloss.float().reshape(1) * inv_n
        C.kd_bwd_inplace(lg, tl, lb, lse3, scale, ctx.valid_vocab, -100, ctx.alpha, ctx.temperature)
        count_launch("kd_bwd")
        return lg.view(ctx.shape), None, None, None, None, None, None


def distill_cross_entropy(logits: torch.Tensor, teacher_logits: torch.Tensor, labels: torch.Tensor, V: int, alpha: float,
                          temperature: float, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """``(1 - alpha)`` mean CE plus ``alpha T^2`` mean forward KL to the teacher's tempered softmax over the rows whose (shifted)
    label is not -100; ``out`` (two fp32), when given, receives the mean CE and the mean KL.  The teacher gets no gradient.
    NOTE (kernel path): ``logits`` is consumed - its storage is reused for the gradient during backward."""
    _check_distill(alpha, temperature, out)
    alpha, temperature = float(alpha), float(temperature)
    if teacher_logits.shape != logits.shape:
        raise ValueError(f"teacher_logits {tuple(teacher_logits.shape)} must match the student logits {tuple(logits.shape)}")
    if use_kernels(logits, teacher_logits) and logits.dtype == torch.bfloat16:
        return _KDFn.apply(logits, teacher_logits.detach(), labels, int(V), alpha, temperature, out)
    return distill_cross_entropy_ref(logits, teacher_logits, labels, V, alpha, temperature, out)


# ------------------------------------------------------------------------------------------------ DPO
def dpo_loss_ref(logits: torch.Tensor, ref_logits: torch.Tensor, labels: torch.Tensor, P: int, valid_vocab: int, beta: float,
                 out: Optional[torch.Tensor] = None, ignore_index: int = -100) -> torch.Tensor:
    """fp32 reference of :func:`dpo_loss` (the CPU and non-bf16 path)."""
    V, P = int(valid_vocab), int(P)
    x = logits[..., :V].float().reshape(-1, V)
    r = ref_logits[..., :V].detach().float().reshape(-1, V)
    lb = labels.reshape(-1)
    mask = lb != ignore_index
    idx = torch.where(mask, lb, torch.zeros_like(lb))[:, None]
    d = torch.log_softmax(x, -1).gather(1, idx)[:, 0] - torch.log_softmax(r, -1).gather(1, idx)[:, 0]
    D = torch.where(mask, d, torch.zeros_like(d)).view(2 * P, -1).sum(1)
    cnt = mask.view(2 * P, -1).sum(1)
    valid = (cnt[:P] > 0) & (cnt[P:] > 0)
    n = valid.sum().clamp(min=1)
    rc, rr = beta * D[:P], beta * D[P:]
    z = rc - rr
    loss = torch.where(valid, F.softplus(-z), torch.zeros_like(z)).sum() / n
    if out is not None:
        zero = torch.zeros_like(z)
        vals = [torch.where(valid, v, zero).sum() / n for v in (rc.detach(), rr.detach(), (z.detach() > 0).float())]
        out.copy_(torch.stack(vals).reshape(out.shape))
    return loss


def _check_dpo(beta: float, out: Optional[torch.Tensor]) -> None:
    if isinstance(beta, bool) or not (math.isfinite(beta) and beta > 0.0):
        raise ValueError(f"beta must be finite and > 0, got {beta!r}")
    if out is not None and (out.numel() != 3 or out.dtype != torch.float32):
        raise ValueError("out must be a three-element fp32 tensor")


class _DPOFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, logits, ref_logits, labels, P, valid_vocab, beta, out):
        C = load_ext(required=True)
        lg = logits.reshape(-1, logits.shape[-1])
        rl = ref_logits.reshape(-1, ref_logits.shape[-1])
        assert lg.is_contiguous() and rl.is_contiguous()
        lb = labels.reshape(-1).contiguous()
        if out is None:
            out = torch.empty(3, device=lg.device, dtype=torch.float32)
        loss, lse, w = C.dpo_fwd(lg, rl, lb, int(P), int(valid_vocab), -100, float(beta), out)
        count_launch("dpo_fwd", 2)
        ctx.save_for_backward(lg, lb, lse, w)
        ctx.P, ctx.valid_vocab, ctx.shape = int(P), int(valid_vocab), logits.shape
        return loss

    @staticmethod
    def backward(ctx, dloss):
        C = load_ext(required=True)
        lg, lb, lse, w = ctx.saved_tensors
        C.dpo_bwd_inplace(lg, lb, lse, w, dloss.float().reshape(1).contiguous(), ctx.P, ctx.valid_vocab, -100)
        count_launch("dpo_bwd")
        return lg.view(ctx.shape), None, None, None, None, None, None


def dpo_loss(logits: torch.Tensor, ref_logits: torch.Tensor, labels: torch.Tensor, P: int, V: int, beta: float,
             out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """The DPO objective of ``P`` preference pairs laid out as ``2P`` rows of ``S`` tokens (chosen rows first); ``labels`` are the
    shifted labels of the ``2P S`` rows, -100 off the responses.  ``out`` (three fp32), when given, receives the mean chosen reward,
    the mean rejected reward and the accuracy.  The reference gets no gradient.
    NOTE (kernel path): ``logits`` is consumed - its storage is reused for the gradient during backward."""
    _check_dpo(beta, out)
    beta, P = float(beta), int(P)
    if ref_logits.shape != logits.shape:
        raise ValueError(f"ref_logits {tuple(ref_logits.shape)} must match the policy logits {tuple(logits.shape)}")
    rows = logits.reshape(-1, logits.shape[-1]).shape[0]
    if P <= 0 or rows % (2 * P) != 0 or labels.numel() != rows:
        raise ValueError(f"dpo_loss needs 2 P S rows and one label per row, got {rows} rows, {labels.numel()} labels and P={P}")
    if use_kernels(logits, ref_logits) and logits.dtype == torch.bfloat16:
        return _DPOFn.apply(logits, ref_logits.detach(), labels, P, int(V), beta, out)
    return dpo_loss_ref(logits, ref_logits, labels, P, V, beta, out)


# ------------------------------------------------------------------------------------------------ SimPO / ORPO
ORPO_MAX_MEAN_LOGP = -(2.0 ** -20)       # ORPO's clamp a' = min(a, -2^-20): log(1 - e^a') stays finite


def _row_mean_logps(logits: torch.Tensor, labels: torch.Tensor, P: int, valid_vocab: int, ignore_index: int):
    """Per row of the ``[2P, S]`` layout: ``l`` (sum of the response tokens' log-probabilities), the token count, ``a = l / count``
    (0 on an empty row), and per pair whether both rows have a response token."""
    V = int(valid_vocab)
    x = logits[..., :V].float().reshape(-1, V)
    lb = labels.reshape(-1)
    mask = lb != ignore_index
    idx = torch.where(mask, lb, torch.zeros_like(lb))[:, None]
    lp = torch.log_softmax(x, -1).gather(1, idx)[:, 0]
    l = torch.where(mask, lp, torch.zeros_like(lp)).view(2 * P, -1).sum(1)
    cnt = mask.view(2 * P, -1).sum(1)
    valid = (cnt[:P] > 0) & (cnt[P:] > 0)
    return l, cnt, l / cnt.clamp(min=1), valid


def log1m_exp(a: torch.Tensor) -> torch.Tensor:
    """``log(1 - e^a)`` for ``a < 0``: ``log(-expm1(a))`` above ``-ln 2``, ``log1p(-exp(a))`` below (no cancellation on either side)."""
    return torch.where(a > -math.log(2.0), torch.log(-torch.expm1(a)), torch.log1p(-torch.exp(a)))


def orpo_log_odds(a: torch.Tensor) -> torch.Tensor:
    """``a - log(1 - e^a')`` with ``a' = min(a, -2^-20)`` taken straight through: the value uses ``a'``, the gradient is
    ``1 / (1 - e^a')`` whether or not the clamp is active."""
    ac = a + (a.clamp(max=ORPO_MAX_MEAN_LOGP) - a).detach()
    return a - log1m_exp(ac)


def simpo_loss_ref(logits: torch.Tensor, labels: torch.Tensor, P: int, valid_vocab: int, beta: float, gamma: float,
                   out: Optional[torch.Tensor] = None, ignore_index: int = -100) -> torch.Tensor:
    """fp32 reference of :func:`simpo_loss` (the CPU and non-bf16 path)."""
    P = int(P)
    _, _, a, valid = _row_mean_logps(logits, labels, P, valid_vocab, ignore_index)
    n = valid.sum().clamp(min=1)
    rc, rr = beta * a[:P], beta * a[P:]
    z = rc - rr - gamma
    zero = torch.zeros_like(z)
    loss = torch.where(valid, F.softplus(-z), zero).sum() / n
    if out is not None:
        vals = [torch.where(valid, v, zero).sum() / n for v in (rc.detach(), rr.detach(), (a[:P] > a[P:]).float())]
        out.copy_(torch.stack(vals).reshape(out.shape))
    return loss


def orpo_loss_ref(logits: torch.Tensor, labels: torch.Tensor, P: int, valid_vocab: int, lam: float, out: Optional[torch.Tensor] = None,
                  ignore_index: int = -100) -> torch.Tensor:
    """fp32 reference of :func:`orpo_loss` (the CPU and non-bf16 path)."""
    P = int(P)
    l, cnt, a, valid = _row_mean_logps(logits, labels, P, valid_vocab, ignore_index)
    n = valid.sum().clamp(min=1)
    lo = orpo_log_odds(a[:P]) - orpo_log_odds(a[P:])
    zero = torch.zeros_like(lo)
    n_c = torch.where(valid, cnt[:P], torch.zeros_like(cnt[:P])).sum().clamp(min=1)
    nll = -torch.where(valid, l[:P], zero).sum() / n_c
    loss = nll + lam * torch.where(valid, F.softplus(-lo), zero).sum() / n
    if out is not None:
        vals = [nll.detach(), torch.where(valid, lo.detach(), zero).sum() / n, torch.where(valid, (lo.detach() > 0).float(), zero).sum() / n]
        out.copy_(torch.stack(vals).reshape(out.shape))
    return loss


def _check_pref(logits: torch.Tensor, labels: torch.Tensor, P: int, coefs, out: Optional[torch.Tensor]) -> None:
    """``coefs``: (name, value, strictly positive) of each hyper-parameter."""
    for name, v, positive in coefs:
        if isinstance(v, bool) or not isinstance(v, (int, float)) or not math.isfinite(v) or v < 0.0 or (positive and v == 0.0):
            raise ValueError(f"{name} must be finite and {'>' if positive else '>='} 0, got {v!r}")
    if out is not None and (out.numel() != 3 or out.dtype != torch.float32):
        raise ValueError("out must be a three-element fp32 tensor")
    rows = logits.reshape(-1, logits.shape[-1]).shape[0]
    if P <= 0 or rows % (2 * P) != 0 or labels.numel() != rows:
        raise ValueError(f"the preference loss needs 2 P S rows and one label per row, got {rows} rows, {labels.numel()} labels and P={P}")


class _PrefFn(torch.autograd.Function):
    """SimPO (``orpo`` false) or ORPO through ``pref_fwd``; the backward is DPO's in-place kernel with the per-row weights."""

    @staticmethod
    def forward(ctx, logits, labels, P, valid_vocab, orpo, coef, gamma, out):
        C = load_ext(required=True)
        lg = logits.reshape(-1, logits.shape[-1])
        assert lg.is_contiguous()
        lb = labels.reshape(-1).contiguous()
        if out is None:
            out = torch.empty(3, device=lg.device, dtype=torch.float32)
        loss, lse, w = C.pref_fwd(lg, lb, int(P), int(valid_vocab), -100, bool(orpo), float(coef), float(gamma), out)
        count_launch("ce_fwd")
        count_launch("pref_reduce")
        ctx.save_for_backward(lg, lb, lse, w)
        ctx.P, ctx.valid_vocab, ctx.shape = int(P), int(valid_vocab), logits.shape
        return loss

    @staticmethod
    def backward(ctx, dloss):
        C = load_ext(required=True)
        lg, lb, lse, w = ctx.saved_tensors
        C.dpo_bwd_inplace(lg, lb, lse, w, dloss.float().reshape(1).contiguous(), ctx.P, ctx.valid_vocab, -100)
        count_launch("dpo_bwd")
        return lg.view(ctx.shape), None, None, None, None, None, None, None


def simpo_loss(logits: torch.Tensor, labels: torch.Tensor, P: int, V: int, beta: float, gamma: float,
               out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """The SimPO objective of ``P`` preference pairs laid out as ``2P`` rows of ``S`` tokens (chosen rows first); ``labels`` are the
    shifted labels of the ``2P S`` rows, -100 off the responses.  ``out`` (three fp32), when given, receives the mean chosen reward,
    the mean rejected reward and the accuracy.
    NOTE (kernel path): ``logits`` is consumed - its storage is reused for the gradient during backward."""
    P = int(P)
    _check_pref(logits, labels, P, (("beta", beta, True), ("gamma", gamma, False)), out)
    if use_kernels(logits) and logits.dtype == torch.bfloat16:
        return _PrefFn.apply(logits, labels, P, int(V), False, float(beta), float(gamma), out)
    return simpo_loss_ref(logits, labels, P, V, float(beta), float(gamma), out)


def orpo_loss(logits: torch.Tensor, labels: torch.Tensor, P: int, V: int, lam: float, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """The ORPO objective (the chosen responses' NLL plus ``lam`` times the mean odds-ratio loss) of ``P`` preference pairs in the
    layout of :func:`simpo_loss`.  ``out`` (three fp32), when given, receives the NLL, the mean log odds ratio and the accuracy.
    NOTE (kernel path): ``logits`` is consumed - its storage is reused for the gradient during backward."""
    P = int(P)
    _check_pref(logits, labels, P, (("lambda", lam, True),), out)
    if use_kernels(logits) and logits.dtype == torch.bfloat16:
        return _PrefFn.apply(logits, labels, P, int(V), True, float(lam), 0.0, out)
    return orpo_loss_ref(logits, labels, P, V, float(lam), out)
