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
mean z-term, so the cross-entropy alone is ``loss - z_loss_out``; it is written on the device, without a host sync."""
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
