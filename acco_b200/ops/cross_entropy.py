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
The kernels take the row sum of the logits in the same streaming pass; ``eps = 0`` runs the unsmoothed kernels."""
from __future__ import annotations

import torch
import torch.nn.functional as F

from . import count_launch, load_ext, use_kernels


def softmax_cross_entropy_ref(logits: torch.Tensor, labels: torch.Tensor, valid_vocab: int, ignore_index: int = -100,
                              label_smoothing: float = 0.0) -> torch.Tensor:
    lg = logits[..., :valid_vocab].float().reshape(-1, valid_vocab)
    return F.cross_entropy(lg, labels.reshape(-1), ignore_index=ignore_index, reduction="mean", label_smoothing=float(label_smoothing))


class _CEFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, logits, labels, valid_vocab, ignore_index, label_smoothing):
        C = load_ext(required=True)
        lg = logits.reshape(-1, logits.shape[-1])
        assert lg.is_contiguous()
        lb = labels.reshape(-1).contiguous()
        loss, inv_n, lse = C.ce_fwd(lg, lb, int(valid_vocab), int(ignore_index), float(label_smoothing))
        count_launch("ce_fwd", 2)
        ctx.save_for_backward(lg, lb, lse, inv_n)
        ctx.valid_vocab, ctx.ignore_index, ctx.shape = int(valid_vocab), int(ignore_index), logits.shape
        ctx.label_smoothing = float(label_smoothing)
        return loss

    @staticmethod
    def backward(ctx, dloss):
        C = load_ext(required=True)
        lg, lb, lse, inv_n = ctx.saved_tensors
        scale = (dloss.float().reshape(1) * inv_n)
        C.ce_bwd_inplace(lg, lb, lse, scale, ctx.valid_vocab, ctx.ignore_index, ctx.label_smoothing)
        count_launch("ce_bwd")
        return lg.view(ctx.shape), None, None, None, None


def softmax_cross_entropy(logits: torch.Tensor, labels: torch.Tensor, valid_vocab: int = None, ignore_index: int = -100,
                          label_smoothing: float = 0.0) -> torch.Tensor:
    """Mean CE, smoothed by ``label_smoothing`` in [0, 1].  NOTE (kernel path): ``logits`` is consumed - its storage is reused
    for the gradient during backward, so it must not be read after this call."""
    V = int(valid_vocab) if valid_vocab is not None else logits.shape[-1]
    if use_kernels(logits) and logits.dtype == torch.bfloat16:
        return _CEFn.apply(logits, labels, V, ignore_index, label_smoothing)
    return softmax_cross_entropy_ref(logits, labels, V, ignore_index, label_smoothing)
