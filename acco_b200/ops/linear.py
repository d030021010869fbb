"""Linear layer with *fused gradient accumulation*.

Autograd would materialise ``dW`` and then run a separate ``grad += dW`` pass over every weight
.  When the weight's ``.grad`` already exists (it is a view of the flat gradient
arena) the wgrad GEMM accumulates straight into it (``beta = 1`` epilogue), and autograd sees
``None`` for the weight gradient.

On CUDA bf16 all three contractions run on the hand-written wgmma kernel (``ops/gemm.py`` ->
``csrc/gemm_wgmma.cu``): forward TN (+ bias in the epilogue), dgrad with the weight as an MN-major B
operand, wgrad with both operands MN-major, split-K and a TMA reduce-add epilogue that adds straight
into the arena view.  ``ACCO_GEMM=cublas`` switches back to the library GEMMs (A/B comparisons);
shapes a TMA tensor map cannot describe (row length not a multiple of 8) and non-bf16 dtypes use the
library path as well.  Reference: every ``nn.Linear`` of `trainer_decoupled.py:18-39`."""
from __future__ import annotations

from typing import Optional

import os

import torch
import torch.nn.functional as F


def _tc(*mats) -> bool:
    """Route to the hand-written wgmma GEMM?"""
    from . import use_kernels
    from .gemm import gemm_supported
    if os.environ.get("ACCO_GEMM", "") == "cublas":
        return False
    return use_kernels(*mats) and gemm_supported(*mats)


class LinearFn(torch.autograd.Function):
    @staticmethod
    @torch.amp.custom_fwd(device_type="cuda")
    def forward(ctx, x, weight, bias, accumulate_into_grad):
        ctx.save_for_backward(x, weight)
        ctx.has_bias = bias is not None
        ctx.accumulate = bool(accumulate_into_grad)
        ctx.weight_ref = weight
        ctx.bias_ref = bias
        x2 = x.reshape(-1, x.shape[-1])
        if _tc(x2, weight) and (bias is None or (bias.dtype == torch.bfloat16 and bias.data_ptr() % 16 == 0)):
            from .gemm import gemm_tn
            return gemm_tn(x2, weight.detach(), bias=None if bias is None else bias.detach()).view(*x.shape[:-1], weight.shape[0])
        return F.linear(x, weight, bias)        # under autocast (fp32 master weights, reference-parity DDP mode) this casts itself

    @staticmethod
    @torch.amp.custom_bwd(device_type="cuda")
    def backward(ctx, dy):
        return _linear_backward(ctx, dy)


_SIDE_STREAMS = {}


def _wgrad_stream(device):
    """``ACCO_WGRAD_STREAM=1``: run the wgrad GEMM on a side stream next to the dgrad GEMM (fork / join, CUDA-graph capturable).  The
    backward GEMMs of a 125M-class layer have 48-72 tiles for 74 CTA pairs, so each leaves 20-35 % of the SMs idle on its own; the two
    are independent (both only read dY) and fill each other's gaps when they run concurrently."""
    if os.environ.get("ACCO_WGRAD_STREAM", "0") != "1" or device.type != "cuda":
        return None
    key = (device.index, torch.cuda.current_stream(device).cuda_stream)
    st = _SIDE_STREAMS.get(key)
    if st is None:
        st = _SIDE_STREAMS[key] = torch.cuda.Stream(device=device)
    return st


def _linear_backward(ctx, dy):
    x, weight = ctx.saved_tensors
    dy2 = dy.reshape(-1, dy.shape[-1])
    x2 = x.reshape(-1, x.shape[-1])
    if dy2.dtype != weight.dtype or x2.dtype != dy2.dtype:
        # autocast forward ran in a lower precision than the stored weight / input: do the backward GEMMs in dy's dtype
        # and let the accumulation below cast back to the gradient's dtype
        weight_c, x2 = weight.to(dy2.dtype), x2.to(dy2.dtype)
    else:
        weight_c = weight
    tc = _tc(dy2, weight_c, x2)
    w = ctx.weight_ref
    acc_tc = (ctx.needs_input_grad[1] and ctx.accumulate and w.grad is not None and tc and w.grad.dtype == torch.bfloat16
              and w.grad.dim() == 2 and w.grad.stride(1) == 1 and w.grad.data_ptr() % 16 == 0)
    dx = dw = db = None
    side = _wgrad_stream(dy2.device) if (acc_tc and ctx.needs_input_grad[0]) else None
    if side is not None:
        # fork BEFORE either GEMM is enqueued: wgrad on the side stream, dgrad on the current one, join below
        from .gemm import gemm_tt_acc
        cur = torch.cuda.current_stream(dy2.device)
        side.wait_stream(cur)
        with torch.cuda.stream(side):
            gemm_tt_acc(dy2, x2, w.grad)
        dy2.record_stream(side)
        x2.record_stream(side)
    if ctx.needs_input_grad[0]:
        if tc:
            from .gemm import gemm_nn
            dx = gemm_nn(dy2, weight_c.detach()).view(x.shape)
        else:
            dx = dy2.matmul(weight_c).view(x.shape).to(x.dtype)
    if side is not None:
        torch.cuda.current_stream(dy2.device).wait_stream(side)     # join: later kernels (and the round that consumes the arena) see dW
    elif ctx.needs_input_grad[1]:
        if ctx.accumulate and w.grad is not None:
            if acc_tc:
                from .gemm import gemm_tt_acc
                gemm_tt_acc(dy2, x2, w.grad)             # split-K adds straight into the arena view
            elif w.grad.dtype == dy2.dtype:
                w.grad.addmm_(dy2.t(), x2)               # accumulate in the (library) GEMM epilogue
            else:
                w.grad.add_(dy2.t().matmul(x2))
        elif tc:
            from .gemm import gemm
            dw = gemm(dy2, x2, a_mn=True, b_mn=True)
        else:
            dw = dy2.t().matmul(x2).to(weight.dtype)
    if ctx.has_bias and ctx.needs_input_grad[2]:
        b = ctx.bias_ref
        if ctx.accumulate and b.grad is not None:
            b.grad.add_(dy2.sum(0))
        else:
            db = dy2.sum(0).to(b.dtype)
    return dx, dw, db, None


class GatherLinearFn(torch.autograd.Function):
    """Forward = KERNEL B (wgmma GEMM that all-gathers the remote row-blocks of ``weight`` over NVLink and
    writes them through to the local copy); backward = the usual dgrad (on the now complete local copy) and
    wgrad accumulation into the gradient arena."""

    @staticmethod
    def forward(ctx, x, weight, gathered, accumulate_into_grad):
        from .gemm import gemm_tn_gather
        ctx.save_for_backward(x, weight)
        ctx.has_bias = False
        ctx.accumulate = bool(accumulate_into_grad)
        ctx.weight_ref = weight
        ctx.bias_ref = None
        x2 = x.reshape(-1, x.shape[-1])
        return gemm_tn_gather(x2, weight.detach(), gathered).view(*x.shape[:-1], weight.shape[0])

    @staticmethod
    def backward(ctx, dy):
        dx, dw, _db, _ = _linear_backward(ctx, dy)
        return dx, dw, None, None


def linear(x: torch.Tensor, weight: torch.Tensor, bias: Optional[torch.Tensor] = None, accumulate_into_grad: bool = True,
           gathered=None) -> torch.Tensor:
    """``gathered``: a :class:`~acco_b200.ops.gemm.GatheredWeight` when this is the first use of ``weight`` after a
    communication round that left its remote row-blocks on their owners (fused all-gather + GEMM)."""
    if gathered is not None and bias is None and x.is_cuda:
        if torch.is_grad_enabled() and (weight.requires_grad or x.requires_grad):
            return GatherLinearFn.apply(x, weight, gathered, accumulate_into_grad)
        from .gemm import gemm_tn_gather
        x2 = x.reshape(-1, x.shape[-1])
        return gemm_tn_gather(x2, weight.detach(), gathered).view(*x.shape[:-1], weight.shape[0])
    if torch.is_grad_enabled() and (weight.requires_grad or x.requires_grad):
        return LinearFn.apply(x, weight, bias, accumulate_into_grad)
    return F.linear(x, weight, bias)
