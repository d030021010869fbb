"""RMSNorm and fused residual-add + RMSNorm (fp32 statistics, bf16 I/O).

HF Llama computes the norm as ~7 eager kernels with an fp32 round trip
(`transformers/models/llama/modeling_llama.py:53-70`); here forward is one pass
(``csrc/norm.cu``) that also emits ``rstd`` for the backward, and the residual add of the
surrounding block is folded in (``h = a + r; y = norm(h) * w``)."""
from __future__ import annotations

from typing import Tuple

import torch

from . import count_launch, load_ext, use_kernels


def rmsnorm_ref(x: torch.Tensor, weight: torch.Tensor, eps: float) -> torch.Tensor:
    xf = x.float()
    rstd = torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + eps)
    return (xf * rstd * weight.float()).to(x.dtype)


def add_rmsnorm_ref(a: torch.Tensor, r: torch.Tensor, weight: torch.Tensor, eps: float) -> Tuple[torch.Tensor, torch.Tensor]:
    h = (a.float() + r.float()).to(a.dtype)
    return rmsnorm_ref(h, weight, eps), h


def _accum_target(weight):
    """The weight's existing bf16 ``.grad`` (a view of the flat gradient arena) if dw can be
    accumulated into it inside the reduction kernel (fused AccumulateGrad), else None."""
    g = getattr(weight, "grad", None)
    if g is not None and g.dtype == torch.bfloat16 and g.is_contiguous() and g.is_cuda:
        return g
    return None


class _RMSNormFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, eps):
        C = load_ext(required=True)
        x2 = x.reshape(-1, x.shape[-1]).contiguous()
        y, rstd = C.rmsnorm_fwd(x2, weight, float(eps))
        count_launch("rmsnorm_fwd")
        ctx.save_for_backward(x2, weight, rstd)
        ctx.weight_ref = weight
        return y.view(x.shape)

    @staticmethod
    def backward(ctx, dy):
        C = load_ext(required=True)
        x2, weight, rstd = ctx.saved_tensors
        dy2 = dy.reshape(-1, dy.shape[-1]).contiguous()
        wg = _accum_target(ctx.weight_ref)
        dx, dw = C.rmsnorm_bwd(dy2, x2, weight, rstd, wg)
        count_launch("rmsnorm_bwd", 2)
        return dx.view(dy.shape), (None if wg is not None else dw.to(weight.dtype)), None


class _AddRMSNormFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, a, r, weight, eps):
        C = load_ext(required=True)
        shp = a.shape
        a2 = a.reshape(-1, shp[-1]).contiguous()
        r2 = r.reshape(-1, shp[-1]).contiguous()
        y, h, rstd = C.add_rmsnorm_fwd(a2, r2, weight, float(eps))
        count_launch("add_rmsnorm_fwd")
        ctx.save_for_backward(h, weight, rstd)
        ctx.weight_ref = weight
        return y.view(shp), h.view(shp)

    @staticmethod
    def backward(ctx, dy, dh_extra):
        C = load_ext(required=True)
        h, weight, rstd = ctx.saved_tensors
        shp = dy.shape
        dy2 = dy.reshape(-1, shp[-1]).contiguous()
        de2 = dh_extra.reshape(-1, shp[-1]).contiguous()
        wg = _accum_target(ctx.weight_ref)
        dh, dw = C.add_rmsnorm_bwd(dy2, de2, h, weight, rstd, wg)
        count_launch("add_rmsnorm_bwd", 2)
        dh = dh.view(shp)
        return dh, dh, (None if wg is not None else dw.to(weight.dtype)), None


def rmsnorm(x: torch.Tensor, weight: torch.Tensor, eps: float = 1e-5) -> torch.Tensor:
    if use_kernels(x, weight):
        return _RMSNormFn.apply(x, weight, eps)
    return rmsnorm_ref(x, weight, eps)


def add_rmsnorm(a: torch.Tensor, r: torch.Tensor, weight: torch.Tensor, eps: float = 1e-5):
    """Returns ``(rmsnorm(a + r) * weight, a + r)``."""
    if use_kernels(a, r, weight):
        return _AddRMSNormFn.apply(a, r, weight, eps)
    return add_rmsnorm_ref(a, r, weight, eps)
