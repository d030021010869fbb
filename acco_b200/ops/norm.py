"""RMSNorm and LayerNorm (weight + bias), each with an optional fused residual add (fp32 statistics, bf16 I/O).

HF Llama computes RMSNorm as ~7 eager kernels with an fp32 round trip
(`transformers/models/llama/modeling_llama.py:53-70`), and GPT-2 / GPT-Neo run LayerNorm as eager ATen ops
(`modeling_gpt_neo.py`).  Here each direction is one sm_90a pass (``csrc/norm.cu``, one kernel template for both norms):
the forward also emits ``rstd`` (and ``mean`` for LayerNorm) for the backward, the residual add of the surrounding block
is folded in (``h = a + r; y = norm(h)``), and dw / db are reduced deterministically and accumulated straight into the
gradient arena."""
from __future__ import annotations

from typing import Tuple

import torch
import torch.nn.functional as F

from . import accum_grad, count_launch, load_ext, main_grad_param, use_kernels

_KERNEL_MAX_H = 16384


def rmsnorm_ref(x: torch.Tensor, weight: torch.Tensor, eps: float) -> torch.Tensor:
    xf = x.float()
    rstd = torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + eps)
    return (xf * rstd * weight.float()).to(x.dtype)


def add_rmsnorm_ref(a: torch.Tensor, r: torch.Tensor, weight: torch.Tensor, eps: float) -> Tuple[torch.Tensor, torch.Tensor]:
    h = (a.float() + r.float()).to(a.dtype)
    return rmsnorm_ref(h, weight, eps), h


def layernorm_ref(x: torch.Tensor, weight: torch.Tensor, bias: torch.Tensor, eps: float) -> torch.Tensor:
    return F.layer_norm(x.float(), (x.shape[-1],), weight.float(), bias.float(), eps).to(x.dtype)


def add_layernorm_ref(a: torch.Tensor, r: torch.Tensor, weight: torch.Tensor, bias: torch.Tensor, eps: float) -> Tuple[torch.Tensor, torch.Tensor]:
    h = (a.float() + r.float()).to(a.dtype)
    return layernorm_ref(h, weight, bias, eps), h


def _kernel_covers(H: int) -> bool:
    return H % 8 == 0 and H <= _KERNEL_MAX_H


def _accum_target(weight):
    """The weight's gradient accumulator (a view of the flat gradient arena: its bf16 ``.grad``, or its fp32 ``main_grad``) if dw can
    be accumulated into it inside the reduction kernel (fused AccumulateGrad), else None."""
    g = None if weight is None else accum_grad(weight)
    if g is not None and g.dtype in (torch.bfloat16, torch.float32) and g.is_contiguous() and g.is_cuda:
        return g
    return None


class _NormFn(torch.autograd.Function):
    """``norm(a (+ r)) * weight (+ bias)``: RMSNorm when ``bias`` is None, LayerNorm otherwise.  With a residual ``r`` it
    returns ``(y, a + r)``, else ``y``."""

    @staticmethod
    def forward(ctx, a, r, weight, bias, eps):
        C = load_ext(required=True)
        shp = a.shape
        a2 = a.reshape(-1, shp[-1]).contiguous()
        r2 = None if r is None else r.reshape(-1, shp[-1]).contiguous()
        y, h, mean, rstd = C.norm_fwd(a2, r2, weight, bias, float(eps))
        count_launch(("add_" if r is not None else "") + ("layernorm_fwd" if bias is not None else "rmsnorm_fwd"))
        ctx.save_for_backward(a2 if h is None else h, weight, mean, rstd)
        ctx.weight_ref, ctx.bias_ref = weight, bias
        ctx.residual = r is not None
        if r is None:
            return y.view(shp)
        return y.view(shp), h.view(shp)

    @staticmethod
    def backward(ctx, dy, dh_extra=None):
        C = load_ext(required=True)
        h, weight, mean, rstd = ctx.saved_tensors
        layer = ctx.bias_ref is not None
        shp = dy.shape
        dy2 = dy.reshape(-1, shp[-1]).contiguous()
        de2 = None if dh_extra is None else dh_extra.reshape(-1, shp[-1]).contiguous()
        wg = _accum_target(ctx.weight_ref)
        bg = _accum_target(ctx.bias_ref)
        if layer and (wg is None or bg is None):     # LayerNorm accumulates both parameters or neither
            wg = bg = None
        if wg is not None and wg.dtype == torch.float32:
            dh, dwdb = C.norm_bwd_acc_f32(dy2, de2, h, weight, mean, rstd, wg, bg), None
        else:
            dh, dwdb = C.norm_bwd(dy2, de2, h, weight, mean, rstd, wg, bg)
        if layer:
            count_launch("layernorm_bwd", 3 if wg is not None else 2)
        else:
            count_launch("add_rmsnorm_bwd" if ctx.residual else "rmsnorm_bwd", 2)
        dh = dh.view(shp)
        dw = db = None
        if wg is None:
            H = shp[-1]
            dw = dwdb[:H].to(weight.dtype)
            if layer:
                db = dwdb[H:].to(weight.dtype)
        return dh, (dh if ctx.residual else None), dw, db, None


def rmsnorm(x: torch.Tensor, weight: torch.Tensor, eps: float = 1e-5) -> torch.Tensor:
    if use_kernels(x, weight) and _kernel_covers(x.shape[-1]):
        return _NormFn.apply(x, None, weight, None, eps)
    return rmsnorm_ref(x, main_grad_param(weight, dtype=torch.float32), eps)


def add_rmsnorm(a: torch.Tensor, r: torch.Tensor, weight: torch.Tensor, eps: float = 1e-5):
    """Returns ``(rmsnorm(a + r) * weight, a + r)``."""
    if use_kernels(a, r, weight) and _kernel_covers(a.shape[-1]):
        return _NormFn.apply(a, r, weight, None, eps)
    return add_rmsnorm_ref(a, r, main_grad_param(weight, dtype=torch.float32), eps)


def layernorm(x: torch.Tensor, weight: torch.Tensor, bias: torch.Tensor, eps: float = 1e-5) -> torch.Tensor:
    if use_kernels(x, weight, bias) and _kernel_covers(x.shape[-1]):
        return _NormFn.apply(x, None, weight, bias, eps)
    return layernorm_ref(x, main_grad_param(weight, dtype=torch.float32), main_grad_param(bias, dtype=torch.float32), eps)


def add_layernorm(a: torch.Tensor, r: torch.Tensor, weight: torch.Tensor, bias: torch.Tensor, eps: float = 1e-5):
    """Returns ``(layernorm(a + r), a + r)``."""
    if use_kernels(a, r, weight, bias) and _kernel_covers(a.shape[-1]):
        return _NormFn.apply(a, r, weight, bias, eps)
    return add_layernorm_ref(a, r, main_grad_param(weight, dtype=torch.float32), main_grad_param(bias, dtype=torch.float32), eps)
