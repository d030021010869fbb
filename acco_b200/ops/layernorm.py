"""LayerNorm (weight + bias) and fused residual-add + LayerNorm, and GELU-new: the normalisation / activation of the
GPT-2 / GPT-Neo family - the reference's default pre-training model (`/root/reference/main.py:39-41`,
``config/model/gpt-neo-125M.json``; HF runs them as eager ATen ops, `modeling_gpt_neo.py`).  One sm_90a pass each
(``csrc/layernorm.cu``); dw / db are reduced deterministically and accumulated straight into the gradient arena."""
from __future__ import annotations

from typing import Tuple

import torch
import torch.nn.functional as F

from . import count_launch, load_ext, use_kernels
from .norm import _accum_target


def layernorm_ref(x: torch.Tensor, weight: torch.Tensor, bias: torch.Tensor, eps: float) -> torch.Tensor:
    return F.layer_norm(x.float(), (x.shape[-1],), weight.float(), bias.float(), eps).to(x.dtype)


def add_layernorm_ref(a: torch.Tensor, r: torch.Tensor, weight: torch.Tensor, bias: torch.Tensor, eps: float) -> Tuple[torch.Tensor, torch.Tensor]:
    h = (a.float() + r.float()).to(a.dtype)
    return layernorm_ref(h, weight, bias, eps), h


def gelu_new_ref(x: torch.Tensor) -> torch.Tensor:
    return F.gelu(x.float(), approximate="tanh").to(x.dtype)


def _bwd(ctx, dy, dh_extra):
    C = load_ext(required=True)
    h, weight, mean, rstd = ctx.saved_tensors
    shp = dy.shape
    dy2 = dy.reshape(-1, shp[-1]).contiguous()
    de2 = None if dh_extra is None else dh_extra.reshape(-1, shp[-1]).contiguous()
    wg, bg = _accum_target(ctx.weight_ref), _accum_target(ctx.bias_ref)
    if wg is None or bg is None:
        wg = bg = None
    dh, dwdb = C.layernorm_bwd(dy2, de2, h, weight, mean, rstd, wg, bg)
    count_launch("layernorm_bwd", 3 if wg is not None else 2)
    H = shp[-1]
    if wg is not None:
        return dh.view(shp), None, None
    return dh.view(shp), dwdb[:H].to(weight.dtype), dwdb[H:].to(weight.dtype)


class _LayerNormFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, bias, eps):
        C = load_ext(required=True)
        x2 = x.reshape(-1, x.shape[-1]).contiguous()
        y, mean, rstd = C.layernorm_fwd(x2, None, weight, bias, float(eps))
        count_launch("layernorm_fwd")
        ctx.save_for_backward(x2, weight, mean, rstd)
        ctx.weight_ref, ctx.bias_ref = weight, bias
        return y.view(x.shape)

    @staticmethod
    def backward(ctx, dy):
        dx, dw, db = _bwd(ctx, dy, None)
        return dx, dw, db, None


class _AddLayerNormFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, a, r, weight, bias, eps):
        C = load_ext(required=True)
        shp = a.shape
        a2 = a.reshape(-1, shp[-1]).contiguous()
        r2 = r.reshape(-1, shp[-1]).contiguous()
        y, h, mean, rstd = C.layernorm_fwd(a2, r2, weight, bias, float(eps))
        count_launch("add_layernorm_fwd")
        ctx.save_for_backward(h, weight, mean, rstd)
        ctx.weight_ref, ctx.bias_ref = weight, bias
        return y.view(shp), h.view(shp)

    @staticmethod
    def backward(ctx, dy, dh_extra):
        dh, dw, db = _bwd(ctx, dy, dh_extra)
        return dh, dh, dw, db, None


class _GeluFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        C = load_ext(required=True)
        xc = x.contiguous()
        ctx.save_for_backward(xc)
        count_launch("gelu_fwd")
        return C.gelu_fwd(xc)

    @staticmethod
    def backward(ctx, dy):
        C = load_ext(required=True)
        (x,) = ctx.saved_tensors
        count_launch("gelu_bwd")
        return C.gelu_bwd(dy.contiguous(), x)


def layernorm(x: torch.Tensor, weight: torch.Tensor, bias: torch.Tensor, eps: float = 1e-5) -> torch.Tensor:
    if use_kernels(x, weight, bias) and x.shape[-1] % 8 == 0 and x.shape[-1] <= 8192:
        return _LayerNormFn.apply(x, weight, bias, eps)
    return layernorm_ref(x, weight, bias, eps)


def add_layernorm(a: torch.Tensor, r: torch.Tensor, weight: torch.Tensor, bias: torch.Tensor, eps: float = 1e-5):
    """Returns ``(layernorm(a + r), a + r)``."""
    if use_kernels(a, r, weight, bias) and a.shape[-1] % 8 == 0 and a.shape[-1] <= 8192:
        return _AddLayerNormFn.apply(a, r, weight, bias, eps)
    return add_layernorm_ref(a, r, weight, bias, eps)


def gelu_new(x: torch.Tensor) -> torch.Tensor:
    if use_kernels(x) and x.numel() % 8 == 0:
        return _GeluFn.apply(x)
    return gelu_new_ref(x)
