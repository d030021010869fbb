"""FP8 training for the transformer-block linear layers (train key ``fp8``): e4m3 / e5m2 wgmma GEMMs with per-tensor current scaling.

Numerics of ``y = x W^T (+ b)`` with ``x [T, K]``, ``W [N, K]``, upstream gradient ``g [T, N]``, all bf16:

* ``amax(t) = max |t|``; ``s(t, f) = 2^floor(log2(max_f / amax))`` with ``max_e4m3 = 448``, ``max_e5m2 = 57344``; ``amax = 0`` gives
  ``s = 1``, a non-finite ``amax`` gives ``s = NaN`` (a NaN / Inf input makes a NaN loss, as in bf16).  ``s`` is capped at ``2^127`` (the
  largest fp32 power of two), which only matters for tensors whose largest value is a bf16 subnormal.
* ``q(t, f) = t * s`` rounded to nearest even in ``f``.  Scales are powers of two, so scaling is exact and nothing overflows: the
  quantiser is reproduced bit for bit by ``torch.float8_e4m3fn`` / ``torch.float8_e5m2`` casts.
* forward ``y = bf16(q(x,e4m3) q(W,e4m3)^T / (s_x s_W) + b)``; dgrad ``dx = bf16(q(g,e5m2) q(W,e4m3) / (s_g s_W))``; wgrad
  ``W.grad += q(g,e5m2)^T q(x,e4m3) / (s_g s_x)`` straight into the bf16 gradient (as ``gemm_tt_acc``), fp32 accumulation throughout.
* the forward's ``q(x)`` is reused by the wgrad and its ``q(W)`` by the dgrad; the backward keeps them (1 byte per element) instead of
  ``x``.

FP8 ``wgmma`` takes no transposed operand, so both GEMM operands are K-major: the quantiser writes ``q(x)`` as ``[T, K]`` (forward A)
and ``[K, T]`` (wgrad B), ``q(W)`` as ``[N, K]`` and ``[K, N]`` (dgrad B), ``q(g)`` as ``[T, N]`` (dgrad A) and ``[N, T]`` (wgrad A).

Each op has a ``*_ref`` twin (float8 casts and fp32 matmuls): the CPU path and the tests' oracle."""
from __future__ import annotations

from typing import Optional, Tuple

import torch

from . import count_launch, load_ext, use_kernels

E4M3, E5M2 = torch.float8_e4m3fn, torch.float8_e5m2
FP8_MAX = {E4M3: 448.0, E5M2: 57344.0}
_E_MAX = {E4M3: 8, E5M2: 15}            # max_f = 1.75 * 2^e_max


def scale_ref(amax: torch.Tensor, fmt) -> Tuple[torch.Tensor, torch.Tensor]:
    """``(s, 1/s)`` (fp32) of a tensor whose ``max |t|`` is ``amax``: the largest power of two with ``amax * s <= max_f``."""
    a = amax.double()
    mant, ex = torch.frexp(a)                                  # a = mant * 2^ex, mant in [0.5, 1)
    k = _E_MAX[fmt] - (ex.double() - 1) - (2 * mant > 1.75).double()
    k = k.clamp(max=127)
    s = torch.pow(2.0, k)
    s = torch.where(a == 0, torch.ones_like(s), s)
    s = torch.where(torch.isfinite(a), s, torch.full_like(s, float("nan")))
    return s.float(), (1.0 / s).float()


def quantize_ref(t: torch.Tensor, fmt, rowmajor: bool = True, transposed: bool = False):
    """``t [R, C]`` -> ``(q [R, C] or None, qT [C, R] or None, scale fp32 {s, 1/s, amax})``."""
    amax = t.detach().abs().max().float()
    s, inv = scale_ref(amax, fmt)
    q = (t.detach().float() * s).to(fmt)
    scale = torch.stack([s, inv, amax])
    return (q if rowmajor else None), (q.t().contiguous() if transposed else None), scale


def quantize(t: torch.Tensor, fmt, rowmajor: bool = True, transposed: bool = False):
    """The sm_90a quantiser (``fp8_amax_kernel`` + ``fp8_cast_kernel``) on CUDA, :func:`quantize_ref` elsewhere.  ``t``: bf16 ``[R, C]``
    with ``R, C`` multiples of 16.  ``scale[:3] = {s, 1/s, amax}`` stays on the device."""
    if not use_kernels(t):
        return quantize_ref(t, fmt, rowmajor, transposed)
    q, qT, scale = load_ext(required=True).fp8_quantize(t.contiguous(), fmt == E5M2, bool(rowmajor), bool(transposed))
    count_launch("fp8_amax")
    count_launch("fp8_cast")
    return (q if rowmajor else None), (qT if transposed else None), scale


def gemm_fp8_ref(a, b, scale_a, scale_b, out=None, bias=None, accumulate=False, dtype=torch.bfloat16):
    """``out[M,N] (+)= a[M,K] b[N,K]^T / (s_a s_b) (+ bias)`` in fp32, rounded once to ``dtype`` (``out``'s when given).  The scale
    product is formed in fp64, as the kernel's epilogue forms it exactly: ``1/s`` runs from ``2^-127`` to ``2^120``, so the product of
    two can leave fp32's range although the output is an ordinary number."""
    y = (a.float() @ b.float().t()).double() * (scale_a[1].double() * scale_b[1].double())
    if bias is not None:
        y = y + bias.double()
    y = y.float()
    if accumulate:
        y = y + out.float()
    if out is not None:
        out.copy_(y.to(out.dtype))
        return out
    return y.to(dtype)


def gemm_fp8(a, b, scale_a, scale_b, out=None, bias=None, accumulate=False, bn: int = 0, splits: int = 0, max_ctas: int = 0):
    """FP8 wgmma GEMM (``csrc/gemm_wgmma.cu``, ``gemm_fp8_kernel``): ``a`` e4m3 or e5m2, ``b`` e4m3, both K-major one-byte ``[rows, K]``;
    bf16 out; ``accumulate`` adds into ``out`` (split-K allowed).  ``bn`` / ``splits``: 0 = heuristic; ``max_ctas`` > 0 caps the
    persistent grid (as in :func:`ops.gemm.gemm`)."""
    if not use_kernels(a, b, bf16_only=False):
        return gemm_fp8_ref(a, b, scale_a, scale_b, out, bias, accumulate)
    if out is not None and out.dtype == torch.float32 and accumulate and bias is None:
        # an fp32 gradient accumulator: the fp32-output instantiation adds the tile's fp32 sum without rounding to bf16
        load_ext(required=True).gemm_fp8_acc_f32(a, b, scale_a, scale_b, out, int(bn), int(splits), int(max_ctas))
        count_launch("gemm_fp8_f32acc")
        return out
    y = load_ext(required=True).gemm_fp8(a, b, scale_a, scale_b, out, bias, bool(accumulate), int(bn), int(splits), int(max_ctas))
    count_launch("gemm_fp8")
    return y


def fp8_supported(x: torch.Tensor, weight: torch.Tensor, bias: Optional[torch.Tensor]) -> bool:
    """Calls the FP8 path takes: bf16 operands (and bias) with ``T``, ``K``, ``N`` multiples of 16 (16-byte FP8 tensor-map strides; the
    transposed copies have rows of ``T`` elements).  Others stay on the bf16 path."""
    if x.dtype != torch.bfloat16 or weight.dtype != torch.bfloat16 or weight.dim() != 2 or x.device != weight.device:
        return False
    if bias is not None and (bias.dtype != torch.bfloat16 or (bias.is_cuda and bias.data_ptr() % 16)):
        return False
    N, K = weight.shape
    return x.shape[-1] == K and x.numel() > 0 and (x.numel() // K) % 16 == 0 and K % 16 == 0 and N % 16 == 0


class Fp8LinearFn(torch.autograd.Function):
    """``y = x W^T (+ b)`` with FP8 GEMMs (module docstring).  Saves ``q(x)^T``, ``q(W)^T`` and their scales for the backward."""

    @staticmethod
    def forward(ctx, x, weight, bias, accumulate_into_grad):
        K = x.shape[-1]
        x2 = x.reshape(-1, K)
        need_dx, need_dw = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
        qx, qxT, sx = quantize(x2, E4M3, True, need_dw)
        qw, qwT, sw = quantize(weight.detach(), E4M3, True, need_dx)
        y = gemm_fp8(qx, qw, sx, sw, bias=None if bias is None else bias.detach())
        ctx.save_for_backward(qxT, qwT, sx, sw)
        ctx.x_shape = x.shape
        ctx.has_bias = bias is not None
        ctx.accumulate = bool(accumulate_into_grad)
        ctx.weight_ref = weight
        ctx.bias_ref = bias
        return y.view(*x.shape[:-1], weight.shape[0])

    @staticmethod
    def backward(ctx, dy):
        from .linear import _bias_grad
        qxT, qwT, sx, sw = ctx.saved_tensors
        g = dy.reshape(-1, dy.shape[-1]).contiguous()
        need_dx, need_dw = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
        dx = dw = None
        if need_dx or need_dw:
            qg, qgT, sg = quantize(g, E5M2, need_dx, need_dw)
            if need_dx:
                dx = gemm_fp8(qg, qwT, sg, sw).view(ctx.x_shape)
            if need_dw:
                w = ctx.weight_ref
                main = getattr(w, "main_grad", None)
                if ctx.accumulate and main is not None:
                    if _arena_view(main, torch.float32):
                        gemm_fp8(qgT, qxT, sg, sx, out=main, accumulate=True)  # fp32 accumulator: fp32 sum added, no bf16 rounding
                    else:
                        main.add_(gemm_fp8_ref(qgT, qxT, sg, sx, dtype=torch.float32))
                elif ctx.accumulate and w.grad is not None and _arena_view(w.grad):
                    gemm_fp8(qgT, qxT, sg, sx, out=w.grad, accumulate=True)     # adds straight into the gradient
                elif ctx.accumulate and w.grad is not None:
                    w.grad.add_(gemm_fp8(qgT, qxT, sg, sx).to(w.grad.dtype))
                else:
                    dw = gemm_fp8(qgT, qxT, sg, sx).to(w.dtype)
        return dx, dw, _bias_grad(ctx, g), None


def _arena_view(grad: torch.Tensor, dtype: torch.dtype = torch.bfloat16) -> bool:
    """A gradient the FP8 GEMM can add into in place: ``dtype`` (bf16, or fp32 for an fp32 accumulator), 2-D, unit inner stride,
    16-byte aligned (CPU tensors: any such matrix)."""
    if grad.dtype != dtype or grad.dim() != 2 or grad.stride(1) != 1:
        return False
    return not grad.is_cuda or (grad.data_ptr() % 16 == 0 and grad.stride(0) % 8 == 0)
