"""MLP activations.

* SwiGLU gate: ``out = silu(gate) * up`` on the fused ``[T, 2I]`` output of the gate|up GEMM
  (HF runs it as separate silu + mul over two GEMM outputs, `modeling_llama.py:171-184`).
* GELU-new (tanh approximation), the activation of the GPT-2 / GPT-Neo family (HF runs it as eager ATen ops,
  `modeling_gpt_neo.py`).

One sm_90a pass each way (``csrc/elementwise.cu``)."""
from __future__ import annotations

import torch
import torch.nn.functional as F

from . import count_launch, load_ext, use_kernels


def gelu_new_ref(x: torch.Tensor) -> torch.Tensor:
    return F.gelu(x.float(), approximate="tanh").to(x.dtype)


def swiglu_ref(gate_up: torch.Tensor) -> torch.Tensor:
    g, u = gate_up.float().chunk(2, dim=-1)
    return (F.silu(g) * u).to(gate_up.dtype)


class _SwiGLUFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, gate_up):
        C = load_ext(required=True)
        gu = gate_up.reshape(-1, gate_up.shape[-1]).contiguous()
        out = C.swiglu_fwd(gu)
        count_launch("swiglu_fwd")
        ctx.save_for_backward(gu)
        ctx.shape = gate_up.shape
        return out.view(*gate_up.shape[:-1], gate_up.shape[-1] // 2)

    @staticmethod
    def backward(ctx, dout):
        C = load_ext(required=True)
        (gu,) = ctx.saved_tensors
        d = dout.reshape(-1, dout.shape[-1]).contiguous()
        dgu = C.swiglu_bwd(d, gu)
        count_launch("swiglu_bwd")
        return dgu.view(ctx.shape)


def swiglu(gate_up: torch.Tensor) -> torch.Tensor:
    if use_kernels(gate_up):
        return _SwiGLUFn.apply(gate_up)
    return swiglu_ref(gate_up)


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


def gelu_new(x: torch.Tensor) -> torch.Tensor:
    if use_kernels(x) and x.numel() % 8 == 0:
        return _GeluFn.apply(x)
    return gelu_new_ref(x)
