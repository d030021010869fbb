"""Token embedding whose backward scatter-adds straight into the (arena-resident) ``weight.grad``
instead of materialising a dense ``[V, H]`` gradient and adding it afterwards.

The backward's contract, on both branches (into an existing ``.grad``, or into a fresh zero ``dw``): for every row ``r``,
``grad[r] = bf16_rn(grad[r] + sum_{i: ids[i] = r} dy[i])`` with the sum in fp32, in a fixed order; rows no id hits are not
touched.  A bf16 ``index_add_`` (or ``index_put_(accumulate=True)``) would instead round the row once per occurrence, so the rows of
frequent tokens - EOS, padding, a tied head's rows already holding the LM-head wgrad - drift from the fp32 sum as their count grows.
On CUDA the ids are stably sorted and ``embedding_bwd_kernel`` (``csrc/elementwise.cu``) sums each run of equal ids; there is no
host sync and no data-dependent size, so the step stays capturable in a CUDA graph."""
from __future__ import annotations

import torch
import torch.nn.functional as F

from . import count_launch, load_ext, use_kernels


def embedding_bwd_ref(grad: torch.Tensor, ids: torch.Tensor, dy: torch.Tensor) -> None:
    """``grad[r] += sum_{i: ids[i] = r} dy[i]`` in place, the sum in fp32 and one rounding to ``grad``'s dtype per row hit.  Every size
    is fixed by ``T``, with no host sync, so the eager path is capturable too: the runs of the sorted ids are summed into ``T`` fp32
    rows, and the rows past the last run repeat the first run's write (same row, same value)."""
    T = ids.numel()
    if T == 0:
        return
    sorted_ids, perm = torch.sort(ids.reshape(-1), stable=True)
    start = torch.ones(T, dtype=torch.bool, device=ids.device)
    start[1:] = sorted_ids[1:] != sorted_ids[:-1]
    run = torch.cumsum(start, 0) - 1
    acc = torch.zeros(T, dy.shape[-1], dtype=torch.float32, device=dy.device).index_add_(0, run, dy[perm].float())
    row = torch.zeros(T, dtype=sorted_ids.dtype, device=ids.device).index_put_((run,), sorted_ids)
    valid = (torch.arange(T, device=ids.device) <= run[-1]).unsqueeze(1)
    row = torch.where(valid.squeeze(1), row, row[0])
    acc = torch.where(valid, acc, acc[0])
    grad.index_put_((row,), (grad[row].float() + acc).to(grad.dtype))


def embedding_bwd_f32(grad: torch.Tensor, ids: torch.Tensor, dy: torch.Tensor) -> None:
    """Add the bf16 rows of ``dy [T, H]`` into an fp32 ``grad [R, H]`` (an fp32 gradient accumulator) at ``ids [T]``: per row hit,
    ``grad[r] += sum_{i: ids[i] = r} dy[i]`` with the sum in fp32, in the order of the module docstring's kernel, and no rounding to
    bf16.  CUDA: the fp32-row instantiation of ``embedding_bwd_kernel``, as capturable as the bf16 one."""
    if use_kernels(grad, dy, bf16_only=False) and dy.dtype == torch.bfloat16:
        sorted_ids, perm = torch.sort(ids.long(), stable=True)
        load_ext(required=True).embedding_bwd_f32(grad, sorted_ids, perm, dy.contiguous())
        count_launch("embedding_bwd_f32")
        return
    grad.index_add_(0, ids, dy.float())


def embedding_bwd(grad: torch.Tensor, ids: torch.Tensor, dy: torch.Tensor) -> None:
    """Add the rows of ``dy [T, H]`` into ``grad [R, H]`` at ``ids [T]`` (see the module docstring)."""
    if use_kernels(grad):
        sorted_ids, perm = torch.sort(ids.long(), stable=True)
        load_ext(required=True).embedding_bwd(grad, sorted_ids, perm, dy.to(grad.dtype).contiguous())
        count_launch("embedding_bwd")
        return
    if grad.dtype in (torch.float32, torch.float64):
        grad.index_add_(0, ids, dy.to(grad.dtype))      # fp32 / fp64 rows: the adds are the sum in the row's own precision
        return
    embedding_bwd_ref(grad, ids, dy.to(grad.dtype))


class EmbeddingFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, ids, weight, accumulate_into_grad):
        ctx.save_for_backward(ids)
        ctx.weight_ref = weight
        ctx.accumulate = bool(accumulate_into_grad)
        return F.embedding(ids, weight)

    @staticmethod
    def backward(ctx, dy):
        (ids,) = ctx.saved_tensors
        w = ctx.weight_ref
        flat_ids = ids.reshape(-1)
        dy2 = dy.reshape(-1, dy.shape[-1])
        if ctx.accumulate and getattr(w, "main_grad", None) is not None:
            embedding_bwd_f32(w.main_grad, flat_ids, dy2)
            return None, None, None
        if ctx.accumulate and w.grad is not None:
            embedding_bwd(w.grad, flat_ids, dy2)
            return None, None, None
        dw = torch.zeros_like(w)
        embedding_bwd(dw, flat_ids, dy2)
        return None, dw, None


def embedding(ids: torch.Tensor, weight: torch.Tensor, accumulate_into_grad: bool = True) -> torch.Tensor:
    if torch.is_grad_enabled() and weight.requires_grad:
        return EmbeddingFn.apply(ids, weight, accumulate_into_grad)
    return F.embedding(ids, weight)
