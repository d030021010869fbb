"""Hand-written wgmma / TMA GEMM (``csrc/gemm_wgmma.cu``) - every contraction of the training step
(`trainer_decoupled.py:18-39`: the ``nn.Linear`` forward / dgrad / wgrad inside ``gradient_step``) - optionally fused
with the all-gather of its weight operand (KERNEL B of the north star).

``gemm(a, b, ...)``            : ``out[M,N] (+)= A @ B^T (+ bias)`` with either operand K-major (``[rows, K]``) or
                                 MN-major (``[K, rows]``, i.e. a transposed view without a copy), ``accumulate=True``
                                 = adding epilogue into ``out`` (beta = 1; split-K for small outputs).
``gemm_tn / gemm_nn / gemm_tt_acc`` : the forward / dgrad / wgrad specialisations used by ``ops.linear``.
``GatheredWeight`` + ``gemm_tn_gather(x, gw)`` : the forward GEMM where the row-blocks of ``w`` that live on
other ranks (they own those slices of the flat arena and have just updated them) are pulled over NVLink
inside the kernel, consumed by the tensor core and written through to the local copy - so the first
forward GEMM after a round *is* the all-gather of that weight."""
from __future__ import annotations

from typing import List

import torch

from . import count_launch, load_ext, use_kernels

TILE_N, TILE_K = 256, 64


def gemm_tn_ref(x: torch.Tensor, w: torch.Tensor) -> torch.Tensor:
    return (x.float() @ w.float().t()).to(x.dtype)


def _rowmajor(t: torch.Tensor) -> torch.Tensor:
    """2-D, unit inner stride, 16-byte aligned rows (what a TMA tensor map can describe); copies otherwise."""
    if t.dim() == 2 and t.stride(1) == 1 and t.stride(0) % 8 == 0 and t.stride(0) >= t.shape[1] and t.data_ptr() % 16 == 0:
        return t
    return t.contiguous()


def gemm_supported(*mats: torch.Tensor) -> bool:
    """Shapes the wgmma kernel takes: bf16 CUDA matrices whose row length is a multiple of 8 (16-byte TMA strides)."""
    return all(m.is_cuda and m.dtype == torch.bfloat16 and m.dim() == 2 and m.shape[1] % 8 == 0 and m.shape[0] > 0 for m in mats)


def gemm_ref(a, b, out=None, bias=None, a_mn=False, b_mn=False, accumulate=False):
    af = (a.t() if a_mn else a).float()
    bf = (b.t() if b_mn else b).float()
    y = af @ bf.t()
    if bias is not None:
        y = y + bias.float()
    if accumulate:
        y = y + out.float()
    y = y.to(a.dtype)
    if out is not None:
        out.copy_(y)
        return out
    return y


def gemm(a: torch.Tensor, b: torch.Tensor, out: torch.Tensor = None, bias: torch.Tensor = None, a_mn: bool = False, b_mn: bool = False,
         accumulate: bool = False, bn: int = 0, splits: int = 0, pm: int = 0, pn: int = 0, msub: int = 0, max_ctas: int = 0) -> torch.Tensor:
    """``out[M,N] (+)= A @ B^T (+ bias)``; ``a``: ``[M,K]`` or (``a_mn``) ``[K,M]``; ``b``: ``[N,K]`` or (``b_mn``) ``[K,N]``.
    ``bn`` / ``splits`` / ``pm, pn`` / ``msub`` override the tile-N / split-K / pair-cluster (TMA multicast) / rows-per-CTA (128 *
    msub) heuristic (0 = automatic)."""
    if not use_kernels(a, b):
        return gemm_ref(a, b, out, bias, a_mn, b_mn, accumulate)
    y = load_ext(required=True).gemm(_rowmajor(a), _rowmajor(b), out, bias, bool(a_mn), bool(b_mn), bool(accumulate), int(bn), int(splits),
                                     int(pm), int(pn), int(msub), int(max_ctas))
    count_launch("gemm")
    return y


def gemm_tn(x: torch.Tensor, w: torch.Tensor, max_ctas: int = 0, bias: torch.Tensor = None) -> torch.Tensor:
    """forward: ``x [M,K] @ w [N,K]^T (+ bias)``"""
    return gemm(x, w, bias=bias, max_ctas=max_ctas)


def gemm_nn(dy: torch.Tensor, w: torch.Tensor) -> torch.Tensor:
    """dgrad: ``dy [M,N] @ w [N,K]`` - the weight is consumed as an MN-major B operand (no transpose copy)"""
    return gemm(dy, w, b_mn=True)


def gemm_tt_acc(dy: torch.Tensor, x: torch.Tensor, grad: torch.Tensor) -> torch.Tensor:
    """wgrad: ``grad [N,K] += dy [M,N]^T @ x [M,K]`` - both operands MN-major, reduce-add epilogue into the arena view"""
    return gemm(dy, x, out=grad, a_mn=True, b_mn=True, accumulate=True)


class GatheredWeight:
    """Book-keeping for one weight matrix ``[N, K]`` inside the symmetric flat parameter buffer.

    ``offset``       : element offset of the matrix in the flat buffer
    ``peer_bases``   : base address of the *flat buffer* on every rank (peer mapped)
    ``size_slice``   : elements per rank in the flat buffer
    A 256-row tile is gathered from rank ``r`` iff all of it lies inside rank ``r``'s slice and ``r`` is not
    this rank; tiles that straddle an ownership boundary (at most one per boundary) are pushed by the round
    kernel as usual (``tile_owner == -1``)."""

    def __init__(self, n: int, k: int, offset: int, peer_bases: List[int], size_slice: int, rank: int, device):
        self.n, self.k, self.offset, self.rank = int(n), int(k), int(offset), int(rank)
        self.peer_ptrs = [int(b) + 2 * self.offset for b in peer_bases]
        num_n = (self.n + TILE_N - 1) // TILE_N
        num_k = (self.k + TILE_K - 1) // TILE_K
        owners = []
        for t in range(num_n):
            lo = self.offset + t * TILE_N * self.k
            hi = self.offset + min((t + 1) * TILE_N, self.n) * self.k - 1
            o_lo, o_hi = lo // size_slice, hi // size_slice
            owners.append(o_lo if (o_lo == o_hi and o_lo != rank) else -1)
        self.owners = owners
        self.tile_owner = torch.tensor(owners, dtype=torch.int32, device=device)
        self.flags = torch.zeros(num_n * num_k * 2, dtype=torch.int32, device=device)   # one per (n_blk, k_blk, half of the B tile)
        self.state = torch.zeros(2, dtype=torch.int32, device=device)

    def pulled_ranges(self, for_rank: int, size_slice: int):
        """Element ranges ``[lo, hi)`` of the flat buffer that rank ``for_rank`` need NOT push because every
        peer pulls them inside the GEMM (whole tiles inside its slice)."""
        out = []
        for t in range((self.n + TILE_N - 1) // TILE_N):
            lo = self.offset + t * TILE_N * self.k
            hi = self.offset + min((t + 1) * TILE_N, self.n) * self.k
            if lo // size_slice == (hi - 1) // size_slice == for_rank:
                out.append((lo, hi))
        return out


def gemm_tn_gather(x: torch.Tensor, w_local: torch.Tensor, gw: GatheredWeight, max_ctas: int = 0) -> torch.Tensor:
    out = load_ext(required=True).gemm_tn(x.contiguous(), w_local, gw.peer_ptrs, gw.tile_owner, gw.flags, gw.state, int(max_ctas))
    count_launch("gemm_gather")
    return out
