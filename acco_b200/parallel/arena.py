"""Flat parameter / gradient arena and shard math.

What the reference does (`trainer_base.py:284-331`, `trainer_decoupled.py:244-315`):
one flat bf16 vector holds all parameters (every ``nn.Parameter.data`` is a view), one flat
vector holds all gradients, a third ``com_buffer`` of ``ceil(N/W)*W`` elements carries grads out /
weights in, and each rank owns an fp32 master copy of slice ``rank``.  Each round flip costs
three full-model memory passes (``params<-com``, ``com<-grad``, ``grad<-0``K15).

GPU-first redesign (no copies on the flip):

* ``theta[0], theta[1]`` - two full parameter buffers.  The model computes on ``theta[live]``
  while the communication round writes the *other* one; a flip re-points the parameter views.
* ``acc[0], acc[1]``   - two gradient accumulators.  Round ``r`` consumes ``acc[r % 2]`` **in place**
  (peers pull their slice straight out of it over NVLink) while backward accumulates into
  ``acc[(r + 1) % 2]``.  The consumer zeroes what it consumed.
* every buffer is padded to ``size_slice * W`` with ``size_slice`` a multiple of ``align``
  elements, so kernels never need a ragged tail (the pad region is an all-zero fixed point of
  AdamW).  ``align=1`` reproduces the reference's slice math exactly.

Buffers come from an ``allocator(numel, dtype) -> Tensor`` callback so the symmetric-memory
backend can hand out NVLink-mapped (P2P + NVLS multicast) storage; the default is plain
``torch.zeros``.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Callable, Dict, List, Optional, Tuple

import torch
import torch.nn as nn

__all__ = ["ShardLayout", "FlatArena", "unique_parameters"]


@dataclass(frozen=True)
class ShardLayout:
    """Slice math for a flat vector of ``numel`` elements over ``world`` owners.

    With ``align == 1`` this is the reference's rule (`trainer_decoupled.py:250-259`):
    ``size_slice = ceil(N / W)``; every rank owns a full slice except possibly the last one,
    whose ``size_local_slice`` is ``N % size_slice`` when that is non-zero.
    """

    numel: int
    world: int
    align: int = 1

    @property
    def size_slice(self) -> int:
        s = math.ceil(self.numel / self.world) if self.numel else 0
        a = max(self.align, 1)
        return ((s + a - 1) // a) * a

    @property
    def padded(self) -> int:
        return self.size_slice * self.world

    def bounds(self, rank: int) -> Tuple[int, int]:
        """Half-open range ``[lo, hi)`` of *real* (un-padded) elements owned by ``rank``."""
        lo = min(rank * self.size_slice, self.numel)
        hi = min((rank + 1) * self.size_slice, self.numel)
        return lo, hi

    def size_local_slice(self, rank: int) -> int:
        lo, hi = self.bounds(rank)
        return hi - lo

    def owner_of(self, index: int) -> int:
        return index // self.size_slice if self.size_slice else 0


def unique_parameters(model: nn.Module, trainable_only: bool = False) -> List[nn.Parameter]:
    """``model.parameters()`` order with tied weights listed once (what HF / torch give the
    reference: GPT-Neo-125M -> 160 tensors, 124 412 160 elements)."""
    seen, out = set(), []
    for p in model.parameters():
        if id(p) in seen:
            continue
        seen.add(id(p))
        if trainable_only and not p.requires_grad:
            continue
        out.append(p)
    return out


Allocator = Callable[[int, torch.dtype], torch.Tensor]


class FlatArena:
    """Owns ``theta[2]`` / ``acc[2]`` and the views that alias model parameters and grads."""

    def __init__(
        self,
        model: nn.Module,
        world: int,
        rank: int,
        dtype: torch.dtype,
        device: torch.device,
        align: int = 1,
        allocator: Optional[Allocator] = None,
        double_buffer: bool = True,
        grad_dtype: Optional[torch.dtype] = None,
    ):
        self.model = model
        self.world, self.rank = world, rank
        self.dtype, self.device = dtype, torch.device(device)
        self.grad_dtype = grad_dtype or dtype
        self.params: List[nn.Parameter] = unique_parameters(model)
        self.shapes = [tuple(p.shape) for p in self.params]
        self.numels = [p.numel() for p in self.params]
        self.offsets: List[int] = []
        off = 0
        for n in self.numels:
            self.offsets.append(off)
            off += n
        self.numel = off
        self.layout = ShardLayout(self.numel, world, align)
        alloc = allocator or (lambda n, dt: torch.zeros(n, dtype=dt, device=self.device))
        nbuf = 2 if double_buffer else 1
        self.theta: List[torch.Tensor] = [alloc(self.layout.padded, self.dtype) for _ in range(nbuf)]
        self.acc: List[torch.Tensor] = [alloc(self.layout.padded, self.grad_dtype) for _ in range(nbuf)]
        for t in self.theta + self.acc:
            assert t.numel() == self.layout.padded and t.is_contiguous()
        # gather current weights into theta[0]
        with torch.no_grad():
            for p, o, n in zip(self.params, self.offsets, self.numels):
                self.theta[0][o : o + n].copy_(p.detach().reshape(-1).to(device=self.device, dtype=self.dtype))
            if nbuf == 2:
                self.theta[1].copy_(self.theta[0])
        self._theta_views = [self._make_views(t) for t in self.theta]
        self._acc_views = [self._make_views(t) for t in self.acc]
        self.live = 0       # index of the theta buffer the model computes on
        self.grad_idx = 0   # index of the accumulator backward writes into
        self._bind_params(0)
        self._bind_grads(0)

    # ------------------------------------------------------------------ views
    def _make_views(self, flat: torch.Tensor) -> List[torch.Tensor]:
        return [flat[o : o + n].view(s) for o, n, s in zip(self.offsets, self.numels, self.shapes)]

    @torch.no_grad()
    def _bind_params(self, idx: int) -> None:
        for p, v in zip(self.params, self._theta_views[idx]):
            p.data = v
        self.live = idx

    @torch.no_grad()
    def _bind_grads(self, idx: int) -> None:
        for p, v in zip(self.params, self._acc_views[idx]):
            if p.requires_grad:
                p.grad = v
        self.grad_idx = idx

    def point_params(self, idx: int) -> None:
        """Make the model compute on ``theta[idx]`` (pointer flip; no data movement)."""
        if idx != self.live:
            self._bind_params(idx)

    def point_grads(self, idx: int) -> None:
        """Make backward accumulate into ``acc[idx]``."""
        if idx != self.grad_idx:
            self._bind_grads(idx)

    def rebind(self) -> None:
        """Re-assert aliasing (e.g. after something replaced ``p.grad`` with ``None``)."""
        self._bind_params(self.live)
        self._bind_grads(self.grad_idx)

    # ------------------------------------------------------------------ accessors
    @property
    def params_flat(self) -> torch.Tensor:
        """The live flat parameter vector (logical length, no padding) - ``self.params`` of the reference."""
        return self.theta[self.live][: self.numel]

    @property
    def grads_flat(self) -> torch.Tensor:
        return self.acc[self.grad_idx][: self.numel]

    def shard(self, flat: torch.Tensor, rank: Optional[int] = None) -> torch.Tensor:
        r = self.rank if rank is None else rank
        s = self.layout.size_slice
        return flat[r * s : (r + 1) * s]

    def param_slices(self) -> Dict[str, Tuple[int, int]]:
        """``name -> (offset, numel)`` of every (de-duplicated) parameter inside the flat vector."""
        by_id = {id(p): (o, n) for p, o, n in zip(self.params, self.offsets, self.numels)}
        out: Dict[str, Tuple[int, int]] = {}
        for name, p in self.model.named_parameters(remove_duplicate=False):
            if id(p) in by_id:
                out[name] = by_id[id(p)]
        return out

    def memory_bytes(self) -> int:
        return sum(t.numel() * t.element_size() for t in self.theta + self.acc)
