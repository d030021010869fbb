"""Symmetric-memory backend: the fused RS + AdamW + AG round kernel over NVLink / NVSwitch.

Plumbing only on the host: buffers are allocated with ``torch.distributed._symmetric_memory``
(CUDA VMM + peer mapping + NVLS multicast binding), which hands back, per buffer, the list of
peer-mapped device pointers and - when the fabric supports it - one *multicast* pointer.  Those raw
pointers go straight into ``csrc/rs_adam_ag.cu``; no NCCL call is made per round
(`trainer_decoupled.py:86-112` issues three: all_reduce(count), reduce_scatter_tensor,
all_gather_into_tensor).

Transport modes (``ACCO_SYMM_MODE=auto|multimem|p2p``): ``multimem`` uses switch-side reduction
and broadcast (``multimem.ld_reduce`` / ``multimem.st``); ``p2p`` uses plain peer loads/stores.
``world == 1`` runs the same kernel on local memory.
"""
from __future__ import annotations

import os
from typing import Callable, Dict, Optional

import torch
import torch.distributed as dist

from ..optim import ShardedAdamW
from .arena import FlatArena
from .backend import CommBackend
from .schedule import RoundPlan

__all__ = ["SymmBackend", "merge_ranges"]


def merge_ranges(ranges):
    """Sort half-open ``(lo, hi)`` ranges and merge the ones that touch or overlap -> list of ``[lo, hi]``."""
    rs = sorted((int(a), int(b)) for a, b in ranges if b > a)
    merged = []
    for a, b in rs:
        if merged and a <= merged[-1][1]:
            merged[-1][1] = max(merged[-1][1], b)
        else:
            merged.append([a, b])
    return merged

_CTRL_WORDS = 1024     # uint32 words in the private signal pad (3*W used, 5*W with max_grad_norm)


class SymmBackend(CommBackend):
    name = "symm"

    def __init__(self, rank: int, world: int, device: torch.device, grid: int = 0):
        super().__init__(rank, world, device)
        from .. import ops
        self.C = ops.load_ext(required=True)
        self._ops = ops
        self.grid = int(os.environ.get("ACCO_ROUND_GRID", grid))
        self._handles: Dict[int, object] = {}
        self._skip = None          # int64 [n, 2] element ranges the round kernel does not push (pulled by KERNEL B)
        self.mode = 0
        self._symm = None
        if world > 1:
            import torch.distributed._symmetric_memory as symm_mem
            self._symm = symm_mem
            self.group = dist.group.WORLD
            self.ctrl = self._alloc_symm(_CTRL_WORDS, torch.int32)
            self.ctrl_handle = self._handles[self.ctrl.data_ptr()]
            want = os.environ.get("ACCO_SYMM_MODE", "auto").lower()
            has_mc = int(getattr(self.ctrl_handle, "multicast_ptr", 0) or 0) != 0
            if want == "multimem" and not has_mc:
                raise RuntimeError("ACCO_SYMM_MODE=multimem but this fabric exposes no multicast pointer")
            self.mode = 2 if (has_mc and want in ("auto", "multimem")) else 1
            self.name = "symm-multimem" if self.mode == 2 else "symm-p2p"
            dist.barrier()
        else:
            self.name = "symm-local"

    # ------------------------------------------------------------------ allocation
    def _alloc_symm(self, numel: int, dtype: torch.dtype) -> torch.Tensor:
        t = self._symm.empty(int(numel), dtype=dtype, device=self.device)
        hdl = self._symm.rendezvous(t, self.group)
        t.zero_()
        self._handles[t.data_ptr()] = hdl
        return t

    def allocator(self) -> Optional[Callable[[int, torch.dtype], torch.Tensor]]:
        if self.world == 1:
            return None
        return self._alloc_symm

    def slice_alignment(self) -> int:
        return 1024

    def attach(self, arena: FlatArena, opt: ShardedAdamW, max_grad_norm: Optional[float] = None) -> None:
        super().attach(arena, opt, max_grad_norm)
        self.scratch = torch.zeros(4, dtype=torch.int32, device=self.device)   # stash_count, total, epoch, done
        self.total_host = torch.zeros(1, dtype=torch.int32).pin_memory()
        if max_grad_norm is not None:
            # round_norm output: norm, inv_eff, sum of squares, one partial per CTA of its grid
            grid = self.grid if self.grid > 0 else 4 * int(self.C.num_sms())
            self.norm_out = torch.zeros(3 + grid, dtype=torch.float32, device=self.device)
            self.norm_host = torch.zeros(1, dtype=torch.float32).pin_memory()
        self._grad_bf16 = arena.grad_dtype == torch.bfloat16
        self._out_bf16 = arena.dtype == torch.bfloat16
        if self.world > 1:
            self._pads = [int(p) for p in self.ctrl_handle.buffer_ptrs]
            self._ptrs = {}
            for name, bufs in (("acc", arena.acc), ("theta", arena.theta)):
                for i, t in enumerate(bufs):
                    h = self._handles[t.data_ptr()]
                    self._ptrs[(name, i)] = ([int(p) for p in h.buffer_ptrs], int(getattr(h, "multicast_ptr", 0) or 0))
            if self.mode == 2 and any(mc == 0 for _, mc in self._ptrs.values()):
                self.mode, self.name = 1, "symm-p2p"
            torch.cuda.synchronize(self.device)
            dist.barrier()

    # ------------------------------------------------------------------ rounds
    @torch.no_grad()
    def launch_round(self, plan: RoundPlan, lr: float, local_count: int) -> None:
        arena, opt = self.arena, self.opt
        acc = arena.acc[plan.read_acc]
        theta = arena.theta[plan.write_theta]
        if self.world > 1:
            acc_ptrs, acc_mc = self._ptrs[("acc", plan.read_acc)]
            th_ptrs, th_mc = self._ptrs[("theta", plan.write_theta)]
            pads = self._pads
        else:
            acc_ptrs, acc_mc, th_ptrs, th_mc, pads = [acc.data_ptr()], 0, [theta.data_ptr()], 0, []
        inv_eff = None
        if self.max_grad_norm is not None:
            # gate (W > 1, gated) + start barrier, then the global norm; the update below reads inv_eff = 1/count * clip coefficient
            self.C.round_norm(acc_ptrs, pads, acc_mc, opt.stash, self.scratch, self.norm_out, arena.layout.size_slice, self.rank,
                              self.world, int(local_count), bool(plan.add_stash), self._grad_bf16, self.mode, self.grid,
                              self.max_grad_norm)
            self._ops.count_launch("round_norm")
            inv_eff = self.norm_out
        self.C.rs_adam_ag(acc_ptrs, th_ptrs, pads, acc_mc, th_mc, opt.master, opt.exp_avg, opt.exp_avg_sq, opt.stash,
                          self.scratch, arena.layout.size_slice, self.rank, self.world, int(local_count),
                          float(lr), opt.beta1, opt.beta2, opt.eps, opt.weight_decay, opt.step + 1, int(plan.commit),
                          bool(plan.add_stash), bool(plan.write_stash), self._grad_bf16, self._out_bf16, self.mode, self.grid,
                          self._skip, inv_eff, opt.no_decay_dev)
        self._ops.count_launch("rs_adam_ag")
        if self.world > 1 and os.environ.get("ACCO_ROUND_GATE", "1") != "0":
            self._ops.count_launch("round_gate")
        opt.after_launch(plan)
        acc.zero_()
        self.total_host.copy_(self.scratch[1:2], non_blocking=True)
        if inv_eff is not None:
            self.norm_host.copy_(self.norm_out[0:1], non_blocking=True)

    def finish_round(self, plan: RoundPlan) -> int:
        if self.max_grad_norm is not None:
            self.last_grad_norm = float(self.norm_host.item())
        return int(self.total_host.item())

    # ------------------------------------------------------------------ fused all-gather + GEMM support (KERNEL B)
    def peer_bases(self, which: str, idx: int):
        """Peer-mapped base addresses of ``arena.theta[idx]`` / ``arena.acc[idx]`` on every rank."""
        return list(self._ptrs[(which, idx)][0])

    def set_pull_ranges(self, ranges) -> None:
        """``ranges``: iterable of ``(lo, hi)`` element ranges of the flat buffer that peers will pull inside their
        first forward GEMM; the round kernel then updates only the owner's copy of them."""
        merged = merge_ranges(ranges)
        assert all(a % 8 == 0 and b % 8 == 0 for a, b in merged), "pull ranges must be 8-element aligned"
        self._skip = torch.tensor(merged, dtype=torch.int64, device=self.device).contiguous() if merged else None

    def kernel_launches_per_round(self) -> int:
        return 1 if self.max_grad_norm is None else 2
