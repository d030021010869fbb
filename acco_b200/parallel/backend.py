"""Communication backends: one interface, three implementations.

==========  ===========================================================================
``symm``    the product: ONE sm_90a kernel per round doing reduce-scatter (NVLS
            ``multimem.ld_reduce`` / P2P loads straight out of the peers' gradient
            accumulators) + count exchange + scale + sharded AdamW (+ stash, commit flags) +
            all-gather push (``multimem.st`` / P2P stores into every peer's shadow parameter
            buffer).  No NCCL call on the path.  See ``parallel/symm.py`` and
            ``csrc/rs_adam_ag.cu``.
``nccl``    the library baseline: ``all_reduce(count)``, ``reduce_scatter_tensor``, one fused
            local AdamW kernel (or PyTorch ops), ``all_gather_into_tensor`` - the same call
            sequence as the reference's ``communication_step`` (`trainer_decoupled.py:67-126`),
            minus the clone/restore passes.
``gloo``    same code as ``nccl`` on CPU tensors (plumbing tests).
==========  ===========================================================================

A backend enqueues a whole *round* on the current stream (:meth:`launch_round`) and later
reports the global micro-gradient count of the update it applied (:meth:`finish_round`, valid
once the round's completion event has fired) - the host never blocks on the device in between.
"""
from __future__ import annotations

from typing import Callable, Optional

import torch
import torch.distributed as dist

from ..optim import ShardedAdamW, adamw_shard_update_
from .arena import FlatArena
from .schedule import RoundPlan

__all__ = ["CommBackend", "TorchDistBackend", "make_backend"]


class CommBackend:
    name = "base"

    def __init__(self, rank: int, world: int, device: torch.device):
        self.rank, self.world, self.device = rank, world, torch.device(device)
        self.arena: Optional[FlatArena] = None
        self.opt: Optional[ShardedAdamW] = None

    # buffers ---------------------------------------------------------------------------
    def allocator(self) -> Optional[Callable[[int, torch.dtype], torch.Tensor]]:
        """Allocator for arena buffers (``None`` -> ordinary device memory)."""
        return None

    def slice_alignment(self) -> int:
        """Required alignment (elements) of ``size_slice``; 1 reproduces the reference math."""
        return 1

    def attach(self, arena: FlatArena, opt: ShardedAdamW) -> None:
        self.arena, self.opt = arena, opt

    # collectives -----------------------------------------------------------------------
    def init_sync(self, flat: torch.Tensor, mode: str = "broadcast") -> None:
        """Make every rank start from the same weights.  ``avg`` is the reference's behaviour
        (`trainer_base.py:180`); ``broadcast`` keeps rank 0's initialisation."""
        if self.world == 1:
            return
        if mode == "avg":
            if flat.dtype in (torch.float16, torch.bfloat16) and flat.device.type == "cpu":
                tmp = flat.float()
                dist.all_reduce(tmp, op=dist.ReduceOp.SUM)
                flat.copy_(tmp / self.world)
            else:
                dist.all_reduce(flat, op=dist.ReduceOp.AVG)
        elif mode == "broadcast":
            dist.broadcast(flat, src=0)
        else:
            raise ValueError("init_sync must be 'broadcast' or 'avg'")

    def launch_round(self, plan: RoundPlan, lr: float, local_count: int) -> None:
        raise NotImplementedError

    def finish_round(self, plan: RoundPlan) -> int:
        raise NotImplementedError

    def barrier(self) -> None:
        if self.world > 1:
            dist.barrier()

    def all_reduce_max(self, value: float) -> float:
        if self.world == 1:
            return float(value)
        t = torch.tensor([float(value)], dtype=torch.float64, device=self.device if self.device.type == "cuda" else "cpu")
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return float(t.item())

    def kernel_launches_per_round(self) -> int:
        """How many of *this repo's* kernels one round launches (for ``gpu_launches``)."""
        return 0

    def close(self) -> None:
        pass


class TorchDistBackend(CommBackend):
    """``torch.distributed`` collectives (NCCL on CUDA, gloo on CPU) around a single-pass AdamW."""

    def __init__(self, rank: int, world: int, device: torch.device, fused_adam: Optional[Callable] = None):
        super().__init__(rank, world, device)
        self.name = "nccl" if self.device.type == "cuda" else "gloo"
        self._fused_adam = fused_adam
        self._launches = 0

    def attach(self, arena: FlatArena, opt: ShardedAdamW) -> None:
        super().attach(arena, opt)
        S = arena.layout.size_slice
        dev = self.device
        self.count = torch.zeros(1, dtype=torch.int32, device=dev)
        self.total = torch.zeros(1, dtype=torch.int32, device=dev)
        self.stash_count = torch.zeros(1, dtype=torch.int32, device=dev)
        self.rs_out = torch.zeros(S, dtype=arena.grad_dtype, device=dev)
        self.shard_out = torch.zeros(S, dtype=arena.dtype, device=dev)
        if dev.type == "cuda":
            self.total_host = torch.zeros(1, dtype=torch.int32).pin_memory()
        else:
            self.total_host = torch.zeros(1, dtype=torch.int32)

    @torch.no_grad()
    def launch_round(self, plan: RoundPlan, lr: float, local_count: int) -> None:
        arena, opt = self.arena, self.opt
        acc = arena.acc[plan.read_acc]
        theta_out = arena.theta[plan.write_theta]
        S = arena.layout.size_slice
        self.count.fill_(int(local_count))
        if self.world > 1:
            work = dist.all_reduce(self.count, op=dist.ReduceOp.SUM, async_op=True)
            dist.reduce_scatter_tensor(self.rs_out, acc, op=dist.ReduceOp.SUM)
            work.wait()
            gsum = self.rs_out
        else:
            gsum = acc[:S]
        self.total.copy_(self.count)
        if plan.add_stash:
            self.total.add_(self.stash_count)
        if plan.write_stash:
            self.stash_count.copy_(self.count)
        inv = 1.0 / self.total.clamp(min=1).to(torch.float32)
        hp = opt.hyper(lr, plan, inv)
        if self._fused_adam is not None:
            self._fused_adam(gsum, opt.master, opt.exp_avg, opt.exp_avg_sq, opt.stash, self.shard_out, hp)
            self._launches = 1
        else:
            adamw_shard_update_(gsum, opt.master, opt.exp_avg, opt.exp_avg_sq, opt.stash, self.shard_out, hp)
        opt.after_launch(plan)
        if self.world > 1:
            dist.all_gather_into_tensor(theta_out, self.shard_out)
        else:
            theta_out.copy_(self.shard_out)
        acc.zero_()
        self.total_host.copy_(self.total, non_blocking=True)

    def finish_round(self, plan: RoundPlan) -> int:
        return int(self.total_host.item())

    def kernel_launches_per_round(self) -> int:
        return self._launches


def make_backend(name: str, rank: int, world: int, device: torch.device, n_nodes: int = 1, **kw) -> CommBackend:
    """``auto`` -> ``symm`` (the fused RS + AdamW + AG kernel over NVLink) on CUDA inside one NVSwitch domain, ``nccl`` across nodes,
    ``gloo`` on CPU.  A single-node CUDA job whose symmetric-memory backend cannot be brought up is an ERROR, not a silent 1.5x
    slower NCCL run - set ``comm_backend=nccl`` explicitly (or ``ACCO_ALLOW_NCCL_FALLBACK=1``) to accept the library path."""
    import os
    device = torch.device(device)
    name = (name or "auto").lower()
    if device.type != "cuda":
        return TorchDistBackend(rank, world, device)
    if name == "auto" and n_nodes > 1:
        name = "nccl"           # peer-mapped symmetric memory / NVLS multicast exist only inside one NVSwitch domain
    if name in ("auto", "symm"):
        try:
            from .symm import SymmBackend
            return SymmBackend(rank, world, device, **kw)
        except Exception as e:  # pragma: no cover - needs a GPU box
            if name == "symm" or os.environ.get("ACCO_ALLOW_NCCL_FALLBACK") != "1":
                raise RuntimeError(f"the fused symmetric-memory backend could not be initialised ({type(e).__name__}: {e}); pass "
                                   f"comm_backend=nccl (or ACCO_ALLOW_NCCL_FALLBACK=1) to run on the NCCL library path instead") from e
            import logging
            logging.getLogger("acco_b200").warning(f"symmetric-memory backend unavailable ({type(e).__name__}: {e}); falling back to NCCL")
    fused = None
    try:
        from ..ops.adam import fused_adamw_shard
        fused = fused_adamw_shard
    except Exception:
        fused = None
    return TorchDistBackend(rank, world, device, fused_adam=fused)
