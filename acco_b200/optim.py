"""Sharded AdamW state (1/W of the model per rank) and the reference math for one update.

Reference: `trainer_decoupled.py:296-315` keeps ``params_opt`` (fp32 master copy of the rank's
slice), its fp32 ``.grad`` and a ``torch.optim.AdamW(capturable=True)`` whose foreach step costs
~17 kernel launches and ~10 passes over the shard , plus 1+3 shard-sized clones and
restores on every tentative round (K1, K2, K11).

Here the state is four flat fp32 tensors of ``size_slice`` elements (``master, exp_avg, exp_avg_sq,
stash``) and an update is *one* pass described by :class:`AdamHyper`:

    g      = (reduced_grad_sum [+ stash]) * inv_count
    master' = master * decay;  m' = lerp(m, g, 1-b1);  v' = b2*v + (1-b2) g^2
              decay = 1 inside the no-decay ranges (train key ``no_decay_1d``), 1 - lr*wd elsewhere
    master' -= lr / (1 - b1^t) * m' / (sqrt(v') / sqrt(1 - b2^t) + eps)
    out_bf16 = cast(master')                       # always produced (it is what gets all-gathered)
    master, m, v <- master', m', v'                # only if the commit flags say so

which is exactly ``torch.optim.AdamW`` (decoupled weight decay, bias-corrected; with a no-decay table, AdamW
with a second parameter group of ``weight_decay=0``) - verified in ``tests/test_optim.py`` and
``tests/test_no_decay.py``.  :func:`adamw_shard_update_` below is the plain-PyTorch implementation
(CPU / gloo path and numerics oracle for the sm_90a kernel in ``csrc/rs_adam_ag.cu``).

Gradient clipping (train key ``max_grad_norm``) is a scalar on ``g``, so it never touches the update
math: every round, whatever its kind, with ``s`` the round's reduced sum (+ stash when ``add_stash``),

    norm    = ||s * inv_count||_2 over the whole flat parameter vector (all ranks' slices)
    inv_eff = inv_count * min(1, max_grad_norm / (norm + 1e-6))      # torch.nn.utils.clip_grad_norm_

and the update runs with ``inv_count = inv_eff`` (:func:`clip_scale`).  The stash keeps the
*unclipped* sum, so a real ACCO round clips the norm of the whole two-half batch, and a tentative
round clips its own half-batch gradient.  ``max_grad_norm = inf`` measures without clipping
(the coefficient is exactly 1).
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Dict, Optional, Sequence, Tuple

import torch

from .parallel.schedule import COMMIT_ALL, COMMIT_PARAM, COMMIT_STATE

__all__ = ["AdamHyper", "ShardedAdamW", "adamw_shard_update_", "clip_scale", "check_max_grad_norm", "check_no_decay_ranges"]


@dataclass
class AdamHyper:
    lr: float
    beta1: float = 0.9
    beta2: float = 0.999
    eps: float = 1e-8
    weight_decay: float = 0.01
    step: int = 1            # 1-based step used for the bias correction of *this* update
    inv_count: object = 1.0  # 1 / (global number of micro-batch gradients in the sum); float or 1-elem tensor
    commit: int = COMMIT_ALL
    add_stash: bool = False
    write_stash: bool = False
    no_decay: Optional[Sequence[Tuple[int, int]]] = None   # sorted, disjoint [lo, hi) ranges of the flat vector updated with decay = 1
    shard_base: int = 0      # flat index of the shard's element 0 (the ranges are global, the shard is a slice)
    no_decay_dev: Optional[torch.Tensor] = None            # the same table as a CUDA int64 [n, 2] tensor, for the sm_90a kernel


@torch.no_grad()
def adamw_shard_update_(
    grad_sum: torch.Tensor,      # [S] any float dtype: this round's reduced gradient *sum* for the shard
    master: torch.Tensor,        # [S] fp32
    exp_avg: torch.Tensor,       # [S] fp32
    exp_avg_sq: torch.Tensor,    # [S] fp32
    stash: Optional[torch.Tensor],  # [S] fp32 or None
    out: torch.Tensor,           # [S] model dtype: receives cast(master')
    hp: AdamHyper,
) -> None:
    g = grad_sum.to(torch.float32)
    if hp.add_stash:
        g = g + stash
    if hp.write_stash:
        stash.copy_(g)
    g = g * hp.inv_count
    m = torch.lerp(exp_avg, g, 1.0 - hp.beta1)
    v = exp_avg_sq * hp.beta2 + (1.0 - hp.beta2) * g * g
    bc1 = 1.0 - hp.beta1 ** hp.step
    bc2 = 1.0 - hp.beta2 ** hp.step
    decay = 1.0 - hp.lr * hp.weight_decay
    if hp.no_decay:
        S = master.numel()
        decay = torch.full_like(master, decay)
        for lo, hi in hp.no_decay:
            decay[max(lo - hp.shard_base, 0):max(min(hi - hp.shard_base, S), 0)] = 1.0
    p = master * decay
    denom = v.sqrt() / (bc2 ** 0.5) + hp.eps
    p = p - (hp.lr / bc1) * (m / denom)
    out.copy_(p)
    if hp.commit & COMMIT_PARAM:
        master.copy_(p)
    if hp.commit & COMMIT_STATE:
        exp_avg.copy_(m)
        exp_avg_sq.copy_(v)


def check_max_grad_norm(value) -> Optional[float]:
    """``max_grad_norm`` as the trainer uses it: ``None`` (off) or a positive float (``inf``: log the norm, never clip)."""
    if value is None:
        return None
    if isinstance(value, bool) or not isinstance(value, (int, float)):
        raise ValueError(f"max_grad_norm must be null or a positive number, got {value!r}")
    v = float(value)
    if math.isnan(v) or v <= 0:
        raise ValueError(f"max_grad_norm must be null or a positive number, got {value!r}")
    return v


def check_no_decay_ranges(ranges) -> Optional[Tuple[Tuple[int, int], ...]]:
    """A no-decay table as the update uses it: ``None`` when empty, else ``(lo, hi)`` pairs with ``0 <= lo < hi``, sorted and
    disjoint (the kernel searches it by bisection)."""
    table = tuple((int(lo), int(hi)) for lo, hi in (ranges or ()))
    prev = 0
    for lo, hi in table:
        if not prev <= lo < hi:
            raise ValueError(f"no-decay ranges must be sorted, disjoint [lo, hi) pairs with lo < hi, got {list(table)}")
        prev = hi
    return table or None


def clip_scale(sumsq, inv_count, max_norm: float) -> Tuple[torch.Tensor, torch.Tensor]:
    """``(norm, inv_eff)`` of a round from the global sum of squares of its gradient *sum* (fp32, 1-element tensor or float).
    ``norm = sqrt(sumsq) * inv_count``; ``inv_eff = inv_count * clamp(max_norm / (norm + 1e-6), max=1)``, the coefficient
    of ``torch.nn.utils.clip_grad_norm_`` (a NaN norm propagates, as there).  Device ops only: the host is not synchronised."""
    sumsq = torch.as_tensor(sumsq, dtype=torch.float32)
    inv = torch.as_tensor(inv_count, dtype=torch.float32, device=sumsq.device)
    norm = torch.sqrt(sumsq) * inv
    coef = torch.clamp(max_norm / (norm + 1e-6), max=1.0)
    return norm, inv * coef


class ShardedAdamW:
    """fp32 optimizer state for the slice ``[rank*size_slice, (rank+1)*size_slice)``."""

    def __init__(self, shard_init: torch.Tensor, lr: float, betas=(0.9, 0.999), eps: float = 1e-8,
                 weight_decay: float = 0.01, allocator=None, no_decay=None, shard_base: int = 0):
        """``no_decay``: ranges of the flat parameter vector (global indices, see ``FlatArena.no_decay_ranges``) that are updated
        without weight decay; ``shard_base``: flat index of this shard's first element."""
        S = shard_init.numel()
        dev = shard_init.device
        alloc = allocator or (lambda n, dt: torch.zeros(n, dtype=dt, device=dev))
        self.master = alloc(S, torch.float32)
        self.master.copy_(shard_init.to(torch.float32))
        self.exp_avg = alloc(S, torch.float32)
        self.exp_avg_sq = alloc(S, torch.float32)
        self.stash = alloc(S, torch.float32)
        self.step = 0                 # committed Adam steps
        self.base_lr = float(lr)
        self.beta1, self.beta2 = float(betas[0]), float(betas[1])
        self.eps, self.weight_decay = float(eps), float(weight_decay)
        self.no_decay = check_no_decay_ranges(no_decay)
        self.shard_base = int(shard_base)
        self.no_decay_dev = None
        if self.no_decay and dev.type == "cuda":
            self.no_decay_dev = torch.tensor(self.no_decay, dtype=torch.int64, device=dev).contiguous()

    def hyper(self, lr: float, plan, inv_count) -> AdamHyper:
        """Hyper-parameters of the update for ``plan``.  ``inv_count`` is ``1 / total`` where
        ``total`` is the global micro-grad count of the sum being applied (a float, or a
        1-element device tensor when the count only exists on the device)."""
        return AdamHyper(
            lr=float(lr), beta1=self.beta1, beta2=self.beta2, eps=self.eps, weight_decay=self.weight_decay,
            step=self.step + 1, inv_count=inv_count, commit=plan.commit,
            add_stash=plan.add_stash, write_stash=plan.write_stash,
            no_decay=self.no_decay, shard_base=self.shard_base, no_decay_dev=self.no_decay_dev,
        )

    def after_launch(self, plan) -> None:
        """Host-side step counter: known as soon as a committing round has been enqueued."""
        if plan.commit & COMMIT_STATE:
            self.step += 1

    # -- checkpoint -----------------------------------------------------------------------
    def state_dict(self) -> Dict[str, object]:
        return {
            "master": self.master.detach().cpu().clone(), "exp_avg": self.exp_avg.detach().cpu().clone(),
            "exp_avg_sq": self.exp_avg_sq.detach().cpu().clone(), "stash": self.stash.detach().cpu().clone(),
            "step": self.step,
        }

    def load_state_dict(self, sd: Dict[str, object]) -> None:
        for k in ("master", "exp_avg", "exp_avg_sq", "stash"):
            getattr(self, k).copy_(sd[k])
        self.step = int(sd["step"])

    def memory_bytes(self) -> int:
        return 4 * 4 * self.master.numel()
