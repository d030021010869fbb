"""Sharded AdamW state (1/W of the model per rank) and the reference math for one update.

Reference: `trainer_decoupled.py:296-315` keeps ``params_opt`` (fp32 master copy of the rank's
slice), its fp32 ``.grad`` and a ``torch.optim.AdamW(capturable=True)`` whose foreach step costs
~17 kernel launches and ~10 passes over the shard , plus 1+3 shard-sized clones and
restores on every tentative round (K1, K2, K11).

Here the state is four flat fp32 tensors of ``size_slice`` elements (``master, exp_avg, exp_avg_sq,
stash``) and an update is *one* pass described by :class:`AdamHyper`:

    g      = (reduced_grad_sum [+ stash]) * inv_count
    master' = master * (1 - lr*wd);  m' = lerp(m, g, 1-b1);  v' = b2*v + (1-b2) g^2
    master' -= lr / (1 - b1^t) * m' / (sqrt(v') / sqrt(1 - b2^t) + eps)
    out_bf16 = cast(master')                       # always produced (it is what gets all-gathered)
    master, m, v <- master', m', v'                # only if the commit flags say so

which is exactly ``torch.optim.AdamW`` (decoupled weight decay, bias-corrected) - verified in
``tests/test_optim.py``.  :func:`adamw_shard_update_` below is the plain-PyTorch implementation
(CPU / gloo path and numerics oracle for the sm_90a kernel in ``csrc/rs_adam_ag.cu``).
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict, Optional

import torch

from .parallel.schedule import COMMIT_ALL, COMMIT_PARAM, COMMIT_STATE

__all__ = ["AdamHyper", "ShardedAdamW", "adamw_shard_update_"]


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
    p = master * (1.0 - hp.lr * hp.weight_decay)
    denom = v.sqrt() / (bc2 ** 0.5) + hp.eps
    p = p - (hp.lr / bc1) * (m / denom)
    out.copy_(p)
    if hp.commit & COMMIT_PARAM:
        master.copy_(p)
    if hp.commit & COMMIT_STATE:
        exp_avg.copy_(m)
        exp_avg_sq.copy_(v)


class ShardedAdamW:
    """fp32 optimizer state for the slice ``[rank*size_slice, (rank+1)*size_slice)``."""

    def __init__(self, shard_init: torch.Tensor, lr: float, betas=(0.9, 0.999), eps: float = 1e-8,
                 weight_decay: float = 0.01, allocator=None):
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

    def hyper(self, lr: float, plan, inv_count) -> AdamHyper:
        """Hyper-parameters of the update for ``plan``.  ``inv_count`` is ``1 / total`` where
        ``total`` is the global micro-grad count of the sum being applied (a float, or a
        1-element device tensor when the count only exists on the device)."""
        return AdamHyper(
            lr=float(lr), beta1=self.beta1, beta2=self.beta2, eps=self.eps, weight_decay=self.weight_decay,
            step=self.step + 1, inv_count=inv_count, commit=plan.commit,
            add_stash=plan.add_stash, write_stash=plan.write_stash,
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
