"""Round state machine and LR schedules - the *semantics* of ACCO / DPU / DDP, with no
tensors, streams or collectives in sight (so it is unit-testable and shared by every backend).

Reference behaviour being reproduced (`trainer_decoupled.py:43-63, 67-126, 431-598`):
rounds are numbered by ``count_after_init = 0, 1, 2, ...``.

* **ACCO** - even rounds are *tentative*: the optimizer consumes the half-batch ``g~_t`` (grads
  evaluated at the estimate ``theta~_t``), produces ``theta~_{t+1}`` and is rolled back
  (`:79-84, 113-121`).  Odd rounds are *real*: the optimizer consumes ``g~_t + g_t``, divides by
  the global micro-batch count, commits ``theta_{t+1}``, steps the LR scheduler (`:102-104`) and
  the global gradient counter advances (`:501-502`).
* **DPU**  - every round commits, using gradients that are one round stale)``, overlapped).
* **DDP**  - every round commits, synchronously, on fresh gradients (the reference pairs torch DDP
  with ZeroRedundancyOptimizer, `:226-241, 732-833`).

Instead of the reference's clone/restore of master weights and Adam state, a plan carries
*commit flags*; instead of copying grads into a com buffer, it names which of the two
accumulators is consumed (``read_acc``) and which parameter buffer receives the gathered
weights (``write_theta``); the half-batch sum of the tentative round is kept in an fp32
*stash* shard on the owner so the real round only has to reduce the second half.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Callable, Dict, Optional

__all__ = [
    "COMMIT_NONE", "COMMIT_PARAM", "COMMIT_STATE", "COMMIT_ALL",
    "RoundPlan", "RoundScheduler", "LRSchedule", "get_lr_lambda",
]

COMMIT_NONE = 0
COMMIT_PARAM = 1   # write the fp32 master weights back
COMMIT_STATE = 2   # write exp_avg / exp_avg_sq back and advance the Adam step
COMMIT_ALL = COMMIT_PARAM | COMMIT_STATE


@dataclass(frozen=True)
class RoundPlan:
    index: int            # round number == the reference's ``count_after_init`` (warm-up rounds: -1)
    kind: str             # "tentative" | "real" | "sync"
    read_acc: int         # accumulator consumed by this round
    write_theta: int      # parameter buffer that receives the all-gathered weights
    commit: int           # COMMIT_* flags
    add_stash: bool       # add the stashed half-batch sum (and its count) before the update
    write_stash: bool     # store this round's reduced sum (and count) into the stash
    lr_step: bool         # advance the LR schedule after this round
    counts_toward_total: bool  # add the global micro-grad count of this update to ``count_grad_tot``
    blocking: bool        # compute must wait for the round before the next micro-batch (DDP / warm-up)


class RoundScheduler:
    """Generates :class:`RoundPlan` s and tracks the counters the reference keeps in
    ``count_after_init`` / ``count_com`` / ``count_grad_tot`` / the LR scheduler."""

    def __init__(self, method: str, n_warmup_rounds: int = 0, reference_quirks: bool = False):
        if method not in ("acco", "dpu", "ddp"):
            raise ValueError("You must select one of the following method_name: 'acco', 'ddp', 'dpu'")
        self.method = method
        self.reference_quirks = reference_quirks
        self.warmup_left = 0 if method == "ddp" else int(n_warmup_rounds)
        self.round = 0            # launched rounds (incl. warm-up)
        self.count_after_init = 0  # rounds launched after warm-up
        self.count_com = 0         # completed rounds (reference ``count_com``)
        self.count_grad_tot = 0    # committed micro-batch gradients, summed over ranks
        self.opt_steps = 0         # committed optimizer steps
        self.lr_steps = 0          # scheduler steps taken

    # -- which buffers a phase uses -------------------------------------------------------
    def compute_buffers(self, round_in_flight: bool) -> Dict[str, int]:
        """Buffers the *compute* side must use now.  ``R = self.round`` is the next round to be
        launched; it will consume what backward is writing now, hence ``acc[R % 2]``.  Round
        ``R - 1`` wrote (or is still writing) ``theta[R % 2]``: if it is still in flight compute
        must stay on the other buffer, ``theta[(R + 1) % 2]``."""
        R = self.round
        return {"theta": (R + 1) % 2 if round_in_flight else R % 2, "acc": R % 2}

    def in_warmup(self) -> bool:
        return self.warmup_left > 0

    def next_plan(self) -> RoundPlan:
        """Plan for the round about to be launched (advances the launch counters)."""
        r = self.round
        read_acc, write_theta = r % 2, (r + 1) % 2
        if self.method == "ddp" or self.warmup_left > 0:
            plan = RoundPlan(-1 if self.warmup_left > 0 else r, "sync", read_acc, write_theta, COMMIT_ALL,
                             False, False, True, True, True)
            if self.warmup_left > 0:
                self.warmup_left -= 1
            else:
                self.count_after_init += 1
        elif self.method == "dpu":
            plan = RoundPlan(self.count_after_init, "real", read_acc, write_theta, COMMIT_ALL,
                             False, False, True, True, False)
            self.count_after_init += 1
        else:  # acco
            c = self.count_after_init
            if c % 2 == 0:
                commit = COMMIT_NONE
                if self.reference_quirks and c == 0:
                    commit = COMMIT_STATE   # round-0 state reset is a no-op in the reference
                plan = RoundPlan(c, "tentative", read_acc, write_theta, commit, False, True, False, False, False)
            else:
                plan = RoundPlan(c, "real", read_acc, write_theta, COMMIT_ALL, True, False, True, True, False)
            self.count_after_init += 1
        self.round += 1
        return plan

    def complete(self, plan: RoundPlan, global_count: int) -> None:
        """Book-keeping when a round has finished (the reference does this at the flip)."""
        self.count_com += 1
        if plan.commit & COMMIT_STATE:
            self.opt_steps += 1
        if plan.lr_step:
            self.lr_steps += 1
        if plan.counts_toward_total:
            self.count_grad_tot += int(global_count)

    def state_dict(self) -> Dict[str, int]:
        return {k: getattr(self, k) for k in
                ("round", "count_after_init", "count_com", "count_grad_tot", "opt_steps", "lr_steps", "warmup_left")}

    def load_state_dict(self, sd: Dict[str, int]) -> None:
        for k, v in sd.items():
            setattr(self, k, int(v))


# ----------------------------------------------------------------------------------------------
# LR schedules (same closed forms as ``transformers.get_scheduler`` which the reference uses,
# `trainer_decoupled.py:236-241, 310-315`)
# ----------------------------------------------------------------------------------------------

def get_lr_lambda(name: str, num_warmup_steps: int, num_training_steps: int) -> Callable[[int], float]:
    name = str(name).lower()
    w, T = int(num_warmup_steps), int(num_training_steps)

    def warm(step: int) -> Optional[float]:
        if step < w:
            return float(step) / float(max(1, w))
        return None

    if name == "cosine":
        def f(step: int) -> float:
            x = warm(step)
            if x is not None:
                return x
            progress = float(step - w) / float(max(1, T - w))
            return max(0.0, 0.5 * (1.0 + math.cos(math.pi * 2.0 * 0.5 * progress)))
    elif name == "linear":
        def f(step: int) -> float:
            x = warm(step)
            if x is not None:
                return x
            return max(0.0, float(T - step) / float(max(1, T - w)))
    elif name == "constant":
        def f(step: int) -> float:
            return 1.0
    elif name == "constant_with_warmup":
        def f(step: int) -> float:
            x = warm(step)
            return 1.0 if x is None else x
    elif name in ("cosine_with_restarts", "polynomial", "inverse_sqrt"):
        if name == "inverse_sqrt":
            def f(step: int) -> float:
                x = warm(step)
                if x is not None:
                    return x
                shift = max(w, 1)
                return math.sqrt(shift / max(step, 1)) if step > 0 else 1.0
        elif name == "polynomial":
            def f(step: int) -> float:
                x = warm(step)
                if x is not None:
                    return x
                if step > T:
                    return 1e-7
                rem = 1 - (step - w) / max(1, T - w)
                return rem * (1.0 - 1e-7) + 1e-7
        else:
            def f(step: int) -> float:
                x = warm(step)
                if x is not None:
                    return x
                progress = float(step - w) / float(max(1, T - w))
                if progress >= 1.0:
                    return 0.0
                return max(0.0, 0.5 * (1.0 + math.cos(math.pi * ((1.0 * progress) % 1.0))))
    else:
        raise ValueError(f"unknown scheduler_name {name!r}")
    return f


@dataclass
class LRSchedule:
    """``lr(k) = base_lr * lambda(k)`` where ``k`` counts scheduler steps.

    ``unit='optimizer_step'`` reproduces the reference;
    ``unit='grads'`` advances by the number of committed gradients (the authors' intent)."""

    base_lr: float
    name: str = "cosine"
    num_warmup_steps: int = 0
    num_training_steps: int = 1
    unit: str = "optimizer_step"
    _fn: Callable[[int], float] = field(init=False, repr=False)

    def __post_init__(self):
        if self.unit not in ("optimizer_step", "grads"):
            raise ValueError("lr_unit must be 'optimizer_step' or 'grads'")
        self._fn = get_lr_lambda(self.name, self.num_warmup_steps, self.num_training_steps)

    def lr_at(self, sched: "RoundScheduler") -> float:
        k = sched.lr_steps if self.unit == "optimizer_step" else sched.count_grad_tot
        return float(self.base_lr) * self._fn(int(k))

    def value(self, k: int) -> float:
        return float(self.base_lr) * self._fn(int(k))
