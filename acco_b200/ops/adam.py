"""Single-pass sharded AdamW on one GPU (``csrc/rs_adam_ag.cu``, local variant).

Used by the NCCL baseline backend after ``reduce_scatter_tensor`` and by the single-GPU path;
the multi-GPU product path runs the same math inside the fused RS+AdamW+AG kernel
(``parallel/symm.py``).  Semantics == :func:`acco_b200.optim.adamw_shard_update_`."""
from __future__ import annotations

import torch

from . import count_launch, load_ext, use_kernels


_SCRATCH = {}
_NORM = {}


def _scratch(device) -> torch.Tensor:
    key = str(device)
    if key not in _SCRATCH:
        _SCRATCH[key] = torch.zeros(4, dtype=torch.int32, device=device)
    return _SCRATCH[key]


def _no_decay_table(hp, device):
    """``hp``'s no-decay ranges on ``device`` (``ShardedAdamW`` builds the tensor once; a hand-made ``AdamHyper`` gets it here)."""
    if not hp.no_decay:
        return None
    if hp.no_decay_dev is None:
        from ..optim import check_no_decay_ranges
        hp.no_decay_dev = torch.tensor(check_no_decay_ranges(hp.no_decay), dtype=torch.int64, device=device).contiguous()
    return hp.no_decay_dev


def fused_adamw_shard(grad_sum, master, exp_avg, exp_avg_sq, stash, out, hp) -> None:
    from ..optim import adamw_shard_update_
    if not use_kernels(grad_sum, master, out, bf16_only=False) or master.numel() % 8 != 0:
        return adamw_shard_update_(grad_sum, master, exp_avg, exp_avg_sq, stash, out, hp)
    C = load_ext(required=True)
    inv = hp.inv_count
    if not torch.is_tensor(inv):
        inv = torch.full((1,), float(inv), dtype=torch.float32, device=master.device)
    C.adamw_shard(grad_sum, master, exp_avg, exp_avg_sq, stash, out, inv.reshape(1).float(), _scratch(master.device),
                  float(hp.lr), float(hp.beta1), float(hp.beta2), float(hp.eps), float(hp.weight_decay),
                  int(hp.step), int(hp.commit), bool(hp.add_stash), bool(hp.write_stash), _no_decay_table(hp, master.device),
                  int(hp.shard_base))
    count_launch("adamw_shard")


def grad_sumsq(grad_sum, stash, add_stash: bool) -> torch.Tensor:
    """fp32 ``[1]``: sum of squares of ``grad_sum (+ stash)`` over the shard, on the device (the local part of a clipped round's
    norm; the NCCL path all-reduces it).  CUDA: ``round_norm_kernel`` in local mode, dispatched like :func:`fused_adamw_shard`."""
    S = stash.numel()
    if not use_kernels(grad_sum, stash, bf16_only=False) or S % 8 != 0:
        g = grad_sum[:S].to(torch.float32)
        if add_stash:
            g = g + stash
        return (g * g).sum().reshape(1)
    C = load_ext(required=True)
    key = str(stash.device)
    if key not in _NORM:
        _NORM[key] = (torch.zeros(4, dtype=torch.int32, device=stash.device),
                      torch.zeros(3 + 4 * int(C.num_sms()), dtype=torch.float32, device=stash.device))
    scratch, out = _NORM[key]
    C.round_norm([grad_sum.data_ptr()], [], 0, stash, scratch, out, S, 0, 1, 1, bool(add_stash),
                 grad_sum.dtype == torch.bfloat16, 0, 0, float("inf"))
    count_launch("round_norm")
    return out[2:3].clone()
