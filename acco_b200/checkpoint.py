"""Checkpoint files: atomic writes, discovery of the latest complete checkpoint, elastic re-sharding of the optimizer state.

The reference only ever *saves* ``model.state_dict()`` (`/root/reference/trainer_decoupled.py:559-574,593-598`; the optimizer
save is commented out and nothing can be loaded back).  Layout kept from it::

    checkpoints/{id_run}_model_{count_grad_tot}.pt      periodic (every >= save_interval_s), HF parameter names
    checkpoints/{id_run}_model.pt                       final      (``dpu_model`` / ``_ddp_model`` variants)

added here (``save_optimizer``), one file per rank next to the model file::

    {stem}_optim_rank{r}of{W}.pt    fp32 master / exp_avg / exp_avg_sq / stash of the slice [r * size_slice, (r+1) * size_slice)
                                    of the flat parameter vector + scheduler counters

A job that lost (or gained) GPUs restarts with a different world size: :func:`reshard_optimizer_state` rebuilds the slice of the
*new* layout from the shards of the old one, reading only the old shards that overlap it."""
from __future__ import annotations

import glob
import os
import re
from typing import Dict, List, Optional, Tuple

import torch

__all__ = ["atomic_save", "shard_path", "shard_sets", "reshard_optimizer_state", "latest_checkpoint", "prune_checkpoints"]

_SHARD_RE = re.compile(r"_optim_rank(\d+)of(\d+)\.pt$")
_STATE_KEYS = ("master", "exp_avg", "exp_avg_sq", "stash")


def atomic_save(obj, path: str) -> None:
    """``torch.save`` through a temporary file + rename: a job killed in the middle of a save leaves the previous file (or no
    file), never a truncated one that a later ``resume_from=auto`` would pick up."""
    d = os.path.dirname(path)
    if d:
        os.makedirs(d, exist_ok=True)
    tmp = f"{path}.tmp{os.getpid()}"
    try:
        torch.save(obj, tmp)
        os.replace(tmp, path)
    finally:
        if os.path.exists(tmp):
            os.remove(tmp)


def shard_path(model_path: str, rank: int, world: int) -> str:
    return f"{os.path.splitext(model_path)[0]}_optim_rank{rank}of{world}.pt"


def shard_sets(model_path: str) -> Dict[int, List[str]]:
    """``{world_size: [shard files in rank order]}`` for every COMPLETE set of optimizer shards next to ``model_path``."""
    stem = os.path.splitext(model_path)[0]
    found: Dict[int, Dict[int, str]] = {}
    for f in glob.glob(f"{glob.escape(stem)}_optim_rank*of*.pt"):
        m = _SHARD_RE.search(f)
        if m:
            found.setdefault(int(m.group(2)), {})[int(m.group(1))] = f
    return {w: [ranks[r] for r in range(w)] for w, ranks in found.items() if all(r in ranks for r in range(w))}


def reshard_optimizer_state(shards: List[str], new_rank: int, new_size_slice: int, numel: Optional[int] = None) -> Tuple[Dict[str, object], Dict[str, object]]:
    """Optimizer state of slice ``[new_rank * new_size_slice, +new_size_slice)`` assembled from a complete set of old shards
    (rank order).  Returns ``(optimizer_state_dict, header)`` where ``header`` holds the rank-independent entries of the old
    shard (scheduler counters, world size, ...).  Elements that no old shard covers (padding beyond the old layout) are zero."""
    lo, hi = new_rank * new_size_slice, (new_rank + 1) * new_size_slice
    out = {k: torch.zeros(new_size_slice, dtype=torch.float32) for k in _STATE_KEYS}
    header: Optional[Dict[str, object]] = None
    step = None
    old_slice = None
    for r_old, f in enumerate(shards):
        if old_slice is not None and (r_old * old_slice >= hi or (r_old + 1) * old_slice <= lo) and header is not None:
            continue                                           # no overlap with the new slice: do not even read the file
        st = torch.load(f, map_location="cpu", weights_only=False)
        old_slice = int(st["size_slice"])
        if header is None:
            header = {k: v for k, v in st.items() if k not in ("optimizer", "rng")}
            if numel is not None and st.get("numel") is not None and int(st["numel"]) != int(numel):
                raise ValueError(f"checkpoint was written for {int(st['numel'])} parameters, this model has {int(numel)}")
        step = int(st["optimizer"]["step"]) if step is None else step
        if int(st["optimizer"]["step"]) != step:
            raise ValueError(f"optimizer shards disagree on the step count ({f})")
        o_lo, o_hi = r_old * old_slice, (r_old + 1) * old_slice
        a, b = max(lo, o_lo), min(hi, o_hi)
        if a >= b:
            continue
        for k in _STATE_KEYS:
            out[k][a - lo:b - lo] = st["optimizer"][k][a - o_lo:b - o_lo].to(torch.float32)
    assert header is not None, "empty shard list"
    opt = dict(out)
    opt["step"] = step
    return opt, header


def _is_model_file(path: str) -> bool:
    return path.endswith(".pt") and not _SHARD_RE.search(path) and ".tmp" not in os.path.basename(path)


def latest_checkpoint(directory: str, require_optimizer: bool = False) -> Optional[str]:
    """Newest model file under ``directory`` (by modification time); with ``require_optimizer`` only checkpoints that have a
    complete set of optimizer shards count (a checkpoint is complete only when every rank's shard is on disk)."""
    cands = [f for f in glob.glob(os.path.join(directory, "*.pt")) if _is_model_file(f)]
    cands.sort(key=lambda f: (os.path.getmtime(f), f), reverse=True)
    for f in cands:
        if not require_optimizer or shard_sets(f):
            return f
    return None


def prune_checkpoints(directory: str, prefix: str, keep: int, rank: int = 0) -> List[str]:
    """Keep the ``keep`` newest PERIODIC checkpoints ``{prefix}{count}.pt`` (count = digits); rank 0 removes older model files,
    every rank removes its own optimizer shards of them.  Returns the removed files."""
    if keep is None or int(keep) <= 0:
        return []
    pat = re.compile(re.escape(prefix) + r"(\d+)\.pt$")
    models = []
    for f in glob.glob(os.path.join(directory, f"{glob.escape(prefix)}*.pt")):
        m = pat.search(os.path.basename(f))
        if m and _is_model_file(f):
            models.append((int(m.group(1)), f))
    # shards whose model file is already gone (removed by rank 0 earlier) are orphans of this rank
    stems = {int(m.group(1)) for m in (re.search(re.escape(prefix) + r"(\d+)_optim_rank", os.path.basename(f))
                                       for f in glob.glob(os.path.join(directory, f"{glob.escape(prefix)}*_optim_rank{rank}of*.pt"))) if m}
    counts = sorted({c for c, _ in models} | stems, reverse=True)
    doomed = set(counts[int(keep):])
    removed = []
    for c in doomed:
        victims = glob.glob(os.path.join(directory, f"{glob.escape(prefix)}{c}_optim_rank{rank}of*.pt"))
        if rank == 0:
            victims += [f for cc, f in models if cc == c]
        for f in victims:
            try:
                os.remove(f)
                removed.append(f)
            except FileNotFoundError:
                pass
    return removed
