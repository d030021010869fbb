"""Rank / device discovery and process-group initialisation.

The reference reads ``SLURM_*`` directly and hard-codes NCCL (`trainer_base.py:135-180`).
Here three launchers are recognised, in this order:

1. **torchrun / torch.distributed.run** – ``RANK, LOCAL_RANK, WORLD_SIZE, MASTER_ADDR, MASTER_PORT``
2. **Slurm ``srun``** – ``SLURM_PROCID, SLURM_LOCALID, SLURM_NTASKS, SLURM_JOB_NODELIST, SLURM_STEP_GPUS``
   (same derivation as the reference: master = first expanded host, port = 12346 + min GPU id,
   but the min is numeric – the reference takes a *string* min)
3. **single process** – world of 1 (no env needed).

One process drives one GPU.  The backend is ``nccl`` on CUDA and ``gloo`` on CPU (plumbing
tests).
"""
from __future__ import annotations

import datetime
import os
import socket
from dataclasses import dataclass, field
from typing import List, Optional

import torch
import torch.distributed as dist

from .utils.hostlist import expand_hostlist

__all__ = ["DistEnv", "discover_env", "init_distributed", "shutdown_distributed", "free_port", "create_id_run"]


@dataclass
class DistEnv:
    rank: int = 0
    local_rank: int = 0
    world_size: int = 1
    node_id: int = 0
    n_nodes: int = 1
    id_run: str = "local"
    master_addr: str = "127.0.0.1"
    master_port: int = 29500
    launcher: str = "single"
    hostnames: List[str] = field(default_factory=lambda: ["localhost"])


def create_id_run() -> str:
    """Unique id of a run outside Slurm: ``Y_M_D_h_m_s_<rand>`` (`utils/logs_utils.py:19-40` of the reference; there every rank draws
    its own, here rank 0's draw is broadcast by :func:`init_distributed` so all ranks name the same checkpoint / TensorBoard dir)."""
    import random
    now = datetime.datetime.now()
    return "_".join(str(v) for v in (now.year, now.month, now.day, now.hour, now.minute, now.second, random.SystemRandom().randint(0, 9999)))


_AUTO_ID = "<auto>"


def free_port() -> int:
    with socket.socket(socket.AF_INET, socket.SOCK_STREAM) as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def discover_env(environ: Optional[dict] = None) -> DistEnv:
    env = os.environ if environ is None else environ
    if "RANK" in env and "WORLD_SIZE" in env:
        world = int(env["WORLD_SIZE"])
        local_world = int(env.get("LOCAL_WORLD_SIZE", world))
        rank = int(env["RANK"])
        return DistEnv(
            rank=rank,
            local_rank=int(env.get("LOCAL_RANK", rank % max(local_world, 1))),
            world_size=world,
            node_id=int(env.get("GROUP_RANK", rank // max(local_world, 1))),
            n_nodes=max(world // max(local_world, 1), 1),
            id_run=_torchrun_id(env),
            master_addr=env.get("MASTER_ADDR", "127.0.0.1"),
            master_port=int(env.get("MASTER_PORT", 29500)),
            launcher="torchrun",
        )
    if "SLURM_PROCID" in env and "SLURM_NTASKS" in env:
        hostnames = expand_hostlist(env.get("SLURM_JOB_NODELIST", "localhost")) or ["localhost"]
        gpu_ids = [g for g in env.get("SLURM_STEP_GPUS", env.get("SLURM_JOB_GPUS", "0")).split(",") if g != ""]
        try:
            port_off = min(int(g) for g in gpu_ids)
        except ValueError:
            port_off = 0
        return DistEnv(
            rank=int(env["SLURM_PROCID"]),
            local_rank=int(env.get("SLURM_LOCALID", 0)),
            world_size=int(env["SLURM_NTASKS"]),
            node_id=int(env.get("SLURM_NODEID", 0)),
            n_nodes=len(hostnames),
            id_run=str(env.get("SLURM_JOBID", env.get("SLURM_JOB_ID", "slurm"))),
            master_addr=env.get("MASTER_ADDR", hostnames[0]),
            master_port=int(env.get("MASTER_PORT", 12346 + port_off)),
            launcher="slurm",
            hostnames=hostnames,
        )
    # single process: any free port will do (a fixed default could collide with another job on the box)
    port = int(env.get("MASTER_PORT", 0)) or free_port()
    return DistEnv(id_run=str(env.get("ACCO_RUN_ID", _AUTO_ID)), master_port=port)


def _torchrun_id(env) -> str:
    """``ACCO_RUN_ID`` wins; a user-chosen ``--rdzv-id`` is kept; torchrun's defaults ("none" / a bare number) are not unique per run, so
    a date-based id is drawn (by rank 0, after the process group exists)."""
    if env.get("ACCO_RUN_ID"):
        return str(env["ACCO_RUN_ID"])
    rid = str(env.get("TORCHELASTIC_RUN_ID", "") or "")
    if rid and rid.lower() != "none" and not rid.isdigit():
        return rid
    return _AUTO_ID


def init_distributed(env: Optional[DistEnv] = None, device_type: Optional[str] = None, timeout_s: int = 1800) -> DistEnv:
    """Initialise the default process group (idempotent).  Returns the resolved :class:`DistEnv`."""
    env = env or discover_env()
    if device_type is None:
        device_type = "cuda" if torch.cuda.is_available() else "cpu"
    if device_type == "cuda":
        torch.cuda.set_device(env.local_rank)
    if dist.is_available() and dist.is_initialized():
        env.rank, env.world_size = dist.get_rank(), dist.get_world_size()
        _resolve_id(env)
        return env
    os.environ.setdefault("MASTER_ADDR", env.master_addr)
    os.environ.setdefault("MASTER_PORT", str(env.master_port))
    backend = "nccl" if device_type == "cuda" else "gloo"
    kwargs = {}
    if device_type == "cuda":
        kwargs["device_id"] = torch.device("cuda", env.local_rank)
    attempt = int(os.environ.get("TORCHELASTIC_RESTART_COUNT", "0") or 0)
    if attempt > 0 and os.environ.get("TORCHELASTIC_USE_AGENT_STORE") == "True":
        # A worker group restarted by `torchrun --max-restarts` under the static rendezvous (--master-addr/--master-port) talks to
        # the SAME agent-hosted store as its previous incarnation, whose keys (gloo pair addresses, NCCL ids) are still in it: a rank
        # that reads before its peer has re-written them connects to a dead process ("Connection refused" / a hang).  Give every
        # incarnation its own key space.
        store = dist.PrefixStore(f"acco_attempt_{attempt}", dist.TCPStore(os.environ["MASTER_ADDR"], int(os.environ["MASTER_PORT"]), env.world_size,
                                                                         False, datetime.timedelta(seconds=timeout_s)))
        kwargs["store"] = store
    dist.init_process_group(
        backend=backend,
        rank=env.rank,
        world_size=env.world_size,
        timeout=datetime.timedelta(seconds=timeout_s),
        **kwargs,
    )
    _resolve_id(env)
    return env


def _resolve_id(env: DistEnv) -> None:
    """Replace the ``<auto>`` placeholder by a unique id shared by every rank (two runs launched from the same directory must not
    overwrite each other's ``checkpoints/{id}_model.pt`` and TensorBoard dir)."""
    if env.id_run != _AUTO_ID:
        return
    box = [create_id_run() if env.rank == 0 else None]
    if env.world_size > 1 and dist.is_initialized():
        dist.broadcast_object_list(box, src=0)
    env.id_run = str(box[0])


def shutdown_distributed() -> None:
    if dist.is_available() and dist.is_initialized():
        try:
            dist.barrier()
        except Exception:
            pass
        dist.destroy_process_group()
