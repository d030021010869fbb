"""``DecoupledTrainer`` - ACCO / DPU / DDP training with a sharded optimizer.

Public surface kept from the reference (`trainer_decoupled.py:170-186`): the
constructor keywords, ``.train()`` dispatching on ``args.method_name``, ``train_acco / train_dpu /
train_ddp``, ``eval_loop``, ``warmup_steps``, ``get_weights / set_weights / get_grads / set_grads``,
``get_train_dataloader / get_eval_dataloader`` and the artefact layout (``tensorboard/``,
``checkpoints/{id_run}_model*.pt`` with HF key names, ``results.csv``).

What is different underneath:

* no Python communication thread, no ``mp.Barrier``: the main thread enqueues a whole round on a
  high-priority *communication stream* the moment the previous one has finished, and polls a CUDA
  event (``query()``) at micro-batch boundaries - "accumulate while you communicate" falls out of
  that poll exactly as in the reference (`:497`);
* no flip copies: two parameter buffers and two gradient accumulators alternate
  (:mod:`acco_b200.parallel.arena`), the round consumes an accumulator in place;
* the tentative (uncommitted) optimizer step is a *flag* on the fused update, not a
  clone/restore of master weights and Adam state;
* one micro-batch is one CUDA-graph launch when batch shapes are static;
* all counters live on the host; the only per-round device->host traffic is a 4-byte global count
  and the 4-byte loss, both landing in pinned memory behind events the host already waits on.
"""
from __future__ import annotations

import contextlib
import logging
import math
import numbers
import os
import threading
import time
from typing import Any, Callable, Dict, List, Optional

import torch
import torch.distributed as dist
import torch.nn as nn

from .config import to_container
from .data import (PREFERENCE_COLUMNS, BatchLoader, DeviceFeeder, DocumentCollator, PackedCollator, PadCollator, PreferenceCollator,
                   make_const_len_tokenize_fn, make_packed_tokenize_fn, make_preference_tokenize_fn, make_truncate_tokenize_fn, pack_sft,
                   stack_collate)
from .launch import DistEnv, discover_env, init_distributed
from .obs import OverlapMeter, ScalarWriter, TrainingPrinter, create_dict_result, log_training_scalars, nvtx_range, save_result
from .optim import ShardedAdamW, check_max_grad_norm
from .parallel.arena import FlatArena
from .parallel.backend import CommBackend, make_backend
from .parallel.graphs import MicroBatchGraphs
from .parallel.schedule import LRSchedule, RoundPlan, RoundScheduler
from .utils.misc import LabelSmoother

__all__ = ["DecoupledTrainer", "TRAIN_DEFAULTS"]

# defaults for every key the trainer reads; reference keys first (`config/train/acco.yaml`), then ours
TRAIN_DEFAULTS: Dict[str, Any] = dict(
    method_name="acco", run_baseline_ddp=False, batch_size=8, n_grad_accumulation=1, max_length=1024,
    learning_rate=6e-4, weight_decay=0.1, adam_beta1=0.9, adam_beta2=0.95, scheduler_name="cosine", warmup=1000,
    nb_steps_tot=50000, n_warmup_steps=0, use_mixed_precision=True, const_len_batch=True, eval=False, eval_step=500,
    save=True, finetune=False, dataloader_num_workers=1, dataloader_pin_memory=True, dataloader_persistent_workers=True,
    label_smoothing_factor=0, group_by_length=False, gradient_accumulation_steps=1, run_expe_slow=False,
    # additions
    comm_backend="auto", lr_unit="optimizer_step", reference_quirks=False, init_sync="broadcast", cuda_graphs=True,
    slow_ranks=(), slow_factor_ms=0, save_interval_s=1800, save_optimizer=False, resume_from=None, save_total_limit=None,
    ddp_weights_dtype="bf16", ddp_impl="native", fused_ag_gemm=False, adam_eps=1e-8, log_every=10, tensorboard=True, seed=None,
    eval_all_ranks=False, max_eval_batches=None, pad_to_multiple_of=None, save_grad_counts=False, save_com_logs=False,
    static_accumulation=False,      # True: never accumulate beyond n_grad_accumulation (wait for the round instead): reproducible A/B runs
    debug_poison=False,             # True (or ACCO_DEBUG_POISON=1): NaN-fill the parameter buffer a round is about to overwrite (race detector)
    preempt_save=False,             # True: SIGTERM / SIGUSR1 (Slurm pre-emption, `scancel --signal`) -> checkpoint at the next committed round, then stop
    fault_inject=None,              # "rank@count" - that rank kills itself (os._exit) once count_grad_tot >= count; fires once per cwd
    packing=False,                  # SFT: pack whole samples into full rows (document-masked attention, per-sample positions)
    max_grad_norm=None,             # global gradient-norm clipping of every round (.inf: log the norm only); logged as grad_norm
    fp8=False,                      # FP8 GEMMs (e4m3 / e5m2, per-tensor current scaling) for the block linears of native models (ops/fp8.py)
    no_decay_1d=False,              # True: trainable parameters with ndim <= 1 (norm gains, biases) are updated without weight decay
    grad_accum_dtype=None,          # "fp32": fp32 gradient accumulators under bf16 weights (bound as p.main_grad); None: the weights' dtype
    document_mask=False,            # const-len rows: no attention across the documents of a row, positions restart per document
    z_loss_weight=0,                # native models: add z * mean lse^2 (PaLM z-loss) to every training micro-batch's loss; logged as z_loss
    distill_teacher=None,           # HF checkpoint dir of a frozen native teacher: train on (1-a) CE + a T^2 KL(teacher || student)
    distill_alpha=0.5,              # a in (0, 1]: weight of the distillation term
    distill_temperature=1.0,        # T > 0: temperature of both softmaxes in the KL
    dpo_beta=None,                  # beta > 0 (TRL's usual 0.1): DPO on preference pairs against a frozen reference; None: off
    dpo_reference=None,             # HF checkpoint dir of the frozen native reference (main.py: model.pretrained when unset)
    simpo_beta=None,                # beta > 0 (e.g. 2.0): SimPO on preference pairs, no reference; None: off
    simpo_gamma=0.5,                # gamma >= 0: SimPO's target reward margin
    orpo_lambda=None,               # lambda > 0 (TRL's usual 0.1): ORPO (SFT + odds-ratio term) on preference pairs, no reference; None: off
)

# the three device scalars each reference-free preference objective logs (ops.simpo_loss / ops.orpo_loss `out`)
PREF_SCALARS = {"simpo": ("simpo_reward_chosen", "simpo_reward_rejected", "simpo_accuracy"),
                "orpo": ("orpo_nll", "orpo_log_odds", "orpo_accuracy")}


class _Args:
    """Attribute view over the user's ``args`` (Hydra DictConfig, AttrDict, Namespace, dict ...)
    that falls back to :data:`TRAIN_DEFAULTS` for keys the user did not provide."""

    def __init__(self, raw: Any):
        object.__setattr__(self, "_raw", raw)

    def _lookup(self, k: str):
        raw = object.__getattribute__(self, "_raw")
        if raw is not None:
            if isinstance(raw, dict):
                if k in raw:
                    return True, raw[k]
            else:
                try:
                    if k in raw:                      # DictConfig supports `in`
                        return True, raw[k]
                except TypeError:
                    pass
                if hasattr(raw, k):
                    return True, getattr(raw, k)
        return False, None

    def __getattr__(self, k: str):
        ok, v = self._lookup(k)
        if ok:
            return v
        if k in TRAIN_DEFAULTS:
            return TRAIN_DEFAULTS[k]
        raise AttributeError(f"training args have no key {k!r}")

    def __setattr__(self, k, v):
        raw = object.__getattribute__(self, "_raw")
        if isinstance(raw, dict):
            raw[k] = v
        else:
            setattr(raw, k, v)

    def to_dict(self) -> Dict[str, Any]:
        raw = object.__getattribute__(self, "_raw")
        d = dict(TRAIN_DEFAULTS)
        d.update(to_container(raw) if raw is not None else {})
        return d


class _InFlight:
    __slots__ = ("plan", "done_evt", "local_count")

    def __init__(self, plan: RoundPlan, done_evt, local_count: int):
        self.plan, self.done_evt, self.local_count = plan, done_evt, local_count

    def done(self) -> bool:
        return True if self.done_evt is None else bool(self.done_evt.query())

    def wait_host(self) -> None:
        if self.done_evt is not None:
            self.done_evt.synchronize()


class DecoupledTrainer:
    """The 'Decoupled Trainer' with sharded optimizer (ACCO, DPU and synchronous DDP modes)."""

    # ================================================================== construction
    def __init__(self, model: nn.Module = None, tokenizer=None, train_dataset=None, eval_dataset=None, args=None,
                 log=None, text_column_name: str = "text", preprocess_dataset_fn: Optional[Callable] = None,
                 run_name: str = "", env: Optional[DistEnv] = None, teacher: Optional[nn.Module] = None,
                 reference: Optional[nn.Module] = None):
        self.model, self.tokenizer = model, tokenizer
        self.train_dataset, self.eval_dataset = train_dataset, eval_dataset
        self.raw_args = args
        self.args = _Args(args)
        self.log = log or logging.getLogger("acco_b200")
        self.text_column_name = text_column_name
        self.preprocess_dataset_fn = preprocess_dataset_fn
        self.run_name = run_name
        self.batch_size = int(self.args.batch_size)
        self.nb_grad_tot = int(self.args.nb_steps_tot)
        self.label_smoothing_factor = self.args.label_smoothing_factor
        self.label_smoother = LabelSmoother(self.label_smoothing_factor) if self.label_smoothing_factor else None
        self.epoch = 0
        self.method = str(self.args.method_name)
        if self.method not in ("acco", "dpu", "ddp"):
            raise ValueError("You must select one of the following method_name: 'acco', 'ddp', 'dpu'")
        self.max_grad_norm = check_max_grad_norm(self.args.max_grad_norm)
        self._grad_norm: Optional[float] = None     # pre-clip norm of the last committed round (max_grad_norm set)
        self._check_fp8()
        self._check_grad_accum_dtype()
        self._fused_smoothing = self._check_label_smoothing()
        self.z_loss_weight = self._check_z_loss()
        teacher_src = self._check_distill(teacher)
        self.pref_objective = self._check_simpo_orpo(reference, teacher_src is not None)
        reference_src = self._check_dpo(reference, teacher_src is not None)
        if not isinstance(self.args.no_decay_1d, bool):
            raise ValueError(f"no_decay_1d must be true or false, got {self.args.no_decay_1d!r}")
        self.no_decay_1d = self.args.no_decay_1d

        self.initialize_com(env)
        self.teacher = self._setup_frozen(teacher_src, "distillation teacher", "student")
        self.reference = self._setup_frozen(reference_src, "DPO reference", "policy")
        if self.teacher is not None and self.rank == 0:
            self.log.info(f">>> distillation: alpha={self.model.distill_alpha}, temperature={self.model.distill_temperature} "
                          f"(eval stays pure cross-entropy)")
        if self.reference is not None and self.rank == 0:
            self.log.info(f">>> DPO: beta={self.model.dpo_beta} on preference pairs, {self.batch_size} pairs = {2 * self.batch_size} rows "
                          f"per micro-batch (eval reports the same objective)")
        if self.pref_objective is not None and self.rank == 0:
            hp = f"beta={self.model.simpo_beta}, gamma={self.model.simpo_gamma}" if self.pref_objective == "simpo" else \
                f"lambda={self.model.orpo_lambda}"
            self.log.info(f">>> {self.pref_objective.upper()}: {hp} on preference pairs, no reference model, {self.batch_size} pairs = "
                          f"{2 * self.batch_size} rows per micro-batch (eval reports the same objective)")
        if self._fused_smoothing and self.rank == 0:
            self.log.info(f">>> label_smoothing_factor={self._fused_smoothing}: smoothed inside the fused cross-entropy kernel "
                          f"of {type(self.model).__name__} (CUDA graphs stay available)")
        if self.z_loss_weight and self.rank == 0:
            self.log.info(f">>> z_loss_weight={self.z_loss_weight}: z-loss inside the fused cross-entropy kernel of "
                          f"{type(self.model).__name__} on every training micro-batch (eval stays pure cross-entropy)")
        self._init_writer()
        self.prepare_data()
        self._tokenize_if_needed()
        self.train_dataloader = self.get_train_dataloader()
        self.eval_dataloader = self.get_eval_dataloader() if self.eval_dataset is not None else None
        self._feeder: Optional[DeviceFeeder] = None
        self.loss_static = torch.zeros(1, device=self.device, dtype=torch.float32)
        self.loss_host = torch.zeros(1, dtype=torch.float32)
        if self.is_cuda:
            self.loss_host = self.loss_host.pin_memory()
        # z_loss_weight > 0: the cross-entropy writes each micro-batch's mean z-term here on the device (also under graph replay);
        # it is copied to the host with the loss
        self.z_loss_static = torch.zeros(1, device=self.device, dtype=torch.float32)
        self.z_loss_host = torch.zeros(1, dtype=torch.float32)
        if self.is_cuda:
            self.z_loss_host = self.z_loss_host.pin_memory()
        if self.z_loss_weight:
            self.model.z_loss_out = self.z_loss_static
        # distillation: each micro-batch's mean CE and mean KL, written on the device like the z-term
        self.distill_static = torch.zeros(2, device=self.device, dtype=torch.float32)
        self.distill_host = torch.zeros(2, dtype=torch.float32)
        if self.is_cuda:
            self.distill_host = self.distill_host.pin_memory()
        if self.teacher is not None:
            self.model.distill_out = self.distill_static
        # DPO: each micro-batch's mean chosen reward, mean rejected reward and accuracy, written on the device like the z-term
        self.dpo_static = torch.zeros(3, device=self.device, dtype=torch.float32)
        self.dpo_host = torch.zeros(3, dtype=torch.float32)
        if self.is_cuda:
            self.dpo_host = self.dpo_host.pin_memory()
        if self.reference is not None:
            self.model.dpo_out = self.dpo_static
        self.eval_dpo_accuracy: Optional[float] = None
        # SimPO / ORPO: each micro-batch's three logged means (PREF_SCALARS), written on the device like the z-term
        self.pref_static = torch.zeros(3, device=self.device, dtype=torch.float32)
        self.pref_host = torch.zeros(3, dtype=torch.float32)
        if self.is_cuda:
            self.pref_host = self.pref_host.pin_memory()
        if self.pref_objective is not None:
            self.model.pref_out = self.pref_static
        self.eval_pref_accuracy: Optional[float] = None
        self.n_grad_acc_ddp = 1
        self._hook_extra_microbatches: Optional[Callable[[int, int], int]] = None   # tests: (rank, round) -> extra
        self._nvtx = os.environ.get("ACCO_NVTX") == "1"
        self._debug_poison = bool(self.args.debug_poison) or os.environ.get("ACCO_DEBUG_POISON") == "1"
        self._graphs: Optional[MicroBatchGraphs] = None
        self.input_override: Optional[Callable[[], Dict[str, torch.Tensor]]] = None   # e.g. device-resident batches
        self.micro_batches = 0
        self._tokens_seen = 0
        self._data_batches_base = 0     # batches of the data stream consumed before this process started (resume)
        self._stop_requested = False    # set by the pre-emption signal handler
        self.callbacks: List[Any] = []  # acco_b200.callbacks.TrainerCallback objects (`add_callback`)
        self._stopped = False           # a pre-emption checkpoint has been written: leave the training loop
        self.stats: Dict[str, Any] = {}
        if self.method == "ddp" and str(self.args.ddp_impl) == "torch":
            self.prepare_ddp()
        else:
            self.prepare_opt()
        if self.args.resume_from:
            ckpt = self._resolve_resume(str(self.args.resume_from))
            if ckpt:
                self.load_checkpoint(ckpt)

    # ------------------------------------------------------------------ process group / weights
    def initialize_com(self, env: Optional[DistEnv] = None) -> None:
        """Rank discovery, device placement, flat arena, weight init sync
        (`trainer_base.py:135-180`)."""
        env = init_distributed(env or discover_env())
        self.env = env
        self.rank, self.local_rank, self.world_size = env.rank, env.local_rank, env.world_size
        self.node_id, self.n_nodes, self.id_run = env.node_id, env.n_nodes, str(env.id_run)
        self.is_cuda = torch.cuda.is_available()
        self.device = torch.device("cuda", self.local_rank) if self.is_cuda else torch.device("cpu")
        if self.rank == 0:
            self.log.info(f">>> Training on {self.n_nodes} nodes and {self.world_size} {'GPUs' if self.is_cuda else 'CPU ranks'}")
        self.log.info("- Process {} corresponds to {} {} of node {}".format(
            self.rank, "GPU" if self.is_cuda else "CPU rank", self.local_rank, self.node_id))
        mixed = bool(self.args.use_mixed_precision)
        self.dtype = torch.bfloat16 if mixed else torch.float32          # compute (autocast) dtype
        fp32_weights = (not mixed) or (self.method == "ddp" and (bool(self.args.run_baseline_ddp) and str(self.args.ddp_weights_dtype) == "fp32"))
        self.param_dtype = torch.float32 if fp32_weights else torch.bfloat16
        self.autocast = mixed and self.param_dtype == torch.float32
        if self.args.seed is not None:
            from .utils.misc import seed_everything
            seed_everything(int(self.args.seed) + 0)
        if self.is_cuda and os.environ.get("ACCO_CARVEOUT_ALL") == "1":
            # experimental: every kernel of this process defaults to the GEMMs' L1 / shared split (co-residency with the round kernel)
            from . import ops
            rc = ops.load_ext(required=True).prefer_shared_carveout()
            self.log.info(f"ACCO_CARVEOUT_ALL=1: cudaDeviceSetCacheConfig(PreferShared) -> {rc}")
        self.model.to(device=self.device, dtype=self.param_dtype)
        torch_ddp = self.method == "ddp" and str(self.args.ddp_impl) == "torch"
        want = "nccl" if torch_ddp else str(self.args.comm_backend)
        if want == "auto" and self.n_nodes > 1:
            want = "nccl"       # peer-mapped symmetric memory / NVLS multicast exist only inside one NVSwitch domain
        self.backend: CommBackend = make_backend(want, self.rank, self.world_size, self.device, n_nodes=self.n_nodes)
        if self.rank == 0:
            self.log.info(f">>> communication backend: {self.backend.name} (requested {str(self.args.comm_backend)!r})")
        fp32_acc = self.args.grad_accum_dtype == "fp32" and self.param_dtype == torch.bfloat16
        self.arena = FlatArena(self.model, self.world_size, self.rank, self.param_dtype, self.device,
                               align=self.backend.slice_alignment(), allocator=self.backend.allocator(),
                               double_buffer=not torch_ddp, grad_dtype=torch.float32 if fp32_acc else None)
        self.len_params = self.arena.numel
        self.size_slice = self.arena.layout.size_slice
        self.size_local_slice = self.arena.layout.size_local_slice(self.rank)
        self.log.info(f"Worker {self.rank} training {self.len_params} parameters")
        with torch.no_grad():
            self.backend.init_sync(self.arena.theta[0], str(self.args.init_sync))
            for t in self.arena.theta[1:]:
                t.copy_(self.arena.theta[0])
        self.process_group = dist.group.WORLD if dist.is_initialized() else None

    @property
    def params(self) -> torch.Tensor:
        """Live flat parameter vector (``self.params`` of the reference)."""
        return self.arena.params_flat

    # ---- read-only views under the reference's attribute names (`trainer_decoupled.py:170-315`), for code that inspects a trainer.
    # The thread machinery (`com_event`, `update_event`, `com_finished`) and `com_buffer` have no counterpart: there is no
    # communication thread and no staging buffer.
    @property
    def scheduler(self):
        """LR schedule object (`trainer_decoupled.py:310-315` builds an HF scheduler); ``get_last_lr()`` like torch schedulers."""
        sch = self.lr_schedule
        if not hasattr(sch, "get_last_lr"):
            sch.get_last_lr = lambda: [float(getattr(self, "_last_lr", sch.lr_at(self.sched)))]
        return sch

    @property
    def count_grad_local(self) -> int:
        """Micro-batch gradients accumulated by this rank since the last flip (`trainer_decoupled.py:437-441`)."""
        return int(getattr(self, "_local_count", 0))

    @property
    def count_grad_this_round(self) -> int:
        """This rank's contribution to the round in flight / last launched (`trainer_decoupled.py:269`)."""
        hist = getattr(self, "round_history", None)
        return int(hist[-1][2]) if hist else 0

    @property
    def master_addr(self) -> str:
        return str(self.env.master_addr)

    @property
    def master_port(self) -> int:
        return int(self.env.master_port)

    @property
    def train_iterator(self):
        """Endless iterator over device-resident training batches (`trainer_decoupled.py:386-397`)."""
        return self._feed()

    def _init_writer(self) -> None:
        tb_dir = os.path.join(os.getcwd(), "tensorboard", str(self.run_name), str(self.id_run))
        self.writer = ScalarWriter(tb_dir, enabled=(self.rank == 0 and bool(self.args.tensorboard)))

    # ------------------------------------------------------------------ data
    def _check_packing(self) -> None:
        """``packing`` needs ragged SFT samples, a fixed row order and a model that masks attention by ``position_ids``."""
        a = self.args
        if not a.packing:
            return
        if a.const_len_batch:
            raise ValueError("packing=True needs const_len_batch=False: const-len pre-training rows are already full")
        if a.group_by_length:
            raise ValueError("packing=True cannot be combined with group_by_length: packed rows all have max_length tokens")
        from .models import NativeCausalLM
        if not isinstance(self.model, NativeCausalLM):
            raise ValueError(f"packing=True needs a native model that masks attention by position_ids; {type(self.model).__name__} "
                             "would attend across the samples of a row")

    def _check_document_mask(self) -> None:
        """``document_mask`` needs const-len rows, a model that masks attention by ``position_ids`` and the EOS id the rows were
        packed with (``DocumentCollator`` finds the documents from it)."""
        a = self.args
        if not isinstance(a.document_mask, bool):
            raise ValueError(f"document_mask must be true or false, got {a.document_mask!r}")
        if not a.document_mask:
            return
        if not a.const_len_batch:
            raise ValueError("document_mask=True needs const_len_batch=True: padded SFT rows hold one sample each, and packed SFT rows "
                             "(packing=True) are already document-masked")
        from .models import NativeCausalLM
        if not isinstance(self.model, NativeCausalLM):
            raise ValueError(f"document_mask=True needs a native model that masks attention by position_ids; {type(self.model).__name__} "
                             "would attend across the documents of a row")
        eos = getattr(self.tokenizer, "eos_token_id", None)
        if isinstance(eos, bool) or not isinstance(eos, numbers.Integral):
            raise ValueError(f"document_mask=True needs a tokenizer with an integer eos_token_id (the token the rows were packed with), "
                             f"got {eos!r}")

    def _check_fp8(self) -> None:
        """``fp8``: the native models' block linears run their training GEMMs in FP8 on bf16 weights and gradients."""
        a = self.args
        if not a.fp8:
            return
        from .models import NativeCausalLM
        if not isinstance(self.model, NativeCausalLM):
            raise ValueError(f"fp8=True needs a native model (LlamaForCausalLM / GPTForCausalLM); {type(self.model).__name__} has no FP8 path")
        if not a.use_mixed_precision or str(a.ddp_weights_dtype) == "fp32":
            raise ValueError("fp8=True quantises bf16 weights and activations: it needs use_mixed_precision=True and ddp_weights_dtype=bf16")
        if a.fused_ag_gemm:
            raise ValueError("fp8=True cannot be combined with fused_ag_gemm: the gathering GEMM has no FP8 instantiation")
        self.model.fp8 = True

    def _check_grad_accum_dtype(self) -> None:
        """``grad_accum_dtype``: None keeps the accumulators in the weights' dtype; "fp32" sums every micro-batch's gradient into fp32
        accumulators (no rounding to bf16 per micro-batch), which only the native models' ops can add into (``p.main_grad``)."""
        a = self.args
        v = a.grad_accum_dtype
        if v is None:
            return
        if v != "fp32":
            raise ValueError(f"grad_accum_dtype must be null or 'fp32', got {v!r}")
        from .models import NativeCausalLM
        if not isinstance(self.model, NativeCausalLM):
            raise ValueError(f"grad_accum_dtype=fp32 needs a native model (LlamaForCausalLM / GPTForCausalLM); {type(self.model).__name__}'s "
                             "backward writes autograd's .grad, which must have the bf16 weights' dtype")
        if self.method == "ddp" and str(a.ddp_impl) == "torch":
            raise ValueError("grad_accum_dtype=fp32 cannot be combined with ddp_impl=torch: its gradient buckets take the parameters' dtype")

    def _check_label_smoothing(self) -> float:
        """``label_smoothing_factor`` on a native model is applied by its fused cross-entropy kernel (``model.label_smoothing``):
        the micro-batch keeps the ``model(..., labels=...)`` path, with no fp32 copy of the logits and CUDA graphs available.
        Every other model keeps :class:`LabelSmoother` on its logits.  Returns the factor the native model smooths with (0 if none)."""
        eps = self.label_smoothing_factor
        from .models import NativeCausalLM
        if not eps or not isinstance(self.model, NativeCausalLM):
            return 0.0
        if isinstance(eps, bool) or not isinstance(eps, (int, float)) or not math.isfinite(eps) or not 0.0 <= eps <= 1.0:
            raise ValueError(f"label_smoothing_factor must be a finite number in [0, 1], got {eps!r}")
        self.model.label_smoothing = float(eps)
        self.label_smoother = None
        return float(eps)

    def _check_z_loss(self) -> float:
        """``z_loss_weight``: the native models add ``z * lse^2`` per non-ignored row inside their fused cross-entropy
        (``model.z_loss_weight``); there is no route for other models.  Returns the weight (0 if off)."""
        z = self.args.z_loss_weight
        if isinstance(z, bool) or not isinstance(z, (int, float)) or not math.isfinite(z) or z < 0:
            raise ValueError(f"z_loss_weight must be a finite number >= 0, got {z!r}")
        if not z:
            return 0.0
        from .models import NativeCausalLM
        if not isinstance(self.model, NativeCausalLM):
            raise ValueError(f"z_loss_weight > 0 needs a native model (LlamaForCausalLM / GPTForCausalLM): the term is computed inside "
                             f"their fused cross-entropy kernel, and {type(self.model).__name__} has no such loss")
        self.model.z_loss_weight = float(z)
        return float(z)

    def _check_distill(self, teacher: Optional[nn.Module]):
        """Validates the distillation keys and returns the teacher source: the ``teacher`` module, the ``distill_teacher``
        checkpoint directory, or None (off).  The student must be native; label smoothing and the z-loss are not combined with it."""
        a = self.args
        path = a.distill_teacher
        if teacher is not None and path is not None:
            raise ValueError("give the distillation teacher either as the trainer's teacher= argument or as distill_teacher, not both")
        src = teacher if teacher is not None else path
        if src is None:
            return None
        if path is not None and not isinstance(path, (str, os.PathLike)):
            raise ValueError(f"distill_teacher must be a checkpoint directory, got {path!r}")
        alpha, temp = a.distill_alpha, a.distill_temperature
        if isinstance(alpha, bool) or not isinstance(alpha, (int, float)) or not math.isfinite(alpha) or not 0.0 < alpha <= 1.0:
            raise ValueError(f"distill_alpha must be a number in (0, 1], got {alpha!r}")
        if isinstance(temp, bool) or not isinstance(temp, (int, float)) or not math.isfinite(temp) or not temp > 0.0:
            raise ValueError(f"distill_temperature must be a finite number > 0, got {temp!r}")
        from .models import NativeCausalLM
        if not isinstance(self.model, NativeCausalLM):
            raise ValueError(f"distillation needs a native student (LlamaForCausalLM / GPTForCausalLM): the loss is computed inside "
                             f"their fused kernels, and {type(self.model).__name__} has no such loss")
        if self.label_smoothing_factor or self.z_loss_weight:
            raise ValueError("distillation cannot be combined with label_smoothing_factor > 0 or z_loss_weight > 0")
        if teacher is self.model:
            raise ValueError("the distillation teacher must be a separate model from the student")
        self.model.distill_alpha, self.model.distill_temperature = float(alpha), float(temp)
        return src

    def _check_dpo(self, reference: Optional[nn.Module], distilling: bool):
        """Validates ``dpo_beta`` and returns the reference source: the ``reference`` module, the ``dpo_reference`` checkpoint directory,
        or None (off).  The policy must be native, the data preference pairs (checked in :meth:`_tokenize_if_needed`), and no other
        loss option may be on."""
        a = self.args
        beta, path = a.dpo_beta, a.dpo_reference
        if beta is None:
            if reference is not None:
                raise ValueError("a DPO reference= was given without dpo_beta")
            return None
        if isinstance(beta, bool) or not isinstance(beta, (int, float)) or not math.isfinite(beta) or not beta > 0.0:
            raise ValueError(f"dpo_beta must be a finite number > 0, got {beta!r}")
        if reference is not None and path is not None:
            raise ValueError("give the DPO reference either as the trainer's reference= argument or as dpo_reference, not both")
        src = reference if reference is not None else path
        if src is None:
            raise ValueError("dpo_beta needs a frozen reference model: set dpo_reference (an HF checkpoint dir) or pass reference=")
        if path is not None and not isinstance(path, (str, os.PathLike)):
            raise ValueError(f"dpo_reference must be a checkpoint directory, got {path!r}")
        from .models import NativeCausalLM
        if not isinstance(self.model, NativeCausalLM):
            raise ValueError(f"DPO needs a native policy (LlamaForCausalLM / GPTForCausalLM): the loss is computed inside their fused "
                             f"kernels, and {type(self.model).__name__} has no such loss")
        if distilling:
            raise ValueError("dpo_beta cannot be combined with distill_teacher: at most one frozen model trains alongside the policy")
        for key, on in (("label_smoothing_factor > 0", self.label_smoothing_factor), ("z_loss_weight > 0", self.z_loss_weight),
                        ("packing", a.packing), ("document_mask", a.document_mask), ("const_len_batch", a.const_len_batch)):
            if on:
                raise ValueError(f"dpo_beta cannot be combined with {key}: DPO trains on padded preference pairs, one sample per row, "
                                 f"with its own loss")
        if reference is self.model:
            raise ValueError("the DPO reference must be a separate model from the policy")
        self.model.dpo_beta = float(beta)
        return src

    def _check_simpo_orpo(self, reference: Optional[nn.Module], distilling: bool) -> Optional[str]:
        """Validates ``simpo_beta`` / ``simpo_gamma`` / ``orpo_lambda`` and returns the objective that is on ("simpo", "orpo") or None.
        Like DPO it needs a native policy and preference pairs (checked in :meth:`_tokenize_if_needed`) and no other loss option; it
        needs no reference, so a reference given with it is rejected."""
        a = self.args
        on = {k: getattr(a, k) for k in ("simpo_beta", "orpo_lambda") if getattr(a, k) is not None}
        if not on:
            return None
        for key, v in on.items():
            if isinstance(v, bool) or not isinstance(v, (int, float)) or not math.isfinite(v) or not v > 0.0:
                raise ValueError(f"{key} must be a finite number > 0, got {v!r}")
        gamma = a.simpo_gamma
        if "simpo_beta" in on and (isinstance(gamma, bool) or not isinstance(gamma, (int, float)) or not math.isfinite(gamma) or gamma < 0.0):
            raise ValueError(f"simpo_gamma must be a finite number >= 0, got {gamma!r}")
        others = [k for k, v in (("dpo_beta", a.dpo_beta), ("distill_teacher", distilling)) if v is not None and v is not False]
        if len(on) + len(others) > 1:
            raise ValueError(f"at most one of dpo_beta, simpo_beta, orpo_lambda and distill_teacher may be set, got {sorted(on) + others}")
        key = next(iter(on))
        if reference is not None or a.dpo_reference is not None:
            raise ValueError(f"{key} is reference-free: a reference= model or dpo_reference is meaningless with it")
        from .models import NativeCausalLM
        if not isinstance(self.model, NativeCausalLM):
            raise ValueError(f"{key} needs a native policy (LlamaForCausalLM / GPTForCausalLM): the loss is computed inside their fused "
                             f"kernels, and {type(self.model).__name__} has no such loss")
        for what, v in (("label_smoothing_factor > 0", self.label_smoothing_factor), ("z_loss_weight > 0", self.z_loss_weight),
                        ("packing", a.packing), ("document_mask", a.document_mask), ("const_len_batch", a.const_len_batch)):
            if v:
                raise ValueError(f"{key} cannot be combined with {what}: it trains on padded preference pairs, one sample per row, "
                                 f"with its own loss")
        if key == "simpo_beta":
            self.model.simpo_beta, self.model.simpo_gamma, self.model.orpo_lambda = float(on[key]), float(gamma), None
            return "simpo"
        self.model.simpo_beta, self.model.orpo_lambda = None, float(on[key])
        return "orpo"

    @property
    def _preference_key(self) -> Optional[str]:
        """The key of the preference objective that is on (its data are preference pairs), or None."""
        if self.args.dpo_beta is not None:
            return "dpo_beta"
        return {"simpo": "simpo_beta", "orpo": "orpo_lambda"}.get(self.pref_objective)

    def _setup_frozen(self, src, role: str, trained: str) -> Optional[nn.Module]:
        """The frozen ``role`` model (distillation teacher or DPO reference) on this rank's device in the trained model's weight dtype (a
        full copy per rank).  It is held by the trainer only, never by the trained model, so its parameters stay out of the arena,
        ``parameters()`` and the checkpoints."""
        if src is None:
            return None
        from .models import NativeCausalLM, from_pretrained
        frozen = from_pretrained(str(src), device=self.device, dtype=self.param_dtype, native=True) if not isinstance(src, nn.Module) else src
        if not isinstance(frozen, NativeCausalLM):
            raise ValueError(f"the {role} must be a native model (LlamaForCausalLM / GPTForCausalLM), got {type(frozen).__name__}")
        if frozen.config.vocab_size != self.model.config.vocab_size or frozen.config.padded_vocab != self.model.config.padded_vocab:
            raise ValueError(f"{role} and {trained} vocabularies differ: {frozen.config.vocab_size} (padded {frozen.config.padded_vocab}) vs "
                             f"{self.model.config.vocab_size} (padded {self.model.config.padded_vocab})")
        frozen.to(device=self.device, dtype=self.param_dtype)
        frozen.requires_grad_(False)
        frozen.eval()
        if self.rank == 0:
            n = sum(p.numel() for p in frozen.parameters())
            self.log.info(f">>> {role}: {type(frozen).__name__} ({n / 1e6:.1f}M parameters, frozen, one copy per rank)")
        return frozen

    def prepare_data(self) -> None:
        """Per-rank sharding (`trainer_base.py:183-200`)."""
        self._check_packing()
        self._check_document_mask()
        if self.train_dataset is not None and isinstance(self.train_dataset, torch.utils.data.IterableDataset) \
                and self.args.group_by_length:
            raise ValueError("the `--group_by_length` option is only available for `Dataset`, not `IterableDataset")
        if self.train_dataset is not None:
            self.train_dataset = self.train_dataset.shard(num_shards=self.world_size, index=self.rank)
        if self.eval_dataset is not None:
            self.eval_dataset = self.eval_dataset.shard(num_shards=self.world_size, index=self.rank)

    def _tokenize_if_needed(self) -> None:
        a = self.args
        if self.preprocess_dataset_fn is not None:
            self.train_dataset = self.train_dataset.map(self.preprocess_dataset_fn, batched=True)
            if self.eval_dataset is not None:
                self.eval_dataset = self.eval_dataset.map(self.preprocess_dataset_fn, batched=True)
        if self.train_dataset is None:
            return
        if self._preference_key is not None:
            self.train_dataset = self._preference_pairs(self.train_dataset)
            if self.eval_dataset is not None:
                self.eval_dataset = self._preference_pairs(self.eval_dataset)
            return
        if "input_ids" in self.train_dataset.column_names:
            if a.packing and "doc_lens" not in self.train_dataset.column_names:
                L = int(a.max_length)
                self.train_dataset = self.train_dataset.map(lambda b: pack_sft(b["input_ids"], L), batched=True,
                                                            remove_columns=self.train_dataset.column_names)
                self._log_packing()
            return
        if self.tokenizer is None:
            raise ValueError("dataset has no 'input_ids' column and no tokenizer was given")
        mk = make_const_len_tokenize_fn if a.const_len_batch else make_truncate_tokenize_fn
        fn = mk(self.tokenizer, self.text_column_name, int(a.max_length))
        train_fn = make_packed_tokenize_fn(self.tokenizer, self.text_column_name, int(a.max_length)) if a.packing else fn
        nproc = int(a.dataloader_num_workers) or None
        self.train_dataset = self.train_dataset.map(train_fn, batched=True, remove_columns=self.train_dataset.column_names, num_proc=nproc)
        if self.eval_dataset is not None:       # eval stays padded: its loss and perplexity compare with unpacked runs
            self.eval_dataset = self.eval_dataset.map(fn, batched=True, remove_columns=self.eval_dataset.column_names, num_proc=nproc)
        if a.packing:
            self._log_packing()

    def _preference_pairs(self, ds):
        """Preference data (DPO, SimPO, ORPO): token columns ``prompt_ids`` / ``chosen_ids`` / ``rejected_ids`` as they are, or TRL's
        ``prompt`` / ``chosen`` / ``rejected`` text columns tokenised; anything else is not preference data."""
        cols = set(ds.column_names)
        if set(PREFERENCE_COLUMNS) <= cols:
            return ds
        if not {"prompt", "chosen", "rejected"} <= cols:
            raise ValueError(f"{self._preference_key} needs preference pairs: columns prompt / chosen / rejected (text) or {' / '.join(PREFERENCE_COLUMNS)} "
                             f"(token ids), got {sorted(cols)}")
        if self.tokenizer is None:
            raise ValueError("the preference dataset has text columns and no tokenizer was given")
        nproc = int(self.args.dataloader_num_workers) or None
        return ds.map(make_preference_tokenize_fn(self.tokenizer), batched=True, remove_columns=ds.column_names, num_proc=nproc)

    def _log_packing(self) -> None:
        if self.rank != 0:
            return
        lens = self.train_dataset["doc_lens"]
        rows, samples, tokens = len(lens), sum(len(r) for r in lens), sum(sum(r) for r in lens)
        eff = tokens / max(rows * int(self.args.max_length), 1)
        self.log.info(f">>> packing: {samples} samples in {rows} rows of {int(self.args.max_length)} tokens, "
                      f"efficiency {eff:.3f} (real tokens / processed tokens)")

    def _collator(self):
        if self.args.const_len_batch:
            return DocumentCollator(self.tokenizer.eos_token_id) if self.args.document_mask else stack_collate
        pad = getattr(self.tokenizer, "pad_token_id", None) if self.tokenizer is not None else None
        if pad is None:
            pad = getattr(self.tokenizer, "eos_token_id", 0) if self.tokenizer is not None else 0
        mult = self.args.pad_to_multiple_of
        if mult is None:
            mult = 64 if self.is_cuda else 1        # few distinct padded lengths -> one CUDA graph per length
            if self.is_cuda and os.environ.get("ACCO_ATTN", "").lower() == "own":
                mult = 128                          # the own attention kernels tile the sequence in blocks of 128
        if self._preference_key is not None:
            return PreferenceCollator(pad_token_id=pad, max_length=int(self.args.max_length), pad_to_multiple_of=int(mult))
        return PadCollator(pad_token_id=pad, max_length=int(self.args.max_length), pad_to_multiple_of=int(mult))

    def get_train_dataloader(self) -> Optional[BatchLoader]:
        if self.train_dataset is None:
            return None
        seed = (int(self.args.seed) if self.args.seed is not None else 0) * 1000 + self.rank
        grouped = bool(self.args.group_by_length) and not bool(self.args.const_len_batch)
        collate = self._collator()
        if self.args.packing:
            collate = PackedCollator(pad_token_id=collate.pad, max_length=int(self.args.max_length))
        return BatchLoader(self.train_dataset, self.batch_size, collate, shuffle=True, drop_last=True, seed=seed,
                           group_by_length=grouped)

    def get_eval_dataloader(self) -> Optional[BatchLoader]:
        if self.eval_dataset is None:
            return None
        return BatchLoader(self.eval_dataset, self.batch_size, self._collator(), shuffle=False, drop_last=True)

    def _feed(self) -> DeviceFeeder:
        if self._feeder is None:
            self._feeder = DeviceFeeder(self.train_dataloader, self.device, prefetch=4, pin=bool(self.args.dataloader_pin_memory),
                                        num_workers=int(self.args.dataloader_num_workers or 0),
                                        persistent_workers=bool(self.args.dataloader_persistent_workers))
        return self._feeder

    def load_next_batch_into_static_memory(self) -> Dict[str, torch.Tensor]:
        """Next training batch on the device (endless; epochs restart automatically,
        `trainer_decoupled.py:386-397`)."""
        return self._feed().next()

    # ------------------------------------------------------------------ optimizer / schedule
    def prepare_opt(self) -> None:
        """fp32 master shard + AdamW state + LR schedule (`trainer_decoupled.py:296-315`)."""
        a = self.args
        no_decay = self.arena.no_decay_ranges() if self.no_decay_1d else None
        if self.no_decay_1d and self.rank == 0:
            excluded = [p for p in self.arena.params if p.requires_grad and p.ndim <= 1]
            self.log.info(f">>> no_decay_1d: {len(excluded)} parameters ({sum(p.numel() for p in excluded)} elements, "
                          f"{len(no_decay)} ranges of the flat vector) are updated without weight decay")
        self.sharded_optimizer = ShardedAdamW(
            self.arena.shard(self.arena.theta[0]), lr=float(a.learning_rate),
            betas=(float(a.adam_beta1), float(a.adam_beta2)), eps=float(a.adam_eps), weight_decay=float(a.weight_decay),
            no_decay=no_decay, shard_base=self.rank * self.size_slice)
        self.params_opt = self.sharded_optimizer.master
        self.backend.attach(self.arena, self.sharded_optimizer, self.max_grad_norm)
        self._setup_fused_ag()
        self.lr_schedule = LRSchedule(float(a.learning_rate), str(a.scheduler_name), int(a.warmup), self.nb_grad_tot, str(a.lr_unit))
        n_warm = int(a.n_warmup_steps) if self.method in ("acco", "dpu") else 0
        self.sched = RoundScheduler(self.method, n_warmup_rounds=n_warm, reference_quirks=bool(a.reference_quirks))
        self._inflight: Optional[_InFlight] = None
        self._local_count = 0
        self.round_history: List = []      # (round index, kind, local micro-batch count) - the reference's `save_grad_acc` data
        self.overlap = OverlapMeter(enabled=self.is_cuda, keep_history=bool(self.args.save_com_logs))
        if self.is_cuda:
            lo, hi = torch.cuda.Stream.priority_range()
            self.com_stream = torch.cuda.Stream(device=self.device, priority=hi)
            self.grad_stream = torch.cuda.current_stream(self.device)
            self.end_of_grad = torch.cuda.Event()
        else:
            self.com_stream = self.grad_stream = self.end_of_grad = None

    # ------------------------------------------------------------------ fused all-gather + first-use GEMM (KERNEL B)
    def _setup_fused_ag(self) -> None:
        """``fused_ag_gemm``: the round kernel stops pushing the row-blocks of the model's GEMM weights; the first
        forward GEMM after every flip pulls them from their owners over NVLink inside the wgmma GEMM kernel."""
        self._ag_on = False
        self._ag_stale = [False, False]     # theta[i] was rewritten by a round and its remote row-blocks are not pulled yet
        from .parallel.symm import SymmBackend
        if not (bool(self.args.fused_ag_gemm) and isinstance(self.backend, SymmBackend) and self.world_size > 1
                and self.param_dtype == torch.bfloat16 and hasattr(self.model, "fused_ag_candidates")):
            return
        from .ops.gemm import fused_ag_tables
        bases = [self.backend.peer_bases("theta", i) for i in range(len(self.arena.theta))]
        table, ranges = fused_ag_tables(self.model, self.arena, bases, self.size_slice, self.rank, self.device)
        self.backend.set_pull_ranges(ranges)
        self.model._ag_table = table
        self._ag_on = bool(table)
        self.stats_fused_ag = {"weights": len(table), "pulled_elements": sum(b - a for a, b in ranges)}
        if self.rank == 0:
            total = sum(int(p.numel()) for p in self.model.fused_ag_candidates())
            pulled = self.stats_fused_ag["pulled_elements"]
            # tiles that straddle an ownership boundary (at most one per boundary and weight) stay on the push path: say so
            self.log.info(f">>> fused all-gather GEMM: {len(table)} weights, {pulled}/{total} elements ({100.0 * pulled / max(total, 1):.1f} %) "
                          f"pulled inside the first forward GEMM, the rest pushed by the round kernel")

    def _ensure_gathered(self) -> None:
        """Complete the local copy of every fused weight now (eval / checkpoint / end of run may come before the
        next training forward): a 128-row dummy GEMM per weight drives the in-kernel gather."""
        idx = self.arena.live
        if not (self._ag_on and self._ag_stale[idx]):
            return
        from .ops.gemm import gemm_tn_gather
        for p in self.model.fused_ag_candidates():
            e = self.model._ag_table.get(id(p))
            if e is None:
                continue
            x = torch.zeros(128, p.shape[1], dtype=torch.bfloat16, device=self.device)
            gemm_tn_gather(x, p.detach(), e[idx])
        self._ag_stale[idx] = False

    def prepare_ddp(self) -> None:
        """Literal torch baseline: ``DDP(model)`` + ``ZeroRedundancyOptimizer(AdamW)``
        (`trainer_decoupled.py:226-241`)."""
        from torch.distributed.optim import ZeroRedundancyOptimizer
        from torch.nn.parallel import DistributedDataParallel as DDP
        a = self.args
        self.ddp_model = DDP(self.model) if self.world_size > 1 or dist.is_initialized() else self.model
        params = list(self.ddp_model.parameters())
        if self.no_decay_1d:
            # the two groups of the sharded update: ndim <= 1 without weight decay, the rest with it
            excluded = [p for p in params if p.requires_grad and p.ndim <= 1]
            ids = {id(p) for p in excluded}
            params = [dict(params=[p for p in params if id(p) not in ids]), dict(params=excluded, weight_decay=0.0)]
            params = [g for g in params if g["params"]]
            if self.rank == 0:
                self.log.info(f">>> no_decay_1d: {len(excluded)} parameters ({sum(p.numel() for p in excluded)} elements) "
                              f"are updated without weight decay")
        self.optimizer = ZeroRedundancyOptimizer(
            params, optimizer_class=torch.optim.AdamW, lr=float(a.learning_rate),
            weight_decay=float(a.weight_decay), betas=(float(a.adam_beta1), float(a.adam_beta2))) \
            if dist.is_initialized() else torch.optim.AdamW(
            params, lr=float(a.learning_rate), weight_decay=float(a.weight_decay),
            betas=(float(a.adam_beta1), float(a.adam_beta2)))
        self.lr_schedule = LRSchedule(float(a.learning_rate), str(a.scheduler_name), int(a.warmup), self.nb_grad_tot, str(a.lr_unit))
        self.sched = RoundScheduler("ddp")
        self.overlap = OverlapMeter(enabled=False)

    # ================================================================== step primitives
    def _forward_loss(self, model: nn.Module, inputs: Dict[str, torch.Tensor], teacher: Optional[nn.Module] = None,
                      reference: Optional[nn.Module] = None) -> torch.Tensor:
        if self.label_smoother is not None and "labels" in inputs:
            return self.compute_loss(model, dict(inputs))
        if reference is not None:
            # the reference scores the same [2P, S] pair rows; its forward is captured with the policy's in one micro-batch graph
            with torch.no_grad():
                r_logits = reference.padded_logits(inputs["input_ids"])
            out = model(**inputs, reference_logits=r_logits)
        elif teacher is not None:
            # the teacher sees the same tokens and positions, so packed / document-masked rows are masked alike for both models
            with torch.no_grad():
                t_logits = teacher.padded_logits(inputs["input_ids"], inputs.get("position_ids"))
            labels = inputs["labels"] if "labels" in inputs else inputs["input_ids"]
            out = model(**{k: v for k, v in inputs.items() if k != "labels"}, labels=labels, teacher_logits=t_logits)
        elif self.pref_objective is not None:
            # SimPO / ORPO: the [2P, S] pair rows score themselves, no frozen model runs
            out = model(**inputs, preference_pairs=True)
        elif "labels" in inputs:
            out = model(**inputs)
        elif self._fused_smoothing:
            # a batch without labels is scored on its own tokens unsmoothed, as on the LabelSmoother route (it smooths labels only)
            self.model.label_smoothing = 0.0
            try:
                out = model(**inputs, labels=inputs["input_ids"])
            finally:
                self.model.label_smoothing = self._fused_smoothing
        else:
            out = model(**inputs, labels=inputs["input_ids"])
        return out["loss"] if isinstance(out, dict) else out[0]

    def _prepare_input(self, data):
        """Move a tensor - or every tensor inside nested dicts / lists / tuples - to this rank's device (`trainer_base.py:240-251`);
        non-tensors pass through.  The training loop itself feeds batches through :class:`DeviceFeeder` (pinned staging + a copy
        stream); this is the public helper for user code that builds its own batches."""
        from collections.abc import Mapping
        if isinstance(data, Mapping):
            return type(data)({k: self._prepare_input(v) for k, v in data.items()})
        if isinstance(data, (tuple, list)):
            return type(data)(self._prepare_input(v) for v in data)
        if isinstance(data, torch.Tensor):
            return data.to(device=self.device, non_blocking=True)
        return data

    def _prepare_inputs(self, inputs):
        return self._prepare_input(inputs)

    def compute_loss(self, model, inputs, return_outputs: bool = False):
        """Loss with optional label smoothing (`trainer_base.py:262-282`): through :class:`LabelSmoother`, or, for a native model,
        inside the model's fused cross-entropy (``model.label_smoothing``, set at construction)."""
        labels = inputs.pop("labels") if (self.label_smoother is not None and "labels" in inputs) else None
        outputs = model(**inputs)
        if labels is not None:
            loss = self.label_smoother(outputs, labels, shift_labels=True)
        else:
            loss = outputs["loss"] if isinstance(outputs, dict) else outputs[0]
        return (loss, outputs) if return_outputs else loss

    def _fwd_bwd(self, inputs: Dict[str, torch.Tensor], model: Optional[nn.Module] = None) -> torch.Tensor:
        """One micro-batch: forward, backward (accumulating into the bound accumulator), returns
        the detached un-scaled loss (`gradient_step`, `trainer_decoupled.py:18-39`)."""
        model = model or self.model
        ctx = torch.autocast(device_type=self.device.type, dtype=self.dtype) if self.autocast else contextlib.nullcontext()
        with ctx:
            frozen = self.teacher is not None or self.reference is not None
            loss = self._forward_loss(model, inputs, self.teacher, self.reference) if frozen else self._forward_loss(model, inputs)
            scaled = loss / self.n_grad_acc_ddp if self.n_grad_acc_ddp != 1 else loss
        scaled.backward()
        return loss.detach()

    def _use_graphs(self) -> bool:
        if getattr(self, "_graphs_disabled", None):
            return False
        static_shapes = bool(self.args.const_len_batch) or bool(self.args.packing) or (self.args.pad_to_multiple_of is None) \
            or int(self.args.pad_to_multiple_of) >= 32
        return bool(self.is_cuda and self.args.cuda_graphs and static_shapes and self.label_smoother is None
                    and os.environ.get("ACCO_NO_GRAPHS") != "1")

    def gradient_step(self, inputs: Optional[Dict[str, torch.Tensor]] = None) -> None:
        """Run one micro-batch on the compute stream (graph replay when shapes are static)."""
        if inputs is None and self.input_override is not None:
            inputs = self.input_override()
        self.micro_batches += 1
        pending = bool(getattr(self, "_ag_on", False) and self._ag_stale[self.arena.live])
        if getattr(self, "_ag_on", False):
            self.model._ag_idx, self.model._ag_pending = self.arena.live, pending
        host = None
        if self._use_graphs():
            host = inputs if inputs is not None else self._feed().next_host()
            key = (self.arena.live, self.arena.grad_idx, pending, MicroBatchGraphs.signature(host))
            if self._graphs is None:
                self._graphs = MicroBatchGraphs(lambda b: self._fwd_bwd(b), self.device)
            if not self._graphs.has(key) and not self._capture(key, host):
                inputs = host               # capture failed: run this very batch eagerly below, graphs stay off
        if self._use_graphs():
            loss = self._graphs.replay(key, host)
            self.loss_static.copy_(loss)
        else:
            dev = inputs if inputs is not None else self.load_next_batch_into_static_memory()
            dev = {k: v.to(self.device, non_blocking=True) for k, v in dev.items()}
            self.loss_static.copy_(self._fwd_bwd(dev).reshape(1))
        self._local_count += 1
        if pending:
            self._ag_stale[self.arena.live] = False     # the forward that just ran completed the local copies
        self._tokens_seen += int(self.batch_size) * int(self.args.max_length)   # upper bound for padded (SFT) batches
        if self.args.run_expe_slow and self.rank in tuple(self.args.slow_ranks or ()) and float(self.args.slow_factor_ms) > 0:
            if self.is_cuda:
                torch.cuda._sleep(int(float(self.args.slow_factor_ms) * 1.5e6))   # ~cycles at ~1.5 GHz
            else:
                time.sleep(float(self.args.slow_factor_ms) / 1e3)

    def _capture(self, key, example: Dict[str, torch.Tensor]) -> bool:
        """Capture the micro-batch graph for the currently bound (theta, acc) pair; the warm-up
        iterations really accumulate gradients, so the accumulator is saved and restored.  Models
        that cannot be captured (host syncs / data-dependent control flow in ``forward``) fall back
        to eager execution for the rest of the run."""
        acc = self.arena.acc[self.arena.grad_idx]
        saved = acc.clone()
        try:
            self._graphs.capture(key, example, cleanup=lambda: acc.copy_(saved))
            return True
        except Exception as e:      # noqa: BLE001 - any capture failure means "this model is not graph-safe"
            torch.cuda.synchronize(self.device)
            try:
                # an aborted capture leaves the device's default RNG generator flagged as "capturing" (every later CUDA RNG call -
                # dropout, randint - would raise "Offset increment outside graph capture"): swap in a clean copy of its state
                gen = torch.cuda.default_generators[self.device.index or 0]
                gen.graphsafe_set_state(gen.clone_state())
            except Exception:       # noqa: BLE001 - best effort, older torch
                pass
            acc.copy_(saved)
            self.arena.rebind()
            self._graphs_disabled = f"{type(e).__name__}: {str(e)[:200]}"
            self.log.warning(f"CUDA-graph capture of the micro-batch failed ({self._graphs_disabled}); continuing without graphs")
            return False
        finally:
            del saved

    # ================================================================== round machinery
    def _launch_round(self) -> None:
        plan = self.sched.next_plan()
        # host-side protocol assertions : the round must never consume the accumulator backward is
        # writing, nor overwrite the parameter buffer the model is bound to
        assert self._inflight is None, "a round is still in flight: complete it before launching the next one"
        if self._debug_poison:
            self._poison(plan)
        self.round_history.append((plan.index, plan.kind, int(self._local_count)))
        lr = self.lr_schedule.lr_at(self.sched)
        self._last_lr = lr
        if self.is_cuda:
            ready = torch.cuda.Event()
            ready.record(self.grad_stream)
            done = torch.cuda.Event()
            e0, e1 = self.overlap.comm_events()
            with torch.cuda.stream(self.com_stream):
                self.com_stream.wait_event(ready)
                if e0 is not None:
                    e0.record(self.com_stream)
                self.backend.launch_round(plan, lr, self._local_count)
                if e1 is not None:
                    e1.record(self.com_stream)
                done.record(self.com_stream)
        else:
            done = None
            self.backend.launch_round(plan, lr, self._local_count)
        self._inflight = _InFlight(plan, done, self._local_count)
        self._local_count = 0

    def _poison(self, plan: RoundPlan) -> None:
        """Debug mode: NaN-fill the shadow parameter buffer right before the round that rewrites ALL of it is enqueued (same stream,
        so the round's writes land after the poison).  Correct schedules never read that buffer while the round is in flight - if
        compute does (a wrong flip, a missing event wait), the NaNs reach the loss immediately instead of silently training on torn
        weights.  The reference's equivalent hazard is its unsynchronised `params <- com_buffer` copy ."""
        buf = self.arena.theta[plan.write_theta]
        if getattr(self, "_ag_on", False) or buf.data_ptr() == self.arena.theta[self.arena.live].data_ptr():
            return                      # fused-AG leaves pulled tiles to the next forward; single-buffer arenas have no shadow
        if self.is_cuda:
            with torch.cuda.stream(self.com_stream):
                self.com_stream.wait_stream(self.grad_stream)
                buf.fill_(float("nan"))
        else:
            buf.fill_(float("nan"))

    def _complete_round(self) -> RoundPlan:
        """Book-keeping for the finished in-flight round; makes compute wait on it (device side)."""
        fl = self._inflight
        if fl.done_evt is not None:
            if self.is_cuda:
                w0, w1 = self.overlap.wait_events()
                if w0 is not None:
                    w0.record(self.grad_stream)
                self.grad_stream.wait_event(fl.done_evt)
                if w1 is not None:
                    w1.record(self.grad_stream)
            fl.wait_host()          # already complete when reached through the poll; blocks in sync mode
        total = self.backend.finish_round(fl.plan)
        if self.max_grad_norm is not None and fl.plan.kind != "tentative":
            self._grad_norm = self.backend.last_grad_norm
        self.sched.complete(fl.plan, total)
        if getattr(self, "_ag_on", False):
            self._ag_stale[fl.plan.write_theta] = True   # fresh weights: remote row-blocks of the GEMM weights still on their owners
        self._inflight = None
        return fl.plan

    def _bind_compute_buffers(self) -> None:
        b = self.sched.compute_buffers(round_in_flight=self._inflight is not None)
        if self._inflight is not None:
            # host-side protocol assertions: never compute on the buffer the in-flight round is rewriting, never accumulate into the
            # accumulator it is consuming
            assert b["theta"] != self._inflight.plan.write_theta and b["acc"] != self._inflight.plan.read_acc, (b, self._inflight.plan)
        self.arena.point_params(b["theta"])
        self.arena.point_grads(b["acc"])

    def _accumulate_phase(self) -> None:
        """``n_grad_accumulation`` micro-batches (+ test-injected extras), then make the loss and the
        end-of-phase event visible to the host (`trainer_decoupled.py:481-495`)."""
        n = int(self.args.n_grad_accumulation)
        if self._hook_extra_microbatches is not None:
            n += int(self._hook_extra_microbatches(self.rank, self.sched.round))
        with nvtx_range(f"acco/phase r{self.sched.round}") if self._nvtx else contextlib.nullcontext():
            for _ in range(n):
                self.gradient_step()
        self._copy_scalars_to_host(non_blocking=self.is_cuda)
        if self.is_cuda:
            self.end_of_grad.record(self.grad_stream)
            self._poll_phase_end()

    def _copy_scalars_to_host(self, non_blocking: bool) -> None:
        """The loss and the loss options' logged device scalars -> their (pinned) host copies."""
        self.loss_host.copy_(self.loss_static, non_blocking=non_blocking)
        if self.z_loss_weight:
            self.z_loss_host.copy_(self.z_loss_static, non_blocking=non_blocking)
        if self.teacher is not None:
            self.distill_host.copy_(self.distill_static, non_blocking=non_blocking)
        if self.reference is not None:
            self.dpo_host.copy_(self.dpo_static, non_blocking=non_blocking)
        if self.pref_objective is not None:
            self.pref_host.copy_(self.pref_static, non_blocking=non_blocking)

    def _poll_phase_end(self) -> None:
        """The flip decision must be taken when the *device* reaches the end of the phase ("if the com finished ... else accumulate
        more", `trainer_decoupled.py:497`), so the host may not run ahead of it - but it does not block in the driver either: it polls
        the phase event (``cudaEventQuery``), yielding the core between polls, and the same loop notices the round event."""
        ev = self.end_of_grad
        spins = 0
        while not ev.query():
            spins += 1
            if spins > 200:                 # ~ the first 100 us are a pure spin (phases are milliseconds; launch jitter is microseconds)
                time.sleep(0)

    def _sync_round(self) -> RoundPlan:
        """accumulate -> round -> wait (DDP mode and the sequential warm-up rounds of ACCO/DPU,
        `trainer_decoupled.py:318-383`)."""
        self._bind_compute_buffers()
        self._accumulate_phase()
        self._launch_round()
        return self._complete_round()

    def warmup_steps(self, n_warmup_steps: int) -> None:
        """``n`` fully sequential sharded steps (no overlap)."""
        self.sched.warmup_left = max(self.sched.warmup_left, 0)
        for _ in range(int(n_warmup_steps)):
            if self.sched.warmup_left == 0:
                self.sched.warmup_left = 1
            self._sync_round()

    # ================================================================== training loops
    def train(self):
        self.t_beg = time.time()
        self.t_last_epoch = self.t_beg
        if self.method == "acco":
            return self.train_acco()
        if self.method == "ddp":
            return self.train_ddp()
        if self.method == "dpu":
            return self.train_dpu()
        raise ValueError("You must select one of the following method_name: 'acco', 'ddp', 'dpu'")

    def train_acco(self):
        return self._train_overlapped()

    def train_dpu(self):
        return self._train_overlapped()

    def _begin_run(self) -> None:
        if not hasattr(self, "t_beg"):
            self.t_beg = time.time()
        if not hasattr(self, "_log_state"):
            self._log_state = dict(last_eval=0, time_checkpoint=time.time(),
                                   printer=TrainingPrinter(self.log, self.rank, int(self.args.log_every)))
            if self.args.preempt_save:
                self._install_preempt_handler()
            self._fire("on_train_begin")

    def finished(self) -> bool:
        return self._stopped or self.sched.count_grad_tot >= self.nb_grad_tot

    def add_callback(self, callback) -> None:
        """Register a :class:`acco_b200.callbacks.TrainerCallback`."""
        self.callbacks.append(callback)

    def request_stop(self) -> None:
        """Leave the training loop after the current round (callbacks; every rank must call it at the same round)."""
        self._stopped = True

    def _fire(self, event: str, *args) -> None:
        for cb in self.callbacks:
            getattr(cb, event)(self, *args)

    def _install_preempt_handler(self) -> None:
        """``preempt_save``: a cluster scheduler announces pre-emption / the end of the allocation with a signal (Slurm: SIGTERM, or
        ``--signal=USR1@120``).  The handler only raises a flag; the training loop looks at it between rounds (`_tail`), where a
        consistent checkpoint can be written, and every rank stops after the same round."""
        import signal
        if threading.current_thread() is not threading.main_thread():
            return                                  # signal handlers can only be installed from the main thread

        def handler(signum, frame):
            self._stop_requested = True
            self.log.info(f"signal {signum} received: checkpoint + stop at the next committed round")

        for sig in (signal.SIGTERM, signal.SIGUSR1):
            signal.signal(sig, handler)

    def step(self) -> bool:
        """One scheduling iteration - the unit the training loops (and ``bench.py``) repeat.

        A *phase* of ``n_grad_accumulation`` micro-batches is enqueued on the buffers the scheduler
        names; then, if the in-flight communication round has finished (event poll - or nothing is
        in flight yet: priming), the round is completed and the next one launched ("flip").
        Otherwise the next call simply accumulates more micro-batches: *accumulate while you
        communicate* (`trainer_decoupled.py:481-520`).  Returns True when a flip happened."""
        self._begin_run()
        sched = self.sched
        if self.method == "ddp" or sched.in_warmup():
            plan = self._sync_round()
            self._tail(plan)
            return True
        self._bind_compute_buffers()
        self._accumulate_phase()
        if self._inflight is not None and bool(self.args.static_accumulation):
            self._inflight.wait_host()          # reproducible mode: exactly n_grad_accumulation micro-batches per round on every rank
        if self._inflight is None or self._inflight.done():
            if self._inflight is not None:
                plan = self._complete_round()
                if self.finished():
                    return True
                # eval / logs / checkpoints run HERE: the round that just finished has landed on every rank, nothing is in flight,
                # so neither the weights nor the optimizer shard can change under the reader
                self._tail(plan)
                if self._stopped:
                    return True
            self._launch_round()
            return True
        return False

    def _train_overlapped(self):
        """ACCO / DPU main loop (`trainer_decoupled.py:431-598`, `:605-730`)."""
        self._begin_run()
        while not self.finished():
            self.step()
        self._drain()
        return self._finish("")

    def train_ddp(self):
        """Synchronous data parallel + sharded optimizer (`trainer_decoupled.py:732-833`)."""
        self._begin_run()
        if str(self.args.ddp_impl) == "torch":
            return self._train_ddp_torch()
        while not self.finished():
            self.step()
        self._drain()
        return self._finish("_ddp")

    def _train_ddp_torch(self):
        a = self.args
        self.n_grad_acc_ddp = int(a.n_grad_accumulation)
        sched = self.sched
        while sched.count_grad_tot < self.nb_grad_tot:
            for _ in range(int(a.n_grad_accumulation)):
                dev = self.load_next_batch_into_static_memory()
                self.loss_static.copy_(self._fwd_bwd(dev, self.ddp_model).reshape(1))
            lr = self.lr_schedule.lr_at(sched)
            for g in self.optimizer.param_groups:
                g["lr"] = lr
            if self.max_grad_norm is not None:
                self._grad_norm = float(torch.nn.utils.clip_grad_norm_(self.ddp_model.parameters(), self.max_grad_norm))
            self.optimizer.step()
            self.optimizer.zero_grad(set_to_none=False)
            sched.round += 1
            sched.count_com += 1
            sched.opt_steps += 1
            sched.lr_steps += 1
            sched.count_grad_tot += self.world_size * int(a.n_grad_accumulation)
            self._copy_scalars_to_host(non_blocking=False)
            self._tail(None)
        return self._finish("_ddp")

    def align_rounds(self) -> None:
        """Collective: make every rank have launched the same number of rounds.  ``train()`` never needs this (ranks stop on
        the same global gradient count, hence after the same round); loops that run a fixed number of ``step()`` calls per
        rank on heterogeneous ranks do - a rank that stopped one round short would leave its peers' last round waiting forever."""
        if self.world_size == 1 or not hasattr(self, "sched") or not self.is_cuda:
            return
        target = int(self.backend.all_reduce_max(float(self.sched.round)))
        while self.sched.round < target:
            if self._inflight is not None:
                self._inflight.wait_host()
                self._complete_round()
            self._bind_compute_buffers()
            self._launch_round()

    def _drain(self) -> None:
        """Wait for the last round and leave the model on the newest weights."""
        if getattr(self, "_align_on_drain", False):
            self.align_rounds()
        if getattr(self, "_inflight", None) is not None:
            self._inflight.wait_host()
            self._complete_round()
        self._bind_compute_buffers()
        self._ensure_gathered()
        if self.is_cuda:
            torch.cuda.synchronize(self.device)

    # ------------------------------------------------------------------ tail of a round: eval / logs / checkpoints
    def _tail(self, plan: Optional[RoundPlan]) -> None:
        """Runs right after a round has completed and before the next one is launched (no communication in flight): the model is
        re-bound to the buffer that round wrote, so eval and checkpoints see one consistent set of weights (never a half-gathered
        buffer), and the optimizer shard is quiescent.  ACCO evaluates / saves only after *real* rounds - the buffer written by a
        tentative round holds the estimate theta~, not committed weights."""
        a, st, sched = self.args, self._log_state, self.sched
        committed = plan is None or self.method != "acco" or plan.kind != "tentative"
        if a.fault_inject:
            self._maybe_inject_fault(str(a.fault_inject))
        if hasattr(self, "arena") and plan is not None:
            self._bind_compute_buffers()                     # nothing in flight -> the newest buffer
        eval_loss = None
        if committed and a.eval and self.eval_dataset is not None and (self.rank == 0 or a.eval_all_ranks) \
                and sched.count_grad_tot - st["last_eval"] > int(a.eval_step):
            eval_loss = self.eval_loop()
            st["last_eval"] = sched.count_grad_tot
            if a.eval_all_ranks and self.world_size > 1:
                # every rank evaluated its own shard at the same round: report the mean (ranks whose shard is empty are skipped)
                from .utils.dist import reduce_mean
                eval_loss = torch.tensor(reduce_mean(float(eval_loss)))
            self._fire("on_evaluate", float(eval_loss))
        if self.rank == 0:
            pr: TrainingPrinter = st["printer"]
            if pr.due(sched.count_grad_tot) or eval_loss is not None:
                loss = float(self.loss_host.item())
                nb_step = sched.count_com // 2 if self.method == "acco" else sched.count_com
                gn = {} if self._grad_norm is None else {"grad_norm": self._grad_norm}
                if self.z_loss_weight:
                    gn["z_loss"] = float(self.z_loss_host.item())    # the loss's z-term: cross-entropy = loss - z_loss
                if self.teacher is not None:                          # loss = (1 - a) distill_ce + a T^2 distill_kl
                    gn["distill_ce"], gn["distill_kl"] = (float(v) for v in self.distill_host.tolist())
                if self.reference is not None:                        # loss = the DPO objective
                    gn["dpo_reward_chosen"], gn["dpo_reward_rejected"], gn["dpo_accuracy"] = (float(v) for v in self.dpo_host.tolist())
                    if eval_loss is not None and self.eval_dpo_accuracy is not None:
                        gn["eval_dpo_accuracy"] = self.eval_dpo_accuracy
                if self.pref_objective is not None:                   # loss = the SimPO / ORPO objective
                    names = PREF_SCALARS[self.pref_objective]
                    gn.update(zip(names, (float(v) for v in self.pref_host.tolist())))
                    if eval_loss is not None and self.eval_pref_accuracy is not None:
                        gn[f"eval_{names[2]}"] = self.eval_pref_accuracy
                log_training_scalars(self.writer, nb_step, sched.count_grad_tot, self.rank, loss, eval_loss, self.t_beg,
                                     extra={"lr": getattr(self, "_last_lr", 0.0), **gn})
                self._fire("on_log", {"step": nb_step, "count_grad_tot": sched.count_grad_tot, "loss": loss,
                                      "eval_loss": None if eval_loss is None else float(eval_loss), "lr": getattr(self, "_last_lr", 0.0), **gn})
                if pr.due(sched.count_grad_tot):
                    # same line as the reference (`utils/logs_utils.py:155-183`) + this rank's throughput since the previous line and the LR
                    now, seen = time.time(), self._tokens_seen
                    t0, n0 = st.get("rate_mark", (self.t_beg, 0))
                    st["rate_mark"] = (now, seen)
                    rate = (seen - n0) / max(now - t0, 1e-9)
                    gn_txt = "" if self._grad_norm is None else f" | grad_norm {self._grad_norm:.4g}"
                    if self.z_loss_weight:
                        gn_txt += f" | z_loss {gn['z_loss']:.4g}"
                    if self.teacher is not None:
                        gn_txt += f" | distill_ce {gn['distill_ce']:.4g} | distill_kl {gn['distill_kl']:.4g}"
                    if self.reference is not None:
                        gn_txt += (f" | dpo_reward_chosen {gn['dpo_reward_chosen']:.4g} | dpo_reward_rejected {gn['dpo_reward_rejected']:.4g}"
                                   f" | dpo_accuracy {gn['dpo_accuracy']:.3f}")
                    if self.pref_objective is not None:
                        c, r, acc = PREF_SCALARS[self.pref_objective]
                        gn_txt += f" | {c} {gn[c]:.4g} | {r} {gn[r]:.4g} | {acc} {gn[acc]:.3f}"
                    pr.emit(sched.count_grad_tot, sched.count_com, loss, extra=f" | {rate:,.0f} tok/s/rank | lr {getattr(self, '_last_lr', 0.0):.3e}{gn_txt}")
                self.epoch = pr.epoch
        if committed and plan is not None and self.callbacks:
            self._fire("on_round_end", plan)
        if a.preempt_save and committed:
            stop = self._stop_requested
            if self.world_size > 1:
                stop = bool(self.backend.all_reduce_max(1.0 if stop else 0.0) > 0.5)      # any rank's signal stops all of them, same round
            if stop:
                tag = {"acco": "_model_", "dpu": "_dpu_model_", "ddp": "_ddp_model_"}[self.method]
                path = os.path.join(os.getcwd(), "checkpoints", f"{self.id_run}{tag}{sched.count_grad_tot}.pt")
                if self.rank == 0 or (a.save_optimizer and hasattr(self, "sharded_optimizer")):
                    self.save_checkpoint(path)
                self.log.info(f"pre-empted: checkpoint {path} written at count_grad_tot={sched.count_grad_tot}; stopping")
                self._stopped = True
                return
        if a.save and committed:
            due = self.rank == 0 and time.time() - st["time_checkpoint"] >= float(a.save_interval_s)
            if a.save_optimizer and self.world_size > 1 and hasattr(self, "sharded_optimizer"):
                # every rank writes its optimizer shard: rank 0's clock decides for all (one tiny collective per committed round,
                # only in this opt-in mode)
                due = bool(self.backend.all_reduce_max(1.0 if due else 0.0) > 0.5)
            if due:
                st["time_checkpoint"] = time.time()
                tag = {"acco": "_model_", "dpu": "_dpu_model_", "ddp": "_ddp_model_"}[self.method]
                self.save_checkpoint(os.path.join(os.getcwd(), "checkpoints", f"{self.id_run}{tag}{sched.count_grad_tot}.pt"))
                if a.save_total_limit and (self.rank == 0 or a.save_optimizer):
                    from .checkpoint import prune_checkpoints
                    prune_checkpoints(os.path.join(os.getcwd(), "checkpoints"), f"{self.id_run}{tag}", int(a.save_total_limit), self.rank)

    def _maybe_inject_fault(self, spec: str) -> None:
        """Failure drill (the reference has no failure handling at all): ``fault_inject="rank@count"`` makes
        that rank die abruptly - no exception, no cleanup, like a lost GPU or an OOM-killed process - the first time the global
        gradient count reaches ``count``.  Its peers then fail in their next collective (NCCL / gloo error, or the signal-pad
        watchdog trap of the fused round kernel), the launcher restarts the group (``torchrun --max-restarts``) and
        ``resume_from=auto`` continues from the newest complete checkpoint.  A marker file makes the fault fire once."""
        rank_s, _, count_s = spec.partition("@")
        if int(rank_s) != self.rank or self.sched.count_grad_tot < int(count_s or 0):
            return
        marker = os.path.join(os.getcwd(), "fault_injected.marker")
        if os.path.exists(marker):
            return
        with open(marker, "w") as f:
            f.write(f"rank {self.rank} killed itself at count_grad_tot={self.sched.count_grad_tot}\n")
        self.log.info(f"fault_inject: rank {self.rank} exits now (count_grad_tot={self.sched.count_grad_tot})")
        logging.shutdown()
        os._exit(17)

    @torch.no_grad()
    def eval_loop(self) -> torch.Tensor:
        """Mean loss over this rank's eval shard (`trainer_decoupled.py:399-415`).  With DPO the loss is the DPO objective (reference
        forward included) and ``eval_dpo_accuracy`` the mean accuracy over the eval micro-batches; with SimPO / ORPO the loss is that
        objective and ``eval_simpo_accuracy`` / ``eval_orpo_accuracy`` (``eval_pref_accuracy``) its mean accuracy."""
        self._ensure_gathered()
        self.model.eval()
        losses: List[torch.Tensor] = []
        accs: List[torch.Tensor] = []
        if self.reference is not None:
            self.model.dpo_out = torch.zeros(3, device=self.device, dtype=torch.float32)   # the training scalars stay as logged
        if self.pref_objective is not None:
            self.model.pref_out = torch.zeros(3, device=self.device, dtype=torch.float32)  # likewise
        ctx = torch.autocast(device_type=self.device.type, dtype=self.dtype) if self.autocast else contextlib.nullcontext()
        if self.z_loss_weight:
            self.model.z_loss_weight = 0.0          # eval loss stays pure cross-entropy, comparable with runs without the key
        try:
            for i, inputs in enumerate(self.eval_dataloader):
                if self.args.max_eval_batches is not None and i >= int(self.args.max_eval_batches):
                    break
                inputs = {k: v.to(self.device, non_blocking=True) for k, v in inputs.items()}
                with ctx:
                    loss = self._forward_loss(self.model, inputs) if self.reference is None else \
                        self._forward_loss(self.model, inputs, reference=self.reference)
                    losses.append(loss.detach().float().reshape(1))
                if self.reference is not None:
                    accs.append(self.model.dpo_out[2:].clone())
                elif self.pref_objective is not None:
                    accs.append(self.model.pref_out[2:].clone())
        finally:
            if self.z_loss_weight:
                self.model.z_loss_weight = self.z_loss_weight
            if self.reference is not None:
                self.model.dpo_out = self.dpo_static
            if self.pref_objective is not None:
                self.model.pref_out = self.pref_static
        self.model.train()
        if not losses:
            return torch.tensor(float("nan"))
        mean = torch.cat(losses).mean().cpu()
        if accs and self.pref_objective is not None:
            self.eval_pref_accuracy = float(torch.cat(accs).mean())
            self.log.info(f"eval loss {float(mean):.4f} | eval {PREF_SCALARS[self.pref_objective][2]} {self.eval_pref_accuracy:.3f}")
        elif accs:
            self.eval_dpo_accuracy = float(torch.cat(accs).mean())
            self.log.info(f"eval loss {float(mean):.4f} | eval dpo_accuracy {self.eval_dpo_accuracy:.3f}")
        else:
            self.log.info(f"eval loss {float(mean):.4f}")
        return mean

    # ------------------------------------------------------------------ end of run
    def _finish(self, tag: str):
        total_time = time.time() - self.t_beg
        ov = self.overlap.summary()
        self.stats = {
            "total_time_s": total_time, "count_grad_tot": self.sched.count_grad_tot, "rounds": self.sched.count_com,
            "optimizer_steps": self.sched.opt_steps, "tokens_local": self._tokens_seen,
            # non-pad tokens this rank really consumed (attention-mask sums of the ragged SFT batches; == tokens_local for const-len)
            "tokens_real_local": (self._feeder.tokens_real if self._feeder is not None else self._tokens_seen),
            "tokens_per_s_local": self._tokens_seen / max(total_time, 1e-9),
            "real_tokens_per_s_local": (self._feeder.tokens_real if self._feeder is not None else self._tokens_seen) / max(total_time, 1e-9),
            "comm_ms_mean": ov["comm_ms_mean"],
            "exposed_comm_ms_per_round": ov["exposed_ms_mean"], "backend": self.backend.name,
        }
        cfg = getattr(self.model, "config", None)
        if hasattr(cfg, "flops_per_token"):
            self.stats["model_tflops_local"] = self.stats["tokens_per_s_local"] * cfg.flops_per_token(int(self.args.max_length)) / 1e12
        if self.rank == 0:
            row = create_dict_result(
                self.args.to_dict(), self.world_size, self.n_nodes,
                torch.cuda.get_device_name() if self.is_cuda else "cpu", total_time, self.id_run,
                float(self.loss_host.item()),
                extra={k: self.stats[k] for k in ("tokens_per_s_local", "comm_ms_mean", "exposed_comm_ms_per_round", "backend")})
            save_result(os.path.join(os.getcwd(), "results.csv"), row)
            self.writer.flush()
        if self.args.save and not self._stopped and (self.rank == 0 or (self.args.save_optimizer and hasattr(self, "sharded_optimizer"))):
            # reference file names: {id}_model.pt / {id}dpu_model.pt (sic) / {id}_ddp_model.pt; rank 0 writes the model, with
            # `save_optimizer` every rank adds its optimizer shard
            name = {"acco": f"{self.id_run}_model.pt", "dpu": f"{self.id_run}dpu_model.pt", "ddp": f"{self.id_run}_ddp_model.pt"}[self.method]
            self.save_checkpoint(os.path.join(os.getcwd(), "checkpoints", name))
        if self.args.save_com_logs and hasattr(self, "round_history"):
            # per-rank communication history (the reference's unused `save_com_logs`, utils/logs_utils.py:141): duration of every round on
            # the communication stream and the time compute really waited for it (CUDA events; empty lists on the CPU path)
            d = os.path.join(os.getcwd(), "com_logs")
            os.makedirs(d, exist_ok=True)
            with open(os.path.join(d, f"{self.id_run}_{self.rank}.txt"), "w") as f:
                f.write(f"{self.rank} rounds : {[k for _, k, _ in self.round_history]}\n")
                f.write(f"{self.rank} comm_ms : {[round(x, 4) for x in (self.overlap.comm_history or [])]}\n")
                f.write(f"{self.rank} exposed_wait_ms : {[round(x, 4) for x in (self.overlap.wait_history or [])]}\n")
        if self.args.save_grad_counts and hasattr(self, "round_history"):
            # per-rank micro-batch counts per round (the reference's unused `save_grad_acc`, utils/logs_utils.py:248)
            d = os.path.join(os.getcwd(), "grad_counts")
            os.makedirs(d, exist_ok=True)
            with open(os.path.join(d, f"{self.id_run}_{self.rank}.txt"), "w") as f:
                f.write(f"{self.rank} # grad acc : {[c for _, _, c in self.round_history]}\n")
                f.write(f"{self.rank} kinds : {[k for _, k, _ in self.round_history]}\n")
        if self._feeder is not None:
            self._feeder.close()
            self._feeder = None
        self._fire("on_train_end", self.stats)
        return self.stats

    # ================================================================== profiling
    def profile(self, steps: int = 4, outdir: Optional[str] = None, warmup: int = 1):
        """Run ``steps`` scheduling iterations under ``torch.profiler`` (CPU + CUDA activities) and export a Chrome trace
        plus a per-op table to ``outdir`` (default ``./profiler/{id_run}``).  The reference has no tracing at all ;
        NVTX ranges are emitted as well when ``ACCO_NVTX=1``.  Returns the path of the trace."""
        from torch.profiler import ProfilerActivity, profile
        outdir = outdir or os.path.join(os.getcwd(), "profiler", str(self.id_run))
        os.makedirs(outdir, exist_ok=True)
        for _ in range(int(warmup)):
            self.step()
        acts = [ProfilerActivity.CPU] + ([ProfilerActivity.CUDA] if self.is_cuda else [])
        with profile(activities=acts, record_shapes=False) as prof:
            for _ in range(int(steps)):
                self.step()
            if self.is_cuda:
                torch.cuda.synchronize(self.device)
        trace = os.path.join(outdir, f"trace_rank{self.rank}.json")
        prof.export_chrome_trace(trace)
        with open(os.path.join(outdir, f"ops_rank{self.rank}.txt"), "w") as f:
            f.write(prof.key_averages().table(sort_by="self_cuda_time_total" if self.is_cuda else "self_cpu_time_total", row_limit=60))
        return trace

    # ================================================================== checkpoints
    def save_checkpoint(self, path: str) -> None:
        """``torch.save(model.state_dict())`` with HF key names (`trainer_decoupled.py:559-574`); with
        ``save_optimizer`` every rank also writes its optimizer shard + counters (enables resume,
        which the reference lacks)."""
        self._ensure_gathered()
        if getattr(self, "_inflight", None) is not None:
            # called by user code in the middle of an overlapped round: finish it first (weights / Adam state must be quiescent)
            self._inflight.wait_host()
            self._complete_round()
            self._bind_compute_buffers()
        if self.is_cuda:
            torch.cuda.current_stream(self.device).synchronize()
        from .checkpoint import atomic_save, shard_path
        with_opt = bool(self.args.save_optimizer) and hasattr(self, "sharded_optimizer")
        if with_opt:
            # shards first, the model file last: `latest_checkpoint` only ever sees a model file whose shards are complete
            atomic_save({"optimizer": self.sharded_optimizer.state_dict(), "scheduler": self.sched.state_dict(),
                         "size_slice": self.size_slice, "numel": int(self.arena.numel), "tokens_seen": self._tokens_seen,
                         "data_batches": self._data_batches_base + (self._feeder.batches_out if self._feeder is not None else 0),
                         "world_size": self.world_size, "rng": torch.get_rng_state()}, shard_path(path, self.rank, self.world_size))
            self.backend.barrier()
        if self.rank == 0:
            atomic_save(self.model.state_dict(), path)
        if with_opt:
            self.backend.barrier()          # nobody moves on (or prunes) before the checkpoint is complete
        self._fire("on_save", path)

    def load_checkpoint(self, path: str) -> None:
        """Resume from ``path`` (a model file written by :meth:`save_checkpoint`; with ``save_optimizer`` shards next to it the
        Adam state, LR schedule position and counters are restored as well).  The shards may come from a run with a DIFFERENT
        world size (elastic restart after losing / gaining GPUs): the slice of the new layout is re-assembled from the old
        shards that overlap it (:func:`acco_b200.checkpoint.reshard_optimizer_state`)."""
        from .checkpoint import reshard_optimizer_state, shard_path, shard_sets
        sd = torch.load(path, map_location="cpu")
        self.model.load_state_dict(sd)
        with torch.no_grad():
            for t in self.arena.theta[1:]:
                t.copy_(self.arena.theta[self.arena.live])
        if not hasattr(self, "sharded_optimizer"):
            return
        stem = os.path.splitext(path)[0]
        own = shard_path(path, self.rank, self.world_size)
        import glob as _glob
        any_shard = sorted(_glob.glob(f"{_glob.escape(stem)}_optim_rank*of*.pt"))
        sets = shard_sets(path)
        st = None
        if self.world_size in sets and os.path.exists(own):
            st = torch.load(own, map_location="cpu", weights_only=False)
            if int(st["size_slice"]) != self.size_slice or int(st.get("numel", self.arena.numel)) != int(self.arena.numel):
                st = None                                   # same world size, different slice alignment (backend): re-shard
            else:
                opt_sd = st["optimizer"]
        if st is None and sets:
            old_world = self.world_size if self.world_size in sets else max(sets)
            opt_sd, st = reshard_optimizer_state(sets[old_world], self.rank, self.size_slice, numel=int(self.arena.numel))
            self.log.info(f"rank {self.rank}: optimizer state re-sharded from {old_world} to {self.world_size} ranks ({os.path.basename(path)})")
            if old_world != self.world_size:
                # per-rank token counters cannot be mapped one to one: split the old total evenly; the dataset is sharded
                # differently now, so the old position in the data stream means nothing
                st["tokens_seen"] = int(st.get("tokens_seen", 0)) * old_world // self.world_size
            st["data_batches"] = 0
        if st is None and any_shard:
            # resuming some ranks with Adam state and others without would desynchronise bias correction, the LR schedule and the
            # stop condition across ranks (-> a hang at the round barrier): refuse instead
            raise FileNotFoundError(
                f"checkpoint {path} has optimizer shards ({os.path.basename(any_shard[0])}, ...) but no complete set: "
                f"{os.path.basename(own)} (or a full set of another world size) is missing")
        if st is not None:
            self.sharded_optimizer.load_state_dict(opt_sd)
            sd_s = dict(st["scheduler"])
            # restart the round parity cleanly: a resumed run begins with a fresh tentative round
            sd_s["round"] = 0
            sd_s["count_after_init"] = 0
            self.sched.load_state_dict(sd_s)
            self._tokens_seen = int(st.get("tokens_seen", 0))
            n = int(st.get("data_batches", 0))
            if n > 0 and self.train_dataloader is not None and self._feeder is None:
                # continue the data stream where this rank stopped (same seed -> same epoch permutations)
                self.train_dataloader.fast_forward(n)
                self._data_batches_base = n
        else:
            self.sharded_optimizer.master.copy_(self.arena.shard(self.arena.theta[self.arena.live]).float())

    def _resolve_resume(self, spec: str) -> Optional[str]:
        """``resume_from=auto`` (or ``latest``): the newest complete checkpoint under ``./checkpoints`` - chosen by rank 0 and
        broadcast, so every rank resumes from the same file; None when there is nothing to resume from (fresh start)."""
        if spec.lower() not in ("auto", "latest"):
            return spec
        from .checkpoint import latest_checkpoint
        box = [None]
        if self.rank == 0:
            box[0] = latest_checkpoint(os.path.join(os.getcwd(), "checkpoints"), require_optimizer=bool(self.args.save_optimizer))
        if self.world_size > 1:
            import torch.distributed as dist
            if dist.is_initialized():
                dist.broadcast_object_list(box, src=0)
        self.log.info(f"resume_from={spec}: " + (f"resuming from {box[0]}" if box[0] else "no checkpoint found, starting fresh"))
        return box[0]

    # ================================================================== flat-vector accessors (API parity)
    @torch.no_grad()
    def get_weights(self) -> torch.Tensor:
        return self.arena.params_flat

    @torch.no_grad()
    def set_weights(self, weights: torch.Tensor) -> None:
        self.arena.params_flat.copy_(weights)

    @torch.no_grad()
    def get_grads(self) -> torch.Tensor:
        return self.arena.grads_flat

    @torch.no_grad()
    def set_grads(self, grads: torch.Tensor) -> None:
        self.arena.grads_flat.copy_(grads)
