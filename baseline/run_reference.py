"""Reference arm of ``bench.py``: run the UNMODIFIED reference trainer (installed verbatim into
``baseline/_ref`` from `/root/reference`) through its own public API and stock code path -
``DecoupledTrainer(model, tokenizer, train_dataset, eval_dataset, args, log, ...).train()`` with
``method_name='acco'`` = NCCL reduce-scatter / all-gather + ``torch.optim.AdamW(capturable=True)`` +
HF ``LlamaForCausalLM`` (cuBLAS / SDPA) under ``torch.autocast(bf16)`` - on the same model config,
batch shape and synthetic data as our arm.  None of this repo's models, kernels or engine is on
that path.

Environment shims (none of them touches reference code):
* ``SLURM_*`` variables are synthesised from torchrun's ``RANK/LOCAL_RANK/WORLD_SIZE`` - the
  reference reads Slurm env directly (`trainer_base.py:137-146`);
* ``omegaconf`` is not installed on this image: a 3-line stand-in provides
  ``OmegaConf.to_container`` (used once for results.csv, `trainer_decoupled.py:582`);
* the final ``torch.save(model.state_dict())`` inside ``train()`` (`:594-598`) is neutralised
  during the *timed* call so a 250 MB checkpoint write is not billed to the reference (our arm
  writes no checkpoint in its timed region either);
* a watchdog aborts the process if the reference hangs (its barrier/reset protocol has a latent
  race).

Warm-up / timed split: ``train()`` is called twice on the same trainer - first with
``nb_grad_tot = warmup rounds``, then (timed) with ``nb_grad_tot = K rounds`` - the only way to
exclude CUDA/NCCL/allocator warm-up without editing the reference's loop.  Work is measured as the
number of micro-batches the model actually ran (a forward hook counts them), exactly as in our arm.
"""
from __future__ import annotations

import logging
import os
import sys
import tempfile
import threading
import time
import types
from typing import Any, Dict

REF_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_ref")


class _Args(dict):
    """attribute-accessible dict (the reference accesses ``args.batch_size`` etc.)."""
    __getattr__ = dict.__getitem__

    def copy(self):
        return _Args(self)


def reference_available() -> str:
    if not os.path.isfile(os.path.join(REF_DIR, "trainer_decoupled.py")):
        return f"reference not installed under {REF_DIR}"
    try:
        import datasets  # noqa: F401
        import transformers  # noqa: F401
    except Exception as e:  # pragma: no cover
        return f"reference dependency missing: {e}"
    return ""


def _install_shims(rank: int, local_rank: int, world: int) -> None:
    os.environ["SLURM_NODEID"] = "0"
    os.environ["SLURM_PROCID"] = str(rank)
    os.environ["SLURM_JOBID"] = os.environ.get("ACCO_RUN_ID", "refbench")
    os.environ["SLURM_LOCALID"] = str(local_rank)
    os.environ["SLURM_NTASKS"] = str(world)
    os.environ["SLURM_JOB_NODELIST"] = os.environ.get("MASTER_ADDR", "127.0.0.1")
    # The reference overwrites MASTER_PORT with 12346 + min(SLURM_STEP_GPUS) (`trainer_base.py:149-153`).  Under torchrun the
    # env:// rendezvous must keep pointing at the agent's store, so choose the "GPU id" that reproduces torchrun's port;
    # stand-alone (no MASTER_PORT) any free offset works.
    if "MASTER_PORT" in os.environ:       # also for a 1-rank torchrun launch (the agent store is used whenever torchrun started us)
        os.environ["SLURM_STEP_GPUS"] = str(int(os.environ["MASTER_PORT"]) - 12346)
    else:
        os.environ["SLURM_STEP_GPUS"] = os.environ.get("ACCO_REF_PORT_OFFSET", "17")
    if "omegaconf" not in sys.modules:
        try:
            import omegaconf  # noqa: F401
        except Exception:
            m = types.ModuleType("omegaconf")
            m.OmegaConf = type("OmegaConf", (), {"to_container": staticmethod(lambda cfg, resolve=True: dict(cfg))})
            sys.modules["omegaconf"] = m
    if REF_DIR not in sys.path:
        sys.path.insert(0, REF_DIR)


def run_reference(steps: int, warmup: int, model_kw: Dict[str, Any], batch_size: int, seq_len: int, n_acc: int,
                  watchdog_s: float = 420.0) -> Dict[str, Any]:
    import numpy as np
    import torch
    import torch.distributed as dist
    rank = int(os.environ.get("RANK", 0))
    local_rank = int(os.environ.get("LOCAL_RANK", 0))
    world = int(os.environ.get("WORLD_SIZE", 1))
    _install_shims(rank, local_rank, world)

    def _abort():
        if rank == 0:
            print('{"impl": "reference", "unavailable": "reference trainer hung (watchdog %.0fs): its unsynchronised params <- com_buffer copy can race"}' % watchdog_s, flush=True)
        os._exit(0)
    wd = threading.Timer(watchdog_s, _abort)
    wd.daemon = True
    wd.start()
    try:
        return _run_reference_guarded(steps, warmup, model_kw, batch_size, seq_len, n_acc, rank, local_rank, world)
    finally:
        wd.cancel()          # never leave the watchdog armed (it hard-exits the process)


def _run_reference_guarded(steps, warmup, model_kw, batch_size, seq_len, n_acc, rank, local_rank, world) -> Dict[str, Any]:
    import numpy as np
    import torch
    import torch.distributed as dist
    import datasets
    import transformers
    torch.cuda.set_device(local_rank)
    torch.manual_seed(1234)
    torch.cuda.manual_seed_all(42)
    hf_cfg = transformers.LlamaConfig(
        vocab_size=model_kw["vocab_size"], hidden_size=model_kw["hidden_size"], intermediate_size=model_kw["intermediate_size"],
        num_hidden_layers=model_kw["num_hidden_layers"], num_attention_heads=model_kw["num_attention_heads"],
        num_key_value_heads=model_kw["num_key_value_heads"], max_position_embeddings=max(model_kw["max_position_embeddings"], seq_len),
        rms_norm_eps=1e-5, rope_theta=model_kw["rope_theta"], tie_word_embeddings=model_kw["tie_word_embeddings"],
        attention_bias=False, mlp_bias=False, use_cache=False)
    model = transformers.LlamaForCausalLM(hf_cfg)
    calls = [0]
    model.register_forward_hook(lambda m, i, o: calls.__setitem__(0, calls[0] + 1))

    rows = 64 * batch_size * world
    rng = np.random.default_rng(7)
    ds = datasets.Dataset.from_dict({"input_ids": rng.integers(0, model_kw["vocab_size"], size=(rows, seq_len), dtype=np.int64).tolist()})

    args = _Args(   # `config/train/acco.yaml` of the reference, verbatim values
        group_by_length=False, batch_size=batch_size, n_grad_accumulation=n_acc, learning_rate=6e-4, weight_decay=0.1,
        adam_beta1=0.9, adam_beta2=0.95, gradient_accumulation_steps=1, nb_steps_tot=max(warmup, 1) * world * n_acc,
        dataloader_num_workers=1, dataloader_pin_memory=True, dataloader_persistent_workers=True, label_smoothing_factor=0,
        max_length=seq_len, scheduler_name="cosine", warmup=1000, use_mixed_precision=True, n_warmup_steps=0,
        run_baseline_ddp=False, method_name="acco", eval=False, save=False, eval_step=500, run_expe_slow=False,
        const_len_batch=True, finetune=False)
    log = logging.getLogger("reference")
    log.setLevel(logging.WARNING)

    cwd = os.getcwd()
    tmp = tempfile.mkdtemp(prefix="acco_ref_")
    os.chdir(tmp)
    try:
        from trainer_decoupled import DecoupledTrainer as RefTrainer   # the reference's own class
        trainer = RefTrainer(model=model, tokenizer=None, train_dataset=ds, eval_dataset=None, args=args, log=log,
                             text_column_name="text", preprocess_dataset_fn=None, run_name="refbench")
        real_save = torch.save
        torch.save = lambda *a, **k: None            # see module docstring
        try:
            trainer.nb_grad_tot = max(warmup, 1) * world * n_acc
            trainer.train()                           # untimed warm-up rounds
            torch.cuda.synchronize()
            dist.barrier()
            torch.cuda.synchronize()
            c0 = calls[0]
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0 = time.perf_counter()
            e0.record()
            trainer.nb_grad_tot = steps * world * n_acc
            trainer.train()                           # timed: ~`steps` communication rounds
            torch.cuda.synchronize()
            e1.record()
            torch.cuda.synchronize()
            wall_ms = (time.perf_counter() - t0) * 1e3
            dev_ms = e0.elapsed_time(e1)
            dist.barrier()
        finally:
            torch.save = real_save
        micro = calls[0] - c0
        t = torch.tensor([dev_ms, wall_ms, float(micro)], dtype=torch.float64, device="cuda")
        tmax = t.clone()
        dist.all_reduce(tmax, op=dist.ReduceOp.MAX)
        tsum = t.clone()
        dist.all_reduce(tsum, op=dist.ReduceOp.SUM)
        loss = float(trainer.loss_static.item())
    finally:
        os.chdir(cwd)
    total_micro = float(tsum[2].item())
    ms = float(tmax[0].item())
    return {
        "ms_total": ms, "wall_ms_total": float(tmax[1].item()), "micro_batches": total_micro,
        "tokens": total_micro * batch_size * seq_len, "loss": loss,
        "h2d_bytes_per_step": n_acc * batch_size * seq_len * 8, "d2h_bytes_per_step": 4,
    }
