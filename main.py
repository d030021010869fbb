#!/usr/bin/env python
"""CLI entry - same command line as the reference (`main.py:25-71`, `README.md:52-58`):

    python main.py train=acco data=openwebtext model=llama125m            # 1 GPU (or CPU)
    torchrun --nproc-per-node 8 main.py train=acco model=llama125m       # 8 GPUs of one box
    srun python -u main.py train=acco-ft data=alpaca model=llama3-1b     # Slurm, one task per GPU

Config groups ``train= data= model=`` and ``key=value`` overrides are composed by
:mod:`acco_b200.config` (Hydra is not required).  The model is built from ``config/model/*.yaml``
(random init; with ``train.finetune=True``, ``model.pretrained=<HF checkpoint dir>`` is loaded like the reference's
``AutoModelForCausalLM.from_pretrained`` - into the native Llama / GPT-Neo when the architecture matches, else as the HF module -
and ``model.checkpoint=<file>`` loads an HF-keyed state dict into the configured architecture); the
dataset is loaded with ``datasets.load_dataset(cfg.data.path)`` and split 95/5 with seed 42 like the
reference, or - offline (``data.synthetic`` true/auto) - replaced by a synthetic corpus of the same
shape.  Artefacts land in the launch directory: ``tensorboard/``, ``checkpoints/``, ``results.csv``.
"""
from __future__ import annotations

import logging
import os
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

logging.basicConfig(stream=sys.stdout, level=logging.INFO)
if os.environ.get("ACCO_HANG_DUMP_S"):
    # host-side hang diagnosis: every N seconds dump the Python stack of every thread to stderr (a stuck rendezvous, a collective
    # waiting for a dead peer, a data-loader dead-lock all show up as the same frames dump after dump)
    import faulthandler
    faulthandler.dump_traceback_later(int(os.environ["ACCO_HANG_DUMP_S"]), repeat=True)
logger = logging.getLogger("distributed_worker")


def load_data(cfg, vocab_size: int, tokenizer):
    """-> (train, test, tokenizer).  Tries the HF hub id first unless ``data.synthetic`` is true."""
    from acco_b200.data import ByteTokenizer, synthetic_pretrain_dataset, synthetic_sft_dataset
    d, t = cfg.data, cfg.train
    mode = str(d.get("synthetic", "auto")).lower()
    if mode not in ("true", "1", "yes") and d.get("path"):
        try:
            import datasets
            if os.path.isdir(str(d.path)):
                ds = datasets.load_from_disk(str(d.path))
            else:
                ds = datasets.load_dataset(d.path)
            split = ds["train"].train_test_split(0.05, seed=42)
            return split["train"], split["test"], tokenizer
        except Exception as e:
            if mode in ("false", "0", "no"):
                raise
            logger.info(f"could not load dataset {d.path!r} ({type(e).__name__}); using a synthetic {d.get('kind', 'pretrain')} corpus")
    n_docs, mean_len = int(d.get("synthetic_docs", 4096)), int(d.get("synthetic_mean_len", 900))
    seed = int(cfg.get("seed", 0))
    if str(d.get("kind", "pretrain")) == "sft" or not t.const_len_batch:
        full = synthetic_sft_dataset(n_docs, mean_len, vocab_size - 1, int(t.max_length), seed=seed)
        if tokenizer is None:
            tokenizer = ByteTokenizer(eos_token_id=vocab_size - 1)
            tokenizer.pad_token_id = tokenizer.eos_token_id
    else:
        full = synthetic_pretrain_dataset(n_docs, mean_len, vocab_size, int(t.max_length), eos_token_id=vocab_size - 1, seed=seed)
    split = full.train_test_split(0.05, seed=42)
    return split["train"], split["test"], tokenizer


def write_run_dir(cfg, overrides) -> None:
    """Hydra's per-run directory (`config/config.yaml:10-12`: ``outputs/<date>/<time>``), written by rank 0 without changing the
    working directory (the reference runs with ``version_base=None``: no chdir, `main.py:25`): ``.hydra/config.yaml`` = the composed
    configuration, ``.hydra/overrides.yaml`` = the command line, ``main.log`` = this job's log."""
    import yaml
    from acco_b200.launch import discover_env
    run_dir = ((cfg.get("hydra") or {}).get("run") or {}).get("dir")
    if not run_dir or discover_env().rank != 0:
        return

    def plain(node):
        if isinstance(node, dict):
            return {k: plain(v) for k, v in node.items()}
        if isinstance(node, (list, tuple)):
            return [plain(v) for v in node]
        return node

    try:
        os.makedirs(os.path.join(run_dir, ".hydra"), exist_ok=True)
        with open(os.path.join(run_dir, ".hydra", "config.yaml"), "w") as f:
            yaml.safe_dump({k: plain(v) for k, v in cfg.items() if k != "hydra"}, f, sort_keys=False)
        with open(os.path.join(run_dir, ".hydra", "overrides.yaml"), "w") as f:
            yaml.safe_dump([str(o) for o in overrides], f)
        handler = logging.FileHandler(os.path.join(run_dir, "main.log"))
        handler.setFormatter(logging.Formatter("[%(asctime)s][%(name)s][%(levelname)s] - %(message)s"))
        logging.getLogger().addHandler(handler)
    except OSError as e:                            # a read-only launch directory must not stop a run
        logger.info(f"could not create the run directory {run_dir!r}: {e}")


def main(argv=None):
    import torch
    from acco_b200 import DecoupledTrainer, compose
    from acco_b200.config import default_config_dir
    from acco_b200.models import build_model
    from acco_b200.utils import seed_everything

    overrides = list(sys.argv[1:] if argv is None else argv)
    cfg = compose(overrides=overrides)
    write_run_dir(cfg, overrides)
    seed_everything(int(cfg.get("seed", 12345)))
    dev = None
    if torch.cuda.is_available():
        from acco_b200.launch import discover_env
        dev = torch.device("cuda", discover_env().local_rank)
    mdtype = torch.bfloat16 if (dev is not None and cfg.train.use_mixed_precision) else None
    pretrained = cfg.model.get("pretrained")
    if cfg.train.finetune and pretrained:
        # reference: AutoModelForCausalLM.from_pretrained(config_path) (`main.py:33-35`)
        from acco_b200.models import from_pretrained
        model = from_pretrained(str(pretrained), device=dev, dtype=mdtype, native=bool(cfg.model.get("native", True)))
        logger.info(f"loaded pretrained model {pretrained} as {type(model).__name__}")
    else:
        model = build_model(cfg.model, config_root=os.path.dirname(default_config_dir()), device=dev, dtype=mdtype)
        if cfg.train.finetune and cfg.model.get("checkpoint"):
            from acco_b200.models import load_hf_state_dict
            model.load_state_dict(load_hf_state_dict(str(cfg.model.checkpoint)))
            logger.info(f"loaded checkpoint {cfg.model.checkpoint}")
    print("model instantiated")
    tokenizer = None
    if cfg.model.get("tokenizer"):
        try:
            from transformers import AutoTokenizer
            tokenizer = AutoTokenizer.from_pretrained(str(cfg.model.tokenizer))
            tokenizer.pad_token_id = tokenizer.eos_token_id
            print("tokenizer loaded")
        except Exception as e:
            logger.info(f"tokenizer {cfg.model.tokenizer!r} unavailable offline ({type(e).__name__})")
    vocab = int(getattr(model.config, "vocab_size", cfg.model.get("vocab_size", 50257)))
    train_ds, test_ds, tokenizer = load_data(cfg, vocab, tokenizer)
    cfg.train["seed"] = cfg.train.get("seed", cfg.get("seed", 12345))
    trainer = DecoupledTrainer(model=model, tokenizer=tokenizer, train_dataset=train_ds, eval_dataset=test_ds,
                               text_column_name="text", args=cfg.train, log=logger, preprocess_dataset_fn=None,
                               run_name=cfg.run_name)
    stats = trainer.train()
    if trainer.rank == 0:
        logger.info(f"done: {stats}")
    from acco_b200.launch import shutdown_distributed
    shutdown_distributed()
    return stats


if __name__ == "__main__":
    main()
