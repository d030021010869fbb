"""acco_b200 - a Hopper (H100, sm_90a) native implementation of ACCO
("Accumulate while you Communicate"), DPU and sharded-optimizer DDP training.

Public API (same shape as the reference repo's, `trainer_decoupled.py:170-186`)::

    from acco_b200 import DecoupledTrainer
    trainer = DecoupledTrainer(model=model, tokenizer=tok, train_dataset=train, eval_dataset=test,
                               args=cfg.train, log=logger, run_name="acco")
    trainer.train()
"""
from .callbacks import EarlyStoppingCallback, TrainerCallback
from .config import AttrDict, compose, to_container
from .trainer import DecoupledTrainer, TRAIN_DEFAULTS

__version__ = "0.1.0"
__all__ = ["DecoupledTrainer", "TRAIN_DEFAULTS", "AttrDict", "compose", "to_container", "TrainerCallback", "EarlyStoppingCallback", "__version__"]
