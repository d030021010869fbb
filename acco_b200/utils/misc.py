"""Small utilities: seeding (the reference seeds CUDA only with a hard-coded 42 and never seeds the
CPU generator that actually initialises the model, `main.py:28`), parameter counting,
and the label-smoothed loss the reference instantiates (`trainer_base.py:63-68`,
`utils/trainer_utils.py:862-902`) but never applies."""
from __future__ import annotations

import random
from typing import Any

import numpy as np
import torch
import torch.nn.functional as F


def seed_everything(seed: int) -> None:
    random.seed(seed)
    np.random.seed(seed % (2 ** 32))
    torch.manual_seed(seed)
    if torch.cuda.is_available():
        torch.cuda.manual_seed_all(seed)


def get_model_param_count(model: torch.nn.Module, trainable_only: bool = False) -> int:
    seen, n = set(), 0
    for p in model.parameters():
        if id(p) in seen or (trainable_only and not p.requires_grad):
            continue
        seen.add(id(p))
        n += p.numel()
    return n


class LabelSmoother:
    """``(1-eps) * nll + eps * mean_over_vocab(-log p)``, averaged over non-ignored positions.

    ``shift_labels=True`` applies the causal-LM shift.  Used by
    :meth:`DecoupledTrainer.compute_loss` when ``label_smoothing_factor != 0`` (unlike the
    reference, where no training path ever calls ``compute_loss``)."""

    def __init__(self, epsilon: float = 0.1, ignore_index: int = -100):
        self.epsilon, self.ignore_index = float(epsilon), int(ignore_index)

    def __call__(self, model_output: Any, labels: torch.Tensor, shift_labels: bool = False) -> torch.Tensor:
        logits = model_output["logits"] if isinstance(model_output, dict) or hasattr(model_output, "keys") else model_output[0]
        if shift_labels:
            logits = logits[..., :-1, :].contiguous()
            labels = labels[..., 1:].contiguous()
        logp = -F.log_softmax(logits.float(), dim=-1)
        labels = labels.unsqueeze(-1)
        pad = labels.eq(self.ignore_index)
        nll = logp.gather(-1, labels.clamp(min=0)).masked_fill(pad, 0.0)
        smooth = logp.sum(-1, keepdim=True).masked_fill(pad, 0.0)
        n = (pad.numel() - pad.long().sum()).clamp(min=1)
        return (1 - self.epsilon) * nll.sum() / n + self.epsilon * smooth.sum() / (n * logits.shape[-1])
