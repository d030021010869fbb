"""Collators.

* :func:`stack_collate` - const-len batches: stack ``input_ids`` rows into one LongTensor
  (`trainer_base.py:131-132`).
* :class:`PadCollator` - ragged SFT batches: right-pad to the longest row, emit ``attention_mask``
  and ``labels`` with pad positions set to -100.  With ``pad == eos`` (the reference sets
  ``tokenizer.pad_token_id = eos_token_id``, `main.py:46`) HF's
  ``DataCollatorForLanguageModeling(mlm=False)`` masks *every* EOS label ; that is
  reproduced with ``mask_all_pad_tokens=True`` (default) and can be switched off.
"""
from __future__ import annotations

from typing import Any, Dict, Sequence

import numpy as np
import torch

__all__ = ["stack_collate", "PadCollator"]


def stack_collate(batch: Sequence[Dict[str, Any]]) -> Dict[str, torch.Tensor]:
    rows = [torch.as_tensor(np.asarray(b["input_ids"]), dtype=torch.long) for b in batch]
    return {"input_ids": torch.stack(rows)}


class PadCollator:
    def __init__(self, pad_token_id: int, label_pad: int = -100, mask_all_pad_tokens: bool = True,
                 pad_to_multiple_of: int = 1, max_length: int = None):
        self.pad, self.label_pad = int(pad_token_id), int(label_pad)
        self.mask_all = mask_all_pad_tokens
        self.mult = max(int(pad_to_multiple_of), 1)
        self.max_length = max_length

    def __call__(self, batch: Sequence[Dict[str, Any]]) -> Dict[str, torch.Tensor]:
        rows = [list(b["input_ids"]) for b in batch]
        L = max(len(r) for r in rows)
        if self.max_length:
            L = min(L, self.max_length)
        L = ((L + self.mult - 1) // self.mult) * self.mult
        ids = torch.full((len(rows), L), self.pad, dtype=torch.long)
        mask = torch.zeros((len(rows), L), dtype=torch.long)
        for i, r in enumerate(rows):
            r = r[:L]
            ids[i, : len(r)] = torch.as_tensor(r, dtype=torch.long)
            mask[i, : len(r)] = 1
        labels = ids.clone()
        if self.mask_all:
            labels[ids == self.pad] = self.label_pad
        else:
            labels[mask == 0] = self.label_pad
        return {"input_ids": ids, "attention_mask": mask, "labels": labels}
