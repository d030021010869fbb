"""Collators.

* :func:`stack_collate` - const-len batches: stack ``input_ids`` rows into one LongTensor
  (`trainer_base.py:131-132`).
* :class:`PadCollator` - ragged SFT batches: right-pad to the longest row, emit ``attention_mask``
  and ``labels`` with pad positions set to -100.  With ``pad == eos`` (the reference sets
  ``tokenizer.pad_token_id = eos_token_id``, `main.py:46`) HF's
  ``DataCollatorForLanguageModeling(mlm=False)`` masks *every* EOS label ; that is
  reproduced with ``mask_all_pad_tokens=True`` (default) and can be switched off.
* :class:`PackedCollator` - packed SFT rows (``pack_sft``): fixed ``[B, max_length]`` batches with per-sample ``position_ids``
  (the models derive document masking from them) and labels that train exactly the (context, target) pairs of ``PadCollator``.
* :class:`DocumentCollator` - const-len pre-training rows with document masking (``document_mask: True``): the same three
  ``[B, S]`` tensors as ``PackedCollator``, with the documents found from the EOS tokens ``pack_const_len`` closed them with.
* :class:`PreferenceCollator` - DPO preference pairs (``prompt_ids`` / ``chosen_ids`` / ``rejected_ids``): ``[2P, S]`` rows, the
  ``P`` chosen responses first, labels only on the response tokens.
"""
from __future__ import annotations

from typing import Any, Dict, Sequence

import numpy as np
import torch

__all__ = ["stack_collate", "PadCollator", "PackedCollator", "DocumentCollator", "PreferenceCollator", "PREFERENCE_COLUMNS"]

PREFERENCE_COLUMNS = ("prompt_ids", "chosen_ids", "rejected_ids")


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


class PackedCollator:
    """Rows of several samples (columns ``input_ids`` and ``doc_lens``) -> ``input_ids``, ``labels``, ``position_ids``, each
    ``[B, max_length]`` int64.  For a sample at ``[a, a+n)``: ``position_ids[a+i] = i``; ``labels[a] = -100`` (the previous
    sample's last token must not learn to predict this one's first); ``labels[a+i] = input_ids[a+i]`` for ``1 <= i < n``, except
    pad ids when ``mask_all_pad_tokens`` (the ``PadCollator`` rule).  The tail ``[used, max_length)`` holds pad ids with labels -100
    and positions restarting at 0: one more segment."""

    def __init__(self, pad_token_id: int, max_length: int, mask_all_pad_tokens: bool = True, label_pad: int = -100):
        self.pad, self.L, self.label_pad = int(pad_token_id), int(max_length), int(label_pad)
        self.mask_all = mask_all_pad_tokens

    def __call__(self, batch: Sequence[Dict[str, Any]]) -> Dict[str, torch.Tensor]:
        B, L = len(batch), self.L
        ids = np.full((B, L), self.pad, dtype=np.int64)
        labels = np.full((B, L), self.label_pad, dtype=np.int64)
        pos = np.zeros((B, L), dtype=np.int64)
        for b, row in enumerate(batch):
            toks = np.asarray(row["input_ids"], dtype=np.int64).reshape(-1)
            lens = [int(n) for n in row["doc_lens"]]
            if any(n <= 0 for n in lens):
                raise ValueError(f"packed row {b}: sample lengths must be positive, got {lens}")
            if sum(lens) != toks.size or toks.size > L:
                raise ValueError(f"packed row {b}: sample lengths sum to {sum(lens)} for a row of {toks.size} tokens (max_length {L})")
            used = toks.size
            ids[b, :used] = toks
            labels[b, :used] = toks
            a = 0
            for n in lens:
                labels[b, a] = self.label_pad
                pos[b, a:a + n] = np.arange(n)
                a += n
            pos[b, used:] = np.arange(L - used)
            if self.mask_all:
                labels[b, :used][toks == self.pad] = self.label_pad
        return {"input_ids": torch.from_numpy(ids), "labels": torch.from_numpy(labels), "position_ids": torch.from_numpy(pos)}


class DocumentCollator:
    """Const-len rows (``pack_const_len``: documents each closed by ``eos_token_id``, cut into rows) -> ``input_ids``, ``labels``,
    ``position_ids``, each ``[B, S]`` int64, following the ``PackedCollator`` rules so the models mask attention by document:

    * a segment starts at column 0 and right after every EOS (the EOS closes its own document; consecutive EOS tokens make
      one-token segments; an EOS in the last column opens no segment).  The first segment usually begins mid-document;
    * ``position_ids[s] = s - start(s)``;
    * ``labels = input_ids`` except ``labels[start] = -100`` at every segment start after column 0 (the models shift labels, so
      this drops the one prediction whose context is the previous document).  EOS stays a target and nothing is masked by pad
      id: const-len rows hold no padding, and with ``pad == eos`` that rule would erase every EOS target.

    Segment starts are a running maximum along the row, so they never decrease within a row: the precondition of the segmented
    attention kernels (``csrc/attention_wgmma.cu``).  Vectorised numpy, no per-token Python loop (it runs in the loader workers)."""

    def __init__(self, eos_token_id: int, label_pad: int = -100):
        self.eos, self.label_pad = int(eos_token_id), int(label_pad)

    def __call__(self, batch: Sequence[Dict[str, Any]]) -> Dict[str, torch.Tensor]:
        ids = np.stack([np.asarray(b["input_ids"], dtype=np.int64).reshape(-1) for b in batch])
        S = ids.shape[1]
        s = np.arange(S, dtype=np.int64)
        opens = np.zeros_like(ids)
        opens[:, 1:] = np.where(ids[:, :-1] == self.eos, s[1:], 0)       # column s opens a segment when column s-1 is an EOS
        start = np.maximum.accumulate(opens, axis=1)
        labels = ids.copy()
        labels[(start == s) & (s > 0)] = self.label_pad
        return {"input_ids": torch.from_numpy(ids), "labels": torch.from_numpy(labels), "position_ids": torch.from_numpy(s - start)}


class PreferenceCollator:
    """``P`` preference pairs (token lists ``prompt_ids``, ``chosen_ids``, ``rejected_ids``) -> ``input_ids``, ``attention_mask``,
    ``labels``, each ``[2P, S]`` int64: row ``i`` is ``prompt + chosen`` of pair ``i``, row ``P + i`` is ``prompt + rejected``, each cut
    at ``max_length`` from the right.  ``S`` is the longest row rounded up to ``pad_to_multiple_of`` (as ``PadCollator``, so CUDA
    graphs replay).  ``labels`` equal the response tokens and are -100 on the prompt and the padding; a row whose response was cut
    away has no label, and its pair then counts as invalid in the DPO loss."""

    def __init__(self, pad_token_id: int, max_length: int, pad_to_multiple_of: int = 1, label_pad: int = -100):
        self.pad, self.L, self.label_pad = int(pad_token_id), int(max_length), int(label_pad)
        self.mult = max(int(pad_to_multiple_of), 1)

    def __call__(self, batch: Sequence[Dict[str, Any]]) -> Dict[str, torch.Tensor]:
        rows, starts = [], []
        for key in ("chosen_ids", "rejected_ids"):
            for b in batch:
                prompt = list(b["prompt_ids"])
                rows.append((prompt + list(b[key]))[: self.L])
                starts.append(len(prompt))
        S = max(max(len(r) for r in rows), 1)
        S = ((S + self.mult - 1) // self.mult) * self.mult
        ids = np.full((len(rows), S), self.pad, dtype=np.int64)
        mask = np.zeros((len(rows), S), dtype=np.int64)
        labels = np.full((len(rows), S), self.label_pad, dtype=np.int64)
        for i, (r, a) in enumerate(zip(rows, starts)):
            ids[i, : len(r)] = r
            mask[i, : len(r)] = 1
            labels[i, a: len(r)] = r[a:]
        return {"input_ids": torch.from_numpy(ids), "attention_mask": torch.from_numpy(mask), "labels": torch.from_numpy(labels)}
