"""Tokenisation post-processing.

* :func:`pack_const_len` - the reference's *const-len packing* (`trainer_base.py:84-97`,
  `dl_dataset.py:8-34`): append EOS to every document, concatenate, cut into rows of
  ``max_length`` tokens, drop the tail; no attention mask is produced.
* :func:`truncate_docs` - the *truncate-only* path for fine-tuning (`trainer_base.py:77-82`).
* :func:`pack_sft` - sample packing for fine-tuning (``packing: True``): whole truncated samples placed into rows of at most
  ``max_length`` tokens by first-fit-decreasing; ``PackedCollator`` turns a row into document-masked training inputs.

Implemented with numpy on flat arrays (one concatenate, one reshape) rather than Python list
appends, since it runs over ~9M documents for openwebtext."""
from __future__ import annotations

from typing import Any, Dict, List, Sequence

import numpy as np

__all__ = ["pack_const_len", "truncate_docs", "pack_sft", "make_const_len_tokenize_fn", "make_truncate_tokenize_fn",
           "make_packed_tokenize_fn"]


def _native():
    """The C++ packer from the in-tree extension (``csrc/host_data.cpp``) if it is built."""
    try:
        from ..ops import load_ext
        ext = load_ext()
        return ext if (ext is not None and hasattr(ext, "pack_const_len")) else None
    except Exception:
        return None


def pack_const_len(docs: Sequence[Sequence[int]], max_length: int, eos_token_id: int) -> np.ndarray:
    """-> int64 array ``[n_rows, max_length]``.  Uses the native C++ packer when the extension is built
    (one memcpy per document), else numpy."""
    if len(docs) == 0:
        return np.zeros((0, max_length), dtype=np.int64)
    ext = _native()
    if ext is not None:
        import torch
        lens_only = np.fromiter((len(d) for d in docs), dtype=np.int64, count=len(docs))
        flat_in = np.concatenate([np.asarray(d, dtype=np.int64) for d in docs]) if lens_only.sum() else np.zeros(0, dtype=np.int64)
        out = ext.pack_const_len(torch.from_numpy(flat_in), torch.from_numpy(lens_only), int(max_length), int(eos_token_id))
        return out.numpy()
    lens = np.fromiter((len(d) + 1 for d in docs), dtype=np.int64, count=len(docs))
    flat = np.empty(int(lens.sum()), dtype=np.int64)
    pos = 0
    for d, n in zip(docs, lens):
        flat[pos: pos + n - 1] = np.asarray(d, dtype=np.int64)
        flat[pos + n - 1] = eos_token_id
        pos += n
    rows = flat.size // max_length
    return flat[: rows * max_length].reshape(rows, max_length)


def truncate_docs(docs: Sequence[Sequence[int]], max_length: int) -> List[List[int]]:
    return [list(d[:max_length]) for d in docs]


def pack_sft(docs: Sequence[Sequence[int]], max_length: int) -> Dict[str, List[List[int]]]:
    """Truncate every sample to ``max_length`` and place the samples into rows of at most ``max_length`` tokens by
    first-fit-decreasing (longest first, ties in input order; each goes into the first row with room, else opens a new row).
    A sample is never split.  Deterministic, no RNG.
    -> ``{"input_ids": [row tokens], "doc_lens": [lengths of the row's samples, in row order]}``; empty samples are dropped."""
    docs = [list(d[:max_length]) for d in docs]
    order = sorted((i for i in range(len(docs)) if docs[i]), key=lambda i: -len(docs[i]))
    rows: List[List[int]] = []
    free: List[int] = []
    for i in order:
        n = len(docs[i])
        r = next((j for j, f in enumerate(free) if f >= n), None)
        if r is None:
            rows.append([])
            free.append(max_length)
            r = len(rows) - 1
        rows[r].append(i)
        free[r] -= n
    return {"input_ids": [[t for i in row for t in docs[i]] for row in rows],
            "doc_lens": [[len(docs[i]) for i in row] for row in rows]}


def make_const_len_tokenize_fn(tokenizer, text_column: str, max_length: int):
    """Batched ``datasets.map`` function: text -> packed ``input_ids`` rows."""
    def fn(batch: Dict[str, Any]) -> Dict[str, Any]:
        ids = tokenizer(batch[text_column], truncation=False)["input_ids"]
        packed = pack_const_len(ids, max_length, tokenizer.eos_token_id)
        return {"input_ids": [row for row in packed]}
    return fn


def make_truncate_tokenize_fn(tokenizer, text_column: str, max_length: int):
    def fn(batch: Dict[str, Any]) -> Dict[str, Any]:
        out = tokenizer(batch[text_column], truncation=True, max_length=max_length)
        res = {"input_ids": out["input_ids"]}
        if "attention_mask" in out:
            res["attention_mask"] = out["attention_mask"]
        return res
    return fn


def make_packed_tokenize_fn(tokenizer, text_column: str, max_length: int):
    """Batched ``datasets.map`` function: text -> packed ``input_ids`` / ``doc_lens`` rows (:func:`pack_sft` within each map batch)."""
    def fn(batch: Dict[str, Any]) -> Dict[str, Any]:
        ids = tokenizer(batch[text_column], truncation=True, max_length=max_length)["input_ids"]
        return pack_sft(ids, max_length)
    return fn


def make_preference_tokenize_fn(tokenizer):
    """Batched ``datasets.map`` function: TRL's ``prompt`` / ``chosen`` / ``rejected`` text columns -> ``prompt_ids``, ``chosen_ids``,
    ``rejected_ids`` token lists, each response closed by the tokenizer's EOS when it has one.  ``PreferenceCollator`` joins the
    prompt and each response and cuts the row at ``max_length``."""
    eos = getattr(tokenizer, "eos_token_id", None)
    tail = [] if eos is None else [int(eos)]

    def fn(batch: Dict[str, Any]) -> Dict[str, Any]:
        out = {"prompt_ids": tokenizer(batch["prompt"])["input_ids"]}
        for key in ("chosen", "rejected"):
            out[f"{key}_ids"] = [list(r) + tail for r in tokenizer(batch[key], add_special_tokens=False)["input_ids"]]
        return out
    return fn
