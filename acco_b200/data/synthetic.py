"""Synthetic corpora shaped like the reference's two datasets (the GPU machines are offline, so
``datasets.load_dataset`` of `config/data/*.yaml` cannot run):

* **openwebtext-shaped** pre-training documents: ragged token sequences with a heavy-tailed
  length distribution (mean ~900 tokens), meant for const-len packing;
* **alpaca-shaped** SFT samples: short ragged prompt+response rows (mean ~180 tokens) that are
  padded per batch (labels -100 on pad/EOS).

Token ids follow a Zipf-like marginal with a first-order Markov dependency so the LM loss can
actually decrease (tests assert it does).  Documents are already token ids (``input_ids``
column) - the trainer skips tokenisation when that column exists, exactly like the reference
(`trainer_base.py:108`); a ``text`` variant exists for exercising the tokeniser path."""
from __future__ import annotations

from typing import Dict, List, Optional

import numpy as np
import torch

from .dataset import TokenDataset
from .packing import pack_const_len

__all__ = ["synthetic_documents", "synthetic_pretrain_dataset", "synthetic_preference_dataset", "synthetic_sft_dataset",
           "synthetic_text_dataset", "synthetic_token_batches"]


def _markov_tokens(rng: np.random.Generator, n: int, vocab: int, reserved_top: int = 1) -> np.ndarray:
    """Zipf marginal + deterministic-ish successor structure: next = (a*prev + noise) mod V."""
    hi = max(vocab - reserved_top, 2)
    z = rng.zipf(1.3, size=n).astype(np.int64)
    base = (z - 1) % hi
    follow = rng.random(n) < 0.6
    follow[0] = False
    # run starts are the non-follow positions; inside a run token_k = f^k(start), f(x) = 31x + 7 (mod hi)
    idx = np.arange(n, dtype=np.int64)
    start = np.maximum.accumulate(np.where(follow, 0, idx))
    k = idx - start
    kmax = int(k.max()) + 1
    A = np.empty(kmax, dtype=np.int64)
    C = np.empty(kmax, dtype=np.int64)
    A[0], C[0] = 1, 0
    for j in range(1, kmax):
        A[j] = (A[j - 1] * 31) % hi
        C[j] = (C[j - 1] * 31 + 7) % hi
    return (A[k] * base[start] + C[k]) % hi


def synthetic_documents(n_docs: int, mean_len: int, vocab_size: int, seed: int = 0, min_len: int = 8,
                        max_len: Optional[int] = None) -> List[np.ndarray]:
    rng = np.random.default_rng(seed)
    lens = np.clip(rng.lognormal(mean=np.log(max(mean_len, 2)) - 0.5, sigma=1.0, size=n_docs).astype(np.int64),
                   min_len, max_len or 16 * mean_len)
    stream = _markov_tokens(rng, int(lens.sum()), vocab_size)
    docs, pos = [], 0
    for n in lens:
        docs.append(stream[pos: pos + n])
        pos += n
    return docs


def synthetic_pretrain_dataset(n_docs: int, mean_len: int, vocab_size: int, max_length: int, eos_token_id: Optional[int] = None,
                               seed: int = 0) -> TokenDataset:
    """Packed const-len rows ready for ``stack_collate`` (column ``input_ids``)."""
    eos = vocab_size - 1 if eos_token_id is None else eos_token_id
    docs = synthetic_documents(n_docs, mean_len, vocab_size, seed)
    rows = pack_const_len(docs, max_length, eos)
    return TokenDataset({"input_ids": torch.from_numpy(rows)})


def synthetic_sft_dataset(n_rows: int, mean_len: int, vocab_size: int, max_length: int, seed: int = 0) -> TokenDataset:
    """Ragged rows (lists), truncated at ``max_length``; EOS is *not* appended - the pad collator
    pads with EOS like the reference."""
    docs = synthetic_documents(n_rows, mean_len, vocab_size, seed, min_len=4, max_len=max_length)
    return TokenDataset({"input_ids": [d[:max_length].tolist() for d in docs]})


def synthetic_preference_dataset(n_pairs: int, mean_len: int, vocab_size: int, seed: int = 0) -> TokenDataset:
    """DPO pairs (columns ``prompt_ids``, ``chosen_ids``, ``rejected_ids``).  The chosen response continues the prompt's Markov source
    (the successor map ``x -> 31 x + 7`` of :func:`_markov_tokens`); the rejected one comes from another source (uniform tokens), so a
    model can learn to prefer the chosen response and the DPO accuracy can rise.  Prompts and responses each average ``mean_len / 2``
    tokens."""
    rng = np.random.default_rng(seed)
    half = max(mean_len // 2, 2)
    prompts, chosen, rejected = [], [], []
    for _ in range(n_pairs):
        lp, lc, lr = (int(v) for v in rng.integers(max(half // 2, 1), half + half // 2 + 1, size=3))
        doc = _markov_tokens(rng, lp + lc, vocab_size)
        prompts.append(doc[:lp].tolist())
        chosen.append(doc[lp:].tolist())
        rejected.append(rng.integers(0, max(vocab_size - 1, 2), size=lr).tolist())
    return TokenDataset({"prompt_ids": prompts, "chosen_ids": chosen, "rejected_ids": rejected})


def synthetic_text_dataset(n_docs: int, mean_words: int, seed: int = 0) -> TokenDataset:
    rng = np.random.default_rng(seed)
    words = ["acco", "grad", "shard", "round", "theta", "nvlink", "tile", "adam", "step", "token", "loss", "comm"]
    texts = []
    for _ in range(n_docs):
        n = max(int(rng.poisson(mean_words)), 1)
        texts.append(" ".join(words[i] for i in rng.integers(0, len(words), n)))
    return TokenDataset({"text": texts})


def synthetic_token_batches(n_batches: int, batch_size: int, seq_len: int, vocab_size: int, seed: int = 0,
                            pin: bool = False) -> List[Dict[str, torch.Tensor]]:
    """Pre-collated random batches on the host (bench input pool)."""
    g = torch.Generator().manual_seed(seed)
    out = []
    for _ in range(n_batches):
        t = torch.randint(0, vocab_size, (batch_size, seq_len), generator=g, dtype=torch.long)
        out.append({"input_ids": t.pin_memory() if pin else t})
    return out
