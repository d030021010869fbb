"""A small in-memory columnar dataset with the slice of the HF ``datasets.Dataset`` API the
reference relies on (`trainer_base.py:100-124,193-200`, `main.py:49-50`): ``column_names``,
``shard(num_shards, index)``, ``map(fn, batched=True, remove_columns=..., num_proc=...)``,
``train_test_split(test_size, seed)``, ``save_to_disk`` / ``load_from_disk``.  Real HF datasets
are accepted everywhere too; this class exists because the GPU machines are offline."""
from __future__ import annotations

import os
import pickle
from typing import Any, Callable, Dict, Iterable, List, Optional, Sequence

import numpy as np
import torch

__all__ = ["TokenDataset", "load_from_disk"]


class TokenDataset:
    def __init__(self, columns: Dict[str, Sequence[Any]]):
        lens = {len(v) for v in columns.values()}
        if len(lens) > 1:
            raise ValueError(f"columns have different lengths: { {k: len(v) for k, v in columns.items()} }")
        self._cols: Dict[str, List[Any]] = {k: list(v) if not isinstance(v, (torch.Tensor, np.ndarray)) else v for k, v in columns.items()}
        self._n = lens.pop() if lens else 0

    # -- construction ------------------------------------------------------------------
    @classmethod
    def from_dict(cls, d: Dict[str, Sequence[Any]]) -> "TokenDataset":
        return cls(d)

    @property
    def column_names(self) -> List[str]:
        return list(self._cols.keys())

    def __len__(self) -> int:
        return self._n

    def __getitem__(self, i):
        if isinstance(i, str):
            return self._cols[i]
        if isinstance(i, slice):
            return {k: v[i] for k, v in self._cols.items()}
        return {k: v[i] for k, v in self._cols.items()}

    def __iter__(self):
        for i in range(self._n):
            yield self[i]

    def select(self, indices: Iterable[int]) -> "TokenDataset":
        idx = list(indices)
        out = {}
        for k, v in self._cols.items():
            if isinstance(v, torch.Tensor):
                out[k] = v[torch.as_tensor(idx, dtype=torch.long)]
            elif isinstance(v, np.ndarray):
                out[k] = v[np.asarray(idx, dtype=np.int64)]
            else:
                out[k] = [v[j] for j in idx]
        return TokenDataset(out)

    # -- HF-like transforms ------------------------------------------------------------
    def shard(self, num_shards: int, index: int, contiguous: bool = False) -> "TokenDataset":
        """Rank ``index`` of ``num_shards``.  Like HF's default this is strided
        (``index, index + num_shards, ...``) unless ``contiguous``."""
        if contiguous:
            per = (self._n + num_shards - 1) // num_shards
            return self.select(range(index * per, min((index + 1) * per, self._n)))
        return self.select(range(index, self._n, num_shards))

    def map(self, fn: Callable, batched: bool = False, remove_columns: Optional[Sequence[str]] = None,
            num_proc: Optional[int] = None, batch_size: int = 1000, **_) -> "TokenDataset":
        remove = set(remove_columns or [])
        out: Dict[str, List[Any]] = {}
        if batched:
            for s in range(0, max(self._n, 1), batch_size):
                if s >= self._n:
                    break
                batch = {k: v[s: s + batch_size] for k, v in self._cols.items()}
                res = fn(batch)
                keep = {k: v for k, v in batch.items() if k not in remove and k not in res}
                n_res = len(next(iter(res.values()))) if res else 0
                for k, v in res.items():
                    out.setdefault(k, []).extend(list(v))
                for k, v in keep.items():
                    if len(v) == n_res:
                        out.setdefault(k, []).extend(list(v))
        else:
            for i in range(self._n):
                row = self[i]
                res = fn(row)
                merged = {k: v for k, v in row.items() if k not in remove}
                merged.update(res)
                for k, v in merged.items():
                    out.setdefault(k, []).append(v)
        return TokenDataset(out)

    def train_test_split(self, test_size: float = 0.05, seed: int = 42, shuffle: bool = True) -> Dict[str, "TokenDataset"]:
        n_test = int(round(self._n * test_size)) if test_size < 1 else int(test_size)
        n_test = min(max(n_test, 1 if self._n > 1 else 0), self._n)
        rng = np.random.default_rng(seed)
        perm = rng.permutation(self._n) if shuffle else np.arange(self._n)
        return {"train": self.select(perm[n_test:].tolist()), "test": self.select(perm[:n_test].tolist())}

    # -- persistence (dl_dataset.py parity) ---------------------------------------------
    def save_to_disk(self, path: str) -> None:
        os.makedirs(path, exist_ok=True)
        with open(os.path.join(path, "token_dataset.pkl"), "wb") as f:
            pickle.dump(self._cols, f, protocol=4)


def load_from_disk(path: str) -> TokenDataset:
    with open(os.path.join(path, "token_dataset.pkl"), "rb") as f:
        return TokenDataset(pickle.load(f))
