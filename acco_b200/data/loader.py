"""Batch loading: random sampling with ``drop_last`` (`trainer_base.py:203-218`), an *endless*
iterator that restarts epochs (`trainer_decoupled.py:386-397`), pinned staging buffers and an
asynchronous host->device copy on a side stream (the reference does a synchronous ``.to()`` per
micro-batch).

The producer is a background thread (collation of in-memory token rows is cheap and releases the
GIL inside numpy/torch); it keeps ``prefetch`` batches ahead, each already resident in pinned
memory, so the training loop's per-step host cost is one ``cudaMemcpyAsync`` + one event wait.
With ``num_workers >= 2`` (the reference's ``dataloader_num_workers`` / ``persistent_workers`` keys,
`trainer_base.py:203-218`) row fetching + collation fan out to that many persistent worker *processes*
(``torch.utils.data.DataLoader`` driven by this loader's own epoch order), which is what a real HF
dataset with on-the-fly tokenisation needs at ~1 M tokens/s per GPU; the thread then only pins and queues."""
from __future__ import annotations

import queue
import threading
import weakref
from typing import Callable, Dict, Iterator

import numpy as np
import torch

__all__ = ["BatchLoader", "DeviceFeeder"]


class BatchLoader:
    """Finite, re-iterable loader: one epoch per ``__iter__`` (shuffled with a fresh permutation)."""

    def __init__(self, dataset, batch_size: int, collate_fn: Callable, shuffle: bool = True, drop_last: bool = True,
                 seed: int = 0, group_by_length: bool = False, mega_batch_mult: int = 50):
        """``group_by_length``: like HF's ``LengthGroupedSampler`` (vendored but unused in the reference,
        `utils/trainer_utils.py:940`): shuffle, cut into mega-batches of ``mega_batch_mult * batch_size`` rows, sort each
        by length (longest first) so that padded SFT batches contain rows of similar length."""
        self.dataset, self.batch_size, self.collate_fn = dataset, int(batch_size), collate_fn
        self.shuffle, self.drop_last = shuffle, drop_last
        self.group_by_length, self.mega = bool(group_by_length), int(mega_batch_mult) * int(batch_size)
        self._lengths = None
        self._rng = np.random.default_rng(seed)
        self._skip = 0                  # batches to drop at the start of the next epoch (set by `fast_forward`)

    def __len__(self) -> int:
        n = len(self.dataset)
        return n // self.batch_size if self.drop_last else (n + self.batch_size - 1) // self.batch_size

    def fast_forward(self, n_batches: int) -> None:
        """Position the loader where a run that has already consumed ``n_batches`` batches would be (resume): whole epochs burn
        one permutation each (same random stream as the original run), the remainder is skipped at the index level when the next
        epoch starts - no row is fetched or collated for it."""
        per = len(self)
        if per <= 0 or n_batches <= 0:
            return
        for _ in range(int(n_batches) // per):
            if self.shuffle:
                self._rng.permutation(len(self.dataset))
        self._skip = int(n_batches) % per

    def __iter__(self) -> Iterator[Dict[str, torch.Tensor]]:
        for idx in self.index_batches():
            yield self.collate_fn([self.dataset[int(i)] for i in idx])

    def index_batches(self) -> Iterator[np.ndarray]:
        """Row indices of every batch of ONE epoch (fresh permutation per call)."""
        n = len(self.dataset)
        order = self._rng.permutation(n) if self.shuffle else np.arange(n)
        if self.group_by_length:
            if self._lengths is None:
                self._lengths = np.asarray([len(self.dataset[int(i)]["input_ids"]) for i in range(n)], dtype=np.int64)
            chunks = [order[s: s + self.mega] for s in range(0, n, self.mega)]
            chunks = [c[np.argsort(-self._lengths[c], kind="stable")] for c in chunks]
            # like HF: put the globally longest row first so an OOM shows up in the very first batch
            if chunks:
                k = int(np.argmax([self._lengths[c[0]] for c in chunks]))
                chunks[0], chunks[k] = chunks[k], chunks[0]
            order = np.concatenate(chunks) if chunks else order
        stop = (n // self.batch_size) * self.batch_size if self.drop_last else n
        start, self._skip = self._skip * self.batch_size, 0
        for s in range(start, stop, self.batch_size):
            yield order[s: s + self.batch_size]

    def worker_loader(self, num_workers: int, persistent: bool = True, prefetch_factor: int = 4):
        """``torch.utils.data.DataLoader`` over the same dataset / collator / epoch order with ``num_workers`` processes."""
        outer = self

        class _EpochBatches(torch.utils.data.Sampler):
            def __iter__(self_inner):
                for idx in outer.index_batches():
                    yield [int(i) for i in idx]

            def __len__(self_inner):
                return len(outer)

        return torch.utils.data.DataLoader(self.dataset, batch_sampler=_EpochBatches(), collate_fn=self.collate_fn, num_workers=int(num_workers),
                                           persistent_workers=bool(persistent), prefetch_factor=int(prefetch_factor))


class DeviceFeeder:
    """Endless stream of device-resident batches with background collation + async H2D."""

    def __init__(self, loader: BatchLoader, device: torch.device, prefetch: int = 4, pin: bool = True, num_workers: int = 0,
                 persistent_workers: bool = True):
        if len(loader) == 0:
            raise ValueError("dataset shard is smaller than one batch (drop_last=True leaves nothing to train on)")
        self.loader, self.device = loader, torch.device(device)
        self.num_workers = int(num_workers) if int(num_workers) >= 2 else 0      # <= 1: this feeder thread IS the worker
        self._source = loader.worker_loader(self.num_workers, persistent_workers) if self.num_workers else loader
        self.cuda = self.device.type == "cuda"
        self.pin = pin and self.cuda
        self.epochs = 0
        self.h2d_bytes = 0
        self.tokens_real = 0            # non-pad tokens handed out so far (attention-mask sum; full batches when there is no mask)
        self.batches_out = 0            # batches handed to the consumer (NOT the producer's position: it runs `prefetch` ahead)
        self._q: "queue.Queue" = queue.Queue(maxsize=max(prefetch, 1))
        self._stop = threading.Event()
        self._copy_stream = torch.cuda.Stream(device=self.device) if self.cuda else None
        self._thread = threading.Thread(target=self._produce, name="acco-feeder", daemon=True)
        self._thread.start()
        self._finalizer = weakref.finalize(self, DeviceFeeder._shutdown, self._stop, self._q, self._thread)

    def _produce(self) -> None:
        try:
            while not self._stop.is_set():
                for batch in self._source:
                    m = batch.get("attention_mask")
                    ntok = int(m.sum()) if m is not None else int(batch["input_ids"].numel())      # on the host, before the copy
                    if self.pin:
                        batch = {k: v.pin_memory() for k, v in batch.items()}
                    while not self._stop.is_set():
                        try:
                            self._q.put((batch, ntok), timeout=0.1)
                            break
                        except queue.Full:
                            continue
                    if self._stop.is_set():
                        return
                self.epochs += 1
        except BaseException as e:  # surface errors in the consumer
            self._q.put(e)

    def next_host(self) -> Dict[str, torch.Tensor]:
        """Next batch still on the host (pinned when feeding a GPU); the caller issues the H2D copy
        (e.g. straight into a CUDA graph's static input buffers)."""
        item = self._q.get()
        if isinstance(item, BaseException):
            raise item
        item, ntok = item
        self.tokens_real += ntok
        self.batches_out += 1
        if self.cuda:
            self.h2d_bytes += sum(v.numel() * v.element_size() for v in item.values())
        return item

    def next(self) -> Dict[str, torch.Tensor]:
        item = self._q.get()
        if isinstance(item, BaseException):
            raise item
        item, ntok = item
        self.tokens_real += ntok
        self.batches_out += 1
        if not self.cuda:
            return item
        self.h2d_bytes += sum(v.numel() * v.element_size() for v in item.values())
        cur = torch.cuda.current_stream(self.device)
        with torch.cuda.stream(self._copy_stream):
            dev = {k: v.to(self.device, non_blocking=True) for k, v in item.items()}
        cur.wait_stream(self._copy_stream)
        for v in dev.values():
            v.record_stream(cur)
        return dev

    __next__ = next

    def __iter__(self):
        return self

    def close(self) -> None:
        """Stop the producer and WAIT for it: a daemon thread that is still inside torch / numpy code when the interpreter
        finalises aborts the process (`terminate called without an active exception`, exit code 134 - a finished training job
        would look like a crashed one to torchrun / Slurm).  Also runs at interpreter exit through `weakref.finalize`."""
        self._finalizer()

    @staticmethod
    def _shutdown(stop: threading.Event, q: "queue.Queue", thread: threading.Thread) -> None:
        stop.set()
        deadline = 50                                    # the producer re-checks `stop` every 0.1 s while the queue is full
        while thread.is_alive() and deadline > 0:
            try:
                while True:
                    q.get_nowait()                       # make room so that a blocked put() returns
            except queue.Empty:
                pass
            if thread is threading.current_thread():
                break
            thread.join(timeout=0.1)
            deadline -= 1
