"""CUDA-graph capture of one micro-batch (forward + backward + loss read-out).

The reference launches ~1.8 k eager kernels per micro-batch from Python and left
``#@torch.compile`` / "static memory" stubs behind (`trainer_decoupled.py:17,199-200,386-397`).  A 125M-parameter micro-batch is a few tens of ms of GPU work
split over ~1.5 k kernels, so launch overhead is first-order; here the whole micro-batch is captured once per
``(parameter buffer, gradient accumulator)`` pair - two graphs cover the ACCO double-buffer
schedule - and replayed with a single ``cudaGraphLaunch``.  Gradients accumulate *inside* the
graph into the flat arena (pointer-stable), inputs arrive in static device buffers filled by an
async H2D copy from pinned memory.
"""
from __future__ import annotations

from typing import Callable, Dict, Optional, Tuple

import torch

__all__ = ["MicroBatchGraphs"]


class MicroBatchGraphs:
    def __init__(self, step_fn: Callable[[Dict[str, torch.Tensor]], torch.Tensor], device: torch.device,
                 warmup_iters: int = 2):
        """``step_fn(inputs) -> loss`` must run forward+backward and return the (detached) loss."""
        self.step_fn = step_fn
        self.device = torch.device(device)
        self.warmup_iters = warmup_iters
        self._graphs: Dict[Tuple, torch.cuda.CUDAGraph] = {}
        self._static_in: Dict[Tuple, Dict[str, torch.Tensor]] = {}
        self._static_loss: Dict[Tuple, torch.Tensor] = {}
        self._kernels: Dict[Tuple, int] = {}
        self._pool = None

    @staticmethod
    def signature(inputs: Dict[str, torch.Tensor]) -> Tuple:
        return tuple(sorted((k, tuple(v.shape), str(v.dtype)) for k, v in inputs.items()))

    def has(self, key: Tuple) -> bool:
        return key in self._graphs

    def static_inputs(self, key: Tuple) -> Dict[str, torch.Tensor]:
        return self._static_in[key]

    def capture(self, key: Tuple, example: Dict[str, torch.Tensor], cleanup: Optional[Callable[[], None]] = None) -> None:
        """Warm up eagerly on a side stream, then capture.  ``cleanup`` is called after the
        warm-up iterations (which really accumulate gradients) so the caller can re-zero them."""
        from .. import ops
        static = {k: torch.empty_like(v, device=self.device) for k, v in example.items()}
        for k, v in example.items():
            static[k].copy_(v)
        side = torch.cuda.Stream(device=self.device)
        side.wait_stream(torch.cuda.current_stream(self.device))
        with torch.cuda.stream(side):
            for _ in range(self.warmup_iters):
                self.step_fn(static)
        torch.cuda.current_stream(self.device).wait_stream(side)
        torch.cuda.synchronize(self.device)
        g = torch.cuda.CUDAGraph()
        before = ops.total_launches()
        kw = {"pool": self._pool} if self._pool is not None else {}
        # thread_local: the feeder thread keeps pinning host batches (cudaHostAlloc) while this thread captures; under the default
        # "global" mode that unrelated call is an error that also invalidates the capture
        with torch.cuda.graph(g, capture_error_mode="thread_local", **kw):
            loss = self.step_fn(static)
            static_loss = loss.detach().reshape(1).float().clone()
        self._kernels[key] = ops.total_launches() - before
        if self._pool is None:
            self._pool = g.pool()
        torch.cuda.synchronize(self.device)
        if cleanup is not None:
            cleanup()
        self._graphs[key], self._static_in[key], self._static_loss[key] = g, static, static_loss

    def replay(self, key: Tuple, host_or_dev_inputs: Dict[str, torch.Tensor]) -> torch.Tensor:
        """Copy inputs into the static buffers (async if the source is pinned) and replay."""
        from .. import ops
        static = self._static_in[key]
        for k, v in host_or_dev_inputs.items():
            static[k].copy_(v, non_blocking=True)
        self._graphs[key].replay()
        ops.count_launch("graph_replay_kernels", self._kernels.get(key, 0))
        return self._static_loss[key]
