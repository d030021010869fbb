"""Device-side timing and overlap accounting (the reference only has ``time.time()``).

:class:`CudaTimer` brackets a region with CUDA events on a stream and resolves lazily (no
host sync at record time).  :class:`OverlapMeter` accumulates, per round, how long the compute
stream had to *wait* for the communication round - the "exposed communication" the north star
wants driven to zero."""
from __future__ import annotations

import contextlib
import time
from typing import Dict, List, Optional

import torch

__all__ = ["CudaTimer", "OverlapMeter", "nvtx_range"]


@contextlib.contextmanager
def nvtx_range(name: str):
    if torch.cuda.is_available():
        torch.cuda.nvtx.range_push(name)
        try:
            yield
        finally:
            torch.cuda.nvtx.range_pop()
    else:
        yield


class CudaTimer:
    def __init__(self, enabled: bool = True):
        self.enabled = enabled and torch.cuda.is_available()
        self._pairs: List = []
        self._cpu: List[float] = []
        self._t0: Optional[float] = None
        self._e0 = None

    def start(self, stream=None) -> None:
        if self.enabled:
            self._e0 = torch.cuda.Event(enable_timing=True)
            self._e0.record(stream)
        else:
            self._t0 = time.perf_counter()

    def stop(self, stream=None) -> None:
        if self.enabled:
            e1 = torch.cuda.Event(enable_timing=True)
            e1.record(stream)
            self._pairs.append((self._e0, e1))
        else:
            self._cpu.append((time.perf_counter() - self._t0) * 1e3)

    def resolve_ms(self) -> List[float]:
        """Durations of all completed regions (synchronises on the last event)."""
        if self.enabled:
            out = []
            for a, b in self._pairs:
                b.synchronize()
                out.append(a.elapsed_time(b))
            return out
        return list(self._cpu)

    def total_ms(self) -> float:
        return float(sum(self.resolve_ms()))

    def reset(self) -> None:
        self._pairs.clear()
        self._cpu.clear()


class OverlapMeter:
    """Per-round record of (comm duration, exposed wait) in ms, resolved lazily.  Completed event pairs are folded into
    running sums once more than ``window`` are pending, so a 50 000-round run does not hold 200 000 CUDA events."""

    def __init__(self, enabled: bool = True, window: int = 256, keep_history: bool = False):
        self.enabled = enabled and torch.cuda.is_available()
        self.window = window
        # keep_history (`save_com_logs`): per-round durations in launch order, like the per-rank communication history the reference's
        # authors dumped in their experiments (`utils/logs_utils.py:141` save_com_logs - unused in the shipped code)
        self.comm_history: Optional[List[float]] = [] if keep_history else None
        self.wait_history: Optional[List[float]] = [] if keep_history else None
        self._comm: List = []     # (start_evt, end_evt) on the comm stream
        self._wait: List = []     # (before_wait_evt, after_wait_evt) on the compute stream
        self._comm_sum, self._comm_n, self._wait_sum, self._wait_n = 0.0, 0, 0.0, 0

    def _fold(self, pairs: List, final: bool = False, sink: Optional[List[float]] = None):
        keep, s, n = [], 0.0, 0
        for a, b in pairs:
            if b.query():
                ms = a.elapsed_time(b)
                s += ms
                n += 1
                if sink is not None:
                    sink.append(ms)
            elif not final:
                keep.append((a, b))
        return keep, s, n

    def _maybe_fold(self) -> None:
        if len(self._comm) > self.window:
            self._comm, s, n = self._fold(self._comm, sink=self.comm_history)
            self._comm_sum += s
            self._comm_n += n
        if len(self._wait) > self.window:
            self._wait, s, n = self._fold(self._wait, sink=self.wait_history)
            self._wait_sum += s
            self._wait_n += n

    def comm_events(self):
        if not self.enabled:
            return None, None
        self._maybe_fold()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        self._comm.append((a, b))
        return a, b

    def wait_events(self):
        if not self.enabled:
            return None, None
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        self._wait.append((a, b))
        return a, b

    def summary(self) -> Dict[str, float]:
        if not self.enabled or (not self._comm and not self._comm_n):
            return {"rounds": 0, "comm_ms_mean": 0.0, "exposed_ms_mean": 0.0, "exposed_ms_total": 0.0}
        torch.cuda.synchronize()
        if self.comm_history is not None:
            # history mode: fold the completed pairs for good, so that no pair is appended to the history twice
            self._comm, cs0, cn0 = self._fold(self._comm, sink=self.comm_history)
            self._wait, ws0, wn0 = self._fold(self._wait, sink=self.wait_history)
            self._comm_sum, self._comm_n, self._wait_sum, self._wait_n = self._comm_sum + cs0, self._comm_n + cn0, self._wait_sum + ws0, self._wait_n + wn0
            cs, cn, ws, wn = 0.0, 0, 0.0, 0
        else:
            _, cs, cn = self._fold(self._comm, final=True)
            _, ws, wn = self._fold(self._wait, final=True)
        cs, cn, ws, wn = cs + self._comm_sum, cn + self._comm_n, ws + self._wait_sum, wn + self._wait_n
        return {
            "rounds": cn,
            "comm_ms_mean": cs / max(cn, 1),
            "exposed_ms_mean": ws / max(wn, 1),
            "exposed_ms_total": ws,
        }

    def reset(self) -> None:
        self._comm.clear()
        self._wait.clear()
        self._comm_sum, self._comm_n, self._wait_sum, self._wait_n = 0.0, 0, 0.0, 0
