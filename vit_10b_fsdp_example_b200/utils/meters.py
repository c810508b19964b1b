"""Windowed meters and device timers (reference: utils.py:60-102 SmoothedValue)."""
from __future__ import annotations

import statistics
from collections import deque


class SmoothedValue:
    """Sliding-window statistics over the last ``window_size`` updates plus a global average.

    Same public surface as the reference meter (update / avg / median / global_avg / get_latest).
    """

    def __init__(self, window_size: int = 20):
        self.window_size = window_size
        self.reset()

    def reset(self) -> None:
        self._weighted = deque(maxlen=self.window_size)
        self._values = deque(maxlen=self.window_size)
        self._weights = deque(maxlen=self.window_size)
        self.total = 0.0
        self.total_samples = 0
        self.count = 0

    def update(self, value: float, batch_size: int = 1) -> None:
        value = float(value)
        self._weighted.append(value * batch_size)
        self._values.append(value)
        self._weights.append(batch_size)
        self.total += value * batch_size
        self.total_samples += batch_size
        self.count += 1

    @property
    def avg(self) -> float:
        return sum(self._weighted) / sum(self._weights)

    @property
    def median(self) -> float:
        return statistics.median(self._values)

    @property
    def global_avg(self) -> float:
        return self.total / self.total_samples

    def get_latest(self) -> float:
        return self._values[-1]


class DeviceTimer:
    """CUDA-event step timer (host clock on CPU).  ``elapsed_ms`` synchronises on the end event only."""

    def __init__(self, device):
        import torch

        self._torch = torch
        self.cuda = device.type == "cuda"
        if self.cuda:
            self._start = torch.cuda.Event(enable_timing=True)
            self._end = torch.cuda.Event(enable_timing=True)
        self._t0 = 0.0
        self._t1 = 0.0

    def start(self) -> None:
        if self.cuda:
            self._start.record()
        else:
            import time

            self._t0 = time.perf_counter()

    def stop(self) -> None:
        if self.cuda:
            self._end.record()
        else:
            import time

            self._t1 = time.perf_counter()

    def elapsed_ms(self) -> float:
        if self.cuda:
            self._end.synchronize()
            return self._start.elapsed_time(self._end)
        return (self._t1 - self._t0) * 1e3
