"""Metrics / logging / observability.

Parity (reference): TB scalars ``cross_entropy`` / ``accuracy`` (+ ``weight_decay_loss`` / ``total_loss``)
written at eval steps to ``<ckpt dir>/train`` (original src/rnn.py:65-68,91,249-250,276-280); tqdm bar
with ``Loss/t_acc`` description (:257,270-271,291-292); the human-readable timing lines (:296,410).
New: CUDA-event device timing, NVTX ranges, JSON lines.
"""
from __future__ import annotations

import contextlib
import json
import os
import time
from typing import Dict, List, Optional

import torch

_ACTIVE: Optional["SummarySink"] = None


class SummarySink:
    """Collects scalars emitted by ``compute_loss`` / ``compute_accuracy`` while active and writes them
    as TensorBoard events under ``logdir`` (the reference's ``tf.summary.FileWriter``)."""

    def __init__(self, logdir: Optional[str] = None):
        self.logdir = logdir
        self.pending: Dict[str, float] = {}
        self.writer = None
        if logdir:
            os.makedirs(logdir, exist_ok=True)
            try:
                from torch.utils.tensorboard import SummaryWriter
                self.writer = SummaryWriter(log_dir=logdir)
            except Exception:                      # tensorboard missing: keep a jsonl of the same scalars
                self.writer = None
            self._jsonl = open(os.path.join(logdir, "scalars.jsonl"), "a")
        else:
            self._jsonl = None

    def add(self, tag: str, value):
        self.pending[tag] = float(value.detach().float().item() if torch.is_tensor(value) else value)

    def flush(self, step: int):
        for tag, v in self.pending.items():
            if self.writer is not None:
                self.writer.add_scalar(tag, v, step)
        if self._jsonl is not None and self.pending:
            self._jsonl.write(json.dumps({"step": step, **self.pending}) + "\n")
            self._jsonl.flush()
        if self.writer is not None:
            self.writer.flush()
        out, self.pending = self.pending, {}
        return out

    def close(self):
        if self.writer is not None:
            self.writer.close()
        if self._jsonl is not None:
            self._jsonl.close()


@contextlib.contextmanager
def capture(sink: SummarySink):
    global _ACTIVE
    prev, _ACTIVE = _ACTIVE, sink
    try:
        yield sink
    finally:
        _ACTIVE = prev


def scalar(tag: str, value):
    if _ACTIVE is not None:
        _ACTIVE.add(tag, value)


# -------------------------------------------------------------------------------------------------
class DeviceTimer:
    """CUDA-event timing on the launching stream (wall clock on CPU)."""

    def __init__(self, device):
        self.cuda = torch.device(device).type == "cuda"
        self.t0 = None

    def start(self):
        if self.cuda:
            self.e0 = torch.cuda.Event(enable_timing=True)
            self.e1 = torch.cuda.Event(enable_timing=True)
            self.e0.record()
        else:
            self.t0 = time.perf_counter()

    def stop_ms(self) -> float:
        if self.cuda:
            self.e1.record()
            self.e1.synchronize()
            return self.e0.elapsed_time(self.e1)
        return (time.perf_counter() - self.t0) * 1e3


class LaggedScalar:
    """Per-step scalar for the progress bar without a per-step host sync: on CUDA the value is copied into a pinned
    buffer asynchronously and the PREVIOUS step's value is returned (its copy has long finished); on the CPU it is exact.
    (The reference's ``sess.run([train_op, loss])`` blocks on the loss every step, original src/rnn.py:264-271.)"""

    def __init__(self, device):
        self.cuda = torch.device(device).type == "cuda"
        self.last = float("nan")
        if self.cuda:
            self.host = torch.empty(2, dtype=torch.float32, pin_memory=True)
            self.evt = [torch.cuda.Event(), torch.cuda.Event()]
            self.k = 0

    def push(self, value: torch.Tensor) -> float:
        if not self.cuda:
            self.last = float(value.detach().float().item())
            return self.last
        k = self.k
        self.host[k & 1].copy_(value.detach().float(), non_blocking=True)
        self.evt[k & 1].record()
        if k > 0:
            self.evt[(k - 1) & 1].synchronize()
            self.last = float(self.host[(k - 1) & 1])
        self.k = k + 1
        return self.last


@contextlib.contextmanager
def nvtx_range(name: str, enabled: bool = True):
    on = enabled and torch.cuda.is_available()
    if on:
        torch.cuda.nvtx.range_push(name)
    try:
        yield
    finally:
        if on:
            torch.cuda.nvtx.range_pop()


class JsonLog:
    def __init__(self, path: str = ""):
        self.f = open(path, "a") if path else None

    def write(self, **kw):
        if self.f:
            self.f.write(json.dumps(kw) + "\n")
            self.f.flush()

    def close(self):
        if self.f:
            self.f.close()
