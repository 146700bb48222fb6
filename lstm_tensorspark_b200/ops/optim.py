"""Flat-buffer optimizers.

Reference: ``tf.train.AdamOptimizer(learning_rate)`` with TF defaults (beta1 .9, beta2 .999, eps 1e-8,
"epsilon-hat" formulation), one ``ApplyAdam`` kernel per variable, injectable via ``train_optimizer``
(original src/rnn.py:180,207,224).  ``asgd`` / ``ntasgd`` are AWD-LSTM's averaged SGD (Merity et al. 2017): the SGD update plus
a running average ``ax`` of the iterates, fused into the same launch.  Here: ONE launch over the flat fp32 master buffer that also
refreshes the bf16 shadow the tensor-core kernels read (csrc/multi_tensor_opt.cu); on the CPU the same
math runs through ops/reference.py.  In ``grad_allreduce`` mode on GPUs the update is not launched here at
all — it is fused into the in-kernel NVLink allreduce (parallel/fused_comm.py).
"""
from __future__ import annotations

import warnings
from typing import Optional, Sequence

import torch

from ..models.flat import FlatParams
from . import reference as ref
from . import functional as F


KINDS = ("adam", "sgd", "asgd", "ntasgd")


def nonmono_trigger(history: Sequence[float], v: float, n: int, averaging: bool) -> bool:
    """NT-ASGD's non-monotone trigger (AWD-LSTM ``main.py``: ``len(h) > n and v > min(h[:-n])``): switch averaging on when the
    validation loss ``v`` is worse than the best of the validations before the last ``n`` ones (``history``: the earlier
    validation losses, oldest first).  Never fires while averaging is already on, nor on a NaN loss."""
    if averaging or n < 1 or len(history) <= n or v != v:
        return False
    return v > min(history[:-n])


class FlatOptimizer:
    def __init__(self, flat: FlatParams, lr: float, kind: str = "adam", beta1: float = 0.9, beta2: float = 0.999,
                 eps: float = 1e-8, weight_decay: float = 0.0):
        self.flat = flat
        self.kind = kind
        self.lr, self.beta1, self.beta2, self.eps, self.weight_decay = lr, beta1, beta2, eps, weight_decay
        self.wd_numel = -1          # weight decay covers flat elements [0, wd_numel); -1 = all (K12: the LSTM variables only)
        self.clip_out = None        # clipping: {norm, coef} of the last step (fp32 [2], on the flat buffer's device)
        self.clip_scratch = None    # the norm kernel's fp64 CTA partials and ticket (allocated by its first launch)
        self.clip_norm = 0.0
        self.step_count = 0
        # device-resident mirror of step_count: the Adam kernels derive the bias correction from it, so a captured
        # CUDA graph of the training step stays exact across replays
        self.step_dev = torch.zeros(1, dtype=torch.int32, device=flat.data.device) if flat.data.is_cuda else None
        if kind not in KINDS:
            raise ValueError(f"unknown optimizer {kind!r}")
        self.m = torch.zeros_like(flat.data) if kind == "adam" else None
        self.v = torch.zeros_like(flat.data) if kind == "adam" else None
        # asgd / ntasgd: ax, the average of the iterates since averaging started, and avg = int32 {on, k} on the flat buffer's
        # device: the update bumps k before it averages when on, so a captured graph stays exact across replays, and switching
        # averaging on is a fill_ outside the graph.  asgd averages from the first step; ntasgd once start_averaging() is called.
        # nonmono_history: the validation losses the trigger has seen
        self.ax = self.avg = None
        self.nonmono_history = []
        if kind in ("asgd", "ntasgd"):
            self.ax = torch.zeros_like(flat.data)
            self.avg = torch.tensor([1 if kind == "asgd" else 0, 0], dtype=torch.int32, device=flat.data.device)

    @property
    def averaging(self) -> bool:
        """Averaging is on (reads the device pair: a host synchronisation on the GPU)."""
        return self.avg is not None and bool(int(self.avg[0]))

    @property
    def averaged_steps(self) -> int:
        """k: the updates averaged into ``ax`` since averaging started (0 without averaging)."""
        return 0 if self.avg is None else int(self.avg[1])

    def has_average(self) -> bool:
        """``ax`` holds an average (averaging on and k >= 1): evaluation then uses it instead of the raw weights."""
        if self.avg is None:
            return False
        on, k = (int(v) for v in self.avg.tolist())
        return bool(on) and k >= 1

    def start_averaging(self) -> None:
        """Switch averaging on from a fresh average (k restarts at 0; the next update copies its weights into ``ax``)."""
        self.avg.copy_(torch.tensor([1, 0], dtype=torch.int32))

    def average_(self) -> None:
        """The averaging half of an update whose SGD half ran elsewhere (the fused allreduce's bucket kernels): bump k when on,
        then ``ax`` += (p - ax) * mu_k over the whole buffer."""
        if self.avg is None:
            return
        if self.flat.data.is_cuda and F.get_backend() != "torch":
            from .cuda_ext import ext
            ext().flat_average(self.flat.data, self.ax, self.avg)
            return
        with torch.no_grad():
            if int(self.avg[0]):
                self.avg[1] += 1
                ref.asgd_average_(self.ax, self.flat.data, int(self.avg[1]))

    def swap_average(self) -> None:
        """Exchange the weights and ``ax`` in place and refresh the bf16 shadow from the new weights; twice is the identity."""
        fl = self.flat
        if fl.data.is_cuda and F.get_backend() != "torch":
            from .cuda_ext import ext
            ext().flat_swap(fl.data, self.ax, fl.shadow)
            return
        with torch.no_grad():
            tmp = fl.data.clone()
            fl.data.copy_(self.ax)
            self.ax.copy_(tmp)
            fl.refresh_shadow()

    @property
    def wd_numel(self) -> int:
        """Weight decay covers flat elements ``[0, wd_numel)``; -1 = all.  The update kernels choose the decay per float4, so
        the cut is a multiple of 4 (``FlatParams.lstm_numel`` is one of ``ALIGN``)."""
        return self._wd_numel

    @wd_numel.setter
    def wd_numel(self, value: int):
        value = int(value)
        if value < -1 or (value >= 0 and value % 4):
            raise ValueError(f"wd_numel must be -1 or a non-negative multiple of 4, got {value}")
        self._wd_numel = value

    @property
    def clip_norm(self) -> float:
        """Clip the gradient by its global norm to this value before the update (0 = off).  The norm is that of the gradient
        the update uses - ``g * grad_scale`` plus the weight-decay term over ``[0, wd_numel)`` - and the update uses
        ``coef * g`` with ``coef = min(clip_norm / (norm + 1e-6), 1)``; ``clip_out`` holds {norm, coef} of the last step."""
        return self._clip_norm

    @clip_norm.setter
    def clip_norm(self, value: float):
        self._clip_norm = float(value)
        if self._clip_norm > 0 and self.clip_out is None:
            self.clip_out = torch.zeros(2, dtype=torch.float32, device=self.flat.data.device)

    def minimize(self, loss: torch.Tensor):
        """``optimizer.minimize(loss)`` of the reference: backward + apply."""
        self.flat.zero_grad()
        loss.backward()
        self.step()

    def step(self, grad_scale: float = 1.0):
        self.step_count += 1
        fl = self.flat
        if fl.data.is_cuda and F.get_backend() != "torch":
            from . import cuda_opt
            cuda_opt.flat_step(self, grad_scale)
            return
        with torch.no_grad():
            n = fl.data.numel()
            cut = n if (self.wd_numel < 0 or not self.weight_decay) else min(self.wd_numel, n)
            segs = [(lo, hi, wd) for lo, hi, wd in ((0, cut, self.weight_decay), (cut, n, 0.0)) if hi > lo]
            coef = None
            if self.clip_norm > 0:
                g_total = [fl.grad[lo:hi] * grad_scale + wd * fl.data[lo:hi] if wd else fl.grad[lo:hi] * grad_scale
                           for lo, hi, wd in segs]
                norm, coef = ref.clip_coefficient(g_total, self.clip_norm)
                self.clip_out[0], self.clip_out[1] = norm, coef
            for lo, hi, wd in segs:
                if self.kind == "adam":
                    ref.adam_step_(fl.data[lo:hi], fl.grad[lo:hi], self.m[lo:hi], self.v[lo:hi], self.step_count, self.lr,
                                   self.beta1, self.beta2, self.eps, wd, grad_scale, coef)
                else:
                    ref.sgd_step_(fl.data[lo:hi], fl.grad[lo:hi], self.lr, wd, grad_scale, coef)
            fl.refresh_shadow()
        self.average_()

    def bias_corrected_lr(self, step: Optional[int] = None) -> float:
        t = self.step_count if step is None else step
        if self.kind != "adam":
            return self.lr
        return self.lr * (1.0 - self.beta2 ** t) ** 0.5 / (1.0 - self.beta1 ** t)

    def state_dict(self):
        sd = {"kind": self.kind, "step": self.step_count, "lr": self.lr,
              "m": None if self.m is None else self.m.detach().cpu(),
              "v": None if self.v is None else self.v.detach().cpu()}
        if self.ax is not None:
            on, k = (int(v) for v in self.avg.tolist())
            sd.update(ax=self.ax.detach().cpu().clone(), on=on, k=k, nonmono_history=list(self.nonmono_history))
        return sd

    def load_state_dict(self, sd):
        """Adam's m / v, and the average: an ``asgd`` / ``ntasgd`` state continues where it stopped; a state without one (an
        ``sgd`` checkpoint) leaves this optimizer's average as it starts (asgd: on from a fresh average; ntasgd: off, with no
        trigger history), and so does an ``ntasgd`` state whose trigger has not fired when loaded into ``asgd`` (its history is
        kept); an average loaded into ``sgd`` / ``adam`` is dropped with a warning."""
        self.step_count = int(sd["step"])
        if self.step_dev is not None:
            self.step_dev.fill_(self.step_count)
        if self.m is not None and sd.get("m") is not None:
            self.m.copy_(sd["m"].to(self.m.device))
            self.v.copy_(sd["v"].to(self.v.device))
        if sd.get("ax") is None:
            return
        if self.ax is None:
            warnings.warn(f"the optimizer state holds a weight average of {int(sd.get('k', 0))} steps; --optimizer {self.kind} "
                          "does not average, so it is dropped (training continues from the raw weights)")
            return
        self.nonmono_history = [float(v) for v in sd.get("nonmono_history", [])]
        if self.kind == "asgd" and not int(sd["on"]):
            return                              # an ntasgd state whose trigger never fired: asgd averages afresh from here
        self.ax.copy_(sd["ax"].to(self.ax.device))
        self.avg.copy_(torch.tensor([int(sd["on"]), int(sd["k"])], dtype=torch.int32))


def AdamOptimizer(learning_rate: float):
    """Factory with the reference's calling convention ``train_optimizer(FLAGS.learning_rate)``."""
    return lambda flat, **kw: FlatOptimizer(flat, learning_rate, "adam", **kw)


def GradientDescentOptimizer(learning_rate: float):
    return lambda flat, **kw: FlatOptimizer(flat, learning_rate, "sgd", **kw)


def ASGDOptimizer(learning_rate: float):
    """``torch.optim.ASGD(params, lr, lambd=0, t0=0)``: SGD that averages its iterates from the first step."""
    return lambda flat, **kw: FlatOptimizer(flat, learning_rate, "asgd", **kw)
