"""Flat parameter / gradient storage.

All trainable tensors of a replica are views into ONE fp32 buffer (``data``) with a same-shaped
gradient buffer (``grad``), so that (a) the optimizer is a single multi-tensor kernel launch instead of
the reference's one ``ApplyAdam`` per variable (14·L+2 launches, src/rnn.py:207,224), and (b) the
cross-replica average / gradient allreduce touches one contiguous, 16 B-aligned message that can live in
NVLink-symmetric memory (replaces the 8 keyed Spark records of src/models/recurrent/rnn.py:27-36).

Order: [LSTM w_x, w_h, bias per layer] [everything else].  The first segment is exactly the reference's
averaged set (``map_data_by_key``); ``lstm_numel`` marks its end.
"""
from __future__ import annotations

from typing import Callable, List, Optional, Sequence, Tuple

import torch
from torch import nn

ALIGN = 64            # elements; 256 B for fp32, 128 B for the bf16 shadow (TMA / vector friendly)
PAD_TOTAL = 16384     # total padded so any world size <= 16 splits it into 16 B-aligned slices


def _round_up(x: int, m: int) -> int:
    return (x + m - 1) // m * m


class FlatParams:
    def __init__(self, lstm_params: Sequence[nn.Parameter], other_params: Sequence[nn.Parameter],
                 allocator: Optional[Callable[[int, torch.dtype, torch.device], torch.Tensor]] = None):
        params = list(lstm_params) + list(other_params)
        assert len(params) > 0
        device = params[0].device
        self.params: List[nn.Parameter] = params
        self.offsets: List[int] = []
        off = 0
        for i, p in enumerate(params):
            self.offsets.append(off)
            off = _round_up(off + p.numel(), ALIGN)
            if i == len(lstm_params) - 1:
                self.lstm_numel = off
        if not lstm_params:
            self.lstm_numel = 0
        self.numel = off
        self.padded_numel = _round_up(off, PAD_TOTAL)
        alloc = allocator or (lambda n, dt, dev: torch.zeros(n, dtype=dt, device=dev))
        self.data = alloc(self.padded_numel, torch.float32, device)
        self.grad = alloc(self.padded_numel, torch.float32, device)
        self.data.zero_()
        self.grad.zero_()
        self.shadow: Optional[torch.Tensor] = None      # bf16 copy maintained by the optimizer kernel
        # Lazy gradient zeroing (CUDA path): parameters whose gradients are WRITTEN by our kernels (first producer of a step
        # overwrites, later ones accumulate) are only marked stale by zero_grad(); no 67 MB memset per step.
        self._direct: set = set()                       # data_ptr of parameters with a direct gradient sink
        self._direct_ids: set = set()                   # the same parameters by identity (addresses change on rebase)
        self._stale: set = set()
        with torch.no_grad():
            for p, o in zip(params, self.offsets):
                self.data[o:o + p.numel()].view_as(p).copy_(p.data)
        self._rebind()

    def _rebind(self):
        for p, o in zip(self.params, self.offsets):
            p.data = self.data[o:o + p.numel()].view(p.shape)
            p.grad = self.grad[o:o + p.numel()].view(p.shape)
        if getattr(self, "_direct_ids", None):
            self._refresh_direct()

    def rebase(self, new_data: torch.Tensor, new_grad: torch.Tensor):
        """Move storage (e.g. into symmetric memory) keeping values."""
        new_data.copy_(self.data)
        new_grad.copy_(self.grad)
        self.data, self.grad = new_data, new_grad
        self._rebind()
        self._register_shadows()

    def ensure_shadow(self) -> torch.Tensor:
        if self.shadow is None:
            self.shadow = self.data.to(torch.bfloat16)
        self._register_shadows()
        return self.shadow

    def _register_shadows(self):
        """Let the CUDA ops find the maintained bf16 copy of a parameter (keyed by the fp32 view's address) instead of
        re-casting the weights every step; also the fp32 grad view so weight-gradient GEMMs accumulate in place."""
        if self.shadow is None or not self.data.is_cuda:
            return
        from ..ops.params import register_param
        for p, o in zip(self.params, self.offsets):
            register_param(p.data_ptr(), self.shadow[o:o + p.numel()].view(p.shape), self.grad[o:o + p.numel()].view(p.shape),
                           owner=self)

    def refresh_shadow(self):
        if self.shadow is not None:
            self.shadow.copy_(self.data)

    def shadow_view(self, p: nn.Parameter) -> torch.Tensor:
        i = next(k for k, q in enumerate(self.params) if q is p)
        o = self.offsets[i]
        return self.ensure_shadow()[o:o + p.numel()].view(p.shape)

    def enable_direct_grads(self, params: Sequence[nn.Parameter]):
        """Declare parameters whose gradients the CUDA ops write straight into ``grad`` (see ``take_sink``)."""
        self._direct_ids = {id(p) for p in params}
        self._refresh_direct()

    def _refresh_direct(self):
        self._direct = {p.data_ptr() for p in self.params if id(p) in self._direct_ids}
        self._stale = set()

    def zero_grad(self):
        if not self._direct:
            self.grad.zero_()
            return
        self._stale = set(self._direct)
        for p in self.params:                           # everything autograd accumulates into (p.grad += g) still needs zeros
            if p.data_ptr() not in self._direct:
                p.grad.zero_()

    def take_sink(self, addr: int) -> bool:
        """A kernel is about to write the gradient of the parameter at ``addr``: returns True when it must ACCUMULATE
        (something was already written this step), False when it must overwrite (first write after zero_grad)."""
        if addr in self._stale:
            self._stale.discard(addr)
            return False
        return True

    def ensure_zeroed(self, addr: int):
        """The gradient of ``addr`` is about to be accumulated by autograd (not by a direct kernel write)."""
        if addr in self._stale:
            self._stale.discard(addr)
            i = next(k for k, q in enumerate(self.params) if q.data_ptr() == addr)
            self.params[i].grad.zero_()

    def finalize_grads(self):
        """After backward: parameters that received no gradient this step hold zeros, not last step's values."""
        for addr in list(self._stale):
            self.ensure_zeroed(addr)

    def segment(self, scope: str) -> Tuple[int, int]:
        """Element range that is synchronised across replicas."""
        if scope == "lstm":
            return 0, _round_up(self.lstm_numel, ALIGN)
        return 0, self.padded_numel
