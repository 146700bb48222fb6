"""How the CUDA ops reach a parameter's bf16 operand and where they write its gradient.

``models.flat.FlatParams`` registers every parameter of its flat buffer here, keyed by the address of the fp32 view: the bf16
shadow the optimizer maintains and the fp32 gradient view.  An op reads a weight through ``lowp`` and takes the tensor its kernel
writes a gradient into from ``grad_out``; whether that write overwrites or accumulates is decided here (by ``FlatParams``), so
no op has to know.

An op ``release``s a parameter to the gradient buckets (``engine.TrainEngine``), which update the flat buffer in place while
backward runs, once it has enqueued the last kernel of this backward pass that writes the parameter's gradient or reads its
weights (fp32 data or bf16 shadow).  A bucket whose parameters are all released is launched behind the next big backward kernel
(a recurrence or a weight-gradient GEMM: ``after_big_launch``) as a programmatic dependent, so it runs next to that kernel."""
from __future__ import annotations

import contextlib
import weakref

import torch

_PARAMS = {}          # fp32 param address -> (bf16 shadow view, fp32 grad view, weakref to the FlatParams or None)
_RELEASED = set()     # addresses released in the current backward pass
_LISTENER = None      # the engine's bucket launcher, for the duration of one backward pass
_QUEUE = []           # big-launch queue: [(generation when queued, closure)]
_GEN = 0              # big launches so far


def register_param(addr: int, shadow: torch.Tensor, grad: torch.Tensor, owner=None) -> None:
    _PARAMS[addr] = (shadow, grad, weakref.ref(owner) if owner is not None else None)


def _lookup(addr: int):
    ent = _PARAMS.get(addr)
    if ent is None:
        return None
    if ent[2] is not None and ent[2]() is None:       # the FlatParams buffer died: its address may have been reused
        del _PARAMS[addr]
        return None
    return ent


def lowp(w: torch.Tensor, cd: torch.dtype) -> torch.Tensor:
    """bf16 copy of a weight: the optimizer-maintained shadow when there is one, a cast otherwise."""
    if cd == torch.bfloat16:
        ent = _lookup(w.data_ptr())
        if ent is not None and ent[0].shape == w.shape:
            return ent[0]
    return w.detach().to(cd).contiguous()


def grad_out(addr: int, shape, device) -> tuple:
    """-> ``(out, accumulate, ret)`` for the gradient of the parameter at ``addr``: the kernel writes the fp32 tensor ``out``
    (adding to it when ``accumulate``), and the op returns ``ret`` to autograd.

    A registered parameter gets its grad view and ``ret = None``: a direct one overwrites on the first write of a step and
    accumulates afterwards (``FlatParams.take_sink``), any other is zeroed on demand and accumulated into.  An unregistered one
    (or one whose ``FlatParams`` is gone) gets a fresh tensor of ``shape``, overwritten and returned."""
    ent = _lookup(addr)
    if ent is None:
        out = torch.empty(shape, dtype=torch.float32, device=device)
        return out, False, out
    owner = ent[2]() if ent[2] is not None else None
    if owner is None or addr not in owner._direct:
        if owner is not None:
            owner.ensure_zeroed(addr)
        return ent[1], True, None
    return ent[1], owner.take_sink(addr), None


def release(*addrs: int) -> None:
    """The calling op has enqueued the last kernel of this backward pass that writes the gradients of the parameters at
    ``addrs`` or reads their weights: a bucket holding them may now be synced and updated."""
    if _LISTENER is not None:
        _RELEASED.update(addrs)
        _LISTENER(_RELEASED)


class Countdown:
    """``n`` ops that write the same gradients, such as the batch chunks of one LSTM layer: ``releaser()``, called once in the
    backward pass of each, gives ``release`` to the one that runs last (in whatever order autograd runs them), a no-op to the rest."""

    def __init__(self, n: int):
        self.left = n

    def releaser(self):
        self.left -= 1
        return release if self.left == 0 else (lambda *addrs: None)


@contextlib.contextmanager
def releases_to(listener):
    """Call ``listener(released addresses)`` after every ``release`` in the block (one backward pass)."""
    global _LISTENER
    _RELEASED.clear()
    _LISTENER = listener
    try:
        yield
    finally:
        _LISTENER = None


def queue_after_big_launch(fn) -> None:
    _QUEUE.append((_GEN, fn))


def big_launch_begin() -> None:
    """An ORDINARY launch of a big backward kernel follows: everything enqueued before it is complete when it starts."""
    global _GEN
    _GEN += 1


def after_big_launch(flush: bool = False) -> None:
    """Run the queued closures (they launch programmatic dependents) behind the kernel just launched - but only those queued
    BEFORE it was launched: a dependent may start while its primary runs, so its inputs must not come from it."""
    while _QUEUE and (flush or _QUEUE[0][0] < _GEN):
        _QUEUE.pop(0)[1]()
