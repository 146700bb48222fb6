"""How the CUDA ops reach a parameter's bf16 operand and where they write its gradient.

``models.flat.FlatParams`` registers every parameter of its flat buffer here, keyed by the address of the fp32 view: the bf16
shadow the optimizer maintains and the fp32 gradient view.  An op reads a weight through ``lowp`` and takes the tensor its kernel
writes a gradient into from ``grad_out``; whether that write overwrites or accumulates is decided here (by ``FlatParams``), so
no op has to know."""
from __future__ import annotations

import weakref

import torch

_PARAMS = {}          # fp32 param address -> (bf16 shadow view, fp32 grad view, weakref to the FlatParams or None)


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
