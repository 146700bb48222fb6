"""Loader for the in-tree sm_90a extension (``lstm_tensorspark_b200/_C*.so``).

There is no eager fallback on the GPU: if a CUDA tensor reaches an op and the extension cannot be imported,
``ext()`` raises with the build command.  ``LSTM_TS_BUILD=1`` builds on demand (used by tests / CI)."""
from __future__ import annotations

import importlib
import os

import torch

_EXT = None
_ERR = None
LAUNCHES = {"n": 0}          # number of OUR kernels launched through the extension (bench.py "gpu_launches")
# which paths the ops took (also read as ``cuda_lstm.STATS``): fixed keys are incremented in place, the others through ``count``
STATS = {"fast_fwd": 0, "fast_bwd": 0, "generic_fwd": 0, "generic_bwd": 0, "tc_gemm": 0, "kernels": 0, "weight_drop": 0,
         "weight_drop_grad": 0, "embed_fwd_dropout": 0, "embed_bwd_dropout": 0}
_NO_KERNEL = {"ar_max_blocks", "ar_flag_words", "ar_slots"}


def count(key: str, n: int = 1) -> None:
    STATS[key] = STATS.get(key, 0) + n


class _Counting:
    """Thin proxy over the pybind module that counts kernel launches."""

    def __init__(self, mod):
        object.__setattr__(self, "_m", mod)

    def __getattr__(self, name):
        fn = getattr(self._m, name)
        if name in _NO_KERNEL or not callable(fn):
            return fn

        def call(*a, **k):
            LAUNCHES["n"] += 1
            return fn(*a, **k)
        object.__setattr__(self, name, call)
        return call

def drop_args(spec, device) -> dict:
    """Keyword arguments of the kernels for a ``reference.DropoutSpec`` (none for None / P = 0): the device-resident step
    counter and the descriptor {key0, key1, thr, c2, row0}."""
    if spec is None or spec.p == 0:
        return {}
    step = spec.step
    if not isinstance(step, torch.Tensor):                       # (a caller without an engine: no graph capture to honour)
        step = torch.tensor([int(step)], dtype=torch.int32, device=device)
    return {"drop_step": step, "drop_desc": spec.desc()}


def ext():
    global _EXT, _ERR
    if _EXT is not None:
        return _EXT
    try:
        _EXT = _Counting(importlib.import_module("lstm_tensorspark_b200._C"))
        return _EXT
    except Exception as e:                       # noqa: BLE001
        _ERR = e
    if os.environ.get("LSTM_TS_BUILD", "0") == "1":
        from .. import build as _b
        _b.build()
        importlib.invalidate_caches()
        _EXT = _Counting(importlib.import_module("lstm_tensorspark_b200._C"))
        return _EXT
    raise RuntimeError(
        "lstm_tensorspark_b200._C (the hand-written sm_90a kernels) is not built/importable: "
        f"{_ERR!r}.  Run `python -m lstm_tensorspark_b200.build` (or __graft_entry__.build()).  "
        "There is deliberately no PyTorch fallback on CUDA tensors.")


def available() -> bool:
    try:
        ext()
        return True
    except Exception:                            # noqa: BLE001
        return False
