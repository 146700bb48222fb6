"""Op dispatch: hand-written sm_90a kernels on CUDA tensors, pure-torch reference elsewhere.

There is exactly one GPU code path (the in-tree ``_C`` extension).  On a CUDA tensor the extension is
mandatory: a missing/unbuilt extension raises instead of silently falling back to eager PyTorch
(``set_backend("torch")`` is an explicit, test-only opt-out used by the numerics tests as ground truth).
"""
from __future__ import annotations

import torch

from . import reference as ref

_BACKEND = "auto"          # auto | cuda_ext | torch


def set_backend(name: str):
    global _BACKEND
    if name not in ("auto", "cuda_ext", "torch"):
        raise ValueError(f"unknown backend {name!r}")
    _BACKEND = name


def get_backend() -> str:
    return _BACKEND


def _use_ext(t: torch.Tensor) -> bool:
    if _BACKEND == "torch":
        return False
    if t.is_cuda:
        return True
    if _BACKEND == "cuda_ext":
        raise RuntimeError("backend 'cuda_ext' requested but the tensor lives on the CPU")
    return False


def lstm_cell_step(x, h, c, w_x, w_h, bias):
    if _use_ext(x):
        from . import cuda_lstm
        h_seq, h_T, c_T = cuda_lstm.lstm_layer_sequence(x.unsqueeze(0), h, c, w_x, w_h, bias)
        return h_T, c_T
    return ref.lstm_cell_step(x, h, c, w_x, w_h, bias)


def lstm_layer_sequence(x_seq, h0, c0, w_x, w_h, bias, lengths=None, reverse=False, dropout=None):
    """``lengths``: optional int32 ``[B]`` per-row sequence lengths (right padding, see ``reference.lstm_layer_sequence``).
    ``reverse``: the reverse-time direction of a bidirectional layer (same reference).  ``dropout``: optional
    ``reference.DropoutSpec``: the first output is then the dropped sequence."""
    if _use_ext(x_seq):
        from . import cuda_lstm
        return cuda_lstm.lstm_layer_sequence(x_seq, h0, c0, w_x, w_h, bias, lengths=lengths, reverse=reverse, dropout=dropout)
    return ref.lstm_layer_sequence(x_seq, h0, c0, w_x, w_h, bias, lengths=lengths, reverse=reverse, dropout=dropout)


def dropout(x, spec, t0: int = 0):
    """``x [B,H]`` (time t0) or ``[T,B,H]`` -> ``x * mask * scale`` of ``spec`` (``reference.dropout``); None / P = 0: x."""
    if _use_ext(x):
        from . import cuda_lstm
        return cuda_lstm.dropout(x, spec, t0)
    return ref.dropout(x, spec, t0)


def head_xent(h, weights, bias, labels):
    """-> (logits [B,C] fp32, mean loss, correct count)."""
    if _use_ext(h):
        from . import cuda_head
        return cuda_head.head_xent(h, weights, bias, labels)
    return ref.head_xent(h, weights, bias, labels)


def lstm_pair_supported(x_seq, h_a: int, h_b: int) -> bool:
    """Can two stacked layers run as one pair op on the GPU (layer wavefront or pipelined, ``cuda_lstm.pair_schedule``)?"""
    if not x_seq.is_cuda or _BACKEND == "torch":
        return False
    from . import cuda_lstm
    return cuda_lstm.wavefront_supported(x_seq, h_a, h_b)


def lstm_pair_sequence(x_seq, la, lb, lengths=None, dropouts=(None, None)):
    from . import cuda_lstm
    return cuda_lstm.lstm_pair_sequence(x_seq, la, lb, lengths=lengths, dropouts=dropouts)
