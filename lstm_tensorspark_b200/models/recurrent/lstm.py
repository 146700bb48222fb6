"""LSTM layer (per-timestep cell + whole-sequence fused path).

Public surface mirrors the reference cell (original src/models/recurrent/lstm.py:16-136):
``LSTMLayer(name, num_hidden, dim_size, batch_size)``, ``fit_next(data, train=True)``,
``restore_state()``, the per-gate accessors ``weight_forget / weight_input / weight_C / weight_output``
(each ``[W_h [H,H], W_x [D,H]]``) and ``biases_*`` ``[H]``, the trainable initial ``ht`` / ``Ct``
(``state`` / ``context_state`` ``[B,H]``), and ``create_variable`` (lstm.py:4-13).

Storage is NOT the reference's 12 separate matrices: each layer owns three fused tensors
(``w_x [4H,D]``, ``w_h [4H,H]``, ``bias [4H]``, gate-interleaved rows, see ops/reference.py) so one
wgmma GEMM tile produces all four gates of a hidden slice; the per-gate accessors are strided views.
"""
from __future__ import annotations

from typing import List, Optional, Tuple

import torch
from torch import nn

from ...ops import functional as F
from ...ops.reference import GATE_INDEX

_WEIGHT_DECAY_COLLECTION: List[torch.Tensor] = []


def truncated_normal_(t: torch.Tensor, std: float = 1.0, generator: Optional[torch.Generator] = None):
    """TF ``truncated_normal_initializer``: N(0, std) re-drawn outside 2 sigma."""
    with torch.no_grad():
        return nn.init.trunc_normal_(t, mean=0.0, std=std, a=-2.0 * std, b=2.0 * std, generator=generator)


def create_variable(name: str, shape, dtype=torch.float32, initializer=truncated_normal_,
                    weight_decay: Optional[float] = None, loss=None, device=None,
                    generator: Optional[torch.Generator] = None) -> nn.Parameter:
    """Variable factory (reference lstm.py:4-13) — lives in HBM, never pinned to the CPU (Q15).

    ``weight_decay``: registers ``loss(var) * weight_decay`` (default L2: sum(var^2)/2) in the
    module-level collection that ``ops.loss.compute_loss`` adds to the total loss."""
    var = nn.Parameter(torch.empty(*shape, dtype=dtype, device=device))
    var._ts_name = name
    if generator is not None:
        initializer(var.data, generator=generator)
    else:
        initializer(var.data)
    if weight_decay:
        fn = loss if loss is not None else (lambda v: 0.5 * (v.float() ** 2).sum())
        _WEIGHT_DECAY_COLLECTION.append((var, fn, float(weight_decay)))
    return var


def weight_decay_terms():
    return [fn(v) * wd for (v, fn, wd) in _WEIGHT_DECAY_COLLECTION]


def weight_decay_collection():
    """``[(variable, loss_fn, coefficient)]`` registered by ``create_variable(..., weight_decay=)``."""
    return list(_WEIGHT_DECAY_COLLECTION)


def clear_weight_decay_collection():
    _WEIGHT_DECAY_COLLECTION.clear()


class LSTMLayer(nn.Module):
    WEIGHT_STATE = 0
    WEIGHT_INPUT = 1

    def __init__(self, name: str, num_hidden: int, dim_size: int, batch_size: int,
                 learn_initial_state: bool = True, init_std: float = 1.0, init: str = "truncated_normal",
                 weight_decay: Optional[float] = None, device=None,
                 generator: Optional[torch.Generator] = None, reverse: bool = False):
        super().__init__()
        self.reverse = reverse                  # reverse-time direction of a bidirectional layer (whole sequences only)
        self.shape = [batch_size, num_hidden, dim_size]
        self.batch_size = batch_size
        self.num_hidden = num_hidden
        self.dim_size = dim_size
        self.node_name = name
        self.learn_initial_state = learn_initial_state
        self.state: List[Tuple[torch.Tensor, torch.Tensor]] = []

        H, D = num_hidden, dim_size
        if init == "scaled":
            sx, sh = init_std / (D ** 0.5), init_std / (H ** 0.5)
        else:
            sx = sh = init_std
        mk = lambda n, shp, s: create_variable(n, shp, initializer=lambda t, generator=None: truncated_normal_(t, s, generator),
                                               weight_decay=weight_decay, device=device, generator=generator)
        self.w_x = mk("weights_x", (4 * H, D), sx)
        self.w_h = mk("weights_h", (4 * H, H), sh)
        self.bias = mk("bias", (4 * H,), init_std)
        if init == "scaled":
            with torch.no_grad():
                self.bias.zero_()
        if learn_initial_state:
            self.h0 = mk("state", (batch_size, H), init_std)
            self.c0 = mk("context_state", (batch_size, H), init_std)
        else:
            self.register_buffer("h0", torch.zeros(batch_size, H, device=device), persistent=False)
            self.register_buffer("c0", torch.zeros(batch_size, H, device=device), persistent=False)
        self._set_state(self.h0, self.c0)

    # (ht, Ct) are plain attributes, NOT registered parameters: they alias h0/c0 only until the first step
    def _set_state(self, h, c):
        object.__setattr__(self, "_ht", h)
        object.__setattr__(self, "_ct", c)

    ht = property(lambda self: self._ht, lambda self, v: object.__setattr__(self, "_ht", v))
    Ct = property(lambda self: self._ct, lambda self, v: object.__setattr__(self, "_ct", v))

    # ---- reference-shaped accessors -----------------------------------------------------------
    def _gate_w(self, gate: str):
        g = GATE_INDEX[gate]
        H, D = self.num_hidden, self.dim_size
        w_h = self.w_h.view(H, 4, H)[:, g, :].t()   # [H_in, H]  == reference weights_<gate>_h
        w_x = self.w_x.view(H, 4, D)[:, g, :].t()   # [D, H]     == reference weights_<gate>_x
        return [w_h, w_x]

    def _gate_b(self, gate: str):
        return self.bias.view(self.num_hidden, 4)[:, GATE_INDEX[gate]]

    weight_forget = property(lambda self: self._gate_w("forget"))
    weight_input = property(lambda self: self._gate_w("input"))
    weight_C = property(lambda self: self._gate_w("C"))
    weight_output = property(lambda self: self._gate_w("output"))
    biases_forget = property(lambda self: self._gate_b("forget"))
    biases_input = property(lambda self: self._gate_b("input"))
    biases_C = property(lambda self: self._gate_b("C"))
    biases_output = property(lambda self: self._gate_b("output"))

    # ---- per-timestep API (reference lstm.py:88-136) --------------------------------------------
    def reset_state(self, batch_size: Optional[int] = None):
        """Start of a new sequence/batch: (ht, Ct) <- the initial state variables."""
        if batch_size is not None and batch_size != self.h0.shape[0]:
            if self.learn_initial_state:
                raise ValueError(f"{self.node_name}: learned initial state has batch {self.h0.shape[0]}, got {batch_size}")
            self._set_state(self.h0.new_zeros(batch_size, self.num_hidden),
                            self.c0.new_zeros(batch_size, self.num_hidden))
        else:
            self._set_state(self.h0, self.c0)
        self.state = []

    def train_layer(self, input_data: torch.Tensor, weight_drop=None):
        h, c = F.lstm_cell_step(input_data, self.ht, self.Ct, self.w_x, self.w_h, self.bias, weight_drop=weight_drop)
        self._set_state(h, c)

    def restore_state(self):
        self._set_state(self.state[-1][0], self.state[-1][1])

    def fit_next(self, data: torch.Tensor, train: bool = True, dropout=None, weight_drop=None) -> torch.Tensor:
        """One step.  ``dropout``: optional ``ops.reference.DropoutSpec`` of the returned output (time 0); the carried state
        is not dropped.  ``weight_drop``: optional weight-drop ``DropoutSpec``: the step reads ``W_h * M * s``."""
        self.train_layer(data, weight_drop)
        out = F.dropout(self.ht, dropout)
        if train:
            self.state.append((self.ht, self.Ct))
            return out
        if self.state:
            self.restore_state()       # roll back: a non-train step must not advance the recurrence
        return out

    # ---- whole-sequence path (the thing the persistent kernel implements) ----------------------
    def fit_sequence(self, x_seq: torch.Tensor, lengths: Optional[torch.Tensor] = None, dropout=None,
                     weight_drop=None, activation_sums: bool = False):
        """``x_seq [T,B,D]`` -> ``h_seq [T,B,H]``; final (ht, Ct) stored on the layer.  ``lengths`` (int32 ``[B]``, right
        padding): the final state is each row's state after its own last step; padded positions of ``h_seq`` carry it.
        A reverse layer runs from the last step to the first: its final state is the one after step 0, and its padded
        positions hold the initial state.  ``dropout``: optional ``ops.reference.DropoutSpec``; the returned sequence is then
        the dropped one (the final state is not dropped).  ``weight_drop``: optional weight-drop ``DropoutSpec``: every step reads
        ``W_h * M * s`` (``ops.reference.weight_drop``) and ``w_h`` gets the masked gradient.  ``activation_sums``: ->
        ``(h_seq, sums)``, ``sums`` the layer's unnormalised AR / TAR sums ``[2]`` (``ops.reference.activation_sums``)."""
        B = x_seq.shape[1]
        if B != self.ht.shape[0]:
            self.reset_state(B)
        outs = F.lstm_layer_sequence(x_seq, self.ht, self.Ct, self.w_x, self.w_h, self.bias, lengths=lengths,
                                     reverse=self.reverse, dropout=dropout, weight_drop=weight_drop, activation_sums=activation_sums)
        h_seq, h_T, c_T = outs[:3]
        self._set_state(h_T, c_T)
        self.state.append((h_T, c_T))
        return (h_seq, outs[3]) if activation_sums else h_seq

    def named_reference_variables(self):
        """(reference variable name, tensor) in the §2.7 checkpoint naming."""
        n = self.node_name
        out = []
        for gate in ("forget", "input", "C", "output"):
            w_h, w_x = self._gate_w(gate)
            out.append((f"{n}/weights_{gate}_h", w_h))
            out.append((f"{n}/weights_{gate}_x", w_x))
            out.append((f"{n}/bias_{gate}", self._gate_b(gate)))
        if self.learn_initial_state:
            out.append((f"{n}/state", self.h0))
            out.append((f"{n}/context_state", self.c0))
        return out
