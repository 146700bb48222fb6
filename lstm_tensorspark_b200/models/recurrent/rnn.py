"""Stack of LSTM layers.

Public surface mirrors original src/models/recurrent/rnn.py:5-53: ``RNN(settings)``,
``fit_layers(x)``, ``map_data_by_key()``, ``add_layer(setting)``, ``add_layers(settings)``.
``settings`` is the list of dicts built by ``Config.net_settings`` (keys ``layer_name``, ``dim_size``,
``num_hidden``, ``batch_size``).  New: ``fit_layers`` also accepts a sequence ``[B,T,D]`` and unrolls it
through time on the fused per-layer sequence op (the reference only ever takes one step), and
``add_reverse_layers()`` makes the stack bidirectional, and ``dropout`` drops the output of every layer but the last while
the module is in training mode (``nn.LSTM(dropout=...)``).  ``weight_drop`` drops connections of every layer direction's
recurrent weights ``W_h`` in training mode, one mask per training step (AWD-LSTM's ``WeightDrop``, Merity et al. 2017).
"""
from __future__ import annotations

from typing import Dict, Iterable, List, Optional

import torch
from torch import nn

from ...ops.reference import DropoutSpec
from .lstm import LSTMLayer

EXPORT_KEYS = ("wf", "wi", "wo", "wc", "bf", "bi", "bc", "bo")


class RNN(nn.Module):
    def __init__(self, settings: Iterable[dict], dropout: float = 0.0, weight_drop: float = 0.0, **layer_kw):
        super().__init__()
        if not 0.0 <= dropout < 1.0:
            raise ValueError(f"dropout must satisfy 0 <= P < 1, got {dropout}")
        if not 0.0 <= weight_drop < 1.0:
            raise ValueError(f"weight_drop must satisfy 0 <= P < 1, got {weight_drop}")
        self.layers = nn.ModuleList()
        self.reverse_layers = nn.ModuleList()      # empty, or one reverse-time layer per entry of ``layers``
        self._layer_kw = layer_kw
        self.dropout = float(dropout)
        self.weight_drop = float(weight_drop)
        # the mask's key (seed, partition) and step counter (training steps completed: an int32 [1] device tensor on the GPU,
        # an int on the CPU); a TrainEngine sets and advances them
        self.dropout_key = (0, 0)
        self.dropout_step = 0
        self.add_layers(settings)

    def dropout_spec(self, layer: int, reverse: bool = False) -> Optional[DropoutSpec]:
        """The dropout of layer ``layer``'s output in this forward pass: None for the top layer, with P = 0 and in eval mode."""
        if not self.training or self.dropout == 0 or layer >= len(self.layers) - 1:
            return None
        return DropoutSpec(self.dropout, self.dropout_key, layer, reverse, self.dropout_step)

    def weight_drop_spec(self, layer: int, reverse: bool = False) -> Optional[DropoutSpec]:
        """The weight drop of layer ``layer``'s ``W_h`` (direction ``reverse``) in this forward pass: every layer, the top one
        included; None with P = 0 and in eval mode.  Same key and step counter as ``dropout_spec``, its own counter stream."""
        if not self.training or self.weight_drop == 0:
            return None
        return DropoutSpec(self.weight_drop, self.dropout_key, layer, reverse, self.dropout_step, weight=True)

    def _make(self, setting: dict, reverse: bool = False) -> LSTMLayer:
        name = setting["layer_name"] + ("_reverse" if reverse else "")
        return LSTMLayer(name=name, num_hidden=setting["num_hidden"], dim_size=setting["dim_size"],
                         batch_size=setting["batch_size"], reverse=reverse, **self._layer_kw)

    def add_layer(self, setting: dict):
        if self.bidirectional:
            raise ValueError("add_layer: add every layer before add_reverse_layers()")
        self.layers.append(self._make(setting))

    def add_reverse_layers(self):
        """Make the stack bidirectional: a reverse-time twin ``<layer_name>_reverse`` of every layer, with its own weights (drawn
        now, after everything drawn so far).  Layer ``l + 1`` then reads ``[h_fwd(t) | h_rev(t)]``, so its ``dim_size`` must be
        ``2 H_l`` (``Config.net_settings`` with ``bidirectional``)."""
        if self.bidirectional:
            raise ValueError("the stack is already bidirectional")
        for i, layer in enumerate(self.layers):
            if i > 0 and layer.dim_size != 2 * self.layers[i - 1].num_hidden:
                raise ValueError(f"{layer.node_name}: a bidirectional stack needs dim_size = 2 * {self.layers[i - 1].num_hidden}, "
                                 f"got {layer.dim_size}")
            self.reverse_layers.append(self._make({"layer_name": layer.node_name, "num_hidden": layer.num_hidden,
                                                   "dim_size": layer.dim_size, "batch_size": layer.batch_size}, reverse=True))

    @property
    def bidirectional(self) -> bool:
        return len(self.reverse_layers) > 0

    def directions(self) -> List[LSTMLayer]:
        """Every layer, forward and reverse of each depth in turn (the order of the averaged / flat parameter set)."""
        if not self.bidirectional:
            return list(self.layers)
        return [l for pair in zip(self.layers, self.reverse_layers) for l in pair]

    def add_layers(self, settings: Iterable[dict]):
        for setting in settings:
            self.add_layer(setting)

    # --------------------------------------------------------------------------------------------
    def reset_state(self, batch_size: Optional[int] = None):
        for layer in self.directions():
            layer.reset_state(batch_size)

    def start_state(self, state: List[tuple]):
        """Start the next pass from ``state = [(h [B,H], c [B,H]) per layer]`` instead of the initial state variables (a carried
        stream state, ``--stateful``).  It is a constant to autograd: no gradient flows into it."""
        if self.bidirectional:
            raise ValueError("a carried state needs a unidirectional stack: the reverse direction has no state to carry forward")
        if len(state) != len(self.layers):
            raise ValueError(f"a carried state needs one (h, c) per layer: {len(self.layers)} layers, got {len(state)}")
        for layer, (h, c) in zip(self.layers, state):
            layer._set_state(h.detach(), c.detach())
            layer.state = []

    def final_state(self) -> List[tuple]:
        """``[(h_T, c_T) per layer]``: the state the last pass ended in (with ``lengths``: each row's state after its own last
        step).  ``h_T`` is in the compute dtype, as the kernels store it."""
        return [(layer.ht, layer.Ct) for layer in self.layers]

    def zero_state(self, batch_size: int, dtype: torch.dtype, device) -> List[tuple]:
        """The state a stream starts from: ``[(h [B,H] zeros in dtype, c [B,H] zeros in fp32 (fp64 for an fp64 model))]``."""
        c_dtype = torch.promote_types(dtype, torch.float32)
        return [(torch.zeros(batch_size, l.num_hidden, dtype=dtype, device=device),
                 torch.zeros(batch_size, l.num_hidden, dtype=c_dtype, device=device)) for l in self.layers]

    def fit_layers(self, input_data: torch.Tensor, train: bool = True, lengths: Optional[torch.Tensor] = None) -> torch.Tensor:
        """``[B,D]``: one step per layer (reference semantics, rnn.py:38-42; ``lengths`` is ignored; not bidirectional).
        ``[B,T,D]``: full unroll; returns the last layer's h at the last step, ``[B,H_last]`` - with ``lengths`` (int32 ``[B]``,
        right padding) at each row's own last step.  Bidirectional: ``[h_fwd_final | h_rev_final]``, ``[B, 2 H_last]``, the
        reverse half being the state after step 0."""
        if input_data.dim() == 2:
            if self.bidirectional:
                raise ValueError("a bidirectional stack needs whole sequences [B,T,D]: the one-step [B,D] path runs forward only")
            state = input_data
            for i, layer in enumerate(self.layers):
                state = layer.fit_next(state, train=train, dropout=self.dropout_spec(i), weight_drop=self.weight_drop_spec(i))
            return state
        if input_data.dim() != 3:
            raise ValueError(f"expected [B,D] or [B,T,D], got {tuple(input_data.shape)}")
        self._run_stack(input_data.transpose(0, 1), lengths)  # time-major [T,B,D]; the kernels index (t, b)
        if self.bidirectional:
            return torch.cat([self.layers[-1].ht, self.reverse_layers[-1].ht], 1)
        return self.layers[-1].ht                   # = seq[-1], as a separate autograd edge (no [T,B,H] gradient for the top layer)

    def fit_sequence_all(self, input_data: torch.Tensor, lengths: Optional[torch.Tensor] = None) -> torch.Tensor:
        """``[B,T,D]`` -> last layer's full ``h_seq [T,B,H]`` (padded positions hold the carried state); bidirectional:
        ``[T,B,2H]``, forward half first."""
        return self._run_stack(input_data.transpose(0, 1), lengths)

    def _run_stack(self, seq: torch.Tensor, lengths: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Layers bottom-up; adjacent pairs run as ONE op where the GPU path supports it (``cuda_lstm.pair_schedule``: a layer
        wavefront with both recurrences co-resident, or, where they do not fit side by side, the recurrences one after the other
        with the upper layer's GEMMs next to them), single layers otherwise.  Bidirectional: both
        directions of a layer run one after the other on the same input, and their outputs are joined into ``[T,B,2H]``
        (one concatenation) for the next layer; no wavefront."""
        from ...ops import functional as F
        if self.bidirectional:
            for i, (la, lr) in enumerate(zip(self.layers, self.reverse_layers)):
                seq = torch.cat([la.fit_sequence(seq, lengths, self.dropout_spec(i), self.weight_drop_spec(i)),
                                 lr.fit_sequence(seq, lengths, self.dropout_spec(i, True), self.weight_drop_spec(i, True))], 2)
            return seq
        i, n = 0, len(self.layers)
        while i < n:
            la = self.layers[i]
            if i + 1 < n and F.lstm_pair_supported(seq, la.num_hidden, self.layers[i + 1].num_hidden):
                lb = self.layers[i + 1]
                B = seq.shape[1]
                for l in (la, lb):
                    if B != l.ht.shape[0]:
                        l.reset_state(B)
                seq, hT_a, cT_a, hT_b, cT_b = F.lstm_pair_sequence(seq, (la.ht, la.Ct, la.w_x, la.w_h, la.bias),
                                                                     (lb.ht, lb.Ct, lb.w_x, lb.w_h, lb.bias), lengths=lengths,
                                                                     dropouts=(self.dropout_spec(i), self.dropout_spec(i + 1)),
                                                                     weight_drops=(self.weight_drop_spec(i),
                                                                                   self.weight_drop_spec(i + 1)))
                la._set_state(hT_a, cT_a); la.state.append((hT_a, cT_a))
                lb._set_state(hT_b, cT_b); lb.state.append((hT_b, cT_b))
                i += 2
            else:
                seq = la.fit_sequence(seq, lengths, self.dropout_spec(i), self.weight_drop_spec(i))
                i += 1
        return seq

    # --------------------------------------------------------------------------------------------
    def map_data_by_key(self):
        """The record set that is averaged across partitions (reference rnn.py:14-36): 8 ``(key, list)``
        pairs; ``w*`` -> per layer ``[W_h [H,H], W_x [D,H]]``; ``b*`` -> per layer ``[H]``."""
        rec: Dict[str, list] = {k: [] for k in EXPORT_KEYS}
        for layer in self.directions():
            rec["wf"].append(layer.weight_forget)
            rec["wi"].append(layer.weight_input)
            rec["wo"].append(layer.weight_output)
            rec["wc"].append(layer.weight_C)
            rec["bf"].append(layer.biases_forget)
            rec["bi"].append(layer.biases_input)
            rec["bc"].append(layer.biases_C)
            rec["bo"].append(layer.biases_output)
        return [(k, rec[k]) for k in EXPORT_KEYS]

    def averaged_parameters(self) -> List[nn.Parameter]:
        """The same set as ``map_data_by_key`` in fused storage (what the allreduce kernel touches)."""
        out = []
        for layer in self.directions():
            out += [layer.w_x, layer.w_h, layer.bias]
        return out
