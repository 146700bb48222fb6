"""Stack of LSTM layers.

Public surface mirrors original src/models/recurrent/rnn.py:5-53: ``RNN(settings)``,
``fit_layers(x)``, ``map_data_by_key()``, ``add_layer(setting)``, ``add_layers(settings)``.
``settings`` is the list of dicts built by ``Config.net_settings`` (keys ``layer_name``, ``dim_size``,
``num_hidden``, ``batch_size``).  New: ``fit_layers`` also accepts a sequence ``[B,T,D]`` and unrolls it
through time on the fused per-layer sequence op (the reference only ever takes one step), and
``add_reverse_layers()`` makes the stack bidirectional, and ``dropout`` drops the output of every layer but the last while
the module is in training mode (``nn.LSTM(dropout=...)``).  ``weight_drop`` drops connections of every layer direction's
recurrent weights ``W_h`` in training mode, one mask per training step (AWD-LSTM's ``WeightDrop``, Merity et al. 2017).
``output_dropout`` drops the top layer's output sequence, ``input_dropout`` the embedding output and ``embedding_dropout``
whole rows of the embedding table (the model's embedding reads ``input_dropout_spec`` / ``embedding_dropout_spec``);
``locked`` shares one mask of ``dropout``, ``output_dropout`` and ``input_dropout`` across every time step (AWD-LSTM's
``LockedDropout``).  ``activation_reg`` / ``temporal_activation_reg`` (AWD-LSTM's AR / TAR coefficients): when either is
non-zero, a forward pass in training mode asks the op of the top layer for its activation sums and leaves the normalised
``(AR, TAR)`` in ``activation_penalties`` (``ops.reference.activation_penalties``) for the training step to weigh into its loss.
"""
from __future__ import annotations

import math
from typing import Dict, Iterable, List, Optional

import torch
from torch import nn

from ...ops.reference import DropoutSpec, activation_penalties
from .lstm import LSTMLayer

EXPORT_KEYS = ("wf", "wi", "wo", "wc", "bf", "bi", "bc", "bo")


class RNN(nn.Module):
    def __init__(self, settings: Iterable[dict], dropout: float = 0.0, weight_drop: float = 0.0, output_dropout: float = 0.0,
                 input_dropout: float = 0.0, embedding_dropout: float = 0.0, locked: bool = False, activation_reg: float = 0.0,
                 temporal_activation_reg: float = 0.0, **layer_kw):
        super().__init__()
        for name, p in (("dropout", dropout), ("weight_drop", weight_drop), ("output_dropout", output_dropout),
                        ("input_dropout", input_dropout), ("embedding_dropout", embedding_dropout)):
            if not 0.0 <= p < 1.0:
                raise ValueError(f"{name} must satisfy 0 <= P < 1, got {p}")
        for name, c in (("activation_reg", activation_reg), ("temporal_activation_reg", temporal_activation_reg)):
            if not (math.isfinite(c) and c >= 0):
                raise ValueError(f"{name} must be a finite number >= 0, got {c}")
        self.layers = nn.ModuleList()
        self.reverse_layers = nn.ModuleList()      # empty, or one reverse-time layer per entry of ``layers``
        self._layer_kw = layer_kw
        self.dropout = float(dropout)
        self.weight_drop = float(weight_drop)
        self.output_dropout = float(output_dropout)
        self.input_dropout = float(input_dropout)
        self.embedding_dropout = float(embedding_dropout)
        self.locked = bool(locked)
        self.activation_reg = float(activation_reg)
        self.temporal_activation_reg = float(temporal_activation_reg)
        self.activation_penalties: Optional[torch.Tensor] = None      # [2] (AR, TAR) of the last training forward pass, or None
        # the mask's key (seed, partition) and step counter (training steps completed: an int32 [1] device tensor on the GPU,
        # an int on the CPU); a TrainEngine sets and advances them
        self.dropout_key = (0, 0)
        self.dropout_step = 0
        self.add_layers(settings)

    def dropout_spec(self, layer: int, reverse: bool = False) -> Optional[DropoutSpec]:
        """The dropout of layer ``layer``'s output in this forward pass: ``dropout`` below the top layer, ``output_dropout`` for
        the top layer; None with P = 0 and in eval mode."""
        p = self.output_dropout if layer >= len(self.layers) - 1 else self.dropout
        if not self.training or p == 0:
            return None
        return DropoutSpec(p, self.dropout_key, layer, reverse, self.dropout_step, locked=self.locked)

    def input_dropout_spec(self) -> Optional[DropoutSpec]:
        """The dropout of the embedding output ``x_t`` (``"input"`` site) in this forward pass; None with P = 0 and in eval
        mode."""
        if not self.training or self.input_dropout == 0:
            return None
        return DropoutSpec(self.input_dropout, self.dropout_key, 0, False, self.dropout_step, site="input", locked=self.locked)

    def embedding_dropout_spec(self) -> Optional[DropoutSpec]:
        """The dropout of whole embedding-table rows (``"rows"`` site, one mask per training step); None with P = 0 and in eval
        mode."""
        if not self.training or self.embedding_dropout == 0:
            return None
        return DropoutSpec(self.embedding_dropout, self.dropout_key, 0, False, self.dropout_step, site="rows")

    @property
    def wants_activation_sums(self) -> bool:
        """Does this forward pass compute AR / TAR (training mode, a coefficient above 0)?"""
        return self.training and (self.activation_reg > 0 or self.temporal_activation_reg > 0)

    @property
    def draws_masks(self) -> bool:
        """Does a training step draw any mask (the step counter must then advance)?"""
        return ((self.dropout > 0 and len(self.layers) > 1) or self.weight_drop > 0 or self.output_dropout > 0
                or self.input_dropout > 0 or self.embedding_dropout > 0)

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
        # the last pass's penalties hold its autograd graph, and with it the parameters' gradient accumulators: let them go before
        # the next pass builds its own (a captured step must not reuse accumulators created on another stream)
        self.activation_penalties = None
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
        (one concatenation) for the next layer; no wavefront.
        ``wants_activation_sums``: the top layer's op (both directions, or the pair whose upper layer is the top one) also
        returns its sums; their total, over the output's width, gives ``activation_penalties``."""
        from ...ops import functional as F
        T, B = seq.shape[0], seq.shape[1]
        n = len(self.layers)
        want = self.wants_activation_sums
        self.activation_penalties = None
        parts = []
        if self.bidirectional:
            for i, (la, lr) in enumerate(zip(self.layers, self.reverse_layers)):
                act = want and i == n - 1
                outs = [l.fit_sequence(seq, lengths, self.dropout_spec(i, r), self.weight_drop_spec(i, r), activation_sums=act)
                        for l, r in ((la, False), (lr, True))]
                if act:
                    parts = [o[1] for o in outs]
                    outs = [o[0] for o in outs]
                seq = torch.cat(outs, 2)
            return self._penalties(seq, parts, T, B, lengths)
        i = 0
        while i < n:
            la = self.layers[i]
            if i + 1 < n and F.lstm_pair_supported(seq, la.num_hidden, self.layers[i + 1].num_hidden):
                lb = self.layers[i + 1]
                B = seq.shape[1]
                for l in (la, lb):
                    if B != l.ht.shape[0]:
                        l.reset_state(B)
                act = want and i + 1 == n - 1
                outs = F.lstm_pair_sequence(seq, (la.ht, la.Ct, la.w_x, la.w_h, la.bias), (lb.ht, lb.Ct, lb.w_x, lb.w_h, lb.bias),
                                            lengths=lengths, dropouts=(self.dropout_spec(i), self.dropout_spec(i + 1)),
                                            weight_drops=(self.weight_drop_spec(i), self.weight_drop_spec(i + 1)),
                                            activation_sums=act)
                seq, hT_a, cT_a, hT_b, cT_b = outs[:5]
                if act:
                    parts = [outs[5]]
                la._set_state(hT_a, cT_a); la.state.append((hT_a, cT_a))
                lb._set_state(hT_b, cT_b); lb.state.append((hT_b, cT_b))
                i += 2
            else:
                act = want and i == n - 1
                seq = la.fit_sequence(seq, lengths, self.dropout_spec(i), self.weight_drop_spec(i), activation_sums=act)
                if act:
                    seq, sums = seq
                    parts = [sums]
                i += 1
        return self._penalties(seq, parts, T, B, lengths)

    def _penalties(self, seq: torch.Tensor, parts: list, T: int, B: int, lengths) -> torch.Tensor:
        """Sets ``activation_penalties`` from the top op's sums ``parts`` (none: left None) -> ``seq``."""
        if parts:
            sums = parts[0] if len(parts) == 1 else parts[0] + parts[1]
            self.activation_penalties = activation_penalties(sums, seq.shape[2], T, B, lengths)
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
