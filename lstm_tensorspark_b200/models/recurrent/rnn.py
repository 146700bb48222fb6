"""Stack of LSTM layers.

Public surface mirrors original src/models/recurrent/rnn.py:5-53: ``RNN(settings)``,
``fit_layers(x)``, ``map_data_by_key()``, ``add_layer(setting)``, ``add_layers(settings)``.
``settings`` is the list of dicts built by ``Config.net_settings`` (keys ``layer_name``, ``dim_size``,
``num_hidden``, ``batch_size``).  New: ``fit_layers`` also accepts a sequence ``[B,T,D]`` and unrolls it
through time on the fused per-layer sequence op (the reference only ever takes one step).
"""
from __future__ import annotations

from typing import Dict, Iterable, List, Optional

import torch
from torch import nn

from .lstm import LSTMLayer

EXPORT_KEYS = ("wf", "wi", "wo", "wc", "bf", "bi", "bc", "bo")


class RNN(nn.Module):
    def __init__(self, settings: Iterable[dict], **layer_kw):
        super().__init__()
        self.layers = nn.ModuleList()
        self._layer_kw = layer_kw
        self.add_layers(settings)

    def _make(self, setting: dict) -> LSTMLayer:
        return LSTMLayer(name=setting["layer_name"], num_hidden=setting["num_hidden"],
                         dim_size=setting["dim_size"], batch_size=setting["batch_size"], **self._layer_kw)

    def add_layer(self, setting: dict):
        self.layers.append(self._make(setting))

    def add_layers(self, settings: Iterable[dict]):
        for setting in settings:
            self.add_layer(setting)

    # --------------------------------------------------------------------------------------------
    def reset_state(self, batch_size: Optional[int] = None):
        for layer in self.layers:
            layer.reset_state(batch_size)

    def fit_layers(self, input_data: torch.Tensor, train: bool = True, lengths: Optional[torch.Tensor] = None) -> torch.Tensor:
        """``[B,D]``: one step per layer (reference semantics, rnn.py:38-42; ``lengths`` is ignored).
        ``[B,T,D]``: full unroll; returns the last layer's h at the last step, ``[B,H_last]`` - with ``lengths`` (int32 ``[B]``,
        right padding) at each row's own last step."""
        if input_data.dim() == 2:
            state = input_data
            for layer in self.layers:
                state = layer.fit_next(state, train=train)
            return state
        if input_data.dim() != 3:
            raise ValueError(f"expected [B,D] or [B,T,D], got {tuple(input_data.shape)}")
        self._run_stack(input_data.transpose(0, 1), lengths)  # time-major [T,B,D]; the kernels index (t, b)
        return self.layers[-1].ht                   # = seq[-1], as a separate autograd edge (no [T,B,H] gradient for the top layer)

    def fit_sequence_all(self, input_data: torch.Tensor, lengths: Optional[torch.Tensor] = None) -> torch.Tensor:
        """``[B,T,D]`` -> last layer's full ``h_seq [T,B,H]`` (padded positions hold the carried state)."""
        return self._run_stack(input_data.transpose(0, 1), lengths)

    def _run_stack(self, seq: torch.Tensor, lengths: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Layers bottom-up; adjacent pairs run as ONE layer-wavefront op where the GPU path supports it (both recurrences
        co-resident, the upper layer trailing by a couple of time steps), single layers otherwise."""
        from ...ops import functional as F
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
                                                                     (lb.ht, lb.Ct, lb.w_x, lb.w_h, lb.bias), lengths=lengths)
                la._set_state(hT_a, cT_a); la.state.append((hT_a, cT_a))
                lb._set_state(hT_b, cT_b); lb.state.append((hT_b, cT_b))
                i += 2
            else:
                seq = la.fit_sequence(seq, lengths)
                i += 1
        return seq

    # --------------------------------------------------------------------------------------------
    def map_data_by_key(self):
        """The record set that is averaged across partitions (reference rnn.py:14-36): 8 ``(key, list)``
        pairs; ``w*`` -> per layer ``[W_h [H,H], W_x [D,H]]``; ``b*`` -> per layer ``[H]``."""
        rec: Dict[str, list] = {k: [] for k in EXPORT_KEYS}
        for layer in self.layers:
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
        for layer in self.layers:
            out += [layer.w_x, layer.w_h, layer.bias]
        return out
