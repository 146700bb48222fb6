"""RNN + dense softmax head = the network the reference trainer assembles inline
(original src/rnn.py:203-228): placeholders -> ``RNN.fit_layers`` -> ``Dense1`` -> loss / accuracy.
"""
from __future__ import annotations

from typing import Callable, Dict, List, Optional, Tuple

import torch
from torch import nn

from ..config import Config
from ..ops import functional as F
from .flat import FlatParams
from .recurrent.lstm import create_variable, truncated_normal_
from .recurrent.rnn import RNN


class DenseHead(nn.Module):
    """``Dense1``: weights ``[H_last, C]`` (bidirectional: ``[2 H_last, C]``), bias ``[C]`` (truncated normal, src/rnn.py:214-221)."""

    def __init__(self, in_features: int, num_classes: int, init_std: float = 1.0, device=None, generator=None):
        super().__init__()
        init = lambda t, generator=None: truncated_normal_(t, init_std, generator)
        self.weights = create_variable("weights", (in_features, num_classes), initializer=init, device=device,
                                       generator=generator)
        self.bias = create_variable("bias", (num_classes,), initializer=init, device=device, generator=generator)

    def forward(self, h: torch.Tensor) -> torch.Tensor:
        h2 = h.reshape(h.shape[0], -1)
        if h2.is_cuda and F.get_backend() != "torch":
            from ..ops import cuda_gemm             # evaluation logits: our own GEMM kernels, no library call on the CUDA path
            return cuda_gemm.matmul(h2, self.weights.detach().t(), bias=self.bias.detach().float(), out_dtype=torch.float32)
        return h2.float() @ self.weights + self.bias


class SequenceClassifier(nn.Module):
    def __init__(self, cfg: Config, batch_size: Optional[int] = None, device=None,
                 generator: Optional[torch.Generator] = None,
                 allocator: Optional[Callable] = None):
        super().__init__()
        self.cfg = cfg
        bs = cfg.batch_size if batch_size is None else batch_size
        settings = cfg.net_settings(bs)
        head_in = settings[-1]["num_hidden"] * (2 if cfg.bidirectional else 1)
        head_std = cfg.init_std if cfg.init != "scaled" else cfg.init_std / (head_in ** 0.5)
        self.rnn = RNN(settings, dropout=cfg.dropout, learn_initial_state=cfg.resolved_learn_initial_state(), init_std=cfg.init_std,
                       init=cfg.init, weight_decay=(cfg.weight_decay or None), device=device, generator=generator)
        self.head = DenseHead(head_in, cfg.num_classes, init_std=head_std, device=device, generator=generator)
        if cfg.bidirectional:
            # drawn after every parameter of the unidirectional model, which therefore keeps its initial weights
            self.rnn.add_reverse_layers()
        self.flat: Optional[FlatParams] = None
        self._allocator = allocator
        self.compute_dtype = torch.float32

    def build_flat(self, allocator: Optional[Callable] = None) -> FlatParams:
        """Re-home every parameter into one flat fp32 buffer (+ grad buffer).  Call AFTER ``.to(device)``."""
        lstm = self.rnn.averaged_parameters()
        ids = {id(p) for p in lstm}
        others = [p for p in self.parameters() if id(p) not in ids]
        self.flat = FlatParams(lstm, others, allocator=allocator or self._allocator)
        return self.flat

    def set_compute_dtype(self, dtype: torch.dtype):
        self.compute_dtype = dtype
        if dtype != torch.float32 and self.flat is not None:
            self.flat.ensure_shadow()
            if self.flat.data.is_cuda and F.get_backend() != "torch":
                # the CUDA ops write these gradients straight into the flat buffer (first write of a step overwrites):
                # zero_grad() then has nothing to memset
                self.flat.enable_direct_grads(self.rnn.averaged_parameters() + [self.head.weights, self.head.bias])

    def features(self, x: torch.Tensor, lengths: Optional[torch.Tensor] = None) -> torch.Tensor:
        """``lengths``: optional int32 ``[B]`` per-sample sequence lengths (right-padded ``x``)."""
        self.rnn.reset_state(x.shape[0])
        return self.rnn.fit_layers(x.to(self.compute_dtype) if x.is_floating_point() else x, lengths=lengths)

    def forward(self, x: torch.Tensor, labels: torch.Tensor, lengths: Optional[torch.Tensor] = None):
        """-> (loss, logits, correct_count)"""
        h = self.features(x, lengths)
        logits, loss, correct = F.head_xent(h, self.head.weights, self.head.bias, labels)
        return loss, logits, correct

    # ---- reference variable naming ------------------------------------------------
    def named_reference_variables(self) -> List[Tuple[str, torch.Tensor]]:
        out = []
        for layer in self.rnn.directions():
            out += layer.named_reference_variables()
        out.append(("Dense1/weights", self.head.weights))
        out.append(("Dense1/bias", self.head.bias))
        return out

    def check_directions(self, variables: Dict[str, torch.Tensor], what: str = "checkpoint") -> None:
        """A checkpoint loads with ``strict=False``: a unidirectional one would leave a bidirectional model's reverse weights at
        their initial values (and the other way round silently drop them).  Raise unless both have the same directions."""
        saved = any("_reverse/" in k for k in variables)
        if saved != self.rnn.bidirectional:
            raise ValueError(f"{what} was written by a {'bidirectional' if saved else 'unidirectional'} model, this run is "
                             f"{'bidirectional' if self.rnn.bidirectional else 'unidirectional'}: "
                             f"{'add' if saved else 'drop'} --bidirectional")

    def reference_state_dict(self) -> Dict[str, torch.Tensor]:
        return {k: v.detach().clone().contiguous().cpu() for k, v in self.named_reference_variables()}

    def load_reference_state_dict(self, sd: Dict[str, torch.Tensor], strict: bool = True):
        with torch.no_grad():
            for k, v in self.named_reference_variables():
                if k in sd:
                    v.copy_(sd[k].to(v.device, v.dtype))
                elif strict:
                    raise KeyError(f"checkpoint is missing variable {k}")
        if self.flat is not None:
            self.flat.refresh_shadow()
