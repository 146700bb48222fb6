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
    """``Dense1``: weights ``[H_last, C]`` (bidirectional: ``[2 H_last, C]``), bias ``[C]`` (truncated normal, src/rnn.py:214-221).
    ``tied`` (``--tie_embeddings``): the weights are drawn as usual, so the bias and every later parameter get the draws of the
    untied model, and then discarded (``weights`` is None): the softmax reads the embedding table instead."""

    def __init__(self, in_features: int, num_classes: int, init_std: float = 1.0, device=None, generator=None, tied: bool = False):
        super().__init__()
        init = lambda t, generator=None: truncated_normal_(t, init_std, generator)
        self.weights = create_variable("weights", (in_features, num_classes), initializer=init, device=device,
                                       generator=generator)
        self.bias = create_variable("bias", (num_classes,), initializer=init, device=device, generator=generator)
        if tied:
            self.weights = None

    def forward(self, h: torch.Tensor, weights: Optional[torch.Tensor] = None, class_major: bool = False) -> torch.Tensor:
        """Evaluation logits ``h W + bias``; ``weights``: the matrix to read instead of ``self.weights`` (``class_major``: it is
        ``[C,H] = W^T``, the tied embedding table)."""
        w = self.weights if weights is None else weights
        h2 = h.reshape(h.shape[0], -1)
        if h2.is_cuda and F.get_backend() != "torch":
            from ..ops import cuda_gemm             # evaluation logits: our own GEMM kernels, no library call on the CUDA path
            w_t = w.detach() if class_major else w.detach().t()
            return cuda_gemm.matmul(h2, w_t, bias=self.bias.detach().float(), out_dtype=torch.float32)
        return h2.float() @ (w.t() if class_major else w) + self.bias


class Attention(nn.Module):
    """Attention pooling over time (``--pooling attention``): ``W_a [H_in, A]``, ``b_a [A]`` and the context vector ``v [A]``
    score every step as ``tanh(h_t W_a + b_a) . v`` (``ops.reference.pool_sequence``).  ``--init scaled``: W_a has std
    init_std / sqrt(H_in), b_a = 0 and v std init_std / sqrt(A); otherwise all three are truncated normal with init_std."""

    def __init__(self, in_features: int, units: int, init_std: float = 1.0, scaled: bool = False, device=None, generator=None):
        super().__init__()
        w_std = init_std / in_features ** 0.5 if scaled else init_std
        v_std = init_std / units ** 0.5 if scaled else init_std
        self.weights = create_variable("weights", (in_features, units), device=device, generator=generator,
                                       initializer=lambda t, generator=None: truncated_normal_(t, w_std, generator))
        self.bias = create_variable("bias", (units,), device=device, generator=generator,
                                    initializer=(lambda t, generator=None: nn.init.zeros_(t)) if scaled
                                    else (lambda t, generator=None: truncated_normal_(t, init_std, generator)))
        self.context = create_variable("context", (units,), device=device, generator=generator,
                                       initializer=lambda t, generator=None: truncated_normal_(t, v_std, generator))

    def params(self) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
        return self.weights, self.bias, self.context


class Embedding(nn.Module):
    """Token embedding in front of the first layer (``--vocab_size V``): ``weights [V, E]``, truncated normal with ``init_std``
    under both ``--init`` modes (the fan-in of a one-hot input is 1)."""

    def __init__(self, vocab_size: int, dim: int, init_std: float = 1.0, device=None, generator=None):
        super().__init__()
        self.weights = create_variable("weights", (vocab_size, dim), device=device, generator=generator,
                                       initializer=lambda t, generator=None: truncated_normal_(t, init_std, generator))

    def forward(self, tokens: torch.Tensor, lengths: Optional[torch.Tensor] = None, dtype=None, input_dropout=None,
                embedding_dropout=None) -> torch.Tensor:
        return F.embedding(tokens, self.weights, lengths, dtype, input_dropout, embedding_dropout)


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
        self.rnn = RNN(settings, dropout=cfg.dropout, weight_drop=getattr(cfg, "weight_drop", 0.0),
                       output_dropout=getattr(cfg, "output_dropout", 0.0), input_dropout=getattr(cfg, "input_dropout", 0.0),
                       embedding_dropout=getattr(cfg, "embedding_dropout", 0.0),
                       locked=getattr(cfg, "locked_dropout", False), learn_initial_state=cfg.resolved_learn_initial_state(), init_std=cfg.init_std,
                       init=cfg.init, weight_decay=(cfg.weight_decay or None), device=device, generator=generator)
        # --tie_embeddings: the softmax reads the embedding table (head_weights); Dense1/weights is drawn and discarded
        self.tied = bool(getattr(cfg, "tie_embeddings", False))
        self.head = DenseHead(head_in, cfg.num_classes, init_std=head_std, device=device, generator=generator, tied=self.tied)
        if cfg.bidirectional:
            # drawn after every parameter of the unidirectional model, which therefore keeps its initial weights
            self.rnn.add_reverse_layers()
        self.pooling = getattr(cfg, "pooling", "last")
        self.attention: Optional[Attention] = None
        if self.pooling == "attention":
            # drawn after everything else (the reverse layers included): every other configuration keeps its initial weights
            self.attention = Attention(head_in, cfg.attention_units, init_std=cfg.init_std, scaled=cfg.init == "scaled",
                                       device=device, generator=generator)
        self.vocab_size = int(getattr(cfg, "vocab_size", 0) or 0)
        self.embedding: Optional[Embedding] = None
        if self.vocab_size > 0:
            # drawn last (after the reverse layers and the attention weights): every run without it keeps its initial weights
            self.embedding = Embedding(self.vocab_size, cfg.in_features, init_std=cfg.init_std, device=device, generator=generator)
        if self.tied and (self.embedding is None or tuple(self.embedding.weights.shape) != (cfg.num_classes, head_in)):
            raise ValueError("--tie_embeddings needs --next_token with --in_features equal to the last --hidden_units: the softmax "
                             "reads the [V, E] embedding table as its [E, V] weights")
        self.flat: Optional[FlatParams] = None
        self._allocator = allocator
        self._decoders: Dict[tuple, "_Decoder"] = {}       # generate(): static buffers (and CUDA graph), one per batch shape
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
                self.flat.enable_direct_grads(self.rnn.averaged_parameters() +
                                              [p for p in (self.head.weights, self.head.bias) if p is not None] +
                                              ([] if self.attention is None else list(self.attention.params())) +
                                              ([] if self.embedding is None else [self.embedding.weights]))

    def head_weights(self) -> Tuple[torch.Tensor, bool]:
        """-> (the matrix the softmax reads, class_major): ``Dense1/weights [H_last, C]``, or with ``--tie_embeddings`` the
        embedding table ``[V, E]`` itself (``W = table^T``: logits_c = h . table[c] + bias_c).  The table is handed over as it is,
        never as a transposed view: the ops find its bf16 shadow and its gradient sink by its address and shape.  Every use of
        the head (training, scoring, evaluation logits, sampling) reads the weights through here."""
        if self.tied:
            return self.embedding.weights, True
        return self.head.weights, False

    def _dense_weights(self) -> torch.Tensor:
        """The head's ``W [H_last, C]`` for the ops that take no class-major operand (the per-step head of fewer than 512
        classes, fp32, the torch backend): with ``--tie_embeddings`` the table's transpose through autograd, so its gradient
        reaches the table in the table's layout."""
        w, class_major = self.head_weights()
        return w.t().contiguous() if class_major else w

    def head_logits(self, h: torch.Tensor) -> torch.Tensor:
        """Evaluation logits ``[rows, C]`` fp32 of ``h [rows, H_last]``."""
        return self.head(h, *self.head_weights())

    def _is_sequence(self, x: torch.Tensor) -> bool:
        """Whole sequences: ``[B,T,D]`` features, or ``[B,T]`` token ids with ``--vocab_size``."""
        return x.dim() == (2 if self.embedding is not None else 3)

    def _input(self, x: torch.Tensor, lengths: Optional[torch.Tensor] = None) -> torch.Tensor:
        """What the stack reads, batch-major: the features in the compute dtype, or with ``--vocab_size`` the embedded tokens
        (``[B,T,E]``, a view of the time-major ``[T,B,E]`` the embedding writes; ``[B,E]`` for one-step ``[B]`` tokens)."""
        if self.embedding is None:
            return x.to(self.compute_dtype) if x.is_floating_point() else x
        if x.is_floating_point() or x.dim() not in (1, 2):
            raise ValueError(f"--vocab_size needs integer token ids [B,T] (one step: [B]), got {x.dtype} {tuple(x.shape)}")
        e = self.embedding(x, lengths if x.dim() == 2 else None, self.compute_dtype, self.rnn.input_dropout_spec(),
                           self.rnn.embedding_dropout_spec())
        return e[0] if x.dim() == 1 else e.transpose(0, 1)

    def _start(self, batch_size: int, state) -> None:
        self.rnn.reset_state(batch_size)
        if state is not None:
            self.rnn.start_state(state)

    @staticmethod
    def _whole_sequences_only(state) -> None:
        if state is not None:
            raise ValueError("a carried state needs a label at every step (--next_token --stateful): a classifier of whole "
                             "sequences starts each one from the initial state")

    def features(self, x: torch.Tensor, lengths: Optional[torch.Tensor] = None) -> torch.Tensor:
        """``lengths``: optional int32 ``[B]`` per-sample sequence lengths (right-padded ``x``).  The top layer's last state, or
        with ``--pooling mean | max | attention`` its outputs pooled over each sample's steps (``ops.reference.pool_sequence``),
        rounded once to the compute dtype.  With ``--vocab_size`` ``x`` holds token ids (``[B,T]``, or ``[B]`` for one step)."""
        if self.pooling != "last":
            if not self._is_sequence(x):
                raise ValueError(f"--pooling {self.pooling} needs sequences [B,T,D] (token ids: [B,T]), got {tuple(x.shape)}")
            h_seq = self.sequence_features(x, lengths)
            s = F.pool_sequence(h_seq, lengths, self.pooling, None if self.attention is None else self.attention.params())
            return s.to(h_seq.dtype)
        self.rnn.reset_state(x.shape[0])
        return self.rnn.fit_layers(self._input(x, lengths), lengths=lengths)

    def check_labels(self, labels: torch.Tensor) -> None:
        """``[B]`` labels classify whole sequences, ``[B,T]`` label every step (``--per_step_labels``): the wrong one is an error."""
        if self.per_step and labels.dim() != 2:
            raise ValueError(f"--per_step_labels needs labels [B,T], got {tuple(labels.shape)}")
        if not self.per_step and labels.dim() == 2 and labels.shape[1] > 1:
            raise ValueError(f"labels {tuple(labels.shape)} of one class per step need --per_step_labels; without it they are [B]")

    @property
    def per_step(self) -> bool:
        return bool(getattr(self.cfg, "per_step_labels", False))

    def sequence_features(self, x: torch.Tensor, lengths: Optional[torch.Tensor] = None, state=None) -> torch.Tensor:
        """The top layer's whole output ``[T,B,H_last]`` (bidirectional ``[T,B,2 H_last]``) of ``x [B,T,D]``.  ``state``: optional
        ``[(h, c) per layer]`` to start from instead of the initial state (``RNN.start_state``); the state the pass ends in is
        ``self.rnn.final_state()``."""
        if not self._is_sequence(x):
            flag = "--per_step_labels" if self.per_step else f"--pooling {self.pooling}"
            raise ValueError(f"{flag} needs sequences [B,T,D] (token ids: [B,T]), got {tuple(x.shape)}")
        self._start(x.shape[0], state)
        return self.rnn.fit_sequence_all(self._input(x, lengths), lengths=lengths)

    def forward(self, x: torch.Tensor, labels: torch.Tensor, lengths: Optional[torch.Tensor] = None, state=None):
        """``state``: optional ``[(h, c) per layer]`` to start from (``sequence_features``), a constant to autograd.
        -> (loss, logits, correct_count); with ``--per_step_labels`` logits are ``[B,T,C]`` and the loss and the count run over
        the counted positions (``ops.reference.head_xent_per_step``).  Where the large-vocabulary head runs
        (``ops.functional.vocab_head_supported``: bf16 on the GPU, 512 classes or more) no logits exist and the slot holds None."""
        self.check_labels(labels)
        if self.per_step:
            h_seq = self.sequence_features(x, lengths, state)
            if F.vocab_head_supported(h_seq, self.cfg.num_classes):
                w, class_major = self.head_weights()
                loss, correct, _n = F.vocab_xent_per_step(h_seq, w, self.head.bias, labels, lengths, class_major=class_major)
                return loss, None, correct
            logits, loss, correct, _n = F.head_xent_per_step(h_seq, self._dense_weights(), self.head.bias, labels, lengths)
            return loss, logits, correct
        self._whole_sequences_only(state)
        h = self.features(x, lengths)
        logits, loss, correct = F.head_xent(h, self.head.weights, self.head.bias, labels)
        return loss, logits, correct

    @torch.no_grad()
    def score(self, x: torch.Tensor, labels: torch.Tensor, lengths: Optional[torch.Tensor] = None, first: int = 0, state=None):
        """Evaluation without gradients (call in eval mode): -> (mean loss, correct count, count) over rows ``first:`` of the
        batch, device tensors (no host sync); ``state`` as in ``forward``.  The count is of the counted positions with ``--per_step_labels``, of the rows
        otherwise.  The whole batch runs through the stack, so a tail can be scored in a batch of the usual static shape."""
        from ..ops import reference as ref
        self.check_labels(labels)
        if self.per_step:
            h_seq = self.sequence_features(x, lengths, state)
            if F.vocab_head_supported(h_seq, self.cfg.num_classes):
                # the tail is a mask, not a slice: rows before `first` get length 0, and no [rows, C] array is ever built
                if first > 0:
                    B, T = labels.shape
                    full = torch.full((B,), T, dtype=torch.int32, device=h_seq.device) if lengths is None else lengths
                    lengths = torch.where(torch.arange(B, device=h_seq.device) < first, torch.zeros_like(full), full)
                w, class_major = self.head_weights()
                return F.vocab_xent_per_step(h_seq, w, self.head.bias, labels, lengths, class_major=class_major)
            labels = labels[first:]
            if first == 0:
                _logits, loss, correct, n = F.head_xent_per_step(h_seq, self._dense_weights(), self.head.bias, labels, lengths)
                return loss, correct, n
            h_seq = h_seq[:, first:]
            logits = self.head_logits(h_seq.reshape(-1, h_seq.shape[2])).float().view(h_seq.shape[0], h_seq.shape[1], -1)
            return ref.softmax_xent_per_step(logits.transpose(0, 1), labels, None if lengths is None else lengths[first:])
        labels = labels[first:]
        self._whole_sequences_only(state)
        logits = self.head_logits(self.features(x, lengths))[first:].float()
        count = torch.full((), labels.shape[0], dtype=torch.int64, device=logits.device)
        return ref.softmax_xent(logits, labels), (logits.argmax(1) == labels).sum(), count

    # ---- text generation -----------------------------------------------------------
    @torch.no_grad()
    def generate(self, prompt: torch.Tensor, lengths: Optional[torch.Tensor], max_new_tokens: int, temperature: float = 1.0,
                 seed: int = 0, graph: Optional[bool] = None, row0: int = 0, top_k: int = 0, top_p: float = 1.0):
        """Continue each prompt (``--next_token`` models): ``prompt`` int ``[B,T]`` right-padded token ids, ``lengths`` int32 ``[B]``
        (None: every row is T long) -> (tokens int32 ``[B,N]``, log p(token) fp32 ``[B,N]`` under the model's softmax),
        ``N = max_new_tokens``, sampled at ``temperature`` with the noise of ``seed`` (``ops.functional.vocab_sample``; step s
        draws token s).  ``row0``: the index of row 0 among all the prompts when they run in batches; row b draws the noise of
        prompt ``row0 + b``, so no two prompts of one generation share it.  ``top_k`` / ``top_p``: draw from the top-k classes
        and then from the nucleus of q-mass ``top_p`` only (0 and 1: off; no effect at temperature 0); the log-probabilities stay
        under the full softmax.

        The prompt runs through the whole-sequence path; token 0 is sampled from the top layer's state after each row's own last
        prompt token.  Every later token embeds the previous one and takes one step of each layer from the carried state (the
        one-step path ``RNN.fit_layers`` in eval mode), then samples.  The state lives in static buffers; on the GPU the decode
        step is captured once per batch shape as a CUDA graph (``graph=False``: eager) and replayed; ``row0`` and the step counter
        live on the device, so one graph serves every batch, and another temperature, seed or filter replaces it (one graph per
        shape is kept).  The graph runs the eager loop's kernels; with the deterministic recurrences (``--deterministic``) both give the
        same bits.  Nothing waits for the device until the caller reads the result."""
        if not getattr(self.cfg, "next_token", False):
            raise ValueError("generate needs a language model trained with --next_token (this one predicts given labels)")
        N = int(max_new_tokens)
        if N < 1:
            raise ValueError(f"max_new_tokens must be >= 1, got {max_new_tokens}")
        if prompt.dim() != 2:
            raise ValueError(f"generate needs prompts [B,T] of token ids, got {tuple(prompt.shape)}")
        from ..ops import reference as ref
        ref.check_sample_filters(top_k, top_p)
        B, dev = prompt.shape[0], prompt.device
        use_graph = dev.type == "cuda" if graph is None else bool(graph)
        was_training = self.training
        self.eval()
        try:
            self.sequence_features(prompt, lengths)
            key = (B, N, str(dev), use_graph)
            noise = (float(temperature), int(seed) & 0xFFFFFFFF, int(top_k), float(top_p))
            dec = self._decoders.get(key)
            if dec is None or (dec.temperature, dec.seed, dec.top_k, dec.top_p) != noise:
                dec = self._decoders[key] = _Decoder(self, B, N, *noise, dev)
            for layer, (h, c) in zip(self.rnn.layers, dec.state):
                h.copy_(layer.ht)
                c.copy_(layer.Ct)
            dec.step.zero_()
            dec.row0.fill_(int(row0))
            dec.sample(self.rnn.layers[-1].ht)
            for s in range(1, N):
                if dec.graph is not None:
                    dec.graph.replay()
                    continue
                dec.run()
                if use_graph and s + 1 < N:
                    dec.capture()
        finally:
            self.train(was_training)
        return dec.tokens_out.clone(), dec.logprob_out.clone()

    # ---- reference variable naming ------------------------------------------------
    def named_reference_variables(self) -> List[Tuple[str, torch.Tensor]]:
        out = []
        for layer in self.rnn.directions():
            out += layer.named_reference_variables()
        if not self.tied:                           # --tie_embeddings: the softmax reads Embedding/weights
            out.append(("Dense1/weights", self.head.weights))
        out.append(("Dense1/bias", self.head.bias))
        if self.attention is not None:
            out.append(("Attention/weights", self.attention.weights))
            out.append(("Attention/bias", self.attention.bias))
            out.append(("Attention/context", self.attention.context))
        if self.embedding is not None:
            out.append(("Embedding/weights", self.embedding.weights))
        return out

    def check_compatible(self, variables: Dict[str, torch.Tensor], settings: Dict, what: str = "checkpoint") -> None:
        """Raise unless ``variables`` and the flags ``settings`` recorded beside them (``utils.checkpoint.recorded_settings``)
        were written by a model this one can load: the same directions, ``--pooling``, ``--vocab_size`` and ``--next_token``,
        checked in that order, then ``--tie_embeddings``."""
        self.check_directions(variables, what)
        self.check_pooling(variables, settings.get("pooling"), what)
        self.check_vocab(variables, settings.get("vocab_size"), what)
        self.check_next_token(settings.get("next_token"), what)
        self.check_tied(variables, settings.get("tie_embeddings"), what)

    def check_tied(self, variables: Dict[str, torch.Tensor], recorded: Optional[bool] = None, what: str = "checkpoint") -> None:
        """Raise unless ``variables`` (and the flag ``recorded`` beside them; nothing recorded counts as untied) were written
        under this model's ``--tie_embeddings``: a checkpoint loads with ``strict=False`` and would otherwise leave an untied
        model's Dense1/weights at their initial values, or silently drop a trained softmax matrix."""
        saved, has_w = bool(recorded), "Dense1/weights" in variables
        if saved == self.tied and has_w == (not self.tied):
            return
        desc = "with" if saved else "without"
        if saved == has_w:
            desc += f" --tie_embeddings but {'with' if has_w else 'without'} a Dense1/weights matrix"
        else:
            desc += " --tie_embeddings"
        raise ValueError(f"{what} was written {desc}, this run is {'with' if self.tied else 'without'} it: "
                         f"{'drop' if self.tied else 'add'} --tie_embeddings")

    def check_next_token(self, recorded: Optional[bool] = None, what: str = "checkpoint") -> None:
        """Raise unless the file was written with this run's ``--next_token`` (nothing recorded counts as off): the variables
        have the same shapes either way, but a head trained on given labels does not predict the next token."""
        saved, mine = bool(recorded), bool(getattr(self.cfg, "next_token", False))
        if saved != mine:
            raise ValueError(f"{what} was written {'with' if saved else 'without'} --next_token, this run is "
                             f"{'with' if mine else 'without'} it: {'add' if saved else 'drop'} --next_token")

    def check_vocab(self, variables: Dict[str, torch.Tensor], recorded: Optional[int] = None, what: str = "checkpoint") -> None:
        """Raise unless ``variables`` (and the vocabulary ``recorded`` beside them; nothing recorded: the table's row count, or 0
        without a table) were written with this model's ``--vocab_size``: a checkpoint loads with ``strict=False`` and would
        otherwise drop or leave behind the embedding table, or read ids against another vocabulary."""
        table = variables.get("Embedding/weights")
        saved = int(recorded) if recorded is not None else (0 if table is None else int(table.shape[0]))
        has_table = table is not None
        if saved == self.vocab_size and has_table == (self.vocab_size > 0) \
                and (table is None or int(table.shape[0]) == self.vocab_size):
            return
        desc = f"--vocab_size {saved}" if has_table == (saved > 0) else \
            f"--vocab_size {saved} ({'with' if has_table else 'without'} an Embedding/weights table)"
        raise ValueError(f"{what} was written with {desc}, this run uses --vocab_size {self.vocab_size}: "
                         f"pass the --vocab_size it was trained with")

    def check_directions(self, variables: Dict[str, torch.Tensor], what: str = "checkpoint") -> None:
        """A checkpoint loads with ``strict=False``: a unidirectional one would leave a bidirectional model's reverse weights at
        their initial values (and the other way round silently drop them).  Raise unless both have the same directions."""
        saved = any("_reverse/" in k for k in variables)
        if saved != self.rnn.bidirectional:
            raise ValueError(f"{what} was written by a {'bidirectional' if saved else 'unidirectional'} model, this run is "
                             f"{'bidirectional' if self.rnn.bidirectional else 'unidirectional'}: "
                             f"{'add' if saved else 'drop'} --bidirectional")

    def check_pooling(self, variables: Dict[str, torch.Tensor], recorded: Optional[str] = None, what: str = "checkpoint") -> None:
        """Raise unless ``variables`` (and the pooling ``recorded`` beside them; nothing recorded counts as ``last``) were written
        under this model's ``--pooling``: a checkpoint loads with ``strict=False`` and would otherwise drop or leave behind the
        attention weights, or silently score another model."""
        saved = recorded or "last"
        has_attn = any(k.startswith("Attention/") for k in variables)
        if saved == self.pooling and has_attn == (self.pooling == "attention"):
            return
        if saved == self.pooling:
            saved = "attention" if has_attn else f"{saved} (without the Attention/* variables)"
        raise ValueError(f"{what} was written with --pooling {saved}, this run uses --pooling {self.pooling}: "
                         f"pass the --pooling it was trained with")

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


class _Decoder:
    """The static buffers of ``SequenceClassifier.generate`` at one batch shape: the carried state of every layer, the previous
    token, the device-resident step counter and row offset and the ``[B,N]`` results, and once captured the CUDA graph of one decode step."""

    def __init__(self, model: SequenceClassifier, B: int, N: int, temperature: float, seed: int, top_k: int, top_p: float, device):
        self.model, self.temperature, self.seed, self.top_k, self.top_p = model, temperature, seed, top_k, top_p
        self.state = [(layer.ht.detach().clone(), layer.Ct.detach().clone()) for layer in model.rnn.layers]
        self.tokens = torch.zeros(B, dtype=torch.int32, device=device)
        self.step = torch.zeros(1, dtype=torch.int32, device=device)
        self.row0 = torch.zeros(1, dtype=torch.int32, device=device)
        self.tokens_out = torch.zeros(B, N, dtype=torch.int32, device=device)
        self.logprob_out = torch.zeros(B, N, dtype=torch.float32, device=device)
        self.graph = None

    def sample(self, h: torch.Tensor) -> None:
        w, class_major = self.model.head_weights()
        F.vocab_sample(h, w, self.model.head.bias, self.temperature, self.seed, self.step, tokens=self.tokens,
                       record=(self.tokens_out, self.logprob_out, 0), row0=self.row0, class_major=class_major, top_k=self.top_k,
                       top_p=self.top_p)

    def run(self) -> None:
        """One decode step: embed the previous token, one step of every layer from the buffers (which get the new state), sample."""
        layers = self.model.rnn.layers
        for layer, (h, c) in zip(layers, self.state):
            layer._set_state(h, c)
            layer.state = []                        # nothing to roll back to: the buffers are the state
        top = self.model.rnn.fit_layers(self.model._input(self.tokens), train=False)
        for layer, (h, c) in zip(layers, self.state):
            h.copy_(layer.ht)
            c.copy_(layer.Ct)
        self.sample(top)

    def capture(self) -> None:
        """Capture ``run`` (after it ran eagerly once at this shape, so every kernel is loaded and every workspace exists)."""
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            self.run()
        self.graph = g
