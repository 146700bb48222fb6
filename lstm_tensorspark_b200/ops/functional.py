"""Op dispatch: hand-written sm_90a kernels on CUDA tensors, pure-torch reference elsewhere.

There is exactly one GPU code path (the in-tree ``_C`` extension).  On a CUDA tensor the extension is
mandatory: a missing/unbuilt extension raises instead of silently falling back to eager PyTorch
(``set_backend("torch")`` is an explicit, test-only opt-out used by the numerics tests as ground truth).
"""
from __future__ import annotations

import math

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


def lstm_cell_step(x, h, c, w_x, w_h, bias, weight_drop=None):
    """One step.  ``weight_drop``: optional weight-drop ``reference.DropoutSpec``: the step reads ``W_h * M * s``
    (``reference.weight_drop``)."""
    if _use_ext(x):
        from . import cuda_lstm
        h_seq, h_T, c_T = cuda_lstm.lstm_layer_sequence(x.unsqueeze(0), h, c, w_x, w_h, bias, weight_drop=weight_drop)
        return h_T, c_T
    return ref.lstm_cell_step(x, h, c, w_x, ref.weight_drop(w_h, weight_drop), bias)


def lstm_layer_sequence(x_seq, h0, c0, w_x, w_h, bias, lengths=None, reverse=False, dropout=None, weight_drop=None,
                        activation_sums=False):
    """``lengths``: optional int32 ``[B]`` per-row sequence lengths (right padding, see ``reference.lstm_layer_sequence``).
    ``reverse``: the reverse-time direction of a bidirectional layer (same reference).  ``dropout``: optional
    ``reference.DropoutSpec``: the first output is then the dropped sequence.  ``weight_drop``: optional weight-drop
    ``reference.DropoutSpec``: every step reads ``W_h * M * s`` and ``W_h`` gets the masked gradient.  ``activation_sums``: one
    more output, the unnormalised AR / TAR sums ``[2]`` of the layer's output (``reference.activation_sums``)."""
    if _use_ext(x_seq):
        from . import cuda_lstm
        return cuda_lstm.lstm_layer_sequence(x_seq, h0, c0, w_x, w_h, bias, lengths=lengths, reverse=reverse, dropout=dropout,
                                             weight_drop=weight_drop, activation_sums=activation_sums)
    return ref.lstm_layer_sequence(x_seq, h0, c0, w_x, w_h, bias, lengths=lengths, reverse=reverse, dropout=dropout,
                                   weight_drop=weight_drop, activation_sums=activation_sums)


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


def head_xent_per_step(h_seq, weights, bias, labels, lengths=None):
    """The head at every time step: ``h_seq [T,B,H]``, ``labels`` int64 ``[B,T]``, ``lengths`` optional int32 ``[B]`` ->
    (logits ``[B,T,C]`` fp32, mean loss over the counted positions, correct count, N = number of counted positions)."""
    if _use_ext(h_seq):
        from . import cuda_head
        return cuda_head.head_xent_per_step(h_seq, weights, bias, labels, lengths)
    return ref.head_xent_per_step(h_seq, weights, bias, labels, lengths)


def vocab_head_supported(h_seq, num_classes: int) -> bool:
    """Does ``vocab_xent_per_step`` run its own GPU kernels on this input (bf16 on the CUDA backend, ``H % 64 == 0``,
    ``C % 8 == 0``, ``C >= 512``)?  Otherwise it is the composition through ``head_xent_per_step``."""
    if not _use_ext(h_seq):
        return False
    from . import cuda_vocab_head
    return cuda_vocab_head.supported(h_seq, num_classes)


def vocab_xent_per_step(h_seq, weights, bias, labels, lengths=None, class_major: bool = False):
    """The per-step head for many classes (a next-token language model's softmax): the loss, the correct count and N of
    ``head_xent_per_step`` - the same mask, normalisation and gradients - without the logits, which are neither returned nor
    stored.  ``lengths`` may hold zeros here (a row that does not count at all).  On the GPU bf16 ``h_seq`` with
    ``H % 64 == 0``, ``C % 8 == 0`` and ``C >= 512`` runs on the tensor cores (csrc/head_vocab.cu); every other input goes
    through ``head_xent_per_step``.  ``class_major``: ``weights`` is ``[C,H]`` (a tied embedding table, ``W^T``), read in place
    by the tensor-core kernels; the other paths read ``weights.t().contiguous()`` through autograd, so the gradient reaches
    ``weights`` in its own layout."""
    C = weights.shape[0 if class_major else 1]
    if vocab_head_supported(h_seq, C):
        from . import cuda_vocab_head
        return cuda_vocab_head.vocab_xent_per_step(h_seq, weights, bias, labels, lengths, class_major)
    w = weights.t().contiguous() if class_major else weights
    if _use_ext(h_seq):
        return head_xent_per_step(h_seq, w, bias, labels, lengths)[1:]
    return ref.vocab_xent_per_step(h_seq, w, bias, labels, lengths)


def vocab_sample(h, weights, bias, temperature: float, seed: int, step, tokens=None, record=None, row0=0, class_major: bool = False,
                 top_k: int = 0, top_p: float = 1.0):
    """Sample the next token of every row from the head's logits ``l = h W + bias`` (``h [B,H]``, ``W [H,C]``) without a host
    round trip -> (tokens int32 ``[B]``, log p(token) under ``softmax(l)`` fp32 ``[B]``).  Temperature 0 is the arg-max; above 0
    Gumbel-max with counter-based noise (``reference.sample_logits`` holds the definition).  ``step``: the decode step, an int
    or an int32 ``[1]`` device tensor that this call advances by one (a captured graph then draws new noise on each replay).
    ``tokens``: an int32 ``[B]`` buffer to write the tokens into; ``record = (tok [B,N], logprob [B,N], s0)``: column
    ``step - s0`` of each also gets them.  ``row0`` (an int or an int32 ``[1]`` device tensor): the noise counter's row word of
    row 0, the index of the batch's first prompt when prompts run in batches, so every prompt draws its own noise.  On the GPU bf16 ``h`` with ``H % 64 == 0``, ``C % 8 == 0`` and ``C >= 512`` runs in
    the head's tensor-core kernel (csrc/head_vocab.cu); every other input computes the fp32 logits with the head GEMM and
    samples them with one more kernel.  Two calls on the same inputs give the same bits.  ``class_major``: ``weights`` is
    ``[C,H]`` (a tied embedding table, ``W^T``), read in place.

    ``top_k`` (int >= 0, 0 = off) and ``top_p`` (in (0, 1], 1 = off): at temperature > 0 the draw is restricted to the row's
    top-k classes, then to its nucleus of q-mass ``top_p`` (``reference.sample_threshold`` holds the definition), with the same
    noise: the token is the unfiltered one whenever that one is kept.  The log-probability stays under the full ``softmax(l)``.
    On the GPU a filter stores the row's fp32 logits (the tensor-core kernel's own values, or the fallback's), computes each
    row's threshold on the device and samples the classes at or above it; with the filters off or at temperature 0 the
    unfiltered kernels run."""
    temperature = float(temperature)
    if not (math.isfinite(temperature) and temperature >= 0):
        raise ValueError(f"temperature must be finite and >= 0, got {temperature}")
    ref.check_sample_filters(top_k, top_p)
    top_k, top_p = int(top_k), float(top_p)
    C = weights.shape[0 if class_major else 1]
    if not ref.sample_filters_active(C, temperature, top_k, top_p):
        top_k, top_p = 0, 1.0
    if vocab_head_supported(h.unsqueeze(0), C):
        from . import cuda_vocab_head
        return cuda_vocab_head.vocab_sample(h, weights, bias, temperature, seed, step, tokens, record, row0, class_major,
                                            top_k, top_p)
    if _use_ext(h):
        from . import cuda_gemm, cuda_vocab_head
        w_t = weights.detach() if class_major else weights.detach().t()          # the GEMM's b_t operand: [C,H]
        logits = cuda_gemm.matmul(h.reshape(h.shape[0], -1), w_t, bias=bias.detach().float(), out_dtype=torch.float32)
        return cuda_vocab_head.vocab_sample_logits(logits, temperature, seed, step, tokens, record, row0, top_k, top_p)
    s = int(step)
    tok, logp = ref.vocab_sample(h, weights, bias, temperature, seed, s, int(row0), class_major=class_major, top_k=top_k,
                                 top_p=top_p)
    logp = logp.float()
    if isinstance(step, torch.Tensor):
        step.add_(1)
    if tokens is not None:
        tok = tokens.copy_(tok)
    if record is not None:
        rec_tok, rec_lp, s0 = record
        if 0 <= s - s0 < rec_tok.shape[1]:
            rec_tok[:, s - s0] = tok
            rec_lp[:, s - s0] = logp
    return tok, logp


def pool_sequence(h_seq, lengths=None, mode: str = "mean", attention=None):
    """Pool ``h_seq [T,B,H]`` over each row's counted steps -> ``s [B,H]`` fp32 (``reference.pool_sequence``); ``mode`` mean,
    max or attention (``attention = (W_a, b_a, v)``)."""
    if _use_ext(h_seq):
        from . import cuda_pool
        return cuda_pool.pool_sequence(h_seq, lengths, mode, attention)
    return ref.pool_sequence(h_seq, lengths, mode, attention)


def embedding(tokens, table, lengths=None, dtype=None, input_dropout=None, embedding_dropout=None):
    """``tokens`` int ``[B,T]`` (int64 is cast to int32) or ``[B]`` -> ``x [T,B,E]``, time-major, in ``dtype`` (the compute dtype;
    default the table's) (``reference.embedding``).  On the GPU the bf16 path reads the table's maintained bf16 shadow.
    ``input_dropout`` / ``embedding_dropout``: optional ``reference.DropoutSpec`` of the ``"input"`` and ``"rows"`` sites."""
    dtype = table.dtype if dtype is None else dtype
    if _use_ext(table):
        from . import cuda_embed
        return cuda_embed.embedding(tokens, table, lengths, dtype, input_dropout, embedding_dropout)
    return ref.embedding(tokens, table, lengths, input_dropout, embedding_dropout).to(dtype)


def lstm_pair_supported(x_seq, h_a: int, h_b: int) -> bool:
    """Can two stacked layers run as one pair op on the GPU (layer wavefront or pipelined, ``cuda_lstm.pair_schedule``)?"""
    if not x_seq.is_cuda or _BACKEND == "torch":
        return False
    from . import cuda_lstm
    return cuda_lstm.wavefront_supported(x_seq, h_a, h_b)


def lstm_pair_sequence(x_seq, la, lb, lengths=None, dropouts=(None, None), weight_drops=(None, None), activation_sums=False):
    """``activation_sums``: one more output, layer b's AR / TAR sums (``lstm_layer_sequence``)."""
    from . import cuda_lstm
    return cuda_lstm.lstm_pair_sequence(x_seq, la, lb, lengths=lengths, dropouts=dropouts, weight_drops=weight_drops,
                                        activation_sums=activation_sums)
