"""CUDA ops of the continuous cache pointer (csrc/cache_pointer.cu): the per-stream history ring's append, the scores of a
segment against it (tensor cores for bf16 with ``H % 64 == 0``, CUDA cores otherwise) with the mixture and the segment's loss
sums, and the model's own log-probability at the label from either softmax head."""
from __future__ import annotations

import torch

from .cuda_ext import count, ext


def tc_supported(h_seq: torch.Tensor) -> bool:
    """Does the segment take the tensor-core kernel (bf16, ``H % 64 == 0``)?  Every other input takes the generic kernel."""
    return h_seq.dtype == torch.bfloat16 and h_seq.shape[2] % 64 == 0


def append(h_seq, labels, keys, key_labels, seen: int) -> None:
    """Write ``h_seq [T,B,H]`` and ``labels [B,T]`` into the ring at positions ``seen .. seen + T - 1``."""
    ext().cache_append(h_seq.contiguous(), keys, key_labels, labels.long().contiguous(), int(seen))
    count("cache_append")


def cache_pointer(h_seq, labels, logp_model, keys, key_labels, seen: int, window: int, theta: float, lam: float, lengths=None):
    """-> (log p ``[T·B]`` fp32, 0 at uncounted positions; ``[2]`` fp32 {sum -log p, sum -log p_model} over the counted ones)."""
    tc = tc_supported(h_seq)
    logp, sums = ext().cache_pointer(h_seq.contiguous(), keys, key_labels, labels.long().contiguous(), logp_model.float().contiguous(),
                                     None if lengths is None else lengths.contiguous(), int(window), int(seen), float(theta),
                                     float(lam), tc)
    count("cache_pointer_tc" if tc else "cache_pointer_generic")
    return logp, sums


def label_logprob_parts(part, lse, labels, num_classes: int):
    """log p_model(y) ``[T·B]`` from the large-vocabulary head's forward partials and ``lse``."""
    return ext().cache_label_logprob_parts(part, lse, labels.long().contiguous(), int(num_classes))


def label_logprob_logits(logits, labels):
    """log p_model(y) ``[T·B]`` from stored fp32 logits ``[B,T,C]``."""
    return ext().cache_label_logprob_logits(logits.float().contiguous(), labels.long().contiguous())
