"""Loss / metric ops with the reference's signatures (original src/rnn.py:55-92):
``compute_loss(labels, logits, sparse=True)`` (+ the ``"weight_decay"`` collection terms of
``create_variable``), ``compute_accuracy(labels, logits, sparse=True)``.  Scalars with the reference's
TensorBoard tags (``cross_entropy``, ``weight_decay_loss``, ``total_loss``, ``accuracy``) are pushed to the
active ``utils.metrics.SummarySink`` if one is installed.
"""
from __future__ import annotations

import torch

from . import reference as ref
from ..utils import metrics as _metrics


def compute_loss(labels, logits, sparse: bool = True):
    return report_loss(ref.softmax_xent(logits, labels, sparse=sparse))


def report_loss(xent):
    """The reference's loss scalars for an already computed mean cross-entropy (also the per-step head's)."""
    _metrics.scalar("cross_entropy", xent)
    from ..models.recurrent.lstm import weight_decay_terms
    wd = weight_decay_terms()
    if len(wd) > 0:
        wd_loss = torch.stack([w.to(xent.device) for w in wd]).sum()
        _metrics.scalar("weight_decay_loss", wd_loss)
        total = xent + wd_loss
        _metrics.scalar("total_loss", total)
        return total
    return xent


def compute_accuracy(labels, logits, sparse: bool = True):
    return report_accuracy(ref.accuracy(logits, labels, sparse=sparse))


def report_accuracy(acc):
    _metrics.scalar("accuracy", acc)
    return acc
