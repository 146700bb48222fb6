"""Pure-PyTorch reference implementations of every op that has a hand-written sm_90a kernel.

These are (a) the CPU execution path, (b) the fp32 ground truth the GPU numerics tests compare against.
Math parity with the reference model: original src/models/recurrent/lstm.py:88-122 (cell),
original src/rnn.py:55-92 (loss / accuracy), TF-1.0 ``ApplyAdam`` (optimizer).

Fused parameter layout (this framework's own, chosen for the kernels): per layer
``w_x [4H, D]``, ``w_h [4H, H]``, ``bias [4H]`` with row ``n = 4*j + g`` = gate ``g`` of hidden unit ``j``
and gate order ``g: 0=input(i) 1=forget(f) 2=candidate(C~) 3=output(o)``.  A CTA that owns a
contiguous slice of rows therefore owns complete (i,f,g,o) quadruples of a hidden slice.
"""
from __future__ import annotations

from typing import Optional, Tuple

import torch

GATE_I, GATE_F, GATE_G, GATE_O = 0, 1, 2, 3
GATE_INDEX = {"input": GATE_I, "forget": GATE_F, "C": GATE_G, "output": GATE_O}


def lstm_gates(pre: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor, torch.Tensor]:
    """``pre [B, 4H]`` (interleaved) -> activated (i, f, g, o), each ``[B, H]``."""
    B = pre.shape[0]
    p = pre.view(B, -1, 4)
    i = torch.sigmoid(p[..., GATE_I])
    f = torch.sigmoid(p[..., GATE_F])
    g = torch.tanh(p[..., GATE_G])
    o = torch.sigmoid(p[..., GATE_O])
    return i, f, g, o


def lstm_cell_step(x, h, c, w_x, w_h, bias):
    """One time step.  ft = σ(h·Wf_h + x·Wf_x + bf) …  Ct = ft*Ct + it*C~ ; ht = ot*tanh(Ct)
    (reference: lstm.py:93-109; ``ot`` uses the OLD ht, as there)."""
    pre = x @ w_x.t() + h @ w_h.t() + bias
    i, f, g, o = lstm_gates(pre)
    c_new = f * c + i * g
    h_new = o * torch.tanh(c_new)
    return h_new, c_new


def check_lengths(lengths: torch.Tensor, B: int, T: int) -> None:
    """Per-row sequence lengths: int32 ``[B]`` with ``1 <= lengths[b] <= T`` (costs a device-to-host read on a GPU tensor)."""
    if lengths.dtype != torch.int32 or lengths.dim() != 1 or lengths.shape[0] != B:
        raise ValueError(f"lengths must be int32 [{B}], got {lengths.dtype} {tuple(lengths.shape)}")
    lo, hi = int(lengths.min()), int(lengths.max())
    if lo < 1 or hi > T:
        raise ValueError(f"lengths must lie in [1, {T}], got [{lo}, {hi}]")


def lstm_layer_sequence(x_seq, h0, c0, w_x, w_h, bias, lengths: Optional[torch.Tensor] = None, reverse: bool = False):
    """Unrolled layer: ``x_seq [T,B,D]`` -> ``(h_seq [T,B,H], h_T, c_T)``.

    ``lengths`` (int32 ``[B]``, right padding): at a step ``t >= lengths[b]`` row ``b`` holds its state (``h_t = h_{t-1}``,
    ``c_t = c_{t-1}``), so ``h_T`` / ``c_T`` are the state after the row's last real step - ``h_n`` / ``c_n`` of ``nn.LSTM`` on
    a packed sequence - and padded inputs get no gradient.

    ``reverse``: the reverse-time direction of a bidirectional layer.  Steps run from ``t = T-1`` down to 0, ``h_seq[t]`` is the
    state after step ``t`` (still in time order) and ``h_T`` / ``c_T`` are the state after step 0.  With ``lengths`` the padded
    steps come first and hold ``h0`` / ``c0``, so each row starts from ``h0`` at its own last real step - the reverse half of
    ``nn.LSTM(bidirectional=True)`` on a packed sequence."""
    T = x_seq.shape[0]
    keep = None
    if lengths is not None:
        check_lengths(lengths, x_seq.shape[1], T)
        keep = lengths.to(x_seq.device).long().view(-1, 1) > torch.arange(T, device=x_seq.device).view(1, -1)   # [B,T]
    h, c = h0, c0
    outs = []
    # hoisted input projection (same arithmetic as per-step x·W_x)
    gx = (x_seq.reshape(-1, x_seq.shape[-1]) @ w_x.t()).view(T, x_seq.shape[1], -1)
    for t in (range(T - 1, -1, -1) if reverse else range(T)):
        pre = gx[t] + h @ w_h.t() + bias
        i, f, g, o = lstm_gates(pre)
        c_new = f * c + i * g
        h_new = o * torch.tanh(c_new)
        if keep is None:
            c, h = c_new, h_new
        else:
            k = keep[:, t:t + 1]
            c, h = torch.where(k, c_new, c), torch.where(k, h_new, h)
        outs.append(h)
    if reverse:
        outs.reverse()
    return torch.stack(outs, 0), h, c


def dense_head(h, weights, bias):
    """logits = h · W + b with ``W [H, C]`` (reference: src/rnn.py:214-221)."""
    return h @ weights + bias


def softmax_xent(logits, labels, sparse: bool = True):
    """Mean softmax cross-entropy (reference: src/rnn.py:55-63)."""
    logp = torch.log_softmax(logits.float(), dim=-1)
    if sparse:
        nll = -logp.gather(1, labels.view(-1, 1).long()).squeeze(1)
    else:
        nll = -(labels.float() * logp).sum(-1)
    return nll.mean()


def accuracy(logits, labels, sparse: bool = True):
    """mean(argmax(logits) == labels) (reference: src/rnn.py:84-92)."""
    pred = logits.argmax(dim=1)
    tgt = labels if sparse else labels.argmax(dim=1)
    return (pred == tgt).float().mean()


def head_xent(h, weights, bias, labels):
    """Fused head: logits, mean loss, number of correct rows."""
    logits = dense_head(h.float(), weights.float(), bias.float())
    loss = softmax_xent(logits, labels)
    correct = (logits.argmax(1) == labels).sum()
    return logits, loss, correct


def adam_step_(p, g, m, v, step: int, lr: float, beta1: float = 0.9, beta2: float = 0.999,
               eps: float = 1e-8, weight_decay: float = 0.0, grad_scale: float = 1.0):
    """TF-1.0 Adam ("epsilon-hat"): lr_t = lr*sqrt(1-b2^t)/(1-b1^t); w -= lr_t*m/(sqrt(v)+eps)."""
    gg = g * grad_scale if grad_scale != 1.0 else g
    if weight_decay:
        gg = gg + weight_decay * p
    m.mul_(beta1).add_(gg, alpha=1.0 - beta1)
    v.mul_(beta2).addcmul_(gg, gg, value=1.0 - beta2)
    lr_t = lr * (1.0 - beta2 ** step) ** 0.5 / (1.0 - beta1 ** step)
    p.addcdiv_(m, v.sqrt().add_(eps), value=-lr_t)
    return p


def sgd_step_(p, g, lr: float, weight_decay: float = 0.0, grad_scale: float = 1.0):
    gg = g * grad_scale if grad_scale != 1.0 else g
    if weight_decay:
        gg = gg + weight_decay * p
    p.add_(gg, alpha=-lr)
    return p
