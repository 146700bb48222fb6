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

import dataclasses
from typing import Optional, Tuple, Union

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


# ---- dropout between stacked layers ---------------------------------------------------------------------------------
# The mask format is shared with the CUDA kernels (csrc/ts_common.cuh dropout_keep8): change both or neither.
PHILOX_M = (0xD2511F53, 0xCD9E8D57)
PHILOX_W = (0x9E3779B9, 0xBB67AE85)
_U32 = 0xFFFFFFFF


def _mulhilo32(a: torch.Tensor, m: int):
    """(hi, lo) 32-bit words of ``a * m`` for int64 tensors holding u32 values (16-bit halves: no int64 overflow)."""
    p = a * (m & 0xFFFF)
    q = a * (m >> 16)
    s = p + ((q & 0xFFFF) << 16)
    return (q >> 16) + (s >> 32), s & _U32


def philox4x32_10(ctr: torch.Tensor, key0, key1) -> torch.Tensor:
    """Philox4x32-10 (Random123): ``ctr [..., 4]`` u32 values in an integer tensor, key words ints or int64 tensors that
    broadcast against ``ctr[..., 0]`` -> ``[..., 4]`` int64 u32 words."""
    c = [ctr[..., i].to(torch.int64) for i in range(4)]
    k0 = torch.as_tensor(key0, dtype=torch.int64) & _U32
    k1 = torch.as_tensor(key1, dtype=torch.int64) & _U32
    for r in range(10):
        if r > 0:
            k0, k1 = (k0 + PHILOX_W[0]) & _U32, (k1 + PHILOX_W[1]) & _U32
        hi0, lo0 = _mulhilo32(c[0], PHILOX_M[0])
        hi1, lo1 = _mulhilo32(c[2], PHILOX_M[1])
        c = [hi1 ^ c[1] ^ k0, lo1, hi0 ^ c[3] ^ k1, lo0]
    return torch.stack(c, -1)


def dropout_threshold(p: float) -> int:
    """A unit is kept iff its 16-bit value is >= this: P quantised to 1/65536."""
    return min(int(round(p * 65536)), 65535)


def dropout_scale(p: float) -> torch.Tensor:
    """fp32 scale of a kept unit, 65536 / (65536 - thr) rounded once (the kernels compute the same fp32 quotient)."""
    return torch.tensor(65536.0, dtype=torch.float32) / torch.tensor(float(65536 - dropout_threshold(p)), dtype=torch.float32)


@dataclasses.dataclass(frozen=True)
class DropoutSpec:
    """Dropout on one layer's output sequence (one direction) in one training step, as ``nn.LSTM(dropout=p)``.

    ``key``: (seed, partition) - replicas draw different masks.  ``layer`` / ``reverse``: counter word c2 = 2 layer + reverse.
    ``step``: training steps completed (counter word c3) - an int32 ``[1]`` device tensor on the CUDA path (a captured graph
    reads its current value), an int on the CPU.  ``row0``: batch row of local row 0 (batch chunks)."""
    p: float
    key: Tuple[int, int]
    layer: int
    reverse: bool
    step: Union[int, torch.Tensor]
    row0: int = 0

    @property
    def thr(self) -> int:
        return dropout_threshold(self.p)

    @property
    def c2(self) -> int:
        return 2 * self.layer + int(self.reverse)

    def desc(self):
        """{key0, key1, thr, c2, row0} as the kernels take it."""
        return [self.key[0] & _U32, self.key[1] & _U32, self.thr, self.c2, self.row0]

    def at_rows(self, row0: int) -> "DropoutSpec":
        return dataclasses.replace(self, row0=self.row0 + row0)


def dropout_mask(spec: DropoutSpec, T: int, B: int, H: int, t0: int = 0, device=None) -> torch.Tensor:
    """Keep mask ``[T,B,H]`` (bool) of ``spec`` at times ``t0 .. t0 + T - 1``: counter (b * ceil(H/8) + j/8, t, c2, step),
    unit 8g + i takes 16-bit half (i & 1) of word i/2 and is kept iff that value >= thr."""
    step = int(spec.step) & _U32
    g = (H + 7) // 8
    t = torch.arange(t0, t0 + T, dtype=torch.int64, device=device).view(T, 1, 1).expand(T, B, g)
    b = torch.arange(B, dtype=torch.int64, device=device).view(1, B, 1) + spec.row0
    c0 = (b * g + torch.arange(g, dtype=torch.int64, device=device).view(1, 1, g)).expand(T, B, g)
    ctr = torch.stack([c0, t, torch.full_like(c0, spec.c2), torch.full_like(c0, step)], -1)
    w = philox4x32_10(ctr, spec.key[0], spec.key[1])                                   # [T,B,g,4]
    vals = torch.stack([w & 0xFFFF, w >> 16], -1).reshape(T, B, 8 * g)                # unit 8g + i: word i/2, half i & 1
    return vals[..., :H] >= spec.thr


def dropout(x: torch.Tensor, spec: Optional[DropoutSpec], t0: int = 0) -> torch.Tensor:
    """``x [T,B,H]`` or ``[B,H]`` (time t0) -> ``x * mask * scale``, rounded to x's dtype once (bf16: from the stored value, as
    the kernels); the gradient is mask * scale.  ``spec`` None or P = 0: x itself."""
    if spec is None or spec.p == 0:
        return x
    x3 = x if x.dim() == 3 else x.unsqueeze(0)
    keep = dropout_mask(spec, x3.shape[0], x3.shape[1], x3.shape[2], t0, device=x.device).view(x.shape)
    scale = dropout_scale(spec.p)
    if x.dtype in (torch.float32, torch.float64):
        y = x * scale.to(x.dtype)
    else:
        y = (x.float() * scale).to(x.dtype)
    return torch.where(keep, y, torch.zeros((), dtype=x.dtype, device=x.device))


def lstm_layer_sequence(x_seq, h0, c0, w_x, w_h, bias, lengths: Optional[torch.Tensor] = None, reverse: bool = False,
                        dropout: Optional[DropoutSpec] = None):
    """Unrolled layer: ``x_seq [T,B,D]`` -> ``(h_seq [T,B,H], h_T, c_T)``.

    ``lengths`` (int32 ``[B]``, right padding): at a step ``t >= lengths[b]`` row ``b`` holds its state (``h_t = h_{t-1}``,
    ``c_t = c_{t-1}``), so ``h_T`` / ``c_T`` are the state after the row's last real step - ``h_n`` / ``c_n`` of ``nn.LSTM`` on
    a packed sequence - and padded inputs get no gradient.

    ``reverse``: the reverse-time direction of a bidirectional layer.  Steps run from ``t = T-1`` down to 0, ``h_seq[t]`` is the
    state after step ``t`` (still in time order) and ``h_T`` / ``c_T`` are the state after step 0.  With ``lengths`` the padded
    steps come first and hold ``h0`` / ``c0``, so each row starts from ``h0`` at its own last real step - the reverse half of
    ``nn.LSTM(bidirectional=True)`` on a packed sequence.

    ``dropout``: the first output is the dropped sequence (``dropout`` below) - the input of the next layer; the final state is
    not dropped."""
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
    return _dropout(torch.stack(outs, 0), dropout), h, c


_dropout = dropout          # (lstm_layer_sequence's argument shadows the function)


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
