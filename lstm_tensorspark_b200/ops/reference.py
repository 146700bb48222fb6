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
import math
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


WEIGHT_DROP_C2 = 0x80000000      # high bit of c2: the weight-drop masks (DropoutSpec.weight)
INPUT_DROP_C2 = 0x40000000       # the embedding output x_t, over its E units (DropoutSpec.site "input")
LOCKED_C2 = 0x20000000           # a locked mask: the counter's time word is 0, one mask for every step (DropoutSpec.locked)
ROW_DROP_C2 = 0x10000000         # whole rows of the embedding table (DropoutSpec.site "rows")
DROPOUT_SITES = ("layer", "input", "rows")


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
    reads its current value), an int on the CPU.  ``row0``: batch row of local row 0 (batch chunks).

    ``weight``: the weight-drop stream instead (DropConnect on the layer direction's ``W_h [4H, H]``, ``weight_drop``): the
    matrix is one time step of 4H rows and c2 = 0x80000000 | (2 layer + reverse), apart from every output stream's c2 < 2^31.

    ``site``: ``"layer"`` (a layer's output: between layers, and the top layer's with ``--output_dropout``), ``"input"`` (the
    embedding output ``x_t [B, E]``, c2 = 0x40000000; ``layer`` / ``reverse`` unused) or ``"rows"`` (whole rows of the ``[V, E]``
    embedding table: one step of one row of V units, c2 = 0x10000000).  ``locked``: one mask per sequence and step, shared by
    every time step (AWD-LSTM's ``LockedDropout``): c2 gains 0x20000000 and the counter's time word is 0 (layer and input sites)."""
    p: float
    key: Tuple[int, int]
    layer: int
    reverse: bool
    step: Union[int, torch.Tensor]
    row0: int = 0
    weight: bool = False
    site: str = "layer"
    locked: bool = False

    def __post_init__(self):
        if self.site not in DROPOUT_SITES:
            raise ValueError(f"dropout site must be one of {', '.join(DROPOUT_SITES)}, got {self.site!r}")
        if self.locked and (self.weight or self.site == "rows"):
            raise ValueError("only the layer and input masks can be locked: weight drop and row masks have no time axis")

    @property
    def thr(self) -> int:
        return dropout_threshold(self.p)

    @property
    def c2(self) -> int:
        if self.weight:
            return WEIGHT_DROP_C2 | (2 * self.layer + int(self.reverse))
        if self.site == "rows":
            return ROW_DROP_C2
        base = INPUT_DROP_C2 if self.site == "input" else 2 * self.layer + int(self.reverse)
        return (LOCKED_C2 if self.locked else 0) | base

    def desc(self):
        """{key0, key1, thr, c2, row0} as the kernels take it."""
        return [self.key[0] & _U32, self.key[1] & _U32, self.thr, self.c2, self.row0]

    def at_rows(self, row0: int) -> "DropoutSpec":
        return dataclasses.replace(self, row0=self.row0 + row0)


def dropout_mask(spec: DropoutSpec, T: int, B: int, H: int, t0: int = 0, device=None) -> torch.Tensor:
    """Keep mask ``[T,B,H]`` (bool) of ``spec`` at times ``t0 .. t0 + T - 1``: counter (b * ceil(H/8) + j/8, t, c2, step),
    unit 8g + i takes 16-bit half (i & 1) of word i/2 and is kept iff that value >= thr.  A locked spec's counter has time word
    0 at every t."""
    step = int(spec.step) & _U32
    g = (H + 7) // 8
    t = torch.arange(t0, t0 + T, dtype=torch.int64, device=device).view(T, 1, 1).expand(T, B, g)
    if spec.c2 & LOCKED_C2:
        t = torch.zeros_like(t)
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


def weight_drop_mask(spec: DropoutSpec, rows: int, H: int, device=None) -> torch.Tensor:
    """Keep mask ``[rows, H]`` (bool) of a weight-drop ``spec``: ``dropout_mask`` of one time step (t = 0) of ``rows`` rows, so row
    r, unit k takes counter (r ceil(H/8) + k/8, 0, c2, step).  Row r is the stored (gate-interleaved) row of ``W_h``."""
    return dropout_mask(spec, 1, rows, H, device=device)[0]


def weight_drop(w_h: torch.Tensor, spec: Optional[DropoutSpec]) -> torch.Tensor:
    """Weight drop (DropConnect on the recurrent weights, AWD-LSTM's ``WeightDrop``): ``W_h * M * s`` of a ``weight`` spec, rounded
    to ``W_h``'s dtype once; the gradient reaching ``W_h`` is ``M * s`` times the gradient of the masked matrix.  ``spec`` None or
    P = 0: ``w_h`` itself."""
    if spec is None or spec.p == 0:
        return w_h
    return dropout(w_h.unsqueeze(0), spec)[0]


def lstm_layer_sequence(x_seq, h0, c0, w_x, w_h, bias, lengths: Optional[torch.Tensor] = None, reverse: bool = False,
                        dropout: Optional[DropoutSpec] = None, weight_drop: Optional[DropoutSpec] = None, activation_sums: bool = False):
    """Unrolled layer: ``x_seq [T,B,D]`` -> ``(h_seq [T,B,H], h_T, c_T)``.

    ``lengths`` (int32 ``[B]``, right padding): at a step ``t >= lengths[b]`` row ``b`` holds its state (``h_t = h_{t-1}``,
    ``c_t = c_{t-1}``), so ``h_T`` / ``c_T`` are the state after the row's last real step - ``h_n`` / ``c_n`` of ``nn.LSTM`` on
    a packed sequence - and padded inputs get no gradient.

    ``reverse``: the reverse-time direction of a bidirectional layer.  Steps run from ``t = T-1`` down to 0, ``h_seq[t]`` is the
    state after step ``t`` (still in time order) and ``h_T`` / ``c_T`` are the state after step 0.  With ``lengths`` the padded
    steps come first and hold ``h0`` / ``c0``, so each row starts from ``h0`` at its own last real step - the reverse half of
    ``nn.LSTM(bidirectional=True)`` on a packed sequence.

    ``dropout``: the first output is the dropped sequence (``dropout`` below) - the input of the next layer; the final state is
    not dropped.

    ``weight_drop``: a ``weight`` ``DropoutSpec``; every step and row reads ``weight_drop(w_h, spec)`` in place of ``w_h``, built
    inside autograd, so ``w_h`` gets the masked gradient.

    ``activation_sums``: a fourth output, ``activation_sums(first output, undropped h_seq, lengths)``."""
    T = x_seq.shape[0]
    w_h = _weight_drop(w_h, weight_drop)
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
    raw = torch.stack(outs, 0)
    out = _dropout(raw, dropout)
    if activation_sums:
        return out, h, c, _activation_sums(out, raw, lengths)
    return out, h, c


def activation_sums(out: torch.Tensor, h: torch.Tensor, lengths: Optional[torch.Tensor] = None) -> torch.Tensor:
    """AWD-LSTM's activation regularisation, unnormalised: ``[2]`` = (sum of ``out[t,b,j]^2`` over the counted positions
    ``t < len_b``, sum of ``(h[t,b,j] - h[t-1,b,j])^2`` over ``1 <= t < len_b``).  ``out`` is the top layer's output as the head
    reads it (after ``--output_dropout``), ``h`` the raw output in time order, both ``[T,B,W]``; ``len_b = T`` without
    ``lengths``.  AR = sums[0] / (W sum_b len_b), TAR = sums[1] / (W sum_b max(len_b - 1, 0)): ``activation_penalties``.  fp32
    (fp64 for fp64 inputs), through autograd."""
    T, B, _ = h.shape
    dt = torch.float64 if h.dtype == torch.float64 else torch.float32
    keep = step_mask(lengths, B, T, device=h.device).t().unsqueeze(2)                       # [T,B,1]
    zero = torch.zeros((), dtype=dt, device=h.device)
    ar = torch.where(keep, out.to(dt), zero).square().sum()
    d = h[1:].to(dt) - h[:-1].to(dt)
    tar = torch.where(keep[1:], d, zero).square().sum()
    return torch.stack([ar, tar])


_activation_sums = activation_sums


def activation_penalties(sums: torch.Tensor, width: int, T: int, B: int, lengths: Optional[torch.Tensor] = None) -> torch.Tensor:
    """``[2]`` = (AR, TAR) from the summed ``activation_sums`` of an output ``width`` units wide: each sum over its count of terms,
    ``N_ar = width * sum_b len_b`` and ``N_tar = width * sum_b max(len_b - 1, 0)`` (``len_b = T`` without ``lengths``), and 0 where
    that count is 0.  Computed on the sums' device from ``lengths`` without reading it on the host."""
    if lengths is None:                       # (host numbers: no copy to the device, which a captured graph could not hold)
        return torch.stack([sums[i] / n if n > 0 else torch.zeros_like(sums[i]) for i, n in enumerate((width * B * T,
                                                                                                     width * B * (T - 1)))])
    lg = lengths.to(sums.device).long()
    n = torch.stack([lg.sum(), (lg - 1).clamp(min=0).sum()]).to(sums.dtype) * width
    return torch.where(n > 0, sums / n.clamp(min=1), torch.zeros((), dtype=sums.dtype, device=sums.device))


_dropout = dropout          # (lstm_layer_sequence's arguments shadow these functions)
_weight_drop = weight_drop


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


def step_mask(lengths: Optional[torch.Tensor], B: int, T: int, device=None) -> torch.Tensor:
    """``[B,T]`` bool: position (b, t) counts iff ``t < lengths[b]`` (every position without lengths)."""
    if lengths is None:
        return torch.ones(B, T, dtype=torch.bool, device=device)
    return lengths.to(device).long().view(B, 1) > torch.arange(T, device=device).view(1, T)


def head_xent_per_step(h_seq, weights, bias, labels, lengths=None):
    """The head at every time step (sequence labelling): ``h_seq [T,B,H]``, ``labels`` int64 ``[B,T]`` -> (logits ``[B,T,C]``,
    loss, correct, N).  Only counted positions (``step_mask``) enter the loss and the accuracy, and their labels alone are
    read; loss = the summed NLL / N, N = the number of counted positions: ``F.cross_entropy`` over the packed outputs."""
    T, B, _ = h_seq.shape
    dt = torch.float64 if h_seq.dtype == torch.float64 else torch.float32
    logits = dense_head(h_seq.to(dt), weights.to(dt), bias.to(dt)).transpose(0, 1)         # [B,T,C]
    keep = step_mask(lengths, B, T, device=h_seq.device)
    lg, lab = logits[keep], labels.to(h_seq.device)[keep].long()
    loss = torch.nn.functional.cross_entropy(lg, lab, reduction="sum") / keep.sum()
    correct = (lg.argmax(1) == lab).sum()
    return logits, loss, correct, keep.sum()


def vocab_xent_per_step(h_seq, weights, bias, labels, lengths=None, class_major: bool = False):
    """``head_xent_per_step`` without the logits -> (loss, correct, N): the reference of the large-vocabulary head.
    ``class_major``: ``weights`` is ``[C,H]`` = ``W^T`` (a tied embedding table)."""
    return head_xent_per_step(h_seq, weights.t() if class_major else weights, bias, labels, lengths)[1:]


# ---- sampling the next token ------------------------------------------------------------------------------------------
# The definition is shared with the CUDA kernels (csrc/head_vocab.cu sample_score): change both or neither.
SAMPLE_KEY1 = 0x53414D50


def sample_noise_words(B: int, C: int, seed: int, step: int, device=None, row0: int = 0) -> torch.Tensor:
    """``[B, C]`` int64 u32 words: class ``c`` of row ``b`` at decode step ``step`` takes word ``c & 3`` of Philox4x32-10 at key
    ``(seed & 0xffffffff, SAMPLE_KEY1)`` and counter ``(c >> 2, row0 + b, step, 0)``.  ``row0`` places the batch in a larger set
    of prompts (the index of its first prompt), so that no two prompts of a generation share a noise stream."""
    G = (C + 3) // 4
    g = torch.arange(G, dtype=torch.int64, device=device).view(1, G).expand(B, G)
    b = ((torch.arange(B, dtype=torch.int64, device=device) + int(row0)) & _U32).view(B, 1).expand(B, G)
    ctr = torch.stack([g, b, torch.full_like(g, int(step) & _U32), torch.zeros_like(g)], -1)
    return philox4x32_10(ctr, int(seed) & _U32, SAMPLE_KEY1).reshape(B, 4 * G)[:, :C]


def sample_uniform(words: torch.Tensor) -> torch.Tensor:
    """u = ((word >> 8) + 0.5) * 2^-24, exact in fp64 and strictly inside (0, 1), so no score is infinite.  (In fp32 u is exact
    below 1/2 and 1 - u above it: the kernels take -log u from whichever is exact.)"""
    return ((words >> 8).double() + 0.5) * 2.0 ** -24


def sample_scores(logits: torch.Tensor, temperature: float, seed: int, step: int, row0: int = 0) -> torch.Tensor:
    """Perturbed scores ``[B, C]`` in fp64: the logits at temperature 0, else ``l / t + g`` with the Gumbel noise
    ``g = -log(-log u)`` of ``sample_noise_words``."""
    l = logits.double()
    if temperature == 0:
        return l
    u = sample_uniform(sample_noise_words(l.shape[0], l.shape[1], seed, step, device=l.device, row0=row0))
    return l / temperature - torch.log(-torch.log(u))


def check_sample_filters(top_k, top_p) -> None:
    """Raise unless ``top_k`` is an int >= 0 (0 = off) and ``top_p`` a finite number in (0, 1] (1 = off)."""
    if isinstance(top_k, bool) or int(top_k) != top_k or top_k < 0:
        raise ValueError(f"top_k must be an integer >= 0 (0 = off), got {top_k}")
    if not (math.isfinite(top_p) and 0 < top_p <= 1):
        raise ValueError(f"top_p must be a finite number in (0, 1] (1 = off), got {top_p}")


def sample_filters_active(num_classes: int, temperature: float, top_k: int = 0, top_p: float = 1.0) -> bool:
    """Does a filter change the draw: temperature > 0 and ``0 < top_k < C`` or ``top_p < 1``?  (Greedy always keeps the arg-max.)"""
    return temperature > 0 and (0 < top_k < num_classes or top_p < 1)


def sample_threshold(logits: torch.Tensor, temperature: float, top_k: int = 0, top_p: float = 1.0) -> torch.Tensor:
    """The kept set's threshold ``tau [B]`` (fp64) of top-k / top-p sampling: row b keeps ``{c : l_c >= tau_b}`` (-inf: every
    class).  In fp64, with the definition of csrc/head_vocab.cu:

    * top-k (``0 < k < C``): ``tau_k`` = the k-th largest logit counted with multiplicity (every class tied at it is kept);
    * top-p (``0 < p < 1``): ``q = softmax(l / t)`` over ``{l >= tau_k}`` (every class without top-k); ``tau`` = the largest
      logit value v whose set ``{l >= v}`` holds q-mass >= p (ties at v are kept).  Top-k first, then top-p: the order of
      Hugging Face's samplers.
    Temperature 0 or both filters off: -inf."""
    check_sample_filters(top_k, top_p)
    l = logits.double()
    B, C = l.shape
    tau = torch.full((B,), float("-inf"), dtype=torch.float64, device=l.device)
    if not sample_filters_active(C, temperature, top_k, top_p):
        return tau
    if 0 < top_k < C:
        tau = l.topk(int(top_k), 1).values[:, -1]
    if top_p < 1:
        keep = l >= tau.unsqueeze(1)
        mx = l.max(1, keepdim=True).values
        e = torch.where(keep, torch.exp((l - mx) / temperature), torch.zeros((), dtype=torch.float64, device=l.device))
        vals, order = l.sort(1, descending=True)
        cum = e.gather(1, order).cumsum(1)
        first = (cum >= top_p * e.sum(1, keepdim=True)).int().argmax(1)      # the first position from the top where it holds
        tau = vals.gather(1, first.view(-1, 1)).squeeze(1)
    return tau


def sample_logits(logits: torch.Tensor, temperature: float, seed: int, step: int, row0: int = 0, top_k: int = 0,
                  top_p: float = 1.0):
    """Sample one token per row of ``logits [B, C]`` -> (tokens int32 [B], log p(token) under softmax(logits), fp64 [B]).

    Temperature 0: the arg-max, the smallest index on a tie, and no noise.  Temperature t > 0: Gumbel-max,
    ``argmax_c (l_c / t + g_c)``, an exact draw from ``softmax(l / t)``; the noise is counter-based (``sample_noise_words``), so
    row b at step s gets the draw of counter row ``row0 + b`` whatever else is in the batch.  ``top_k`` / ``top_p``
    (``sample_threshold``): the argmax runs over the kept classes only, with the same noise, an exact draw from ``softmax(l / t)``
    restricted to them and renormalised; the token is the unfiltered one whenever that one is kept.  The log-probability is under
    the model's own full ``softmax(l)`` at every temperature and filter."""
    if not (math.isfinite(temperature) and temperature >= 0):
        raise ValueError(f"temperature must be finite and >= 0, got {temperature}")
    check_sample_filters(top_k, top_p)
    l = logits.double()
    s = sample_scores(l, temperature, seed, step, row0)
    if sample_filters_active(l.shape[1], temperature, top_k, top_p):
        keep = l >= sample_threshold(l, temperature, top_k, top_p).unsqueeze(1)
        s = torch.where(keep, s, torch.full((), float("-inf"), dtype=torch.float64, device=l.device))
    tok = s.argmax(1)
    logp = torch.log_softmax(l, 1).gather(1, tok.view(-1, 1)).squeeze(1)
    return tok.to(torch.int32), logp


def vocab_sample(h, weights, bias, temperature: float, seed: int, step, row0: int = 0, class_major: bool = False, top_k: int = 0,
                 top_p: float = 1.0):
    """``sample_logits`` of ``l = h W + bias`` (``h [B,H]``, ``W [H,C]``; ``class_major``: ``weights`` is ``[C,H]`` = ``W^T``)
    computed in fp64: the reference of the sampling op."""
    w = weights.t() if class_major else weights
    return sample_logits(dense_head(h.double(), w.double(), bias.double()), temperature, seed, int(step), int(row0), top_k, top_p)


def softmax_xent_per_step(logits, labels, lengths=None):
    """``logits [B,T,C]``, ``labels [B,T]`` -> (mean NLL over counted positions, correct count among them, N)."""
    keep = step_mask(lengths, logits.shape[0], logits.shape[1], device=logits.device)
    lg, lab = logits[keep].float(), labels.to(logits.device)[keep].long()
    n = keep.sum()
    return torch.nn.functional.cross_entropy(lg, lab, reduction="sum") / n, (lg.argmax(1) == lab).sum(), n


def label_logprob(logits, labels):
    """``logits [B,T,C]``, ``labels [B,T]`` -> ``log softmax(logits)[label]`` ``[T·B]`` in time-major row order (row t·B + b)."""
    lp = torch.log_softmax(logits, dim=2).gather(2, labels.to(logits.device).long().unsqueeze(2)).squeeze(2)
    return lp.transpose(0, 1).reshape(-1)


# ---- continuous cache pointer (Grave et al. 2017) ----------------------------------------------------------------------
# The definition is shared with the CUDA kernels (csrc/cache_pointer.cu): change both or neither.
def cache_ring_positions(capacity: int, end: int, device=None) -> torch.Tensor:
    """The stream position each ring slot holds once positions ``0 .. end - 1`` have been written to slot ``position % capacity``:
    the largest ``q < end`` with ``q % capacity == slot``, -1 where none is."""
    slot = torch.arange(capacity, device=device, dtype=torch.int64)
    last = end - 1
    q = last - ((last - slot) % capacity)
    return torch.where(q >= 0, q, torch.full_like(q, -1))


def cache_pointer(h_seq, labels, logp_model, keys, key_labels, seen: int, window: int, theta: float, lam: float, lengths=None):
    """The continuous cache pointer's log p(y) of one segment of ``B`` streams, in the dtype of ``h_seq`` / ``keys``.

    ``h_seq [T,B,H]``: the segment's top-layer outputs (queries), ``labels [B,T]``: y_p, the id after position p,
    ``logp_model [T·B]``: the model's log p_v(y_p) in time-major row order, ``keys [B,Cap,H]`` / ``key_labels [B,Cap]``: each
    stream's ring with the segment already written (position j in slot j % Cap, Cap >= window + T), ``seen``: positions of each
    stream before the segment, ``lengths``: optional ``[B]`` counted positions per stream (a tail segment).  For the query at
    absolute position p, J(p) = {j : max(0, p - window) <= j < p}, s_j = theta (h_p . h_j), and

        log p(y_p) = logaddexp(log1p(-lam) + log p_v(y_p), log lam + log sum_{j in J, y_j = y_p} e^{s_j} - log sum_{j in J} e^{s_j})

    (J empty: log p_v(y_p)).  -> (log p ``[T·B]``, 0 at uncounted positions; counted mask ``[T·B]``)."""
    T, B, _ = h_seq.shape
    dev = h_seq.device
    cap = keys.shape[1]
    if cap < window + T:
        raise ValueError(f"the ring holds {cap} positions, fewer than the window {window} plus the segment {T}")
    pos = cache_ring_positions(cap, seen + T, dev)                                       # [Cap]
    p = seen + torch.arange(T, device=dev, dtype=torch.int64)                             # [T]
    valid = (pos.view(1, -1) >= (p.view(-1, 1) - window).clamp(min=0)) & (pos.view(1, -1) < p.view(-1, 1))   # [T,Cap]
    s = theta * torch.einsum("tbh,bch->btc", h_seq, keys.to(h_seq.dtype))                # [B,T,Cap]
    s = s.masked_fill(~valid.unsqueeze(0), float("-inf"))
    same = key_labels.to(dev).long().unsqueeze(1) == labels.to(dev).long().unsqueeze(2)  # [B,T,Cap]
    lz = torch.logsumexp(s, dim=2)                                                        # [B,T]
    lm = torch.logsumexp(s.masked_fill(~same, float("-inf")), dim=2)
    lv = logp_model.to(h_seq.dtype).view(T, B).t()
    empty = ~valid.any(1).view(1, T).expand(B, T)
    neg_inf = torch.full_like(lv, float("-inf"))
    a = math.log1p(-lam) + lv
    c = (math.log(lam) + (lm - lz)) if lam > 0 else neg_inf
    c = torch.where(torch.isfinite(c), c, neg_inf)
    lp = torch.where(empty, lv, torch.where(torch.isinf(c), a, torch.logaddexp(a, c)))
    keep = step_mask(lengths, B, T, device=dev)
    lp = torch.where(keep, lp, torch.zeros_like(lp))
    return lp.t().reshape(-1), keep.t().reshape(-1)


POOLING_MODES = ("last", "mean", "max", "attention")


def pool_sequence(h_seq, lengths=None, mode: str = "mean", attention=None):
    """Pool the top layer's output over the counted steps (``step_mask``): ``h_seq [T,B,H]`` -> ``s [B,H]`` (fp32; fp64 for
    fp64 ``h_seq``).  ``mean``: the mean over t < len_b.  ``max``: the per-unit max; its gradient goes to the smallest t that
    attains it.  ``attention`` with ``attention = (W_a [H,A], b_a [A], v [A])``: u = tanh(h W_a + b_a), e = u . v, alpha =
    softmax over the counted t (0 elsewhere), s = sum_t alpha_t h_t.  Uncounted positions are replaced by zeros before anything
    reads them, so their values reach neither the result nor a gradient (theirs is 0)."""
    T, B, _ = h_seq.shape
    dt = torch.float64 if h_seq.dtype == torch.float64 else torch.float32
    keep = step_mask(lengths, B, T, device=h_seq.device).t()                                 # [T,B]
    h = torch.where(keep.unsqueeze(2), h_seq.to(dt), torch.zeros((), dtype=dt, device=h_seq.device))
    if mode == "mean":
        n = keep.sum(0).to(dt)
        return h.sum(0) / n.unsqueeze(1)
    if mode == "max":
        hm = torch.where(keep.unsqueeze(2), h, torch.full((), float("-inf"), dtype=dt, device=h.device))
        top = hm.max(0, keepdim=True).values
        t_idx = torch.arange(T, device=h.device).view(T, 1, 1).expand_as(hm)
        first = torch.where(hm == top, t_idx, T).min(0, keepdim=True).values                  # the smallest t at the max
        return h.gather(0, first).squeeze(0)
    if mode == "attention":
        if attention is None:
            raise ValueError("attention pooling needs its parameters (W_a, b_a, v)")
        w_a, b_a, v = (p.to(dt) for p in attention)
        u = torch.tanh(h @ w_a + b_a)
        e = torch.where(keep, u @ v, torch.full((), float("-inf"), dtype=dt, device=h.device))
        alpha = torch.softmax(e, 0)
        return (alpha.unsqueeze(2) * h).sum(0)
    raise ValueError(f"unknown pooling {mode!r}: one of {', '.join(POOLING_MODES)}")


def embedding_row_mask(spec: DropoutSpec, V: int, device=None) -> torch.Tensor:
    """Keep mask ``[V]`` (bool) of a ``"rows"`` spec (embedding dropout): ``dropout_mask`` of one step of one row of V units, so id
    v takes unit v % 8 of counter (v / 8, 0, c2, step)."""
    return dropout_mask(spec, 1, 1, V, device=device)[0, 0]


def dropout_factor(*specs: Optional[DropoutSpec]) -> torch.Tensor:
    """fp32 factor of a unit kept by every active spec: the scale of the one spec on, or the fp32 product of the scales."""
    on = [s for s in specs if s is not None and s.p > 0]
    f = dropout_scale(on[0].p)
    for s in on[1:]:
        f = dropout_scale(s.p) * f
    return f


def embedding(tokens, table, lengths=None, input_dropout: Optional[DropoutSpec] = None,
              embedding_dropout: Optional[DropoutSpec] = None):
    """Token embedding in front of the first layer (``--vocab_size``): ``nn.Embedding`` read time-major.  ``tokens`` int ``[B,T]``
    (or ``[B]``, one step), ``table [V,E]``, ``lengths`` optional int ``[B]`` -> ``x [T,B,E]`` of the table's dtype with
    ``x[t,b] = table[tokens[b,t]]`` at counted positions (``t < lengths[b]``, id in ``[0, V)``) and 0 elsewhere.  Uncounted
    positions give the table no gradient; a counted one adds its ``dx`` to its id's row.

    ``input_dropout``: an ``"input"`` spec; unit e of position (t, b) is kept where ``dropout_mask(spec, T, B, E)`` is.
    ``embedding_dropout``: a ``"rows"`` spec; a position reads 0 where its id's row is dropped (``embedding_row_mask``).  A
    kept unit is ``w * f`` (``dropout_factor``), rounded once to the table's dtype (bf16: from float(w); fp64: ``w`` times each
    scale); the gradient follows through autograd."""
    tok = tokens.long()
    if tok.dim() == 1:
        tok = tok.unsqueeze(1)
    tok = tok.t()                                                    # [T,B]
    T, B = tok.shape
    V, E = table.shape
    keep = (tok >= 0) & (tok < V)
    if lengths is not None:
        keep = keep & (torch.arange(T, device=tok.device).unsqueeze(1) < lengths.to(tok.device).long().unsqueeze(0))
    safe = torch.where(keep, tok, torch.zeros_like(tok))
    rows = table[safe]                                               # [T,B,E]
    specs = [s for s in (input_dropout, embedding_dropout) if s is not None and s.p > 0]
    if not specs:
        return rows * keep.unsqueeze(2).to(table.dtype)
    if embedding_dropout is not None and embedding_dropout.p > 0:
        keep = keep & embedding_row_mask(embedding_dropout, V, device=tok.device)[safe]
    keep = keep.unsqueeze(2).expand(T, B, E)
    if input_dropout is not None and input_dropout.p > 0:
        keep = keep & dropout_mask(input_dropout, T, B, E, device=tok.device)
    if rows.dtype == torch.float64:                                   # (fp64: one product per scale, no fp32 rounding)
        y = rows
        for s in specs:
            y = y * dropout_scale(s.p).double()
    elif rows.dtype == torch.float32:
        y = rows * dropout_factor(*specs)
    else:
        y = (rows.float() * dropout_factor(*specs)).to(rows.dtype)
    return torch.where(keep, y, torch.zeros((), dtype=table.dtype, device=table.device))


def clip_coefficient(g_total_segments, max_norm: float):
    """Clipping by the global norm (``torch.nn.utils.clip_grad_norm_``): ``norm = ||g_total||_2`` over all segments, summed in
    fp64 and rounded to the segments' dtype, and ``coef = min(max_norm / (norm + 1e-6), 1)`` in that dtype (a NaN norm gives a
    NaN coef, an infinite one 0).  -> (norm, coef), 0-dim tensors."""
    segs = [s.reshape(-1) for s in g_total_segments]
    dtype = segs[0].dtype
    sq = sum(s.double().square().sum() for s in segs)
    norm = sq.sqrt().to(dtype)
    coef = torch.clamp(max_norm / (norm + 1e-6), max=1.0)
    return norm, coef


def adam_step_(p, g, m, v, step: int, lr: float, beta1: float = 0.9, beta2: float = 0.999,
               eps: float = 1e-8, weight_decay: float = 0.0, grad_scale: float = 1.0, clip_coef=None):
    """TF-1.0 Adam ("epsilon-hat"): lr_t = lr*sqrt(1-b2^t)/(1-b1^t); w -= lr_t*m/(sqrt(v)+eps).  ``clip_coef``: the update
    uses clip_coef * (g * grad_scale + weight_decay * p)."""
    gg = g * grad_scale if grad_scale != 1.0 else g
    if weight_decay:
        gg = gg + weight_decay * p
    if clip_coef is not None:
        gg = gg * clip_coef
    m.mul_(beta1).add_(gg, alpha=1.0 - beta1)
    v.mul_(beta2).addcmul_(gg, gg, value=1.0 - beta2)
    lr_t = lr * (1.0 - beta2 ** step) ** 0.5 / (1.0 - beta1 ** step)
    p.addcdiv_(m, v.sqrt().add_(eps), value=-lr_t)
    return p


def sgd_step_(p, g, lr: float, weight_decay: float = 0.0, grad_scale: float = 1.0, clip_coef=None):
    gg = g * grad_scale if grad_scale != 1.0 else g
    if weight_decay:
        gg = gg + weight_decay * p
    if clip_coef is not None:
        gg = gg * clip_coef
    p.add_(gg, alpha=-lr)
    return p


def asgd_average_(ax, p, k: int):
    """The k-th (k = 1, 2, ...) averaging step of ``torch.optim.ASGD(lambd=0, t0=0)``, in torch's indexing and order: k <= 2
    copies ``ax = p``; after that ``ax += (p - ax) * mu_k`` with ``mu_k = fp32(1 / (k - 1))``, each operation rounded on its own
    (no fused multiply-add).  So ``ax_k = mean(p_2 .. p_k)`` for k >= 2."""
    if k <= 2:
        return ax.copy_(p)
    mu = torch.tensor(1.0 / (k - 1), dtype=torch.float32, device=ax.device)
    return ax.add_(p.sub(ax).mul_(mu))
