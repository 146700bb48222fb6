"""A reference for the persistent LSTM kernels (csrc/lstm_seq_wgmma.cu) that knows where their fast path rounds.

``layer`` / ``pair`` run one layer / a stacked pair forward AND backward with a hand-written backward loop (no autograd: at
T = 512, B = 64, H = 2048 a single fp64 [T, B, 4H] tensor is 2.1 GB, and the rounding points sit inside the backward):
  * ``rounding=None``: fp64 - the exact result of the operation on the inputs the kernels get;
  * ``rounding=Bf16(...)``: fp32 with every bf16 rounding of the fast path in its place - what an ideal kernel with those
    rounding points computes.  Its distance from fp64 is the error the bf16 storage alone explains;
  * ``rounding=Generic()``: the same for the bf16 generic path (H % 64 != 0 and other shapes the persistent kernels do not
    take: a CUDA-core GEMM per time step and the fused cell kernels of csrc/lstm_pointwise.cu);
  * ``rounding=Fp32()``: the fp32 generic path (``--dtype fp32``) - every operation in fp32, nothing rounded to bf16, exact
    activations.
``check_budget`` then holds a kernel's error against fp64 to ALPHA x the emulation's error (plus a small floor: FLOOR for the
bf16 arms, FLOOR_F32 for the fp32 one), per time step for the sequences, so that a defect confined to one step of hundreds
cannot hide in a global norm.  ``model`` composes the layers into the whole classifier (stacked, bidirectional, dropout, head)
with the same arms.

Rounding points of the fast path (ops/cuda_lstm.py, csrc/lstm_seq_wgmma.cu), all round-to-nearest-even:
  forward   gx = x W_x^T is stored bf16 (_gemm_tn); with the forward K-split (cluster of 2) a member adds the PEER's half of the
            recurrent product as bf16 to its own fp32 half; pre = rec + gx + bias (fp32 bias); h and the saved activations
            (i, f, g, o) are stored bf16, c stays fp32; h0 enters as bf16, c0 as fp32.
  backward  dh_seq enters as bf16, dh_T / dc_T as fp32; the recurrent product dG W_h is split into ``bwd_split`` K parts (4 with
            the weights resident, 2 streamed), each an fp32 partial sum rounded to bf16 for the DSMEM exchange and summed in
            fp32; the cell backward reads the bf16 activations and fp32 c, and stores dG as bf16; dW_x / dW_h are fp32 products
            of bf16 operands, db the fp32 column sum of the bf16 dG, dx = dG W_x is stored bf16.
  pair      h_seq of layer a (bf16) is layer b's input; dx of layer b (bf16) is layer a's dh_seq (ops/cuda_lstm._LSTMPairFn).

Rounding points of the bf16 generic path (ops/cuda_lstm._LSTMSeqFn with ``fast_path_supported`` false), where they differ:
  forward   pre = bf16(gx + h W_h^T): the GEMM adds the fp32 product to the bf16 gx in fp32 and stores the bf16 pre buffer,
            the fp32 bias is added to it afterwards by the cell kernel; no forward K-split;
  backward  the recurrent product dG W_h is fp32 and never rounded (the fp32 output of the GEMM, or accumulated into the fp32
            dh handed to the step before); gx, the activations, h, dG and dx are bf16 and c fp32 as on the fast path;
  dropout   the standalone dropout kernel masks the output (bf16(h x scale), as the fast path) and the incoming gradient,
            which it stores as bf16(dh x scale) before the cell kernel reads it.
The fp32 generic path has no rounding point besides fp32 arithmetic: its GEMMs accumulate in fp32 into fp32 outputs, and its
cell kernels compute the activations in fp64 and round them once (csrc/ts_common.cuh tanhf_acc / sigmoidf_acc).

The optimizer update (csrc/multi_tensor_opt.cu, TF-1.0 Adam with "epsilon-hat" or SGD over the flat fp32 master buffer) has no
bf16 rounding point and no emulation arm: ``adam_update`` / ``sgd_update`` compute it in fp64 from the kernel's own fp32
inputs, and ``check_update`` holds each element of the kernel's p, m, v to a worst-case bound built from sums of magnitudes
(m and gg = g s + wd p can cancel, so a bound relative to the result would not hold).  With u = 2^-24:
  gg        fp32 product and sum: <= 2u (|g| s + wd |p|) =: 2u |gg|_abs;
  m         b1 m + (1 - b1) gg (1 - b1 is exact in fp32, Sterbenz): three roundings on top of gg's, 8u (b1 |m| + (1 - b1) |gg|_abs);
  v         b2 v + (1 - b2) gg^2 likewise, 8u (b2 v + (1 - b2) |gg|_abs^2);
  p         p - D with D = lr_t m' / (sqrt(v') + eps): 2u |p| for the subtraction, RHO |D| for the relative error of D itself,
            and lr_t (bound on m') / (sqrt(v') + eps) for the error m' brings along;
  floor     2^-100 absolute everywhere: build.py compiles with --use_fast_math, which flushes denormals to zero.
RHO = 2^-11 is D's relative error under --use_fast_math, derived from the documented intrinsic bounds (not measured):
  lr_t = lr sqrt(1 - b2^t) / (1 - b1^t) from step_dev: powf becomes __powf = ex2.approx(t __log2f(b2)).  __log2f's absolute
            error of about 2^-21.4 becomes a relative error of t ln2 2^-21.4 in b2^t, and ex2.approx adds 2^-22.5; 1 - b2^t
            magnifies it by b2^t / (1 - b2^t), whose product with t is largest at t = 1 (1 / (1 - b2) = 1000): <= 4.2e-4 in
            1 - b2^t, 2.1e-4 in its square root.  The same term for b1 (1 / (1 - b1) = 10) is below 2e-6;
  D         sqrt.approx and the approximate division add a few ulp (< 1e-6).
So D is within 2.2e-4 of its exact value and RHO leaves a factor of 2.2.  SGD (p - lr (g s + wd p)) has no approximate
operation: 2u |p| + 4u lr |gg|_abs.  The bf16 shadow the update kernels write has no tolerance: it must be the master rounded
to nearest even, bit for bit (``check_shadow``).
"""
from __future__ import annotations

import dataclasses
import math
from typing import NamedTuple, Optional

import torch

KB = 64            # columns of one operand k-block of the persistent kernels
ROWS = 16          # rows of one wgmma row group

# The kernel's error may be at most ALPHA times the emulation's (both measured against fp64) ...
ALPHA = 2.0
# ... plus FLOOR x |fp64|.  The emulation computes tanh / sigmoid exactly; the kernels use tanh.approx.f32 (relative error
# <= 2^-11; sigmoid(x) = 0.5 tanh(x / 2) + 0.5).  One step's h = o * tanh(c) carries two such approximations, so a kernel
# that is exact up to them may sit 2 x 2^-11 away from the emulation where the emulation itself happens to be exact.
FLOOR = 2.0 * 2.0 ** -11
# The fp32 path's floor: its activations are correctly rounded up to a last-bit error, so the floor only has to absorb fp32
# rounding of a different order than the emulation's where the emulation happens to be close to fp64 - a few ulp.  A kernel
# whose tanh were off by 2^-15 (let alone tanh.approx's 2^-11) exceeds it.
FLOOR_F32 = 2.0 ** -20


@dataclasses.dataclass(frozen=True)
class Bf16:
    """The fast path's rounding: ``fwd_split`` K parts of the forward recurrent product (2 = forward K-split), ``bwd_split``
    K parts of the backward one (4 resident weights, 2 streamed).  ``approx``: relative error put on every tanh (a
    deterministic function of its argument, like tanh.approx's) - only for stand-ins of a kernel in tests of this module."""
    fwd_split: int = 1
    bwd_split: int = 4
    approx: float = 0.0

    @classmethod
    def for_layer(cls, H: int, B: int, variant: int = 0) -> "Bf16":
        """The splits the kernels use for H, B and a variant (``lstm_seq_config``: no device needed)."""
        from lstm_tensorspark_b200.ops.cuda_ext import ext
        fwd = ext().lstm_seq_config(False, H, B, variant)
        bwd = ext().lstm_seq_config(True, H, B, variant)
        return cls(fwd_split=2 if fwd[3] else 1, bwd_split=2 if bwd[2] else 4)


@dataclasses.dataclass(frozen=True)
class Generic:
    """The bf16 generic path's rounding (module docstring).  ``approx``: as ``Bf16.approx``."""
    approx: float = 0.0


@dataclasses.dataclass(frozen=True)
class Fp32:
    """The fp32 generic path: fp32 arithmetic, no bf16 rounding, exact sigmoid and tanh.  ``split``: the recurrent products
    as the fp32 sum of that many K parts (another order of the same fp32 sums); ``approx``: as ``Bf16.approx`` - both only for
    stand-ins of a kernel in tests of this module."""
    split: int = 1
    approx: float = 0.0


@dataclasses.dataclass(frozen=True)
class Defect:
    """A defect to plant into a run (tests of the budget's sensitivity).  ``step``: processing step (0 = the first step of
    the direction); ``index``: the k-block (``drop_kblock``: of h in the forward recurrent product; ``zero_dg``: of dG) or the
    16-row group (``stale_rows``: its recurrent operand is h from one step earlier).
    Defects of the model composition (``model``; every layer / layer boundary):
      ``fwd_dx_only``      at time ``step`` the lower layer's incoming gradient is the forward upper direction's dx alone;
      ``mask_next_step``   the backward masks dropout with the mask of training step ``step + 1``;
      ``lost_chunk``       weight and bias gradients lose batch rows [0, ``index``) (a second batch chunk overwrote the sink);
      ``reverse_unmasked`` the reverse direction ignores ``lengths`` and starts at T - 1."""
    kind: str
    step: int
    index: int


class LayerOut(NamedTuple):
    h_seq: torch.Tensor
    h_T: torch.Tensor
    c_T: torch.Tensor
    dx: torch.Tensor
    dh0: torch.Tensor
    dc0: torch.Tensor
    dw_x: torch.Tensor
    dw_h: torch.Tensor
    db: torch.Tensor


def _round(r, x: torch.Tensor) -> torch.Tensor:
    return x if r is None or isinstance(r, Fp32) else x.to(torch.bfloat16).to(x.dtype)


def _tanh(r, x: torch.Tensor) -> torch.Tensor:
    y = torch.tanh(x)
    if r is not None and r.approx:
        y = y * (1.0 + r.approx * torch.sin(x * 4099.0))
    return y


def _sigmoid(r, x: torch.Tensor) -> torch.Tensor:
    if r is None or (isinstance(r, Fp32) and not r.approx):
        return torch.sigmoid(x)
    return 0.5 * _tanh(r, 0.5 * x) + 0.5


def _split_mm(a, b, parts):
    """a @ b as the fp32 sum of ``parts`` products over K slices (Fp32.split)."""
    q = -(-a.shape[1] // parts)
    return sum(a[:, s:s + q] @ b[s:s + q] for s in range(0, a.shape[1], q))


def _keep(lengths, T, B, device):
    if lengths is None:
        return None
    return lengths.to(device).long().view(B, 1) > torch.arange(T, device=device).view(1, T)      # [B, T]


def _rec_fwd(r, h, w_h):
    """h_{t-1} W_h^T.  Forward K-split: gate column n belongs to cluster member m = (n % 128) // 64, which contracts K half m
    itself (fp32) and receives the other half from its peer as bf16."""
    if isinstance(r, Fp32) and r.split > 1:
        return _split_mm(h, w_h.t(), r.split)
    if r is None or not isinstance(r, Bf16) or r.fwd_split == 1:
        return h @ w_h.t()
    hk = h.shape[1] // 2
    p0 = h[:, :hk] @ w_h[:, :hk].t()
    p1 = h[:, hk:] @ w_h[:, hk:].t()
    own0 = (torch.arange(w_h.shape[0], device=h.device) % (2 * KB)) < KB
    return torch.where(own0, p0 + _round(r, p1), p1 + _round(r, p0))


def _rec_bwd(r, dg, w_h):
    """dG W_h: ``bwd_split`` fp32 partial sums over K quarters / halves, each rounded to bf16, summed in fp32 (the fast path);
    one fp32 product, not rounded (the generic paths)."""
    if isinstance(r, Fp32) and r.split > 1:
        return _split_mm(dg, w_h, r.split)
    if r is None or not isinstance(r, Bf16):
        return dg @ w_h
    q = dg.shape[1] // r.bwd_split
    out = None
    for s in range(r.bwd_split):
        part = _round(r, dg[:, s * q:(s + 1) * q] @ w_h[s * q:(s + 1) * q])
        out = part if out is None else out + part
    return out


def _forward(x, h0, c0, w_x, w_h, bias, keep, reverse, r, defect):
    dt = torch.float64 if r is None else torch.float32
    T, B, D = x.shape
    H = w_h.shape[1]
    w_h = w_h.to(dt)
    gx = _round(r, x.reshape(T * B, D).to(dt) @ w_x.to(dt).t()).view(T, B, 4 * H)
    bias = bias.to(dt)
    h, c = _round(r, h0.to(dt)), c0.to(dt)
    hs = torch.empty(T + 1, B, H, dtype=dt, device=x.device)
    cs = torch.empty(T + 1, B, H, dtype=dt, device=x.device)
    acts = torch.empty(T, B, H, 4, dtype=dt, device=x.device)
    s0 = T if reverse else 0
    hs[s0], cs[s0] = h, c
    h_before = h
    for n, t in enumerate(range(T - 1, -1, -1) if reverse else range(T)):
        hin = h
        if defect is not None and defect.step == n and defect.kind in ("drop_kblock", "stale_rows"):
            hin = h.clone()
            if defect.kind == "drop_kblock":
                hin[:, KB * defect.index:KB * (defect.index + 1)] = 0
            else:
                rows = slice(ROWS * defect.index, ROWS * (defect.index + 1))
                hin[rows] = h_before[rows]
        rec = _rec_fwd(r, hin, w_h) + gx[t]
        if isinstance(r, Generic):
            rec = _round(r, rec)                      # the GEMM's bf16 output buffer, before the cell kernel adds the bias
        pre = (rec + bias).view(B, H, 4)
        i, f = _sigmoid(r, pre[..., 0]), _sigmoid(r, pre[..., 1])
        g, o = _tanh(r, pre[..., 2]), _sigmoid(r, pre[..., 3])
        c_new = f * c + i * g
        h_new = _round(r, o * _tanh(r, c_new))
        acts[t] = _round(r, torch.stack((i, f, g, o), -1))
        if keep is not None:
            k = keep[:, t:t + 1]
            c_new, h_new = torch.where(k, c_new, c), torch.where(k, h_new, h)
        h_before = h
        h, c = h_new, c_new
        sn = t if reverse else t + 1
        hs[sn], cs[sn] = h, c
    return hs, cs, acts


def _backward(fw, x, w_x, w_h, dh_seq, dh_T, dc_T, keep, reverse, r, defect, dh_scale=None):
    """``dh_scale`` [T,B,H]: dropout's mask x scale on this layer's output, applied to the bf16 dh_seq as it is loaded."""
    hs, cs, acts = fw
    dt = hs.dtype
    T, B, H = acts.shape[:3]
    D = x.shape[2]
    w_h = w_h.to(dt)
    zeros = lambda: torch.zeros(B, H, dtype=dt, device=hs.device)
    dh = dh_T.to(dt) if dh_T is not None else zeros()
    dc = dc_T.to(dt) if dc_T is not None else zeros()
    dgs = torch.empty(T, B, 4 * H, dtype=dt, device=hs.device)
    for n, t in enumerate(range(T) if reverse else range(T - 1, -1, -1)):
        sp, sn = (t + 1, t) if reverse else (t, t + 1)
        if dh_seq is None:
            dht = dh
        elif dh_scale is None:
            dht = dh + _round(r, dh_seq[t].to(dt))
        elif isinstance(r, Generic):                  # the standalone dropout kernel stores bf16(dh_seq x mask x scale)
            dht = dh + _round(r, _round(r, dh_seq[t].to(dt)) * dh_scale[t])
        else:
            dht = dh + _round(r, dh_seq[t].to(dt)) * dh_scale[t]
        i, f, g, o = acts[t].unbind(-1)
        tcn = _tanh(r, cs[sn])
        dct = dc + dht * o * (1 - tcn * tcn)
        dg = torch.stack((dct * g * i * (1 - i), dct * cs[sp] * f * (1 - f), dct * i * (1 - g * g), dht * tcn * o * (1 - o)), -1)
        dg = _round(r, dg.view(B, 4 * H))
        if defect is not None and defect.step == n and defect.kind == "zero_dg":
            dg[:, KB * defect.index:KB * (defect.index + 1)] = 0
        if keep is None:
            dc = dct * f
            dh = _rec_bwd(r, dg, w_h)
        else:                                 # padded step: no gate gradient, dh / dc pass through to the step before
            k = keep[:, t:t + 1]
            dg = torch.where(k, dg, 0.0)
            dc = torch.where(k, dct * f, dc)
            dh = torch.where(k, 0.0, dht) + _rec_bwd(r, dg, w_h)
        dgs[t] = dg
    dg2d = dgs.view(T * B, 4 * H)
    h_prev = hs[1:] if reverse else hs[:T]
    rows = slice(defect.index, None) if defect is not None and defect.kind == "lost_chunk" else slice(None)
    dg_w = dgs[:, rows].reshape(-1, 4 * H)
    dw_x = dg_w.t() @ x[:, rows].reshape(-1, D).to(dt)
    dw_h = dg_w.t() @ h_prev[:, rows].reshape(-1, H)
    dx = _round(r, dg2d @ w_x.to(dt)).view(T, B, D)
    return dx, dh, dc, dw_x, dw_h, dg_w.sum(0)


def _state_out(fw, reverse):
    hs, cs, _ = fw
    T = hs.shape[0] - 1
    return (hs[:T], hs[0], cs[0]) if reverse else (hs[1:], hs[T], cs[T])


def layer(x, h0, c0, w_x, w_h, bias, dh_seq, dh_T, dc_T, lengths=None, reverse=False, rounding: Optional[Bf16] = None,
          defect: Optional[Defect] = None) -> LayerOut:
    """One layer forward and backward (``ops/reference.lstm_layer_sequence`` semantics, masking and reverse included) for
    the loss whose gradients into h_seq / h_T / c_T are ``dh_seq`` / ``dh_T`` / ``dc_T`` (each may be None = zero)."""
    T, B, _ = x.shape
    keep = _keep(lengths, T, B, x.device)
    fw = _forward(x, h0, c0, w_x, w_h, bias, keep, reverse, rounding, defect)
    return LayerOut(*_state_out(fw, reverse), *_backward(fw, x, w_x, w_h, dh_seq, dh_T, dc_T, keep, reverse, rounding, defect))


def pair(x, la, lb, dh_seq, dh_T_a, dc_T_a, dh_T_b, dc_T_b, lengths=None, rounding=None):
    """Two stacked layers as ``ops/cuda_lstm._LSTMPairFn`` composes them; ``la`` / ``lb`` = (h0, c0, w_x, w_h, bias).
    ``rounding``: None, one Bf16 for both layers or a (layer a, layer b) tuple.  -> (LayerOut of a, LayerOut of b): the
    pair's outputs are b.h_seq, a.h_T, a.c_T, b.h_T, b.c_T; its input gradient is a.dx (b.dx is the gradient into a.h_seq)."""
    ra, rb = rounding if isinstance(rounding, tuple) else (rounding, rounding)
    T, B, _ = x.shape
    keep = _keep(lengths, T, B, x.device)
    fa = _forward(x, *la, keep, False, ra, None)
    h_seq_a = fa[0][1:]
    fb = _forward(h_seq_a, *lb, keep, False, rb, None)
    gb = _backward(fb, h_seq_a, lb[2], lb[3], dh_seq, dh_T_b, dc_T_b, keep, False, rb, None)
    ga = _backward(fa, x, la[2], la[3], gb[0], dh_T_a, dc_T_a, keep, False, ra, None)
    return LayerOut(*_state_out(fa, False), *ga), LayerOut(*_state_out(fb, False), *gb)


class Dropout(NamedTuple):
    """Dropout between stacked layers in one training step: ``RNN.dropout_spec``'s P, (seed, partition) key and step count."""
    p: float
    key: tuple
    step: int


class ModelOut(NamedTuple):
    loss: Optional[torch.Tensor]     # mean cross-entropy (None without a head)
    h_T: torch.Tensor                # the classifier's input [B, H_last] (bidirectional: [B, 2 H_last], forward half first)
    grads: dict                      # "LSTMLayer<l>[_reverse]/<h0|c0|w_x|w_h|bias>", "Dense1/weights", "Dense1/bias" -> gradient


def _drop_scale(dropout, layer, reverse, T, B, H, dt, device):
    """mask x scale [T,B,H] of one layer direction's output (``reference.dropout_mask``, keyed as ``RNN.dropout_spec``)."""
    from lstm_tensorspark_b200.ops import reference as ref
    spec = ref.DropoutSpec(dropout.p, tuple(dropout.key), layer, reverse, int(dropout.step))
    keep = ref.dropout_mask(spec, T, B, H, device=device)
    return keep.to(dt) * ref.dropout_scale(dropout.p).to(dt).to(device)


def model(x, layers, head, labels, lengths=None, bidirectional=False, dropout: Optional[Dropout] = None, rounding=None,
          defect: Optional[Defect] = None, dh_T=None, backward=True) -> ModelOut:
    """The whole classifier (``models.classifier.SequenceClassifier`` in training mode on the CUDA path) forward and backward,
    composed from the layer loops above.  ``x [B,T,D]`` batch-major; ``layers``: per layer (h0, c0, w_x, w_h, bias) - for a
    bidirectional stack a (forward, reverse) pair of them; ``head``: (W [H_in, C], b [C]) and ``labels`` [B] - or None and
    ``dh_T``, the gradient into h_T; ``dropout``: None or ``Dropout``.  ``rounding``: None (fp64) or the fast path's: one
    Bf16 for every layer, or one per layer (each a Bf16 or a (forward, reverse) pair).  ``backward=False``: loss and h_T only.

    Rounding points on top of the layers' (module docstring), all in the emulation only:
      between layers  the next layer reads the bf16 h_seq; with dropout bf16(h * scale) under the mask, and the lower layer
                      multiplies the bf16 dx it receives by the same mask x scale in fp32 as it loads it;
      bidirectional   the next layer reads [h_fwd | h_rev]; the lower layer's incoming gradient is the sum of the two upper
                      directions' bf16 dx, rounded to bf16 once (autograd adds the two bf16 gradients of the shared input);
      head            logits = bf16 h_T x bf16(W) in fp32 + fp32 bias; softmax, NLL, dlogits = (p - onehot) / B in fp32;
                      dh = dlogits W^T with the fp32 W, stored bf16; dW = h_T^T dlogits and db in fp32.  The top layer
                      receives dh as dh_T (no dh_seq, dc_T = 0)."""
    dt = torch.float64 if rounding is None else torch.float32
    dev = x.device
    B, T, _ = x.shape
    L = len(layers)
    dirs = (False, True) if bidirectional else (False,)
    keep = _keep(lengths, T, B, dev)

    def rnd(l, d):
        r = rounding[l] if isinstance(rounding, (list, tuple)) else rounding
        return r[d] if isinstance(r, tuple) else r

    def params(l, d):
        return layers[l][d] if bidirectional else layers[l]

    def name(l, d):
        return f"LSTMLayer{l}" + ("_reverse" if dirs[d] else "")

    seq = x.transpose(0, 1).to(dt)                                          # time-major [T,B,D], as RNN.fit_layers feeds it
    saved = []                                                              # per layer: [(forward state, input, keep, scale)]
    for l in range(L):
        outs, sv = [], []
        for d, rev in enumerate(dirs):
            r, p = rnd(l, d), params(l, d)
            kp = None if rev and defect is not None and defect.kind == "reverse_unmasked" else keep
            fw = _forward(seq, *p, kp, rev, r, None)
            h_seq = _state_out(fw, rev)[0]
            sc = None
            if dropout is not None and dropout.p > 0 and l < L - 1:
                sc = _drop_scale(dropout, l, rev, T, B, h_seq.shape[2], dt, dev)
                h_seq = _round(r, h_seq * sc)
            outs.append(h_seq)
            sv.append((fw, seq, kp, sc))
        saved.append(sv)
        seq = torch.cat(outs, 2) if bidirectional else outs[0]
    r_top = rnd(L - 1, 0)
    h_T = torch.cat([_state_out(saved[L - 1][d][0], rev)[1] for d, rev in enumerate(dirs)], 1)
    loss = None
    grads = {}
    if head is not None:
        W, b = head[0].to(dt), head[1].to(dt)
        logits = h_T @ _round(r_top, W) + b
        logp = torch.log_softmax(logits, 1)
        lab = labels.long().view(-1, 1).to(dev)
        loss = -logp.gather(1, lab).mean()
        if backward:
            dlogits = (logp.exp() - torch.zeros_like(logp).scatter_(1, lab, 1.0)) / B
            dh_T = _round(r_top, dlogits @ W.t())
            grads["Dense1/weights"] = h_T.t() @ dlogits
            grads["Dense1/bias"] = dlogits.sum(0)
    if not backward:
        return ModelOut(loss, h_T, grads)
    H_top = h_T.shape[1] // len(dirs)
    incoming = [None] * len(dirs)                       # the gradient into each direction's output sequence (bf16 dx above)
    for l in range(L - 1, -1, -1):
        dxs = []
        for d, rev in enumerate(dirs):
            fw, x_in, kp, sc = saved[l][d]
            p, r = params(l, d), rnd(l, d)
            if sc is not None and defect is not None and defect.kind == "mask_next_step":
                sc = _drop_scale(dropout._replace(step=dropout.step + 1), l, rev, T, B, sc.shape[2], dt, dev)
            top = dh_T[:, d * H_top:(d + 1) * H_top] if l == L - 1 else None
            g = _backward(fw, x_in, p[2], p[3], incoming[d], top, None, kp, rev, r, defect, dh_scale=sc)
            for k, v in zip(("h0", "c0", "w_x", "w_h", "bias"), g[1:]):
                grads[f"{name(l, d)}/{k}"] = v
            dxs.append(g[0])
        if l == 0:
            break
        if bidirectional:
            total = _round(rnd(l, 0), dxs[0] + dxs[1])
            if defect is not None and defect.kind == "fwd_dx_only":
                total[defect.step] = dxs[0][defect.step]
            H_low = total.shape[2] // 2
            incoming = [total[..., :H_low], total[..., H_low:]]
        else:
            incoming = [dxs[0]]
    return ModelOut(loss, h_T, grads)


def check_budget(name: str, got: torch.Tensor, fp64: torch.Tensor, emulated: torch.Tensor, per_step: bool = False,
                 alpha: float = ALPHA, floor: float = FLOOR) -> float:
    """Assert |got - fp64| <= alpha |emulated - fp64| + floor |fp64| (L2 norms: per time step along dim 0 with
    ``per_step``, else over the whole tensor) and return the worst ratio of the left side to the right side."""
    ref = fp64.double()
    g = got.detach().double().to(ref.device)
    e = emulated.double().to(ref.device)
    if not per_step:
        ref, g, e = ref.reshape(1, -1), g.reshape(1, -1), e.reshape(1, -1)
    dims = tuple(range(1, ref.dim()))
    ek = torch.linalg.vector_norm(g - ref, dim=dims)
    ee = torch.linalg.vector_norm(e - ref, dim=dims)
    sc = torch.linalg.vector_norm(ref, dim=dims)
    bound = alpha * ee + floor * sc
    ratio = torch.where(bound > 0, ek / bound.clamp_min(1e-300), torch.where(ek > 0, float("inf"), 0.0))
    ratio = torch.where(torch.isnan(ratio), float("inf"), ratio)
    s = int(ratio.argmax())
    worst = float(ratio[s])
    if not worst <= 1.0:
        where = f" at step {s}" if per_step else ""
        raise AssertionError(
            f"{name}{where}: error vs fp64 {float(ek[s]):.3e} exceeds {alpha} x the emulation's {float(ee[s]):.3e} + "
            f"{floor:.2e} x |fp64| {float(sc[s]):.3e} (ratio {worst:.2f}; kernel / emulation error "
            f"{float(ek[s]) / max(float(ee[s]), 1e-300):.2f})")
    return worst


# ---- the optimizer update (module docstring) -------------------------------------------------------------------------------
U = 2.0 ** -24
RHO = 2.0 ** -11
UPDATE_FLOOR = 2.0 ** -100


class Update(NamedTuple):
    """One update in fp64 and the element-wise bound on a kernel's error in each tensor (m / v None for SGD)."""
    p: torch.Tensor
    m: Optional[torch.Tensor]
    v: Optional[torch.Tensor]
    bound_p: torch.Tensor
    bound_m: Optional[torch.Tensor]
    bound_v: Optional[torch.Tensor]


def f32(x: float) -> float:
    """``x`` as the fp32 value a ``float`` kernel argument receives."""
    return float(torch.tensor(float(x), dtype=torch.float32))


def _decayed(p, g, wd, grad_scale, wd_numel):
    """gg = g s + wd p in fp64, the weight decay on flat elements [0, ``wd_numel``) only (-1: all), and |g| s + wd |p|."""
    p, g = p.double(), g.double()
    w = torch.zeros_like(p)
    w.view(-1)[:p.numel() if wd_numel < 0 else wd_numel] = f32(wd)
    s = f32(grad_scale)
    return g * s + w * p, g.abs() * s + w * p.abs()


def adam_update(p, m, v, g, t: Optional[int], lr: float, b1: float = 0.9, b2: float = 0.999, eps: float = 1e-8,
                wd: float = 0.0, grad_scale: float = 1.0, wd_numel: int = -1) -> Update:
    """``flat_adam_kernel`` (``ops/reference.adam_step_``'s math) on the kernel's fp32 ``p``, ``m``, ``v`` before the step and
    gradient ``g`` (flat, contiguous).  ``t``: the step count the kernel reads from ``step_dev`` after its increment - ``lr``
    is then the base learning rate; None: ``lr`` is the host-computed lr_t.  The scalars are taken as the fp32 values the
    kernel receives."""
    lr, b1, b2, eps = f32(lr), f32(b1), f32(b2), f32(eps)
    gg, ga = _decayed(p, g, wd, grad_scale, wd_numel)
    m, v = m.double(), v.double()
    lr_t = lr if t is None else lr * math.sqrt(1.0 - b2 ** t) / (1.0 - b1 ** t)
    m1 = b1 * m + (1.0 - b1) * gg
    v1 = b2 * v + (1.0 - b2) * gg * gg
    den = v1.sqrt() + eps
    step = lr_t * m1 / den
    bm = 8 * U * (b1 * m.abs() + (1.0 - b1) * ga) + UPDATE_FLOOR
    bv = 8 * U * (b2 * v + (1.0 - b2) * ga * ga) + UPDATE_FLOOR
    bp = 2 * U * p.double().abs() + RHO * step.abs() + lr_t * bm / den + UPDATE_FLOOR
    return Update(p.double() - step, m1, v1, bp, bm, bv)


def sgd_update(p, g, lr: float, wd: float = 0.0, grad_scale: float = 1.0, wd_numel: int = -1) -> Update:
    """``flat_sgd_kernel`` (``ops/reference.sgd_step_``'s math), as ``adam_update``."""
    lr = f32(lr)
    gg, ga = _decayed(p, g, wd, grad_scale, wd_numel)
    bp = 2 * U * p.double().abs() + 4 * U * lr * ga + UPDATE_FLOOR
    return Update(p.double() - lr * gg, None, None, bp, None, None)


def check_update(name: str, got: torch.Tensor, ref: torch.Tensor, bound: torch.Tensor) -> float:
    """Assert |got - ref| <= bound element by element and return the worst ratio of the two sides."""
    g = got.detach().double().to(ref.device).reshape(-1)
    r, b = ref.reshape(-1), bound.reshape(-1)
    ratio = (g - r).abs() / b
    ratio = torch.where(torch.isnan(ratio), float("inf"), ratio)
    i = int(ratio.argmax())
    worst = float(ratio[i])
    if not worst <= 1.0:
        at = tuple(int(k) for k in torch.unravel_index(torch.tensor(i), tuple(ref.shape)))
        over = int((~(ratio <= 1.0)).sum())
        raise AssertionError(
            f"{name}: element {at}: {float(g[i]):.9e} vs fp64 {float(r[i]):.9e}, error {abs(float(g[i]) - float(r[i])):.3e} "
            f"exceeds the bound {float(b[i]):.3e} (ratio {worst:.2f}; {over} of {r.numel()} elements over)")
    return worst


def check_shadow(name: str, shadow: torch.Tensor, master: torch.Tensor) -> None:
    """Assert the bf16 ``shadow`` is ``master`` rounded to nearest even, bit for bit."""
    want = master.detach().to(torch.bfloat16).reshape(-1)
    got = shadow.detach().reshape(-1)
    bad = got.view(torch.int16) != want.view(torch.int16)
    if bool(bad.any()):
        i = int(bad.nonzero()[0])
        raise AssertionError(f"{name}: the bf16 shadow differs from the rounded master at {int(bad.sum())} of {bad.numel()} "
                             f"elements; first at {i}: {float(got[i]):.6e} vs {float(want[i]):.6e} (master "
                             f"{float(master.reshape(-1)[i]):.9e})")
