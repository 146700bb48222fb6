"""CUDA LSTM layer ops = autograd.Functions around the hand-written kernels.

Fast path (bf16, H % 64 == 0, grid <= #SMs): hoisted input projection on the wgmma GEMM (csrc/gemm2_wgmma.cu) + ONE
persistent wgmma kernel for the whole recurrence in each direction (csrc/lstm_seq_wgmma.cu; weights resident in SMEM
up to H = 1024, streamed through the ring above).  Two stacked layers run as ONE layer wavefront (``_LSTMPairFn``: both
recurrences co-resident, the upper layer's x-projection / dX as a dataflow-gated GEMM on the idle SMs).  Generic path (any
shape / fp32): our CUDA-core GEMM per step (csrc/gemm_generic.cu) + the fused pointwise cell kernels (csrc/lstm_pointwise.cu).
Weight gradients are wgmma GEMMs over all T at once (``[4H, T·B] x [T·B, D | H]``, both operands MN-major and read in
place), fp32, written straight into the flat gradient buffer; bias gradients are deterministic column sums running next to
them, or, for the lower layer of the pipelined pair, row sums of dG^T computed by its dW_h GEMM itself.  Nothing in here reaches cuBLAS / cuDNN.  Math parity: original src/models/recurrent/lstm.py:88-122.
"""
from __future__ import annotations

import os
from typing import Optional

import torch

from .cuda_ext import STATS, count, ext
from .cuda_ext import drop_args as _drop_args
from .params import Countdown, after_big_launch, big_launch_begin, grad_out, lowp, release
from . import cuda_gemm as G

_SYNC_WS = {}
_SM_COUNT = {}
FORCE_GENERIC = os.environ.get("LSTM_TS_FORCE_GENERIC", "0") == "1"
# Tuning knob of the persistent kernels (0 = defaults), bit fields as decoded in csrc/lstm_seq_wgmma.cu seq_config():
#   [0:4) batch tiles per CTA (2 = one CTA alternates two tiles), [4:8) ring stages (0 = auto), [12:15) 3 = in-order operand
#   stream (--deterministic), bit 16 sync mode (0 per-k-block dataflow counters, 1 one counter per batch tile = grid barrier).
#   The kernels refuse any other bit, and any other value in [12:15).
SEQ_VARIANT = int(os.environ.get("LSTM_TS_SEQ_VARIANT", "0"))


def _grad_gemm(w_addr: int, a_t: torch.Tensor, b: torch.Tensor, b_folded: bool = False, pdl: bool = False, max_ctas: int = 0,
               ctas: int = 0, rowsum=None, masked: bool = False) -> tuple:
    """dW = a_t @ b in fp32 (``a_t`` = dG^T as a transposed view, ``b`` = the layer input: both operands MN-major, read in
    place by the wgmma GEMM; ``b_folded``: ``b`` is the batch-major [B,T,D] array standing for the time-major [T*B, D]
    matrix).  When the parameter lives in a FlatParams buffer the product lands straight in its grad
    view (overwrite on the first write of a step, accumulate afterwards) and None is returned to autograd.
    ``pdl``: launch as a programmatic dependent of the previous kernel (single-CTA tiles on at most ``max_ctas`` SMs, next to a
    recurrence that is still running).  Such a GEMM is no "big launch" for the gradient buckets: what precedes it in the stream
    may still be running when it starts, so no bucket's allreduce is launched under it.  ``ctas``: CTAs per tile cluster of
    an ordinary launch (0 = ``cuda_gemm.GEMM_CTAS``).  ``rowsum``: see ``cuda_gemm.matmul`` (the bias gradient, summed by the
    same launch).  ``masked``: an accumulating sink gets the product in an fp32 scratch, for ``_weight_drop_grad`` to add in.
    -> ``(product, sink, what autograd gets)``, where ``product is sink`` unless it is that scratch."""
    ops = dict(a=a_t, b_t=None, b_folded=b, ctas=ctas) if b_folded else dict(a=a_t, b_t=b.t(), ctas=ctas)
    ops["rowsum"] = rowsum
    if pdl:
        ops.update(pdl=True, ctas=1, max_ctas=max_ctas)
    out, acc, ret = grad_out(w_addr, (a_t.shape[0], b.shape[-1]), a_t.device)
    scratch = masked and acc
    big = ret is None and not pdl
    if big:
        big_launch_begin()
    part = G.matmul(out_dtype=torch.float32, **ops) if scratch else G.matmul(out=out, accumulate=acc, **ops)
    if big:
        after_big_launch()               # finished buckets of earlier gradients: allreduce them under this GEMM
    return (part if scratch else out), out, ret


def _accumulate_grad(w_addr: int, a_t: torch.Tensor, b: torch.Tensor, wdrop=None, **gemm):
    """``_grad_gemm``, then with ``wdrop`` (``_drop_args`` of a weight-drop spec) ``_weight_drop_grad`` -> what autograd gets."""
    part, out, ret = _grad_gemm(w_addr, a_t, b, masked=bool(wdrop), **gemm)
    if wdrop:
        _weight_drop_grad(part, out, wdrop, part is not out)
    return ret


def _bias_grad(b_addr: int, dg2d: torch.Tensor, under_gemm: bool = False, part: int = -1, max_ctas: int = 0, sink=None):
    """db = column sums of dG; straight into the flat grad view when there is one.  ``under_gemm``: the previous launch of the
    stream is a weight-gradient GEMM over the same dG that leaves SMs idle - run next to it (programmatic dependent launch).
    ``part`` 0 / 1: only the first / second half of the columns (one half under each of the layer's two weight-gradient GEMMs:
    on the ~20 idle SMs a half takes about as long as the GEMM it hides under).  Part 0 returns its ``sink`` (None when the columns
    do not split), which the caller passes to part 1; otherwise -> what autograd gets.
    ``max_ctas`` (whole-column launches): at most that many CTAs, each walking several slabs (the same sums)."""
    n = dg2d.shape[1]
    if part >= 0 and dg2d.is_cuda and dg2d.dtype == torch.bfloat16 and n % 512 == 0 and dg2d.is_contiguous():
        out, acc, ret = sink = sink or grad_out(b_addr, (n,), dg2d.device)
        STATS["kernels"] += 1
        ext().colsum_bf16_into(dg2d, out, not acc, under_gemm, part * (n // 2), n // 2)
        return sink if part == 0 else ret
    if part == 0:
        return None                                   # everything happens with the part-1 call
    out, acc, ret = grad_out(b_addr, (n,), dg2d.device)
    if dg2d.is_cuda and dg2d.dtype == torch.bfloat16 and n % 256 == 0 and dg2d.is_contiguous():
        STATS["kernels"] += 1
        ext().colsum_bf16_into(dg2d, out, not acc, under_gemm and part < 0, max_ctas=max_ctas)
    else:
        ones = torch.ones(1, dg2d.shape[0], dtype=dg2d.dtype, device=dg2d.device)
        G.matmul(ones, dg2d.t(), out=out.view(1, -1), accumulate=acc)
    return ret


SYNC_WORDS = 8192        # csrc/lstm_seq_wgmma.cu kSyncWords; the last word is the sticky error flag


def _sync_ws(device) -> torch.Tensor:
    key = (device.type, device.index)
    if key not in _SYNC_WS:
        _SYNC_WS[key] = torch.zeros(SYNC_WORDS, dtype=torch.int32, device=device)
    return _SYNC_WS[key]


def check_kernel_errors(device) -> None:
    """Raise if a persistent kernel hit its bounded-spin timeout (sticky flag, costs one D2H read)."""
    ws = _SYNC_WS.get((device.type, device.index))
    if ws is not None and int(ws[SYNC_WORDS - 1].item()) != 0:
        raise RuntimeError("lstm_seq kernel aborted: an in-kernel wait timed out (see csrc/lstm_seq_wgmma.cu)")
    for (di, _tag), ent in list(globals().get("_WS_PAIR", {}).items()):
        if di == device.index and (int(ent[SYNC_WORDS - 1].item()) != 0 or int(ent[2 * SYNC_WORDS - 1].item()) != 0):
            raise RuntimeError("lstm_seq kernel (layer wavefront) aborted: an in-kernel wait timed out")


def _sms(device) -> int:
    key = device.index
    if key not in _SM_COUNT:
        _SM_COUNT[key] = torch.cuda.get_device_properties(device).multi_processor_count
    return _SM_COUNT[key]


_CORES = {}


def _coresident_ctas(device, cluster: int = 4) -> int:
    """CTAs of the persistent kernels that can be co-resident in thread-block clusters of ``cluster``: the backward kernel runs
    in clusters of 4 (resident weights) or 2 (streamed weights), and a GPC's SM count is not always a multiple of 4 (an H100
    co-schedules 120 CTAs in clusters of 4: fewer than the 128 of B = 256, H = 1024 at one batch tile per CTA)."""
    key = (device.index, cluster)
    if key not in _CORES:
        n = _sms(device)
        try:
            with torch.cuda.device(device):
                c = int(ext().lstm_seq_cluster_probe(cluster))
            if c > 0:
                n = min(n, cluster * c)
        except Exception:                                   # noqa: BLE001
            pass
        _CORES[key] = n
    return _CORES[key]


def _bwd_cluster(H: int) -> int:
    """Cluster size of the backward recurrence kernel: 4 with the weight slice resident (H <= 1024), 2 once it is streamed."""
    return 4 if H <= 1024 else 2


def tiles_per_cta(B: int, H: int, coresident: int) -> Optional[int]:
    """Batch tiles per CTA of the persistent kernels (1, or 2 when one tile per CTA needs more CTAs than can be co-resident),
    None when neither fits, with ``coresident`` CTAs of the backward kernel co-resident in its clusters (``_coresident_ctas``).
    H / 16 CTAs per batch tile (pair); all of them must be co-resident (dataflow sync between CTAs), in clusters for the
    backward pass.  Two tiles per CTA need the resident weight slice (H <= 1024); larger H streams it through the ring
    (csrc/lstm_seq_wgmma.cu, kStream; the streamed backward takes H <= 2048)."""
    if H > 2048:
        return None
    tiles_m = (B + 127) // 128
    if tiles_m * (H // 16) <= coresident:
        return 1
    if H <= 1024 and tiles_m % 2 == 0 and (tiles_m // 2) * (H // 16) <= coresident:
        return 2
    return None


def _tiles_per_cta(B: int, H: int, device) -> Optional[int]:
    return tiles_per_cta(B, H, _coresident_ctas(device, _bwd_cluster(H)))


def fwd_tiles_per_cta(B: int, H: int, sms: int, coresident) -> Optional[int]:
    """Batch tiles per CTA of a forward recurrence that has the GPU to itself, on a device with ``sms`` SMs;
    ``coresident(cluster)``: CTAs co-resident in thread-block clusters of that size (``_coresident_ctas``).
    ``tiles_per_cta`` picks the tile count from the backward kernel's clusters of 4, which an H100 co-schedules on only 120
    of its 132 SMs: at B = 256, H = 1024 that means two tiles on 64 CTAs.  The forward kernel runs without clusters (or in
    clusters of 2 with its K-split), so its 128 one-tile CTAs fit, and each then has half the MMA work per step and no second
    tile to wait behind.  1 where ``tiles_m * H / 16`` one-tile CTAs fit the forward kernel's own co-residency, else what
    ``tiles_per_cta`` returns."""
    tiles = tiles_per_cta(B, H, coresident(_bwd_cluster(H)))
    if tiles != 2:
        return tiles
    fsplit = ext().lstm_seq_config(False, H, B, SEQ_VARIANT & ~15)[3]      # the one-tile launch's K-split (no device needed)
    return 1 if (B + 127) // 128 * (H // 16) <= (coresident(2) if fsplit else sms) else 2


def _seq_variant(B: int, H: int, device) -> int:
    if SEQ_VARIANT & 15 or _tiles_per_cta(B, H, device) != 2:
        return SEQ_VARIANT
    return SEQ_VARIANT | 2


def _fwd_full_width(B: int, H: int, device) -> bool:
    """Does a forward recurrence that runs alone take one batch tile per CTA where ``_seq_variant`` (which the backward
    pass needs) takes two?  Decided from the device's SM count and cluster co-residency up front, not by a failed launch."""
    if SEQ_VARIANT & 15 or _tiles_per_cta(B, H, device) != 2:
        return False
    return fwd_tiles_per_cta(B, H, _sms(device), lambda c: _coresident_ctas(device, c)) == 1


def _fwd_variant(B: int, H: int, device) -> int:
    """Variant of a forward recurrence with nothing co-resident beside it (``_fwd_full_width``)."""
    return SEQ_VARIANT if _fwd_full_width(B, H, device) else _seq_variant(B, H, device)


def bwd_tiles_per_cta(B: int, H: int, sms: int, coresident: int) -> Optional[int]:
    """Batch tiles per CTA of a backward recurrence that has the GPU to itself, on a device with ``sms`` SMs, ``coresident`` of
    which hold backward CTAs in clusters of 4 (``_coresident_ctas``).  ``tiles_per_cta`` needs those clusters for the DSMEM
    reduce-scatter of the K-split, and an H100 co-schedules only 120 such CTAs: at B = 256, H = 1024 that means two tiles on
    64 CTAs.  With the reduce-scatter through L2 instead (csrc/lstm_seq_wgmma.cu, kXchgL2) the kernel needs no cluster, so its
    128 one-tile CTAs fit the 132 SMs.  1 where ``tiles_m * H / 16`` cluster-free one-tile CTAs fit ``sms`` (resident weights,
    H <= 1024), else what ``tiles_per_cta`` returns."""
    tiles = tiles_per_cta(B, H, coresident)
    if tiles != 2:
        return tiles
    return 1 if (B + 127) // 128 * (H // 16) <= sms else 2


def _bwd_full_width(B: int, H: int, device) -> bool:
    """Does a backward recurrence that runs alone take one batch tile per CTA with the L2 exchange where ``_seq_variant``
    takes two?  Decided from the device's SM count and cluster co-residency up front, not by a failed launch."""
    if SEQ_VARIANT & 15 or _tiles_per_cta(B, H, device) != 2:
        return False
    return bwd_tiles_per_cta(B, H, _sms(device), _coresident_ctas(device, _bwd_cluster(H))) == 1


def _xchg_buffer(B: int, H: int, device) -> torch.Tensor:
    """Exchange buffer of the one-tile backward kernel that reduce-scatters through L2: two step parities x H / 16 CTAs per
    batch tile x a [128 x 64] bf16 partial (4 MiB at B = 256, H = 1024)."""
    return torch.empty(2 * ((B + 127) // 128) * (H // 16) * 128 * 64, dtype=torch.bfloat16, device=device)


def fast_path_supported(B: int, H: int, dtype: torch.dtype, device) -> bool:
    if FORCE_GENERIC or dtype != torch.bfloat16 or H % 64 != 0:
        return False
    return (B + 127) // 128 <= 16 and _tiles_per_cta(B, H, device) is not None


def _batch_chunk(B: int, H: int, dtype: torch.dtype, device) -> Optional[int]:
    """Largest multiple of 128 rows whose CTAs fit the device, when the whole batch does not (else None)."""
    if FORCE_GENERIC or dtype != torch.bfloat16 or H % 64 != 0 or fast_path_supported(B, H, dtype, device):
        return None
    if H > 2048:
        return None
    tiles = _coresident_ctas(device, _bwd_cluster(H)) // (H // 16) * (2 if H <= 1024 else 1)
    if tiles < 1:
        return None
    chunk = min(tiles, 16) * 128
    return chunk if chunk < B else None


def _mm_f32(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """a [M,K] @ b [K,N] -> fp32 (own kernels: wgmma when bf16 and aligned, CUDA-core GEMM otherwise)."""
    return G.matmul(a, b.t(), out_dtype=torch.float32)


def _transposed(w: torch.Tensor) -> torch.Tensor:
    """``w [R,C]`` -> contiguous ``[C,R]`` (tile-transpose kernel for 16-bit CUDA tensors)."""
    if w.is_cuda and w.dim() == 2 and w.element_size() == 2 and w.is_contiguous():
        STATS["kernels"] += 1
        return ext().transpose2d(w)
    return w.t().contiguous()


def _gemm_tn(a: torch.Tensor, w: torch.Tensor) -> torch.Tensor:
    """a [M,K] @ w[N,K]^T -> [M,N] in a.dtype."""
    STATS["tc_gemm"] += 1
    STATS["kernels"] += 1
    return G.matmul(a, w, out_dtype=a.dtype)


def _check_lengths_arg(lengths: Optional[torch.Tensor], B: int, device) -> None:
    """Shape / dtype / device of per-row lengths; the values are not read (that would synchronise with the device)."""
    if lengths is not None and (lengths.dtype != torch.int32 or lengths.shape != (B,) or lengths.device != device
                                or not lengths.is_contiguous()):
        raise ValueError(f"lengths must be a contiguous int32 [{B}] tensor on {device}, got {lengths.dtype} "
                         f"{tuple(lengths.shape)} on {lengths.device}")


def _weight_image(w_h_c: torch.Tensor, spec) -> torch.Tensor:
    """Weight drop: ``W_h' = W_h * M * s`` of a weight-drop spec (``reference.weight_drop``), computed from the compute-dtype copy
    (the bf16 shadow, or fp32) by the dropout kernel over its ``[1, 4H, H]`` view; ``w_h_c`` itself for None / P = 0."""
    d = _drop_args(spec, w_h_c.device)
    if not d:
        return w_h_c
    STATS["weight_drop"] += 1
    STATS["kernels"] += 1
    return ext().dropout(w_h_c.unsqueeze(0), d["drop_step"], d["drop_desc"], 0)[0]


def _weight_drop_grad(src: torch.Tensor, dst: torch.Tensor, wdrop: dict, accumulate: bool) -> None:
    """``dst (+)= src * M * s``: the gradient of the masked matrix -> the gradient of ``W_h`` (csrc/lstm_pointwise.cu)."""
    STATS["weight_drop_grad"] += 1
    STATS["kernels"] += 1
    ext().weight_drop_grad(src, dst, wdrop["drop_step"], wdrop["drop_desc"], accumulate)


class _DropoutFn(torch.autograd.Function):
    """Standalone dropout (csrc/lstm_pointwise.cu ts_dropout), forward and backward with the same mask: the one-step path and
    the shapes the persistent kernels do not fuse it into.  ``x [..., B, H]``, leading dims = times t0, t0 + 1, ..."""
    @staticmethod
    def forward(ctx, x, spec, t0):
        ctx.spec, ctx.t0 = spec, t0
        STATS["kernels"] += 1
        d = _drop_args(spec, x.device)
        return ext().dropout(x.contiguous(), d["drop_step"], d["drop_desc"], t0)

    @staticmethod
    def backward(ctx, g):
        STATS["kernels"] += 1
        d = _drop_args(ctx.spec, g.device)
        return ext().dropout(g.contiguous(), d["drop_step"], d["drop_desc"], ctx.t0), None, None


def dropout(x: torch.Tensor, spec, t0: int = 0) -> torch.Tensor:
    """``x * mask * scale`` (``reference.dropout``) on our own kernel; ``spec`` None or P = 0: x itself, no launch."""
    if spec is None or spec.p == 0:
        return x
    return _DropoutFn.apply(x, spec, t0)


_ACT_SCRATCH = {}


def _activation_sums(out: Optional[torch.Tensor], h: torch.Tensor, lengths) -> torch.Tensor:
    """fp32 ``[2]`` = (sum out^2, sum (h_t - h_{t-1})^2) over the counted positions of the top layer's output (csrc/activation_reg.cu):
    ``h`` the raw output ``[T,B,H]`` in time order, ``out`` the dropped one the head reads (None: ``h`` itself)."""
    T, B, H = h.shape
    n = ext().act_reg_scratch(T, B, H, h.dtype == torch.bfloat16)
    key = (h.device.index, n)
    if key not in _ACT_SCRATCH:          # one buffer per size, never freed: a captured graph keeps its address
        _ACT_SCRATCH[key] = torch.zeros(n, dtype=torch.float64, device=h.device)   # (every launch leaves its ticket 0)
    STATS["act_reg_fwd"] += 1
    STATS["kernels"] += 1
    return ext().act_reg_fwd(out, h, lengths, _ACT_SCRATCH[key])


def _activation_grad(dh: Optional[torch.Tensor], out: Optional[torch.Tensor], h: torch.Tensor, lengths, g: torch.Tensor,
                     drop: dict) -> torch.Tensor:
    """The gradient into the top layer's raw output ``h``: the head's ``dh`` (w.r.t. ``out``, None: zero) and that of the two sums
    (``g = d loss / d sums``), with the output dropout's mask ``drop`` (``_drop_args``) applied, in one pass; the recurrence's
    backward then reads it unmasked."""
    STATS["act_reg_bwd"] += 1
    STATS["kernels"] += 1
    return ext().act_reg_bwd(dh, out, h, lengths, g.float().contiguous(), **drop)


class _LSTMSeqFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x_seq, h0, c0, w_x, w_h, bias, lengths=None, reverse=False, dropout=None, weight_drop=None, chunks=None,
                act_sums=False):
        E = ext()
        T, B, D = x_seq.shape
        H = w_h.shape[1]
        cd = x_seq.dtype
        x2d = x_seq.reshape(T * B, D).contiguous()
        w_x_c = lowp(w_x, cd)
        ctx.wdrop = _drop_args(weight_drop, x_seq.device)
        w_h_c = _weight_image(lowp(w_h, cd), weight_drop)             # every step reads the masked image (weight drop)
        bias_f = bias.detach().float().contiguous()
        gx = _gemm_tn(x2d, w_x_c).view(T, B, 4 * H)
        fast = fast_path_supported(B, H, cd, x_seq.device)
        c0f = c0.detach().float().contiguous()
        h0c = h0.detach().to(cd).contiguous()
        drop = _drop_args(dropout, x_seq.device)
        h_drop = None
        if fast:
            # the only recurrence on the GPU: the forward kernel's own co-residency decides its tile count (_fwd_full_width)
            full = _fwd_full_width(B, H, x_seq.device)
            outs = E.lstm_seq_fwd(gx, w_h_c, bias_f, h0c, c0f, _sync_ws(x_seq.device), _fwd_variant(B, H, x_seq.device),
                                  lengths=lengths, reverse=reverse, **drop)
            h_seq, c_seq, act = outs[:3]
            if drop:
                h_drop = outs[3]                                          # written next to h_seq by the recurrence kernel
            STATS["fast_fwd"] += 1
            STATS["kernels"] += 1
            if full:
                count("fwd_full_width")
        else:
            h_seq = torch.empty(T + 1, B, H, dtype=cd, device=x_seq.device)
            c_seq = torch.empty(T + 1, B, H, dtype=torch.float32, device=x_seq.device)
            act = torch.empty(T, B, 4 * H, dtype=cd, device=x_seq.device)
            s0 = T if reverse else 0                                      # state row of h0 / c0 (see lstm_layer_sequence)
            h_seq[s0].copy_(h0c)
            c_seq[s0].copy_(c0f)
            pre = torch.empty(B, 4 * H, dtype=cd, device=x_seq.device)
            for t in (range(T - 1, -1, -1) if reverse else range(T)):
                sp, sn = (t + 1, t) if reverse else (t, t + 1)            # state rows before / after step t
                pre.copy_(gx[t])
                G.matmul(h_seq[sp], w_h_c, out=pre, accumulate=True)      # pre = gx[t] + h_prev W_h^T
                h, c, a = E.lstm_pointwise_fwd(pre, bias_f, c_seq[sp], h_seq[sp], lengths, t)
                h_seq[sn].copy_(h)
                c_seq[sn].copy_(c)
                act[t].copy_(a)
            STATS["generic_fwd"] += 1
            STATS["kernels"] += T
            if drop:
                h_drop = E.dropout(h_seq[:T] if reverse else h_seq[1:], drop["drop_step"], drop["drop_desc"], 0)
                STATS["kernels"] += 1
        ctx.drop = drop
        h_out = h_seq[:T] if reverse else h_seq[1:]
        ctx.act_sums = act_sums
        ctx.save_for_backward(x2d, h_seq, c_seq, act, w_x_c, w_h_c, h_drop if act_sums else None)
        ctx.set_materialize_grads(False)       # an unused output must arrive as None, not as a zero-filled [T,B,H] tensor
        ctx.fast = fast
        ctx.lengths = lengths
        ctx.reverse = reverse
        ctx.chunks = chunks                    # a params.Countdown shared by the batch chunks of one layer, or None
        ctx.dims = (T, B, D, H)
        ctx.w_addrs = (w_x.data_ptr(), w_h.data_ptr(), bias.data_ptr())
        ctx.in_dtypes = (h0.dtype, c0.dtype)
        # h_T is its own output (not a slice of the first one taken by the caller): a consumer of the final state only - the
        # classifier on top of the stack - then sends back a [B,H] gradient instead of a zero-filled [T,B,H] one
        outs = (h_out if h_drop is None else h_drop), h_seq[0 if reverse else T], c_seq[0 if reverse else T]
        if act_sums:                           # AR / TAR: the sums over this op's rows and positions, one more output
            return outs + (_activation_sums(h_drop, h_out, lengths),)
        return outs

    @staticmethod
    def backward(ctx, dh_seq, dh_T, dc_T, d_sums=None):
        E = ext()
        x2d, h_seq, c_seq, act, w_x_c, w_h_c, h_drop = ctx.saved_tensors
        T, B, D, H = ctx.dims
        cd = act.dtype
        dev = act.device
        drop = ctx.drop if dh_seq is not None else {}          # (the mask only matters where a gradient arrives)
        if dh_seq is not None:
            dh_seq = dh_seq.to(cd).contiguous()
        if ctx.act_sums and d_sums is not None:
            # the sums' gradient joins the head's and the output dropout's mask is applied to both in one pass: the recurrence
            # below (and the generic path) then reads dh_seq unmasked
            dh_seq = _activation_grad(dh_seq, h_drop, h_seq[:T] if ctx.reverse else h_seq[1:], ctx.lengths, d_sums, ctx.drop)
            drop = {}
        if dh_seq is not None:
            if drop and not ctx.fast:
                dh_seq = E.dropout(dh_seq, drop["drop_step"], drop["drop_desc"], 0)
                STATS["kernels"] += 1
        elif not ctx.fast:
            dh_seq = torch.zeros(T, B, H, dtype=cd, device=dev)
        dcT = (dc_T.float().contiguous() if dc_T is not None else torch.zeros(B, H, dtype=torch.float32, device=dev))
        dhT = (dh_T.float().contiguous() if dh_T is not None else torch.zeros(B, H, dtype=torch.float32, device=dev))
        if ctx.fast:
            w_hT = _transposed(w_h_c)
            # the only recurrence on the GPU: one tile per CTA with the L2 exchange where that fits (_bwd_full_width)
            full = _bwd_full_width(B, H, dev)
            big_launch_begin()
            dpre, dh0, dc0 = E.lstm_seq_bwd(dh_seq, w_hT, act, c_seq, dhT, dcT, _sync_ws(dev),
                                            SEQ_VARIANT if full else _seq_variant(B, H, dev), lengths=ctx.lengths,
                                            reverse=ctx.reverse, xchg=_xchg_buffer(B, H, dev) if full else None, **drop)
            STATS["fast_bwd"] += 1
            STATS["kernels"] += 1
            if full:
                count("bwd_full_width")
            after_big_launch()                   # finished gradient buckets of the layers above: sync them under this recurrence
        else:
            dpre = torch.empty_like(act)
            dh_rec: Optional[torch.Tensor] = dhT if dh_T is not None else None
            dc = dcT
            for t in (range(T) if ctx.reverse else range(T - 1, -1, -1)):
                sp, sn = (t + 1, t) if ctx.reverse else (t, t + 1)
                if ctx.lengths is None:
                    dp, dc = E.lstm_pointwise_bwd(dh_seq[t], dh_rec, dc, act[t], c_seq[sp], c_seq[sn])
                    dh_rec = _mm_f32(dp, w_h_c)
                else:                            # padded rows hand their dh on directly (dh_pass), the others through W_h
                    dp, dc, dh_pass = E.lstm_pointwise_bwd(dh_seq[t], dh_rec, dc, act[t], c_seq[sp], c_seq[sn], ctx.lengths, t)
                    G.matmul(dp, w_h_c.t(), out=dh_pass, accumulate=True)
                    dh_rec = dh_pass
                dpre[t].copy_(dp)
            dh0, dc0 = dh_rec, dc
            STATS["generic_bwd"] += 1
            STATS["kernels"] += T
        dg2d = dpre.view(T * B, 4 * H)
        dg_t = dg2d.t()
        a, rel = ctx.w_addrs, (release if ctx.chunks is None else ctx.chunks.releaser())
        dw_x = _accumulate_grad(a[0], dg_t, x2d)
        if not ctx.needs_input_grad[0]:
            rel(a[0])                                              # (else W_x is released after the dX GEMM reads it)
        h_prev = h_seq[1:] if ctx.reverse else h_seq[:T]          # the h each step's dG pairs with
        dw_h = _accumulate_grad(a[1], dg_t, h_prev.reshape(T * B, H), wdrop=ctx.wdrop)
        db = _bias_grad(a[2], dg2d)
        rel(a[1], a[2])
        dx = None
        if ctx.needs_input_grad[0]:
            dx = G.matmul(dg2d, w_x_c.t(), out_dtype=cd).view(T, B, D)        # dG · W_x: W_x read in place as an MN-major operand
            STATS["kernels"] += 1
            rel(a[0])
        h0_dt, c0_dt = ctx.in_dtypes
        return dx, dh0.to(h0_dt), dc0.to(c0_dt), dw_x, dw_h, db, None, None, None, None, None, None


def lstm_layer_sequence(x_seq, h0, c0, w_x, w_h, bias, lengths=None, reverse=False, dropout=None, weight_drop=None,
                        activation_sums=False):
    """``x_seq [T,B,D]`` (bf16 or fp32) -> ``(h_seq [T,B,H], h_T, c_T)``.  ``lengths``: optional int32 ``[B]`` on the batch's
    device, right padding (``ops/reference.py``); the persistent kernels then run their masked instantiations.  ``reverse``:
    the reverse-time direction (time T-1 down to 0; ``h_T`` / ``c_T`` are then the state after time 0).  ``dropout``: a
    ``reference.DropoutSpec``; the first output is then the dropped sequence (the persistent kernels store it next to h_seq
    and mask the incoming gradient as they load it; other shapes run the standalone dropout kernel).  ``weight_drop``: a weight-drop
    ``reference.DropoutSpec``: the kernels read the masked image ``W_h * M * s`` in place of ``W_h`` and the weight gradient is
    masked on its way into the sink (one mask for every batch chunk).  ``activation_sums``: one more output, fp32 ``[2]`` =
    (sum out^2, sum (h_t - h_{t-1})^2) over the counted positions, ``out`` the first output and ``h`` the undropped one
    (``reference.activation_sums``; csrc/activation_reg.cu); its gradient is combined with the first output's by one more kernel
    ahead of the backward recurrence."""
    if (not x_seq.is_contiguous() and not x_seq.requires_grad and x_seq.transpose(0, 1).is_contiguous()
            and (x_seq.shape[2] * x_seq.element_size()) % 16 == 0):
        x_seq = ext().transpose01(x_seq.transpose(0, 1))     # batch-major feed -> time-major, a row permutation at copy speed
        STATS["kernels"] += 1
    T, B, _ = x_seq.shape
    H = w_h.shape[1]
    _check_lengths_arg(lengths, B, x_seq.device)
    chunk = _batch_chunk(B, H, x_seq.dtype, x_seq.device)
    if chunk is not None:
        # more batch tiles than the persistent kernels can keep co-resident: the sequences are independent, so run the fast
        # path per batch chunk (weight-gradient contributions accumulate across chunks) instead of the per-step generic path;
        # the chunk whose backward runs last releases the parameters
        chunks = Countdown((B + chunk - 1) // chunk)
        outs = [_LSTMSeqFn.apply(x_seq[:, b0:b0 + chunk].contiguous(), h0[b0:b0 + chunk], c0[b0:b0 + chunk], w_x, w_h, bias,
                                 None if lengths is None else lengths[b0:b0 + chunk], reverse,
                                 None if dropout is None else dropout.at_rows(b0), weight_drop, chunks, activation_sums)
                for b0 in range(0, B, chunk)]
        count("batch_chunks", len(outs))
        cat = (torch.cat([o[0] for o in outs], dim=1), torch.cat([o[1] for o in outs], dim=0),
               torch.cat([o[2] for o in outs], dim=0))
        if activation_sums:                  # unnormalised: the chunks' parts add up, in chunk order
            sums = outs[0][3]
            for o in outs[1:]:
                sums = sums + o[3]
            cat = cat + (sums,)
        return cat
    return _LSTMSeqFn.apply(x_seq.contiguous(), h0, c0, w_x, w_h, bias, lengths, reverse, dropout, weight_drop, None, activation_sums)


# =====================================================================================================================
# Layer wavefront: two stacked layers' recurrences run CO-RESIDENT (64 + 64 CTAs, two batch tiles per CTA over the same resident
# weight slice), chained through a dataflow-gated wgmma GEMM on the ~20 SMs they leave idle:
#     forward :  L_a step t  ->  gx_b[t] = h_a[t] W_xb^T (gated GEMM)  ->  L_b step t
#     backward:  L_b step t  ->  dh_a[t] = dG_b[t] W_xb  (gated GEMM)  ->  L_a step t
# The reference stacks layers strictly one after the other (original src/models/recurrent/rnn.py:38-42); here layer l+1
# trails layer l by a couple of time steps and the next layer's input projection leaves the critical path altogether.
# Where both recurrences do not fit side by side (an H100 at H = 1024: 64 + 64 + 8 > 132 SMs), the pair is PIPELINED instead:
# the recurrences run one after the other and the GEMMs move onto the SMs the running recurrence leaves idle (L_a's own input
# projection gx_a too: L_a waits for it block by block)
#     forward :  L_a  || gx_a, gx_b (gated)              ->  L_b
#     backward:  L_b  || dx_b (gated)                    ->  L_a  || dW_xb, dW_hb, db_b
#            or  L_b alone, one tile per CTA             ->  L_a  || dx_b, dW_xb, dW_hb, db_b   (where that fits: _bwd_full_width)
# =====================================================================================================================
FOLDED_FEED = os.environ.get("LSTM_TS_FOLDED_FEED", "1") != "0"   # batch-major input read in place by the first layer's GEMMs
WAVEFRONT = os.environ.get("LSTM_TS_WAVEFRONT", "1") == "1"
_WS_PAIR = {}


_WARM = set()


def _warm_wavefront_kernels(device):
    """CUDA loads kernels lazily, and loading one may wait for every running kernel to finish.  The wavefront's kernels WAIT
    FOR EACH OTHER on the device, so a kernel that is loaded for the first time while its producers are already spinning would
    deadlock (until the bounded spins time out).  Load the gated GEMM instantiations and the pipelined pair's ungated
    ``done``-publishing x-projection (the same instantiation, contiguous or folded input) once, before the first concurrent use."""
    if device.index in _WARM:
        return
    a = torch.zeros(256, 64, dtype=torch.bfloat16, device=device)
    w = torch.zeros(256, 64, dtype=torch.bfloat16, device=device)
    wt = torch.zeros(64, 256, dtype=torch.bfloat16, device=device)
    ext().gemm2(a, w, ctas=1, bn=256)
    ext().gemm2(a, wt, b_mn=True, ctas=1, bn=256)
    torch.cuda.synchronize(device)
    _WARM.add(device.index)


def _pair_ws(device, tag: str, n_done: int):
    """[sync ws of the head kernel | sync ws of the tail kernel | completion counters of the gated GEMM] in one allocation."""
    key = (device.index, tag)
    ent = _WS_PAIR.get(key)
    if ent is None or ent.numel() < 2 * SYNC_WORDS + n_done:
        ent = torch.zeros(2 * SYNC_WORDS + max(n_done, 1), dtype=torch.int32, device=device)
        _WS_PAIR[key] = ent
    return ent[:SYNC_WORDS], ent[SYNC_WORDS:2 * SYNC_WORDS], ent[2 * SYNC_WORDS:2 * SYNC_WORDS + n_done]


def pair_schedule(T: int, B: int, D: int, h_a: int, h_b: int, sms: int, coresident: int) -> Optional[str]:
    """How two stacked layers run as one op on a device with ``sms`` SMs, ``coresident`` of which hold backward-kernel CTAs in
    clusters of 4 (``_coresident_ctas``).  Every recurrence runs two batch tiles per CTA, H/16 CTAs (except the pipelined
    L_b forward, which runs alone: one tile per CTA where that fits, ``_fwd_full_width``).  Both schedules need
    B = 256 (one GEMM tile row per time step), resident weights (H <= 1024) and 256-aligned widths.
      "wavefront": both recurrences co-resident, the gated GEMM on the SMs they leave free (H_a/16 + H_b/16 + 8 SMs).
      "pipelined": the recurrences run one after the other, GEMMs next to them (forward: L_a with its own gx_a and with gx_b;
                   backward: L_b with dx_b, then L_a with dW_xb, dW_hb and db_b; where L_b's backward fits one tile per
                   CTA, L_b alone, then L_a with dx_b too).  Needs max(H)/16 + 8 SMs.
      None: two separate layers."""
    if B != 256 or T < 2 or D % 8 != 0 or any(h % 256 != 0 or h > 1024 for h in (h_a, h_b)):
        return None
    both = h_a // 16 + h_b // 16 + 8
    if both <= coresident + 16 and both <= sms:
        return "wavefront"
    if max(h_a, h_b) // 16 <= coresident and max(h_a, h_b) // 16 + 8 <= sms:
        return "pipelined"
    return None


def pipelined_fwd_split(sms: int, d: int, h_a: int, h_b: int) -> tuple:
    """SMs of the pipelined pair's forward side GEMMs -> (gx_a CTAs, gx_b CTAs).  Both run next to L_a on the ``sms - h_a / 16``
    SMs its CTAs leave free, one single-CTA 128 x 256 tile per SM, and both must keep pace with it: L_a waits for gx_a(t) at its
    step t, and L_b (after L_a) for the last gx_b rows.  Their work per step is 2·B·4h_a·d and 2·B·4h_b·h_a FLOP, so the free
    SMs are split in the ratio d : h_b: 34 + 34 at the headline 2 x 1024 on a 132-SM H100, where a step of L_a takes about
    20 us and 34 SMs compute a step's 2.1 GFLOP of either GEMM in about 12 us (5.2 TFLOP/s per SM with single-CTA tiles,
    bench/side_gemms.py on an H100 80GB HBM3 at 700 W)."""
    free = max(2, sms - h_a // 16)
    n_a = min(free - 1, max(1, round(free * d / (d + h_b)))) if d > 0 else 0     # d = 0: gx_a computed before L_a
    return n_a, free - n_a


def pipelined_bwd_split(sms: int, h_a: int, h_b: int) -> tuple:
    """SMs of the pipelined pair's backward side GEMMs when L_b's backward runs alone at one tile per CTA -> (dx_b CTAs, CTAs of
    each of dW_xb and dW_hb).  All three run next to L_a's backward on the ``sms - h_a / 16 - _COLSUM_SMS`` SMs its CTAs and
    the bias column sums leave free, one single-CTA 128 x 256 tile per SM.  Their work is 2·T·B·4h_b·h_a (dx_b),
    2·T·B·4h_b·h_a (dW_xb) and 2·T·B·4h_b·h_b (dW_hb) FLOP.  L_a waits for dx_b(t) at its step t, while dW_xb and dW_hb only
    have to end with it, so dx_b gets a third more than its share of the work: the free SMs are split in the ratio
    4h_a : 3h_a : 3h_b, 26 + 19 + 19 at the headline 2 x 1024 on a 132-SM H100.  There a step of L_a's backward takes about
    20 us, and 26 SMs compute a step's 2.1 GFLOP of dx_b (eight 128 x 256 tiles) in about 16 us at 5.2 TFLOP/s per SM
    (bench/side_gemms.py).  On an H100 80GB HBM3 at 700 W the headline step took 9.84 ms with 26 dx_b CTAs, against 9.87-9.88
    with 21 (the plain work ratio), 9.87-9.88 with 30 and 9.92-9.96 with 34, two runs each."""
    free = max(3, sms - h_a // 16 - _COLSUM_SMS)
    n_dx = min(free - 2, max(1, round(free * 4 * h_a / (7 * h_a + 3 * h_b))))
    return n_dx, (free - n_dx) // 2


def _pair_schedule_of(x_seq: torch.Tensor, h_a: int, h_b: int) -> Optional[str]:
    """``pair_schedule`` for an input on its device; None off the bf16 fast path, with ``LSTM_TS_WAVEFRONT=0`` (serial layers,
    for tools that serialise kernels) or with a tile-count override in ``LSTM_TS_SEQ_VARIANT``."""
    if not (WAVEFRONT and x_seq.is_cuda and x_seq.dtype == torch.bfloat16 and not FORCE_GENERIC and x_seq.dim() == 3):
        return None
    if (SEQ_VARIANT & 15) > 2:
        return None
    T, B, D = x_seq.shape
    return pair_schedule(T, B, D, h_a, h_b, _sms(x_seq.device), _coresident_ctas(x_seq.device))


def wavefront_supported(x_seq: torch.Tensor, h_a: int, h_b: int) -> bool:
    """Can two stacked layers run as one pair op (``lstm_pair_sequence``, either schedule of ``pair_schedule``)?"""
    return _pair_schedule_of(x_seq, h_a, h_b) is not None


WAVE_SYNC_MODE = int(os.environ.get("LSTM_TS_WAVE_SYNC", "1"))      # 1: one arrival counter per batch tile (measured 2.5 % faster with two
                                                                    # tiles per CTA), 0: one per operand k-block


def _wave_variant() -> int:
    return (SEQ_VARIANT & ~(15 | (3 << 16))) | 2 | ((WAVE_SYNC_MODE & 1) << 16)


_COLSUM_SMS = 4            # pipelined backward: SMs kept for layer b's bias column sums (4 CTAs of 256 threads each)


def _pair_variant(schedule: str) -> int:
    """Variant of the four recurrences of a layer pair.  Pipelined: per-k-block counters (sync mode 0), the layout a single
    layer's recurrence uses; one counter per batch tile only pays off when two recurrences are co-resident."""
    var = _wave_variant()
    return var & ~(3 << 16) if schedule == "pipelined" else var


def _gate_off(var: int) -> int:
    return 0 if (var >> 16) & 3 == 1 else 512


def _gate_cfg(var: int, tiles_m: int, nkb: int, per_kb_step: int, ctas_per_tile: int, base_steps: int, step_sign: int, rows: int, bwd: bool):
    """Gate of the wavefront GEMM on the producer layer's arrival counters: [count, stride, base, per_step, rows_per_step, use_last,
    reverse_m].  A time step's natural-layout rows are complete with the producer's (step + 1)-th signal, hence base = 2 steps
    (forward: target(t) = per_step * (t + 2)) or T + 1 (backward: target(t) = per_step * (T + 1 - t))."""
    if (var >> 16) & 3 == 1:                # one counter per batch tile, every CTA of the tile arrives once per step
        per = ctas_per_tile
        return [tiles_m, 1, per * base_steps, per * step_sign, rows, 0 if bwd else 1, 1 if bwd else 0]
    per = per_kb_step                       # one counter per operand k-block (fwd: 4 producer CTAs, bwd: 1)
    return [tiles_m * nkb, 32, per * base_steps, per * step_sign, rows, 0 if bwd else 1, 1 if bwd else 0]


class _LSTMPairFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x_seq, h0a, c0a, w_xa, w_ha, b_a, h0b, c0b, w_xb, w_hb, b_b, lengths=None, schedule="wavefront", drop_a=None,
                drop_b=None, wdrop_a=None, wdrop_b=None, act_sums=False):
        E = ext()
        pipelined = schedule == "pipelined"
        dev = x_seq.device
        T, B, D = x_seq.shape
        Ha, Hb = w_ha.shape[1], w_hb.shape[1]
        cd = x_seq.dtype
        # a batch-major input ([B,T,D] storage behind a transposed view) is read in place by the x-projection and by the
        # weight-gradient GEMM of the first layer (folded tensor map, csrc/gemm2_wgmma.cu): no transpose pass
        x_bm = x_seq.transpose(0, 1) if not x_seq.is_contiguous() else None
        x2d = x_seq.reshape(T * B, D) if x_bm is None else x_bm
        wxa, wha, wxb, whb = lowp(w_xa, cd), lowp(w_ha, cd), lowp(w_xb, cd), lowp(w_hb, cd)
        wha, whb = _weight_image(wha, wdrop_a), _weight_image(whb, wdrop_b)          # weight drop: the masked images
        ctx.wdrop = (_drop_args(wdrop_a, dev), _drop_args(wdrop_b, dev))
        ba_f, bb_f = b_a.detach().float().contiguous(), b_b.detach().float().contiguous()
        h0a_c, h0b_c = h0a.detach().to(cd).contiguous(), h0b.detach().to(cd).contiguous()
        c0a_f, c0b_f = c0a.detach().float().contiguous(), c0b.detach().float().contiguous()
        _warm_wavefront_kernels(dev)
        opt = dict(dtype=cd, device=dev)
        side_a = pipelined and D >= 64                                   # gx_a next to L_a (the tensor-core GEMM needs K >= 64)
        if side_a:
            gx_a = torch.empty(T, B, 4 * Ha, **opt)                      # written next to L_a (see below)
        elif x_bm is None:
            gx_a = _gemm_tn(x2d, wxa).view(T, B, 4 * Ha)
        else:
            STATS["tc_gemm"] += 1; STATS["kernels"] += 1; count("folded_feed")
            gx_a = G.matmul(None, wxa, out_dtype=cd, a_folded=x_bm).view(T, B, 4 * Ha)
        h_seq_a = torch.empty(T + 1, B, Ha, **opt); c_seq_a = torch.empty(T + 1, B, Ha, dtype=torch.float32, device=dev)
        act_a = torch.empty(T, B, 4 * Ha, **opt); til_a = torch.empty((T + 1) * 2 * 128 * Ha, **opt)
        h_seq_b = torch.empty(T + 1, B, Hb, **opt); c_seq_b = torch.empty(T + 1, B, Hb, dtype=torch.float32, device=dev)
        act_b = torch.empty(T, B, 4 * Hb, **opt); til_b = torch.empty((T + 1) * 2 * 128 * Hb, **opt)
        gx_b = torch.empty(T, B, 4 * Hb, **opt)
        # dropout: L_a stores h_drop_a next to h_seq_a (the gated gx_b GEMM reads it), L_b stores h_drop_b (the pair's output)
        dra, drb = _drop_args(drop_a, dev), _drop_args(drop_b, dev)
        h_drop_a = torch.empty(T, B, Ha, **opt) if dra else None
        h_drop_b = torch.empty(T, B, Hb, **opt) if drb else None
        hin_b = h_seq_a[1:] if h_drop_a is None else h_drop_a            # layer b's input sequence
        tn, tn_a = 4 * Hb // 256, 4 * Ha // 256
        ws_a, ws_b, done = _pair_ws(dev, "fwd", T * 2 * (tn + (tn_a if side_a else 0)))
        done.zero_()                                                     # (the prologue kernels zero ws_a / ws_b)
        done, done_a = done[:T * 2 * tn], done[T * 2 * tn:]
        var = _pair_variant(schedule)                                    # two batch tiles per CTA: 64 CTAs per layer at H = 1024
        # ONE stream, a programmatic-dependent-launch chain: L_a -> L_b (starts once every CTA of L_a is resident) -> gated GEMM
        # (starts once every CTA of L_b is resident, on the SMs that are left).  The order in which the three grids take their
        # SMs is thereby fixed (a kernel that is still queueing could otherwise starve the chain head of co-resident SMs).
        # Everything the later kernels need up front (prologues, zeroed counters) is enqueued before the chain head.
        # Pipelined: L_a -> gx_a GEMM -> gated gx_b GEMM (programmatic dependents, on the SMs L_a leaves free) -> L_b, an ordinary
        # launch that starts once all three are complete (each GEMM waits for its predecessor before it exits).  L_a waits for
        # gx_a's 128 x 256 blocks as the wavefront's L_b does for gx_b's; the gx_a GEMM is ungated, so nothing it waits for
        # depends on L_a, and its capped grid walks the M tiles (time steps) in order.
        E.lstm_seq_prologue(h0a_c, c0a_f, h_seq_a, c_seq_a, til_a, ws_a)
        E.lstm_seq_prologue(h0b_c, c0b_f, h_seq_b, c_seq_b, til_b, ws_b)
        E.lstm_seq_fwd_into(gx_a, wha, ba_f, h0a_c, c0a_f, h_seq_a, c_seq_a, act_a, til_a, ws_a, var, done_a if side_a else None,
                            tn_a if side_a else 0, True, 0, 1, lengths, h_drop=h_drop_a, **dra)
        if pipelined:
            ctas_a, free_ctas = pipelined_fwd_split(_sms(dev), D if side_a else 0, Ha, Hb)
        if side_a:
            a_op = dict(A=x2d, a_fold=0) if x_bm is None else dict(A=x_bm.reshape(B, T * D), a_fold=B, fold_cols=D)
            E.gemm2(B=wxa, out=gx_a.view(T * B, 4 * Ha), ctas=1, bn=256, max_ctas=ctas_a, done=done_a, pdl=True, **a_op)
            STATS["tc_gemm"] += 1; STATS["kernels"] += 1; count("pipelined_side_gemms")
            if x_bm is not None:
                count("folded_feed")
        if not pipelined:
            E.lstm_seq_fwd_into(gx_b, whb, bb_f, h0b_c, c0b_f, h_seq_b, c_seq_b, act_b, til_b, ws_b, var, done, tn, False, 0, 3, lengths,
                                h_drop=h_drop_b, **drb)
            # single-CTA tiles: the recurrences' CTAs are spread one per TPC, the SMs they leave free rarely form CTA pairs
            free_ctas = max(1, _sms(dev) - Ha // 16 - Hb // 16)
        E.gemm2(hin_b.view(T * B, Ha), wxb, out=gx_b.view(T * B, 4 * Hb), ctas=1, bn=256, max_ctas=free_ctas,
                gate=ws_a[_gate_off(var):], gate_cfg=_gate_cfg(var, 2, Ha // 64, 4, 4 * Ha // 64, 2, 1, B, False), done=done,
                gate_err=ws_a[SYNC_WORDS - 1:], pdl=True)
        if pipelined:
            # L_b is an ordinary launch after gx_a / gx_b are complete: nothing runs beside it, so it takes one batch tile per CTA
            # where that fits (128 CTAs at B = 256, H_b = 1024; _fwd_full_width).  Its counters stay per k-block (sync mode 0 of
            # the pipelined variant), and til_b is sized per batch tile, whatever the tiles per CTA.  No warm-up is needed for
            # this instantiation (_warm_wavefront_kernels): its first launch comes after its producers have finished.
            var_b = var
            if _fwd_full_width(B, Hb, dev):
                var_b = var & ~15
                count("fwd_full_width")
            E.lstm_seq_fwd_into(gx_b, whb, bb_f, h0b_c, c0b_f, h_seq_b, c_seq_b, act_b, til_b, ws_b, var_b, None, 0, False, 0, 1, lengths,
                                h_drop=h_drop_b, **drb)
        STATS["fast_fwd"] += 2
        STATS["kernels"] += 3
        count(schedule + "_fwd")
        ctx.save_for_backward(x2d, h_seq_a, c_seq_a, act_a, h_seq_b, c_seq_b, act_b, wxa, wha, wxb, whb, hin_b,
                              h_drop_b if act_sums else None)
        ctx.set_materialize_grads(False)
        ctx.act_sums = act_sums
        ctx.drop = (dra, drb)
        ctx.dims = (T, B, D, Ha, Hb)
        ctx.lengths = lengths
        ctx.pipelined = pipelined
        ctx.x_folded = x_bm is not None
        ctx.addrs = (w_xa.data_ptr(), w_ha.data_ptr(), b_a.data_ptr(), w_xb.data_ptr(), w_hb.data_ptr(), b_b.data_ptr())
        ctx.in_dtypes = (h0a.dtype, c0a.dtype, h0b.dtype, c0b.dtype)
        outs = (h_seq_b[1:] if h_drop_b is None else h_drop_b), h_seq_a[T], c_seq_a[T], h_seq_b[T], c_seq_b[T]
        if act_sums:                          # AR / TAR of layer b, the top layer (an ordinary launch: L_b has finished)
            return outs + (_activation_sums(h_drop_b, h_seq_b[1:], lengths),)
        return outs

    @staticmethod
    def backward(ctx, dh_seq_b, dhT_a, dcT_a, dhT_b, dcT_b, d_sums=None):
        E = ext()
        x2d, h_seq_a, c_seq_a, act_a, h_seq_b, c_seq_b, act_b, wxa, wha, wxb, whb, hin_b, h_drop_b = ctx.saved_tensors
        dra, drb = ctx.drop
        wda, wdb = ctx.wdrop
        if dh_seq_b is None:
            drb = {}
        T, B, D, Ha, Hb = ctx.dims
        cd, dev = act_a.dtype, act_a.device
        if dh_seq_b is not None:
            dh_seq_b = dh_seq_b.to(cd).contiguous()
        if ctx.act_sums and d_sums is not None:
            # the sums' gradient joins the head's, masked by layer b's output dropout in the same pass: L_b reads it unmasked
            dh_seq_b = _activation_grad(dh_seq_b, h_drop_b, h_seq_b[1:], ctx.lengths, d_sums, ctx.drop[1])
            drb = {}
        f32 = dict(dtype=torch.float32, device=dev)
        z = lambda g, H: g.float().contiguous().clone() if g is not None else torch.zeros(B, H, **f32)
        dh0a, dc0a, dh0b, dc0b = z(dhT_a, Ha), z(dcT_a, Ha), z(dhT_b, Hb), z(dcT_b, Hb)
        whT_a, whT_b = _transposed(wha), _transposed(whb)
        dpre_a = torch.empty_like(act_a); dpre_b = torch.empty_like(act_b)
        til_a = torch.empty(T * 2 * 128 * 4 * Ha, dtype=cd, device=dev); til_b = torch.empty(T * 2 * 128 * 4 * Hb, dtype=cd, device=dev)
        dx_b = torch.empty(T, B, Ha, dtype=cd, device=dev)                # = the gradient into every h_a[t]
        tn = Ha // 256
        ws_b, ws_a, done = _pair_ws(dev, "bwd", T * tn * 2)               # head of the backward chain is layer b
        ws_a[:SYNC_WORDS - 1].zero_(); ws_b[:SYNC_WORDS - 1].zero_(); done.zero_()
        var = _pair_variant("pipelined" if ctx.pipelined else "wavefront")
        # programmatic-dependent-launch chain on one stream (see forward): L_b -> L_a -> gated dX GEMM.  Pipelined: L_b -> gated
        # dX GEMM -> L_a (ordinary launch: dx_b is complete when it starts)
        pipelined = ctx.pipelined
        # pipelined, where L_b's backward fits one tile per CTA with the L2 exchange (_bwd_full_width): it runs alone on 128 SMs,
        # and dx_b moves next to L_a's backward, which waits for it block by block (as L_a's forward does for gx_a)
        full_b = pipelined and _bwd_full_width(B, Hb, dev)
        # dropout: each recurrence masks the gradient into its output sequence as it loads it (dx_b stays the raw dL/dh_drop_a)
        if full_b:
            # L_b: an ordinary launch.  L_a: the chain head, gated on dx_b's 128 x 256 blocks.  dx_b: its programmatic dependent,
            # ungated (L_b is complete) on its capped grid, walking the M tiles (time steps) from the last, the order in which L_a
            # consumes them.  dW_xb, dW_hb and db_b follow as programmatic dependents (below).
            n_dx, side = pipelined_bwd_split(_sms(dev), Ha, Hb)
            E.lstm_seq_bwd_into(dh_seq_b, whT_b, act_b, c_seq_b, dpre_b, dh0b, dc0b, til_b, ws_b, var & ~15, None, 0, False, 0, 1,
                                ctx.lengths, xchg=_xchg_buffer(B, Hb, dev), **drb)
            E.lstm_seq_bwd_into(dx_b, whT_a, act_a, c_seq_a, dpre_a, dh0a, dc0a, til_a, ws_a, var, done, tn, False, 0, 1, ctx.lengths,
                                **dra)
            E.gemm2(dpre_b.view(T * B, 4 * Hb), wxb, out=dx_b.view(T * B, Ha), b_mn=True, ctas=1, bn=256, max_ctas=n_dx, done=done,
                    pdl=True, reverse_m=True)
            count("bwd_full_width")
        else:
            E.lstm_seq_bwd_into(dh_seq_b, whT_b, act_b, c_seq_b, dpre_b, dh0b, dc0b, til_b, ws_b, var, None, 0, True, 0, 1, ctx.lengths,
                                **drb)
            if not pipelined:
                E.lstm_seq_bwd_into(dx_b, whT_a, act_a, c_seq_a, dpre_a, dh0a, dc0a, til_a, ws_a, var, done, tn, False, 0, 3,
                                    ctx.lengths, **dra)
            free_ctas = max(1, _sms(dev) - Hb // 16 - (0 if pipelined else Ha // 16))
            E.gemm2(dpre_b.view(T * B, 4 * Hb), wxb, out=dx_b.view(T * B, Ha), b_mn=True, ctas=1, bn=256, max_ctas=free_ctas,
                    gate=ws_b[_gate_off(var):], gate_cfg=_gate_cfg(var, 2, 4 * Hb // 64, 1, 4 * Hb // 64, T + 1, -1, B, True), done=done,
                    gate_err=ws_b[SYNC_WORDS - 1:], pdl=True)
            if pipelined:
                E.lstm_seq_bwd_into(dx_b, whT_a, act_a, c_seq_a, dpre_a, dh0a, dc0a, til_a, ws_a, var, None, 0, False, 0, 1, ctx.lengths,
                                    **dra)
            side = max(1, (_sms(dev) - Ha // 16 - _COLSUM_SMS) // 2)
        STATS["fast_bwd"] += 2
        STATS["kernels"] += 5
        a = ctx.addrs
        dg_b = dpre_b.view(T * B, 4 * Hb)
        if pipelined:
            # layer b's weight and bias gradients read nothing L_a writes: programmatic dependents of L_a, next to it on the SMs it
            # leaves free.  dW_xb and dW_hb split those SMs between them: a dependent that has finished its tiles stays resident
            # until L_a ends (it waits for its predecessor before exiting), so a second GEMM behind it would get no SMs.  A GEMM
            # CTA holds nearly all registers of its SM, so the bias column sums get SMs of their own (_COLSUM_SMS; at H = 1024
            # the GEMMs still take 4 rounds of tiles on 32 instead of 34 CTAs): ONE launch of a few CTAs that all stay resident
            # and walk every slab while L_a runs (with one CTA per slab, the CTAs that find no SM would start after L_a; two
            # concurrent column-sum launches would share the slab scratch).  Gradient buckets are launched under the next
            # ordinary launch (dW_xa), not under these: a programmatic dependent may start before the kernels ahead of it in
            # the stream are complete.
            # Weight drop: dW_hb's mask is an ordinary launch behind the column sums (it runs after L_a, before dW_xa), and W_hb is
            # released only from then on.  With dx_b beside L_a too (full_b), they share what dx_b leaves (pipelined_bwd_split).
            dw_xb = _accumulate_grad(a[3], dg_b.t(), hin_b.reshape(T * B, Ha), pdl=True, max_ctas=side)
            release(a[3])
            part, out, dw_hb = _grad_gemm(a[4], dg_b.t(), h_seq_b[:T].reshape(T * B, Hb), pdl=True, max_ctas=side, masked=bool(wdb))
            db_b = _bias_grad(a[5], dg_b, under_gemm=True, max_ctas=4 * _COLSUM_SMS)
            if wdb:
                _weight_drop_grad(part, out, wdb, part is not out)
        else:
            # the bias column sums run NEXT TO the first weight-gradient GEMM of their layer (same dG, idle SMs), not after it
            # (each GEMM is followed by: finished gradient buckets [programmatic dependents of the GEMM], then half of the layer's
            # bias column sums [programmatic dependent of whatever was launched last] - all three run side by side)
            dw_xb = _accumulate_grad(a[3], dg_b.t(), hin_b.reshape(T * B, Ha))
            release(a[3])
            sink = _bias_grad(a[5], dg_b, under_gemm=dw_xb is None, part=0)
            dw_hb = _accumulate_grad(a[4], dg_b.t(), h_seq_b[:T].reshape(T * B, Hb), wdrop=wdb)
            db_b = _bias_grad(a[5], dg_b, under_gemm=dw_hb is None and not wdb, part=1, sink=sink)
        release(a[4], a[5])
        dg_a = dpre_a.view(T * B, 4 * Ha)
        # pipelined, 2 x 1024 on a 132-SM H100: single-CTA 128 x 256 tiles put the 128 tiles of each of layer a's weight-gradient
        # GEMMs on 128 SMs in one wave, at the per-SM rate of the capped side GEMMs; 2-CTA clusters ran them at about half that
        # rate per SM (bench/side_gemms.py).  The tile's K order, and with it every bit of dW, is the same either way.  db_a comes
        # out of the dW_ha launch as the row sums of dG_a^T (csrc/gemm2_wgmma.cu): the column-sum kernels beside these GEMMs only
        # found the 4 SMs the GEMMs leave free and ran on after them.
        dw_xa = _accumulate_grad(a[0], dg_a.t(), x2d, b_folded=ctx.x_folded, ctas=1 if pipelined else 0)
        if not ctx.needs_input_grad[0]:
            release(a[0])                                                 # (else W_xa is released after the dX GEMM reads it)
        if pipelined:
            db_out, db_acc, db_a = grad_out(a[2], (4 * Ha,), dev)
            dw_ha = _accumulate_grad(a[1], dg_a.t(), h_seq_a[:T].reshape(T * B, Ha), ctas=1, rowsum=(db_out, db_acc), wdrop=wda)
            count("fused_bias_grads")
        else:
            sink = _bias_grad(a[2], dg_a, under_gemm=dw_xa is None, part=0)
            dw_ha = _accumulate_grad(a[1], dg_a.t(), h_seq_a[:T].reshape(T * B, Ha), wdrop=wda)
            db_a = _bias_grad(a[2], dg_a, under_gemm=dw_ha is None and not wda, part=1, sink=sink)
        release(a[1], a[2])
        dx = None
        if ctx.needs_input_grad[0]:                                       # (never with a folded input: lstm_pair_sequence)
            dx = G.matmul(dg_a, wxa.t(), out_dtype=cd).view(T, B, D)
            STATS["kernels"] += 1
            release(a[0])
        t = ctx.in_dtypes
        return (dx, dh0a.to(t[0]), dc0a.to(t[1]), dw_xa, dw_ha, db_a, dh0b.to(t[2]), dc0b.to(t[3]), dw_xb, dw_hb, db_b, None, None,
                None, None, None, None, None)


def lstm_pair_sequence(x_seq, la, lb, lengths=None, schedule=None, dropouts=(None, None), weight_drops=(None, None),
                       activation_sums=False):
    """Two stacked layers as one op.  ``la`` / ``lb`` = (h0, c0, w_x, w_h, bias).  -> (h_seq_b, hT_a, cT_a, hT_b, cT_b).
    ``lengths``: optional int32 ``[B]`` per-row lengths (both layers run their masked kernels; the gated GEMM is unchanged).
    ``schedule``: "wavefront" or "pipelined" (see ``pair_schedule``); None = the one ``pair_schedule`` picks for the device.
    ``dropouts``: ``reference.DropoutSpec`` (or None) of layer a's output (the input of layer b) and of layer b's output (the
    first result).  ``weight_drops``: weight-drop ``reference.DropoutSpec`` (or None) of layer a's and layer b's ``W_h``: the
    recurrences read the masked images, and each ``dW_h`` is masked on its way into the sink.  ``activation_sums``: one more
    output, layer b's sums of ``lstm_layer_sequence``."""
    _check_lengths_arg(lengths, x_seq.shape[1], x_seq.device)
    if schedule is None:
        schedule = _pair_schedule_of(x_seq, la[3].shape[1], lb[3].shape[1])
    if schedule not in ("wavefront", "pipelined"):
        raise ValueError(f"no layer-pair schedule for x {tuple(x_seq.shape)} {x_seq.dtype}, H = {la[3].shape[1]}, "
                         f"{lb[3].shape[1]} (schedule={schedule!r}); check wavefront_supported first")
    if (not x_seq.is_contiguous() and not x_seq.requires_grad and x_seq.transpose(0, 1).is_contiguous()
            and (x_seq.shape[2] * x_seq.element_size()) % 16 == 0):
        if FOLDED_FEED and G.folded_ok(x_seq.transpose(0, 1)):
            return _LSTMPairFn.apply(x_seq, *la, *lb, lengths, schedule, *dropouts, *weight_drops,   # read in place (see forward)
                                     activation_sums)
        x_seq = ext().transpose01(x_seq.transpose(0, 1))
        STATS["kernels"] += 1
    return _LSTMPairFn.apply(x_seq.contiguous(), *la, *lb, lengths, schedule, *dropouts, *weight_drops, activation_sums)
