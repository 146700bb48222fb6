"""CUDA op of the large-vocabulary per-step head (csrc/head_vocab.cu): softmax cross-entropy over ``C >= 512`` classes at every
time step without storing the logits ``[B,T,C]`` or an fp32 dlogits ``[T·B,C]``.

Forward: one fused TMA + wgmma launch reduces every 128 x 256 logit tile to four numbers per row in its epilogue, a second small
launch merges them into ``lse [T·B]``, the loss, the correct count and N.  Backward, in chunks of ``ROW_CHUNK`` rows, in index
order on one stream: the logits of the chunk are recomputed and turned into bf16 dlogits in a reused scratch ``[ROW_CHUNK, C]``,
then ``dh = dlogits W^T``, ``dW += h^T dlogits`` (straight into the flat gradient buffer) and ``db += column sums`` - every sum in
a fixed order, so two calls on the same inputs give the same bits.  N, lse and the masks stay on the device: a captured CUDA
graph holds across batches with other lengths.

``class_major=True`` (tied embeddings): ``weights`` is the embedding table ``[C,H] = W^T`` itself, which the head kernels read in
place as a K-major operand.  Backward then computes ``dh = dlogits · table`` and ``dTable (+)= dlogits^T h`` into the table's
gradient sink, where the embedding's scatter-add later in the same backward pass adds its own part.
"""
from __future__ import annotations

import torch

from . import cuda_gemm as G
from .cuda_ext import count, ext
from .params import grad_out, lowp, release

ROW_CHUNK = 4096          # rows of h per backward chunk: the schedule depends on the shapes only
MIN_CLASSES = 512


def supported(h_seq: torch.Tensor, num_classes: int) -> bool:
    """Does this op take the head (bf16 activations on the GPU, ``H % 64 == 0``, ``C % 8 == 0``, ``C >= 512``)?  Everything
    else stays with ``cuda_head.head_xent_per_step``."""
    return (h_seq.is_cuda and h_seq.dtype == torch.bfloat16 and h_seq.dim() == 3 and h_seq.shape[2] % 64 == 0
            and num_classes % 8 == 0 and num_classes >= MIN_CLASSES)


def _weights_lowp(weights: torch.Tensor, class_major: bool) -> torch.Tensor:
    """The bf16 operand of the head kernels: the maintained shadow, or one rounding of the fp32 weights.  ``class_major``: the
    table ``[C,H]`` itself (never a transposed view: the shadow and the gradient sink are found by the parameter's address and
    shape), read by TMA in place, which needs a 16-byte aligned base (FlatParams places every parameter at a multiple of 64
    elements, so a shadow view always is) and ``H % 8 == 0`` (implied by ``H % 64 == 0``)."""
    wb = lowp(weights, torch.bfloat16)
    if class_major:
        assert wb.is_contiguous() and wb.data_ptr() % 16 == 0, "the tied table's bf16 operand must be packed and 16-byte aligned"
    return wb


class _VocabXentFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, h_seq, weights, bias, labels, lengths, class_major=False):
        E = ext()
        T, B, H = h_seq.shape
        hc = h_seq.detach()
        h2 = hc.reshape(T * B, H) if hc.is_contiguous() else hc.contiguous().view(T * B, H)
        wb = _weights_lowp(weights, class_major)
        b = bias.detach().float().contiguous()
        lab = labels.long().contiguous()
        ln = None if lengths is None else lengths.contiguous()
        C = wb.shape[0 if class_major else 1]
        part = torch.empty(T * B * E.vocab_head_parts(C) * 4, dtype=torch.float32, device=h2.device)
        lse, loss, correct, n = E.vocab_head_fwd(h2, wb, bool(class_major), b, lab, ln, T, part)
        count("vocab_head_fwd")
        if class_major:
            count("vocab_head_fwd_tied")
        ctx.save_for_backward(h2, wb, b, lab, ln, lse, n)
        ctx.shape, ctx.class_major = (T, B, H), bool(class_major)
        ctx.addrs = (weights.data_ptr(), bias.data_ptr())
        ctx.mark_non_differentiable(correct, n)
        return loss.squeeze(0), correct.squeeze(0), n.squeeze(0)

    @staticmethod
    def backward(ctx, dloss, _dcorrect_unused, _dcount_unused):
        E = ext()
        h2, wb, b, lab, ln, lse, n = ctx.saved_tensors
        T, cm = ctx.shape[0], ctx.class_major
        R, H = h2.shape
        C = wb.shape[0 if cm else 1]
        dw, acc_w, ret_w = grad_out(ctx.addrs[0], (C, H) if cm else (H, C), h2.device)
        db, acc_b, ret_b = grad_out(ctx.addrs[1], (C,), h2.device)
        scale = dloss.detach().float().reshape(1).contiguous()
        dh = torch.empty_like(h2)
        dl = torch.empty(min(ROW_CHUNK, R), C, dtype=torch.bfloat16, device=h2.device)
        for r0 in range(0, R, ROW_CHUNK):
            rows = min(ROW_CHUNK, R - r0)
            d = dl[:rows]
            E.vocab_head_dlogits(h2, wb, cm, b, lab, ln, T, lse, n, scale, r0, rows, d)
            acc = bool(acc_w or r0 > 0)
            if cm:
                G.matmul(d, wb.t(), out=dh[r0:r0 + rows])                                      # dh = dlogits table
                G.matmul(d.t(), h2[r0:r0 + rows].t(), out=dw, accumulate=acc)                   # dTable (+)= dlogits^T h
            else:
                G.matmul(d, wb, out=dh[r0:r0 + rows])                                          # dh = dlogits W^T
                G.matmul(h2[r0:r0 + rows].t(), d.t(), out=dw, accumulate=acc)                   # dW (+)= h^T dlogits
            E.vocab_head_colsum(d, db.view(-1), bool(acc_b or r0 > 0))
        count("vocab_head_bwd")
        release(*(ctx.addrs[1:] if cm else ctx.addrs))    # (a tied table's gradient is finished by the embedding's backward)
        return dh.view(ctx.shape), ret_w, ret_b, None, None, None


def vocab_xent_per_step(h_seq, weights, bias, labels, lengths=None, class_major=False):
    """-> (mean loss over the counted positions, correct count, N); see ``ops.functional.vocab_xent_per_step``."""
    return _VocabXentFn.apply(h_seq, weights, bias, labels, lengths, bool(class_major))


def _device_int(v, device):
    return v if isinstance(v, torch.Tensor) else torch.full((1,), int(v), dtype=torch.int32, device=device)


def _sample_args(step, row0, tokens, record, B, device):
    tok = torch.empty(B, dtype=torch.int32, device=device) if tokens is None else tokens
    rec_tok, rec_lp, s0 = (None, None, 0) if record is None else record
    return _device_int(step, device), _device_int(row0, device), tok, rec_tok, rec_lp, s0


def vocab_sample(h, weights, bias, temperature: float, seed: int, step, tokens=None, record=None, row0=0, class_major=False,
                 top_k: int = 0, top_p: float = 1.0):
    """Sample the next token from ``h [B,H]`` bf16 through the head's tensor-core kernel (``kSample``), without storing the
    logits; see ``ops.functional.vocab_sample``.  With a filter on (the caller passes ``top_k = 0`` and ``top_p = 1`` when it is
    off) the same main loop stores the fp32 logits (``kLogits``) and ``vocab_sample_logits`` samples them."""
    wb = _weights_lowp(weights, class_major)
    hc, bc = h.detach().contiguous(), bias.detach().float().contiguous()
    if class_major:
        count("vocab_sample_tied")
    if top_k > 0 or top_p < 1:
        logits = ext().vocab_head_logits(hc, wb, bool(class_major), bc)
        return vocab_sample_logits(logits, temperature, seed, step, tokens, record, row0, top_k, top_p)
    step_t, row_t, tok, rec_tok, rec_lp, s0 = _sample_args(step, row0, tokens, record, h.shape[0], h.device)
    lp = ext().vocab_sample(hc, wb, bool(class_major), bc, float(temperature), int(seed), step_t, row_t, tok, rec_tok, rec_lp, int(s0))
    count("vocab_sample")
    return tok, lp


def vocab_sample_logits(logits, temperature: float, seed: int, step, tokens=None, record=None, row0=0, top_k: int = 0,
                        top_p: float = 1.0):
    """The same sampling from stored fp32 logits ``[B,C]`` (bias included): the inputs the tensor-core kernel does not take, and
    top-k / top-p (on: ``top_k > 0`` or ``top_p < 1``, at temperature > 0), where ``vocab_threshold`` computes each row's
    threshold first and the sampling kernel scores only the classes at or above it."""
    step_t, row_t, tok, rec_tok, rec_lp, s0 = _sample_args(step, row0, tokens, record, logits.shape[0], logits.device)
    lg = logits.float().contiguous()
    tau = None
    if top_k > 0 or top_p < 1:
        tau = ext().vocab_threshold(lg, int(top_k), float(top_p), float(temperature))
        count("vocab_sample_filtered")
    lp = ext().vocab_sample_logits(lg, float(temperature), int(seed), step_t, row_t, tok, rec_tok, rec_lp, int(s0), tau)
    count("vocab_sample")
    return tok, lp
