"""CUDA head op: dense layer + softmax cross-entropy + accuracy in ONE launch on the tensor cores (csrc/head_wgmma.cu:
TMA-fed wgmma tile, logits in registers, softmax / NLL / accuracy / dlogits in the epilogue) and the whole backward
(dh, dW, db) in ONE launch that writes dW / db straight into the flat gradient buffer.
Parity: original src/rnn.py:214-221 (Dense1), :55-63 (loss), :84-92 (accuracy), :224 (autodiff)."""
from __future__ import annotations

import torch

from .cuda_ext import count, ext
from .params import grad_out, release


class _HeadXentFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, h, weights, bias, labels):
        E = ext()
        B = h.shape[0]
        hc = h.detach()
        if hc.dtype not in (torch.bfloat16, torch.float32):
            hc = hc.float()
        if hc.stride(-1) != 1:
            hc = hc.contiguous()
        w = weights.detach().float().contiguous()
        b = bias.detach().float().contiguous()
        lab = labels.long().contiguous()
        logits, dlogits, loss_sum, correct = E.head_fwd(hc, w, b, lab)
        ctx.save_for_backward(hc, w, dlogits)
        ctx.h_dtype = h.dtype
        ctx.addrs = (weights.data_ptr(), bias.data_ptr())
        loss = (loss_sum / B).squeeze(0)
        ctx.mark_non_differentiable(logits, correct)
        return logits, loss, correct.squeeze(0)

    @staticmethod
    def backward(ctx, _dlogits_unused, dloss, _dcorrect_unused):
        hc, w, dlogits = ctx.saved_tensors
        hcc = hc if hc.is_contiguous() else hc.contiguous()
        dw, acc_w, ret_w = grad_out(ctx.addrs[0], w.shape, w.device)
        db, acc_b, ret_b = grad_out(ctx.addrs[1], (w.shape[1],), w.device)
        dl = dloss.detach().float().reshape(1).contiguous()
        dh = ext().head_bwd(hcc, w, dlogits, dl, dw, db, acc_w, acc_b)
        release(*ctx.addrs)
        return dh.to(ctx.h_dtype), ret_w, ret_b, None


def head_xent(h, weights, bias, labels):
    return _HeadXentFn.apply(h, weights, bias, labels)


class _HeadXentStepFn(torch.autograd.Function):
    """The head at every time step of ``h_seq [T,B,H]`` (read in place as ``T·B`` time-major rows): one forward launch (logits,
    loss over the counted positions, correct count, N, dlogits) and one backward launch (dh_seq, dW, db).  N stays on the
    device, so a captured graph holds across batches with different lengths."""

    @staticmethod
    def forward(ctx, h_seq, weights, bias, labels, lengths):
        E = ext()
        T, B, H = h_seq.shape
        hc = h_seq.detach()
        if hc.dtype not in (torch.bfloat16, torch.float32):
            hc = hc.float()
        h2 = hc.reshape(T * B, H) if hc.is_contiguous() else hc.contiguous().view(T * B, H)
        w = weights.detach().float().contiguous()
        b = bias.detach().float().contiguous()
        lab = labels.long().contiguous()
        ln = None if lengths is None else lengths.contiguous()
        logits, dlogits, loss, correct, n, used_tc = E.head_step_fwd(h2, w, b, lab, ln, T)
        count("head_per_step")
        if int(used_tc[0]):
            count("head_per_step_tc")
        ctx.save_for_backward(h2, w, dlogits)
        ctx.shape, ctx.h_dtype = (T, B, H), h_seq.dtype
        ctx.addrs = (weights.data_ptr(), bias.data_ptr())
        ctx.mark_non_differentiable(logits, correct, n)
        return logits, loss.squeeze(0), correct.squeeze(0), n.squeeze(0)

    @staticmethod
    def backward(ctx, _dlogits_unused, dloss, _dcorrect_unused, _dcount_unused):
        h2, w, dlogits = ctx.saved_tensors
        dw, acc_w, ret_w = grad_out(ctx.addrs[0], w.shape, w.device)
        db, acc_b, ret_b = grad_out(ctx.addrs[1], (w.shape[1],), w.device)
        dl = dloss.detach().float().reshape(1).contiguous()
        dh = ext().head_step_bwd(h2, w, dlogits, dl, dw, db, acc_w, acc_b)
        release(*ctx.addrs)
        return dh.view(ctx.shape).to(ctx.h_dtype), ret_w, ret_b, None, None


def head_xent_per_step(h_seq, weights, bias, labels, lengths=None):
    return _HeadXentStepFn.apply(h_seq, weights, bias, labels, lengths)
