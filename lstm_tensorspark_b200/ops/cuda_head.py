"""CUDA head op: dense layer + softmax cross-entropy + accuracy in ONE launch on the tensor cores (csrc/head_wgmma.cu:
TMA-fed wgmma tile, logits in registers, softmax / NLL / accuracy / dlogits in the epilogue) and the whole backward
(dh, dW, db) in ONE launch that writes dW / db straight into the flat gradient buffer.
Parity: original src/rnn.py:214-221 (Dense1), :55-63 (loss), :84-92 (accuracy), :224 (autodiff)."""
from __future__ import annotations

import torch

from .cuda_ext import ext


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
        from .cuda_lstm import grad_sink
        E = ext()
        hc, w, dlogits = ctx.saved_tensors
        hcc = hc if hc.is_contiguous() else hc.contiguous()
        sw, sb = grad_sink(ctx.addrs[0]), grad_sink(ctx.addrs[1])
        dl = dloss.detach().float().reshape(1).contiguous()
        if sw is not None and sb is not None and sw[1] == sb[1]:
            dh = E.head_bwd(hcc, w, dlogits, dl, sw[0], sb[0], sw[1])
            return dh.to(ctx.h_dtype), None, None, None
        if sw is not None and sb is not None:             # one of the two already holds a gradient: bring both to "accumulate"
            if not sw[1]:
                sw[0].zero_()
            if not sb[1]:
                sb[0].zero_()
            dh = E.head_bwd(hcc, w, dlogits, dl, sw[0], sb[0], True)
            return dh.to(ctx.h_dtype), None, None, None
        dw = torch.empty_like(w)
        db = torch.empty(w.shape[1], dtype=torch.float32, device=w.device)
        dh = E.head_bwd(hcc, w, dlogits, dl, dw, db, False)
        return dh.to(ctx.h_dtype), dw, db, None


def head_xent(h, weights, bias, labels):
    return _HeadXentFn.apply(h, weights, bias, labels)


class _HeadXentStepFn(torch.autograd.Function):
    """The head at every time step of ``h_seq [T,B,H]`` (read in place as ``T·B`` time-major rows): one forward launch (logits,
    loss over the counted positions, correct count, N, dlogits) and one backward launch (dh_seq, dW, db).  N stays on the
    device, so a captured graph holds across batches with different lengths."""

    @staticmethod
    def forward(ctx, h_seq, weights, bias, labels, lengths):
        from .cuda_lstm import STATS
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
        logits, dlogits, loss, correct, count, used_tc = E.head_step_fwd(h2, w, b, lab, ln, T)
        STATS["head_per_step"] = STATS.get("head_per_step", 0) + 1
        if int(used_tc[0]):
            STATS["head_per_step_tc"] = STATS.get("head_per_step_tc", 0) + 1
        ctx.save_for_backward(h2, w, dlogits)
        ctx.shape, ctx.h_dtype = (T, B, H), h_seq.dtype
        ctx.addrs = (weights.data_ptr(), bias.data_ptr())
        ctx.mark_non_differentiable(logits, correct, count)
        return logits, loss.squeeze(0), correct.squeeze(0), count.squeeze(0)

    @staticmethod
    def backward(ctx, _dlogits_unused, dloss, _dcorrect_unused, _dcount_unused):
        from .cuda_lstm import grad_sink
        E = ext()
        h2, w, dlogits = ctx.saved_tensors
        sw, sb = grad_sink(ctx.addrs[0]), grad_sink(ctx.addrs[1])
        dl = dloss.detach().float().reshape(1).contiguous()
        dw = db = None
        if (sw is None) != (sb is None):
            # one of the two has a sink: a tied head (--tie_embeddings) reads the table's transpose, a tensor of its own, next to
            # the registered bias.  That sink is taken by now, so it gets its gradient here; the other goes back to autograd
            dw = torch.empty_like(w)
            db = torch.empty(w.shape[1], dtype=torch.float32, device=w.device)
            dh = E.head_step_bwd(h2, w, dlogits, dl, dw, db, False)
            for sink, g in ((sw, dw), (sb, db)):
                if sink is not None and sink[1]:
                    sink[0].add_(g)
                elif sink is not None:
                    sink[0].copy_(g)
            return dh.view(ctx.shape).to(ctx.h_dtype), None if sw is not None else dw, None if sb is not None else db, None, None
        if sw is not None and sb is not None:
            if sw[1] != sb[1]:                             # one of the two already holds a gradient: bring both to "accumulate"
                if not sw[1]:
                    sw[0].zero_()
                if not sb[1]:
                    sb[0].zero_()
            dh = E.head_step_bwd(h2, w, dlogits, dl, sw[0], sb[0], bool(sw[1] or sb[1]))
        else:
            dw = torch.empty_like(w)
            db = torch.empty(w.shape[1], dtype=torch.float32, device=w.device)
            dh = E.head_step_bwd(h2, w, dlogits, dl, dw, db, False)
        return dh.view(ctx.shape).to(ctx.h_dtype), dw, db, None, None


def head_xent_per_step(h_seq, weights, bias, labels, lengths=None):
    return _HeadXentStepFn.apply(h_seq, weights, bias, labels, lengths)
