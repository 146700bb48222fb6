"""CUDA pooling over time (csrc/seq_pool.cu): the top layer's ``h_seq [T,B,H]`` -> ``s [B,H]`` fp32 over each row's counted
steps, read in place as ``T·B`` time-major rows with per-row lengths on the device (no host sync, so a captured graph holds
across batches with different lengths).

  mean / max  one forward launch, one backward launch (max keeps an int32 argmax ``[B,H]``);
  attention   forward: ``h W_a`` on the wgmma GEMM (fp32 out), one fused launch for ``+ b_a``, tanh, ``. v`` and the masked
              softmax (``u`` is kept for the backward pass), one pooling launch;
              backward: one launch for dU and the dv / db_a sums, ``dU W_a^T`` and ``dW_a = h^T dU`` on the wgmma GEMM (dW_a
              straight into its flat gradient sink), one launch that adds ``alpha_t ds`` and rounds dh_seq once.
Semantics: ``reference.pool_sequence``."""
from __future__ import annotations

import torch

from .cuda_ext import count, ext
from .params import grad_out, lowp, release

MODES = {"mean": 0, "max": 1, "attention": 2}


class _PoolFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, h_seq, lengths, mode, w_a, b_a, v):
        from . import cuda_gemm
        E = ext()
        T, B, H = h_seq.shape
        hc = h_seq.detach()
        if hc.dtype not in (torch.bfloat16, torch.float32):
            hc = hc.float()
        h2 = hc.reshape(T * B, H) if hc.is_contiguous() else hc.contiguous().view(T * B, H)
        ln = None if lengths is None else lengths.contiguous()
        m = MODES[mode]
        ctx.mode, ctx.T, ctx.h_dtype, ctx.ln = m, T, h_seq.dtype, ln
        if m == 2:
            wa = lowp(w_a, torch.bfloat16) if h2.dtype == torch.bfloat16 else w_a.detach().float().contiguous()
            ba, vv = b_a.detach().float().contiguous(), v.detach().float().contiguous()
            u = cuda_gemm.matmul(h2, wa.t(), out_dtype=torch.float32)          # h W_a [T·B, A]; tanh(. + b_a) in place below
            alpha = E.seq_pool_attn_scores(u, ba, vv, ln, T, exact=h2.dtype == torch.float32)
            s, _ = E.seq_pool_fwd(h2, ln, T, m, alpha)
            count("pool_attention_fwd")
            ctx.save_for_backward(h2, alpha, u, wa, vv)
            ctx.addrs = (w_a.data_ptr(), b_a.data_ptr(), v.data_ptr())
        else:
            s, am = E.seq_pool_fwd(h2, ln, T, m, None)
            ctx.save_for_backward(am if m == 1 else None)
        count("pool_fwd")
        return s

    @staticmethod
    def backward(ctx, ds):
        E = ext()
        T, m, ln = ctx.T, ctx.mode, ctx.ln
        dsf = ds.detach().float().contiguous()
        B, H = dsf.shape
        out_bf16 = ctx.h_dtype == torch.bfloat16
        count("pool_bwd")
        if m != 2:
            (am,) = ctx.saved_tensors
            dh = E.seq_pool_bwd(dsf, ln, T, m, am, None, None, out_bf16)
            return dh.view(T, B, H).to(ctx.h_dtype), None, None, None, None, None
        from . import cuda_gemm
        h2, alpha, u, wa, vv = ctx.saved_tensors
        A = u.shape[1]
        dwa, acc_dwa, ret_dwa = grad_out(ctx.addrs[0], wa.shape, dsf.device)
        dba, acc_dba, ret_dba = grad_out(ctx.addrs[1], (A,), dsf.device)
        dv, acc_dv, ret_dv = grad_out(ctx.addrs[2], (A,), dsf.device)
        dU = E.seq_pool_attn_bwd(h2, dsf, alpha, u, vv, ln, T, dv, dba, acc_dv, acc_dba)       # dtype of h
        G = cuda_gemm.matmul(dU, wa, out_dtype=torch.float32)                                 # dU W_a^T [T·B, H]
        cuda_gemm.matmul(h2.t(), dU.t(), out=dwa, accumulate=acc_dwa)                         # dW_a = h^T dU
        dh = E.seq_pool_bwd(dsf, ln, T, m, None, alpha, G, out_bf16)
        count("pool_attention_bwd")
        release(*ctx.addrs)
        return dh.view(T, B, H).to(ctx.h_dtype), None, None, ret_dwa, ret_dba, ret_dv


def pool_sequence(h_seq, lengths=None, mode: str = "mean", attention=None):
    if mode not in MODES:
        raise ValueError(f"unknown pooling {mode!r} for the CUDA op: one of {', '.join(MODES)}")
    if mode == "attention":
        if attention is None:
            raise ValueError("attention pooling needs its parameters (W_a, b_a, v)")
        w_a, b_a, v = attention
    else:
        w_a = b_a = v = None
    return _PoolFn.apply(h_seq, lengths, mode, w_a, b_a, v)
