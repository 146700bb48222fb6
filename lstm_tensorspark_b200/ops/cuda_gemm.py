"""Matrix products of the CUDA path: every one of them runs on this framework's own kernels.

  * ``csrc/gemm2_wgmma.cu`` - TMA + wgmma (128 x 256 tiles, 2-CTA clusters sharing B), K-major or MN-major operands, bf16 / fp32 / accumulating
    fp32 output: the hoisted input projection, dX, and the weight gradients of the LSTM layers;
  * ``csrc/gemm_generic.cu``  - any shape / stride / dtype on the CUDA cores: the reference's own tiny configuration (iris:
    in_features 4, hidden 16, original src/rnn.py:312-321) and the fp32 parity path.

No call in here (or anywhere on the CUDA path) reaches cuBLAS.
"""
from __future__ import annotations

import os
from typing import Optional

import torch

from .cuda_ext import ext

GEMM_CTAS = int(os.environ.get("LSTM_TS_GEMM_CTAS", "2"))      # 2 = 2-CTA clusters sharing the B tile (TMA multicast), 1 = single CTA
GEMM_BN = int(os.environ.get("LSTM_TS_GEMM_BN", "256"))
STATS = {"tc": 0, "generic": 0}


def _major(t: torch.Tensor):
    """(is_mn_major, storage view with unit inner stride) of a logical [rows, contraction] operand, or None."""
    if t.dim() != 2:
        return None
    if t.stride(1) == 1 and t.stride(0) >= t.shape[1]:
        return False, t                      # contraction dim contiguous: K-major
    if t.stride(0) == 1 and t.stride(1) >= t.shape[0]:
        return True, t.t()                   # row dim contiguous: MN-major, stored as [contraction, rows]
    return None


def _tc_ok(a_k: torch.Tensor, b_k: torch.Tensor, M: int, N: int, K: int) -> bool:
    if a_k.dtype != torch.bfloat16 or b_k.dtype != torch.bfloat16:
        return False
    if M < 128 or N < 16 or K < 64 or K % 8 or N % 8 or M % 8:
        return False
    for t in (a_k, b_k):
        if t.stride(0) % 8 or t.data_ptr() % 16:
            return False
    return True


def folded_ok(x_bm: torch.Tensor) -> bool:
    """Can a batch-major ``[B, T, F]`` array be read in place as the time-major matrix ``[T*B, F]`` by the tensor-core GEMM
    (see ``Gemm2Params::a_fold`` in csrc/gemm2_wgmma.cu)?  Saves the transpose pass over the input of the first layer."""
    return (x_bm.is_cuda and x_bm.dim() == 3 and x_bm.dtype == torch.bfloat16 and x_bm.is_contiguous() and x_bm.shape[0] % 128 == 0
            and x_bm.shape[2] % max(64, GEMM_BN) == 0 and x_bm.data_ptr() % 16 == 0 and GEMM_BN in (128, 256))


def matmul(a: Optional[torch.Tensor], b_t: Optional[torch.Tensor], out: Optional[torch.Tensor] = None, accumulate: bool = False,
           out_dtype: Optional[torch.dtype] = None, bias: Optional[torch.Tensor] = None, max_ctas: int = 0,
           a_folded: Optional[torch.Tensor] = None, b_folded: Optional[torch.Tensor] = None, pdl: bool = False,
           ctas: int = 0, rowsum: Optional[tuple] = None) -> torch.Tensor:
    """``a [M,K] @ b_t[N,K]^T`` (+ bias[N]); either operand may be a transposed view (then it is MN-major and is read in
    place).  ``out`` fp32 + ``accumulate`` -> ``out += a @ b_t^T``.

    ``a_folded`` / ``b_folded`` (instead of ``a`` / ``b_t``): a batch-major ``[B, T, F]`` array (``folded_ok``) standing for the
    time-major matrix ``X = [T*B, F]``: ``a = X`` resp. ``b_t = X^T``.

    ``pdl``: programmatic dependent launch of the tensor-core GEMM (it starts once every CTA of the previous kernel is resident
    and waits for that kernel before it exits).  ``ctas``: CTAs per tile cluster, 1 or 2 (0 = ``LSTM_TS_GEMM_CTAS``).

    ``rowsum`` = (fp32 [M] tensor, accumulate flag): the same launch also writes (or adds) the row sums of ``a`` over K into it
    (tensor-core path with fp32 output only: a bias gradient next to its weight gradient)."""
    E = ext()
    ctas = ctas or GEMM_CTAS
    rs = dict(rowsum=rowsum[0], rowsum_acc=rowsum[1]) if rowsum is not None else {}
    if a_folded is not None or b_folded is not None:
        assert rowsum is None or a_folded is None, "row sums of a folded A are not supported"
        xb = a_folded if a_folded is not None else b_folded
        Bsz, T, F = xb.shape
        store = xb.view(Bsz, T * F)
        other = _major(b_t if a_folded is not None else a)
        assert folded_ok(xb) and other is not None and other[1].dtype == torch.bfloat16 and (a_folded is None or b_folded is None)
        if out_dtype is None:
            out_dtype = out.dtype if out is not None else torch.bfloat16
        STATS["tc"] += 1
        if a_folded is not None:
            return E.gemm2(store, other[1], bias=bias, out=out, a_mn=False, b_mn=other[0], out_fp32=out_dtype == torch.float32,
                           accumulate=accumulate, ctas=ctas, bn=GEMM_BN if b_t.shape[0] > 128 else 128, max_ctas=max_ctas, pdl=pdl,
                           a_fold=Bsz, fold_cols=F)
        return E.gemm2(other[1], store, bias=bias, out=out, a_mn=other[0], b_mn=True, out_fp32=out_dtype == torch.float32,
                       accumulate=accumulate, ctas=ctas, bn=GEMM_BN, max_ctas=max_ctas, pdl=pdl, b_fold=Bsz, fold_cols=F, **rs)
    M, K = a.shape
    N = b_t.shape[0]
    assert b_t.shape[1] == K, (a.shape, b_t.shape)
    if out_dtype is None:
        out_dtype = out.dtype if out is not None else a.dtype
    ma, mb = _major(a), _major(b_t)
    if ma is not None and mb is not None and _tc_ok(ma[1], mb[1], M, N, K) and out_dtype in (torch.bfloat16, torch.float32) \
            and not (accumulate and out_dtype != torch.float32) \
            and (out is None or (out.stride(1) == 1 and out.stride(0) % 4 == 0 and out.data_ptr() % 16 == 0)):
        STATS["tc"] += 1
        return E.gemm2(ma[1], mb[1], bias=bias, out=out, a_mn=ma[0], b_mn=mb[0], out_fp32=out_dtype == torch.float32,
                       accumulate=accumulate, ctas=ctas, bn=GEMM_BN if N > 128 else 128, max_ctas=max_ctas, pdl=pdl, **rs)
    assert a_folded is None and b_folded is None, "folded operands need the tensor-core path (check folded_ok first)"
    assert rowsum is None, "row sums need the tensor-core path"
    STATS["generic"] += 1
    a_g = a if a.dtype in (torch.float32, torch.bfloat16) else a.float()
    b_g = b_t if b_t.dtype in (torch.float32, torch.bfloat16) else b_t.float()
    if out is None:
        res = E.gemm_generic(a_g, b_g.t(), bias=bias, out_fp32=out_dtype == torch.float32)
        return res if res.dtype == out_dtype else res.to(out_dtype)
    return E.gemm_generic(a_g, b_g.t(), bias=bias, out=out, beta=1.0 if accumulate else 0.0)
