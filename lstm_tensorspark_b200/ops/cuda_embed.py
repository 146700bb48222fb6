"""CUDA token embedding (csrc/embedding.cu): ``x [T,B,E] = table[tokens]`` in front of the first LSTM layer, time-major and
contiguous, so the first layer (or layer pair) reads it with no transpose.  Tokens stay int32 ``[B,T]`` on the device and the
lengths are read there too (no host sync: a captured graph holds across token batches).

  forward   one gather launch from the table's maintained bf16 shadow (bf16 path) or the fp32 table;
  backward  the first layer's ``dx`` (its wgmma dX GEMM) -> ``dEmbedding`` straight into the table's flat gradient sink, in three
            launches (rank, plan, sum): a stable counting sort of the counted positions by id and a fixed-order fp32 sum per id,
            so the result is bitwise reproducible and independent of the grid.
Semantics: ``reference.embedding``."""
from __future__ import annotations

import torch

from .cuda_ext import LAUNCHES, count, ext
from .params import grad_out, lowp


def _tokens(tokens: torch.Tensor) -> torch.Tensor:
    tok = tokens if tokens.dim() == 2 else tokens.unsqueeze(1)          # [B] = one step
    return tok.to(torch.int32).contiguous()


class _EmbedFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, tokens, table, lengths, dtype):
        tok = _tokens(tokens)
        if tok.device != table.device:
            raise ValueError(f"tokens on {tok.device}, the embedding table on {table.device}")
        tab = lowp(table, torch.bfloat16) if dtype == torch.bfloat16 else table.detach().float().contiguous()
        ln = None if lengths is None else lengths.contiguous()
        x = ext().embed_fwd(tab, tok, ln)
        count("embed_fwd")
        ctx.tok, ctx.ln, ctx.addr, ctx.shape = tok, ln, table.data_ptr(), tuple(table.shape)
        return x if x.dtype == dtype else x.to(dtype)

    @staticmethod
    def backward(ctx, dx):
        E = ext()
        d = dx.detach()
        if d.dtype not in (torch.bfloat16, torch.float32):
            d = d.float()
        d = d.contiguous()
        out, acc, ret = grad_out(ctx.addr, ctx.shape, d.device)
        E.embed_bwd(d, ctx.tok, ctx.ln, out, acc)
        LAUNCHES["n"] += E.EMBED_BWD_LAUNCHES - 1
        count("embed_bwd")
        return None, ret, None, None


def embedding(tokens, table, lengths=None, dtype=None):
    if tokens.is_floating_point():
        raise ValueError(f"--vocab_size needs integer token ids, got {tokens.dtype}")
    return _EmbedFn.apply(tokens, table, lengths, table.dtype if dtype is None else dtype)
