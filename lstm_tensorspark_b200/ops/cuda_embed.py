"""CUDA token embedding (csrc/embedding.cu): ``x [T,B,E] = table[tokens]`` in front of the first LSTM layer, time-major and
contiguous, so the first layer (or layer pair) reads it with no transpose.  Tokens stay int32 ``[B,T]`` on the device and the
lengths are read there too (no host sync: a captured graph holds across token batches).

  forward   one gather launch from the table's maintained bf16 shadow (bf16 path) or the fp32 table;
  backward  the first layer's ``dx`` (its wgmma dX GEMM) -> ``dEmbedding`` straight into the table's flat gradient sink, in three
            launches (rank, plan, sum): a stable counting sort of the counted positions by id and a fixed-order fp32 sum per id,
            so the result is bitwise reproducible and independent of the grid.
Dropout (``input_dropout`` over each position's E units, ``embedding_dropout`` over whole table rows): the gather and the sum
launch their masked instantiations, which draw the masks in place (``reference.embedding``); the launch count is unchanged.
Semantics: ``reference.embedding``."""
from __future__ import annotations

import torch

from .cuda_ext import LAUNCHES, count, drop_args, ext
from .params import grad_out, lowp, release


def _tokens(tokens: torch.Tensor) -> torch.Tensor:
    tok = tokens if tokens.dim() == 2 else tokens.unsqueeze(1)          # [B] = one step
    return tok.to(torch.int32).contiguous()


class _EmbedFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, tokens, table, lengths, dtype, input_dropout, embedding_dropout):
        tok = _tokens(tokens)
        if tok.device != table.device:
            raise ValueError(f"tokens on {tok.device}, the embedding table on {table.device}")
        tab = lowp(table, torch.bfloat16) if dtype == torch.bfloat16 else table.detach().float().contiguous()
        ln = None if lengths is None else lengths.contiguous()
        di, de = drop_args(input_dropout, tab.device), drop_args(embedding_dropout, tab.device)
        drop = {"in_step": di.get("drop_step"), "in_desc": di.get("drop_desc", []),
                "row_step": de.get("drop_step"), "row_desc": de.get("drop_desc", [])}
        x = ext().embed_fwd(tab, tok, ln, **drop)
        count("embed_fwd")
        if di or de:
            count("embed_fwd_dropout")
        ctx.tok, ctx.ln, ctx.addr, ctx.shape, ctx.drop = tok, ln, table.data_ptr(), tuple(table.shape), drop
        return x if x.dtype == dtype else x.to(dtype)

    @staticmethod
    def backward(ctx, dx):
        E = ext()
        d = dx.detach()
        if d.dtype not in (torch.bfloat16, torch.float32):
            d = d.float()
        d = d.contiguous()
        out, acc, ret = grad_out(ctx.addr, ctx.shape, d.device)
        E.embed_bwd(d, ctx.tok, ctx.ln, out, acc, **ctx.drop)
        LAUNCHES["n"] += E.EMBED_BWD_LAUNCHES - 1
        release(ctx.addr)
        count("embed_bwd")
        if ctx.drop["in_step"] is not None or ctx.drop["row_step"] is not None:
            count("embed_bwd_dropout")
        return None, ret, None, None, None, None


def embedding(tokens, table, lengths=None, dtype=None, input_dropout=None, embedding_dropout=None):
    if tokens.is_floating_point():
        raise ValueError(f"--vocab_size needs integer token ids, got {tokens.dtype}")
    return _EmbedFn.apply(tokens, table, lengths, table.dtype if dtype is None else dtype, input_dropout, embedding_dropout)
