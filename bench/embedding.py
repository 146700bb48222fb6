"""Training throughput on token sequences (``--vocab_size``, one GPU): the headline model (2-layer-1024 LSTM, T = 128, B = 256,
bf16, Adam, CUDA graph) behind a learned embedding table of V = 32768 rows and E = 1024 columns.

    python bench/embedding.py --steps 50 --warmup 10

Arms, each device-timed with CUDA events around ``--steps`` steps after ``--warmup`` steps:
  * ``ours_<uniform|zipf>`` / ``..._variable_length``: ``TrainEngine.step`` with ``vocab_size=V`` on int32 token batches (ids
    uniform over V, or Zipf(1.1)), fixed-length and ragged (lengths in [T // 4, T]), the step captured as a CUDA graph on each of
    the 4 rotating device batches;
  * ``ours_dense``: the same model on dense bf16 features of the same shape, for the step-cost delta of the table;
  * ``cudnn_embedding``: the stand-in of ``baseline/harness.py`` (``variant="tuned"``) with ``nn.Embedding`` in front;
  * ``embed_kernels``: the gather and the gradient launches alone at the headline shape, next to their bandwidth bounds computed
    from the shapes at ``--hbm_gbps`` (computed, not measured).
Prints one JSON line, with the card's name and power limit.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "bench"))

import numpy as np
import torch

from variable_length import _card, _timed     # noqa: E402  (the shared helpers)


def _tokens(kind, n, T, V, seed):
    rng = np.random.default_rng(seed)
    if kind == "uniform":
        return rng.integers(0, V, size=(n, T)).astype(np.int32)
    return ((rng.zipf(1.1, size=(n, T)) - 1) % V).astype(np.int32)


def ours(args, x, ys, ls, dev, vocab):
    from lstm_tensorspark_b200.config import Config
    from lstm_tensorspark_b200.engine import TrainEngine
    from lstm_tensorspark_b200.ops import cuda_lstm
    B, T, nb = args.batch_size, args.seq_len, 4
    cfg = Config(hidden_units=args.hidden_units, in_features=args.in_features, seq_len=T, batch_size=B, num_classes=args.num_classes,
                 partitions=1, sync_mode="none", init="scaled", learn_initial_state=False, dtype="bf16", device="cuda",
                 learning_rate=1e-3, quiet=True, variable_length=ls is not None, vocab_size=vocab)
    eng = TrainEngine(cfg, 0, 1, None, batch_size=B, device=dev, dtype=torch.bfloat16)
    dx = torch.as_tensor(x).to(dev, torch.int32 if vocab else torch.bfloat16)
    dy = torch.as_tensor(ys).to(dev)
    dl = None if ls is None else torch.as_tensor(ls).to(dev)
    batches = [(dx[i * B:(i + 1) * B], dy[i * B:(i + 1) * B], None if dl is None else dl[i * B:(i + 1) * B]) for i in range(nb)]
    n_embed = cuda_lstm.STATS.get("embed_bwd", 0)
    eng.step(*batches[0])
    if args.cuda_graph:
        eng.capture(*batches[0][:2], lengths=batches[0][2], bind=batches[1:] if dl is not None else [b[:2] for b in batches[1:]])
    it = {"i": 0}

    def step():
        eng.step(*batches[it["i"] % nb])
        it["i"] += 1
    ms = _timed(step, args.steps, args.warmup)
    cuda_lstm.check_kernel_errors(dev)
    return {"ms_per_step": ms, "value": B * 1e3 / ms, "cuda_graph": bool(args.cuda_graph),
            "embed_launched": cuda_lstm.STATS.get("embed_bwd", 0) > n_embed,
            "pipelined": cuda_lstm.STATS.get("pipelined_fwd", 0) > 0}


def cudnn(args, x, ys, dev):
    from baseline import harness
    B, nb = args.batch_size, 4
    hidden = [int(h) for h in args.hidden_units.split(",")]
    runner = harness.BaselineRunner(hidden, args.in_features, args.num_classes, B, args.seq_len, 0, 1, dev, variant="tuned",
                                    vocab_size=args.vocab_size)
    dx = torch.as_tensor(x).to(dev, torch.int64)
    dy = torch.as_tensor(ys).to(dev)
    batches = [(dx[i * B:(i + 1) * B], dy[i * B:(i + 1) * B]) for i in range(nb)]
    graphed = runner.capture(*batches[0], bind=batches)
    it = {"i": 0}

    def step():
        runner.train_step(*batches[it["i"] % nb])
        it["i"] += 1
    ms = _timed(step, args.steps, args.warmup)
    return {"ms_per_step": ms, "value": B * 1e3 / ms, "cuda_graph": graphed}


def embed_kernels(args, dev, reps=100):
    """Device time of the gather and of the gradient (rank, plan, sum) alone, uniform and Zipf ids, ragged lengths.  Bytes they
    must move at least: the gather writes x (T·B·E bf16) and reads as many table rows; the gradient reads dx once and writes the
    whole fp32 table gradient (V·E·4, overwrite mode)."""
    from lstm_tensorspark_b200.ops.cuda_ext import ext
    B, T, V, E = args.batch_size, args.seq_len, args.vocab_size, args.in_features
    g = torch.Generator(device="cpu").manual_seed(0)
    table = torch.randn(V, E, generator=g).to(dev, torch.bfloat16)
    lengths = torch.randint(T // 4, T + 1, (B,), generator=g, dtype=torch.int32).to(dev)
    dx = torch.randn(T * B, E, generator=g).to(dev, torch.bfloat16)
    dW = torch.empty(V, E, dtype=torch.float32, device=dev)
    xb = T * B * E * 2
    out = {"rows": T * B, "V": V, "E": E, "x_MiB": xb / 2 ** 20, "table_grad_MiB": V * E * 4 / 2 ** 20,
           "hbm_gbps_assumed": args.hbm_gbps, "bwd_launches": int(ext().EMBED_BWD_LAUNCHES),
           "fwd_bound_us": 2 * xb / (args.hbm_gbps * 1e3), "bwd_bound_us": (xb + V * E * 4) / (args.hbm_gbps * 1e3)}
    for kind in ("uniform", "zipf"):
        tok = torch.as_tensor(_tokens(kind, B, T, V, 5)).to(dev)
        out[kind] = {"fwd_us": _timed(lambda: ext().embed_fwd(table, tok, lengths), reps, 10) * 1e3,
                     "bwd_us": _timed(lambda: ext().embed_bwd(dx, tok, lengths, dW, False), reps, 10) * 1e3}
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--hidden_units", default="1024,1024")
    ap.add_argument("--in_features", type=int, default=1024)
    ap.add_argument("--vocab_size", type=int, default=32768)
    ap.add_argument("--seq_len", type=int, default=128)
    ap.add_argument("--batch_size", type=int, default=256)
    ap.add_argument("--num_classes", type=int, default=10)
    ap.add_argument("--cuda_graph", type=int, default=1)
    ap.add_argument("--hbm_gbps", type=float, default=3350.0, help="HBM bandwidth for the computed bound (H100 SXM: 3.35 TB/s)")
    ap.add_argument("--no_baseline", action="store_true")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    from lstm_tensorspark_b200 import data as Dm
    n, T, V = 4 * args.batch_size, args.seq_len, args.vocab_size
    xf, yf = Dm.synthetic_sequences(n, T, args.in_features, args.num_classes, seed=1234)
    ls = Dm.synthetic_lengths(n, T, 1234)
    out = {"metric": "samples/sec", "unit": "samples/s", "n_gpus": 1, "steps": args.steps, "warmup": args.warmup,
           "card": _card(), "dtype": "bf16",
           "config": {"hidden_units": args.hidden_units, "in_features": args.in_features, "vocab_size": V, "seq_len": T,
                      "batch_size": args.batch_size, "num_classes": args.num_classes},
           "lengths": {"min": int(ls.min()), "mean": float(ls.mean()), "max": int(ls.max())}}
    out["embed_kernels"] = embed_kernels(args, dev)
    for kind in ("uniform", "zipf"):
        tok = _tokens(kind, n, T, V, 77)
        torch.cuda.empty_cache()
        out[f"ours_{kind}"] = ours(args, tok, yf, None, dev, V)
        torch.cuda.empty_cache()
        out[f"ours_{kind}_variable_length"] = ours(args, tok, yf, ls, dev, V)
    torch.cuda.empty_cache()
    out["ours_dense"] = ours(args, xf, yf, None, dev, 0)
    out["table_step_cost_ms"] = out["ours_uniform"]["ms_per_step"] - out["ours_dense"]["ms_per_step"]
    if not args.no_baseline:
        torch.cuda.empty_cache()
        out["cudnn_embedding"] = cudnn(args, _tokens("uniform", n, T, V, 77), yf, dev)
    out["value"], out["ms_per_step"] = out["ours_uniform"]["value"], out["ours_uniform"]["ms_per_step"]
    print(json.dumps(out))


if __name__ == "__main__":
    sys.exit(main())
