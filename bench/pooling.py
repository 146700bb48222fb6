"""Training throughput of sequence classification from a pooled summary of every time step (one GPU): the headline model
(2-layer-1024 LSTM, T = 128, B = 256, D = 1024, bf16, Adam, CUDA graph) with ``--pooling last | mean | max | attention``
(A = 128), on fixed-length and on ragged synthetic batches (lengths in [T // 4, T]).

    python bench/pooling.py --steps 50 --warmup 10

Arms, each device-timed with CUDA events around ``--steps`` steps after ``--warmup`` steps:
  * ``ours_<mode>`` / ``ours_<mode>_variable_length``: ``TrainEngine.step`` with ``pooling=<mode>``, the step captured as a CUDA
    graph on each of the 4 rotating device batches;
  * ``cudnn_<mode>``: the stand-in of ``baseline/harness.py`` (``variant="tuned"``: bf16 ``nn.LSTM`` weights, fp32 masters + fused
    Adam, CUDA graph) with ``pooling=<mode>``: ``nn.LSTM`` + pool + ``nn.Linear``, fixed-length batches;
  * ``pool_kernels``: the pooling launches alone at the headline shape (``h_seq`` [T·B, H] bf16, ragged lengths): forward and
    backward device time per mode (attention: its GEMMs included), next to the bandwidth bound computed from the shapes at
    ``--hbm_gbps`` (computed, not measured).
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

import torch

from variable_length import _card, _timed     # noqa: E402  (the shared helpers)

MODES = ("last", "mean", "max", "attention")


def ours(args, mode, xs, ys, ls, dev):
    from lstm_tensorspark_b200.config import Config
    from lstm_tensorspark_b200.engine import TrainEngine
    from lstm_tensorspark_b200.ops import cuda_lstm
    B, T, D, C, nb = args.batch_size, args.seq_len, args.in_features, args.num_classes, 4
    cfg = Config(hidden_units=args.hidden_units, in_features=D, seq_len=T, batch_size=B, num_classes=C, partitions=1,
                 sync_mode="none", init="scaled", learn_initial_state=False, dtype="bf16", device="cuda", learning_rate=1e-3,
                 quiet=True, variable_length=ls is not None, pooling=mode, attention_units=args.attention_units)
    eng = TrainEngine(cfg, 0, 1, None, batch_size=B, device=dev, dtype=torch.bfloat16)
    dx = torch.as_tensor(xs).to(dev, torch.bfloat16)
    dy = torch.as_tensor(ys).to(dev)
    dl = None if ls is None else torch.as_tensor(ls).to(dev)
    batches = [(dx[i * B:(i + 1) * B], dy[i * B:(i + 1) * B], None if dl is None else dl[i * B:(i + 1) * B]) for i in range(nb)]
    n_pool = cuda_lstm.STATS.get("pool_fwd", 0)
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
            "pool_launched": cuda_lstm.STATS.get("pool_fwd", 0) > n_pool,
            "pipelined": cuda_lstm.STATS.get("pipelined_fwd", 0) > 0}


def cudnn(args, mode, xs, ys, dev):
    from baseline import harness
    B, nb = args.batch_size, 4
    hidden = [int(h) for h in args.hidden_units.split(",")]
    runner = harness.BaselineRunner(hidden, args.in_features, args.num_classes, B, args.seq_len, 0, 1, dev, variant="tuned",
                                    pooling=mode)
    dx = torch.as_tensor(xs).to(dev, torch.bfloat16)
    dy = torch.as_tensor(ys).to(dev)
    batches = [(dx[i * B:(i + 1) * B], dy[i * B:(i + 1) * B]) for i in range(nb)]
    graphed = runner.capture(*batches[0], bind=batches)
    it = {"i": 0}

    def step():
        runner.train_step(*batches[it["i"] % nb])
        it["i"] += 1
    ms = _timed(step, args.steps, args.warmup)
    return {"ms_per_step": ms, "value": B * 1e3 / ms, "cuda_graph": graphed}


def pool_kernels(args, dev, reps=100):
    """Device time of the pooling op alone (forward; backward = forward + backward minus forward) per mode at this shape, and
    the bytes each must move at least: forward reads h_seq once (attention: plus u written and read back, alpha); backward
    writes dh_seq (attention: reads h_seq again, u, writes dU and reads it twice, writes and reads G = dU W_a^T in fp32)."""
    from lstm_tensorspark_b200.ops import functional as F
    B, T, A = args.batch_size, args.seq_len, args.attention_units
    H = int(args.hidden_units.split(",")[-1])
    g = torch.Generator(device="cpu").manual_seed(0)
    h = torch.randn(T, B, H, generator=g).to(dev, torch.bfloat16).requires_grad_(True)
    lengths = torch.randint(T // 4, T + 1, (B,), generator=g, dtype=torch.int32).to(dev)
    att = tuple(t.to(dev).requires_grad_(True) for t in (torch.randn(H, A, generator=g) / H ** 0.5, torch.zeros(A),
                                                           torch.randn(A, generator=g) / A ** 0.5))
    ds = torch.randn(B, H, generator=g).to(dev)
    hs, ss = T * B * H * 2, B * H * 4
    out = {"rows": T * B, "H": H, "A": A, "h_seq_MiB": hs / 2 ** 20, "hbm_gbps_assumed": args.hbm_gbps}
    for mode in MODES[1:]:
        a = att if mode == "attention" else None
        fwd = lambda: F.pool_sequence(h, lengths, mode, a)
        both = lambda: torch.autograd.grad(F.pool_sequence(h, lengths, mode, a), (h,) + (a or ()), ds)
        f_us = _timed(fwd, reps, 10) * 1e3
        fb_us = _timed(both, reps, 10) * 1e3
        if mode == "attention":
            u = T * B * A * 4
            fwd_bytes = 2 * hs + 2 * u + ss
            bwd_bytes = 2 * hs + 2 * u + 3 * T * B * A * 2 + 2 * T * B * H * 4 + hs
        else:
            fwd_bytes, bwd_bytes = hs + ss + (ss if mode == "max" else 0), hs + ss + (ss if mode == "max" else 0)
        out[mode] = {"fwd_us": f_us, "bwd_us": fb_us - f_us,
                     "fwd_bound_us": fwd_bytes / (args.hbm_gbps * 1e3), "bwd_bound_us": bwd_bytes / (args.hbm_gbps * 1e3)}
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--hidden_units", default="1024,1024")
    ap.add_argument("--in_features", type=int, default=1024)
    ap.add_argument("--seq_len", type=int, default=128)
    ap.add_argument("--batch_size", type=int, default=256)
    ap.add_argument("--num_classes", type=int, default=10)
    ap.add_argument("--attention_units", type=int, default=128)
    ap.add_argument("--cuda_graph", type=int, default=1)
    ap.add_argument("--hbm_gbps", type=float, default=3350.0, help="HBM bandwidth for the computed bound (H100 SXM: 3.35 TB/s)")
    ap.add_argument("--no_baseline", action="store_true")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    from lstm_tensorspark_b200 import data as Dm
    n = 4 * args.batch_size
    xf, yf = Dm.synthetic_sequences(n, args.seq_len, args.in_features, args.num_classes, seed=1234)
    xs, ys, ls = Dm.synthetic_sequences(n, args.seq_len, args.in_features, args.num_classes, seed=1234, variable_length=True)
    out = {"metric": "samples/sec", "unit": "samples/s", "n_gpus": 1, "steps": args.steps, "warmup": args.warmup,
           "card": _card(), "dtype": "bf16",
           "config": {"hidden_units": args.hidden_units, "in_features": args.in_features, "seq_len": args.seq_len,
                      "batch_size": args.batch_size, "num_classes": args.num_classes, "attention_units": args.attention_units},
           "lengths": {"min": int(ls.min()), "mean": float(ls.mean()), "max": int(ls.max())}}
    out["pool_kernels"] = pool_kernels(args, dev)
    for mode in MODES:
        torch.cuda.empty_cache()
        out[f"ours_{mode}"] = ours(args, mode, xf, yf, None, dev)
        torch.cuda.empty_cache()
        out[f"ours_{mode}_variable_length"] = ours(args, mode, xs, ys, ls, dev)
        if not args.no_baseline:
            torch.cuda.empty_cache()
            out[f"cudnn_{mode}"] = cudnn(args, mode, xf, yf, dev)
    out["value"], out["ms_per_step"] = out["ours_attention"]["value"], out["ours_attention"]["ms_per_step"]
    print(json.dumps(out))


if __name__ == "__main__":
    sys.exit(main())
