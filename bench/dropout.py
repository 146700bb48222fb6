"""Training throughput with dropout between the layers (one GPU): the headline model (2-layer-1024 LSTM, T = 128, B = 256,
D = 1024, bf16, Adam, CUDA graph) with ``--dropout 0`` and ``--dropout 0.2``, and the tuned cuDNN stand-in with
``nn.LSTM(dropout=0.2)``.

    python bench/dropout.py --steps 50 --warmup 10

Arms, each device-timed with CUDA events around ``--steps`` steps after ``--warmup`` steps, over 4 rotating device batches:
  * ``ours_p0`` / ``ours``: ``TrainEngine.step(x, y)`` with ``dropout`` 0 / ``--dropout``, the step captured as a CUDA graph on
    each batch (the mask's step counter advances inside the graph);
  * ``cudnn``: ``baseline/harness.py`` (``variant="tuned"``: bf16 ``nn.LSTM`` weights, fp32 masters + fused Adam, CUDA graph when
    the capture succeeds) with ``dropout=--dropout``.
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

from variable_length import _card, _timed     # noqa: E402  (the shared timing helpers)


def ours(args, p, xs, ys, dev):
    from lstm_tensorspark_b200.config import Config
    from lstm_tensorspark_b200.engine import TrainEngine
    from lstm_tensorspark_b200.ops import cuda_lstm
    B, T, D, C, nb = args.batch_size, args.seq_len, args.in_features, args.num_classes, 4
    cfg = Config(hidden_units=args.hidden_units, in_features=D, seq_len=T, batch_size=B, num_classes=C, partitions=1,
                 sync_mode="none", init="scaled", learn_initial_state=False, dtype="bf16", device="cuda", learning_rate=1e-3,
                 quiet=True, dropout=p)
    eng = TrainEngine(cfg, 0, 1, None, batch_size=B, device=dev, dtype=torch.bfloat16)
    dx = torch.as_tensor(xs).to(dev, torch.bfloat16)
    dy = torch.as_tensor(ys).to(dev)
    batches = [(dx[i * B:(i + 1) * B], dy[i * B:(i + 1) * B]) for i in range(nb)]
    eng.step(*batches[0])
    eng.capture(*batches[0], bind=batches[1:])
    it = {"i": 0}

    def step():
        eng.step(*batches[it["i"] % nb])
        it["i"] += 1
    ms = _timed(step, args.steps, args.warmup)
    cuda_lstm.check_kernel_errors(dev)
    return {"ms_per_step": ms, "value": B * 1e3 / ms, "dropout": p}


def cudnn(args, xs, ys, dev):
    from baseline import harness
    B, nb = args.batch_size, 4
    hidden = [int(h) for h in args.hidden_units.split(",")]
    runner = harness.BaselineRunner(hidden, args.in_features, args.num_classes, B, args.seq_len, 0, 1, dev, variant="tuned",
                                    dropout=args.dropout)
    dx = torch.as_tensor(xs).to(dev, torch.bfloat16)
    dy = torch.as_tensor(ys).to(dev)
    batches = [(dx[i * B:(i + 1) * B], dy[i * B:(i + 1) * B]) for i in range(nb)]
    graphed = runner.capture(*batches[0], bind=batches)
    it = {"i": 0}

    def step():
        runner.train_step(*batches[it["i"] % nb])
        it["i"] += 1
    ms = _timed(step, args.steps, args.warmup)
    return {"ms_per_step": ms, "value": B * 1e3 / ms, "dropout": args.dropout, "cuda_graph": graphed,
            "capture_error": getattr(runner, "capture_error", None)}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--dropout", type=float, default=0.2)
    ap.add_argument("--hidden_units", default="1024,1024")
    ap.add_argument("--in_features", type=int, default=1024)
    ap.add_argument("--seq_len", type=int, default=128)
    ap.add_argument("--batch_size", type=int, default=256)
    ap.add_argument("--num_classes", type=int, default=10)
    ap.add_argument("--no_baseline", action="store_true")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    from lstm_tensorspark_b200 import data as Dm
    xs, ys = Dm.synthetic_sequences(4 * args.batch_size, args.seq_len, args.in_features, args.num_classes, seed=1234)
    out = {"metric": "samples/sec", "unit": "samples/s", "n_gpus": 1, "steps": args.steps, "warmup": args.warmup,
           "card": _card(), "dtype": "bf16", "dropout": args.dropout,
           "config": {"hidden_units": args.hidden_units, "in_features": args.in_features, "seq_len": args.seq_len,
                      "batch_size": args.batch_size, "num_classes": args.num_classes}}
    out["ours_p0"] = ours(args, 0.0, xs, ys, dev)
    torch.cuda.empty_cache()
    out["ours"] = ours(args, args.dropout, xs, ys, dev)
    out["value"], out["ms_per_step"] = out["ours"]["value"], out["ours"]["ms_per_step"]
    out["cost_vs_p0"] = out["ours"]["ms_per_step"] / out["ours_p0"]["ms_per_step"] - 1.0
    if not args.no_baseline:
        torch.cuda.empty_cache()
        out["cudnn"] = cudnn(args, xs, ys, dev)
        out["vs_cudnn"] = out["value"] / out["cudnn"]["value"]
    print(json.dumps(out))


if __name__ == "__main__":
    sys.exit(main())
