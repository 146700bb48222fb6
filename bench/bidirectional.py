"""Training throughput of bidirectional layers (one GPU): the headline model (2-layer-1024 LSTM, T = 128, B = 256, D = 1024, bf16,
Adam, CUDA graph) with ``--bidirectional``, on fixed-length and on ragged synthetic batches.

    python bench/bidirectional.py --steps 50 --warmup 10

Arms, each device-timed with CUDA events around ``--steps`` steps after ``--warmup`` steps:
  * ``ours``: ``TrainEngine.step(x, y)`` with ``bidirectional=True``, the step captured as a CUDA graph on each of the 4 rotating
    device batches;
  * ``cudnn``: the stand-in of ``baseline/harness.py`` (``variant="tuned"``: bf16 ``nn.LSTM`` weights, fp32 masters + fused Adam,
    CUDA graph) with ``bidirectional=True``, classifying ``[h_n[-2] | h_n[-1]]`` like our model;
  * ``ours_variable_length`` / ``packed_cudnn``: the same on batches with lengths drawn from ``[T // 4, T]``, against cuDNN on
    ``pack_padded_sequence`` (eager: packing takes host lengths), as in ``bench/variable_length.py``.
Prints one JSON line, with the card's name and power limit.  The two directions of a layer run one after the other.
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

from variable_length import _card, _timed, ours, packed_cudnn     # noqa: E402  (the shared arms and helpers)


def cudnn_fixed(args, xs, ys, dev):
    from baseline import harness
    B, nb = args.batch_size, 4
    hidden = [int(h) for h in args.hidden_units.split(",")]
    runner = harness.BaselineRunner(hidden, args.in_features, args.num_classes, B, args.seq_len, 0, 1, dev, variant="tuned",
                                    bidirectional=True)
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


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--hidden_units", default="1024,1024")
    ap.add_argument("--in_features", type=int, default=1024)
    ap.add_argument("--seq_len", type=int, default=128)
    ap.add_argument("--batch_size", type=int, default=256)
    ap.add_argument("--num_classes", type=int, default=10)
    ap.add_argument("--cuda_graph", type=int, default=1)
    ap.add_argument("--variable_length", type=int, default=1, help="also time ragged batches (and packed cuDNN)")
    ap.add_argument("--no_baseline", action="store_true")
    args = ap.parse_args()
    args.bidirectional = True
    assert torch.cuda.is_available(), "needs a GPU"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    from lstm_tensorspark_b200 import data as Dm
    xs, ys, ls = Dm.synthetic_sequences(4 * args.batch_size, args.seq_len, args.in_features, args.num_classes, seed=1234,
                                        variable_length=True)
    xf, yf = Dm.synthetic_sequences(4 * args.batch_size, args.seq_len, args.in_features, args.num_classes, seed=1234)
    out = {"metric": "samples/sec", "unit": "samples/s", "n_gpus": 1, "steps": args.steps, "warmup": args.warmup,
           "card": _card(), "dtype": "bf16", "bidirectional": True,
           "config": {"hidden_units": args.hidden_units, "in_features": args.in_features, "seq_len": args.seq_len,
                      "batch_size": args.batch_size, "num_classes": args.num_classes}}
    out["ours"] = ours(args, xf, yf, None, dev)
    out["value"], out["ms_per_step"] = out["ours"]["value"], out["ours"]["ms_per_step"]
    if not args.no_baseline:
        torch.cuda.empty_cache()
        out["cudnn"] = cudnn_fixed(args, xf, yf, dev)
        out["vs_cudnn"] = out["value"] / out["cudnn"]["value"]
    if args.variable_length:
        torch.cuda.empty_cache()
        out["lengths"] = {"min": int(ls.min()), "mean": float(ls.mean()), "max": int(ls.max())}
        out["ours_variable_length"] = ours(args, xs, ys, ls, dev)
        if not args.no_baseline:
            torch.cuda.empty_cache()
            out["packed_cudnn"] = packed_cudnn(args, xs, ys, ls, dev)
            out["variable_length_vs_packed_cudnn"] = out["ours_variable_length"]["value"] / out["packed_cudnn"]["value"]
    print(json.dumps(out))


if __name__ == "__main__":
    sys.exit(main())
