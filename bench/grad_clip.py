"""Cost of clipping the gradient by its global norm (one GPU): the headline model (2-layer-1024 LSTM, T = 128, B = 256, D = 1024,
bf16, Adam, CUDA graph) without and with ``--clip_grad_norm 1e-6``, and the norm kernel alone.  The clip is active: with the
``scaled`` init the headline gradient's norm is about 1e-5, so a limit of 1.0 would never clip (the cost is the same either way:
the norm kernel runs and the update reads coef every step).

    python bench/grad_clip.py --steps 50 --warmup 10

  * ``no_clip`` / ``clip``: ``TrainEngine.step`` replaying the captured step on 4 rotating device batches, device-timed with CUDA
    events around ``--steps`` steps after ``--warmup``; the two arms alternate over ``--runs`` runs (other work shares the host);
  * ``norm_kernel``: ``flat_grad_norm`` alone over the headline flat buffer, CUDA events around ``--launches`` back-to-back launches,
    against the bound of its bytes (the fp32 gradient read once; the weights are not read without weight decay) at the data
    sheet's 3.35 TB/s of HBM3.
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

HBM3_BYTES_PER_S = 3.35e12                     # H100 SXM data sheet


def engine(args, clip, dev):
    from lstm_tensorspark_b200.config import Config
    from lstm_tensorspark_b200.engine import TrainEngine
    cfg = Config(hidden_units=args.hidden_units, in_features=args.in_features, seq_len=args.seq_len, batch_size=args.batch_size,
                 num_classes=args.num_classes, partitions=1, sync_mode="none", init="scaled", learn_initial_state=False,
                 dtype="bf16", device="cuda", learning_rate=1e-3, quiet=True, clip_grad_norm=clip).validate()
    return TrainEngine(cfg, 0, 1, None, batch_size=args.batch_size, device=dev, dtype=torch.bfloat16)


def timed_arm(args, eng, batches):
    it = {"i": 0}

    def step():
        eng.step(*batches[it["i"] % len(batches)])
        it["i"] += 1
    return _timed(step, args.steps, args.warmup)


def norm_kernel(args, n, dev):
    from lstm_tensorspark_b200.ops.cuda_ext import ext
    E = ext()
    g = torch.randn(n, device=dev)
    p = torch.randn(n, device=dev)
    out = torch.zeros(2, device=dev)
    scratch = torch.zeros(E.flat_grad_norm_scratch(n), dtype=torch.float64, device=dev)
    for _ in range(10):
        E.flat_grad_norm(g, p, out, scratch, 1.0)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.launches):
        E.flat_grad_norm(g, p, out, scratch, 1.0)
    e1.record()
    torch.cuda.synchronize()
    us = e0.elapsed_time(e1) * 1e3 / args.launches
    bound_us = 4 * n / HBM3_BYTES_PER_S * 1e6
    return {"n": n, "bytes": 4 * n, "us_per_launch": us, "bound_us": bound_us, "share_of_bound": bound_us / us,
            "achieved_GB_per_s": 4 * n / (us * 1e-6) / 1e9}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--launches", type=int, default=100)
    ap.add_argument("--clip", type=float, default=1e-6)
    ap.add_argument("--hidden_units", default="1024,1024")
    ap.add_argument("--in_features", type=int, default=1024)
    ap.add_argument("--seq_len", type=int, default=128)
    ap.add_argument("--batch_size", type=int, default=256)
    ap.add_argument("--num_classes", type=int, default=10)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    from lstm_tensorspark_b200 import data as Dm
    B, nb = args.batch_size, 4
    xs, ys = Dm.synthetic_sequences(nb * B, args.seq_len, args.in_features, args.num_classes, seed=1234)
    dx = torch.as_tensor(xs).to(dev, torch.bfloat16)
    dy = torch.as_tensor(ys).to(dev)
    batches = [(dx[i * B:(i + 1) * B], dy[i * B:(i + 1) * B]) for i in range(nb)]
    arms = {"no_clip": engine(args, 0.0, dev), "clip": engine(args, args.clip, dev)}
    for eng in arms.values():
        eng.step(*batches[0])
        eng.capture(*batches[0], bind=batches[1:])
    times = {k: [] for k in arms}
    for _ in range(args.runs):
        for name, eng in arms.items():
            times[name].append(timed_arm(args, eng, batches))
    clip_eng = arms["clip"]
    coef = float(clip_eng.optimizer.clip_out[1])
    out = {"metric": "ms/step", "unit": "ms", "n_gpus": 1, "steps": args.steps, "warmup": args.warmup, "runs": args.runs,
           "card": _card(), "dtype": "bf16",
           "config": {"hidden_units": args.hidden_units, "in_features": args.in_features, "seq_len": args.seq_len,
                      "batch_size": B, "num_classes": args.num_classes, "optimizer": "adam", "cuda_graph": True},
           "no_clip_ms": times["no_clip"], "clip_ms": times["clip"], "clip_grad_norm": args.clip,
           "last_grad_norm": float(clip_eng.grad_norm()), "last_coef": coef, "clip_active": coef < 1.0,
           "flat_numel": clip_eng.flat.padded_numel}
    del arms, clip_eng
    torch.cuda.empty_cache()
    out["norm_kernel"] = norm_kernel(args, out["flat_numel"], dev)
    print(json.dumps(out))


if __name__ == "__main__":
    sys.exit(main())
