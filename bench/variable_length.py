"""Training throughput on variable-length samples (one GPU): the headline model (2-layer-1024 LSTM, T = 128, B = 256, bf16, Adam)
on ragged synthetic batches, against cuDNN on ``pack_padded_sequence``.

    python bench/variable_length.py --steps 50 --warmup 10

Lengths are drawn uniformly from ``[T // 4, T]`` (``data.synthetic_sequences(variable_length=True)``), inputs are right-padded with
zeros.  Our arm is ``TrainEngine.step(x, y, lengths)`` with the step captured as a CUDA graph on each of the 4 rotating device
batches; the bar is ``torch.nn.LSTM`` (cuDNN, bf16 weights, fp32 master copies + fused Adam) on
``pack_padded_sequence(enforce_sorted=False)`` of the same batches, reading ``h_n`` of the top layer.  Packing takes the lengths on
the host, so that arm runs eagerly: it cannot be captured in a CUDA graph.  Both are device-timed with CUDA events around
``--steps`` steps after ``--warmup`` steps.  Prints one JSON line, with the card's name and power limit.

Our persistent kernels run every sample for all T steps (padded steps hold the state), while cuDNN's packed mode skips the padding.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np
import torch


def _timed(step, steps, warmup):
    for _ in range(warmup):
        step()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        step()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def _card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        return r.stdout.strip()
    except Exception as e:                                  # noqa: BLE001
        return f"unavailable ({e!r})"


def ours(args, xs, ys, ls, dev):
    """``ls`` None: fixed-length batches.  ``args.bidirectional`` (absent = False): bench/bidirectional.py."""
    from lstm_tensorspark_b200.config import Config
    from lstm_tensorspark_b200.engine import TrainEngine
    from lstm_tensorspark_b200.ops import cuda_lstm
    B, T, D, C, nb = args.batch_size, args.seq_len, args.in_features, args.num_classes, 4
    cfg = Config(hidden_units=args.hidden_units, in_features=D, seq_len=T, batch_size=B, num_classes=C, partitions=1,
                 sync_mode="none", init="scaled", learn_initial_state=False, dtype="bf16", device="cuda", learning_rate=1e-3,
                 quiet=True, variable_length=ls is not None, bidirectional=getattr(args, "bidirectional", False))
    eng = TrainEngine(cfg, 0, 1, None, batch_size=B, device=dev, dtype=torch.bfloat16)
    dx = torch.as_tensor(xs).to(dev, torch.bfloat16)
    dy = torch.as_tensor(ys).to(dev)
    dl = None if ls is None else torch.as_tensor(ls).to(dev)
    batches = [(dx[i * B:(i + 1) * B], dy[i * B:(i + 1) * B], None if dl is None else dl[i * B:(i + 1) * B]) for i in range(nb)]
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
            "fast_path": cuda_lstm.STATS["fast_fwd"] > 0, "generic_path": cuda_lstm.STATS["generic_fwd"] > 0,
            "wavefront": cuda_lstm.STATS.get("wavefront_fwd", 0) > 0}


def packed_cudnn(args, xs, ys, ls, dev):
    import torch.nn as nn
    import torch.nn.functional as Fn
    from torch.nn.utils.rnn import pack_padded_sequence
    B, T, D, C, nb = args.batch_size, args.seq_len, args.in_features, args.num_classes, 4
    hidden = [int(h) for h in args.hidden_units.split(",")]
    bidir = getattr(args, "bidirectional", False)
    torch.manual_seed(0)
    lstm = nn.LSTM(D, hidden[0], num_layers=len(hidden), device=dev, dtype=torch.bfloat16,     # weights in one cuDNN buffer
                   bidirectional=bidir)
    lstm.flatten_parameters()
    head = nn.Linear(hidden[-1] * (2 if bidir else 1), C, device=dev, dtype=torch.bfloat16)
    params = list(lstm.parameters()) + list(head.parameters())
    masters = [p.detach().float().clone().requires_grad_(True) for p in params]
    for m in masters:
        m.grad = torch.zeros_like(m)
    opt = torch.optim.Adam(masters, lr=1e-3, fused=True)
    dx = torch.as_tensor(xs).to(dev, torch.bfloat16).transpose(0, 1)            # time-major view [T, nb*B, D]
    dy = torch.as_tensor(ys).to(dev)
    lens = [torch.as_tensor(ls[i * B:(i + 1) * B]).long() for i in range(nb)]   # host lengths, as packing wants them
    it = {"i": 0}

    def step():
        i = it["i"] % nb
        it["i"] += 1
        for p in params:
            p.grad = None
        _, (h_n, _) = lstm(pack_padded_sequence(dx[:, i * B:(i + 1) * B], lens[i], enforce_sorted=False))
        feat = torch.cat([h_n[-2], h_n[-1]], 1) if bidir else h_n[-1]
        loss = Fn.cross_entropy(head(feat).float(), dy[i * B:(i + 1) * B])
        loss.backward()
        with torch.no_grad():
            torch._foreach_copy_([m.grad for m in masters], [p.grad for p in params])       # bf16 grads -> fp32 masters
        opt.step()
        with torch.no_grad():
            torch._foreach_copy_(params, masters)
    ms = _timed(step, args.steps, args.warmup)
    return {"ms_per_step": ms, "value": B * 1e3 / ms, "cuda_graph": False,
            "note": "pack_padded_sequence(enforce_sorted=False) takes host lengths: eager, not capturable"}


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
    ap.add_argument("--no_baseline", action="store_true")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    from lstm_tensorspark_b200 import data as Dm
    xs, ys, ls = Dm.synthetic_sequences(4 * args.batch_size, args.seq_len, args.in_features, args.num_classes, seed=1234,
                                        variable_length=True)
    out = {"metric": "samples/sec", "unit": "samples/s", "n_gpus": 1, "steps": args.steps, "warmup": args.warmup,
           "card": _card(), "dtype": "bf16",
           "config": {"hidden_units": args.hidden_units, "in_features": args.in_features, "seq_len": args.seq_len,
                      "batch_size": args.batch_size, "num_classes": args.num_classes},
           "lengths": {"min": int(ls.min()), "mean": float(ls.mean()), "max": int(ls.max())}}
    out["ours"] = ours(args, xs, ys, ls, dev)
    out["value"], out["ms_per_step"] = out["ours"]["value"], out["ours"]["ms_per_step"]
    if not args.no_baseline:
        torch.cuda.empty_cache()
        out["packed_cudnn"] = packed_cudnn(args, xs, ys, ls, dev)
        out["vs_packed_cudnn"] = out["value"] / out["packed_cudnn"]["value"]
    print(json.dumps(out))


if __name__ == "__main__":
    sys.exit(main())
