"""Training throughput with a label at every time step (one GPU): the headline model (2-layer-1024 LSTM, T = 128, B = 256, D = 1024,
bf16, Adam, CUDA graph) with ``--per_step_labels``, on fixed-length and on ragged synthetic batches.

    python bench/per_step_labels.py --steps 50 --warmup 10

Arms, each device-timed with CUDA events around ``--steps`` steps after ``--warmup`` steps:
  * ``ours``: ``TrainEngine.step(x, y)`` with ``per_step_labels=True`` and ``y [B,T]``, the step captured as a CUDA graph on each of
    the 4 rotating device batches;
  * ``ours_variable_length``: the same on batches with lengths drawn from ``[T // 4, T]`` (loss over the real positions);
  * ``cudnn``: the stand-in of ``baseline/harness.py`` (``variant="tuned"``: bf16 ``nn.LSTM`` weights, fp32 masters + fused Adam,
    CUDA graph) with ``per_step=True``: ``nn.Linear`` over every output, cross-entropy over all ``T·B`` positions;
  * ``packed_cudnn``: cuDNN on ``pack_padded_sequence`` of the ragged batches with the head applied to ``packed.data`` (eager:
    packing takes host lengths);
  * ``head_kernels``: the per-step head's forward and backward launches alone (each includes its small scratch allocations).
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


def ours(args, xs, ys, ls, dev):
    from lstm_tensorspark_b200.config import Config
    from lstm_tensorspark_b200.engine import TrainEngine
    from lstm_tensorspark_b200.ops import cuda_lstm
    B, T, D, C, nb = args.batch_size, args.seq_len, args.in_features, args.num_classes, 4
    cfg = Config(hidden_units=args.hidden_units, in_features=D, seq_len=T, batch_size=B, num_classes=C, partitions=1,
                 sync_mode="none", init="scaled", learn_initial_state=False, dtype="bf16", device="cuda", learning_rate=1e-3,
                 quiet=True, variable_length=ls is not None, per_step_labels=True)
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
            "head_per_step_tc": cuda_lstm.STATS.get("head_per_step_tc", 0) > 0,
            "pipelined": cuda_lstm.STATS.get("pipelined_fwd", 0) > 0, "wavefront": cuda_lstm.STATS.get("wavefront_fwd", 0) > 0}


def cudnn_fixed(args, xs, ys, dev):
    from baseline import harness
    B, nb = args.batch_size, 4
    hidden = [int(h) for h in args.hidden_units.split(",")]
    runner = harness.BaselineRunner(hidden, args.in_features, args.num_classes, B, args.seq_len, 0, 1, dev, variant="tuned",
                                    per_step=True)
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


def packed_cudnn(args, xs, ys, ls, dev):
    import torch.nn as nn
    import torch.nn.functional as Fn
    from torch.nn.utils.rnn import pack_padded_sequence
    B, T, D, C, nb = args.batch_size, args.seq_len, args.in_features, args.num_classes, 4
    hidden = [int(h) for h in args.hidden_units.split(",")]
    torch.manual_seed(0)
    lstm = nn.LSTM(D, hidden[0], num_layers=len(hidden), device=dev, dtype=torch.bfloat16)
    lstm.flatten_parameters()
    head = nn.Linear(hidden[-1], C, device=dev, dtype=torch.bfloat16)
    params = list(lstm.parameters()) + list(head.parameters())
    masters = [p.detach().float().clone().requires_grad_(True) for p in params]
    for m in masters:
        m.grad = torch.zeros_like(m)
    opt = torch.optim.Adam(masters, lr=1e-3, fused=True)
    dx = torch.as_tensor(xs).to(dev, torch.bfloat16).transpose(0, 1)            # time-major view [T, nb*B, D]
    dy = torch.as_tensor(ys).to(dev).t()                                        # [T, nb*B]
    lens = [torch.as_tensor(ls[i * B:(i + 1) * B]).long() for i in range(nb)]   # host lengths, as packing wants them
    # the labels in packed order, once per batch (packing the labels the same way as the inputs)
    ylab = [pack_padded_sequence(dy[:, i * B:(i + 1) * B], lens[i], enforce_sorted=False).data for i in range(nb)]
    it = {"i": 0}

    def step():
        i = it["i"] % nb
        it["i"] += 1
        for p in params:
            p.grad = None
        out, _ = lstm(pack_padded_sequence(dx[:, i * B:(i + 1) * B], lens[i], enforce_sorted=False))
        loss = Fn.cross_entropy(head(out.data).float(), ylab[i])
        loss.backward()
        with torch.no_grad():
            torch._foreach_copy_([m.grad for m in masters], [p.grad for p in params])       # bf16 grads -> fp32 masters
        opt.step()
        with torch.no_grad():
            torch._foreach_copy_(params, masters)
    ms = _timed(step, args.steps, args.warmup)
    return {"ms_per_step": ms, "value": B * 1e3 / ms, "cuda_graph": False,
            "note": "pack_padded_sequence(enforce_sorted=False) takes host lengths: eager, not capturable"}


def head_kernels(args, dev, reps=200):
    """Device time of the per-step head alone at this shape (ragged lengths): the forward launch and the backward launch, each
    averaged over ``reps`` back-to-back launches between CUDA events."""
    from lstm_tensorspark_b200.ops.cuda_ext import ext
    E = ext()
    B, T, C = args.batch_size, args.seq_len, args.num_classes
    H = int(args.hidden_units.split(",")[-1])
    g = torch.Generator(device="cpu").manual_seed(0)
    h = torch.randn(T * B, H, generator=g).to(dev, torch.bfloat16)
    W = (torch.randn(H, C, generator=g) / H ** 0.5).to(dev)
    b = torch.zeros(C, device=dev)
    y = torch.randint(0, C, (B, T), generator=g).to(dev)
    lengths = torch.randint(T // 4, T + 1, (B,), generator=g, dtype=torch.int32).to(dev)
    dW, db = torch.empty_like(W), torch.empty_like(b)
    dloss = torch.ones(1, device=dev)
    fwd = lambda: E.head_step_fwd(h, W, b, y, lengths, T)
    dlogits = fwd()[1]
    bwd = lambda: E.head_step_bwd(h, W, dlogits, dloss, dW, db, False, False)
    return {"rows": T * B, "H": H, "C": C, "fwd_us": _timed(fwd, reps, 10) * 1e3, "bwd_us": _timed(bwd, reps, 10) * 1e3}


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
    assert torch.cuda.is_available(), "needs a GPU"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    from lstm_tensorspark_b200 import data as Dm
    n = 4 * args.batch_size
    xf, yf = Dm.synthetic_per_step(n, args.seq_len, args.in_features, args.num_classes, seed=1234)
    out = {"metric": "samples/sec", "unit": "samples/s", "n_gpus": 1, "steps": args.steps, "warmup": args.warmup,
           "card": _card(), "dtype": "bf16", "per_step_labels": True,
           "config": {"hidden_units": args.hidden_units, "in_features": args.in_features, "seq_len": args.seq_len,
                      "batch_size": args.batch_size, "num_classes": args.num_classes}}
    out["head_kernels"] = head_kernels(args, dev)
    out["ours"] = ours(args, xf, yf, None, dev)
    out["value"], out["ms_per_step"] = out["ours"]["value"], out["ours"]["ms_per_step"]
    if not args.no_baseline:
        torch.cuda.empty_cache()
        out["cudnn"] = cudnn_fixed(args, xf, yf, dev)
        out["vs_cudnn"] = out["value"] / out["cudnn"]["value"]
    if args.variable_length:
        xs, ys, ls = Dm.synthetic_per_step(n, args.seq_len, args.in_features, args.num_classes, seed=1234, variable_length=True)
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
