"""Training throughput of next-token language models (``--next_token``, one GPU): the headline model (2-layer-1024 LSTM, T = 128,
B = 256, bf16, Adam, CUDA graph) behind an embedding table and under a softmax over the whole vocabulary, V in {4096, 32768}.

    python bench/next_token.py --steps 30 --warmup 5

Arms, each device-timed with CUDA events around ``--steps`` steps after ``--warmup`` steps:
  * ``ours_V<V>`` / ``ours_V<V>_variable_length``: ``TrainEngine.step`` with ``vocab_size=V, next_token=True`` on batches of the
    synthetic Markov language, fixed-length and ragged (lengths in [T // 4, T]), the step captured as a CUDA graph on each of
    the 4 rotating device batches;
  * ``cudnn_V<V>``: the stand-in of ``baseline/harness.py`` (``variant="tuned"``): ``nn.Embedding`` -> ``nn.LSTM`` -> ``nn.Linear``
    and ``F.cross_entropy`` over every output (it materialises the logits);
  * ``head_op_V<V>``: the large-vocabulary head's launches alone, forward and backward, with the floating-point operations and
    the bytes they need computed from the shapes below, the achieved TFLOP/s and their share of the data sheet's dense bf16
    peak (``--peak_tflops``, H100 SXM at 700 W: 989; a card with a lower power limit reaches less).
Prints one JSON line, with the card's name and power limit.  Needs a GPU; there is no fallback.
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


def ours(args, V, ragged, dev):
    from lstm_tensorspark_b200 import data as Dm
    from lstm_tensorspark_b200.config import Config
    from lstm_tensorspark_b200.engine import TrainEngine
    from lstm_tensorspark_b200.ops import cuda_lstm
    B, T, nb = args.batch_size, args.seq_len, 4
    cfg = Config(hidden_units=args.hidden_units, in_features=args.in_features, seq_len=T, batch_size=B, partitions=1,
                 sync_mode="none", init="scaled", learn_initial_state=False, dtype="bf16", device="cuda", learning_rate=1e-3,
                 quiet=True, variable_length=ragged, vocab_size=V, next_token=True).validate()
    eng = TrainEngine(cfg, 0, 1, None, batch_size=B, device=dev, dtype=torch.bfloat16)
    x, y, *ls = Dm.synthetic_next_token(nb * B, T, V, seed=1234, variable_length=ragged)
    dx, dy = torch.as_tensor(x).to(dev), torch.as_tensor(y).to(dev)
    dl = torch.as_tensor(ls[0]).to(dev) if ragged else None
    batches = [(dx[i * B:(i + 1) * B], dy[i * B:(i + 1) * B], None if dl is None else dl[i * B:(i + 1) * B]) for i in range(nb)]
    n_head = cuda_lstm.STATS.get("vocab_head_bwd", 0)
    eng.step(*batches[0])
    if args.cuda_graph:
        eng.capture(*batches[0][:2], lengths=batches[0][2], bind=batches[1:] if ragged else [b[:2] for b in batches[1:]])
    it = {"i": 0}

    def step():
        it["loss"] = eng.step(*batches[it["i"] % nb])
        it["i"] += 1
    ms = _timed(step, args.steps, args.warmup)
    cuda_lstm.check_kernel_errors(dev)
    return {"ms_per_step": ms, "value": B * 1e3 / ms, "cuda_graph": bool(args.cuda_graph), "loss": float(it["loss"]),
            "vocab_head_launched": cuda_lstm.STATS.get("vocab_head_bwd", 0) > n_head,
            "pipelined": cuda_lstm.STATS.get("pipelined_fwd", 0) > 0}


def cudnn(args, V, dev):
    from baseline import harness
    from lstm_tensorspark_b200 import data as Dm
    B, T, nb = args.batch_size, args.seq_len, 4
    hidden = [int(h) for h in args.hidden_units.split(",")]
    runner = harness.BaselineRunner(hidden, args.in_features, V, B, T, 0, 1, dev, variant="tuned", per_step=True, vocab_size=V)
    x, y = Dm.synthetic_next_token(nb * B, T, V, seed=1234)
    dx, dy = torch.as_tensor(x).to(dev, torch.int64), torch.as_tensor(y).to(dev)
    batches = [(dx[i * B:(i + 1) * B], dy[i * B:(i + 1) * B]) for i in range(nb)]
    graphed = runner.capture(*batches[0], bind=batches)
    it = {"i": 0}

    def step():
        runner.train_step(*batches[it["i"] % nb])
        it["i"] += 1
    ms = _timed(step, args.steps, args.warmup)
    return {"ms_per_step": ms, "value": B * 1e3 / ms, "cuda_graph": graphed}


def head_costs(R, H, C, chunk):
    """What the head needs, from the shapes alone.  Forward: one GEMM, 2·R·H·C operations; it reads h and W (bf16) once per band of
    ``chunk`` rows and writes 16 B per row and 256-class tile.  Backward: the recomputed logits, dh and dW, three such GEMMs;
    per chunk it reads h and W for the recompute, writes and twice reads the bf16 dlogits chunk (a third time for db), reads W
    and writes dh, reads h and reads and writes the fp32 dW."""
    gemm = 2.0 * R * H * C
    bands = (R + chunk - 1) // chunk
    fwd_bytes = R * H * 2 + bands * H * C * 2 + R * ((C + 255) // 256) * 16
    bwd_bytes = bands * (2 * H * C * 2 + 2 * H * C * 4) + R * (2 * H * 2 + H * 2) + R * C * 2 * 4
    return {"fwd_flop": gemm, "bwd_flop": 3.0 * gemm, "fwd_bytes": float(fwd_bytes), "bwd_bytes": float(bwd_bytes)}


def head_op(args, V, dev, reps=10):
    from lstm_tensorspark_b200.ops import cuda_vocab_head
    T, B = args.seq_len, args.batch_size
    H = int(args.hidden_units.split(",")[-1])
    g = torch.Generator(device="cpu").manual_seed(0)
    h = torch.randn(T, B, H, generator=g).to(dev, torch.bfloat16).requires_grad_(True)
    W = (torch.randn(H, V, generator=g) / H ** 0.5).to(dev).requires_grad_(True)
    b = torch.zeros(V, device=dev, requires_grad=True)
    labels = torch.randint(0, V, (B, T), generator=g).to(dev)
    out = {}

    def fwd():
        out["loss"] = cuda_vocab_head.vocab_xent_per_step(h, W, b, labels, None)[0]

    def bwd():
        out["loss"].backward(retain_graph=True)
    fwd_ms = _timed(fwd, reps, 3)
    bwd_ms = _timed(bwd, reps, 3)
    costs = head_costs(T * B, H, V, cuda_vocab_head.ROW_CHUNK)
    res = {"rows": T * B, "H": H, "V": V, "fwd_ms": fwd_ms, "bwd_ms": bwd_ms, **costs,
           "logits_not_stored_GiB": T * B * V * 4 / 2 ** 30, "fp32_dlogits_not_stored_GiB": T * B * V * 4 / 2 ** 30,
           "peak_tflops_assumed": args.peak_tflops, "hbm_gbps_assumed": args.hbm_gbps}
    for k, ms in (("fwd", fwd_ms), ("bwd", bwd_ms)):
        tflops = costs[f"{k}_flop"] / (ms * 1e-3) / 1e12
        least_ms = max(costs[f"{k}_flop"] / (args.peak_tflops * 1e12), costs[f"{k}_bytes"] / (args.hbm_gbps * 1e9)) * 1e3
        res[f"{k}_tflops"] = tflops
        res[f"{k}_share_of_bf16_peak"] = tflops / args.peak_tflops
        res[f"{k}_bound_ms"] = least_ms
        res[f"{k}_bound_by"] = "compute" if costs[f"{k}_flop"] / (args.peak_tflops * 1e12) >= costs[f"{k}_bytes"] / (args.hbm_gbps * 1e9) \
            else "memory"
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--hidden_units", default="1024,1024")
    ap.add_argument("--in_features", type=int, default=1024)
    ap.add_argument("--vocab_sizes", default="4096,32768")
    ap.add_argument("--seq_len", type=int, default=128)
    ap.add_argument("--batch_size", type=int, default=256)
    ap.add_argument("--cuda_graph", type=int, default=1)
    ap.add_argument("--peak_tflops", type=float, default=989.0, help="dense bf16 peak for the share of peak (H100 SXM data sheet)")
    ap.add_argument("--hbm_gbps", type=float, default=3350.0, help="HBM bandwidth for the computed bound (H100 SXM: 3.35 TB/s)")
    ap.add_argument("--no_baseline", action="store_true")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    out = {"metric": "samples/sec", "unit": "samples/s", "n_gpus": 1, "steps": args.steps, "warmup": args.warmup,
           "card": _card(), "dtype": "bf16",
           "config": {"hidden_units": args.hidden_units, "in_features": args.in_features, "seq_len": args.seq_len,
                      "batch_size": args.batch_size, "vocab_sizes": args.vocab_sizes}}
    for V in (int(v) for v in args.vocab_sizes.split(",")):
        torch.cuda.empty_cache()
        out[f"head_op_V{V}"] = head_op(args, V, dev)
        for ragged in (False, True):
            torch.cuda.empty_cache()
            out[f"ours_V{V}" + ("_variable_length" if ragged else "")] = ours(args, V, ragged, dev)
        if not args.no_baseline:
            torch.cuda.empty_cache()
            out[f"cudnn_V{V}"] = cudnn(args, V, dev)
        out["value"], out["ms_per_step"] = out[f"ours_V{V}"]["value"], out[f"ours_V{V}"]["ms_per_step"]
    print(json.dumps(out))


if __name__ == "__main__":
    sys.exit(main())
