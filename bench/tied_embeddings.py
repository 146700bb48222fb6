"""Tied embeddings (``--tie_embeddings``, one GPU) against the untied language model: the headline model (2-layer-1024 LSTM,
T = 128, B = 256, E = 1024, bf16, Adam, CUDA graph) behind an embedding table and under a softmax over the whole vocabulary,
V in {4096, 32768}.

    python bench/tied_embeddings.py --steps 30 --warmup 5 --rounds 3

Per V, for the arms ``untied`` and ``tied``:
  * ``train``: ``TrainEngine.step`` on 4 rotating device batches of the synthetic Markov language, captured as a CUDA graph,
    device-timed with CUDA events around ``--steps`` steps after ``--warmup``; the two arms alternate ``--rounds`` times in one
    process (so drift of the card's clock hits both alike); the median is reported;
  * ``params`` / ``flat_bytes``: the parameter count and the bytes the flat buffer, its gradient, Adam's m and v (fp32 each) and
    the bf16 shadow take (18 B per element, padding included);
  * ``perplexity``: a fresh engine of each arm (the same seed) trained for ``--ppl_steps`` steps, each on new walks of the
    chain, then scored on walks it never saw: exp of that loss (a reported figure, not a pass/fail; the chain's own
    perplexity is 2.97);
  * ``head_op``: the large-vocabulary head's launches alone, forward and backward, on W [H, V] (untied) or the table [V, H]
    (tied, read in place as a K-major operand), with TFLOP/s and bytes from the shapes (``bench/next_token.head_costs``);
  * ``decode``: ms per generated token of the captured decode step at B = 1 and 256.
Prints one JSON line, with the card's name, power limit and maximum SM clock.  Needs a GPU; there is no fallback.
"""
from __future__ import annotations

import argparse
import json
import math
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "bench"))

import torch

from next_token import head_costs                 # noqa: E402  (the shared helpers)
from variable_length import _card, _timed         # noqa: E402

BYTES_PER_ELEMENT = 4 + 4 + 4 + 4 + 2             # fp32 weights, gradient, Adam m and v; bf16 shadow


def _cfg(args, V, tied, B, T):
    from lstm_tensorspark_b200.config import Config
    return Config(hidden_units=args.hidden_units, in_features=args.in_features, seq_len=T, batch_size=B, partitions=1,
                  sync_mode="none", init="scaled", learn_initial_state=False, dtype="bf16", device="cuda", learning_rate=1e-3,
                  quiet=True, vocab_size=V, next_token=True, tie_embeddings=tied).validate()


def train_arm(args, V, tied, dev):
    from lstm_tensorspark_b200 import data as Dm
    from lstm_tensorspark_b200.engine import TrainEngine
    B, T, nb = args.batch_size, args.seq_len, 4
    eng = TrainEngine(_cfg(args, V, tied, B, T), 0, 1, None, batch_size=B, device=dev, dtype=torch.bfloat16)
    x, y = Dm.synthetic_next_token(nb * B, T, V, seed=1234)
    dx, dy = torch.as_tensor(x).to(dev), torch.as_tensor(y).to(dev)
    batches = [(dx[i * B:(i + 1) * B], dy[i * B:(i + 1) * B]) for i in range(nb)]
    eng.step(*batches[0])
    if args.cuda_graph:
        eng.capture(*batches[0], bind=batches[1:])
    params = sum(p.numel() for p in eng.model.parameters())
    return {"eng": eng, "batches": batches, "it": 0, "times": [],
            "params": params, "flat_elements": eng.flat.padded_numel, "flat_bytes": eng.flat.padded_numel * BYTES_PER_ELEMENT}


def timed_steps(args, arm):
    def step():
        arm["loss"] = arm["eng"].step(*arm["batches"][arm["it"] % len(arm["batches"])])
        arm["it"] += 1
    return _timed(step, args.steps, args.warmup)


def held_out_perplexity(args, V, tied, dev):
    """Train ``--ppl_steps`` steps on new walks of the chain each, then score ``B`` walks that were not trained on."""
    from lstm_tensorspark_b200 import data as Dm
    from lstm_tensorspark_b200.engine import TrainEngine
    B, T, K = args.batch_size, args.seq_len, args.ppl_steps
    eng = TrainEngine(_cfg(args, V, tied, B, T), 0, 1, None, batch_size=B, device=dev, dtype=torch.bfloat16)
    x, y = (torch.as_tensor(a).to(dev) for a in Dm.synthetic_next_token((K + 1) * B, T, V, seed=1234))
    for k in range(K):
        eng.step(x[k * B:(k + 1) * B], y[k * B:(k + 1) * B])
    m = eng.model
    m.eval()
    with torch.no_grad():
        loss = float(m.score(x[K * B:], y[K * B:])[0])
    del eng, m
    return {"steps": K, "held_out_loss": loss, "perplexity": math.exp(loss)}


def head_op(args, V, tied, dev, reps=10):
    from lstm_tensorspark_b200.ops import cuda_vocab_head
    T, B = args.seq_len, args.batch_size
    H = int(args.hidden_units.split(",")[-1])
    g = torch.Generator(device="cpu").manual_seed(0)
    h = torch.randn(T, B, H, generator=g).to(dev, torch.bfloat16).requires_grad_(True)
    W = (torch.randn(H, V, generator=g) / H ** 0.5).to(dev)
    # bf16, as the shadow the op reads in training (no cast per call); no autograd leaf: the backward computes dW all the same
    W = (W.t().contiguous() if tied else W).bfloat16()
    b = torch.zeros(V, device=dev, requires_grad=True)
    labels = torch.randint(0, V, (B, T), generator=g).to(dev)
    out = {}

    def fwd():
        out["loss"] = cuda_vocab_head.vocab_xent_per_step(h, W, b, labels, None, class_major=tied)[0]

    def bwd():
        out["loss"].backward(retain_graph=True)
    fwd_ms = _timed(fwd, reps, 3)
    bwd_ms = _timed(bwd, reps, 3)
    costs = head_costs(T * B, H, V, cuda_vocab_head.ROW_CHUNK)
    res = {"fwd_ms": fwd_ms, "bwd_ms": bwd_ms}
    for k, ms in (("fwd", fwd_ms), ("bwd", bwd_ms)):
        res[f"{k}_tflops"] = costs[f"{k}_flop"] / (ms * 1e-3) / 1e12
        res[f"{k}_share_of_bf16_peak"] = res[f"{k}_tflops"] / args.peak_tflops
    return res


def decode(args, V, tied, B, dev, N=16):
    """ms per token of the captured decode step (embedding, one step per layer, sampling) at batch B."""
    from lstm_tensorspark_b200.engine import TrainEngine
    m = TrainEngine(_cfg(args, V, tied, B, args.prompt_len), 0, 1, None, batch_size=B, device=dev, dtype=torch.bfloat16).model
    m.eval()
    g = torch.Generator().manual_seed(B + V)
    x = torch.randint(0, V, (B, args.prompt_len), generator=g, dtype=torch.int32).to(dev)
    lengths = torch.full((B,), args.prompt_len, dtype=torch.int32, device=dev)
    m.generate(x, lengths, N, 1.0, 1)                             # captures the decode step
    dec = next(d for k, d in m._decoders.items() if k[0] == B and k[1] == N)
    ms = _timed(dec.graph.replay, args.reps, 5)
    del m, dec
    return ms


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--hidden_units", default="1024,1024")
    ap.add_argument("--in_features", type=int, default=1024)
    ap.add_argument("--vocab_sizes", default="4096,32768")
    ap.add_argument("--seq_len", type=int, default=128)
    ap.add_argument("--batch_size", type=int, default=256)
    ap.add_argument("--prompt_len", type=int, default=16)
    ap.add_argument("--decode_batches", default="1,256")
    ap.add_argument("--reps", type=int, default=200, help="decode steps timed per arm and batch")
    ap.add_argument("--ppl_steps", type=int, default=300, help="training steps before the held-out perplexity")
    ap.add_argument("--cuda_graph", type=int, default=1)
    ap.add_argument("--peak_tflops", type=float, default=989.0, help="dense bf16 peak for the share of peak (H100 SXM data sheet)")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    out = {"metric": "ms/step", "unit": "ms", "n_gpus": 1, "steps": args.steps, "warmup": args.warmup, "rounds": args.rounds,
           "card": _card(), "dtype": "bf16",
           "config": {"hidden_units": args.hidden_units, "in_features": args.in_features, "seq_len": args.seq_len,
                      "batch_size": args.batch_size, "vocab_sizes": args.vocab_sizes, "cuda_graph": bool(args.cuda_graph)}}
    from lstm_tensorspark_b200.ops import cuda_lstm
    for V in (int(v) for v in args.vocab_sizes.split(",")):
        torch.cuda.empty_cache()
        n_tied = cuda_lstm.STATS.get("vocab_head_fwd_tied", 0)          # the eager step before each capture counts
        arms = {"untied": train_arm(args, V, False, dev), "tied": train_arm(args, V, True, dev)}
        for _ in range(args.rounds):
            for arm in arms.values():
                arm["times"].append(timed_steps(args, arm))
        res = {}
        for k, arm in arms.items():
            res[k] = {"ms_per_step": statistics.median(arm["times"]), "ms_per_step_rounds": arm["times"],
                      "loss": float(arm["loss"]),
                      "params": arm["params"], "flat_elements": arm["flat_elements"], "flat_bytes": arm["flat_bytes"]}
        res["tied_head_launched"] = cuda_lstm.STATS.get("vocab_head_fwd_tied", 0) > n_tied
        cuda_lstm.check_kernel_errors(dev)
        del arms
        torch.cuda.empty_cache()
        for k, tied in (("untied", False), ("tied", True)):
            torch.cuda.empty_cache()
            res[k]["held_out"] = held_out_perplexity(args, V, tied, dev)
            torch.cuda.empty_cache()
            res[k]["head_op"] = head_op(args, V, tied, dev)
            res[k]["decode_ms_per_token"] = {}
            for B in (int(b) for b in args.decode_batches.split(",")):
                torch.cuda.empty_cache()
                res[k]["decode_ms_per_token"][f"B{B}"] = decode(args, V, tied, B, dev)
        res["tied_over_untied_step"] = res["tied"]["ms_per_step"] / res["untied"]["ms_per_step"]
        res["params_saved"] = res["untied"]["params"] - res["tied"]["params"]
        res["flat_bytes_saved"] = res["untied"]["flat_bytes"] - res["tied"]["flat_bytes"]
        out[f"V{V}"] = res
        cuda_lstm.check_kernel_errors(dev)
    print(json.dumps(out))


if __name__ == "__main__":
    sys.exit(main())
