"""Weight drop (``--weight_drop``, AWD-LSTM's DropConnect on W_h, one GPU): what it costs per training step, what its two launches
cost alone, and what it does to a model that overfits.

    python bench/weight_drop.py --steps 30 --warmup 5 --rounds 3

  * ``step``: the headline model (2 x 1024, T = 128, B = 256, D = 1024, bf16, Adam, CUDA graph) and the language model
    (``--next_token --vocab_size 32768 --stateful --tie_embeddings``, E = 1024) at ``--weight_drop`` 0 and 0.5 (AWD-LSTM's
    default).  ``TrainEngine.step`` on 4 rotating device batches, device-timed with CUDA events around ``--steps`` steps after
    ``--warmup``; the arms alternate ``--rounds`` times in one process and the median is reported.
  * ``launches``: the masked image (the dropout kernel over a bf16 [1, 4H, H] view of W_h) and the masked weight gradient
    (fp32 [4H, H], in place and accumulating) at H = 1024, device-timed over ``--reps`` launches each; GB/s and the share of the
    data sheet's 3.35 TB/s from the bytes the shapes say each launch must move.
  * ``regularisation`` (a reported figure, not pass/fail): a fixed set of ``--reg_batches`` batches of the synthetic Markov
    language, trained on for ``--reg_epochs`` epochs by a fresh engine per arm (same seed) at ``--weight_drop`` 0 and 0.5; the
    training and held-out perplexity (walks never trained on) after it.  The chain's own perplexity is 2.97: a training
    perplexity below it means the model memorised its set.
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

from variable_length import _card, _timed         # noqa: E402  (the shared helpers)

HBM_TBS = 3.35                                      # H100 SXM data sheet
ROTATE = 8


def _cfg(args, wd, lm, **kw):
    from lstm_tensorspark_b200.config import Config
    base = dict(hidden_units=args.hidden_units, in_features=args.in_features, seq_len=args.seq_len, batch_size=args.batch_size,
                partitions=1, sync_mode="none", init="scaled", learn_initial_state=False, dtype="bf16", device="cuda",
                learning_rate=1e-3, quiet=True, weight_drop=wd)
    if lm:
        base.update(vocab_size=args.vocab_size, next_token=True, stateful=True, tie_embeddings=True)
    else:
        base.update(num_classes=10)
    base.update(kw)
    return Config(**base).validate()


def train_arm(args, wd, lm, dev):
    from lstm_tensorspark_b200 import data as Dm
    from lstm_tensorspark_b200.engine import TrainEngine
    B, T, nb = args.batch_size, args.seq_len, 4
    eng = TrainEngine(_cfg(args, wd, lm), 0, 1, None, batch_size=B, device=dev, dtype=torch.bfloat16)
    if lm:
        x, y = Dm.synthetic_next_token(nb * B, T, args.vocab_size, seed=1234)
        dx, dy = torch.as_tensor(x).to(dev), torch.as_tensor(y).to(dev)
    else:
        x, y = Dm.synthetic_sequences(nb * B, T, args.in_features, 10, seed=1234)
        dx, dy = torch.as_tensor(x).to(dev).bfloat16(), torch.as_tensor(y).to(dev)
    batches = [(dx[i * B:(i + 1) * B], dy[i * B:(i + 1) * B]) for i in range(nb)]
    eng.step(*batches[0])
    if args.cuda_graph:
        eng.capture(*batches[0], bind=batches[1:])
    return {"eng": eng, "batches": batches, "it": 0, "times": []}


def timed_steps(args, arm):
    def step():
        arm["loss"] = arm["eng"].step(*arm["batches"][arm["it"] % len(arm["batches"])])
        arm["it"] += 1
    return _timed(step, args.steps, args.warmup)


def step_times(args, lm, dev):
    from lstm_tensorspark_b200.ops import cuda_lstm
    n0 = cuda_lstm.STATS["weight_drop"], cuda_lstm.STATS["weight_drop_grad"]
    arms = {"p0": train_arm(args, 0.0, lm, dev), "p0.5": train_arm(args, 0.5, lm, dev)}
    for _ in range(args.rounds):
        for arm in arms.values():
            arm["times"].append(timed_steps(args, arm))
    res = {k: {"ms_per_step": statistics.median(a["times"]), "ms_per_step_rounds": a["times"], "loss": float(a["loss"]),
               "mask_counter": int(a["eng"].model.rnn.dropout_step)} for k, a in arms.items()}
    res["weight_drop_launches_recorded"] = [cuda_lstm.STATS["weight_drop"] - n0[0], cuda_lstm.STATS["weight_drop_grad"] - n0[1]]
    res["p0.5_over_p0"] = res["p0.5"]["ms_per_step"] / res["p0"]["ms_per_step"]
    res["p0.5_minus_p0_us"] = (res["p0.5"]["ms_per_step"] - res["p0"]["ms_per_step"]) * 1e3
    cuda_lstm.check_kernel_errors(dev)
    del arms
    torch.cuda.empty_cache()
    return res


def launch_costs(H: int) -> dict:
    """Bytes each launch must move at [4H, H]: the image reads and writes bf16; the gradient reads fp32 src and writes fp32 dst,
    and reads dst too when it accumulates."""
    n = 4 * H * H
    return {"image": 2 * n + 2 * n, "grad_in_place": 4 * n + 4 * n, "grad_accumulate": 4 * n + 4 * n + 4 * n}


def launches(args, dev):
    from lstm_tensorspark_b200.ops import cuda_lstm
    from lstm_tensorspark_b200.ops.reference import DropoutSpec
    H = args.launch_h
    spec = DropoutSpec(0.5, (1, 0), 0, False, torch.zeros(1, dtype=torch.int32, device=dev), weight=True)
    d = cuda_lstm._drop_args(spec, dev)
    # consecutive launches rotate over ROTATE sets of operands (>= 128 MiB at H = 1024), so that they do not find their operands
    # in the 50 MB L2 the previous launch left them in, as in a training step
    w = [(torch.randn(4 * H, H, device=dev) / H ** 0.5).bfloat16() for _ in range(ROTATE)]
    g = [torch.randn(4 * H, H, device=dev) for _ in range(ROTATE)]
    acc = [torch.randn(4 * H, H, device=dev) for _ in range(ROTATE)]
    it = {"n": 0}

    def nxt():
        it["n"] += 1
        return it["n"] % ROTATE
    runs = {"image": lambda: cuda_lstm._weight_image(w[nxt()], spec),
            "grad_in_place": lambda: (lambda i: cuda_lstm._weight_drop_grad(g[i], g[i], d, False))(nxt()),
            "grad_accumulate": lambda: (lambda i: cuda_lstm._weight_drop_grad(g[i], acc[i], d, True))(nxt())}
    costs = launch_costs(H)
    out = {"H": H, "shape": [4 * H, H], "operand_sets_rotated": ROTATE}
    for k, fn in runs.items():
        us = _timed(fn, args.reps, 10) * 1e3
        gbs = costs[k] / (us * 1e-6) / 1e9
        out[k] = {"us": us, "bytes": costs[k], "GB_per_s": gbs, "share_of_hbm_peak": gbs / (HBM_TBS * 1e3)}
    layers = len(args.hidden_units.split(","))
    out["per_step_from_shapes_us"] = {
        "bytes": layers * (costs["image"] + costs["grad_in_place"]),
        "us_at_hbm_peak": layers * (costs["image"] + costs["grad_in_place"]) / (HBM_TBS * 1e12) * 1e6,
        "note": "computed from the shapes at the data sheet's bandwidth, not measured"}
    return out


def regularisation(args, dev):
    """A fixed training set, many epochs; training and held-out perplexity of a fresh engine per arm."""
    from lstm_tensorspark_b200 import data as Dm
    from lstm_tensorspark_b200.engine import TrainEngine
    B, T, V, nb = args.reg_batch_size, args.reg_seq_len, args.reg_vocab, args.reg_batches
    x, y = (torch.as_tensor(a).to(dev) for a in Dm.synthetic_next_token((nb + 4) * B, T, V, seed=99))
    train = [(x[i * B:(i + 1) * B], y[i * B:(i + 1) * B]) for i in range(nb)]
    held = (x[nb * B:], y[nb * B:])
    out = {"batches": nb, "batch_size": B, "seq_len": T, "vocab_size": V, "hidden_units": args.reg_hidden, "epochs": args.reg_epochs,
           "chain_perplexity": math.exp(Dm.NEXT_TOKEN_ENTROPY)}
    for k, wd in (("p0", 0.0), ("p0.5", 0.5)):
        h = int(args.reg_hidden.split(",")[-1])
        cfg = _cfg(args, wd, False, hidden_units=args.reg_hidden, in_features=h, seq_len=T, batch_size=B, vocab_size=V,
                   next_token=True, num_classes=V, learning_rate=args.reg_lr, seed=7)
        eng = TrainEngine(cfg, 0, 1, None, batch_size=B, device=dev, dtype=torch.bfloat16)
        for _ in range(args.reg_epochs):
            for xb, yb in train:
                eng.step(xb, yb)
        m = eng.model
        m.eval()
        with torch.no_grad():
            tr = statistics.mean(float(m.score(xb, yb)[0]) for xb, yb in train)
            ho = statistics.mean(float(m.score(held[0][i * B:(i + 1) * B], held[1][i * B:(i + 1) * B])[0]) for i in range(4))
        out[k] = {"train_loss": tr, "train_perplexity": math.exp(tr), "held_out_loss": ho, "held_out_perplexity": math.exp(ho)}
        del eng, m
        torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--hidden_units", default="1024,1024")
    ap.add_argument("--in_features", type=int, default=1024)
    ap.add_argument("--seq_len", type=int, default=128)
    ap.add_argument("--batch_size", type=int, default=256)
    ap.add_argument("--vocab_size", type=int, default=32768)
    ap.add_argument("--cuda_graph", type=int, default=1)
    ap.add_argument("--launch_h", type=int, default=1024)
    ap.add_argument("--reps", type=int, default=200, help="launches timed per kernel")
    ap.add_argument("--reg_batches", type=int, default=4)
    ap.add_argument("--reg_batch_size", type=int, default=64)
    ap.add_argument("--reg_seq_len", type=int, default=64)
    ap.add_argument("--reg_vocab", type=int, default=512)
    ap.add_argument("--reg_hidden", default="512,512")
    ap.add_argument("--reg_epochs", type=int, default=150)
    ap.add_argument("--reg_lr", type=float, default=2e-3)
    ap.add_argument("--skip", default="", help="comma list of sections to skip: step, lm, launches, regularisation")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    skip = set(s for s in args.skip.split(",") if s)
    out = {"metric": "ms/step", "unit": "ms", "n_gpus": 1, "steps": args.steps, "warmup": args.warmup, "rounds": args.rounds,
           "card": _card(), "dtype": "bf16",
           "config": {"hidden_units": args.hidden_units, "in_features": args.in_features, "seq_len": args.seq_len,
                      "batch_size": args.batch_size, "vocab_size": args.vocab_size, "cuda_graph": bool(args.cuda_graph)}}
    if "step" not in skip:
        out["headline"] = step_times(args, False, dev)
    if "lm" not in skip:
        out["language_model"] = step_times(args, True, dev)
    if "launches" not in skip:
        out["launches"] = launches(args, dev)
    if "regularisation" not in skip:
        out["regularisation"] = regularisation(args, dev)
    print(json.dumps(out))


if __name__ == "__main__":
    sys.exit(main())
