"""AWD-LSTM's activation regularisation (``--activation_reg 2 --temporal_activation_reg 1`` on top of AWD's dropout recipe, one
GPU): what AR / TAR cost per language-model step, what their two kernels cost alone, and what they do to a model that overfits.

    python bench/activation_reg.py --steps 30 --warmup 5 --rounds 3

  * ``step``: the language model of ``bench/awd_dropout.py`` (``--next_token --vocab_size 32768 --stateful --tie_embeddings``,
    2 x 1024, T = 128, B = 256, bf16, Adam, CUDA graph) with AWD's PTB dropout recipe, without and with alpha = 2, beta = 1.
    Device-timed with CUDA events around ``--steps`` steps after ``--warmup``; the arms alternate ``--rounds`` times in one
    process and the median is reported.
  * ``kernels``: the sum kernel and the combine kernel of csrc/activation_reg.cu alone at T = 128, B = 256, H = 1024, bf16, with
    the locked output dropout on, device-timed over ``--reps`` calls each; GB/s and the share of the data sheet's 3.35 TB/s from
    the bytes the shapes say each call must move (sum: reads out and h; combine: reads dh, out and h, writes dh_total).
  * ``regularisation`` (a reported figure, not pass/fail): the protocol of ``bench/awd_dropout.py`` (4 fixed batches of the
    synthetic Markov language, 2 x 512, V = 512, 150 epochs, training and held-out perplexity) for the full dropout recipe
    without and with AR / TAR.
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

from awd_dropout import RECIPE, _cfg                # noqa: E402  (the dropout recipe and its language model)
from variable_length import _card, _timed           # noqa: E402  (the shared helpers)

HBM_TBS = 3.35                                      # H100 SXM data sheet
AWD = dict(activation_reg=2.0, temporal_activation_reg=1.0)
ARMS = {"recipe": RECIPE, "recipe_ar_tar": {**RECIPE, **AWD}}


def train_arm(args, kw, dev):
    from lstm_tensorspark_b200 import data as Dm
    from lstm_tensorspark_b200.engine import TrainEngine
    B, T, nb = args.batch_size, args.seq_len, 4
    eng = TrainEngine(_cfg(args, kw), 0, 1, None, batch_size=B, device=dev, dtype=torch.bfloat16)
    x, y = Dm.synthetic_next_token(nb * B, T, args.vocab_size, seed=1234)
    dx, dy = torch.as_tensor(x).to(dev), torch.as_tensor(y).to(dev)
    batches = [(dx[i * B:(i + 1) * B], dy[i * B:(i + 1) * B]) for i in range(nb)]
    eng.step(*batches[0])
    if args.cuda_graph:
        eng.capture(*batches[0], bind=batches[1:])
    return {"eng": eng, "batches": batches, "it": 0, "times": []}


def step_times(args, dev):
    from lstm_tensorspark_b200.ops import cuda_lstm

    def timed(arm):
        def step():
            arm["loss"] = arm["eng"].step(*arm["batches"][arm["it"] % len(arm["batches"])])
            arm["it"] += 1
        return _timed(step, args.steps, args.warmup)
    arms = {k: train_arm(args, kw, dev) for k, kw in ARMS.items()}
    for _ in range(args.rounds):
        for arm in arms.values():
            arm["times"].append(timed(arm))
    res = {k: {"ms_per_step": statistics.median(a["times"]), "ms_per_step_rounds": a["times"], "loss": float(a["loss"])}
           for k, a in arms.items()}
    pen = arms["recipe_ar_tar"]["eng"].activation_penalties()
    res["recipe_ar_tar"]["ar_tar"] = [float(v) for v in pen.tolist()]
    res["ar_tar_over_recipe"] = res["recipe_ar_tar"]["ms_per_step"] / res["recipe"]["ms_per_step"]
    res["ar_tar_minus_recipe_us"] = (res["recipe_ar_tar"]["ms_per_step"] - res["recipe"]["ms_per_step"]) * 1e3
    cuda_lstm.check_kernel_errors(dev)
    del arms
    torch.cuda.empty_cache()
    return res


def kernels(args, dev):
    from lstm_tensorspark_b200.ops import cuda_lstm
    from lstm_tensorspark_b200.ops.cuda_ext import drop_args
    from lstm_tensorspark_b200.ops.reference import DropoutSpec
    T, B, H = args.seq_len, args.batch_size, int(args.hidden_units.split(",")[-1])
    step = torch.zeros(1, dtype=torch.int32, device=dev)
    spec = DropoutSpec(RECIPE["output_dropout"], (1, 0), 1, False, step, locked=True)
    h = (torch.randn(T, B, H, device=dev) * 0.3).bfloat16()
    out = cuda_lstm.dropout(h, spec)
    dh = (torch.randn(T, B, H, device=dev) * 1e-4).bfloat16()
    g = torch.tensor([1e-6, 1e-6], device=dev)
    drop = drop_args(spec, dev)
    arr = T * B * H * 2
    runs = {"sum": (lambda: cuda_lstm._activation_sums(out, h, None), 2 * arr),
            "combine": (lambda: cuda_lstm._activation_grad(dh, out, h, None, g, drop), 4 * arr)}
    res = {"T": T, "B": B, "H": H, "output_dropout": spec.p, "locked": True}
    for k, (fn, nbytes) in runs.items():
        us = _timed(fn, args.reps, 10) * 1e3
        gbs = nbytes / (us * 1e-6) / 1e9
        res[k] = {"us": us, "bytes": nbytes, "GB_per_s": gbs, "share_of_hbm_peak": gbs / (HBM_TBS * 1e3)}
    return res


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
    for k, kw in ARMS.items():
        h = int(args.reg_hidden.split(",")[-1])
        cfg = _cfg(args, kw, hidden_units=args.reg_hidden, in_features=h, seq_len=T, batch_size=B, vocab_size=V,
                   stateful=False, tie_embeddings=False, learning_rate=args.reg_lr, seed=7)
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
    ap.add_argument("--reps", type=int, default=200, help="calls timed per kernel")
    ap.add_argument("--reg_batches", type=int, default=4)
    ap.add_argument("--reg_batch_size", type=int, default=64)
    ap.add_argument("--reg_seq_len", type=int, default=64)
    ap.add_argument("--reg_vocab", type=int, default=512)
    ap.add_argument("--reg_hidden", default="512,512")
    ap.add_argument("--reg_epochs", type=int, default=150)
    ap.add_argument("--reg_lr", type=float, default=2e-3)
    ap.add_argument("--skip", default="", help="comma list of sections to skip: step, kernels, regularisation")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    skip = set(s for s in args.skip.split(",") if s)
    out = {"metric": "ms/step", "unit": "ms", "n_gpus": 1, "steps": args.steps, "warmup": args.warmup, "rounds": args.rounds,
           "card": _card(), "dtype": "bf16", "recipe": RECIPE, "ar_tar": AWD,
           "config": {"hidden_units": args.hidden_units, "in_features": args.in_features, "seq_len": args.seq_len,
                      "batch_size": args.batch_size, "vocab_size": args.vocab_size, "cuda_graph": bool(args.cuda_graph)}}
    if "step" not in skip:
        out["language_model"] = step_times(args, dev)
    if "kernels" not in skip:
        out["kernels"] = kernels(args, dev)
    if "regularisation" not in skip:
        out["regularisation"] = regularisation(args, dev)
    print(json.dumps(out))


if __name__ == "__main__":
    sys.exit(main())
