"""AWD-LSTM's dropouts (``--locked_dropout --input_dropout --dropout --output_dropout --embedding_dropout --weight_drop``, one
GPU): what the full recipe costs per language-model step, what the masked embedding launches cost alone, and what the recipe does
to a model that overfits.

    python bench/awd_dropout.py --steps 30 --warmup 5 --rounds 3

  * ``step``: the language model (``--next_token --vocab_size 32768 --stateful --tie_embeddings``, 2 x 1024, T = 128, B = 256,
    E = 1024, bf16, Adam, CUDA graph) with no dropout and with AWD-LSTM's PTB recipe (``--locked_dropout --input_dropout 0.65
    --dropout 0.3 --output_dropout 0.4 --embedding_dropout 0.1 --weight_drop 0.5``).  ``TrainEngine.step`` on 4 rotating device
    batches, device-timed with CUDA events around ``--steps`` steps after ``--warmup``; the arms alternate ``--rounds`` times
    in one process and the median is reported.
  * ``launches``: the embedding gather and the table gradient's three launches (rank, plan, sum; one call) at T·B = 32768,
    E = 1024, V = 32768, bf16, unmasked and with both masks, device-timed over ``--reps`` calls each; GB/s and the share of the
    data sheet's 3.35 TB/s from the bytes the shapes say each call must move.
  * ``regularisation`` (a reported figure, not pass/fail): the protocol of ``bench/weight_drop.py`` (a fixed set of batches of the
    synthetic Markov language, many epochs, training and held-out perplexity) with three arms: no dropout, weight drop 0.5
    alone, and the full recipe.
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
RECIPE = dict(locked_dropout=True, input_dropout=0.65, dropout=0.3, output_dropout=0.4, embedding_dropout=0.1, weight_drop=0.5)
ARMS = {"none": {}, "weight_drop": dict(weight_drop=0.5), "recipe": RECIPE}


def _cfg(args, drop, **kw):
    from lstm_tensorspark_b200.config import Config
    base = dict(hidden_units=args.hidden_units, in_features=args.in_features, seq_len=args.seq_len, batch_size=args.batch_size,
                partitions=1, sync_mode="none", init="scaled", learn_initial_state=False, dtype="bf16", device="cuda",
                learning_rate=1e-3, quiet=True, vocab_size=args.vocab_size, next_token=True, stateful=True, tie_embeddings=True)
    base.update(drop)
    base.update(kw)
    return Config(**base).validate()


def train_arm(args, drop, dev):
    from lstm_tensorspark_b200 import data as Dm
    from lstm_tensorspark_b200.engine import TrainEngine
    B, T, nb = args.batch_size, args.seq_len, 4
    eng = TrainEngine(_cfg(args, drop), 0, 1, None, batch_size=B, device=dev, dtype=torch.bfloat16)
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
    arms = {"none": train_arm(args, {}, dev), "recipe": train_arm(args, RECIPE, dev)}
    for _ in range(args.rounds):
        for arm in arms.values():
            arm["times"].append(timed(arm))
    res = {k: {"ms_per_step": statistics.median(a["times"]), "ms_per_step_rounds": a["times"], "loss": float(a["loss"]),
               "mask_counter": int(a["eng"].model.rnn.dropout_step)} for k, a in arms.items()}
    res["recipe_over_none"] = res["recipe"]["ms_per_step"] / res["none"]["ms_per_step"]
    res["recipe_minus_none_us"] = (res["recipe"]["ms_per_step"] - res["none"]["ms_per_step"]) * 1e3
    B, T, H = args.batch_size, args.seq_len, int(args.hidden_units.split(",")[-1])
    res["top_layer_h_drop_store_MiB_from_shapes"] = T * B * H * 2 / 2 ** 20
    cuda_lstm.check_kernel_errors(dev)
    del arms
    torch.cuda.empty_cache()
    return res


def launch_costs(N: int, E: int, V: int) -> dict:
    """Bytes each call must move (bf16 rows, fp32 table gradient, int32 ids): the gather reads N rows and writes N rows; the
    gradient reads the N ids (rank), writes and reads back its sort (plan, about 6 int32 words per position), reads N rows of
    dx and writes every row of dW.  Dropped rows need not be read, so the masked arms may move less than this."""
    gather = 2 * N * E * 2 + N * 4
    grad = N * 4 + 6 * N * 4 + N * E * 2 + V * E * 4
    return {"gather": gather, "table_gradient": grad}


def launches(args, dev):
    from lstm_tensorspark_b200.ops.cuda_ext import ext
    from lstm_tensorspark_b200.ops.reference import DropoutSpec
    N, E, V = args.launch_rows, args.launch_e, args.launch_v
    B = 256
    T = N // B
    step = torch.zeros(1, dtype=torch.int32, device=dev)
    si = DropoutSpec(0.65, (1, 0), 0, False, step, site="input", locked=True)
    se = DropoutSpec(0.1, (1, 0), 0, False, step, site="rows")
    masked = {"in_step": step, "in_desc": si.desc(), "row_step": step, "row_desc": se.desc()}
    table = (torch.randn(V, E, device=dev) * 0.1).bfloat16()
    tok = torch.randint(0, V, (B, T), device=dev, dtype=torch.int32)
    dx = torch.randn(T, B, E, device=dev).bfloat16()
    dW = torch.empty(V, E, device=dev)
    costs = launch_costs(N, E, V)
    out = {"rows": N, "E": E, "V": V, "input_dropout": si.p, "embedding_dropout": se.p, "locked": True}
    for arm, kw in (("plain", {}), ("masked", masked)):
        runs = {"gather": lambda: ext().embed_fwd(table, tok, None, **kw),
                "table_gradient": lambda: ext().embed_bwd(dx, tok, None, dW, False, **kw)}
        out[arm] = {}
        for k, fn in runs.items():
            us = _timed(fn, args.reps, 10) * 1e3
            gbs = costs[k] / (us * 1e-6) / 1e9
            out[arm][k] = {"us": us, "bytes": costs[k], "GB_per_s": gbs, "share_of_hbm_peak": gbs / (HBM_TBS * 1e3)}
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
    for k, drop in ARMS.items():
        h = int(args.reg_hidden.split(",")[-1])
        cfg = _cfg(args, drop, hidden_units=args.reg_hidden, in_features=h, seq_len=T, batch_size=B, vocab_size=V,
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
    ap.add_argument("--launch_rows", type=int, default=32768)
    ap.add_argument("--launch_e", type=int, default=1024)
    ap.add_argument("--launch_v", type=int, default=32768)
    ap.add_argument("--reps", type=int, default=100, help="calls timed per launch")
    ap.add_argument("--reg_batches", type=int, default=4)
    ap.add_argument("--reg_batch_size", type=int, default=64)
    ap.add_argument("--reg_seq_len", type=int, default=64)
    ap.add_argument("--reg_vocab", type=int, default=512)
    ap.add_argument("--reg_hidden", default="512,512")
    ap.add_argument("--reg_epochs", type=int, default=150)
    ap.add_argument("--reg_lr", type=float, default=2e-3)
    ap.add_argument("--skip", default="", help="comma list of sections to skip: step, launches, regularisation")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    skip = set(s for s in args.skip.split(",") if s)
    out = {"metric": "ms/step", "unit": "ms", "n_gpus": 1, "steps": args.steps, "warmup": args.warmup, "rounds": args.rounds,
           "card": _card(), "dtype": "bf16", "recipe": RECIPE,
           "config": {"hidden_units": args.hidden_units, "in_features": args.in_features, "seq_len": args.seq_len,
                      "batch_size": args.batch_size, "vocab_size": args.vocab_size, "cuda_graph": bool(args.cuda_graph)}}
    if "step" not in skip:
        out["language_model"] = step_times(args, dev)
    if "launches" not in skip:
        out["launches"] = launches(args, dev)
    if "regularisation" not in skip:
        out["regularisation"] = regularisation(args, dev)
    print(json.dumps(out))


if __name__ == "__main__":
    sys.exit(main())
