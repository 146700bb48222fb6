"""NT-ASGD (``--optimizer asgd | ntasgd``, one GPU): what averaging costs per training step, what its kernels cost alone, what one
validation pass costs, and what the averaged model does on held-out data.

    python bench/asgd.py --steps 30 --warmup 5 --rounds 3

  * ``step``: the headline model (2 x 1024, T = 128, B = 256, D = 1024, bf16, CUDA graph) and the language model (``--next_token
    --vocab_size 32768 --stateful --tie_embeddings``, E = 1024, with AWD-LSTM's dropout recipe and weight drop) under ``sgd`` and
    under ``asgd`` with averaging on (the fused update + average).  ``TrainEngine.step`` on 4 rotating device batches,
    device-timed with CUDA events around ``--steps`` steps after ``--warmup``; the arms alternate ``--rounds`` times in one
    process and the median is reported.
  * ``launches``: ``flat_sgd``, the fused ``flat_asgd`` (averaging on, k large), ``flat_average`` and ``flat_swap`` over a flat
    buffer of the language model's size, device-timed over ``--reps`` launches each on rotating operand sets (each larger than
    L2); GB/s and the share of the data sheet's 3.35 TB/s from the bytes the shapes say each launch must move.
  * ``validation``: one pass of ``trainer.validation_scorer`` over a held-out stream of ``--valid_segments`` segments of the
    language model (B x T positions each), with the averaged weights swapped in and out around it, device-timed.
  * ``regularisation`` (a reported figure, not pass/fail): the synthetic Markov language, a small training set trained on for
    ``--reg_epochs`` epochs through ``trainer.run_job`` (validated once per epoch) under ``sgd`` and ``ntasgd`` at the same
    learning rate and clip; the held-out perplexity of the last validation (the averaged model once ntasgd has fired) and the
    step it fired at.  The chain's own perplexity is 2.97.
Prints one JSON line, with the card's name, power limit and maximum SM clock.  Needs a GPU; there is no fallback.  Run-time files
(checkpoints of the regularisation runs) go to a temporary directory.
"""
from __future__ import annotations

import argparse
import json
import math
import os
import statistics
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "bench"))

import torch

from variable_length import _card, _timed         # noqa: E402  (the shared helpers)

HBM_TBS = 3.35                                      # H100 SXM data sheet
ROTATE = 2                                          # operand sets per kernel: each is hundreds of MB, far beyond the 50 MB L2
AWD_RECIPE = dict(locked_dropout=True, input_dropout=0.65, dropout=0.3, output_dropout=0.4, embedding_dropout=0.1, weight_drop=0.5)


def _cfg(args, kind, lm, **kw):
    from lstm_tensorspark_b200.config import Config
    base = dict(hidden_units=args.hidden_units, in_features=args.in_features, seq_len=args.seq_len, batch_size=args.batch_size,
                partitions=1, sync_mode="none", init="scaled", learn_initial_state=False, dtype="bf16", device="cuda",
                learning_rate=1e-3, quiet=True, optimizer=kind)
    if lm:
        base.update(vocab_size=args.vocab_size, next_token=True, stateful=True, tie_embeddings=True, **AWD_RECIPE)
    else:
        base.update(num_classes=10)
    base.update(kw)
    return Config(**base).validate()


def _lm_batches(args, n, dev, seed=1234):
    from lstm_tensorspark_b200 import data as Dm
    B, T = args.batch_size, args.seq_len
    x, y = Dm.synthetic_next_token(n * B, T, args.vocab_size, seed=seed)
    dx, dy = torch.as_tensor(x).to(dev), torch.as_tensor(y).to(dev)
    return [(dx[i * B:(i + 1) * B], dy[i * B:(i + 1) * B]) for i in range(n)]


def train_arm(args, kind, lm, dev):
    from lstm_tensorspark_b200 import data as Dm
    from lstm_tensorspark_b200.engine import TrainEngine
    B, T, nb = args.batch_size, args.seq_len, 4
    eng = TrainEngine(_cfg(args, kind, lm), 0, 1, None, batch_size=B, device=dev, dtype=torch.bfloat16)
    if lm:
        batches = _lm_batches(args, nb, dev)
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
    arms = {"sgd": train_arm(args, "sgd", lm, dev), "asgd": train_arm(args, "asgd", lm, dev)}
    for _ in range(args.rounds):
        for arm in arms.values():
            arm["times"].append(timed_steps(args, arm))
    res = {k: {"ms_per_step": statistics.median(a["times"]), "ms_per_step_rounds": a["times"], "loss": float(a["loss"])}
           for k, a in arms.items()}
    opt = arms["asgd"]["eng"].optimizer
    res["asgd"].update(averaging=opt.averaging, averaged_steps=opt.averaged_steps)
    res["flat_numel"] = int(arms["sgd"]["eng"].flat.data.numel())
    res["asgd_over_sgd"] = res["asgd"]["ms_per_step"] / res["sgd"]["ms_per_step"]
    res["asgd_minus_sgd_us"] = (res["asgd"]["ms_per_step"] - res["sgd"]["ms_per_step"]) * 1e3
    cuda_lstm.check_kernel_errors(dev)
    del arms, opt
    torch.cuda.empty_cache()
    return res


def launch_bytes(n: int) -> dict:
    """Bytes each launch must move over n fp32 elements with a bf16 shadow: SGD reads p, g and writes p, shadow (14 B); the fused
    ASGD also reads and writes ax (22 B); the average reads p, ax and writes ax (12 B); the swap reads and writes p and ax and
    writes the shadow (18 B)."""
    return {"flat_sgd": 14 * n, "flat_asgd": 22 * n, "flat_average": 12 * n, "flat_swap": 18 * n}


def launches(args, n, dev):
    from lstm_tensorspark_b200.ops.cuda_ext import ext
    E = ext()
    n = (n + 3) // 4 * 4
    sets = []
    for _ in range(ROTATE):
        sets.append({"p": torch.randn(n, device=dev) * 0.05, "g": torch.randn(n, device=dev) * 1e-3,
                     "ax": torch.randn(n, device=dev) * 0.05, "s": torch.empty(n, dtype=torch.bfloat16, device=dev)})
    # k far past 2, averaging on: every launch takes the averaging branch; the bump advances k, which changes no byte count
    avg = torch.tensor([1, 1000], dtype=torch.int32, device=dev)
    it = {"n": 0}

    def nxt():
        it["n"] += 1
        return sets[it["n"] % ROTATE]
    runs = {"flat_sgd": lambda: (lambda o: E.flat_sgd(o["p"], o["g"], o["s"], 1e-3, 0.0, 1.0))(nxt()),
            "flat_asgd": lambda: (lambda o: E.flat_asgd(o["p"], o["g"], o["ax"], avg, o["s"], 1e-3, 0.0, 1.0))(nxt()),
            "flat_average": lambda: (lambda o: E.flat_average(o["p"], o["ax"], avg))(nxt()),
            "flat_swap": lambda: (lambda o: E.flat_swap(o["p"], o["ax"], o["s"]))(nxt())}
    costs = launch_bytes(n)
    out = {"n": n, "operand_sets_rotated": ROTATE}
    for k, fn in runs.items():
        us = _timed(fn, args.reps, 10) * 1e3
        gbs = costs[k] / (us * 1e-6) / 1e9
        out[k] = {"us": us, "bytes": costs[k], "GB_per_s": gbs, "share_of_hbm_peak": gbs / (HBM_TBS * 1e3),
                  "us_at_hbm_peak_not_measured": costs[k] / (HBM_TBS * 1e12) * 1e6}
    del sets
    torch.cuda.empty_cache()
    return out


def validation(args, dev):
    from lstm_tensorspark_b200 import data as Dm
    from lstm_tensorspark_b200.engine import TrainEngine
    from lstm_tensorspark_b200.trainer import validation_scorer
    cfg = _cfg(args, "asgd", True)
    eng = TrainEngine(cfg, 0, 1, None, batch_size=args.batch_size, device=dev, dtype=torch.bfloat16)
    for xb, yb in _lm_batches(args, 2, dev):
        eng.step(xb, yb)
    stream = Dm.synthetic_stream(args.batch_size * args.valid_segments, args.seq_len, args.vocab_size, seed=5, valid=True)
    score = validation_scorer(stream, cfg, args.batch_size, dev, torch.bfloat16)
    res = {}

    def one():
        with torch.no_grad(), eng.averaged_weights():
            eng.model.eval()
            res["val"] = score(eng.model)
            eng.model.train()
    ms = _timed(one, 3, 1)
    out = {"segments": args.valid_segments, "streams": args.batch_size, "seq_len": args.seq_len,
           "positions": res["val"][2], "ms_per_pass": ms, "val_loss": res["val"][0]}
    del eng
    torch.cuda.empty_cache()
    return out


def regularisation(args):
    from lstm_tensorspark_b200.config import Config
    from lstm_tensorspark_b200.trainer import run_job
    from lstm_tensorspark_b200 import data as Dm
    B, T, V, nb = args.reg_batch_size, args.reg_seq_len, args.reg_vocab, args.reg_batches
    h = int(args.reg_hidden.split(",")[-1])
    out = {"batches_per_epoch": nb, "batch_size": B, "seq_len": T, "vocab_size": V, "hidden_units": args.reg_hidden,
           "epochs": args.reg_epochs, "learning_rate": args.reg_lr, "clip_grad_norm": args.reg_clip, "nonmono": args.reg_nonmono,
           "valid_samples": 4 * B, "chain_perplexity": math.exp(Dm.NEXT_TOKEN_ENTROPY)}
    with tempfile.TemporaryDirectory() as tmp:
        for kind in ("sgd", "ntasgd"):
            log = os.path.join(tmp, kind + ".jsonl")
            cfg = Config(hidden_units=args.reg_hidden, in_features=h, seq_len=T, batch_size=B, vocab_size=V, next_token=True,
                         synthetic=nb * B, valid_synthetic=4 * B, partitions=1, sync_mode="none", init="scaled",
                         learn_initial_state=False, dtype="bf16", device="cuda", quiet=True, optimizer=kind,
                         learning_rate=args.reg_lr, clip_grad_norm=args.reg_clip, nonmono=args.reg_nonmono, seed=7,
                         max_steps=nb * args.reg_epochs, evaluate_every=nb, cuda_graph=True, json_log=log,
                         checkpoint_path=os.path.join(tmp, kind), output_path=os.path.join(tmp, kind + "_out")).validate()
            run_job(cfg, standalone=True)
            evals = [r for r in map(json.loads, open(log).read().splitlines()) if "val_loss" in r]
            last = evals[-1]
            fired = [r["step"] for r in evals if r.get("averaging")]
            out[kind] = {"held_out_loss": last["val_loss"], "held_out_perplexity": last["val_perplexity"],
                         "best_held_out_perplexity": min(r["val_perplexity"] for r in evals),
                         "train_batch_loss": last["loss"], "averaging_from_validation_at_step": fired[0] if fired else None,
                         "averaged_steps": last.get("averaged_steps")}
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
    ap.add_argument("--reps", type=int, default=200, help="launches timed per kernel")
    ap.add_argument("--launch_n", type=int, default=50380800, help="flat elements of the kernel timings when the lm section is skipped")
    ap.add_argument("--valid_segments", type=int, default=8)
    ap.add_argument("--reg_batches", type=int, default=4)
    ap.add_argument("--reg_batch_size", type=int, default=64)
    ap.add_argument("--reg_seq_len", type=int, default=64)
    ap.add_argument("--reg_vocab", type=int, default=512)
    ap.add_argument("--reg_hidden", default="512,512")
    ap.add_argument("--reg_epochs", type=int, default=150)
    ap.add_argument("--reg_lr", type=float, default=20.0)
    ap.add_argument("--reg_clip", type=float, default=0.25)
    ap.add_argument("--reg_nonmono", type=int, default=5)
    ap.add_argument("--skip", default="", help="comma list of sections to skip: step, lm, launches, validation, regularisation")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    skip = set(s for s in args.skip.split(",") if s)
    out = {"metric": "ms/step", "unit": "ms", "n_gpus": 1, "steps": args.steps, "warmup": args.warmup, "rounds": args.rounds,
           "card": _card(), "dtype": "bf16",
           "config": {"hidden_units": args.hidden_units, "in_features": args.in_features, "seq_len": args.seq_len,
                      "batch_size": args.batch_size, "vocab_size": args.vocab_size, "cuda_graph": bool(args.cuda_graph),
                      "lm_dropout_recipe": AWD_RECIPE}}
    if "step" not in skip:
        out["headline"] = step_times(args, False, dev)
    if "lm" not in skip:
        out["language_model"] = step_times(args, True, dev)
    if "launches" not in skip:
        out["launches"] = launches(args, out.get("language_model", {}).get("flat_numel", args.launch_n), dev)
    if "validation" not in skip:
        out["validation"] = validation(args, dev)
    if "regularisation" not in skip:
        out["regularisation"] = regularisation(args)
    print(json.dumps(out))


if __name__ == "__main__":
    sys.exit(main())
