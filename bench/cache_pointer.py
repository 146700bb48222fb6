"""The continuous cache pointer (``--mode eval --stateful --cache_window W``, one GPU): what it adds to stream evaluation, what
its kernels reach alone, and what it does to held-out perplexity.

    python bench/cache_pointer.py --segments 8 --rounds 3

  * ``eval``: the tied language model (V = 32768, 2 x 1024, E = 1024, T = 128, bf16, random weights: the time does not depend on
    them) scores a random stream with the state carried, as ``trainer.score_stream`` does, without the cache and with it at each
    W in ``--windows``, for each B in ``--batches``.  The first ceil(max W / T) segments fill every arm's window and are not
    timed; the ``--segments`` after them are, so every timed query has a full window.  The arms alternate ``--rounds`` times in
    one process; the medians of ms per steady-state segment are reported.
  * ``kernels``: ``ops.functional.cache_pointer`` alone (ring append, scores, combine) on a segment whose history is full,
    device-timed over ``--reps`` calls.  The useful operations are those of the definition at steady state, 2 B T H W (every
    query has W keys); the kernel also multiplies the masked parts of its 128-key tiles, ``issued`` below.  TFLOP/s and the
    share of the data sheet's 989 TFLOP/s dense bf16 are of the useful count.  ``grid_ctas`` against the SM count says whether
    the key split fills the GPU at small B.
  * ``perplexity`` (a reported figure, not pass/fail, run once, untuned): the synthetic Markov language, trained with
    ``--optimizer ntasgd`` through ``trainer.run_job`` as bench/asgd.py's regularisation protocol does, then a held-out walk
    of the same chain scored with and without the cache at pointer.py's theta and lambda.
Prints one JSON line, with the card's name, power limit and maximum SM clock.  Needs a GPU; there is no fallback.  Run-time files
(the trained model's checkpoints) go to a temporary directory.
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

PEAK_TFLOPS = 989.0                                 # H100 SXM data sheet, dense bf16
KEY_TILE, QUERY_TILE = 128, 64


def useful_flops(B: int, T: int, H: int, W: int) -> int:
    """Multiply-adds of the definition for a segment whose every query has W earlier positions: 2 B T H W."""
    return 2 * B * T * H * W


def issued_flops(B: int, T: int, H: int, W: int, seen: int) -> int:
    """What the tensor-core kernel multiplies: every query tile against every 128-key tile its window touches."""
    total = 0
    for q0 in range(seen, seen + T, QUERY_TILE):
        lo, hi = max(0, q0 - W) // KEY_TILE, (q0 + QUERY_TILE - 2) // KEY_TILE
        total += (hi - lo + 1) * KEY_TILE * QUERY_TILE * H * 2
    return total * B


def _model(args, B, dev):
    from lstm_tensorspark_b200.config import Config
    from lstm_tensorspark_b200.engine import TrainEngine
    cfg = Config(hidden_units=args.hidden_units, in_features=args.hidden, seq_len=args.seq_len, batch_size=B,
                 vocab_size=args.vocab_size, next_token=True, stateful=True, tie_embeddings=True, partitions=1, sync_mode="none",
                 init="scaled", learn_initial_state=False, dtype="bf16", device="cuda", quiet=True).validate()
    eng = TrainEngine(cfg, 0, 1, None, batch_size=B, device=dev, dtype=torch.bfloat16)
    eng.model.eval()
    return eng.model


def steady_segment_ms(model, xs, ys, B: int, cache, warm: int) -> float:
    """One pass over the stream as ``trainer.score_stream`` makes it (state carried, the history reset first, a host read of the
    loss after every segment); device-timed over the segments after the first ``warm``, whose history is full."""
    segs = xs.shape[0] // B
    state = model.rnn.zero_state(B, torch.bfloat16, xs.device)
    if cache is not None:
        cache.reset()
    kw = {} if cache is None else {"cache": cache}
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for k in range(segs):
        if k == warm:
            torch.cuda.synchronize()
            e0.record()
        out = model.score(xs[k * B:(k + 1) * B], ys[k * B:(k + 1) * B], None, state=state, **kw)
        state = model.rnn.final_state()
        float(out[0])
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / (segs - warm)


def eval_times(args, dev):
    from lstm_tensorspark_b200.ops import functional as F
    out = []
    T, V = args.seq_len, args.vocab_size
    warm = -(-max(args.windows) // T)                        # segments before every query of every arm has a full window
    segs = warm + args.segments
    for B in args.batches:
        model = _model(args, B, dev)
        g = torch.Generator(device=dev).manual_seed(B)
        xs = torch.randint(0, V, (segs * B, T), generator=g, device=dev, dtype=torch.int32)
        ys = torch.randint(0, V, (segs * B, T), generator=g, device=dev)
        arms = {"none": None}
        for W in args.windows:
            arms[f"W{W}"] = F.CacheHistory(W, 0.6625523432485668, 0.12785920428335693, B, T, args.hidden, torch.bfloat16, dev)
        times = {k: [] for k in arms}
        for _ in range(args.rounds + 1):                    # the first round warms every shape up and is dropped
            for k, cache in arms.items():
                times[k].append(steady_segment_ms(model, xs, ys, B, cache, warm))
        row = {"B": B, "warm_segments": warm, "history_at_first_timed_segment": warm * T, "timed_segments": args.segments,
               "ms_per_segment": {k: statistics.median(v[1:]) for k, v in times.items()}}
        row["added_ms_per_segment"] = {k: row["ms_per_segment"][k] - row["ms_per_segment"]["none"] for k in arms if k != "none"}
        row["ring_gb"] = {k: (c.keys.numel() * 2 + c.key_labels.numel() * 4) / 1e9 for k, c in arms.items() if c is not None}
        out.append(row)
        del arms, model
        torch.cuda.empty_cache()
    return out


def kernel_times(args, dev):
    from lstm_tensorspark_b200.ops import functional as F
    from lstm_tensorspark_b200.ops.cuda_ext import ext
    T, H = args.seq_len, args.hidden
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    out = []
    for B in args.batches:
        for W in args.windows:
            g = torch.Generator(device=dev).manual_seed(W + B)
            hist = F.CacheHistory(W, 0.6625523432485668, 0.12785920428335693, B, T, H, torch.bfloat16, dev)
            h = (torch.rand(T, B, H, generator=g, device=dev) * 2 - 1).bfloat16()
            y = torch.randint(0, 1000, (B, T), generator=g, device=dev)
            lv = torch.full((T * B,), -5.0, device=dev)
            seen = -(-W // T) * T                           # a full window before the segment
            hist.keys.uniform_(-1, 1)

            def one():
                hist.seen = seen
                F.cache_pointer(h, y, lv, hist)
            ms = _timed(one, args.reps, 10)
            chunks = ext().cache_chunks(T, B, H, W)
            flops = useful_flops(B, T, H, W)
            tflops = flops / (ms * 1e-3) / 1e12
            out.append({"B": B, "W": W, "ms": ms, "useful_gflop": flops / 1e9, "issued_gflop": issued_flops(B, T, H, W, seen) / 1e9,
                        "tflops": tflops, "share_of_989": tflops / PEAK_TFLOPS, "grid_ctas": chunks * (-(-T // QUERY_TILE)) * B,
                        "sms": sms})
            del hist
            torch.cuda.empty_cache()
    return out


def perplexity(args):
    from lstm_tensorspark_b200 import data as Dm
    from lstm_tensorspark_b200.config import Config
    from lstm_tensorspark_b200.ops import functional as F
    from lstm_tensorspark_b200.trainer import _find_trained_model, _load_trained_model, run_job, score_stream
    B, T, V, nb, hid = 32, 32, 256, 60, "256,256"
    dev = torch.device("cuda")
    with tempfile.TemporaryDirectory() as tmp:
        common = dict(hidden_units=hid, in_features=256, seq_len=T, batch_size=B, vocab_size=V, next_token=True, stateful=True,
                      tie_embeddings=True, partitions=1, sync_mode="none", init="scaled", learn_initial_state=False, dtype="bf16",
                      device="cuda", quiet=True, seed=7, checkpoint_path=os.path.join(tmp, "m"), output_path=os.path.join(tmp, "o"))
        run_job(Config(synthetic=nb * B, valid_synthetic=8, optimizer="ntasgd", learning_rate=5.0, clip_grad_norm=0.25,
                       max_steps=nb * args.reg_epochs, evaluate_every=nb, **common).validate(), standalone=True)
        cfg = Config(mode="eval", synthetic=nb * B, **common).validate()
        found = _find_trained_model(cfg, True)
        eng = _load_trained_model(cfg, found, B, dev, torch.bfloat16)
        stream = Dm.synthetic_stream(16 * B, T, V, 7, valid=True)
        x, y, tail = Dm.stream_layout(stream, B, T, tail=True)
        xs, ys = torch.as_tensor(x).to(dev), torch.as_tensor(y).to(dev)
        out = {"vocab_size": V, "hidden_units": hid, "streams": B, "seq_len": T, "train_steps": nb * args.reg_epochs,
               "held_out_positions": int(xs.numel()), "chain_perplexity": math.exp(Dm.NEXT_TOKEN_ENTROPY)}
        plain = score_stream(eng.model, xs, ys, B, tail, torch.bfloat16)
        out["perplexity_model"] = math.exp(plain[0])
        for W in (100, 500):
            cache = F.CacheHistory(W, 0.6625523432485668, 0.12785920428335693, B, T, 256, torch.bfloat16, dev)
            r = score_stream(eng.model, xs, ys, B, tail, torch.bfloat16, cache=cache)
            out[f"perplexity_cache_W{W}"] = math.exp(r[0])
            out[f"perplexity_model_same_pass_W{W}"] = math.exp(r[3])
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--batches", type=lambda s: [int(v) for v in s.split(",")], default=[1, 16, 256])
    ap.add_argument("--windows", type=lambda s: [int(v) for v in s.split(",")], default=[500, 2048, 3785])
    ap.add_argument("--hidden_units", default="1024,1024")
    ap.add_argument("--hidden", type=int, default=1024)
    ap.add_argument("--vocab_size", type=int, default=32768)
    ap.add_argument("--seq_len", type=int, default=128)
    ap.add_argument("--segments", type=int, default=8)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--reg_epochs", type=int, default=6)
    ap.add_argument("--skip", default="", help="comma list of sections to skip: eval, kernels, perplexity")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench/cache_pointer.py needs a GPU")
    dev = torch.device("cuda")
    skip = set(filter(None, args.skip.split(",")))
    out = {"card": _card()}
    if "kernels" not in skip:
        out["kernels"] = kernel_times(args, dev)
    if "eval" not in skip:
        out["eval"] = eval_times(args, dev)
    if "perplexity" not in skip:
        out["perplexity"] = perplexity(args)
    out["card_after"] = _card()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
