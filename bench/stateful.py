"""Training throughput of stateful next-token language models (``--stateful``, one GPU) against the same model trained on
independent rows: the headline model (2-layer-1024 LSTM, T = 128, B = 256, bf16, Adam, CUDA graph) behind an embedding table and
under a softmax over the whole vocabulary, V in {4096, 32768}.

    python bench/stateful.py --steps 30 --warmup 5 --rounds 3

Arms, device-timed with CUDA events around ``--steps`` steps after ``--warmup`` steps, the two training arms alternating
``--rounds`` times in one process (so drift of the card's clock hits both alike):
  * ``rows_V<V>``: ``TrainEngine.step`` with ``next_token=True`` on 4 rotating device batches of the synthetic Markov language,
    each row starting from zero (what ``bench/next_token.py`` times);
  * ``stateful_V<V>``: the same model with ``stateful=True`` on 4 consecutive segments of one synthetic stream in 256 parallel
    streams (``data.stream_layout``): every step copies the carried state in and out, and batch 0 of each pass resets it;
  * ``carry_copies``: those copies alone (``state -> state_prev`` and the final states -> ``state`` of every layer), with the
    bytes they move computed from the shapes.
Prints one JSON line, with the card's name, power limit and maximum SM clock.  Needs a GPU; there is no fallback.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "bench"))

import torch

from variable_length import _card, _timed     # noqa: E402  (the shared helpers)


def engine(args, V, stateful, dev):
    """A captured training step and its 4 device batches -> (engine, batches)."""
    from lstm_tensorspark_b200 import data as Dm
    from lstm_tensorspark_b200.config import Config
    from lstm_tensorspark_b200.engine import TrainEngine
    B, T, nb = args.batch_size, args.seq_len, 4
    cfg = Config(hidden_units=args.hidden_units, in_features=args.in_features, seq_len=T, batch_size=B, partitions=1,
                 sync_mode="none", init="scaled", learn_initial_state=False, dtype="bf16", device="cuda", learning_rate=1e-3,
                 quiet=True, vocab_size=V, next_token=True, stateful=stateful).validate()
    eng = TrainEngine(cfg, 0, 1, None, batch_size=B, device=dev, dtype=torch.bfloat16)
    if stateful:
        x, y, _ = Dm.stream_layout(Dm.synthetic_stream(nb * B, T, V, seed=1234), B, T)
    else:
        x, y = Dm.synthetic_next_token(nb * B, T, V, seed=1234)
    dx, dy = torch.as_tensor(x).to(dev), torch.as_tensor(y).to(dev)
    batches = [(dx[i * B:(i + 1) * B], dy[i * B:(i + 1) * B]) for i in range(nb)]
    eng.step(*batches[0], reset=True)
    if args.cuda_graph:
        eng.capture(*batches[0], bind=batches[1:])
    return eng, batches


def timed_steps(args, eng, batches):
    it = {"i": 0}

    def step():
        k = it["i"] % len(batches)
        it["loss"] = eng.step(*batches[k], reset=k == 0)
        it["i"] += 1
    ms = _timed(step, args.steps, args.warmup)
    return ms, float(it["loss"])


def carry_copies(eng, reps=200):
    """The carry's copies alone: ``state -> state_prev``, then ``state_prev -> state`` standing in for the final states."""
    def copies():
        for (h, c), (hp, cp) in zip(eng.state, eng.state_prev):
            hp.copy_(h)
            cp.copy_(c)
        for (h, c), (hp, cp) in zip(eng.state, eng.state_prev):
            h.copy_(hp)
            c.copy_(cp)
    ms = _timed(copies, reps, 10)
    written = 2 * sum(h.numel() * h.element_size() + c.numel() * c.element_size() for h, c in eng.state)
    return {"ms_per_step": ms, "bytes_written_per_step": written, "bytes_moved_per_step": 2 * written,
            "launches_per_step": 4 * len(eng.state), "GB_per_s": 2 * written / (ms * 1e-3) / 1e9}


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
    ap.add_argument("--cuda_graph", type=int, default=1)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    out = {"metric": "ms/step", "unit": "ms", "n_gpus": 1, "steps": args.steps, "warmup": args.warmup, "rounds": args.rounds,
           "card": _card(), "dtype": "bf16",
           "config": {"hidden_units": args.hidden_units, "in_features": args.in_features, "seq_len": args.seq_len,
                      "batch_size": args.batch_size, "vocab_sizes": args.vocab_sizes, "cuda_graph": bool(args.cuda_graph)}}
    for V in (int(v) for v in args.vocab_sizes.split(",")):
        torch.cuda.empty_cache()
        arms = {"rows": engine(args, V, False, dev), "stateful": engine(args, V, True, dev)}
        times = {k: [] for k in arms}
        losses = {}
        for _ in range(args.rounds):
            for k, (eng, batches) in arms.items():
                ms, losses[k] = timed_steps(args, eng, batches)
                times[k].append(ms)
        for k in arms:
            out[f"{k}_V{V}"] = {"ms_per_step": statistics.median(times[k]), "ms_per_step_rounds": times[k],
                                "loss": losses[k], "value": args.batch_size * 1e3 / statistics.median(times[k])}
        out[f"stateful_over_rows_V{V}"] = out[f"stateful_V{V}"]["ms_per_step"] / out[f"rows_V{V}"]["ms_per_step"]
        out["carry_copies"] = carry_copies(arms["stateful"][0])
        from lstm_tensorspark_b200.ops import cuda_lstm
        cuda_lstm.check_kernel_errors(dev)
        del arms
    print(json.dumps(out))


if __name__ == "__main__":
    sys.exit(main())
