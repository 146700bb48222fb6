"""Decode cost of top-k / top-p sampling (``SequenceClassifier.generate(..., top_k, top_p)``, one GPU): the headline language
model (2-layer-1024 LSTM, E = 1024, bf16, untrained ``--init scaled`` weights) under a V-way softmax, V in {4096, 32768}, batch
sizes 1, 64 and 256, prompts of 32 tokens, 64 new tokens at temperature 1.

    python bench/generate_filters.py --rounds 3

Arms: ``off`` (the unfiltered kernels), ``top_k`` 50, ``top_p`` 0.9 and ``both``.  Every arm's decode step is captured once (each
keeps its own graph and buffers), then the arms' decode loops (one replay per new token) alternate in ``--rounds`` rounds in
this process; the median ms per token is reported with the spread.  ``launches`` times the sampling launches alone, many per
captured graph, at each shape: the unfiltered sampling op, and the filtered path's parts - the ``kLogits`` GEMM, the threshold
kernel and the filtered sampling kernel with the combine - with the bytes each must move, computed from the shapes (the threshold
counted as if every pass over the logits reached HBM), the achieved GB/s and the share of the data sheet's HBM3 bandwidth
(``--hbm_gbps``, H100 SXM: 3.35 TB/s).  Prints one JSON line, with the card's name and power limit.  Needs a GPU.
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

from generate import _events, _graph, _model, _prompts, sample_bytes     # noqa: E402  (the decode benchmark's helpers)
from variable_length import _card                                       # noqa: E402

ARMS = {"off": (0, 1.0), "top_k": (50, 1.0), "top_p": (0, 0.9), "both": (50, 0.9)}


def launch_bytes(B, H, V, passes):
    """Bytes from the shapes: the kLogits GEMM reads W (bf16), h and the bias and writes the fp32 logits; the threshold reads
    the logits ``passes`` times and writes tau; the filtered sampling kernel reads the logits and tau and writes the partials,
    which the combine reads back."""
    tiles = (V + 255) // 256
    logits = B * V * 4.0
    return {"logits_gemm": H * V * 2.0 + B * H * 2 + V * 4 + logits,
            "threshold": passes * logits + B * 4,
            "filtered_sample": logits + B * 4 + 2 * B * tiles * 20}


def launches(args, m, B, V, dev, top_k, top_p):
    """The sampling launches alone, ``args.sample_launches`` per captured graph -> ms per call, bytes, GB/s, share of peak."""
    from lstm_tensorspark_b200.ops import functional as F
    from lstm_tensorspark_b200.ops.cuda_ext import ext
    from lstm_tensorspark_b200.ops.cuda_vocab_head import _weights_lowp
    K, t = args.sample_launches, args.temperature
    top, head = m.rnn.layers[-1].ht.detach().contiguous(), m.head
    wb, bias = _weights_lowp(head.weights, False), head.bias.detach().float().contiguous()
    step = torch.zeros(1, dtype=torch.int32, device=dev)
    row0 = torch.zeros(1, dtype=torch.int32, device=dev)
    tok = torch.zeros(B, dtype=torch.int32, device=dev)
    H = top.shape[1]
    passes = (4 if top_k else 0) + (5 if top_p < 1 else 0)
    nbytes = launch_bytes(B, H, V, passes)
    with torch.no_grad():
        logits = ext().vocab_head_logits(top, wb, False, bias)
        tau = ext().vocab_threshold(logits, top_k, top_p, t)
        parts = {
            "op": (lambda: F.vocab_sample(top, head.weights, head.bias, t, 1, step, top_k=top_k, top_p=top_p),
                   sum(nbytes.values()) if (top_k or top_p < 1) else sample_bytes(B, H, V)),
            "logits_gemm": (lambda: ext().vocab_head_logits(top, wb, False, bias), nbytes["logits_gemm"]),
            "threshold": (lambda: ext().vocab_threshold(logits, top_k, top_p, t), nbytes["threshold"]),
            "filtered_sample": (lambda: ext().vocab_sample_logits(logits, t, 1, step, row0, tok, None, None, 0, tau),
                                nbytes["filtered_sample"]),
        }
        if not (top_k or top_p < 1):
            parts = {"op": parts["op"]}
        graphs = {k: (_graph(lambda f=f: [f() for _ in range(K)]), b) for k, (f, b) in parts.items()}
    out = {}
    for k, (g, b) in graphs.items():
        ms = _events(g.replay, args.reps) / K
        out[k] = {"ms": ms, "bytes": b, "GBps": b / (ms * 1e-3) / 1e9, "share_of_hbm_peak": b / (ms * 1e-3) / (args.hbm_gbps * 1e9)}
    return out


def shape(args, B, V, dev):
    m = _model(args, B, V, dev)
    x, lengths = _prompts(args, B, V, dev)
    N = args.new_tokens
    decs = {}
    for arm, (k, p) in ARMS.items():
        m.generate(x, lengths, N, args.temperature, 1, top_k=k, top_p=p)              # captures this arm's decode step
        decs[arm] = next(d for key, d in m._decoders.items() if key[0] == B and key[1] == N)
    times = {arm: [] for arm in ARMS}
    for _ in range(args.rounds):
        for arm, dec in decs.items():
            times[arm].append(_events(lambda: [dec.graph.replay() for _ in range(N - 1)], args.reps) / (N - 1))
    out = {"B": B, "V": V, "new_tokens": N}
    for arm, ts in times.items():
        med = statistics.median(ts)
        out[arm] = {"decode_ms_per_token": med, "min": min(ts), "max": max(ts), "decode_tokens_per_s": B * 1e3 / med}
        if arm != "off":
            out[arm]["vs_off"] = med / statistics.median(times["off"])
    out["launches"] = {arm: launches(args, m, B, V, dev, *ARMS[arm]) for arm in ARMS}
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--hidden_units", default="1024,1024")
    ap.add_argument("--in_features", type=int, default=1024)
    ap.add_argument("--vocab_sizes", default="4096,32768")
    ap.add_argument("--batch_sizes", default="1,64,256")
    ap.add_argument("--prompt_len", type=int, default=32)
    ap.add_argument("--new_tokens", type=int, default=64)
    ap.add_argument("--temperature", type=float, default=1.0)
    ap.add_argument("--sample_launches", type=int, default=50, help="sampling launches per captured graph in the launches arm")
    ap.add_argument("--hbm_gbps", type=float, default=3350.0, help="HBM bandwidth for the share of peak (H100 SXM: 3.35 TB/s)")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    out = {"metric": "decode ms per token by sampling filter", "unit": "ms", "n_gpus": 1, "card": _card(), "dtype": "bf16",
           "arms": {k: {"top_k": v[0], "top_p": v[1]} for k, v in ARMS.items()},
           "config": {k: getattr(args, k) for k in ("hidden_units", "in_features", "vocab_sizes", "batch_sizes", "prompt_len",
                                                    "new_tokens", "temperature", "rounds", "reps")}}
    for V in (int(v) for v in args.vocab_sizes.split(",")):
        for B in (int(b) for b in args.batch_sizes.split(",")):
            torch.cuda.empty_cache()
            out[f"V{V}_B{B}"] = shape(args, B, V, dev)
    from lstm_tensorspark_b200.ops import cuda_lstm
    cuda_lstm.check_kernel_errors(dev)
    print(json.dumps(out))


if __name__ == "__main__":
    sys.exit(main())
