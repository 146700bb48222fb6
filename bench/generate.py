"""Text generation throughput (``SequenceClassifier.generate``, one GPU): the headline language model (2-layer-1024 LSTM, E = 1024,
bf16, untrained ``--init scaled`` weights) behind a V-token embedding and under a V-way softmax, V in {4096, 32768}, prompts of
32 tokens and 128 new tokens at temperature 1, batch sizes 1, 64 and 256.

    python bench/generate.py --reps 5

Arms, each device-timed with CUDA events after a warm-up that captures every graph:
  * ``ours``: ``generate`` end to end, and its two parts: the prefill (the prompt through the whole-sequence path) and the decode
    loop (one replay of the captured decode step per new token), reported as ms per token and tokens/s;
  * ``split``: one decode step taken apart: the embedding and the LSTM layers' one-step launches, against the sampling launches
    (the head's tensor-core GEMM with the sampling epilogue, and the combine), each captured alone;
  * ``sample_op``: the sampling launches alone, many per graph: the bytes they must move computed from the shapes (bf16 W read
    once, h, the fp32 bias, the partials written and read back), the achieved GB/s and the share of the data sheet's HBM3
    bandwidth (``--hbm_gbps``, H100 SXM: 3.35 TB/s);
  * ``cudnn``: the stand-in ``nn.Embedding`` -> ``nn.LSTM`` with ``(h, c)`` carried -> ``nn.Linear`` -> Gumbel-max in torch ops, one
    decode step per token, captured as a CUDA graph where capture works and eager otherwise (``cuda_graph`` says which).
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

from variable_length import _card     # noqa: E402  (the shared helper)


def _events(fn, reps):
    """Device ms per call of ``fn`` over ``reps`` calls (after one call outside the window)."""
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def _graph(fn):
    fn()                                              # every kernel loaded, every workspace allocated
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
    return g


def _model(args, B, V, dev):
    from lstm_tensorspark_b200.config import Config
    from lstm_tensorspark_b200.engine import TrainEngine
    cfg = Config(hidden_units=args.hidden_units, in_features=args.in_features, seq_len=args.prompt_len, batch_size=B, partitions=1,
                 sync_mode="none", init="scaled", learn_initial_state=False, dtype="bf16", device="cuda", quiet=True,
                 vocab_size=V, next_token=True).validate()
    m = TrainEngine(cfg, 0, 1, None, batch_size=B, device=dev, dtype=torch.bfloat16).model
    m.eval()
    return m


def _prompts(args, B, V, dev):
    g = torch.Generator().manual_seed(B + V)
    x = torch.randint(0, V, (B, args.prompt_len), generator=g, dtype=torch.int32).to(dev)
    lengths = torch.full((B,), args.prompt_len, dtype=torch.int32, device=dev)
    return x, lengths


def sample_bytes(B, H, V):
    """Bytes the sampling launches must move, from the shapes: W (bf16) once, h (bf16), the bias (fp32), and the partials
    (16 + 4 B per row and 256-class tile) written by the GEMM and read by the combine; the outputs are negligible."""
    tiles = (V + 255) // 256
    return float(H * V * 2 + B * H * 2 + V * 4 + 2 * B * tiles * 20)


def ours(args, B, V, dev):
    from lstm_tensorspark_b200.ops import cuda_lstm
    from lstm_tensorspark_b200.ops import functional as F
    m = _model(args, B, V, dev)
    x, lengths = _prompts(args, B, V, dev)
    N = args.new_tokens
    n0 = cuda_lstm.STATS.get("vocab_sample", 0)
    m.generate(x, lengths, N, args.temperature, 1)                 # captures the decode step
    launched = cuda_lstm.STATS.get("vocab_sample", 0) > n0
    dec = next(d for k, d in m._decoders.items() if k[0] == B and k[1] == N)
    total_ms = _events(lambda: m.generate(x, lengths, N, args.temperature, 1), args.reps)
    with torch.no_grad():
        prefill_ms = _events(lambda: (m.sequence_features(x, lengths), dec.sample(m.rnn.layers[-1].ht)), args.reps)
    decode_ms = _events(lambda: [dec.graph.replay() for _ in range(N - 1)], args.reps) / (N - 1)

    # the decode step taken apart: layers (embedding + one step per layer + state copies) vs the sampling launches
    top = m.rnn.layers[-1].ht
    head = m.head

    def layers():
        for layer, (h, c) in zip(m.rnn.layers, dec.state):
            layer._set_state(h, c)
            layer.state = []
        m.rnn.fit_layers(m._input(dec.tokens), train=False)
        for layer, (h, c) in zip(m.rnn.layers, dec.state):
            h.copy_(layer.ht)
            c.copy_(layer.Ct)
    with torch.no_grad():
        g_layers = _graph(layers)
        step = torch.zeros(1, dtype=torch.int32, device=dev)
        K = args.sample_launches
        g_sample = _graph(lambda: [F.vocab_sample(top, head.weights, head.bias, args.temperature, 1, step) for _ in range(K)])
    layers_ms = _events(g_layers.replay, args.reps * 10)
    sample_ms = _events(g_sample.replay, args.reps) / K
    H = top.shape[1]
    nbytes = sample_bytes(B, H, V)
    return {"B": B, "V": V, "prompt_len": args.prompt_len, "new_tokens": N, "sample_launched": launched,
            "generate_ms": total_ms, "prefill_ms": prefill_ms, "decode_ms_per_token": decode_ms,
            "decode_tokens_per_s": B * 1e3 / decode_ms, "generate_tokens_per_s": B * N * 1e3 / total_ms,
            "split": {"layers_ms": layers_ms, "sample_ms": sample_ms, "sample_share": sample_ms / (layers_ms + sample_ms)},
            "sample_op": {"ms": sample_ms, "bytes": nbytes, "GBps": nbytes / (sample_ms * 1e-3) / 1e9,
                          "share_of_hbm_peak": nbytes / (sample_ms * 1e-3) / (args.hbm_gbps * 1e9),
                          "hbm_gbps_assumed": args.hbm_gbps}}


def cudnn(args, B, V, dev):
    hidden = [int(h) for h in args.hidden_units.split(",")]
    assert len(set(hidden)) == 1, "the stand-in is one nn.LSTM of equal layers"
    E, H, L = args.in_features, hidden[0], len(hidden)
    emb = torch.nn.Embedding(V, E).to(dev, torch.bfloat16)
    lstm = torch.nn.LSTM(E, H, num_layers=L).to(dev, torch.bfloat16)
    lin = torch.nn.Linear(H, V).to(dev, torch.bfloat16)
    tok = torch.randint(0, V, (B,), device=dev)
    h = torch.zeros(L, B, H, device=dev, dtype=torch.bfloat16)
    c = torch.zeros(L, B, H, device=dev, dtype=torch.bfloat16)
    inv_t = 1.0 / args.temperature

    @torch.no_grad()
    def step():
        y, (h2, c2) = lstm(emb(tok).unsqueeze(0), (h, c))
        h.copy_(h2)
        c.copy_(c2)
        logits = lin(y[0]).float()
        u = torch.rand(logits.shape, device=dev).clamp_(1e-12, 1 - 1e-7)
        tok.copy_((logits * inv_t - torch.log(-torch.log(u))).argmax(1))
    graphed = True
    try:
        g = _graph(step)
        fn = g.replay
    except Exception:                                           # noqa: BLE001  (the stand-in runs eagerly then)
        graphed, fn = False, step
    ms = _events(fn, args.reps * 20)
    return {"B": B, "V": V, "decode_ms_per_token": ms, "decode_tokens_per_s": B * 1e3 / ms, "cuda_graph": graphed}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--hidden_units", default="1024,1024")
    ap.add_argument("--in_features", type=int, default=1024)
    ap.add_argument("--vocab_sizes", default="4096,32768")
    ap.add_argument("--batch_sizes", default="1,64,256")
    ap.add_argument("--prompt_len", type=int, default=32)
    ap.add_argument("--new_tokens", type=int, default=128)
    ap.add_argument("--temperature", type=float, default=1.0)
    ap.add_argument("--sample_launches", type=int, default=50, help="sampling launches per captured graph in the sample_op arm")
    ap.add_argument("--hbm_gbps", type=float, default=3350.0, help="HBM bandwidth for the share of peak (H100 SXM: 3.35 TB/s)")
    ap.add_argument("--no_baseline", action="store_true")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    out = {"metric": "generated tokens/sec", "unit": "tokens/s", "n_gpus": 1, "card": _card(), "dtype": "bf16",
           "config": {k: getattr(args, k) for k in ("hidden_units", "in_features", "vocab_sizes", "batch_sizes", "prompt_len",
                                                    "new_tokens", "temperature", "reps")}}
    for V in (int(v) for v in args.vocab_sizes.split(",")):
        for B in (int(b) for b in args.batch_sizes.split(",")):
            torch.cuda.empty_cache()
            out[f"ours_V{V}_B{B}"] = ours(args, B, V, dev)
            if not args.no_baseline:
                torch.cuda.empty_cache()
                out[f"cudnn_V{V}_B{B}"] = cudnn(args, B, V, dev)
    last = out[f"ours_V{V}_B{B}"]
    out["value"], out["decode_ms_per_token"] = last["generate_tokens_per_s"], last["decode_ms_per_token"]
    from lstm_tensorspark_b200.ops import cuda_lstm
    cuda_lstm.check_kernel_errors(dev)
    print(json.dumps(out))


if __name__ == "__main__":
    sys.exit(main())
