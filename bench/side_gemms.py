"""Per-SM rate of the wgmma GEMM (csrc/gemm2_wgmma.cu) with single-CTA 128 x 256 tiles on a capped grid: the configuration the
pipelined layer pair runs next to a recurrence, on the SMs it leaves free.  The three shapes are the first layer's full-GPU GEMMs
of the headline step (2 x 1024 LSTM, T = 128, B = 256, D = 1024):

    gx_a  = x · W_xa^T     32768 x 4096 x 1024   (TN, bf16 out)
    dW_xa = dG_a^T · x      4096 x 1024 x 32768  (both operands MN-major, fp32 accumulate)
    dW_ha = dG_a^T · h_a    4096 x 1024 x 32768  (same kernel and shape as dW_xa)

    python bench/side_gemms.py [--reps 10]

(dW_ha is not timed separately.)  Each configuration is timed with CUDA events around ``--reps`` back-to-back launches after two
warm-up launches; the whole GPU without a cap, in 2-CTA clusters and in single CTAs, is included for reference.  Prints one JSON
line per configuration, then one with the card.
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    from lstm_tensorspark_b200.ops.cuda_ext import ext
    E = ext()
    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev).manual_seed(0)
    T, B, D, H = 128, 256, 1024, 1024
    rnd = lambda *s: (torch.randn(*s, device=dev, generator=g) * 0.1).bfloat16()
    x, w, dg = rnd(T * B, D), rnd(4 * H, D), rnd(T * B, 4 * H)
    out_bf = torch.empty(T * B, 4 * H, dtype=torch.bfloat16, device=dev)
    out_f = torch.zeros(4 * H, D, dtype=torch.float32, device=dev)
    shapes = {
        "gx_a": (lambda **k: E.gemm2(x, w, out=out_bf, bn=256, **k), T * B, 4 * H, D),
        "dW_xa": (lambda **k: E.gemm2(dg, x, out=out_f, a_mn=True, b_mn=True, accumulate=True, bn=256, **k), 4 * H, D, T * B),
    }
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    for name, (fn, M, N, K) in shapes.items():
        for ctas, cap in ((2, 0), (1, 0), (1, 16), (1, 32), (1, 64)):
            run = lambda: fn(ctas=ctas, max_ctas=cap)
            for _ in range(2):
                run()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.reps):
                run()
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / args.reps
            n_sm = cap or sms
            tflops = 2.0 * M * N * K / (ms * 1e-3) / 1e12
            print(json.dumps({"gemm": name, "shape": [M, N, K], "ctas": ctas, "max_ctas": cap, "ms": round(ms, 4),
                              "tflops": round(tflops, 1), "tflops_per_sm": round(tflops / n_sm, 3)}))
    print(json.dumps({"card": _card()}))


if __name__ == "__main__":
    main()
