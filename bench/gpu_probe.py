#!/usr/bin/env python
"""GPU bring-up probe: runs every kernel check in its OWN subprocess under a timeout (a faulting kernel poisons
its CUDA context — it must not take the other checks down) and appends results to gpurun_out/probe.jsonl.

    python bench/gpu_probe.py [check ...]        # no args = all checks
"""
from __future__ import annotations

import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
OUT = os.path.join(ROOT, "gpurun_out")


def _emit(name, **kw):
    os.makedirs(OUT, exist_ok=True)
    rec = {"check": name, **kw}
    with open(os.path.join(OUT, "probe.jsonl"), "a") as f:
        f.write(json.dumps(rec, default=str) + "\n")
    print("PROBE", json.dumps(rec, default=str), flush=True)


def _time_ms(fn, iters=10, warm=3):
    import torch
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


# ---------------------------------------------------------------------------------------------------------
def check_env():
    import torch
    p = torch.cuda.get_device_properties(0)
    _emit("env", gpu=p.name, sms=p.multi_processor_count, mem_gb=p.total_memory / 2**30, cc=f"{p.major}.{p.minor}",
          torch=torch.__version__, n_gpus=torch.cuda.device_count())


def check_simple():
    import torch
    from lstm_tensorspark_b200.ops.cuda_ext import ext
    from lstm_tensorspark_b200.ops import reference as ref
    E = ext()
    dev = torch.device("cuda")
    torch.manual_seed(0)
    for dt in (torch.float32, torch.bfloat16):
        B, H = 37, 24
        pre = torch.randn(B, 4 * H, device=dev).to(dt)
        bias = torch.randn(4 * H, device=dev)
        c = torch.randn(B, H, device=dev)
        h, cn, act = E.lstm_pointwise_fwd(pre, bias, c)
        i, f, g, o = ref.lstm_gates(pre.float() + bias)
        c_ref = f * c + i * g
        h_ref = o * torch.tanh(c_ref)
        _emit("pointwise_fwd", dtype=str(dt), h_err=float((h.float() - h_ref).abs().max()), c_err=float((cn - c_ref).abs().max()))
    # head
    B, H, C = 50, 96, 7
    hh = torch.randn(B, H, device=dev)
    W = torch.randn(H, C, device=dev) * 0.1
    b = torch.randn(C, device=dev)
    y = torch.randint(0, C, (B,), device=dev)
    logits, dlog, loss, corr = E.head_fwd(hh, W, b, y)
    lr, lossr, corrr = ref.head_xent(hh, W, b, y)
    _emit("head_xent", logit_err=float((logits - lr).abs().max()), loss=float(loss / B), loss_ref=float(lossr), correct=int(corr), correct_ref=int(corrr))
    # adam
    n = 16384
    p = torch.randn(n, device=dev); g = torch.randn(n, device=dev); m = torch.zeros(n, device=dev); v = torch.zeros(n, device=dev)
    p2, m2, v2 = p.clone(), m.clone(), v.clone()
    sh = torch.empty(n, dtype=torch.bfloat16, device=dev)
    lr_t = 1e-3 * (1 - 0.999) ** 0.5 / (1 - 0.9)
    E.flat_adam(p, g, m, v, sh, lr_t, 0.9, 0.999, 1e-8, 0.0, 1.0)
    ref.adam_step_(p2, g, m2, v2, 1, 1e-3)
    _emit("flat_adam", p_err=float((p - p2).abs().max()), shadow_err=float((sh.float() - p).abs().max()))


def check_gemm2():
    """General wgmma GEMM: every operand-major combination, 1- and 2-CTA tiles, accumulate, ragged shapes, then timing
    of the training-step shapes against cuBLAS."""
    import torch
    from lstm_tensorspark_b200.ops.cuda_ext import ext
    E = ext()
    dev = torch.device("cuda")
    torch.manual_seed(0)
    small = [(128, 128, 64), (256, 256, 128), (512, 512, 256), (1000, 520, 264), (384, 1024, 1024)]
    for ctas, bn in ((1, 128), (1, 256), (2, 128), (2, 256)):
        for a_mn in (False, True):
            for b_mn in (False, True):
                worst = 0.0
                for (M, N, K) in small:
                    A = (torch.randn(K, M, device=dev) * 0.5).bfloat16() if a_mn else (torch.randn(M, K, device=dev) * 0.5).bfloat16()
                    Bm = (torch.randn(K, N, device=dev) * 0.5).bfloat16() if b_mn else (torch.randn(N, K, device=dev) * 0.5).bfloat16()
                    R = (A.float().t() if a_mn else A.float()) @ (Bm.float() if b_mn else Bm.float().t())
                    try:
                        C16 = E.gemm2(A, Bm, a_mn=a_mn, b_mn=b_mn, ctas=ctas, bn=bn)
                        C32 = E.gemm2(A, Bm, a_mn=a_mn, b_mn=b_mn, out_fp32=True, ctas=ctas, bn=bn)
                        acc = torch.ones(M, N, device=dev)
                        E.gemm2(A, Bm, out=acc, a_mn=a_mn, b_mn=b_mn, accumulate=True, ctas=ctas, bn=bn)
                        torch.cuda.synchronize()
                        scale = float(R.abs().max())
                        e16 = float((C16.float() - R).abs().max()) / scale
                        e32 = float((C32 - R).abs().max()) / scale
                        eac = float((acc - 1.0 - R).abs().max()) / scale
                        worst = max(worst, e16 / 8.0, e32, eac)       # bf16 output rounding allowed 8x
                        if max(e32, eac) > 2e-3 or e16 > 1.6e-2:
                            _emit("gemm2_MISMATCH", ctas=ctas, bn=bn, a_mn=a_mn, b_mn=b_mn, M=M, N=N, K=K, e16=e16, e32=e32, eacc=eac)
                    except Exception as e:            # noqa: BLE001
                        _emit("gemm2_ERROR", ctas=ctas, bn=bn, a_mn=a_mn, b_mn=b_mn, M=M, N=N, K=K, error=repr(e)[:300])
                        raise
                _emit("gemm2", ctas=ctas, bn=bn, a_mn=a_mn, b_mn=b_mn, worst_rel_err=worst)
    # strided operands (views of wider buffers)
    big = (torch.randn(512, 1536, device=dev) * 0.5).bfloat16()
    A, Bm = big[:, :512], big[:256, 512:1024]
    C = E.gemm2(A, Bm, out_fp32=True)
    R = A.float() @ Bm.float().t()
    _emit("gemm2_strided", rel_err=float((C - R).abs().max() / R.abs().max()))
    # timing: x-projection (TN), dX (NN), dW (NT = both MN-major), head-sized
    TB, H4, D = 32768, 4096, 1024
    X = (torch.randn(TB, D, device=dev) * 0.5).bfloat16()
    W = (torch.randn(H4, D, device=dev) * 0.05).bfloat16()
    dG = (torch.randn(TB, H4, device=dev) * 0.5).bfloat16()
    gw = torch.zeros(H4, D, device=dev)
    for ctas, bn in ((1, 256), (2, 256), (2, 128)):
        ms = _time_ms(lambda: E.gemm2(X, W, ctas=ctas, bn=bn))
        _emit("gemm2_time", what="gx = X Wx^T", ctas=ctas, bn=bn, ms=ms, tflops=2.0 * TB * H4 * D / ms / 1e9)
        ms = _time_ms(lambda: E.gemm2(dG, W, b_mn=True, ctas=ctas, bn=bn))
        _emit("gemm2_time", what="dX = dG Wx", ctas=ctas, bn=bn, ms=ms, tflops=2.0 * TB * H4 * D / ms / 1e9)
        ms = _time_ms(lambda: E.gemm2(dG, X, out=gw, a_mn=True, b_mn=True, accumulate=True, ctas=ctas, bn=bn))
        _emit("gemm2_time", what="dW += dG^T X", ctas=ctas, bn=bn, ms=ms, tflops=2.0 * TB * H4 * D / ms / 1e9)
    ms = _time_ms(lambda: X @ W.t())
    _emit("gemm2_time", what="cuBLAS gx", ms=ms, tflops=2.0 * TB * H4 * D / ms / 1e9)
    ms = _time_ms(lambda: dG @ W)
    _emit("gemm2_time", what="cuBLAS dX", ms=ms, tflops=2.0 * TB * H4 * D / ms / 1e9)
    ms = _time_ms(lambda: torch.addmm(gw, dG.t(), X, out_dtype=torch.float32, out=gw))
    _emit("gemm2_time", what="cuBLAS dW", ms=ms, tflops=2.0 * TB * H4 * D / ms / 1e9)
    R = dG[:, :256].float().t() @ X.float()
    gw.zero_()
    E.gemm2(dG, X, out=gw, a_mn=True, b_mn=True, accumulate=True)
    _emit("gemm2_dw_check", rel_err=float((gw[:256] - R).abs().max() / R.abs().max()))


def check_gemm2_dw():
    """Why is the NT (both MN-major) weight-gradient product slower than the TN ones?  Isolate operand major, K length, grid."""
    import torch
    from lstm_tensorspark_b200.ops.cuda_ext import ext
    E = ext()
    dev = torch.device("cuda")
    torch.manual_seed(0)
    TB, H4, D = 32768, 4096, 1024
    X = (torch.randn(TB, D, device=dev) * 0.5).bfloat16()
    XT = X.t().contiguous()                      # [D, TB]
    W = (torch.randn(H4, D, device=dev) * 0.05).bfloat16()
    WT = W.t().contiguous()                      # [D, 4H]
    dG = (torch.randn(TB, H4, device=dev) * 0.5).bfloat16()
    dGT = dG.t().contiguous()                    # [4H, TB]
    gw = torch.zeros(H4, D, device=dev)
    fl = 2.0 * TB * H4 * D
    def t(what, fn):
        ms = _time_ms(fn)
        _emit("gemm2_dw", what=what, ms=ms, tflops=fl / ms / 1e9)
    t("gx TN (A K-major, B K-major)", lambda: E.gemm2(X, W))
    t("gx with A MN-major (X^T stored)", lambda: E.gemm2(XT, W, a_mn=True))
    t("gx with B MN-major (W^T stored)", lambda: E.gemm2(X, WT, b_mn=True))
    t("gx both MN-major", lambda: E.gemm2(XT, WT, a_mn=True, b_mn=True))
    t("dW NT both MN (dG, X)", lambda: E.gemm2(dG, X, out=gw, a_mn=True, b_mn=True, accumulate=True))
    t("dW NT overwrite", lambda: E.gemm2(dG, X, out=gw, a_mn=True, b_mn=True, out_fp32=True))
    t("dW TN on transposed copies (dG^T, X^T K-major)", lambda: E.gemm2(dGT, XT, out=gw, out_fp32=True))
    t("dW A K-major (dG^T), B MN (X)", lambda: E.gemm2(dGT, X, out=gw, b_mn=True, out_fp32=True))
    t("dW A MN (dG), B K-major (X^T)", lambda: E.gemm2(dG, XT, out=gw, a_mn=True, out_fp32=True))
    for mc in (64, 96, 128, 132):
        t(f"dW NT max_ctas={mc}", lambda: E.gemm2(dG, X, out=gw, a_mn=True, b_mn=True, out_fp32=True, max_ctas=mc))
    t("dW NT 1-CTA bn256", lambda: E.gemm2(dG, X, out=gw, a_mn=True, b_mn=True, out_fp32=True, ctas=1, bn=256))
    t("dW NT 2-CTA bn128", lambda: E.gemm2(dG, X, out=gw, a_mn=True, b_mn=True, out_fp32=True, ctas=2, bn=128))
    for mc in (96, 128):
        t(f"gx TN max_ctas={mc}", lambda: E.gemm2(X, W, max_ctas=mc))


def check_wave():
    """Layer-wavefront bring-up: the three co-resident kernels piece by piece, dumping the dataflow counters after each stage."""
    import torch
    from lstm_tensorspark_b200.ops import cuda_lstm as CL
    from lstm_tensorspark_b200.ops.cuda_ext import ext
    E = ext()
    dev = torch.device("cuda")
    torch.manual_seed(0)
    T, B, D, Ha, Hb = 6, 256, 256, 1024, 1024
    cd = torch.bfloat16
    x2d = (torch.randn(T * B, D, device=dev) * 0.5).to(cd)
    wxa = (torch.randn(4 * Ha, D, device=dev) * D ** -0.5).to(cd); wha = (torch.randn(4 * Ha, Ha, device=dev) * Ha ** -0.5).to(cd)
    wxb = (torch.randn(4 * Hb, Ha, device=dev) * Ha ** -0.5).to(cd); whb = (torch.randn(4 * Hb, Hb, device=dev) * Hb ** -0.5).to(cd)
    ba = torch.zeros(4 * Ha, device=dev); bb = torch.zeros(4 * Hb, device=dev)
    h0a = torch.zeros(B, Ha, device=dev, dtype=cd); c0a = torch.zeros(B, Ha, device=dev)
    h0b = torch.zeros(B, Hb, device=dev, dtype=cd); c0b = torch.zeros(B, Hb, device=dev)
    gx_a = E.gemm2(x2d, wxa).view(T, B, 4 * Ha)
    opt = dict(dtype=cd, device=dev)
    def bufs(H):
        return (torch.empty(T + 1, B, H, **opt), torch.empty(T + 1, B, H, dtype=torch.float32, device=dev), torch.empty(T, B, 4 * H, **opt),
                torch.empty((T + 1) * 2 * 128 * H, **opt))
    tn = 4 * Hb // 256
    ws_a, ws_b, done = CL._pair_ws(dev, "probe", T * tn * 2)
    var = 2
    def ctrs(ws, n):
        return [int(v) for v in ws[512:512 + 32 * n:32].cpu()]
    # stage 1: L_a alone, two tiles per CTA, extra signal
    ws_a.zero_(); ws_b.zero_(); done.zero_()
    ha, ca, aa, ta = bufs(Ha)
    E.lstm_seq_fwd_into(gx_a, wha, ba, h0a, c0a, ha, ca, aa, ta, ws_a, var, None, 0, True, 0)
    torch.cuda.synchronize()
    ref_h, _, _ = E.lstm_seq_fwd(gx_a, wha, ba, h0a, c0a, CL._sync_ws(dev), 0)
    torch.cuda.synchronize()
    _emit("wave_stage1", err=int(ws_a[-1]), counters=ctrs(ws_a, 32)[:6], expect=4 * (T + 1), h_diff=float((ha.float() - ref_h.float()).abs().max()))
    # stage 2: + gated GEMM on a side stream (L_a re-run so that the GEMM really waits)
    ws_a.zero_(); done.zero_()
    gx_b = torch.zeros(T, B, 4 * Hb, **opt)
    s1 = torch.cuda.Stream()
    main = torch.cuda.current_stream()
    ev = torch.cuda.Event(); ev.record(main); s1.wait_event(ev)
    E.lstm_seq_fwd_into(gx_a, wha, ba, h0a, c0a, ha, ca, aa, ta, ws_a, var, None, 0, True, main.cuda_stream)
    E.gemm2(ha[1:].view(T * B, Ha), wxb, out=gx_b.view(T * B, 4 * Hb), ctas=1, bn=256, max_ctas=20, gate=ws_a[512:],
            gate_cfg=[2 * (Ha // 64), 32, 8, 4, B, 1, 0], done=done, gate_err=ws_a[-1:], stream=s1.cuda_stream)
    torch.cuda.synchronize()
    ref_gx = (ha[1:].reshape(T * B, Ha).float() @ wxb.float().t()).view(T, B, 4 * Hb)
    _emit("wave_stage2", err=int(ws_a[-1]), done_min=int(done.min()), done_max=int(done.max()), done_n=int(done.numel()),
          gx_rel=float((gx_b.float() - ref_gx).abs().max() / ref_gx.abs().max()))
    # stage 3: all three
    ws_a.zero_(); ws_b.zero_(); done.zero_()
    hb, cb, ab, tb = bufs(Hb)
    s2 = torch.cuda.Stream()
    ev = torch.cuda.Event(); ev.record(main); s1.wait_event(ev); s2.wait_event(ev)
    E.lstm_seq_fwd_into(gx_a, wha, ba, h0a, c0a, ha, ca, aa, ta, ws_a, var, None, 0, True, main.cuda_stream)
    E.lstm_seq_fwd_into(gx_b, whb, bb, h0b, c0b, hb, cb, ab, tb, ws_b, var, done, tn, False, s2.cuda_stream)
    E.gemm2(ha[1:].view(T * B, Ha), wxb, out=gx_b.view(T * B, 4 * Hb), ctas=1, bn=256, max_ctas=20, gate=ws_a[512:],
            gate_cfg=[2 * (Ha // 64), 32, 8, 4, B, 1, 0], done=done, gate_err=ws_a[-1:], stream=s1.cuda_stream)
    try:
        torch.cuda.synchronize()
        ref_hb, _, _ = E.lstm_seq_fwd(ref_gx.to(cd), whb, bb, h0b, c0b, CL._sync_ws(dev), 0)
        torch.cuda.synchronize()
        _emit("wave_stage3", err_a=int(ws_a[-1]), err_b=int(ws_b[-1]), a_ctr=ctrs(ws_a, 32)[:4], b_ctr=ctrs(ws_b, 32)[:4],
              done_min=int(done.min()), done_max=int(done.max()), hb_diff=float((hb.float() - ref_hb.float()).abs().max()))
    except Exception as e:           # noqa: BLE001
        _emit("wave_stage3_EXC", error=repr(e)[:300])
        raise


def check_wave_bwd():
    """Backward half of the wavefront through the autograd op; dumps the dataflow counters of all three kernels afterwards."""
    import torch
    from lstm_tensorspark_b200.ops import cuda_lstm as CL
    dev = torch.device("cuda")
    torch.manual_seed(11)
    import os
    last_only = os.environ.get("LAST_ONLY", "0") == "1"
    for (T, Ha, Hb, D) in ((6, 1024, 1024, 256), (128, 1024, 1024, 1024)):
        B = 256
        mk = lambda *s, sc=1.0: (torch.randn(*s, device=dev) * sc)
        x = mk(T, B, D, sc=0.5).bfloat16()
        pa = [mk(B, Ha, sc=0.1), mk(B, Ha, sc=0.1), mk(4 * Ha, D, sc=D ** -0.5), mk(4 * Ha, Ha, sc=Ha ** -0.5), mk(4 * Ha, sc=0.1)]
        pb = [mk(B, Hb, sc=0.1), mk(B, Hb, sc=0.1), mk(4 * Hb, Ha, sc=Ha ** -0.5), mk(4 * Hb, Hb, sc=Hb ** -0.5), mk(4 * Hb, sc=0.1)]
        wgt = mk(T, B, Hb)
        def run(pair):
            xa = x.clone().requires_grad_(True)
            a = [p.clone().requires_grad_(True) for p in pa]
            b = [p.clone().requires_grad_(True) for p in pb]
            if pair:
                hs, hTa, cTa, hTb, cTb = CL.lstm_pair_sequence(xa, a, b)
            else:
                hs_a, hTa, cTa = CL.lstm_layer_sequence(xa, *a)
                hs, hTb, cTb = CL.lstm_layer_sequence(hs_a, *b)
            loss = hTb.float().sum() if last_only else (hs.float() * wgt).sum() + hTa.float().sum() + hTb.float().sum()
            torch.cuda.synchronize()
            t0 = time.time()
            loss.backward()
            torch.cuda.synchronize()
            return [hs.detach().float(), xa.grad.float()] + [p.grad.float() for p in a + b if p.grad is not None], time.time() - t0
        ref, _ = run(False)
        try:
            got, dt = run(True)
        except Exception as e:       # noqa: BLE001
            got, dt = None, -1.0
            _emit("wave_bwd_EXC", T=T, error=repr(e)[:200])
        def c(tag, i, n):
            ent = CL._WS_PAIR.get((0, tag))
            if ent is None:
                return None
            ws = ent[i * 8192:(i + 1) * 8192]
            return {"err": int(ws[-1]), "ctr": [int(v) for v in ws[512:512 + 32 * n:32].cpu()][:5]}
        ent = CL._WS_PAIR.get((0, "bwd"))
        dn = ent[2 * 8192:2 * 8192 + T * (Ha // 256) * 2] if ent is not None else None
        rel = None
        if got is not None:
            rel = [float((g - r).norm() / (r.norm() + 1e-30)) for g, r in zip(got, ref)]
        _emit("wave_bwd", T=T, seconds=dt, head_b=c("bwd", 0, 128), tail_a=c("bwd", 1, 128), fwd_a=c("fwd", 0, 32), fwd_b=c("fwd", 1, 32),
              done_min=None if dn is None else int(dn.min()), done_zero=None if dn is None else int((dn == 0).sum()), rel=rel)


def _seq_case(T, B, H, D, check_bwd=True, time_it=False):
    import torch
    from lstm_tensorspark_b200.ops import cuda_lstm, reference as ref
    from lstm_tensorspark_b200.ops.cuda_ext import ext
    dev = torch.device("cuda")
    torch.manual_seed(1)
    x = (torch.randn(T, B, D, device=dev) * 0.5)
    w_x = (torch.randn(4 * H, D, device=dev) / D ** 0.5)
    w_h = (torch.randn(4 * H, H, device=dev) / H ** 0.5)
    bias = torch.randn(4 * H, device=dev) * 0.1
    h0 = torch.randn(B, H, device=dev) * 0.1
    c0 = torch.randn(B, H, device=dev) * 0.1
    params = [x, h0, c0, w_x, w_h, bias]
    # reference in fp32 on bf16-rounded operands
    pr = [p.bfloat16().float().requires_grad_(True) if i != 2 else p.clone().requires_grad_(True) for i, p in enumerate(params)]
    hs_r, hT_r, cT_r = ref.lstm_layer_sequence(*pr)
    wgt = torch.randn_like(hs_r)
    (hs_r * wgt).sum().backward()
    pc = [p.clone().requires_grad_(True) for p in params]
    xb = pc[0].bfloat16()
    hs, hT, cT = cuda_lstm.lstm_layer_sequence(xb, pc[1], pc[2], pc[3], pc[4], pc[5])
    torch.cuda.synchronize()
    cuda_lstm.check_kernel_errors(dev)
    out = dict(T=T, B=B, H=H, D=D, fast=cuda_lstm.STATS["fast_fwd"] > 0,
               h_err=float((hs.float() - hs_r).abs().max()), c_err=float((cT - cT_r).abs().max()), h_ref_max=float(hs_r.abs().max()))
    if check_bwd:
        (hs.float() * wgt).sum().backward()
        torch.cuda.synchronize()
        cuda_lstm.check_kernel_errors(dev)
        names = ["dx", "dh0", "dc0", "dw_x", "dw_h", "db"]
        for n, a, b in zip(names, pc, pr):
            out[n + "_rel"] = float((a.grad.float() - b.grad).abs().max() / (b.grad.abs().max() + 1e-12))
    if time_it:
        E = ext()
        gx = (xb.reshape(T * B, D) @ w_x.bfloat16().t()).view(T, B, 4 * H).contiguous()
        whb = w_h.bfloat16().contiguous()
        ws = cuda_lstm._sync_ws(dev)
        out["fwd_kernel_ms"] = _time_ms(lambda: E.lstm_seq_fwd(gx, whb, bias, h0.bfloat16(), c0, ws, 0), iters=5, warm=2)
        out["fwd_us_per_step"] = out["fwd_kernel_ms"] * 1e3 / T
        hseq, cseq, act = E.lstm_seq_fwd(gx, whb, bias, h0.bfloat16(), c0, ws, 0)
        whT = whb.t().contiguous()
        dh = torch.randn(T, B, H, device=dev).bfloat16()
        z = torch.zeros(B, H, device=dev)
        out["bwd_kernel_ms"] = _time_ms(lambda: E.lstm_seq_bwd(dh, whT, act, cseq, z, z, ws, 0), iters=5, warm=2)
        out["bwd_us_per_step"] = out["bwd_kernel_ms"] * 1e3 / T
        cuda_lstm.check_kernel_errors(dev)
    _emit("lstm_seq", **out)


def check_seq_small():
    _seq_case(3, 128, 64, 64)
    _seq_case(5, 100, 128, 72)
    _seq_case(4, 256, 256, 128)


def check_seq_big():
    _seq_case(16, 256, 1024, 1024, check_bwd=True, time_it=True)
    _seq_case(128, 256, 1024, 1024, check_bwd=False, time_it=True)


def check_seq_tune():
    """Per-phase timestamps of CTA 0 (wait-done / accumulator-ready / signalled) + per-k-block TMA issue -> landed times."""
    import torch
    from lstm_tensorspark_b200.ops import cuda_lstm
    from lstm_tensorspark_b200.ops.cuda_ext import ext
    E = ext()
    dev = torch.device("cuda")
    for (T, B, H) in ((128, 256, 1024),):
        torch.manual_seed(0)
        gx = (torch.randn(T, B, 4 * H, device=dev) * 0.5).bfloat16()
        whb = (torch.randn(4 * H, H, device=dev) / H ** 0.5).bfloat16()
        bias = torch.zeros(4 * H, device=dev)
        h0 = torch.zeros(B, H, device=dev).bfloat16(); c0 = torch.zeros(B, H, device=dev)
        ws = cuda_lstm._sync_ws(dev)
        for (tiles, st, mode, sync, acq, nosplit) in ((1, 0, 0, 1, 0, 1), (1, 0, 0, 0, 0, 1), (1, 0, 0, 1, 0, 0), (1, 0, 0, 0, 0, 0), (1, 4, 0, 0, 0, 0), (1, 0, 5, 0, 0, 0)):
            v = tiles + 16 * st + 4096 * mode + 65536 * sync + 262144 * acq + 524288 * nosplit
            try:
                ms = _time_ms(lambda: E.lstm_seq_fwd(gx, whb, bias, h0, c0, ws, v), iters=5, warm=2)
                dbg = torch.zeros(4 * (T + 2) + 64 + 512, dtype=torch.int64, device=dev)
                E.lstm_seq_fwd(gx, whb, bias, h0, c0, ws, v, dbg)
                torch.cuda.synchronize()
                cuda_lstm.check_kernel_errors(dev)
                d = dbg[:4 * (T + 2)].view(-1, 4)[8:24].cpu()
                waited, accum, sig = d[:, 0], d[:, 1], d[:, 2]
                nk = H // 64
                kb = dbg[4 * (T + 2):].cpu()
                t0 = int(d[0, 0])
                issue = [(int(x) - t0) for x in kb[:nk]]
                landed = [(int(x) - t0) for x in kb[32:32 + nk]]
                w3 = dbg[:4 * (T + 2)].view(-1, 4)[8:24, 3].cpu()
                mma_first = [int(x) & 0xFFFFF for x in w3]
                mma_wait = [(int(x) >> 20) & 0xFFFFF for x in w3]
                mma_total = [(int(x) >> 40) & 0xFFFFF for x in w3]
                e = dbg[4 * (T + 2):4 * (T + 2) + 3].cpu()
                acc8, sig8 = int(d[0, 1]), int(d[0, 2])
                _emit("fwd_variant", T=T, B=B, H=H, tiles=tiles, stages=st, debug_mode=mode, sync=sync, acq=acq, nosplit=nosplit, us_per_step=ms * 1e3 / T,
                      mma_first_wait_cyc=sum(mma_first) / 16, mma_later_wait_cyc=sum(mma_wait) / 16, mma_step_cyc=sum(mma_total) / 16,
                      epi_ld_ns=int(e[0]) - acc8, epi_math_store_ns=int(e[1]) - int(e[0]), epi_bar_ns=int(e[2]) - int(e[1]), epi_signal_ns=sig8 - int(e[2]),
                      load_mma_us=float((accum - waited).float().mean()) / 1e3, epi_us=float((sig - accum).float().mean()) / 1e3,
                      sync_us=float((waited[1:] - sig[:-1]).float().mean()) / 1e3, 
                      accum_ns=int(d[0, 1]) - t0)
            except Exception as e:                     # noqa: BLE001
                _emit("fwd_variant", T=T, B=B, H=H, tiles=tiles, stages=st, error=repr(e)[:300])


def check_tiles2_tune():
    """The two-tiles-per-CTA kernels the layer wavefront launches (64 CTAs per layer), one layer alone: ring depth / sync mode."""
    import torch
    from lstm_tensorspark_b200.ops import cuda_lstm
    from lstm_tensorspark_b200.ops.cuda_ext import ext
    E = ext()
    dev = torch.device("cuda")
    T, B, H = 128, 256, 1024
    torch.manual_seed(0)
    gx = (torch.randn(T, B, 4 * H, device=dev) * 0.5).bfloat16()
    whb = (torch.randn(4 * H, H, device=dev) / H ** 0.5).bfloat16()
    whT = whb.t().contiguous()
    bias = torch.zeros(4 * H, device=dev)
    h0 = torch.zeros(B, H, device=dev).bfloat16(); c0 = torch.zeros(B, H, device=dev)
    ws = cuda_lstm._sync_ws(dev)
    hseq, cseq, act = E.lstm_seq_fwd(gx, whb, bias, h0, c0, ws, 2)
    dh = torch.randn(T, B, H, device=dev).bfloat16()
    z = torch.zeros(B, H, device=dev)
    for st in (0, 4, 5, 6):
        for sync in (0, 1, 2):
            v = 2 + 16 * st + 65536 * sync
            try:
                ms = _time_ms(lambda: E.lstm_seq_fwd(gx, whb, bias, h0, c0, ws, v), iters=5, warm=2)
                cuda_lstm.check_kernel_errors(dev)
                _emit("tiles2_fwd", stages=st, sync=sync, us_per_step=ms * 1e3 / T)
            except Exception as e:        # noqa: BLE001
                _emit("tiles2_fwd", stages=st, sync=sync, error=repr(e)[:200])
    for st in (0, 3, 4):
        for sync in (0, 1, 2):
            v = 2 + 16 * st + 65536 * sync
            try:
                ms = _time_ms(lambda: E.lstm_seq_bwd(dh, whT, act, cseq, z, z, ws, v), iters=5, warm=2)
                cuda_lstm.check_kernel_errors(dev)
                _emit("tiles2_bwd", stages=st, sync=sync, us_per_step=ms * 1e3 / (T + 1))
            except Exception as e:        # noqa: BLE001
                _emit("tiles2_bwd", stages=st, sync=sync, error=repr(e)[:200])
    # one tile per CTA on 128 CTAs (the single-layer default), for reference
    for v, nm in ((0, "ksplit_default"), (524288, "nosplit")):
        ms = _time_ms(lambda: E.lstm_seq_fwd(gx, whb, bias, h0, c0, ws, v), iters=5, warm=2)
        _emit("tiles1_fwd", variant=nm, us_per_step=ms * 1e3 / T)
    ms = _time_ms(lambda: E.lstm_seq_bwd(dh, whT, act, cseq, z, z, ws, 0), iters=5, warm=2)
    _emit("tiles1_bwd", us_per_step=ms * 1e3 / (T + 1))


def check_tiles2_phase():
    """Per-step phase split of the two-tiles-per-CTA kernels (64 CTAs per layer, the headline's recurrences), from the time
    stamps of CTA 0's first tile: first operand block ready -> accumulator ready (load_mma_us), accumulator ready -> dataflow
    signal sent (epi_us), signal -> next step's first block ready (sync_us).  debug_mode 1 skips the operand loads (garbage
    results): how much of the step the operand stream costs.
    Per warpgroup (= tile, ping-pong schedule): MMA start -> accumulator ready (wgN_mma_us), accumulator ready -> signal
    (wgN_epi_us), and how much of warpgroup 1's MMA window falls inside warpgroup 0's epilogue (wg1_mma_in_wg0_epi_us)."""
    import torch
    from lstm_tensorspark_b200.ops import cuda_lstm
    from lstm_tensorspark_b200.ops.cuda_ext import ext
    E = ext()
    dev = torch.device("cuda")
    T, B, H = 128, 256, 1024
    torch.manual_seed(0)
    gx = (torch.randn(T, B, 4 * H, device=dev) * 0.5).bfloat16()
    whb = (torch.randn(4 * H, H, device=dev) / H ** 0.5).bfloat16()
    whT = whb.t().contiguous()
    bias = torch.zeros(4 * H, device=dev)
    h0 = torch.zeros(B, H, device=dev).bfloat16(); c0 = torch.zeros(B, H, device=dev)
    ws = cuda_lstm._sync_ws(dev)
    _, cseq, act = E.lstm_seq_fwd(gx, whb, bias, h0, c0, ws, 2)
    dh = (torch.randn(T, B, H, device=dev) * 0.1).bfloat16()
    z = torch.zeros(B, H, device=dev)
    runs = {"fwd": lambda v, dbg=None: E.lstm_seq_fwd(gx, whb, bias, h0, c0, ws, v, dbg),
            "bwd": lambda v, dbg=None: E.lstm_seq_bwd(dh, whT, act, cseq, z, z, ws, v, dbg)}
    for direction, run in runs.items():
        steps = T if direction == "fwd" else T + 1
        first = 8 if direction == "fwd" else 9              # skip the first steps (the backward pass stamps from s = 1)
        for mode in (0, 1):
            v = 2 + 4096 * mode
            try:
                ms = _time_ms(lambda: run(v), iters=5, warm=2)
                tile1 = 4 * (T + 2) + 64 + 512                # the second tile's [steps][4] stamps start here
                dbg = torch.zeros(tile1 + 4 * (T + 2), dtype=torch.int64, device=dev)
                run(v, dbg)
                torch.cuda.synchronize()
                cuda_lstm.check_kernel_errors(dev)
                d = dbg[:4 * (T + 2)].view(-1, 4)[first:steps - 8].cpu()
                d1 = dbg[tile1:].view(-1, 4)[first:steps - 8].cpu()
                waited, accum, sig = d[:, 0], d[:, 1], d[:, 2]

                def us(x):
                    return float(x.double().mean()) / 1e3
                overlap = (torch.minimum(d1[:, 1], d[:, 2]) - torch.maximum(d1[:, 3], d[:, 1])).clamp(min=0)
                _emit("tiles2_phase", direction=direction, debug_mode=mode, us_per_step=ms * 1e3 / steps,
                      load_mma_us=us(accum - waited), epi_us=us(sig - accum), sync_us=us(waited[1:] - sig[:-1]),
                      wg0_mma_us=us(d[:, 1] - d[:, 3]), wg0_epi_us=us(d[:, 2] - d[:, 1]),
                      wg1_mma_us=us(d1[:, 1] - d1[:, 3]), wg1_epi_us=us(d1[:, 2] - d1[:, 1]),
                      wg1_mma_start_after_wg0_acc_us=us(d1[:, 3] - d[:, 1]), wg1_mma_in_wg0_epi_us=us(overlap))
            except Exception as e:                     # noqa: BLE001
                _emit("tiles2_phase", direction=direction, debug_mode=mode, error=repr(e)[:300])


def check_bwd_tune():
    """Backward kernel: per-phase timestamps of CTA 0 (first operand block ready / accumulator ready / signalled)."""
    import torch
    from lstm_tensorspark_b200.ops import cuda_lstm
    from lstm_tensorspark_b200.ops.cuda_ext import ext
    E = ext()
    dev = torch.device("cuda")
    T, B, H = 128, 256, 1024
    torch.manual_seed(0)
    gx = (torch.randn(T, B, 4 * H, device=dev) * 0.5).bfloat16()
    whb = (torch.randn(4 * H, H, device=dev) / H ** 0.5).bfloat16()
    bias = torch.zeros(4 * H, device=dev)
    h0 = torch.zeros(B, H, device=dev).bfloat16(); c0 = torch.zeros(B, H, device=dev)
    ws = cuda_lstm._sync_ws(dev)
    h_seq, c_seq, act = E.lstm_seq_fwd(gx, whb, bias, h0, c0, ws, 0)
    dh_seq = (torch.randn(T, B, H, device=dev) * 0.1).bfloat16()
    w_hT = whb.t().contiguous()
    z = torch.zeros(B, H, device=dev)
    for (mode, sync) in ((0, 0), (0, 1), (1, 0), (2, 0)):
        v = 4096 * mode + 65536 * sync
        try:
            ms = _time_ms(lambda: E.lstm_seq_bwd(dh_seq, w_hT, act, c_seq, z, z, ws, v), iters=5, warm=2)
            dbg = torch.zeros(4 * (T + 2) + 64 + 512, dtype=torch.int64, device=dev)
            E.lstm_seq_bwd(dh_seq, w_hT, act, c_seq, z, z, ws, v, dbg)
            torch.cuda.synchronize()
            cuda_lstm.check_kernel_errors(dev)
            d = dbg[:4 * (T + 2)].view(-1, 4)[8:40].cpu()
            waited, accum, sig = d[:, 0], d[:, 1], d[:, 2]
            w3 = d[:, 3]
            mma_first = [int(x) & 0xFFFFF for x in w3]
            mma_wait = [(int(x) >> 20) & 0xFFFFF for x in w3]
            mma_total = [(int(x) >> 40) & 0xFFFFF for x in w3]
            n = len(mma_first)
            _emit("bwd_variant", debug_mode=mode, sync=sync, us_per_step=ms * 1e3 / (T + 1),
                  mma_first_wait_us=sum(mma_first) / n / 1965, mma_later_wait_us=sum(mma_wait) / n / 1965, mma_step_us=sum(mma_total) / n / 1965,
                  load_mma_us=float((accum - waited).float().mean()) / 1e3, epi_us=float((sig - accum).float().mean()) / 1e3,
                  sync_us=float((waited[1:] - sig[:-1]).float().mean()) / 1e3)
        except Exception as e:                     # noqa: BLE001
            _emit("bwd_variant", debug_mode=mode, sync=sync, error=repr(e)[:300])


def check_skew():
    """Per-CTA time stamps at step 8 of the forward kernel: when each CTA's accumulator was ready and when it signalled."""
    import torch
    from lstm_tensorspark_b200.ops import cuda_lstm
    from lstm_tensorspark_b200.ops.cuda_ext import ext
    E = ext()
    dev = torch.device("cuda")
    T, B, H = 32, 256, 1024
    gx = (torch.randn(T, B, 4 * H, device=dev) * 0.5).bfloat16()
    whb = (torch.randn(4 * H, H, device=dev) / H ** 0.5).bfloat16()
    bias = torch.zeros(4 * H, device=dev)
    h0 = torch.zeros(B, H, device=dev).bfloat16(); c0 = torch.zeros(B, H, device=dev)
    ws = cuda_lstm._sync_ws(dev)
    for rep in range(2):
        dbg = torch.zeros(4 * (T + 2) + 64 + 2 * 160, dtype=torch.int64, device=dev)
        E.lstm_seq_fwd(gx, whb, bias, h0, c0, ws, 0, dbg)
        torch.cuda.synchronize()
        st = dbg[4 * (T + 2) + 64:].view(-1, 2)[:128].cpu()
        acc, sig = st[:, 0], st[:, 1]
        base = int(acc.min())
        a = (acc - base).tolist(); g = (sig - base).tolist()
        for mb in (0, 1):
            aa = a[64 * mb:64 * mb + 64]; gg = g[64 * mb:64 * mb + 64]
            _emit("skew", rep=rep, mb=mb, acc_min=min(aa), acc_max=max(aa), acc_sorted=sorted(aa)[::8], sig_min=min(gg), sig_max=max(gg),
                  slowest=[i for i, _ in sorted(enumerate(aa), key=lambda kv: -kv[1])[:8]])


def check_seq_tiles():
    """Kernel time of the persistent fwd / bwd kernels with 1 vs 2 batch tiles per CTA (T=128, B=256, H=1024)."""
    import torch
    from lstm_tensorspark_b200.ops import cuda_lstm
    from lstm_tensorspark_b200.ops.cuda_ext import ext
    E = ext()
    dev = torch.device("cuda")
    T, B, H = 128, 256, 1024
    torch.manual_seed(0)
    gx = (torch.randn(T, B, 4 * H, device=dev) * 0.5).bfloat16()
    whb = (torch.randn(4 * H, H, device=dev) / H ** 0.5).bfloat16()
    whT = whb.t().contiguous()
    bias = torch.zeros(4 * H, device=dev)
    h0 = torch.zeros(B, H, device=dev).bfloat16(); c0 = torch.zeros(B, H, device=dev)
    dh = (torch.randn(T, B, H, device=dev) * 0.1).bfloat16()
    z = torch.zeros(B, H, device=dev)
    ws = cuda_lstm._sync_ws(dev)
    ref = None
    for tiles in (1, 2):
        hs, cs, act = E.lstm_seq_fwd(gx, whb, bias, h0, c0, ws, tiles)
        dpre, dh0, dc0 = E.lstm_seq_bwd(dh, whT, act, cs, z, z, ws, tiles)
        torch.cuda.synchronize()
        cuda_lstm.check_kernel_errors(dev)
        if ref is None:
            ref = (hs, dpre, dh0)
        f = _time_ms(lambda: E.lstm_seq_fwd(gx, whb, bias, h0, c0, ws, tiles), iters=5, warm=2)
        b = _time_ms(lambda: E.lstm_seq_bwd(dh, whT, act, cs, z, z, ws, tiles), iters=5, warm=2)
        _emit("seq_tiles", tiles=tiles, fwd_ms=f, fwd_us_per_step=f * 1e3 / T, bwd_ms=b, bwd_us_per_step=b * 1e3 / T,
              h_same=bool(torch.equal(hs, ref[0])), dpre_maxdiff=float((dpre.float() - ref[1].float()).abs().max()),
              dh0_maxdiff=float((dh0 - ref[2]).abs().max()))


def check_seq_h2048():
    """Streamed-weights variant (BASELINE.json config 4 shape: H = 2048, B = 64)."""
    _seq_case(6, 64, 2048, 256, check_bwd=True, time_it=True)
    _seq_case(32, 64, 2048, 2048, check_bwd=False, time_it=True)


def check_generic():
    os.environ["LSTM_TS_FORCE_GENERIC"] = "1"
    from lstm_tensorspark_b200.ops import cuda_lstm
    cuda_lstm.FORCE_GENERIC = True
    _seq_case(3, 10, 16, 4)
    _seq_case(6, 33, 48, 20)


def check_engine():
    import torch
    sys.path.insert(0, ROOT)
    import __graft_entry__ as g
    g.smoke()
    _emit("smoke", ok=True)


def check_iris_gpu():
    r = subprocess.run([sys.executable, os.path.join(ROOT, "lstm-no-spark.py"), "--training_path", os.path.join(ROOT, "dataset/iris.data"),
                        "--hidden_units", "16", "--epochs", "30", "--checkpoint_path", "/tmp/ck_gpu", "--output_path", "/tmp/out_gpu",
                        "--quiet"], capture_output=True, text=True, timeout=600)
    _emit("iris_gpu_standalone", rc=r.returncode, tail=(r.stdout + r.stderr)[-600:])


CHECKS = {"tiles2": check_tiles2_tune, "tiles2_phase": check_tiles2_phase,"wave": check_wave, "wave_bwd": check_wave_bwd, "gemm2": check_gemm2, "gemm2_dw": check_gemm2_dw, "seq_h2048": check_seq_h2048, "bwd_tune": check_bwd_tune, "skew": check_skew, "seq_tiles": check_seq_tiles, "seq_tune": check_seq_tune, "env": check_env, "simple": check_simple, "generic": check_generic, "seq_small": check_seq_small,
          "seq_big": check_seq_big, "engine": check_engine, "iris_gpu": check_iris_gpu}


def main():
    if len(sys.argv) >= 3 and sys.argv[1] == "--one":
        CHECKS[sys.argv[2]]()
        return 0
    names = sys.argv[1:] or list(CHECKS)
    for n in names:
        t0 = time.time()
        try:
            r = subprocess.run([sys.executable, os.path.abspath(__file__), "--one", n], capture_output=True, text=True,
                               timeout=float(os.environ.get("PROBE_TIMEOUT", "300")))
            sys.stdout.write(r.stdout[-6000:])
            if r.returncode != 0:
                _emit(n + "_FAILED", rc=r.returncode, stderr=r.stderr[-3000:])
        except subprocess.TimeoutExpired as e:
            _emit(n + "_TIMEOUT", seconds=time.time() - t0, stdout=(e.stdout or b"")[-2000:] if e.stdout else "")
    return 0


if __name__ == "__main__":
    sys.exit(main())
