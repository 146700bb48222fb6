"""The rounding-aware LSTM reference (tests/lstm_numerics.py) on the CPU: its fp64 arm against autograd, its pair against two
chained layers, and the error budget's sensitivity to defects confined to one step of a long sequence.  Also the sync-workspace
guard of the persistent kernels' launch configuration."""
import pytest
import torch

import lstm_numerics as N
from lstm_numerics import Bf16, Defect


def _bf(t):
    return t.bfloat16().double()


def _inputs(T, B, H, D, seed, dtype=torch.float64):
    """bf16-representable x, h0, W (what the kernels read), fp32-valued c0 and bias; bf16-representable loss weights."""
    g = torch.Generator().manual_seed(seed)
    rn = lambda *s: torch.randn(*s, generator=g, dtype=torch.float64)
    x = _bf(rn(T, B, D) * 0.5)
    h0, c0 = _bf(rn(B, H) * 0.1), (rn(B, H) * 0.1).float().double()
    w_x, w_h = _bf(rn(4 * H, D) / D ** 0.5), _bf(rn(4 * H, H) / H ** 0.5)
    bias = (rn(4 * H) * 0.1).float().double()
    dh_seq, dh_T, dc_T = _bf(rn(T, B, H)), _bf(rn(B, H)), _bf(rn(B, H))
    return [t.to(dtype) for t in (x, h0, c0, w_x, w_h, bias)], (dh_seq.to(dtype), dh_T.to(dtype), dc_T.to(dtype))


def _lengths(T, B, seed):
    g = torch.Generator().manual_seed(seed)
    lengths = torch.randint(1, T + 1, (B,), generator=g, dtype=torch.int32)
    lengths[0], lengths[-1] = 1, T
    return lengths


def _rel(a, b):
    a, b = a.detach().double(), b.detach().double()
    return float((a - b).norm() / (b.norm() + 1e-300))


@pytest.mark.parametrize("masked,reverse", [(False, False), (True, False), (False, True), (True, True)])
@pytest.mark.parametrize("loss", ["h_seq", "h_T", "all"])
def test_fp64_layer_matches_autograd_on_the_reference(masked, reverse, loss):
    from lstm_tensorspark_b200.ops import reference as ref
    T, B, H, D = 7, 6, 8, 5
    params, (dh_seq, dh_T, dc_T) = _inputs(T, B, H, D, seed=1)
    dh_seq = dh_seq if loss in ("h_seq", "all") else None
    dh_T = dh_T if loss in ("h_T", "all") else None
    dc_T = dc_T if loss == "all" else None
    lengths = _lengths(T, B, 2) if masked else None
    leaves = [p.clone().requires_grad_(True) for p in params]
    hs, hT, cT = ref.lstm_layer_sequence(*leaves, lengths=lengths, reverse=reverse)
    obj = sum((o * w).sum() for o, w in ((hs, dh_seq), (hT, dh_T), (cT, dc_T)) if w is not None)
    obj.backward()
    got = N.layer(*params, dh_seq, dh_T, dc_T, lengths=lengths, reverse=reverse)
    for name, a, b in [("h_seq", got.h_seq, hs), ("h_T", got.h_T, hT), ("c_T", got.c_T, cT)] + \
            [(n, getattr(got, n), p.grad) for n, p in zip(("dx", "dh0", "dc0", "dw_x", "dw_h", "db"), leaves)]:
        assert a.dtype == torch.float64 and _rel(a, b) < 1e-10, (name, _rel(a, b))


@pytest.mark.parametrize("masked", [False, True])
def test_fp64_pair_equals_two_chained_layers(masked):
    T, B, D, Ha, Hb = 6, 5, 4, 8, 12
    pa, (_, dhTa, dcTa) = _inputs(T, B, Ha, D, seed=3)
    x, la = pa[0], pa[1:]
    pb, (dh_seq, dhTb, dcTb) = _inputs(T, B, Hb, Ha, seed=4)
    lb = pb[1:]
    lengths = _lengths(T, B, 5) if masked else None
    a, b = N.pair(x, la, lb, dh_seq, dhTa, dcTa, dhTb, dcTb, lengths=lengths)
    fa = N.layer(x, *la, None, None, None, lengths=lengths)
    fb = N.layer(fa.h_seq, *lb, dh_seq, dhTb, dcTb, lengths=lengths)
    ga = N.layer(x, *la, fb.dx, dhTa, dcTa, lengths=lengths)
    for want, got in ((fb, b), (ga, a)):
        for name, u, v in zip(N.LayerOut._fields, want, got):
            assert torch.allclose(u, v, rtol=1e-12, atol=1e-14), name


# --- the budget against defects confined to one step ------------------------------------------------------------------
T_LONG, B_CPU, H_CPU, D_CPU = 128, 64, 512, 256
STEP = 64
STANDIN = Bf16(fwd_split=1, bwd_split=4, approx=2.0 ** -11)      # a "kernel": other rounding realisations, tanh.approx-sized error


@pytest.fixture(scope="module")
def long_case():
    params64, grads64 = _inputs(T_LONG, B_CPU, H_CPU, D_CPU, seed=7)
    params32, grads32 = [p.float() for p in params64], [g.float() for g in grads64]
    fp64 = N.layer(*params64, *grads64)
    emu = N.layer(*params32, *grads32, rounding=Bf16(fwd_split=1, bwd_split=4))
    run = lambda defect=None: N.layer(*params32, *grads32, rounding=STANDIN, defect=defect)
    return fp64, emu, run


def _budget_all(got, fp64, emu):
    """Every output's worst budget ratio; raises on the first tensor over budget."""
    return {name: N.check_budget(name, g, f, e, per_step=name in ("h_seq", "dx"))
            for name, g, f, e in zip(N.LayerOut._fields, got, fp64, emu)}


def test_emulation_sits_inside_the_budget_of_a_second_realisation(long_case):
    fp64, emu, run = long_case
    ratios = _budget_all(run(), fp64, emu)
    assert max(ratios.values()) <= 1.0, ratios
    # the emulation is a bf16-sized distance from fp64 (not a copy of it, nor far off)
    assert 1e-4 < _rel(emu.h_seq, fp64.h_seq) < 1e-2 and 1e-4 < _rel(emu.dx, fp64.dx) < 2e-2


@pytest.mark.parametrize("defect,tensor", [
    (Defect("drop_kblock", STEP, 3), "h_seq"),       # one k-block of the recurrent product dropped at one step
    (Defect("stale_rows", STEP, 1), "h_seq"),        # one 16-row group reads h_{t-2} instead of h_{t-1} at one step
    (Defect("zero_dg", STEP, 5), "dx"),              # one k-block of dG zeroed at one (backward) step
])
def test_a_defect_at_one_step_breaks_the_budget(long_case, defect, tensor):
    fp64, emu, run = long_case
    got = run(defect)
    with pytest.raises(AssertionError, match=rf"{tensor} at step \d+: .*ratio"):
        _budget_all(got, fp64, emu)
    # the defect's own time step is over budget, the steps computed before it are not
    t = STEP if tensor == "h_seq" else T_LONG - 1 - STEP
    before = slice(0, t) if tensor == "h_seq" else slice(t + 1, T_LONG)
    g, f, e = getattr(got, tensor), getattr(fp64, tensor), getattr(emu, tensor)
    with pytest.raises(AssertionError, match=rf"{tensor} at step 0:"):
        N.check_budget(tensor, g[t:t + 1], f[t:t + 1], e[t:t + 1], per_step=True)
    assert N.check_budget(tensor, g[before], f[before], e[before], per_step=True) <= 1.0
    if defect.kind == "zero_dg":
        # what the per-tensor criterion of the older kernel tests (relative L2 < 2e-2 on every gradient) makes of it: a pass
        rel = {n: _rel(getattr(got, n), getattr(fp64, n)) for n in ("dx", "dh0", "dc0", "dw_x", "dw_h", "db")}
        assert max(rel.values()) < 2e-2, rel
        assert _rel(got.dx[t], fp64.dx[t]) > 0.1


# --- launch configuration -----------------------------------------------------------------------------------------------
def test_seq_config_rejects_layouts_whose_arrival_counters_overflow_the_sync_workspace():
    from lstm_tensorspark_b200.ops.cuda_ext import ext
    E = ext()
    # backward H = 256, B = 2048, two tiles per CTA: 16 tiles x 64 dG k-blocks = 1024 counters (128 CTAs in clusters of 4)
    with pytest.raises(RuntimeError, match="sync workspace"):
        E.lstm_seq_config(True, 256, 2048, 2)
    with pytest.raises(RuntimeError, match="sync workspace"):
        E.lstm_seq_config(True, 1024, 512, 2)                # 4 tiles x 64 = 256 counters
    assert E.lstm_seq_config(True, 960, 512, 2)[1] == 2       # 4 tiles x 60 = 240: the last counter at word 8160 < 8191
    assert E.lstm_seq_config(False, 256, 2048, 2)[1] == 2     # the forward has a quarter of the counters
    assert E.lstm_seq_config(True, 1024, 256, 2) == (4, 2, False, False)
    assert E.lstm_seq_config(True, 2048, 64, 0)[2] is True
