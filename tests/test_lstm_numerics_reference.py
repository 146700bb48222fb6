"""The rounding-aware LSTM reference (tests/lstm_numerics.py) on the CPU: its fp64 arm against autograd, its pair against two
chained layers, and the error budget's sensitivity to defects confined to one step of a long sequence; its whole-model arm
against autograd on the plain composition of ops/reference, against ``pair``, and the budget's sensitivity to defects of the
model's composition.  Also the sync-workspace guard of the persistent kernels' launch configuration."""
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


# --- the generic path's arms: bf16 (Generic) and fp32 (Fp32) --------------------------------------------------------------
G_T, G_B, G_H, G_D = 128, 64, 96, 40           # H % 64 != 0: a bf16 layer of this shape runs on the generic path
G_LENGTHS = _lengths(G_T, G_B, 8)


@pytest.fixture(scope="module")
def generic_case():
    """fp64 and both generic arms of one masked reverse layer: (fp64, {arm: emulation}, fp32 inputs)."""
    params64, grads64 = _inputs(G_T, G_B, G_H, G_D, seed=9)
    args32 = [p.float() for p in params64] + [g.float() for g in grads64]
    kw = dict(lengths=G_LENGTHS, reverse=True)
    fp64 = N.layer(*params64, *grads64, **kw)
    emu = {"generic": N.layer(*args32, rounding=N.Generic(), **kw), "fp32": N.layer(*args32, rounding=N.Fp32(), **kw)}
    return fp64, emu, lambda rounding, defect=None: N.layer(*args32, rounding=rounding, defect=defect, **kw)


def _budget_floor(got, fp64, emu, floor):
    return {name: N.check_budget(name, g, f, e, per_step=name in ("h_seq", "dx"), floor=floor)
            for name, g, f, e in zip(N.LayerOut._fields, got, fp64, emu)}


@pytest.mark.parametrize("arm,standin,floor", [
    ("generic", N.Generic(approx=2.0 ** -11), N.FLOOR),            # tanh.approx-sized activations, as the bf16 cell kernels
    ("fp32", N.Fp32(split=2, approx=2.0 ** -24), N.FLOOR_F32),      # other fp32 sums, activations off by an ulp
])
def test_generic_arms_sit_inside_the_budget_of_a_second_realisation(generic_case, arm, standin, floor):
    fp64, emu, run = generic_case
    ratios = _budget_floor(run(standin), fp64, emu[arm], floor)
    assert max(ratios.values()) <= 1.0, ratios
    lo, hi = (1e-4, 2e-2) if arm == "generic" else (1e-8, 1e-5)     # bf16-sized / fp32-sized distances from fp64
    assert lo < _rel(emu[arm].h_seq, fp64.h_seq) < hi and lo < _rel(emu[arm].dw_h, fp64.dw_h) < hi


def test_generic_arm_differs_from_the_fast_path_emulation(generic_case):
    """The generic arm rounds pre before the bias and never the recurrent gradient product: not the fast path's numbers."""
    fp64, emu, run = generic_case
    fast = run(Bf16(fwd_split=1, bwd_split=4))
    assert not torch.equal(fast.h_seq, emu["generic"].h_seq) and not torch.equal(fast.dx, emu["generic"].dx)


def test_fp32_budget_rejects_a_tanh_off_by_2_to_the_minus_15(generic_case):
    """A 128-step fp32 layer whose every tanh (and sigmoid) carries a relative error of 2^-15 - sixteen times smaller than
    tanh.approx's - is over the fp32 budget."""
    fp64, emu, run = generic_case
    with pytest.raises(AssertionError, match=r"error vs fp64 .*ratio"):
        _budget_floor(run(N.Fp32(approx=2.0 ** -15)), fp64, emu["fp32"], N.FLOOR_F32)


def test_a_defect_at_one_step_breaks_the_generic_budget(generic_case):
    """One k-block of h dropped from the recurrent product at one step, on the bf16 generic arm."""
    fp64, emu, run = generic_case
    with pytest.raises(AssertionError, match=r"h_seq at step \d+: .*ratio"):
        _budget_floor(run(N.Generic(approx=2.0 ** -11), Defect("drop_kblock", STEP, 0)), fp64, emu["generic"], N.FLOOR)


# --- the whole model ----------------------------------------------------------------------------------------------------
def _model_inputs(hidden, T, B, D, C, seed, bidirectional=False, initial_state=False, dtype=torch.float64):
    """x [B,T,D], per-layer (direction) (h0, c0, w_x, w_h, bias), head (W, b), labels: bf16-representable where the kernels
    read bf16.  ``initial_state``: nonzero h0 / c0 (learned), else zeros (the engine's default)."""
    g = torch.Generator().manual_seed(seed)
    rn = lambda *s: torch.randn(*s, generator=g, dtype=torch.float64)
    x = _bf(rn(B, T, D) * 0.5)
    layers, d_in = [], D
    for H in hidden:
        def one():
            z = torch.zeros(B, H, dtype=torch.float64)
            h0, c0 = (_bf(rn(B, H) * 0.3), _bf(rn(B, H) * 0.3)) if initial_state else (z, z.clone())
            return (h0, c0, _bf(rn(4 * H, d_in) / d_in ** 0.5), _bf(rn(4 * H, H) / H ** 0.5), _bf(rn(4 * H) * 0.1))
        layers.append((one(), one()) if bidirectional else one())
        d_in = H * (2 if bidirectional else 1)
    W, b = _bf(rn(d_in, C) / d_in ** 0.5), _bf(rn(C) * 0.1)
    labels = torch.randint(0, C, (B,), generator=g)
    cast = lambda t: t.to(dtype)
    layers = [tuple(tuple(map(cast, p)) for p in l) if bidirectional else tuple(map(cast, l)) for l in layers]
    return cast(x), layers, (cast(W), cast(b)), labels


def _autograd_model(x, layers, head, labels, lengths, bidirectional, dropout):
    """The same classifier as a plain composition of ops/reference under autograd -> (loss, h_T, {name: grad})."""
    from lstm_tensorspark_b200.ops import reference as ref
    dirs = (False, True) if bidirectional else (False,)
    leaves = {}
    for l, lp in enumerate(layers):
        for d, rev in enumerate(dirs):
            p = lp[d] if bidirectional else lp
            for k, v in zip(("h0", "c0", "w_x", "w_h", "bias"), p):
                leaves[f"LSTMLayer{l}{'_reverse' if rev else ''}/{k}"] = v.clone().requires_grad_(True)
    leaves["Dense1/weights"], leaves["Dense1/bias"] = (t.clone().requires_grad_(True) for t in head)
    seq = x.transpose(0, 1)
    for l in range(len(layers)):
        outs, finals = [], []
        for rev in dirs:
            n = f"LSTMLayer{l}{'_reverse' if rev else ''}/"
            spec = None
            if dropout is not None and l < len(layers) - 1:
                spec = ref.DropoutSpec(dropout.p, dropout.key, l, rev, dropout.step)
            hs, hT, _ = ref.lstm_layer_sequence(seq, *(leaves[n + k] for k in ("h0", "c0", "w_x", "w_h", "bias")),
                                                lengths=lengths, reverse=rev, dropout=spec)
            outs.append(hs)
            finals.append(hT)
        seq = torch.cat(outs, 2)
    h_T = torch.cat(finals, 1)
    logits = ref.dense_head(h_T, leaves["Dense1/weights"], leaves["Dense1/bias"])
    # ref.softmax_xent, in fp64 (it casts the logits to fp32)
    loss = -torch.log_softmax(logits, -1).gather(1, labels.view(-1, 1).long()).mean()
    loss.backward()
    return loss, h_T, {k: v.grad for k, v in leaves.items()}


@pytest.mark.parametrize("case", ["three layers", "bidirectional lengths", "dropout", "bidirectional dropout",
                                  "learned initial state"])
def test_fp64_model_matches_autograd_on_the_reference(case):
    T, B, D, C = 6, 5, 4, 3
    bidir = case.startswith("bidirectional")
    hidden = [8, 12, 8] if case == "three layers" else [8, 12]
    x, layers, head, labels = _model_inputs(hidden, T, B, D, C, seed=11, bidirectional=bidir,
                                            initial_state=case == "learned initial state")
    lengths = _lengths(T, B, 12) if case == "bidirectional lengths" else None
    dropout = N.Dropout(0.3, (5, 1), 3) if "dropout" in case else None
    loss, h_T, want = _autograd_model(x, layers, head, labels, lengths, bidir, dropout)
    got = N.model(x, layers, head, labels, lengths=lengths, bidirectional=bidir, dropout=dropout)
    assert _rel(got.loss, loss) < 1e-10 and _rel(got.h_T, h_T) < 1e-10
    assert set(got.grads) == set(want)
    for k, v in want.items():
        assert got.grads[k].dtype == torch.float64 and _rel(got.grads[k], v) < 1e-10, (k, _rel(got.grads[k], v))
    if dropout is not None:                           # the masks drop something, and the step count selects them
        other = N.model(x, layers, head, labels, bidirectional=bidir, dropout=dropout._replace(step=4), lengths=lengths)
        assert _rel(other.loss, loss) > 1e-6


@pytest.mark.parametrize("rounding", [None, Bf16(fwd_split=1, bwd_split=4)])
def test_model_without_dropout_or_head_equals_pair(rounding):
    T, B, D = 7, 6, 4
    x, layers, _, _ = _model_inputs([8, 12], T, B, D, 3, seed=13, initial_state=True,
                                    dtype=torch.float64 if rounding is None else torch.float32)
    dh_T = _bf(torch.randn(B, 12, generator=torch.Generator().manual_seed(14), dtype=torch.float64)).to(x.dtype)
    lengths = _lengths(T, B, 15)
    got = N.model(x, layers, None, None, lengths=lengths, dh_T=dh_T, rounding=rounding)
    a, b = N.pair(x.transpose(0, 1), layers[0], layers[1], None, None, None, dh_T, None, lengths=lengths, rounding=rounding)
    assert torch.equal(got.h_T, b.h_T)
    for l, out in enumerate((a, b)):
        for k in ("dh0", "dc0", "dw_x", "dw_h", "db"):
            n = {"dh0": "h0", "dc0": "c0", "dw_x": "w_x", "dw_h": "w_h", "db": "bias"}[k]
            assert torch.allclose(got.grads[f"LSTMLayer{l}/{n}"], getattr(out, k), rtol=1e-12, atol=1e-14), (l, k)


# --- the budget against defects of the model's composition --------------------------------------------------------------
M_T, M_B, M_H, M_D, M_C = 64, 64, 256, 128, 10
M_DROP = N.Dropout(0.2, (7, 0), 2)
M_LOST = 40                          # rows of the first batch chunk, 256 of B = 400 scaled to B = 64


@pytest.fixture(scope="module")
def model_case():
    """A bidirectional 2-layer stack with lengths (1 and T included) and dropout: fp64, the emulation and a stand-in run."""
    x, layers, head, labels = _model_inputs([M_H, M_H], M_T, M_B, M_D, M_C, seed=17, bidirectional=True)
    lengths = _lengths(M_T, M_B, 18)
    f32 = lambda t: t.float()
    l32 = [tuple(tuple(map(f32, p)) for p in l) for l in layers]
    kw = dict(lengths=lengths, bidirectional=True, dropout=M_DROP)
    fp64 = N.model(x, layers, head, labels, **kw)
    emu = N.model(x.float(), l32, tuple(map(f32, head)), labels, rounding=Bf16(fwd_split=1, bwd_split=4), **kw)
    run = lambda defect=None: N.model(x.float(), l32, tuple(map(f32, head)), labels, rounding=STANDIN, defect=defect, **kw)
    return fp64, emu, run


def _model_budget(got, fp64, emu):
    """Loss, h_T per row and every gradient; raises on the first one over budget."""
    ratios = {"loss": N.check_budget("loss", got.loss, fp64.loss, emu.loss),
              "h_T": N.check_budget("h_T", got.h_T, fp64.h_T, emu.h_T, per_step=True)}
    for k in fp64.grads:
        ratios[k] = N.check_budget(k, got.grads[k], fp64.grads[k], emu.grads[k])
    return ratios


def test_model_emulation_sits_inside_the_budget_of_a_second_realisation(model_case):
    fp64, emu, run = model_case
    ratios = _model_budget(run(), fp64, emu)
    assert max(ratios.values()) <= 1.0, ratios
    assert 1e-4 < _rel(emu.grads["LSTMLayer0/w_x"], fp64.grads["LSTMLayer0/w_x"]) < 2e-2


@pytest.mark.parametrize("defect,tensor", [
    (Defect("fwd_dx_only", 1, 0), "LSTMLayer0"),                   # the reverse upper direction's dx lost at t = 1 (near its h_T)
    (Defect("mask_next_step", 0, 0), "LSTMLayer0"),                # backward masks drawn for the next training step
    (Defect("lost_chunk", 0, M_LOST), "LSTMLayer"),                # the second batch chunk overwrote the weight sinks
    (Defect("reverse_unmasked", 0, 0), ""),                        # the reverse direction runs over the padding
])
def test_a_composition_defect_breaks_the_model_budget(model_case, defect, tensor):
    fp64, emu, run = model_case
    got = run(defect)
    with pytest.raises(AssertionError, match=rf"^{tensor}[^:]*: error vs fp64 .*ratio"):
        _model_budget(got, fp64, emu)
    grads = {k: v for k, v in got.grads.items() if k in fp64.grads}
    over = sorted(k for k in grads if not _rel(grads[k], fp64.grads[k]) <= 1e-2)
    print(f"\n{defect.kind}: the per-gradient relative L2 <= 1e-2 criterion {'catches it on ' + ', '.join(over) if over else 'misses it'}")


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


# --- the optimizer update -----------------------------------------------------------------------------------------------
STRIDE = 132 * 8 * 256 * 4           # floats one grid-stride pass of the update kernels covers (grid_for, multi_tensor_opt.cu)
U_N = 2 * STRIDE + 300 * 1024        # a flat buffer of three passes, the last one partial
U_WD = 2 * STRIDE + 128 * 1024       # end of the LSTM segment: weight decay covers [0, U_WD)
U_BIAS = 4096                        # the last LSTM variable, a bias, ends at U_WD; a dense head follows it
U_PAD = 64                           # trailing alignment padding: every value 0
LR_T_APPROX = 2.2e-4                 # the worst relative error of the in-kernel lr_t under --use_fast_math (lstm_numerics)
ADAM = dict(lr=1e-3, b1=0.9, b2=0.999, eps=1e-8, wd=0.1, grad_scale=0.37, wd_numel=U_WD)


def _update_state(seed, n=U_N):
    """fp32 p, m, v and two consecutive gradients with magnitudes from 1e-4 to 1 (padding all zero)."""
    gen = torch.Generator().manual_seed(seed)
    scale = 10.0 ** (torch.rand(n, generator=gen) * 4 - 4)
    p = torch.randn(n, generator=gen) * 0.05
    g = torch.randn(n, generator=gen) * scale
    g_prev = torch.randn(n, generator=gen) * scale
    m = torch.randn(n, generator=gen) * scale * 0.3
    v = scale * scale * (0.5 + torch.rand(n, generator=gen))
    for t in (p, g, g_prev, m, v):
        t[-U_PAD:] = 0
    return p, m, v, g, g_prev


def _adam_f32(p, m, v, g, t, lr, b1, b2, eps, wd, grad_scale, wd_numel, defect=None):
    """flat_adam_kernel with the bias correction from step_dev, in fp32 arithmetic with lr_t off by the worst fast-math
    error - and ``defect`` planted."""
    f = lambda x: torch.tensor(x, dtype=torch.float32)
    if defect == "b1 b2 swapped":
        b1, b2 = b2, b1
    tt = t + 1 if defect == "lr_t of t + 1" else t
    lr_t = f(lr) * torch.sqrt(1 - f(b2) ** tt) / (1 - f(b1) ** tt) * f(1 + LR_T_APPROX)
    hi = {"wd missing on the bias": wd_numel - U_BIAS, "wd past wd_numel": wd_numel + 64}.get(defect, wd_numel)
    w = torch.zeros_like(p)
    w[:hi] = f(wd)
    gg = g * f(grad_scale) + w * p
    m1 = f(b1) * m + (1 - f(b1)) * gg
    v1 = f(b2) * v + (1 - f(b2)) * gg * gg
    p1 = p - lr_t * m1 / (torch.sqrt(v1) + f(eps))
    skip = {"last float4 not updated": slice(p.numel() - U_PAD - 4, p.numel() - U_PAD),
            "one grid-stride pass not updated": slice(STRIDE, 2 * STRIDE)}.get(defect)
    if skip is not None:
        p1[skip], m1[skip], v1[skip] = p[skip], m[skip], v[skip]
    return p1, m1, v1


def _check_adam(got, ref):
    return max(N.check_update(k, a, b, bnd) for k, a, b, bnd in zip("pmv", got, ref[:3], ref[3:]))


@pytest.mark.parametrize("t", [1, 2, 1000, 100000])
def test_fp64_update_matches_the_reference_optimizer(t):
    """adam_update / sgd_update == ops/reference.adam_step_ / sgd_step_ run in fp64 on the fp32 scalars, the weight decay over
    [0, wd_numel) as FlatOptimizer applies it."""
    from lstm_tensorspark_b200.ops import reference as ref
    p, m, v, g, _ = _update_state(7, n=1 << 16)
    wd_n = 40000
    f = N.f32
    got = N.adam_update(p, m, v, g, t, **{**ADAM, "wd_numel": wd_n})
    p64, m64, v64, g64 = (x.double() for x in (p, m, v, g))
    for lo, hi, wd in ((0, wd_n, f(0.1)), (wd_n, p.numel(), 0.0)):
        ref.adam_step_(p64[lo:hi], g64[lo:hi], m64[lo:hi], v64[lo:hi], t, f(1e-3), f(0.9), f(0.999), f(1e-8), wd, f(0.37))
    for a, b, bound in ((got.p, p64, got.bound_p), (got.m, m64, got.bound_m), (got.v, v64, got.bound_v)):
        assert bool(((a - b).abs() <= 1e-8 * bound).all())            # fp64 rounding only: 1e-8 of the fp32 bound
    sgd = N.sgd_update(p, g, 0.05, 0.1, 0.37, wd_n)
    q64 = p.double()
    for lo, hi, wd in ((0, wd_n, f(0.1)), (wd_n, p.numel(), 0.0)):
        ref.sgd_step_(q64[lo:hi], g64[lo:hi], f(0.05), wd, f(0.37))
    assert bool(((sgd.p - q64).abs() <= 1e-8 * sgd.bound_p).all())
    assert bool((got.p[-U_PAD:] == 0).all()) and bool((sgd.p[-U_PAD:] == 0).all())


@pytest.mark.parametrize("t", [1, 2, 5, 100, 1000, 100000])
def test_fp32_update_sits_inside_the_bound(t):
    """An fp32 realisation of the update kernels (Adam's lr_t off by its worst fast-math error) passes check_update."""
    p, m, v, g, _ = _update_state(3)
    worst = _check_adam(_adam_f32(p, m, v, g, t, **ADAM), N.adam_update(p, m, v, g, t, **ADAM))
    lr, wd, gs = N.f32(0.05), N.f32(0.1), N.f32(0.37)
    w = torch.zeros_like(p)
    w[:U_WD] = wd
    q = p - torch.tensor(lr) * (g * torch.tensor(gs) + w * p)
    ref = N.sgd_update(p, g, 0.05, 0.1, 0.37, U_WD)
    worst_sgd = N.check_update("p", q, ref.p, ref.bound_p)
    assert 0.05 < worst <= 1.0 and worst_sgd <= 1.0, (worst, worst_sgd)


@pytest.mark.parametrize("defect,t", [("lr_t of t + 1", 1), ("lr_t of t + 1", 5), ("lr_t of t + 1", 100),
                                      ("wd missing on the bias", 1000), ("wd past wd_numel", 1000), ("b1 b2 swapped", 1000),
                                      ("previous gradient", 1000), ("last float4 not updated", 1000),
                                      ("one grid-stride pass not updated", 1000)])
def test_an_update_defect_breaks_the_bound(defect, t):
    p, m, v, g, g_prev = _update_state(5)
    got = _adam_f32(p, m, v, g_prev if defect == "previous gradient" else g, t, defect=defect, **ADAM)
    with pytest.raises(AssertionError, match=r"^[pmv]: element .* exceeds the bound"):
        _check_adam(got, N.adam_update(p, m, v, g, t, **ADAM))


def test_shadow_is_checked_bit_for_bit():
    p = torch.randn(4096) * 0.05
    N.check_shadow("shadow", p.bfloat16(), p)
    sh = p.bfloat16()
    sh.view(torch.int16)[1000] += 1                     # one ulp off at one element
    with pytest.raises(AssertionError, match=r"^shadow: .* at 1 of 4096 elements; first at 1000"):
        N.check_shadow("shadow", sh, p)
    with pytest.raises(AssertionError, match="shadow"):
        N.check_shadow("shadow", (p * (1 + 2.0 ** -10)).bfloat16(), p)      # the shadow of the weights before a step
