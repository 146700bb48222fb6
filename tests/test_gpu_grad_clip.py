"""Gradient clipping by the global norm on the GPU: the norm kernel (csrc/multi_tensor_opt.cu flat_grad_norm_kernel) against fp64
at awkward and headline sizes, its special values and its determinism across calls and graph replays; the clipped Adam and SGD
kernels against the fp64 clipped update (coef = 1: bit for bit the unclipped kernels); whole TrainEngine steps with an active
clip, checked after every step against the fp64 norm of the kernel's own gradient buffer and the fp64 clipped update of the
state before the step; an inactive clip giving the bits of no clip, eager and from a captured graph; a captured graph replayed
on batches with different norms, each replay checked the same way and against a second engine's replays."""
import math
from typing import Optional

import pytest
import torch

import lstm_numerics as N

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
N_HEADLINE = 1025 * 16384        # about the headline flat buffer (2 x 1024 LSTM + head)


@pytest.fixture(scope="module")
def E():
    from lstm_tensorspark_b200.ops.cuda_ext import ext
    return ext()


# ---- fp64 references ---------------------------------------------------------------------------------------------------------------
def _g_total(g, p, wd, gscale, wd_numel):
    """fp64 g * s + wd * p (decay on [0, wd_numel); -1 all) and |g| s + wd |p|, with the fp32 scalars the kernels receive."""
    w = torch.zeros(g.numel(), dtype=torch.float64, device=g.device)
    w[:g.numel() if wd_numel < 0 else wd_numel] = N.f32(wd)
    s = N.f32(gscale)
    g, p = g.double().reshape(-1), p.double().reshape(-1)
    return g * s + w * p, g.abs() * s + w * p.abs()


def _coef32(norm: torch.Tensor, max_norm: float) -> float:
    """min(max_norm / (norm + 1e-6), 1) in fp32 from the fp32 norm (IEEE division, as the kernel's __fdiv_rn)."""
    c = torch.tensor(max_norm, dtype=torch.float32) / (norm.float().cpu() + torch.tensor(1e-6, dtype=torch.float32))
    return float(torch.clamp(c, max=1.0))


def clipped_update(kind, p, m, v, g, coef, t: Optional[int], lr, wd=0.0, gscale=1.0, wd_numel=-1, b1=0.9, b2=0.999, eps=1e-8):
    """The clipped update kernels' math in fp64: lstm_numerics.adam_update / sgd_update with gg = coef * (g s + wd p).  The
    kernel rounds gg three times (wd p, the fma with g s, the coef product): 3u coef |gg|_abs, one u more than the unclipped
    kernel, so the m bound keeps its 8u and v's, where gg enters squared, grows from 8u to 10u."""
    U, F = N.U, N.UPDATE_FLOOR
    c = float(coef)
    gg, ga = _g_total(g, p, wd, gscale, wd_numel)
    gg, ga = c * gg, c * ga
    p0 = p.double().reshape(-1)
    if kind == "sgd":
        lr = N.f32(lr)
        return N.Update(p0 - lr * gg, None, None, 2 * U * p0.abs() + 5 * U * lr * ga + F, None, None)
    lr, b1, b2, eps = N.f32(lr), N.f32(b1), N.f32(b2), N.f32(eps)
    m, v = m.double().reshape(-1), v.double().reshape(-1)
    lr_t = lr if t is None else lr * math.sqrt(1.0 - b2 ** t) / (1.0 - b1 ** t)
    m1 = b1 * m + (1.0 - b1) * gg
    v1 = b2 * v + (1.0 - b2) * gg * gg
    den = v1.sqrt() + eps
    step = lr_t * m1 / den
    bm = 8 * U * (b1 * m.abs() + (1.0 - b1) * ga) + F
    bv = 10 * U * (b2 * v + (1.0 - b2) * ga * ga) + F
    bp = 2 * U * p0.abs() + N.RHO * step.abs() + lr_t * bm / den + F
    return N.Update(p0 - step, m1, v1, bp, bm, bv)


def _check_state(name, kind, p, m, v, shadow, ref):
    worst = N.check_update(f"{name} p", p, ref.p, ref.bound_p)
    if kind == "adam":
        worst = max(worst, N.check_update(f"{name} m", m, ref.m, ref.bound_m), N.check_update(f"{name} v", v, ref.v, ref.bound_v))
    if shadow is not None:
        N.check_shadow(name, shadow, p)
    return worst


# ---- the norm kernel alone -------------------------------------------------------------------------------------------------------
def _norm(E, g, p, max_norm, wd=0.0, gscale=1.0, wd_numel=-1, out=None, scratch=None):
    out = torch.full((2,), -1.0, device=DEV) if out is None else out
    if scratch is None:
        scratch = torch.zeros(E.flat_grad_norm_scratch(g.numel()), dtype=torch.float64, device=DEV)
    E.flat_grad_norm(g, p, out, scratch, max_norm, wd, gscale, wd_numel)
    return out


@pytest.mark.parametrize("n", [4, 1028, 10 ** 6 + 4, N_HEADLINE])
def test_norm_kernel_against_fp64(E, n):
    """g with magnitudes from 1e-4 to 1, weight decay 0.1 over a prefix, gradient scale 0.37: relative error <= 2e-5, coef as
    clip_grad_norm_ computes it in fp32 from that norm."""
    gen = torch.Generator(device=DEV).manual_seed(n % 977)
    g = torch.randn(n, generator=gen, device=DEV) * 10.0 ** (torch.rand(n, generator=gen, device=DEV) * 4 - 4)
    p = torch.randn(n, generator=gen, device=DEV)
    wd_numel = max(4, (n * 3 // 4) // 4 * 4)
    want = _g_total(g, p, 0.1, 0.37, wd_numel)[0].norm()
    for max_norm in (0.5 * float(want), 2.0 * float(want)):            # active / inactive
        out = _norm(E, g, p, max_norm, 0.1, 0.37, wd_numel)
        assert abs(float(out[0]) - float(want)) <= 2e-5 * float(want), (float(out[0]), float(want))
        assert float(out[1]) == _coef32(out[0], max_norm)
    assert float(_norm(E, g, p, 1.0, 0.1, 0.37, wd_numel)[0]) != float(_norm(E, g, p, 1.0, 0.0, 0.37, wd_numel)[0])
    # wd == 0 never reads p: a NaN there changes nothing
    pn = torch.full_like(p, float("nan"))
    assert torch.equal(_norm(E, g, p, 1.0, 0.0, 0.37), _norm(E, g, pn, 1.0, 0.0, 0.37))


def test_norm_kernel_special_values(E):
    n = 10 ** 6 + 4
    p = torch.zeros(n, device=DEV)
    g = torch.zeros(n, device=DEV)
    out = _norm(E, g, p, 0.5)
    assert float(out[0]) == 0.0 and float(out[1]) == 1.0
    g = torch.randn(n, device=DEV)
    g[n // 3] = float("inf")
    out = _norm(E, g, p, 0.5)
    assert math.isinf(float(out[0])) and float(out[1]) == 0.0
    g[n // 3] = float("nan")
    out = _norm(E, g, p, 0.5)
    assert math.isnan(float(out[0])) and math.isnan(float(out[1]))             # not fminf(NaN, 1) = 1
    g = torch.full((n,), 1e30, device=DEV)                                      # squares past fp32's range: summed in fp64
    out = _norm(E, g, p, 0.5)
    assert abs(float(out[0]) - 1e30 * math.sqrt(n)) <= 2e-5 * 1e30 * math.sqrt(n)


def test_norm_kernel_is_deterministic_across_calls_and_graph_replays(E):
    gen = torch.Generator(device=DEV).manual_seed(5)
    g = torch.randn(N_HEADLINE, generator=gen, device=DEV)
    p = torch.randn(N_HEADLINE, generator=gen, device=DEV)
    out = torch.zeros(2, device=DEV)
    scratch = torch.zeros(E.flat_grad_norm_scratch(N_HEADLINE), dtype=torch.float64, device=DEV)
    first = _norm(E, g, p, 1.0, 0.1, 0.5, N_HEADLINE // 2, out, scratch).clone()
    for _ in range(20):
        assert torch.equal(_norm(E, g, p, 1.0, 0.1, 0.5, N_HEADLINE // 2, out, scratch), first)
    graph = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        _norm(E, g, p, 1.0, 0.1, 0.5, N_HEADLINE // 2, out, scratch)
    torch.cuda.current_stream().wait_stream(s)
    with torch.cuda.graph(graph):
        _norm(E, g, p, 1.0, 0.1, 0.5, N_HEADLINE // 2, out, scratch)
    for k in range(5):
        out.zero_()
        graph.replay()
        assert torch.equal(out, first), k
    g2 = g * 3.0                                                              # new values in the captured buffer
    g.copy_(g2)
    want = _norm(E, g, p, 1.0, 0.1, 0.5, N_HEADLINE // 2).clone()
    out.zero_()
    graph.replay()
    assert torch.equal(out, want) and not torch.equal(want, first)
    assert int(scratch[-1:].view(torch.int64)[0] & 0xFFFFFFFF) == 0                 # the ticket is left 0


# ---- the clipped update kernels --------------------------------------------------------------------------------------------------
def _update_state(n, seed):
    gen = torch.Generator(device=DEV).manual_seed(seed)
    scale = 10.0 ** (torch.rand(n, generator=gen, device=DEV) * 4 - 4)
    p = torch.randn(n, generator=gen, device=DEV) * 0.05
    g = torch.randn(n, generator=gen, device=DEV) * scale
    m = torch.randn(n, generator=gen, device=DEV) * scale * 0.3
    v = scale * scale * (0.5 + torch.rand(n, generator=gen, device=DEV))
    for x in (p, g, m, v):
        x[-64:] = 0
    return p, g, m, v


@pytest.mark.parametrize("coef", [0.3125, 0.0123, 1.0])
@pytest.mark.parametrize("kind,t0", [("adam", None), ("adam", 1000), ("sgd", None)], ids=["adam-host-lr_t", "adam-t1000", "sgd"])
@pytest.mark.parametrize("n", [16384, N_HEADLINE])
def test_clipped_update_kernels_against_fp64(E, n, kind, t0, coef):
    """Two consecutive clipped updates with weight decay over [0, wd_numel) and a gradient scale, against the fp64 clipped update;
    coef = 1 also bit for bit against the unclipped kernel."""
    p, g, m, v = _update_state(n, seed=n % 1000 + int(coef * 1e4))
    wd, gscale, wd_numel = 0.1, 0.37, (n * 3 // 4) // 64 * 64 + 20
    lr = 0.05 if kind == "sgd" else 1e-3
    clip = torch.tensor([123.0, coef], device=DEV)
    sh = torch.empty_like(p, dtype=torch.bfloat16)
    step_dev = None if t0 is None else torch.full((1,), t0 - 1, dtype=torch.int32, device=DEV)
    plain = [x.clone() for x in (p, m, v)] + [torch.empty_like(sh), None if t0 is None else step_dev.clone()]
    worst = 0.0
    for k, gk in enumerate([g, g.roll(4096)]):
        gk[-64:] = 0
        p0, m0, v0 = p.clone(), m.clone(), v.clone()
        if kind == "sgd":
            E.flat_sgd(p, gk, sh, lr, wd, gscale, wd_numel, clip)
            ref = clipped_update("sgd", p0, None, None, gk, coef, None, lr, wd, gscale, wd_numel)
            E.flat_sgd(plain[0], gk, plain[3], lr, wd, gscale, wd_numel)
        else:
            t = k + 1 if t0 is None else t0 + k
            lr_k = lr * (1 - 0.999 ** t) ** 0.5 / (1 - 0.9 ** t) if t0 is None else lr
            E.flat_adam(p, gk, m, v, sh, lr_k, 0.9, 0.999, 1e-8, wd, gscale, step_dev, wd_numel, clip)
            ref = clipped_update("adam", p0, m0, v0, gk, coef, None if t0 is None else t, lr_k, wd, gscale, wd_numel)
            E.flat_adam(plain[0], gk, plain[1], plain[2], plain[3], lr_k, 0.9, 0.999, 1e-8, wd, gscale, plain[4], wd_numel)
        worst = max(worst, _check_state(f"step {k}", kind, p, m, v, sh, ref))
        assert not bool(p[-64:].any() or m[-64:].any() or v[-64:].any())
        same = torch.equal(p, plain[0]) and torch.equal(m, plain[1]) and torch.equal(v, plain[2]) and torch.equal(sh, plain[3])
        assert same == (coef == 1.0), (k, same)
        if coef != 1.0:
            plain = [x.clone() for x in (p, m, v)] + [sh.clone(), plain[4]]          # follow the clipped trajectory
    print(f"\nclipped {kind} n={n} t0={t0} coef={coef}: worst update ratio {worst:.3f}")


# ---- whole engine steps ----------------------------------------------------------------------------------------------------------
def _engine(clip: float = 0.0, **kw):
    from lstm_tensorspark_b200.config import Config
    from lstm_tensorspark_b200.engine import TrainEngine
    base = dict(partitions=1, sync_mode="none", init="scaled", device="cuda", quiet=True, learn_initial_state=False,
                dtype="bf16", learning_rate=1e-3, num_classes=10, deterministic=True)     # bitwise comparisons between engines
    base.update(kw)
    cfg = Config(clip_grad_norm=clip, **base).validate()
    return TrainEngine(cfg, 0, 1, None, batch_size=cfg.batch_size, device=DEV, dtype=torch.bfloat16)


def _batches(n, B, T, D, C=10, seed=0, scales=None):
    gen = torch.Generator(device=DEV).manual_seed(seed)
    out = []
    for k in range(n):
        s = 1.0 if scales is None else scales[k]
        out.append(((torch.randn(B, T, D, generator=gen, device=DEV) * s).bfloat16(),
                    torch.randint(0, C, (B,), generator=gen, device=DEV)))
    return out


def _state(eng):
    opt = eng.optimizer
    return [eng.flat.data.clone(), None if opt.m is None else opt.m.clone(), None if opt.v is None else opt.v.clone(),
            eng.flat.shadow.clone()]


@pytest.mark.parametrize("case", ["headline-adam", "sgd-wd-initial-state"])
def test_engine_steps_with_an_active_clip(case):
    if case == "headline-adam":
        kw = dict(hidden_units="1024,1024", in_features=1024, seq_len=128, batch_size=256, optimizer="adam")
        max_norm, steps = 1e-3, 3
    else:
        kw = dict(hidden_units="256,256,256", in_features=128, seq_len=16, batch_size=64, optimizer="sgd", weight_decay=0.01,
                  learn_initial_state=True, learning_rate=0.05)
        max_norm, steps = 1e-3, 4
    eng = _engine(max_norm, **kw)
    fl, opt, cfg = eng.flat, eng.optimizer, eng.cfg
    wd = cfg.weight_decay
    prev_coef, worst, controls = None, 0.0, 0
    scales = [1.0, 0.3, 2.0, 0.5][:steps]                                      # norms that differ: the negative control bites
    for k, (x, y) in enumerate(_batches(steps, cfg.batch_size, cfg.seq_len, cfg.in_features, seed=7, scales=scales)):
        p0, m0, v0, _ = _state(eng)
        eng.step(x, y)
        torch.cuda.synchronize()
        g = fl.grad                                                           # the kernel's own gradient, not modified by the clip
        norm64 = float(_g_total(g, p0, wd, 1.0, fl.lstm_numel)[0].norm())
        norm, coef = float(eng.grad_norm()), float(opt.clip_out[1])
        assert abs(norm - norm64) <= 2e-5 * norm64, (k, norm, norm64)
        assert coef == _coef32(opt.clip_out[0], max_norm) and coef < 1.0, (k, coef)
        t = opt.step_count
        ref = clipped_update(cfg.optimizer, p0, m0, v0, g, coef, t, cfg.learning_rate, wd, 1.0, fl.lstm_numel)
        worst = max(worst, _check_state(f"{case} step {k}", cfg.optimizer, fl.data, opt.m, opt.v, fl.shadow, ref))
        if prev_coef is not None and abs(prev_coef - coef) > 1e-3 * coef:       # negative control: last step's coef fails
            stale = clipped_update(cfg.optimizer, p0, m0, v0, g, prev_coef, t, cfg.learning_rate, wd, 1.0, fl.lstm_numel)
            with pytest.raises(AssertionError):
                _check_state("stale coef", cfg.optimizer, fl.data, opt.m, opt.v, None, stale)
            controls += 1
        prev_coef = coef
        assert not bool(fl.data[fl.numel:].any())                             # padding stays 0
    assert controls >= 1
    print(f"\n{case}: worst update ratio {worst:.3f}")


@pytest.mark.parametrize("graph", [False, True], ids=["eager", "graph"])
def test_inactive_clip_gives_the_bits_of_no_clip(graph):
    kw = dict(hidden_units="256,256", in_features=128, seq_len=16, batch_size=64, optimizer="adam", weight_decay=0.01)
    a, b = _engine(1e30, **kw), _engine(0.0, **kw)
    batches = _batches(4, 64, 16, 128, seed=3)
    if graph:
        a.capture(*batches[0]); b.capture(*batches[0])
    for x, y in batches[1:]:
        la, lb = a.step(x, y), b.step(x, y)
        assert abs(float(la) - float(lb)) <= 1e-6 * abs(float(lb))      # the reported loss's last bits vary between runs, clip or not
        assert float(a.optimizer.clip_out[1]) == 1.0
        for sa, sb in zip(_state(a), _state(b)):
            assert torch.equal(sa, sb)


def test_captured_graph_replays_batches_with_changing_norms():
    """Every replay writes its own norm and coef: checked against the fp64 norm of the gradient buffer that replay left and the fp64
    clipped update of the state before it; a second engine with the same seed replays the same bits, norms included."""
    kw = dict(hidden_units="256,256", in_features=128, seq_len=16, batch_size=64, optimizer="adam")
    batches = _batches(5, 64, 16, 128, seed=11, scales=[1.0, 0.05, 3.0, 0.2, 1.5])
    graphed, twin = _engine(1e-6, **kw), _engine(1e-6, **kw)
    for eng in (graphed, twin):
        eng.capture(batches[0][0].clone(), batches[0][1].clone())
    fl, opt = graphed.flat, graphed.optimizer
    norms, coefs = [], []
    for k, (x, y) in enumerate(batches):
        p0, m0, v0, _ = _state(graphed)
        lg, lt = graphed.step(x, y), twin.step(x, y)
        torch.cuda.synchronize()
        assert abs(float(lg) - float(lt)) <= 1e-6 * abs(float(lt)) and torch.equal(opt.clip_out, twin.optimizer.clip_out)
        assert torch.equal(fl.grad, twin.flat.grad)
        for sg, st in zip(_state(graphed), _state(twin)):
            assert torch.equal(sg, st)
        norm, coef = float(graphed.grad_norm()), float(opt.clip_out[1])
        norm64 = float(_g_total(fl.grad, p0, 0.0, 1.0, -1)[0].norm())
        assert abs(norm - norm64) <= 2e-5 * norm64, (k, norm, norm64)
        assert coef == _coef32(opt.clip_out[0], 1e-6)
        ref = clipped_update("adam", p0, m0, v0, fl.grad, coef, opt.step_count, 1e-3)
        _check_state(f"replay {k}", "adam", fl.data, opt.m, opt.v, fl.shadow, ref)
        norms.append(norm)
        coefs.append(coef)
    assert len(set(norms)) == len(norms) and len(set(coefs)) > 1, (norms, coefs)
