"""The fused allreduce-and-update kernel (csrc/fused_allreduce.cu) against the fp64 update, element by element.

With ``--comm fused`` and ``--sync_mode grad_allreduce`` this kernel is the only thing that updates the weights of a multi-GPU
run: it sums the replicas' gradients, applies SGD or Adam with weight decay over ``[0, wd_numel)`` and writes the fp32 master
and its bf16 shadow into every replica, once per gradient bucket.  The update is held to the bound of the single-GPU update
kernels (``lstm_numerics.adam_update`` / ``sgd_update`` / ``check_update``), and the shadow must be the master rounded to
nearest even, bit for bit (``check_shadow``).

A. One GPU.  At world = 1 the kernel runs on ordinary device memory (``_solo``: a ``FusedComm`` whose one-rank arena is a plain
   allocation, so every launch goes through ``FusedComm._launch``'s offset, slot and weight-decay-cut arithmetic).  The barrier
   then waits only on the flag its own CTA just wrote, and the sum is ``g * 1.0``, which isolates the epilogue: every mode,
   both variants (one-shot, two-shot), grids of 1 to 300 CTAs (clamped to 256), the weight-decay cut, the bias correction
   from ``step_dev`` at resumed steps, bucket launches at element offsets in their own barrier slots, and the refusals.
B. Replicas (>= 2 GPUs, skipped otherwise): the peer-pointer sum in rank order (exact on the host) and the multicast sum
   (order free, bound widened), two-shot slices that do not divide evenly, bitwise-identical replicas, the Adam state that
   two-shot splits across ranks and ``optimizer_state()`` reassembles, resume from it, and parameter averaging.
C. Whole training steps (>= 2 GPUs): ``--comm fused`` with gradient buckets against ``--comm nccl`` on the same batches.

Negative controls apply a plausible slip to the REFERENCE side and require the bound to catch it: the weight-decay term dropped
for the last float4 below ``wd_numel``, the bias correction of step t - 1, and (B) the gradient sum without the 1 / W.

Agreement with ``flat_adam`` / ``flat_sgd`` (``test_agrees_with_the_flat_update_kernels``): on the same inputs at world = 1
both kernels are within the fp64 bound.  Adam's results are bitwise equal; SGD's are not (they differ in the last bits of
some elements).
"""
import math
import types

import pytest
import torch

import lstm_numerics as N

pytestmark = pytest.mark.gpu

MODE_AVG, MODE_SGD, MODE_ADAM = 0, 1, 2
N_HEADLINE = 1025 * 16384           # about the headline flat buffer (2 x 1024 LSTM + head), as in test_gpu_kernels.py
THREADS = 512                       # threads per CTA of the fused kernel: one float4 each per grid-stride pass
B1, B2, EPS = 0.9, 0.999, 1e-8


@pytest.fixture(scope="module")
def E():
    from lstm_tensorspark_b200.ops.cuda_ext import ext
    return ext()


@pytest.fixture(scope="module")
def dev():
    return torch.device("cuda", 0)


# ---- A. one GPU --------------------------------------------------------------------------------------------------------------
def _solo(dev, n):
    """A ``FusedComm`` of one rank whose "symmetric" arena is an ordinary zeroed allocation, carved as ``FusedComm.adopt``
    carves it: data, grad, stage, shadow, flags.  No process group and no symmetric memory are involved."""
    from lstm_tensorspark_b200.ops.cuda_ext import ext
    from lstm_tensorspark_b200.parallel.fused_comm import FusedComm, SymmetricArena, _align
    E = ext()
    total = 3 * _align(4 * n) + _align(2 * n) + _align(4 * E.ar_flag_words()) + 4096
    A = object.__new__(SymmetricArena)
    A.buf = torch.zeros(total, dtype=torch.uint8, device=dev)
    A.rank, A.world, A.off, A.nbytes = 0, 1, 0, total
    A.base, A.mc_base = [A.buf.data_ptr()], 0
    c = object.__new__(FusedComm)
    c.rank, c.world_size, c.device, c.timeout_s = 0, 1, dev, 60.0
    c.arena, c.use_multicast, c.blocks_override, c.launches = A, "0", 0, 0
    c._state_buckets, c._gs = [], None
    c.data, c.off_data = A.carve(n, torch.float32)
    c.grad, c.off_grad = A.carve(n, torch.float32)
    c.stage, c.off_stage = A.carve(n, torch.float32)
    c.shadow, c.off_shadow = A.carve(n, torch.bfloat16)
    c.flags, c.off_flags = A.carve(E.ar_flag_words(), torch.int32)
    c.slots = E.ar_slots()
    c.epochs = torch.zeros(E.ar_max_blocks() * c.slots, dtype=torch.int32, device=dev)
    c.err = torch.zeros(1, dtype=torch.int32, device=dev)
    return c


def _state(n, dev, seed):
    """fp32 p, m, v and a gradient with magnitudes from 1e-4 to 1; from 256 elements up the last 64 (the flat buffer's
    alignment padding) are all zero and must stay zero."""
    gen = torch.Generator(device=dev).manual_seed(seed)
    scale = 10.0 ** (torch.rand(n, generator=gen, device=dev) * 4 - 4)
    p = torch.randn(n, generator=gen, device=dev) * 0.05
    g = torch.randn(n, generator=gen, device=dev) * scale
    m = torch.randn(n, generator=gen, device=dev) * scale * 0.3
    v = scale * scale * (0.5 + torch.rand(n, generator=gen, device=dev))
    if n >= 256:
        for x in (p, g, m, v):
            x[-64:] = 0
    return p, g, m, v


def _mid(n):
    """A weight-decay cut inside the message: a multiple of 4 that is not one of 64."""
    return (n * 3 // 4) // 64 * 64 + 20 if n >= 128 else n // 2 // 4 * 4


def _lr_t(t):
    return 1e-3 * (1 - B2 ** t) ** 0.5 / (1 - B1 ** t)


def _launch(c, kind, n, *, force, blocks, lr, wd=0.0, wd_numel=-1, m=None, v=None, step_dev=None, bump=True, slot=0,
            elem_off=0, pdl=False):
    if kind == "sgd":
        return c._launch(MODE_SGD, c.off_grad, n, lr, wd=wd, force=force, elem_off=elem_off, wd_numel=wd_numel, pdl=pdl,
                         blocks=blocks, slot=slot)
    return c._launch(MODE_ADAM, c.off_grad, n, lr, B1, B2, EPS, wd, m, v, force=force, step_dev=step_dev, elem_off=elem_off,
                     wd_numel=wd_numel, bump_step=bump, pdl=pdl, blocks=blocks, slot=slot)


def _steps(c, kind, n, grads, *, force, blocks, wd, wd_numel, m=None, v=None, t0=None, bump=True, lr=None, check=True):
    """One launch per gradient (in place on c.data, m, v), each against the fp64 update of the state before it.  Adam: ``t0``
    None = the host's lr_t of steps 1, 2, ...; else step_dev preset to ``t0`` - 1 as a resumed run's, bumped by the launch
    (``bump``) or, as ``FusedComm.begin_grad_step`` does, by ``ar_bump_step`` before it.  -> (worst ratio, last reference,
    the inputs of the last step)."""
    from lstm_tensorspark_b200.ops.cuda_ext import ext
    p = c.data[:n]
    lr = lr if lr is not None else (0.05 if kind == "sgd" else 1e-3)
    step_dev = None if t0 is None else torch.full((1,), t0 - 1, dtype=torch.int32, device=c.device)
    worst, ref, before = 0.0, None, None
    for k, g in enumerate(grads):
        c.grad[:n].copy_(g)
        before = (p.clone(), None if m is None else m.clone(), None if v is None else v.clone(), g)
        padded = n >= 256 and not any(bool(x[-64:].any()) for x in before if x is not None)
        if kind == "sgd":
            _launch(c, kind, n, force=force, blocks=blocks, lr=lr, wd=wd, wd_numel=wd_numel)
            ref = N.sgd_update(before[0], g, lr, wd, 1.0, wd_numel)
        elif t0 is None:
            lr_t = lr * (1 - B2 ** (k + 1)) ** 0.5 / (1 - B1 ** (k + 1))
            _launch(c, kind, n, force=force, blocks=blocks, lr=lr_t, wd=wd, wd_numel=wd_numel, m=m, v=v)
            ref = N.adam_update(before[0], before[1], before[2], g, None, lr_t, B1, B2, EPS, wd, 1.0, wd_numel)
        else:
            if not bump:
                ext().ar_bump_step(step_dev)
            _launch(c, kind, n, force=force, blocks=blocks, lr=lr, wd=wd, wd_numel=wd_numel, m=m, v=v, step_dev=step_dev,
                    bump=bump)
            assert int(step_dev) == t0 + k                                  # once per step, by the launch or before it
            ref = N.adam_update(before[0], before[1], before[2], g, t0 + k, lr, B1, B2, EPS, wd, 1.0, wd_numel)
        torch.cuda.synchronize()
        assert int(c.err) == 0
        if not check:
            continue
        worst = max(worst, N.check_update(f"{kind} step {k} p", p, ref.p, ref.bound_p))
        if kind == "adam":
            worst = max(worst, N.check_update(f"step {k} m", m, ref.m, ref.bound_m),
                        N.check_update(f"step {k} v", v, ref.v, ref.bound_v))
        N.check_shadow(f"{kind} step {k}", c.shadow[:n], p)
        if padded:                                      # zero padding (p, g, m, v all 0) stays zero
            assert not bool(p[-64:].any()) and (m is None or not bool(m[-64:].any() or v[-64:].any()))
    return worst, ref, before


def _geometry(c, blocks, launches_per_slot):
    """The barrier bookkeeping of ``launches_per_slot[s]`` launches in slot s with ``blocks`` CTAs: the grid is clamped to 256,
    each CTA's epoch and its own flag advance by exactly 2 per launch, and nothing outside the slot's first CTAs is touched."""
    from lstm_tensorspark_b200.ops.cuda_ext import ext
    mb = ext().ar_max_blocks()
    nb = min(max(blocks, 1), mb)
    ep = c.epochs.view(c.slots, mb).cpu()
    fl = c.flags.view(c.slots, mb, -1).cpu()                # [slot][CTA][rank]
    for s in range(c.slots):
        want = 2 * launches_per_slot.get(s, 0)
        assert bool((ep[s, :nb] == want).all()) and not bool(ep[s, nb:].any()), (s, ep[s])
        assert bool((fl[s, :nb, 0] == want).all()) and not bool(fl[s, nb:].any()) and not bool(fl[s, :, 1:].any()), s


def _n_case(case, blocks):
    return {"one": 4, "small": 1028, "second_pass": 4 * THREADS * min(blocks, 256) + 4, "headline": N_HEADLINE}[case]


@pytest.mark.parametrize("blocks", [1, 64, 256, 300])
@pytest.mark.parametrize("case", ["one", "small", "second_pass", "headline"])
@pytest.mark.parametrize("force", ["one_shot", "two_shot"])
def test_update_against_fp64_at_every_grid(E, dev, force, case, blocks):
    """Two Adam steps (bias correction from step_dev at a resumed step 1000) and one SGD step, weight decay 0.1 over a cut inside
    the message, at 4 elements, one CTA pass, a second grid-stride pass and the headline size, on 1 to 300 CTAs.  300 must
    behave as 256: the same bits, and only 256 CTAs' barrier state touched."""
    n = _n_case(case, blocks)
    c = _solo(dev, n)
    p, g, m, v = _state(n, dev, seed=n % 997 + blocks)
    c.data.copy_(p)
    g2 = g.roll(4)
    if n >= 256:
        g2[-64:] = 0
    cut = _mid(n) if n > 4 else n
    worst = _steps(c, "adam", n, [g, g2], force=force, blocks=blocks, wd=0.1, wd_numel=cut, m=m, v=v, t0=1000)[0]
    worst = max(worst, _steps(c, "sgd", n, [g], force=force, blocks=blocks, wd=0.1, wd_numel=cut)[0])
    _geometry(c, blocks, {0: 3})
    assert c.launches == 3
    print(f"\n{force} n={n} blocks={blocks}: worst update ratio {worst:.3f}")
    if blocks == 300:                                     # bit for bit what 256 CTAs compute
        c256 = _solo(dev, n)
        c256.data.copy_(p)
        m2, v2 = _state(n, dev, seed=n % 997 + blocks)[2:]
        _steps(c256, "adam", n, [g, g2], force=force, blocks=256, wd=0.1, wd_numel=cut, m=m2, v=v2, t0=1000, check=False)
        _steps(c256, "sgd", n, [g], force=force, blocks=256, wd=0.1, wd_numel=cut, check=False)
        assert torch.equal(c256.data, c.data) and torch.equal(m2, m) and torch.equal(v2, v)


N_CUT = 4 * THREADS * 64 + 4        # two grid-stride passes of 64 CTAs; the second holds one float4


@pytest.mark.parametrize("wd,cut", [(0.0, -1), (0.1, -1), (0.1, 0), (0.1, "mid"), (0.1, "last"), (0.1, "n")],
                         ids=["no-wd", "wd-all", "wd-none", "wd-mid", "wd-all-but-last-float4", "wd-n"])
@pytest.mark.parametrize("kind", ["sgd", "adam"])
@pytest.mark.parametrize("force", ["one_shot", "two_shot"])
def test_weight_decay_cut(E, dev, force, kind, wd, cut):
    """Weight decay over [0, wd_numel): all (-1), none (0), a cut inside the first pass, one that leaves only the float4 of the
    second grid-stride pass undecayed, and n."""
    n = N_CUT
    cut = {"mid": _mid(n), "last": n - 4, "n": n}.get(cut, cut)
    c = _solo(dev, n)
    p, g, m, v = _state(n, dev, seed=11)
    p[-64:] = 0.05                          # no zero padding here: the last float4's decay must show
    g[-64:] = 1e-3
    m[-64:] = 1e-4
    v[-64:] = 1e-6
    c.data.copy_(p)
    _steps(c, kind, n, [g, g.flip(0)], force=force, blocks=64, wd=wd, wd_numel=cut, m=m if kind == "adam" else None,
           v=v if kind == "adam" else None, t0=None if kind == "sgd" else 3)


@pytest.mark.parametrize("t0,bump", [(None, False)] + [(t, b) for t in (1, 2, 1000, 100000) for b in (True, False)],
                         ids=["host-lr_t"] + [f"t{t}-{b}" for t in (1, 2, 1000, 100000)
                                              for b in ("bump-in-launch", "bumped-before")])
@pytest.mark.parametrize("force", ["one_shot", "two_shot"])
def test_adam_bias_correction(E, dev, force, t0, bump):
    """Adam with the host's lr_t (step_dev None), or the bias correction from step_dev preset to t0 - 1 as a resumed run's,
    bumped by the launch or before it (``FusedComm.begin_grad_step``): three steps over two grid-stride passes; the counter
    ends at t0 + 2."""
    n = N_CUT
    c = _solo(dev, n)
    p, g, m, v = _state(n, dev, seed=5 + (t0 or 0))
    c.data.copy_(p)
    _steps(c, "adam", n, [g, g.roll(8), g.roll(-4)], force=force, blocks=64, wd=0.1, wd_numel=_mid(n), m=m, v=v, t0=t0,
           bump=bump)


@pytest.mark.parametrize("force", ["one_shot", "two_shot"])
def test_average_at_one_rank(E, dev, force):
    """Parameter averaging of one replica: w * fp32(1 / 1), exactly (as values: the sum starts from +0, so -0 comes out +0;
    the kernels are built with --use_fast_math, which flushes denormals, so none are fed); the shadow rounded from it;
    one-shot stages w first."""
    n = N_CUT
    c = _solo(dev, n)
    w = _state(n, dev, seed=2)[0]
    w[:8] = torch.tensor([0.0, -0.0, 1e-30, -3.5, 65504.0, 1e30, -1.5e-38, 7.0])
    c.data.copy_(w)
    c._launch(MODE_AVG, c.off_data, n, force=force, blocks=64)
    torch.cuda.synchronize()
    assert int(c.err) == 0
    one = torch.tensor(N.f32(1.0 / 1), dtype=torch.float32, device=dev)
    assert torch.equal(c.data, w * one)
    N.check_shadow("average", c.shadow, c.data)
    if force == "one_shot":
        assert torch.equal(c.stage, w)
    _geometry(c, 64, {0: 1})


def _opt(kind, n, dev, wd, cut, t0, m, v):
    """What ``FusedComm.begin_grad_step`` / ``launch_bucket`` read of a ``FlatOptimizer``."""
    return types.SimpleNamespace(kind=kind, lr=1e-3 if kind == "adam" else 0.05, beta1=B1, beta2=B2, eps=EPS, weight_decay=wd,
                                 wd_numel=cut, m=m, v=v, step_count=t0 - 1,
                                 step_dev=torch.full((1,), t0 - 1, dtype=torch.int32, device=dev))


@pytest.mark.parametrize("kind", ["sgd", "adam"])
@pytest.mark.parametrize("force", ["one_shot", "two_shot"])
def test_buckets_equal_one_whole_launch(E, dev, force, kind):
    """One flat buffer in 3 buckets at multiples of 4 (not of 64), launched in sequence through ``FusedComm.launch_bucket``
    (slots 0, 1, 2; the second one a programmatic dependent), with the weight-decay cut inside the second bucket: two steps
    equal two whole-buffer launches bit for bit (master, shadow, m, v, step counter), each launch leaves err == 0, and the
    epochs of each slot advance by exactly 2 per step.  The whole-buffer run is also held to the fp64 update."""
    n = 3 * 4 * THREADS * 64 + 1028
    lo = [0, 4 * THREADS * 64 + 36, 2 * 4 * THREADS * 64 + 500, n]
    cut = lo[1] + 4 * 1000 + 8
    p, g, m, v = _state(n, dev, seed=21)
    grads = [g, g.roll(12)]
    grads[1][-64:] = 0
    runs = {}
    for split in (True, False):
        c = _solo(dev, n)
        c.data.copy_(p)
        mk, vk = (m.clone(), v.clone()) if kind == "adam" else (None, None)
        opt = _opt(kind, n, dev, 0.1, cut, 4, mk, vk)
        for k, gk in enumerate(grads):
            c.grad.copy_(gk)
            before = (c.data.clone(), None if mk is None else mk.clone(), None if vk is None else vk.clone())
            c.begin_grad_step(None, opt)
            bounds = list(zip(lo[:-1], lo[1:])) if split else [(0, n)]
            for b, (a, z) in enumerate(bounds):
                c.launch_bucket(a, z, pdl=split and b == 1, force=force, blocks=64)
                torch.cuda.synchronize()
                assert int(c.err) == 0
            assert c._gs["buckets"] == [(a, z, force == "two_shot") for a, z in bounds]
            if kind == "adam":
                assert int(opt.step_dev) == 4 + k and opt.step_count == 4 + k
                ref = N.adam_update(*before, gk, 4 + k, opt.lr, B1, B2, EPS, 0.1, 1.0, cut)
            else:
                ref = N.sgd_update(before[0], gk, opt.lr, 0.1, 1.0, cut)
            N.check_update(f"split={split} step {k} p", c.data, ref.p, ref.bound_p)
            if kind == "adam":
                N.check_update(f"split={split} step {k} m", mk, ref.m, ref.bound_m)
                N.check_update(f"split={split} step {k} v", vk, ref.v, ref.bound_v)
            N.check_shadow(f"split={split} step {k}", c.shadow, c.data)
        _geometry(c, 64, {s: 2 for s in range(len(lo) - 1 if split else 1)})
        runs[split] = (c.data.clone(), c.shadow.clone(), mk, vk)
    for a, b in zip(runs[True], runs[False]):
        assert a is None or torch.equal(a.view(torch.int16) if a.dtype == torch.bfloat16 else a.view(torch.int32),
                                        b.view(torch.int16) if b.dtype == torch.bfloat16 else b.view(torch.int32))


@pytest.mark.parametrize("kind", ["sgd", "adam"])
@pytest.mark.parametrize("n", [1028, N_HEADLINE])
@pytest.mark.parametrize("force", ["one_shot", "two_shot"])
def test_agrees_with_the_flat_update_kernels(E, dev, force, n, kind):
    """The fused kernel at world = 1 and flat_adam / flat_sgd on the same inputs (weight decay over a cut, Adam's bias
    correction from step_dev): both within the fp64 bound.  Adam is also equal bit for bit (the sum g * 1.0 is exact and the
    two epilogues round alike).  SGD is not: the two kernels' results differ in the last bits of some elements, so only the
    bound is asserted for it."""
    p, g, m, v = _state(n, dev, seed=n % 1000 + 3)
    cut = _mid(n)
    c = _solo(dev, n)
    c.data.copy_(p)
    mf, vf = (m.clone(), v.clone()) if kind == "adam" else (None, None)
    _steps(c, kind, n, [g, g.roll(4)], force=force, blocks=64, wd=0.1, wd_numel=cut, m=mf, v=vf, t0=None if kind == "sgd" else 7)
    pk, sh = p.clone(), torch.empty(n, dtype=torch.bfloat16, device=dev)
    step_dev = torch.full((1,), 6, dtype=torch.int32, device=dev)
    for gk in (g, g.roll(4)):
        before = (pk.clone(), m.clone(), v.clone())
        if kind == "sgd":
            E.flat_sgd(pk, gk, sh, 0.05, 0.1, 1.0, cut)
            ref = N.sgd_update(before[0], gk, 0.05, 0.1, 1.0, cut)
        else:
            E.flat_adam(pk, gk, m, v, sh, 1e-3, B1, B2, EPS, 0.1, 1.0, step_dev, cut)
            ref = N.adam_update(*before, gk, int(step_dev), 1e-3, B1, B2, EPS, 0.1, 1.0, cut)
        N.check_update("flat p", pk, ref.p, ref.bound_p)
        N.check_shadow("flat", sh, pk)
    if kind == "adam":
        assert torch.equal(pk.view(torch.int32), c.data.view(torch.int32))
        assert torch.equal(m.view(torch.int32), mf.view(torch.int32)) and torch.equal(v.view(torch.int32), vf.view(torch.int32))


def test_refusals_launch_nothing(E, dev):
    """A message that is not whole float4s, more than 16 ranks, and a weight-decay cut inside a float4 are refused before
    anything runs: not the step counter's bump, not an update, not the barrier."""
    from lstm_tensorspark_b200.parallel.fused_comm import FusedComm
    n = 1024
    c = _solo(dev, n)
    p, g, m, v = _state(n, dev, seed=9)
    c.data.copy_(p)
    c.grad.copy_(g)
    step_dev = torch.full((1,), 5, dtype=torch.int32, device=dev)
    snap = [t.clone() for t in (c.arena.buf, m, v, c.epochs, c.err, step_dev)]
    with pytest.raises(RuntimeError):
        _launch(c, "adam", n - 2, force="two_shot", blocks=64, lr=1e-3, m=m, v=v, step_dev=step_dev)
    with pytest.raises(RuntimeError):
        _launch(c, "adam", n, force="one_shot", blocks=64, lr=1e-3, wd=0.1, wd_numel=6, m=m, v=v, step_dev=step_dev)
    with pytest.raises(RuntimeError):
        _launch(c, "sgd", n, force="two_shot", blocks=64, lr=0.05, wd=0.1, wd_numel=1022)
    ptr = [c.arena.buf.data_ptr()]
    rows = torch.tensor([ptr * 17] * 4, dtype=torch.int64)
    with pytest.raises(RuntimeError):
        E.fused_allreduce(rows, 0, 0, 0, m, v, c.epochs[:256], c.err, n, 0, 17, MODE_ADAM, True, False, 64, 1e-3, B1, B2, EPS,
                          0.0, 60.0, step_dev, -1, True, False)
    with pytest.raises(AssertionError):                 # a bucket must start on a float4
        FusedComm._launch(c, MODE_SGD, c.off_grad, n - 4, 0.05, elem_off=2, force="two_shot")
    torch.cuda.synchronize()
    for a, b in zip(snap, (c.arena.buf, m, v, c.epochs, c.err, step_dev)):
        assert torch.equal(a, b)
    for bad in (E.flat_adam, E.flat_sgd):               # the flat kernels take the same cuts
        with pytest.raises(RuntimeError):
            if bad is E.flat_adam:
                bad(p, g, m, v, None, 1e-3, B1, B2, EPS, 0.1, 1.0, None, 6)
            else:
                bad(p, g, None, 0.05, 0.1, 1.0, 6)


@pytest.mark.parametrize("force", ["one_shot", "two_shot"])
def test_negative_controls_fail(E, dev, force):
    """The bound resolves the slips it exists for.  Applied to the reference, each must fail:
      * the weight-decay term dropped for the last float4 below wd_numel (SGD: p; Adam: m);
      * the bias correction of step t - 1 (at t = 2 and t = 100: it changes lr_t by more than the bound's RHO = 2^-11 while
        t stays below about 700; beyond, one step moves lr_t by less and the bound cannot tell the two apart).
    The correct reference passes on the same outputs."""
    n = N_CUT
    cut = _mid(n)
    p, g, m, v = _state(n, dev, seed=17)
    for kind in ("sgd", "adam"):
        c = _solo(dev, n)
        c.data.copy_(p)
        mk, vk = (m.clone(), v.clone()) if kind == "adam" else (None, None)
        _, ref, (p0, m0, v0, g0) = _steps(c, kind, n, [g], force=force, blocks=64, wd=0.1, wd_numel=cut, m=mk, v=vk,
                                          t0=None if kind == "sgd" else 2)
        if kind == "sgd":
            bad = N.sgd_update(p0, g0, 0.05, 0.1, 1.0, cut - 4)
            with pytest.raises(AssertionError):
                N.check_update("sgd without the last float4's decay", c.data, bad.p, bad.bound_p)
        else:
            bad = N.adam_update(p0, m0, v0, g0, 2, 1e-3, B1, B2, EPS, 0.1, 1.0, cut - 4)
            N.check_update("adam p", c.data, ref.p, ref.bound_p)
            with pytest.raises(AssertionError):
                N.check_update("adam without the last float4's decay", mk, bad.m, bad.bound_m)
    for t0 in (2, 100):
        c = _solo(dev, n)
        c.data.copy_(p)
        mk, vk = m.clone(), v.clone()
        _, ref, (p0, m0, v0, g0) = _steps(c, "adam", n, [g], force=force, blocks=64, wd=0.1, wd_numel=cut, m=mk, v=vk, t0=t0)
        bad = N.adam_update(p0, m0, v0, g0, t0 - 1, 1e-3, B1, B2, EPS, 0.1, 1.0, cut)
        with pytest.raises(AssertionError):
            N.check_update(f"adam at t {t0} with the bias correction of t - 1", c.data, bad.p, bad.bound_p)


# ---- B. replicas (>= 2 GPUs) -------------------------------------------------------------------------------------------------
def _grads(n, world, seed):
    """Every rank's gradient, identical on every rank (drawn on the host)."""
    gen = torch.Generator().manual_seed(seed)
    out = []
    for _ in range(world):
        scale = 10.0 ** (torch.rand(n, generator=gen) * 3 - 3)
        out.append(torch.randn(n, generator=gen) * scale)
    return out


def _peer_grad(gs, dev):
    """The peer-pointer kernel's gradient, exactly: the fp32 sum in rank order, times fp32(1 / W)."""
    s = gs[0].to(dev).clone()
    for g in gs[1:]:
        s = s + g.to(dev)
    return s * torch.tensor(N.f32(1.0 / len(gs)), dtype=torch.float32, device=dev), s


def _multicast_update(kind, p, m, v, gs, t, lr, wd, cut):
    """The update from the fp64 mean of the replicas' gradients, with its bound widened for a sum in any order.

    The switch adds the W fp32 gradients in an order of its own, so the kernel's gradient is not a function of the inputs the
    host can reproduce.  Its fp32 sum S differs from the exact sum by at most (W - 1) u sum_r |g_r| (W - 1 roundings of
    partial sums each bounded by sum_r |g_r|, to first order in u = 2^-24); fp32(1 / W) carries a relative error of at most u
    and the product one more rounding, so the kernel's g = S fp32(1/W) is within Delta = (W + 1) u sum_r |g_r| / W <= W u
    sum_r |g_r| of the mean for W >= 2 (the second-order terms fit in the difference).  The fp64 update of the mean plus the
    update's sensitivity to its gradient times Delta then bounds the kernel:
      SGD    p' = p - lr (g + wd p):           d p' / d g = lr;
      Adam   m' = b1 m + (1 - b1) gg:          (1 - b1) Delta;
             v' = b2 v + (1 - b2) gg^2:        (1 - b2) (2 |gg|_abs + Delta) Delta  (|gg + d|^2 - gg^2 <= 2 |gg| |d| + d^2);
             p' = p - lr_t m' / (sqrt(v') + eps): with S = sqrt(v'), d/dgg [m' / (S + eps)] = (1 - b1) / (S + eps) -
                    m' (1 - b2) gg / (S (S + eps)^2), and (1 - b2) |gg| / S <= sqrt(1 - b2) since S >= sqrt(1 - b2) |gg|, so
                    the derivative is at most [(1 - b1) + sqrt(1 - b2) |m'| / (S + eps)] / (S + eps).  Over gg +- Delta, S is
                    at least S_lo = sqrt(b2 v + (1 - b2) max(|gg| - Delta, 0)^2) and |m'| at most |m'| + (1 - b1) Delta, so
                    lr_t Delta [(1 - b1) + sqrt(1 - b2) (|m'| + (1 - b1) Delta) / (S_lo + eps)] / (S_lo + eps).
    The kernel's own roundings are bounded as in part A by the unwidened terms (computed at the mean: their change with the
    gradient is u times the widening)."""
    g64 = sum(g.double() for g in gs) / len(gs)
    delta = len(gs) * N.U * sum(g.double().abs() for g in gs)
    p, g64, delta = p.double(), g64.to(p.device), delta.to(p.device)
    if kind == "sgd":
        ref = N.sgd_update(p, g64, lr, wd, 1.0, cut)
        return ref._replace(bound_p=ref.bound_p + N.f32(lr) * delta)
    ref = N.adam_update(p, m, v, g64, t, lr, B1, B2, EPS, wd, 1.0, cut)
    gg, ga = N._decayed(p, g64, wd, 1.0, cut)
    b1, b2, eps = N.f32(B1), N.f32(B2), N.f32(EPS)
    lr_t = N.f32(lr) * math.sqrt(1.0 - b2 ** t) / (1.0 - b1 ** t)
    s_lo = (b2 * v.double() + (1 - b2) * (gg.abs() - delta).clamp_min(0) ** 2).sqrt()
    sens = ((1 - b1) + math.sqrt(1 - b2) * (ref.m.abs() + (1 - b1) * delta) / (s_lo + eps)) / (s_lo + eps)
    return ref._replace(bound_m=ref.bound_m + (1 - b1) * delta, bound_v=ref.bound_v + (1 - b2) * (2 * ga + delta) * delta,
                        bound_p=ref.bound_p + lr_t * delta * sens)


def _gather_equal(t):
    import torch.distributed as dist
    out = [torch.empty_like(t) for _ in range(dist.get_world_size())]
    dist.all_gather(out, t.contiguous())
    return all(torch.equal(out[0].view(torch.int16 if t.dtype == torch.bfloat16 else torch.int32),
                           o.view(torch.int16 if t.dtype == torch.bfloat16 else torch.int32)) for o in out)


def _replica_worker(rank, world):
    import torch.distributed as dist
    from lstm_tensorspark_b200.models.flat import FlatParams
    from lstm_tensorspark_b200.ops.optim import FlatOptimizer
    from lstm_tensorspark_b200.parallel.fused_comm import FusedComm
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    comm = FusedComm(rank, world, dev, 60)
    sizes = [4, 4 * (3 * world + 1), 4 * (20000 * world + world - 1)]    # n4 < W; n4 % W != 0 (small, several passes)
    flat = FlatParams([torch.nn.Parameter(torch.zeros(max(sizes), device=dev))], [])
    comm.adopt(flat)
    out = {"multicast": bool(comm.arena.mc_base), "checked": []}
    variants = [("one_shot", "0"), ("two_shot", "0")] + ([("two_shot", "1")] if comm.arena.mc_base else [])

    def sync():
        torch.cuda.synchronize()
        dist.barrier(device_ids=[rank])

    # ---- gradient sum + SGD / Adam, every variant and edge size ----------------------------------------------------------
    for n in sizes:
        cut = _mid(n) if n > 4 else n
        p0, _, m0, v0 = _state(n, dev, seed=n % 1000)                  # identical on every rank
        for force, mc in variants:
            comm.use_multicast = mc
            for kind, t0 in (("sgd", 1), ("adam", 1), ("adam", 1000)):
                gs = _grads(n, world, seed=n + t0)
                opt = FlatOptimizer(flat, 1e-3 if kind == "adam" else 0.05, kind, weight_decay=0.1)
                opt.wd_numel = cut
                flat.data.zero_()
                flat.data[:n].copy_(p0)
                flat.grad.zero_()
                flat.grad[:n].copy_(gs[rank])
                if kind == "adam":
                    opt.m[:n].copy_(m0)
                    opt.v[:n].copy_(v0)
                    opt.step_count = t0 - 1
                    opt.step_dev.fill_(t0 - 1)
                sync()
                comm.begin_grad_step(flat, opt)
                comm.launch_bucket(0, n, force=force)
                sync()
                comm.check_errors()
                full = comm.optimizer_state(opt) if kind == "adam" else None
                if mc == "1":
                    ref = _multicast_update(kind, p0, m0, v0, gs, t0, opt.lr, 0.1, cut)
                else:
                    g, s = _peer_grad(gs, dev)
                    if kind == "sgd":
                        ref = N.sgd_update(p0, g, opt.lr, 0.1, 1.0, cut)
                        bad = N.sgd_update(p0, s, opt.lr, 0.1, 1.0, cut)
                    else:
                        ref = N.adam_update(p0, m0, v0, g, t0, opt.lr, B1, B2, EPS, 0.1, 1.0, cut)
                        bad = N.adam_update(p0, m0, v0, s, t0, opt.lr, B1, B2, EPS, 0.1, 1.0, cut)
                    try:                                                 # negative control: the sum without 1 / W
                        N.check_update("gradient sum without 1/W", flat.data[:n], bad.p, bad.bound_p)
                        raise RuntimeError(f"the bound missed a gradient sum without 1/W ({force}, n={n}, {kind})")
                    except AssertionError:
                        pass
                name = f"{force} mc={mc} n={n} {kind} t={t0}"
                N.check_update(name + " p", flat.data[:n], ref.p, ref.bound_p)
                N.check_shadow(name, flat.shadow[:n], flat.data[:n])
                if kind == "adam":
                    N.check_update(name + " m", full["m"][:n].to(dev), ref.m, ref.bound_m)
                    N.check_update(name + " v", full["v"][:n].to(dev), ref.v, ref.bound_v)
                    assert int(opt.step_dev) == t0
                assert _gather_equal(flat.data) and _gather_equal(flat.shadow), name
                out["checked"].append(name)

    # ---- Adam state split by two-shot across ranks: 3 steps of 3 buckets, reassembled, then resumed --------------------------
    comm.use_multicast = "0"
    n = sizes[-1]
    lo = [0, (n // 3) // 4 * 4 + 4, (2 * n // 3) // 4 * 4 - 12, n]
    cut = lo[1] + 404

    def step(c, fl, op, k):
        fl.grad.zero_()
        fl.grad[:n].copy_(_grads(n, world, seed=100 + k)[rank])
        sync()
        c.begin_grad_step(fl, op)
        for b in range(3):
            c.launch_bucket(lo[b], lo[b + 1], pdl=b == 1, force="two_shot")
        sync()
        c.check_errors()

    p0, _, _, _ = _state(n, dev, seed=31)
    opt = FlatOptimizer(flat, 1e-3, "adam", weight_decay=0.1)
    opt.wd_numel = cut
    flat.data.zero_()
    flat.data[:n].copy_(p0)
    state = comm.optimizer_state(opt)
    for k in range(3):
        before = (flat.data[:n].clone(), state["m"][:n].to(dev), state["v"][:n].to(dev))
        step(comm, flat, opt, k)
        state = comm.optimizer_state(opt)
        g = _peer_grad(_grads(n, world, seed=100 + k), dev)[0]
        ref = N.adam_update(*before, g, k + 1, 1e-3, B1, B2, EPS, 0.1, 1.0, cut)
        N.check_update(f"state step {k} p", flat.data[:n], ref.p, ref.bound_p)
        N.check_update(f"state step {k} m", state["m"][:n].to(dev), ref.m, ref.bound_m)
        N.check_update(f"state step {k} v", state["v"][:n].to(dev), ref.v, ref.bound_v)
        assert _gather_equal(flat.data) and _gather_equal(flat.shadow)
    p3 = flat.data.clone()
    step(comm, flat, opt, 3)
    after = comm.optimizer_state(opt)
    comm2 = FusedComm(rank, world, dev, 60)
    flat2 = FlatParams([torch.nn.Parameter(p3[:max(sizes)].clone())], [])
    comm2.adopt(flat2)
    opt2 = FlatOptimizer(flat2, 1e-3, "adam", weight_decay=0.1)
    opt2.wd_numel = cut
    comm2.load_optimizer_state(opt2, state)
    step(comm2, flat2, opt2, 3)
    after2 = comm2.optimizer_state(opt2)
    out["resume_bitwise"] = (torch.equal(flat2.data.view(torch.int32), flat.data.view(torch.int32))
                             and torch.equal(flat2.shadow.view(torch.int16), flat.shadow.view(torch.int16))
                             and all(torch.equal(after[k].view(torch.int32), after2[k].view(torch.int32)) for k in ("m", "v"))
                             and after["step"] == after2["step"] == 4)
    comm2.check_errors()

    # ---- parameter averaging ------------------------------------------------------------------------------------------------
    gen = torch.Generator().manual_seed(77)
    ws = [torch.randn(flat.padded_numel, generator=gen) * (10.0 ** (torch.rand(flat.padded_numel, generator=gen) * 4 - 2))
          for _ in range(world)]
    for force, mc in [("one_shot", "0")] + variants[1:]:
        comm.use_multicast = mc
        flat.data.copy_(ws[rank])
        sync()
        comm.average_params_(flat, "all", force=force)
        sync()
        comm.check_errors()
        mean = sum(w.double() for w in ws) / world
        bound = (world + 2) * N.U * sum(w.double().abs() for w in ws) / world + N.UPDATE_FLOOR
        name = f"average {force} mc={mc}"
        N.check_update(name, flat.data, mean.to(dev), bound.to(dev))
        if mc == "0":                                   # rank order: exactly the host's fp32 emulation
            assert torch.equal(flat.data.view(torch.int32), _peer_grad(ws, dev)[0].view(torch.int32)), name
        N.check_shadow(name, flat.shadow, flat.data)
        assert _gather_equal(flat.data) and _gather_equal(flat.shadow), name
        out["checked"].append(name)
    comm2.close()
    comm.close()
    return out


def _worlds():
    n = torch.cuda.device_count()
    return sorted({2, min(n, 8)}) if n >= 2 else []


@pytest.mark.parametrize("which", ["two", "all"])
def test_replicas_against_fp64(which):
    """Part B at world = 2 and at min(device count, 8): every variant, edge sizes, the reassembled Adam state, resume and
    averaging (``_replica_worker``)."""
    worlds = _worlds()
    if not worlds:
        pytest.skip("needs >= 2 GPUs")
    world = worlds[0] if which == "two" else worlds[-1]
    if which == "all" and world == 2:
        pytest.skip("only 2 GPUs: covered by the world = 2 case")
    from lstm_tensorspark_b200.parallel.launch import launch
    res = launch(_replica_worker, world)
    for r in res:
        assert r["resume_bitwise"], r
        assert len(r["checked"]) == len(res[0]["checked"]) > 0


# ---- C. whole training steps (>= 2 GPUs) ---------------------------------------------------------------------------------------
def _engine_worker(rank, world, comm_kind, steps):
    from lstm_tensorspark_b200 import data as D
    from lstm_tensorspark_b200.config import Config
    from lstm_tensorspark_b200.engine import TrainEngine
    from lstm_tensorspark_b200.parallel.comm import make_communicator
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    cfg = Config(hidden_units="128,128", in_features=64, seq_len=8, batch_size=128, num_classes=10, partitions=world,
                 sync_mode="grad_allreduce", comm=comm_kind, grad_buckets=True, optimizer="adam", learning_rate=1e-3,
                 weight_decay=0.01, init="scaled", learn_initial_state=False, dtype="bf16", device="cuda", deterministic=True,
                 quiet=True)
    comm = make_communicator(comm_kind, rank, world, dev, 60)
    eng = TrainEngine(cfg, rank, world, comm, batch_size=128, device=dev, dtype=torch.bfloat16)
    flat, opt = eng.flat, eng.optimizer
    bound = torch.zeros_like(flat.data, dtype=torch.float64)
    for k in range(steps):
        x, y = D.synthetic_sequences(128, 8, 64, 10, seed=1000 * k + rank)
        before = (flat.data.clone(), opt.m.clone(), opt.v.clone())
        eng.step(torch.as_tensor(x).to(dev, torch.bfloat16), torch.as_tensor(y).to(dev))
        torch.cuda.synchronize()
        if comm_kind == "nccl":                            # flat.grad holds the summed gradient the update used
            ref = N.adam_update(*before, flat.grad, k + 1, opt.lr, B1, B2, EPS, 0.01, 1.0 / world, opt.wd_numel)
            N.check_update(f"nccl step {k} p", flat.data, ref.p, ref.bound_p)
            bound += ref.bound_p
    out = {"p": flat.data.cpu(), "bound": bound.cpu(), "launches": getattr(comm, "launches", 0), "wd_numel": opt.wd_numel}
    if comm_kind == "fused":
        comm.check_errors()
        out["identical"] = _gather_equal(flat.data) and _gather_equal(flat.shadow)
    comm.close()
    return out


def test_engine_fused_buckets_match_nccl():
    """Three two-GPU training steps with ``--comm fused`` (gradient buckets, Adam, weight decay over the LSTM segment) against
    the same steps with ``--comm nccl`` (all_reduce, then flat_adam) on the same batches.  The NCCL run is held to the fp64
    update step by step; the two runs' parameters may then differ by both runs' update bounds summed over the steps."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    from lstm_tensorspark_b200.parallel.launch import launch
    steps = 3
    fused = launch(_engine_worker, 2, args=("fused", steps))
    nccl = launch(_engine_worker, 2, args=("nccl", steps))
    for f, c in zip(fused, nccl):
        assert f["identical"]
        assert f["launches"] > steps, f["launches"]             # more than one bucket per step
        assert 0 < f["wd_numel"] < f["p"].numel()
        N.check_update("fused vs nccl", f["p"], c["p"].double(), 2 * c["bound"])
