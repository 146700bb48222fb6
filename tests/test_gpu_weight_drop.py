"""Weight drop on the GPU (`pytest -m gpu`): the masked image (the dropout kernel over W_h's [1, 4H, H] view) and the masked
weight-gradient kernel against the reference bit for bit; the layer op and both layer-pair schedules with a weight-drop spec
against the same op fed the explicit image, under the deterministic recurrences; whole headline training steps with Adam against
the fp64 model of tests/lstm_numerics.py; a captured step drawing a new mask on each replay; the gradient-bucket hook seeing only
masked gradients; and eval, generation and P = 0 launching nothing extra.  Every case asserts the kernels it targets through
cuda_lstm.STATS."""
import pytest
import torch

import lstm_numerics as N
from lstm_tensorspark_b200.ops import reference as ref
from lstm_tensorspark_b200.ops.reference import DropoutSpec

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
KEYS = ("fast_fwd", "fast_bwd", "generic_fwd", "generic_bwd", "batch_chunks", "pipelined_fwd", "wavefront_fwd", "weight_drop",
        "weight_drop_grad")
IN_ORDER = 3 << 12                 # the persistent kernels' in-order operand stream (--deterministic)


def _stats():
    from lstm_tensorspark_b200.ops import cuda_lstm
    return {k: cuda_lstm.STATS.get(k, 0) for k in KEYS}


def _delta(before):
    return {k: v - before[k] for k, v in _stats().items() if v != before[k]}


def _wspec(p=0.5, layer=0, reverse=False, step=5, key=(123, 4)):
    return DropoutSpec(p, key, layer, reverse, torch.tensor([step], dtype=torch.int32, device=DEV), weight=True)


def _masked_grad(g, spec):
    """M * s * g in fp32 (fp64 stays fp64): the gradient that reaches W_h."""
    keep = ref.weight_drop_mask(spec, *g.shape, device=g.device)
    return torch.where(keep, g * ref.dropout_scale(spec.p).to(g.dtype).to(g.device), torch.zeros((), dtype=g.dtype, device=g.device))


# ---- the kernels ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("H", [64, 1024])
def test_image_is_the_reference_weight_drop_bit_for_bit(dt, H):
    from lstm_tensorspark_b200.ops import cuda_lstm
    w = (torch.randn(4 * H, H, device=DEV) / H ** 0.5).to(dt)
    spec = _wspec(0.5, layer=1, reverse=True)
    n0 = _stats()
    img = cuda_lstm._weight_image(w, spec)
    assert _delta(n0) == {"weight_drop": 1}
    want = ref.weight_drop(w, spec)
    assert img.dtype == dt and torch.equal(img.view(torch.int16 if dt == torch.bfloat16 else torch.int32),
                                           want.view(torch.int16 if dt == torch.bfloat16 else torch.int32))
    assert cuda_lstm._weight_image(w, _wspec(0.0)) is w and _delta(n0) == {"weight_drop": 1}


@pytest.mark.parametrize("H", [64, 1024, 1280, 2048])
@pytest.mark.parametrize("mode", ["overwrite", "accumulate", "in_place"])
def test_gradient_kernel_is_src_times_mask_times_scale(H, mode):
    from lstm_tensorspark_b200.ops import cuda_lstm
    spec = _wspec(0.3, layer=0, step=17)
    src = torch.randn(4 * H, H, device=DEV)
    dst0 = torch.randn(4 * H, H, device=DEV)
    d = cuda_lstm._drop_args(spec, DEV)
    want = _masked_grad(src, spec)
    if mode == "accumulate":
        want = dst0 + want
    dst = src.clone() if mode == "in_place" else dst0.clone()
    n0 = _stats()
    cuda_lstm._weight_drop_grad(dst if mode == "in_place" else src, dst, d, mode == "accumulate")
    torch.cuda.synchronize()
    assert _delta(n0) == {"weight_drop_grad": 1}
    assert torch.equal(dst.view(torch.int32), want.view(torch.int32))
    keep = float((dst != (dst0 if mode == "accumulate" else 0)).float().mean())
    assert abs(keep - 0.7) < 0.01


# ---- the op with a spec against the op fed the explicit image --------------------------------------------------------------------
def _bits(t):
    return t.contiguous().view(torch.int16 if t.dtype == torch.bfloat16 else torch.int32)


def _lengths(T, B, seed):
    g = torch.Generator().manual_seed(seed)
    lengths = torch.randint(1, T + 1, (B,), generator=g, dtype=torch.int32)
    lengths[0], lengths[-1] = 1, T
    return lengths.to(DEV)


@pytest.mark.parametrize("T,B,D,H,cfg,masked,reverse,dt,path", [
    (16, 128, 64, 64, (6, 1, False, False), False, False, torch.bfloat16, {"fast_fwd": 1, "fast_bwd": 1}),     # one tile
    (32, 256, 256, 1024, (6, 2, False, False), False, False, torch.bfloat16, {"fast_fwd": 1, "fast_bwd": 1}),  # two tiles
    (32, 128, 256, 512, (5, 1, False, True), False, False, torch.bfloat16, {"fast_fwd": 1, "fast_bwd": 1}),   # forward K-split
    (16, 64, 256, 1280, (8, 1, True, False), False, False, torch.bfloat16, {"fast_fwd": 1, "fast_bwd": 1}),   # streamed weights
    (32, 256, 256, 1024, (6, 2, False, False), True, True, torch.bfloat16, {"fast_fwd": 1, "fast_bwd": 1}),   # lengths, reverse
    (16, 400, 256, 1024, None, False, False, torch.bfloat16, {"fast_fwd": 2, "fast_bwd": 2, "batch_chunks": 2}),   # batch chunks
    (6, 9, 12, 20, None, False, True, torch.float32, {"generic_fwd": 1, "generic_bwd": 1}),                   # generic fp32
])
def test_layer_op_equals_the_op_fed_the_masked_image(monkeypatch, T, B, D, H, cfg, masked, reverse, dt, path):
    from lstm_tensorspark_b200.ops import cuda_lstm
    from lstm_tensorspark_b200.ops.cuda_ext import ext
    if cfg is not None:
        assert ext().lstm_seq_config(False, H, B, cuda_lstm._seq_variant(B, H, DEV)) == cfg
    monkeypatch.setattr(cuda_lstm, "SEQ_VARIANT", IN_ORDER)
    g = torch.Generator(device=DEV).manual_seed(T + B + H)
    rn = lambda *s: torch.randn(*s, generator=g, device=DEV)
    x = (rn(T, B, D) * 0.5).to(dt)
    p = [rn(B, H) * 0.1, rn(B, H) * 0.1, rn(4 * H, D) / D ** 0.5, rn(4 * H, H) / H ** 0.5, rn(4 * H) * 0.1]
    lengths = _lengths(T, B, 4) if masked else None
    w, wT = rn(T, B, H), rn(B, H)
    spec = _wspec(0.5, layer=1, reverse=reverse)
    image = ref.weight_drop(p[3].to(dt), spec).float()              # the explicit W_h' (the op casts it back to dt exactly)

    def run(with_spec):
        leaves = [x.clone().requires_grad_(True)] + [t.clone().requires_grad_(True) for t in p]
        if not with_spec:
            leaves[4] = image.clone().requires_grad_(True)
        n0 = _stats()
        hs, hT, cT = cuda_lstm.lstm_layer_sequence(*leaves, lengths=lengths, reverse=reverse,
                                                   weight_drop=spec if with_spec else None)
        ((hs.float() * w).sum() + (hT.float() * wT).sum() + cT.sum()).backward()
        torch.cuda.synchronize()
        cuda_lstm.check_kernel_errors(DEV)
        return [hs.detach(), hT.detach(), cT.detach()] + [t.grad for t in leaves], _delta(n0)

    got, dg = run(True)
    want, dw = run(False)
    n = path.get("batch_chunks", 1)
    assert dw == path and dg == {**path, "weight_drop": n, "weight_drop_grad": n}, (dg, dw)
    for i in (0, 1, 2, 3, 4, 5, 6, 8):                     # h_seq, h_T, c_T, dx, dh0, dc0, dW_x, db
        assert torch.equal(_bits(got[i]), _bits(want[i])), i
    if n == 1:
        assert torch.equal(_bits(got[7]), _bits(_masked_grad(want[7], spec)))      # dW_h = M s dW_h'
    else:                                                 # per chunk: M s dW_h'(chunk), summed by autograd in another order
        assert torch.allclose(got[7], _masked_grad(want[7], spec), rtol=1e-5, atol=1e-6)


@pytest.mark.parametrize("schedule,T,Ha,Hb,D,p", [("pipelined", 32, 1024, 1024, 1024, 0.0), ("pipelined", 32, 1024, 1024, 1024, 0.3),
                                                 ("wavefront", 12, 512, 256, 256, 0.0), ("wavefront", 12, 512, 256, 256, 0.3)])
def test_layer_pair_equals_the_pair_fed_the_masked_images(monkeypatch, schedule, T, Ha, Hb, D, p):
    """The pipelined pair at the headline widths (dW_hb is a programmatic-dependent GEMM beside L_a, its mask an ordinary launch
    behind it; dW_ha carries db_a's row sums), the wavefront forced at a small shape; with and without --dropout."""
    from lstm_tensorspark_b200.ops import cuda_lstm
    monkeypatch.setattr(cuda_lstm, "SEQ_VARIANT", IN_ORDER)
    torch.manual_seed(11)
    B = 256
    mk = lambda *s, sc=1.0: (torch.randn(*s, device=DEV) * sc)
    x = mk(T, B, D, sc=0.5).bfloat16()
    pa = [mk(B, Ha, sc=0.1), mk(B, Ha, sc=0.1), mk(4 * Ha, D, sc=D ** -0.5), mk(4 * Ha, Ha, sc=Ha ** -0.5), mk(4 * Ha, sc=0.1)]
    pb = [mk(B, Hb, sc=0.1), mk(B, Hb, sc=0.1), mk(4 * Hb, Ha, sc=Ha ** -0.5), mk(4 * Hb, Hb, sc=Hb ** -0.5), mk(4 * Hb, sc=0.1)]
    wgt = mk(T, B, Hb)
    drops = (DropoutSpec(p, (9, 0), 0, False, torch.tensor([3], dtype=torch.int32, device=DEV)),
             DropoutSpec(p, (9, 0), 1, False, torch.tensor([3], dtype=torch.int32, device=DEV)))
    wds = (_wspec(0.5, layer=0, step=3, key=(9, 0)), _wspec(0.5, layer=1, step=3, key=(9, 0)))
    imgs = (ref.weight_drop(pa[3].bfloat16(), wds[0]).float(), ref.weight_drop(pb[3].bfloat16(), wds[1]).float())

    def run(with_spec):
        xa = x.clone().requires_grad_(True)
        a = [t.clone().requires_grad_(True) for t in pa]
        b = [t.clone().requires_grad_(True) for t in pb]
        if not with_spec:
            a[3], b[3] = imgs[0].clone().requires_grad_(True), imgs[1].clone().requires_grad_(True)
        n0 = _stats()
        hs, hTa, cTa, hTb, cTb = cuda_lstm.lstm_pair_sequence(xa, a, b, schedule=schedule, dropouts=drops,
                                                              weight_drops=wds if with_spec else (None, None))
        loss = (hs.float() * wgt).sum() + hTa.float().sum() + cTa.float().sum() * 0.5 + hTb.float().sum() + cTb.float().sum() * 0.25
        loss.backward()
        torch.cuda.synchronize()
        cuda_lstm.check_kernel_errors(DEV)
        return [hs.detach(), hTa.detach(), cTa.detach(), hTb.detach(), cTb.detach(), xa.grad] + [t.grad for t in a + b], _delta(n0)

    got, dg = run(True)
    want, dw = run(False)
    path = {"fast_fwd": 2, "fast_bwd": 2, f"{schedule}_fwd": 1}
    assert dw == path and dg == {**path, "weight_drop": 2, "weight_drop_grad": 2}, (dg, dw)
    for i, (a_, b_) in enumerate(zip(got, want)):
        if i == 6 + 3:
            b_ = _masked_grad(b_, wds[0])
        elif i == 6 + 5 + 3:
            b_ = _masked_grad(b_, wds[1])
        assert torch.equal(_bits(a_), _bits(b_)), i


# ---- whole training steps ---------------------------------------------------------------------------------------------------------
@pytest.fixture
def _fp32_matmuls(monkeypatch):
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)


def test_headline_adam_steps_against_fp64(_fp32_matmuls):
    """2 x 1024, T = 128, B = 256, D = 1024, --weight_drop 0.5, Adam at lr 1e-3 over 2 steps: the loss and every gradient of the
    flat buffer within the bf16 budget of the fp64 model fed the masked weights (its W_h gradients masked here), and the update
    of every tensor within check_update."""
    import test_gpu_model_numerics as M
    from lstm_tensorspark_b200 import data as Dm
    from lstm_tensorspark_b200.ops import cuda_lstm
    T, B, D, C, P, steps = 128, 256, 1024, 10, 0.5, 2
    hs = [1024, 1024]
    eng = M._engine(hidden_units="1024,1024", in_features=D, seq_len=T, batch_size=B, num_classes=C, weight_drop=P,
                    learning_rate=1e-3)
    flat, opt, rnn = eng.flat, eng.optimizer, eng.model.rnn
    xs, ys = Dm.synthetic_sequences(steps * B, T, D, C, seed=5)
    xs, ys = torch.as_tensor(xs).to(DEV).bfloat16(), torch.as_tensor(ys).to(DEV)
    names = M._names(eng)
    seg = M._segments(eng, names)
    rounding = M._roundings(hs, T, B, D, False)
    for s in range(steps):
        x, y = xs[s * B:(s + 1) * B], ys[s * B:(s + 1) * B]
        before = {"p": flat.data.clone(), "m": opt.m.clone(), "v": opt.v.clone(), "drop": int(rnn.dropout_step)}
        assert before["drop"] == s
        n0 = _stats()
        loss = eng.step(x, y)
        torch.cuda.synchronize()
        cuda_lstm.check_kernel_errors(DEV)
        assert _delta(n0) == {"fast_fwd": 2, "fast_bwd": 2, "pipelined_fwd": 1, "weight_drop": 2, "weight_drop_grad": 2}
        got = {"loss": loss.float()}
        for k, (o, shape) in seg.items():
            got[k] = flat.grad[o:o + shape.numel()].view(shape).clone()
        upd = N.adam_update(before["p"], before["m"], before["v"], flat.grad, int(opt.step_dev), opt.lr, opt.beta1, opt.beta2,
                            opt.eps, 0.0, 1.0, 0)
        for k, (o, shape) in seg.items():
            sl = slice(o, o + shape.numel())
            for what, now, r, bound in (("p", flat.data, upd.p, upd.bound_p), ("m", opt.m, upd.m, upd.bound_m),
                                        ("v", opt.v, upd.v, upd.bound_v)):
                N.check_update(f"step {s} {k} {what}", now[sl], r[sl], bound[sl])
        del upd
        specs = [DropoutSpec(P, rnn.dropout_key, l, False, before["drop"], weight=True) for l in range(len(hs))]
        with torch.no_grad():
            arms = {}
            for arm, dt, r in (("fp64", torch.float64, None), ("emu", torch.float32, rounding)):
                layers, head = M._reference_params(eng, seg, before["p"], dt)
                layers = [(h0, c0, wx, ref.weight_drop(wh.bfloat16(), sp).to(dt), b) for (h0, c0, wx, wh, b), sp in zip(layers, specs)]
                full = N.model(x.to(dt), layers, head, y, rounding=r)
                arms[arm] = {"loss": full.loss, **full.grads}
                for l, sp in enumerate(specs):
                    arms[arm][f"LSTMLayer{l}/w_h"] = _masked_grad(arms[arm][f"LSTMLayer{l}/w_h"], sp)
                del full
            worst = max(N.check_budget(f"step {s} {k}", g, arms["fp64"][k], arms["emu"][k]) for k, g in got.items())
            del arms
        print(f"\nweight drop headline step {s}: worst budget ratio {worst:.3f}")


def _headline_engine(**kw):
    from lstm_tensorspark_b200.config import Config
    from lstm_tensorspark_b200.engine import TrainEngine
    cfg = Config(**{**dict(hidden_units="1024,1024", in_features=1024, seq_len=128, batch_size=256, num_classes=10, partitions=1,
                           sync_mode="none", init="scaled", learn_initial_state=False, device="cuda", quiet=True, seed=3), **kw})
    return TrainEngine(cfg, 0, 1, None, batch_size=256, device=DEV, dtype=torch.bfloat16)


def _headline_batch():
    from lstm_tensorspark_b200 import data as Dm
    xs, ys = Dm.synthetic_sequences(256, 128, 1024, 10, seed=5)
    return torch.as_tensor(xs).to(DEV).bfloat16(), torch.as_tensor(ys).to(DEV)


def test_graph_replays_draw_a_new_mask_each(monkeypatch):
    """5 replays of a captured --weight_drop 0.5 step give the losses of 5 eager steps (within the one-ulp difference two
    identical --deterministic runs have shown at this shape), the counter advances inside the graph, and every loss differs."""
    from lstm_tensorspark_b200.ops import cuda_lstm
    monkeypatch.setattr(cuda_lstm, "SEQ_VARIANT", cuda_lstm.SEQ_VARIANT)
    x, y = _headline_batch()
    eager = _headline_engine(weight_drop=0.5, deterministic=True)
    want = [float(eager.step(x, y)) for _ in range(5)]
    graphed = _headline_engine(weight_drop=0.5, deterministic=True)
    n0 = _stats()
    graphed.capture(x, y)
    assert _delta(n0)["weight_drop"] == 2 * 4 and int(graphed.model.rnn.dropout_step) == 0
    got = [float(graphed.step(x, y)) for _ in range(5)]
    assert int(graphed.model.rnn.dropout_step) == int(eager.model.rnn.dropout_step) == 5
    assert all(abs(a - b) <= 1e-6 * abs(b) for a, b in zip(got, want)), (got, want)
    assert len(set(want)) == 5
    cuda_lstm.check_kernel_errors(DEV)


@pytest.mark.parametrize("hidden", ["1024,1024", "1024"])
def test_every_released_w_h_gradient_is_masked(hidden):
    """A single-replica stand-in for the gradient buckets: whenever a parameter is released to them, a listener snapshots (in
    stream order, where a bucket launched then would read) every W_h gradient already released.  Each snapshot must be the
    final, masked gradient: zero wherever the mask dropped.  The stand-in needs one GPU; the buckets' allreduce itself needs two."""
    from lstm_tensorspark_b200.ops import params
    x, y = _headline_batch()
    eng = _headline_engine(weight_drop=0.5, hidden_units=hidden)
    flat, rnn = eng.flat, eng.model.rnn
    snaps = {}

    def hook(released):
        for l, layer in enumerate(rnn.layers):
            if l not in snaps and layer.w_h.data_ptr() in flat._direct and layer.w_h.data_ptr() in released:
                snaps[l] = layer.w_h.grad.clone()

    flat.zero_grad()
    assert params._LISTENER is None
    n0 = _stats()
    with params.releases_to(hook):
        eng.step(x, y)
    torch.cuda.synchronize()
    assert _delta(n0)["weight_drop_grad"] == len(rnn.layers)
    assert sorted(snaps) == list(range(len(rnn.layers)))
    for l, layer in enumerate(rnn.layers):
        keep = ref.weight_drop_mask(DropoutSpec(0.5, rnn.dropout_key, l, False, 0, weight=True), *layer.w_h.shape, device=DEV)
        assert torch.equal(snaps[l], layer.w_h.grad), l
        assert not bool(snaps[l][~keep].any()) and bool(snaps[l][keep].any()), l


def test_zero_p_eval_and_generate_launch_nothing_extra(monkeypatch):
    from lstm_tensorspark_b200.ops import cuda_lstm
    from lstm_tensorspark_b200.ops.cuda_ext import LAUNCHES
    monkeypatch.setattr(cuda_lstm, "SEQ_VARIANT", cuda_lstm.SEQ_VARIANT)
    x, y = _headline_batch()
    runs = []
    for kw in ({}, {"weight_drop": 0.0}, {"weight_drop": 0.5}):
        e = _headline_engine(deterministic=True, **kw)
        k0, l0, n0 = cuda_lstm.STATS["kernels"], LAUNCHES["n"], _stats()
        losses = [float(e.step(x, y)) for _ in range(2)]
        torch.cuda.synchronize()
        runs.append((losses, e.flat.data.clone(), cuda_lstm.STATS["kernels"] - k0, LAUNCHES["n"] - l0, _delta(n0)))
    assert runs[0][2:4] == runs[1][2:4] and "weight_drop" not in runs[1][4]
    assert all(abs(a - b) <= 1e-6 * abs(b) for a, b in zip(runs[1][0], runs[0][0]))
    assert float((runs[1][1] - runs[0][1]).norm() / runs[0][1].norm()) < 1e-6
    assert runs[2][4]["weight_drop"] == 4 and runs[2][4]["weight_drop_grad"] == 4
    assert abs(runs[2][0][-1] - runs[0][0][-1]) > 1e-4 * abs(runs[0][0][-1])
    # evaluation: the raw weights, no weight-drop launch
    on, off = _headline_engine(deterministic=True, weight_drop=0.5), _headline_engine(deterministic=True)
    n0 = _stats()
    a, b = on.evaluate(x, y), off.evaluate(x, y)
    assert "weight_drop" not in _delta(n0)
    assert float(a[0]) == float(b[0]) and float(a[1]) == float(b[1])


def test_generate_uses_the_raw_weights():
    from lstm_tensorspark_b200.config import Config
    from lstm_tensorspark_b200.engine import TrainEngine
    mods = []
    for wd in (0.0, 0.5):
        cfg = Config(next_token=True, vocab_size=1024, hidden_units="256", in_features=256, seq_len=16, batch_size=128,
                     partitions=1, sync_mode="none", init="scaled", learn_initial_state=False, device="cuda", quiet=True, seed=2,
                     weight_drop=wd).validate()
        mods.append(TrainEngine(cfg, 0, 1, None, batch_size=128, device=DEV, dtype=torch.bfloat16).model)
    prompt = torch.randint(0, 1024, (128, 16), device=DEV, dtype=torch.int32)
    n0 = _stats()
    outs = [m.generate(prompt, None, 8, 1.0, 5, graph=False) for m in mods]
    torch.cuda.synchronize()
    assert "weight_drop" not in _delta(n0) and "weight_drop_grad" not in _delta(n0)
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
    assert all(m.training for m in mods)
