"""AWD-LSTM's activation regularisation on the GPU (`pytest -m gpu`): the sum kernel against fp64 sums of its own inputs and bit
for bit across calls, the combine kernel element by element against the fp64 formula, the layer and pair ops' gradients with
``activation_sums=True`` against fp64 autograd on the reference, a whole language-model step with AWD's recipe and alpha = 2,
beta = 1 against the fp64 model, launch counts, and graph replays."""
import pytest
import torch

from lstm_tensorspark_b200.ops import reference as ref
from lstm_tensorspark_b200.ops.reference import DropoutSpec

import lstm_numerics as N

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
RECIPE = dict(locked_dropout=True, input_dropout=0.65, dropout=0.3, output_dropout=0.4, embedding_dropout=0.1,
              weight_drop=0.5)
AWD = dict(activation_reg=2.0, temporal_activation_reg=1.0)


def _rel_l2(a, b):
    return float((a.double() - b.double()).norm() / (b.double().norm() + 1e-30))


def _spec(p=0.4, locked=True, step=5, layer=1, reverse=False):
    return DropoutSpec(p, (123, 4), layer, reverse, torch.tensor([step], dtype=torch.int32, device=DEV), locked=locked)


def _lengths(T, B, seed):
    g = torch.Generator().manual_seed(seed)
    lengths = torch.randint(1, T + 1, (B,), generator=g, dtype=torch.int32)
    lengths[0], lengths[-1] = 1, T
    return lengths.to(DEV)


def _stats(keys=("act_reg_fwd", "act_reg_bwd", "fast_fwd", "fast_bwd", "generic_fwd", "generic_bwd", "batch_chunks")):
    from lstm_tensorspark_b200.ops import cuda_lstm
    return {k: cuda_lstm.STATS.get(k, 0) for k in keys}


def _delta(before):
    return {k: v - before[k] for k, v in _stats().items() if v != before[k]}


# ---- the kernels ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("H", [64, 1024, 100])
@pytest.mark.parametrize("ragged", [False, True])
@pytest.mark.parametrize("dropped", [False, True])
def test_sums_against_fp64_and_bitwise_across_calls(dt, H, ragged, dropped):
    from lstm_tensorspark_b200.ops import cuda_lstm
    T, B = 37, 24
    g = torch.Generator(device=DEV).manual_seed(H + T)
    h = torch.randn(T, B, H, generator=g, device=DEV).to(dt)
    out = ref.dropout(h, _spec()) if dropped else None
    lengths = _lengths(T, B, H) if ragged else None
    got = cuda_lstm._activation_sums(out, h, lengths)
    want = ref.activation_sums((h if out is None else out).double(), h.double(), lengths)
    assert torch.allclose(got.double(), want, rtol=1e-6, atol=0), (got, want)
    again = cuda_lstm._activation_sums(out, h, lengths)
    assert torch.equal(got.view(torch.int32), again.view(torch.int32))


def _combine_fp64(dh, out, h, lengths, g, spec):
    """keep * s * (dh + 2 g0 out) + 2 g1 (TAR stencil of h) at counted positions, keep * s * dh elsewhere, in fp64, and the
    magnitude of its terms (what fp32 arithmetic may lose)."""
    T, B, H = h.shape
    hd, g0, g1 = h.double(), 2 * float(g[0]), 2 * float(g[1])
    o = hd if out is None else out.double()
    keep = ref.step_mask(lengths, B, T, device=DEV).t().unsqueeze(2)
    fwd = torch.zeros_like(hd)
    fwd[1:] = hd[1:] - hd[:-1]
    bwd = torch.zeros_like(hd)
    bwd[:-1] = hd[1:] - hd[:-1]
    nxt = torch.zeros_like(keep)
    nxt[:-1] = keep[1:]
    st = fwd - torch.where(nxt, bwd, 0.0)
    a, mag_a = dh.double() + g0 * o, dh.double().abs() + abs(g0) * o.abs()
    if spec is not None:
        ms = ref.dropout_mask(spec, T, B, H, device=DEV).double() * float(ref.dropout_scale(spec.p))
        a, mag_a = a * ms, mag_a * ms
    hn = torch.zeros_like(hd)
    hn[:-1] = hd[1:].abs()
    hp = torch.zeros_like(hd)
    hp[1:] = hd[:-1].abs()
    plain = dh.double() if spec is None else dh.double() * ms
    want = torch.where(keep, a + g1 * st, plain)
    mag = torch.where(keep, mag_a + abs(g1) * (2 * hd.abs() + hp + hn), plain.abs())
    return want, mag


@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("H", [1024, 100])
@pytest.mark.parametrize("mask", ["off", "per_step", "locked"])
@pytest.mark.parametrize("ragged", [False, True])
def test_combine_against_the_fp64_formula(dt, H, mask, ragged):
    from lstm_tensorspark_b200.ops import cuda_lstm
    from lstm_tensorspark_b200.ops.cuda_ext import drop_args
    T, B = 35, 16
    gen = torch.Generator(device=DEV).manual_seed(H + len(mask))
    h = torch.randn(T, B, H, generator=gen, device=DEV).to(dt)
    dh = (torch.randn(T, B, H, generator=gen, device=DEV) * 1e-2).to(dt)
    g = torch.tensor([3e-3, 5e-3], device=DEV)
    spec = None if mask == "off" else _spec(locked=mask == "locked")
    out = None if spec is None else ref.dropout(h, spec)
    lengths = _lengths(T, B, H + 1) if ragged else None
    got = cuda_lstm._activation_grad(dh, out, h, lengths, g, drop_args(spec, DEV))
    want, mag = _combine_fp64(dh, out, h, lengths, g, spec)
    rnd = 2.0 ** -8 if dt == torch.bfloat16 else 2.0 ** -24
    f32 = 8 * 2.0 ** -24 * mag
    err = (got.double() - want).abs()
    assert bool((err <= rnd * (want.abs() + f32) + f32).all()), float((err / (rnd * want.abs() + f32 + 1e-300)).max())


# ---- the layer and pair ops --------------------------------------------------------------------------------------------------
def _params(T, B, D, H, dt, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    rn = lambda *s: torch.randn(*s, generator=g, device=DEV)
    x = (rn(T, B, D) * 0.5).to(dt)
    return x, [rn(B, H) * 0.1, rn(B, H) * 0.1, rn(4 * H, D) / D ** 0.5, rn(4 * H, H) / H ** 0.5, rn(4 * H) * 0.1]


COEF = torch.tensor([0.5, 0.5], dtype=torch.float64)         # d loss / d sums: the penalty's gradient is the head's size


def _loss(outs, w, sums):
    return (outs[0].double() * w).sum() + outs[1].double().sum() + outs[2].double().sum() + (COEF.to(DEV) * sums.double()).sum()


def _grads(fn, x, p):
    leaves = [x.clone().requires_grad_(True)] + [t.clone().requires_grad_(True) for t in p]
    fn(leaves).backward()
    torch.cuda.synchronize()
    return [t.grad for t in leaves]


@pytest.mark.parametrize("T,B,D,H,dt,ragged,reverse,mask", [
    (24, 128, 256, 256, torch.bfloat16, False, False, "locked"),      # one batch tile per CTA
    (24, 256, 256, 1024, torch.bfloat16, False, False, "per_step"),   # two tiles per CTA
    (24, 128, 256, 256, torch.bfloat16, True, True, "locked"),        # reverse, ragged
    (24, 256, 256, 1024, torch.bfloat16, True, False, "off"),         # ragged
    (16, 400, 256, 1024, torch.bfloat16, False, False, "locked"),     # batch chunks
    (16, 64, 32, 100, torch.bfloat16, True, False, "per_step"),       # generic path (H % 64 != 0)
    (16, 64, 32, 96, torch.float32, False, True, "locked"),           # generic path, fp32
])
def test_layer_op_gradients_against_fp64(T, B, D, H, dt, ragged, reverse, mask):
    """The op with ``activation_sums=True`` against fp64 autograd on ``reference.lstm_layer_sequence`` within ``check_budget``,
    whose comparison arm is the same op without the sums, its dropout and sums composed by torch on its output."""
    from lstm_tensorspark_b200.ops import cuda_lstm
    x, p = _params(T, B, D, H, dt, T + B + H)
    w = torch.randn(T, B, H, device=DEV, dtype=torch.float64)
    lengths = _lengths(T, B, 7) if ragged else None
    spec = None if mask == "off" else _spec(locked=mask == "locked", reverse=reverse)
    kw = dict(lengths=lengths, reverse=reverse)

    def fused(l):
        outs = cuda_lstm.lstm_layer_sequence(*l, dropout=spec, activation_sums=True, **kw)
        return _loss(outs, w, outs[3])

    def composed(l):
        raw, hT, cT = cuda_lstm.lstm_layer_sequence(*l, **kw)
        out = ref.dropout(raw.float(), spec)
        return _loss((out, hT, cT), w, ref.activation_sums(out, raw.float(), lengths))

    def fp64(l):
        outs = ref.lstm_layer_sequence(*[t.double() for t in l], dropout=spec, activation_sums=True, **kw)
        return _loss(outs, w, outs[3])

    n0 = _stats()
    got = _grads(fused, x, p)
    d = _delta(n0)
    assert d["act_reg_fwd"] == d["act_reg_bwd"] == (2 if B == 400 else 1), d
    emu, want = _grads(composed, x, p), _grads(fp64, x, p)
    for name, a, e, f in zip(("dx", "dh0", "dc0", "dW_x", "dW_h", "db"), got, emu, want):
        N.check_budget(name, a, f, e, floor=N.FLOOR if dt == torch.bfloat16 else N.FLOOR_F32)


@pytest.mark.parametrize("schedule", ["pipelined", "wavefront"])
def test_pair_op_gradients_against_fp64(schedule):
    from lstm_tensorspark_b200.ops import cuda_lstm
    T, B, D, Ha, Hb = 12, 256, 256, 512, 256
    x, pa = _params(T, B, D, Ha, torch.bfloat16, 11)
    _, pb = _params(T, B, Ha, Hb, torch.bfloat16, 12)
    w = torch.randn(T, B, Hb, device=DEV, dtype=torch.float64)
    sa, sb = _spec(0.3, layer=0), _spec(0.4, layer=1)

    def fused(l):
        outs = cuda_lstm.lstm_pair_sequence(l[0], l[1:6], l[6:], schedule=schedule, dropouts=(sa, sb), activation_sums=True)
        return _loss((outs[0], outs[3], outs[4]), w, outs[5])

    def composed(l):
        outs = cuda_lstm.lstm_pair_sequence(l[0], l[1:6], l[6:], schedule=schedule, dropouts=(sa, None))
        out = ref.dropout(outs[0].float(), sb)
        return _loss((out, outs[3], outs[4]), w, ref.activation_sums(out, outs[0].float()))

    def fp64(l):
        l = [t.double() for t in l]
        ha, _, _ = ref.lstm_layer_sequence(l[0], *l[1:6], dropout=sa)
        outs = ref.lstm_layer_sequence(ha, *l[6:], dropout=sb, activation_sums=True)
        return _loss(outs, w, outs[3])

    n0 = _stats()
    got = _grads(fused, x, pa + pb)
    assert _delta(n0) == {"act_reg_fwd": 1, "act_reg_bwd": 1, "fast_fwd": 2, "fast_bwd": 2}
    emu, want = _grads(composed, x, pa + pb), _grads(fp64, x, pa + pb)
    names = ["dx"] + [f"{n}_{l}" for l in "ab" for n in ("dh0", "dc0", "dW_x", "dW_h", "db")]
    for name, a, e, f in zip(names, got, emu, want):
        N.check_budget(name, a, f, e)


# ---- whole language-model steps -------------------------------------------------------------------------------------------------
def _lm_engine(deterministic=True, **kw):
    from lstm_tensorspark_b200.config import Config
    from lstm_tensorspark_b200.engine import TrainEngine
    cfg = Config(**{**dict(next_token=True, vocab_size=1024, hidden_units="256,256", in_features=256, seq_len=16, batch_size=64,
                           partitions=1, sync_mode="none", init="truncated_normal", init_std=0.1, learn_initial_state=False,
                           device="cuda", quiet=True, seed=2, deterministic=deterministic), **kw}).validate()
    return TrainEngine(cfg, 0, 1, None, batch_size=64, device=DEV, dtype=torch.bfloat16)


def _lm_batch(seed=3):
    from lstm_tensorspark_b200 import data as Dm
    x, y = Dm.synthetic_next_token(64, 16, 1024, seed=seed)[:2]
    return torch.as_tensor(x).to(DEV), torch.as_tensor(y).to(DEV)


def _fp64_grads(cpu, x, y, penalty):
    cpu.zero_grad()
    loss, _logits, _ = cpu(x, y)
    pen = cpu.rnn.activation_penalties
    total = loss + (2.0 * pen[0] + 1.0 * pen[1] if penalty else 0.0)
    total.backward()
    return float(loss), pen.detach(), {n: p.grad.clone() for n, p in cpu.named_parameters() if p.grad is not None}


@pytest.mark.parametrize("tied", [False, True])
@pytest.mark.parametrize("graph", [False, True])
def test_awd_step_against_the_fp64_model_fed_the_same_masks(tied, graph):
    """AWD's recipe with alpha = 2, beta = 1: the GPU step's loss, (AR, TAR) and every gradient against the fp64 model (the
    reference ops on the CPU) with the same weights and masks, with the tolerances of the recipe step without the penalties.
    The penalty must matter beyond them: without it the fp64 gradients of the top layer move by more than 10x the tolerance."""
    from lstm_tensorspark_b200.models.classifier import SequenceClassifier
    from lstm_tensorspark_b200.ops import cuda_lstm
    eng = _lm_engine(tie_embeddings=tied, **RECIPE, **AWD)
    x, y = _lm_batch()
    model = eng.model
    cpu = SequenceClassifier(eng.cfg, batch_size=64, device="cpu").double()
    cpu.load_state_dict({k: v.detach().double().cpu() for k, v in model.state_dict().items()})
    cpu.set_compute_dtype(torch.float64)
    cpu.rnn.dropout_key, cpu.rnn.dropout_step = model.rnn.dropout_key, 0
    want_loss, want_pen, want = _fp64_grads(cpu, x.cpu(), y.cpu(), True)
    _, _, plain = _fp64_grads(cpu, x.cpu(), y.cpu(), False)
    for n in want:
        if n.startswith("rnn.layers.1."):
            assert _rel_l2(want[n], plain[n]) >= 10 * 3e-2, (n, _rel_l2(want[n], plain[n]))
    if graph:
        eng.capture(x, y)
    n0 = _stats()
    loss = float(eng.step(x, y))
    torch.cuda.synchronize()
    cuda_lstm.check_kernel_errors(DEV)
    if not graph:
        assert {k: v for k, v in _delta(n0).items() if k.startswith("act_reg")} == {"act_reg_fwd": 1, "act_reg_bwd": 1}
    got = {n: p.grad.detach().double().cpu() for n, p in model.named_parameters() if p.grad is not None}
    assert abs(loss - want_loss) <= 5e-3 * abs(want_loss), (loss, want_loss)
    assert torch.allclose(eng.activation_penalties().double().cpu(), want_pen, rtol=2e-2), (eng.activation_penalties(), want_pen)
    assert got.keys() == want.keys()
    for n in want:
        assert _rel_l2(got[n], want[n]) < 3e-2, (n, _rel_l2(got[n], want[n]))


def test_launches_and_the_unmasked_top_recurrence(monkeypatch):
    """A coefficient on: one act_reg_fwd and one act_reg_bwd per step, and the top recurrence's backward gets no dropout mask
    (the combine applied it); both off: no new launch, and the kernels and results of the run without the flags."""
    from lstm_tensorspark_b200.ops import cuda_lstm
    from lstm_tensorspark_b200.ops.cuda_ext import LAUNCHES
    real = cuda_lstm.ext()
    calls = []

    class Spy:
        def __getattr__(self, name):
            fn = getattr(real, name)
            if not name.startswith("lstm_seq_bwd"):
                return fn
            return lambda *a, **k: (calls.append("drop_step" in k), fn(*a, **k))[1]

    monkeypatch.setattr(cuda_lstm, "ext", lambda: Spy())
    x, y = _lm_batch()
    for kw in (dict(temporal_activation_reg=1.0), dict(activation_reg=2.0)):
        e = _lm_engine(**RECIPE, **kw)
        calls.clear()
        n0 = _stats()
        e.step(x, y)
        torch.cuda.synchronize()
        d = _delta(n0)
        assert d["act_reg_fwd"] == 1 and d["act_reg_bwd"] == 1, d
        assert calls[0] is False                                      # the top layer's backward runs first, unmasked
    runs = []
    for kw in ({}, dict(activation_reg=0.0, temporal_activation_reg=0.0)):
        e = _lm_engine(**RECIPE, **kw)
        calls.clear()
        k0, l0, n0 = cuda_lstm.STATS["kernels"], LAUNCHES["n"], _stats()
        losses = [float(e.step(x, y)) for _ in range(2)]
        torch.cuda.synchronize()
        runs.append((losses, e.flat.data.clone(), cuda_lstm.STATS["kernels"] - k0, LAUNCHES["n"] - l0, _delta(n0), list(calls)))
        assert e.activation_penalties() is None
    assert runs[0][2:] == runs[1][2:] and "act_reg_fwd" not in runs[1][4] and runs[1][5][0] is True
    assert runs[0][0] == runs[1][0] and torch.equal(runs[0][1], runs[1][1])


def test_graph_replays_rewrite_the_penalties():
    x, y = _lm_batch()
    eager = _lm_engine(**RECIPE, **AWD)
    want = []
    for _ in range(3):
        eager.step(x, y)
        want.append(eager.activation_penalties().clone())
    graphed = _lm_engine(**RECIPE, **AWD)
    graphed.capture(x, y)
    buf = graphed.activation_penalties()
    got = []
    for _ in range(3):
        graphed.step(x, y)
        assert graphed.activation_penalties() is buf
        got.append(buf.clone())
    assert len({tuple(g.tolist()) for g in got}) == 3
    for a, b in zip(got, want):
        assert torch.allclose(a, b, rtol=1e-5), (a, b)
