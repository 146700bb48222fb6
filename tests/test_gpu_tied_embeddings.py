"""Tied embeddings on the GPU (``--tie_embeddings``): the large-vocabulary head reading the embedding table ``[C,H] = W^T`` in
place as a K-major operand, against an fp64 reference within the bf16 budget of tests/test_gpu_next_token.py; its forward, lse,
dlogits and sampling bit for bit against the MN-major kernels fed ``W = table.t().contiguous()`` (the same bf16 values, the same
products in the same k order: only the shared-memory layout of B differs); whole tied training steps against the fp64 model
(the table's gradient the sum of the softmax's and the embedding's), an Adam update, eager against graph replay; the fallback
heads with tying and direct gradient sinks; a stateful tied step from the carried state; and generation, graph against eager.

Rounding points: unchanged from the untied head (bf16 h x bf16 table accumulated in fp32, plus the fp32 bias).  The table's
gradient is fp32: ``dlogits^T h`` (bf16 x bf16 in fp32) written first, the embedding's fixed-order scatter-add on top."""
import pytest
import torch

import lstm_numerics as N
from test_gpu_model_numerics import _engine, _names, _reference_params, _roundings, _segments, DEV
from test_gpu_next_token import _batch, _head, _inputs, _keep_tb, model_next_token

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _fp32_matmuls(monkeypatch):
    from lstm_tensorspark_b200.ops import cuda_lstm
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)
    monkeypatch.setattr(cuda_lstm, "SEQ_VARIANT", cuda_lstm.SEQ_VARIANT)     # (--deterministic sets a module-level knob)


def _stat(k):
    from lstm_tensorspark_b200.ops import cuda_lstm
    return cuda_lstm.STATS.get(k, 0)


# ---- the op alone ----------------------------------------------------------------------------------------------------------------
def _run_tied(h, table, b, labels, lengths, dloss=0.37):
    from lstm_tensorspark_b200.ops import functional as F
    hp, tp, bp = h.clone().requires_grad_(True), table.clone().requires_grad_(True), b.clone().requires_grad_(True)
    loss, correct, n = F.vocab_xent_per_step(hp, tp, bp, labels, lengths, class_major=True)
    (loss * dloss).backward()
    return loss.detach(), correct, n, hp.grad, tp.grad, bp.grad


@pytest.mark.parametrize("H", [64, 1024])
@pytest.mark.parametrize("Cn", [512, 1000, 4096])
def test_op_class_major_against_fp64(H, Cn):
    T, B = 9, 60                                                                 # 540 rows: a ragged row tile
    h, W, b, labels, lengths = _inputs(T, B, H, Cn, True, seed=H + Cn)
    table = W.t().contiguous()
    n_fwd, n_tied, n_old = _stat("vocab_head_fwd"), _stat("vocab_head_fwd_tied"), _stat("head_per_step")
    first = _run_tied(h, table, b, labels, lengths)
    assert (_stat("vocab_head_fwd"), _stat("vocab_head_fwd_tied"), _stat("head_per_step")) == (n_fwd + 1, n_tied + 1, n_old)
    loss, correct, n, dh, dT, db = first
    assert dT.shape == (Cn, H)
    keep = _keep_tb(lengths, T, B)
    lab = torch.where(keep.t(), labels, 0)
    assert int(n) == int(keep.sum())
    logits = h.double() @ W.bfloat16().double() + b.double()
    assert int(correct) == int(((logits.argmax(2) == lab.t()) & keep).sum()) and int(correct) > 0
    arms = {}
    for arm, dt, emu in (("fp64", torch.float64, False), ("emu", torch.float32, True)):
        l_, dh_, dW_, db_ = _head(h.to(dt), W, b, lab, lengths, emu, dloss=0.37)
        arms[arm] = {"loss": l_, "dh": dh_, "dT": dW_.t(), "db": db_}
    for k, v in {"loss": loss, "dh": dh, "dT": dT, "db": db}.items():
        N.check_budget(f"tied head H={H} C={Cn} {k}", v, arms["fp64"][k], arms["emu"][k])
    second = _run_tied(h, table, b, labels, lengths)
    for k, (x, y) in enumerate(zip(first, second)):
        assert torch.equal(x, y), k


@pytest.mark.parametrize("H,Cn", [(64, 1000), (1024, 4096), (256, 32768)])
def test_class_major_kernels_equal_the_mn_major_ones_bitwise(H, Cn):
    """Forward loss / lse / correct, the dlogits of the backward, and sampling at temperatures 0 and 1 for B = 1 and 256: the
    K-major table against the MN-major kernels fed ``table.t().contiguous()``, bit for bit."""
    from lstm_tensorspark_b200.ops import functional as F
    from lstm_tensorspark_b200.ops.cuda_ext import ext
    E = ext()
    T, B = 8, 70
    h, W, b, labels, lengths = _inputs(T, B, H, Cn, True, seed=Cn)
    tab = W.t().contiguous().bfloat16()
    wmn = tab.t().contiguous()
    h2 = h.reshape(T * B, H)
    out = {}
    for cm, w in ((True, tab), (False, wmn)):
        part = torch.empty(T * B * E.vocab_head_parts(Cn) * 4, dtype=torch.float32, device=DEV)
        lse, loss, correct, count = E.vocab_head_fwd(h2, w, cm, b, labels, lengths, T, part)
        dl = torch.empty(T * B, Cn, dtype=torch.bfloat16, device=DEV)
        scale = torch.full((1,), 0.5, device=DEV)
        E.vocab_head_dlogits(h2, w, cm, b, labels, lengths, T, lse, count, scale, 0, T * B, dl)
        out[cm] = [lse, loss, correct, count, dl]
    for k, (x, y) in enumerate(zip(out[True], out[False])):
        assert torch.equal(x, y), k
    for Bs in (1, 256):
        hs = torch.randn(Bs, H, generator=torch.Generator().manual_seed(Bs)).to(DEV, torch.bfloat16)
        for temperature in (0.0, 1.0):
            t = F.vocab_sample(hs, tab, b, temperature, 7, 3, class_major=True)
            u = F.vocab_sample(hs, wmn, b, temperature, 7, 3)
            assert torch.equal(t[0], u[0]) and torch.equal(t[1], u[1]), (Bs, temperature)


def test_class_major_needs_a_packed_aligned_table():
    from lstm_tensorspark_b200.ops.cuda_ext import ext
    E = ext()
    T, B, H, Cn = 2, 64, 64, 512
    h, W, b, labels, _ = _inputs(T, B, H, Cn, False)
    labels = labels.contiguous()
    buf = torch.zeros(Cn * H + 8, dtype=torch.bfloat16, device=DEV)
    off = buf[1:1 + Cn * H].view(Cn, H)                                          # 2 B past a 16-byte boundary
    part = torch.empty(T * B * E.vocab_head_parts(Cn) * 4, dtype=torch.float32, device=DEV)
    with pytest.raises(RuntimeError, match="16-byte aligned"):
        E.vocab_head_fwd(h.reshape(T * B, H), off, True, b, labels, None, T, part)


def test_op_gradients_with_and_without_a_flat_buffer():
    """A table and bias outside any flat buffer: their gradients leave the op through autograd in the table's layout, with the
    same bits as the ones written straight into the flat buffer's sinks."""
    from lstm_tensorspark_b200.models.flat import FlatParams
    from lstm_tensorspark_b200.ops import functional as F
    T, B, H, Cn = 6, 50, 128, 1024
    h, W, b, labels, lengths = _inputs(T, B, H, Cn, True, seed=4)
    table = torch.nn.Parameter(W.t().contiguous().bfloat16().float())
    bias = torch.nn.Parameter(b.clone())
    plain = (torch.nn.Parameter(table.detach().clone()), torch.nn.Parameter(bias.detach().clone()))
    flat = FlatParams([], [table, bias])
    flat.ensure_shadow()
    flat.enable_direct_grads([table, bias])
    flat.zero_grad()
    want = _run_tied(h, table.detach(), bias.detach(), labels, lengths, dloss=1.0)
    for direct, (tp, bp) in ((True, (table, bias)), (False, plain)):
        hp = h.clone().requires_grad_(True)
        F.vocab_xent_per_step(hp, tp, bp, labels, lengths, class_major=True)[0].backward()
        assert torch.equal(tp.grad, want[4]) and torch.equal(bp.grad, want[5]) and torch.equal(hp.grad, want[3]), direct


# ---- whole training steps ------------------------------------------------------------------------------------------------------
def _tied_reference(tok, table, layers, bias, labels, lengths, dropout, rounding):
    """model_next_token with the softmax matrix = table^T; the table's gradient is the sum of both uses."""
    loss, g = model_next_token(tok, table, layers, (table.t(), bias), labels, lengths, dropout, rounding)
    g["Embedding/weights"] = g["Embedding/weights"] + g.pop("Dense1/weights").t()
    return loss, g


def _tied_engine(**kw):
    eng = _engine(next_token=True, tie_embeddings=True, **kw)
    assert eng.model.head.weights is None and eng.model.tied
    names = _names(eng)
    names[id(eng.model.embedding.weights)] = "Embedding/weights"
    seg = _segments(eng, names)
    assert "Dense1/weights" not in seg
    return eng, seg


def _check_step(case, eng, seg, rounding, tok, y, lengths, data, loss, state=None):
    got = {"loss": loss.float()}
    for k, (o, shape) in seg.items():
        got[k] = eng.flat.grad[o:o + shape.numel()].view(shape).clone()
    with torch.no_grad():
        arms = {}
        for arm, dt, r in (("fp64", torch.float64, None), ("emu", torch.float32, rounding)):
            layers, head = _reference_params(eng, {**seg, "Dense1/weights": seg["Embedding/weights"]}, data, dt)
            if state is not None:
                layers = [(h.to(dt), c.to(dt)) + tuple(p[2:]) for p, (h, c) in zip(layers, state)]
            o, shape = seg["Embedding/weights"]
            table = data[o:o + shape.numel()].view(shape).bfloat16().to(dt)
            l_, g_ = _tied_reference(tok, table, layers, head[1], y, lengths, None, r)
            arms[arm] = {"loss": l_, **g_}
        assert set(got) <= set(arms["fp64"]) and "Embedding/weights" in got, sorted(got)
        for k, g in got.items():
            N.check_budget(f"{case} {k}", g, arms["fp64"][k], arms["emu"][k])


@pytest.mark.parametrize("ragged", [False, True])
def test_training_steps_against_fp64_with_an_adam_update(ragged):
    hidden, T, B, E, V = "256,256", 32, 128, 256, 1024
    eng, seg = _tied_engine(hidden_units=hidden, in_features=E, seq_len=T, batch_size=B, vocab_size=V, variable_length=ragged,
                            learning_rate=1e-3)
    flat, opt = eng.flat, eng.optimizer
    rounding = _roundings([256, 256], T, B, E, False)
    for s in range(2):
        tok, y, lengths = _batch(B, T, V, 5 + s, ragged)
        before = {"p": flat.data.clone(), "m": opt.m.clone(), "v": opt.v.clone()}
        n_tied, n_emb = _stat("vocab_head_fwd_tied"), _stat("embed_bwd")
        loss = eng.step(tok, y, lengths)
        torch.cuda.synchronize()
        assert (_stat("vocab_head_fwd_tied"), _stat("embed_bwd")) == (n_tied + 1, n_emb + 1)
        _check_step(f"tied step {s}", eng, seg, rounding, tok, y, lengths, before["p"], loss)
        t = int(opt.step_dev)
        upd = N.adam_update(before["p"], before["m"], before["v"], flat.grad, t, opt.lr, opt.beta1, opt.beta2, opt.eps,
                            0.0, 1.0, flat.lstm_numel)
        for k, (o, shape) in seg.items():
            sl = slice(o, o + shape.numel())
            for what, now, ref, bound in (("p", flat.data, upd.p, upd.bound_p), ("m", opt.m, upd.m, upd.bound_m),
                                          ("v", opt.v, upd.v, upd.bound_v)):
                N.check_update(f"tied step {s} {k} {what}", now[sl], ref[sl], bound[sl])


def test_eager_and_graph_steps_give_the_same_bits():
    kw = dict(hidden_units="256,256", in_features=256, seq_len=32, batch_size=128, vocab_size=1024, deterministic=True,
              learning_rate=1e-3, variable_length=True, dropout=0.1)
    (eager, _), (graphed, _) = _tied_engine(**kw), _tied_engine(**kw)
    assert torch.equal(eager.flat.data, graphed.flat.data)
    for s in range(4):
        tok, y, lengths = _batch(128, 32, 1024, 11 + s, True)
        if s == 1:
            graphed.capture(tok, y, lengths=lengths)
        le, lg = eager.step(tok, y, lengths), graphed.step(tok, y, lengths)
        torch.cuda.synchronize()
        assert torch.equal(le, lg) and torch.equal(eager.flat.data, graphed.flat.data), s
    assert graphed._graph is not None or graphed._bound


@pytest.mark.parametrize("V,dtype", [(256, torch.bfloat16), (1024, torch.float32)])
def test_fallback_heads_sum_both_gradients(V, dtype):
    """Inputs the tensor-core head does not take (C < 512; fp32) run the per-step head on ``table.t().contiguous()``: the
    tied engine's table gradient is the untied engine's embedding gradient plus its Dense1 gradient transposed, with the
    untied Dense1/weights set to the table's transpose.  bf16 runs with the direct gradient sinks on.  Both engines run the
    recurrences with the in-order operand stream (``deterministic``): the two are compared element by element, and the default
    stream does not give the same bits from run to run."""
    from lstm_tensorspark_b200.config import Config
    from lstm_tensorspark_b200.engine import TrainEngine
    hidden, T, B, E = "128,128", 16, 64, 128
    engines = []
    for tied in (True, False):
        cfg = Config(partitions=1, sync_mode="none", init="scaled", device="cuda", quiet=True, hidden_units=hidden, in_features=E,
                     seq_len=T, batch_size=B, vocab_size=V, next_token=True, tie_embeddings=tied, learning_rate=0.0,
                     variable_length=True, deterministic=True)
        eng = TrainEngine(cfg, 0, 1, None, batch_size=B, device=DEV, dtype=dtype)
        assert bool(eng.flat._direct) == (dtype == torch.bfloat16)
        engines.append(eng)
    tied, untied = engines
    with torch.no_grad():
        for name, v in tied.model.named_reference_variables():
            dict(untied.model.named_reference_variables())[name].copy_(v)
        untied.model.head.weights.copy_(tied.model.embedding.weights.t())
        for e in engines:
            e.flat.refresh_shadow()
    n_old, n_vocab = _stat("head_per_step"), _stat("vocab_head_fwd")
    for s in range(2):                                                          # the second step finds stale sinks
        tok, y, lengths = _batch(B, T, V, 3 + s, True)
        lt, lu = tied.step(tok, y, lengths), untied.step(tok, y, lengths)
        torch.cuda.synchronize()
        assert float(lt) == pytest.approx(float(lu), rel=1e-5)
        gt = tied.model.embedding.weights.grad
        gu = untied.model.embedding.weights.grad + untied.model.head.weights.grad.t()
        assert torch.allclose(gt, gu, rtol=1e-4, atol=1e-7 * float(gu.abs().max())), s
        assert float(tied.model.embedding.weights.grad.abs().max()) > 0
        assert torch.allclose(tied.model.head.bias.grad, untied.model.head.bias.grad, rtol=1e-4, atol=1e-7)
    assert _stat("head_per_step") == n_old + 4 and _stat("vocab_head_fwd") == n_vocab


def test_stateful_tied_step_from_the_carried_state():
    hidden, T, B, E, V = "256,256", 32, 128, 256, 1024
    eng, seg = _tied_engine(hidden_units=hidden, in_features=E, seq_len=T, batch_size=B, vocab_size=V, stateful=True)
    from lstm_tensorspark_b200 import data as D
    s = D.synthetic_stream(B * 2 + 1, T, V, seed=3)
    x, y, _ = D.stream_layout(s, B, T)
    x, y = torch.as_tensor(x).to(DEV), torch.as_tensor(y).to(DEV)
    eng.step(x[:B], y[:B], reset=True)
    data = eng.flat.data.clone()
    loss = eng.step(x[B:], y[B:])
    torch.cuda.synchronize()
    carried = [(h.clone(), c.clone()) for h, c in eng.state_prev]
    assert all(float(h.float().abs().max()) > 0 for h, _ in carried)
    _check_step("stateful tied step", eng, seg, _roundings([256, 256], T, B, E, False), x[B:], y[B:], None, data, loss,
                state=carried)


def test_generation_graph_equals_eager(monkeypatch):
    from lstm_tensorspark_b200.ops import cuda_lstm
    monkeypatch.setattr(cuda_lstm, "SEQ_VARIANT", (cuda_lstm.SEQ_VARIANT & ~(7 << 12)) | (3 << 12))   # --deterministic
    B, T, V = 64, 16, 4096
    eng, _ = _tied_engine(hidden_units="256,256", in_features=256, seq_len=T, batch_size=B, vocab_size=V)
    m = eng.model.eval()
    g = torch.Generator().manual_seed(2)
    x = torch.randint(0, V, (B, T), generator=g, dtype=torch.int32).to(DEV)
    lengths = torch.randint(1, T + 1, (B,), generator=g, dtype=torch.int32).to(DEV)
    n_tied = _stat("vocab_sample_tied")
    eager = m.generate(x, lengths, 8, 1.0, 5, graph=False)
    assert _stat("vocab_sample_tied") == n_tied + 8                              # one draw per token, from the table
    first = m.generate(x, lengths, 8, 1.0, 5)                                    # captures the decode step
    again = m.generate(x, lengths, 8, 1.0, 5)                                    # replays it
    for a in (first, again):
        assert torch.equal(a[0], eager[0]) and torch.equal(a[1], eager[1])
    assert bool(torch.isfinite(eager[1]).all()) and bool((eager[1] <= 0).all())
