"""Next-token language modelling on the GPU: the large-vocabulary head op alone against an fp64 reference within the budget of its
bf16 emulation (tests/lstm_numerics.py), its bitwise determinism, the memory it does not allocate, its dispatch, both gradient
sink states, whole training steps of TrainEngine with ``next_token`` against an fp64 model reference, and tail scoring.

Rounding points of the large-vocabulary head (csrc/head_vocab.cu, ops/cuda_vocab_head.py):
  logits   bf16 h x bf16(W) accumulated in fp32, + fp32 bias, never rounded and never stored;
  lse      fp32;
  dlogits  (softmax - onehot) * dloss / N in fp32 at counted positions, 0 elsewhere, rounded once to bf16 after the scale;
  dh       bf16 dlogits x bf16(W) accumulated in fp32, stored bf16 - the top layer's dh_seq;
  dW, db   fp32 sums of bf16 h x bf16 dlogits and of the bf16 dlogits.
The model reference composes the layer loops of lstm_numerics behind the embedding, as tests/test_gpu_embedding.py does, with
this head at every step of the top layer's output, as tests/test_gpu_per_step_labels.py does."""
import pytest
import torch

import lstm_numerics as N
from test_gpu_model_numerics import _engine, _is_h100, _lengths, _names, _reference_params, _roundings, _sched, _segments, DEV

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _fp32_matmuls(monkeypatch):
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)


def _stat(k):
    from lstm_tensorspark_b200.ops import cuda_lstm
    return cuda_lstm.STATS.get(k, 0)


def _keep_tb(lengths, T, B):
    k = N._keep(lengths, T, B, DEV)
    return torch.ones(T, B, dtype=torch.bool, device=DEV) if k is None else k.t()


def _head(h_seq, W, b, labels, lengths, emulate, dloss=1.0, norm_all=False):
    """The head forward and backward in the precision of ``h_seq`` (fp64: exact; fp32 with ``emulate``: the rounding points at
    the top of this file).  -> (loss, dh_seq [T,B,H], dW, db).  ``norm_all``: divide by T·B instead of N (negative control)."""
    T, B, _ = h_seq.shape
    dt = h_seq.dtype
    r = N.Bf16() if emulate else None
    keep = _keep_tb(lengths, T, B).to(dt)
    Wr = N._round(r, W.to(dt))
    logp = torch.log_softmax(h_seq @ Wr + b.to(dt), 2)
    lab = (labels.long().t() * keep.long()).unsqueeze(2)                       # uncounted positions: any class, masked below
    n = float(T * B) if norm_all else keep.sum()
    loss = -(logp.gather(2, lab).squeeze(2) * keep).sum() / n
    dlogits = N._round(r, (logp.exp_().scatter_add_(2, lab, -torch.ones_like(lab, dtype=dt))) * keep.unsqueeze(2) * (dloss / n))
    dh = N._round(r, dlogits @ Wr.t())
    dW = h_seq.reshape(T * B, -1).t() @ dlogits.reshape(T * B, -1)
    return loss, dh, dW, dlogits.sum((0, 1))


# ---- the op alone ------------------------------------------------------------------------------------------------------------
def _inputs(T, B, H, Cn, ragged, seed=0):
    g = torch.Generator().manual_seed(seed)
    h = torch.randn(T, B, H, generator=g).to(DEV, torch.bfloat16)
    W = (torch.randn(H, Cn, generator=g) * (2.0 / H ** 0.5)).to(DEV)
    b = torch.randn(Cn, generator=g).to(DEV)
    labels = torch.randint(0, Cn, (B, T), generator=g).to(DEV)
    # half of the labels are the arg-max where it is clear of the runner-up, so that `correct` counts something
    top = (h.float() @ W.bfloat16().float() + b).topk(2, dim=2)
    clear = ((top.values[..., 0] - top.values[..., 1]) > 1e-3).t() & (torch.rand(B, T, generator=g).to(DEV) < 0.5)
    labels = torch.where(clear, top.indices[..., 0].t(), labels)
    lengths = None
    if ragged:
        lengths = torch.randint(1, T + 1, (B,), generator=g, dtype=torch.int32)
        lengths[0], lengths[1], lengths[-1] = 1, 0, T                             # a row that counts nothing, a full one
        lengths = lengths.to(DEV)
        labels = torch.where(_keep_tb(lengths, T, B).t(), labels, 10 ** 6)        # never read
    return h, W, b, labels, lengths


def _run(h, W, b, labels, lengths, dloss=0.37):
    from lstm_tensorspark_b200.ops import functional as F
    hp, Wp, bp = h.clone().requires_grad_(True), W.clone().requires_grad_(True), b.clone().requires_grad_(True)
    loss, correct, n = F.vocab_xent_per_step(hp, Wp, bp, labels, lengths)
    (loss * dloss).backward()
    return loss.detach(), correct, n, hp.grad, Wp.grad, bp.grad


@pytest.mark.parametrize("T,B,H,Cn,ragged", [
    (7, 19, 128, 512, True),            # T·B = 133: one full row tile and a ragged one, the backward GEMMs on the CUDA cores
    (5, 60, 256, 1000, False),          # C not a multiple of the class tile
    (6, 50, 2048, 520, True),           # the longest contraction
    (18, 250, 128, 32768, True),        # 4500 rows: two backward chunks, the last one ragged
    (33, 128, 192, 2048, True),         # 4224 rows: a last chunk of exactly one row tile
])
def test_op_against_fp64(T, B, H, Cn, ragged):
    h, W, b, labels, lengths = _inputs(T, B, H, Cn, ragged, seed=T + Cn)
    n_fwd, n_bwd, n_old = _stat("vocab_head_fwd"), _stat("vocab_head_bwd"), _stat("head_per_step")
    loss, correct, n, dh, dW, db = _run(h, W, b, labels, lengths)
    assert (_stat("vocab_head_fwd"), _stat("vocab_head_bwd"), _stat("head_per_step")) == (n_fwd + 1, n_bwd + 1, n_old)
    keep = _keep_tb(lengths, T, B)
    lab = torch.where(keep.t(), labels, 0)
    assert int(n) == int(keep.sum())
    logits = (h.double() @ W.bfloat16().double() + b.double())
    assert int(correct) == int(((logits.argmax(2) == lab.t()) & keep).sum()) and int(correct) > 0
    del logits
    arms = {}
    for arm, dt, emu in (("fp64", torch.float64, False), ("emu", torch.float32, True)):
        l_, dh_, dW_, db_ = _head(h.to(dt), W, b, lab, lengths, emu, dloss=0.37)
        arms[arm] = {"loss": l_, "dh": dh_, "dW": dW_, "db": db_}
    for k, v in {"loss": loss, "dh": dh, "dW": dW, "db": db}.items():
        N.check_budget(f"vocab head T={T} B={B} H={H} C={Cn} {k}", v, arms["fp64"][k], arms["emu"][k])
    assert float(dh.float()[~keep].abs().max() if (~keep).any() else 0.0) == 0.0      # no gradient into uncounted positions


def test_op_is_deterministic_and_stores_no_logits():
    """The headline shape (32768 rows x 32768 classes: logits and fp32 dlogits would be 4 GiB each): two calls give identical
    bits, and the call's peak memory grows by less than 1 GiB."""
    h, W, b, labels, lengths = _inputs(128, 256, 1024, 32768, True, seed=3)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    first = _run(h, W, b, labels, lengths)
    torch.cuda.synchronize()
    assert torch.cuda.max_memory_allocated() - base < 2 ** 30
    second = _run(h, W, b, labels, lengths)
    for k, (x, y) in enumerate(zip(first, second)):
        assert torch.equal(x, y), k
    assert bool(torch.isfinite(first[0])) and int(first[2]) == int(lengths.sum())


@pytest.mark.parametrize("Cn,dtype,vocab", [(512, torch.bfloat16, True), (300, torch.bfloat16, False), (504, torch.bfloat16, False),
                                            (512, torch.float32, False)])
def test_dispatch(Cn, dtype, vocab):
    from lstm_tensorspark_b200.ops import functional as F
    h, W, b, labels, lengths = _inputs(6, 21, 128, Cn, True)
    n_new, n_old = _stat("vocab_head_fwd"), _stat("head_per_step")
    loss, correct, n = F.vocab_xent_per_step(h.to(dtype), W, b, torch.where(labels > Cn, 0, labels), lengths)
    assert (_stat("vocab_head_fwd") - n_new, _stat("head_per_step") - n_old) == ((1, 0) if vocab else (0, 1))
    assert bool(torch.isfinite(loss)) and int(n) == int(lengths.sum())


def test_gradient_sinks_overwrite_then_accumulate():
    """Dense1's weights in a flat buffer: after zero_grad the first backward overwrites whatever the gradient views hold, a
    second one without zero_grad adds to them; each reads the maintained bf16 shadow."""
    from lstm_tensorspark_b200.models.classifier import DenseHead
    from lstm_tensorspark_b200.models.flat import FlatParams
    from lstm_tensorspark_b200.ops import functional as F
    T, B, H, Cn = 20, 250, 128, 1024                                               # 5000 rows: two chunks
    h, W, b, labels, lengths = _inputs(T, B, H, Cn, True, seed=9)
    want = _run(h, W.bfloat16().float(), b, labels, lengths, dloss=1.0)
    head = DenseHead(H, Cn, device=DEV)
    flat = FlatParams([], [head.weights, head.bias])
    with torch.no_grad():
        head.weights.copy_(W.bfloat16().float())
        head.bias.copy_(b)
    flat.ensure_shadow()
    flat.refresh_shadow()
    flat.enable_direct_grads([head.weights, head.bias])
    flat.grad.fill_(7.5)
    flat.zero_grad()
    hp = h.clone().requires_grad_(True)
    F.vocab_xent_per_step(hp, head.weights, head.bias, labels, lengths)[0].backward()
    assert torch.equal(head.weights.grad, want[4]) and torch.equal(head.bias.grad, want[5]) and torch.equal(hp.grad, want[3])
    F.vocab_xent_per_step(hp, head.weights, head.bias, labels, lengths)[0].backward()
    assert torch.allclose(head.weights.grad, 2 * want[4], rtol=1e-5, atol=1e-9)
    assert torch.allclose(head.bias.grad, 2 * want[5], rtol=1e-5, atol=1e-9)


# ---- whole training steps ------------------------------------------------------------------------------------------------------
def model_next_token(tok, table, layers, head, labels, lengths, dropout, rounding, norm_all=False):
    """Embedding -> the stacked layers -> the head at every step -> (loss, every gradient by name, the table's included)."""
    emulate = rounding is not None
    dt = torch.float32 if emulate else torch.float64
    B, T = tok.shape
    V, L = table.shape[0], len(layers)
    keep = N._keep(lengths, T, B, DEV)
    keep_tb = _keep_tb(lengths, T, B)
    ids = tok.t().long()
    rnd = (lambda l: rounding[l]) if emulate else (lambda l: None)
    seq = table.to(dt)[ids] * keep_tb.unsqueeze(2).to(dt)
    saved = []
    for l in range(L):
        fw = N._forward(seq, *layers[l], keep, False, rnd(l), None)
        h_seq = N._state_out(fw, False)[0]
        sc = None
        if dropout is not None and dropout.p > 0 and l < L - 1:
            sc = N._drop_scale(dropout, l, False, T, B, h_seq.shape[2], dt, DEV)
            h_seq = N._round(rnd(l), h_seq * sc)
        saved.append((fw, seq, sc))
        seq = h_seq
    loss, incoming, dW, db = _head(seq, head[0], head[1], labels, lengths, emulate, norm_all=norm_all)
    grads = {"Dense1/weights": dW, "Dense1/bias": db}
    for l in range(L - 1, -1, -1):
        fw, x_in, sc = saved[l]
        p = layers[l]
        g = N._backward(fw, x_in, p[2], p[3], incoming, None, None, keep, False, rnd(l), None, dh_scale=sc)
        for k, v in zip(("h0", "c0", "w_x", "w_h", "bias"), g[1:]):
            grads[f"LSTMLayer{l}/{k}"] = v
        incoming = g[0]
    grads["Embedding/weights"] = torch.zeros(table.shape, dtype=dt, device=DEV).index_add_(0, ids[keep_tb], incoming[keep_tb])
    return loss, grads


def _batch(B, T, V, seed, ragged):
    from lstm_tensorspark_b200 import data as Dm
    x, y, *l = Dm.synthetic_next_token(B, T, V, seed=seed, variable_length=False)
    lengths = _lengths(T, B, seed + 100) if ragged else None
    return torch.as_tensor(x).to(DEV), torch.as_tensor(y).to(DEV), lengths


def _case(case, hidden, T, B, E, V, path, steps=2, ragged=False, dropout=0.0, learning_rate=0.0, graph=False, clip=0.0,
          negative=False):
    """Training steps, each checked (loss and every gradient of the flat buffer) against the fp64 reference at the weights it
    read.  ``path``: a STATS key one step must bump (besides the large-vocabulary head).  ``graph``: captured on the first batch
    and replayed on every batch, each with lengths of its own.  ``negative``: the reference normalises by T·B."""
    eng = _engine(hidden_units=hidden, in_features=E, seq_len=T, batch_size=B, vocab_size=V, next_token=True, dropout=dropout,
                  variable_length=ragged, learning_rate=learning_rate, clip_grad_norm=clip)
    assert eng.cfg.per_step_labels and eng.cfg.num_classes == V
    flat = eng.flat
    names = _names(eng)
    names[id(eng.model.embedding.weights)] = "Embedding/weights"
    seg = _segments(eng, names)
    rounding = _roundings([int(h) for h in hidden.split(",")], T, B, E, False)
    worst = {}
    for s in range(steps):
        tok, y, lengths = _batch(B, T, V, 5 + s, ragged)
        before = {"p": flat.data.clone(), "drop": int(eng.model.rnn.dropout_step)}
        n_head, n_old, n_path = _stat("vocab_head_bwd"), _stat("head_per_step"), _stat(path)
        if graph and s == 0:
            eng.capture(tok, y, lengths=lengths)
            assert _stat("vocab_head_bwd") > n_head and _stat(path) > n_path, case
            n_head, n_path = _stat("vocab_head_bwd"), _stat(path)
        loss = eng.step(tok, y, lengths)
        torch.cuda.synchronize()
        if not graph:
            assert _stat("vocab_head_bwd") == n_head + 1 and _stat(path) > n_path, (case, s)
        assert _stat("head_per_step") == n_old
        got = {"loss": loss.float()}
        for k, (o, shape) in seg.items():
            got[k] = flat.grad[o:o + shape.numel()].view(shape).clone()
        drop = N.Dropout(dropout, eng.model.rnn.dropout_key, before["drop"]) if dropout > 0 else None
        with torch.no_grad():
            arms = {}
            for arm, dt, r in (("fp64", torch.float64, None), ("emu", torch.float32, rounding)):
                layers, head = _reference_params(eng, seg, before["p"], dt)
                o, shape = seg["Embedding/weights"]
                table = before["p"][o:o + shape.numel()].view(shape).bfloat16().to(dt)
                l_, g_ = model_next_token(tok, table, layers, head, y, lengths, drop, r, norm_all=negative)
                arms[arm] = {"loss": l_, **g_}
            if negative:
                with pytest.raises(AssertionError):
                    N.check_budget(f"{case} loss", got["loss"], arms["fp64"]["loss"], arms["emu"]["loss"])
                return
            assert set(got) <= set(arms["fp64"]), sorted(got)
            for k, g in got.items():
                worst[k] = max(worst.get(k, 0.0), N.check_budget(f"{case} step {s} {k}", g, arms["fp64"][k], arms["emu"][k]))
            if clip > 0:
                total = torch.sqrt(sum(arms["fp64"][k].double().square().sum() for k in got if k != "loss"))
                assert float(eng.grad_norm()) == pytest.approx(float(total), rel=2e-2)
            del arms
    top = sorted(worst.items(), key=lambda kv: -kv[1])[:3]
    print(f"\n{case}: worst budget ratio " + ", ".join(f"{k} {v:.3f}" for k, v in top))


def test_headline_pipelined_pair():
    if _is_h100():
        assert _sched(128, 256, 1024, 1024, 1024) == "pipelined"
    _case("next-token headline", "1024,1024", 128, 256, 1024, 4096, "pipelined_fwd")


def test_ragged_wavefront_pair():
    _case("next-token ragged", "512,512", 64, 256, 512, 2048, "fast_fwd", ragged=True)


def test_dropout():
    _case("next-token dropout", "512,512", 64, 256, 512, 1024, "fast_fwd", dropout=0.2)


def test_batch_chunks():
    """B = 400 at H = 1024: every layer runs as two persistent chunks; the top chunks' dh_seq slices come from one head."""
    _case("next-token batch chunks", "1024,1024", 32, 400, 256, 1000, "batch_chunks", steps=1)


def test_clip_grad_norm():
    _case("next-token clip", "256,256", 32, 128, 256, 512, "fast_fwd", steps=1, ragged=True, clip=0.5)


def test_adam_graph_replays_with_changing_lengths():
    """Captured once, replayed on 3 batches with lengths of their own: N, lse and the masks are computed on the device."""
    _case("next-token adam graph", "512,512", 64, 256, 512, 2048, "fast_fwd", steps=3, ragged=True, learning_rate=1e-3, graph=True)


def test_negative_control_normalised_by_all_positions():
    _case("next-token negative control", "256,256", 32, 128, 256, 512, "fast_fwd", steps=1, ragged=True, negative=True)


# ---- evaluation ----------------------------------------------------------------------------------------------------------------
def test_tail_scoring_masks_rows_and_builds_no_logits():
    """``score(first > 0)``: the tail rows' loss, correct count and N, with no ``[rows, C]`` array (1 GiB here) allocated."""
    from lstm_tensorspark_b200.ops import reference as ref
    T, B, V, first = 64, 256, 32768, 128
    eng = _engine(hidden_units="256,256", in_features=128, seq_len=T, batch_size=B, vocab_size=V, next_token=True,
                  variable_length=True)
    eng.model.eval()
    tok, y, lengths = _batch(B, T, V, 3, True)
    eng.model.score(tok, y, lengths, first)                                        # warm-up: modules, workspaces
    n_head, n_old = _stat("vocab_head_fwd"), _stat("head_per_step")
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    loss, ok, n = eng.model.score(tok, y, lengths, first)
    torch.cuda.synchronize()
    assert torch.cuda.max_memory_allocated() - base < (B - first) * T * V * 4 // 2
    assert (_stat("vocab_head_fwd"), _stat("head_per_step")) == (n_head + 1, n_old)
    with torch.no_grad():
        h_seq = eng.model.sequence_features(tok, lengths)[:, first:].double()
        W = eng.flat.shadow_view(eng.model.head.weights).double()
        _, l_ref, ok_ref, n_ref = ref.head_xent_per_step(h_seq, W, eng.model.head.bias.double(), y[first:], lengths[first:])
    assert int(n) == int(n_ref) == int(lengths[first:].sum()) and int(ok) == int(ok_ref)
    assert float(loss) == pytest.approx(float(l_ref), rel=1e-4)
