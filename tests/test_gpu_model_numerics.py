"""Whole training steps of the public TrainEngine (bf16, CUDA kernels) against the fp64 model reference of
tests/lstm_numerics.py, within the error budget of its bf16 emulation: the loss, h_T per batch row and every gradient segment
of the flat buffer, per tensor, by parameter name - step after step on different batches (dropout: a new mask each step).
This reaches what the layer-level tests do not: the direct gradient sinks (first write of a step overwrites, later ones
accumulate; split bias column sums; dW GEMMs launched beside the recurrence), batch chunks sharing those sinks, stacked /
bidirectional / dropout compositions, learned initial states, per-row lengths through the classifier and the head inside the
step.  Every case names the path it targets and asserts it through cuda_lstm.STATS (`pytest -m gpu`; `-s` prints each case's
worst budget ratios and its worst update ratio).
The cases with a learning rate train: each step is checked at the weights it read (the bf16 shadow the previous update wrote,
W^T derived from it, moved biases), and its update of the master weights and of Adam's m and v against the fp64 update of the
state before it (lstm_numerics.check_update), eager or replayed from a captured graph, with weight decay, from a resumed
state.  The cases at learning rate 0 keep the weights bf16-representable; Adam's m and v still move and are checked.
The file runs in about 40 s on an H100 80GB HBM3 at a 700 W power limit, fp64 arms included (the training cases take 13 s of
it); the worst budget ratio of any case was 0.52 there, the worst update ratio 0.75."""
import pytest
import torch

import lstm_numerics as N
from lstm_numerics import Bf16

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
STEPS = 3
C = 10
KEYS = ("fast_fwd", "fast_bwd", "generic_fwd", "generic_bwd", "batch_chunks", "pipelined_fwd", "wavefront_fwd", "folded_feed")


@pytest.fixture(autouse=True)
def _fp32_matmuls(monkeypatch):
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)     # the emulation's fp32 products stay fp32


def _stats():
    from lstm_tensorspark_b200.ops import cuda_lstm
    return {k: cuda_lstm.STATS.get(k, 0) for k in KEYS}


def _engine(dtype=torch.bfloat16, **kw):
    """A one-rank engine computing in ``dtype``: bf16 (weights made bf16-representable, so that learning rate 0 keeps the
    shadow exact) or fp32 (``--dtype fp32``: the kernels read the fp32 master itself; the weights are left as initialised)."""
    from lstm_tensorspark_b200.config import Config
    from lstm_tensorspark_b200.engine import TrainEngine
    cfg = Config(partitions=1, sync_mode="none", init="scaled", device="cuda", quiet=True, backend="auto",
                 **{"learning_rate": 0.0, **kw})
    eng = TrainEngine(cfg, 0, 1, None, batch_size=cfg.batch_size, device=DEV, dtype=dtype)
    if dtype == torch.bfloat16:
        with torch.no_grad():
            eng.flat.data.copy_(eng.flat.data.bfloat16().float())     # bf16-representable initial weights
            eng.flat.refresh_shadow()
    return eng


def _roundings(hidden, T, B, D, bidirectional):
    """The Bf16 of every layer: the pairs RNN._run_stack forms use the pair variant, single layers their own (per batch chunk)."""
    from lstm_tensorspark_b200.ops import cuda_lstm
    out, i, d_in = [], 0, D
    sms, cores = cuda_lstm._sms(DEV), cuda_lstm._coresident_ctas(DEV)
    while i < len(hidden):
        sched = None if bidirectional or i + 1 == len(hidden) else \
            cuda_lstm.pair_schedule(T, B, d_in, hidden[i], hidden[i + 1], sms, cores)
        if sched is not None:
            var = cuda_lstm._pair_variant(sched)
            out += [Bf16.for_layer(hidden[i], B, var), Bf16.for_layer(hidden[i + 1], B, var)]
            d_in, i = hidden[i + 1], i + 2
            continue
        rows = cuda_lstm._batch_chunk(B, hidden[i], torch.bfloat16, DEV) or B
        out.append(Bf16.for_layer(hidden[i], rows, cuda_lstm._seq_variant(rows, hidden[i], DEV)))
        d_in, i = hidden[i] * (2 if bidirectional else 1), i + 1
    return out


def _lengths(T, B, seed):
    g = torch.Generator().manual_seed(seed)
    lengths = torch.randint(1, T + 1, (B,), generator=g, dtype=torch.int32)
    lengths[0], lengths[B // 2], lengths[-1] = 1, T, T            # a one-step row, full-length rows (one in a later tile)
    return lengths.to(DEV)


def _names(eng):
    """id(parameter) -> the model reference's gradient name, for every tensor of the flat buffer."""
    rnn, out = eng.model.rnn, {}
    for l, layer in enumerate(rnn.layers):
        for lay in (layer,) + ((rnn.reverse_layers[l],) if rnn.bidirectional else ()):
            n = f"LSTMLayer{l}" + ("_reverse" if lay.reverse else "")
            for k in ("w_x", "w_h", "bias") + (("h0", "c0") if lay.learn_initial_state else ()):
                out[id(getattr(lay, k))] = f"{n}/{k}"
    out[id(eng.model.head.weights)] = "Dense1/weights"
    out[id(eng.model.head.bias)] = "Dense1/bias"
    return out


def _segments(eng, names):
    """name -> (offset, shape) of every tensor of the flat buffer."""
    return {names[id(p)]: (o, p.shape) for p, o in zip(eng.flat.params, eng.flat.offsets)}


def _reference_params(eng, seg, data, dt, bf16_weights=True):
    """The weights a step reads, from ``data`` (a snapshot of the fp32 master buffer): W_x / W_h rounded to bf16 here (the
    kernels read them from the shadow; ``bf16_weights=False``: an fp32 engine, which reads the master), the rest fp32.  Initial
    states that are not learned are the layers' zero buffers."""
    rnn = eng.model.rnn

    def get(name, k, lay):
        if f"{name}/{k}" not in seg:
            return getattr(lay, k).detach().to(dt)
        o, shape = seg[f"{name}/{k}"]
        t = data[o:o + shape.numel()].view(shape)
        return (t.bfloat16() if bf16_weights and k in ("w_x", "w_h") else t).to(dt)

    def one(l, lay):
        name = f"LSTMLayer{l}" + ("_reverse" if lay.reverse else "")
        return tuple(get(name, k, lay) for k in ("h0", "c0", "w_x", "w_h", "bias"))
    if rnn.bidirectional:
        layers = [(one(l, a), one(l, b)) for l, (a, b) in enumerate(zip(rnn.layers, rnn.reverse_layers))]
    else:
        layers = [one(l, a) for l, a in enumerate(rnn.layers)]
    return layers, (get("Dense1", "weights", None), get("Dense1", "bias", None))


def _load_resumed_state(eng, step, seed):
    """What a resumed run loads: the model's weights (its learned initial states scaled to 0.1, so that their L2 term stays
    small next to the loss in fp32) and Adam's m and v after ``step`` steps - nonzero on every parameter, zero in the padding."""
    model, opt = eng.model, eng.optimizer
    sd = model.reference_state_dict()
    for k in sd:
        if k.endswith("/state") or k.endswith("/context_state"):
            sd[k] = sd[k] * 0.1
    model.load_reference_state_dict(sd)
    gen = torch.Generator().manual_seed(seed)
    n = eng.flat.padded_numel
    scale = 10.0 ** (torch.rand(n, generator=gen) * 3 - 5)                   # |m| and sqrt(v) from 1e-5 to 1e-2
    m, v = torch.randn(n, generator=gen) * scale, scale * scale * (0.5 + torch.rand(n, generator=gen))
    real = torch.zeros(n, dtype=torch.bool)
    for p, o in zip(eng.flat.params, eng.flat.offsets):
        real[o:o + p.numel()] = True
    opt.load_state_dict({"kind": "adam", "step": step, "lr": opt.lr, "m": m * real, "v": v * real})
    eng.set_dropout_step(step)


def _model_case(case, hidden, T, B, D, per_step, steps=STEPS, lengths_seed=None, bidirectional=False, dropout=0.0,
                learn_initial_state=False, free_engine=False, learning_rate=0.0, optimizer="adam", weight_decay=0.0,
                graph=False, resume_at=None, stale_shadow=False, dtype=torch.bfloat16, rounding=None, weight_drop=0.0):
    """One training step after the other, each checked against the weights it read:
      * before the step: the bf16 shadow is the master rounded to nearest even, bit for bit;
      * the loss, h_T (eval mode, computed before the step) and every gradient of the flat buffer within the budget of the fp64
        model reference at the weights the step read;
      * the update: the master p and Adam's m and v after the step, element by element within ``lstm_numerics.check_update``
        of the fp64 update of the state before it and the step's gradient, weight decay on [0, end of the LSTM variables);
        every padding element of the flat buffer keeps a gradient and a parameter of 0.
    ``per_step``: the STATS deltas one training step must show (the path the case targets).  ``graph``: the step is captured
    once (on the first batch; STATS count only there) and replayed on every batch.  ``resume_at``: the run starts from a state
    loaded as a resumed run would at that step.  ``stale_shadow``: the shadow of the weights before step 1 is put back after
    it, standing in for a missing refresh (the shadow assertion is off): step 2's check must raise.
    ``dtype``: the engine's compute dtype; fp32 checks against the ``lstm_numerics.Fp32`` arm with the fp32 floor, and reads
    unrounded weights.  ``rounding``: the emulation arm's rounding in place of the fast path's (the bf16 generic path).
    ``weight_drop``: P of --weight_drop; both arms read the masked W_h of the step and mask its gradient."""
    from lstm_tensorspark_b200 import data as Dm
    from lstm_tensorspark_b200.models.flat import ALIGN
    from lstm_tensorspark_b200.ops import cuda_lstm
    hs = [int(h) for h in hidden.split(",")]
    from lstm_tensorspark_b200.ops import reference as ops_ref
    from test_gpu_weight_drop import _masked_grad
    bf16 = dtype == torch.bfloat16
    eng = _engine(dtype, hidden_units=hidden, in_features=D, seq_len=T, batch_size=B, num_classes=C, bidirectional=bidirectional,
                  dropout=dropout, learn_initial_state=learn_initial_state, variable_length=lengths_seed is not None,
                  learning_rate=learning_rate, optimizer=optimizer, weight_decay=weight_decay, weight_drop=weight_drop)
    flat, opt = eng.flat, eng.optimizer
    if resume_at is not None:
        _load_resumed_state(eng, resume_at, seed=3)
    xs, ys = Dm.synthetic_sequences(steps * B, T, D, C, seed=5)
    xs, ys = torch.as_tensor(xs).to(DEV).to(dtype), torch.as_tensor(ys).to(DEV)
    names = _names(eng)
    assert len(names) == len(flat.params)
    seg = _segments(eng, names)
    lstm_end = max(o + shape.numel() for k, (o, shape) in seg.items()
                   if k.startswith("LSTMLayer") and k.split("/")[1] in ("w_x", "w_h", "bias"))
    wd_numel = (lstm_end + ALIGN - 1) // ALIGN * ALIGN                     # weight decay covers the LSTM weights and biases
    decayed = [k for k in seg if k.startswith("LSTMLayer")] if weight_decay else []
    real = torch.zeros(flat.padded_numel, dtype=torch.bool, device=DEV)
    for o, shape in seg.values():
        real[o:o + shape.numel()] = True
    adam = optimizer == "adam"
    if rounding is None:
        rounding = _roundings(hs, T, B, D, bidirectional) if bf16 else N.Fp32()
    floor = N.FLOOR if bf16 else N.FLOOR_F32
    t0 = opt.step_count
    drop0 = int(eng.model.rnn.dropout_step)
    worst, worst_update = {}, 0.0
    for s in range(steps):
        x, y = xs[s * B:(s + 1) * B], ys[s * B:(s + 1) * B]
        lengths = None if lengths_seed is None else _lengths(T, B, lengths_seed + s)
        before = {"p": flat.data.clone(), "m": opt.m.clone() if adam else None, "v": opt.v.clone() if adam else None,
                  "shadow": None if flat.shadow is None else flat.shadow.clone(), "t": int(opt.step_dev),
                  "drop": int(eng.model.rnn.dropout_step)}
        if not stale_shadow and bf16:
            N.check_shadow(f"{case} before step {s}", flat.shadow, flat.data)
        assert before["drop"] == drop0 + (s if dropout > 0 or weight_drop > 0 else 0), (case, s, before["drop"])
        assert not adam or before["t"] == t0 + s, (case, s, before["t"])
        eng.model.eval()
        with torch.no_grad():
            h_T = eng.model.features(x, lengths)                        # the weights the step reads
        eng.model.train()
        n0 = _stats()
        if graph and s == 0:
            warmup = 3
            eng.capture(x, y, warmup=warmup, lengths=lengths)
            delta = {k: v - n0[k] for k, v in _stats().items()}
            assert delta == {**dict.fromkeys(KEYS, 0), **{k: v * (warmup + 1) for k, v in per_step.items()}}, (case, delta)
            # capture ran real steps: the training state it restored is the one before them
            for k, now in (("p", flat.data), ("m", opt.m), ("v", opt.v), ("shadow", flat.shadow)):
                assert now is None or torch.equal(now, before[k]), (case, "capture() did not restore", k)
            assert int(opt.step_dev) == before["t"] and int(eng.model.rnn.dropout_step) == before["drop"]
            n0 = _stats()
        loss = eng.step(x, y, lengths)
        torch.cuda.synchronize()
        cuda_lstm.check_kernel_errors(DEV)
        delta = {k: v - n0[k] for k, v in _stats().items()}
        assert delta == {**dict.fromkeys(KEYS, 0), **({} if graph else per_step)}, (case, s, delta)
        t = int(opt.step_dev)
        assert not adam or t == opt.step_count == t0 + s + 1, (case, s, t, opt.step_count)
        got = {"loss": loss.float(), "h_T": h_T.float()}
        for k, (o, shape) in seg.items():
            got[k] = flat.grad[o:o + shape.numel()].view(shape).clone()
        # the update, against the fp64 one of the state before the step and the step's own gradient
        if adam:
            upd = N.adam_update(before["p"], before["m"], before["v"], flat.grad, t, opt.lr, opt.beta1, opt.beta2, opt.eps,
                                weight_decay, 1.0, wd_numel)
        else:
            upd = N.sgd_update(before["p"], flat.grad, opt.lr, weight_decay, 1.0, wd_numel)
        for k, (o, shape) in seg.items():
            sl = slice(o, o + shape.numel())
            for what, now, ref, bound in (("p", flat.data, upd.p, upd.bound_p), ("m", opt.m, upd.m, upd.bound_m),
                                          ("v", opt.v, upd.v, upd.bound_v)):
                if ref is not None:
                    worst_update = max(worst_update, N.check_update(f"{case} step {s} {k} {what}", now[sl], ref[sl], bound[sl]))
        pad = ~real
        assert not bool(flat.grad[pad].any() or flat.data[pad].any()), (case, s, "padding of the flat buffer is not 0")
        del upd
        if stale_shadow and s == 0:
            flat.shadow.copy_(before["shadow"])                         # the refresh after step 1 "did not happen"
        if free_engine:                                          # room for the fp64 arm next to the engine
            del loss, h_T
            torch.cuda.empty_cache()
        drop = N.Dropout(dropout, eng.model.rnn.dropout_key, before["drop"]) if dropout > 0 else None
        wspecs = {}
        if weight_drop > 0:
            for l in range(len(hs)):
                for rev in ((False, True) if bidirectional else (False,)):
                    wspecs[f"LSTMLayer{l}" + ("_reverse" if rev else "")] = ops_ref.DropoutSpec(
                        weight_drop, eng.model.rnn.dropout_key, l, rev, before["drop"], weight=True)
        with torch.no_grad():
            arms = {}
            for arm, dt, r in (("fp64", torch.float64, None), ("emu", torch.float32, rounding)):
                layers, head = _reference_params(eng, seg, before["p"], dt, bf16_weights=bf16)
                raw = layers                                        # eval mode: no dropout, no weight drop
                if wspecs:                                          # W_h * M * s of the step, from the weights the kernels read
                    mask = lambda p, n: (*p[:3], ops_ref.weight_drop(p[3].to(dtype), wspecs[n]).to(dt), p[4])
                    layers = [(mask(p[0], f"LSTMLayer{l}"), mask(p[1], f"LSTMLayer{l}_reverse")) if bidirectional
                              else mask(p, f"LSTMLayer{l}") for l, p in enumerate(layers)]
                kw = dict(lengths=lengths, bidirectional=bidirectional, rounding=r)
                full = N.model(x.to(dt), layers, head, y, dropout=drop, **kw)
                h_eval = full.h_T if drop is None and not wspecs else N.model(x.to(dt), raw, head, y, backward=False, **kw).h_T
                arms[arm] = {"loss": full.loss, "h_T": h_eval, **full.grads}
                for n, sp in wspecs.items():
                    arms[arm][f"{n}/w_h"] = _masked_grad(arms[arm][f"{n}/w_h"], sp)
                for k in decayed:                                       # the L2 term of create_variable
                    o, shape = seg[k]
                    if k.split("/")[1] in ("h0", "c0"):                 # ... through autograd: in the gradient
                        arms[arm][k] = arms[arm][k] + N.f32(weight_decay) * before["p"][o:o + shape.numel()].view(shape).to(dt)
                del full
            l2 = sum(N.f32(weight_decay) * 0.5 * float((before["p"][o:o + sh.numel()].double() ** 2).sum())
                     for o, sh in (seg[k] for k in decayed))
            got["loss"] = got["loss"].double() - l2                     # the reported loss includes the L2 value
            ratios = {k: N.check_budget(f"{case} step {s} {k}", g, arms["fp64"][k], arms["emu"][k], per_step=k == "h_T",
                                        floor=floor) for k, g in got.items()}
            del arms
        for k, v in ratios.items():
            worst[k] = max(worst.get(k, 0.0), v)
    top = sorted(worst.items(), key=lambda kv: -kv[1])[:4]
    print(f"\n{case}: worst budget ratio {top[0][1]:.3f} over {steps} steps (" + ", ".join(f"{k} {v:.3f}" for k, v in top) +
          f"); alpha {N.ALPHA}, floor {floor:.2e}; worst update ratio {worst_update:.3f}")


def _sched(T, B, D, ha, hb):
    from lstm_tensorspark_b200.ops import cuda_lstm
    return cuda_lstm.pair_schedule(T, B, D, ha, hb, cuda_lstm._sms(DEV), cuda_lstm._coresident_ctas(DEV))


def _pair_step(schedule):
    return {"fast_fwd": 2, "fast_bwd": 2, f"{schedule}_fwd": 1, "folded_feed": 1}


def _is_h100():
    from lstm_tensorspark_b200.ops import cuda_lstm
    return cuda_lstm._sms(DEV) == 132


def test_headline():
    """2 x 1024: the pipelined pair with the folded batch-major feed; layer b's dW GEMMs and capped bias column sums beside
    layer a's recurrence, layer a's bias column sums in two halves under its own dW GEMMs."""
    if _is_h100():
        assert _sched(128, 256, 1024, 1024, 1024) == "pipelined"
    _model_case("headline", "1024,1024", 128, 256, 1024, _pair_step("pipelined"))


def test_wavefront():
    """2 x 512: both recurrences co-resident (the wavefront pair)."""
    if _is_h100():
        assert _sched(128, 256, 512, 512, 512) == "wavefront"
    _model_case("wavefront", "512,512", 128, 256, 512, _pair_step("wavefront"))


def test_three_layers_learned_initial_state():
    """3 x 256: a pair then a single layer; the learned h0 / c0 reach the flat buffer through autograd, not a direct sink."""
    if _is_h100():
        assert _sched(64, 256, 128, 256, 256) == "wavefront"
    _model_case("three layers", "256,256,256", 64, 256, 128, {**_pair_step("wavefront"), "fast_fwd": 3, "fast_bwd": 3, "folded_feed": 0},
                learn_initial_state=True)


def test_ragged():
    """The headline pair's masked kernels, lengths 1 and T included: h_T is each row's own last state."""
    _model_case("ragged", "1024,1024", 128, 256, 1024, _pair_step("pipelined"), lengths_seed=31)


def test_dropout():
    """The headline pair with its dropout masks fused into the recurrences; the step counter advances over the 3 steps."""
    _model_case("dropout", "1024,1024", 128, 256, 1024, _pair_step("pipelined"), dropout=0.2)


def test_bidirectional_ragged():
    """2 x 1024 bidirectional with lengths: 4 directions one after the other, [h_fwd | h_rev] into layer 1, the two upper
    directions' dx summed into layer 0, a [2H, C] head."""
    _model_case("bidirectional ragged", "1024,1024", 128, 256, 1024, {"fast_fwd": 4, "fast_bwd": 4}, lengths_seed=41,
                bidirectional=True)


def test_bidirectional_dropout():
    """2 x 256 bidirectional: a mask per direction of layer 0."""
    _model_case("bidirectional dropout", "256,256", 64, 256, 128, {"fast_fwd": 4, "fast_bwd": 4}, bidirectional=True,
                dropout=0.3)


def test_batch_chunks():
    """B = 400 at H = 1024: each layer runs as two persistent chunks (256 + 144 rows) whose weight and bias gradients land in
    the same sinks - the first chunk overwrites, the second accumulates."""
    _model_case("batch chunks", "1024,1024", 32, 400, 256, {"fast_fwd": 4, "fast_bwd": 4, "batch_chunks": 4})


def test_headline_adam():
    """The pipelined pair and the folded feed over 4 Adam steps at lr 1e-3: from step 2 on, every kernel reads weights the
    update kernel moved (master no longer bf16-representable, shadow refreshed by the update)."""
    _model_case("headline adam", "1024,1024", 128, 256, 1024, _pair_step("pipelined"), steps=4, learning_rate=1e-3)


def test_dropout_graph_replays():
    """The headline pair with dropout 0.2, captured once and replayed on 4 batches: Adam's step counter and the dropout
    counter advance inside the graph, and the first replay starts from the state capture() restored (t = 1)."""
    _model_case("dropout graph", "1024,1024", 128, 256, 1024, _pair_step("pipelined"), steps=4, dropout=0.2,
                learning_rate=1e-3, graph=True)


def test_resumed_three_layers_weight_decay():
    """3 x 256 with learned initial states, Adam with weight decay 0.1 from a state loaded at step 1000 (nonzero m and v): the
    decay in the update kernel over the LSTM weights and biases, through autograd for h0 / c0, and the bias correction of t > 1000."""
    _model_case("resumed three layers", "256,256,256", 64, 256, 128,
                {**_pair_step("wavefront"), "fast_fwd": 3, "fast_bwd": 3, "folded_feed": 0}, learn_initial_state=True,
                learning_rate=1e-3, weight_decay=0.1, resume_at=1000)


def test_bidirectional_ragged_sgd_weight_decay():
    """2 x 256 bidirectional with lengths, SGD at lr 0.05 with weight decay 0.1: the reverse directions' weights move too."""
    _model_case("bidirectional ragged sgd", "256,256", 64, 256, 128, {"fast_fwd": 4, "fast_bwd": 4}, lengths_seed=51,
                bidirectional=True, optimizer="sgd", learning_rate=0.05, weight_decay=0.1)


def test_batch_chunks_adam():
    """B = 400 at H = 1024 under Adam: the two batch chunks write the same sinks at moved weights."""
    _model_case("batch chunks adam", "1024,1024", 32, 400, 256, {"fast_fwd": 4, "fast_bwd": 4, "batch_chunks": 4},
                learning_rate=1e-3)


def test_a_stale_shadow_fails_the_next_step():
    """Negative control: with the shadow of the weights before step 1 put back after it (a missing refresh), step 2 computes
    with the old weights, and its check against the weights the update wrote must fail."""
    with pytest.raises(AssertionError, match=r"^stale shadow step 1 [^:]*: error vs fp64"):
        _model_case("stale shadow", "512,512", 128, 256, 512, _pair_step("wavefront"), steps=2, learning_rate=1e-3,
                    stale_shadow=True)


def test_config4():
    """BASELINE config 4 (4 x 2048, T = 512, B = 64), one step: streamed weights, backward in clusters of 2, the head at
    H = 2048."""
    _model_case("config 4", "2048,2048,2048,2048", 512, 64, 2048, {"fast_fwd": 4, "fast_bwd": 4}, steps=1, free_engine=True)
