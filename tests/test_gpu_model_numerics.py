"""Whole training steps of the public TrainEngine (bf16, CUDA kernels) against the fp64 model reference of
tests/lstm_numerics.py, within the error budget of its bf16 emulation: the loss, h_T per batch row and every gradient segment
of the flat buffer, per tensor, by parameter name - over 3 steps on different batches (dropout: a new mask each step).
This reaches what the layer-level tests do not: the direct gradient sinks (first write of a step overwrites, later ones
accumulate; split bias column sums; dW GEMMs launched beside the recurrence), batch chunks sharing those sinks, stacked /
bidirectional / dropout compositions, learned initial states, per-row lengths through the classifier and the head inside the
step.  Every case names the path it targets and asserts it through cuda_lstm.STATS (`pytest -m gpu`; `-s` prints each case's
worst budget ratios).  The file runs in about 37 s on an H100 80GB HBM3 at a 700 W power limit, fp64 arms included; the worst
ratio of any case was 0.52 there."""
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


def _engine(**kw):
    from lstm_tensorspark_b200.config import Config
    from lstm_tensorspark_b200.engine import TrainEngine
    cfg = Config(partitions=1, sync_mode="none", init="scaled", device="cuda", quiet=True, learning_rate=0.0, backend="auto",
                 **kw)                                                 # lr = 0: the weights stay put across the 3 steps
    eng = TrainEngine(cfg, 0, 1, None, batch_size=cfg.batch_size, device=DEV, dtype=torch.bfloat16)
    with torch.no_grad():
        eng.flat.data.copy_(eng.flat.data.bfloat16().float())         # bf16-representable: both arms read the same weights
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


def _reference_params(eng, dt):
    rnn = eng.model.rnn
    cast = lambda t: t.detach().to(dt)

    def one(lay):
        return tuple(cast(t) for t in (lay.h0, lay.c0, lay.w_x, lay.w_h, lay.bias))
    if rnn.bidirectional:
        layers = [(one(a), one(b)) for a, b in zip(rnn.layers, rnn.reverse_layers)]
    else:
        layers = [one(a) for a in rnn.layers]
    return layers, (cast(eng.model.head.weights), cast(eng.model.head.bias))


def _model_case(case, hidden, T, B, D, per_step, steps=STEPS, lengths_seed=None, bidirectional=False, dropout=0.0,
                learn_initial_state=False, free_engine=False):
    """``per_step``: the STATS deltas one training step must show (the path the case targets)."""
    from lstm_tensorspark_b200 import data as Dm
    from lstm_tensorspark_b200.ops import cuda_lstm
    hs = [int(h) for h in hidden.split(",")]
    eng = _engine(hidden_units=hidden, in_features=D, seq_len=T, batch_size=B, num_classes=C, bidirectional=bidirectional,
                  dropout=dropout, learn_initial_state=learn_initial_state, variable_length=lengths_seed is not None)
    xs, ys = Dm.synthetic_sequences(steps * B, T, D, C, seed=5)
    xs, ys = torch.as_tensor(xs).to(DEV).bfloat16(), torch.as_tensor(ys).to(DEV)
    names = _names(eng)
    assert len(names) == len(eng.flat.params)
    rounding = _roundings(hs, T, B, D, bidirectional)
    worst = {}
    for s in range(steps):
        x, y = xs[s * B:(s + 1) * B], ys[s * B:(s + 1) * B]
        lengths = None if lengths_seed is None else _lengths(T, B, lengths_seed + s)
        n0 = _stats()
        loss = eng.step(x, y, lengths)
        torch.cuda.synchronize()
        cuda_lstm.check_kernel_errors(DEV)
        delta = {k: v - n0[k] for k, v in _stats().items()}
        assert delta == {**dict.fromkeys(KEYS, 0), **per_step}, (case, s, delta)
        eng.model.eval()
        with torch.no_grad():
            h_T = eng.model.features(x, lengths)
        eng.model.train()
        got = {"loss": loss.float(), "h_T": h_T.float()}
        for p, o in zip(eng.flat.params, eng.flat.offsets):
            got[names[id(p)]] = eng.flat.grad[o:o + p.numel()].view(p.shape).clone()
        if free_engine:                                          # room for the fp64 arm next to the engine
            del loss, h_T
            torch.cuda.empty_cache()
        drop = N.Dropout(dropout, eng.model.rnn.dropout_key, s) if dropout > 0 else None
        with torch.no_grad():
            arms = {}
            for arm, dt, r in (("fp64", torch.float64, None), ("emu", torch.float32, rounding)):
                layers, head = _reference_params(eng, dt)
                kw = dict(lengths=lengths, bidirectional=bidirectional, rounding=r)
                full = N.model(x.to(dt), layers, head, y, dropout=drop, **kw)
                h_eval = full.h_T if drop is None else N.model(x.to(dt), layers, head, y, backward=False, **kw).h_T
                arms[arm] = {"loss": full.loss, "h_T": h_eval, **full.grads}
                del full
            ratios = {k: N.check_budget(f"{case} step {s} {k}", g, arms["fp64"][k], arms["emu"][k], per_step=k == "h_T")
                      for k, g in got.items()}
            del arms
        for k, v in ratios.items():
            worst[k] = max(worst.get(k, 0.0), v)
    top = sorted(worst.items(), key=lambda kv: -kv[1])[:4]
    print(f"\n{case}: worst budget ratio {top[0][1]:.3f} over {steps} steps (" + ", ".join(f"{k} {v:.3f}" for k, v in top) +
          f"); alpha {N.ALPHA}, floor {N.FLOOR:.2e}")


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


def test_config4():
    """BASELINE config 4 (4 x 2048, T = 512, B = 64), one step: streamed weights, backward in clusters of 2, the head at
    H = 2048."""
    _model_case("config 4", "2048,2048,2048,2048", 512, 64, 2048, {"fast_fwd": 4, "fast_bwd": 4}, steps=1, free_engine=True)
