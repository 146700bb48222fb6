"""Stateful language-model training on the GPU (``--stateful``): continuity of the carried state through the persistent kernels
(one layer, the layer pair in both schedules, streamed weights) bit for bit against one long pass, a stateful training step
against the fp64 model reference of tests/lstm_numerics.py started from the same carried state, CUDA-graph replay against eager
steps across a pass boundary, capture leaving the carry alone, resume, and stream evaluation against the CPU reference.

Continuity is bitwise with ``--deterministic``: a step of the recurrence reads only bf16 h_{t-1}, fp32 c_{t-1} and the bf16
gx_t = x_t W_x^T, whose K order does not depend on how many time steps the launch covers."""
import math

import pytest
import torch

import lstm_numerics as N
from test_gpu_model_numerics import _engine, _names, _reference_params, _roundings, _segments, DEV
from test_gpu_next_token import model_next_token

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _fp32_matmuls(monkeypatch):
    from lstm_tensorspark_b200.ops import cuda_lstm
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)
    monkeypatch.setattr(cuda_lstm, "SEQ_VARIANT", cuda_lstm.SEQ_VARIANT)     # (--deterministic sets a module-level knob)


def _stat(k):
    from lstm_tensorspark_b200.ops import cuda_lstm
    return cuda_lstm.STATS.get(k, 0)


def _segments_of(B, T, K, V, seed):
    from lstm_tensorspark_b200 import data as D
    s = D.synthetic_stream(B * K + 1, T, V, seed=seed)
    x, y, _ = D.stream_layout(s, B, T)
    return torch.as_tensor(x).to(DEV), torch.as_tensor(y).to(DEV)


@pytest.mark.parametrize("hidden,B,T,E,path", [
    ("256", 128, 32, 128, "fast_fwd"),                   # one layer
    ("256,256", 256, 32, 128, "wavefront_fwd"),          # the layer pair, both recurrences co-resident
    ("1024,1024", 256, 32, 1024, "pipelined_fwd"),       # the pair's pipelined schedule (the headline model)
    ("2048", 64, 16, 256, "fast_fwd"),                   # H = 2048: the weight slice streamed through the ring
])
def test_segments_equal_one_long_pass_bitwise(hidden, B, T, E, path):
    K, V = 4, 1024
    eng = _engine(hidden_units=hidden, in_features=E, seq_len=T, batch_size=B, vocab_size=V, next_token=True, stateful=True,
                  deterministic=True)
    m = eng.model.eval()
    x, y = _segments_of(B, T, K, V, seed=1)
    with torch.no_grad():
        before = _stat(path)
        h_long = m.sequence_features(torch.cat([x[k * B:(k + 1) * B] for k in range(K)], 1)).clone()
        final_long = [(h.clone(), c.clone()) for h, c in m.rnn.final_state()]
        assert _stat(path) > before
        state = m.rnn.zero_state(B, torch.bfloat16, DEV)
        hs = []
        before = _stat(path)
        for k in range(K):
            hs.append(m.sequence_features(x[k * B:(k + 1) * B], state=state).clone())
            state = [(h.clone(), c.clone()) for h, c in m.rnn.final_state()]
        assert _stat(path) >= before + K
    torch.cuda.synchronize()
    assert hs[0].dtype == torch.bfloat16 and state[0][1].dtype == torch.float32
    assert torch.equal(torch.cat(hs), h_long), hidden
    for (h, c), (h1, c1) in zip(state, final_long):
        assert torch.equal(h, h1) and torch.equal(c, c1)


def test_a_stateful_step_against_fp64_from_the_carried_state():
    """The second step of a pass: loss and every gradient against the fp64 model started from the state the first step ended in
    (the layer pair), within the bf16 budget."""
    hidden, T, B, E, V = "512,512", 32, 128, 256, 2048
    eng = _engine(hidden_units=hidden, in_features=E, seq_len=T, batch_size=B, vocab_size=V, next_token=True, stateful=True)
    names = _names(eng)
    names[id(eng.model.embedding.weights)] = "Embedding/weights"
    seg = _segments(eng, names)
    rounding = _roundings([int(h) for h in hidden.split(",")], T, B, E, False)
    x, y = _segments_of(B, T, 2, V, seed=3)
    eng.step(x[:B], y[:B], reset=True)
    data = eng.flat.data.clone()
    loss = eng.step(x[B:], y[B:])
    torch.cuda.synchronize()
    carried = [(h.clone(), c.clone()) for h, c in eng.state_prev]
    assert all(float(h.float().abs().max()) > 0 for h, _ in carried)
    got = {"loss": loss.float()}
    for k, (o, shape) in seg.items():
        got[k] = eng.flat.grad[o:o + shape.numel()].view(shape).clone()
    with torch.no_grad():
        arms = {}
        for arm, dt, r in (("fp64", torch.float64, None), ("emu", torch.float32, rounding)):
            layers, head = _reference_params(eng, seg, data, dt)
            layers = [(h.to(dt), c.to(dt)) + tuple(p[2:]) for p, (h, c) in zip(layers, carried)]
            o, shape = seg["Embedding/weights"]
            table = data[o:o + shape.numel()].view(shape).bfloat16().to(dt)
            l_, g_ = model_next_token(x[B:], table, layers, head, y[B:], None, None, r)
            arms[arm] = {"loss": l_, **g_}
        for k, g in got.items():
            N.check_budget(f"stateful step {k}", g, arms["fp64"][k], arms["emu"][k])


def test_graph_replays_equal_eager_steps_across_a_pass_boundary():
    """Two engines from the same seed, ``--deterministic``, Adam: one eager, one captured after its first step and replayed.
    Every step's loss, weights and carried state agree bit for bit over 5 steps of 2-segment passes (resets at steps 0, 2, 4);
    capturing leaves the carried state as it was."""
    kw = dict(hidden_units="256,256", in_features=128, seq_len=32, batch_size=128, vocab_size=1024, next_token=True,
              stateful=True, deterministic=True, learning_rate=1e-3, dropout=0.1)
    eager, graphed = _engine(**kw), _engine(**kw)
    B, K = 128, 2
    x, y = _segments_of(B, 32, K, 1024, seed=5)
    for step in range(5):
        k = step % K
        bx, by = x[k * B:(k + 1) * B], y[k * B:(k + 1) * B]
        if step == 1:
            before = [t.clone() for pair in graphed.state + graphed.state_prev for t in pair]
            graphed.capture(bx, by)
            after = [t for pair in graphed.state + graphed.state_prev for t in pair]
            assert all(torch.equal(u, v) for u, v in zip(before, after))
        le = eager.step(bx, by, reset=k == 0)
        lg = graphed.step(bx, by, reset=k == 0)
        torch.cuda.synchronize()
        assert torch.equal(le, lg), step
        assert torch.equal(eager.flat.data, graphed.flat.data), step
        for (h, c), (h1, c1) in zip(eager.carried_state(), graphed.carried_state()):
            assert torch.equal(h, h1) and torch.equal(c, c1), step
    assert graphed._graph is not None


def _run_cfg(tmp_path, name, **kw):
    from lstm_tensorspark_b200.config import Config
    base = dict(next_token=True, stateful=True, vocab_size=512, seq_len=16, batch_size=64, hidden_units="128,128",
                in_features=64, synthetic=300, device="cuda", quiet=True, init="scaled", learning_rate=1e-3, dropout=0.1,
                deterministic=True, checkpoint_path=str(tmp_path / name), output_path=str(tmp_path / (name + "_out")))
    base.update(kw)
    return Config(**base).validate()


def _latest(path):
    from lstm_tensorspark_b200.utils import checkpoint as ckpt
    return ckpt.load(ckpt.latest_checkpoint(ckpt.find_latest_run(str(path), None)))


def test_resume_continues_bit_for_bit(tmp_path):
    """5 steps, a checkpoint, 5 more after resuming = 10 uninterrupted steps, with a CUDA graph: weights, Adam's state and the
    carried state.  A pass is 4 segments (300 * 16 + 1 ids in 64 streams), so the resumed run starts in the middle of a pass,
    from the saved state."""
    from lstm_tensorspark_b200.trainer import run_job
    k = 5
    run_job(_run_cfg(tmp_path, "a", epochs=1, max_steps=k, evaluate_every=k, cuda_graph=True), standalone=True)
    run_job(_run_cfg(tmp_path, "a", epochs=1, max_steps=2 * k, evaluate_every=k, cuda_graph=True, use_pretrained_model=True),
            standalone=True)
    run_job(_run_cfg(tmp_path, "b", epochs=1, max_steps=2 * k, evaluate_every=k, cuda_graph=True), standalone=True)
    va, ma, oa = _latest(tmp_path / "a")
    vb, mb, ob = _latest(tmp_path / "b")
    assert ma["global_step"] == mb["global_step"] == 2 * k - 1
    assert all(torch.equal(va[n], vb[n]) for n in va)
    assert all(torch.equal(u, v) for p, q in zip(oa["state"], ob["state"]) for u, v in zip(p, q))
    assert oa["state"][0][0].dtype == torch.bfloat16 and oa["state"][0][1].dtype == torch.float32
    for key, v in oa["optimizer"].items():
        assert (torch.equal(v, ob["optimizer"][key]) if isinstance(v, torch.Tensor) else v == ob["optimizer"][key]), key


def test_stream_eval_on_the_gpu_against_the_cpu_reference(tmp_path):
    """``--mode eval --stateful`` of one trained model on the GPU (bf16 kernels) and on the CPU (fp32 reference): the same
    positions, and losses within 1 % (bf16 storage of h and of the recurrent operands over 300 steps of carried state)."""
    from lstm_tensorspark_b200.trainer import run_job
    run_job(_run_cfg(tmp_path, "e", epochs=1, max_steps=6, dropout=0.0), standalone=True)
    gpu = run_job(_run_cfg(tmp_path, "e", mode="eval", synthetic=301), standalone=True)
    cpu = run_job(_run_cfg(tmp_path, "e", mode="eval", synthetic=301, device="cpu", deterministic=False), standalone=True)
    L = (301 * 16) // 64
    assert gpu["positions"] == cpu["positions"] == 64 * L and L % 16 != 0
    assert gpu["loss"] == pytest.approx(cpu["loss"], rel=1e-2)
    assert math.isfinite(gpu["perplexity"]) and gpu["perplexity"] < 512
