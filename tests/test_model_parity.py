"""Numerical parity (CPU): LSTM cell / stack vs a NumPy transcription of the reference equations
(original src/models/recurrent/lstm.py:88-109), loss/accuracy closed forms, TF-Adam values, gradcheck."""
import numpy as np
import pytest
import torch

from lstm_tensorspark_b200.config import Config
from lstm_tensorspark_b200.models import RNN, LSTMLayer, SequenceClassifier
from lstm_tensorspark_b200.models.flat import FlatParams
from lstm_tensorspark_b200.ops import reference as ref
from lstm_tensorspark_b200.ops.loss import compute_accuracy, compute_loss
from lstm_tensorspark_b200.ops.optim import FlatOptimizer


def sig(v):
    return 1.0 / (1.0 + np.exp(-v))


def numpy_reference_step(layer: LSTMLayer, x, ht, Ct):
    """Per-gate math exactly as written in the reference (12 separate matrices)."""
    g = lambda t: t.detach().double().numpy()
    Wf, Wi, Wc, Wo = layer.weight_forget, layer.weight_input, layer.weight_C, layer.weight_output
    bf, bi, bc, bo = layer.biases_forget, layer.biases_input, layer.biases_C, layer.biases_output
    step = lambda W, b: ht @ g(W[0]) + x @ g(W[1]) + g(b)
    ft = sig(step(Wf, bf))
    it = sig(step(Wi, bi))
    c_ta = np.tanh(step(Wc, bc))
    Ct = ft * Ct + it * c_ta
    ot = sig(step(Wo, bo))
    return ot * np.tanh(Ct), Ct


def test_cell_matches_reference_equations():
    torch.manual_seed(0)
    layer = LSTMLayer("LSTMLayer0", num_hidden=6, dim_size=4, batch_size=5).double()
    x = torch.randn(5, 4, dtype=torch.float64)
    h_np, c_np = numpy_reference_step(layer, x.numpy(), layer.h0.detach().numpy(), layer.c0.detach().numpy())
    h = layer.fit_next(x)
    assert np.allclose(h.detach().numpy(), h_np, atol=1e-10)
    assert np.allclose(layer.Ct.detach().numpy(), c_np, atol=1e-10)
    assert len(layer.state) == 1


def test_per_gate_views_have_reference_shapes():
    layer = LSTMLayer("L", num_hidden=6, dim_size=4, batch_size=5)
    w_h, w_x = layer.weight_forget
    assert tuple(w_h.shape) == (6, 6) and tuple(w_x.shape) == (4, 6) and tuple(layer.biases_C.shape) == (6,)
    names = [n for n, _ in layer.named_reference_variables()]
    assert names[:3] == ["L/weights_forget_h", "L/weights_forget_x", "L/bias_forget"]
    assert "L/state" in names and "L/context_state" in names


def test_fit_next_eval_does_not_advance_state():
    torch.manual_seed(0)
    layer = LSTMLayer("L", 6, 4, 5)
    x = torch.randn(5, 4)
    layer.fit_next(x)
    h1 = layer.ht.clone()
    layer.fit_next(x, train=False)
    assert torch.equal(layer.ht, h1) and len(layer.state) == 1


def test_stack_sequence_equals_stepwise():
    torch.manual_seed(1)
    cfg = Config(hidden_units="8,5", in_features=3, batch_size=4, seq_len=6, learn_initial_state=True)
    net = RNN(cfg.net_settings(), learn_initial_state=True)
    x = torch.randn(4, 6, 3)
    net.reset_state(4)
    out_seq = net.fit_layers(x)
    net.reset_state(4)
    for t in range(6):
        out_step = net.fit_layers(x[:, t])
    assert torch.allclose(out_seq, out_step, atol=1e-5)


def test_map_data_by_key_layout():
    net = RNN(Config(hidden_units="8,5", in_features=3).net_settings())
    rec = net.map_data_by_key()
    assert [k for k, _ in rec] == ["wf", "wi", "wo", "wc", "bf", "bi", "bc", "bo"]
    wf = dict(rec)["wf"]
    assert len(wf) == 2 and tuple(wf[0][0].shape) == (8, 8) and tuple(wf[0][1].shape) == (3, 8)
    assert tuple(wf[1][0].shape) == (5, 5) and tuple(wf[1][1].shape) == (8, 5)
    assert tuple(dict(rec)["bo"][1].shape) == (5,)


def test_add_layer():
    net = RNN([])
    net.add_layer({"layer_name": "LSTMLayer0", "dim_size": 3, "num_hidden": 4, "batch_size": 2})
    net.add_layers([{"layer_name": "LSTMLayer1", "dim_size": 4, "num_hidden": 5, "batch_size": 2}])
    assert len(net.layers) == 2 and net.fit_layers(torch.randn(2, 3)).shape == (2, 5)


def test_loss_and_accuracy_closed_form():
    logits = torch.tensor([[2.0, 0.0, 0.0], [0.0, 0.0, 3.0]])
    labels = torch.tensor([0, 1])
    l = compute_loss(labels=labels, logits=logits)
    e = np.array([[np.e ** 2, 1, 1], [1, 1, np.e ** 3]])
    p = e / e.sum(1, keepdims=True)
    assert float(l) == pytest.approx(-(np.log(p[0, 0]) + np.log(p[1, 1])) / 2, rel=1e-6)
    assert float(compute_accuracy(labels=labels, logits=logits)) == pytest.approx(0.5)
    onehot = torch.tensor([[1.0, 0, 0], [0, 1.0, 0]])
    assert float(compute_loss(labels=onehot, logits=logits, sparse=False)) == pytest.approx(float(l), rel=1e-6)


def test_tf_adam_formulation():
    p = torch.tensor([1.0, -2.0]); g = torch.tensor([0.5, 0.25]); m = torch.zeros(2); v = torch.zeros(2)
    ref.adam_step_(p, g, m, v, step=1, lr=1e-3)
    lr_t = 1e-3 * np.sqrt(1 - 0.999) / (1 - 0.9)
    exp = np.array([1.0, -2.0]) - lr_t * (0.1 * np.array([0.5, 0.25])) / (np.sqrt(0.001 * np.array([0.25, 0.0625])) + 1e-8)
    assert np.allclose(p.numpy(), exp, rtol=1e-6)


def test_sequence_gradcheck_fp64():
    torch.manual_seed(0)
    T, B, D, H = 3, 2, 3, 4
    mk = lambda *s: torch.randn(*s, dtype=torch.float64, requires_grad=True)
    args = (mk(T, B, D), mk(B, H), mk(B, H), mk(4 * H, D), mk(4 * H, H), mk(4 * H))
    assert torch.autograd.gradcheck(lambda *a: ref.lstm_layer_sequence(*a)[0], args, atol=1e-6)


def test_flat_params_views_and_optimizer():
    torch.manual_seed(0)
    cfg = Config(hidden_units="8", in_features=4, batch_size=5)
    model = SequenceClassifier(cfg, batch_size=5)
    flat = model.build_flat()
    assert flat.lstm_numel >= 4 * (8 * 8 + 4 * 8 + 8)
    w = model.rnn.layers[0].w_x
    assert w.data_ptr() == flat.data[flat.offsets[0]:].data_ptr()
    x = torch.randn(5, 4); y = torch.randint(0, 3, (5,))
    opt = FlatOptimizer(flat, 1e-2, "adam")
    l0 = None
    for _ in range(30):
        flat.zero_grad()
        loss, _, _ = model(x, y)
        loss.backward()
        assert w.grad.data_ptr() == flat.grad[flat.offsets[0]:].data_ptr()
        opt.step()
        l0 = l0 if l0 is not None else float(loss)
    assert float(loss) < l0


def test_reference_state_dict_roundtrip():
    cfg = Config(hidden_units="8,6", in_features=4, batch_size=5)
    m1 = SequenceClassifier(cfg, batch_size=5); m1.build_flat()
    m2 = SequenceClassifier(cfg, batch_size=5); m2.build_flat()
    sd = m1.reference_state_dict()
    assert "LSTMLayer1/weights_C_x" in sd and tuple(sd["LSTMLayer1/weights_C_x"].shape) == (8, 6)
    assert "Dense1/weights" in sd and tuple(sd["Dense1/weights"].shape) == (6, 3)
    m2.load_reference_state_dict(sd)
    x = torch.randn(5, 4)
    assert torch.allclose(m1.features(x), m2.features(x))


def test_fit_layers_returns_final_state_edge():
    """fit_layers([B,T,D]) hands back the top layer's final state (a separate autograd edge, so the top layer never sees a
    dense [T,B,H] gradient on the GPU path); value and gradients must equal the explicit seq[-1] route."""
    import torch
    from lstm_tensorspark_b200.models.recurrent.rnn import RNN
    torch.manual_seed(0)
    from lstm_tensorspark_b200.config import Config
    rnn = RNN(Config(hidden_units="6,4", in_features=5, batch_size=3).net_settings(), init="scaled", learn_initial_state=False)
    x = torch.randn(3, 7, 5)
    out = rnn.fit_layers(x)
    assert out.shape == (3, 4)
    w = torch.randn_like(out)
    (out * w).sum().backward()
    g1 = [p.grad.clone() for p in rnn.parameters() if p.grad is not None]
    for p in rnn.parameters():
        p.grad = None
    rnn.reset_state(3)
    seq = x.transpose(0, 1)
    for layer in rnn.layers:
        seq = layer.fit_sequence(seq)
    assert torch.allclose(seq[-1], out, atol=1e-6)
    (seq[-1] * w).sum().backward()
    g2 = [p.grad.clone() for p in rnn.parameters() if p.grad is not None]
    assert len(g1) == len(g2) and all(torch.allclose(a, b, atol=1e-6) for a, b in zip(g1, g2))
