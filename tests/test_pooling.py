"""Pooling over time (``--pooling mean | max | attention``) on the CPU: the reference semantics against a hand-written fp64
nn.LSTM + masked pool + nn.Linear (loss and every gradient; fixed, ragged, bidirectional ragged and dropout), gradcheck of the
pool op, padded positions that never reach a result, max ties, the flags' errors and warning, unchanged initial weights under
``--pooling last``, checkpoints written under another pooling, the standalone CLI (train, resume, eval) and 2-rank gloo runs."""
import os
import subprocess
import sys
import warnings

import pytest
import torch
import torch.nn.functional as Fn

from lstm_tensorspark_b200 import data as D
from lstm_tensorspark_b200.config import Config
from lstm_tensorspark_b200.ops import reference as ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MODES = ("mean", "max", "attention")


def _blocks(w):
    """Gate-interleaved rows (n = 4 j + g) -> torch's [i; f; g; o] blocks."""
    H = w.shape[0] // 4
    return w.view(H, 4, *w.shape[1:]).transpose(0, 1).reshape(w.shape)


def _model(mode, bidirectional, dropout, ragged, T=6, B=5, D_=3, H=4, C=3, A=5, seed=0):
    """A 2-layer SequenceClassifier with ``--pooling mode`` (fp64, CPU reference path) and the same weights in nn.LSTM."""
    from lstm_tensorspark_b200.models.classifier import SequenceClassifier
    from lstm_tensorspark_b200.ops import functional as F
    F.set_backend("torch")
    cfg = Config(hidden_units=f"{H},{H}", in_features=D_, seq_len=T, batch_size=B, num_classes=C, bidirectional=bidirectional,
                 dropout=dropout, pooling=mode, attention_units=A, learn_initial_state=False, init="scaled", device="cpu",
                 variable_length=ragged)
    g = torch.Generator().manual_seed(seed)
    m = SequenceClassifier(cfg, batch_size=B, device="cpu", generator=g).double()
    m.compute_dtype = torch.float64
    lstm = torch.nn.LSTM(D_, H, num_layers=2, bidirectional=bidirectional, dropout=0.0).double()
    dirs = m.rnn.directions()
    with torch.no_grad():
        for k, lay in enumerate(dirs):
            l, suf = (k // 2, "_reverse" if k % 2 else "") if bidirectional else (k, "")
            getattr(lstm, f"weight_ih_l{l}{suf}").copy_(_blocks(lay.w_x))
            getattr(lstm, f"weight_hh_l{l}{suf}").copy_(_blocks(lay.w_h))
            getattr(lstm, f"bias_ih_l{l}{suf}").copy_(_blocks(lay.bias))
            getattr(lstm, f"bias_hh_l{l}{suf}").zero_()
    return m, lstm, dirs


def _hand_pool(out, lengths, mode, att):
    """The pool written out over nn.LSTM's padded output ``out [T,B,H]``: one sample at a time over its own steps."""
    rows = []
    for b in range(out.shape[1]):
        hb = out[:int(lengths[b]), b]                                      # [len_b, H]
        if mode == "mean":
            rows.append(hb.mean(0))
        elif mode == "max":
            rows.append(hb.max(0).values)
        else:
            W, bias, v = att
            alpha = torch.softmax(torch.tanh(hb @ W + bias) @ v, 0)
            rows.append((alpha.unsqueeze(1) * hb).sum(0))
    return torch.stack(rows)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("bidirectional,ragged", [(False, False), (False, True), (True, True)])
def test_reference_matches_nn_lstm_pool_linear_fp64(mode, bidirectional, ragged):
    """The pooled features and every gradient through them in fp64 (the last-state head computes its loss in fp32, so the whole
    model's loss and head gradients are compared at fp32 precision)."""
    from torch.nn.utils.rnn import pack_padded_sequence, pad_packed_sequence
    T, B, C = 6, 5, 3
    lengths = torch.tensor([6, 1, 3, 6, 2], dtype=torch.int32) if ragged else None
    m, lstm, dirs = _model(mode, bidirectional, 0.0, ragged)
    g = torch.Generator().manual_seed(1)
    x = torch.randn(B, T, 3, generator=g, dtype=torch.float64)
    y = torch.randint(0, C, (B,), generator=g)
    lt = lengths.long() if ragged else torch.full((B,), T)
    out, _ = lstm(pack_padded_sequence(x.transpose(0, 1), lt, enforce_sorted=False))
    out, _ = pad_packed_sequence(out, total_length=T)
    att = None if mode != "attention" else [p.detach().clone().requires_grad_(True) for p in m.attention.params()]
    want_s = _hand_pool(out, lt, mode, att)
    R = torch.randn(want_s.shape, generator=g, dtype=torch.float64)
    s = m.features(x, lengths)
    assert s.dtype == torch.float64 and torch.allclose(s, want_s, atol=1e-12)
    (s * R).sum().backward()
    (want_s * R).sum().backward()
    if att is not None:
        for p, q in zip(m.attention.params(), att):
            assert torch.allclose(p.grad, q.grad, atol=1e-12)
    for k, lay in enumerate(dirs):
        l, suf = (k // 2, "_reverse" if k % 2 else "") if bidirectional else (k, "")
        assert torch.allclose(_blocks(lay.w_x.grad), getattr(lstm, f"weight_ih_l{l}{suf}").grad, atol=1e-12), lay.node_name
        assert torch.allclose(_blocks(lay.w_h.grad), getattr(lstm, f"weight_hh_l{l}{suf}").grad, atol=1e-12), lay.node_name
        assert torch.allclose(_blocks(lay.bias.grad), getattr(lstm, f"bias_hh_l{l}{suf}").grad, atol=1e-12), lay.node_name
    W = m.head.weights.detach().clone().requires_grad_(True)
    bias = m.head.bias.detach().clone().requires_grad_(True)
    want_logits = want_s.detach() @ W + bias
    want = Fn.cross_entropy(want_logits, y)
    want.backward()
    loss, logits, correct = m(x, y, lengths)
    loss.backward()
    assert abs(float(loss) - float(want)) < 1e-6
    assert torch.allclose(logits.double(), want_logits, atol=1e-6) and int(correct) == int((want_logits.argmax(1) == y).sum())
    assert torch.allclose(m.head.weights.grad, W.grad, atol=1e-6) and torch.allclose(m.head.bias.grad, bias.grad, atol=1e-6)


@pytest.mark.parametrize("mode", MODES)
def test_reference_with_dropout_matches_hand_composed_masks_fp64(mode):
    """Dropout 0.4 between the layers: the first layer's output times reference.dropout_mask x scale feeds layer 2; the pooled
    top layer's output is not dropped."""
    T, B, C, H = 6, 5, 3, 4
    lengths = torch.tensor([6, 1, 3, 6, 2], dtype=torch.int32)
    m, _lstm, dirs = _model(mode, False, 0.4, True)
    m.rnn.dropout_key, m.rnn.dropout_step = (7, 1), 3
    g = torch.Generator().manual_seed(2)
    x = torch.randn(B, T, 3, generator=g, dtype=torch.float64)
    R = torch.randn(B, H, generator=g, dtype=torch.float64)
    (m.features(x, lengths) * R).sum().backward()                               # fp64 throughout (the head's loss is fp32)
    own = [dirs[0].w_x, dirs[0].w_h, dirs[0].bias, dirs[1].w_x, dirs[1].w_h, dirs[1].bias]
    own += list(m.attention.params()) if m.attention is not None else []
    ps = [p.detach().clone().requires_grad_(True) for p in own]
    z = torch.zeros(B, H, dtype=torch.float64)
    h1, _, _ = ref.lstm_layer_sequence(x.transpose(0, 1), z, z, *ps[:3], lengths=lengths)
    spec = ref.DropoutSpec(0.4, (7, 1), 0, False, 3)
    h1 = h1 * ref.dropout_mask(spec, T, B, H).double() * ref.dropout_scale(0.4).double()
    h2, _, _ = ref.lstm_layer_sequence(h1, z, z, *ps[3:6], lengths=lengths)
    (_hand_pool(h2, lengths, mode, ps[6:] or None) * R).sum().backward()
    for p, q in zip(own, ps):
        assert torch.allclose(p.grad, q.grad, atol=1e-12)


def _op_inputs(T=5, B=4, H=3, A=4, seed=0):
    g = torch.Generator().manual_seed(seed)
    h = torch.randn(T, B, H, generator=g, dtype=torch.float64)
    att = tuple(torch.randn(*s, generator=g, dtype=torch.float64) for s in ((H, A), (A,), (A,)))
    return h, att, torch.tensor([5, 1, 3, 2], dtype=torch.int32)


@pytest.mark.parametrize("mode", MODES)
def test_gradcheck(mode):
    h, att, lengths = _op_inputs()
    if mode == "attention":
        args = (h.requires_grad_(True),) + tuple(a.requires_grad_(True) for a in att)
        fn = lambda hh, w, b, v: ref.pool_sequence(hh, lengths, mode, (w, b, v))
    else:
        args = (h.requires_grad_(True),)
        fn = lambda hh: ref.pool_sequence(hh, lengths, mode)
    assert torch.autograd.gradcheck(fn, args)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("poison", [1e30, float("inf"), float("nan")])
def test_poisoned_padding_changes_nothing(mode, poison):
    h, att, lengths = _op_inputs(seed=3)
    keep = ref.step_mask(lengths, 4, 5).t().unsqueeze(2)                       # [T,B,1]
    dirty = torch.where(keep, h, torch.full_like(h, poison))
    out = []
    for hh in (h, dirty):
        hp = hh.clone().requires_grad_(True)
        ap = tuple(a.clone().requires_grad_(True) for a in att)
        s = ref.pool_sequence(hp, lengths, mode, ap if mode == "attention" else None)
        s.backward(torch.linspace(-1, 1, s.numel(), dtype=s.dtype).view(s.shape))
        out.append([s.detach(), hp.grad] + ([a.grad for a in ap] if mode == "attention" else []))
    for a, b in zip(*out):
        assert torch.equal(a, b)
    assert float(out[1][1][~keep.expand_as(h)].abs().max()) == 0.0


def test_max_ties_send_the_gradient_to_the_smallest_t():
    h = torch.tensor([[[1.0, 2.0]], [[3.0, 2.0]], [[3.0, 0.5]], [[3.0, 2.0]]], dtype=torch.float64, requires_grad=True)  # [4,1,2]
    s = ref.pool_sequence(h, torch.tensor([4], dtype=torch.int32), "max")
    s.backward(torch.tensor([[10.0, 20.0]], dtype=torch.float64))
    assert s.tolist() == [[3.0, 2.0]]
    assert h.grad[:, 0, 0].tolist() == [0, 10, 0, 0] and h.grad[:, 0, 1].tolist() == [20, 0, 0, 0]
    assert torch.max(h.detach(), 0).indices.tolist() == [[1, 0]]                  # what torch.max(dim).indices picks
    h2 = h.detach().clone().requires_grad_(True)                                  # the tie beyond len_b = 3 does not count
    ref.pool_sequence(h2, torch.tensor([1], dtype=torch.int32), "max").sum().backward()
    assert h2.grad[:, 0, :].tolist() == [[1, 1], [0, 0], [0, 0], [0, 0]]


# ---- flags ---------------------------------------------------------------------------------------------------------------------
def test_flag_errors_and_warning():
    from lstm_tensorspark_b200.config import parse_args
    assert parse_args(["--seq_len", "4"]).pooling == "last" and parse_args(["--seq_len", "4"]).attention_units == 128
    cfg = parse_args(["--seq_len", "4", "--pooling", "attention", "--attention_units", "7"])
    assert (cfg.pooling, cfg.attention_units) == ("attention", 7)
    with pytest.raises(ValueError, match="--pooling"):
        Config(pooling="sum", seq_len=4).validate()
    with pytest.raises(ValueError, match="--attention_units"):
        Config(pooling="attention", seq_len=4, attention_units=0).validate()
    for mode in MODES:
        with pytest.raises(ValueError, match="--seq_len"):
            Config(pooling=mode, seq_len=1).validate()
        with pytest.raises(ValueError, match="--pooling.*--per_step_labels"):
            Config(pooling=mode, seq_len=4, per_step_labels=True).validate()
    with warnings.catch_warnings():
        warnings.simplefilter("error")
        Config(pooling="attention", seq_len=4, attention_units=7).validate()
        Config(pooling="mean", seq_len=4).validate()
    with pytest.warns(UserWarning, match="--attention_units"):
        cfg = Config(pooling="mean", seq_len=4, attention_units=7).validate()
    from lstm_tensorspark_b200.models.classifier import SequenceClassifier
    assert SequenceClassifier(cfg, device="cpu").attention is None                # the warning changes nothing


# ---- initial weights ---------------------------------------------------------------------------------------------------------
# sum_i (i + 1) x_i over every reference variable of a fresh SequenceClassifier (hidden 6,5, in_features 3, C 3, init_std 0.5,
# generator seed 11), as the model without --pooling drew them
PARENT_INIT = {(False, "truncated_normal"): -119.97647917456925, (False, "scaled"): -50.35229337849887,
               (True, "truncated_normal"): -207.6873937957571, (True, "scaled"): -69.92901020066347}


def _fresh(bidirectional, init, pooling, A=4):
    from lstm_tensorspark_b200.models.classifier import SequenceClassifier
    cfg = Config(hidden_units="6,5", in_features=3, seq_len=4, batch_size=2, num_classes=3, bidirectional=bidirectional,
                 init=init, device="cpu", init_std=0.5, pooling=pooling, attention_units=A)
    return SequenceClassifier(cfg, batch_size=2, device="cpu", generator=torch.Generator().manual_seed(11))


def _checksum(sd):
    return sum(float((v.double() * (1 + torch.arange(v.numel(), dtype=torch.float64).view(v.shape))).sum()) for v in sd.values())


@pytest.mark.parametrize("bidirectional", [False, True])
@pytest.mark.parametrize("init", ["truncated_normal", "scaled"])
def test_initial_weights_unchanged(bidirectional, init):
    """``--pooling last`` draws the weights the model drew before pooling existed; every other mode draws the same ones and then
    the attention weights."""
    last = _fresh(bidirectional, init, "last").reference_state_dict()
    assert _checksum(last) == PARENT_INIT[(bidirectional, init)]
    for mode in MODES:
        sd = _fresh(bidirectional, init, mode).reference_state_dict()
        assert {k: v for k, v in sd.items() if not k.startswith("Attention/")}.keys() == last.keys()
        assert all(torch.equal(sd[k], last[k]) for k in last)
        assert any(k.startswith("Attention/") for k in sd) == (mode == "attention")
    att = _fresh(bidirectional, init, "attention", A=64).attention
    H_in = 10 if bidirectional else 5
    assert att.weights.shape == (H_in, 64) and att.bias.shape == (64,) and att.context.shape == (64,)
    if init == "scaled":
        assert float(att.bias.abs().max()) == 0.0
        assert 0.5 * 0.5 / H_in ** 0.5 < float(att.weights.std()) < 1.5 * 0.5 / H_in ** 0.5
        assert 0.5 * 0.5 / 8 < float(att.context.std()) < 1.5 * 0.5 / 8


# ---- checkpoints and the CLI ---------------------------------------------------------------------------------------------------
def _base(tmp_path, **kw):
    kw.setdefault("attention_units", 8 if kw.get("pooling", "attention") == "attention" else 128)
    return dict(dict(synthetic=120, hidden_units="12", in_features=3, seq_len=6, num_classes=3, variable_length=True,
                     batch_size=20, checkpoint_path=str(tmp_path / "ck"), output_path=str(tmp_path / "out"), device="cpu",
                     quiet=True, learning_rate=2e-2, init="scaled", steps_mode="epochs", evaluate_every=5, pooling="attention"),
                **kw)


def test_cli_trains_resumes_and_evaluates_with_attention(tmp_path):
    import json
    from lstm_tensorspark_b200.trainer import run_job
    base = _base(tmp_path)
    flags = [f"--{k}={v}" for k, v in dict(base, epochs=8).items()]
    r = subprocess.run([sys.executable, os.path.join(ROOT, "lstm-no-spark.py")] + flags, capture_output=True, text=True,
                       timeout=600, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-3000:]
    runs = os.listdir(base["checkpoint_path"])
    scal = [json.loads(s) for s in open(os.path.join(base["checkpoint_path"], runs[0], "train", "scalars.jsonl"))]
    assert scal[-1]["cross_entropy"] < scal[0]["cross_entropy"]                     # it learns
    out2 = run_job(Config(epochs=10, use_pretrained_model=True, **base).validate(), standalone=True)
    assert out2["results"][0]["steps"] == 12                                       # 60 total - 48 already done
    assert any(k.startswith("Attention/") for k in out2["results"][0]["variables"])
    ev = run_job(Config(mode="eval", **dict(base, batch_size=50)).validate(), standalone=True)    # 2 full batches + a tail
    assert ev["samples"] == 120 and ev["accuracy"] > 1 / 3


@pytest.mark.parametrize("written,loaded", [("attention", "last"), ("last", "attention"), ("mean", "max"), ("max", "last"),
                                            ("last", "mean")])
def test_checkpoint_under_another_pooling_is_refused(tmp_path, written, loaded):
    from lstm_tensorspark_b200.trainer import run_job
    run_job(Config(epochs=1, max_steps=2, **_base(tmp_path, pooling=written)).validate(), standalone=True)
    with pytest.raises(ValueError, match=f"--pooling {written}.*--pooling {loaded}"):
        run_job(Config(epochs=1, max_steps=3, use_pretrained_model=True, **_base(tmp_path, pooling=loaded)).validate(),
                standalone=True)
    with pytest.raises(ValueError, match="--pooling"):
        run_job(Config(mode="eval", **_base(tmp_path, pooling=loaded)).validate(), standalone=True)


def test_averaged_model_records_pooling_and_is_checked(tmp_path):
    from lstm_tensorspark_b200.trainer import run_job
    base = _base(tmp_path, partitions=2, max_workers=1, epochs=1, max_steps=2)
    run_job(Config(**base).validate(), standalone=False)
    blob = torch.load(os.path.join(base["output_path"], "averaged_model.pt"), weights_only=False)
    assert blob["meta"]["pooling"] == "attention" and blob["meta"]["attention_units"] == 8
    assert "Attention/context" in blob["variables"]
    ev = run_job(Config(mode="eval", **dict(base, partitions=1)).validate(), standalone=False)
    assert ev["samples"] == 120
    with pytest.raises(ValueError, match="--pooling attention.*--pooling mean"):
        run_job(Config(mode="eval", **dict(base, partitions=1, pooling="mean", attention_units=128)).validate(), standalone=False)
    # a file that records no pooling counts as last
    from lstm_tensorspark_b200.models.classifier import SequenceClassifier
    m = SequenceClassifier(Config(**dict(base, pooling="last")), device="cpu")
    m.check_pooling(m.reference_state_dict(), None)
    with pytest.raises(ValueError, match="--pooling last.*--pooling attention"):
        SequenceClassifier(Config(**base), device="cpu").check_pooling(m.reference_state_dict(), None)


# ---- two ranks -----------------------------------------------------------------------------------------------------------------
def _sync_check(rank, world, sync_mode):
    """4 steps on rank-specific batches -> (the attention weights moved, the flat buffers of both ranks are identical)."""
    import torch.distributed as dist
    from lstm_tensorspark_b200.engine import TrainEngine
    from lstm_tensorspark_b200.parallel.comm import make_communicator
    dev = torch.device("cpu")
    comm = make_communicator("gloo", rank, world, dev, 60)
    cfg = Config(hidden_units="8,8", in_features=4, batch_size=6, seq_len=5, sync_mode=sync_mode, average_scope="all",
                 device="cpu", learn_initial_state=False, init="scaled", partitions=world, variable_length=True,
                 pooling="attention", attention_units=6, independent_init=sync_mode == "param_avg")
    eng = TrainEngine(cfg, rank, world, comm, batch_size=6, device=dev, dtype=torch.float32)
    x, y, l = D.synthetic_sequences(6, 5, 4, 3, seed=rank, variable_length=True)
    start = [p.detach().clone() for p in eng.model.attention.params()]
    for _ in range(4):
        eng.step(torch.as_tensor(x), torch.as_tensor(y), torch.as_tensor(l))
    eng.maybe_average(force=True)
    moved = all(not torch.equal(a, p) for a, p in zip(start, eng.model.attention.params()))
    all_w = [torch.zeros_like(eng.flat.data) for _ in range(world)]
    dist.all_gather(all_w, eng.flat.data)
    comm.close()
    return moved and all(torch.equal(all_w[0], w) for w in all_w)


@pytest.mark.parametrize("sync_mode", ["grad_allreduce", "param_avg"])
def test_two_ranks_end_with_identical_attention_weights(sync_mode):
    """grad_allreduce: the replicas start equal and average every gradient, the attention weights' included.  param_avg with
    ``--average_scope all``: each replica draws its own initial weights (``--independent_init``) and the final average covers
    the attention weights too."""
    from functools import partial
    from lstm_tensorspark_b200.parallel.launch import launch
    assert launch(partial(_sync_check, sync_mode=sync_mode), 2) == [True, True]
