"""Dropout between stacked layers (CPU): the Philox4x32-10 mask shared with the kernels, the reference op, the stack on the torch
backend against a hand-composed reference, and the engine / trainer semantics (training mode only, a step counter that makes a
resumed run draw the masks of an uninterrupted one, replicas that stay equal under a gradient allreduce)."""
import math
import os
import runpy
import sys

import pytest
import torch

from lstm_tensorspark_b200.config import Config, parse_args
from lstm_tensorspark_b200.ops import reference as ref
from lstm_tensorspark_b200.ops.reference import DropoutSpec
from lstm_tensorspark_b200.utils import checkpoint as ckpt

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("ctr,key,want", [
    ((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
    ((0xffffffff,) * 4, (0xffffffff, 0xffffffff), (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
    ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0), (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1)),
])
def test_philox_known_answers(ctr, key, want):
    got = ref.philox4x32_10(torch.tensor(ctr, dtype=torch.int64), *key)
    assert [int(v) for v in got] == list(want)


def test_mask_layout_follows_the_counter_definition():
    """Unit 8g + i of row b at time t: word i/2 (low half for even i) of Philox((b ceil(H/8) + g, t, 2 layer + reverse, step))."""
    spec = DropoutSpec(0.3, (7, 3), layer=2, reverse=True, step=11, row0=5)
    H = 20                                                       # 3 groups, the last one partial
    keep = ref.dropout_mask(spec, 2, 3, H, t0=4)
    for t, b, j in [(0, 0, 0), (1, 2, 19), (0, 1, 9), (1, 0, 14)]:
        w = ref.philox4x32_10(torch.tensor([(b + 5) * 3 + j // 8, 4 + t, 5, 11]), 7, 3)
        v = (int(w[(j % 8) // 2]) >> (16 * (j % 2))) & 0xFFFF
        assert bool(keep[t, b, j]) == (v >= spec.thr), (t, b, j)


@pytest.mark.parametrize("p", [0.1, 0.2, 0.5, 0.9])
def test_kept_fraction_and_exact_scale(p):
    spec = DropoutSpec(p, (1, 0), 0, False, 3)
    keep = ref.dropout_mask(spec, 16, 256, 256)                  # ~1M units
    n = keep.numel()
    q = 1 - spec.thr / 65536
    assert abs(float(keep.float().mean()) - q) <= 5 * math.sqrt(q * (1 - q) / n)
    scale = ref.dropout_scale(p)
    assert scale.dtype == torch.float32 and float(scale) == float(torch.tensor(65536.0) / (65536 - spec.thr))
    assert float(scale.double() * (65536 - spec.thr) / 65536) == pytest.approx(1.0, abs=1e-7)    # exact expectation
    assert float(ref.dropout_scale(0.25)) == float(torch.tensor(4.0 / 3.0, dtype=torch.float32))
    x = torch.randn(16, 256, 256)
    y = ref.dropout(x, spec)
    assert torch.equal(y, torch.where(keep, x * scale, torch.zeros(())))


def test_zero_p_is_the_identity_and_masks_differ_by_every_counter_word():
    x = torch.randn(3, 4, 8)
    assert ref.dropout(x, DropoutSpec(0.0, (0, 0), 0, False, 0)) is x
    assert ref.dropout(x, None) is x
    base = DropoutSpec(0.5, (0, 0), 0, False, 0)
    m = ref.dropout_mask(base, 4, 8, 64)
    import dataclasses
    for kw in [dict(key=(1, 0)), dict(key=(0, 1)), dict(layer=1), dict(reverse=True), dict(step=1), dict(row0=8)]:
        assert not torch.equal(m, ref.dropout_mask(dataclasses.replace(base, **kw), 4, 8, 64)), kw


def test_gradient_is_mask_times_scale():
    spec = DropoutSpec(0.4, (5, 2), 1, False, 9)
    x = torch.randn(3, 4, 24, dtype=torch.float64, requires_grad=True)
    assert torch.autograd.gradcheck(lambda v: ref.dropout(v, spec), (x,))
    g = torch.randn(3, 4, 24, dtype=torch.float64)
    ref.dropout(x, spec).backward(g)
    keep = ref.dropout_mask(spec, 3, 4, 24)
    assert torch.equal(x.grad, torch.where(keep, g * ref.dropout_scale(0.4).double(), torch.zeros((), dtype=torch.float64)))


def test_bf16_rounds_once_from_the_stored_value():
    spec = DropoutSpec(0.2, (0, 0), 0, False, 0)
    h = torch.randn(2, 8, 64).bfloat16()
    keep = ref.dropout_mask(spec, 2, 8, 64)
    want = torch.where(keep, (h.float() * ref.dropout_scale(0.2)).bfloat16(), torch.zeros((), dtype=torch.bfloat16))
    assert torch.equal(ref.dropout(h, spec).view(torch.int16), want.view(torch.int16))


# ---- the stack on the torch backend --------------------------------------------------------------------------------------
def _rnn(hidden, D, B, p, bidirectional=False, seed=0):
    from lstm_tensorspark_b200.models.recurrent.rnn import RNN
    settings = [{"layer_name": f"LSTMLayer{i}", "num_hidden": h, "batch_size": B,
                 "dim_size": D if i == 0 else (2 if bidirectional else 1) * hidden[i - 1]} for i, h in enumerate(hidden)]
    g = torch.Generator().manual_seed(seed)
    rnn = RNN(settings, dropout=p, learn_initial_state=False, init="scaled", generator=g)
    if bidirectional:
        rnn.add_reverse_layers()
    rnn.dropout_key, rnn.dropout_step = (42, 1), 6
    return rnn


def _by_hand(rnn, x, lengths, p):
    """layer, mask, layer, ...: the reference layers composed with reference.dropout; the top layer's output is not dropped."""
    seq = x.transpose(0, 1)
    n = len(rnn.layers)
    for i in range(n):
        dirs = [rnn.layers[i]] + ([rnn.reverse_layers[i]] if rnn.bidirectional else [])
        outs, finals = [], []
        for l in dirs:
            B, H = seq.shape[1], l.num_hidden
            h, hT, _ = ref.lstm_layer_sequence(seq, torch.zeros(B, H), torch.zeros(B, H), l.w_x, l.w_h, l.bias, lengths=lengths,
                                               reverse=l.reverse)
            if i < n - 1:
                h = ref.dropout(h, DropoutSpec(p, (42, 1), i, l.reverse, 6))
            outs.append(h)
            finals.append(hT)
        seq = torch.cat(outs, 2)
    return torch.cat(finals, 1), seq


@pytest.mark.parametrize("hidden,lengths,bidirectional", [
    ((12, 8), False, False), ((12, 8, 8), False, False), ((12, 8, 8), True, False), ((8, 8), True, True), ((8, 6, 8), False, True)])
def test_stack_equals_layers_composed_with_masks(hidden, lengths, bidirectional):
    from lstm_tensorspark_b200.ops import functional as F
    F.set_backend("torch")
    try:
        B, T, D, p = 5, 7, 6, 0.5
        x = torch.randn(B, T, D)
        ln = torch.tensor([7, 3, 1, 5, 7], dtype=torch.int32) if lengths else None
        rnn = _rnn(list(hidden), D, B, p, bidirectional)
        got = rnn.fit_layers(x, lengths=ln)
        want, want_seq = _by_hand(rnn, x, ln, p)
        assert torch.equal(got, want)
        rnn.reset_state(B)
        assert torch.equal(rnn.fit_sequence_all(x, ln), want_seq)      # the top layer's sequence is not dropped either
        rnn.eval()
        rnn.reset_state(B)
        off = rnn.fit_layers(x, lengths=ln)
        assert not torch.equal(off, got)
        assert torch.equal(off, _by_hand(rnn, x, ln, 0.0)[0])
        if bidirectional:
            a, b = (ref.dropout_mask(DropoutSpec(p, (42, 1), 0, r, 6), T, B, hidden[0]) for r in (False, True))
            assert not torch.equal(a, b)                               # each direction has its own mask
    finally:
        F.set_backend("auto")


def test_one_step_path_drops_the_output_at_time_zero_but_not_the_state():
    rnn = _rnn([10, 10, 6], 4, 3, 0.5)
    rnn.reset_state(3)
    x = torch.randn(3, 4)
    out = rnn.fit_layers(x)
    state = x
    for i, l in enumerate(rnn.layers):
        h, _c = ref.lstm_cell_step(state, torch.zeros(3, l.num_hidden), torch.zeros(3, l.num_hidden), l.w_x, l.w_h, l.bias)
        assert torch.equal(l.ht, h)                                    # the carried state is the undropped one
        state = ref.dropout(h, DropoutSpec(0.5, (42, 1), i, False, 6)) if i < 2 else h
    assert torch.equal(out, state)


# ---- engine / trainer ------------------------------------------------------------------------------------------------------
def _engine(p, hidden="8,8", seed=0, **kw):
    from lstm_tensorspark_b200.engine import TrainEngine
    cfg = Config(hidden_units=hidden, in_features=4, batch_size=6, seq_len=5, device="cpu", learn_initial_state=False, init="scaled",
                 dropout=p, seed=seed, partitions=1, sync_mode="none", quiet=True, **kw)
    return TrainEngine(cfg, 0, 1, None, batch_size=6, device=torch.device("cpu"), dtype=torch.float32)


def _batch(seed=0):
    from lstm_tensorspark_b200 import data as D
    x, y = D.synthetic_sequences(6, 5, 4, 3, seed=seed)
    return torch.as_tensor(x), torch.as_tensor(y)


def _train(eng, n):
    x, y = _batch()
    losses = [float(eng.step(x, y)) for _ in range(n)]
    return losses, eng.flat.data.clone()


def test_zero_p_trains_bit_identically_and_positive_p_differs():
    l0, w0 = _train(_engine(0.0), 4)
    lc, wc = _train(_engine(Config().dropout), 4)
    assert l0 == lc and torch.equal(w0, wc)
    e = _engine(0.3)
    l1, w1 = _train(e, 4)
    assert l1 != l0 and not torch.equal(w1, w0)
    assert e.model.rnn.dropout_step == 4
    single = _engine(0.3, hidden="8")                                  # one layer: nothing to drop, no counter either
    assert _train(single, 2)[0] == _train(_engine(0.0, hidden="8"), 2)[0] and single.model.rnn.dropout_step == 0


def test_evaluate_ignores_dropout():
    x, y = _batch(1)
    a, b = _engine(0.6), _engine(0.0)
    assert torch.equal(a.flat.data, b.flat.data)
    la, aa = a.evaluate(x, y)
    lb, ab = b.evaluate(x, y)
    assert float(la) == float(lb) and float(aa) == float(ab)
    assert a.model.training
    with torch.no_grad():
        assert float(a.model(x, y)[0]) != float(la)                   # training mode does drop


def test_in_loop_and_mode_eval_score_without_dropout(tmp_path, iris_path, monkeypatch):
    from lstm_tensorspark_b200.models.classifier import SequenceClassifier
    from lstm_tensorspark_b200.trainer import run_job
    seen = []
    orig = SequenceClassifier.features

    def spy(self, x, lengths=None):
        seen.append((torch.is_grad_enabled(), self.training))
        return orig(self, x, lengths)

    monkeypatch.setattr(SequenceClassifier, "features", spy)
    cfg = Config(training_path=iris_path, hidden_units="16,16", dropout=0.5, checkpoint_path=str(tmp_path / "ck"),
                 output_path=str(tmp_path / "o"), device="cpu", quiet=True, max_steps=6, evaluate_every=2).validate()
    run_job(cfg, standalone=True)
    assert (True, True) in seen and (False, False) in seen and (False, True) not in seen and (True, False) not in seen
    seen.clear()
    run_job(Config(**dict(cfg.__dict__, mode="eval", batch_size=40)).validate(), standalone=True)
    assert seen and all(not tr for _g, tr in seen)


def _final(cfg):
    d = ckpt.find_latest_run(cfg.checkpoint_path, None)
    return ckpt.load(ckpt.latest_checkpoint(d))


def test_resume_draws_the_masks_of_an_uninterrupted_run(tmp_path, iris_path):
    from lstm_tensorspark_b200.trainer import run_job
    common = dict(training_path=iris_path, hidden_units="16,16", dropout=0.5, device="cpu", quiet=True, evaluate_every=1,
                  learning_rate=1e-2, batch_size=10)
    mk = lambda d, **kw: Config(checkpoint_path=str(tmp_path / d), output_path=str(tmp_path / (d + "o")), **common, **kw).validate()
    run_job(mk("a", max_steps=8), standalone=True)
    run_job(mk("b", max_steps=4), standalone=True)
    out = run_job(mk("b", max_steps=8, use_pretrained_model=True), standalone=True)
    assert out["results"][0]["steps"] == 4
    va, _, oa = _final(mk("a"))
    vb, _, ob = _final(mk("b"))
    for k in va:
        assert torch.equal(va[k], vb[k]), k
    # and a resumed run with another P is allowed (a hyperparameter, not a weight)
    run_job(Config(**dict(mk("b", max_steps=10, use_pretrained_model=True).__dict__, dropout=0.1)).validate(), standalone=True)


def _grad_sync_dropout(rank, world):
    import torch
    import torch.distributed as dist
    from lstm_tensorspark_b200 import data as D
    from lstm_tensorspark_b200.config import Config
    from lstm_tensorspark_b200.engine import TrainEngine
    from lstm_tensorspark_b200.parallel.comm import make_communicator
    dev = torch.device("cpu")
    comm = make_communicator("gloo", rank, world, dev, 60)
    cfg = Config(hidden_units="8,8,8", in_features=4, batch_size=6, seq_len=3, sync_mode="grad_allreduce", device="cpu",
                 learn_initial_state=False, init="scaled", partitions=world, dropout=0.5)
    eng = TrainEngine(cfg, rank, world, comm, batch_size=6, device=dev, dtype=torch.float32, partition_key=rank)
    x, y = D.synthetic_sequences(6, 3, 4, 3, seed=0)                   # the same batch: only the masks tell the replicas apart
    g = []
    for _ in range(3):
        eng.step(torch.as_tensor(x), torch.as_tensor(y))
        g.append(eng.flat.grad.clone())
    all_w = [torch.zeros_like(eng.flat.data) for _ in range(world)]
    dist.all_gather(all_w, eng.flat.data)
    comm.close()
    return bool(all(torch.equal(all_w[0], w) for w in all_w)), eng.model.rnn.dropout_key


def test_grad_allreduce_with_dropout_keeps_replicas_equal():
    from lstm_tensorspark_b200.parallel.launch import launch
    res = launch(_grad_sync_dropout, 2)
    assert [r[0] for r in res] == [True, True]
    assert res[0][1] != res[1][1]                                      # each replica draws its own masks


def test_standalone_cli_trains_and_scores(tmp_path, iris_path, monkeypatch, capsys):
    args = ["--training_path", iris_path, "--hidden_units", "16,16", "--dropout", "0.5", "--device", "cpu", "--quiet",
            "--checkpoint_path", str(tmp_path / "ck"), "--output_path", str(tmp_path / "o"), "--epochs", "2",
            "--learning_rate", "0.01"]
    monkeypatch.setattr(sys, "argv", ["lstm-no-spark.py"] + args)
    runpy.run_path(os.path.join(ROOT, "lstm-no-spark.py"), run_name="__main__")
    assert "DROPOUT = 0.5" in capsys.readouterr().out
    monkeypatch.setattr(sys, "argv", ["lstm-no-spark.py"] + args + ["--mode", "eval", "--batch_size", "50"])
    runpy.run_path(os.path.join(ROOT, "lstm-no-spark.py"), run_name="__main__")
    from lstm_tensorspark_b200.trainer import run_job
    ev = run_job(parse_args(args + ["--mode", "eval", "--batch_size", "50"], standalone=True), standalone=True)
    assert ev["samples"] == 150 and 0 <= ev["accuracy"] <= 1 and ev["loss"] == ev["loss"]


@pytest.mark.parametrize("bad", ["1.0", "-0.1", "1.5", "nan"])
def test_flag_validation(bad):
    with pytest.raises(ValueError, match="--dropout"):
        parse_args(["--hidden_units", "8,8", "--dropout", bad])


def test_one_layer_warns_and_zero_or_stack_does_not(recwarn):
    with pytest.warns(UserWarning, match="--dropout"):
        parse_args(["--hidden_units", "8", "--dropout", "0.3"])
    parse_args(["--hidden_units", "8", "--dropout", "0"])
    parse_args(["--hidden_units", "8,8", "--dropout", "0.3"])
    assert not [w for w in recwarn.list if "--dropout" in str(w.message)]
