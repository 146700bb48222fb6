"""AWD-LSTM's activation regularisation without a GPU (``--activation_reg`` AR, ``--temporal_activation_reg`` TAR): flags and the
head rule, the reference sums against AWD's expressions and the packed definition, a training step in fp64 against AWD-LSTM built
from torch modules, zero coefficients as the run without the flags, evaluation, the ``--stateful`` segment boundary, logging,
resume and two gloo ranks."""
import json
import math

import pytest
import torch

from lstm_tensorspark_b200 import data as D
from lstm_tensorspark_b200.config import Config, parse_args
from lstm_tensorspark_b200.models.classifier import SequenceClassifier
from lstm_tensorspark_b200.ops import reference as ref
from lstm_tensorspark_b200.ops.reference import DropoutSpec
from lstm_tensorspark_b200.utils import checkpoint as ckpt

FLAGS = ("activation_reg", "temporal_activation_reg")
RECIPE = dict(locked_dropout=True, input_dropout=0.65, dropout=0.3, output_dropout=0.4, embedding_dropout=0.1)
AWD = dict(activation_reg=2.0, temporal_activation_reg=1.0)


def _lm(**kw):
    base = dict(hidden_units="16,16", in_features=16, seq_len=6, batch_size=5, vocab_size=64, next_token=True, init="scaled",
                learn_initial_state=False, device="cpu")
    base.update(kw)
    return Config(**base).validate()


# ---- flags --------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("flag", FLAGS)
@pytest.mark.parametrize("bad", [-0.5, float("nan"), float("inf")])
def test_bad_coefficient_names_the_flag(flag, bad):
    with pytest.raises(ValueError, match=f"--{flag}"):
        _lm(**{flag: bad})


@pytest.mark.parametrize("flag", FLAGS)
def test_coefficients_need_a_sequence_head(flag):
    with pytest.raises(ValueError) as ei:
        Config(hidden_units="8", in_features=4, seq_len=4, **{flag: 1.0}).validate()
    assert f"--{flag}" in str(ei.value) and "--pooling" in str(ei.value) and "--per_step_labels" in str(ei.value)
    for ok in (dict(per_step_labels=True), dict(pooling="mean"), dict(pooling="max"), dict(pooling="attention")):
        Config(hidden_units="8", in_features=4, seq_len=4, **{flag: 1.0}, **ok).validate()
    Config(hidden_units="8", in_features=4, seq_len=4, **{flag: 0.0}).validate()


def test_flags_parse_on_both_entry_points_and_default_off():
    argv = ["--next_token", "--vocab_size", "64", "--in_features", "16", "--hidden_units", "16,16", "--seq_len", "4",
            "--activation_reg", "2", "--temporal_activation_reg", "1"]
    for standalone in (False, True):
        cfg = parse_args(argv, standalone=standalone)
        assert (cfg.activation_reg, cfg.temporal_activation_reg) == (2.0, 1.0)
    d = Config()
    assert d.activation_reg == d.temporal_activation_reg == 0.0


# ---- the reference sums -------------------------------------------------------------------------------------------------------
def test_fixed_length_sums_are_awds_means():
    g = torch.Generator().manual_seed(0)
    T, B, W = 7, 4, 12
    out, h = torch.randn(T, B, W, generator=g, dtype=torch.float64), torch.randn(T, B, W, generator=g, dtype=torch.float64)
    pen = ref.activation_penalties(ref.activation_sums(out, h), W, T, B)
    assert torch.allclose(pen[0], out.pow(2).mean(), rtol=1e-14)
    assert torch.allclose(pen[1], (h[1:] - h[:-1]).pow(2).mean(), rtol=1e-14)


def test_ragged_sums_are_the_packed_definition():
    g = torch.Generator().manual_seed(1)
    T, B, W = 6, 5, 3
    out, h = torch.randn(T, B, W, generator=g, dtype=torch.float64), torch.randn(T, B, W, generator=g, dtype=torch.float64)
    lengths = torch.tensor([1, 6, 3, 1, 4], dtype=torch.int32)
    sums = ref.activation_sums(out, h, lengths)
    ar = sum(float(out[t, b].pow(2).sum()) for b in range(B) for t in range(int(lengths[b])))
    tar = sum(float((h[t, b] - h[t - 1, b]).pow(2).sum()) for b in range(B) for t in range(1, int(lengths[b])))
    assert math.isclose(float(sums[0]), ar, rel_tol=1e-13) and math.isclose(float(sums[1]), tar, rel_tol=1e-13)
    pen = ref.activation_penalties(sums, W, T, B, lengths)
    assert math.isclose(float(pen[0]), ar / (W * 15), rel_tol=1e-13)
    assert math.isclose(float(pen[1]), tar / (W * 10), rel_tol=1e-13)
    # every row of length 1: no TAR term, and a penalty whose count is 0 is 0
    ones = torch.ones(B, dtype=torch.int32)
    pen1 = ref.activation_penalties(ref.activation_sums(out, h, ones), W, T, B, ones)
    assert float(pen1[1]) == 0.0 and float(pen1[0]) > 0
    assert float(ref.activation_penalties(ref.activation_sums(out[:1], h[:1]), W, 1, B)[1]) == 0.0


def test_layer_op_returns_the_sums_of_its_outputs():
    g = torch.Generator().manual_seed(2)
    T, B, D, H = 5, 3, 4, 6
    x = torch.randn(T, B, D, generator=g, dtype=torch.float64)
    p = [torch.zeros(B, H, dtype=torch.float64), torch.zeros(B, H, dtype=torch.float64),
         torch.randn(4 * H, D, generator=g, dtype=torch.float64), torch.randn(4 * H, H, generator=g, dtype=torch.float64),
         torch.randn(4 * H, generator=g, dtype=torch.float64)]
    lengths = torch.tensor([5, 1, 3], dtype=torch.int32)
    spec = DropoutSpec(0.4, (3, 1), 0, False, 2, locked=True)
    for reverse in (False, True):
        raw, _, _ = ref.lstm_layer_sequence(x, *p, lengths=lengths, reverse=reverse)
        drop, _, _, sums = ref.lstm_layer_sequence(x, *p, lengths=lengths, reverse=reverse, dropout=spec, activation_sums=True)
        assert torch.equal(sums, ref.activation_sums(ref.dropout(raw, spec), raw, lengths))


# ---- fp64 against AWD-LSTM built from torch modules ----------------------------------------------------------------------------
def _torch_awd(m, x, y, key, step, cfg):
    """AWD-LSTM's loss around nn.Embedding / nn.LSTM / F.linear in fp64: the regularisers as in AWD's code (a masked copy of the
    table, LockedDropout masks ``[1, B, H]`` from ``reference.dropout_mask`` with T = 1) and its training loss
    ``xent + alpha * dropped_h.pow(2).mean() + beta * (raw_h[1:] - raw_h[:-1]).pow(2).mean()`` on the last layer's output."""
    B, T = x.shape
    V, E = m.embedding.weights.shape
    order = [ref.GATE_I, ref.GATE_F, ref.GATE_G, ref.GATE_O]
    perm = lambda w: torch.cat([w[g::4] for g in order])
    table = m.embedding.weights.detach().clone().requires_grad_(True)
    lstms = []
    for layer in m.rnn.layers:
        l = torch.nn.LSTM(layer.w_x.shape[1], layer.w_h.shape[1], dtype=torch.float64)
        with torch.no_grad():
            l.weight_ih_l0.copy_(perm(layer.w_x.detach()))
            l.weight_hh_l0.copy_(perm(layer.w_h.detach()))
            l.bias_ih_l0.copy_(perm(layer.bias.detach()))
            l.bias_hh_l0.zero_()
        lstms.append(l)
    head_w = None if m.tied else m.head.weights.detach().clone().requires_grad_(True)
    bias = m.head.bias.detach().clone().requires_grad_(True)

    def locked(p, H, **kw):
        spec = DropoutSpec(p, key, step=step, locked=True, **kw)
        return ref.dropout_mask(spec, 1, B, H).double() * float(ref.dropout_scale(p))

    rows = ref.embedding_row_mask(DropoutSpec(cfg.embedding_dropout, key, 0, False, step, site="rows"), V)
    masked = table * rows.double().unsqueeze(1) * float(ref.dropout_scale(cfg.embedding_dropout))
    h = torch.nn.functional.embedding(x.long(), masked).transpose(0, 1)
    h = h * locked(cfg.input_dropout, E, layer=0, reverse=False, site="input")
    n = len(lstms)
    for l, lstm in enumerate(lstms):
        raw, _ = lstm(h)
        h = raw * locked(cfg.dropout if l < n - 1 else cfg.output_dropout, raw.shape[2], layer=l, reverse=False)
    w = table if m.tied else head_w.t()
    logits = torch.nn.functional.linear(h.transpose(0, 1), w, bias)
    xent = torch.nn.functional.cross_entropy(logits.reshape(-1, V), y.reshape(-1).long())
    ar = h.pow(2).mean()
    tar = (raw[1:] - raw[:-1]).pow(2).mean()
    (xent + cfg.activation_reg * ar + cfg.temporal_activation_reg * tar).backward()
    grads = {"table": table.grad, "bias": bias.grad, "head": None if m.tied else head_w.grad}
    for l, lstm in enumerate(lstms):
        grads[l] = (lstm.weight_ih_l0.grad, lstm.weight_hh_l0.grad, lstm.bias_ih_l0.grad)
    return xent, torch.stack([ar, tar]).detach(), grads, perm


@pytest.mark.parametrize("tied", [False, True])
def test_training_step_equals_awd_lstm_from_torch_modules_in_fp64(tied):
    cfg = _lm(tie_embeddings=tied, **RECIPE, **AWD)
    m = SequenceClassifier(cfg, batch_size=5, device="cpu", generator=torch.Generator().manual_seed(7)).to(torch.float64)
    m.set_compute_dtype(torch.float64)
    key, step = (12, 1), 4
    m.rnn.dropout_key, m.rnn.dropout_step = key, step
    x, y = (torch.as_tensor(a) for a in D.synthetic_next_token(5, 6, 64, seed=3)[:2])
    loss, _logits, _ = m(x, y)
    pen = m.rnn.activation_penalties
    (loss + cfg.activation_reg * pen[0] + cfg.temporal_activation_reg * pen[1]).backward()     # TrainEngine._step_eager's loss
    want_loss, want_pen, g, perm = _torch_awd(m, x, y, key, step, cfg)
    close = lambda a, b: torch.allclose(a, b, rtol=1e-10, atol=1e-12)
    assert close(loss, want_loss) and close(pen.detach(), want_pen)
    assert float(want_pen[0]) > 0 and float(want_pen[1]) > 0
    assert close(m.embedding.weights.grad, g["table"]) and close(m.head.bias.grad, g["bias"])
    if not tied:
        assert close(m.head.weights.grad, g["head"])
    for l, layer in enumerate(m.rnn.layers):
        for got, w in zip((layer.w_x.grad, layer.w_h.grad, layer.bias.grad), g[l]):
            assert close(perm(got), w), l


# ---- engine ---------------------------------------------------------------------------------------------------------------------
def _engine(seed=0, **kw):
    from lstm_tensorspark_b200.engine import TrainEngine
    cfg = _lm(seed=seed, partitions=1, sync_mode="none", quiet=True, **kw)
    return TrainEngine(cfg, 0, 1, None, batch_size=5, device=torch.device("cpu"), dtype=torch.float32)


def _batch(seed=0):
    return tuple(torch.as_tensor(a) for a in D.synthetic_next_token(5, 6, 64, seed=seed)[:2])


def _train(eng, n):
    x, y = _batch()
    return [float(eng.step(x, y)) for _ in range(n)], eng.flat.data.clone()


@pytest.mark.parametrize("tied", [False, True])
def test_zero_coefficients_are_the_run_without_flags(tied):
    l0, w0 = _train(_engine(tie_embeddings=tied, **RECIPE), 3)
    ez = _engine(tie_embeddings=tied, activation_reg=0.0, temporal_activation_reg=0.0, **RECIPE)
    lz, wz = _train(ez, 3)
    assert l0 == lz and torch.equal(w0, wz) and ez.activation_penalties() is None
    for kw in (dict(activation_reg=2.0), dict(temporal_activation_reg=1.0)):
        lr, wr = _train(_engine(tie_embeddings=tied, **RECIPE, **kw), 3)
        assert lr[0] == l0[0] and not torch.equal(wr, w0)             # same first loss (reported), another update


def test_evaluation_ignores_the_flags():
    a, b = _engine(**RECIPE, **AWD), _engine(**RECIPE)
    assert torch.equal(a.flat.data, b.flat.data)
    x, y = _batch(1)
    assert [float(v) for v in a.evaluate(x, y)] == [float(v) for v in b.evaluate(x, y)]
    assert a.model.rnn.activation_penalties is None
    a.model.train()
    a.model(x, y)
    assert a.model.rnn.activation_penalties is not None


def test_tar_stays_inside_a_stateful_segment():
    """--stateful: the carried state is the start of the segment, not a step of it (AWD's TAR is over raw_h[1:] - raw_h[:-1])."""
    eng = _engine(stateful=True, optimizer="sgd", learning_rate=0.0, temporal_activation_reg=1.0)
    m = eng.model
    x, y = _batch(2)
    eng.step(x, y, reset=True)
    eng.step(x, y)                                                    # starts from a non-zero carried state
    start = [(h.clone(), c.clone()) for h, c in eng.state_prev]
    assert float(start[-1][0].abs().sum()) > 0
    got = float(eng.activation_penalties()[1])
    m.train()
    h = m.sequence_features(x, None, state=start).detach()            # no output dropout: the raw output
    want = float((h[1:] - h[:-1]).pow(2).mean())
    across = float((torch.cat([start[-1][0].unsqueeze(0), h]).diff(dim=0)).pow(2).mean())
    assert math.isclose(got, want, rel_tol=1e-5) and not math.isclose(got, across, rel_tol=1e-3)


def _run_cfg(tmp_path, name, **kw):
    base = dict(next_token=True, stateful=True, vocab_size=32, seq_len=6, batch_size=4, hidden_units="8,8", in_features=8,
                synthetic=30, device="cpu", quiet=True, init="scaled", learning_rate=1e-2, tie_embeddings=True,
                checkpoint_path=str(tmp_path / name), output_path=str(tmp_path / (name + "_out")), **RECIPE)
    base.update(kw)
    return Config(**base).validate()


def _latest(path):
    return ckpt.load(ckpt.latest_checkpoint(ckpt.find_latest_run(str(path), None)))


def test_json_log_has_ar_and_tar(tmp_path):
    from lstm_tensorspark_b200.trainer import run_job
    log = tmp_path / "log.jsonl"
    run_job(_run_cfg(tmp_path, "a", epochs=1, max_steps=4, evaluate_every=2, json_log=str(log), **AWD), standalone=True)
    rows = [json.loads(l) for l in log.read_text().splitlines()]
    evals = [r for r in rows if "loss" in r]
    assert evals and all(r["ar"] > 0 and r["tar"] > 0 and math.isfinite(r["perplexity"]) for r in evals)
    log0 = tmp_path / "log0.jsonl"
    run_job(_run_cfg(tmp_path, "b", epochs=1, max_steps=4, evaluate_every=2, json_log=str(log0)), standalone=True)
    assert all("ar" not in json.loads(l) and "tar" not in json.loads(l) for l in log0.read_text().splitlines())


def test_resume_under_other_coefficients(tmp_path):
    from lstm_tensorspark_b200.trainer import run_job
    k = 3
    run_job(_run_cfg(tmp_path, "a", epochs=1, max_steps=k, **AWD), standalone=True)
    out = run_job(_run_cfg(tmp_path, "a", epochs=1, max_steps=2 * k, use_pretrained_model=True, activation_reg=0.5),
                  standalone=True)
    assert out["results"][0]["steps"] == k
    run_job(_run_cfg(tmp_path, "b", epochs=1, max_steps=k), standalone=True)
    va, ma, _ = _latest(tmp_path / "a")
    vb, _, _ = _latest(tmp_path / "b")
    assert ma["global_step"] == 2 * k - 1 and va.keys() == vb.keys()          # the flags add no variable
    ev = run_job(_run_cfg(tmp_path, "a", mode="eval", **AWD), standalone=True)
    ev0 = run_job(_run_cfg(tmp_path, "a", mode="eval"), standalone=True)
    assert ev["loss"] == ev0["loss"] and math.isfinite(ev["loss"])


def _gloo_rank(rank, world):
    import torch.distributed as dist
    from lstm_tensorspark_b200.engine import TrainEngine
    from lstm_tensorspark_b200.parallel.comm import make_communicator
    dev = torch.device("cpu")
    comm = make_communicator("gloo", rank, world, dev, 60)
    cfg = _lm(partitions=world, sync_mode="grad_allreduce", **RECIPE, **AWD)
    eng = TrainEngine(cfg, rank, world, comm, batch_size=5, device=dev, dtype=torch.float32)
    x, y = _batch(rank)
    pens = []
    for _ in range(3):
        eng.step(x, y)
        pens.append(eng.activation_penalties().clone())
    all_w = [torch.zeros_like(eng.flat.data) for _ in range(world)]
    dist.all_gather(all_w, eng.flat.data)
    comm.close()
    return all(torch.equal(all_w[0], w) for w in all_w), [p.tolist() for p in pens]


def test_two_gloo_ranks_train():
    from lstm_tensorspark_b200.parallel.launch import launch
    (same0, p0), (same1, p1) = launch(_gloo_rank, 2)
    assert same0 and same1
    assert all(v > 0 and math.isfinite(v) for p in p0 + p1 for v in p)
    assert p0 != p1                                                   # each replica's penalty is its own
