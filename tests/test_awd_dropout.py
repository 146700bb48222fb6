"""AWD-LSTM's remaining dropouts without a GPU (``--locked_dropout``, ``--input_dropout``, ``--output_dropout``,
``--embedding_dropout``): flags, the mask streams (locked and per-step, every site's counter word c2), the per-step masks of
``--dropout`` as they were, kept fractions, a training step in fp64 against an independent construction from torch modules,
P = 0 and eval mode as the unmasked model, the step counter, and resume."""
import dataclasses
import math
import warnings

import pytest
import torch

from lstm_tensorspark_b200 import data as D
from lstm_tensorspark_b200.config import Config, parse_args
from lstm_tensorspark_b200.models.classifier import SequenceClassifier
from lstm_tensorspark_b200.ops import reference as ref
from lstm_tensorspark_b200.ops.reference import DropoutSpec
from lstm_tensorspark_b200.utils import checkpoint as ckpt

NEW_FLAGS = ("input_dropout", "output_dropout", "embedding_dropout")
RECIPE = dict(locked_dropout=True, input_dropout=0.65, dropout=0.3, output_dropout=0.4, embedding_dropout=0.1)


def _lm(**kw):
    base = dict(hidden_units="16,16", in_features=16, seq_len=6, batch_size=5, vocab_size=64, next_token=True, init="scaled",
                learn_initial_state=False, device="cpu")
    base.update(kw)
    return Config(**base).validate()


# ---- flags --------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("flag", NEW_FLAGS)
@pytest.mark.parametrize("bad", [-0.1, 1.0, 1.5])
def test_p_out_of_range_names_the_flag(flag, bad):
    with pytest.raises(ValueError, match=f"--{flag}"):
        _lm(**{flag: bad})


@pytest.mark.parametrize("flag", ["input_dropout", "embedding_dropout"])
def test_embedding_dropouts_need_token_ids(flag):
    with pytest.raises(ValueError) as ei:
        Config(hidden_units="8", in_features=4, seq_len=4, per_step_labels=True, **{flag: 0.2}).validate()
    assert f"--{flag}" in str(ei.value) and "--vocab_size" in str(ei.value)


def test_output_dropout_needs_a_sequence_head():
    with pytest.raises(ValueError) as ei:
        Config(hidden_units="8", in_features=4, seq_len=4, output_dropout=0.2).validate()
    assert "--output_dropout" in str(ei.value) and "--pooling" in str(ei.value) and "--per_step_labels" in str(ei.value)
    for ok in (dict(per_step_labels=True), dict(pooling="mean"), dict(pooling="attention")):
        Config(hidden_units="8", in_features=4, seq_len=4, output_dropout=0.2, **ok).validate()


def test_locked_without_a_dropout_warns():
    with pytest.warns(UserWarning, match="--locked_dropout"):
        _lm(locked_dropout=True, embedding_dropout=0.1, weight_drop=0.5)
    with warnings.catch_warnings():
        warnings.simplefilter("error")
        for p in NEW_FLAGS[:2] + ("dropout",):
            _lm(locked_dropout=True, **{p: 0.2})


def test_flags_parse_on_both_entry_points_and_default_off():
    argv = ["--next_token", "--vocab_size", "64", "--in_features", "16", "--hidden_units", "16,16", "--seq_len", "4",
            "--locked_dropout", "--input_dropout", "0.65", "--dropout", "0.3", "--output_dropout", "0.4",
            "--embedding_dropout", "0.1"]
    for standalone in (False, True):
        cfg = parse_args(argv, standalone=standalone)
        assert (cfg.locked_dropout, cfg.input_dropout, cfg.output_dropout, cfg.embedding_dropout) == (True, 0.65, 0.4, 0.1)
    d = Config()
    assert not d.locked_dropout and d.input_dropout == d.output_dropout == d.embedding_dropout == 0.0


# ---- masks --------------------------------------------------------------------------------------------------------------------
def test_every_site_has_its_own_stream():
    key, step = (7, 3), 5
    specs = {}
    for layer in (0, 1, 2):
        for rev in (False, True):
            for locked in (False, True):
                specs[("layer", layer, rev, locked)] = DropoutSpec(0.5, key, layer, rev, step, locked=locked)
            specs[("weight", layer, rev)] = DropoutSpec(0.5, key, layer, rev, step, weight=True)
    for locked in (False, True):
        specs[("input", locked)] = DropoutSpec(0.5, key, 0, False, step, site="input", locked=locked)
    specs["rows"] = DropoutSpec(0.5, key, 0, False, step, site="rows")
    c2 = [s.c2 for s in specs.values()]
    assert len(set(c2)) == len(c2)
    assert specs[("input", True)].c2 == ref.LOCKED_C2 | ref.INPUT_DROP_C2 and specs["rows"].c2 == ref.ROW_DROP_C2
    assert specs[("layer", 1, True, True)].c2 == ref.LOCKED_C2 | 3
    masks = [ref.dropout_mask(s, 1, 4, 64)[0] for s in specs.values()]
    for i in range(len(masks)):
        for j in range(i):
            assert not torch.equal(masks[i], masks[j])
    with pytest.raises(ValueError):
        DropoutSpec(0.5, key, 0, False, step, weight=True, locked=True)
    with pytest.raises(ValueError):
        DropoutSpec(0.5, key, 0, False, step, site="rows", locked=True)


@pytest.mark.parametrize("site", ["layer", "input"])
def test_locked_masks_are_one_mask_for_every_step(site):
    spec = DropoutSpec(0.4, (11, 2), 1, False, 9, site=site, locked=True)
    m = ref.dropout_mask(spec, 7, 5, 24, t0=3)
    assert all(torch.equal(m[t], m[0]) for t in range(7))
    assert torch.equal(m[0], ref.dropout_mask(spec, 1, 5, 24)[0])
    # the locked mask at t is the per-step counter at time 0 of the locked stream (its own c2)
    w = ref.philox4x32_10(torch.tensor([2 * 3 + 1, 0, spec.c2, 9]), 11, 2)
    assert bool(m[4, 2, 10]) == (((int(w[1]) >> 0) & 0xFFFF) >= spec.thr)
    per_step = ref.dropout_mask(dataclasses.replace(spec, locked=False), 7, 5, 24)
    assert not all(torch.equal(per_step[t], per_step[0]) for t in range(7))
    assert not torch.equal(per_step[0], m[0])


def test_per_step_dropout_masks_are_unchanged():
    """Bit patterns of ``--dropout``'s per-step masks, recorded before locked masks existed."""
    m = ref.dropout_mask(DropoutSpec(0.3, (1234, 1), 0, False, 7), 5, 3, 20)
    assert int(m.sum()) == 199
    bits = [int(x) for x in (m.reshape(5, -1).to(torch.int64) * (2 ** torch.arange(60))).sum(1)]
    assert bits == [52043996024462199, 574842269895392138, 790802054054000526, 1147440833099857871, 609811099938912175]
    m = ref.dropout_mask(DropoutSpec(0.5, (99, 0), 1, True, 123456), 2, 2, 16, t0=3)
    assert [int(x) for x in (m.reshape(2, -1).to(torch.int64) * (2 ** torch.arange(32))).sum(1)] == [257062371, 1727482316]


@pytest.mark.parametrize("site,p", [("layer", 0.3), ("input", 0.65), ("rows", 0.1), ("layer", 0.4)])
def test_kept_fraction_within_a_binomial_bound(site, p):
    spec = DropoutSpec(p, (3, 0), 0, False, 2, site=site, locked=site != "rows")
    m = ref.embedding_row_mask(spec, 32768) if site == "rows" else ref.dropout_mask(spec, 1, 64, 512)
    n, q = m.numel(), 1 - ref.dropout_threshold(p) / 65536
    assert abs(float(m.float().mean()) - q) <= 5 * math.sqrt(q * (1 - q) / n)


def test_reference_embedding_masks():
    g = torch.Generator().manual_seed(0)
    V, E, B, T = 40, 12, 3, 5
    table = torch.randn(V, E, generator=g)
    tok = torch.randint(-2, V + 2, (B, T), generator=g)
    lengths = torch.tensor([5, 2, 4], dtype=torch.int32)
    si = DropoutSpec(0.3, (1, 2), 0, False, 4, site="input", locked=True)
    se = DropoutSpec(0.25, (1, 2), 0, False, 4, site="rows")
    x0 = ref.embedding(tok, table, lengths)
    rows = ref.embedding_row_mask(se, V)
    mi = ref.dropout_mask(si, T, B, E)
    f = ref.dropout_scale(0.3) * ref.dropout_scale(0.25)
    for i, e in ((si, None), (None, se), (si, se)):
        x = ref.embedding(tok, table, lengths, input_dropout=i, embedding_dropout=e)
        keep = torch.ones(T, B, E, dtype=torch.bool)
        if e is not None:
            keep &= rows[tok.t().clamp(0, V - 1)].unsqueeze(2)
        if i is not None:
            keep &= mi
        s = f if (i and e) else ref.dropout_scale((i or e).p)
        assert torch.equal(x, torch.where(keep, x0 * s, torch.zeros(())))
    assert torch.equal(ref.embedding(tok, table, lengths, input_dropout=dataclasses.replace(si, p=0.0)), x0)


# ---- fp64 against AWD-LSTM built from torch modules ----------------------------------------------------------------------------
def _torch_awd(m, x, y, key, step, cfg):
    """AWD-LSTM's regularisers around nn.Embedding / nn.LSTM / F.linear in fp64: a masked copy of the table (dropoute) and
    LockedDropout masks ``[1, B, H]`` broadcast over T, each mask taken from ``reference.dropout_mask`` with T = 1."""
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
        return ref.dropout_mask(spec, 1, B, H).double() * float(ref.dropout_scale(p))        # [1, B, H]

    rows = ref.embedding_row_mask(DropoutSpec(cfg.embedding_dropout, key, 0, False, step, site="rows"), V)
    masked = table * rows.double().unsqueeze(1) * float(ref.dropout_scale(cfg.embedding_dropout))
    h = torch.nn.functional.embedding(x.long(), masked).transpose(0, 1)                     # [T, B, E]
    h = h * locked(cfg.input_dropout, E, layer=0, reverse=False, site="input")
    n = len(lstms)
    for l, lstm in enumerate(lstms):
        h, _ = lstm(h)
        h = h * locked(cfg.dropout if l < n - 1 else cfg.output_dropout, h.shape[2], layer=l, reverse=False)
    w = table if m.tied else head_w.t()
    logits = torch.nn.functional.linear(h.transpose(0, 1), w, bias)
    loss = torch.nn.functional.cross_entropy(logits.reshape(-1, V), y.reshape(-1).long())
    loss.backward()
    grads = {"table": table.grad, "bias": bias.grad, "head": None if m.tied else head_w.grad}
    for l, lstm in enumerate(lstms):
        grads[l] = (lstm.weight_ih_l0.grad, lstm.weight_hh_l0.grad, lstm.bias_ih_l0.grad)
    return loss, grads, perm


@pytest.mark.parametrize("tied", [False, True])
def test_training_step_equals_awd_lstm_from_torch_modules_in_fp64(tied):
    cfg = _lm(tie_embeddings=tied, **RECIPE)
    m = SequenceClassifier(cfg, batch_size=5, device="cpu", generator=torch.Generator().manual_seed(7)).to(torch.float64)
    m.set_compute_dtype(torch.float64)
    key, step = (12, 1), 4
    m.rnn.dropout_key, m.rnn.dropout_step = key, step
    x, y = (torch.as_tensor(a) for a in D.synthetic_next_token(5, 6, 64, seed=3)[:2])
    loss, _logits, _ = m(x, y)
    loss.backward()
    want, g, perm = _torch_awd(m, x, y, key, step, cfg)
    close = lambda a, b: torch.allclose(a, b, rtol=1e-10, atol=1e-12)
    assert close(loss, want)
    assert close(m.embedding.weights.grad, g["table"]) and close(m.head.bias.grad, g["bias"])
    if not tied:
        assert close(m.head.weights.grad, g["head"])
    for l, layer in enumerate(m.rnn.layers):
        for got, w in zip((layer.w_x.grad, layer.w_h.grad, layer.bias.grad), g[l]):
            assert close(perm(got), w), l
    # the masks mattered: the unmasked model has another loss
    m.zero_grad()
    m.eval()
    plain, _, _ = m(x, y)
    assert not close(plain, want)


# ---- engine: P = 0, eval, counter, resume --------------------------------------------------------------------------------------
def _engine(seed=0, **kw):
    from lstm_tensorspark_b200.engine import TrainEngine
    cfg = _lm(seed=seed, partitions=1, sync_mode="none", quiet=True, **kw)
    return TrainEngine(cfg, 0, 1, None, batch_size=5, device=torch.device("cpu"), dtype=torch.float32)


def _batch(seed=0):
    return tuple(torch.as_tensor(a) for a in D.synthetic_next_token(5, 6, 64, seed=seed)[:2])


def _train(eng, n):
    x, y = _batch()
    return [float(eng.step(x, y)) for _ in range(n)], eng.flat.data.clone()


@pytest.mark.filterwarnings("ignore:--locked_dropout has no effect")
@pytest.mark.parametrize("tied", [False, True])
def test_zero_p_is_the_model_without_flags(tied):
    l0, w0 = _train(_engine(tie_embeddings=tied), 3)
    lz, wz = _train(_engine(tie_embeddings=tied, locked_dropout=True, input_dropout=0.0, output_dropout=0.0,
                            embedding_dropout=0.0), 3)
    assert l0 == lz and torch.equal(w0, wz)
    lr, wr = _train(_engine(tie_embeddings=tied, **RECIPE), 3)
    assert lr != l0 and not torch.equal(wr, w0)


def test_evaluation_ignores_the_flags():
    a, b = _engine(**RECIPE), _engine()
    assert torch.equal(a.flat.data, b.flat.data)
    x, y = _batch(1)
    assert [float(v) for v in a.evaluate(x, y)] == [float(v) for v in b.evaluate(x, y)]


@pytest.mark.parametrize("flag", NEW_FLAGS)
def test_step_counter_advances_with_only_a_new_flag(flag):
    e = _engine(hidden_units="16", **{flag: 0.3})
    assert e._dropout_on
    losses, _ = _train(e, 3)
    assert e.model.rnn.dropout_step == 3 and len(set(losses)) == 3
    assert not _engine(hidden_units="16")._dropout_on


def test_locked_only_changes_the_masks():
    a, _ = _train(_engine(dropout=0.3, output_dropout=0.4, input_dropout=0.5), 2)
    b, _ = _train(_engine(locked_dropout=True, dropout=0.3, output_dropout=0.4, input_dropout=0.5), 2)
    assert a != b


def _run_cfg(tmp_path, name, **kw):
    base = dict(next_token=True, stateful=True, vocab_size=32, seq_len=6, batch_size=4, hidden_units="8,8", in_features=8,
                synthetic=30, device="cpu", quiet=True, init="scaled", learning_rate=1e-2, tie_embeddings=True,
                checkpoint_path=str(tmp_path / name), output_path=str(tmp_path / (name + "_out")), **RECIPE)
    base.update(kw)
    return Config(**base).validate()


def _latest(path):
    return ckpt.load(ckpt.latest_checkpoint(ckpt.find_latest_run(str(path), None)))


def test_resume_draws_the_masks_of_the_uninterrupted_run(tmp_path):
    from lstm_tensorspark_b200.trainer import run_job
    k = 3
    run_job(_run_cfg(tmp_path, "a", epochs=1, max_steps=k, evaluate_every=k), standalone=True)
    run_job(_run_cfg(tmp_path, "a", epochs=1, max_steps=2 * k, evaluate_every=k, use_pretrained_model=True), standalone=True)
    run_job(_run_cfg(tmp_path, "b", epochs=1, max_steps=2 * k, evaluate_every=k), standalone=True)
    va, ma, _ = _latest(tmp_path / "a")
    vb, mb, _ = _latest(tmp_path / "b")
    assert ma["global_step"] == mb["global_step"]
    assert va.keys() == vb.keys() and all(torch.equal(va[n], vb[n]) for n in va)
    # a checkpoint written without the flags resumes with them, and the flags add no variable
    run_job(_run_cfg(tmp_path, "c", epochs=1, max_steps=k, **{f: 0.0 for f in RECIPE if f != "locked_dropout"},
                     locked_dropout=False), standalone=True)
    out = run_job(_run_cfg(tmp_path, "c", epochs=1, max_steps=2 * k, use_pretrained_model=True), standalone=True)
    assert out["results"][0]["steps"] == k
    vc, _, _ = _latest(tmp_path / "c")
    assert vc.keys() == va.keys()
    ev = run_job(_run_cfg(tmp_path, "a", mode="eval"), standalone=True)
    ev0 = run_job(_run_cfg(tmp_path, "a", mode="eval", **{f: 0.0 for f in RECIPE if f != "locked_dropout"},
                           locked_dropout=False), standalone=True)
    assert ev["loss"] == ev0["loss"] and math.isfinite(ev["loss"])
