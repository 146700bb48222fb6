"""Weight drop (AWD-LSTM's DropConnect on the recurrent weights, ``--weight_drop``) without a GPU: the mask is the dropout mask of
its own counter stream, the reference layer equals the layer fed ``W_h * M * s`` explicitly (outputs and every gradient), eval
mode and P = 0 are the unmasked model bit for bit, flags, and end-to-end runs (a stateful language model, resume, a checkpoint
written without the flag, two replicas under a gradient allreduce)."""
import dataclasses
import math

import pytest
import torch

from lstm_tensorspark_b200.config import Config, parse_args
from lstm_tensorspark_b200.ops import reference as ref
from lstm_tensorspark_b200.ops.reference import DropoutSpec
from lstm_tensorspark_b200.utils import checkpoint as ckpt


def _wspec(p=0.5, key=(7, 3), layer=0, reverse=False, step=4):
    return DropoutSpec(p, key, layer, reverse, step, weight=True)


# ---- the mask -----------------------------------------------------------------------------------------------------------------
def test_mask_is_the_dropout_mask_of_the_weight_counter_stream():
    spec = _wspec(0.3, layer=2, reverse=True, step=11)
    assert spec.c2 == 0x80000000 | 5 and spec.desc()[3] == 0x80000000 | 5
    H = 20                                                       # 3 Philox groups per row, the last one partial
    m = ref.weight_drop_mask(spec, 4 * H, H)
    assert m.shape == (4 * H, H)
    assert torch.equal(m, ref.dropout_mask(spec, 1, 4 * H, H)[0])
    for r, k in [(0, 0), (79, 19), (33, 9), (41, 16)]:           # counter (r ceil(H/8) + k/8, 0, c2, step)
        w = ref.philox4x32_10(torch.tensor([r * 3 + k // 8, 0, 0x80000005, 11]), 7, 3)
        v = (int(w[(k % 8) // 2]) >> (16 * (k % 2))) & 0xFFFF
        assert bool(m[r, k]) == (v >= spec.thr), (r, k)


@pytest.mark.parametrize("p", [0.1, 0.5])
def test_kept_fraction_within_a_binomial_bound(p):
    H = 256
    m = ref.weight_drop_mask(_wspec(p), 4 * H, H)
    n, q = m.numel(), 1 - ref.dropout_threshold(p) / 65536
    assert abs(float(m.float().mean()) - q) <= 5 * math.sqrt(q * (1 - q) / n)


def test_masks_differ_by_layer_direction_step_and_partition():
    base = _wspec()
    m = ref.weight_drop_mask(base, 256, 64)
    for kw in [dict(layer=1), dict(reverse=True), dict(step=5), dict(key=(7, 4)), dict(key=(8, 3))]:
        assert not torch.equal(m, ref.weight_drop_mask(dataclasses.replace(base, **kw), 256, 64)), kw


def test_mask_is_disjoint_from_the_output_dropout_stream():
    """Same (key, layer, reverse, step): the weight stream's counters carry c2's high bit, the output stream's never do."""
    w = _wspec(0.5, layer=1, step=9)
    out = dataclasses.replace(w, weight=False)
    assert out.c2 == 2 and w.c2 == out.c2 | ref.WEIGHT_DROP_C2 and out.c2 < 2 ** 31
    assert not torch.equal(ref.weight_drop_mask(w, 256, 64), ref.dropout_mask(out, 1, 256, 64)[0])


def _rnn(hidden, D, B, wd, p=0.0, bidirectional=False, seed=0):
    from lstm_tensorspark_b200.models.recurrent.rnn import RNN
    settings = [{"layer_name": f"LSTMLayer{i}", "num_hidden": h, "batch_size": B,
                 "dim_size": D if i == 0 else (2 if bidirectional else 1) * hidden[i - 1]} for i, h in enumerate(hidden)]
    rnn = RNN(settings, dropout=p, weight_drop=wd, learn_initial_state=False, init="scaled",
              generator=torch.Generator().manual_seed(seed))
    if bidirectional:
        rnn.add_reverse_layers()
    rnn.dropout_key, rnn.dropout_step = (42, 1), 6
    return rnn


def test_mask_does_not_depend_on_the_batch():
    """The spec of a layer has no row offset and nothing in it depends on B or T; the CUDA path hands the same spec to every batch
    chunk (no ``at_rows``)."""
    a, b = _rnn([8, 8], 4, 3, 0.5), _rnn([8, 8], 4, 11, 0.5)
    for layer in (0, 1):
        sa, sb = a.weight_drop_spec(layer), b.weight_drop_spec(layer)
        assert sa == sb and sa.row0 == 0 and sa.weight
        assert torch.equal(ref.weight_drop_mask(sa, 32, 8), ref.weight_drop_mask(sb, 32, 8))


# ---- the reference layer ------------------------------------------------------------------------------------------------------
def _masked(w_h, spec):
    keep = ref.weight_drop_mask(spec, *w_h.shape)
    return keep, torch.where(keep, w_h * ref.dropout_scale(spec.p).to(w_h.dtype), torch.zeros((), dtype=w_h.dtype))


@pytest.mark.parametrize("reverse,lengths,T", [(False, False, 7), (True, False, 7), (False, True, 7), (True, True, 7),
                                               (False, False, 1)])
def test_reference_layer_equals_the_layer_fed_the_masked_weights(reverse, lengths, T):
    torch.manual_seed(0)
    B, D, H = 5, 6, 12
    spec = _wspec(0.4, layer=1, reverse=reverse)
    x = torch.randn(T, B, D, dtype=torch.float64)
    p = [torch.randn(B, H, dtype=torch.float64) * 0.3, torch.randn(B, H, dtype=torch.float64) * 0.3,
         torch.randn(4 * H, D, dtype=torch.float64) / D ** 0.5, torch.randn(4 * H, H, dtype=torch.float64) / H ** 0.5,
         torch.randn(4 * H, dtype=torch.float64) * 0.1]
    ln = torch.tensor([T, max(1, T - 4), 1, max(1, T - 1), T], dtype=torch.int32) if lengths else None
    wo, wh = torch.randn(T, B, H, dtype=torch.float64), torch.randn(B, H, dtype=torch.float64)
    keep, w_masked = _masked(p[3], spec)

    def run(explicit):
        leaves = [t.clone().requires_grad_(True) for t in [x] + p]
        if explicit:
            w_h_prime = leaves[4].detach().clone().requires_grad_(True)
            w_h_prime.data.copy_(w_masked)
            hs, hT, cT = ref.lstm_layer_sequence(leaves[0], leaves[1], leaves[2], leaves[3], w_h_prime, leaves[5], lengths=ln,
                                                 reverse=reverse)
        else:
            hs, hT, cT = ref.lstm_layer_sequence(*leaves, lengths=ln, reverse=reverse, weight_drop=spec)
        ((hs * wo).sum() + (hT * wh).sum() + cT.sum()).backward()
        grads = [t.grad for t in leaves]
        if explicit:
            grads[4] = w_h_prime.grad
        return [hs.detach(), hT.detach(), cT.detach()] + grads

    got, want = run(False), run(True)
    for i in range(3):
        assert torch.equal(got[i], want[i]), i
    for i in (3, 4, 5, 6, 8):                                   # dx, dh0, dc0, dW_x, db
        assert torch.equal(got[i], want[i]), i
    s = ref.dropout_scale(spec.p).double()
    assert torch.equal(got[7], torch.where(keep, want[7] * s, torch.zeros((), dtype=torch.float64)))     # dW_h = M s dW_h'


def test_one_step_path_reads_the_masked_weights():
    from lstm_tensorspark_b200.ops import functional as F
    torch.manual_seed(1)
    B, D, H = 3, 4, 8
    x, h, c = torch.randn(B, D), torch.randn(B, H), torch.randn(B, H)
    w_x, w_h, b = torch.randn(4 * H, D), torch.randn(4 * H, H), torch.randn(4 * H)
    spec = _wspec(0.5)
    got = F.lstm_cell_step(x, h, c, w_x, w_h, b, weight_drop=spec)
    want = ref.lstm_cell_step(x, h, c, w_x, _masked(w_h, spec)[1], b)
    assert all(torch.equal(a, w) for a, w in zip(got, want))
    rnn = _rnn([8, 6], D, B, 0.5)
    rnn.reset_state(B)
    out = rnn.fit_layers(x)
    state = x
    for i, l in enumerate(rnn.layers):
        state, _ = ref.lstm_cell_step(state, torch.zeros(B, l.num_hidden), torch.zeros(B, l.num_hidden), l.w_x,
                                      ref.weight_drop(l.w_h, rnn.weight_drop_spec(i)), l.bias)
    assert torch.equal(out.detach(), state.detach())


# ---- eval mode and P = 0 --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bidirectional", [False, True])
def test_eval_and_zero_p_are_the_unmasked_model(bidirectional):
    from lstm_tensorspark_b200.ops import functional as F
    F.set_backend("torch")
    try:
        B, T, D = 4, 6, 5
        x = torch.randn(B, T, D)
        base = _rnn([8, 8], D, B, 0.0, bidirectional=bidirectional)
        on = _rnn([8, 8], D, B, 0.5, bidirectional=bidirectional)
        assert base.weight_drop_spec(0) is None and on.weight_drop_spec(1, bidirectional) is not None
        want = base.fit_layers(x)
        got = on.fit_layers(x)
        assert not torch.equal(got, want)
        on.eval()
        on.reset_state(B)
        assert on.weight_drop_spec(0) is None
        assert torch.equal(on.fit_layers(x), want)
        assert ref.weight_drop(on.layers[0].w_h, DropoutSpec(0.0, (0, 0), 0, False, 0, weight=True)) is on.layers[0].w_h
    finally:
        F.set_backend("auto")


# ---- flags ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bad", ["1.0", "-0.1", "1.5", "nan"])
def test_flag_validation_names_the_flag(bad):
    with pytest.raises(ValueError, match="--weight_drop"):
        parse_args(["--hidden_units", "8", "--weight_drop", bad])


def test_default_is_off_and_a_one_layer_model_is_masked(recwarn):
    assert Config().weight_drop == 0.0
    cfg = parse_args(["--hidden_units", "8", "--weight_drop", "0.3"])
    assert cfg.weight_drop == 0.3 and "WEIGHT_DROP = 0.3" in cfg.params_str()
    assert not [w for w in recwarn.list if "--weight_drop" in str(w.message)]
    single = _rnn([8], 4, 3, 0.3)
    assert single.weight_drop_spec(0) is not None


# ---- engine / trainer ---------------------------------------------------------------------------------------------------------
def _engine(wd, hidden="8", seed=0, **kw):
    from lstm_tensorspark_b200.engine import TrainEngine
    cfg = Config(hidden_units=hidden, in_features=4, batch_size=6, seq_len=5, device="cpu", learn_initial_state=False, init="scaled",
                 weight_drop=wd, seed=seed, partitions=1, sync_mode="none", quiet=True, **kw)
    return TrainEngine(cfg, 0, 1, None, batch_size=6, device=torch.device("cpu"), dtype=torch.float32)


def _train(eng, n):
    from lstm_tensorspark_b200 import data as D
    x, y = (torch.as_tensor(a) for a in D.synthetic_sequences(6, 5, 4, 3, seed=0))
    return [float(eng.step(x, y)) for _ in range(n)], eng.flat.data.clone()


def test_engine_one_layer_counter_and_zero_p():
    l0, w0 = _train(_engine(0.0), 3)
    lc, wc = _train(_engine(Config().weight_drop), 3)
    assert l0 == lc and torch.equal(w0, wc)
    e = _engine(0.5)
    l1, w1 = _train(e, 3)
    assert l1 != l0 and e.model.rnn.dropout_step == 3 and len(set(l1)) == 3
    from lstm_tensorspark_b200 import data as D
    x, y = (torch.as_tensor(a) for a in D.synthetic_sequences(6, 5, 4, 3, seed=1))
    a, b = _engine(0.6), _engine(0.0)
    assert torch.equal(a.flat.data, b.flat.data)
    assert [float(v) for v in a.evaluate(x, y)] == [float(v) for v in b.evaluate(x, y)]       # evaluation: the raw weights


def test_weight_decay_acts_on_the_raw_parameter_and_gradients_are_masked():
    """One SGD step: the gradient of W_h is zero where the mask dropped, so the update there is weight decay alone."""
    e = _engine(0.5, optimizer="sgd", weight_decay=0.1, learning_rate=0.5)
    w0 = e.model.rnn.layers[0].w_h.detach().clone()
    _train(e, 1)
    spec = DropoutSpec(0.5, e.model.rnn.dropout_key, 0, False, 0, weight=True)
    keep = ref.weight_drop_mask(spec, *w0.shape)
    g = e.model.rnn.layers[0].w_h.grad
    assert torch.all(g[~keep] == 0) and float(g[keep].abs().max()) > 0
    w1 = e.model.rnn.layers[0].w_h.detach()
    assert torch.allclose(w1[~keep], w0[~keep] * (1 - 0.5 * 0.1), rtol=1e-6, atol=0)


def _lm_cfg(tmp_path, name, **kw):
    base = dict(next_token=True, stateful=True, vocab_size=32, seq_len=6, batch_size=4, hidden_units="8,8", in_features=6,
                synthetic=30, device="cpu", quiet=True, init="scaled", learning_rate=1e-2, weight_drop=0.5,
                checkpoint_path=str(tmp_path / name), output_path=str(tmp_path / (name + "_out")))
    base.update(kw)
    return Config(**base).validate()


def _latest(path):
    return ckpt.load(ckpt.latest_checkpoint(ckpt.find_latest_run(str(path), None)))


def test_stateful_language_model_trains_and_scores(tmp_path):
    from lstm_tensorspark_b200.trainer import run_job
    out = run_job(_lm_cfg(tmp_path, "lm", epochs=1, max_steps=6, evaluate_every=3, tie_embeddings=True,
                                  hidden_units="8,6"), standalone=True)
    assert out["results"][0]["steps"] == 6
    ev = run_job(_lm_cfg(tmp_path, "lm", mode="eval", tie_embeddings=True, hidden_units="8,6"), standalone=True)
    assert math.isfinite(ev["loss"])
    ev0 = run_job(_lm_cfg(tmp_path, "lm", mode="eval", tie_embeddings=True, hidden_units="8,6", weight_drop=0.0),
                  standalone=True)
    assert ev0["loss"] == ev["loss"]                          # scoring uses the raw weights whatever the flag says


def test_resume_reproduces_the_uninterrupted_run(tmp_path):
    from lstm_tensorspark_b200.trainer import run_job
    k = 4
    run_job(_lm_cfg(tmp_path, "a", epochs=1, max_steps=k, evaluate_every=k), standalone=True)
    run_job(_lm_cfg(tmp_path, "a", epochs=1, max_steps=2 * k, evaluate_every=k, use_pretrained_model=True), standalone=True)
    run_job(_lm_cfg(tmp_path, "b", epochs=1, max_steps=2 * k, evaluate_every=k), standalone=True)
    va, ma, oa = _latest(tmp_path / "a")
    vb, mb, ob = _latest(tmp_path / "b")
    assert ma["global_step"] == mb["global_step"]
    assert va.keys() == vb.keys() and all(torch.equal(va[n], vb[n]) for n in va)
    run_job(_lm_cfg(tmp_path, "c", epochs=1, max_steps=2 * k, evaluate_every=k, weight_drop=0.0), standalone=True)
    vc, _, _ = _latest(tmp_path / "c")
    assert vc.keys() == va.keys() and not all(torch.equal(va[n], vc[n]) for n in va)    # no new variables; the masks mattered


def test_checkpoint_without_the_flag_resumes_with_it(tmp_path):
    from lstm_tensorspark_b200.trainer import run_job
    run_job(_lm_cfg(tmp_path, "n", epochs=1, max_steps=2, weight_drop=0.0), standalone=True)
    out = run_job(_lm_cfg(tmp_path, "n", epochs=1, max_steps=4, use_pretrained_model=True), standalone=True)
    assert out["results"][0]["steps"] == 2


def _grad_sync(rank, world):
    import torch
    import torch.distributed as dist
    from lstm_tensorspark_b200 import data as D
    from lstm_tensorspark_b200.config import Config
    from lstm_tensorspark_b200.engine import TrainEngine
    from lstm_tensorspark_b200.ops import reference as ref
    from lstm_tensorspark_b200.parallel.comm import make_communicator
    dev = torch.device("cpu")
    comm = make_communicator("gloo", rank, world, dev, 60)
    cfg = Config(hidden_units="8", in_features=4, batch_size=6, seq_len=3, sync_mode="grad_allreduce", device="cpu",
                 learn_initial_state=False, init="scaled", partitions=world, weight_drop=0.5)
    eng = TrainEngine(cfg, rank, world, comm, batch_size=6, device=dev, dtype=torch.float32, partition_key=rank)
    spec = eng.model.rnn.weight_drop_spec(0)
    mask = ref.weight_drop_mask(spec, 32, 8).to(torch.int32)
    x, y = D.synthetic_sequences(6, 3, 4, 3, seed=0)                     # the same batch: only the masks tell the replicas apart
    for _ in range(2):
        eng.step(torch.as_tensor(x), torch.as_tensor(y))
    all_w = [torch.zeros_like(eng.flat.data) for _ in range(world)]
    dist.all_gather(all_w, eng.flat.data)
    masks = [torch.zeros_like(mask) for _ in range(world)]
    dist.all_gather(masks, mask)
    comm.close()
    return bool(all(torch.equal(all_w[0], w) for w in all_w)), bool(torch.equal(masks[0], masks[1]))


def test_two_ranks_draw_different_masks_and_stay_equal():
    from lstm_tensorspark_b200.parallel.launch import launch
    res = launch(_grad_sync, 2)
    assert [r[0] for r in res] == [True, True]
    assert [r[1] for r in res] == [False, False]
