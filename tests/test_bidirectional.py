"""Bidirectional layers on the CPU: the reverse-time reference against torch.nn.LSTM(bidirectional=True) with and without a
packed sequence, gradcheck, the bidirectional SequenceClassifier against nn.LSTM + Linear, config, checkpoint names and
direction checks, initial weights, gradient buckets, and training / resume / eval / 2-rank runs with --bidirectional."""
import hashlib

import numpy as np
import pytest
import torch

from lstm_tensorspark_b200 import data as D
from lstm_tensorspark_b200.config import Config, parse_args
from lstm_tensorspark_b200.models.classifier import SequenceClassifier
from lstm_tensorspark_b200.ops import reference as ref
from lstm_tensorspark_b200.utils import checkpoint as ckpt


def _to_torch_blocks(w):
    """Gate-interleaved rows (n = 4 j + g, g = i f g o) -> torch's [i; f; g; o] blocks."""
    H = w.shape[0] // 4
    return w.view(H, 4, *w.shape[1:]).transpose(0, 1).reshape(w.shape)


def _set_lstm_dir(lstm, layer, sfx, w_x, w_h, b):
    with torch.no_grad():
        getattr(lstm, f"weight_ih_l{layer}{sfx}").copy_(_to_torch_blocks(w_x.detach()))
        getattr(lstm, f"weight_hh_l{layer}{sfx}").copy_(_to_torch_blocks(w_h.detach()))
        getattr(lstm, f"bias_ih_l{layer}{sfx}").copy_(_to_torch_blocks(b.detach()))
        getattr(lstm, f"bias_hh_l{layer}{sfx}").zero_()


@pytest.mark.parametrize("packed", [False, True])
def test_reverse_reference_matches_bidirectional_nn_lstm_fp64(packed):
    from torch.nn.utils.rnn import pack_padded_sequence, pad_packed_sequence
    torch.manual_seed(0)
    T, B, D, H = 7, 8, 5, 4
    lengths = torch.tensor([7, 1, 3, 7, 2, 5, 6, 4], dtype=torch.int32) if packed else None     # spans 1..T
    dt = dict(dtype=torch.float64)
    x = torch.randn(T, B, D, **dt, requires_grad=True)
    p = {d: [torch.randn(B, H, **dt), torch.randn(B, H, **dt), torch.randn(4 * H, D, **dt), torch.randn(4 * H, H, **dt),
             torch.randn(4 * H, **dt)] for d in ("f", "r")}
    for d in p:
        for t in p[d]:
            t.requires_grad_(True)
    hs_f, hT_f, cT_f = ref.lstm_layer_sequence(x, *p["f"], lengths=lengths)
    hs_r, hT_r, cT_r = ref.lstm_layer_sequence(x, *p["r"], lengths=lengths, reverse=True)

    lstm = torch.nn.LSTM(D, H, bidirectional=True).double()
    _set_lstm_dir(lstm, 0, "", *p["f"][2:])
    _set_lstm_dir(lstm, 0, "_reverse", *p["r"][2:])
    x2 = x.detach().clone().requires_grad_(True)
    h02 = torch.stack([p["f"][0], p["r"][0]]).detach().clone().requires_grad_(True)
    c02 = torch.stack([p["f"][1], p["r"][1]]).detach().clone().requires_grad_(True)
    inp = pack_padded_sequence(x2, lengths.long(), enforce_sorted=False) if packed else x2
    out, (hn, cn) = lstm(inp, (h02, c02))
    if packed:
        out, _ = pad_packed_sequence(out, total_length=T)
    valid = (torch.arange(T).view(T, 1) < (lengths if packed else torch.full((B,), T)).view(1, B)).view(T, B, 1)
    ours = torch.cat([hs_f, hs_r], 2)
    assert torch.allclose(torch.where(valid, ours, 0.0), out, atol=1e-12)
    assert torch.allclose(hT_f, hn[0], atol=1e-12) and torch.allclose(hT_r, hn[1], atol=1e-12)
    assert torch.allclose(cT_f, cn[0], atol=1e-12) and torch.allclose(cT_r, cn[1], atol=1e-12)
    if packed:                                           # reverse padding holds h0: the row starts at its own last step
        pad = ~valid.view(T, B)
        assert torch.equal(hs_r[pad], p["r"][0].detach().expand(T, B, H)[pad])

    g_out, g_h, g_c = torch.randn(T, B, 2 * H, **dt) * valid, torch.randn(2, B, H, **dt), torch.randn(2, B, H, **dt)
    ((ours * g_out).sum() + (torch.stack([hT_f, hT_r]) * g_h).sum() + (torch.stack([cT_f, cT_r]) * g_c).sum()).backward()
    ((out * g_out).sum() + (hn * g_h).sum() + (cn * g_c).sum()).backward()
    assert torch.allclose(x.grad, x2.grad, atol=1e-12)
    assert torch.allclose(p["r"][0].grad, h02.grad[1], atol=1e-12) and torch.allclose(p["r"][1].grad, c02.grad[1], atol=1e-12)
    assert torch.allclose(_to_torch_blocks(p["r"][2].grad), lstm.weight_ih_l0_reverse.grad, atol=1e-12)
    assert torch.allclose(_to_torch_blocks(p["r"][3].grad), lstm.weight_hh_l0_reverse.grad, atol=1e-12)
    assert torch.allclose(_to_torch_blocks(p["r"][4].grad), lstm.bias_ih_l0_reverse.grad, atol=1e-12)
    if packed:
        assert float(x.grad[~valid.view(T, B)].abs().max()) == 0.0                 # padded inputs get no gradient


def test_reverse_reference_gradcheck_with_lengths():
    torch.manual_seed(1)
    T, B, D, H = 4, 3, 2, 3
    lengths = torch.tensor([4, 1, 2], dtype=torch.int32)
    args = [torch.randn(T, B, D), torch.randn(B, H) * 0.5, torch.randn(B, H) * 0.5, torch.randn(4 * H, D) * 0.5,
            torch.randn(4 * H, H) * 0.5, torch.randn(4 * H) * 0.1]
    args = [a.double().requires_grad_(True) for a in args]
    assert torch.autograd.gradcheck(lambda *a: ref.lstm_layer_sequence(*a, lengths=lengths, reverse=True), args)


def test_reverse_is_forward_on_flipped_time():
    torch.manual_seed(2)
    T, B, D, H = 5, 2, 3, 4
    p = [torch.randn(T, B, D), torch.randn(B, H), torch.randn(B, H), torch.randn(4 * H, D), torch.randn(4 * H, H), torch.randn(4 * H)]
    hs_r, hT_r, cT_r = ref.lstm_layer_sequence(*p, reverse=True)
    hs_f, hT_f, cT_f = ref.lstm_layer_sequence(p[0].flip(0), *p[1:])
    assert torch.equal(hs_r, hs_f.flip(0)) and torch.equal(hT_r, hT_f) and torch.equal(cT_r, cT_f)


@pytest.mark.parametrize("packed", [False, True])
def test_bidirectional_classifier_matches_nn_lstm_and_linear(packed):
    from torch.nn.utils.rnn import pack_padded_sequence
    T, B, F, H, C = 6, 5, 4, 3, 3
    cfg = Config(hidden_units=f"{H},{H}", in_features=F, seq_len=T, num_classes=C, batch_size=B, bidirectional=True,
                 learn_initial_state=False, variable_length=packed).validate()
    model = SequenceClassifier(cfg, generator=torch.Generator().manual_seed(3)).double()
    model.set_compute_dtype(torch.float64)
    assert model.head.weights.shape == (2 * H, C)
    lstm = torch.nn.LSTM(F, H, num_layers=2, bidirectional=True).double()
    for i, (lf, lr) in enumerate(zip(model.rnn.layers, model.rnn.reverse_layers)):
        assert lf.dim_size == (F if i == 0 else 2 * H) and lr.node_name == f"LSTMLayer{i}_reverse"
        _set_lstm_dir(lstm, i, "", lf.w_x, lf.w_h, lf.bias)
        _set_lstm_dir(lstm, i, "_reverse", lr.w_x, lr.w_h, lr.bias)
    lin = torch.nn.Linear(2 * H, C).double()
    with torch.no_grad():
        lin.weight.copy_(model.head.weights.t()); lin.bias.copy_(model.head.bias)
    torch.manual_seed(4)
    x = torch.randn(B, T, F, dtype=torch.float64)
    lengths = torch.tensor([6, 1, 3, 5, 2], dtype=torch.int32) if packed else None
    feats = model.features(x, lengths)
    model.rnn.reset_state(B)
    seq = model.rnn.fit_sequence_all(x, lengths)
    inp = x.transpose(0, 1)
    if packed:
        inp = pack_padded_sequence(inp, lengths.long(), enforce_sorted=False)
    out, (hn, _) = lstm(inp)
    want = torch.cat([hn[-2], hn[-1]], 1)
    assert feats.shape == (B, 2 * H) and seq.shape == (T, B, 2 * H)
    assert torch.allclose(feats, want, atol=1e-12)
    assert torch.allclose(feats @ model.head.weights + model.head.bias, lin(want), atol=1e-12)
    if not packed:
        assert torch.allclose(seq, out, atol=1e-12)
    with pytest.raises(ValueError, match="bidirectional"):
        model.rnn.fit_layers(x[:, 0])                          # the one-step path is forward-only


def test_config_validation_and_widths():
    with pytest.raises(ValueError, match="--bidirectional"):
        Config(seq_len=1, bidirectional=True).validate()
    cfg = parse_args(["--bidirectional", "--seq_len", "4", "--hidden_units", "8,6,5", "--in_features", "3"], standalone=True)
    assert cfg.bidirectional and [s["dim_size"] for s in cfg.net_settings()] == [3, 16, 12]
    assert [s["dim_size"] for s in Config(hidden_units="8,6,5", in_features=3).net_settings()] == [3, 8, 6]
    assert not parse_args([], standalone=True).bidirectional


def _digest(model):
    h = hashlib.sha256()
    for k, v in model.named_reference_variables():
        h.update(k.encode()); h.update(v.detach().contiguous().numpy().tobytes())
    return h.hexdigest()


def test_unidirectional_initial_weights_unchanged_and_reverse_drawn_last():
    # digests of the initial weights before bidirectional layers existed
    want = ["95e11e2f9ede0b95790da193dabf9b973dbc64a5f76d4cdb5d58f459d5d8922b",
            "c3734d24bc68595f3c9d9cc48ca5a8636e716a0dbea68cc6490c15e0eba42db3"]
    kws = (dict(hidden_units="8,6", in_features=5, seq_len=4, num_classes=3, init="scaled"),
           dict(hidden_units="7", in_features=3, seq_len=1, num_classes=4))
    for kw, w in zip(kws, want):
        m = SequenceClassifier(Config(batch_size=3, **kw).validate(), generator=torch.Generator().manual_seed(11))
        assert _digest(m) == w
    cfg = dict(hidden_units="8", in_features=5, seq_len=4, num_classes=3, batch_size=3)
    uni = SequenceClassifier(Config(**cfg).validate(), generator=torch.Generator().manual_seed(5))
    bi = SequenceClassifier(Config(bidirectional=True, **cfg).validate(), generator=torch.Generator().manual_seed(5))
    for a, b in zip(uni.rnn.layers.parameters(), bi.rnn.layers.parameters()):
        assert torch.equal(a, b)                              # the forward direction is drawn first, as before


def test_checkpoint_names_round_trip_and_direction_mismatch(tmp_path):
    kw = dict(hidden_units="6,4", in_features=3, seq_len=5, num_classes=3, batch_size=2)
    a = SequenceClassifier(Config(bidirectional=True, **kw).validate(), generator=torch.Generator().manual_seed(0))
    names = [k for k, _ in a.named_reference_variables()]
    assert "LSTMLayer1_reverse/weights_forget_h" in names and "LSTMLayer0_reverse/bias_output" in names
    assert "LSTMLayer0/weights_input_x" in names and len(names) == len(set(names))
    saver = ckpt.Saver(str(tmp_path), "m")
    saver.save(a.reference_state_dict(), global_step=3)
    variables, _, _ = ckpt.load(ckpt.latest_checkpoint(str(tmp_path)))
    b = SequenceClassifier(Config(bidirectional=True, **kw).validate(), generator=torch.Generator().manual_seed(1))
    b.check_directions(variables)
    b.load_reference_state_dict(variables)
    for (k, va), (_, vb) in zip(a.named_reference_variables(), b.named_reference_variables()):
        assert torch.equal(va, vb), k
    uni = SequenceClassifier(Config(**kw).validate())
    with pytest.raises(ValueError, match="--bidirectional"):
        uni.check_directions(variables)
    with pytest.raises(ValueError, match="--bidirectional"):
        b.check_directions(uni.reference_state_dict())


def test_bucket_plan_covers_both_directions_once():
    from lstm_tensorspark_b200.engine import TrainEngine
    cfg = Config(hidden_units="8,6", in_features=4, seq_len=3, num_classes=3, batch_size=4, bidirectional=True, device="cpu",
                 learn_initial_state=False).validate()
    eng = TrainEngine(cfg, device=torch.device("cpu"), dtype=torch.float32)
    rnn = eng.model.rnn
    assert len(rnn.averaged_parameters()) == 12 and len(rnn.map_data_by_key()[0][1]) == 4
    eng.flat.enable_direct_grads(rnn.averaged_parameters() + [eng.model.head.weights, eng.model.head.bias])
    plan = eng._make_bucket_plan()
    assert len(plan) == 8
    hit = np.zeros(eng.flat.padded_numel, dtype=int)
    for b in plan:
        hit[b["lo"]:b["hi"]] += 1
    assert (hit[:eng.flat.lstm_numel] == 1).all() and (hit <= 1).all()
    owners = set().union(*[b["need"] for b in plan])
    assert all(p.data_ptr() in owners for p in rnn.averaged_parameters())


def _final_state(path):
    return ckpt.load(ckpt.latest_checkpoint(ckpt.find_latest_run(path, None)))


def test_standalone_bidirectional_ragged_trains_resumes_and_scores(tmp_path):
    from lstm_tensorspark_b200.trainer import run_job
    base = dict(synthetic=96, hidden_units="10,6", in_features=3, seq_len=6, num_classes=3, variable_length=True,
                bidirectional=True, batch_size=16, device="cpu", quiet=True, learning_rate=2e-2, init="scaled",
                evaluate_every=2, output_path=str(tmp_path / "out"))
    a = Config(max_steps=8, checkpoint_path=str(tmp_path / "a"), **base).validate()
    run_job(a, standalone=True)
    va, ma, oa = _final_state(a.checkpoint_path)
    assert any(k.startswith("LSTMLayer1_reverse/") for k in va) and va["Dense1/weights"].shape == (12, 3)
    b1 = Config(max_steps=4, checkpoint_path=str(tmp_path / "b"), **base).validate()
    run_job(b1, standalone=True)
    b2 = Config(max_steps=8, checkpoint_path=str(tmp_path / "b"), use_pretrained_model=True, **base).validate()
    assert run_job(b2, standalone=True)["results"][0]["steps"] == 4
    vb, mb, ob = _final_state(b2.checkpoint_path)
    assert ma["global_step"] == mb["global_step"] == 7
    for k in va:
        assert torch.equal(va[k], vb[k]), k
    assert torch.equal(oa["optimizer"]["m"], ob["optimizer"]["m"]) and torch.equal(oa["optimizer"]["v"], ob["optimizer"]["v"])
    ev = run_job(Config(mode="eval", checkpoint_path=a.checkpoint_path, **dict(base, batch_size=40)).validate(), standalone=True)
    assert ev["samples"] == 96 and np.isfinite(ev["loss"])
    # a unidirectional run cannot resume from / score a bidirectional checkpoint (and the other way round)
    uni = dict(base, bidirectional=False)
    with pytest.raises(ValueError, match="--bidirectional"):
        run_job(Config(max_steps=10, checkpoint_path=a.checkpoint_path, use_pretrained_model=True, **uni).validate(), standalone=True)
    with pytest.raises(ValueError, match="--bidirectional"):
        run_job(Config(mode="eval", checkpoint_path=a.checkpoint_path, **uni).validate(), standalone=True)
    run_job(Config(max_steps=2, checkpoint_path=str(tmp_path / "u"), **uni).validate(), standalone=True)
    with pytest.raises(ValueError, match="--bidirectional"):
        run_job(Config(max_steps=4, checkpoint_path=str(tmp_path / "u"), use_pretrained_model=True, **base).validate(),
                standalone=True)


def _grad_sync_check_bidirectional(rank, world):
    import torch.distributed as dist
    from lstm_tensorspark_b200.engine import TrainEngine
    from lstm_tensorspark_b200.parallel.comm import make_communicator
    dev = torch.device("cpu")
    comm = make_communicator("gloo", rank, world, dev, 60)
    cfg = Config(hidden_units="8,8", in_features=4, batch_size=6, seq_len=5, sync_mode="grad_allreduce", device="cpu",
                 learn_initial_state=True, init="scaled", partitions=world, variable_length=True, bidirectional=True)
    eng = TrainEngine(cfg, rank, world, comm, batch_size=6, device=dev, dtype=torch.float32)
    x, y, l = D.synthetic_sequences(6, 5, 4, 3, seed=rank, variable_length=True)
    for _ in range(4):
        eng.step(torch.as_tensor(x), torch.as_tensor(y), torch.as_tensor(l))
    all_w = [torch.zeros_like(eng.flat.data) for _ in range(world)]
    dist.all_gather(all_w, eng.flat.data)
    comm.close()
    return bool(all(torch.equal(all_w[0], w) for w in all_w))


def test_grad_allreduce_bidirectional_keeps_replicas_identical():
    from lstm_tensorspark_b200.parallel.launch import launch
    assert launch(_grad_sync_check_bidirectional, 2) == [True, True]
