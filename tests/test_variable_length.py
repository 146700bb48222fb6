"""Variable-length sequences on the CPU: the masked reference against torch.nn.LSTM on a packed sequence, gradcheck, the
ragged CSV format, synthetic lengths, loaders that carry lengths, and training / resume / eval / 2-rank runs with
--variable_length."""
import os

import numpy as np
import pytest
import torch
from hypothesis import given, settings, strategies as st

from lstm_tensorspark_b200 import data as D
from lstm_tensorspark_b200.config import Config
from lstm_tensorspark_b200.ops import reference as ref


def _to_torch_blocks(w):
    """Gate-interleaved rows (n = 4 j + g, g = i f g o) -> torch's [i; f; g; o] blocks."""
    H = w.shape[0] // 4
    return w.view(H, 4, *w.shape[1:]).transpose(0, 1).reshape(w.shape)


def test_masked_reference_matches_packed_nn_lstm_fp64():
    from torch.nn.utils.rnn import pack_padded_sequence
    torch.manual_seed(0)
    T, B, D, H = 7, 6, 5, 4
    lengths = torch.tensor([7, 1, 3, 7, 2, 5], dtype=torch.int32)
    x = torch.randn(T, B, D, dtype=torch.float64, requires_grad=True)
    h0 = torch.randn(B, H, dtype=torch.float64, requires_grad=True)
    c0 = torch.randn(B, H, dtype=torch.float64, requires_grad=True)
    w_x = torch.randn(4 * H, D, dtype=torch.float64, requires_grad=True)
    w_h = torch.randn(4 * H, H, dtype=torch.float64, requires_grad=True)
    b = torch.randn(4 * H, dtype=torch.float64, requires_grad=True)
    _, hT, cT = ref.lstm_layer_sequence(x, h0, c0, w_x, w_h, b, lengths=lengths)

    lstm = torch.nn.LSTM(D, H).double()
    with torch.no_grad():
        lstm.weight_ih_l0.copy_(_to_torch_blocks(w_x.detach()))
        lstm.weight_hh_l0.copy_(_to_torch_blocks(w_h.detach()))
        lstm.bias_ih_l0.copy_(_to_torch_blocks(b.detach()))
        lstm.bias_hh_l0.zero_()
    x2 = x.detach().clone().requires_grad_(True)
    h02 = h0.detach().clone().requires_grad_(True)
    c02 = c0.detach().clone().requires_grad_(True)
    packed = pack_padded_sequence(x2, lengths.long(), enforce_sorted=False)
    _, (hn, cn) = lstm(packed, (h02.unsqueeze(0), c02.unsqueeze(0)))
    assert torch.allclose(hT, hn[0], atol=1e-12) and torch.allclose(cT, cn[0], atol=1e-12)

    gh, gc = torch.randn(B, H, dtype=torch.float64), torch.randn(B, H, dtype=torch.float64)
    ((hT * gh).sum() + (cT * gc).sum()).backward()
    ((hn[0] * gh).sum() + (cn[0] * gc).sum()).backward()
    assert torch.allclose(x.grad, x2.grad, atol=1e-12)
    assert torch.allclose(h0.grad, h02.grad, atol=1e-12) and torch.allclose(c0.grad, c02.grad, atol=1e-12)
    assert torch.allclose(_to_torch_blocks(w_x.grad), lstm.weight_ih_l0.grad, atol=1e-12)
    assert torch.allclose(_to_torch_blocks(w_h.grad), lstm.weight_hh_l0.grad, atol=1e-12)
    assert torch.allclose(_to_torch_blocks(b.grad), lstm.bias_ih_l0.grad, atol=1e-12)
    assert torch.allclose(_to_torch_blocks(b.grad), lstm.bias_hh_l0.grad, atol=1e-12)
    pad = torch.arange(T).view(T, 1) >= lengths.view(1, B)
    assert float(x.grad[pad].abs().max()) == 0.0                  # padded inputs get no gradient


def test_masked_reference_gradcheck():
    torch.manual_seed(1)
    T, B, D, H = 4, 3, 2, 3
    lengths = torch.tensor([4, 1, 2], dtype=torch.int32)
    args = [torch.randn(T, B, D), torch.randn(B, H) * 0.5, torch.randn(B, H) * 0.5, torch.randn(4 * H, D) * 0.5,
            torch.randn(4 * H, H) * 0.5, torch.randn(4 * H) * 0.1]
    args = [a.double().requires_grad_(True) for a in args]

    def f(*a):
        hs, hT, cT = ref.lstm_layer_sequence(*a, lengths=lengths)
        return hs, hT, cT
    assert torch.autograd.gradcheck(f, args)


def test_masked_reference_holds_state_and_checks_lengths():
    torch.manual_seed(2)
    T, B, D, H = 5, 2, 3, 4
    p = [torch.randn(T, B, D), torch.randn(B, H), torch.randn(B, H), torch.randn(4 * H, D), torch.randn(4 * H, H), torch.randn(4 * H)]
    hs, hT, cT = ref.lstm_layer_sequence(*p, lengths=torch.tensor([2, 5], dtype=torch.int32))
    assert torch.equal(hs[1:, 0], hs[1:2, 0].expand(4, H)) and torch.equal(hT[0], hs[1, 0])     # carried after step 1
    hs_full, hT_full, cT_full = ref.lstm_layer_sequence(*p)
    hs_T, hT_T, cT_T = ref.lstm_layer_sequence(*p, lengths=torch.full((B,), T, dtype=torch.int32))
    assert torch.equal(hs_full, hs_T) and torch.equal(hT_full, hT_T) and torch.equal(cT_full, cT_T)
    for bad in (torch.tensor([0, 5], dtype=torch.int32), torch.tensor([1, 6], dtype=torch.int32), torch.tensor([1, 5])):
        with pytest.raises(ValueError):
            ref.lstm_layer_sequence(*p, lengths=bad)


def test_ragged_csv_rows_pad_and_validate():
    rows = [["1", "2", "3", "4", "0"], ["5", "6", "1"], ["7", "8", "9", "10", "11", "12", "2"]]
    x, y, l = D.process_batch_ragged(rows, seq_len=3, in_features=2)
    assert x.shape == (3, 3, 2) and x.dtype == np.float32 and l.dtype == np.int32
    assert l.tolist() == [2, 1, 3] and y.tolist() == [0, 1, 2]
    assert x[0].tolist() == [[1, 2], [3, 4], [0, 0]] and x[1].tolist() == [[5, 6], [0, 0], [0, 0]]
    with pytest.raises(ValueError, match="row 1"):
        D.process_batch_ragged([["1", "2", "0"], ["1", "2", "3", "1"]], seq_len=3, in_features=2)     # not whole steps
    with pytest.raises(ValueError, match="row 0"):
        D.process_batch_ragged([["1"] * 8 + ["0"]], seq_len=3, in_features=2)                       # longer than seq_len
    xn, _, _ = D.process_batch_ragged([["-1", "1", "0"], ["3", "5", "7", "1", "1"]], seq_len=3, in_features=2, normalize=True)
    # min / max over the real values only (-1 and 7): padding (0) neither takes part nor is rescaled
    assert np.allclose(xn[0, 0], [0.0, 0.25]) and np.allclose(xn[1, :2].ravel(), [0.5, 0.75, 1.0, 0.25])
    assert xn[0, 1:].tolist() == [[0, 0], [0, 0]] and xn[1, 2].tolist() == [0, 0]


def test_synthetic_lengths_are_additive_and_seeded():
    x0, y0 = D.synthetic_sequences(64, 12, 5, 3, seed=4)
    x1, y1, l1 = D.synthetic_sequences(64, 12, 5, 3, seed=4, variable_length=True)
    x2, y2, l2 = D.synthetic_sequences(64, 12, 5, 3, seed=4, variable_length=True)
    _, _, l3 = D.synthetic_sequences(64, 12, 5, 3, seed=5, variable_length=True)
    assert np.array_equal(y0, y1) and np.array_equal(l1, l2) and not np.array_equal(l1, l3)
    assert l1.dtype == np.int32 and l1.min() >= 3 and l1.max() <= 12
    pad = np.arange(12)[None, :] >= l1[:, None]
    assert np.array_equal(x1[~pad], x0[~pad]) and not x1[pad].any()
    # with the flag off the data is what it was before lengths existed (digest of the earlier output for seed 4)
    import hashlib
    assert hashlib.sha256(x0.tobytes() + y0.tobytes()).hexdigest() == \
        "84eec319f1c13265ffb051350a417cc9e8518f45a226b1c0338cdd3743d0b5aa"
    with pytest.raises(ValueError):
        Config(seq_len=1, variable_length=True).validate()


def test_device_shard_and_pinned_loader_carry_lengths():
    x, y, l = D.synthetic_sequences(40, 6, 3, 4, seed=0, variable_length=True)
    ds = D.DeviceShard(x.copy(), y.copy(), 8, "cpu", lengths=l.copy(), seed=3)
    pl = D.PinnedHostLoader(x.copy(), y.copy(), 8, "cpu", lengths=l.copy(), seed=3, depth=3)   # (permutes its arrays in place)
    assert len(pl.dev[0]) == 3
    for _ in range(12):                                          # across a reshuffle
        bx, by, bl = ds.next()
        px, py, pll = pl.next()
        assert torch.equal(bx, px) and torch.equal(by, py) and torch.equal(bl, pll) and bl.dtype == torch.int32
        for i in range(8):                                       # every length follows its row
            row = int(np.nonzero((x == bx[i].numpy()).all(axis=(1, 2)))[0][0])
            assert int(bl[i]) == int(l[row])
    out = (torch.empty(8, 6, 3), torch.empty(8, dtype=torch.int64), torch.empty(8, dtype=torch.int32))
    r = ds.next(out=out)
    assert r[2] is out[2]


@settings(max_examples=15, deadline=None)
@given(consumed=st.integers(0, 17), depth=st.integers(2, 4))
def test_pinned_loader_with_lengths_resumes_at_any_position(consumed, depth):
    x, y, l = D.synthetic_sequences(30, 5, 2, 3, seed=1, variable_length=True)
    a = D.PinnedHostLoader(x.copy(), y.copy(), 7, "cpu", lengths=l.copy(), seed=9, depth=depth)
    for _ in range(consumed):
        a.next()
    st_ = a.state_dict()
    want = [tuple(t.clone() for t in a.next()) for _ in range(6)]
    b = D.PinnedHostLoader(x.copy(), y.copy(), 7, "cpu", lengths=l.copy(), seed=9, depth=depth)
    b.load_state_dict(st_)
    got = [tuple(t.clone() for t in b.next()) for _ in range(6)]
    assert all(torch.equal(p, q) for w, g in zip(want, got) for p, q in zip(w, g))


def _ragged_csv(path, n=120, T=6, F=3, seed=0):
    x, y, l = D.synthetic_sequences(n, T, F, 3, seed=seed, variable_length=True)
    with open(path, "w") as f:
        for i in range(n):
            vals = x[i, :l[i]].ravel().tolist() + [int(y[i])]
            f.write(",".join(f"{v:.5f}" if isinstance(v, float) else str(v) for v in vals) + "\n")


def test_standalone_ragged_csv_trains_resumes_and_scores(tmp_path):
    from lstm_tensorspark_b200.trainer import run_job
    csv_path = str(tmp_path / "ragged.csv")
    _ragged_csv(csv_path)
    base = dict(training_path=csv_path, hidden_units="12", in_features=3, seq_len=6, num_classes=3, variable_length=True,
                batch_size=20, checkpoint_path=str(tmp_path / "ck"), output_path=str(tmp_path / "out"), device="cpu",
                quiet=True, learning_rate=2e-2, init="scaled", steps_mode="epochs", evaluate_every=5)
    out = run_job(Config(epochs=8, **base).validate(), standalone=True)
    res = out["results"][0]
    import json
    runs = os.listdir(base["checkpoint_path"])
    scal = [json.loads(s) for s in open(os.path.join(base["checkpoint_path"], runs[0], "train", "scalars.jsonl"))]
    assert scal[-1]["cross_entropy"] < scal[0]["cross_entropy"]                        # it learns
    out2 = run_job(Config(epochs=10, use_pretrained_model=True, **base).validate(), standalone=True)
    assert out2["results"][0]["steps"] == 12                                          # 60 total - 48 already done
    ev = run_job(Config(mode="eval", **dict(base, batch_size=50)).validate(), standalone=True)    # 2 full batches + a tail of 20
    assert ev["samples"] == 120 and np.isfinite(ev["loss"]) and ev["accuracy"] > 1 / 3
    assert res["steps"] == 48


def _grad_sync_check_ragged(rank, world):
    import torch.distributed as dist
    from lstm_tensorspark_b200.engine import TrainEngine
    from lstm_tensorspark_b200.parallel.comm import make_communicator
    dev = torch.device("cpu")
    comm = make_communicator("gloo", rank, world, dev, 60)
    cfg = Config(hidden_units="8,8", in_features=4, batch_size=6, seq_len=5, sync_mode="grad_allreduce", device="cpu",
                 learn_initial_state=False, init="scaled", partitions=world, variable_length=True)
    eng = TrainEngine(cfg, rank, world, comm, batch_size=6, device=dev, dtype=torch.float32)
    x, y, l = D.synthetic_sequences(6, 5, 4, 3, seed=rank, variable_length=True)
    for _ in range(4):
        eng.step(torch.as_tensor(x), torch.as_tensor(y), torch.as_tensor(l))
    all_w = [torch.zeros_like(eng.flat.data) for _ in range(world)]
    dist.all_gather(all_w, eng.flat.data)
    comm.close()
    return bool(all(torch.equal(all_w[0], w) for w in all_w))


def test_grad_allreduce_with_variable_length_keeps_replicas_identical():
    from lstm_tensorspark_b200.parallel.launch import launch
    assert launch(_grad_sync_check_ragged, 2) == [True, True]
