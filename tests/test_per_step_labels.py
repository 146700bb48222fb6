"""Per-step labels (sequence labelling) on the CPU: the reference semantics against nn.LSTM + nn.Linear + F.cross_entropy on the
packed outputs in fp64 (loss and every gradient; fixed, ragged, bidirectional and dropout), the CSV format and the rows it
rejects, both loaders with [B,T] labels including resume, the flag's errors, the standalone CLI (train, resume, position-weighted
eval) and a 2-rank gloo run."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as Fn

from lstm_tensorspark_b200 import data as D
from lstm_tensorspark_b200.config import Config
from lstm_tensorspark_b200.ops import reference as ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _blocks(w):
    """Gate-interleaved rows (n = 4 j + g) -> torch's [i; f; g; o] blocks."""
    H = w.shape[0] // 4
    return w.view(H, 4, *w.shape[1:]).transpose(0, 1).reshape(w.shape)


def _model(bidirectional, dropout, lengths, T=6, B=5, D_=3, H=4, C=3, seed=0):
    """A 2-layer SequenceClassifier (fp64, CPU reference path) and the same weights in nn.LSTM + nn.Linear."""
    from lstm_tensorspark_b200.models.classifier import SequenceClassifier
    from lstm_tensorspark_b200.ops import functional as F
    F.set_backend("torch")
    cfg = Config(hidden_units=f"{H},{H}", in_features=D_, seq_len=T, batch_size=B, num_classes=C, bidirectional=bidirectional,
                 dropout=dropout, per_step_labels=True, learn_initial_state=False, init="scaled", device="cpu",
                 variable_length=lengths is not None)
    g = torch.Generator().manual_seed(seed)
    m = SequenceClassifier(cfg, batch_size=B, device="cpu", generator=g).double()
    m.compute_dtype = torch.float64
    lstm = torch.nn.LSTM(D_, H, num_layers=2, bidirectional=bidirectional).double()
    dirs = m.rnn.directions()
    with torch.no_grad():
        for k, lay in enumerate(dirs):
            l, suf = (k // 2, "_reverse" if k % 2 else "") if bidirectional else (k, "")
            getattr(lstm, f"weight_ih_l{l}{suf}").copy_(_blocks(lay.w_x))
            getattr(lstm, f"weight_hh_l{l}{suf}").copy_(_blocks(lay.w_h))
            getattr(lstm, f"bias_ih_l{l}{suf}").copy_(_blocks(lay.bias))
            getattr(lstm, f"bias_hh_l{l}{suf}").zero_()
    lin = torch.nn.Linear(m.head.weights.shape[0], C).double()
    with torch.no_grad():
        lin.weight.copy_(m.head.weights.t())
        lin.bias.copy_(m.head.bias)
    return m, lstm, lin, dirs


@pytest.mark.parametrize("bidirectional,ragged", [(False, False), (False, True), (True, True)])
def test_reference_matches_nn_lstm_linear_cross_entropy_fp64(bidirectional, ragged):
    from torch.nn.utils.rnn import pack_padded_sequence
    T, B, C = 6, 5, 3
    lengths = torch.tensor([6, 1, 3, 6, 2], dtype=torch.int32) if ragged else None
    m, lstm, lin, dirs = _model(bidirectional, 0.0, lengths)
    g = torch.Generator().manual_seed(1)
    x = torch.randn(B, T, 3, generator=g, dtype=torch.float64)
    y = torch.randint(0, C, (B, T), generator=g)
    loss, logits, correct = m(x, y, lengths)
    loss.backward()
    lt = lengths.long() if ragged else torch.full((B,), T)
    packed = pack_padded_sequence(x.transpose(0, 1), lt, enforce_sorted=False)
    out, _ = lstm(packed)
    ylab = pack_padded_sequence(y.t(), lt, enforce_sorted=False).data
    want = Fn.cross_entropy(lin(out.data), ylab)
    want.backward()
    assert abs(float(loss) - float(want)) < 1e-12
    assert int(correct) == int((lin(out.data).argmax(1) == ylab).sum())
    assert logits.shape == (B, T, C)
    assert torch.allclose(m.head.weights.grad, lin.weight.grad.t(), atol=1e-12)
    assert torch.allclose(m.head.bias.grad, lin.bias.grad, atol=1e-12)
    for k, lay in enumerate(dirs):
        l, suf = (k // 2, "_reverse" if k % 2 else "") if bidirectional else (k, "")
        assert torch.allclose(_blocks(lay.w_x.grad), getattr(lstm, f"weight_ih_l{l}{suf}").grad, atol=1e-12), lay.node_name
        assert torch.allclose(_blocks(lay.w_h.grad), getattr(lstm, f"weight_hh_l{l}{suf}").grad, atol=1e-12), lay.node_name
        assert torch.allclose(_blocks(lay.bias.grad), getattr(lstm, f"bias_hh_l{l}{suf}").grad, atol=1e-12), lay.node_name


def test_reference_with_dropout_matches_hand_composed_masks_fp64():
    """Dropout 0.4 between the layers: the first layer's output times reference.dropout_mask x scale feeds layer 2; the top
    layer's output is not dropped."""
    T, B, C, H = 6, 5, 3, 4
    m, _lstm, _lin, dirs = _model(False, 0.4, None)
    m.rnn.dropout_key, m.rnn.dropout_step = (7, 1), 3
    g = torch.Generator().manual_seed(2)
    x = torch.randn(B, T, 3, generator=g, dtype=torch.float64)
    y = torch.randint(0, C, (B, T), generator=g)
    loss, _, _ = m(x, y)
    loss.backward()
    got = [p.grad.clone() for p in m.parameters()]
    ps = [p.detach().clone().requires_grad_(True) for p in (dirs[0].w_x, dirs[0].w_h, dirs[0].bias, dirs[1].w_x, dirs[1].w_h,
                                                              dirs[1].bias, m.head.weights, m.head.bias)]
    z = torch.zeros(B, H, dtype=torch.float64)
    h1, _, _ = ref.lstm_layer_sequence(x.transpose(0, 1), z, z, *ps[:3])
    spec = ref.DropoutSpec(0.4, (7, 1), 0, False, 3)
    h1 = h1 * ref.dropout_mask(spec, T, B, H).double() * ref.dropout_scale(0.4).double()
    h2, _, _ = ref.lstm_layer_sequence(h1, z, z, *ps[3:6])
    want = Fn.cross_entropy((h2 @ ps[6] + ps[7]).reshape(-1, C), y.t().reshape(-1))
    want.backward()
    assert abs(float(loss) - float(want)) < 1e-12
    byid = {id(p): gr for p, gr in zip(m.parameters(), got)}
    for p, q in zip((dirs[0].w_x, dirs[0].w_h, dirs[0].bias, dirs[1].w_x, dirs[1].w_h, dirs[1].bias, m.head.weights,
                     m.head.bias), ps):
        assert torch.allclose(byid[id(p)], q.grad, atol=1e-12)


def test_op_never_reads_uncounted_labels_and_counts_positions():
    T, B, C = 4, 3, 5
    h = torch.randn(T, B, 6, dtype=torch.float64)
    W, b = torch.randn(6, C, dtype=torch.float64), torch.randn(C, dtype=torch.float64)
    lengths = torch.tensor([4, 1, 2], dtype=torch.int32)
    y = torch.randint(0, C, (B, T))
    y2 = y.clone()
    y2[1, 1:] = 10 ** 6                                  # garbage at uncounted positions
    y2[2, 2:] = -5
    a = ref.head_xent_per_step(h, W, b, y, lengths)
    c = ref.head_xent_per_step(h, W, b, y2, lengths)
    assert int(a[3]) == 7 and torch.equal(a[1], c[1]) and int(a[2]) == int(c[2])


# ---- CSV -----------------------------------------------------------------------------------------------------------------------
def test_csv_rows_fixed_and_ragged():
    rows = [["1", "2", "3", "4", "0", "2"], ["5", "6", "7", "8", "1", "1"]]          # 2 steps of 2 features, 2 labels
    x, y = D.process_batch_per_step(rows, 2, 2, 3)
    assert x.shape == (2, 2, 2) and y.tolist() == [[0, 2], [1, 1]] and x[1, 1].tolist() == [7, 8]
    rows = [["1", "2", "3", "4", "0", "2"], ["5", "6", "1"]]
    x, y, l = D.process_batch_per_step(rows, 3, 2, 3, variable_length=True, normalize=True)
    assert x.shape == (2, 3, 2) and l.tolist() == [2, 1] and y.tolist() == [[0, 2, 0], [1, 0, 0]]
    assert x.max() == 1.0 and x[0, 0, 0] == 0.0 and x[1, 1:].sum() == 0                # normalised features only, padding 0


@pytest.mark.parametrize("rows,kw,msg", [
    ([["1", "2", "3", "4", "0"]], {}, "row 0"),                                       # does not split into steps + labels
    ([["1", "2", "0"]], {}, "row 0"),                                                 # one step where seq_len = 2 (fixed)
    ([["1", "2", "3", "4", "0", "1"], ["1", "2", "3", "4", "0", "3"]], {}, "row 1: label 3"),
    ([["1", "2", "-1"]], {"variable_length": True}, "row 0: label -1"),
    ([["1", "2", "3", "4", "5", "6", "0", "0", "0"]], {"variable_length": True}, "row 0"),   # 3 steps > seq_len
])
def test_csv_rejects(rows, kw, msg):
    with pytest.raises(ValueError, match=msg):
        D.process_batch_per_step(rows, 2, 2, 3, **kw)


def test_synthetic_per_step_is_seeded_and_leaves_the_old_draws_alone():
    a = D.synthetic_sequences(10, 5, 3, 4, seed=2)
    x, y = D.synthetic_per_step(10, 5, 3, 4, seed=2)
    b = D.synthetic_sequences(10, 5, 3, 4, seed=2)
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
    assert y.shape == (10, 5) and y.dtype == np.int64 and np.array_equal(x, D.synthetic_per_step(10, 5, 3, 4, seed=2)[0])
    x, y, l = D.synthetic_per_step(10, 8, 3, 4, seed=2, variable_length=True)
    assert np.array_equal(l, D.synthetic_lengths(10, 8, 2))
    pad = np.arange(8)[None, :] >= l[:, None]
    assert not x[pad].any() and not y[pad].any()


# ---- loaders -------------------------------------------------------------------------------------------------------------------
def test_loaders_carry_per_step_labels_and_resume():
    x, y, l = D.synthetic_per_step(40, 6, 3, 4, seed=0, variable_length=True)
    ds = D.DeviceShard(x.copy(), y.copy(), 8, "cpu", lengths=l.copy(), seed=3)
    pl = D.PinnedHostLoader(x.copy(), y.copy(), 8, "cpu", lengths=l.copy(), seed=3, depth=3)
    assert pl.dev[0][1].shape == (8, 6) and pl.bytes_per_batch == 8 * 6 * 3 * 4 + 8 * 6 * 8 + 8 * 4
    for _ in range(7):
        a, b = ds.next(), pl.next()
        assert all(torch.equal(p, q) for p, q in zip(a, b)) and a[1].shape == (8, 6)
    for loader_cls in (D.DeviceShard, D.PinnedHostLoader):
        kw = {"depth": 3} if loader_cls is D.PinnedHostLoader else {}
        first = loader_cls(x.copy(), y.copy(), 8, "cpu", lengths=l.copy(), seed=5, **kw)
        for _ in range(6):
            first.next()
        st = first.state_dict()
        want = [tuple(t.clone() for t in first.next()) for _ in range(5)]
        second = loader_cls(x.copy(), y.copy(), 8, "cpu", lengths=l.copy(), seed=5, **kw)
        second.load_state_dict(st)
        got = [tuple(t.clone() for t in second.next()) for _ in range(5)]
        assert all(torch.equal(p, q) for w, g in zip(want, got) for p, q in zip(w, g)), loader_cls.__name__


# ---- flag --------------------------------------------------------------------------------------------------------------------
def test_config_and_label_shape_errors():
    from lstm_tensorspark_b200.engine import TrainEngine
    with pytest.raises(ValueError, match="--per_step_labels"):
        Config(per_step_labels=True, seq_len=1).validate()
    from lstm_tensorspark_b200.config import parse_args
    assert parse_args(["--per_step_labels", "--seq_len", "4"]).per_step_labels
    assert not parse_args(["--seq_len", "4"]).per_step_labels
    x = torch.randn(4, 5, 3)
    for flag, y in ((True, torch.zeros(4, dtype=torch.int64)), (False, torch.zeros(4, 5, dtype=torch.int64))):
        cfg = Config(hidden_units="6", in_features=3, seq_len=5, batch_size=4, per_step_labels=flag, device="cpu")
        eng = TrainEngine(cfg, 0, 1, None, batch_size=4)
        with pytest.raises(ValueError, match="--per_step_labels"):
            eng.step(x, y)


# ---- CLI --------------------------------------------------------------------------------------------------------------------
def _csv(path, n=120, T=6, F=3, ragged=False, seed=0):
    data = D.synthetic_per_step(n, T, F, 3, seed=seed, variable_length=ragged)
    x, y = data[0], data[1]
    l = data[2] if ragged else np.full(n, T)
    with open(path, "w") as f:
        for i in range(n):
            vals = [f"{v:.5f}" for v in x[i, :l[i]].ravel()] + [str(int(v)) for v in y[i, :l[i]]]
            f.write(",".join(vals) + "\n")
    return l


@pytest.mark.parametrize("ragged", [False, True])
def test_cli_trains_resumes_and_scores_by_position(tmp_path, ragged):
    from lstm_tensorspark_b200.trainer import run_job
    csv_path = str(tmp_path / "steps.csv")
    lengths = _csv(csv_path, ragged=ragged)
    base = dict(training_path=csv_path, hidden_units="12", in_features=3, seq_len=6, num_classes=3, per_step_labels=True,
                variable_length=ragged, batch_size=20, checkpoint_path=str(tmp_path / "ck"), output_path=str(tmp_path / "out"),
                device="cpu", quiet=True, learning_rate=2e-2, init="scaled", steps_mode="epochs", evaluate_every=5)
    flags = [f"--{k}={v}" for k, v in dict(base, epochs=8).items()]
    r = subprocess.run([sys.executable, os.path.join(ROOT, "lstm-no-spark.py")] + flags, capture_output=True, text=True,
                       timeout=600, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-3000:]
    runs = os.listdir(base["checkpoint_path"])
    scal = [json.loads(s) for s in open(os.path.join(base["checkpoint_path"], runs[0], "train", "scalars.jsonl"))]
    assert scal[-1]["cross_entropy"] < scal[0]["cross_entropy"]                     # it learns
    out2 = run_job(Config(epochs=10, use_pretrained_model=True, **base).validate(), standalone=True)
    assert out2["results"][0]["steps"] == 12                                       # 60 total - 48 already done
    ev = run_job(Config(mode="eval", **dict(base, batch_size=50)).validate(), standalone=True)   # 2 full batches + a tail of 20
    assert ev["samples"] == 120 and ev["positions"] == int(lengths.sum())
    # position-weighted: the whole-file numbers equal one pass over every counted position
    from lstm_tensorspark_b200.engine import TrainEngine
    from lstm_tensorspark_b200.trainer import _find_trained_model
    cfg = Config(mode="eval", **dict(base, batch_size=120)).validate()
    eng = TrainEngine(cfg, 0, 1, None, batch_size=120)
    eng.model.load_reference_state_dict(_find_trained_model(cfg, True)[0], strict=False)
    data = D.process_batch_per_step(D.read_dataset_from_path(csv_path), 6, 3, 3, variable_length=ragged)
    loss, acc = eng.evaluate(torch.as_tensor(data[0]), torch.as_tensor(data[1]),
                             torch.as_tensor(data[2]) if ragged else None)
    assert abs(ev["loss"] - float(loss)) < 1e-5 and abs(ev["accuracy"] - float(acc)) < 1e-6
    assert ev["accuracy"] > 1 / 3


def _grad_sync_check(rank, world):
    import torch.distributed as dist
    from lstm_tensorspark_b200.engine import TrainEngine
    from lstm_tensorspark_b200.parallel.comm import make_communicator
    dev = torch.device("cpu")
    comm = make_communicator("gloo", rank, world, dev, 60)
    cfg = Config(hidden_units="8,8", in_features=4, batch_size=6, seq_len=5, sync_mode="grad_allreduce", device="cpu",
                 learn_initial_state=False, init="scaled", partitions=world, variable_length=True, per_step_labels=True)
    eng = TrainEngine(cfg, rank, world, comm, batch_size=6, device=dev, dtype=torch.float32)
    x, y, l = D.synthetic_per_step(6, 5, 4, 3, seed=rank, variable_length=True)
    for _ in range(4):
        eng.step(torch.as_tensor(x), torch.as_tensor(y), torch.as_tensor(l))
    all_w = [torch.zeros_like(eng.flat.data) for _ in range(world)]
    dist.all_gather(all_w, eng.flat.data)
    comm.close()
    return bool(all(torch.equal(all_w[0], w) for w in all_w))


def test_two_rank_grad_allreduce_keeps_replicas_identical():
    from lstm_tensorspark_b200.parallel.launch import launch
    assert launch(_grad_sync_check, 2) == [True, True]
