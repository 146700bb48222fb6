"""Token embedding in front of the first layer (``--vocab_size``), on the CPU: the flags, the three CSV row formats and their
errors, the synthetic token task, initial weights, the reference op against ``torch.nn.functional.embedding``, checkpoints and
their refusals, the loaders and two gloo ranks."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from lstm_tensorspark_b200 import data as D
from lstm_tensorspark_b200.config import Config

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---- flags -------------------------------------------------------------------------------------------------------------------
def test_flag_validation():
    assert Config().vocab_size == 0
    with pytest.raises(ValueError, match="--vocab_size"):
        Config(vocab_size=-1).validate()
    with pytest.raises(ValueError, match="--normalize.*--vocab_size"):
        Config(vocab_size=10, normalize=True).validate()
    Config(vocab_size=10, seq_len=4, pooling="attention").validate()
    from lstm_tensorspark_b200.config import parse_args
    assert parse_args(["--vocab_size", "7"]).vocab_size == 7


# ---- CSV rows ------------------------------------------------------------------------------------------------------------------
def test_fixed_rows():
    x, y = D.process_tokens([["1", "2", "3", "0"], ["4", "5", "6", "2"], []], 3, 10)
    assert x.dtype == np.int32 and x.tolist() == [[1, 2, 3], [4, 5, 6]] and y.tolist() == [0, 2]
    x1, y1 = D.process_tokens([["7", "1"], ["0", "0"]], 1, 10)           # one step: [N] ids
    assert x1.shape == (2,) and x1.tolist() == [7, 0] and y1.tolist() == [1, 0]


def test_ragged_rows():
    x, y, l = D.process_tokens([["1", "2"], ["3", "4", "5", "1"]], 4, 10, variable_length=True)
    assert x.tolist() == [[1, 0, 0, 0], [3, 4, 5, 0]] and y.tolist() == [2, 1] and l.tolist() == [1, 3]
    assert l.dtype == np.int32


def test_per_step_rows():
    x, y = D.process_tokens([["1", "2", "0", "1"]], 2, 10, num_classes=2, per_step_labels=True)
    assert x.tolist() == [[1, 2]] and y.tolist() == [[0, 1]]
    x, y, l = D.process_tokens([["3", "1"], ["1", "2", "3", "0", "1", "1"]], 3, 10, num_classes=2, variable_length=True,
                               per_step_labels=True)
    assert x.tolist() == [[3, 0, 0], [1, 2, 3]] and y.tolist() == [[1, 0, 0], [0, 1, 1]] and l.tolist() == [1, 3]


@pytest.mark.parametrize("rows,kw,match", [
    ([["1", "2", "0"], ["1", "x", "0"]], {}, "row 1: token id 'x' is not an integer"),
    ([["1", "2.5", "0"]], {}, "row 0: token id '2.5'"),
    ([["1", "10", "0"]], {}, r"row 0: token id 10 outside \[0, 10\)"),
    ([["1", "-1", "0"]], {}, r"row 0: token id -1 outside"),
    ([["1", "2", "0"], ["1", "0"]], {}, "row 1: 2 fields is not 2 token ids"),
    ([["1", "2", "3", "4", "0"]], {"variable_length": True}, "row 0: 5 fields is not 1..2 token ids"),
    ([["1", "2", "0"]], {"per_step_labels": True, "num_classes": 2}, "row 0: 3 fields is not 2 token ids followed by one label"),
    ([["1", "2", "0", "5"]], {"per_step_labels": True, "num_classes": 2}, r"row 0: label 5 outside \[0, 2\)"),
])
def test_row_errors(rows, kw, match):
    with pytest.raises(ValueError, match=match):
        D.process_tokens(rows, 2, 10, **kw)


# ---- the synthetic task --------------------------------------------------------------------------------------------------------
def test_synthetic_tokens():
    before = D.synthetic_sequences(16, 5, 3, 3, seed=4, variable_length=True)
    x, y, l = D.synthetic_tokens(400, 6, 50, 3, seed=4, variable_length=True)
    assert x.dtype == np.int32 and x.shape == (400, 6) and 0 <= x.min() and x.max() < 50 and y.shape == (400,)
    assert (x[np.arange(6)[None, :] >= l[:, None]] == 0).all()
    xs, ys = D.synthetic_tokens(200, 4, 20, 2, seed=1, per_step_labels=True)
    assert ys.shape == (200, 4) and xs.max() < 20
    x1, _ = D.synthetic_tokens(10, 1, 5, 2)
    assert x1.shape == (10,)
    # a generator of its own: the feature draws are those of before
    after = D.synthetic_sequences(16, 5, 3, 3, seed=4, variable_length=True)
    assert all(np.array_equal(a, b) for a, b in zip(before, after))
    assert np.array_equal(np.asarray(D.synthetic_lengths(400, 6, 4)), l)


def test_loss_falls_on_the_synthetic_task():
    from lstm_tensorspark_b200.engine import TrainEngine
    cfg = Config(hidden_units="16", in_features=8, seq_len=6, batch_size=32, num_classes=3, partitions=1, sync_mode="none",
                 vocab_size=40, device="cpu", quiet=True, variable_length=True, learning_rate=1e-2, init="scaled")
    eng = TrainEngine(cfg, 0, 1, None, batch_size=32)
    x, y, l = (torch.as_tensor(a) for a in D.synthetic_tokens(128, 6, 40, 3, seed=0, variable_length=True))
    losses = [float(eng.step(x[i % 4 * 32:][:32], y[i % 4 * 32:][:32], l[i % 4 * 32:][:32])) for i in range(60)]
    assert np.mean(losses[-8:]) < 0.5 * np.mean(losses[:4])


# ---- model ---------------------------------------------------------------------------------------------------------------------
def _fresh(vocab, bidirectional=False, pooling="last", init="truncated_normal"):
    from lstm_tensorspark_b200.models.classifier import SequenceClassifier
    cfg = Config(hidden_units="6,5", in_features=3, seq_len=4, batch_size=2, num_classes=3, bidirectional=bidirectional,
                 init=init, device="cpu", init_std=0.5, pooling=pooling, attention_units=4, vocab_size=vocab)
    return SequenceClassifier(cfg, batch_size=2, device="cpu", generator=torch.Generator().manual_seed(11))


@pytest.mark.parametrize("bidirectional,pooling,init", [(False, "last", "truncated_normal"), (True, "attention", "scaled")])
def test_initial_weights_of_everything_else_unchanged(bidirectional, pooling, init):
    off = _fresh(0, bidirectional, pooling, init).reference_state_dict()
    on = _fresh(9, bidirectional, pooling, init).reference_state_dict()
    assert list(on) == list(off) + ["Embedding/weights"]
    assert all(torch.equal(on[k], off[k]) for k in off)
    tab = on["Embedding/weights"]
    assert tab.shape == (9, 3) and float(tab.abs().max()) <= 1.0 and float(tab.std()) > 0.1   # std init_std under both inits


def test_reference_op_against_torch_embedding():
    from lstm_tensorspark_b200.ops import reference as ref
    g = torch.Generator().manual_seed(0)
    V, E, B, T = 7, 5, 4, 6
    table = torch.randn(V, E, generator=g, dtype=torch.float64, requires_grad=True)
    tok = torch.randint(-2, V + 2, (B, T), generator=g)
    lengths = torch.tensor([1, 6, 3, 4], dtype=torch.int32)
    x = ref.embedding(tok, table, lengths)
    keep = (tok.t() >= 0) & (tok.t() < V) & (torch.arange(T)[:, None] < lengths[None, :].long())
    want = torch.nn.functional.embedding(tok.t().clamp(0, V - 1), table) * keep.unsqueeze(2)
    assert x.shape == (T, B, E) and torch.equal(x, want)
    dx = torch.randn(T, B, E, generator=g, dtype=torch.float64)
    x.backward(dx)
    dW = torch.zeros(V, E, dtype=torch.float64)
    for t in range(T):
        for b in range(B):
            if keep[t, b]:
                dW[tok[b, t]] += dx[t, b]
    assert torch.allclose(table.grad, dW, rtol=0, atol=1e-12)
    x1 = ref.embedding(torch.tensor([2, 9]), table)                    # one step, an id out of range
    assert x1.shape == (1, 2, E) and torch.equal(x1[0, 0], table[2]) and float(x1[0, 1].detach().abs().sum()) == 0


def test_model_reads_ids_and_rejects_floats():
    m = _fresh(9)
    with pytest.raises(ValueError, match="--vocab_size needs integer token ids"):
        m.features(torch.zeros(2, 4, 3))
    assert m.features(torch.zeros(2, 4, dtype=torch.int64)).shape == (2, 5)


# ---- checkpoints and the CLI ---------------------------------------------------------------------------------------------------
def _base(tmp_path, **kw):
    return dict(dict(synthetic=120, hidden_units="12", in_features=6, seq_len=6, num_classes=3, variable_length=True,
                     batch_size=20, checkpoint_path=str(tmp_path / "ck"), output_path=str(tmp_path / "out"), device="cpu",
                     quiet=True, learning_rate=2e-2, init="scaled", steps_mode="epochs", evaluate_every=5, vocab_size=30), **kw)


def test_cli_trains_resumes_and_evaluates(tmp_path):
    import json
    from lstm_tensorspark_b200.trainer import run_job
    base = _base(tmp_path)
    flags = [f"--{k}={v}" for k, v in dict(base, epochs=8).items()]
    r = subprocess.run([sys.executable, os.path.join(ROOT, "lstm-no-spark.py")] + flags, capture_output=True, text=True,
                       timeout=600, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-3000:]
    runs = os.listdir(base["checkpoint_path"])
    scal = [json.loads(s) for s in open(os.path.join(base["checkpoint_path"], runs[0], "train", "scalars.jsonl"))]
    assert scal[-1]["cross_entropy"] < scal[0]["cross_entropy"]
    out2 = run_job(Config(epochs=10, use_pretrained_model=True, **base).validate(), standalone=True)
    assert out2["results"][0]["steps"] == 12
    assert out2["results"][0]["variables"]["Embedding/weights"].shape == (30, 6)
    ev = run_job(Config(mode="eval", **dict(base, batch_size=50)).validate(), standalone=True)
    assert ev["samples"] == 120 and ev["accuracy"] > 1 / 3


@pytest.mark.parametrize("written,loaded", [(30, 0), (0, 30), (30, 31)])
def test_checkpoint_with_another_vocabulary_is_refused(tmp_path, written, loaded):
    from lstm_tensorspark_b200.trainer import run_job
    run_job(Config(epochs=1, max_steps=2, **_base(tmp_path, vocab_size=written)).validate(), standalone=True)
    with pytest.raises(ValueError, match=f"--vocab_size {written}.*--vocab_size {loaded}"):
        run_job(Config(epochs=1, max_steps=3, use_pretrained_model=True, **_base(tmp_path, vocab_size=loaded)).validate(),
                standalone=True)
    with pytest.raises(ValueError, match="--vocab_size"):
        run_job(Config(mode="eval", **_base(tmp_path, vocab_size=loaded)).validate(), standalone=True)


def test_averaged_model_records_vocab_and_eval_never_averages_table_rows(tmp_path):
    from lstm_tensorspark_b200.models.classifier import SequenceClassifier
    from lstm_tensorspark_b200.trainer import run_job
    base = _base(tmp_path, partitions=2, max_workers=1, epochs=1, max_steps=2)
    run_job(Config(**base).validate(), standalone=False)
    path = os.path.join(base["output_path"], "averaged_model.pt")
    blob = torch.load(path, weights_only=False)
    assert blob["meta"]["vocab_size"] == 30 and blob["variables"]["Embedding/weights"].shape == (30, 6)
    ev = run_job(Config(mode="eval", **dict(base, partitions=1)).validate(), standalone=False)
    assert ev["samples"] == 120
    with pytest.raises(ValueError, match="--vocab_size 30.*--vocab_size 20"):
        run_job(Config(mode="eval", **dict(base, partitions=1, vocab_size=20)).validate(), standalone=False)
    # a file without a recorded vocabulary: the table's rows are its vocabulary, never averaged to fit another one
    blob["meta"].pop("vocab_size")
    torch.save(blob, path)
    with pytest.raises(ValueError, match="--vocab_size 30.*--vocab_size 20"):
        run_job(Config(mode="eval", resume=path, **dict(base, partitions=1, vocab_size=20)).validate(), standalone=False)
    m = SequenceClassifier(Config(**dict(base, vocab_size=0)), device="cpu")
    with pytest.raises(ValueError, match="without an Embedding/weights table"):
        SequenceClassifier(Config(**base), device="cpu").check_vocab(m.reference_state_dict(), 30)


# ---- loaders -------------------------------------------------------------------------------------------------------------------
def test_loaders_keep_int32_and_the_batch_order():
    """The same seed draws the same rows for token ids as for float features (labels = row numbers identify them)."""
    x, _, l = D.synthetic_tokens(40, 5, 17, 3, seed=2, variable_length=True)
    xf, _ = D.synthetic_sequences(40, 5, 2, 3, seed=2)
    y = np.arange(40, dtype=np.int64)
    for cls in (D.DeviceShard, D.PinnedHostLoader):
        # (copies: the pinned loader permutes its host arrays in place)
        tok = cls(x.copy(), y.copy(), 8, "cpu", dtype=torch.int32, seed=3, lengths=l.copy())
        flt = cls(xf.copy(), y.copy(), 8, "cpu", dtype=torch.float32, seed=3, lengths=l.copy())
        for _ in range(12):                                              # across reshuffles
            bt, bf = tok.next(), flt.next()
            assert bt[0].dtype == torch.int32 and torch.equal(bt[1], bf[1]) and torch.equal(bt[2], bf[2])
            assert np.array_equal(bt[0].numpy(), x[bt[1].numpy()]) and np.array_equal(bf[0].numpy(), xf[bf[1].numpy()])
    pl = D.PinnedHostLoader(x.copy(), y.copy(), 8, "cpu", dtype=torch.int32, seed=3, lengths=l.copy())
    assert pl.bytes_per_batch == 8 * 5 * 4 + 8 * 8 + 8 * 4


# ---- two ranks -----------------------------------------------------------------------------------------------------------------
def _sync_check(rank, world):
    import torch.distributed as dist
    from lstm_tensorspark_b200.engine import TrainEngine
    from lstm_tensorspark_b200.parallel.comm import make_communicator
    dev = torch.device("cpu")
    comm = make_communicator("gloo", rank, world, dev, 60)
    cfg = Config(hidden_units="8,8", in_features=4, batch_size=6, seq_len=5, sync_mode="grad_allreduce", device="cpu",
                 learn_initial_state=False, init="scaled", partitions=world, variable_length=True, vocab_size=11,
                 clip_grad_norm=1.0)
    eng = TrainEngine(cfg, rank, world, comm, batch_size=6, device=dev, dtype=torch.float32)
    x, y, l = D.synthetic_tokens(6, 5, 11, 3, seed=rank, variable_length=True)
    start = eng.model.embedding.weights.detach().clone()
    for _ in range(4):
        eng.step(torch.as_tensor(x), torch.as_tensor(y), torch.as_tensor(l))
    moved = not torch.equal(start, eng.model.embedding.weights)
    all_w = [torch.zeros_like(eng.flat.data) for _ in range(world)]
    dist.all_gather(all_w, eng.flat.data)
    comm.close()
    return moved and all(torch.equal(all_w[0], w) for w in all_w)


def test_two_ranks_grad_allreduce_end_with_identical_tables():
    from lstm_tensorspark_b200.parallel.launch import launch
    assert all(launch(_sync_check, 2, args=()))


@pytest.mark.parametrize("kw", [dict(per_step_labels=True), dict(pooling="attention", attention_units=5),
                                dict(bidirectional=True, dropout=0.2)])
def test_combines_with_per_step_labels_pooling_and_bidirectional(kw):
    """Token batches through the other sequence features: the table gets a gradient and the loss falls."""
    from lstm_tensorspark_b200.engine import TrainEngine
    cfg = Config(hidden_units="12,12", in_features=6, seq_len=5, batch_size=16, num_classes=3, partitions=1, sync_mode="none",
                 vocab_size=25, device="cpu", quiet=True, variable_length=True, learning_rate=2e-2, init="scaled", **kw)
    eng = TrainEngine(cfg, 0, 1, None, batch_size=16)
    x, y, l = (torch.as_tensor(a) for a in D.synthetic_tokens(16, 5, 25, 3, seed=3, variable_length=True,
                                                              per_step_labels=cfg.per_step_labels))
    start = eng.model.embedding.weights.detach().clone()
    losses = [float(eng.step(x, y, l)) for _ in range(40)]
    assert not torch.equal(start, eng.model.embedding.weights) and losses[-1] < 0.7 * losses[0]
