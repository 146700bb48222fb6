"""Unit tests for the flag system and the data layer (: sharder, process_batch, next_batch, normaliser,
flag defaults, net_settings)."""
import numpy as np
import pytest
import torch

from lstm_tensorspark_b200 import data as D
from lstm_tensorspark_b200.config import Config, parse_args


def test_reference_flag_defaults():
    cfg = parse_args([], standalone=False)
    # original src/rnn.py:310-334
    assert (cfg.master, cfg.spark_exec_memory, cfg.partitions, cfg.epochs) == ("local", "4g", 4, 1)
    assert (cfg.hidden_units, cfg.batch_size, cfg.num_classes, cfg.in_features) == ("128,256", 10, 3, 4)
    assert cfg.learning_rate == pytest.approx(1e-3) and cfg.evaluate_every == 10
    assert (cfg.training_path, cfg.labels_path, cfg.output_path) == ("train", "train_labels", "output_path")
    assert cfg.mode == "train" and cfg.checkpoint_path == "train_dir"


def test_standalone_defaults_and_unknown_args_ignored():
    cfg = parse_args(["--bogus", "1", "--hidden_units=16"], standalone=True)
    assert cfg.epochs == 5                      # original src/lstm-no-spark.py:12
    assert cfg.partitions == 1 and cfg.hidden_units == "16"


def test_spark_flags_accepted():
    cfg = parse_args(["--master", "spark://x", "--spark_exec_memory", "8g", "--partitions", "2"])
    assert cfg.master == "spark://x" and cfg.partitions == 2


def test_net_settings():
    cfg = Config(hidden_units="128,256", in_features=4, batch_size=10)
    ns = cfg.net_settings()
    assert [s["layer_name"] for s in ns] == ["LSTMLayer0", "LSTMLayer1"]
    assert [(s["dim_size"], s["num_hidden"]) for s in ns] == [(4, 128), (128, 256)]
    assert all(s["batch_size"] == 10 and s["normalize"] is True for s in ns)


def test_params_str_format():
    s = Config().params_str()
    lines = s.strip().split("\n")
    keys = [l.split(" = ")[0].lower() for l in lines]
    assert keys == sorted(keys) and "BATCH_SIZE = 10" in lines       # sorted by flag name, then upper-cased


def test_bad_mode_rejected():
    with pytest.raises(ValueError):
        parse_args(["--mode", "predict"])


# ---------------------------------------------------------------------------------------------------------
def test_sharder_sizes_and_determinism(iris_path):
    lines = D.read_lines(iris_path)
    a = D.csv_to_partitions(lines, 4, shuffle=True, seed=3)
    b = D.csv_to_partitions(lines, 4, shuffle=True, seed=3)
    assert [k for k, _ in a] == [0, 1, 2, 3]
    assert all(len(rows) == 37 for _, rows in a)          # floor(150/4); the reference's 5th 2-row shard is gone (Q2)
    assert a == b
    c = D.csv_to_partitions(lines, 4, shuffle=True, seed=4)
    assert a != c
    s = D.csv_to_partitions(lines, 4, shuffle=False, remainder="spread")
    assert sorted(len(r) for _, r in s) == [37, 37, 38, 38]


def test_sharder_rejects_too_many_partitions():
    with pytest.raises(ValueError):
        D.csv_to_partitions(["1,2,0", "3,4,1"], 3)


def test_process_batch(iris_path):
    rows = D.read_dataset_from_path(iris_path)
    x, y = D.process_batch(rows)
    assert x.shape == (150, 4) and x.dtype == np.float32 and y.dtype == np.int64
    assert sorted(set(y.tolist())) == [0, 1, 2]
    xn, _ = D.process_batch(rows, normalize=True)
    assert xn.min() == pytest.approx(0.0) and xn.max() == pytest.approx(1.0)


def test_min_max_normalizer_is_global():
    out = np.array(D.min_max_normalizer([[0.0, 10.0], [5.0, 2.5]]))
    assert out.tolist() == [[0.0, 1.0], [0.5, 0.25]]


def test_process_batch_sequences():
    rows = [[str(v) for v in range(6)] + ["1"], [str(v) for v in range(6, 12)] + ["0"]]
    x, y = D.process_batch(rows, seq_len=3, in_features=2)
    assert x.shape == (2, 3, 2) and y.tolist() == [1, 0]


def test_next_batch_full_batches_and_reshuffle():
    x = np.arange(25, dtype=np.float32).reshape(25, 1)
    y = np.arange(25)
    it = D.next_batch(x, y, batch_size=10, shuffle=True, rng=np.random.default_rng(0))
    seen = [next(it) for _ in range(4)]
    assert all(b[0].shape == (10, 1) for b in seen)
    first_pass = np.concatenate([seen[0][1], seen[1][1]])
    second_pass = np.concatenate([seen[2][1], seen[3][1]])
    assert len(set(first_pass.tolist())) == 20 and not np.array_equal(first_pass, second_pass)


def test_next_batch_small_shard_is_an_error_not_a_hang():
    with pytest.raises(ValueError):
        next(D.next_batch(np.zeros((2, 4), np.float32), np.zeros(2, np.int64), batch_size=10))


def test_batch_size_zero_is_whole_shard():
    assert D.resolve_batch_size(0, 37) == 37
    with pytest.raises(ValueError):
        D.resolve_batch_size(50, 37)


def test_device_shard_and_pinned_loader_cpu():
    x, y = D.synthetic_sequences(40, 5, 3, 4, seed=0)
    ds = D.DeviceShard(x, y, 8, "cpu")
    xb, yb = ds.next()
    assert xb.shape == (8, 5, 3) and yb.shape == (8,)
    pl = D.PinnedHostLoader(x, y, 8, "cpu", shuffle=False)
    xb2, yb2 = pl.next()
    assert np.allclose(xb2.numpy(), x[:8]) and pl.bytes_per_batch == 8 * 5 * 3 * 4 + 64


def test_pinned_loader_yields_batches_in_order_cpu():
    x = np.arange(40 * 3, dtype=np.float32).reshape(40, 3)
    y = np.arange(40, dtype=np.int64)
    pl = D.PinnedHostLoader(x, y, 8, "cpu", shuffle=False)
    seen = [pl.next()[1].clone().numpy() for _ in range(7)]       # crosses an epoch boundary (5 batches per pass)
    assert [int(b[0]) for b in seen] == [0, 8, 16, 24, 32, 0, 8]
    assert all(len(b) == 8 for b in seen)


def test_pinned_loader_depth_three_same_order_cpu():
    x = np.arange(40 * 3, dtype=np.float32).reshape(40, 3)
    y = np.arange(40, dtype=np.int64)
    pl = D.PinnedHostLoader(x, y, 8, "cpu", shuffle=False, depth=3)
    seen = []
    for _ in range(7):
        xb, yb = pl.next()
        assert np.allclose(xb.numpy(), x[int(yb[0]):int(yb[0]) + 8])   # the slot still holds ITS batch when it is handed out
        seen.append(int(yb[0]))
    assert seen == [0, 8, 16, 24, 32, 0, 8] and len(pl.dev) == 3


@pytest.mark.parametrize("depth,per_pass", [(2, 5), (3, 5), (3, 2), (4, 1)])
def test_pinned_loader_resume_is_exact(depth, per_pass):
    """state_dict() = position of the next batch to be handed out, whatever has been prefetched (also across reshuffles and
    when the prefetch runs more than one pass ahead of a tiny shard): a fresh loader continues with exactly the same batches."""
    bs = 8
    n = bs * per_pass
    x = np.arange(n * 3, dtype=np.float32).reshape(n, 3)
    y = np.arange(n, dtype=np.int64)
    mk = lambda: D.PinnedHostLoader(x.copy(), y.copy(), bs, "cpu", shuffle=True, seed=5, depth=depth)
    ref = mk()
    want = [ref.next()[1].clone() for _ in range(14)]
    for k in (0, 1, per_pass, per_pass + 1, 2 * per_pass, 7):
        a = mk()
        for j in range(k):
            assert torch.equal(a.next()[1], want[j])
        st = a.state_dict()
        b = mk()
        b.load_state_dict(st)
        for j in range(k, 14):
            xb, yb = b.next()
            assert torch.equal(yb, want[j]), (depth, per_pass, k, j)
            assert np.allclose(xb.numpy(), x[yb.numpy()])                       # rows and labels stay together
        assert b.state_dict()["i"] == ref.state_dict()["i"]
