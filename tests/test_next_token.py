"""Next-token language modelling without a GPU: the reference of the large-vocabulary head, ``--next_token`` flag validation, row
parsing, the synthetic Markov language, a small training run with perplexity, checkpoints, ``--mode eval`` and two gloo ranks."""
import json
import math
import os

import numpy as np
import pytest
import torch

from lstm_tensorspark_b200 import data as D
from lstm_tensorspark_b200.config import Config
from lstm_tensorspark_b200.ops import functional as F
from lstm_tensorspark_b200.ops import reference as ref


# ---- the op's reference -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("ragged", [False, True])
def test_reference_op_matches_head_xent_per_step_and_autograd(ragged):
    g = torch.Generator().manual_seed(3)
    T, B, H, C = 6, 5, 8, 20
    h = torch.randn(T, B, H, generator=g, dtype=torch.float64, requires_grad=True)
    W = torch.randn(H, C, generator=g, dtype=torch.float64, requires_grad=True)
    b = torch.randn(C, generator=g, dtype=torch.float64, requires_grad=True)
    labels = torch.randint(0, C, (B, T), generator=g)
    lengths = torch.tensor([6, 1, 3, 0, 4], dtype=torch.int32) if ragged else None      # a zero length counts nothing
    loss, correct, n = F.vocab_xent_per_step(h, W, b, labels, lengths)
    _, l0, c0, n0 = ref.head_xent_per_step(h, W, b, labels, lengths)
    assert torch.equal(loss, l0) and int(correct) == int(c0) and int(n) == int(n0) == (14 if ragged else T * B)
    (loss * 0.7).backward()
    got = [t.grad.clone() for t in (h, W, b)]
    for t in (h, W, b):
        t.grad = None
    keep = ref.step_mask(lengths, B, T)
    logits = (h @ W + b).transpose(0, 1)[keep]
    (torch.nn.functional.cross_entropy(logits, labels[keep]) * 0.7).backward()
    for a, t in zip(got, (h, W, b)):
        assert torch.allclose(a, t.grad, rtol=1e-12, atol=1e-14)
    if ragged:
        assert float(got[0][:, 3].abs().max()) == 0.0 and float(got[0][1:, 1].abs().max()) == 0.0


def test_cpu_dispatch_is_the_reference():
    h = torch.randn(3, 2, 64)
    assert not F.vocab_head_supported(h.bfloat16(), 512)


# ---- flags ------------------------------------------------------------------------------------------------------------------
def test_flag_sets_per_step_labels_and_num_classes():
    cfg = Config(next_token=True, vocab_size=50, seq_len=4).validate()
    assert cfg.per_step_labels and cfg.num_classes == 50
    assert Config(next_token=True, vocab_size=50, seq_len=4, num_classes=50).validate().num_classes == 50
    from lstm_tensorspark_b200.config import parse_args
    cfg = parse_args(["--next_token", "--vocab_size", "40", "--seq_len", "3"])
    assert cfg.next_token and cfg.per_step_labels and cfg.num_classes == 40
    assert "NEXT_TOKEN = True" in cfg.params_str()
    assert not Config().next_token


@pytest.mark.parametrize("kw,names", [
    (dict(vocab_size=0), ["--next_token", "--vocab_size"]),
    (dict(seq_len=1), ["--next_token", "--seq_len"]),
    (dict(num_classes=7), ["--next_token", "--num_classes", "--vocab_size"]),
    (dict(pooling="mean"), ["--next_token", "--pooling mean"]),
    (dict(bidirectional=True), ["--next_token", "--bidirectional"]),
])
def test_flag_errors_name_their_flags(kw, names):
    base = dict(next_token=True, vocab_size=50, seq_len=4)
    base.update(kw)
    with pytest.raises(ValueError) as ei:
        Config(**base).validate()
    for name in names:
        assert name in str(ei.value)


# ---- rows -------------------------------------------------------------------------------------------------------------------
def _cfg(**kw):
    return Config(**dict(dict(next_token=True, vocab_size=10, seq_len=4), **kw)).validate()


def test_fixed_rows_are_shifted():
    x, y, l = D.parse_rows([["1", "2", "3", "4", "5"], ["9", "0", "9", "0", "9"]], _cfg())
    assert l is None and x.dtype == np.int32 and y.dtype == np.int64
    assert x.tolist() == [[1, 2, 3, 4], [9, 0, 9, 0]] and y.tolist() == [[2, 3, 4, 5], [0, 9, 0, 9]]


def test_ragged_rows_are_shifted_and_padded():
    x, y, l = D.parse_rows([["1", "2"], ["3", "4", "5", "6", "7"], ["8", "9", "1"]], _cfg(variable_length=True))
    assert l.tolist() == [1, 4, 2]
    assert x.tolist() == [[1, 0, 0, 0], [3, 4, 5, 6], [8, 9, 0, 0]] and y.tolist() == [[2, 0, 0, 0], [4, 5, 6, 7], [9, 1, 0, 0]]


@pytest.mark.parametrize("rows,ragged,msg", [
    ([["1", "2", "3", "4", "5"], ["1", "2", "3", "4"]], False, "row 1: 4 fields is not 5 token ids"),
    ([["1", "2", "3", "4", "5", "6"]], True, "row 0: 6 fields is not 2..5 token ids"),
    ([["1", "2"], ["7"]], True, "row 1: 1 fields is not 2..5 token ids"),
    ([["1", "2", "3.5", "4", "5"]], False, "row 0: token id '3.5' is not an integer"),
    ([["1", "2", "3", "4", "10"]], False, r"row 0: token id 10 outside \[0, 10\)"),
    ([["1", "2", "3", "4", "5"], ["1", "-1", "3", "4", "5"]], False, r"row 1: token id -1 outside \[0, 10\)"),
])
def test_malformed_rows_name_the_row(rows, ragged, msg):
    with pytest.raises(ValueError, match=msg):
        D.parse_rows(rows, _cfg(variable_length=ragged))


def test_rows_without_the_flag_parse_as_before():
    cfg = Config(vocab_size=10, seq_len=4, num_classes=3).validate()
    x, y, _ = D.parse_rows([["1", "2", "3", "4", "2"]], cfg)
    assert x.tolist() == [[1, 2, 3, 4]] and y.tolist() == [2]


# ---- the synthetic language -------------------------------------------------------------------------------------------------
def test_synthetic_chain_is_reproducible_and_has_the_stated_statistics():
    V, T = 64, 32
    x, y = D.synthetic_next_token(4000, T, V, seed=5)
    x2, y2 = D.synthetic_next_token(4000, T, V, seed=5)
    assert np.array_equal(x, x2) and np.array_equal(y, y2)
    assert not np.array_equal(x, D.synthetic_next_token(4000, T, V, seed=6)[0])
    assert x.dtype == np.int32 and y.dtype == np.int64 and np.array_equal(x[:, 1:], y[:, :-1])
    xt, _ = D.synthetic_tokens(4000, T, V, V, seed=5, per_step_labels=True)
    assert not np.array_equal(x, xt)
    succ = D.next_token_chain(V, 5)
    assert succ.shape == (V, 4) and all(len(set(r)) == 4 for r in succ.tolist())
    which = (y[:, :, None] == succ[x]).astype(np.float64)                   # [n, T, 4]: which successor followed
    assert np.all(which.sum(2) == 1)
    assert np.allclose(which.mean((0, 1)), D.NEXT_TOKEN_PROBS, atol=0.01)
    assert D.NEXT_TOKEN_ENTROPY == pytest.approx(1.0889, abs=1e-4) and math.exp(D.NEXT_TOKEN_ENTROPY) == pytest.approx(2.97, abs=0.01)
    xr, yr, l = D.synthetic_next_token(50, T, V, seed=5, variable_length=True)
    assert np.array_equal(l, D.synthetic_lengths(50, T, 5))
    pad = np.arange(T)[None, :] >= l[:, None]
    assert np.all(xr[pad] == 0) and np.all(yr[pad] == 0) and np.array_equal(xr[~pad], D.synthetic_next_token(50, T, V, seed=5)[0][~pad])


def test_runs_without_the_flag_draw_what_they_drew_before():
    """``synthetic`` dispatches on the flag alone: the other tasks' arrays are those of their own generators."""
    cfg = Config(vocab_size=20, seq_len=5, num_classes=3, per_step_labels=True, variable_length=True).validate()
    a = D.synthetic(cfg, 30, 4)
    b = D.synthetic_tokens(30, 5, 20, 3, seed=4, variable_length=True, per_step_labels=True)
    assert all(np.array_equal(u, v) for u, v in zip(a, b))
    nt = D.synthetic(_cfg(vocab_size=20, seq_len=5), 30, 4)
    assert np.array_equal(nt[0], D.synthetic_next_token(30, 5, 20, seed=4)[0]) and nt[2] is None


# ---- training ---------------------------------------------------------------------------------------------------------------
def _base(tmp_path, **kw):
    base = dict(hidden_units="32", in_features=16, seq_len=12, batch_size=32, vocab_size=64, next_token=True, synthetic=512,
                device="cpu", quiet=True, init="scaled", learning_rate=2e-2, steps_mode="epochs", evaluate_every=20,
                checkpoint_path=str(tmp_path / "ck"), output_path=str(tmp_path / "out"), json_log=str(tmp_path / "log.jsonl"))
    base.update(kw)
    return base


def _log(tmp_path):
    return [json.loads(s) for s in open(tmp_path / "log.jsonl") if "perplexity" in s]


def test_training_run_lowers_perplexity_and_checkpoints_round_trip(tmp_path):
    from lstm_tensorspark_b200.trainer import run_job
    out = run_job(Config(epochs=25, **_base(tmp_path)).validate(), standalone=True)
    rows = _log(tmp_path)
    assert rows[0]["perplexity"] > 30 and rows[-1]["perplexity"] < 8
    assert all(r["perplexity"] == pytest.approx(math.exp(r["loss"])) for r in rows)
    run = os.path.join(tmp_path / "ck", os.listdir(tmp_path / "ck")[0])
    scal = [json.loads(s) for s in open(os.path.join(run, "train", "scalars.jsonl"))]
    assert "perplexity" in scal[-1]
    steps = out["results"][0]["steps"]
    # resume: continues at the next step with the recorded flag
    out2 = run_job(Config(epochs=26, use_pretrained_model=True, **_base(tmp_path)).validate(), standalone=True)
    assert out2["results"][0]["steps"] == 16 and steps == 400
    ev = run_job(Config(mode="eval", **_base(tmp_path, json_log="")).validate(), standalone=True)
    assert ev["perplexity"] == pytest.approx(math.exp(ev["loss"])) and ev["perplexity"] < 8 and ev["positions"] == 512 * 12


def test_eval_prints_the_perplexity_the_last_evaluation_logged(tmp_path, capsys):
    """One batch is the whole data set: the last training evaluation and ``--mode eval`` score the same positions of the same
    weights."""
    from lstm_tensorspark_b200.trainer import run_job
    base = _base(tmp_path, synthetic=32, quiet=False)
    run_job(Config(epochs=6, **base).validate(), standalone=True)
    last = _log(tmp_path)[-1]
    capsys.readouterr()
    ev = run_job(Config(mode="eval", **dict(base, json_log="")).validate(), standalone=True)
    assert ev["perplexity"] == pytest.approx(last["perplexity"], rel=1e-5)
    assert f"perplexity {ev['perplexity']:.4f}" in capsys.readouterr().out


def test_checkpoint_written_with_the_other_setting_is_refused(tmp_path):
    from lstm_tensorspark_b200.trainer import run_job
    plain = dict(_base(tmp_path), next_token=False, per_step_labels=True, num_classes=64)
    run_job(Config(epochs=1, max_steps=2, **plain).validate(), standalone=True)
    with pytest.raises(ValueError, match="written without --next_token.*drop --next_token"):
        run_job(Config(epochs=1, max_steps=3, use_pretrained_model=True, **_base(tmp_path)).validate(), standalone=True)
    with pytest.raises(ValueError, match="--next_token"):
        run_job(Config(mode="eval", **_base(tmp_path)).validate(), standalone=True)


def test_averaged_model_records_the_flag(tmp_path):
    from lstm_tensorspark_b200.trainer import run_job
    base = _base(tmp_path, partitions=2, max_workers=1, epochs=1, max_steps=2, synthetic=128)
    run_job(Config(**base).validate(), standalone=False)
    blob = torch.load(os.path.join(base["output_path"], "averaged_model.pt"), weights_only=False)
    assert blob["meta"]["next_token"] is True
    ev = run_job(Config(mode="eval", **dict(base, partitions=1)).validate(), standalone=False)
    assert "perplexity" in ev
    other = dict(base, partitions=1, next_token=False, per_step_labels=True, num_classes=64)
    with pytest.raises(ValueError, match="written with --next_token.*add --next_token"):
        run_job(Config(mode="eval", **other).validate(), standalone=False)


def test_tail_scoring_on_the_cpu_counts_the_tail_only():
    from lstm_tensorspark_b200.models.classifier import SequenceClassifier
    cfg = _cfg(hidden_units="8", in_features=4, batch_size=6, variable_length=True, device="cpu")
    m = SequenceClassifier(cfg, batch_size=6, device="cpu").eval()
    x, y, l = (torch.as_tensor(a) for a in D.synthetic_next_token(6, 4, 10, seed=1, variable_length=True))
    loss, ok, n = m.score(x, y, l, first=4)
    assert int(n) == int(l[4:].sum())
    l2, ok2, n2 = m.score(torch.cat([x[4:], x[4:], x[4:]]), torch.cat([y[4:], y[4:], y[4:]]), torch.cat([l[4:], l[4:], l[4:]]))
    assert float(loss) == pytest.approx(float(l2), rel=1e-5) and int(ok2) == 3 * int(ok)


# ---- two ranks --------------------------------------------------------------------------------------------------------------
def _sync_check(rank, world):
    import torch.distributed as dist
    from lstm_tensorspark_b200.engine import TrainEngine
    from lstm_tensorspark_b200.parallel.comm import make_communicator
    dev = torch.device("cpu")
    comm = make_communicator("gloo", rank, world, dev, 60)
    cfg = Config(hidden_units="8,8", in_features=4, batch_size=6, seq_len=5, sync_mode="grad_allreduce", device="cpu",
                 learn_initial_state=False, init="scaled", partitions=world, variable_length=True, vocab_size=16, next_token=True)
    eng = TrainEngine(cfg, rank, world, comm, batch_size=6, device=dev, dtype=torch.float32)
    x, y, l = (torch.as_tensor(a) for a in D.synthetic_next_token(6, 5, 16, seed=rank, variable_length=True))
    for _ in range(4):
        eng.step(x, y, l)
    eng.model.eval()
    probe = [torch.as_tensor(a) for a in D.synthetic_next_token(6, 5, 16, seed=9, variable_length=True)]
    loss = eng.model.score(*probe)[0].reshape(1).clone()
    losses = [torch.zeros_like(loss) for _ in range(world)]
    dist.all_gather(losses, loss)
    all_w = [torch.zeros_like(eng.flat.data) for _ in range(world)]
    dist.all_gather(all_w, eng.flat.data)
    comm.close()
    return all(torch.equal(losses[0], v) for v in losses) and all(torch.equal(all_w[0], w) for w in all_w)


def test_two_ranks_grad_allreduce_agree_on_the_loss():
    from lstm_tensorspark_b200.parallel.launch import launch
    assert all(launch(_sync_check, 2, args=()))
