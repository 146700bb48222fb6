"""Stateful language-model training without a GPU (``--stateful``, truncated backpropagation through time): the refused flag
combinations, the stream parser, the (segment, stream) layout and the partition split, continuity of the carried state against
one long pass in fp64, a training step's gradient against fp64 autograd from the detached carried state, the reset at a pass
boundary, resume, ``--mode eval --stateful`` against a direct fp64 computation over the streams, and checkpoint compatibility."""
import json
import math
import os

import numpy as np
import pytest
import torch

from lstm_tensorspark_b200 import data as D
from lstm_tensorspark_b200.config import Config
from lstm_tensorspark_b200.utils import checkpoint as ckpt


def _cfg(**kw):
    base = dict(next_token=True, stateful=True, vocab_size=16, seq_len=4, batch_size=3, hidden_units="6", in_features=5,
                device="cpu", quiet=True, init="scaled")
    base.update(kw)
    return Config(**base).validate()


# ---- flags ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kw,names", [
    (dict(next_token=False), ["--stateful", "--next_token"]),
    (dict(variable_length=True), ["--stateful", "--variable_length"]),
    (dict(learn_initial_state=True), ["--stateful", "--learn_initial_state true"]),
    (dict(pooling="mean"), ["--stateful", "--pooling mean"]),
    (dict(batch_size=0), ["--stateful", "--batch_size"]),
])
def test_refused_flag_combinations_name_both_flags(kw, names):
    with pytest.raises(ValueError) as ei:
        _cfg(**kw)
    for name in names:
        assert name in str(ei.value)


def test_flag_defaults_off_and_is_recorded():
    assert not Config().stateful
    from lstm_tensorspark_b200.config import parse_args
    cfg = parse_args(["--next_token", "--vocab_size", "8", "--seq_len", "3", "--stateful"])
    assert cfg.stateful and "STATEFUL = True" in cfg.params_str()


# ---- the stream -------------------------------------------------------------------------------------------------------------
def test_rows_concatenate_in_file_order():
    s = D.token_stream([["1", "2", "3"], ["4"], ["5", "6"]], 10)
    assert s.dtype == np.int64 and s.tolist() == [1, 2, 3, 4, 5, 6]


@pytest.mark.parametrize("rows,msg", [
    ([["1", "2"], ["3", "x"]], "row 1: token id 'x' is not an integer"),
    ([["1", "2.5"]], "row 0: token id '2.5' is not an integer"),
    ([["1"], ["2"], ["10"]], r"row 2: token id 10 outside \[0, 10\)"),
    ([["-1"]], r"row 0: token id -1 outside \[0, 10\)"),
    ([["1"], ["", " "]], "row 1: no token ids"),
])
def test_bad_ids_name_the_row(rows, msg):
    with pytest.raises(ValueError, match=msg):
        D.token_stream(rows, 10)


def test_layout_of_a_hand_built_stream():
    s = np.arange(100, 123)                       # n = 23 ids, B = 3 streams: L = 7, T = 2: K = 3, one position dropped
    x, y, tail = D.stream_layout(s, 3, 2)
    L, K, B, T = 7, 3, 3, 2
    assert x.shape == (K * B, T) and x.dtype == np.int32 and y.dtype == np.int64 and tail == 0
    for k in range(K):
        for b in range(B):
            p = np.arange(k * T, k * T + T)
            assert x[k * B + b].tolist() == (100 + b * L + p).tolist()
            assert y[k * B + b].tolist() == (100 + b * L + p + 1).tolist()
    dropped = {100 + b * L + K * T for b in range(B)}                         # position 6 of every stream
    assert not dropped & set(x.ravel().tolist())
    xt, yt, tail = D.stream_layout(s, 3, 2, tail=True)                        # evaluation: the dropped positions as a tail
    assert tail == 1 and np.array_equal(xt[:K * B], x) and np.array_equal(yt[:K * B], y)
    assert xt[K * B:, 0].tolist() == sorted(dropped) and yt[K * B:, 0].tolist() == [d + 1 for d in sorted(dropped)]
    assert np.all(xt[K * B:, 1:] == 0) and np.all(yt[K * B:, 1:] == 0)


def test_too_short_a_shard_names_its_size_b_and_t():
    with pytest.raises(ValueError, match=r"shard of 6 ids.*--batch_size 3.*--seq_len 2.*at least 7 ids"):
        D.stream_layout(np.arange(6), 3, 2)
    x, y, tail = D.stream_layout(np.arange(6), 3, 2, tail=True)               # evaluation still scores it, as one tail segment
    assert tail == 1 and x.shape == (3, 2)


def test_partitions_are_contiguous_pieces_sharing_one_id(tmp_path):
    s = np.arange(22)                                                          # 21 transitions: 3 pieces of 7, none left
    pieces = D.split_stream(s, 3)
    assert [p.tolist() for p in pieces] == [list(range(0, 8)), list(range(7, 15)), list(range(14, 22))]
    path = tmp_path / "ids.csv"
    path.write_text("0,1,2,3,4\n5,6\n7,8,9,10,11,12,13,14,15,16,17,18,19,20,21\n")
    from lstm_tensorspark_b200.trainer import load_shards
    shards = load_shards(_cfg(training_path=str(path), partitions=3, vocab_size=32), 3, standalone=False)
    assert [(k, p.tolist()) for k, p in shards] == [(k, p.tolist()) for k, p in enumerate(pieces)]


def test_synthetic_stream_is_one_walk_of_its_own():
    V, T, n = 32, 5, 40
    s = D.synthetic_stream(n, T, V, seed=3)
    assert len(s) == n * T + 1 and np.array_equal(s, D.synthetic_stream(n, T, V, seed=3))
    succ = D.next_token_chain(V, 3)
    assert (succ[s[:-1]] == s[1:, None]).any(1).all()                          # every transition is one of the chain's
    x, y = D.synthetic_next_token(n, T, V, seed=3)                              # the row task draws what it drew before
    assert np.array_equal(x, D.synthetic(Config(next_token=True, vocab_size=V, seq_len=T).validate(), n, 3)[0])


# ---- continuity and truncation in fp64 --------------------------------------------------------------------------------------
def _model(cfg, B, seed=0):
    from lstm_tensorspark_b200.models.classifier import SequenceClassifier
    gen = torch.Generator().manual_seed(seed)
    m = SequenceClassifier(cfg, batch_size=B, device="cpu", generator=gen).double()
    m.set_compute_dtype(torch.float64)
    return m


def _position_losses(m, h_seq, labels):
    logp = torch.log_softmax(h_seq @ m.head.weights + m.head.bias, 2)          # [T,B,C]
    return -logp.gather(2, labels.t().unsqueeze(2)).squeeze(2)


@pytest.mark.parametrize("hidden", ["6", "6,5"])
def test_segments_carry_the_state_of_one_long_pass(hidden):
    B, T, K = 3, 4, 5
    cfg = _cfg(hidden_units=hidden)
    m = _model(cfg, B).eval()
    s = D.synthetic_stream(B * K * T // T + 2, T, cfg.vocab_size, seed=1)[:B * K * T + 1]
    x, y, _ = D.stream_layout(s, B, T)
    x, y = torch.as_tensor(x), torch.as_tensor(y)
    # one pass over every stream's K*T positions from zero
    long_x = torch.cat([x[k * B:(k + 1) * B] for k in range(K)], 1)
    long_y = torch.cat([y[k * B:(k + 1) * B] for k in range(K)], 1)
    with torch.no_grad():
        h_long = m.sequence_features(long_x)
        l_long = _position_losses(m, h_long, long_y)
        state = m.rnn.zero_state(B, torch.float64, "cpu")
        hs, ls = [], []
        for k in range(K):
            h = m.sequence_features(x[k * B:(k + 1) * B], state=state)
            state = m.rnn.final_state()
            hs.append(h)
            ls.append(_position_losses(m, h, y[k * B:(k + 1) * B]))
    assert torch.allclose(torch.cat(hs), h_long, rtol=1e-12, atol=1e-14)
    assert torch.allclose(torch.cat(ls), l_long, rtol=1e-12, atol=1e-14)
    # without the carry every segment but the first differs
    with torch.no_grad():
        h_cold = m.sequence_features(x[B:2 * B])
    assert not torch.allclose(h_cold, h_long[T:2 * T])


def _engine(cfg, B, lr=0.0, optimizer="sgd"):
    from lstm_tensorspark_b200.engine import TrainEngine
    cfg.learning_rate, cfg.optimizer = lr, optimizer
    return TrainEngine(cfg, 0, 1, None, batch_size=B, device=torch.device("cpu"), dtype=torch.float32)


def test_a_step_is_truncated_at_the_segment_boundary():
    """One stateful step's gradient equals fp64 autograd of the same segment from the carried state, detached: no gradient
    crosses into the previous segment (and the carried state matters: from zero the gradient is another)."""
    B, T = 3, 4
    cfg = _cfg(hidden_units="6,5")
    eng = _engine(cfg, B)
    s = D.synthetic_stream(B * 2 * T, T, cfg.vocab_size, seed=2)
    x, y, _ = (torch.as_tensor(a) if isinstance(a, np.ndarray) else a for a in D.stream_layout(s, B, T))
    eng.step(x[:B], y[:B], reset=True)
    eng.step(x[B:2 * B], y[B:2 * B])
    got = {k: p.grad.double().clone() for k, p in eng.model.named_parameters()}
    carried = [(h.double(), c.double()) for h, c in eng.state_prev]
    assert all(float(h.abs().max()) > 0 for h, _ in carried)

    def fp64_grads(state):
        ref = _model(cfg, B)
        ref.load_reference_state_dict(eng.model.reference_state_dict())
        st = [(h.clone().requires_grad_(True), c.clone().requires_grad_(True)) for h, c in state]
        loss = ref(x[B:2 * B], y[B:2 * B], state=st)[0]
        loss.backward()
        assert all(h.grad is None and c.grad is None for h, c in st)         # the carried state is a constant
        return {k: p.grad for k, p in ref.named_parameters() if p.grad is not None}

    want = fp64_grads(carried)
    assert set(want) == set(got)
    for k in want:
        assert torch.allclose(got[k], want[k], rtol=1e-4, atol=1e-6), k
    cold = fp64_grads([(torch.zeros_like(h), torch.zeros_like(c)) for h, c in carried])
    assert not torch.allclose(got["rnn.layers.0.w_h"], cold["rnn.layers.0.w_h"], rtol=1e-3, atol=1e-5)


def test_a_new_pass_starts_from_zero():
    B, T, K = 3, 4, 2
    cfg = _cfg(hidden_units="6,5", learn_initial_state=False)
    eng = _engine(cfg, B, lr=1e-2, optimizer="adam")
    x, y, _ = D.stream_layout(D.synthetic_stream(B * K, T, cfg.vocab_size, seed=4), B, T)
    loader = D.DeviceShard(x, y, B, "cpu", dtype=torch.int32, shuffle=False)
    opened = []
    for step in range(2 * K + 1):
        bx, by = loader.next()
        opened.append(loader.opened_pass())
        eng.step(bx, by, reset=loader.opened_pass())
        zero = all(float(h.abs().max()) == 0 and float(c.abs().max()) == 0 for h, c in eng.state_prev)
        assert zero == (step % K == 0), step
        assert all(float(h.abs().max()) > 0 for h, _ in eng.carried_state())
    assert opened == [True, False, True, False, True]


# ---- training runs ----------------------------------------------------------------------------------------------------------
def _run_cfg(tmp_path, name, **kw):
    base = dict(next_token=True, stateful=True, vocab_size=32, seq_len=6, batch_size=4, hidden_units="8,8", in_features=6,
                synthetic=30, device="cpu", quiet=True, init="scaled", learning_rate=1e-2, dropout=0.2,
                checkpoint_path=str(tmp_path / name), output_path=str(tmp_path / (name + "_out")))
    base.update(kw)
    return Config(**base).validate()


def _latest(path):
    run = ckpt.find_latest_run(str(path), None)
    return ckpt.load(ckpt.latest_checkpoint(run))


def test_resume_continues_the_stream_and_its_state(tmp_path):
    """k steps, a checkpoint, k more after resuming = 2k uninterrupted steps: weights, optimizer state and carried state.  A pass
    is 7 segments (30 * 6 + 1 ids in 4 streams: L = 45, K = 7), so the 2k = 10 steps cross a pass boundary."""
    from lstm_tensorspark_b200.trainer import run_job
    k = 5
    run_job(_run_cfg(tmp_path, "a", epochs=1, max_steps=k, evaluate_every=k), standalone=True)
    run_job(_run_cfg(tmp_path, "a", epochs=1, max_steps=2 * k, evaluate_every=k, use_pretrained_model=True), standalone=True)
    run_job(_run_cfg(tmp_path, "b", epochs=1, max_steps=2 * k, evaluate_every=k), standalone=True)
    va, ma, oa = _latest(tmp_path / "a")
    vb, mb, ob = _latest(tmp_path / "b")
    assert ma["global_step"] == mb["global_step"] == 2 * k - 1
    assert va.keys() == vb.keys() and all(torch.equal(va[n], vb[n]) for n in va)
    assert oa["stateful"] is True and ob["stateful"] is True
    assert len(oa["state"]) == 2 and all(torch.equal(u, v) for p, q in zip(oa["state"], ob["state"]) for u, v in zip(p, q))
    assert all(float(h.abs().max()) > 0 for h, _ in oa["state"])
    sa, sb = oa["optimizer"], ob["optimizer"]
    for key in sa:
        if isinstance(sa[key], torch.Tensor):
            assert torch.equal(sa[key], sb[key]), key
        else:
            assert sa[key] == sb[key], key
    assert not any(n.endswith("state") for n in va)                           # no new model variables


def test_checkpoints_of_the_other_setting_are_refused_for_resume_and_scored_by_eval(tmp_path):
    from lstm_tensorspark_b200.trainer import run_job
    run_job(_run_cfg(tmp_path, "s", epochs=1, max_steps=2, dropout=0.0), standalone=True)
    with pytest.raises(ValueError, match="written with --stateful.*add --stateful"):
        run_job(_run_cfg(tmp_path, "s", stateful=False, epochs=1, max_steps=3, use_pretrained_model=True, dropout=0.0),
                standalone=True)
    run_job(_run_cfg(tmp_path, "p", stateful=False, epochs=1, max_steps=2, dropout=0.0), standalone=True)
    with pytest.raises(ValueError, match="written without --stateful.*drop --stateful"):
        run_job(_run_cfg(tmp_path, "p", epochs=1, max_steps=3, use_pretrained_model=True, dropout=0.0), standalone=True)
    for name in ("s", "p"):
        for stateful in (True, False):
            ev = run_job(_run_cfg(tmp_path, name, mode="eval", stateful=stateful, dropout=0.0), standalone=True)
            assert math.isfinite(ev["perplexity"]) and ev["perplexity"] == pytest.approx(math.exp(ev["loss"]))


def test_stream_eval_equals_a_direct_fp64_computation(tmp_path):
    """``--mode eval --stateful`` on a tiny file: B streams, the state carried over every segment, the tail included, equals
    one fp64 pass per stream over all of its L positions."""
    from lstm_tensorspark_b200.trainer import run_job
    rng = np.random.default_rng(7)
    rows = [rng.integers(0, 32, size=rng.integers(1, 9)).tolist() for _ in range(20)]
    path = tmp_path / "ids.csv"
    path.write_text("".join(",".join(map(str, r)) + "\n" for r in rows))
    kw = dict(synthetic=0, training_path=str(path), dropout=0.0)
    run_job(_run_cfg(tmp_path, "e", epochs=1, max_steps=3, **kw), standalone=True)
    ev = run_job(_run_cfg(tmp_path, "e", mode="eval", json_log=str(tmp_path / "ev.jsonl"), **kw), standalone=True)
    s = D.token_stream([[str(v) for v in r] for r in rows], 32)
    B, T = 4, 6
    L = (len(s) - 1) // B
    assert L % T != 0 and ev["positions"] == B * L and ev["streams"] == B and ev["stream"] == len(s)
    variables, _, _ = _latest(tmp_path / "e")
    m = _model(_run_cfg(tmp_path, "e", **kw), B)
    m.load_reference_state_dict(variables)
    inp = torch.as_tensor(s[:B * L].reshape(B, L))
    lab = torch.as_tensor(s[1:B * L + 1].reshape(B, L))
    with torch.no_grad():
        losses = _position_losses(m, m.sequence_features(inp), lab)
        correct = int(((m.sequence_features(inp) @ m.head.weights + m.head.bias).argmax(2) == lab.t()).sum())
    assert ev["loss"] == pytest.approx(float(losses.mean()), rel=1e-5)
    assert ev["accuracy"] == pytest.approx(correct / (B * L), abs=0.5 / (B * L))
    assert json.loads(open(tmp_path / "ev.jsonl").read().splitlines()[-1])["positions"] == B * L


def test_evaluations_score_the_batch_from_the_state_it_was_trained_from(tmp_path):
    """The loss logged at an evaluation is that of the step's batch from ``state_prev``: with one segment per pass (zero state
    every step) it equals the stateless score; with several it does not have to."""
    from lstm_tensorspark_b200.trainer import run_job
    log = tmp_path / "log.jsonl"
    run_job(_run_cfg(tmp_path, "v", epochs=1, max_steps=4, evaluate_every=1, json_log=str(log), dropout=0.0,
                     learning_rate=0.0), standalone=True)
    rows = [json.loads(r) for r in open(log) if "perplexity" in r]
    variables, _, _ = _latest(tmp_path / "v")
    cfg = _run_cfg(tmp_path, "v", dropout=0.0)
    m = _model(cfg, 4)
    m.load_reference_state_dict(variables)
    s = D.synthetic_stream(30, 6, 32, 0)
    x, y, _ = D.stream_layout(s, 4, 6)
    x, y = torch.as_tensor(x), torch.as_tensor(y)
    state = m.rnn.zero_state(4, torch.float64, "cpu")
    with torch.no_grad():
        for step in range(4):
            loss, _, _ = m.score(x[4 * step:4 * step + 4], y[4 * step:4 * step + 4], state=state)
            state = m.rnn.final_state()
            assert rows[step]["loss"] == pytest.approx(float(loss), rel=1e-5), step
