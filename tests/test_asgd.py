"""AWD-LSTM's NT-ASGD without a GPU (``--optimizer asgd | ntasgd``, ``--valid_path`` / ``--valid_synthetic``, ``--nonmono``): the
non-monotone trigger on hand-worked histories, the flat optimizer against ``torch.optim.ASGD`` in fp64, ntasgd before the trigger as
sgd, the held-out draws, the flags, two gloo ranks, checkpoints and resume, ``--mode eval`` on the average and the export."""
import hashlib
import json
import math

import numpy as np
import pytest
import torch

from lstm_tensorspark_b200 import data as D
from lstm_tensorspark_b200.config import Config, parse_args
from lstm_tensorspark_b200.models.flat import FlatParams
from lstm_tensorspark_b200.ops import reference as ref
from lstm_tensorspark_b200.ops.optim import FlatOptimizer, nonmono_trigger
from lstm_tensorspark_b200.utils import checkpoint as ckpt


# ---- the trigger --------------------------------------------------------------------------------------------------------------
def _fire_step(losses, n):
    """The index of the validation at which AWD-LSTM's main.py switches to ASGD, by the trainer's own bookkeeping."""
    hist, on, fired = [], False, []
    for i, v in enumerate(losses):
        if nonmono_trigger(hist, v, n, on):
            on = True
            fired.append(i)
        hist.append(v)
    return fired


def test_trigger_fires_at_awds_step_once():
    # n = 2: validation i fires iff i > 2 and v_i > min(v_0 .. v_{i-3})
    assert _fire_step([5.0, 4.0, 3.0, 2.0, 1.0, 0.5], 2) == []                  # monotone: never
    assert _fire_step([5.0, 4.0, 3.0, 4.5, 6.0, 7.0], 2) == [4]                 # 4.5 <= min(5.0); 6.0 > min(5.0, 4.0)
    assert _fire_step([3.0, 4.0, 5.0, 3.0, 3.5, 9.0, 9.0], 2) == [4]            # 3.0 == min: not worse; 3.5 > 3.0
    assert _fire_step([1.0, 2.0, 3.0], 2) == []                                  # len(h) > n is needed first
    assert _fire_step([1.0, 2.0, 3.0, 4.0], 2) == [3]
    assert _fire_step([1.0, 2.0, 3.0, 4.0, 5.0, 6.0, 7.0], 5) == [6]            # AWD's default n = 5


def test_trigger_never_fires_on_nan_nor_while_averaging():
    assert _fire_step([1.0, 2.0, 3.0, float("nan"), float("nan")], 2) == []
    assert _fire_step([1.0, 2.0, 3.0, float("nan"), 4.0], 2) == [4]
    assert not nonmono_trigger([1.0, 1.0, 1.0], 5.0, 1, averaging=True)
    assert nonmono_trigger([1.0, 1.0, 1.0], 5.0, 1, averaging=False)
    assert not nonmono_trigger([float("nan"), 1.0], 5.0, 1, averaging=False)     # min over a NaN: no number beats it


# ---- the optimizer against torch.optim.ASGD -----------------------------------------------------------------------------------
def _flat(n_lstm, n_other, seed=0, dtype=torch.float64):
    g = torch.Generator().manual_seed(seed)
    a = torch.nn.Parameter(torch.randn(n_lstm, generator=g))
    b = torch.nn.Parameter(torch.randn(n_other, generator=g))
    fl = FlatParams([a], [b])
    fl.data = fl.data.to(dtype)
    fl.grad = fl.grad.to(dtype)
    fl._rebind()
    return fl, a, b


@pytest.mark.parametrize("wd,cut,clip", [(0.0, False, 0.0), (0.125, False, 0.0), (0.125, True, 0.0), (0.0, False, 0.75)])
def test_flat_asgd_equals_torch_asgd_in_fp64(wd, cut, clip):
    """20 steps of random gradients: p and ax equal torch.optim.ASGD(lambd=0, t0=0, weight_decay) in fp64 (lr a power of two,
    which torch's fp32 eta holds exactly); the decay over the first segment only (the wd_numel cut) is two parameter groups there.
    Clipping is clip_grad_norm_ before the step, whose norm of per-tensor norms rounds differently from the one fp64 sum of
    squares here: equal to within fp64 rounding."""
    lr, steps = 0.25, 20
    fl, a, b = _flat(64, 48)
    opt = FlatOptimizer(fl, lr, "asgd", weight_decay=wd)
    if cut:
        opt.wd_numel = fl.lstm_numel
    opt.clip_norm = clip
    ta, tb = (torch.nn.Parameter(p.detach().clone()) for p in (a, b))
    groups = [{"params": [ta]}, {"params": [tb], "weight_decay": 0.0 if cut else wd}]
    topt = torch.optim.ASGD(groups, lr=lr, lambd=0.0, alpha=0.75, t0=0.0, weight_decay=wd)
    g = torch.Generator().manual_seed(1)
    for _ in range(steps):
        ga, gb = torch.randn(64, generator=g, dtype=torch.float64), torch.randn(48, generator=g, dtype=torch.float64)
        a.grad.copy_(ga); b.grad.copy_(gb)
        ta.grad, tb.grad = ga.clone(), gb.clone()
        opt.step()
        if clip:
            torch.nn.utils.clip_grad_norm_([ta, tb], clip)
        topt.step()
    assert opt.averaged_steps == steps and opt.averaging
    tol = dict(rtol=1e-13, atol=1e-15) if clip else dict(rtol=0, atol=0)
    oa, ob = fl.offsets
    for mine, theirs in ((a.detach(), ta.detach()), (b.detach(), tb.detach()), (opt.ax[oa:oa + 64], topt.state[ta]["ax"]),
                         (opt.ax[ob:ob + 48], topt.state[tb]["ax"])):
        torch.testing.assert_close(mine, theirs, **tol)


def test_average_is_the_mean_of_the_iterates_from_the_second():
    p = torch.zeros(8, dtype=torch.float64)
    ax = torch.zeros_like(p)
    iterates = []
    for k in range(1, 9):
        p.copy_(torch.arange(8, dtype=torch.float64) * k)
        iterates.append(p.clone())
        ref.asgd_average_(ax, p, k)
    torch.testing.assert_close(ax, torch.stack(iterates[1:]).mean(0))


def test_ntasgd_before_the_trigger_is_sgd_bitwise_then_averages_afresh():
    fl1, a1, _ = _flat(64, 48, dtype=torch.float32)
    fl2, a2, _ = _flat(64, 48, dtype=torch.float32)
    sgd = FlatOptimizer(fl1, 0.1, "sgd", weight_decay=0.01)
    nt = FlatOptimizer(fl2, 0.1, "ntasgd", weight_decay=0.01)
    for o in (sgd, nt):
        o.wd_numel = o.flat.lstm_numel
        o.clip_norm = 2.0
    g = torch.Generator().manual_seed(2)
    for step in range(8):
        gr = torch.randn(fl1.grad.numel(), generator=g)
        fl1.grad.copy_(gr); fl2.grad.copy_(gr)
        sgd.step(); nt.step()
        assert torch.equal(fl1.data, fl2.data)
        if step == 4:
            assert not nt.averaging and nt.averaged_steps == 0 and not nt.ax.any()
            nt.start_averaging()
    assert nt.averaging and nt.averaged_steps == 3
    assert not torch.equal(nt.ax, fl2.data)


# ---- held-out draws -----------------------------------------------------------------------------------------------------------
def _h(*arrs):
    g = hashlib.sha256()
    for a in arrs:
        if a is not None:
            g.update(np.ascontiguousarray(a).tobytes())
    return g.hexdigest()[:16]


TASKS = [(dict(hidden_units="8", in_features=4, seq_len=5, num_classes=3), "5859e765296fe7c3"),
         (dict(hidden_units="8", in_features=4, seq_len=5, num_classes=3, per_step_labels=True, variable_length=True),
          "b1ca46e5caca74f7"),
         (dict(hidden_units="8", in_features=4, seq_len=5, vocab_size=50, num_classes=3), "c055768535e55fdf"),
         (dict(hidden_units="8", in_features=4, seq_len=5, vocab_size=50, next_token=True), "22d9ab21abeb1477")]


@pytest.mark.parametrize("kw,train_hash", TASKS)
def test_validation_draws_are_new_samples_of_the_training_task(kw, train_hash):
    cfg = Config(**kw).validate()
    train = D.synthetic(cfg, 40, 3)
    assert _h(*train) == train_hash                                 # the training draws are those of the parent commit
    valid = D.synthetic(cfg, 40, 3, valid_of=40)
    assert train[0].shape == valid[0].shape and not np.array_equal(train[0], valid[0])
    if cfg.variable_length:                                          # the held-out lengths are new draws too
        assert not np.array_equal(train[2], valid[2])
    if cfg.next_token:                                               # the same chain: every held-out transition is legal
        succ = D.next_token_chain(cfg.vocab_size, 3)
        tok = np.concatenate([valid[0][:, :1], valid[1]], 1)
        assert D.legal_fraction(tok[:, :1], np.ones(len(tok), np.int32), tok[:, 1:], succ) == 1.0
    elif cfg.vocab_size == 0 and not cfg.per_step_labels:            # the same class centres as the 40 training samples
        rng = np.random.default_rng(3)
        rng.integers(0, cfg.num_classes, size=40)
        centers = rng.standard_normal((cfg.num_classes, cfg.in_features))
        big = D.synthetic(cfg, 3000, 3, valid_of=40)
        for c in range(cfg.num_classes):
            assert np.abs(big[0][big[1] == c].mean((0, 1)) - centers[c]).max() < 0.05


def test_validation_stream_is_a_new_walk_of_the_chain():
    train = D.synthetic_stream(20, 5, 50, 3)
    assert _h(train) == "e976df247d3475cd"
    valid = D.synthetic_stream(20, 5, 50, 3, valid=True)
    assert len(valid) == len(train) and not np.array_equal(train, valid)
    succ = D.next_token_chain(50, 3)
    assert D.legal_fraction(valid[None, :1], np.ones(1, np.int32), valid[None, 1:], succ) == 1.0


# ---- flags --------------------------------------------------------------------------------------------------------------------
def _lm(**kw):
    base = dict(hidden_units="8,8", in_features=8, seq_len=6, batch_size=4, vocab_size=32, next_token=True, init="scaled",
                learn_initial_state=False, device="cpu", synthetic=40)
    base.update(kw)
    return Config(**base).validate()


def test_flags_parse_and_default():
    cfg = parse_args(["--optimizer", "ntasgd", "--nonmono", "3", "--valid_synthetic", "12", "--synthetic", "40"])
    assert (cfg.optimizer, cfg.nonmono, cfg.valid_synthetic) == ("ntasgd", 3, 12)
    d = Config()
    assert (d.optimizer, d.nonmono, d.valid_path, d.valid_synthetic) == ("adam", 5, "", 0)
    _lm(optimizer="asgd")


def test_refusals_name_the_flags():
    with pytest.raises(ValueError) as ei:
        _lm(optimizer="ntasgd")
    assert "--valid_path" in str(ei.value) and "--valid_synthetic" in str(ei.value)
    with pytest.raises(ValueError, match="--nonmono"):
        _lm(optimizer="ntasgd", valid_synthetic=8, nonmono=0)
    with pytest.raises(ValueError, match="one of them"):
        _lm(valid_synthetic=8, valid_path="v.csv")
    with pytest.raises(ValueError, match="--synthetic"):
        _lm(synthetic=0, training_path="t.csv", valid_synthetic=8)
    with pytest.raises(ValueError, match="--optimizer"):
        _lm(optimizer="rmsprop")


def test_warnings_for_flags_without_effect():
    with pytest.warns(UserWarning, match="--nonmono"):
        _lm(optimizer="asgd", nonmono=3)
    with pytest.warns(UserWarning, match="--valid_path"):
        _lm(mode="eval", valid_synthetic=8)


# ---- training runs ------------------------------------------------------------------------------------------------------------
def _run_cfg(tmp_path, name, **kw):
    base = dict(hidden_units="8,8", in_features=8, seq_len=6, batch_size=4, vocab_size=32, next_token=True, init="scaled",
                learn_initial_state=False, device="cpu", synthetic=48, valid_synthetic=12, quiet=True, partitions=1,
                optimizer="asgd", learning_rate=0.5, epochs=1, checkpoint_path=str(tmp_path / name),
                output_path=str(tmp_path / (name + "_out")))
    base.update(kw)
    return Config(**base).validate()


def _latest(path, partition=None):
    return ckpt.load(ckpt.latest_checkpoint(ckpt.find_latest_run(str(path), partition)))


def test_json_log_has_validation_and_averaging(tmp_path):
    from lstm_tensorspark_b200.trainer import run_job
    log = tmp_path / "log.jsonl"
    run_job(_run_cfg(tmp_path, "a", max_steps=6, evaluate_every=2, json_log=str(log)), standalone=True)
    evals = [r for r in map(json.loads, log.read_text().splitlines()) if "loss" in r]
    assert [r["step"] for r in evals] == [0, 2, 4, 5]
    for r in evals:
        assert math.isfinite(r["val_loss"]) and 0 <= r["val_accuracy"] <= 1
        assert r["val_perplexity"] == pytest.approx(math.exp(r["val_loss"]))
        assert r["averaging"] == 1 and r["averaged_steps"] == r["step"] + 1


def test_ntasgd_fires_prints_the_step_and_every_later_step_averages(tmp_path, capsys):
    from lstm_tensorspark_b200.trainer import run_job
    log = tmp_path / "log.jsonl"
    # a learning rate this large makes the held-out loss rise: the trigger fires at the first validation it can
    cfg = _run_cfg(tmp_path, "n", optimizer="ntasgd", nonmono=1, learning_rate=40.0, max_steps=10, evaluate_every=1,
                   json_log=str(log), quiet=False)
    run_job(cfg, standalone=True)
    evals = [r for r in map(json.loads, log.read_text().splitlines()) if "loss" in r]
    on = [r["averaging"] for r in evals]
    assert 1 in on and on[0] == 0
    first = on.index(1)
    assert all(on[first:]) and evals[first]["averaged_steps"] == 0
    assert [r["averaged_steps"] for r in evals[first:]] == list(range(len(evals) - first))
    assert f"averaging the weights from step {evals[first]['step'] + 1}" in capsys.readouterr().out


def test_resume_continues_the_average_and_the_trigger(tmp_path):
    from lstm_tensorspark_b200.trainer import run_job
    # validations at steps 0, 3, 6 (the interrupted run's last step), 9, 12 and 13 in both runs
    kw = dict(optimizer="ntasgd", nonmono=1, learning_rate=40.0, evaluate_every=3)
    run_job(_run_cfg(tmp_path, "a", max_steps=7, **kw), standalone=True)
    run_job(_run_cfg(tmp_path, "a", max_steps=14, use_pretrained_model=True, **kw), standalone=True)
    run_job(_run_cfg(tmp_path, "b", max_steps=14, **kw), standalone=True)
    va, ma, oa = _latest(tmp_path / "a")
    vb, mb, ob = _latest(tmp_path / "b")
    sa, sb = oa["optimizer"], ob["optimizer"]
    assert ma["global_step"] == mb["global_step"] == 13
    assert (sa["on"], sa["k"]) == (sb["on"], sb["k"]) and sa["on"] == 1 and sa["k"] >= 1
    assert sa["nonmono_history"] == sb["nonmono_history"] and len(sa["nonmono_history"]) == 6
    assert torch.equal(sa["ax"], sb["ax"])
    assert all(torch.equal(va[k], vb[k]) for k in va)


def test_sgd_checkpoint_resumed_under_asgd_starts_a_fresh_average_and_back_warns(tmp_path):
    from lstm_tensorspark_b200.trainer import run_job
    run_job(_run_cfg(tmp_path, "s", optimizer="sgd", max_steps=3), standalone=True)
    run_job(_run_cfg(tmp_path, "s", optimizer="asgd", max_steps=6, use_pretrained_model=True), standalone=True)
    _, _, o = _latest(tmp_path / "s")
    assert (o["optimizer"]["on"], o["optimizer"]["k"]) == (1, 3)
    with pytest.warns(UserWarning, match="dropped"):
        run_job(_run_cfg(tmp_path, "s", optimizer="sgd", max_steps=8, use_pretrained_model=True), standalone=True)
    _, _, o = _latest(tmp_path / "s")
    assert "ax" not in o["optimizer"]


def test_unfired_ntasgd_checkpoint_resumed_under_asgd_starts_a_fresh_average(tmp_path):
    """AWD's main.py under NT-ASGD, then finetune.py under ASGD: a checkpoint whose trigger never fired averages from the
    resumed run's first step, and keeps the trigger's history."""
    from lstm_tensorspark_b200.trainer import run_job
    run_job(_run_cfg(tmp_path, "u", optimizer="ntasgd", nonmono=100, max_steps=3, evaluate_every=1), standalone=True)
    _, _, o = _latest(tmp_path / "u")
    assert (o["optimizer"]["on"], o["optimizer"]["k"], len(o["optimizer"]["nonmono_history"])) == (0, 0, 3)
    run_job(_run_cfg(tmp_path, "u", optimizer="asgd", max_steps=7, evaluate_every=1, use_pretrained_model=True), standalone=True)
    _, _, o = _latest(tmp_path / "u")
    assert (o["optimizer"]["on"], o["optimizer"]["k"]) == (1, 4)
    assert len(o["optimizer"]["nonmono_history"]) == 3
    ev = run_job(_run_cfg(tmp_path, "u", mode="eval", valid_synthetic=0), standalone=True)
    assert ev["weights"] == "averaged"


def test_ntasgd_refuses_replicas_that_train_in_turn(tmp_path):
    from lstm_tensorspark_b200.trainer import run_job
    with pytest.raises(ValueError, match="cannot decide together"):
        run_job(_run_cfg(tmp_path, "o", optimizer="ntasgd", partitions=3, max_workers=1, max_steps=2), standalone=False)


def test_eval_scores_the_average_and_the_export_is_the_average(tmp_path):
    from lstm_tensorspark_b200.trainer import run_job, _find_trained_model, _averaged_variables
    cfg = _run_cfg(tmp_path, "e", max_steps=5, evaluate_every=100)
    out = run_job(cfg, standalone=False)
    _, meta, opt = _latest(tmp_path / "e", "0")
    sd = opt["optimizer"]
    assert sd["on"] == 1 and sd["k"] == 5
    # the checkpoint holds the raw iterate; --mode eval on it scores the average
    run = ckpt.find_latest_run(str(tmp_path / "e"), "0")
    ev = run_job(_run_cfg(tmp_path, "e", mode="eval", resume=run), standalone=False)
    assert ev["weights"] == "averaged"
    ev_out = run_job(_run_cfg(tmp_path, "e", mode="eval", resume=str(tmp_path / "e_out")), standalone=False)
    assert ev_out["weights"] == "averaged" and ev_out["loss"] == ev["loss"]
    # the export is ax
    blob = torch.load(tmp_path / "e_out" / "averaged_model.pt", weights_only=False)
    found = _find_trained_model(_run_cfg(tmp_path, "e", mode="eval", resume=run), False)
    expect = _averaged_variables(cfg, found[0], sd["ax"], 4)
    assert blob["meta"]["weights"] == "averaged"
    assert blob["variables"].keys() == expect.keys()
    assert all(torch.equal(blob["variables"][k], expect[k]) for k in expect)
    assert all(torch.equal(found[0][k], expect[k]) for k in expect)
    assert out["results"][0]["averaged"]


def test_sgd_eval_reports_raw_weights(tmp_path):
    from lstm_tensorspark_b200.trainer import run_job
    run_job(_run_cfg(tmp_path, "r", optimizer="sgd", max_steps=3), standalone=True)
    ev = run_job(_run_cfg(tmp_path, "r", optimizer="sgd", mode="eval"), standalone=True)
    assert ev["weights"] == "raw"


def test_validation_reads_a_file_like_training(tmp_path):
    from lstm_tensorspark_b200.trainer import run_job
    x, y = D.synthetic_next_token(10, 6, 32, seed=0, valid_of=1)
    path = tmp_path / "valid.csv"
    path.write_text("".join(",".join(str(int(v)) for v in np.concatenate([r, l[-1:]])) + "\n" for r, l in zip(x, y)))
    log = tmp_path / "log.jsonl"
    run_job(_run_cfg(tmp_path, "f", valid_synthetic=0, valid_path=str(path), max_steps=3, json_log=str(log)), standalone=True)
    evals = [r for r in map(json.loads, log.read_text().splitlines()) if "loss" in r]
    assert all(math.isfinite(r["val_loss"]) for r in evals)


def test_stateful_validation_leaves_the_carried_state_alone(tmp_path):
    from lstm_tensorspark_b200.trainer import run_job
    kw = dict(stateful=True, optimizer="sgd", max_steps=6, evaluate_every=1, learning_rate=0.1)
    run_job(_run_cfg(tmp_path, "v", **kw), standalone=True)
    run_job(_run_cfg(tmp_path, "w", valid_synthetic=0, **kw), standalone=True)
    va, _, oa = _latest(tmp_path / "v")
    vb, _, ob = _latest(tmp_path / "w")
    assert all(torch.equal(va[k], vb[k]) for k in va)
    assert all(torch.equal(h1, h2) and torch.equal(c1, c2) for (h1, c1), (h2, c2) in zip(oa["state"], ob["state"]))


def _gloo_run(rank, world, tmp):
    from lstm_tensorspark_b200 import trainer as T
    # each rank's own decision differs: rank 1 fires at its 4th validation (step 3), rank 0 never; the ranks take the max
    T.nonmono_trigger = (lambda h, v, n, averaging: not averaging and len(h) == 3) if rank == 1 else (lambda *a: False)
    cfg = _run_cfg(tmp, "g", optimizer="ntasgd", nonmono=1, learning_rate=0.5, max_steps=10, evaluate_every=1,
                   partitions=world, sync_mode="param_avg", comm="gloo")
    shards = T.load_shards(cfg, world, False)
    valid = D.load_validation(cfg, cfg.synthetic // world)
    T._rank_main(rank, world, cfg, shards, False, valid)
    run = ckpt.find_latest_run(str(tmp / "g"), str(rank))
    _, _, o = ckpt.load(ckpt.latest_checkpoint(run))
    return o["optimizer"]["on"], o["optimizer"]["k"], len(o["optimizer"]["nonmono_history"])


def test_two_gloo_ranks_fire_at_the_same_step(tmp_path):
    from lstm_tensorspark_b200.parallel.launch import launch
    r0, r1 = launch(_gloo_run, 2, args=(tmp_path,))
    assert r0 == r1 == (1, 6, 10)                      # averaging over steps 4 .. 9 on both ranks
