"""Gradient clipping by the global norm (``--clip_grad_norm``) on the CPU: the reference norm and coefficient against
``torch.nn.utils.clip_grad_norm_``, whole ``TrainEngine`` steps against a hand-written loop (backward, L2 term, clip_grad_norm_,
plain update), an inactive clip giving the bits of no clip, the flag's errors and the communicator it selects, a 2-rank gloo
``grad_allreduce`` run, and the standalone CLI's logs."""
import json
import math
import os
import subprocess
import sys

import pytest
import torch

from lstm_tensorspark_b200 import data as D
from lstm_tensorspark_b200.config import FUSED_CLIP_ERROR, Config, parse_args
from lstm_tensorspark_b200.ops import reference as ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---- reference -----------------------------------------------------------------------------------------------------------------
def _torch_clip(segments, max_norm):
    """clip_grad_norm_ over parameters whose gradients are ``segments`` (fp64) -> (norm, clipped gradients)."""
    ps = [torch.nn.Parameter(torch.zeros_like(s)) for s in segments]
    for p, s in zip(ps, segments):
        p.grad = s.clone()
    norm = torch.nn.utils.clip_grad_norm_(ps, max_norm)
    return norm, [p.grad for p in ps]


@pytest.mark.parametrize("case", ["random", "zeros", "huge", "inf", "nan", "inactive"])
def test_reference_matches_clip_grad_norm(case):
    gen = torch.Generator().manual_seed(3)
    segs = [torch.randn(37, generator=gen, dtype=torch.float64), torch.randn(5, 4, generator=gen, dtype=torch.float64) * 1e-3]
    max_norm = 0.5
    if case == "zeros":
        segs = [torch.zeros_like(s) for s in segs]
    elif case == "huge":
        segs = [s * 1e150 for s in segs]
    elif case == "inf":
        segs[1][2, 1] = float("inf")
    elif case == "nan":
        segs[0][7] = float("nan")
    elif case == "inactive":
        max_norm = 1e30
    norm, coef = ref.clip_coefficient(segs, max_norm)
    want_norm, want = _torch_clip(segs, max_norm)
    assert norm.dtype == coef.dtype == torch.float64
    if case == "nan":
        assert math.isnan(norm) and math.isnan(coef)
    elif case == "inf":
        assert math.isinf(norm) and float(coef) == 0.0
    else:
        assert math.isclose(float(norm), float(want_norm), rel_tol=1e-13)
        for s, w in zip(segs, want):
            assert torch.allclose(s * coef, w, rtol=1e-13, atol=0)
    if case in ("zeros", "inactive"):
        assert float(coef) == 1.0
    elif case in ("random", "huge"):
        assert float(coef) < 1.0


def test_reference_update_with_coef_one_is_the_plain_update():
    gen = torch.Generator().manual_seed(0)
    p, g = torch.randn(64, generator=gen), torch.randn(64, generator=gen)
    m, v = torch.zeros(64), torch.zeros(64)
    a = [t.clone() for t in (p, m, v)]
    b = [t.clone() for t in (p, m, v)]
    ref.adam_step_(a[0], g, a[1], a[2], 1, 1e-2, weight_decay=0.1, grad_scale=0.5)
    ref.adam_step_(b[0], g, b[1], b[2], 1, 1e-2, weight_decay=0.1, grad_scale=0.5, clip_coef=torch.tensor(1.0))
    assert all(torch.equal(x, y) for x, y in zip(a, b))


# ---- engine steps ----------------------------------------------------------------------------------------------------------------
def _cfg(**kw):
    base = dict(hidden_units="6,5", in_features=3, seq_len=4, batch_size=5, num_classes=3, device="cpu", init="scaled",
                learning_rate=1e-2, quiet=True, partitions=1, sync_mode="none")
    base.update(kw)
    return Config(**base).validate()


def _batches(n, seed=0, B=5, T=4, F=3, C=3, scale=1.0):
    gen = torch.Generator().manual_seed(seed)
    return [(torch.randn(B, T, F, generator=gen) * scale, torch.randint(0, C, (B,), generator=gen)) for _ in range(n)]


def _engine(cfg):
    from lstm_tensorspark_b200.engine import TrainEngine
    return TrainEngine(cfg, 0, 1, None, batch_size=cfg.batch_size, device=torch.device("cpu"), dtype=torch.float32)


def _hand_step(eng, x, y, max_norm, t):
    """One step of ``eng``'s model by hand: backward of the loss with the autograd L2 terms of the variables outside the LSTM
    segment, the L2 gradient wd * p added over the LSTM segment, torch's clip_grad_norm_, then the reference update without
    weight decay.  -> the norm clip_grad_norm_ returned."""
    from lstm_tensorspark_b200.models.recurrent.lstm import weight_decay_collection
    fl, opt, cfg = eng.flat, eng.optimizer, eng.cfg
    seg = {id(p) for p in eng.model.rnn.averaged_parameters()}
    fl.zero_grad()
    loss, _, _ = eng.model(x, y)
    extra = [fn(v) * wd for (v, fn, wd) in weight_decay_collection() if id(v) not in seg]
    if extra:
        loss = loss + torch.stack(extra).sum()
    loss.backward()
    fl.finalize_grads()
    with torch.no_grad():
        g = fl.grad.clone()
        g[:fl.lstm_numel] += cfg.weight_decay * fl.data[:fl.lstm_numel]
        holder = torch.nn.Parameter(fl.data.clone())
        holder.grad = g
        norm = torch.nn.utils.clip_grad_norm_([holder], max_norm)
        if cfg.optimizer == "adam":
            ref.adam_step_(fl.data, holder.grad, opt.m, opt.v, t, cfg.learning_rate)
        else:
            ref.sgd_step_(fl.data, holder.grad, cfg.learning_rate)
    return float(norm)


@pytest.mark.parametrize("optimizer", ["adam", "sgd"])
def test_engine_steps_match_a_hand_written_loop(optimizer):
    """Adam and SGD, weight decay (in the update over the LSTM segment, by autograd on the learned initial states), active clip."""
    max_norm = 0.05
    kw = dict(optimizer=optimizer, weight_decay=0.01, learn_initial_state=True, seq_len=4)
    eng = _engine(_cfg(clip_grad_norm=max_norm, **kw))
    hand = _engine(_cfg(**kw))                 # same seed: same initial weights; its own step() is never called
    assert torch.equal(eng.flat.data, hand.flat.data)
    assert len(hand._wd_autograd) > 0          # the learned initial states carry an autograd L2 term
    for t, (x, y) in enumerate(_batches(4, seed=1), start=1):
        eng.step(x, y)
        want = _hand_step(hand, x, y, max_norm, t)
        got = float(eng.grad_norm())
        assert math.isclose(got, want, rel_tol=1e-5), (t, got, want)
        assert float(eng.optimizer.clip_out[1]) < 1.0                   # the clip is active
        assert torch.allclose(eng.flat.data, hand.flat.data, rtol=1e-5, atol=1e-6), t
        if optimizer == "adam":
            assert torch.allclose(eng.optimizer.m, hand.optimizer.m, rtol=1e-4, atol=1e-8)
            assert torch.allclose(eng.optimizer.v, hand.optimizer.v, rtol=1e-4, atol=1e-10)


@pytest.mark.parametrize("optimizer", ["adam", "sgd"])
def test_inactive_clip_gives_the_bits_of_no_clip(optimizer):
    kw = dict(optimizer=optimizer, weight_decay=0.01, learn_initial_state=True)
    a, b = _engine(_cfg(clip_grad_norm=1e30, **kw)), _engine(_cfg(**kw))
    assert b.grad_norm() is None
    for x, y in _batches(3, seed=2):
        la, lb = a.step(x, y), b.step(x, y)
        assert torch.equal(la, lb)
        assert float(a.optimizer.clip_out[1]) == 1.0 and float(a.grad_norm()) > 0
    assert torch.equal(a.flat.data, b.flat.data)
    if optimizer == "adam":
        assert torch.equal(a.optimizer.m, b.optimizer.m) and torch.equal(a.optimizer.v, b.optimizer.v)


# ---- flag ---------------------------------------------------------------------------------------------------------------------------
def test_flag_validation_and_comm_resolution():
    from lstm_tensorspark_b200.parallel.comm import Communicator, resolve_comm
    assert parse_args([]).clip_grad_norm == 0.0
    assert parse_args(["--clip_grad_norm", "1.5"]).clip_grad_norm == 1.5
    for bad in ("-1", "nan", "inf"):
        with pytest.raises(ValueError, match="--clip_grad_norm"):
            parse_args(["--clip_grad_norm", bad])
    grad_ar = dict(clip_grad_norm=1.0, sync_mode="grad_allreduce", partitions=2)
    with pytest.raises(ValueError, match="--comm nccl"):
        Config(comm="fused", **grad_ar).validate()
    for ok in (dict(grad_ar, comm="nccl"), dict(grad_ar, comm="auto"), dict(grad_ar, comm="fused", partitions=1),
               dict(grad_ar, comm="fused", sync_mode="param_avg"), dict(grad_ar, comm="fused", clip_grad_norm=0.0)):
        Config(**ok).validate()
    assert Config(comm="auto", **grad_ar).clips_synced_grads()
    assert not Config(comm="auto", **dict(grad_ar, sync_mode="param_avg")).clips_synced_grads()
    cuda, cpu = torch.device("cuda"), torch.device("cpu")
    assert resolve_comm("auto", cuda, clip_synced_grads=True) == "nccl"
    assert resolve_comm("auto", cuda, clip_synced_grads=False) == "fused"
    assert resolve_comm("auto", cpu, clip_synced_grads=True) == "gloo"
    assert resolve_comm("fused", cuda, clip_synced_grads=False) == "fused"

    class FusedLike(Communicator):              # what TrainEngine sees of parallel.fused_comm.FusedComm
        name = "fused"
    from lstm_tensorspark_b200.engine import TrainEngine
    cfg = _cfg(clip_grad_norm=1.0, sync_mode="grad_allreduce")
    with pytest.raises(ValueError) as e:
        TrainEngine(cfg, 0, 2, FusedLike(0, 2), batch_size=5, device=torch.device("cpu"))
    assert str(e.value) == FUSED_CLIP_ERROR
    TrainEngine(_cfg(clip_grad_norm=1.0, sync_mode="param_avg"), 0, 2, FusedLike(0, 2), batch_size=5, device=torch.device("cpu"))


# ---- two ranks ----------------------------------------------------------------------------------------------------------------------
def _grad_clip_sync_check(rank, world):
    import torch.distributed as dist
    from lstm_tensorspark_b200.engine import TrainEngine
    from lstm_tensorspark_b200.parallel.comm import make_communicator
    dev = torch.device("cpu")
    comm = make_communicator("gloo", rank, world, dev, 60)
    kw = dict(hidden_units="8,8", in_features=4, batch_size=6, seq_len=5, sync_mode="grad_allreduce", device="cpu",
              learn_initial_state=False, init="scaled", partitions=world, weight_decay=0.01, quiet=True)
    eng = TrainEngine(Config(clip_grad_norm=0.05, **kw), rank, world, comm, batch_size=6, device=dev, dtype=torch.float32)
    local = TrainEngine(Config(**kw), rank, world, None, batch_size=6, device=dev, dtype=torch.float32)   # gradients by hand
    ok = []
    for x, y in _batches(4, seed=10 + rank, B=6, T=5, F=4):
        local.flat.data.copy_(eng.flat.data)
        local.flat.zero_grad()
        local.model(x, y)[0].backward()
        local.flat.finalize_grads()
        grads = [torch.zeros_like(local.flat.grad) for _ in range(world)]
        dist.all_gather(grads, local.flat.grad)
        avg = torch.stack([g.double() for g in grads]).mean(0)
        avg[:local.flat.lstm_numel] += 0.01 * local.flat.data[:local.flat.lstm_numel].double()
        eng.step(x, y)
        ok.append(math.isclose(float(eng.grad_norm()), float(avg.norm()), rel_tol=1e-5))
        ok.append(float(eng.optimizer.clip_out[1]) < 1.0)
    all_w = [torch.zeros_like(eng.flat.data) for _ in range(world)]
    dist.all_gather(all_w, eng.flat.data)
    ok.append(all(torch.equal(all_w[0], w) for w in all_w))
    comm.close()
    return all(ok)


def test_two_rank_grad_allreduce_clips_the_averaged_gradient():
    from lstm_tensorspark_b200.parallel.launch import launch
    assert launch(_grad_clip_sync_check, 2) == [True, True]


# ---- CLI ----------------------------------------------------------------------------------------------------------------------------
def _json_lines(path):
    return [json.loads(s) for s in open(path)] if os.path.isfile(path) else []


@pytest.mark.parametrize("clip", [0.0, 0.5])
def test_cli_logs_grad_norm_at_evaluation_steps(tmp_path, clip):
    from lstm_tensorspark_b200.trainer import run_job
    log = str(tmp_path / "log.jsonl")
    base = dict(synthetic=60, hidden_units="12", in_features=3, seq_len=5, num_classes=3, batch_size=10,
                checkpoint_path=str(tmp_path / "ck"), output_path=str(tmp_path / "out"), device="cpu", quiet=True,
                learning_rate=2e-2, steps_mode="epochs", evaluate_every=4, json_log=log, clip_grad_norm=clip)
    flags = [f"--{k}={v}" for k, v in dict(base, epochs=2).items()]
    r = subprocess.run([sys.executable, os.path.join(ROOT, "lstm-no-spark.py")] + flags, capture_output=True, text=True,
                       timeout=600, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-3000:]
    out2 = run_job(Config(epochs=3, use_pretrained_model=True, **base).validate(), standalone=True)
    assert out2["results"][0]["steps"] == 6                                       # 18 total - 12 already done
    run_job(Config(mode="eval", **base).validate(), standalone=True)
    lines = _json_lines(log)
    steps = [l for l in lines if "step" in l]
    assert [l["step"] for l in steps] == [0, 4, 8, 11, 12, 16, 17]
    if clip:
        assert all(math.isfinite(l["grad_norm"]) and l["grad_norm"] > 0 for l in steps)
        assert all("grad_norm" not in l for l in lines if "step" not in l)            # done / eval lines
        run = sorted(os.listdir(base["checkpoint_path"]))[0]
        scal = _json_lines(os.path.join(base["checkpoint_path"], run, "train", "scalars.jsonl"))
        assert [s["grad_norm"] for s in scal] == [l["grad_norm"] for l in steps[:4]]
    else:
        assert not any("grad_norm" in l for l in lines)
    assert any(l.get("mode") == "eval" for l in lines)
