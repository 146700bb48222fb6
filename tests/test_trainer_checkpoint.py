"""Integration (CPU): standalone run on iris (BASELINE.json config 1), checkpoint tree, cadence,
retention, resume, compat step count (Q5), batch_size 0 (Q3)."""
import glob
import json
import os

import pytest
import torch

from lstm_tensorspark_b200.config import Config
from lstm_tensorspark_b200.trainer import compute_max_steps, run_job
from lstm_tensorspark_b200.utils import checkpoint as ckpt


def _cfg(tmp_path, iris_path, **kw):
    base = dict(training_path=iris_path, hidden_units="16", checkpoint_path=str(tmp_path / "ck"),
                output_path=str(tmp_path / "out"), device="cpu", quiet=True, epochs=3)
    base.update(kw)
    return Config(**base).validate()


def test_standalone_iris_layout_and_learning(tmp_path, iris_path):
    cfg = _cfg(tmp_path, iris_path, epochs=40, learning_rate=1e-2)
    out = run_job(cfg, standalone=True)
    res = out["results"][0]
    assert res["steps"] == 400                                   # epochs * batch_size (src/rnn.py:256)
    runs = os.listdir(cfg.checkpoint_path)
    assert len(runs) == 1 and float(runs[0]) > 0                 # <checkpoint_path>/<unix-time>/
    d = os.path.join(cfg.checkpoint_path, runs[0])
    names = set(os.listdir(d))
    assert {"params_settings", "checkpoint", "train"} <= names
    steps = sorted(int(f.split("-")[1].split(".")[0]) for f in names if f.endswith(".index"))
    assert steps == [360, 370, 380, 390, 399]                    # every evaluate_every + last step, keep 5
    assert all(f"lstm_no_spark-{s}.data-00000-of-00001" in names and f"lstm_no_spark-{s}.meta" in names for s in steps)
    assert glob.glob(os.path.join(d, "train", "events.out.tfevents.*"))
    text = open(os.path.join(d, "params_settings")).read()
    assert "HIDDEN_UNITS = 16" in text and "LEARNING_RATE = 0.01" in text
    assert ckpt.latest_checkpoint(d).endswith("lstm_no_spark-399")
    variables, meta, opt = ckpt.load(ckpt.latest_checkpoint(d))
    assert set(variables) == {f"LSTMLayer0/{n}" for n in
                              ["weights_forget_h", "weights_forget_x", "bias_forget", "weights_input_h", "weights_input_x",
                               "bias_input", "weights_C_h", "weights_C_x", "bias_C", "weights_output_h", "weights_output_x",
                               "bias_output", "state", "context_state"]} | {"Dense1/weights", "Dense1/bias"}
    assert tuple(variables["LSTMLayer0/weights_forget_x"].shape) == (4, 16)
    assert tuple(variables["LSTMLayer0/state"].shape) == (10, 16)
    assert meta["global_step"] == 399 and opt is not None
    scal = [json.loads(l) for l in open(os.path.join(d, "train", "scalars.jsonl"))]
    assert {"cross_entropy", "accuracy"} <= set(scal[0])
    assert scal[-1]["cross_entropy"] < scal[0]["cross_entropy"]  # it learns
    assert res["acc"] > 0.5


def test_resume_continues_from_last_step(tmp_path, iris_path):
    cfg = _cfg(tmp_path, iris_path, epochs=2)
    run_job(cfg, standalone=True)
    cfg2 = _cfg(tmp_path, iris_path, epochs=4, use_pretrained_model=True)
    out = run_job(cfg2, standalone=True)
    assert out["results"][0]["steps"] == 20                      # 40 total - 20 already done


def test_step_count_modes():
    cfg = Config(epochs=3, batch_size=10)
    assert compute_max_steps(cfg, 10, 15) == 30
    cfg.steps_mode = "epochs"
    assert compute_max_steps(cfg, 10, 15) == 45
    cfg.max_steps = 7
    assert compute_max_steps(cfg, 10, 15) == 7


def test_batch_size_zero_uses_whole_shard(tmp_path, iris_path):
    cfg = _cfg(tmp_path, iris_path, batch_size=0, max_steps=3)
    out = run_job(cfg, standalone=True)
    assert out["results"][0]["samples"] == 3 * 150


def test_sequence_training_synthetic_cpu(tmp_path):
    cfg = Config(synthetic=64, seq_len=5, in_features=6, num_classes=4, hidden_units="12,8", batch_size=16, max_steps=30,
                 learning_rate=1e-2, init="scaled", checkpoint_path=str(tmp_path / "ck"), output_path=str(tmp_path / "o"),
                 device="cpu", quiet=True, evaluate_every=29).validate()
    out = run_job(cfg, standalone=True)
    assert out["results"][0]["loss"] < 1.3


def test_saver_retention_and_index(tmp_path):
    s = ckpt.Saver(str(tmp_path), "spark_lstm", max_to_keep=2)
    for step in (0, 10, 20):
        s.save({"a": torch.zeros(2)}, step)
    assert sorted(f for f in os.listdir(tmp_path) if f.endswith(".index")) == ["spark_lstm-10.index", "spark_lstm-20.index"]
    idx = open(tmp_path / "checkpoint").read()
    assert 'model_checkpoint_path: "spark_lstm-20"' in idx and idx.count("all_model_checkpoint_paths") == 2


def _final_state(cfg):
    d = ckpt.find_latest_run(cfg.checkpoint_path, None)
    return ckpt.load(ckpt.latest_checkpoint(d))


@pytest.mark.parametrize("residency,bs,steps", [("device", 10, 8), ("host", 10, 8), ("host", 60, 8)])
def test_resume_is_equivalent_to_an_uninterrupted_run(tmp_path, iris_path, residency, bs, steps):
    """8 steps straight == 4 steps + resume + 4 steps, bit for bit: weights, Adam slots, step counter AND the position in
    the data order (the loader state is restored, not replayed from the first permutation).  ``host``: the pinned-memory feed
    with its prefetched-but-unconsumed batches; batch 60 of 150 rows = 2 batches per pass, so the resume point sits on a
    reshuffle boundary that the prefetch has already crossed."""
    common = dict(evaluate_every=1, learning_rate=1e-2, data_residency=residency, batch_size=bs)
    a = _cfg(tmp_path / "a", iris_path, max_steps=8, **common)
    run_job(a, standalone=True)
    va, ma, oa = _final_state(a)
    b1 = _cfg(tmp_path / "b", iris_path, max_steps=4, **common)
    run_job(b1, standalone=True)
    b2 = _cfg(tmp_path / "b", iris_path, max_steps=8, use_pretrained_model=True, **common)
    out = run_job(b2, standalone=True)
    assert out["results"][0]["steps"] == 4
    vb, mb, ob = _final_state(b2)
    assert ma["global_step"] == mb["global_step"] == 7
    for k in va:
        assert torch.equal(va[k], vb[k]), k
    assert oa["optimizer"]["step"] == ob["optimizer"]["step"] == 8
    assert torch.equal(oa["optimizer"]["m"], ob["optimizer"]["m"]) and torch.equal(oa["optimizer"]["v"], ob["optimizer"]["v"])
    key = "perm" if residency == "device" else "order"
    assert oa["loader"]["i"] == ob["loader"]["i"] and torch.equal(oa["loader"][key], ob["loader"][key])


def test_mode_eval_scores_a_trained_model(tmp_path, iris_path):
    """--mode eval: the checkpoint a standalone run left / an averaged model of a distributed run is scored on the whole file
    (full batches + the remainder), and a trained model beats an untrained one."""
    from lstm_tensorspark_b200.ops import reference as ref
    cfg = _cfg(tmp_path, iris_path, epochs=6, learning_rate=2e-2)
    run_job(cfg, standalone=True)
    ev = run_job(_cfg(tmp_path, iris_path, mode="eval", batch_size=40), standalone=True)       # 150 rows: 3 full batches + 30
    assert ev["mode"] == "eval" and ev["samples"] == 150 and 0.0 < ev["loss"] < 1.0 and ev["accuracy"] > 0.45
    whole = run_job(_cfg(tmp_path, iris_path, mode="eval", batch_size=0), standalone=True)      # one batch = the whole file
    assert whole["samples"] == 150 and abs(whole["loss"] - ev["loss"]) < 1e-5 and abs(whole["accuracy"] - ev["accuracy"]) < 1e-6
    # distributed job -> <output_path>/averaged_model.pt -> eval picks it up
    d = Config(training_path=iris_path, hidden_units="16", checkpoint_path=str(tmp_path / "ck2"), partitions=2, comm="gloo",
               output_path=str(tmp_path / "out2"), device="cpu", quiet=True, epochs=2, sync_mode="grad_allreduce",
               average_scope="all", learning_rate=2e-2, timeout_s=120).validate()
    run_job(d, standalone=False)
    d.mode = "eval"
    ev2 = run_job(d.validate(), standalone=False)
    assert ev2["model"].endswith("averaged_model.pt") and ev2["samples"] == 150 and ev2["accuracy"] > 0.4
    with pytest.raises(FileNotFoundError):
        run_job(_cfg(tmp_path / "none", iris_path, mode="eval"), standalone=True)
