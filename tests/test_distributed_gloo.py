"""Distributed tests without GPUs: world_size > 1 on CPU + gloo (our analogue of Spark ``local[N]``):
shard->rank mapping, averaging schedule, identical-weights-after-average, per-rank checkpoint layout, output_path,
per-step gradient allreduce, failure detection."""
import os

import pytest
import torch

from lstm_tensorspark_b200.config import Config
from lstm_tensorspark_b200.parallel.launch import RankFailure, launch
from lstm_tensorspark_b200.trainer import run_job


def _cfg(tmp_path, iris_path, **kw):
    base = dict(training_path=iris_path, hidden_units="16", checkpoint_path=str(tmp_path / "ck"), partitions=2,
                output_path=str(tmp_path / "out"), device="cpu", comm="gloo", quiet=True, epochs=1, timeout_s=120)
    base.update(kw)
    return Config(**base).validate()


def _avg_check(rank, world, tmpdir):
    """Each rank builds a different replica; after average_params_ all replicas are identical and equal the mean."""
    import torch
    import torch.distributed as dist
    from lstm_tensorspark_b200.config import Config
    from lstm_tensorspark_b200.models import SequenceClassifier
    from lstm_tensorspark_b200.parallel.comm import make_communicator
    comm = make_communicator("gloo", rank, world, torch.device("cpu"), 60)
    cfg = Config(hidden_units="8", in_features=4, batch_size=5)
    g = torch.Generator().manual_seed(100 + rank)
    model = SequenceClassifier(cfg, batch_size=5, generator=g)
    flat = model.build_flat()
    before = flat.data.clone()
    gathered = [torch.zeros_like(before) for _ in range(world)]
    dist.all_gather(gathered, before)
    comm.average_params_(flat, "lstm")
    lo, hi = flat.segment("lstm")
    mean = torch.stack(gathered).mean(0)
    ok_avg = torch.allclose(flat.data[lo:hi], mean[lo:hi], atol=1e-6)
    ok_head_untouched = torch.equal(flat.data[hi:], before[hi:])       # Dense head / states are NOT averaged (reference)
    after = [torch.zeros_like(before) for _ in range(world)]
    dist.all_gather(after, flat.data)
    ok_same = all(torch.equal(after[0][lo:hi], a[lo:hi]) for a in after)
    comm.close()
    return bool(ok_avg and ok_head_untouched and ok_same)


def test_param_average_invariants(tmp_path):
    assert launch(_avg_check, 3, args=(str(tmp_path),)) == [True, True, True]


def test_rnn_job_two_partitions(tmp_path, iris_path):
    cfg = _cfg(tmp_path, iris_path)
    out = run_job(cfg, standalone=False)
    assert out["world_size"] == 2
    runs = os.listdir(cfg.checkpoint_path)
    assert len(runs) == 1                                   # ONE shared run timestamp (rank 0 broadcasts it)
    assert sorted(os.listdir(os.path.join(cfg.checkpoint_path, runs[0]))) == ["0", "1"]
    d0 = os.path.join(cfg.checkpoint_path, runs[0], "0")
    assert {"params_settings", "checkpoint", "train", "spark_lstm-9.index"} <= set(os.listdir(d0))
    avg = torch.load(os.path.join(cfg.output_path, "averaged_model.pt"), weights_only=False)
    assert list(avg["records"].keys()) == ["wf", "wi", "wo", "wc", "bf", "bi", "bc", "bo"]
    assert tuple(avg["records"]["wf"][0][0].shape) == (16, 16) and tuple(avg["records"]["wf"][0][1].shape) == (4, 16)


def _grad_sync_check(rank, world, iris_path):
    """Per-step gradient allreduce keeps replicas bit-identical when they start identical."""
    import torch
    import torch.distributed as dist
    from lstm_tensorspark_b200 import data as D
    from lstm_tensorspark_b200.config import Config
    from lstm_tensorspark_b200.engine import TrainEngine
    from lstm_tensorspark_b200.parallel.comm import make_communicator
    dev = torch.device("cpu")
    comm = make_communicator("gloo", rank, world, dev, 60)
    cfg = Config(hidden_units="8,8", in_features=4, batch_size=6, seq_len=3, sync_mode="grad_allreduce", device="cpu",
                 learn_initial_state=False, init="scaled", partitions=world)
    eng = TrainEngine(cfg, rank, world, comm, batch_size=6, device=dev, dtype=torch.float32)
    x, y = D.synthetic_sequences(6, 3, 4, 3, seed=rank)
    for _ in range(4):
        eng.step(torch.as_tensor(x), torch.as_tensor(y))
    all_w = [torch.zeros_like(eng.flat.data) for _ in range(world)]
    dist.all_gather(all_w, eng.flat.data)
    comm.close()
    return bool(all(torch.equal(all_w[0], w) for w in all_w))


def test_grad_allreduce_keeps_replicas_identical(iris_path):
    assert launch(_grad_sync_check, 2, args=(iris_path,)) == [True, True]


def test_rank_failure_is_an_error_not_a_hang(tmp_path, iris_path):
    cfg = _cfg(tmp_path, iris_path, fault_inject="1:3", timeout_s=30)
    with pytest.raises(RankFailure) as ei:
        run_job(cfg, standalone=False)
    assert ei.value.exit_codes[1] == 17


def test_more_partitions_than_workers_round_robin(tmp_path, iris_path, capfd):
    """--partitions 4 on 2 workers (Spark local[2] with 4 tasks, original src/rnn.py:355-358): every partition gets
    its own replica + checkpoint dir, ranks take their partitions in turn, the final average runs over all 4."""
    cfg = _cfg(tmp_path, iris_path, partitions=4, max_workers=2)
    out = run_job(cfg, standalone=False)
    assert out["world_size"] == 2 and out["partitions"] == 4
    assert "4 partitions on 2 workers" in capfd.readouterr().err
    runs = os.listdir(cfg.checkpoint_path)
    assert len(runs) == 1
    assert sorted(os.listdir(os.path.join(cfg.checkpoint_path, runs[0]))) == ["0", "1", "2", "3"]
    avg = torch.load(os.path.join(cfg.output_path, "averaged_model.pt"), weights_only=False)
    # the exported average equals the mean of the four replicas' final checkpoints
    from lstm_tensorspark_b200.utils import checkpoint as ckpt
    finals = [ckpt.load(ckpt.latest_checkpoint(os.path.join(cfg.checkpoint_path, runs[0], str(k))))[0] for k in range(4)]
    mean_wf_h = torch.stack([f["LSTMLayer0/weights_forget_h"] for f in finals]).mean(0)
    assert torch.allclose(avg["records"]["wf"][0][0], mean_wf_h, atol=1e-6)
    assert out["results"][0]["partitions_trained"] == [0, 2] and out["results"][1]["partitions_trained"] == [1, 3]


def test_oversubscription_needs_the_one_shot_average(tmp_path, iris_path):
    cfg = _cfg(tmp_path, iris_path, partitions=4, max_workers=2, sync_mode="grad_allreduce")
    with pytest.raises(ValueError):
        run_job(cfg, standalone=False)


def test_host_resident_feed_matches_the_device_resident_one(tmp_path, iris_path):
    """--data_residency host (pinned host shard, every batch copied to the device by the prefetch pipeline - the reference's
    per-step feed) draws the same batches as the device-resident gather: two ranks, per-step gradient allreduce, same result."""
    outs = {}
    for res in ("device", "host"):
        cfg = _cfg(tmp_path / res, iris_path, sync_mode="grad_allreduce", average_scope="all", max_steps=6, batch_size=15,
                   data_residency=res, evaluate_every=5)
        out = run_job(cfg, standalone=False)
        outs[res] = [r["loss"] for r in out["results"]]
        assert out["world_size"] == 2 and all(r["steps"] == 6 for r in out["results"])
    # both loaders permute a pass with torch.randperm from the same seeded generator -> identical batches -> identical losses
    assert outs["device"] == pytest.approx(outs["host"], rel=1e-6)
