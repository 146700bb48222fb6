"""The gradient buckets against the kernels backward still runs, on one GPU.

With ``--sync_mode grad_allreduce`` the engine syncs and updates the flat buffer one bucket at a time, in place, while backward
still runs.  Here a fake communicator stands in for the fused allreduce and update: at each ``launch_bucket``, in stream order,
it snapshots the bucket's gradient and overwrites the bucket's weights and bf16 shadow with NaN, as an update would change them.
One eager ``--deterministic`` step must then give the loss of the same step without buckets (to the last bits, which the head's
atomic loss sum leaves free), every snapshot must be that step's gradient bitwise, and no gradient may hold a NaN: no bucket is
launched before the last kernel that writes its gradient or reads its weights.  Each case asserts through ``STATS`` that the
path it is about ran."""
import pytest
import torch

from lstm_tensorspark_b200.parallel.comm import Communicator

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)


class _NaNUpdate(Communicator):
    """A two-rank communicator that replaces each bucket's update with NaN and records what the bucket would have read."""

    def __init__(self):
        super().__init__(0, 2)
        self.launches = []              # (lo, hi, our kernels launched in backward before it, snapshot of the gradient)

    def begin_grad_step(self, flat, optimizer):
        from lstm_tensorspark_b200.ops.cuda_ext import LAUNCHES
        self.flat, self.n0 = flat, LAUNCHES["n"]

    def launch_bucket(self, lo, hi, **_kw):
        from lstm_tensorspark_b200.ops.cuda_ext import LAUNCHES
        f = self.flat
        self.launches.append((lo, hi, LAUNCHES["n"] - self.n0, f.grad[lo:hi].clone()))
        f.data[lo:hi].fill_(float("nan"))
        f.shadow[lo:hi].fill_(float("nan"))


CASES = {
    # two single-layer ops (B != 256: no layer pair); the top one computes dX through its W_x
    "two_layers_dx": (dict(hidden_units="128,128", in_features=64, seq_len=8, batch_size=128), {"fast_bwd": 2}),
    # a wavefront pair whose dX goes into the embedding table
    "next_token_pair": (dict(hidden_units="256,256", in_features=256, seq_len=16, batch_size=256, vocab_size=1024,
                             num_classes=1024, next_token=True), {"wavefront_fwd": 1, "embed_bwd": 1, "vocab_head_bwd": 1}),
    # more batch tiles than fit the device: the layer runs in batch chunks that add to one gradient (8 classes: the head's
    # backward then takes all 1024 rows in one slab, without the atomics that would make its own gradient differ in the last bits)
    "batch_chunks": (dict(hidden_units="1024", in_features=256, seq_len=4, batch_size=1024, num_classes=8), {"batch_chunks": 2}),
    "headline": (dict(hidden_units="1024,1024", in_features=1024, seq_len=128, batch_size=256), {"pipelined_fwd": 1}),
    "headline_weight_drop": (dict(hidden_units="1024,1024", in_features=1024, seq_len=128, batch_size=256, weight_drop=0.5),
                             {"pipelined_fwd": 1, "weight_drop_grad": 2}),
    "wavefront_weight_drop": (dict(hidden_units="256,256", in_features=256, seq_len=16, batch_size=256, weight_drop=0.5),
                              {"wavefront_fwd": 1, "weight_drop_grad": 2}),
}


def _engine(kw, world, comm=None):
    from lstm_tensorspark_b200.config import Config
    from lstm_tensorspark_b200.engine import TrainEngine
    cfg = Config(**{**dict(num_classes=10, partitions=world, sync_mode="grad_allreduce" if comm else "none", grad_buckets=True,
                           init="scaled", learn_initial_state=False, device="cuda", deterministic=True, quiet=True, seed=7), **kw})
    return TrainEngine(cfg, 0, world, comm, batch_size=cfg.batch_size, device=DEV, dtype=torch.bfloat16)


def _batch(cfg):
    from lstm_tensorspark_b200 import data as D
    if cfg.vocab_size:
        x, y = D.synthetic_next_token(cfg.batch_size, cfg.seq_len, cfg.vocab_size, seed=3)[:2]
        return torch.as_tensor(x).to(DEV), torch.as_tensor(y).to(DEV)
    x, y = D.synthetic_sequences(cfg.batch_size, cfg.seq_len, cfg.in_features, cfg.num_classes, seed=3)
    return torch.as_tensor(x).to(DEV, torch.bfloat16), torch.as_tensor(y).to(DEV)


@pytest.mark.parametrize("case", list(CASES))
def test_no_bucket_updates_what_backward_still_needs(case, monkeypatch):
    from lstm_tensorspark_b200.ops import cuda_lstm
    monkeypatch.setattr(cuda_lstm, "SEQ_VARIANT", cuda_lstm.SEQ_VARIANT)     # (--deterministic sets it)
    kw, path = CASES[case]
    ref = _engine(kw, 1)
    x, y = _batch(ref.cfg)
    want = ref.step(x, y)
    comm = _NaNUpdate()
    eng = _engine(kw, 2, comm)
    assert eng._bucket_plan is not None and len(eng._bucket_plan) >= 2
    n0 = {k: cuda_lstm.STATS.get(k, 0) for k in path}
    got = eng.step(x, y)
    torch.cuda.synchronize()
    ran = {k: cuda_lstm.STATS.get(k, 0) - n0[k] for k in path}
    assert all(ran[k] >= n for k, n in path.items()), ran
    print(f"bucket launches of {case}: {[(lo, hi, pos) for lo, hi, pos, _ in comm.launches]}")
    assert sorted((lo, hi) for lo, hi, _, _ in comm.launches) == sorted((b["lo"], b["hi"]) for b in eng._bucket_plan)
    assert abs(float(got) - float(want)) <= 1e-6 * abs(float(want)), (float(got), float(want))
    assert not bool(torch.isnan(eng.flat.grad).any())
    for lo, hi, pos, g in comm.launches:
        assert torch.equal(g, ref.flat.grad[lo:hi]), (case, lo, hi, pos)
    cuda_lstm.check_kernel_errors(DEV)
