"""NT-ASGD on the GPU (csrc/multi_tensor_opt.cu flat_asgd_kernel, flat_average_kernel, flat_swap_kernel): the fused update against
fp64 with ax bit-exact to torch's fp32 expression on the kernel's own p at k = 1, 2, 3 and a large k, with and without clipping and
the weight-decay cut; averaging off as flat_sgd bit for bit; the standalone average as the fused one; two swaps as the identity; a
captured graph replayed across a trigger flip as the eager steps; validation that leaves training bitwise alone; a short ntasgd
run whose trigger fires; the standalone average after the fused allreduce's gradient buckets, inside a captured step (one GPU),
and ``--comm fused`` against ``--comm nccl`` (two GPUs or more, skipped otherwise)."""
import json

import pytest
import torch

import lstm_numerics as N

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
N_ELEMS = 4 * 100003             # not a multiple of the grid's stride: the grid-stride tail runs


@pytest.fixture(scope="module")
def E():
    from lstm_tensorspark_b200.ops.cuda_ext import ext
    return ext()


def _state(n=N_ELEMS, seed=0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    p = torch.randn(n, device=DEV, generator=g)
    grad = torch.randn(n, device=DEV, generator=g)
    ax = torch.randn(n, device=DEV, generator=g)
    return p, grad, ax


def _torch_average(ax, p, k):
    """torch.optim.ASGD's fp32 averaging step k (ops/reference.asgd_average_) on the GPU."""
    from lstm_tensorspark_b200.ops import reference as ref
    out = ax.clone()
    return ref.asgd_average_(out, p, k)


@pytest.mark.parametrize("k", [1, 2, 3, 1000])
@pytest.mark.parametrize("clip", [False, True])
@pytest.mark.parametrize("wd_numel", [-1, 4 * 30000])
def test_fused_update_and_average(E, k, clip, wd_numel):
    lr, wd, gscale = 0.05, 0.01, 0.5
    p, g, ax = _state()
    p0, ax0 = p.clone(), ax.clone()
    shadow = torch.empty(p.numel(), dtype=torch.bfloat16, device=DEV)
    avg = torch.tensor([1, k - 1], dtype=torch.int32, device=DEV)
    clip_out = None
    if clip:                                           # a clip that is active: the norm kernel's coef < 1
        clip_out = torch.zeros(2, dtype=torch.float32, device=DEV)
        scratch = torch.zeros(E.flat_grad_norm_scratch(p.numel()), dtype=torch.float64, device=DEV)
        E.flat_grad_norm(g, p, clip_out, scratch, 10.0, wd, gscale, wd_numel)
        assert float(clip_out[1]) < 1.0
    E.flat_asgd(p, g, ax, avg, shadow, lr, wd, gscale, wd_numel, clip_out)
    torch.cuda.synchronize()
    assert avg.tolist() == [1, k]
    # p: flat_sgd's bits (and so its fp64 bound); without the clip also against fp64 directly
    ps, ss = p0.clone(), torch.empty_like(shadow)
    E.flat_sgd(ps, g, ss, lr, wd, gscale, wd_numel, clip_out)
    assert torch.equal(p, ps) and torch.equal(shadow.view(torch.int16), ss.view(torch.int16))
    if not clip:
        ref = N.sgd_update(p0, g, lr, wd, gscale, wd_numel)
        N.check_update("p", p, ref.p, ref.bound_p)
    N.check_shadow("shadow", shadow, p)
    # ax: bit-exact to torch's fp32 expression on the kernel's own p
    assert torch.equal(ax, _torch_average(ax0, p, k))


def test_averaging_off_is_flat_sgd_and_leaves_ax(E):
    for clip in (False, True):
        p, g, ax = _state(seed=1)
        p0, ax0 = p.clone(), ax.clone()
        shadow, ss = (torch.empty(p.numel(), dtype=torch.bfloat16, device=DEV) for _ in range(2))
        avg = torch.tensor([0, 7], dtype=torch.int32, device=DEV)
        clip_out = torch.tensor([0.0, 0.3], dtype=torch.float32, device=DEV) if clip else None
        E.flat_asgd(p, g, ax, avg, shadow, 0.1, 0.02, 1.0, -1, clip_out)
        ps = p0.clone()
        E.flat_sgd(ps, g, ss, 0.1, 0.02, 1.0, -1, clip_out)
        torch.cuda.synchronize()
        assert torch.equal(p, ps) and torch.equal(shadow.view(torch.int16), ss.view(torch.int16))
        assert torch.equal(ax, ax0) and avg.tolist() == [0, 7]


@pytest.mark.parametrize("k", [1, 2, 3, 57])
def test_standalone_average_is_the_fused_one(E, k):
    p, g, ax = _state(seed=2)
    ax0 = ax.clone()
    shadow = torch.empty(p.numel(), dtype=torch.bfloat16, device=DEV)
    avg = torch.tensor([1, k - 1], dtype=torch.int32, device=DEV)
    E.flat_asgd(p, g, ax, avg, shadow, 0.1, 0.0, 1.0)
    ax2 = ax0.clone()
    avg2 = torch.tensor([1, k - 1], dtype=torch.int32, device=DEV)
    E.flat_average(p, ax2, avg2)
    off = torch.tensor([0, k - 1], dtype=torch.int32, device=DEV)
    ax3 = ax0.clone()
    E.flat_average(p, ax3, off)
    torch.cuda.synchronize()
    assert torch.equal(ax, ax2) and avg2.tolist() == [1, k]
    assert torch.equal(ax3, ax0) and off.tolist() == [0, k - 1]


def test_two_swaps_are_the_identity(E):
    p, _, ax = _state(seed=3)
    shadow = p.to(torch.bfloat16)
    p0, ax0, s0 = p.clone(), ax.clone(), shadow.clone()
    E.flat_swap(p, ax, shadow)
    torch.cuda.synchronize()
    assert torch.equal(p, ax0) and torch.equal(ax, p0)
    N.check_shadow("swapped shadow", shadow, p)
    E.flat_swap(p, ax, shadow)
    torch.cuda.synchronize()
    assert torch.equal(p, p0) and torch.equal(ax, ax0) and torch.equal(shadow.view(torch.int16), s0.view(torch.int16))


# ---- whole steps --------------------------------------------------------------------------------------------------------------
def _engine(kind, **kw):
    from lstm_tensorspark_b200.config import Config
    from lstm_tensorspark_b200.engine import TrainEngine
    base = dict(hidden_units="128,128", in_features=64, seq_len=16, batch_size=64, vocab_size=512, next_token=True, init="scaled",
                learn_initial_state=False, device="cuda", quiet=True, optimizer=kind, learning_rate=0.5, weight_decay=1e-4,
                clip_grad_norm=0.5, deterministic=True, sync_mode="none", partitions=1)
    base.update(kw)
    cfg = Config(**base)
    torch.cuda.set_device(0)
    return TrainEngine(cfg, 0, 1, None, batch_size=cfg.batch_size, device=DEV, dtype=torch.bfloat16)


def _batches(n, seed=0):
    from lstm_tensorspark_b200 import data as D
    x, y = D.synthetic_next_token(64 * n, 16, 512, seed=seed)
    return [(torch.as_tensor(x[i * 64:(i + 1) * 64]).to(DEV), torch.as_tensor(y[i * 64:(i + 1) * 64]).to(DEV)) for i in range(n)]


def test_graph_replays_equal_eager_steps_across_a_trigger_flip():
    batches = _batches(12)
    eager, graph = _engine("ntasgd"), _engine("ntasgd")
    before = (graph.flat.data.clone(), graph.optimizer.ax.clone(), graph.optimizer.avg.clone())
    graph.capture(*batches[0])
    torch.cuda.synchronize()
    assert torch.equal(graph.flat.data, before[0]) and torch.equal(graph.optimizer.ax, before[1])
    assert torch.equal(graph.optimizer.avg, before[2])                # capturing does not advance the average
    for i, (x, y) in enumerate(batches[:10]):
        if i == 4:                                                    # the trigger fires between replays: no recapture
            eager.optimizer.start_averaging()
            graph.optimizer.start_averaging()
        eager.step(x, y)
        graph.step(x, y)
    torch.cuda.synchronize()
    assert torch.equal(eager.flat.data, graph.flat.data)
    assert torch.equal(eager.optimizer.ax, graph.optimizer.ax)
    assert eager.optimizer.avg.tolist() == graph.optimizer.avg.tolist() == [1, 6]
    # evaluation on the average puts the raw weights and their shadow back bit for bit
    w, s = graph.flat.data.clone(), graph.flat.shadow.clone()
    with graph.averaged_weights() as swapped:
        assert swapped and torch.equal(graph.flat.data, eager.optimizer.ax)
        graph.evaluate(*batches[11])
    torch.cuda.synchronize()
    assert torch.equal(graph.flat.data, w) and torch.equal(graph.flat.shadow.view(torch.int16), s.view(torch.int16))
    # ... and scores what a model holding ax as its weights scores: no derived copy of the weights goes stale
    fresh = _engine("sgd")
    with torch.no_grad():
        fresh.flat.data.copy_(graph.optimizer.ax)
        fresh.flat.refresh_shadow()
    with graph.averaged_weights():
        got = graph.evaluate(*batches[11])
    want = fresh.evaluate(*batches[11])
    assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1])


def _run_cfg(tmp_path, name, **kw):
    from lstm_tensorspark_b200.config import Config
    base = dict(next_token=True, vocab_size=512, seq_len=16, batch_size=64, hidden_units="128,128", in_features=64,
                synthetic=640, device="cuda", quiet=True, init="scaled", learning_rate=0.5, optimizer="sgd", deterministic=True,
                cuda_graph=True, learn_initial_state=False, partitions=1, evaluate_every=3, epochs=1,
                checkpoint_path=str(tmp_path / name), output_path=str(tmp_path / (name + "_out")))
    base.update(kw)
    return Config(**base).validate()


def _latest(path):
    from lstm_tensorspark_b200.utils import checkpoint as ckpt
    return ckpt.load(ckpt.latest_checkpoint(ckpt.find_latest_run(str(path), None)))


@pytest.mark.parametrize("stateful", [False, True])
def test_validation_leaves_training_bitwise_alone(tmp_path, stateful):
    from lstm_tensorspark_b200.trainer import run_job
    kw = dict(stateful=stateful, max_steps=9, dropout=0.1)
    run_job(_run_cfg(tmp_path, "v", valid_synthetic=200, **kw), standalone=True)
    run_job(_run_cfg(tmp_path, "n", **kw), standalone=True)
    va, _, oa = _latest(tmp_path / "v")
    vb, _, ob = _latest(tmp_path / "n")
    assert all(torch.equal(va[k], vb[k]) for k in va)
    if stateful:
        assert all(torch.equal(h1, h2) and torch.equal(c1, c2) for (h1, c1), (h2, c2) in zip(oa["state"], ob["state"]))


def test_ntasgd_run_fires_and_exports_the_average(tmp_path):
    import numpy as np
    from lstm_tensorspark_b200 import data as D
    from lstm_tensorspark_b200.trainer import run_job
    # held out: walks of another chain (seed 99), whose loss rises as the model learns the training chain: the trigger fires
    x, y = D.synthetic_next_token(128, 16, 512, seed=99)
    path = tmp_path / "valid.csv"
    path.write_text("".join(",".join(str(int(v)) for v in np.concatenate([r, l[-1:]])) + "\n" for r, l in zip(x, y)))
    log = tmp_path / "log.jsonl"
    run_job(_run_cfg(tmp_path, "t", optimizer="ntasgd", nonmono=1, learning_rate=20.0, clip_grad_norm=0.25, valid_path=str(path),
                     max_steps=20, evaluate_every=2, json_log=str(log)), standalone=True)
    evals = [r for r in map(json.loads, log.read_text().splitlines()) if "loss" in r]
    on = [r["averaging"] for r in evals]
    assert on[0] == 0 and 1 in on and all(on[on.index(1):]), [(r["val_loss"], r["averaging"]) for r in evals]
    assert evals[-1]["averaged_steps"] >= 1
    ev = run_job(_run_cfg(tmp_path, "t", mode="eval", optimizer="ntasgd"), standalone=True)
    assert ev["weights"] == "averaged"


# ---- the average after the fused allreduce's buckets --------------------------------------------------------------------------
def _solo_fused():
    """A ``FusedComm`` of one rank whose "symmetric" arena is an ordinary allocation, carved as ``FusedComm.adopt`` carves it (no
    process group, no symmetric memory): every gradient bucket goes through ``FusedComm.launch_bucket`` and the fused kernel as at
    any world size, and the kernel's sum over one rank is the gradient itself."""
    from lstm_tensorspark_b200.ops.cuda_ext import ext
    from lstm_tensorspark_b200.parallel.comm import Communicator
    from lstm_tensorspark_b200.parallel.fused_comm import FusedComm, SymmetricArena, _align

    class SoloFused(FusedComm):
        def __init__(self):
            Communicator.__init__(self, 0, 1)
            self.name, self.device, self.timeout_s = "fused", DEV, 60.0
            self.arena, self.use_multicast, self.blocks_override, self.launches = None, "0", 0, 0
            self._state_buckets, self._gs = [], None

        def adopt(self, flat):
            E = ext()
            n = flat.padded_numel
            total = 3 * _align(4 * n) + _align(2 * n) + _align(4 * E.ar_flag_words()) + 4096
            A = object.__new__(SymmetricArena)
            A.buf = torch.zeros(total, dtype=torch.uint8, device=DEV)
            A.rank, A.world, A.off, A.nbytes = 0, 1, 0, total
            A.base, A.mc_base = [A.buf.data_ptr()], 0
            self.arena = A
            self.data, self.off_data = A.carve(n, torch.float32)
            self.grad, self.off_grad = A.carve(n, torch.float32)
            self.stage, self.off_stage = A.carve(n, torch.float32)
            self.shadow, self.off_shadow = A.carve(n, torch.bfloat16)
            self.flags, self.off_flags = A.carve(E.ar_flag_words(), torch.int32)
            flat.rebase(self.data, self.grad)
            flat.shadow = self.shadow
            flat.refresh_shadow()
            self.slots = E.ar_slots()
            self.epochs = torch.zeros(E.ar_max_blocks() * self.slots, dtype=torch.int32, device=DEV)
            self.err = torch.zeros(1, dtype=torch.int32, device=DEV)
            self.flat = flat
            return flat

        def close(self):
            torch.cuda.synchronize(DEV)
            self.check_errors()

    return SoloFused()


def test_bucketed_fused_step_averages_once_after_every_bucket_inside_the_graph():
    """``--comm fused --sync_mode grad_allreduce`` with gradient buckets (the engine sees two replicas, the communicator one): a
    captured step replayed 8 times, the trigger flipped between replays.  After every step ``ax`` must be bitwise the fp32 torch
    average of the step's final weights (so it ran once, after the last bucket wrote its part of ``p``, and inside the graph),
    ``k`` must count the steps since the flip, and both must agree with the same steps through ``flat_asgd``."""
    from lstm_tensorspark_b200.config import Config
    from lstm_tensorspark_b200.engine import TrainEngine
    from lstm_tensorspark_b200.ops import reference as ref
    comm = _solo_fused()
    cfg = Config(hidden_units="128,128", in_features=64, seq_len=16, batch_size=64, vocab_size=512, next_token=True, init="scaled",
                 learn_initial_state=False, device="cuda", quiet=True, optimizer="ntasgd", learning_rate=0.1, weight_decay=1e-4,
                 deterministic=True, sync_mode="grad_allreduce", comm="fused", grad_buckets=True, partitions=2)
    eng = TrainEngine(cfg, 0, 2, comm, batch_size=64, device=DEV, dtype=torch.bfloat16)
    assert eng._bucket_plan is not None and len(eng._bucket_plan) >= 2
    flat_path = _engine("ntasgd", learning_rate=0.1, weight_decay=1e-4, clip_grad_norm=0.0)
    batches = _batches(8)
    eng.capture(*batches[0])
    n_capture = comm.launches                                         # every bucket launch is recorded in the graph
    opt = eng.optimizer
    dp = 0.0
    for i, (x, y) in enumerate(batches):
        if i == 2:
            opt.start_averaging()
            flat_path.optimizer.start_averaging()
        ax0 = opt.ax.clone()
        eng.step(x, y)
        flat_path.step(x, y)
        torch.cuda.synchronize()
        k = max(0, i - 1)
        assert opt.avg.tolist() == [int(i >= 2), k] == flat_path.optimizer.avg.tolist()
        want = ref.asgd_average_(ax0.clone(), eng.flat.data, k) if i >= 2 else ax0
        assert torch.equal(opt.ax, want), i
        if i >= 2:
            dp = max(dp, float((eng.flat.data - flat_path.flat.data).abs().max()))
    assert comm.launches == n_capture                                 # the steps were replays
    # the bucket kernel's SGD and flat_sgd differ in the last bits, and the runs drift apart from there; ax is a mean of the
    # weights since the flip, so the averages differ by no more than the weights did at some step (plus the average's rounding)
    assert float((opt.ax - flat_path.optimizer.ax).abs().max()) <= dp * (1 + 1e-3) + 8 * N.U * float(opt.ax.abs().max())
    comm.close()


def _fused_vs_nccl_worker(rank, world, comm_kind, steps):
    from lstm_tensorspark_b200 import data as D
    from lstm_tensorspark_b200.config import Config
    from lstm_tensorspark_b200.engine import TrainEngine
    from lstm_tensorspark_b200.ops import reference as ref
    from lstm_tensorspark_b200.parallel.comm import make_communicator
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    cfg = Config(hidden_units="128,128", in_features=64, seq_len=8, batch_size=128, num_classes=10, partitions=world,
                 sync_mode="grad_allreduce", comm=comm_kind, grad_buckets=True, optimizer="asgd", learning_rate=0.1,
                 weight_decay=0.01, init="scaled", learn_initial_state=False, dtype="bf16", device="cuda", deterministic=True,
                 quiet=True)
    comm = make_communicator(comm_kind, rank, world, dev, 60)
    eng = TrainEngine(cfg, rank, world, comm, batch_size=128, device=dev, dtype=torch.bfloat16)
    flat, opt = eng.flat, eng.optimizer
    bound = torch.zeros_like(flat.data, dtype=torch.float64)
    for k in range(steps):
        x, y = D.synthetic_sequences(128, 8, 64, 10, seed=1000 * k + rank)
        before, ax0 = flat.data.clone(), opt.ax.clone()
        eng.step(torch.as_tensor(x).to(dev, torch.bfloat16), torch.as_tensor(y).to(dev))
        torch.cuda.synchronize()
        assert torch.equal(opt.ax, ref.asgd_average_(ax0, flat.data, k + 1)), (comm_kind, k)
        if comm_kind == "nccl":                            # flat.grad holds the summed gradient the update used
            upd = N.sgd_update(before, flat.grad, opt.lr, 0.01, 1.0 / world, opt.wd_numel)
            N.check_update(f"nccl step {k} p", flat.data, upd.p, upd.bound_p)
            bound += upd.bound_p
    out = {"p": flat.data.cpu(), "ax": opt.ax.cpu(), "k": opt.averaged_steps, "bound": bound.cpu()}
    comm.close()
    return out


def test_fused_buckets_average_as_nccl():
    """Two GPUs or more: three ``asgd`` steps with ``--comm fused`` (gradient buckets, then ``flat_average``) against ``--comm
    nccl`` (all_reduce, then ``flat_asgd``) on the same batches.  Each run's ``ax`` is bitwise the torch average of its own
    weights at every step; ``ax`` is a mean of the weights, so the two runs' averages differ by at most the two runs' update
    bounds summed over the steps."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    from lstm_tensorspark_b200.parallel.launch import launch
    steps = 3
    fused = launch(_fused_vs_nccl_worker, 2, args=("fused", steps))
    nccl = launch(_fused_vs_nccl_worker, 2, args=("nccl", steps))
    for f, c in zip(fused, nccl):
        assert f["k"] == c["k"] == steps
        N.check_update("fused vs nccl p", f["p"], c["p"].double(), 2 * c["bound"])
        N.check_update("fused vs nccl ax", f["ax"], c["ax"].double(), 2 * c["bound"] + 2 * N.U * c["ax"].double().abs())
