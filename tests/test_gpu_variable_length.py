"""Variable-length sequences on the GPU (`pytest -m gpu`): the masked persistent kernels, the masked generic path, the layer
wavefront and the engine with per-sample lengths, against the masked fp32 reference (ops/reference.py)."""
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    return torch.device("cuda", 0)


def _rel_l2(a, b):
    return float((a.float() - b.float()).norm() / (b.float().norm() + 1e-20))


def _lengths(B, T, seed):
    g = torch.Generator().manual_seed(seed)
    l = torch.randint(1, T + 1, (B,), generator=g, dtype=torch.int32)
    l[0], l[-1] = 1, T                                   # both ends of the range
    return l


def _inputs(dev, T, B, H, D, seed=1):
    torch.manual_seed(seed)
    return [torch.randn(T, B, D, device=dev) * 0.5, torch.randn(B, H, device=dev) * 0.1, torch.randn(B, H, device=dev) * 0.1,
            torch.randn(4 * H, D, device=dev) / D ** 0.5, torch.randn(4 * H, H, device=dev) / H ** 0.5,
            torch.randn(4 * H, device=dev) * 0.1]


def _loss(loss_on, hs, hT, cT, w):
    if loss_on == "last":
        return (hT.float() * w[1]).sum()
    return (hs.float() * w[0]).sum() + (hT.float() * w[1]).sum() + (cT.float() * w[2]).sum()


def _run_cuda(params, lengths, dtype, loss_on, w):
    from lstm_tensorspark_b200.ops import cuda_lstm
    pc = [p.clone().requires_grad_(True) for p in params]
    hs, hT, cT = cuda_lstm.lstm_layer_sequence(pc[0].to(dtype), pc[1], pc[2], pc[3], pc[4], pc[5], lengths=lengths)
    _loss(loss_on, hs, hT, cT, w).backward()
    torch.cuda.synchronize()
    return (hs, hT, cT), [p.grad for p in pc]


def _masked_case(dev, T, B, H, D, loss_on, dtype=torch.bfloat16, tol=3e-2):
    from lstm_tensorspark_b200.ops import cuda_lstm, reference as ref
    params = _inputs(dev, T, B, H, D)
    lengths = _lengths(B, T, seed=T * 1000 + B).to(dev)
    cast = (lambda p: p.bfloat16().float()) if dtype == torch.bfloat16 else (lambda p: p.clone())
    pr = [cast(p).requires_grad_(True) if i != 2 else p.clone().requires_grad_(True) for i, p in enumerate(params)]
    hs_r, hT_r, cT_r = ref.lstm_layer_sequence(*pr, lengths=lengths)
    w = (torch.randn_like(hs_r), torch.randn_like(hT_r), torch.randn_like(cT_r))
    _loss(loss_on, hs_r, hT_r, cT_r, w).backward()
    (hs, hT, cT), grads = _run_cuda(params, lengths, dtype, loss_on, w)
    cuda_lstm.check_kernel_errors(dev)
    assert (hs.float() - hs_r).abs().max() < tol and (cT - cT_r).abs().max() < tol and (hT.float() - hT_r).abs().max() < tol
    assert _rel_l2(hs, hs_r) < 1e-2 and _rel_l2(cT, cT_r) < 1e-2 and _rel_l2(hT, hT_r) < 1e-2
    for g, p in zip(grads, pr):
        assert _rel_l2(g, p.grad) < 2e-2, (tuple(p.shape), _rel_l2(g, p.grad))
    pad = (torch.arange(T, device=dev).view(T, 1) >= lengths.view(1, B))
    if pad.any():
        assert float(grads[0][pad].abs().max()) == 0.0                   # no gradient into padded inputs


SHAPES = [(1, 128, 64, 64), (1, 96, 128, 40), (2, 256, 256, 64), (3, 128, 64, 64), (5, 100, 128, 72),
          (4, 256, 256, 128), (8, 256, 1024, 1024), (3, 64, 2048, 256), (3, 64, 1280, 256)]


@pytest.mark.parametrize("loss_on", ["last", "all"])
@pytest.mark.parametrize("T,B,H,D", SHAPES)
def test_masked_persistent_lstm_sequence(dev, T, B, H, D, loss_on):
    from lstm_tensorspark_b200.ops import cuda_lstm
    n0 = cuda_lstm.STATS["fast_fwd"], cuda_lstm.STATS["fast_bwd"]
    _masked_case(dev, T, B, H, D, loss_on)
    assert cuda_lstm.STATS["fast_fwd"] == n0[0] + 1 and cuda_lstm.STATS["fast_bwd"] == n0[1] + 1


def test_masked_large_batch_runs_in_chunks(dev):
    from lstm_tensorspark_b200.ops import cuda_lstm
    n0 = cuda_lstm.STATS["fast_fwd"], cuda_lstm.STATS["generic_fwd"]
    _masked_case(dev, 4, 400, 1024, 256, "all")
    assert cuda_lstm.STATS["fast_fwd"] == n0[0] + 2 and cuda_lstm.STATS["generic_fwd"] == n0[1]


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("loss_on", ["last", "all"])
@pytest.mark.parametrize("T,B,H,D", [(1, 10, 16, 4), (6, 33, 48, 20)])
def test_masked_generic_path(dev, T, B, H, D, loss_on, dtype):
    from lstm_tensorspark_b200.ops import cuda_lstm
    n0 = cuda_lstm.STATS["generic_fwd"], cuda_lstm.STATS["generic_bwd"]
    _masked_case(dev, T, B, H, D, loss_on, dtype=dtype)
    assert cuda_lstm.STATS["generic_fwd"] == n0[0] + 1 and cuda_lstm.STATS["generic_bwd"] == n0[1] + 1


def _deterministic():
    """The recurrence kernels consume operand blocks in index order (the engine's deterministic mode): bitwise repeatable."""
    from lstm_tensorspark_b200.ops import cuda_lstm
    old = cuda_lstm.SEQ_VARIANT
    cuda_lstm.SEQ_VARIANT = (old & ~(7 << 12)) | (3 << 12)
    return old


@pytest.mark.parametrize("T,B,H,D", [(5, 100, 128, 72), (8, 256, 1024, 1024), (3, 64, 1280, 256), (6, 33, 48, 20)])
def test_full_lengths_equal_no_lengths_bitwise(dev, T, B, H, D):
    from lstm_tensorspark_b200.ops import cuda_lstm
    old = _deterministic()
    try:
        params = _inputs(dev, T, B, H, D, seed=5)
        w = (torch.randn(T, B, H, device=dev), torch.randn(B, H, device=dev), torch.randn(B, H, device=dev))
        full = torch.full((B,), T, dtype=torch.int32, device=dev)
        out_a, g_a = _run_cuda(params, None, torch.bfloat16, "all", w)
        out_b, g_b = _run_cuda(params, full, torch.bfloat16, "all", w)
    finally:
        cuda_lstm.SEQ_VARIANT = old
    cuda_lstm.check_kernel_errors(dev)
    for a, b in zip(list(out_a) + g_a, list(out_b) + g_b):
        assert torch.equal(a, b)


@pytest.mark.parametrize("T,B,H,D", [(5, 100, 128, 72), (8, 256, 1024, 1024), (3, 64, 2048, 256), (6, 33, 48, 20)])
def test_padded_input_values_change_nothing(dev, T, B, H, D):
    from lstm_tensorspark_b200.ops import cuda_lstm
    old = _deterministic()
    try:
        params = _inputs(dev, T, B, H, D, seed=6)
        lengths = _lengths(B, T, seed=7).to(dev)
        pad = (torch.arange(T, device=dev).view(T, 1) >= lengths.view(1, B))
        params[0] = torch.where(pad.unsqueeze(-1), torch.zeros_like(params[0]), params[0])
        noisy = list(params)
        noisy[0] = torch.where(pad.unsqueeze(-1), torch.randn_like(params[0]) * 100.0, params[0])
        w = (torch.randn(T, B, H, device=dev), torch.randn(B, H, device=dev), torch.randn(B, H, device=dev))
        out_a, g_a = _run_cuda(params, lengths, torch.bfloat16, "all", w)
        out_b, g_b = _run_cuda(noisy, lengths, torch.bfloat16, "all", w)
    finally:
        cuda_lstm.SEQ_VARIANT = old
    cuda_lstm.check_kernel_errors(dev)
    for a, b in zip(list(out_a) + g_a, list(out_b) + g_b):
        assert torch.equal(a, b)


def test_layer_wavefront_with_lengths_matches_sequential_layers(dev):
    from lstm_tensorspark_b200.ops import cuda_lstm
    torch.manual_seed(11)
    T, B, D, Ha, Hb = 6, 256, 256, 512, 256
    x = (torch.randn(T, B, D, device=dev) * 0.5).bfloat16()
    lengths = _lengths(B, T, seed=12).to(dev)

    def layer(H, Din):
        return [torch.randn(B, H, device=dev) * 0.1, torch.randn(B, H, device=dev) * 0.1, torch.randn(4 * H, Din, device=dev) / Din ** 0.5,
                torch.randn(4 * H, H, device=dev) / H ** 0.5, torch.randn(4 * H, device=dev) * 0.1]
    la, lb = layer(Ha, D), layer(Hb, Ha)
    assert cuda_lstm.wavefront_supported(x, Ha, Hb)
    w = torch.randn(T, B, Hb, device=dev)

    def run(pair):
        a = [p.clone().requires_grad_(True) for p in la]
        b = [p.clone().requires_grad_(True) for p in lb]
        if pair:
            hs_b, hTa, cTa, hTb, cTb = cuda_lstm.lstm_pair_sequence(x, a, b, lengths=lengths)
        else:
            hs_a, hTa, cTa = cuda_lstm.lstm_layer_sequence(x, *a, lengths=lengths)
            hs_b, hTb, cTb = cuda_lstm.lstm_layer_sequence(hs_a, *b, lengths=lengths)
        ((hs_b.float() * w).sum() + hTa.float().sum() + cTb.float().sum()).backward()
        torch.cuda.synchronize()
        return [hs_b, hTa, cTa, hTb, cTb] + [p.grad for p in a + b]
    n0 = cuda_lstm.STATS.get("wavefront_fwd", 0)
    got = run(True)
    assert cuda_lstm.STATS.get("wavefront_fwd", 0) == n0 + 1
    want = run(False)
    cuda_lstm.check_kernel_errors(dev)
    for g, r in zip(got, want):
        assert _rel_l2(g, r) < 2e-2, _rel_l2(g, r)


def _engine(dev, deterministic=True):
    from lstm_tensorspark_b200.config import Config
    from lstm_tensorspark_b200.engine import TrainEngine
    cfg = Config(hidden_units="256,256", in_features=128, seq_len=12, batch_size=256, num_classes=10, partitions=1,
                 sync_mode="none", init="scaled", learn_initial_state=False, dtype="bf16", device="cuda", quiet=True,
                 deterministic=deterministic, variable_length=True)
    return TrainEngine(cfg, 0, 1, None, batch_size=256, device=dev, dtype=torch.bfloat16)


def test_engine_with_lengths_eager_captured_and_bound_follow_one_trajectory(dev):
    from lstm_tensorspark_b200 import data as D
    from lstm_tensorspark_b200.ops import cuda_lstm
    x, y, l = D.synthetic_sequences(3 * 256, 12, 128, 10, seed=0, variable_length=True)
    xs = torch.as_tensor(x).to(dev, torch.bfloat16)
    ys, ls = torch.as_tensor(y).to(dev), torch.as_tensor(l).to(dev)
    batches = [(xs[i * 256:(i + 1) * 256], ys[i * 256:(i + 1) * 256], ls[i * 256:(i + 1) * 256]) for i in range(3)]
    eager = _engine(dev)
    want = [float(eager.step(*batches[k % 3])) for k in range(6)]
    graphed = _engine(dev)
    graphed.capture(*batches[0][:2], lengths=batches[0][2], bind=batches[1:])
    assert len(graphed.graph_inputs()) == 3 and graphed.graph_inputs()[2] is not None
    got = [float(graphed.step(*batches[k % 3])) for k in range(6)]
    torch.cuda.synchronize()
    cuda_lstm.check_kernel_errors(dev)
    assert want[-1] < want[0]
    for a, b in zip(want, got):
        assert abs(a - b) <= 1e-3 * max(1.0, abs(a)), (want, got)
    assert torch.allclose(eager.flat.data, graphed.flat.data, rtol=0, atol=1e-4)


def test_synthetic_variable_length_graph_job_trains_and_resumes(dev, tmp_path):
    from lstm_tensorspark_b200.config import Config
    from lstm_tensorspark_b200.ops import cuda_lstm
    from lstm_tensorspark_b200.trainer import run_job
    import json
    import os
    base = dict(synthetic=2048, seq_len=16, in_features=64, num_classes=5, hidden_units="128,128", batch_size=256,
                variable_length=True, cuda_graph=True, init="scaled", learning_rate=3e-3, steps_mode="epochs", device="cuda",
                checkpoint_path=str(tmp_path / "ck"), output_path=str(tmp_path / "out"), quiet=True, evaluate_every=8)
    n0 = cuda_lstm.STATS["fast_fwd"]
    run_job(Config(epochs=4, **base).validate(), standalone=True)
    assert cuda_lstm.STATS["fast_fwd"] > n0
    runs = os.listdir(base["checkpoint_path"])
    scal = [json.loads(s) for s in open(os.path.join(base["checkpoint_path"], runs[0], "train", "scalars.jsonl"))]
    assert scal[-1]["cross_entropy"] < scal[0]["cross_entropy"]
    out = run_job(Config(epochs=5, use_pretrained_model=True, **base).validate(), standalone=True)
    assert out["results"][0]["steps"] == 8                     # 40 total - 32 already done
    cuda_lstm.check_kernel_errors(dev)
