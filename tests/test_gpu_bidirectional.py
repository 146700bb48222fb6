"""Bidirectional layers on the GPU (`pytest -m gpu`): the reverse-time persistent kernels (masked and unmasked), batch chunks and
the generic path against the reverse fp32 reference, bitwise identities of the reverse direction in deterministic mode, and the
engine / trainer with --bidirectional."""
import pytest
import torch

from test_gpu_variable_length import SHAPES, _deterministic, _inputs, _lengths, _loss, _rel_l2

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    return torch.device("cuda", 0)


def _run_cuda(params, lengths, dtype, loss_on, w, reverse=True):
    from lstm_tensorspark_b200.ops import cuda_lstm
    pc = [p.clone().requires_grad_(True) for p in params]
    hs, hT, cT = cuda_lstm.lstm_layer_sequence(pc[0].to(dtype), pc[1], pc[2], pc[3], pc[4], pc[5], lengths=lengths, reverse=reverse)
    _loss(loss_on, hs, hT, cT, w).backward()
    torch.cuda.synchronize()
    return (hs, hT, cT), [p.grad for p in pc]


def _reverse_case(dev, T, B, H, D, loss_on, masked, dtype=torch.bfloat16, tol=3e-2):
    from lstm_tensorspark_b200.ops import cuda_lstm, reference as ref
    params = _inputs(dev, T, B, H, D)
    lengths = _lengths(B, T, seed=T * 1000 + B + 7).to(dev) if masked else None
    cast = (lambda p: p.bfloat16().float()) if dtype == torch.bfloat16 else (lambda p: p.clone())
    pr = [cast(p).requires_grad_(True) if i != 2 else p.clone().requires_grad_(True) for i, p in enumerate(params)]
    hs_r, hT_r, cT_r = ref.lstm_layer_sequence(*pr, lengths=lengths, reverse=True)
    w = (torch.randn_like(hs_r), torch.randn_like(hT_r), torch.randn_like(cT_r))
    _loss(loss_on, hs_r, hT_r, cT_r, w).backward()
    (hs, hT, cT), grads = _run_cuda(params, lengths, dtype, loss_on, w)
    cuda_lstm.check_kernel_errors(dev)
    assert (hs.float() - hs_r).abs().max() < tol and (cT - cT_r).abs().max() < tol and (hT.float() - hT_r).abs().max() < tol
    assert _rel_l2(hs, hs_r) < 1e-2 and _rel_l2(cT, cT_r) < 1e-2 and _rel_l2(hT, hT_r) < 1e-2
    for g, p in zip(grads, pr):
        assert _rel_l2(g, p.grad) < 2e-2, (tuple(p.shape), _rel_l2(g, p.grad))
    if masked:
        pad = (torch.arange(T, device=dev).view(T, 1) >= lengths.view(1, B))
        if pad.any():
            assert float(grads[0][pad].abs().max()) == 0.0                   # no gradient into padded inputs


@pytest.mark.parametrize("masked", [False, True])
@pytest.mark.parametrize("loss_on", ["last", "all"])
@pytest.mark.parametrize("T,B,H,D", SHAPES)
def test_reverse_persistent_lstm_sequence(dev, T, B, H, D, loss_on, masked):
    from lstm_tensorspark_b200.ops import cuda_lstm
    n0 = cuda_lstm.STATS["fast_fwd"], cuda_lstm.STATS["fast_bwd"]
    _reverse_case(dev, T, B, H, D, loss_on, masked)
    assert cuda_lstm.STATS["fast_fwd"] == n0[0] + 1 and cuda_lstm.STATS["fast_bwd"] == n0[1] + 1


def test_reverse_large_batch_runs_in_chunks(dev):
    from lstm_tensorspark_b200.ops import cuda_lstm
    n0 = cuda_lstm.STATS["fast_fwd"], cuda_lstm.STATS["generic_fwd"]
    _reverse_case(dev, 4, 400, 1024, 256, "all", masked=True)
    assert cuda_lstm.STATS["fast_fwd"] == n0[0] + 2 and cuda_lstm.STATS["generic_fwd"] == n0[1]


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("masked", [False, True])
@pytest.mark.parametrize("T,B,H,D", [(1, 10, 16, 4), (6, 33, 48, 20)])
def test_reverse_generic_path(dev, T, B, H, D, masked, dtype):
    from lstm_tensorspark_b200.ops import cuda_lstm
    n0 = cuda_lstm.STATS["generic_fwd"], cuda_lstm.STATS["generic_bwd"]
    _reverse_case(dev, T, B, H, D, "all", masked, dtype=dtype)
    assert cuda_lstm.STATS["generic_fwd"] == n0[0] + 1 and cuda_lstm.STATS["generic_bwd"] == n0[1] + 1


DET_SHAPES = [(5, 100, 128, 72), (8, 256, 1024, 1024), (3, 64, 1280, 256), (3, 64, 2048, 256), (6, 33, 48, 20)]


@pytest.mark.parametrize("T,B,H,D", DET_SHAPES)
def test_reverse_equals_forward_on_flipped_time_bitwise(dev, T, B, H, D):
    """Same operand stream, same arithmetic: only the time index of the saved arrays differs.  (The weight and bias gradients
    sum over time in another order and are not compared bitwise.)"""
    from lstm_tensorspark_b200.ops import cuda_lstm
    old = _deterministic()
    try:
        params = _inputs(dev, T, B, H, D, seed=8)
        w = (torch.randn(T, B, H, device=dev), torch.randn(B, H, device=dev), torch.randn(B, H, device=dev))
        (hs_r, hT_r, cT_r), g_r = _run_cuda(params, None, torch.bfloat16, "all", w, reverse=True)
        flipped = [params[0].flip(0).contiguous()] + params[1:]
        (hs_f, hT_f, cT_f), g_f = _run_cuda(flipped, None, torch.bfloat16, "all", (w[0].flip(0), w[1], w[2]), reverse=False)
    finally:
        cuda_lstm.SEQ_VARIANT = old
    cuda_lstm.check_kernel_errors(dev)
    assert torch.equal(hs_r, hs_f.flip(0)) and torch.equal(hT_r, hT_f) and torch.equal(cT_r, cT_f)
    assert torch.equal(g_r[0], g_f[0].flip(0))                              # dx
    assert torch.equal(g_r[1], g_f[1]) and torch.equal(g_r[2], g_f[2])      # dh0, dc0


@pytest.mark.parametrize("T,B,H,D", DET_SHAPES)
def test_reverse_full_lengths_equal_no_lengths_bitwise(dev, T, B, H, D):
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


def test_reverse_rejects_wavefront_gating(dev):
    from lstm_tensorspark_b200.ops import cuda_lstm
    from lstm_tensorspark_b200.ops.cuda_ext import ext
    T, B, H = 2, 128, 64
    gx = torch.zeros(T, B, 4 * H, device=dev, dtype=torch.bfloat16)
    w_h = torch.zeros(4 * H, H, device=dev, dtype=torch.bfloat16)
    with pytest.raises(RuntimeError, match="wavefront"):
        ext().lstm_seq_fwd(gx, w_h, torch.zeros(4 * H, device=dev), torch.zeros(B, H, device=dev, dtype=torch.bfloat16),
                           torch.zeros(B, H, device=dev), cuda_lstm._sync_ws(dev), extra_signal=True, reverse=True)


def _engine(dev, deterministic=True):
    from lstm_tensorspark_b200.config import Config
    from lstm_tensorspark_b200.engine import TrainEngine
    cfg = Config(hidden_units="256,256", in_features=128, seq_len=12, batch_size=256, num_classes=10, partitions=1,
                 sync_mode="none", init="scaled", learn_initial_state=False, dtype="bf16", device="cuda", quiet=True,
                 deterministic=deterministic, variable_length=True, bidirectional=True)
    return TrainEngine(cfg, 0, 1, None, batch_size=256, device=dev, dtype=torch.bfloat16)


def test_bidirectional_engine_eager_captured_and_bound_follow_one_trajectory(dev):
    from lstm_tensorspark_b200 import data as D
    from lstm_tensorspark_b200.ops import cuda_lstm
    x, y, l = D.synthetic_sequences(3 * 256, 12, 128, 10, seed=0, variable_length=True)
    xs = torch.as_tensor(x).to(dev, torch.bfloat16)
    ys, ls = torch.as_tensor(y).to(dev), torch.as_tensor(l).to(dev)
    batches = [(xs[i * 256:(i + 1) * 256], ys[i * 256:(i + 1) * 256], ls[i * 256:(i + 1) * 256]) for i in range(3)]
    n0 = cuda_lstm.STATS["fast_fwd"], cuda_lstm.STATS.get("wavefront_fwd", 0), cuda_lstm.STATS["generic_fwd"]
    eager = _engine(dev)
    want = [float(eager.step(*batches[k % 3])) for k in range(6)]
    assert cuda_lstm.STATS["fast_fwd"] == n0[0] + 6 * 4                    # 2 layers x 2 directions per step
    assert cuda_lstm.STATS.get("wavefront_fwd", 0) == n0[1] and cuda_lstm.STATS["generic_fwd"] == n0[2]
    graphed = _engine(dev)
    graphed.capture(*batches[0][:2], lengths=batches[0][2], bind=batches[1:])
    got = [float(graphed.step(*batches[k % 3])) for k in range(6)]
    torch.cuda.synchronize()
    cuda_lstm.check_kernel_errors(dev)
    assert want[-1] < want[0]
    for a, b in zip(want, got):
        assert abs(a - b) <= 1e-3 * max(1.0, abs(a)), (want, got)
    assert torch.allclose(eager.flat.data, graphed.flat.data, rtol=0, atol=1e-4)
    assert cuda_lstm.STATS.get("wavefront_fwd", 0) == n0[1]


def test_synthetic_bidirectional_graph_job_trains_and_resumes(dev, tmp_path):
    from lstm_tensorspark_b200.config import Config
    from lstm_tensorspark_b200.ops import cuda_lstm
    from lstm_tensorspark_b200.trainer import run_job
    import json
    import os
    base = dict(synthetic=2048, seq_len=16, in_features=64, num_classes=5, hidden_units="128,128", batch_size=256,
                variable_length=True, bidirectional=True, cuda_graph=True, init="scaled", learning_rate=3e-3, steps_mode="epochs",
                device="cuda", checkpoint_path=str(tmp_path / "ck"), output_path=str(tmp_path / "out"), quiet=True, evaluate_every=8)
    n0 = cuda_lstm.STATS["fast_fwd"]
    run_job(Config(epochs=4, **base).validate(), standalone=True)
    assert cuda_lstm.STATS["fast_fwd"] > n0
    cuda_lstm.check_kernel_errors(dev)
    runs = os.listdir(base["checkpoint_path"])
    scal = [json.loads(s) for s in open(os.path.join(base["checkpoint_path"], runs[0], "train", "scalars.jsonl"))]
    assert scal[-1]["cross_entropy"] < scal[0]["cross_entropy"]
    out = run_job(Config(epochs=5, use_pretrained_model=True, **base).validate(), standalone=True)
    assert out["results"][0]["steps"] == 8                     # 40 total - 32 already done
    ev = run_job(Config(mode="eval", **base).validate(), standalone=True)
    assert ev["samples"] == 2048 and ev["loss"] == ev["loss"]
    cuda_lstm.check_kernel_errors(dev)
