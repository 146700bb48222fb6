"""Operand-ring depth of the persistent LSTM kernels (csrc/lstm_seq_wgmma.cu): the fp32 accumulator is staged in drained
ring stages, so the ring gets the shared memory a separate staging buffer used to take.  The stage counts the kernels pick,
every forced depth of the two-tiles-per-CTA kernels, and the configurations that stage differently (forward K-split,
streamed weights, masked, reverse) against the fp32 reference."""
import pytest
import torch


def _ext():
    from lstm_tensorspark_b200.ops.cuda_ext import ext
    return ext()


def test_headline_ring_depths():
    # 2 x 1024, B = 256: two batch tiles per CTA on an H100.  (stages, tiles, streamed, K-split)
    assert _ext().lstm_seq_config(False, 1024, 256, 2) == (6, 2, False, False)
    assert _ext().lstm_seq_config(True, 1024, 256, 2) == (4, 2, False, False)


def test_ring_depth_limits_and_weight_streaming_boundary():
    E = _ext()
    assert E.lstm_seq_config(True, 1024, 256, 2 + 16 * 4)[0] == 4
    with pytest.raises(RuntimeError, match="does not fit"):
        E.lstm_seq_config(True, 1024, 256, 2 + 16 * 5)
    # resident weights up to H = 1152 (forward) / 1024 (backward), streamed above
    assert E.lstm_seq_config(False, 1152, 128, 0)[2] is False
    assert E.lstm_seq_config(False, 1280, 128, 0)[2] is True
    assert E.lstm_seq_config(True, 1024, 128, 0)[2] is False
    assert E.lstm_seq_config(True, 1088, 128, 0)[2] is True
    # H = 64 keeps a dedicated staging buffer; the forward K-split keeps its own
    assert E.lstm_seq_config(False, 64, 128, 0)[0] == 6
    assert E.lstm_seq_config(False, 256, 128, 0)[3] is True


def _case(T, B, H, D, lengths=None, reverse=False, backward=True):
    from lstm_tensorspark_b200.ops import cuda_lstm, reference as ref
    dev = torch.device("cuda", 0)
    torch.manual_seed(3)
    params = [torch.randn(T, B, D, device=dev) * 0.5, torch.randn(B, H, device=dev) * 0.1, torch.randn(B, H, device=dev) * 0.1,
              torch.randn(4 * H, D, device=dev) / D ** 0.5, torch.randn(4 * H, H, device=dev) / H ** 0.5,
              torch.randn(4 * H, device=dev) * 0.1]
    lens = None if lengths is None else lengths.to(dev, torch.int32)
    pr = [p.bfloat16().float().requires_grad_(True) if i != 2 else p.clone().requires_grad_(True) for i, p in enumerate(params)]
    hs_r, hT_r, cT_r = ref.lstm_layer_sequence(*pr, lengths=lens, reverse=reverse)
    wgt, w2 = torch.randn_like(hs_r), torch.randn_like(hT_r)
    pc = [p.clone().requires_grad_(True) for p in params]
    n0 = cuda_lstm.STATS["fast_fwd"], cuda_lstm.STATS["fast_bwd"]
    hs, hT, cT = cuda_lstm.lstm_layer_sequence(pc[0].bfloat16(), *pc[1:], lengths=lens, reverse=reverse)
    if backward:
        ((hs_r * wgt).sum() + (hT_r * w2).sum()).backward()
        ((hs.float() * wgt).sum() + (hT.float() * w2).sum()).backward()
    torch.cuda.synchronize()
    cuda_lstm.check_kernel_errors(dev)
    assert cuda_lstm.STATS["fast_fwd"] == n0[0] + 1 and cuda_lstm.STATS["fast_bwd"] == n0[1] + int(backward)

    def rel_l2(a, b):
        return float((a.float() - b.float()).norm() / (b.float().norm() + 1e-20))
    assert (hs.float() - hs_r).abs().max() < 3e-2 and (cT - cT_r).abs().max() < 3e-2
    assert rel_l2(hs, hs_r) < 1e-2 and rel_l2(cT, cT_r) < 1e-2
    if backward:
        for a, b in zip(pc, pr):
            assert rel_l2(a.grad, b.grad) < 2e-2, (tuple(b.shape), rel_l2(a.grad, b.grad))


@pytest.mark.gpu
@pytest.mark.parametrize("stages", [2, 3, 4, 5, 6])
def test_two_tile_kernels_at_every_ring_depth(monkeypatch, stages):
    from lstm_tensorspark_b200.ops import cuda_lstm
    monkeypatch.setattr(cuda_lstm, "SEQ_VARIANT", 2 + 16 * stages)
    # the backward ring holds at most 4 stages next to the two exchange buffers: deeper rings are forward-only
    _case(T=4, B=256, H=1024, D=256, backward=stages <= 4)


@pytest.mark.gpu
@pytest.mark.parametrize("T,B,H,D,masked,reverse", [
    (3, 128, 256, 64, False, False),      # forward K-split (dedicated staging buffer)
    (3, 128, 64, 64, False, False),       # one k-block per tile (dedicated staging buffer)
    (3, 64, 1280, 256, False, False),     # streamed weights, kNarrow backward
    (3, 64, 2048, 256, False, False),
    (5, 200, 256, 64, True, False),       # masked
    (5, 200, 256, 64, False, True),       # reverse
    (5, 256, 1024, 128, True, True),      # masked reverse, two tiles per CTA
])
def test_ring_staging_configurations(T, B, H, D, masked, reverse):
    lengths = torch.randint(1, T + 1, (B,)) if masked else None
    _case(T, B, H, D, lengths=lengths, reverse=reverse)
