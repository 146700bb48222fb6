"""Two batch tiles per CTA (csrc/lstm_seq_wgmma.cu, kTiles = 2): each consumer warpgroup owns one tile and the two run
their steps independently.  Here the tiles are unbalanced - B = 200 leaves the second tile 72 valid rows of 128 - with
per-row lengths, so the warpgroups differ in valid rows, padded steps and operand bytes, against the fp32 reference."""
import pytest
import torch


def _rel_l2(a, b):
    return float((a.float() - b.float()).norm() / (b.float().norm() + 1e-20))


@pytest.mark.gpu
@pytest.mark.parametrize("reverse", [False, True])
def test_unbalanced_two_tile_layer_with_lengths(monkeypatch, reverse):
    from lstm_tensorspark_b200.ops import cuda_lstm, reference as ref
    from lstm_tensorspark_b200.ops.cuda_ext import ext
    T, B, H, D = 5, 200, 1024, 128
    monkeypatch.setattr(cuda_lstm, "SEQ_VARIANT", 2)
    assert ext().lstm_seq_config(False, H, B, 2)[1] == 2 and ext().lstm_seq_config(True, H, B, 2)[1] == 2
    dev = torch.device("cuda", 0)
    torch.manual_seed(11)
    lens = torch.randint(1, T + 1, (B,)).to(dev, torch.int32)
    params = [torch.randn(T, B, D, device=dev) * 0.5, torch.randn(B, H, device=dev) * 0.1, torch.randn(B, H, device=dev) * 0.1,
              torch.randn(4 * H, D, device=dev) / D ** 0.5, torch.randn(4 * H, H, device=dev) / H ** 0.5,
              torch.randn(4 * H, device=dev) * 0.1]
    pr = [p.bfloat16().float().requires_grad_(True) if i != 2 else p.clone().requires_grad_(True) for i, p in enumerate(params)]
    hs_r, hT_r, cT_r = ref.lstm_layer_sequence(*pr, lengths=lens, reverse=reverse)
    wgt, w2 = torch.randn_like(hs_r), torch.randn_like(hT_r)
    pc = [p.clone().requires_grad_(True) for p in params]
    n0 = cuda_lstm.STATS["fast_fwd"], cuda_lstm.STATS["fast_bwd"]
    hs, hT, cT = cuda_lstm.lstm_layer_sequence(pc[0].bfloat16(), *pc[1:], lengths=lens, reverse=reverse)
    ((hs_r * wgt).sum() + (hT_r * w2).sum()).backward()
    ((hs.float() * wgt).sum() + (hT.float() * w2).sum()).backward()
    torch.cuda.synchronize()
    cuda_lstm.check_kernel_errors(dev)
    assert cuda_lstm.STATS["fast_fwd"] == n0[0] + 1 and cuda_lstm.STATS["fast_bwd"] == n0[1] + 1
    assert (hs.float() - hs_r).abs().max() < 3e-2 and (cT - cT_r).abs().max() < 3e-2
    assert _rel_l2(hs, hs_r) < 1e-2 and _rel_l2(cT, cT_r) < 1e-2
    for a, b in zip(pc, pr):
        assert _rel_l2(a.grad, b.grad) < 2e-2, (tuple(b.shape), _rel_l2(a.grad, b.grad))
