"""The pipelined layer pair's first-layer input projection (gx_a) runs next to L_a's forward recurrence, which waits for it block
by block (ops/cuda_lstm.py, _LSTMPairFn): a batch-major input read in place (folded), with dropout, against two separate
layers (`pytest -m gpu`)."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _rel_l2(a, b):
    return float((a.float() - b.float()).norm() / (b.float().norm() + 1e-20))


@pytest.mark.parametrize("drop", [0.0, 0.25])
def test_pipelined_pair_with_folded_input_matches_sequential_layers(drop):
    """x is a transposed view of batch-major storage without grad: the pair reads it in place for gx_a (and dW_xa), the separate
    layers transpose it first.  Forward states and every weight gradient."""
    from lstm_tensorspark_b200.ops import cuda_lstm
    from lstm_tensorspark_b200.ops.reference import DropoutSpec
    dev = torch.device("cuda", 0)
    torch.manual_seed(21)
    T, B, D, Ha, Hb = 10, 256, 256, 512, 256
    mk = lambda *s, sc=1.0: (torch.randn(*s, device=dev) * sc)
    x = mk(B, T, D, sc=0.5).bfloat16().transpose(0, 1)                       # [T, B, D] view of [B, T, D] storage
    pa = [mk(B, Ha, sc=0.1), mk(B, Ha, sc=0.1), mk(4 * Ha, D, sc=D ** -0.5), mk(4 * Ha, Ha, sc=Ha ** -0.5), mk(4 * Ha, sc=0.1)]
    pb = [mk(B, Hb, sc=0.1), mk(B, Hb, sc=0.1), mk(4 * Hb, Ha, sc=Ha ** -0.5), mk(4 * Hb, Hb, sc=Hb ** -0.5), mk(4 * Hb, sc=0.1)]
    wgt = mk(T, B, Hb)
    step = torch.tensor([3], dtype=torch.int32, device=dev)
    specs = (DropoutSpec(drop, (9, 0), 0, False, step), None) if drop else (None, None)

    def run(pair):
        a = [p.clone().requires_grad_(True) for p in pa]
        b = [p.clone().requires_grad_(True) for p in pb]
        if pair:
            hs, hTa, cTa, hTb, cTb = cuda_lstm.lstm_pair_sequence(x, a, b, schedule="pipelined", dropouts=specs)
        else:
            hs_a, hTa, cTa = cuda_lstm.lstm_layer_sequence(x, *a, dropout=specs[0])
            hs, hTb, cTb = cuda_lstm.lstm_layer_sequence(hs_a, *b)
        loss = (hs.float() * wgt).sum() + hTa.float().sum() + cTb.float().sum() * 0.25
        loss.backward()
        torch.cuda.synchronize()
        cuda_lstm.check_kernel_errors(dev)
        return [hs.detach().float(), hTa.detach().float(), cTa.detach().float()] + [p.grad.float() for p in a + b]

    ref = run(False)
    n0 = {k: cuda_lstm.STATS.get(k, 0) for k in ("pipelined_fwd", "pipelined_side_gemms", "folded_feed")}
    got = run(True)
    n1 = {k: cuda_lstm.STATS.get(k, 0) for k in n0}
    assert all(n1[k] == n0[k] + 1 for k in n0), (n0, n1)
    for i, (g, r) in enumerate(zip(got, ref)):
        assert _rel_l2(g, r) <= 5e-3, (i, tuple(r.shape), _rel_l2(g, r))


@pytest.mark.parametrize("ctas,folded", [(1, False), (1, True), (2, False)])
def test_gemm_row_sums_of_a_ride_along_with_the_weight_gradient(ctas, folded):
    """dW = dG^T · X with rowsum: dW is bit for bit the product without it, and the row sums of dG^T (the bias gradient) match
    an fp64 column sum of dG, overwritten and then accumulated."""
    from lstm_tensorspark_b200.ops import cuda_gemm as G
    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev).manual_seed(5)
    T, B, D, G4 = 6, 256, 256, 1024 + 128
    dg = torch.randn(T * B, G4, device=dev, generator=g).bfloat16()
    xb = torch.randn(B, T, D, device=dev, generator=g).bfloat16()            # batch-major storage
    x = xb.transpose(0, 1).reshape(T * B, D)                                 # the time-major matrix it stands for
    ops = dict(a=dg.t(), b_t=None, b_folded=xb) if folded else dict(a=dg.t(), b_t=x.t())
    want = G.matmul(out_dtype=torch.float32, ctas=ctas, **ops)
    rs = torch.full((G4,), float("nan"), device=dev)
    got = G.matmul(out_dtype=torch.float32, ctas=ctas, rowsum=(rs, False), **ops)
    ref = dg.double().sum(0)
    assert torch.equal(got, want)
    assert float((rs.double() - ref).norm() / ref.norm()) < 1e-5
    acc = torch.zeros(G4, D, device=dev)
    G.matmul(out=acc, accumulate=True, ctas=ctas, rowsum=(rs, True), **ops)
    assert float((rs.double() - 2 * ref).norm() / (2 * ref).norm()) < 1e-5 and torch.equal(acc, want)
