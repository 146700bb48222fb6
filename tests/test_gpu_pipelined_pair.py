"""The pipelined layer pair (ops/cuda_lstm.py, schedule "pipelined": the two recurrences one after the other, the upper layer's
GEMMs and bias column sums on the SMs the running recurrence leaves idle) against two separate layers, and the column-sum
kernel with a capped grid (`pytest -m gpu`)."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _rel_l2(a, b):
    return float((a.float() - b.float()).norm() / (b.float().norm() + 1e-20))


@pytest.mark.parametrize("ragged", [False, True])
def test_pipelined_pair_matches_sequential_layers(ragged):
    """Forced at a small shape (where the device would pick the wavefront): forward states and every gradient, full-sequence
    loss so that dh_seq flows into the top layer too; with per-row lengths, both layers run their masked kernels."""
    from lstm_tensorspark_b200.ops import cuda_lstm
    dev = torch.device("cuda", 0)
    torch.manual_seed(11)
    T, B, D, Ha, Hb = 12, 256, 256, 512, 256
    mk = lambda *s, sc=1.0: (torch.randn(*s, device=dev) * sc)
    x = mk(T, B, D, sc=0.5).bfloat16()
    pa = [mk(B, Ha, sc=0.1), mk(B, Ha, sc=0.1), mk(4 * Ha, D, sc=D ** -0.5), mk(4 * Ha, Ha, sc=Ha ** -0.5), mk(4 * Ha, sc=0.1)]
    pb = [mk(B, Hb, sc=0.1), mk(B, Hb, sc=0.1), mk(4 * Hb, Ha, sc=Ha ** -0.5), mk(4 * Hb, Hb, sc=Hb ** -0.5), mk(4 * Hb, sc=0.1)]
    wgt = mk(T, B, Hb)
    lengths = None
    if ragged:
        g = torch.Generator().manual_seed(12)
        lengths = torch.randint(1, T + 1, (B,), generator=g, dtype=torch.int32)
        lengths[0], lengths[-1] = 1, T
        lengths = lengths.to(dev)

    def run(pair):
        xa = x.clone().requires_grad_(True)
        a = [p.clone().requires_grad_(True) for p in pa]
        b = [p.clone().requires_grad_(True) for p in pb]
        if pair:
            hs, hTa, cTa, hTb, cTb = cuda_lstm.lstm_pair_sequence(xa, a, b, lengths=lengths, schedule="pipelined")
        else:
            hs_a, hTa, cTa = cuda_lstm.lstm_layer_sequence(xa, *a, lengths=lengths)
            hs, hTb, cTb = cuda_lstm.lstm_layer_sequence(hs_a, *b, lengths=lengths)
        loss = (hs.float() * wgt).sum() + hTa.float().sum() + cTa.float().sum() * 0.5 + hTb.float().sum() + cTb.float().sum() * 0.25
        loss.backward()
        torch.cuda.synchronize()
        cuda_lstm.check_kernel_errors(dev)
        return [hs.detach().float(), hTa.detach().float(), cTa.detach().float(), cTb.detach().float(), xa.grad.float()] + \
               [p.grad.float() for p in a + b]

    ref = run(False)
    n0 = cuda_lstm.STATS.get("pipelined_fwd", 0)
    got = run(True)
    assert cuda_lstm.STATS.get("pipelined_fwd", 0) == n0 + 1
    for i, (g, r) in enumerate(zip(got, ref)):
        assert _rel_l2(g, r) <= (2e-2 if ragged else 5e-3), (i, tuple(r.shape), _rel_l2(g, r))


def test_headline_step_runs_the_schedule_pair_schedule_picks():
    """One training step of the headline model (2 x 1024, T = 128, B = 256) goes through the pair op with the schedule that
    pair_schedule picks for this device - "pipelined" on a 132-SM H100 - with its gradients written into the flat buffer."""
    from lstm_tensorspark_b200.config import Config
    from lstm_tensorspark_b200.engine import TrainEngine
    from lstm_tensorspark_b200 import data as Dm
    from lstm_tensorspark_b200.ops import cuda_lstm
    dev = torch.device("cuda", 0)
    T, B, D, H, C = 128, 256, 1024, 1024, 10
    sched = cuda_lstm.pair_schedule(T, B, D, H, H, cuda_lstm._sms(dev), cuda_lstm._coresident_ctas(dev))
    if cuda_lstm._sms(dev) == 132:
        assert sched == "pipelined"
    cfg = Config(hidden_units="1024,1024", in_features=D, seq_len=T, batch_size=B, num_classes=C, partitions=1, sync_mode="none",
                 init="scaled", learn_initial_state=False, device="cuda", quiet=True)
    eng = TrainEngine(cfg, 0, 1, None, batch_size=B, device=dev, dtype=torch.bfloat16)
    xs, ys = Dm.synthetic_sequences(B, T, D, C, seed=1)
    n0 = cuda_lstm.STATS.get(f"{sched}_fwd", 0)
    loss = float(eng.step(torch.as_tensor(xs).to(dev).bfloat16(), torch.as_tensor(ys).to(dev)))
    torch.cuda.synchronize()
    cuda_lstm.check_kernel_errors(dev)
    assert loss == loss and cuda_lstm.STATS.get(f"{sched}_fwd", 0) == n0 + 1, cuda_lstm.STATS
    assert bool(torch.isfinite(eng.flat.grad).all()) and float(eng.flat.grad.abs().sum()) > 0


@pytest.mark.parametrize("max_ctas", [1, 16, 100])
def test_column_sums_with_a_capped_grid_are_bit_identical(max_ctas):
    """colsum_bf16_into with fewer CTAs than (column blocks x row slabs) walks the same slabs in the same order."""
    from lstm_tensorspark_b200.ops.cuda_ext import ext
    dev = torch.device("cuda", 0)
    torch.manual_seed(3)
    x = torch.randn(32768 + 300, 4096, device=dev).bfloat16()
    want = torch.empty(4096, device=dev)
    ext().colsum_bf16_into(x, want, True)
    got = torch.full((4096,), float("nan"), device=dev)
    ext().colsum_bf16_into(x, got, True, max_ctas=max_ctas)
    assert torch.equal(got, want)
    acc = want.clone()
    ext().colsum_bf16_into(x, acc, False, False, 1024, 2048, max_ctas)       # accumulate into a column range
    assert torch.equal(acc[:1024], want[:1024]) and torch.equal(acc[3072:], want[3072:])
    assert torch.equal(acc[1024:3072], want[1024:3072] * 2)
    assert _rel_l2(want, x.float().sum(0)) < 1e-5
