"""The persistent LSTM kernels (csrc/lstm_seq_wgmma.cu) over long sequences - where the operand ring and the mbarrier phases
wrap hundreds of times and the dataflow counters run far past their early values - against an fp64 reference, within the
error budget of a bf16 emulation of the fast path (tests/lstm_numerics.py): per time step for h_seq and dx, per tensor for the
rest.  Every case names the instantiation it targets and asserts it (`pytest -m gpu`; `-s` prints each case's worst budget
ratios).  The file runs in about 13 s on an H100 80GB HBM3 at a 400 W power limit, fp64 references included."""
import pytest
import torch

import lstm_numerics as N
from lstm_numerics import Bf16

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
PER_STEP = ("h_seq", "dx")


@pytest.fixture(autouse=True)
def _fp32_matmuls(monkeypatch):
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)     # the emulation's fp32 products stay fp32


def _bf(t):
    return t.bfloat16().float()


def _layer_inputs(T, B, H, D, seed, default_init=False):
    """bf16-representable x, h0 and weights, fp32 c0 and bias (both arms get exactly these); bf16-representable loss weights on
    h_seq and h_T (they reach the kernel as bf16), an fp32 one on c_T."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    rn = lambda *s: torch.randn(*s, generator=g, device=DEV)
    if default_init:
        # Config.init's default: the reference's truncated normal with std 1 (saturated gates, |c| grows with T); inputs in the
        # synthetic loader's range, zero initial state
        from lstm_tensorspark_b200 import data as Dm
        from lstm_tensorspark_b200.models.recurrent import truncated_normal_
        cpu = torch.Generator().manual_seed(seed)
        tn = lambda *s: truncated_normal_(torch.empty(*s), 1.0, cpu).to(DEV)
        xs, _ = Dm.synthetic_sequences(B, T, D, 10, seed=seed)
        x = _bf(torch.as_tensor(xs).to(DEV).transpose(0, 1).contiguous())
        params = [x, torch.zeros(B, H, device=DEV), torch.zeros(B, H, device=DEV), _bf(tn(4 * H, D)), _bf(tn(4 * H, H)), tn(4 * H)]
    else:
        params = [_bf(rn(T, B, D) * 0.5), _bf(rn(B, H) * 0.1), rn(B, H) * 0.1, _bf(rn(4 * H, D) / D ** 0.5),
                  _bf(rn(4 * H, H) / H ** 0.5), rn(4 * H) * 0.1]
    return params, (_bf(rn(T, B, H)), _bf(rn(B, H)), rn(B, H))


def _lengths(T, B, seed):
    g = torch.Generator().manual_seed(seed)
    lengths = torch.randint(1, T + 1, (B,), generator=g, dtype=torch.int32)
    lengths[0], lengths[-1] = 1, T                      # both ends: a one-step row and a full-length row
    return lengths.to(DEV)


def _stats():
    from lstm_tensorspark_b200.ops import cuda_lstm
    return {k: cuda_lstm.STATS.get(k, 0) for k in ("fast_fwd", "fast_bwd", "batch_chunks", "pipelined_fwd", "wavefront_fwd")}


def _delta(before):
    return {k: v - before[k] for k, v in _stats().items()}


def _check_all(case, got, fp64, emu, names):
    ratios = {n: N.check_budget(f"{case} {n}", getattr(got, n), getattr(fp64, n), getattr(emu, n), per_step=n in PER_STEP)
              for n in names}
    print(f"\n{case}: worst budget ratio {max(ratios.values()):.3f} (" +
          ", ".join(f"{n} {r:.3f}" for n, r in ratios.items()) + f"); alpha {N.ALPHA}, floor {N.FLOOR:.2e}")


def _layer_case(case, T, B, H, D, cfg_fwd, cfg_bwd, stats, lengths=None, reverse=False, backward=True, default_init=False,
                seed=5, chunk=None):
    """Kernel arm through ops.cuda_lstm.lstm_layer_sequence; fp64 and bf16-emulation arms through lstm_numerics.layer.
    ``chunk``: rows of the persistent batch chunks the op splits B into (the kernels are picked for the chunk)."""
    from lstm_tensorspark_b200.ops import cuda_lstm
    from lstm_tensorspark_b200.ops.cuda_ext import ext
    B_cfg = chunk or B
    variant = cuda_lstm._seq_variant(B_cfg, H, DEV)
    assert ext().lstm_seq_config(False, H, B_cfg, variant) == cfg_fwd
    if backward:
        assert ext().lstm_seq_config(True, H, B_cfg, variant) == cfg_bwd
    params, (dh_seq, dh_T, dc_T) = _layer_inputs(T, B, H, D, seed, default_init)
    x = params[0].bfloat16().requires_grad_(True)
    leaves = [p.clone().requires_grad_(True) for p in params[1:]]
    n0 = _stats()
    hs, hT, cT = cuda_lstm.lstm_layer_sequence(x, *leaves, lengths=lengths, reverse=reverse)
    if backward:
        ((hs.float() * dh_seq).sum() + (hT.float() * dh_T).sum() + (cT * dc_T).sum()).backward()
    torch.cuda.synchronize()
    cuda_lstm.check_kernel_errors(DEV)
    assert _delta(n0) == {**dict.fromkeys(n0, 0), "fast_fwd": 1, "fast_bwd": int(backward), **stats}, _delta(n0)
    got = N.LayerOut(hs, hT, cT, x.grad, *[p.grad for p in leaves]) if backward else N.LayerOut(hs, hT, cT, *[None] * 6)
    names = N.LayerOut._fields if backward else ("h_seq", "h_T", "c_T")
    rounding = Bf16.for_layer(H, B_cfg, variant & ~0xF0)        # (the K splits do not depend on a forced ring depth)
    with torch.no_grad():
        emu = N.layer(*params, dh_seq, dh_T, dc_T, lengths=lengths, reverse=reverse, rounding=rounding)
        fp64 = N.layer(*[p.double() for p in params], dh_seq.double(), dh_T.double(), dc_T.double(), lengths=lengths,
                       reverse=reverse)
        _check_all(case, got, fp64, emu, names)


TWO_TILES = ((6, 2, False, False), (4, 2, False, False))


def test_headline_layer():
    """2 x 1024 headline layer shape: two batch tiles per CTA, ring 6 forward / 4 backward."""
    _layer_case("headline", 128, 256, 1024, 1024, *TWO_TILES, {})


def test_headline_layer_masked_reverse():
    """Masked reverse-time kernels with two tiles per CTA; lengths 1 and T both present."""
    _layer_case("masked reverse", 128, 256, 1024, 1024, *TWO_TILES, {}, lengths=_lengths(128, 256, 1), reverse=True)


def test_unbalanced_tiles_masked():
    """B = 200: two tiles per CTA, the second with 72 valid rows (partial operand loads), per-row lengths."""
    _layer_case("unbalanced tiles", 128, 200, 1024, 128, *TWO_TILES, {}, lengths=_lengths(128, 200, 2))


def test_forward_k_split():
    """One tile per CTA, forward K-split across a cluster of 2 (the peer's half arrives as bf16)."""
    _layer_case("forward K-split", 128, 128, 512, 256, (5, 1, False, True), (6, 1, False, False), {})


def test_one_k_block():
    """H = 64: a single k-block per tile, the accumulator in the dedicated staging buffer."""
    _layer_case("one k-block", 256, 128, 64, 64, (6, 1, False, False), (6, 1, False, False), {})


def test_config4_streamed_layer():
    """BASELINE config 4's layer (4 x 2048, T = 512, B = 64): streamed weights, 8 ring stages, backward in clusters of 2."""
    _layer_case("config-4 layer", 512, 64, 2048, 2048, (8, 1, True, False), (8, 1, True, False), {})


def test_streamed_at_the_resident_boundary():
    """H = 1280: just above the resident limit, streamed in both directions (narrow backward)."""
    _layer_case("streamed narrow", 128, 64, 1280, 256, (8, 1, True, False), (8, 1, True, False), {})


def test_batch_chunks():
    """B = 400 at H = 1024 does not fit co-resident: two persistent chunks (256 + 144 rows), weight gradients accumulated."""
    _layer_case("batch chunks", 64, 400, 1024, 256, *TWO_TILES, {"fast_fwd": 2, "fast_bwd": 2, "batch_chunks": 2},
                chunk=256)


@pytest.mark.parametrize("stages", [2, 3, 4, 5, 6])
def test_every_forced_ring_depth(monkeypatch, stages):
    """Two-tile kernels at every ring depth; the backward ring holds at most 4 stages, deeper rings are forward-only."""
    from lstm_tensorspark_b200.ops import cuda_lstm
    monkeypatch.setattr(cuda_lstm, "SEQ_VARIANT", 2 + 16 * stages)
    bwd = stages <= 4
    _layer_case(f"ring depth {stages}", 64, 256, 1024, 256, (stages, 2, False, False), (stages, 2, False, False) if bwd else None,
                {}, backward=bwd)


def test_reference_default_init():
    """Config.init's default (truncated normal, std 1): saturated gates and a cell state that grows with T."""
    _layer_case("default init", 128, 256, 1024, 1024, *TWO_TILES, {}, default_init=True)


@pytest.mark.parametrize("schedule,H", [("pipelined", 1024), ("wavefront", 512)])
def test_layer_pair(schedule, H):
    """Two stacked layers as one op (ops.cuda_lstm.lstm_pair_sequence) with the schedule pair_schedule picks on an H100:
    pipelined at 2 x 1024, wavefront at 2 x 512."""
    from lstm_tensorspark_b200.ops import cuda_lstm
    T, B, D = 128, 256, H
    if cuda_lstm._sms(DEV) == 132:
        assert cuda_lstm.pair_schedule(T, B, D, H, H, 132, cuda_lstm._coresident_ctas(DEV)) == schedule
    pa, (_, dhTa, dcTa) = _layer_inputs(T, B, H, D, seed=21)
    pb, (dh_seq, dhTb, dcTb) = _layer_inputs(T, B, H, H, seed=22)
    x = pa[0].bfloat16().requires_grad_(True)
    a = [p.clone().requires_grad_(True) for p in pa[1:]]
    b = [p.clone().requires_grad_(True) for p in pb[1:]]
    n0 = _stats()
    hs, hTa, cTa, hTb, cTb = cuda_lstm.lstm_pair_sequence(x, a, b, schedule=schedule)
    loss = (hs.float() * dh_seq).sum() + (hTa.float() * dhTa).sum() + (cTa * dcTa).sum() + (hTb.float() * dhTb).sum() + \
        (cTb * dcTb).sum()
    loss.backward()
    torch.cuda.synchronize()
    cuda_lstm.check_kernel_errors(DEV)
    assert _delta(n0) == {**dict.fromkeys(n0, 0), "fast_fwd": 2, "fast_bwd": 2, f"{schedule}_fwd": 1}, _delta(n0)
    rounding = Bf16.for_layer(H, B, cuda_lstm._pair_variant(schedule))
    with torch.no_grad():
        la, lb = pa[1:], pb[1:]
        emu = N.pair(pa[0], la, lb, dh_seq, dhTa, dcTa, dhTb, dcTb, rounding=rounding)
        d = lambda ts: [t.double() for t in ts]
        fp64 = N.pair(pa[0].double(), d(la), d(lb), *d((dh_seq, dhTa, dcTa, dhTb, dcTb)))
        got_a = N.LayerOut(None, hTa, cTa, x.grad, *[p.grad for p in a])
        got_b = N.LayerOut(hs, hTb, cTb, None, *[p.grad for p in b])
        _check_all(f"{schedule} pair, layer a", got_a, fp64[0], emu[0], [n for n in N.LayerOut._fields if n != "h_seq"])
        _check_all(f"{schedule} pair, layer b", got_b, fp64[1], emu[1], [n for n in N.LayerOut._fields if n != "dx"])
