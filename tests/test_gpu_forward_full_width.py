"""A forward recurrence that has the GPU to itself runs one batch tile per CTA where its own co-residency allows it
(ops/cuda_lstm.py fwd_tiles_per_cta): at B = 256, H = 1024 that is 128 CTAs on an H100 instead of the 64 two-tile CTAs the
backward kernel's clusters of 4 need.  The tile choice is host logic (no GPU); the one-tile forward kernel is held against an
fp64 reference within the bf16 budget of tests/lstm_numerics.py and against the two-tile kernel on the same inputs, alone and
inside the single-layer op and the pipelined layer pair (`pytest -m gpu` for those)."""
import pytest
import torch

from lstm_tensorspark_b200.ops import cuda_lstm as CL

DEV = torch.device("cuda", 0)
H100 = {4: 120, 2: 132}          # an H100 SXM: 132 SMs, 120 CTAs co-resident in clusters of 4


def test_fwd_tiles_per_cta_table():
    h100 = lambda c: H100[c]
    # the headline layer: the backward needs two tiles on 64 CTAs, the unclustered forward fits 128 one-tile CTAs
    assert CL.tiles_per_cta(256, 1024, 120) == 2
    assert CL.fwd_tiles_per_cta(256, 1024, 132, h100) == 1
    # 114 SMs: 128 one-tile CTAs do not fit, the forward keeps two tiles
    assert CL.fwd_tiles_per_cta(256, 1024, 114, lambda c: 112) == 2
    # one tile already (32 CTAs, forward K-split in clusters of 2)
    assert CL.fwd_tiles_per_cta(128, 512, 132, h100) == 1
    # forward K-split at one tile per CTA (clusters of 2): decided by the co-residency of clusters of 2, not the SM count
    assert CL.fwd_tiles_per_cta(512, 512, 132, h100) == 1
    assert CL.fwd_tiles_per_cta(512, 512, 132, lambda c: 120) == 2
    # streamed weights (H > 1152): whatever tiles_per_cta says
    for B, H in ((64, 2048), (128, 1280), (256, 2048), (128, 4096)):
        assert CL.fwd_tiles_per_cta(B, H, 132, h100) == CL.tiles_per_cta(B, H, h100(CL._bwd_cluster(H))), (B, H)
    # the one-tile forward's default ring at H >= 1024 holds 4 stages; smaller H and two tiles keep the deepest ring that fits
    from lstm_tensorspark_b200.ops.cuda_ext import ext
    assert ext().lstm_seq_config(False, 1024, 256, 0) == (4, 1, False, False)
    assert ext().lstm_seq_config(False, 1152, 128, 0) == (4, 1, False, False)
    assert ext().lstm_seq_config(False, 1024, 256, 2) == (6, 2, False, False)
    assert ext().lstm_seq_config(False, 960, 128, 0)[0] == 6
    # never more tiles than the shared choice, and the same answer wherever that is not 2
    for B in range(128, 2049, 128):
        for H in range(64, 2049, 64):
            shared, fwd = CL.tiles_per_cta(B, H, h100(CL._bwd_cluster(H))), CL.fwd_tiles_per_cta(B, H, 132, h100)
            assert fwd == shared or (shared, fwd) == (2, 1), (B, H, shared, fwd)


# ---- on the GPU ------------------------------------------------------------------------------------------------------------
T, B, H = 32, 256, 1024
ONE_TILE, TWO_TILES = (4, 1, False, False), (6, 2, False, False)


@pytest.fixture
def _fp32_matmuls(monkeypatch):
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)     # the emulation's fp32 products stay fp32


def _bf(t):
    return t.bfloat16().float()


def _lengths(seed):
    g = torch.Generator().manual_seed(seed)
    lengths = torch.randint(1, T + 1, (B,), generator=g, dtype=torch.int32)
    lengths[0], lengths[-1] = 1, T                      # both ends: a one-step row and a full-length row
    return lengths.to(DEV)


def _needs_full_width():
    if CL.fwd_tiles_per_cta(B, H, CL._sms(DEV), lambda c: CL._coresident_ctas(DEV, c)) != 1:
        pytest.skip("128 one-tile CTAs do not fit this device")
    assert CL._fwd_full_width(B, H, DEV)


def _check_kernels(case, one, two, fp64, emu, per_step):
    """The one-tile kernel's output against fp64 within the budget, and against the two-tile kernel's within the same
    allowance: |one - two| <= ALPHA |emulation - fp64| + FLOOR |fp64| (the two kernels accumulate the k-blocks in arrival
    order with different wgmma shapes, so their bits may differ)."""
    import lstm_numerics as N
    N.check_budget(f"{case}: one tile vs fp64", one, fp64, emu, per_step=per_step)
    N.check_budget(f"{case}: two tiles vs fp64", two, fp64, emu, per_step=per_step)
    N.check_budget(f"{case}: one tile vs two tiles", one.double(), two.double(), two.double() + (emu.double() - fp64.double()),
                   per_step=per_step)


@pytest.mark.gpu
@pytest.mark.parametrize("masked,reverse,dropout", [(False, False, False), (False, False, True), (True, False, False),
                                                    (False, True, False)])
def test_one_tile_forward_kernel(_fp32_matmuls, masked, reverse, dropout):
    """h_seq, c_seq and the saved activations of the forward kernel at one tile per CTA (the variant ``_fwd_variant`` picks)
    and at two (``_seq_variant``) on the same inputs; with dropout, h_drop is the reference mask on the kernel's own h_seq."""
    import lstm_numerics as N
    from lstm_tensorspark_b200.ops import reference as ref
    from lstm_tensorspark_b200.ops.cuda_ext import ext
    from lstm_tensorspark_b200.ops.reference import DropoutSpec
    _needs_full_width()
    E = ext()
    v1, v2 = CL._fwd_variant(B, H, DEV), CL._seq_variant(B, H, DEV)
    assert E.lstm_seq_config(False, H, B, v1) == ONE_TILE and E.lstm_seq_config(False, H, B, v2) == TWO_TILES
    D = 256
    g = torch.Generator(device=DEV).manual_seed(31 + 2 * masked + 4 * reverse + 8 * dropout)
    rn = lambda *s: torch.randn(*s, generator=g, device=DEV)
    x, h0, c0 = _bf(rn(T, B, D) * 0.5), _bf(rn(B, H) * 0.1), rn(B, H) * 0.1
    w_x, w_h, bias = _bf(rn(4 * H, D) / D ** 0.5), _bf(rn(4 * H, H) / H ** 0.5), rn(4 * H) * 0.1
    rounding = N.Bf16.for_layer(H, B, v1)
    assert rounding.fwd_split == 1
    gx = N._round(rounding, x.reshape(T * B, D) @ w_x.t()).view(T, B, 4 * H).bfloat16()     # the emulation's gx, bit for bit
    lengths = _lengths(7) if masked else None
    spec = DropoutSpec(0.2, (123, 4), 1, reverse, torch.tensor([5], dtype=torch.int32, device=DEV)) if dropout else None
    drop = dict(drop_step=spec.step, drop_desc=spec.desc()) if dropout else {}
    outs = {}
    for name, v in (("one", v1), ("two", v2)):
        outs[name] = E.lstm_seq_fwd(gx, w_h.bfloat16(), bias, h0.bfloat16(), c0, CL._sync_ws(DEV), v, lengths=lengths,
                                    reverse=reverse, **drop)
        torch.cuda.synchronize()
        CL.check_kernel_errors(DEV)
    keep = N._keep(lengths, T, B, DEV)
    with torch.no_grad():
        emu = N._forward(x, h0, c0, w_x, w_h, bias, keep, reverse, rounding, None)
        fp64 = N._forward(*[t.double() for t in (x, h0, c0, w_x, w_h, bias)], keep, reverse, None, None)
    case = f"masked={masked} reverse={reverse} dropout={dropout}"
    rows = slice(0, T) if reverse else slice(1, T + 1)      # the computed states (the other row is h0 / c0)
    one, two = outs["one"], outs["two"]
    _check_kernels(f"{case} h_seq", one[0][rows].float(), two[0][rows].float(), fp64[0][rows], emu[0][rows], True)
    _check_kernels(f"{case} c_seq", one[1][rows], two[1][rows], fp64[1][rows], emu[1][rows], True)
    _check_kernels(f"{case} act", one[2].float(), two[2].float(), fp64[2].reshape(T, B, 4 * H), emu[2].reshape(T, B, 4 * H),
                   False)
    if dropout:
        want = ref.dropout(one[0][rows], spec)
        assert torch.equal(one[3].view(torch.int16), want.contiguous().view(torch.int16))


def _counts():
    return {k: CL.STATS.get(k, 0) for k in ("fast_fwd", "fast_bwd", "fwd_full_width", "pipelined_fwd")}


def _delta(before):
    return {k: v - before[k] for k, v in _counts().items()}


def _layer_inputs(D, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    rn = lambda *s: torch.randn(*s, generator=g, device=DEV)
    params = [_bf(rn(T, B, D) * 0.5), _bf(rn(B, H) * 0.1), rn(B, H) * 0.1, _bf(rn(4 * H, D) / D ** 0.5),
              _bf(rn(4 * H, H) / H ** 0.5), rn(4 * H) * 0.1]
    return params, (_bf(rn(T, B, H)), _bf(rn(B, H)), rn(B, H))


@pytest.mark.gpu
def test_single_layer_op_runs_the_one_tile_forward(_fp32_matmuls):
    """``lstm_layer_sequence`` at the headline layer shape: the forward at one tile per CTA, the backward at two; outputs
    and every gradient against fp64 within the budget."""
    import lstm_numerics as N
    _needs_full_width()
    params, (dh_seq, dh_T, dc_T) = _layer_inputs(256, 41)
    x = params[0].bfloat16().requires_grad_(True)
    leaves = [p.clone().requires_grad_(True) for p in params[1:]]
    n0 = _counts()
    hs, hT, cT = CL.lstm_layer_sequence(x, *leaves)
    ((hs.float() * dh_seq).sum() + (hT.float() * dh_T).sum() + (cT * dc_T).sum()).backward()
    torch.cuda.synchronize()
    CL.check_kernel_errors(DEV)
    assert _delta(n0) == {"fast_fwd": 1, "fast_bwd": 1, "fwd_full_width": 1, "pipelined_fwd": 0}, _delta(n0)
    got = N.LayerOut(hs, hT, cT, x.grad, *[p.grad for p in leaves])
    with torch.no_grad():
        emu = N.layer(*params, dh_seq, dh_T, dc_T, rounding=N.Bf16.for_layer(H, B, CL._seq_variant(B, H, DEV)))
        fp64 = N.layer(*[p.double() for p in params], dh_seq.double(), dh_T.double(), dc_T.double())
    for n in N.LayerOut._fields:
        N.check_budget(f"single layer {n}", getattr(got, n), getattr(fp64, n), getattr(emu, n), per_step=n in ("h_seq", "dx"))


@pytest.mark.gpu
def test_pipelined_pair_runs_layer_b_forward_at_one_tile(_fp32_matmuls):
    """The pipelined pair at the headline shape (T = 32): L_b's forward, which runs alone after the side GEMMs, takes one tile
    per CTA; L_a's forward and both backward recurrences keep two.  Both layers' outputs and gradients against fp64."""
    import lstm_numerics as N
    _needs_full_width()
    pa, (_, dhTa, dcTa) = _layer_inputs(1024, 51)
    pb, (dh_seq, dhTb, dcTb) = _layer_inputs(H, 52)
    x = pa[0].bfloat16().requires_grad_(True)
    a = [p.clone().requires_grad_(True) for p in pa[1:]]
    b = [p.clone().requires_grad_(True) for p in pb[1:]]
    n0 = _counts()
    hs, hTa, cTa, hTb, cTb = CL.lstm_pair_sequence(x, a, b, schedule="pipelined")
    loss = (hs.float() * dh_seq).sum() + (hTa.float() * dhTa).sum() + (cTa * dcTa).sum() + (hTb.float() * dhTb).sum() + \
        (cTb * dcTb).sum()
    loss.backward()
    torch.cuda.synchronize()
    CL.check_kernel_errors(DEV)
    assert _delta(n0) == {"fast_fwd": 2, "fast_bwd": 2, "fwd_full_width": 1, "pipelined_fwd": 1}, _delta(n0)
    rounding = N.Bf16.for_layer(H, B, CL._pair_variant("pipelined"))
    assert rounding == N.Bf16.for_layer(H, B, CL._pair_variant("pipelined") & ~15)          # fwd_split stays 1 at one tile
    with torch.no_grad():
        la, lb = pa[1:], pb[1:]
        emu = N.pair(pa[0], la, lb, dh_seq, dhTa, dcTa, dhTb, dcTb, rounding=rounding)
        d = lambda ts: [t.double() for t in ts]
        fp64 = N.pair(pa[0].double(), d(la), d(lb), *d((dh_seq, dhTa, dcTa, dhTb, dcTb)))
    got_a = N.LayerOut(None, hTa, cTa, x.grad, *[p.grad for p in a])
    got_b = N.LayerOut(hs, hTb, cTb, None, *[p.grad for p in b])
    for tag, got, f, e, skip in (("a", got_a, fp64[0], emu[0], "h_seq"), ("b", got_b, fp64[1], emu[1], "dx")):
        for n in N.LayerOut._fields:
            if n != skip:
                N.check_budget(f"pipelined pair, layer {tag} {n}", getattr(got, n), getattr(f, n), getattr(e, n),
                               per_step=n in ("h_seq", "dx"))
