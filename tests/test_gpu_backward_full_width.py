"""A backward recurrence that has the GPU to itself runs one batch tile per CTA with its K-split reduce-scattered through L2
instead of a cluster's DSMEM (csrc/lstm_seq_wgmma.cu kXchgL2; ops/cuda_lstm.py bwd_tiles_per_cta): at B = 256, H = 1024 that
is 128 CTAs on an H100 instead of the 64 two-tile CTAs its clusters of 4 fit.  The tile choice, the side-GEMM split of the
pipelined pair, the ring depths and the variant fields the kernels accept are host logic (no GPU).  On the GPU
(`pytest -m gpu`) the L2 exchange is held bit for bit against the clustered one-tile kernel where both fit, and the
single-layer op and the pipelined layer pair that take the path against fp64 within the bf16 budget of
tests/lstm_numerics.py."""
import pytest
import torch

from lstm_tensorspark_b200.ops import cuda_lstm as CL
from lstm_tensorspark_b200.ops.cuda_ext import ext


def test_bwd_tiles_per_cta_table():
    # (SMs, CTAs co-resident in clusters of 4) -> {(B, H): tiles per CTA}
    table = {
        (132, 120): {(128, 256): 1, (128, 1024): 1, (128, 2048): None, (256, 256): 1, (256, 1024): 1, (256, 2048): None,
                     (512, 256): 1, (512, 1024): None, (512, 2048): None},
        (128, 128): {(128, 256): 1, (128, 1024): 1, (128, 2048): 1, (256, 256): 1, (256, 1024): 1, (256, 2048): None,
                     (512, 256): 1, (512, 1024): 2, (512, 2048): None},
        (120, 120): {(128, 256): 1, (128, 1024): 1, (128, 2048): None, (256, 256): 1, (256, 1024): 2, (256, 2048): None,
                     (512, 256): 1, (512, 1024): None, (512, 2048): None},
    }
    for (sms, cores), want in table.items():
        for (B, H), tiles in want.items():
            assert CL.bwd_tiles_per_cta(B, H, sms, cores) == tiles, (sms, cores, B, H)
    # never more tiles than the shared choice, and the same answer wherever that is not 2
    for B in range(128, 2049, 128):
        for H in range(64, 2049, 64):
            shared, bwd = CL.tiles_per_cta(B, H, 120), CL.bwd_tiles_per_cta(B, H, 132, 120)
            assert bwd == shared or (shared, bwd) == (2, 1), (B, H, shared, bwd)


def test_pipelined_bwd_split_table():
    # (SMs, H_a, H_b) -> (dx_b CTAs, CTAs of each of dW_xb / dW_hb): free = SMs - H_a / 16 - 4 in the ratio 4H_a : 3H_a : 3H_b
    table = {(132, 1024, 1024): (26, 19), (132, 512, 1024): (30, 33), (132, 1024, 512): (30, 17), (114, 1024, 1024): (18, 14),
             (132, 256, 256): (45, 33)}
    for (sms, h_a, h_b), want in table.items():
        n_dx, side = CL.pipelined_bwd_split(sms, h_a, h_b)
        assert (n_dx, side) == want, (sms, h_a, h_b, n_dx, side)
        assert h_a // 16 + n_dx + 2 * side + CL._COLSUM_SMS <= sms


def test_l2_exchange_configs():
    E = ext()
    # the one-tile L2-exchange backward: 4 ring stages at H >= 1024 (measured fastest), the deepest ring that fits below
    assert E.lstm_seq_config(True, 1024, 256, 0, True) == (4, 1, False, False)
    assert E.lstm_seq_config(True, 512, 256, 0, True) == (6, 1, False, False)
    # unchanged: the clustered one-tile and two-tile backward
    assert E.lstm_seq_config(True, 1024, 128, 0) == (5, 1, False, False)
    assert E.lstm_seq_config(True, 1024, 256, 2) == (4, 2, False, False)
    # one tile per CTA with resident weights only
    for H, B, var in ((1024, 256, 2), (2048, 128, 0)):
        with pytest.raises(RuntimeError, match="L2 exchange"):
            E.lstm_seq_config(True, H, B, var, True)
    with pytest.raises(RuntimeError, match="L2 exchange"):
        E.lstm_seq_config(False, 1024, 256, 0, True)
    # instantiated ring depths: 4 to 6
    assert E.lstm_seq_config(True, 1024, 256, 16 * 4, True)[0] == 4
    with pytest.raises(RuntimeError, match="4 to 6"):
        E.lstm_seq_config(True, 1024, 256, 16 * 3, True)
    # the exchange counters follow the k-block counters in the sync workspace: a layout whose k-block counters still fit
    # (5 tiles x 48 = 240 lines) is rejected once the 5 x 12 exchange counters are added
    assert E.lstm_seq_config(True, 768, 640, 0)[1] == 1
    with pytest.raises(RuntimeError, match="sync workspace"):
        E.lstm_seq_config(True, 768, 640, 0, True)
    # the variant's fields: [0:4) tiles per CTA, [4:8) ring stages, [12:15) = 3 the in-order stream, bit 16 one counter per
    # batch tile.  Any other bit, or another value in [12:15), is refused.
    for bwd, want in ((False, {3 << 12: (4, 1, False, False), 1 << 16: (4, 1, False, False), 2 + 16 * 4: (4, 2, False, False)}),
                      (True, {3 << 12: (5, 1, False, False), 1 << 16: (5, 1, False, False), 2 + 16 * 4: (4, 2, False, False)})):
        for var, cfg in want.items():
            assert E.lstm_seq_config(bwd, 1024, 256, var) == cfg, (bwd, var)
        refused = [m << 12 for m in (1, 2, 4, 5, 6, 7)] + [2 << 16, 3 << 16] + [1 << b for b in (8, 9, 15, 18, 19, 20, 21, 30)]
        for var in refused + [2 + 16 * 4 + (1 << 19), (3 << 12) | (1 << 20), -1]:
            with pytest.raises(RuntimeError, match="unsupported variant"):
                E.lstm_seq_config(bwd, 1024, 256, var)


# ---- on the GPU ------------------------------------------------------------------------------------------------------------
DEV = torch.device("cuda", 0)
T, H = 32, 1024
IN_ORDER = 4096 * 3          # debug mode 3: operand k-blocks issued (and accumulated) in index order, real results


@pytest.fixture
def _fp32_matmuls(monkeypatch):
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)     # the emulation's fp32 products stay fp32


def _bf(t):
    return t.bfloat16().float()


def _lengths(B, seed):
    g = torch.Generator().manual_seed(seed)
    lengths = torch.randint(1, T + 1, (B,), generator=g, dtype=torch.int32)
    lengths[0], lengths[-1] = 1, T                      # both ends: a one-step row and a full-length row
    return lengths.to(DEV)


def _needs_full_width(B):
    if CL.bwd_tiles_per_cta(B, H, CL._sms(DEV), CL._coresident_ctas(DEV, 4)) != 1:
        pytest.skip("the one-tile backward CTAs do not fit this device")


@pytest.mark.gpu
@pytest.mark.parametrize("masked,reverse,dropout", [(False, False, False), (False, False, True), (True, False, False),
                                                    (False, True, False)])
def test_l2_exchange_matches_the_cluster_exchange_bit_for_bit(masked, reverse, dropout):
    """B = 128, where the clustered one-tile kernel fits too (64 CTAs): with the k-blocks accumulated in index order by both,
    the L2 exchange sums the same bf16 partials in the same source order, so dpre, dh0 and dc0 are the same bits."""
    from lstm_tensorspark_b200.ops.reference import DropoutSpec
    B = 128
    _needs_full_width(B)
    E = ext()
    assert E.lstm_seq_config(True, H, B, 0) == (5, 1, False, False)
    g = torch.Generator(device=DEV).manual_seed(61 + 2 * masked + 4 * reverse + 8 * dropout)
    rn = lambda *s: torch.randn(*s, generator=g, device=DEV)
    gx = (rn(T, B, 4 * H) * 0.5).bfloat16()
    w_h = (rn(4 * H, H) / H ** 0.5).bfloat16()
    lengths = _lengths(B, 9) if masked else None
    _, c_seq, act = E.lstm_seq_fwd(gx, w_h, rn(4 * H) * 0.1, (rn(B, H) * 0.1).bfloat16(), rn(B, H) * 0.1, CL._sync_ws(DEV), 0,
                                   lengths=lengths, reverse=reverse)
    dh_seq, dh_T, dc_T = (rn(T, B, H) * 0.1).bfloat16(), rn(B, H) * 0.1, rn(B, H) * 0.1
    spec = DropoutSpec(0.2, (321, 4), 1, reverse, torch.tensor([3], dtype=torch.int32, device=DEV)) if dropout else None
    drop = dict(drop_step=spec.step, drop_desc=spec.desc()) if dropout else {}
    w_hT = w_h.t().contiguous()
    outs = {}
    for name, xchg in (("cluster", None), ("l2", CL._xchg_buffer(B, H, DEV))):
        outs[name] = E.lstm_seq_bwd(dh_seq, w_hT, act, c_seq, dh_T, dc_T, CL._sync_ws(DEV), IN_ORDER, lengths=lengths,
                                    reverse=reverse, xchg=xchg, **drop)
        torch.cuda.synchronize()
        CL.check_kernel_errors(DEV)
    for n, a, b in zip(("dpre", "dh0", "dc0"), outs["l2"], outs["cluster"]):
        assert torch.equal(a, b), (n, float((a.float() - b.float()).abs().max()))


def _counts():
    return {k: CL.STATS.get(k, 0) for k in ("fast_fwd", "fast_bwd", "bwd_full_width", "pipelined_fwd")}


def _delta(before):
    return {k: v - before[k] for k, v in _counts().items()}


def _layer_inputs(B, D, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    rn = lambda *s: torch.randn(*s, generator=g, device=DEV)
    params = [_bf(rn(T, B, D) * 0.5), _bf(rn(B, H) * 0.1), rn(B, H) * 0.1, _bf(rn(4 * H, D) / D ** 0.5),
              _bf(rn(4 * H, H) / H ** 0.5), rn(4 * H) * 0.1]
    return params, (_bf(rn(T, B, H)), _bf(rn(B, H)), rn(B, H))


@pytest.mark.gpu
@pytest.mark.parametrize("masked,reverse", [(False, False), (True, False), (False, True)])
def test_single_layer_op_runs_the_one_tile_backward(_fp32_matmuls, masked, reverse):
    """``lstm_layer_sequence`` at the headline layer shape (B = 256): the backward at one tile per CTA with the L2 exchange;
    outputs and every gradient against fp64 within the budget."""
    import lstm_numerics as N
    B = 256
    _needs_full_width(B)
    assert CL._bwd_full_width(B, H, DEV)
    params, (dh_seq, dh_T, dc_T) = _layer_inputs(B, 256, 71 + masked + 2 * reverse)
    lengths = _lengths(B, 5) if masked else None
    x = params[0].bfloat16().requires_grad_(True)
    leaves = [p.clone().requires_grad_(True) for p in params[1:]]
    n0 = _counts()
    hs, hT, cT = CL.lstm_layer_sequence(x, *leaves, lengths=lengths, reverse=reverse)
    ((hs.float() * dh_seq).sum() + (hT.float() * dh_T).sum() + (cT * dc_T).sum()).backward()
    torch.cuda.synchronize()
    CL.check_kernel_errors(DEV)
    assert _delta(n0) == {"fast_fwd": 1, "fast_bwd": 1, "bwd_full_width": 1, "pipelined_fwd": 0}, _delta(n0)
    got = N.LayerOut(hs, hT, cT, x.grad, *[p.grad for p in leaves])
    with torch.no_grad():
        emu = N.layer(*params, dh_seq, dh_T, dc_T, lengths=lengths, reverse=reverse,
                      rounding=N.Bf16.for_layer(H, B, CL._fwd_variant(B, H, DEV)))
        fp64 = N.layer(*[p.double() for p in params], dh_seq.double(), dh_T.double(), dc_T.double(), lengths=lengths,
                       reverse=reverse)
    for n in N.LayerOut._fields:
        N.check_budget(f"single layer masked={masked} reverse={reverse} {n}", getattr(got, n), getattr(fp64, n),
                       getattr(emu, n), per_step=n in ("h_seq", "dx"))


@pytest.mark.gpu
def test_pipelined_pair_runs_layer_b_backward_at_one_tile(_fp32_matmuls):
    """The pipelined pair at the headline shape (T = 32): L_b's backward runs alone at one tile per CTA, dx_b next to L_a's
    backward (which waits for it block by block) with dW_xb, dW_hb and db_b.  Both layers' outputs and gradients against fp64."""
    import lstm_numerics as N
    B = 256
    _needs_full_width(B)
    pa, (_, dhTa, dcTa) = _layer_inputs(B, 1024, 81)
    pb, (dh_seq, dhTb, dcTb) = _layer_inputs(B, H, 82)
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
    assert _delta(n0) == {"fast_fwd": 2, "fast_bwd": 2, "bwd_full_width": 1, "pipelined_fwd": 1}, _delta(n0)
    rounding = N.Bf16.for_layer(H, B, CL._pair_variant("pipelined"))
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
