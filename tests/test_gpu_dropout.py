"""Dropout between stacked layers on the GPU (`pytest -m gpu`): the persistent kernels store h_drop bit for bit as the reference
mask applied to their own h_seq, in every forward configuration; gradients with the mask applied on load; the layer pairs; the
standalone kernel of the generic and one-step paths; and, at the headline shape, a step counter that advances inside a captured
CUDA graph.  Every kernel case asserts the instantiation it targets."""
import pytest
import torch

from lstm_tensorspark_b200.ops import reference as ref
from lstm_tensorspark_b200.ops.reference import DropoutSpec

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
TWO_TILES = (6, 2, False, False)


def _rel_l2(a, b):
    return float((a.float() - b.float()).norm() / (b.float().norm() + 1e-20))


def _spec(p=0.2, layer=0, reverse=False, step=5, key=(123, 4)):
    return DropoutSpec(p, key, layer, reverse, torch.tensor([step], dtype=torch.int32, device=DEV))


def _stats():
    from lstm_tensorspark_b200.ops import cuda_lstm
    return {k: cuda_lstm.STATS.get(k, 0) for k in ("fast_fwd", "fast_bwd", "generic_fwd", "generic_bwd", "batch_chunks",
                                                    "pipelined_fwd", "wavefront_fwd")}


def _delta(before):
    return {k: v - before[k] for k, v in _stats().items() if v != before[k]}


def _lengths(T, B, seed):
    g = torch.Generator().manual_seed(seed)
    lengths = torch.randint(1, T + 1, (B,), generator=g, dtype=torch.int32)
    lengths[0], lengths[-1] = 1, T
    return lengths.to(DEV)


def _bits(t):
    return t.contiguous().view(torch.int16)


@pytest.mark.parametrize("T,B,H,cfg,masked,reverse", [
    (16, 128, 64, (6, 1, False, False), False, False),           # one tile, one k-block
    (32, 256, 1024, TWO_TILES, False, False),                    # two tiles per CTA (ping-pong)
    (32, 128, 512, (5, 1, False, True), False, False),           # forward K-split
    (16, 64, 1280, (8, 1, True, False), False, False),           # streamed weights
    (32, 256, 1024, TWO_TILES, True, False),                     # masked
    (32, 256, 1024, TWO_TILES, False, True),                     # reverse
    (32, 256, 1024, TWO_TILES, True, True),                      # masked reverse
    (16, 200, 1024, TWO_TILES, True, False),                     # a partial second tile
])
def test_forward_h_drop_is_the_reference_mask_on_the_kernels_h_seq(T, B, H, cfg, masked, reverse):
    from lstm_tensorspark_b200.ops import cuda_lstm
    from lstm_tensorspark_b200.ops.cuda_ext import ext
    variant = cuda_lstm._seq_variant(B, H, DEV)
    assert ext().lstm_seq_config(False, H, B, variant) == cfg
    g = torch.Generator(device=DEV).manual_seed(T + B + H)
    rn = lambda *s: torch.randn(*s, generator=g, device=DEV)
    gx = (rn(T, B, 4 * H) * 0.5).bfloat16()
    w_h = (rn(4 * H, H) / H ** 0.5).bfloat16()
    lengths = _lengths(T, B, 3) if masked else None
    spec = _spec(0.2, layer=1, reverse=reverse)
    h_seq, _c, _a, h_drop = ext().lstm_seq_fwd(gx, w_h, rn(4 * H) * 0.1, (rn(B, H) * 0.1).bfloat16(), rn(B, H) * 0.1,
                                               cuda_lstm._sync_ws(DEV), variant, lengths=lengths, reverse=reverse,
                                               drop_step=spec.step, drop_desc=spec.desc())
    torch.cuda.synchronize()
    cuda_lstm.check_kernel_errors(DEV)
    h_out = h_seq[:T] if reverse else h_seq[1:]
    want = ref.dropout(h_out, spec)
    assert torch.equal(_bits(h_drop), _bits(want))
    kept = float((h_drop != 0).float().mean())
    assert 0.75 < kept < 0.85


def test_batch_chunks_draw_the_masks_of_the_whole_batch(monkeypatch):
    """B = 400 at H = 1024: two persistent chunks; rows of the second chunk get the masks of their row in the whole batch."""
    from lstm_tensorspark_b200.ops import cuda_lstm
    monkeypatch.setattr(cuda_lstm, "SEQ_VARIANT", 3 << 12)            # in-order operand stream: both runs give the same h_seq
    T, B, D, H = 16, 400, 256, 1024
    g = torch.Generator(device=DEV).manual_seed(7)
    rn = lambda *s: torch.randn(*s, generator=g, device=DEV)
    x = (rn(T, B, D) * 0.5).bfloat16()
    p = [rn(B, H) * 0.1, rn(B, H) * 0.1, rn(4 * H, D) / D ** 0.5, rn(4 * H, H) / H ** 0.5, rn(4 * H) * 0.1]
    spec = _spec(0.3)
    n0 = _stats()
    h_drop, _, _ = cuda_lstm.lstm_layer_sequence(x, *p, dropout=spec)
    assert _delta(n0) == {"fast_fwd": 2, "batch_chunks": 2}
    h_seq, _, _ = cuda_lstm.lstm_layer_sequence(x, *p)
    torch.cuda.synchronize()
    assert torch.equal(_bits(h_drop), _bits(ref.dropout(h_seq, spec)))


def test_generic_fp32_path_and_its_gradients():
    from lstm_tensorspark_b200.ops import cuda_lstm
    T, B, D, H = 6, 9, 12, 20
    g = torch.Generator(device=DEV).manual_seed(8)
    rn = lambda *s: torch.randn(*s, generator=g, device=DEV)
    x = rn(T, B, D)
    p = [rn(B, H) * 0.1, rn(B, H) * 0.1, rn(4 * H, D) / D ** 0.5, rn(4 * H, H) / H ** 0.5, rn(4 * H) * 0.1]
    w = rn(T, B, H)
    spec = _spec(0.4, layer=2, reverse=True)

    def run(fused):
        leaves = [t.clone().requires_grad_(True) for t in [x] + p]
        if fused:
            hs, hT, _ = cuda_lstm.lstm_layer_sequence(*leaves, reverse=True, dropout=spec)
        else:
            hs, hT, _ = cuda_lstm.lstm_layer_sequence(*leaves, reverse=True)
            hs = ref.dropout(hs, spec)
        ((hs * w).sum() + hT.sum()).backward()
        return [hs.detach()] + [t.grad for t in leaves]

    n0 = _stats()
    got = run(True)
    assert _delta(n0) == {"generic_fwd": 1, "generic_bwd": 1}
    want = run(False)
    assert torch.equal(got[0], want[0])
    for a, b in zip(got[1:], want[1:]):
        assert _rel_l2(a, b) < 1e-5


def test_standalone_kernel_one_step_path():
    """The one-step [B,D] path's dropout (time 0) and its backward, bf16 and fp32."""
    from lstm_tensorspark_b200.ops import cuda_lstm
    spec = _spec(0.5, step=77)
    for dt in (torch.bfloat16, torch.float32):
        h = torch.randn(33, 100, device=DEV).to(dt).requires_grad_(True)
        y = cuda_lstm.dropout(h, spec)
        assert torch.equal(_bits(y.detach()) if dt == torch.bfloat16 else y.detach(),
                           _bits(ref.dropout(h.detach(), spec)) if dt == torch.bfloat16 else ref.dropout(h.detach(), spec))
        gy = torch.randn(33, 100, device=DEV).to(dt)
        y.backward(gy)
        assert torch.equal(h.grad.float(), ref.dropout(gy, spec).float())
    x = torch.randn(4, 1, 256, device=DEV).bfloat16()
    assert cuda_lstm.dropout(x, DropoutSpec(0.0, (0, 0), 0, False, spec.step)) is x


@pytest.mark.parametrize("masked,reverse,drop_only", [(False, False, False), (False, False, True), (True, True, False)])
def test_layer_gradients_with_the_mask_on_load(masked, reverse, drop_only):
    """Fused dropout (h_drop stored by the forward kernel, dh_seq masked as the backward kernel loads it) against the layer
    without dropout composed with the reference mask; ``drop_only``: the loss reads h_drop and nothing else."""
    from lstm_tensorspark_b200.ops import cuda_lstm
    T, B, D, H = 32, 256, 256, 1024
    g = torch.Generator(device=DEV).manual_seed(9)
    rn = lambda *s: torch.randn(*s, generator=g, device=DEV)
    x = (rn(T, B, D) * 0.5).bfloat16()
    p = [rn(B, H) * 0.1, rn(B, H) * 0.1, rn(4 * H, D) / D ** 0.5, rn(4 * H, H) / H ** 0.5, rn(4 * H) * 0.1]
    w, wT = rn(T, B, H), rn(B, H)
    lengths = _lengths(T, B, 4) if masked else None
    spec = _spec(0.25, reverse=reverse)

    def run(fused):
        leaves = [x.clone().requires_grad_(True)] + [t.clone().requires_grad_(True) for t in p]
        if fused:
            hs, hT, cT = cuda_lstm.lstm_layer_sequence(*leaves, lengths=lengths, reverse=reverse, dropout=spec)
        else:
            hs, hT, cT = cuda_lstm.lstm_layer_sequence(*leaves, lengths=lengths, reverse=reverse)
            hs = ref.dropout(hs, spec)
        loss = (hs.float() * w).sum()
        if not drop_only:
            loss = loss + (hT.float() * wT).sum() + cT.sum()
        loss.backward()
        torch.cuda.synchronize()
        cuda_lstm.check_kernel_errors(DEV)
        return [hs.detach()] + [t.grad for t in leaves]

    n0 = _stats()
    got = run(True)
    assert _delta(n0) == {"fast_fwd": 1, "fast_bwd": 1}
    want = run(False)
    assert _rel_l2(got[0], want[0]) < 5e-3
    for i, (a, b) in enumerate(zip(got[1:], want[1:])):
        assert _rel_l2(a, b) < 5e-3, (i, _rel_l2(a, b))


@pytest.mark.parametrize("schedule", ["pipelined", "wavefront"])
def test_layer_pair_with_dropout_on_both_layers_matches_separate_layers(schedule):
    """Forced at a small shape: layer a's mask feeds the gated gx_b GEMM and dW_xb; layer b's output is dropped too (the lower
    pair of a 3-layer stack)."""
    from lstm_tensorspark_b200.ops import cuda_lstm
    torch.manual_seed(11)
    T, B, D, Ha, Hb = 12, 256, 256, 512, 256
    mk = lambda *s, sc=1.0: (torch.randn(*s, device=DEV) * sc)
    x = mk(T, B, D, sc=0.5).bfloat16()
    pa = [mk(B, Ha, sc=0.1), mk(B, Ha, sc=0.1), mk(4 * Ha, D, sc=D ** -0.5), mk(4 * Ha, Ha, sc=Ha ** -0.5), mk(4 * Ha, sc=0.1)]
    pb = [mk(B, Hb, sc=0.1), mk(B, Hb, sc=0.1), mk(4 * Hb, Ha, sc=Ha ** -0.5), mk(4 * Hb, Hb, sc=Hb ** -0.5), mk(4 * Hb, sc=0.1)]
    wgt = mk(T, B, Hb)
    sa, sb = _spec(0.3, layer=0), _spec(0.3, layer=1)

    def run(pair):
        xa = x.clone().requires_grad_(True)
        a = [t.clone().requires_grad_(True) for t in pa]
        b = [t.clone().requires_grad_(True) for t in pb]
        if pair:
            hs, hTa, cTa, hTb, cTb = cuda_lstm.lstm_pair_sequence(xa, a, b, schedule=schedule, dropouts=(sa, sb))
        else:
            hs_a, hTa, cTa = cuda_lstm.lstm_layer_sequence(xa, *a, dropout=sa)
            hs, hTb, cTb = cuda_lstm.lstm_layer_sequence(hs_a, *b, dropout=sb)
        loss = (hs.float() * wgt).sum() + hTa.float().sum() + cTa.float().sum() * 0.5 + hTb.float().sum() + cTb.float().sum() * 0.25
        loss.backward()
        torch.cuda.synchronize()
        cuda_lstm.check_kernel_errors(DEV)
        return [hs.detach().float(), hTa.detach().float(), cTa.detach().float(), cTb.detach().float(), xa.grad.float()] + \
               [t.grad.float() for t in a + b]

    ref_out = run(False)
    n0 = _stats()
    got = run(True)
    assert _delta(n0) == {"fast_fwd": 2, "fast_bwd": 2, f"{schedule}_fwd": 1}
    assert float((got[0] == 0).float().mean()) > 0.25                 # the pair's output is the dropped sequence
    for i, (g_, r) in enumerate(zip(got, ref_out)):
        assert _rel_l2(g_, r) <= 5e-3, (i, tuple(r.shape), _rel_l2(g_, r))


def _headline_engine(p, **kw):
    from lstm_tensorspark_b200.config import Config
    from lstm_tensorspark_b200.engine import TrainEngine
    cfg = Config(hidden_units="1024,1024", in_features=1024, seq_len=128, batch_size=256, num_classes=10, partitions=1,
                 sync_mode="none", init="scaled", learn_initial_state=False, device="cuda", quiet=True, dropout=p, seed=3,
                 **kw)
    return TrainEngine(cfg, 0, 1, None, batch_size=256, device=DEV, dtype=torch.bfloat16)


def _headline_batch():
    from lstm_tensorspark_b200 import data as Dm
    xs, ys = Dm.synthetic_sequences(256, 128, 1024, 10, seed=5)
    return torch.as_tensor(xs).to(DEV).bfloat16(), torch.as_tensor(ys).to(DEV)


def test_headline_graph_replays_advance_the_mask_counter(monkeypatch):
    """P = 0.2, --deterministic: 5 replays of a captured step give the losses of 5 eager steps - the counter the masks are keyed
    on advances inside the graph (and capture() puts it back after its warm-up steps).  The losses agree bit for bit in most
    runs; one run on an H100 showed a one-ulp difference in one of them, hence the 1e-6 relative bound (a replay that drew the
    wrong masks is off by orders of magnitude more)."""
    from lstm_tensorspark_b200.ops import cuda_lstm
    monkeypatch.setattr(cuda_lstm, "SEQ_VARIANT", cuda_lstm.SEQ_VARIANT)     # (--deterministic sets a module-level knob)
    x, y = _headline_batch()
    eager = _headline_engine(0.2, deterministic=True)
    want = [float(eager.step(x, y)) for _ in range(5)]
    graphed = _headline_engine(0.2, deterministic=True)
    graphed.capture(x, y)
    assert int(graphed.model.rnn.dropout_step) == 0
    got = [float(graphed.step(x, y)) for _ in range(5)]
    assert int(graphed.model.rnn.dropout_step) == int(eager.model.rnn.dropout_step) == 5
    assert all(abs(a - b) <= 1e-6 * abs(b) for a, b in zip(got, want)), (got, want)
    assert len(set(want)) == 5
    cuda_lstm.check_kernel_errors(DEV)


def test_headline_kept_fraction():
    from lstm_tensorspark_b200.ops import cuda_lstm
    from lstm_tensorspark_b200.ops.cuda_ext import ext
    T, B, H = 128, 256, 1024
    g = torch.Generator(device=DEV).manual_seed(1)
    rn = lambda *s: torch.randn(*s, generator=g, device=DEV)
    spec = _spec(0.2)
    h_seq, _c, _a, h_drop = ext().lstm_seq_fwd((rn(T, B, 4 * H) * 0.5).bfloat16(), (rn(4 * H, H) / H ** 0.5).bfloat16(), rn(4 * H) * 0.1,
                                               torch.zeros(B, H, device=DEV).bfloat16(), torch.zeros(B, H, device=DEV),
                                               cuda_lstm._sync_ws(DEV), cuda_lstm._seq_variant(B, H, DEV), drop_step=spec.step,
                                               drop_desc=spec.desc())
    nz = h_seq[1:] != 0
    kept = float(((h_drop != 0) & nz).sum()) / float(nz.sum())
    assert abs(kept - 0.8) < 1e-3, kept


def test_headline_zero_p_is_the_build_without_dropout(monkeypatch):
    """P = 0: the same kernels (not one extra launch) and the same training; P = 0.2 trains differently.  (Two runs of the
    identical configuration under --deterministic have been seen to differ in the last bit of a loss at this shape on an
    H100, so the losses and weights are compared to within that.)"""
    from lstm_tensorspark_b200.ops import cuda_lstm
    from lstm_tensorspark_b200.ops.cuda_ext import LAUNCHES
    monkeypatch.setattr(cuda_lstm, "SEQ_VARIANT", cuda_lstm.SEQ_VARIANT)     # (--deterministic sets a module-level knob)
    x, y = _headline_batch()
    runs = []
    for kw in ({}, {"dropout": 0.0}, {"dropout": 0.2}):
        from lstm_tensorspark_b200.config import Config
        from lstm_tensorspark_b200.engine import TrainEngine
        cfg = Config(hidden_units="1024,1024", in_features=1024, seq_len=128, batch_size=256, num_classes=10, partitions=1,
                     sync_mode="none", init="scaled", learn_initial_state=False, device="cuda", quiet=True, seed=3,
                     deterministic=True, **kw)
        e = TrainEngine(cfg, 0, 1, None, batch_size=256, device=DEV, dtype=torch.bfloat16)
        k0, l0 = cuda_lstm.STATS["kernels"], LAUNCHES["n"]
        losses = [float(e.step(x, y)) for _ in range(3)]
        torch.cuda.synchronize()
        runs.append((losses, e.flat.data.clone(), cuda_lstm.STATS["kernels"] - k0, LAUNCHES["n"] - l0))
    assert runs[0][2:] == runs[1][2:]
    assert all(abs(a - b) <= 1e-6 * abs(b) for a, b in zip(runs[1][0], runs[0][0])), (runs[1][0], runs[0][0])
    assert _rel_l2(runs[1][1], runs[0][1]) < 1e-6
    assert abs(runs[2][0][-1] - runs[0][0][-1]) > 1e-4 * abs(runs[0][0][-1])
