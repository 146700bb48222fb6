"""AWD-LSTM's remaining dropouts on the GPU (`pytest -m gpu`): locked masks in every persistent-kernel configuration (h_drop bit
for bit against the reference mask of the kernel's own h_seq), layer and pair gradients under locked masks, the masked embedding
gather (bit for bit) and table gradient (against fp64), a whole language-model step with AWD's PTB recipe against the fp64 model
fed the same masks, graph replays and resume, P = 0, evaluation and generation."""
import dataclasses

import pytest
import torch

from lstm_tensorspark_b200.ops import reference as ref
from lstm_tensorspark_b200.ops.reference import DropoutSpec

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
TWO_TILES = (6, 2, False, False)
RECIPE = dict(locked_dropout=True, input_dropout=0.65, dropout=0.3, output_dropout=0.4, embedding_dropout=0.1,
              weight_drop=0.5)


def _rel_l2(a, b):
    return float((a.double() - b.double()).norm() / (b.double().norm() + 1e-30))


def _step(n):
    return torch.tensor([n], dtype=torch.int32, device=DEV)


def _spec(p=0.2, layer=0, reverse=False, step=5, key=(123, 4), **kw):
    return DropoutSpec(p, key, layer, reverse, _step(step), locked=True, **kw)


def _stats(keys=("fast_fwd", "fast_bwd", "batch_chunks", "pipelined_fwd", "wavefront_fwd", "embed_fwd", "embed_bwd",
                 "embed_fwd_dropout", "embed_bwd_dropout")):
    from lstm_tensorspark_b200.ops import cuda_lstm
    return {k: cuda_lstm.STATS.get(k, 0) for k in keys}


def _delta(before):
    return {k: v - before[k] for k, v in _stats().items() if v != before[k]}


def _bits(t):
    return t.contiguous().view(torch.int16) if t.dtype == torch.bfloat16 else t.contiguous().view(torch.int32)


def _lengths(T, B, seed):
    g = torch.Generator().manual_seed(seed)
    lengths = torch.randint(1, T + 1, (B,), generator=g, dtype=torch.int32)
    lengths[0], lengths[-1] = 1, T
    return lengths.to(DEV)


# ---- locked masks in the persistent kernels ---------------------------------------------------------------------------------
@pytest.mark.parametrize("T,B,H,cfg,masked,reverse", [
    (16, 128, 64, (6, 1, False, False), False, False),           # one tile, one k-block
    (32, 256, 1024, TWO_TILES, False, False),                    # two tiles per CTA (ping-pong)
    (32, 128, 512, (5, 1, False, True), False, False),           # forward K-split
    (16, 64, 1280, (8, 1, True, False), False, False),           # streamed weights
    (32, 256, 1024, TWO_TILES, True, False),                     # masked
    (32, 256, 1024, TWO_TILES, True, True),                      # masked reverse
])
def test_locked_h_drop_is_the_reference_mask_on_the_kernels_h_seq(T, B, H, cfg, masked, reverse):
    from lstm_tensorspark_b200.ops import cuda_lstm
    from lstm_tensorspark_b200.ops.cuda_ext import ext
    variant = cuda_lstm._seq_variant(B, H, DEV)
    assert ext().lstm_seq_config(False, H, B, variant) == cfg
    g = torch.Generator(device=DEV).manual_seed(T + B + H)
    rn = lambda *s: torch.randn(*s, generator=g, device=DEV)
    lengths = _lengths(T, B, 3) if masked else None
    spec = _spec(0.3, layer=1, reverse=reverse)
    h_seq, _c, _a, h_drop = ext().lstm_seq_fwd((rn(T, B, 4 * H) * 0.5).bfloat16(), (rn(4 * H, H) / H ** 0.5).bfloat16(),
                                               rn(4 * H) * 0.1, (rn(B, H) * 0.1).bfloat16(), rn(B, H) * 0.1,
                                               cuda_lstm._sync_ws(DEV), variant, lengths=lengths, reverse=reverse,
                                               drop_step=spec.step, drop_desc=spec.desc())
    torch.cuda.synchronize()
    cuda_lstm.check_kernel_errors(DEV)
    h_out = h_seq[:T] if reverse else h_seq[1:]
    assert torch.equal(_bits(h_drop), _bits(ref.dropout(h_out, spec)))
    dropped = (h_drop == 0) & (h_out != 0)
    assert all(torch.equal(dropped[t] | (h_out[t] == 0), dropped[0] | (h_out[t] == 0)) for t in range(T))   # one mask, every t


def test_locked_batch_chunks_draw_the_masks_of_the_whole_batch(monkeypatch):
    from lstm_tensorspark_b200.ops import cuda_lstm
    monkeypatch.setattr(cuda_lstm, "SEQ_VARIANT", 3 << 12)            # in-order operand stream: both runs give the same h_seq
    T, B, D, H = 16, 400, 256, 1024
    g = torch.Generator(device=DEV).manual_seed(7)
    rn = lambda *s: torch.randn(*s, generator=g, device=DEV)
    x = (rn(T, B, D) * 0.5).bfloat16()
    p = [rn(B, H) * 0.1, rn(B, H) * 0.1, rn(4 * H, D) / D ** 0.5, rn(4 * H, H) / H ** 0.5, rn(4 * H) * 0.1]
    spec = _spec(0.4)
    n0 = _stats()
    h_drop, _, _ = cuda_lstm.lstm_layer_sequence(x, *p, dropout=spec)
    assert _delta(n0) == {"fast_fwd": 2, "batch_chunks": 2}
    h_seq, _, _ = cuda_lstm.lstm_layer_sequence(x, *p)
    torch.cuda.synchronize()
    assert torch.equal(_bits(h_drop), _bits(ref.dropout(h_seq, spec)))


@pytest.mark.parametrize("masked,reverse", [(False, False), (True, True)])
def test_locked_layer_gradients_with_the_mask_on_load(masked, reverse):
    from lstm_tensorspark_b200.ops import cuda_lstm
    T, B, D, H = 32, 256, 256, 1024
    g = torch.Generator(device=DEV).manual_seed(9)
    rn = lambda *s: torch.randn(*s, generator=g, device=DEV)
    x = (rn(T, B, D) * 0.5).bfloat16()
    p = [rn(B, H) * 0.1, rn(B, H) * 0.1, rn(4 * H, D) / D ** 0.5, rn(4 * H, H) / H ** 0.5, rn(4 * H) * 0.1]
    w = rn(T, B, H)
    lengths = _lengths(T, B, 4) if masked else None
    spec = _spec(0.4, reverse=reverse)

    def run(fused):
        leaves = [x.clone().requires_grad_(True)] + [t.clone().requires_grad_(True) for t in p]
        if fused:
            hs, hT, cT = cuda_lstm.lstm_layer_sequence(*leaves, lengths=lengths, reverse=reverse, dropout=spec)
        else:
            hs, hT, cT = cuda_lstm.lstm_layer_sequence(*leaves, lengths=lengths, reverse=reverse)
            hs = ref.dropout(hs, spec)
        ((hs.float() * w).sum() + hT.float().sum() + cT.sum()).backward()
        torch.cuda.synchronize()
        cuda_lstm.check_kernel_errors(DEV)
        return [hs.detach()] + [t.grad for t in leaves]

    n0 = _stats()
    got = run(True)
    assert _delta(n0) == {"fast_fwd": 1, "fast_bwd": 1}
    want = run(False)
    for i, (a, b) in enumerate(zip(got, want)):
        assert _rel_l2(a, b) < 5e-3, (i, _rel_l2(a, b))


@pytest.mark.parametrize("schedule", ["pipelined", "wavefront"])
def test_layer_pair_with_the_top_layer_dropped(schedule):
    """A two-layer stack: layer a's locked mask between the layers, layer b's (the top layer's, --output_dropout) on the pair's
    output, against the two layers run one after the other."""
    from lstm_tensorspark_b200.ops import cuda_lstm
    torch.manual_seed(11)
    T, B, D, Ha, Hb = 12, 256, 256, 512, 256
    mk = lambda *s, sc=1.0: (torch.randn(*s, device=DEV) * sc)
    x = mk(T, B, D, sc=0.5).bfloat16()
    pa = [mk(B, Ha, sc=0.1), mk(B, Ha, sc=0.1), mk(4 * Ha, D, sc=D ** -0.5), mk(4 * Ha, Ha, sc=Ha ** -0.5), mk(4 * Ha, sc=0.1)]
    pb = [mk(B, Hb, sc=0.1), mk(B, Hb, sc=0.1), mk(4 * Hb, Ha, sc=Ha ** -0.5), mk(4 * Hb, Hb, sc=Hb ** -0.5), mk(4 * Hb, sc=0.1)]
    wgt = mk(T, B, Hb)
    sa, sb = _spec(0.3, layer=0), _spec(0.4, layer=1)

    def run(pair):
        xa = x.clone().requires_grad_(True)
        a = [t.clone().requires_grad_(True) for t in pa]
        b = [t.clone().requires_grad_(True) for t in pb]
        if pair:
            hs, hTa, cTa, hTb, cTb = cuda_lstm.lstm_pair_sequence(xa, a, b, schedule=schedule, dropouts=(sa, sb))
        else:
            hs_a, hTa, cTa = cuda_lstm.lstm_layer_sequence(xa, *a, dropout=sa)
            hs, hTb, cTb = cuda_lstm.lstm_layer_sequence(hs_a, *b, dropout=sb)
        ((hs.float() * wgt).sum() + hTb.float().sum()).backward()
        torch.cuda.synchronize()
        cuda_lstm.check_kernel_errors(DEV)
        return [hs.detach().float(), hTb.detach().float(), xa.grad.float()] + [t.grad.float() for t in a + b]

    want = run(False)
    n0 = _stats()
    got = run(True)
    assert _delta(n0) == {"fast_fwd": 2, "fast_bwd": 2, f"{schedule}_fwd": 1}
    zero = got[0] == 0
    assert 0.35 < float(zero.float().mean()) < 0.45 and all(torch.equal(zero[t], zero[0]) for t in range(T))
    for i, (a, b) in enumerate(zip(got, want)):
        assert _rel_l2(a, b) <= 5e-3, (i, _rel_l2(a, b))


# ---- the masked embedding kernels ---------------------------------------------------------------------------------------------
def _tokens(B, T, V, seed, hot=False):
    g = torch.Generator().manual_seed(seed)
    tok = torch.randint(-1, V + 1, (B, T), generator=g, dtype=torch.int32)
    if hot:                                                          # one id at a third of the positions: a multi-piece segment
        tok[torch.rand(B, T, generator=g) < 0.33] = 5
    return tok.to(DEV)


def _drop_kw(si, se):
    kw = {}
    if si is not None:
        kw.update(in_step=si.step, in_desc=si.desc())
    if se is not None:
        kw.update(row_step=se.step, row_desc=se.desc())
    return kw


MASKS = {"input": (True, False), "rows": (False, True), "both": (True, True)}


@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("E", [256, 20])
@pytest.mark.parametrize("T,ragged", [(9, False), (9, True), (1, False)])
@pytest.mark.parametrize("masks", list(MASKS))
def test_gather_is_the_reference_bit_for_bit(dt, E, T, ragged, masks):
    from lstm_tensorspark_b200.ops.cuda_ext import ext
    V, B = 300, 37
    table = torch.randn(V, E, device=DEV).to(dt)
    tok = _tokens(B, T, V, T + E)
    lengths = _lengths(T, B, 2) if ragged else None
    use_i, use_e = MASKS[masks]
    si = _spec(0.65, site="input") if use_i else None
    se = DropoutSpec(0.3, (123, 4), 0, False, _step(5), site="rows") if use_e else None
    x = ext().embed_fwd(table, tok, lengths, **_drop_kw(si, se))
    want = ref.embedding(tok, table, lengths, input_dropout=si, embedding_dropout=se)
    assert torch.equal(_bits(x), _bits(want))


def _table_grad_fp64(dx, tok, lengths, V, si, se):
    T, B, E = dx.shape
    t = tok.t().long()
    keep = (t >= 0) & (t < V)
    if lengths is not None:
        keep &= torch.arange(T, device=DEV).unsqueeze(1) < lengths.long().unsqueeze(0)
    d = dx.double()
    if si is not None:
        d = d * ref.dropout_mask(si, T, B, E, device=DEV).double() * float(ref.dropout_scale(si.p))
    out = torch.zeros(V, E, dtype=torch.float64, device=DEV)
    out.index_add_(0, t[keep], d[keep])
    mag = torch.zeros(V, E, dtype=torch.float64, device=DEV).index_add_(0, t[keep], d[keep].abs())
    if se is not None:
        rows = ref.embedding_row_mask(se, V, device=DEV).double().unsqueeze(1)
        out, mag = out * rows * float(ref.dropout_scale(se.p)), mag * rows * float(ref.dropout_scale(se.p))
    return out, mag


@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("E", [256, 20])
@pytest.mark.parametrize("ragged", [False, True])
@pytest.mark.parametrize("masks", list(MASKS))
def test_table_gradient_against_fp64(dt, E, ragged, masks):
    from lstm_tensorspark_b200.ops.cuda_ext import ext
    V, B, T = 300, 64, 12
    tok = _tokens(B, T, V, E + 1, hot=True)
    lengths = _lengths(T, B, 6) if ragged else None
    dx = torch.randn(T, B, E, device=DEV).to(dt)
    use_i, use_e = MASKS[masks]
    si = _spec(0.65, site="input") if use_i else None
    se = DropoutSpec(0.3, (123, 4), 0, False, _step(5), site="rows") if use_e else None
    kw = _drop_kw(si, se)
    dW = torch.full((V, E), float("nan"), device=DEV)
    n0 = _stats()
    ext().embed_bwd(dx, tok, lengths, dW, False, **kw)
    want, mag = _table_grad_fp64(dx, tok, lengths, V, si, se)
    n = int((tok.t().long() == 5).sum())
    assert n > 2 * 64                                                # id 5 spans several pieces
    assert bool(((dW.double() - want).abs() <= 4 * n * 2 ** -24 * mag + 1e-30).all())
    again = torch.empty_like(dW)
    ext().embed_bwd(dx, tok, lengths, again, False, **kw)
    assert torch.equal(_bits(again), _bits(dW))
    if se is not None:
        dropped = ~ref.embedding_row_mask(se, V, device=DEV)
        assert bool((dW[dropped] == 0).all()) and bool(dropped.any())
        base = torch.randn(V, E, device=DEV)
        acc = base.clone()
        ext().embed_bwd(dx, tok, lengths, acc, True, **kw)
        assert torch.equal(acc[dropped], base[dropped])
        kept = ~dropped
        assert bool(((acc[kept].double() - base[kept].double() - want[kept]).abs()
                     <= 4 * n * 2 ** -24 * (mag[kept] + base[kept].double().abs()) + 1e-30).all())


def test_op_counts_masked_launches_and_zero_p_launches_the_plain_kernels():
    from lstm_tensorspark_b200.ops import cuda_embed
    V, E, B, T = 300, 256, 16, 8
    table = torch.randn(V, E, device=DEV).requires_grad_(True)
    tok = _tokens(B, T, V, 1)
    n0 = _stats()
    x0 = cuda_embed.embedding(tok, table)
    x0.sum().backward()
    assert _delta(n0) == {"embed_fwd": 1, "embed_bwd": 1}
    g0 = table.grad.clone()
    table.grad = None
    zero = DropoutSpec(0.0, (1, 1), 0, False, _step(0), site="input")
    n0 = _stats()
    xz = cuda_embed.embedding(tok, table, input_dropout=zero, embedding_dropout=dataclasses.replace(zero, site="rows"))
    xz.sum().backward()
    assert _delta(n0) == {"embed_fwd": 1, "embed_bwd": 1}
    assert torch.equal(xz, x0) and torch.equal(table.grad, g0)
    table.grad = None
    n0 = _stats()
    cuda_embed.embedding(tok, table, input_dropout=_spec(0.5, site="input")).sum().backward()
    assert _delta(n0) == {"embed_fwd": 1, "embed_bwd": 1, "embed_fwd_dropout": 1, "embed_bwd_dropout": 1}


# ---- whole language-model steps -------------------------------------------------------------------------------------------------
def _lm_engine(deterministic=True, **kw):
    from lstm_tensorspark_b200.config import Config
    from lstm_tensorspark_b200.engine import TrainEngine
    cfg = Config(**{**dict(next_token=True, vocab_size=1024, hidden_units="256,256", in_features=256, seq_len=16, batch_size=64,
                           partitions=1, sync_mode="none", init="scaled", learn_initial_state=False, device="cuda", quiet=True,
                           seed=2, deterministic=deterministic), **kw}).validate()
    return TrainEngine(cfg, 0, 1, None, batch_size=64, device=DEV, dtype=torch.bfloat16)


def _lm_batch(seed=3):
    from lstm_tensorspark_b200 import data as Dm
    x, y = Dm.synthetic_next_token(64, 16, 1024, seed=seed)[:2]
    return torch.as_tensor(x).to(DEV), torch.as_tensor(y).to(DEV)


@pytest.mark.parametrize("tied", [False, True])
@pytest.mark.parametrize("graph", [False, True])
def test_recipe_step_against_the_fp64_model_fed_the_same_masks(tied, graph):
    """AWD's PTB recipe (every dropout and weight drop): the GPU step's loss and every parameter's gradient against the fp64 model
    (the reference ops on the CPU) with the same weights, key and step counter, within a bf16 budget; the rows the row mask drops
    get no embedding gradient (with --tie_embeddings only the softmax's)."""
    from lstm_tensorspark_b200.models.classifier import SequenceClassifier
    from lstm_tensorspark_b200.ops import cuda_lstm
    eng = _lm_engine(tie_embeddings=tied, **RECIPE)
    x, y = _lm_batch()
    model = eng.model
    cpu = SequenceClassifier(eng.cfg, batch_size=64, device="cpu").double()
    cpu.load_state_dict({k: v.detach().double().cpu() for k, v in model.state_dict().items()})
    cpu.set_compute_dtype(torch.float64)
    cpu.rnn.dropout_key, cpu.rnn.dropout_step = model.rnn.dropout_key, 0
    if graph:
        eng.capture(x, y)
        assert int(model.rnn.dropout_step) == 0
    n0 = _stats()
    loss = float(eng.step(x, y))
    torch.cuda.synchronize()
    cuda_lstm.check_kernel_errors(DEV)
    if not graph:
        d = _delta(n0)
        assert d["embed_fwd_dropout"] == 1 and d["embed_bwd_dropout"] == 1
    got = {n: p.grad.detach().double().cpu() for n, p in model.named_parameters() if p.grad is not None}
    want_loss, _logits, _ = cpu(x.cpu(), y.cpu())
    want_loss.backward()
    want_loss = float(want_loss)
    want = {n: p.grad for n, p in cpu.named_parameters() if p.grad is not None}
    assert abs(loss - want_loss) <= 5e-3 * abs(want_loss), (loss, want_loss)
    assert got.keys() == want.keys()
    for n in want:
        assert _rel_l2(got[n], want[n]) < 3e-2, (n, _rel_l2(got[n], want[n]))
    se = cpu.rnn.embedding_dropout_spec()
    dropped = ~ref.embedding_row_mask(se, 1024)
    table = [n for n in want if n.startswith("embedding")][0]
    assert bool(dropped.any())
    if not tied:
        assert bool((got[table][dropped] == 0).all()) and bool((want[table][dropped] == 0).all())
    assert int(model.rnn.dropout_step) == 1


def test_graph_replays_draw_new_masks_and_resume_draws_the_uninterrupted_ones():
    x, y = _lm_batch()
    eager = _lm_engine(**RECIPE)
    want = [float(eager.step(x, y)) for _ in range(4)]
    graphed = _lm_engine(**RECIPE)
    graphed.capture(x, y)
    got = [float(graphed.step(x, y)) for _ in range(4)]
    assert int(graphed.model.rnn.dropout_step) == 4 and len(set(want)) == 4
    assert all(abs(a - b) <= 1e-5 * abs(b) for a, b in zip(got, want)), (got, want)
    # resume: at learning rate 0 only the masks change from step to step, so an engine set to step 2 must see step 2's loss
    frozen = _lm_engine(optimizer="sgd", learning_rate=0.0, **RECIPE)
    steps = [float(frozen.step(x, y)) for _ in range(3)]
    resumed = _lm_engine(optimizer="sgd", learning_rate=0.0, **RECIPE)
    resumed.set_dropout_step(2)
    assert len(set(steps)) == 3
    assert abs(float(resumed.step(x, y)) - steps[2]) <= 1e-5 * abs(steps[2])


def test_zero_p_adds_no_launch_and_trains_the_same():
    from lstm_tensorspark_b200.ops import cuda_lstm
    from lstm_tensorspark_b200.ops.cuda_ext import LAUNCHES
    x, y = _lm_batch()
    runs = []
    for kw in ({}, dict(input_dropout=0.0, output_dropout=0.0, embedding_dropout=0.0)):
        e = _lm_engine(tie_embeddings=True, **kw)
        k0, l0, n0 = cuda_lstm.STATS["kernels"], LAUNCHES["n"], _stats()
        losses = [float(e.step(x, y)) for _ in range(2)]
        torch.cuda.synchronize()
        runs.append((losses, e.flat.data.clone(), cuda_lstm.STATS["kernels"] - k0, LAUNCHES["n"] - l0, _delta(n0)))
    assert runs[0][2:] == runs[1][2:] and "embed_fwd_dropout" not in runs[1][4]
    assert all(abs(a - b) <= 1e-6 * abs(b) for a, b in zip(runs[1][0], runs[0][0]))
    assert _rel_l2(runs[1][1], runs[0][1]) < 1e-6


def test_evaluation_and_generation_ignore_the_flags():
    x, y = _lm_batch(4)
    on, off = _lm_engine(tie_embeddings=True, **RECIPE), _lm_engine(tie_embeddings=True)
    assert torch.equal(on.flat.data, off.flat.data)
    n0 = _stats()
    a, b = on.evaluate(x, y), off.evaluate(x, y)
    assert "embed_fwd_dropout" not in _delta(n0)
    assert [float(v) for v in a] == [float(v) for v in b]
    outs = [e.model.generate(x[:, :8].int(), None, 6, 1.0, 5, graph=False) for e in (on, off)]
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
