"""Pooling over time on the GPU (``--pooling mean | max | attention``): whole training steps of TrainEngine against an fp64
reference of the pooled classifier, within the budget of its bf16 emulation (tests/lstm_numerics.py), the pool op alone at
awkward shapes, its bitwise determinism and a negative control.

The model reference composes the layer loops of lstm_numerics as ``lstm_numerics.model`` does, with the pooled ``s`` in place of
h_T; the top layer receives the pool's gradient as its dh_seq (no dh_T).  Rounding points of the pooling (csrc/seq_pool.cu):
  mean       s = (sum_{t<len} h_t) / len in fp32;  dh_t = ds / len in fp32, stored bf16;
  max        s = max h_t (exact);  dh = ds at the first argmax, stored bf16;
  attention  P = bf16 h x bf16(W_a) accumulated in fp32 (wgmma GEMM); u = tanh(P + b_a), e = u . v, the softmax alpha and
             s = sum alpha_t h_t in fp32;
             backward dalpha = ds . h_t, de = alpha (dalpha - sum alpha dalpha), dU = de v (1 - u^2) in fp32; the GEMMs read
             bf16(dU): G = bf16(dU) x bf16(W_a)^T and dW_a = h^T bf16(dU) in fp32; dh_t = alpha_t ds + G stored bf16 once;
             db_a = sum of the fp32 dU, dv = sum de u_t, in fp32;
  all        s is stored bf16 and read by the last-state head (``lstm_numerics.model``'s head rounding: logits = bf16 s x bf16(W)
             + b; ds = dlogits W^T with the fp32 W, stored bf16; dW = bf16(s)^T dlogits and db in fp32);
             positions t >= len_b are read by nothing and get dh = 0."""
import pytest
import torch

import lstm_numerics as N
from test_gpu_model_numerics import (_engine, _is_h100, _lengths, _names, _roundings, _reference_params, _sched, _segments,
                                     DEV)

pytestmark = pytest.mark.gpu
C = 10


@pytest.fixture(autouse=True)
def _fp32_matmuls(monkeypatch):
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)


def _stat(k):
    from lstm_tensorspark_b200.ops import cuda_lstm
    return cuda_lstm.STATS.get(k, 0)


def _keep_tb(lengths, T, B, dev):
    k = N._keep(lengths, T, B, dev)
    return torch.ones(T, B, dtype=torch.bool, device=dev) if k is None else k.t()


def pool_forward(h, keep, mode, att, r, norm_all=False):
    """``h [T,B,H]`` -> (s [B,H], what the backward needs).  ``norm_all``: the mean divides by T (the negative control)."""
    T = h.shape[0]
    kf = keep.to(h.dtype).unsqueeze(2)
    hm = h * kf
    if mode == "mean":
        n = torch.full_like(keep.sum(0), T) if norm_all else keep.sum(0)
        n = n.to(h.dtype).unsqueeze(1)
        return hm.sum(0) / n, (n,)
    if mode == "max":
        hx = torch.where(keep.unsqueeze(2), h, float("-inf"))
        top = hx.max(0, keepdim=True).values
        t_idx = torch.arange(T, device=h.device).view(T, 1, 1).expand_as(hx)
        first = torch.where(hx == top, t_idx, T).min(0, keepdim=True).values
        return top.squeeze(0), (first,)
    Wa, ba, v = att
    u = torch.tanh(hm @ N._round(r, Wa) + ba)
    e = torch.where(keep, u @ v, float("-inf"))
    alpha = torch.softmax(e, 0)
    return (alpha.unsqueeze(2) * hm).sum(0), (alpha, u, kf)


def pool_backward(ds, h, keep, mode, att, saved, r):
    """-> (dh_seq [T,B,H] in the reference's precision, grads of the attention parameters by name)."""
    kf = keep.to(h.dtype).unsqueeze(2)
    if mode == "mean":
        return N._round(r, (ds / saved[0]).unsqueeze(0) * kf), {}
    if mode == "max":
        dh = torch.zeros_like(h).scatter_(0, saved[0], ds.unsqueeze(0))
        return N._round(r, dh), {}
    Wa, ba, v = att
    alpha, u, _ = saved
    hm = h * kf
    dalpha = (ds.unsqueeze(0) * hm).sum(2)
    de = alpha * (dalpha - (alpha * dalpha).sum(0, keepdim=True))
    dU = de.unsqueeze(2) * v * (1 - u * u) * kf
    dUr = N._round(r, dU)
    G = dUr @ N._round(r, Wa).t()
    dh = N._round(r, (alpha.unsqueeze(2) * ds.unsqueeze(0) + G) * kf)
    A = u.shape[2]
    grads = {"Attention/weights": hm.reshape(-1, hm.shape[2]).t() @ dUr.reshape(-1, A), "Attention/bias": dU.sum((0, 1)),
             "Attention/context": (de.unsqueeze(2) * u).sum((0, 1))}
    return dh, grads


def model_pooled(x, layers, head, att, labels, mode, lengths=None, bidirectional=False, dropout=None, rounding=None,
                 norm_all=False):
    """``lstm_numerics.model`` with the head on the pooled top-layer output -> (loss, grads by name)."""
    dt = torch.float64 if rounding is None else torch.float32
    dev = x.device
    B, T, _ = x.shape
    L = len(layers)
    dirs = (False, True) if bidirectional else (False,)
    keep = N._keep(lengths, T, B, dev)

    def rnd(l, d):
        r = rounding[l] if isinstance(rounding, (list, tuple)) else rounding
        return r[d] if isinstance(r, tuple) else r

    def params(l, d):
        return layers[l][d] if bidirectional else layers[l]

    seq = x.transpose(0, 1).to(dt)
    saved = []
    for l in range(L):
        outs, sv = [], []
        for d, rev in enumerate(dirs):
            r, p = rnd(l, d), params(l, d)
            fw = N._forward(seq, *p, keep, rev, r, None)
            h_seq = N._state_out(fw, rev)[0]
            sc = None
            if dropout is not None and dropout.p > 0 and l < L - 1:
                sc = N._drop_scale(dropout, l, rev, T, B, h_seq.shape[2], dt, dev)
                h_seq = N._round(r, h_seq * sc)
            outs.append(h_seq)
            sv.append((fw, seq, keep, sc))
        saved.append(sv)
        seq = torch.cat(outs, 2) if bidirectional else outs[0]
    r_top = rnd(L - 1, 0)
    keep_tb = _keep_tb(lengths, T, B, dev)
    att = None if att is None else tuple(a.to(dt) for a in att)
    s, ps = pool_forward(seq, keep_tb, mode, att, r_top, norm_all)
    s = N._round(r_top, s)
    W, b = head[0].to(dt), head[1].to(dt)
    logp = torch.log_softmax(s @ N._round(r_top, W) + b, 1)
    lab = labels.long().view(-1, 1).to(dev)
    loss = -logp.gather(1, lab).mean()
    dlogits = (logp.exp() - torch.zeros_like(logp).scatter_(1, lab, 1.0)) / B
    ds = N._round(r_top, dlogits @ W.t())
    grads = {"Dense1/weights": s.t() @ dlogits, "Dense1/bias": dlogits.sum(0)}
    dh_top, g_att = pool_backward(ds, seq, keep_tb, mode, att, ps, r_top)
    grads.update(g_att)
    H_top = seq.shape[2] // len(dirs)
    incoming = [dh_top[..., d * H_top:(d + 1) * H_top] for d in range(len(dirs))]
    for l in range(L - 1, -1, -1):
        dxs = []
        for d, rev in enumerate(dirs):
            fw, x_in, kp, sc = saved[l][d]
            p, r = params(l, d), rnd(l, d)
            g = N._backward(fw, x_in, p[2], p[3], incoming[d], None, None, kp, rev, r, None, dh_scale=sc)
            for k, v in zip(("h0", "c0", "w_x", "w_h", "bias"), g[1:]):
                grads[f"LSTMLayer{l}" + ("_reverse" if rev else "") + f"/{k}"] = v
            dxs.append(g[0])
        if l == 0:
            break
        if bidirectional:
            total = N._round(rnd(l, 0), dxs[0] + dxs[1])
            H_low = total.shape[2] // 2
            incoming = [total[..., :H_low], total[..., H_low:]]
        else:
            incoming = [dxs[0]]
    return loss, grads


def _pool_names(eng):
    out = _names(eng)
    a = eng.model.attention
    if a is not None:
        out[id(a.weights)], out[id(a.bias)], out[id(a.context)] = "Attention/weights", "Attention/bias", "Attention/context"
    return out


def _case(case, mode, hidden, T, B, D, path, steps=2, lengths_seed=None, bidirectional=False, dropout=0.0, learning_rate=0.0,
          graph=False, negative=False, A=128, dtype=torch.bfloat16):
    """Training steps, each checked (loss and every gradient of the flat buffer) against the fp64 reference at the weights it
    read.  ``path``: a STATS key one step must bump (besides the pooling launches).  ``graph``: captured on the first batch and
    replayed on every batch, each with lengths of its own.  ``negative``: the reference (both arms) takes the mean over T - the
    check must fail.  ``dtype``: the engine's compute dtype (fp32: the lstm_numerics.Fp32 arm and floor)."""
    from lstm_tensorspark_b200 import data as Dm
    bf16 = dtype == torch.bfloat16
    eng = _engine(dtype, hidden_units=hidden, in_features=D, seq_len=T, batch_size=B, num_classes=C, bidirectional=bidirectional,
                  dropout=dropout, variable_length=lengths_seed is not None, learning_rate=learning_rate, pooling=mode,
                  attention_units=A)
    flat = eng.flat
    xs, ys = Dm.synthetic_sequences(steps * B, T, D, C, seed=5)
    xs, ys = torch.as_tensor(xs).to(DEV).to(dtype), torch.as_tensor(ys).to(DEV)
    seg = _segments(eng, _pool_names(eng))
    rounding = _roundings([int(h) for h in hidden.split(",")], T, B, D, bidirectional) if bf16 else N.Fp32()
    floor = N.FLOOR if bf16 else N.FLOOR_F32
    worst = {}
    for s in range(steps):
        x, y = xs[s * B:(s + 1) * B], ys[s * B:(s + 1) * B]
        lengths = None if lengths_seed is None else _lengths(T, B, lengths_seed + s)
        before = {"p": flat.data.clone(), "drop": int(eng.model.rnn.dropout_step)}
        n_fwd, n_bwd, n_path = _stat("pool_fwd"), _stat("pool_bwd"), _stat(path)
        if graph and s == 0:
            eng.capture(x, y, lengths=lengths)
            assert _stat("pool_fwd") > n_fwd and _stat("pool_bwd") > n_bwd and _stat(path) > n_path, case
            n_fwd, n_bwd, n_path = _stat("pool_fwd"), _stat("pool_bwd"), _stat(path)
        loss = eng.step(x, y, lengths)
        torch.cuda.synchronize()
        if not graph:
            assert _stat("pool_fwd") == n_fwd + 1 and _stat("pool_bwd") == n_bwd + 1 and _stat(path) > n_path, (case, s)
        got = {"loss": loss.float()}
        for k, (o, shape) in seg.items():
            got[k] = flat.grad[o:o + shape.numel()].view(shape).clone()
        drop = N.Dropout(dropout, eng.model.rnn.dropout_key, before["drop"]) if dropout > 0 else None
        with torch.no_grad():
            arms = {}
            for arm, dt, r in (("fp64", torch.float64, None), ("emu", torch.float32, rounding)):
                layers, head = _reference_params(eng, seg, before["p"], dt, bf16_weights=bf16)
                att = None
                if mode == "attention":
                    att = tuple(before["p"][o:o + sh.numel()].view(sh).to(dt)
                                for o, sh in (seg[f"Attention/{k}"] for k in ("weights", "bias", "context")))
                l_, g_ = model_pooled(x.to(dt), layers, head, att, y, mode, lengths, bidirectional, drop, r, norm_all=negative)
                arms[arm] = {"loss": l_, **g_}
            if negative:
                with pytest.raises(AssertionError):
                    for k in ("loss", "Dense1/weights"):
                        N.check_budget(f"{case} {k}", got[k], arms["fp64"][k], arms["emu"][k])
                return
            assert set(got) <= set(arms["fp64"]) and (mode != "attention" or "Attention/context" in got), sorted(got)
            for k, g in got.items():
                worst[k] = max(worst.get(k, 0.0), N.check_budget(f"{case} step {s} {k}", g, arms["fp64"][k], arms["emu"][k],
                                                                 floor=floor))
            del arms
    top = sorted(worst.items(), key=lambda kv: -kv[1])[:3]
    print(f"\n{case}: worst budget ratio " + ", ".join(f"{k} {v:.3f}" for k, v in top))


MODES = ("mean", "max", "attention")


@pytest.mark.parametrize("mode", MODES)
def test_headline_pipelined_pair(mode):
    if _is_h100():
        assert _sched(128, 256, 1024, 1024, 1024) == "pipelined"
    _case(f"{mode} headline", mode, "1024,1024", 128, 256, 1024, "pipelined_fwd")


@pytest.mark.parametrize("mode", MODES)
def test_wavefront_pair(mode):
    if _is_h100():
        assert _sched(128, 256, 512, 512, 512) == "wavefront"
    _case(f"{mode} wavefront", mode, "512,512", 128, 256, 512, "wavefront_fwd")


@pytest.mark.parametrize("mode", MODES)
def test_ragged(mode):
    """Lengths 1 and T included: padded positions are not pooled and get no gradient."""
    _case(f"{mode} ragged", mode, "1024,1024", 128, 256, 1024, "pipelined_fwd", lengths_seed=31)


@pytest.mark.parametrize("mode", MODES)
def test_bidirectional_ragged(mode):
    """[h_fwd(t) | h_rev(t)] pooled into a [2H] feature; each direction receives its half of the pool's dh_seq."""
    _case(f"{mode} bidirectional ragged", mode, "512,512", 64, 256, 256, "fast_bwd", lengths_seed=41, bidirectional=True)


@pytest.mark.parametrize("mode", MODES)
def test_dropout(mode):
    _case(f"{mode} dropout", mode, "1024,1024", 128, 256, 1024, "pipelined_fwd", dropout=0.2)


@pytest.mark.parametrize("mode", MODES)
def test_batch_chunks(mode):
    """B = 400 at H = 1024: every layer runs as two persistent chunks below one pool."""
    _case(f"{mode} batch chunks", mode, "1024,1024", 32, 400, 256, "batch_chunks")


@pytest.mark.parametrize("mode", MODES)
def test_adam_graph_replays_with_changing_lengths(mode):
    """Captured once, replayed on 3 batches with lengths of their own: the pool reads the lengths on the device each replay."""
    _case(f"{mode} adam graph", mode, "1024,1024", 128, 256, 1024, "pipelined_fwd", steps=3, lengths_seed=51,
          learning_rate=1e-3, graph=True)


def test_negative_control_mean_over_all_steps():
    """A reference that averages over T instead of len_b must fail the budget."""
    _case("mean negative control", "mean", "512,512", 64, 128, 256, "fast_fwd", steps=1, lengths_seed=61, negative=True)


def test_last_launches_no_pooling():
    """The default ``--pooling last`` is the parent model: no pooling launch."""
    from lstm_tensorspark_b200 import data as Dm
    eng = _engine(hidden_units="512,512", in_features=256, seq_len=16, batch_size=128, num_classes=C)
    assert eng.model.attention is None
    xs, ys = Dm.synthetic_sequences(128, 16, 256, C, seed=5)
    before = (_stat("pool_fwd"), _stat("pool_bwd"), _stat("pool_attention_fwd"), _stat("pool_attention_bwd"))
    eng.step(torch.as_tensor(xs).to(DEV).bfloat16(), torch.as_tensor(ys).to(DEV))
    eng.evaluate(torch.as_tensor(xs).to(DEV).bfloat16(), torch.as_tensor(ys).to(DEV))
    torch.cuda.synchronize()
    assert (_stat("pool_fwd"), _stat("pool_bwd"), _stat("pool_attention_fwd"), _stat("pool_attention_bwd")) == before


# ---- the op alone ------------------------------------------------------------------------------------------------------------
def _op_case(mode, T, B, H, A, ragged, dtype=torch.bfloat16, seed=0, poison=False):
    from lstm_tensorspark_b200.ops import functional as F
    g = torch.Generator().manual_seed(seed)
    h = torch.randn(T, B, H, generator=g).to(DEV, dtype)
    if dtype == torch.bfloat16 and mode == "max":
        h = (h * 4).round().to(dtype) / 4                           # many ties: the gradient goes to the first t
    att = None
    if mode == "attention":
        att = ((torch.randn(H, A, generator=g) / H ** 0.5).to(DEV), (0.1 * torch.randn(A, generator=g)).to(DEV),
               (torch.randn(A, generator=g) / A ** 0.5).to(DEV))
    ds = torch.randn(B, H, generator=g).to(DEV)
    lengths = None
    if ragged:
        lengths = torch.randint(1, T + 1, (B,), generator=g, dtype=torch.int32)
        lengths[0], lengths[-1] = 1, T
        lengths = lengths.to(DEV)
        if poison:
            keep = _keep_tb(lengths, T, B, DEV).unsqueeze(2)
            h = torch.where(keep, h, torch.full_like(h, float("nan") if mode != "attention" else 1e30))
    hp = h.clone().requires_grad_(True)
    ap = None if att is None else tuple(a.clone().requires_grad_(True) for a in att)
    s = F.pool_sequence(hp, lengths, mode, ap)
    s.backward(ds)
    grads = {"s": s.detach(), "dh": hp.grad}
    if ap is not None:
        grads.update({"Attention/weights": ap[0].grad, "Attention/bias": ap[1].grad, "Attention/context": ap[2].grad})
    return h, att, ds, lengths, grads


OP_SHAPES = [
    (7, 19, 96, 40, True, torch.bfloat16),          # B, H and A off every tile size: the generic GEMM
    (5, 130, 200, 72, True, torch.bfloat16),        # B not a multiple of 128, H and A not multiples of 64
    (9, 33, 128, 64, False, torch.bfloat16),
    (16, 160, 256, 128, True, torch.bfloat16),      # T·B, H, A on the tensor-core GEMM
    (6, 21, 80, 24, True, torch.float32),           # fp32 h: the generic fp32 path
]


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("T,B,H,A,ragged,dtype", OP_SHAPES)
def test_pool_op_against_fp64(mode, T, B, H, A, ragged, dtype):
    h, att, ds, lengths, got = _op_case(mode, T, B, H, A, ragged, dtype)
    keep = _keep_tb(lengths, T, B, DEV)
    arms = {}
    for arm, dt, r in (("fp64", torch.float64, None), ("emu", torch.float32, N.Bf16())):
        rr = r if dtype == torch.bfloat16 else None
        a = None if att is None else tuple(x.to(dt) for x in att)
        s, saved = pool_forward(h.to(dt), keep, mode, a, rr)
        dh, g = pool_backward(ds.to(dt), h.to(dt), keep, mode, a, saved, rr)
        arms[arm] = {"s": s, "dh": dh, **g}
    assert set(got) == set(arms["fp64"])
    floor = N.FLOOR if dtype == torch.bfloat16 else N.FLOOR_F32            # fp32 h: exact tanh, the fp32 floor
    for k, v in got.items():
        N.check_budget(f"{mode} T={T} B={B} H={H} A={A} {k}", v, arms["fp64"][k], arms["emu"][k], floor=floor)
    if lengths is not None:
        assert float(got["dh"].float().transpose(0, 1)[~keep.t()].abs().max()) == 0.0     # no gradient into uncounted steps
    if mode == "max" and dtype == torch.bfloat16:
        assert torch.equal(got["dh"].float(), arms["emu"]["dh"].float())       # the first t of a tie, exactly


@pytest.mark.parametrize("mode", MODES)
def test_pool_op_ignores_poisoned_padding(mode):
    """NaN (attention: 1e30) at every uncounted position changes neither s nor a gradient.  Attention's dW_a GEMM reads every
    row of h against a dU that is 0 at uncounted steps, so only finite values vanish there; an LSTM's padded outputs are its
    carried state, always finite."""
    clean = _op_case(mode, 9, 70, 128, 64, True, seed=4)[4]
    dirty = _op_case(mode, 9, 70, 128, 64, True, seed=4, poison=True)[4]
    for k in clean:
        assert torch.equal(clean[k], dirty[k]), k


@pytest.mark.parametrize("mode", MODES)
def test_pool_op_is_deterministic(mode):
    """The headline shape (T = 128, B = 256, H = 1024, A = 128): two calls, identical bits."""
    outs = [_op_case(mode, 128, 256, 1024, 128, True, seed=3)[4] for _ in range(2)]
    for k in outs[0]:
        assert torch.equal(outs[0][k], outs[1][k]), k


@pytest.mark.parametrize("mode", MODES)
def test_graph_replays_match_eager_calls(mode):
    """Forward and backward of the op captured once in a CUDA graph, replayed on batches whose lengths change in place: each
    replay gives the bits of an eager call with those lengths."""
    from lstm_tensorspark_b200.ops import functional as F
    T, B, H, A = 32, 160, 256, 128
    h, att, ds, lengths, _ = _op_case(mode, T, B, H, A, True, seed=5)
    hp = h.clone().requires_grad_(True)
    ap = None if att is None else tuple(a.clone().requires_grad_(True) for a in att)
    leaves = (hp,) + (ap or ())

    def run():
        for p in leaves:
            p.grad = None
        s = F.pool_sequence(hp, lengths, mode, ap)
        s.backward(ds)
        return [s.detach()] + [p.grad for p in leaves]

    def eager(ln):
        lengths.copy_(ln)
        return [t.clone() for t in run()]

    draws = [_lengths(T, B, 80 + k) for k in range(3)]
    want = [eager(ln) for ln in draws]
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        run()
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    for p in leaves:
        p.grad = None
    with torch.cuda.graph(g):
        s = F.pool_sequence(hp, lengths, mode, ap)
        grads = torch.autograd.grad(s, leaves, ds)
        outs = [s.detach()] + list(grads)
    for ln, w in zip(draws, want):
        lengths.copy_(ln)
        g.replay()
        torch.cuda.synchronize()
        for k, (a, b) in enumerate(zip(outs, w)):
            assert torch.equal(a, b), (k, ln[:4])
