"""Per-step labels on the GPU: whole training steps of TrainEngine with ``per_step_labels`` against an fp64 reference of the
sequence-labelling model, within the budget of its bf16 emulation (tests/lstm_numerics.py), and the per-step head op alone at
awkward shapes, its bitwise determinism and a negative control.

The model reference composes the layer loops of lstm_numerics as ``lstm_numerics.model`` does, with the head at every time step
instead of on h_T.  Rounding points of the per-step head (csrc/head_wgmma.cu):
  logits   bf16 h_top(t) x bf16(W) accumulated in fp32, + fp32 bias (generic path, fp32 h or C > 256: fp32 W);
  dlogits  (softmax - onehot) / N in fp32 at counted positions, 0 elsewhere;
  dh       dlogits W^T with the fp32 W, stored bf16 - the top layer's dh_seq (no dh_T);
  dW, db   fp32 sums of h x dlogits and of dlogits."""
import pytest
import torch

import lstm_numerics as N
from test_gpu_model_numerics import (_engine, _is_h100, _lengths, _names, _reference_params, _roundings, _sched, _segments,
                                     DEV)

pytestmark = pytest.mark.gpu
C = 10


@pytest.fixture(autouse=True)
def _fp32_matmuls(monkeypatch):
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)


def _stat(k):
    from lstm_tensorspark_b200.ops import cuda_lstm
    return cuda_lstm.STATS.get(k, 0)


def _head(h_seq, W, b, labels, lengths, rounding, tc=True, norm_all=False):
    """The per-step head forward and backward in the reference's precision.  ``h_seq [T,B,H]``, ``labels [B,T]`` -> (loss,
    dh_seq [T,B,H], dW, db).  ``norm_all``: divide by T·B instead of N (the negative control's wrong reference)."""
    T, B, _ = h_seq.shape
    dt = h_seq.dtype
    keep = N._keep(lengths, T, B, h_seq.device)
    keep = torch.ones(B, T, dtype=torch.bool, device=h_seq.device) if keep is None else keep
    keep = keep.t().to(dt)                                                   # [T,B]
    Wr = W.to(dt)
    logits = h_seq @ (N._round(rounding, Wr) if tc else Wr) + b.to(dt)
    logp = torch.log_softmax(logits, 2)
    lab = (labels.to(h_seq.device).long().t() * keep.long()).unsqueeze(2)    # uncounted positions: any class, masked below
    n = float(T * B) if norm_all else keep.sum()
    loss = -(logp.gather(2, lab).squeeze(2) * keep).sum() / n
    dlogits = (logp.exp() - torch.zeros_like(logp).scatter_(2, lab, 1.0)) * keep.unsqueeze(2) / n
    dh = dlogits @ Wr.t()
    dW = h_seq.reshape(T * B, -1).t() @ dlogits.reshape(T * B, -1)
    return loss, dh, dW, dlogits.sum((0, 1))


def model_per_step(x, layers, head, labels, lengths=None, bidirectional=False, dropout=None, rounding=None, norm_all=False):
    """``lstm_numerics.model`` with the head at every step of the top layer's output (``[h_fwd(t) | h_rev(t)]`` when
    bidirectional) -> (loss, grads by name).  The top layer receives dh as its dh_seq."""
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
    loss, dh_top, dW, db = _head(seq, head[0], head[1], labels, lengths, rnd(L - 1, 0), norm_all=norm_all)
    grads = {"Dense1/weights": dW, "Dense1/bias": db}
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


def _per_step_labels(n, T, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, C, (n, T), generator=g).to(DEV)


def _case(case, hidden, T, B, D, path, steps=2, lengths_seed=None, bidirectional=False, dropout=0.0, learning_rate=0.0,
          graph=False, negative=False, dtype=torch.bfloat16):
    """Training steps, each checked (loss and every gradient of the flat buffer) against the fp64 reference at the weights it
    read.  ``path``: a STATS key one step must bump (besides the per-step head: on the tensor cores in bf16, on the generic
    kernels in fp32).  ``graph``: captured on the first batch and replayed on every batch, each with lengths of its own.
    ``negative``: the reference (both arms) normalises by T·B - the loss check must fail.  ``dtype``: the engine's compute
    dtype (fp32: the lstm_numerics.Fp32 arm and floor, and the reference reads the fp32 master)."""
    from lstm_tensorspark_b200 import data as Dm
    bf16 = dtype == torch.bfloat16
    head_key = "head_per_step_tc" if bf16 else "head_per_step"
    eng = _engine(dtype, hidden_units=hidden, in_features=D, seq_len=T, batch_size=B, num_classes=C, bidirectional=bidirectional,
                  dropout=dropout, variable_length=lengths_seed is not None, learning_rate=learning_rate, per_step_labels=True)
    flat = eng.flat
    xs, _ = Dm.synthetic_sequences(steps * B, T, D, C, seed=5)
    xs, ys = torch.as_tensor(xs).to(DEV).to(dtype), _per_step_labels(steps * B, T, 7)
    seg = _segments(eng, _names(eng))
    rounding = _roundings([int(h) for h in hidden.split(",")], T, B, D, bidirectional) if bf16 else N.Fp32()
    floor = N.FLOOR if bf16 else N.FLOOR_F32
    worst = {}
    for s in range(steps):
        x, y = xs[s * B:(s + 1) * B], ys[s * B:(s + 1) * B]
        lengths = None if lengths_seed is None else _lengths(T, B, lengths_seed + s)
        before = {"p": flat.data.clone(), "drop": int(eng.model.rnn.dropout_step)}
        n_tc, n_path, n_tc_any = _stat(head_key), _stat(path), _stat("head_per_step_tc")
        if graph and s == 0:
            eng.capture(x, y, lengths=lengths)
            assert _stat(head_key) > n_tc and _stat(path) > n_path, case
            n_tc, n_path = _stat(head_key), _stat(path)
        loss = eng.step(x, y, lengths)
        torch.cuda.synchronize()
        if not graph:
            assert _stat(head_key) == n_tc + 1 and _stat(path) > n_path, (case, s)
            assert bf16 or _stat("head_per_step_tc") == n_tc_any, (case, s)           # fp32: the generic kernels
        got = {"loss": loss.float()}
        for k, (o, shape) in seg.items():
            got[k] = flat.grad[o:o + shape.numel()].view(shape).clone()
        drop = N.Dropout(dropout, eng.model.rnn.dropout_key, before["drop"]) if dropout > 0 else None
        with torch.no_grad():
            arms = {}
            for arm, dt, r in (("fp64", torch.float64, None), ("emu", torch.float32, rounding)):
                layers, head = _reference_params(eng, seg, before["p"], dt, bf16_weights=bf16)
                l_, g_ = model_per_step(x.to(dt), layers, head, y, lengths, bidirectional, drop, r,
                                        norm_all=negative)
                arms[arm] = {"loss": l_, **g_}
            if negative:
                with pytest.raises(AssertionError):
                    N.check_budget(f"{case} loss", got["loss"], arms["fp64"]["loss"], arms["emu"]["loss"])
                return
            for k, g in got.items():
                worst[k] = max(worst.get(k, 0.0), N.check_budget(f"{case} step {s} {k}", g, arms["fp64"][k], arms["emu"][k],
                                                                 floor=floor))
            del arms
    top = sorted(worst.items(), key=lambda kv: -kv[1])[:3]
    print(f"\n{case}: worst budget ratio " + ", ".join(f"{k} {v:.3f}" for k, v in top))


def test_headline_pipelined_pair():
    if _is_h100():
        assert _sched(128, 256, 1024, 1024, 1024) == "pipelined"
    _case("per-step headline", "1024,1024", 128, 256, 1024, "pipelined_fwd")


def test_wavefront_pair():
    if _is_h100():
        assert _sched(128, 256, 512, 512, 512) == "wavefront"
    _case("per-step wavefront", "512,512", 128, 256, 512, "wavefront_fwd")


def test_ragged():
    """Lengths 1 and T included: padded positions are not counted and get no gradient."""
    _case("per-step ragged", "1024,1024", 128, 256, 1024, "pipelined_fwd", lengths_seed=31)


def test_bidirectional_ragged():
    """[h_fwd(t) | h_rev(t)] at every step into a [2H, C] head; each direction receives its half of dh as dh_seq."""
    _case("per-step bidirectional ragged", "512,512", 64, 256, 256, "fast_bwd", lengths_seed=41, bidirectional=True)


def test_dropout():
    _case("per-step dropout", "1024,1024", 128, 256, 1024, "pipelined_fwd", dropout=0.2)


def test_batch_chunks():
    """B = 400 at H = 1024: every layer runs as two persistent chunks; the top chunks' dh_seq slices come from one head."""
    _case("per-step batch chunks", "1024,1024", 32, 400, 256, "batch_chunks")


def test_adam_graph_replays_with_changing_lengths():
    """Captured once, replayed on 3 batches with lengths of their own: N is computed on the device at every replay."""
    _case("per-step adam graph", "1024,1024", 128, 256, 1024, "pipelined_fwd", steps=3, lengths_seed=51, learning_rate=1e-3,
          graph=True)


def test_fp32_ragged_adam():
    """``--dtype fp32`` with lengths, two Adam steps: the layers and the per-step head on the generic kernels (the head's
    softmax in xent_steps_kernel, its backward on the CUDA cores), against the Fp32 arm with the fp32 floor."""
    _case("per-step fp32 ragged adam", "48,48", 32, 20, 12, "generic_fwd", lengths_seed=71, learning_rate=1e-3,
          dtype=torch.float32)


def test_negative_control_normalised_by_all_positions():
    """A reference that divides by T·B instead of the number of counted positions must fail the budget."""
    _case("per-step negative control", "512,512", 64, 128, 256, "fast_fwd", steps=1, lengths_seed=61, negative=True)


# ---- the op alone ------------------------------------------------------------------------------------------------------------
def _op_case(T, B, H, Cn, ragged, dtype=torch.bfloat16, seed=0):
    from lstm_tensorspark_b200.ops import functional as F
    g = torch.Generator().manual_seed(seed)
    h = torch.randn(T, B, H, generator=g).to(DEV, dtype)
    W = (torch.randn(H, Cn, generator=g) / H ** 0.5).to(DEV)
    b = torch.randn(Cn, generator=g).to(DEV)
    labels = torch.randint(0, Cn, (B, T), generator=g).to(DEV)
    lengths = None
    if ragged:
        lengths = torch.randint(1, T + 1, (B,), generator=g, dtype=torch.int32)
        lengths[0], lengths[-1] = 1, T
        lengths = lengths.to(DEV)
        labels = torch.where(torch.arange(T, device=DEV).view(1, T) < lengths.view(B, 1).long(), labels, 10 ** 6)  # never read
    hp = h.clone().requires_grad_(True)
    Wp, bp = W.clone().requires_grad_(True), b.clone().requires_grad_(True)
    logits, loss, correct, n = F.head_xent_per_step(hp, Wp, bp, labels, lengths)
    (loss * 0.37).backward()
    return h, W, b, labels, lengths, logits, loss, correct, n, hp.grad, Wp.grad, bp.grad


@pytest.mark.parametrize("T,B,H,Cn,ragged,dtype", [
    (7, 19, 256, 2, True, torch.bfloat16),          # T·B = 133: one full row tile and a ragged one
    (5, 37, 512, 10, False, torch.bfloat16),
    (9, 33, 128, 17, True, torch.bfloat16),
    (3, 50, 192, 33, True, torch.bfloat16),         # C > 32: the per-output backward
    (4, 45, 128, 200, False, torch.bfloat16),
    (6, 21, 128, 300, True, torch.bfloat16),        # C > 256: the generic forward
    (5, 30, 96, 10, True, torch.float32),           # fp32 activations: the generic forward
])
def test_head_op_against_fp64(T, B, H, Cn, ragged, dtype):
    h, W, b, labels, lengths, logits, loss, correct, n, dh, dW, db = _op_case(T, B, H, Cn, ragged, dtype)
    tc = dtype == torch.bfloat16 and Cn <= 256
    assert (_stat("head_per_step_tc") > 0) or not tc
    keep = N._keep(lengths, T, B, DEV)
    keep = torch.ones(B, T, dtype=torch.bool, device=DEV) if keep is None else keep
    assert int(n) == int(keep.sum())
    lab = torch.where(keep, labels, 0)
    arms = {}
    for arm, dt, r in (("fp64", torch.float64, None), ("emu", torch.float32, N.Bf16())):
        hd = h.to(dt)
        rr = r if dtype == torch.bfloat16 else None
        l_, dh_, dW_, db_ = _head(hd, W.to(dt), b.to(dt), lab, lengths, rr, tc=tc)
        lg = (hd @ (N._round(rr, W.to(dt)) if tc else W.to(dt)) + b.to(dt)).transpose(0, 1)
        arms[arm] = {"logits": lg, "loss": l_, "dh": N._round(rr, dh_ * 0.37) if rr is not None else dh_ * 0.37,
                     "dW": dW_ * 0.37, "db": db_ * 0.37}
    got = {"logits": logits, "loss": loss, "dh": dh, "dW": dW, "db": db}
    floor = N.FLOOR if dtype == torch.bfloat16 else N.FLOOR_F32
    for k, v in got.items():
        N.check_budget(f"head T={T} B={B} C={Cn} {k}", v, arms["fp64"][k], arms["emu"][k], per_step=k == "logits", floor=floor)
    pred = logits.argmax(2)
    assert int(correct) == int(((pred == labels) & keep).sum())
    if lengths is not None:
        assert float(dh.float().transpose(0, 1)[~keep].abs().max()) == 0.0     # no gradient into uncounted positions


def test_head_op_is_deterministic():
    """The headline shape (T·B = 32768 rows, beyond one backward slab): two calls, identical bits."""
    outs = [_op_case(128, 256, 1024, 10, True, seed=3) for _ in range(2)]
    for k, (a, b) in enumerate(zip(outs[0][5:], outs[1][5:])):
        assert torch.equal(a, b), k
