"""Token embedding on the GPU (``--vocab_size``): the gather and the table gradient alone at awkward shapes, their bitwise
determinism, both gradient-sink modes, whole training steps of TrainEngine against an fp64 model reference within the budget of
its bf16 emulation (tests/lstm_numerics.py), graph replays against eager steps, a negative control and a CLI run.

Rounding points of the embedding (csrc/embedding.cu):
  forward   x[t,b] = the bf16 shadow's row tok[b,t], copied exactly; 0 at padded positions and for ids outside [0, V);
  backward  the first layer's dx = bf16(dG W_x) (its wgmma dX GEMM, fp32 accumulation, stored bf16; bidirectional: the two
            directions' bf16 dx added by autograd and rounded to bf16 once); dEmbedding[v] = the fp32 sum of the bf16 dx rows of the
            counted positions holding v, in increasing row order t·B + b, in pieces of 64 rows whose partials are summed in piece
            order; rows of absent ids are exactly 0.
The model reference composes the layer loops of lstm_numerics as ``lstm_numerics.model`` does, with the embedded tokens as the
first layer's input and the first layer's dx carried on into the table's gradient."""
import os
import subprocess
import sys

import pytest
import torch

import lstm_numerics as N
from test_gpu_model_numerics import _engine, _lengths, _names, _reference_params, _roundings, _segments, DEV

pytestmark = pytest.mark.gpu
C = 10
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(autouse=True)
def _fp32_matmuls(monkeypatch):
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)


def _stat(k):
    from lstm_tensorspark_b200.ops import cuda_lstm
    return cuda_lstm.STATS.get(k, 0)


def _keep_tb(lengths, T, B):
    k = N._keep(lengths, T, B, DEV)
    return torch.ones(T, B, dtype=torch.bool, device=DEV) if k is None else k.t()


def _tokens(kind, B, T, V, seed):
    g = torch.Generator().manual_seed(seed)
    if kind == "uniform":
        tok = torch.randint(0, V, (B, T), generator=g)
    elif kind == "zipf":
        import numpy as np
        tok = torch.as_tensor((np.random.default_rng(seed).zipf(1.2, size=(B, T)) - 1) % V)
    else:                                                               # one id at every position
        tok = torch.full((B, T), V // 2, dtype=torch.int64)
    return tok.to(DEV, torch.int32)


# ---- the gather --------------------------------------------------------------------------------------------------------------
GATHER = [  # (T, B, V, E)
    (4, 3, 5, 1), (6, 7, 11, 3), (5, 33, 40, 100), (8, 16, 64, 1024), (1, 9, 7, 100), (3, 5, 1, 8), (2, 3, 1000, 24),
]


@pytest.mark.parametrize("T,B,V,E", GATHER)
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
def test_gather_is_the_shadow_rows(T, B, V, E, dtype):
    from lstm_tensorspark_b200.ops import functional as F
    g = torch.Generator().manual_seed(T * 100 + E)
    table = torch.randn(V, E, generator=g).to(DEV)
    tok = torch.randint(-3, V + 3, (B, T), generator=g, dtype=torch.int32).to(DEV)  # ids outside [0, V) read zero rows
    lengths = torch.randint(1, T + 1, (B,), generator=g, dtype=torch.int32).to(DEV)
    for ln in (None, lengths):
        n = _stat("embed_fwd")
        x = F.embedding(tok, table, ln, dtype)
        assert _stat("embed_fwd") == n + 1
        keep = _keep_tb(ln, T, B) & (tok.t() >= 0) & (tok.t() < V)
        want = table.to(dtype)[tok.t().clamp(0, V - 1).long()] * keep.unsqueeze(2)
        assert x.shape == (T, B, E) and x.dtype == dtype and x.is_contiguous()
        assert torch.equal(x, want)
        assert (x[~keep] == 0).all() and not torch.signbit(x[~keep]).any()


def test_one_step_tokens():
    from lstm_tensorspark_b200.ops import functional as F
    table = torch.randn(9, 16, device=DEV)
    tok = torch.tensor([0, 8, 3, 12], device=DEV)                       # int64 is cast, 12 reads a zero row
    x = F.embedding(tok, table, None, torch.bfloat16)
    assert x.shape == (1, 4, 16) and torch.equal(x[0, :3], table.bfloat16()[[0, 8, 3]]) and float(x[0, 3].abs().sum()) == 0


# ---- the gradient --------------------------------------------------------------------------------------------------------------
def _grad(tok, V, E, dx, lengths, dtype=torch.bfloat16):
    from lstm_tensorspark_b200.ops import functional as F
    table = torch.zeros(V, E, device=DEV, requires_grad=True)
    x = F.embedding(tok, table, lengths, dtype)
    n = _stat("embed_bwd")
    x.backward(dx)
    assert _stat("embed_bwd") == n + 1
    return table.grad


def _fp64_grad(tok, V, E, dx, lengths):
    T, B = tok.shape[1], tok.shape[0]
    keep = _keep_tb(lengths, T, B) & (tok.t() >= 0) & (tok.t() < V)
    ids = tok.t()[keep].long()
    out = torch.zeros(V, E, dtype=torch.float64, device=DEV).index_add_(0, ids, dx[keep].double())
    cnt = torch.zeros(V, dtype=torch.float64, device=DEV).index_add_(0, ids, torch.ones_like(ids, dtype=torch.float64))
    mag = torch.zeros(V, E, dtype=torch.float64, device=DEV).index_add_(0, ids, dx[keep].double().abs())
    return out, cnt, mag


GRAD = [  # (T, B, V, E, kind)
    (7, 5, 3, 100, "uniform"), (16, 33, 1000, 3, "uniform"), (32, 64, 50, 256, "zipf"), (64, 128, 700, 64, "single"),
    (1, 9, 2, 40, "uniform"), (4, 3, 1, 8, "uniform"), (128, 256, 32768, 1024, "zipf"),
]


@pytest.mark.parametrize("T,B,V,E,kind", GRAD)
@pytest.mark.parametrize("ragged", [False, True])
def test_gradient_against_fp64(T, B, V, E, kind, ragged):
    """Within the fp32 bound of its order: |got - fp64| <= n u sum |dx| per element (n rows of the id, u = 2^-24), plus the
    pieces' partial sums (n / 64 + 1 more roundings).  Absent rows are exactly 0."""
    g = torch.Generator().manual_seed(T + B + V)
    tok = _tokens(kind, B, T, V, T + B)
    tok[0, 0] = -1                                                      # an id outside [0, V): no gradient
    lengths = _lengths(T, B, 7) if ragged and T > 1 else None
    dx = torch.randn(T, B, E, generator=g).to(DEV, torch.bfloat16)
    got = _grad(tok, V, E, dx, lengths)
    ref, cnt, mag = _fp64_grad(tok, V, E, dx, lengths)
    bound = (cnt.unsqueeze(1) + cnt.unsqueeze(1) / 64 + 2) * 2.0 ** -24 * mag
    assert ((got.double() - ref).abs() <= bound).all()
    assert (got[cnt == 0] == 0).all()


@pytest.mark.parametrize("kind", ["uniform", "zipf", "single"])
def test_gradient_is_bitwise_reproducible(kind):
    T, B, V, E = 64, 256, 4096, 512
    tok = _tokens(kind, B, T, V, 3)
    dx = torch.randn(T, B, E, generator=torch.Generator().manual_seed(1)).to(DEV, torch.bfloat16)
    a = _grad(tok, V, E, dx, None)
    b = _grad(tok, V, E, dx, None)
    assert torch.equal(a, b)


def test_overwrite_and_accumulate_sinks():
    from lstm_tensorspark_b200.ops.cuda_ext import ext
    T, B, V, E = 10, 24, 300, 72
    tok = _tokens("zipf", B, T, V, 5)
    lengths = _lengths(T, B, 9)
    dx = torch.randn(T, B, E, generator=torch.Generator().manual_seed(2)).to(DEV, torch.bfloat16)
    fresh = _grad(tok, V, E, dx, lengths)
    present = fresh.abs().sum(1) > 0
    junk = torch.full((V, E), 7.5, device=DEV)
    over = junk.clone()
    ext().embed_bwd(dx.view(T * B, E), tok, lengths, over, False)      # every row written, zeros included
    assert torch.equal(over, fresh)
    acc = junk.clone()
    ext().embed_bwd(dx.view(T * B, E), tok, lengths, acc, True)        # only the rows present move
    assert torch.equal(acc[~present], junk[~present]) and torch.equal(acc[present], junk[present] + fresh[present])


# ---- whole training steps ------------------------------------------------------------------------------------------------------
def model_embedded(tok, table, layers, head, labels, lengths=None, bidirectional=False, rounding=None):
    """``lstm_numerics.model`` behind the embedding: the loss and every gradient by name, ``Embedding/weights`` included."""
    dt = torch.float64 if rounding is None else torch.float32
    B, T = tok.shape
    V = table.shape[0]
    L = len(layers)
    dirs = (False, True) if bidirectional else (False,)
    keep = N._keep(lengths, T, B, DEV)
    keep_tb = _keep_tb(lengths, T, B) & (tok.t() >= 0) & (tok.t() < V)
    ids = tok.t().long().clamp(0, V - 1)

    def rnd(l, d):
        r = rounding[l] if isinstance(rounding, (list, tuple)) else rounding
        return r[d] if isinstance(r, tuple) else r

    def params(l, d):
        return layers[l][d] if bidirectional else layers[l]

    seq = table.to(dt)[ids] * keep_tb.unsqueeze(2).to(dt)
    saved = []
    for l in range(L):
        outs, sv = [], []
        for d, rev in enumerate(dirs):
            fw = N._forward(seq, *params(l, d), keep, rev, rnd(l, d), None)
            outs.append(N._state_out(fw, rev)[0])
            sv.append((fw, seq))
        saved.append(sv)
        seq = torch.cat(outs, 2) if bidirectional else outs[0]
    r_top = rnd(L - 1, 0)
    h_T = torch.cat([N._state_out(saved[L - 1][d][0], rev)[1] for d, rev in enumerate(dirs)], 1)
    W, b = head[0].to(dt), head[1].to(dt)
    logp = torch.log_softmax(h_T @ N._round(r_top, W) + b, 1)
    lab = labels.long().view(-1, 1)
    loss = -logp.gather(1, lab).mean()
    dlogits = (logp.exp() - torch.zeros_like(logp).scatter_(1, lab, 1.0)) / B
    dh_T = N._round(r_top, dlogits @ W.t())
    grads = {"Dense1/weights": h_T.t() @ dlogits, "Dense1/bias": dlogits.sum(0)}
    H_top = h_T.shape[1] // len(dirs)
    incoming = [None] * len(dirs)
    for l in range(L - 1, -1, -1):
        dxs = []
        for d, rev in enumerate(dirs):
            fw, x_in = saved[l][d]
            p, r = params(l, d), rnd(l, d)
            top = dh_T[:, d * H_top:(d + 1) * H_top] if l == L - 1 else None
            g = N._backward(fw, x_in, p[2], p[3], incoming[d], top, None, keep, rev, r, None)
            for k, v in zip(("h0", "c0", "w_x", "w_h", "bias"), g[1:]):
                grads[f"LSTMLayer{l}" + ("_reverse" if rev else "") + f"/{k}"] = v
            dxs.append(g[0])
        total = N._round(rnd(l, 0), dxs[0] + dxs[1]) if bidirectional else dxs[0]
        if l == 0:
            grads["Embedding/weights"] = torch.zeros(table.shape, dtype=dt, device=DEV).index_add_(
                0, ids[keep_tb], total[keep_tb])
            break
        H_low = total.shape[2] // len(dirs)
        incoming = [total[..., :H_low], total[..., H_low:]] if bidirectional else [total]
    return loss, grads


def _case(case, hidden, T, B, E, V, path, steps=2, ragged=False, bidirectional=False, negative=False):
    """Steps at learning rate 0, each checked (loss and every gradient of the flat buffer, the table's included) against the fp64
    reference.  ``negative``: the reference ignores the lengths (padded positions are embedded and reach the gradient)."""
    eng = _engine(hidden_units=hidden, in_features=E, seq_len=T, batch_size=B, num_classes=C, bidirectional=bidirectional,
                  variable_length=ragged, vocab_size=V)
    names = _names(eng)
    names[id(eng.model.embedding.weights)] = "Embedding/weights"
    seg = _segments(eng, names)
    rounding = _roundings([int(h) for h in hidden.split(",")], T, B, E, bidirectional)
    worst = {}
    for s in range(steps):
        tok = _tokens("zipf" if s % 2 else "uniform", B, T, V, 10 + s)
        y = torch.randint(0, C, (B,), generator=torch.Generator().manual_seed(s)).to(DEV)
        lengths = _lengths(T, B, 20 + s) if ragged else None
        before = eng.flat.data.clone()
        n_path = _stat(path)
        loss = eng.step(tok, y, lengths)
        torch.cuda.synchronize()
        assert _stat(path) > n_path, case
        got = {"loss": loss.float()}
        for k, (o, shape) in seg.items():
            got[k] = eng.flat.grad[o:o + shape.numel()].view(shape).clone()
        arms = {}
        with torch.no_grad():
            for arm, dt, r in (("fp64", torch.float64, None), ("emu", torch.float32, rounding)):
                layers, head = _reference_params(eng, seg, before, dt)
                o, shape = seg["Embedding/weights"]
                table = before[o:o + shape.numel()].view(shape).bfloat16().to(dt)
                l_, g_ = model_embedded(tok, table, layers, head, y, None if negative else lengths, bidirectional, r)
                arms[arm] = {"loss": l_, **g_}
        if negative:
            with pytest.raises(AssertionError):
                for k in ("loss", "Embedding/weights"):
                    N.check_budget(f"{case} {k}", got[k], arms["fp64"][k], arms["emu"][k])
            return
        assert set(got) <= set(arms["fp64"]), sorted(got)
        for k, gk in got.items():
            worst[k] = max(worst.get(k, 0.0), N.check_budget(f"{case} step {s} {k}", gk, arms["fp64"][k], arms["emu"][k]))
    top = sorted(worst.items(), key=lambda kv: -kv[1])[:3]
    print(f"\n{case}: worst budget ratio " + ", ".join(f"{k} {v:.3f}" for k, v in top))


def test_headline_pair_fixed():
    _case("fixed", "1024,1024", 128, 256, 1024, 32768, "pipelined_fwd")


def test_ragged():
    _case("ragged", "512,512", 64, 256, 512, 5000, "embed_bwd", ragged=True)


def test_bidirectional_ragged():
    _case("bidirectional ragged", "256,256", 32, 128, 256, 3000, "fast_bwd", ragged=True, bidirectional=True)


def test_negative_control_padding_reaches_the_gradient():
    _case("negative control", "256,256", 32, 128, 256, 3000, "embed_bwd", steps=1, ragged=True, negative=True)


@pytest.mark.parametrize("optimizer", ["adam", "sgd"])
def test_graph_replays_equal_eager_steps(optimizer):
    """A step captured on one token batch and replayed on others (lengths of their own) follows the eager steps: the same loss to
    fp32 rounding and the same weights to well within one update (the replay does not read the capture batch's tokens)."""
    kw = dict(hidden_units="512,512", in_features=512, seq_len=64, batch_size=256, num_classes=C, variable_length=True,
              vocab_size=4000, learning_rate=1e-3, optimizer=optimizer, deterministic=True)
    eager, graph = _engine(**kw), _engine(**kw)
    assert torch.equal(eager.flat.data, graph.flat.data)
    batches = [(_tokens("zipf", 256, 64, 4000, 40 + s), torch.randint(0, C, (256,)).to(DEV), _lengths(64, 256, 50 + s))
               for s in range(4)]
    graph.capture(*batches[0][:2], lengths=batches[0][2])
    for tok, y, ln in batches[1:]:
        le, lg = eager.step(tok, y, ln), graph.step(tok, y, ln)
        torch.cuda.synchronize()
        assert abs(float(le) - float(lg)) <= 1e-4 * abs(float(le))
        assert float((eager.flat.data - graph.flat.data).abs().max()) <= 1e-5
    o = next(o for p, o in zip(eager.flat.params, eager.flat.offsets) if p is eager.model.embedding.weights)
    assert not torch.equal(eager.flat.data[o:o + 4000 * 512], _engine(**kw).flat.data[o:o + 4000 * 512])   # the table trained


def test_cli_learns_resumes_and_evaluates(tmp_path):
    import json
    from lstm_tensorspark_b200.config import Config
    from lstm_tensorspark_b200.trainer import run_job
    base = dict(synthetic=2048, hidden_units="256,256", in_features=128, seq_len=32, num_classes=4, variable_length=True,
                batch_size=256, checkpoint_path=str(tmp_path / "ck"), output_path=str(tmp_path / "out"), quiet=True,
                learning_rate=3e-3, init="scaled", steps_mode="epochs", evaluate_every=8, vocab_size=1000, cuda_graph=True)
    flags = [f"--{k}={v}" for k, v in dict(base, epochs=6).items()]
    r = subprocess.run([sys.executable, os.path.join(ROOT, "lstm-no-spark.py")] + flags, capture_output=True, text=True,
                       timeout=900, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-3000:]
    runs = os.listdir(base["checkpoint_path"])
    scal = [json.loads(s) for s in open(os.path.join(base["checkpoint_path"], runs[0], "train", "scalars.jsonl"))]
    assert scal[-1]["cross_entropy"] < 0.7 * scal[0]["cross_entropy"], scal
    out2 = run_job(Config(epochs=8, use_pretrained_model=True, **base).validate(), standalone=True)
    assert out2["results"][0]["steps"] == 16
    ev = run_job(Config(mode="eval", **dict(base, batch_size=300)).validate(), standalone=True)
    assert ev["samples"] == 2048 and ev["accuracy"] > 0.5
