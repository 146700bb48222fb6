"""Every softmax head and the sampling kernels on the designed cases of tests/head_edges.py: exact logits with ties at each merge
level, near ties one ulp apart, all-negative rows beside padded classes, rows spread over +-2000, constant rows, labels at the
edges and uncounted rows.

Exact (bit for bit or integer-equal): the small heads' logits; ``correct`` and N; greedy tokens and tokens a gap of 21 t forces;
the two vocabulary-head layouts' loss, correct, N, dh and db; runs whose uncounted rows of h hold +-2^100 against runs with zeros
there (loss, correct, N, dW, db and dh at counted rows; dh at uncounted rows is 0); dloss = 0 gives zero gradients and -dloss
flips every gradient's sign.  Within the budget of tests/lstm_numerics.py against the fp64 arm (the exact logits) and the fp32
emulation at the kernels' rounding points: loss (and through it lse), dh, dW and db (and through them dlogits), and the sampled
log-probability.  Each case asserts the path it targets through STATS, and for the small heads the NP / CP instantiation the
shape selects (head_edges.small_head_path)."""
import pytest
import torch

import head_edges as E
import lstm_numerics as N

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
BF, F32 = torch.bfloat16, torch.float32
DLOSS = 0.37

SMALL = [(C, H, dt) for C in (2, 16, 17, 32, 33, 64, 65, 128, 129, 256, 257) for H in (64, 1024) for dt in (BF, F32)]
# (C, H, T, B, dtype): rows around the backward slabs step_bwd_rows<CP> (1024, 512, 192), and more row tiles than a persistent grid
STEP_ROWS = [(2, 64, 5, 205, BF), (8, 64, 1, 1023, F32), (16, 64, 1, 512, BF), (16, 1024, 1, 513, BF), (32, 64, 3, 64, BF),
             (32, 64, 1, 193, F32), (10, 64, 64, 2113, BF)]
# (C, H, T, B): R = T·B at CTA (128), cluster (256), band and ROW_CHUNK (4096) edges; R = 127 / 257: a cluster whose second CTA has
# no row.  C % 256 = 0, 8, 128; C = 8200: 33 class tiles, so one combine lane merges tiles 0 and 32.
VOCAB = [(512, 64, 1, 1), (520, 64, 1, 127), (520, 1024, 3, 43), (640, 64, 5, 51), (640, 4096, 1, 257), (4104, 1024, 63, 65),
         (4104, 64, 64, 64), (512, 4096, 17, 241), (8200, 1024, 3, 2731), (8200, 64, 5, 51)]
# (C, H, dtype, tied): the tensor-core kernel, and the fallbacks (fp32 h, C < 512, H % 64 != 0)
SAMPLE = [(512, 64, BF, False), (520, 1024, BF, True), (4104, 64, BF, False), (8200, 1024, BF, False), (8200, 64, BF, True),
          (520, 64, F32, False), (264, 64, BF, False), (520, 96, BF, False)]


@pytest.fixture(autouse=True)
def _fp32_matmuls(monkeypatch):
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)


def _stat(k):
    from lstm_tensorspark_b200.ops import cuda_lstm
    return cuda_lstm.STATS.get(k, 0)


def _regimes(C):
    return [r for r in E.REGIMES if r != "spread" or C >= 15]


def _poisoned(c, value):
    """h with every uncounted position set to +-value (0: zeros)."""
    off = ~c.keep
    g = torch.Generator().manual_seed(1)
    sign = (torch.randint(0, 2, c.h.shape, generator=g) * 2 - 1).to(c.h.device, c.h.dtype)
    return torch.where(off.unsqueeze(2), sign * value, c.h)


def _assert_sign_and_poison(name, c, run):
    """dloss = 0: zero gradients; -dloss: every gradient negated exactly; +-2^100 at uncounted rows of h: the same bits as zeros."""
    base = run(c.h, DLOSS)
    zero = run(c.h, 0.0)
    neg = run(c.h, -DLOSS)
    for k in ("dh", "dW", "db"):
        assert not bool(zero[k].float().ne(0).any()), (name, "dloss 0", k)
        assert torch.equal(neg[k], -base[k]), (name, "-dloss", k)
    if c.lengths is None:
        return base
    a, b = run(_poisoned(c, 2.0 ** 100), DLOSS), run(_poisoned(c, 0.0), DLOSS)
    keep = c.keep
    for k in ("loss", "correct", "n", "dW", "db"):
        assert torch.equal(a[k], b[k]), (name, "poisoned", k)
    dha, dhb = a["dh"].view(c.h.shape), b["dh"].view(c.h.shape)
    assert torch.equal(dha[keep], dhb[keep]), (name, "poisoned dh")
    assert not bool(dha[~keep].float().ne(0).any()), (name, "poisoned dh at uncounted rows")
    return base


# ---- the small heads -------------------------------------------------------------------------------------------------------------
def _per_step(c, dtype):
    from lstm_tensorspark_b200.ops import functional as F
    W, b = c.W.float(), c.bias.float()

    def run(h, dloss):
        hp = h.to(dtype).requires_grad_(True)
        Wp, bp = W.clone().requires_grad_(True), b.clone().requires_grad_(True)
        logits, loss, correct, n = F.head_xent_per_step(hp, Wp, bp, c.labels, c.lengths)
        (loss * dloss).backward()
        return {"logits": logits, "loss": loss.detach(), "correct": correct, "n": n, "dh": hp.grad, "dW": Wp.grad, "db": bp.grad}
    return run


def _last_state(c, dtype):
    from lstm_tensorspark_b200.ops import functional as F
    W, b, y = c.W.float(), c.bias.float(), c.labels[:, 0].contiguous()

    def run(h, dloss):
        hp = h[0].to(dtype).requires_grad_(True)
        Wp, bp = W.clone().requires_grad_(True), b.clone().requires_grad_(True)
        logits, loss, correct = F.head_xent(hp, Wp, bp, y)
        (loss * dloss).backward()
        return {"logits": logits.unsqueeze(1), "loss": loss.detach(), "correct": correct, "n": torch.tensor(y.numel()),
                "dh": hp.grad, "dW": Wp.grad, "db": bp.grad}
    return run


def _small(name, c, dtype, per_step):
    H, C = c.W.shape
    np_, cp = E.small_head_path(dtype, H, C, per_step)
    n_any, n_tc = _stat("head_per_step"), _stat("head_per_step_tc")
    run = (_per_step if per_step else _last_state)(c, dtype)
    got = _assert_sign_and_poison(name, c, run)
    if per_step:
        runs = 3 + 2 * (c.lengths is not None)
        assert (_stat("head_per_step") - n_any, _stat("head_per_step_tc") - n_tc) == (runs, runs * (np_ is not None)), name
    assert torch.equal(got["logits"].double(), c.logits.transpose(0, 1)), (name, "logits")
    E.assert_counts(c, got["correct"], got["n"])
    floor = N.FLOOR if dtype == BF else N.FLOOR_F32
    rd = (lambda x: x.bfloat16().float()) if dtype == BF else None
    worst = E.check_head(name, c, got, DLOSS, vocab=False, floor=floor, round_dh=rd)
    path = f"NP={np_}" if np_ else "generic"
    return f"{path} CP={cp or 'generic'} worst {worst:.3f}"


@pytest.mark.parametrize("C,H,dtype", SMALL)
def test_last_state_head(C, H, dtype):
    """The last-state head (B = 200: a padded batch tile) on every regime."""
    out = []
    for regime in _regimes(C):
        c = E.make_case(regime, 1, 200, H, C, lengths=False, seed=C, device=DEV)
        out.append(f"{regime}: " + _small(f"last-state {c.describe()}", c, dtype, False))
    print(f"\nlast-state head C={C} H={H} {str(dtype)[6:]}: " + "; ".join(out))


@pytest.mark.parametrize("C,H,dtype", SMALL)
def test_per_step_head(C, H, dtype):
    """The per-step head (T·B = 129 with lengths) on every regime."""
    out = []
    for regime in _regimes(C):
        c = E.make_case(regime, 3, 43, H, C, seed=C, device=DEV)
        out.append(f"{regime}: " + _small(f"per-step {c.describe()}", c, dtype, True))
    print(f"\nper-step head C={C} H={H} {str(dtype)[6:]}: " + "; ".join(out))


@pytest.mark.parametrize("C,H,T,B,dtype", STEP_ROWS)
def test_per_step_row_edges(C, H, T, B, dtype):
    R = T * B
    if R > 100000:
        sms = torch.cuda.get_device_properties(DEV).multi_processor_count
        assert R > sms * (2048 // 384) * 128                       # more row tiles than the persistent grid can hold
    out = []
    for regime in ("ties", "negative"):
        c = E.make_case(regime, T, B, H, C, seed=R, device=DEV)
        out.append(f"{regime}: " + _small(f"per-step {c.describe()}", c, dtype, True))
    print(f"\nper-step R={R} C={C} H={H} {str(dtype)[6:]}: " + "; ".join(out))


# ---- the large-vocabulary head ----------------------------------------------------------------------------------------------------
def _vocab(c, tied):
    from lstm_tensorspark_b200.ops import functional as F
    W = c.W.float()
    w = W.t().contiguous() if tied else W

    def run(h, dloss):
        hp = h.to(BF).requires_grad_(True)
        Wp, bp = w.clone().requires_grad_(True), c.bias.float().requires_grad_(True)
        loss, correct, n = F.vocab_xent_per_step(hp, Wp, bp, c.labels, c.lengths, class_major=tied)
        (loss * dloss).backward()
        return {"loss": loss.detach(), "correct": correct, "n": n, "dh": hp.grad, "dW": Wp.grad.t() if tied else Wp.grad,
                "db": bp.grad}
    return run


@pytest.mark.parametrize("C,H,T,B", VOCAB)
def test_vocab_head(C, H, T, B):
    out = []
    for regime in _regimes(C):
        c = E.make_case(regime, T, B, H, C, seed=T * B, device=DEV)
        got, worst = {}, 0.0
        for tied in (False, True):
            name = f"vocab {'tied ' if tied else ''}{c.describe()}"
            n = {k: _stat(k) for k in ("vocab_head_fwd", "vocab_head_fwd_tied", "head_per_step")}
            runs = 3 + 2 * (c.lengths is not None)
            got[tied] = _assert_sign_and_poison(name, c, _vocab(c, tied))
            assert {k: _stat(k) - v for k, v in n.items()} == {"vocab_head_fwd": runs, "vocab_head_fwd_tied": runs * tied,
                                                                "head_per_step": 0}, name
            E.assert_counts(c, got[tied]["correct"], got[tied]["n"])
            worst = max(worst, E.check_head(name, c, got[tied], DLOSS, vocab=True, floor=N.FLOOR))
        # dW is not compared bit for bit: the general GEMM computes dW = h^T dlogits as [H, C] in one layout and the table's
        # gradient dlogits^T h as [C, H] in the other, and it picks its kernel and tile width from the output shape, so the two
        # may add the rows in another order (they do at C = 4104, H = 64, R = 4096).  Both are held to the budget above.
        for k in ("loss", "correct", "n", "dh", "db"):
            assert torch.equal(got[False][k], got[True][k]), (c.describe(), "layouts", k)
        out.append(f"{regime} worst {worst:.3f}")
    print(f"\nvocab head C={C} H={H} R={T * B}: " + "; ".join(out))


# ---- sampling ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("C,H,dtype,tied", SAMPLE)
def test_sample(C, H, dtype, tied):
    """Greedy tokens are the first arg-max (ties, near ties, padded classes); at t = 0.5 rows whose max leads by 14 > 21 t give
    the arg-max or one of the two tied classes, and the tied rows take both classes; top_k = 1 keeps both tied classes and a
    tiny top_p keeps the classes at the max."""
    from lstm_tensorspark_b200.ops import cuda_vocab_head
    from lstm_tensorspark_b200.ops import functional as F
    B = 300
    tc = dtype == BF and H % 64 == 0 and C % 8 == 0 and C >= 512
    out = []
    for regime in _regimes(C):
        c = E.make_case(regime, 1, B, H, C, lengths=False, seed=C + H, device=DEV)
        assert cuda_vocab_head.supported(c.h.to(dtype), C) == tc
        h = c.h[0].to(dtype)
        w = c.W.float().t().contiguous().bfloat16() if tied else c.W.float()
        b = c.bias.float()
        worst = 0.0
        filters = [(0, 1.0)] + ([(1, 1.0), (0, 1e-6)] if regime == "ties" else [])
        for temperature in (0.0, 0.5):
            for top_k, top_p in filters:
                if temperature == 0 and (top_k, top_p) != (0, 1.0):
                    continue
                n = {k: _stat(k) for k in ("vocab_sample", "vocab_sample_tied", "vocab_sample_filtered")}
                tok, lp = F.vocab_sample(h, w, b, temperature, 17, 3, class_major=tied, top_k=top_k, top_p=top_p)
                filt = (top_k, top_p) != (0, 1.0)
                assert {k: _stat(k) - v for k, v in n.items()} == {"vocab_sample": 1, "vocab_sample_tied": int(tied),
                                                                    "vocab_sample_filtered": int(filt)}
                what = f"sample {c.describe()} t={temperature} k={top_k} p={top_p}"
                checked = E.assert_tokens(c, tok, temperature)
                if temperature > 0 and regime != "negative":
                    assert checked >= B // 2, (what, checked)
                if temperature > 0 and regime == "ties":
                    pairs = [(p, k.pair) for p, k in enumerate(c.kinds) if k.name.startswith("tie")]
                    t = tok.long().to(DEV)
                    second = sum(int((t[c.kind_of[0] == p] == bb).sum()) for p, (_, bb) in pairs)
                    first = sum(int((t[c.kind_of[0] == p] == a).sum()) for p, (a, _) in pairs)
                    assert first > 0 and second > 0, (what, first, second)
                worst = max(worst, E.check_logprob(what, c, tok, lp))
        out.append(f"{regime} worst {worst:.3f}")
    print(f"\nsample C={C} H={H} {str(dtype)[6:]}{' tied' if tied else ''} {'kSample' if tc else 'fallback'}: " + "; ".join(out))
