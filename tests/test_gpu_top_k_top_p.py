"""Top-k and nucleus (top-p) sampling on the GPU: the filtered op (the head's ``kLogits`` main loop, the threshold kernel and the
filtered sampling kernel; the fallback's GEMM logits for the inputs the tensor-core kernel does not take) against the fp64
reference, the threshold kernel exactly on designed logits, the coupling with the unfiltered op bit for bit, the off values, the
determinism and graph replay, the distribution of the draws, the decode loop without a host sync and a tiny trained model.

Budgets.  Logits: ALPHA x the largest error of an fp32 evaluation of the same products, plus 2^-20 x the largest logit.  A class
is surely kept (surely dropped) when it stays above (below) the top-k threshold by twice that, and when the tempered mass of the
classes that may rank above it stays below p (above p) after scaling every mass by exp(+-4 err / t) and adding MASS_BUDGET, the
threshold kernel's own rounding (fixed point at 2^-32 of the max's mass, C x 2^-33 <= 4e-6 of the total at C = 32768, and fp32
exp); the rest are boundary classes, which may go either way.  Scores: the budget of tests/test_gpu_generate.py."""
import math

import numpy as np
import pytest
import torch

import lstm_numerics as N

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
MASS_BUDGET = 1e-5
FILTERS = [(50, 1.0), (0, 0.9), (50, 0.9), (1, 1.0), (0, 0.3)]


@pytest.fixture(autouse=True)
def _fp32_matmuls(monkeypatch):
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)


def _stat(k):
    from lstm_tensorspark_b200.ops import cuda_lstm
    return cuda_lstm.STATS.get(k, 0)


def _inputs(B, H, V, seed, dtype=torch.bfloat16):
    g = torch.Generator().manual_seed(seed)
    h = torch.randn(B, H, generator=g).to(DEV, dtype)
    W = (torch.randn(H, V, generator=g) * (2.0 / H ** 0.5)).bfloat16().float().to(DEV)
    b = torch.randn(V, generator=g).to(DEV)
    return h, W, b


def _above(l, e, x):
    """Per row: the sum of e over the classes with l > x (x [B, C]) -> [B, C]."""
    v, order = l.sort(1)
    suffix = e.gather(1, order).flip(1).cumsum(1).flip(1)
    suffix = torch.cat([suffix, torch.zeros_like(suffix[:, :1])], 1)
    idx = torch.searchsorted(v.contiguous(), x.contiguous(), right=True)
    return suffix.gather(1, idx)


def _kept_bounds(l64, err, temperature, top_k, top_p):
    """(surely kept, possibly kept) [B, C] under a logit error of at most ``err`` [B] (module docstring)."""
    from lstm_tensorspark_b200.ops import reference as ref
    B, C = l64.shape
    e2 = 2 * err.view(-1, 1)
    sure = torch.ones_like(l64, dtype=torch.bool)
    maybe = sure.clone()
    if 0 < top_k < C:
        tk = l64.topk(top_k, 1).values[:, -1:]
        sure, maybe = l64 > tk + e2, l64 >= tk - e2
    if top_p < 1:
        f = torch.exp(4 * err / temperature).view(-1, 1)
        w = torch.exp((l64 - l64.amax(1, keepdim=True)) / temperature)
        w_sure, w_maybe = w * sure, w * maybe
        z_lo, z_hi = w_sure.sum(1, keepdim=True), w_maybe.sum(1, keepdim=True)
        m_lo = _above(l64, w_sure, l64 + e2)                                  # surely ranked above c
        m_hi = _above(l64, w_maybe, l64 - e2) - w_maybe                       # possibly ranked above c (c itself excluded)
        sure = sure & (m_hi / z_lo * f + MASS_BUDGET < top_p)
        maybe = maybe & ~(m_lo / z_hi / f - MASS_BUDGET >= top_p)
    assert not bool((sure & (l64 < ref.sample_threshold(l64, temperature, top_k, top_p).unsqueeze(1))).any())
    return sure, maybe


def _check(h, W, b, temperature, seed, step, top_k, top_p, tok, lp, row0=0):
    """The GPU's filtered tokens and log-probabilities against the fp64 reference -> the number of rows with a clear decision."""
    from lstm_tensorspark_b200.ops import reference as ref
    l64 = h.double() @ W.double() + b.double()
    l32 = h.float() @ W.float() + b.float()
    err = N.ALPHA * (l32.double() - l64).abs().amax(1) + 2.0 ** -20 * l64.abs().amax(1)
    sure, maybe = _kept_bounds(l64, err, temperature, top_k, top_p)
    s64 = ref.sample_scores(l64, temperature, seed, step, row0)
    g = -torch.log(-torch.log(ref.sample_uniform(ref.sample_noise_words(h.shape[0], W.shape[1], seed, step, device=DEV, row0=row0))))
    s32 = (l32 * torch.tensor(1.0 / temperature, dtype=torch.float32) + g.float()).double()
    tol = N.ALPHA * (s32 - s64).abs().amax(1) + N.FLOOR * s64.abs().amax(1)
    t = tok.long().view(-1, 1)
    assert bool(((t >= 0) & (t < W.shape[1])).all())
    assert bool(maybe.gather(1, t).all()), "a token outside every possible kept set"
    ninf = torch.tensor(float("-inf"), dtype=torch.float64, device=DEV)
    best_sure = torch.where(sure, s64, ninf).amax(1)
    got = s64.gather(1, t).squeeze(1)
    assert bool((got >= best_sure - tol).all()), float((best_sure - got - tol).max())
    cand = torch.where(maybe, s64, ninf)
    top2 = cand.topk(2, dim=1)
    lead = top2.indices[:, :1]
    clear = sure.gather(1, lead).squeeze(1) & ((top2.values[:, 0] - top2.values[:, 1]) > tol)
    want = ref.sample_logits(l64, temperature, seed, step, row0, top_k, top_p)[0].long()
    assert torch.equal(want[clear], lead.squeeze(1)[clear])
    assert bool((t.squeeze(1)[clear] == want[clear]).all())
    lp64 = torch.log_softmax(l64, 1).gather(1, t).squeeze(1)
    lp32 = torch.log_softmax(l32.double(), 1).gather(1, t).squeeze(1)
    N.check_budget("logprob", lp, lp64, lp32)
    return int(clear.sum())


# ---- the op against fp64 --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("tied", [False, True])
@pytest.mark.parametrize("B", [1, 3, 130, 256])
@pytest.mark.parametrize("H", [64, 1024])
@pytest.mark.parametrize("V", [512, 4104, 32768])
def test_op_against_fp64(B, H, V, tied):
    from lstm_tensorspark_b200.ops import functional as F
    h, W, b = _inputs(B, H, V, seed=B + H + V + tied)
    w = W.t().contiguous().bfloat16() if tied else W
    clear = total = 0
    for temperature in (0.7, 1.0):
        for top_k, top_p in FILTERS:
            n0, nt = _stat("vocab_sample_filtered"), _stat("vocab_sample_tied")
            step = torch.full((1,), 5, dtype=torch.int32, device=DEV)
            tok, lp = F.vocab_sample(h, w, b, temperature, 11, step, class_major=tied, top_k=top_k, top_p=top_p)
            assert _stat("vocab_sample_filtered") == n0 + 1 and _stat("vocab_sample_tied") == nt + int(tied)
            assert int(step) == 6 and tok.dtype == torch.int32 and lp.dtype == torch.float32
            clear += _check(h, W, b, temperature, 11, 5, top_k, top_p, tok, lp)
            total += B
    assert clear >= total // 2, (clear, total)


@pytest.mark.parametrize("B,H,V,dtype", [(5, 64, 512, torch.float32), (130, 128, 300, torch.bfloat16), (7, 96, 1000, torch.bfloat16),
                                         (3, 64, 4100, torch.bfloat16)])
def test_fallback_against_fp64(B, H, V, dtype):
    """fp32 activations, C < 512, H % 64 != 0, C % 8 != 0: the head GEMM's fp32 logits, then the same threshold and sampling."""
    from lstm_tensorspark_b200.ops import cuda_vocab_head
    from lstm_tensorspark_b200.ops import functional as F
    h, W, b = _inputs(B, H, V, seed=V, dtype=dtype)
    assert not cuda_vocab_head.supported(h.unsqueeze(0), V)
    for top_k, top_p in FILTERS:
        n0 = _stat("vocab_sample_filtered")
        tok, lp = F.vocab_sample(h, W, b, 1.0, 3, 2, top_k=top_k, top_p=top_p)
        assert _stat("vocab_sample_filtered") == n0 + 1
        _check(h, W, b, 1.0, 3, 2, top_k, top_p, tok, lp)


# ---- the threshold kernel exactly -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("V", [512, 4104, 32768])
def test_threshold_is_exact_on_designed_logits(V):
    """h = 0: the kLogits kernel's logits are the bias itself.  Rows of values on a grid of 1/8 (gaps far above any rounding)
    with many ties, some rows all tied; every (k, p, t) whose nucleus cut keeps a margin of 1e-3 from every class's cumulative
    mass must give the reference's threshold bit for bit."""
    from lstm_tensorspark_b200.ops import reference as ref
    from lstm_tensorspark_b200.ops.cuda_ext import ext
    B = 6
    g = torch.Generator().manual_seed(V)
    bias = (torch.randint(-40, 24, (V,), generator=g).float() / 8).to(DEV)
    h = torch.zeros(B, 64, dtype=torch.bfloat16, device=DEV)
    W = torch.randn(64, V, device=DEV).bfloat16()
    logits = ext().vocab_head_logits(h, W, False, bias)
    assert torch.equal(logits, bias.expand(B, V))
    rows = logits.clone()
    rows[1] = rows[1][torch.randperm(V, generator=g).to(DEV)]
    rows[2] = 0.25                                                           # all tied
    rows[3, : V // 2] = -1e30                                                # half the classes far out of reach
    rows[4] = (torch.randn(V, generator=g) * 3).round().to(DEV)              # integers: large tie groups
    rows[5, 7] = 40.0                                                        # one dominant class
    checked = 0
    for temperature in (0.5, 1.0, 2.0):
        for top_k in (0, 1, 3, 50, V // 3, V - 1, V, V + 5):
            for top_p in (1.0, 0.97, 0.9, 0.5, 0.1, 1e-6):
                want = ref.sample_threshold(rows.double(), temperature, top_k, top_p)
                if top_p < 1:
                    keep_k = rows.double() >= ref.sample_threshold(rows.double(), temperature, top_k, 1.0).unsqueeze(1)
                    w = torch.exp((rows.double() - rows.double().amax(1, keepdim=True)) / temperature) * keep_k
                    frac = _above(rows.double(), w, rows.double()) / w.sum(1, keepdim=True)
                    if bool((((frac - top_p).abs() < 1e-3) & (frac > 0)).any()):
                        continue                                             # a cut too close to call: not a designed case
                got = ext().vocab_threshold(rows, top_k, top_p, temperature)
                assert torch.equal(got.double(), want), (temperature, top_k, top_p, got, want)
                checked += 1
    assert checked >= 100, checked


def test_threshold_binding_refuses_bad_arguments():
    from lstm_tensorspark_b200.ops.cuda_ext import ext
    l = torch.zeros(2, 16, device=DEV)
    for args, msg in (((-1, 1.0, 1.0), "top_k"), ((0, 0.0, 1.0), "top_p"), ((0, 1.5, 1.0), "top_p"), ((0, float("nan"), 1.0), "top_p"),
                      ((0, 0.5, 0.0), "temperature"), ((0, 0.5, float("inf")), "temperature")):
        with pytest.raises(RuntimeError, match=msg):
            ext().vocab_threshold(l, *args)
    with pytest.raises(RuntimeError, match="contiguous"):
        ext().vocab_threshold(torch.zeros(16, 2, device=DEV).t(), 1, 1.0, 1.0)


# ---- the coupling, the off values, determinism ----------------------------------------------------------------------------------
@pytest.mark.parametrize("tied,H,V,dtype", [(False, 1024, 32768, torch.bfloat16), (True, 1024, 32768, torch.bfloat16),
                                            (False, 256, 4104, torch.bfloat16), (False, 96, 1000, torch.bfloat16),
                                            (False, 64, 512, torch.float32)])
def test_filtered_token_is_the_unfiltered_one_whenever_it_is_kept(tied, H, V, dtype):
    from lstm_tensorspark_b200.ops import functional as F
    from lstm_tensorspark_b200.ops.cuda_ext import ext
    B = 256
    h, W, b = _inputs(B, H, V, seed=H + V, dtype=dtype)
    w = W.t().contiguous().bfloat16() if tied else W
    inside = 0
    for step in range(4):
        free, flp = F.vocab_sample(h, w, b, 1.0, 21, step, class_major=tied)
        for top_k, top_p in FILTERS + [(V - 1, 1.0), (0, 0.999)]:
            tok, lp = F.vocab_sample(h, w, b, 1.0, 21, step, class_major=tied, top_k=top_k, top_p=top_p)
            if dtype == torch.bfloat16 and H % 64 == 0 and V % 8 == 0:
                logits = ext().vocab_head_logits(h, w if tied else W.bfloat16(), tied, b)
            else:
                from lstm_tensorspark_b200.ops import cuda_gemm
                logits = cuda_gemm.matmul(h, W.t(), bias=b, out_dtype=torch.float32)
            tau = ext().vocab_threshold(logits, top_k, top_p, 1.0)
            keep = logits >= tau.unsqueeze(1)
            assert bool(keep.gather(1, tok.long().view(-1, 1)).all())
            kept = keep.gather(1, free.long().view(-1, 1)).squeeze(1)
            assert torch.equal(tok[kept], free[kept]), (top_k, top_p)
            assert torch.equal(lp[kept], flp[kept]) or bool(((lp[kept] - flp[kept]).abs() <= 1e-5 * (1 + flp[kept].abs())).all())
            inside += int(kept.sum())
    assert inside >= B


@pytest.mark.parametrize("V,dtype", [(32768, torch.bfloat16), (1004, torch.bfloat16)])
def test_filters_off_or_greedy_run_the_unfiltered_kernels(V, dtype):
    from lstm_tensorspark_b200.ops import functional as F
    h, W, b = _inputs(64, 128, V, seed=3, dtype=dtype)
    for temperature, top_k, top_p in ((1.0, 0, 1.0), (1.0, V, 1.0), (1.0, V + 7, 1.0), (0.0, 5, 0.5), (0.0, 1, 1.0), (0.0, 0, 1e-3)):
        want = F.vocab_sample(h, W, b, temperature, 4, 2)
        n0 = _stat("vocab_sample_filtered")
        got = F.vocab_sample(h, W, b, temperature, 4, 2, top_k=top_k, top_p=top_p)
        assert _stat("vocab_sample_filtered") == n0
        assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1])


def test_filtered_op_is_deterministic_and_a_graph_replays_it():
    from lstm_tensorspark_b200.ops import functional as F
    h, W, b = _inputs(256, 1024, 32768, seed=1)
    kw = dict(top_k=50, top_p=0.9)
    a = F.vocab_sample(h, W, b, 1.0, 9, 3, **kw)
    c = F.vocab_sample(h, W, b, 1.0, 9, 3, **kw)
    assert torch.equal(a[0], c[0]) and torch.equal(a[1], c[1])
    step = torch.full((1,), 3, dtype=torch.int32, device=DEV)
    tok = torch.zeros(256, dtype=torch.int32, device=DEV)
    F.vocab_sample(h, W, b, 1.0, 9, step, tokens=tok, **kw)                          # warm-up outside the capture
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        F.vocab_sample(h, W, b, 1.0, 9, step, tokens=tok, **kw)
    step.fill_(3)
    g.replay()
    assert torch.equal(tok, a[0]) and int(step) == 4
    g.replay()
    assert torch.equal(tok, F.vocab_sample(h, W, b, 1.0, 9, 4, **kw)[0]) and int(step) == 5


@pytest.mark.parametrize("V", [512, 300])
def test_distribution(V):
    """The chi-square test of tests/test_top_k_top_p.py on the GPU: h = 0, so the logits are the bias exactly."""
    from test_generate import designed_logits
    from test_top_k_top_p import chi_square_kept_ok
    from lstm_tensorspark_b200.ops import functional as F
    from lstm_tensorspark_b200.ops import reference as ref
    B, S = 256, 40
    bias = designed_logits(V).to(DEV)
    h = torch.zeros(B, 64, dtype=torch.bfloat16, device=DEV)
    W = torch.randn(64, V, device=DEV)
    for temperature in (0.5, 1.0, 2.0):
        for top_k, top_p in ((5, 1.0), (0, 0.8), (6, 0.9)):
            keep = bias.cpu().double() >= ref.sample_threshold(bias.cpu().double().view(1, V), temperature, top_k, top_p)
            step = torch.zeros(1, dtype=torch.int32, device=DEV)
            rec = (torch.zeros(B, S, dtype=torch.int32, device=DEV), torch.zeros(B, S, device=DEV), 0)
            for _ in range(S):
                F.vocab_sample(h, W, bias, temperature, 1234, step, record=rec, top_k=top_k, top_p=top_p)
            draws = rec[0].cpu().numpy().ravel()
            assert chi_square_kept_ok(draws, bias.cpu().double(), temperature, keep), (temperature, top_k, top_p)


# ---- the decode loop ------------------------------------------------------------------------------------------------------------
def test_generate_with_filters_replays_without_a_sync(monkeypatch):
    """The headline shape (2 x 1024, V = 32768, B = 256) with deterministic recurrences, as tests/test_gpu_generate.py."""
    from test_gpu_generate import _lm, _prompts
    from lstm_tensorspark_b200.ops import cuda_lstm
    monkeypatch.setattr(cuda_lstm, "SEQ_VARIANT", (cuda_lstm.SEQ_VARIANT & ~(7 << 12)) | (3 << 12))
    B, T, V, Nn = 256, 32, 32768, 8
    m = _lm("1024,1024", V, 1024, B, T)
    x, lengths = _prompts(B, T, V, 2)
    kw = dict(top_k=50, top_p=0.9)
    eager = m.generate(x, lengths, Nn, 1.0, 5, graph=False, **kw)
    n0 = _stat("vocab_sample_filtered")
    first = m.generate(x, lengths, Nn, 1.0, 5, **kw)                          # captures the decode step
    assert _stat("vocab_sample_filtered") > n0
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        tok, lp = m.generate(x, lengths, Nn, 1.0, 5, **kw)                    # replays it
    finally:
        torch.cuda.set_sync_debug_mode(0)
    for a in (first, (tok, lp)):
        assert torch.equal(a[0], eager[0]) and torch.equal(a[1], eager[1])
    assert bool(torch.isfinite(lp).all()) and bool((lp <= 0).all())
    free = m.generate(x, lengths, Nn, 1.0, 5)
    assert sum(k[3] for k in m._decoders) == 1 and not torch.equal(free[0], tok)   # another filter replaced the graph: other tokens
    assert torch.equal(m.generate(x, lengths, Nn, 0.0, 5, **kw)[0], m.generate(x, lengths, Nn, 0.0, 5)[0])


def test_tiny_trained_model_generates_the_chain_with_filters(tmp_path):
    from lstm_tensorspark_b200.config import Config
    from lstm_tensorspark_b200.trainer import run_job
    base = dict(hidden_units="32", in_features=16, seq_len=12, batch_size=32, vocab_size=64, next_token=True, synthetic=512,
                device="cuda", quiet=True, init="scaled", learning_rate=2e-2, steps_mode="epochs", evaluate_every=20,
                checkpoint_path=str(tmp_path / "ck"), output_path=str(tmp_path / "out"))
    run_job(Config(epochs=25, **base).validate(), standalone=True)
    gen = dict(base, synthetic=100)
    free = run_job(Config(mode="generate", temperature=1.0, **gen).validate(), standalone=True)
    nucleus = run_job(Config(mode="generate", temperature=1.0, top_p=0.5, **gen).validate(), standalone=True)
    top4 = run_job(Config(mode="generate", temperature=1.0, top_k=4, **gen).validate(), standalone=True)
    assert nucleus["top_p"] == 0.5 and top4["top_k"] == 4
    assert nucleus["legal_fraction"] >= 0.9, nucleus["legal_fraction"]
    assert top4["legal_fraction"] >= free["legal_fraction"], (top4["legal_fraction"], free["legal_fraction"])
    for out in (free, nucleus, top4):
        assert out["tokens"] == 100 * 32 and math.isfinite(out["mean_logprob"]) and out["mean_logprob"] <= 0
