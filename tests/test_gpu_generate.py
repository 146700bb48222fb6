"""Text generation on the GPU: the sampling op (the head's tensor-core kernel and the fallback for the inputs it does not take)
against the fp64 reference within the budget of tests/lstm_numerics.py, the distribution it draws from, its determinism, the
decode loop (graph replay equals eager, no host sync until the result is read, agreement with the whole-sequence path) and a
tiny trained model.

Budget of one row's perturbed scores: ALPHA x the largest error of an fp32 evaluation of the same definition (the rounding points
of the kernels: fp32 logits from bf16 operands, fp32 score) plus FLOOR x the largest score magnitude."""
import math

import numpy as np
import pytest
import torch

import lstm_numerics as N

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)


@pytest.fixture(autouse=True)
def _fp32_matmuls(monkeypatch):
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)


def _stat(k):
    from lstm_tensorspark_b200.ops import cuda_lstm
    return cuda_lstm.STATS.get(k, 0)


def _inputs(B, H, V, seed, dtype=torch.bfloat16):
    g = torch.Generator().manual_seed(seed)
    h = torch.randn(B, H, generator=g).to(DEV, dtype)
    W = (torch.randn(H, V, generator=g) * (2.0 / H ** 0.5)).to(DEV)
    b = torch.randn(V, generator=g).to(DEV)
    return h, W, b


def _check(h, W, b, temperature, seed, step, tok, lp, row0=0):
    """The GPU's tokens and log-probabilities against the fp64 reference of the same definition."""
    from lstm_tensorspark_b200.ops import reference as ref
    Wr = W.bfloat16()
    l64 = h.double() @ Wr.double() + b.double()
    l32 = h.float() @ Wr.float() + b.float()
    s64 = ref.sample_scores(l64, temperature, seed, step, row0)
    if temperature == 0:
        s32 = l32.double()
    else:
        g = -torch.log(-torch.log(ref.sample_uniform(ref.sample_noise_words(h.shape[0], W.shape[1], seed, step, device=DEV, row0=row0))))
        s32 = (l32 * torch.tensor(1.0 / temperature, dtype=torch.float32) + g.float()).double()
    tol = N.ALPHA * (s32 - s64).abs().amax(1) + N.FLOOR * s64.abs().amax(1)
    top2 = s64.topk(2, dim=1).values
    t = tok.long()
    assert bool(((t >= 0) & (t < W.shape[1])).all())
    got = s64.gather(1, t.view(-1, 1)).squeeze(1)
    assert bool((got >= top2[:, 0] - tol).all()), float((top2[:, 0] - got - tol).max())
    clear = (top2[:, 0] - top2[:, 1]) > tol
    ref_tok = s64.argmax(1)
    assert bool((t[clear] == ref_tok[clear]).all())
    lp64 = torch.log_softmax(l64, 1).gather(1, t.view(-1, 1)).squeeze(1)
    lp32 = torch.log_softmax(l32, 1).gather(1, t.view(-1, 1)).squeeze(1)
    N.check_budget("logprob", lp, lp64, lp32)
    return int(clear.sum())


# ---- the op --------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B", [1, 3, 130, 256])
@pytest.mark.parametrize("H", [64, 1024])
@pytest.mark.parametrize("V", [512, 4104, 32768])
def test_op_against_fp64(B, H, V):
    from lstm_tensorspark_b200.ops import functional as F
    h, W, b = _inputs(B, H, V, seed=B + H + V)
    for temperature in (0.0, 0.7, 1.0, 2.0):
        n0 = _stat("vocab_sample")
        step = torch.full((1,), 5, dtype=torch.int32, device=DEV)
        tok, lp = F.vocab_sample(h, W, b, temperature, 11, step)
        assert _stat("vocab_sample") == n0 + 1 and int(step) == 6 and tok.dtype == torch.int32 and lp.dtype == torch.float32
        clear = _check(h, W, b, temperature, 11, 5, tok, lp)
        assert clear >= B // 2


@pytest.mark.parametrize("H,V,dtype", [(1024, 4104, torch.bfloat16), (96, 1000, torch.bfloat16)])
def test_row_offset(H, V, dtype):
    """``row0`` as an int and as a device tensor, on the head kernel and on the fallback: the reference at that counter row."""
    from lstm_tensorspark_b200.ops import functional as F
    h, W, b = _inputs(130, H, V, seed=5, dtype=dtype)
    W = W.bfloat16().float()
    a = F.vocab_sample(h, W, b, 1.0, 4, 2, row0=1000)
    c = F.vocab_sample(h, W, b, 1.0, 4, 2, row0=torch.full((1,), 1000, dtype=torch.int32, device=DEV))
    assert torch.equal(a[0], c[0]) and torch.equal(a[1], c[1])
    assert not torch.equal(a[0], F.vocab_sample(h, W, b, 1.0, 4, 2)[0])
    _check(h, W, b, 1.0, 4, 2, a[0], a[1], row0=1000)


@pytest.mark.parametrize("B,H,V,dtype", [(5, 64, 512, torch.float32), (130, 128, 300, torch.bfloat16), (7, 96, 1000, torch.bfloat16),
                                         (3, 64, 4100, torch.bfloat16)])
def test_fallback_against_fp64(B, H, V, dtype):
    """fp32 activations, C < 512, H % 64 != 0, C % 8 != 0: the head GEMM's fp32 logits, then the sampling kernel."""
    from lstm_tensorspark_b200.ops import cuda_vocab_head
    from lstm_tensorspark_b200.ops import functional as F
    h, W, b = _inputs(B, H, V, seed=V, dtype=dtype)
    W = W.bfloat16().float()                                     # whatever the GEMM reads of W, it is these values
    assert not cuda_vocab_head.supported(h.unsqueeze(0), V)
    for temperature in (0.0, 1.0):
        tok, lp = F.vocab_sample(h, W, b, temperature, 3, 2)
        _check(h, W, b, temperature, 3, 2, tok, lp)


@pytest.mark.parametrize("V", [512, 300])
def test_distribution(V):
    """The same chi-square test as on the CPU (tests/test_generate.py): h = 0, so the logits are the bias exactly."""
    from test_generate import chi_square_ok, designed_logits
    from lstm_tensorspark_b200.ops import functional as F
    B, S = 256, 40
    bias = designed_logits(V).to(DEV)
    h = torch.zeros(B, 64, dtype=torch.bfloat16, device=DEV)
    W = torch.randn(64, V, device=DEV)
    for temperature in (0.5, 1.0, 2.0):
        step = torch.zeros(1, dtype=torch.int32, device=DEV)
        rec = (torch.zeros(B, S, dtype=torch.int32, device=DEV), torch.zeros(B, S, device=DEV), 0)
        for _ in range(S):
            F.vocab_sample(h, W, bias, temperature, 1234, step, record=rec)
        draws = rec[0].cpu().numpy().ravel()
        assert chi_square_ok(draws, bias.cpu().double(), temperature), temperature


def test_op_is_deterministic_and_a_graph_replays_it():
    from lstm_tensorspark_b200.ops import functional as F
    h, W, b = _inputs(256, 1024, 32768, seed=1)
    a = F.vocab_sample(h, W, b, 1.0, 9, 3)
    c = F.vocab_sample(h, W, b, 1.0, 9, 3)
    assert torch.equal(a[0], c[0]) and torch.equal(a[1], c[1])
    step = torch.full((1,), 3, dtype=torch.int32, device=DEV)
    tok = torch.zeros(256, dtype=torch.int32, device=DEV)
    F.vocab_sample(h, W, b, 1.0, 9, step, tokens=tok)                     # warm-up outside the capture
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        F.vocab_sample(h, W, b, 1.0, 9, step, tokens=tok)
    step.fill_(3)
    g.replay()
    assert torch.equal(tok, a[0]) and int(step) == 4
    g.replay()                                                            # a replay reads the advanced step: new noise
    assert torch.equal(tok, F.vocab_sample(h, W, b, 1.0, 9, 4)[0]) and int(step) == 5


# ---- the decode loop -----------------------------------------------------------------------------------------------------
def _lm(hidden, V, E, B, T):
    from lstm_tensorspark_b200.config import Config
    from lstm_tensorspark_b200.engine import TrainEngine
    cfg = Config(hidden_units=hidden, in_features=E, seq_len=T, batch_size=B, vocab_size=V, next_token=True, partitions=1,
                 sync_mode="none", init="scaled", device="cuda", quiet=True).validate()
    eng = TrainEngine(cfg, 0, 1, None, batch_size=B, device=DEV, dtype=torch.bfloat16)
    eng.model.eval()
    return eng.model


def _prompts(B, T, V, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randint(0, V, (B, T), generator=g, dtype=torch.int32)
    lengths = torch.randint(1, T + 1, (B,), generator=g, dtype=torch.int32)
    lengths[0] = T
    return x.to(DEV), lengths.to(DEV)


def test_generate_graph_equals_eager_and_replays_without_a_sync(monkeypatch):
    """The headline shape: 2 x 1024, V = 32768, B = 256.  The recurrences consume their operand blocks in index order (what
    --deterministic selects; by default arrival order makes h differ in its last bits from run to run, and untrained logits
    over 32768 classes hold near-ties that such bits decide), so every run below can be compared bit for bit."""
    from lstm_tensorspark_b200.ops import cuda_lstm
    monkeypatch.setattr(cuda_lstm, "SEQ_VARIANT", (cuda_lstm.SEQ_VARIANT & ~(7 << 12)) | (3 << 12))
    B, T, V, Nn = 256, 32, 32768, 8
    m = _lm("1024,1024", V, 1024, B, T)
    x, lengths = _prompts(B, T, V, 2)
    eager = m.generate(x, lengths, Nn, 1.0, 5, graph=False)
    first = m.generate(x, lengths, Nn, 1.0, 5)                               # captures the decode step
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        tok, lp = m.generate(x, lengths, Nn, 1.0, 5)                         # replays it
    finally:
        torch.cuda.set_sync_debug_mode(0)
    for a in (first, (tok, lp)):
        assert torch.equal(a[0], eager[0]) and torch.equal(a[1], eager[1])
    assert bool(torch.isfinite(lp).all()) and bool((lp <= 0).all())
    greedy = m.generate(x, lengths, Nn, 0.0, 5)
    assert torch.equal(greedy[0], m.generate(x, lengths, Nn, 0.0, 6)[0])    # the seed does not enter a greedy run


@pytest.mark.parametrize("hidden,E,schedule", [("1024,1024", 1024, "pipelined"), ("256,256", 128, "wavefront"), ("256", 128, None)])
def test_decode_agrees_with_the_sequence_path(hidden, E, schedule):
    """Rerun prompt + generated tokens through ``sequence_features``: each generated token is the sample of the logits there."""
    from lstm_tensorspark_b200.ops import cuda_lstm
    from lstm_tensorspark_b200.ops import reference as ref
    B, T, V, Nn = 256, 16, 4096, 12
    if schedule is not None and cuda_lstm._sms(DEV) == 132:
        h = int(hidden.split(",")[0])
        assert cuda_lstm.pair_schedule(T, B, E, h, h, 132, cuda_lstm._coresident_ctas(DEV)) == schedule
    m = _lm(hidden, V, E, B, T + Nn)
    x, lengths = _prompts(B, T, V, 7)
    for temperature in (0.0, 1.0):
        key = f"{schedule}_fwd"
        n0 = cuda_lstm.STATS.get(key, 0)
        tok, lp = m.generate(x, lengths, Nn, temperature, 3)
        if schedule is not None:
            assert cuda_lstm.STATS.get(key, 0) > n0
        full = torch.zeros(B, T + Nn, dtype=torch.int32, device=DEV)
        full[:, :T] = x
        pos = lengths.long().view(B, 1) + torch.arange(Nn, device=DEV).view(1, Nn)          # where generated token j lands
        full.scatter_(1, pos, tok)
        with torch.no_grad():
            h_seq = m.sequence_features(full, lengths + Nn)                                   # [T + N, B, H]
            l = m.head(h_seq.reshape(-1, h_seq.shape[2])).view(T + Nn, B, V).transpose(0, 1)  # [B, T + N, V]
        prev = pos - 1                                                                        # token j is sampled after position prev
        same = 0
        for j in range(Nn):
            lj = l[torch.arange(B, device=DEV), prev[:, j]].double()
            s = ref.sample_scores(lj, temperature, 3, j)
            best = s.max(1).values
            got = s.gather(1, tok[:, j].long().view(-1, 1)).squeeze(1)
            tol = 0.05 * (1.0 + best.abs())
            assert bool((got >= best - tol).all()), (hidden, temperature, j)
            same += int((s.argmax(1) == tok[:, j].long()).sum())
        assert same >= 0.9 * B * Nn, (hidden, temperature, same)


def test_tiny_trained_model_generates_the_chain(tmp_path):
    from lstm_tensorspark_b200.config import Config
    from lstm_tensorspark_b200.trainer import run_job
    base = dict(hidden_units="32", in_features=16, seq_len=12, batch_size=32, vocab_size=64, next_token=True, synthetic=512,
                device="cuda", quiet=True, init="scaled", learning_rate=2e-2, steps_mode="epochs", evaluate_every=20,
                checkpoint_path=str(tmp_path / "ck"), output_path=str(tmp_path / "out"))
    run_job(Config(epochs=25, **base).validate(), standalone=True)
    ev = run_job(Config(mode="eval", **base).validate(), standalone=True)
    assert ev["perplexity"] < 8
    out = run_job(Config(mode="generate", temperature=0.0, **dict(base, synthetic=100)).validate(), standalone=True)
    assert out["legal_fraction"] >= 0.9 and out["tokens"] == 100 * 32
    assert math.isfinite(out["mean_logprob"]) and out["mean_logprob"] <= 0
