"""Text generation without a GPU: the sampling definition (reference against a direct evaluation, the Philox counters, the noise's
range, the distribution it draws from), the decode loop (batch independence, agreement with the whole-sequence path), flags,
prompt rows, refusals and ``--mode generate`` end to end on a small trained language model."""
import math
import os
import warnings

import numpy as np
import pytest
import torch
from scipy.stats import chi2

from lstm_tensorspark_b200 import data as D
from lstm_tensorspark_b200.config import Config
from lstm_tensorspark_b200.ops import functional as F
from lstm_tensorspark_b200.ops import reference as ref

# ---- the distribution test, shared with tests/test_gpu_generate.py -----------------------------------------------------------
# Eight classes with logits 2, 1.5, ..., -1.5 at spread-out indices, every other class at -30 (merged into the last bin); the
# draws pass when the chi-square statistic over the eight bins stays below its 0.999 quantile (7 degrees of freedom, 24.3):
# with a fixed seed the test is deterministic, and a correct sampler fails it with probability 1e-3 over seeds.
BINS = 8
CHI2_QUANTILE = 0.999


def designed_logits(V: int) -> torch.Tensor:
    l = torch.full((V,), -30.0)
    idx = torch.linspace(0, V - 1, BINS).round().long()
    l[idx] = torch.arange(BINS, dtype=torch.float32) * -0.5 + 2.0
    return l


def chi_square_ok(draws: np.ndarray, logits: torch.Tensor, temperature: float) -> bool:
    p = torch.softmax(logits.double() / temperature, 0).numpy()
    idx = torch.linspace(0, len(p) - 1, BINS).round().long().numpy()
    expected = p[idx].copy()
    expected[-1] += 1.0 - expected.sum()                     # every other class joins the last bin
    counts = np.array([np.sum(draws == i) for i in idx], dtype=np.float64)
    counts[-1] += len(draws) - counts.sum()
    expected *= len(draws)
    assert expected.min() >= 5, "too few draws per bin for the chi-square approximation"
    stat = float(((counts - expected) ** 2 / expected).sum())
    return stat < chi2.ppf(CHI2_QUANTILE, BINS - 1)


# ---- the definition ----------------------------------------------------------------------------------------------------------
def _direct(logits, temperature, seed, step):
    """The definition written out one class at a time, in fp64."""
    B, C = logits.shape
    toks, lps = [], []
    for b in range(B):
        scores = []
        for c in range(C):
            l = float(logits[b, c])
            if temperature == 0:
                scores.append(l)
                continue
            w = int(ref.philox4x32_10(torch.tensor([c >> 2, b, step, 0]), seed & 0xFFFFFFFF, 0x53414D50)[c & 3])
            u = ((w >> 8) + 0.5) * 2.0 ** -24
            scores.append(l / temperature - math.log(-math.log(u)))
        t = max(range(C), key=lambda c: (scores[c], -c))                     # the smallest index on a tie
        lse = math.log(sum(math.exp(float(v)) for v in logits[b]))
        toks.append(t)
        lps.append(float(logits[b, t]) - lse)
    return toks, lps


@pytest.mark.parametrize("temperature", [0.0, 0.7, 1.0, 2.0])
def test_reference_matches_the_definition(temperature):
    g = torch.Generator().manual_seed(1)
    h, W, b = torch.randn(3, 5, generator=g), torch.randn(5, 10, generator=g), torch.randn(10, generator=g)
    tok, lp = ref.vocab_sample(h, W, b, temperature, 77, 4)
    toks, lps = _direct(h.double() @ W.double() + b.double(), temperature, 77, 4)
    assert tok.dtype == torch.int32 and tok.tolist() == toks
    assert np.allclose(lp.numpy(), lps, rtol=1e-12, atol=1e-12)


def test_greedy_is_the_argmax_with_the_smallest_index_on_a_tie_and_ignores_the_seed():
    logits = torch.tensor([[1.0, 3.0, 3.0, 0.0], [5.0, 5.0, 5.0, 5.0], [0.0, -1.0, 2.0, 2.0]], dtype=torch.float64)
    for seed, step in ((0, 0), (123, 9)):
        tok, lp = ref.sample_logits(logits, 0.0, seed, step)
        assert tok.tolist() == [1, 0, 2]
        assert torch.allclose(lp, torch.log_softmax(logits, 1)[[0, 1, 2], [1, 0, 2]])


def test_noise_words_are_philox_at_the_stated_counters():
    B, C, seed, step = 3, 10, 0x1234567890, 6
    words = ref.sample_noise_words(B, C, seed, step)
    for b in range(B):
        for c in range(C):
            w = ref.philox4x32_10(torch.tensor([c >> 2, b, step, 0]), seed & 0xFFFFFFFF, ref.SAMPLE_KEY1)[c & 3]
            assert int(words[b, c]) == int(w)
    assert ref.SAMPLE_KEY1 == int.from_bytes(b"SAMP", "big")
    # the streams differ from the dropout masks' (key (seed, partition)) and between steps and rows
    assert not torch.equal(words, ref.sample_noise_words(B, C, seed, step + 1))
    assert not torch.equal(words[0], words[1])


def test_row_offset_moves_the_counter_row():
    words = ref.sample_noise_words(10, 9, 5, 3)
    assert torch.equal(ref.sample_noise_words(4, 9, 5, 3, row0=6), words[6:])
    l = torch.randn(1, 9, dtype=torch.float64, generator=torch.Generator().manual_seed(0)).expand(10, 9)
    assert torch.equal(ref.sample_logits(l[6:], 1.0, 5, 3, row0=6)[0], ref.sample_logits(l, 1.0, 5, 3)[0][6:])
    step, row0 = torch.tensor([3], dtype=torch.int32), torch.tensor([6], dtype=torch.int32)
    h, W, b = torch.randn(4, 8), torch.randn(8, 30), torch.randn(30)
    assert torch.equal(F.vocab_sample(h, W, b, 1.0, 5, step, row0=row0)[0], ref.vocab_sample(h, W, b, 1.0, 5, 3, row0=6)[0])


def test_uniform_stays_inside_the_open_interval():
    u = ref.sample_uniform(torch.tensor([0, 0xFFFFFFFF, 0x80000000, 0x7FFFFFFF], dtype=torch.int64))
    assert u.tolist() == [2.0 ** -25, 1.0 - 2.0 ** -25, 0.5 + 2.0 ** -25, 0.5 - 2.0 ** -25]
    assert bool(((u > 0) & (u < 1)).all())
    g = -torch.log(-torch.log(u))
    assert bool(torch.isfinite(g).all()) and float(g[1]) == pytest.approx(-math.log(2.0 ** -25), rel=1e-6)
    # fp32 holds u below 1/2 and 1 - u above it exactly (what the kernels compute -log u from), not u itself above 1/2
    low, high = u < 0.5, u >= 0.5
    assert torch.equal(u[low].float().double(), u[low]) and torch.equal((1 - u[high]).float().double(), 1 - u[high])
    assert float(u[1].float()) == 1.0


@pytest.mark.parametrize("temperature", [0.5, 1.0, 2.0])
def test_draws_follow_the_tempered_softmax(temperature):
    V, B, S = 64, 256, 40
    logits = designed_logits(V)
    draws = np.concatenate([ref.sample_logits(logits.expand(B, V), temperature, 1234, s)[0].numpy() for s in range(S)])
    assert chi_square_ok(draws, logits.double(), temperature)
    # the same statistic rejects the untempered softmax (a negative control of the test's power)
    assert not chi_square_ok(draws, logits.double(), 1.0 if temperature != 1.0 else 0.5)


def test_functional_cpu_path_advances_the_step_and_records():
    g = torch.Generator().manual_seed(2)
    h, W, b = torch.randn(4, 8, generator=g), torch.randn(8, 30, generator=g), torch.randn(30, generator=g)
    step = torch.tensor([2], dtype=torch.int32)
    rec = (torch.full((4, 3), -1, dtype=torch.int32), torch.zeros(4, 3), 1)
    tokens = torch.zeros(4, dtype=torch.int32)
    tok, lp = F.vocab_sample(h, W, b, 1.0, 5, step, tokens=tokens, record=rec)
    want, wlp = ref.vocab_sample(h, W, b, 1.0, 5, 2)
    assert int(step) == 3 and tok is tokens and torch.equal(tok, want) and lp.dtype == torch.float32
    assert torch.equal(rec[0][:, 1], want) and bool((rec[0][:, [0, 2]] == -1).all()) and torch.allclose(rec[1][:, 1], wlp.float())
    for bad in (-1.0, float("nan"), float("inf")):
        with pytest.raises(ValueError, match="temperature"):
            F.vocab_sample(h, W, b, bad, 5, 0)


# ---- the decode loop ---------------------------------------------------------------------------------------------------------
def _model(hidden="16,16", V=40, E=8, B=6, T=10, **kw):
    from lstm_tensorspark_b200.models.classifier import SequenceClassifier
    cfg = Config(hidden_units=hidden, in_features=E, seq_len=T, batch_size=B, vocab_size=V, next_token=True, device="cpu",
                 init="scaled", **kw).validate()
    return SequenceClassifier(cfg, batch_size=B, device="cpu", generator=torch.Generator().manual_seed(3)).eval()


def _prompts(B, T, V, seed=0):
    g = torch.Generator().manual_seed(seed)
    lengths = torch.randint(1, T + 1, (B,), generator=g, dtype=torch.int32)
    x = torch.randint(0, V, (B, T), generator=g, dtype=torch.int32) * (torch.arange(T) < lengths.view(B, 1))
    return x.to(torch.int32), lengths


def test_ragged_batch_gives_each_prompt_its_own_tokens():
    m = _model()
    x, lengths = _prompts(6, 7, 40)
    tok, lp = m.generate(x, lengths, 5, 0.0, 1)
    assert tok.shape == (6, 5) and tok.dtype == torch.int32 and lp.shape == (6, 5) and bool((lp <= 0).all())
    for b in range(6):
        k = int(lengths[b])
        alone, alp = m.generate(x[b:b + 1, :k], lengths[b:b + 1], 5, 0.0, 1)
        assert torch.equal(alone[0], tok[b]) and torch.allclose(alp[0], lp[b], atol=1e-5)
    # with noise a row's draws depend on (seed, row, step) only: other prompts in the other rows change nothing
    t1, _ = m.generate(x, lengths, 5, 1.0, 1)
    x2, l2 = _prompts(6, 7, 40, seed=9)
    x2[2], l2[2] = x[2], lengths[2]
    t2, _ = m.generate(x2, l2, 5, 1.0, 1)
    assert torch.equal(t1[2], t2[2]) and not torch.equal(t1, t2)


@pytest.mark.parametrize("hidden", ["16,16", "16"])
@pytest.mark.parametrize("temperature", [0.0, 1.0])
def test_decode_agrees_with_the_sequence_path(hidden, temperature):
    """Rerun prompt + generated tokens through ``sequence_features``: each generated token is the reference sample of the logits
    there (fp32 on the CPU: the one-step and whole-sequence paths differ only in summation order)."""
    B, T, V, Nn = 6, 7, 40, 5
    m = _model(hidden=hidden, T=T + Nn)
    x, lengths = _prompts(B, T, V, seed=4)
    tok, lp = m.generate(x, lengths, Nn, temperature, 8)
    full = torch.zeros(B, T + Nn, dtype=torch.int32)
    full[:, :T] = x
    pos = lengths.long().view(B, 1) + torch.arange(Nn).view(1, Nn)
    full.scatter_(1, pos, tok)
    with torch.no_grad():
        h_seq = m.sequence_features(full, lengths + Nn)
        l = m.head(h_seq.reshape(-1, h_seq.shape[2])).view(T + Nn, B, V).transpose(0, 1).double()
    for j in range(Nn):
        lj = l[torch.arange(B), pos[:, j] - 1]
        want, wlp = ref.sample_logits(lj, temperature, 8, j)
        s = ref.sample_scores(lj, temperature, 8, j)
        got = s.gather(1, tok[:, j].long().view(-1, 1)).squeeze(1)
        assert bool((got >= s.max(1).values - 1e-4).all())
        assert int((want == tok[:, j]).sum()) >= B - 1
        assert torch.allclose(lp[:, j].double(), wlp, atol=1e-4)


def test_row_offset_places_a_batch_among_the_prompts_and_one_decoder_is_kept_per_shape():
    m = _model()
    x, lengths = _prompts(6, 7, 40)
    full = m.generate(x, lengths, 5, 1.0, 1)
    part = _model(B=2).generate(x[2:4], lengths[2:4], 5, 1.0, 1, row0=2)
    assert torch.equal(part[0], full[0][2:4]) and torch.allclose(part[1], full[1][2:4], atol=1e-5)
    for seed in range(4):
        m.generate(x, lengths, 5, 1.0, seed)
    assert len(m._decoders) == 1


def test_state_does_not_grow_per_token():
    m = _model()
    x, lengths = _prompts(6, 7, 40)
    m.generate(x, lengths, 20, 1.0, 0)
    assert all(len(layer.state) <= 1 for layer in m.rnn.layers)


def test_a_model_without_next_token_is_refused():
    from lstm_tensorspark_b200.models.classifier import SequenceClassifier
    cfg = Config(hidden_units="8", in_features=4, seq_len=5, batch_size=2, vocab_size=10, per_step_labels=True, num_classes=10,
                 device="cpu").validate()
    m = SequenceClassifier(cfg, batch_size=2, device="cpu")
    with pytest.raises(ValueError, match="--next_token"):
        m.generate(torch.zeros(2, 3, dtype=torch.int32), None, 2)


# ---- flags and prompt rows ---------------------------------------------------------------------------------------------------
def _gen_cfg(**kw):
    return Config(**dict(dict(mode="generate", next_token=True, vocab_size=10, seq_len=4), **kw))


def test_generate_flags():
    cfg = _gen_cfg().validate()
    assert cfg.max_new_tokens == 32 and cfg.temperature == 1.0
    from lstm_tensorspark_b200.config import parse_args
    cfg = parse_args(["--mode", "generate", "--next_token", "--vocab_size", "10", "--seq_len", "4", "--max_new_tokens", "7",
                      "--temperature", "0"])
    assert cfg.max_new_tokens == 7 and cfg.temperature == 0.0
    with warnings.catch_warnings():
        warnings.simplefilter("error")
        Config(next_token=True, vocab_size=10, seq_len=4).validate()             # the defaults outside --mode generate: silent


@pytest.mark.parametrize("kw,msg", [
    (dict(max_new_tokens=0), "--max_new_tokens must be >= 1"),
    (dict(temperature=-0.5), "--temperature must be a finite number >= 0"),
    (dict(temperature=float("nan")), "--temperature"),
    (dict(temperature=float("inf")), "--temperature"),
    (dict(next_token=False, per_step_labels=True, num_classes=10), "--mode generate needs --next_token"),
    (dict(mode="sample"), "generate"),
])
def test_generate_flag_errors(kw, msg):
    with pytest.raises(ValueError, match=msg):
        _gen_cfg(**kw).validate()


@pytest.mark.parametrize("flag,value", [("max_new_tokens", 5), ("temperature", 0.5)])
def test_generate_flags_warn_outside_generate(flag, value):
    with pytest.warns(UserWarning, match=f"--{flag} .* no effect without --mode generate"):
        Config(next_token=True, vocab_size=10, seq_len=4, **{flag: value}).validate()


def test_prompt_rows_are_right_padded():
    x, l = D.process_prompts([["1", "2"], ["3", " 4", "5", "6"], ["7"]], 4, 10)
    assert x.dtype == np.int32 and l.dtype == np.int32
    assert x.tolist() == [[1, 2, 0, 0], [3, 4, 5, 6], [7, 0, 0, 0]] and l.tolist() == [2, 4, 1]


@pytest.mark.parametrize("rows,msg", [
    ([["1", "2"], ["1", "2", "3", "4", "5"]], "row 1: a prompt of 5 token ids is longer than --seq_len 4"),
    ([["1"], ["", ""]], "row 1: an empty prompt"),
    ([["1", "x"]], "row 0: token id 'x' is not an integer"),
    ([["1"], ["2", "10"]], r"row 1: token id 10 outside \[0, 10\)"),
    ([["-1"]], r"row 0: token id -1 outside \[0, 10\)"),
    ([], "no prompts"),
])
def test_malformed_prompt_rows_name_the_row(rows, msg):
    with pytest.raises(ValueError, match=msg):
        D.process_prompts(rows, 4, 10)


def test_synthetic_prompts_and_legal_fraction():
    x, l = D.synthetic_prompts(5, 12, 64, seed=3)
    walks = D.synthetic_next_token(5, 12, 64, seed=3)[0]
    assert x.shape == (5, 3) and np.array_equal(x, walks[:, :3]) and l.tolist() == [3] * 5
    succ = D.next_token_chain(64, 3)
    legal = walks[:, 3:7]                                                       # the walk's own continuation: always allowed
    assert D.legal_fraction(x, l, legal, succ) == 1.0
    bad = legal.copy()
    bad[0, 0] = next(v for v in range(64) if v not in succ[x[0, 2]])            # the prompt -> first token transition
    bad[1, 3] = next(v for v in range(64) if v not in succ[legal[1, 2]])         # the last one
    illegal = 2 + int(bad[0, 1] not in succ[bad[0, 0]])                          # (the changed first token's own successor)
    assert D.legal_fraction(x, l, bad, succ) == pytest.approx(1 - illegal / 20)


# ---- end to end --------------------------------------------------------------------------------------------------------------
def _base(tmp_path, **kw):
    base = dict(hidden_units="32", in_features=16, seq_len=12, batch_size=32, vocab_size=64, next_token=True, synthetic=512,
                device="cpu", quiet=True, init="scaled", learning_rate=2e-2, steps_mode="epochs", evaluate_every=20,
                checkpoint_path=str(tmp_path / "ck"), output_path=str(tmp_path / "out"))
    base.update(kw)
    return base


def test_generate_end_to_end(tmp_path):
    from lstm_tensorspark_b200.trainer import run_job
    run_job(Config(epochs=25, **_base(tmp_path)).validate(), standalone=True)
    assert run_job(Config(mode="eval", **_base(tmp_path)).validate(), standalone=True)["perplexity"] < 8
    csv = tmp_path / "out" / "generated.csv"
    log = tmp_path / "gen.jsonl"

    def gen(**kw):
        out = run_job(Config(mode="generate", **_base(tmp_path, **kw)).validate(), standalone=True)
        return out, [list(map(int, r.split(","))) for r in open(csv).read().splitlines()]

    out, rows = gen(synthetic=70, temperature=0.0, max_new_tokens=9, json_log=str(log), batch_size=32)   # a short last batch
    assert len(rows) == 70 and all(len(r) == 9 and all(0 <= v < 64 for v in r) for r in rows)
    assert out["prompts"] == 70 and out["tokens"] == 630 and out["legal_fraction"] >= 0.9         # chance: 4/64
    import json
    logged = json.loads(open(log).read().splitlines()[-1])
    assert logged["legal_fraction"] == out["legal_fraction"] and logged["mean_logprob"] == out["mean_logprob"]
    # prompts from a file, in order, ragged
    prompts = tmp_path / "prompts.csv"
    prompts.write_text("1,2,3\n5\n7,8,9,10,11,12,13,14,15,16,17,18\n" * 3)
    a = gen(training_path=str(prompts), synthetic=0, temperature=1.0, seed=0, batch_size=4)[1]
    b = gen(training_path=str(prompts), synthetic=0, temperature=1.0, seed=0, batch_size=4)[1]
    c = gen(training_path=str(prompts), synthetic=0, temperature=1.0, seed=1, batch_size=4)[1]
    assert len(a) == 9 and a == b and a != c
    assert a[0] != a[3] or a[1] != a[4]                            # the same prompt in another row draws other noise
    # one prompt repeated across batches: every copy draws its own noise, and the batch size changes nothing
    same = tmp_path / "same.csv"
    same.write_text("3,4,5\n" * 8)
    r4 = gen(training_path=str(same), synthetic=0, temperature=1.0, seed=0, batch_size=4)[1]
    r8 = gen(training_path=str(same), synthetic=0, temperature=1.0, seed=0, batch_size=8)[1]
    r3 = gen(training_path=str(same), synthetic=0, temperature=1.0, seed=0, batch_size=3)[1]
    assert r4 == r8 == r3 and len({tuple(r) for r in r4}) == 8
    g0 = gen(training_path=str(prompts), synthetic=0, temperature=0.0, seed=0, batch_size=4)[1]
    g1 = gen(training_path=str(prompts), synthetic=0, temperature=0.0, seed=1, batch_size=9)[1]
    assert g0 == g1 and g0[0] == g0[3] == g0[6]                   # greedy: no noise, no dependence on the row or the batch


def test_generate_refuses_a_model_trained_without_next_token(tmp_path):
    from lstm_tensorspark_b200.trainer import run_job
    plain = dict(_base(tmp_path), next_token=False, per_step_labels=True, num_classes=64)
    run_job(Config(epochs=1, max_steps=2, **plain).validate(), standalone=True)
    with pytest.raises(ValueError, match="written without --next_token"):
        run_job(Config(mode="generate", **_base(tmp_path)).validate(), standalone=True)
    with pytest.raises(FileNotFoundError, match="--mode generate: no trained model"):
        run_job(Config(mode="generate", **_base(tmp_path, checkpoint_path=str(tmp_path / "none"))).validate(), standalone=True)
