"""Top-k and nucleus (top-p) sampling without a GPU: the reference's kept set against a class-by-class fp64 evaluation of the
definition (ties at the top-k boundary and at the nucleus boundary), the off values, the coupling with the unfiltered draw, the
distribution of the draws, flags, and ``--mode generate`` end to end with both filters."""
import json
import math
import warnings

import numpy as np
import pytest
import torch
from scipy.stats import chi2

from lstm_tensorspark_b200.config import Config
from lstm_tensorspark_b200.ops import functional as F
from lstm_tensorspark_b200.ops import reference as ref
from test_generate import BINS, CHI2_QUANTILE, designed_logits


def brute_kept(row, temperature, top_k, top_p):
    """The definition one class at a time, in fp64: c survives top-k iff fewer than k classes have a strictly larger logit;
    c then survives top-p iff the tempered mass of the survivors with a strictly larger logit is below p times their total."""
    l = [float(v) for v in row]
    C = len(l)
    alive = [True] * C
    if 0 < top_k < C:
        alive = [sum(1 for o in l if o > v) < top_k for v in l]
    if top_p < 1:
        mx = max(l)
        e = [math.exp((v - mx) / temperature) if a else 0.0 for v, a in zip(l, alive)]
        z = math.fsum(e)
        alive = [a and math.fsum(e[o] for o in range(C) if l[o] > l[c]) < top_p * z for c, a in enumerate(alive)]
    return alive


# Designed rows (t = 1): ties at the k-th value, and nucleus cuts that fall inside a tie group.
TIES = torch.tensor([
    [3.0, 1.0, 2.0, 3.0, 2.0, 0.0, 2.0, -1.0, 1.0, -4.0, 2.0, 0.5],     # k = 3, 4, 5, 6: the k-th largest is a tied 2
    [0.0, 0.0, 0.0, 0.0, 1.0, 1.0, -2.0, -2.0, -2.0, 5.0, -9.0, 0.0],    # one dominant class, then tie groups
    [1.0] * 12,                                                          # everything tied: every filter keeps all
], dtype=torch.float64)


@pytest.mark.parametrize("top_k", [0, 1, 2, 3, 4, 6, 7, 11, 12, 40])
@pytest.mark.parametrize("top_p", [1.0, 0.999, 0.9, 0.6, 0.35, 0.05])
@pytest.mark.parametrize("temperature", [0.5, 1.0, 3.0])
def test_kept_set_matches_the_class_by_class_definition(top_k, top_p, temperature):
    tau = ref.sample_threshold(TIES, temperature, top_k, top_p)
    for b in range(TIES.shape[0]):
        got = (TIES[b] >= tau[b]).tolist()
        assert got == brute_kept(TIES[b], temperature, top_k, top_p), (b, tau[b])


def test_random_rows_match_the_definition():
    g = torch.Generator().manual_seed(0)
    l = (torch.randn(40, 30, generator=g) * 2).round(decimals=1).double()        # rounded: many exact ties
    for top_k, top_p, t in ((5, 1.0, 1.0), (0, 0.8, 0.7), (7, 0.5, 1.3), (12, 0.95, 2.0)):
        tau = ref.sample_threshold(l, t, top_k, top_p)
        for b in range(l.shape[0]):
            assert (l[b] >= tau[b]).tolist() == brute_kept(l[b], t, top_k, top_p)


def test_ties_at_the_boundary_are_kept():
    row = TIES[:1]
    assert int((row >= ref.sample_threshold(row, 1.0, 3, 1.0).unsqueeze(1)).sum()) == 6     # 3, 3 and the four 2s
    # the nucleus: q of the two 3s is 2e^3 / Z; the cut lands in the 2s and keeps all four of them
    l = row[0].tolist()
    z = sum(math.exp(v) for v in l)
    p = (2 * math.exp(3) + 0.5 * math.exp(2)) / z
    assert int((row >= ref.sample_threshold(row, 1.0, 0, p).unsqueeze(1)).sum()) == 6


def test_off_values_give_the_unfiltered_tokens():
    g = torch.Generator().manual_seed(1)
    l = torch.randn(16, 50, generator=g).double()
    for t in (0.5, 1.0):
        want = ref.sample_logits(l, t, 3, 4)
        for k, p in ((0, 1.0), (50, 1.0), (51, 1.0), (10 ** 9, 1.0)):
            got = ref.sample_logits(l, t, 3, 4, top_k=k, top_p=p)
            assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1])
            assert bool(torch.isinf(ref.sample_threshold(l, t, k, p)).all())
    # greedy: the filters have no effect
    assert torch.equal(ref.sample_logits(l, 0.0, 3, 4, top_k=1, top_p=0.01)[0], ref.sample_logits(l, 0.0, 3, 4)[0])
    assert not ref.sample_filters_active(50, 0.0, 5, 0.5) and ref.sample_filters_active(50, 1.0, 49, 1.0)


def test_coupling_and_no_draw_outside_the_kept_set():
    g = torch.Generator().manual_seed(2)
    l = (torch.randn(64, 200, generator=g) * 3).double()
    kept_same = 0
    for step in range(6):
        for k, p in ((1, 1.0), (10, 1.0), (0, 0.9), (0, 0.3), (20, 0.7)):
            free, flp = ref.sample_logits(l, 1.0, 9, step)
            tok, lp = ref.sample_logits(l, 1.0, 9, step, top_k=k, top_p=p)
            keep = l >= ref.sample_threshold(l, 1.0, k, p).unsqueeze(1)
            assert bool(keep.gather(1, tok.long().view(-1, 1)).all())                       # never outside K
            inside = keep.gather(1, free.long().view(-1, 1)).squeeze(1)
            assert torch.equal(tok[inside], free[inside])                                   # the coupling
            kept_same += int(inside.sum())
            # log p(token) stays under the full softmax
            assert torch.allclose(lp, torch.log_softmax(l, 1).gather(1, tok.long().view(-1, 1)).squeeze(1), rtol=0, atol=0)
    assert kept_same > 0


def test_tiny_top_p_keeps_only_the_argmax_or_its_ties():
    l = torch.tensor([[1.0, 4.0, 2.0, 4.0, -1.0], [0.0, 0.0, 3.0, 1.0, 2.0]], dtype=torch.float64)
    tau = ref.sample_threshold(l, 1.0, 0, 1e-9)
    assert (l >= tau.unsqueeze(1)).tolist() == [[False, True, False, True, False], [False, False, True, False, False]]
    for s in range(20):
        assert ref.sample_logits(l, 1.0, 5, s, top_p=1e-9)[0].tolist()[1] == 2


def chi_square_kept_ok(draws: np.ndarray, logits: torch.Tensor, temperature: float, keep: torch.Tensor) -> bool:
    """The chi-square test of tests/test_generate.py over the designed bins that the filter keeps, against softmax(l / t)
    restricted to the kept set and renormalised (a kept class outside the bins would join the last bin; the designed rows
    below keep none)."""
    idx = torch.linspace(0, len(logits) - 1, BINS).round().long()
    assert torch.equal(keep.nonzero().squeeze(1), idx[keep[idx]]), "the kept set must be made of designed bins"
    idx = idx[keep[idx]].numpy()
    p = torch.softmax(torch.where(keep, logits.double() / temperature, torch.tensor(float("-inf"), dtype=torch.float64)), 0).numpy()
    expected = p[idx] * len(draws)
    counts = np.array([np.sum(draws == i) for i in idx], dtype=np.float64)
    assert counts.sum() == len(draws), "a draw fell outside the kept set"
    assert expected.min() >= 5, "too few draws per bin for the chi-square approximation"
    stat = float(((counts - expected) ** 2 / expected).sum())
    return stat < chi2.ppf(CHI2_QUANTILE, len(idx) - 1)


@pytest.mark.parametrize("top_k,top_p", [(5, 1.0), (0, 0.8), (6, 0.9)])
@pytest.mark.parametrize("temperature", [0.5, 1.0, 2.0])
def test_draws_follow_the_truncated_tempered_softmax(top_k, top_p, temperature):
    V, B, S = 64, 256, 40
    logits = designed_logits(V).double()
    keep = logits >= ref.sample_threshold(logits.view(1, V), temperature, top_k, top_p)
    assert 2 <= int(keep.sum()) < BINS
    draws = np.concatenate([ref.sample_logits(logits.expand(B, V), temperature, 1234, s, top_k=top_k, top_p=top_p)[0].numpy()
                            for s in range(S)])
    assert chi_square_kept_ok(draws, logits, temperature, keep)
    assert not chi_square_kept_ok(draws, logits, temperature * 2, keep)                 # the test's power: another temperature


def test_functional_cpu_path_and_argument_errors():
    g = torch.Generator().manual_seed(3)
    h, W, b = torch.randn(4, 8, generator=g), torch.randn(8, 30, generator=g), torch.randn(30, generator=g)
    step = torch.tensor([2], dtype=torch.int32)
    tok, lp = F.vocab_sample(h, W, b, 1.0, 5, step, top_k=3, top_p=0.9)
    want, wlp = ref.vocab_sample(h, W, b, 1.0, 5, 2, top_k=3, top_p=0.9)
    assert int(step) == 3 and torch.equal(tok, want) and torch.allclose(lp, wlp.float())
    for kw, msg in ((dict(top_k=-1), "top_k must be an integer >= 0.*-1"), (dict(top_k=1.5), "top_k.*1.5"),
                    (dict(top_p=0.0), r"top_p must be a finite number in \(0, 1\].*0.0"), (dict(top_p=1.5), "top_p.*1.5"),
                    (dict(top_p=float("nan")), "top_p.*nan"), (dict(top_p=float("inf")), "top_p.*inf"), (dict(top_p=-0.2), "top_p")):
        with pytest.raises(ValueError, match=msg):
            F.vocab_sample(h, W, b, 1.0, 5, 0, **kw)
        with pytest.raises(ValueError, match=msg):
            ref.sample_logits(h @ W, 1.0, 5, 0, **kw)


# ---- flags -------------------------------------------------------------------------------------------------------------------
def _gen_cfg(**kw):
    return Config(**dict(dict(mode="generate", next_token=True, vocab_size=10, seq_len=4), **kw))


def test_filter_flags_defaults_and_parsing():
    cfg = _gen_cfg().validate()
    assert cfg.top_k == 0 and cfg.top_p == 1.0
    from lstm_tensorspark_b200.config import parse_args
    cfg = parse_args(["--mode", "generate", "--next_token", "--vocab_size", "10", "--seq_len", "4", "--top_k", "5", "--top_p",
                      "0.9"]).validate()
    assert cfg.top_k == 5 and cfg.top_p == 0.9
    with warnings.catch_warnings():
        warnings.simplefilter("error")
        _gen_cfg(top_k=3, top_p=0.5).validate()                                  # with sampling: silent
        Config(next_token=True, vocab_size=10, seq_len=4).validate()             # the defaults outside --mode generate: silent


@pytest.mark.parametrize("kw,msg", [
    (dict(top_k=-1), r"--top_k must be an integer >= 0 \(0 = off\), got -1"),
    (dict(top_p=0.0), r"--top_p must be a number in \(0, 1\] \(1 = off\), got 0.0"),
    (dict(top_p=1.01), "--top_p .* got 1.01"),
    (dict(top_p=float("nan")), "--top_p .* got nan"),
    (dict(top_p=-1.0), "--top_p"),
])
def test_filter_flag_errors(kw, msg):
    with pytest.raises(ValueError, match=msg):
        _gen_cfg(**kw).validate()


@pytest.mark.parametrize("flag,value", [("top_k", 5), ("top_p", 0.5)])
def test_filter_flags_warn(flag, value):
    with pytest.warns(UserWarning, match=f"--{flag} .* no effect without --mode generate"):
        Config(next_token=True, vocab_size=10, seq_len=4, **{flag: value}).validate()
    with pytest.warns(UserWarning, match=f"--{flag} .* no effect with --temperature 0"):
        _gen_cfg(temperature=0.0, **{flag: value}).validate()


# ---- the decode loop and the CLI ---------------------------------------------------------------------------------------------
def test_decoder_is_keyed_by_the_filters():
    from test_generate import _model, _prompts
    m = _model()
    x, lengths = _prompts(6, 7, 40)
    free = m.generate(x, lengths, 6, 1.0, 1)
    k1 = m.generate(x, lengths, 6, 1.0, 1, top_k=1)
    assert len(m._decoders) == 1 and next(iter(m._decoders.values())).top_k == 1
    greedy = m.generate(x, lengths, 6, 0.0, 1)
    assert torch.equal(k1[0], greedy[0])                                         # top_k 1 is the arg-max at any temperature
    assert torch.equal(m.generate(x, lengths, 6, 1.0, 1)[0], free[0])            # and back: the unfiltered decoder again
    nuc = m.generate(x, lengths, 6, 1.0, 1, top_p=0.5)
    assert bool(torch.isfinite(nuc[1]).all()) and bool((nuc[1] <= 0).all())
    with pytest.raises(ValueError, match="top_p"):
        m.generate(x, lengths, 6, 1.0, 1, top_p=0.0)


def test_generate_with_both_filters_end_to_end(tmp_path, capsys):
    from test_generate import _base
    from lstm_tensorspark_b200.trainer import run_job
    run_job(Config(epochs=3, **_base(tmp_path)).validate(), standalone=True)
    log = tmp_path / "gen.jsonl"
    out = run_job(Config(mode="generate", **dict(_base(tmp_path), quiet=False, synthetic=20, max_new_tokens=6, top_k=4,
                                                  top_p=0.8, json_log=str(log))).validate(), standalone=True)
    assert out["top_k"] == 4 and out["top_p"] == 0.8 and out["tokens"] == 120
    logged = json.loads(open(log).read().splitlines()[-1])
    assert logged["top_k"] == 4 and logged["top_p"] == 0.8
    assert "top_k 4, top_p 0.8" in capsys.readouterr().out
    rows = [list(map(int, r.split(","))) for r in open(tmp_path / "out" / "generated.csv").read().splitlines()]
    assert len(rows) == 20 and all(len(r) == 6 and all(0 <= v < 64 for v in r) for r in rows)
