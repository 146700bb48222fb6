"""The continuous cache pointer (``--cache_window``) on the CPU: its flags, the reference definition against a literal
per-position loop in fp64, independence of the segment length, lambda = 0, and ``--mode eval --stateful`` end to end."""
import json
import math
import warnings

import pytest
import torch

from lstm_tensorspark_b200.config import CACHE_LAMBDA_DEFAULT, CACHE_THETA_DEFAULT, Config, parse_args
from lstm_tensorspark_b200.ops import functional as F
from lstm_tensorspark_b200.ops import reference as ref


def _cfg(**kw):
    base = dict(next_token=True, stateful=True, vocab_size=16, seq_len=4, batch_size=3, hidden_units="6", in_features=5,
                device="cpu", quiet=True, init="scaled", mode="eval")
    base.update(kw)
    return Config(**base).validate()


# ---- flags ------------------------------------------------------------------------------------------------------------------
def test_defaults_are_pointer_py_and_off():
    c = Config()
    assert c.cache_window == 0 and c.cache_theta == CACHE_THETA_DEFAULT == 0.6625523432485668
    assert c.cache_lambda == CACHE_LAMBDA_DEFAULT == 0.12785920428335693
    a = parse_args(["--cache_window", "500", "--cache_theta", "0.3", "--cache_lambda", "0.1"], standalone=True)
    assert (a.cache_window, a.cache_theta, a.cache_lambda) == (500, 0.3, 0.1)
    with warnings.catch_warnings():
        warnings.simplefilter("error")
        _cfg()
        _cfg(cache_window=8)
        Config().validate()


@pytest.mark.parametrize("kw,names", [
    (dict(cache_window=-1), ["--cache_window"]),
    (dict(cache_window=8, cache_theta=-0.5), ["--cache_theta"]),
    (dict(cache_window=8, cache_theta=float("inf")), ["--cache_theta"]),
    (dict(cache_window=8, cache_theta=float("nan")), ["--cache_theta"]),
    (dict(cache_window=8, cache_lambda=1.0), ["--cache_lambda"]),
    (dict(cache_window=8, cache_lambda=-0.1), ["--cache_lambda"]),
    (dict(cache_window=8, stateful=False), ["--cache_window", "--next_token --stateful"]),
    (dict(cache_window=8, stateful=False, next_token=False, per_step_labels=True), ["--cache_window", "--next_token --stateful"]),
])
def test_refusals_name_their_flags(kw, names):
    with pytest.raises(ValueError) as e:
        _cfg(**kw)
    for n in names:
        assert n in str(e.value)


@pytest.mark.parametrize("kw,names", [
    (dict(mode="train", cache_window=8), ["--cache_window 8", "--mode train"]),
    (dict(mode="generate", cache_window=8), ["--cache_window 8", "--mode generate"]),
    (dict(mode="train", cache_lambda=0.2), ["--cache_lambda 0.2", "--mode train"]),
    (dict(cache_theta=0.3), ["--cache_theta 0.3", "--cache_window"]),
    (dict(cache_lambda=0.2), ["--cache_lambda 0.2", "--cache_window"]),
])
def test_warnings_name_their_flags(kw, names):
    with pytest.warns(UserWarning) as w:
        _cfg(**kw)
    msg = " ".join(str(x.message) for x in w)
    for n in names:
        assert n in msg


# ---- the definition -----------------------------------------------------------------------------------------------------------
def naive(h, y, lv, W, theta, lam):
    """The formula one query at a time: ``h [B,L,H]``, ``y [B,L]``, ``lv [B,L]`` -> log p ``[B,L]`` (fp64)."""
    B, L, _ = h.shape
    out = torch.empty(B, L, dtype=torch.float64)
    for b in range(B):
        for p in range(L):
            J = list(range(max(0, p - W), p))
            if not J:
                out[b, p] = lv[b, p]
                continue
            s = theta * (h[b, J] @ h[b, p])
            m = s.max()
            e = torch.exp(s - m)
            Z = e.sum()
            M = e[y[b, J] == y[b, p]].sum()
            a = math.log1p(-lam) + float(lv[b, p])
            c = math.log(lam) + math.log(M) - math.log(Z) if (lam > 0 and M > 0) else -math.inf
            out[b, p] = a if c == -math.inf else max(a, c) + math.log1p(math.exp(min(a, c) - max(a, c)))
    return out


def stream_scores(h, y, lv, W, theta, lam, T):
    """Score the streams through ``F.cache_pointer`` in segments of T (the last one a tail) -> (log p ``[B,L]``, sums)."""
    B, L, H = h.shape
    hist = F.CacheHistory(W, theta, lam, B, T, H, h.dtype, "cpu")
    out = torch.empty(B, L, dtype=h.dtype)
    sums = torch.zeros(2, dtype=h.dtype)
    for t0 in range(0, L, T):
        n = min(T, L - t0)
        hs = torch.zeros(T, B, H, dtype=h.dtype)
        hs[:n] = h[:, t0:t0 + n].transpose(0, 1)
        ys = torch.zeros(B, T, dtype=torch.int64)
        ys[:, :n] = y[:, t0:t0 + n]
        ls = torch.zeros(T, B, dtype=h.dtype)
        ls[:n] = lv[:, t0:t0 + n].t()
        lengths = torch.full((B,), n, dtype=torch.int32) if n < T else None
        lp, s = F.cache_pointer(hs, ys, ls.reshape(-1), hist, lengths)
        out[:, t0:t0 + n] = lp.view(T, B)[:n].t()
        sums += s
    return out, sums


def _stream(B, L, H, V, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    h = (torch.rand(B, L, H, generator=g, dtype=torch.float64) * 2 - 1) * scale
    y = torch.randint(0, V, (B, L), generator=g)
    lv = torch.log(torch.rand(B, L, generator=g, dtype=torch.float64) * 0.9 + 0.05)
    return h, y, lv


@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("W,T", [(3, 5), (5, 5), (12, 5), (7, 16), (30, 4)])
def test_reference_matches_the_per_position_loop(B, W, T):
    """Several segments and a tail; W below, at and above the segment length; the first position has no history."""
    h, y, lv = _stream(B, 23, 6, 4, seed=W * 31 + T + B)
    want = naive(h, y, lv, W, 0.7, 0.3)
    got, sums = stream_scores(h, y, lv, W, 0.7, 0.3, T)
    torch.testing.assert_close(got, want, rtol=1e-12, atol=1e-12)
    assert torch.equal(got[:, 0], lv[:, 0])                        # empty history: the model alone
    assert float(sums[0]) == pytest.approx(-float(want.sum()), rel=1e-12)
    assert float(sums[1]) == pytest.approx(-float(lv.sum()), rel=1e-12)


def test_absent_target_all_equal_labels_theta_zero_and_saturation():
    B, L, H, W = 2, 19, 5, 6
    h, y, lv = _stream(B, L, H, 50, seed=3)
    # M = 0: every label distinct, so no earlier position shares the target: log p = log1p(-lam) + log p_v after the first
    yd = torch.arange(B * L).view(B, L)
    got, _ = stream_scores(h, yd, lv, W, 0.7, 0.3, 4)
    torch.testing.assert_close(got[:, 1:], lv[:, 1:] + math.log1p(-0.3), rtol=1e-13, atol=1e-13)
    torch.testing.assert_close(got, naive(h, yd, lv, W, 0.7, 0.3), rtol=1e-12, atol=1e-12)
    # M = Z: one label everywhere, log p = logaddexp(log1p(-lam) + log p_v, log lam)
    y1 = torch.zeros(B, L, dtype=torch.int64)
    got, _ = stream_scores(h, y1, lv, W, 0.7, 0.3, 4)
    torch.testing.assert_close(got[:, 1:], torch.logaddexp(lv[:, 1:] + math.log1p(-0.3), torch.tensor(math.log(0.3), dtype=torch.float64)),
                               rtol=1e-13, atol=1e-13)
    # theta = 0: uniform over the window, p_cache(y) = (count of y in the window) / |J|
    got, _ = stream_scores(h, y, lv, W, 0.0, 0.5, 4)
    for b in range(B):
        for p in range(1, L):
            J = range(max(0, p - W), p)
            share = sum(int(y[b, j] == y[b, p]) for j in J) / len(J)
            want = math.log(0.5 * math.exp(float(lv[b, p])) + 0.5 * share)
            assert float(got[b, p]) == pytest.approx(want, rel=1e-12, abs=1e-12)
    # a large theta on large activations: scores of order 1e5 saturate the softmax without overflow
    hs, ys, lvs = _stream(B, L, H, 3, seed=4, scale=40.0)
    got, _ = stream_scores(hs, ys, lvs, W, 50.0, 0.3, 4)
    assert torch.isfinite(got).all()
    torch.testing.assert_close(got, naive(hs, ys, lvs, W, 50.0, 0.3), rtol=1e-12, atol=1e-12)


def test_segment_length_does_not_matter():
    h, y, lv = _stream(3, 61, 7, 5, seed=11)
    a, _ = stream_scores(h, y, lv, 20, 0.66, 0.13, 5)
    b, _ = stream_scores(h, y, lv, 20, 0.66, 0.13, 16)
    torch.testing.assert_close(a, b, rtol=1e-14, atol=1e-14)


def test_lambda_zero_gives_the_model_loss_exactly():
    h, y, lv = _stream(3, 30, 4, 3, seed=5)
    for dt in (torch.float64, torch.float32):
        got, sums = stream_scores(h.to(dt), y, lv.to(dt), 9, 0.66, 0.0, 7)
        assert torch.equal(got, lv.to(dt))
        assert float(sums[0]) == float(sums[1])


def test_the_ring_holds_window_plus_segment_in_whole_key_tiles():
    hist = F.CacheHistory(3785, 0.6, 0.1, 2, 128, 8, torch.float32, "cpu")
    assert hist.keys.shape == (2, 3968, 8) and hist.key_labels.shape == (2, 3968) and 3968 % F.CACHE_KEY_TILE == 0
    with pytest.raises(ValueError, match="at most 128"):
        hist.append(torch.zeros(129, 2, 8), torch.zeros(2, 129, dtype=torch.int64))
    assert ref.cache_ring_positions(4, 6).tolist() == [4, 5, 2, 3]
    assert ref.cache_ring_positions(4, 2).tolist() == [0, 1, -1, -1]


# ---- --mode eval end to end ------------------------------------------------------------------------------------------------
def _run_cfg(tmp_path, name, **kw):
    base = dict(next_token=True, stateful=True, vocab_size=32, seq_len=6, batch_size=4, hidden_units="8,8", in_features=6,
                synthetic=30, device="cpu", quiet=True, init="scaled", learning_rate=1e-2, dropout=0.0,
                checkpoint_path=str(tmp_path / name), output_path=str(tmp_path / (name + "_out")))
    base.update(kw)
    return Config(**base).validate()


@pytest.mark.parametrize("tie", [False, True])
def test_stream_eval_with_the_cache_end_to_end(tmp_path, tie):
    from lstm_tensorspark_b200.trainer import run_job
    kw = dict(tie_embeddings=True, in_features=8) if tie else {}
    run_job(_run_cfg(tmp_path, "c", epochs=1, max_steps=3, **kw), standalone=True)
    plain = run_job(_run_cfg(tmp_path, "c", mode="eval", json_log=str(tmp_path / "a.jsonl"), **kw), standalone=True)
    cached = run_job(_run_cfg(tmp_path, "c", mode="eval", cache_window=10, json_log=str(tmp_path / "b.jsonl"), **kw),
                     standalone=True)
    assert set(plain) == {"mode", "model", "stream", "streams", "positions", "loss", "accuracy", "seconds", "weights", "perplexity"}
    assert cached["positions"] == plain["positions"] and cached["accuracy"] == plain["accuracy"]
    assert cached["loss_model"] == pytest.approx(plain["loss"], rel=1e-6)
    assert cached["perplexity"] == pytest.approx(math.exp(cached["loss"]))
    assert cached["perplexity_model"] == pytest.approx(math.exp(cached["loss_model"]))
    assert (cached["cache_window"], cached["cache_theta"], cached["cache_lambda"]) == (10, CACHE_THETA_DEFAULT, CACHE_LAMBDA_DEFAULT)
    assert cached["loss"] != cached["loss_model"]
    logged = json.loads(open(tmp_path / "b.jsonl").read().splitlines()[-1])
    for k in ("loss", "loss_model", "perplexity_model", "cache_window", "cache_theta", "cache_lambda"):
        assert k in logged
    assert "loss_model" not in json.loads(open(tmp_path / "a.jsonl").read().splitlines()[-1])
    zero = run_job(_run_cfg(tmp_path, "c", mode="eval", cache_window=10, cache_lambda=0.0, **kw), standalone=True)
    assert zero["loss"] == zero["loss_model"]
