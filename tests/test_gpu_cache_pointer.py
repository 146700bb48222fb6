"""The continuous cache pointer's kernels (csrc/cache_pointer.cu) against the fp64 reference (``ops.reference.cache_pointer``) fed
the same stored h and the same log p_model, the model's log-probability at the label against fp64 log_softmax, bitwise
repeatability, and ``--mode eval --stateful --cache_window`` on the GPU against the CPU.

Error budget of one position (derived, not tuned).  The kernels form s_j = theta (h_p . h_j) from the stored operands with fp32
accumulation over H products; the products of bf16 values are exact in fp32, so the dot is off by at most gamma_H A_pj, with
A_pj = sum_k |h_pk h_jk| and gamma_n = n u / (1 - n u).  u is taken as 2^-23, twice the unit roundoff, because the tensor cores'
fp32 adder is not documented to round to nearest.  Scaling by theta log2(e) adds 2 u |s|.  log-sum-exp is 1-Lipschitz in the max
norm, so log M - log Z moves by at most 2 theta max_j A_pj (gamma_H + 2u).  Z and M are fp32 sums of at most W + 1 terms <= 1
(relative gamma_{W+1}), each made by ex2.approx (relative 2^-22) and rescaled once per merge of running sums (at most W / 64 + 16
merges, relative 2^-22 each): twice that relative error bounds their log ratio.  The final logs, exp and log1p (lg2.approx,
ex2.approx: absolute 2^-21 each, five of them) add 5 2^-21, and rounding the result to fp32 |log p| 2^-23.  The mixture's
logaddexp is 1-Lipschitz in the cache term, so the sum of these bounds |log p_kernel - log p_fp64|."""
import math

import pytest
import torch

from lstm_tensorspark_b200.ops import functional as F
from lstm_tensorspark_b200.ops import reference as ref

pytestmark = pytest.mark.gpu
DEV = "cuda"
U = 2.0 ** -23


def gamma(n):
    return n * U / (1 - n * U)


def _stream(B, L, H, V, seed, dtype=torch.bfloat16, scale=1.0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    h = ((torch.rand(B, L, H, generator=g, device=DEV) * 2 - 1) * scale).to(dtype)
    y = torch.randint(0, V, (B, L), generator=g, device=DEV)
    lv = torch.log(torch.rand(B, L, generator=g, device=DEV) * 0.9 + 0.05)
    return h, y, lv


def run(h, y, lv, W, theta, lam, T, check=True):
    """Score the streams in segments of T (the last one a tail) with the kernels and, with ``check``, the fp64 reference on an
    fp64 copy of the same ring -> (log p kernel ``[B,L]``, log p fp64, bound, kernel sums, fp64 sums)."""
    B, L, H = h.shape
    hist = F.CacheHistory(W, theta, lam, B, T, H, h.dtype, DEV)
    keys = torch.zeros(B, hist.keys.shape[1], H, dtype=torch.float64, device=DEV)
    klab = torch.zeros(B, hist.keys.shape[1], dtype=torch.int64, device=DEV)
    got = torch.empty(B, L, device=DEV)
    want = torch.empty(B, L, dtype=torch.float64, device=DEV)
    bound = torch.empty(B, L, dtype=torch.float64, device=DEV)
    sums = torch.zeros(2, dtype=torch.float64, device=DEV)
    sums64 = torch.zeros(2, dtype=torch.float64, device=DEV)
    nmerge = W / 64 + 16
    for t0 in range(0, L, T):
        n = min(T, L - t0)
        hs = torch.zeros(T, B, H, dtype=h.dtype, device=DEV)
        hs[:n] = h[:, t0:t0 + n].transpose(0, 1)
        ys = torch.zeros(B, T, dtype=torch.int64, device=DEV)
        ys[:, :n] = y[:, t0:t0 + n]
        ls = torch.zeros(T, B, device=DEV)
        ls[:n] = lv[:, t0:t0 + n].t()
        lengths = torch.full((B,), n, dtype=torch.int32, device=DEV) if n < T else None
        seen = hist.seen
        lp, s = F.cache_pointer(hs, ys, ls.reshape(-1), hist, lengths)
        got[:, t0:t0 + n] = lp.view(T, B)[:n].t()
        sums += s.double()
        if not check:
            continue
        slots = (seen + torch.arange(T, device=DEV)) % keys.shape[1]
        keys[:, slots] = hs.double().transpose(0, 1)
        klab[:, slots] = ys
        assert torch.equal(hist.keys.double(), keys) and torch.equal(hist.key_labels.long(), klab)     # the append kernel
        lp64, keep = ref.cache_pointer(hs.double(), ys, ls.double().reshape(-1), keys, klab, seen, W, theta, lam, lengths)
        want[:, t0:t0 + n] = lp64.view(T, B)[:n].t()
        sums64 += torch.stack([-(lp64[keep]).sum(), -(ls.double().reshape(-1)[keep]).sum()])
        # max_j A_pj over J(p)
        pos = ref.cache_ring_positions(keys.shape[1], seen + T, DEV)
        p = seen + torch.arange(T, device=DEV)
        valid = (pos.view(1, -1) >= (p.view(-1, 1) - W).clamp(min=0)) & (pos.view(1, -1) < p.view(-1, 1))
        A = torch.einsum("tbh,bch->btc", hs.double().abs(), keys.abs()).masked_fill(~valid.unsqueeze(0), 0).amax(2)   # [B,T]
        b = (2 * theta * A * (gamma(H) + 2 * U) + 2 * (gamma(W + 1) + nmerge * 2.0 ** -22) + 5 * 2.0 ** -21
             + lp64.view(T, B).t().abs() * U)
        bound[:, t0:t0 + n] = b[:, :n]
    return got, want, bound, sums, sums64


def _check(got, want, bound):
    err = (got.double() - want).abs()
    worst = float((err - bound).max())
    assert worst <= 0, f"error above the bound by {worst:.3g} (max error {float(err.max()):.3g})"


TC_CASES = [
    # H, B, T, W, L (L > T: several segments and a tail unless L % T == 0)
    (64, 1, 1, 1, 7),
    (64, 7, 63, 63, 200),
    (64, 7, 64, 64, 256),
    (512, 7, 64, 100, 330),          # ring of 256 slots: wrapped
    (512, 1, 128, 500, 300),         # partly full history
    (1024, 1, 128, 3785, 520),
    (1024, 7, 200, 500, 900),
    (512, 256, 128, 2048, 256),
    (1024, 16, 128, 3785, 384),
    (1024, 256, 64, 64, 192),
]


@pytest.mark.parametrize("H,B,T,W,L", TC_CASES)
def test_tensor_core_path_against_fp64(H, B, T, W, L):
    from lstm_tensorspark_b200.ops import cuda_cache
    h, y, lv = _stream(B, L, H, 37, seed=H + B + T + W)
    assert cuda_cache.tc_supported(h.transpose(0, 1))
    got, want, bound, sums, sums64 = run(h, y, lv, W, 0.6625523432485668, 0.12785920428335693, T)
    _check(got, want, bound)
    assert float(sums[0]) == pytest.approx(float(sums64[0]), rel=1e-4)


@pytest.mark.parametrize("lam", [0.0, 0.1279, 0.9])
def test_absent_targets_one_label_and_saturated_scores(lam):
    B, L, H, W, T = 3, 300, 128, 100, 64
    h, y, lv = _stream(B, L, H, 5, seed=1)
    yd = torch.arange(B * L, device=DEV).view(B, L)                # M = 0
    got, want, bound, _, _ = run(h, yd, lv, W, 0.66, lam, T)
    _check(got, want, bound)
    torch.testing.assert_close(got[:, 1:].double(), lv[:, 1:].double() + math.log1p(-lam), rtol=0, atol=4 * 2.0 ** -21)
    y1 = torch.zeros(B, L, dtype=torch.int64, device=DEV)          # M = Z
    got, want, bound, _, _ = run(h, y1, lv, W, 0.66, lam, T)
    _check(got, want, bound)
    hs, ys, lvs = _stream(B, L, H, 4, seed=2, scale=8.0)           # theta large: scores of order 1e4
    got, want, bound, _, _ = run(hs, ys, lvs, W, 40.0, lam, T)
    assert torch.isfinite(got).all()
    _check(got, want, bound)


# rows of 16-byte multiples, and rows the ring append copies in 4-byte (fp32 H = 30, bf16 H = 650) and 2-byte (bf16 H = 75) words
@pytest.mark.parametrize("dtype,H", [(torch.float32, 64), (torch.float32, 400), (torch.bfloat16, 400), (torch.bfloat16, 72),
                                     (torch.float32, 30), (torch.bfloat16, 650), (torch.bfloat16, 75)])
def test_generic_path_against_fp64(dtype, H):
    from lstm_tensorspark_b200.ops import cuda_cache
    B, L, T, W = 5, 260, 70, 150
    h, y, lv = _stream(B, L, H, 23, seed=H, dtype=dtype)
    assert not cuda_cache.tc_supported(h.transpose(0, 1))
    before = F.get_backend()
    got, want, bound, sums, sums64 = run(h, y, lv, W, 0.66, 0.3, T)
    assert F.get_backend() == before
    _check(got, want, bound)


def test_two_calls_give_the_same_bits_and_lambda_zero_the_model_loss():
    h, y, lv = _stream(4, 400, 256, 30, seed=9)
    a = run(h, y, lv, 300, 0.66, 0.13, 128, check=False)
    b = run(h, y, lv, 300, 0.66, 0.13, 128, check=False)
    assert torch.equal(a[0], b[0]) and torch.equal(a[3], b[3])
    for dtype, H in ((torch.bfloat16, 256), (torch.float32, 40)):
        h, y, lv = _stream(4, 200, H, 30, seed=10, dtype=dtype)
        got, _, _, sums, _ = run(h, y, lv, 90, 0.66, 0.0, 64, check=False)
        assert torch.equal(got, lv)
        assert float(sums[0]) == float(sums[1])


# ---- log p_model(y) --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("tied", [False, True])
def test_label_logprob_of_the_vocab_head_against_fp64(tied):
    T, B, H, C = 16, 24, 128, 1000
    g = torch.Generator(device=DEV).manual_seed(3)
    h = (torch.rand(T, B, H, generator=g, device=DEV) * 2 - 1).bfloat16()
    w = torch.randn(C, H, generator=g, device=DEV) * 0.2 if tied else torch.randn(H, C, generator=g, device=DEV) * 0.2
    bias = torch.randn(C, generator=g, device=DEV)
    y = torch.randint(0, C, (B, T), generator=g, device=DEV)
    assert F.vocab_head_supported(h, C)
    _loss, _ok, n, lp = F.vocab_xent_logprob(h, w, bias, y, None, class_major=tied)
    w64 = w.bfloat16().double()
    W = w64.t() if tied else w64
    logits = torch.einsum("tbh,hc->btc", h.double(), W) + bias.double()
    want = ref.label_logprob(logits, y)
    # the logits: fp32 accumulation over H bf16 products plus the bias; lse moves by at most the largest logit error
    A = torch.einsum("tbh,hc->btc", h.double().abs(), W.abs()).amax(2).t().reshape(-1)
    bound = 2 * (A * gamma(H + 1) + logits.abs().amax(2).t().reshape(-1) * U) + gamma(C) + 4 * 2.0 ** -21 + want.abs() * U
    assert int(n) == T * B
    assert float(((lp.double() - want).abs() - bound).max()) <= 0


def test_label_logprob_of_stored_logits_against_fp64():
    B, T, C = 6, 9, 300
    g = torch.Generator(device=DEV).manual_seed(4)
    logits = torch.randn(B, T, C, generator=g, device=DEV) * 4
    y = torch.randint(0, C, (B, T), generator=g, device=DEV)
    from lstm_tensorspark_b200.ops import cuda_cache
    lp = cuda_cache.label_logprob_logits(logits, y)
    want = ref.label_logprob(logits.double(), y)
    bound = gamma(C) + 4 * 2.0 ** -21 + (want.abs() + logits.abs().amax(2).t().reshape(-1).double()) * U
    assert float(((lp.double() - want).abs() - bound).max()) <= 0


# ---- end to end ------------------------------------------------------------------------------------------------------------
def _run_cfg(tmp_path, name, **kw):
    from lstm_tensorspark_b200.config import Config
    base = dict(next_token=True, stateful=True, vocab_size=512, seq_len=16, batch_size=64, hidden_units="128,128",
                in_features=64, synthetic=300, device="cuda", quiet=True, init="scaled", learning_rate=1e-3, dropout=0.1,
                deterministic=True, checkpoint_path=str(tmp_path / name), output_path=str(tmp_path / (name + "_out")))
    base.update(kw)
    return Config(**base).validate()


def test_stream_eval_with_the_cache_on_the_gpu_against_the_cpu_reference(tmp_path):
    """The same trained model scored with the cache on the GPU (bf16 kernels) and on the CPU (fp32 reference): the same
    positions, and losses within the 1 % of the stream evaluation's own GPU-CPU test."""
    from lstm_tensorspark_b200.ops.cuda_ext import STATS
    from lstm_tensorspark_b200.trainer import run_job
    run_job(_run_cfg(tmp_path, "e", epochs=1, max_steps=6, dropout=0.0), standalone=True)
    before = STATS.get("cache_pointer_tc", 0)
    gpu = run_job(_run_cfg(tmp_path, "e", mode="eval", synthetic=301, cache_window=200), standalone=True)
    assert STATS.get("cache_pointer_tc", 0) > before
    cpu = run_job(_run_cfg(tmp_path, "e", mode="eval", synthetic=301, cache_window=200, device="cpu", deterministic=False),
                  standalone=True)
    plain = run_job(_run_cfg(tmp_path, "e", mode="eval", synthetic=301), standalone=True)
    assert gpu["positions"] == cpu["positions"] == plain["positions"]
    assert gpu["loss"] == pytest.approx(cpu["loss"], rel=1e-2)
    assert gpu["loss_model"] == pytest.approx(cpu["loss_model"], rel=1e-2)
    assert gpu["loss_model"] == pytest.approx(plain["loss"], rel=1e-5)
    assert math.isfinite(gpu["perplexity"]) and gpu["accuracy"] == plain["accuracy"]
