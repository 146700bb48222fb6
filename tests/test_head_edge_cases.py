"""The designed cases of tests/head_edges.py on the CPU: the premises the GPU tests rest on (exact logits, the claimed ties, gaps,
padding and bounds), the dispatch rules the GPU tests mirror, and negative controls: torch models of kernels with a reversed tie
rule, padded classes let in as logit 0, a dropped rescale or gradients at uncounted rows must fail the GPU tests' assertions."""
import math

import pytest
import torch

import head_edges as E
import lstm_numerics as N
from test_gpu_head_edges import SAMPLE, SMALL, STEP_ROWS, VOCAB

SHAPES = [(C, H, T, B) for C, H, T, B in [(2, 64, 3, 43), (16, 64, 1, 200), (17, 64, 3, 43), (33, 1024, 2, 9), (65, 64, 3, 43),
                                          (129, 64, 2, 40), (257, 64, 3, 43), (520, 64, 3, 43), (640, 96, 2, 30),
                                          (4104, 64, 1, 40), (8200, 64, 1, 40)]]


def _cases():
    for C, H, T, B in SHAPES:
        for regime in E.REGIMES:
            if regime == "spread" and C < 15:
                continue
            yield pytest.param(regime, C, H, T, B, id=f"{regime}-C{C}-H{H}-T{T}-B{B}")


@pytest.mark.parametrize("regime,C,H,T,B", list(_cases()))
def test_logits_are_exact(regime, C, H, T, B):
    """h and W are exact in bf16, every partial sum is below 2^24, and fp32 logits equal the fp64 logits bit for bit."""
    c = E.make_case(regime, T, B, H, C)
    h, W = c.h.reshape(T * B, H), c.W
    assert torch.equal(h.bfloat16().double(), h) and torch.equal(W.bfloat16().double(), W)
    assert int(h.abs().max()) <= 2 and int(W.abs().max()) <= 4
    assert torch.equal(c.bias.float().double(), c.bias)
    assert float((h.abs() @ W.abs() + c.bias.abs()).max()) < 2 ** 24
    assert torch.equal((h @ W + c.bias).view(T, B, C), c.logits)
    l32 = (h.float() @ W.float() + c.bias.float()).view(T, B, C)
    assert torch.equal(l32.double(), c.logits)
    assert bool((c.logits.float().double() == c.logits).all())


@pytest.mark.parametrize("regime,C,H,T,B", list(_cases()))
def test_claimed_properties(regime, C, H, T, B):
    c = E.make_case(regime, T, B, H, C)
    l, keep = c.logits, c.keep
    top = l.amax(2)
    first = E.first_argmax(l)
    lead = E.lead(c)
    for p, k in enumerate(c.kinds):
        rows = c.kind_of == p
        assert bool(rows.any()), k.name
        lk = l[rows]
        assert bool((lk == lk[:1]).all()), k.name                              # every row of a kind has the same logits
        row = lk[0]
        if k.name.startswith("tie"):
            a, b = k.pair
            assert row[a] == row[b] == row.max() and int((row == row.max()).sum()) == 2, k.name
            assert bool((first[rows] == a).all()) and set(k.labels) == {a, b}
            if regime == "ties":
                assert bool((lead[rows] >= 14).all()), k.name
        elif k.name.startswith("near"):
            a, b = k.pair
            x = row[a].float()
            assert row[b] == torch.nextafter(x, torch.tensor(math.inf)).double() and row[b] == row.max(), k.name
            assert int((row == row.max()).sum()) == 1 and row[b] - row[a] == E.NEG_ULP and b > a
            assert bool((first[rows] == b).all()) and k.labels[0] == b
        elif k.name == "const":
            assert bool((row == row[0]).all()) and bool((first[rows] == 0).all())
        elif k.name.startswith("max"):
            m = k.labels[0]
            assert int((row == row.max()).sum()) == 1 and row[m] == row.max()
            assert 0 in k.labels and C - 1 in k.labels
            last0 = E.TILE * ((C - 1) // E.TILE)
            assert any(last0 <= y < C for y in k.labels)
            if regime == "ties":
                assert bool((lead[rows] >= 14).all()), k.name
        elif k.name.startswith("spread"):
            assert float(row.max()) == E.SPREAD + 8 and float(row[k.labels[0]]) <= -E.SPREAD + 4
            assert int(row.argmax()) == (C - 3 if k.name == "spread max last" else 2)     # the last class tile, or tile 0
            nll = torch.logsumexp(row, 0) - row[k.labels[0]]
            assert 3990 < float(nll) < 4020
            assert bool((lead[rows] >= 16).all())
    if regime == "negative":
        assert bool((l < 0).all()) and float(top.max()) <= -990 + E.NEG_ULP
    # labels: in range where counted, never read elsewhere; uncounted rows exist when there are lengths
    lab = c.labels.t()
    assert bool(((lab[keep] >= 0) & (lab[keep] < C)).all()) and bool((lab[~keep] == E.UNREAD).all())
    assert bool((c.lengths == 0).any()) and bool((~keep).any()) and bool(keep.any())
    if T > 1:
        assert bool(((c.lengths > 0) & (c.lengths < T)).any()) or B < 3
    if regime != "spread":
        assert bool((c.lab[keep] == 0).any()) and bool((c.lab[keep] == C - 1).any())


def test_small_head_dispatch_rules():
    """The rules of ts_head_fwd_tc, ts_head_step_fwd, launch_bwd and launch_step_bwd (head_wgmma.cu) the GPU tests mirror, and
    the GPU shapes reach every instantiation."""
    bf, f32 = torch.bfloat16, torch.float32
    assert E.small_head_path(bf, 1024, 64, True) == (64, None) and E.small_head_path(bf, 1024, 65, True) == (None, None)
    assert E.small_head_path(bf, 64, 257, False) == (None, None) and E.small_head_path(f32, 64, 16, True) == (None, 16)
    assert E.small_head_path(bf, 64, 2, True) == (16, 8) and E.small_head_path(bf, 64, 17, False) == (32, 32)
    nps, cps = set(), set()
    for C, H, dtype in SMALL:
        for per_step in (False, True):
            np_, cp = E.small_head_path(dtype, H, C, per_step)
            nps.add(np_)
            cps.add(cp)
    assert nps == {16, 32, 64, 128, 256, None} and cps == {8, 16, 32, None}
    slabs = set()
    for C, H, T, B, dtype in STEP_ROWS:
        cp = E.small_head_path(dtype, H, C, True)[1]
        rpb = E.STEP_BWD_ROWS[cp]
        slabs.add((cp, (T * B) % rpb in (0, 1, rpb - 1)))
    assert {(8, True), (16, True), (32, True)} <= slabs


def test_gpu_shapes_reach_every_edge():
    Cs, Hs, Rs = {v[0] for v in VOCAB}, {v[1] for v in VOCAB}, {v[2] * v[3] for v in VOCAB}
    assert Cs == {512, 520, 640, 4104, 8200} and Hs == {64, 1024, 4096}
    assert Rs == {1, 127, 129, 255, 257, 4095, 4096, 4097, 8193}
    assert {C % E.TILE for C in Cs} >= {0, 8, 128}
    fallback = {(dtype, C < 512, H % 64 != 0) for C, H, dtype, _ in SAMPLE}
    assert {(torch.float32, False, False), (torch.bfloat16, True, False), (torch.bfloat16, False, True)} <= fallback
    assert any(t for *_, t in SAMPLE) and any(C >= 8200 for C, *_ in SAMPLE)


# ---- negative controls ----------------------------------------------------------------------------------------------------------
def _vocab_case(regime, C=520, T=3, B=43):
    return E.make_case(regime, T, B, 64, C)


def _passes(c, sim):
    E.assert_counts(c, sim["correct"], sim["n"])
    return E.check_head("sim", c, sim, 0.37, vocab=True, floor=N.FLOOR)


@pytest.mark.parametrize("regime,C", [("ties", 520), ("ties", 8200), ("negative", 520), ("negative", 4104), ("spread", 520),
                                      ("spread", 8200)])
def test_the_faithful_model_passes(regime, C):
    c = _vocab_case(regime, C, T=1 if C > 4096 else 3, B=40 if C > 4096 else 43)
    assert _passes(c, E.simulate(c, 0.37)) <= 1.0
    if regime != "spread":
        c1 = E.make_case(regime, 1, 40, 64, C, lengths=False)
        assert E.assert_tokens(c1, E.simulate(c1)["tokens"][0], 0.0) == 40


@pytest.mark.parametrize("C", [520, 8200])
def test_control_last_index_on_a_tie_fails(C):
    c = _vocab_case("ties", C, T=1, B=40)
    sim = E.simulate(c, 0.37, tie="last")
    with pytest.raises(AssertionError, match="correct"):
        E.assert_counts(c, sim["correct"], sim["n"])
    c1 = E.make_case("ties", 1, 40, 64, C, lengths=False)
    with pytest.raises(AssertionError, match="greedy"):
        E.assert_tokens(c1, E.simulate(c1, tie="last")["tokens"][0], 0.0)


@pytest.mark.parametrize("C", [520, 640, 4104])
def test_control_padded_classes_as_zero_fail(C):
    c = _vocab_case("negative", C, T=1 if C > 4096 else 3, B=40 if C > 4096 else 43)
    sim = E.simulate(c, 0.37, pad=0.0)
    with pytest.raises(AssertionError):
        E.assert_counts(c, sim["correct"], sim["n"])
    with pytest.raises(AssertionError):
        E.check_head("pad 0", c, sim, 0.37, vocab=True, floor=N.FLOOR)
    c1 = E.make_case("negative", 1, 40, 64, C, lengths=False)
    with pytest.raises(AssertionError, match="outside"):                     # the token is a padded class
        E.assert_tokens(c1, E.simulate(c1, pad=0.0)["tokens"][0], 0.0)


@pytest.mark.parametrize("C", [520, 8200])
def test_control_dropped_rescale_fails(C):
    c = _vocab_case("spread", C, T=1 if C > 4096 else 3, B=40 if C > 4096 else 43)
    sim = E.simulate(c, 0.37, rescale=False)
    E.assert_counts(c, sim["correct"], sim["n"])                              # the arg-max does not see it ...
    with pytest.raises(AssertionError):                                       # ... the sums do
        E.check_head("no rescale", c, sim, 0.37, vocab=True, floor=N.FLOOR)


@pytest.mark.parametrize("regime", E.REGIMES)
def test_control_gradients_at_uncounted_rows_fail(regime):
    c = _vocab_case(regime)
    sim = E.simulate(c, 0.37, mask=False)
    with pytest.raises(AssertionError):
        E.check_head("unmasked", c, sim, 0.37, vocab=True, floor=N.FLOOR)
