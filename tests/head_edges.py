"""Designed inputs for the softmax heads and the sampling kernels, and the assertions that hold the kernels to them.

Every case has exact logits.  h takes integers in [-2, 2] and W integers in [-4, 4], so both are exact in bf16 (rounding W to
bf16 for the tensor cores changes nothing and every path sees the same W); the bias is an integer or a dyadic fraction, and
every partial sum stays far below 2^24.  So the fp32 logits of any kernel equal the fp64 logits bit for bit, whatever its
summation order, and fp64 ``log_softmax`` of those logits is the exact reference.

A case is built from row kinds, each a logit template ``S [C]`` added to the case's bias.  Template p lives in its own group of
dimensions of h (k = p mod P): a row of kind p has h = 1 on its group and 0 on the other groups, and W on the group holds S on
four dimensions spread over H plus zero-sum noise pairs, so the contraction runs over every k-block.  Dimensions past the groups
carry random h in [-2, 2] against W = 0.

Kinds, and the code each one puts under pressure (kernels of head_vocab.cu, head_wgmma.cu and head_xent.cu, by name):
  tie pair (c, c+1), tie thread (c, c+8)
      the arg-max inside one thread: ascending columns with a strict ``>`` (vocab_head_gemm_kernel's kFwd and kSample
      epilogues), ``l > mx || (l == mx && c < arg)`` (head_fwd_tc_kernel, head_step_fwd_tc_kernel); in
      vocab_sample_logits_kernel the pair sits in one lane.
  tie quad (c, c+2)
      the lane-quad shuffle merge of the same epilogues (sample_take in kSample).
  tie warp (c, c+32)
      the lane-strided loop and the warp tree of the generic softmax (xent_steps_kernel, xent_rows_kernel).
  tie tile (c, c+256)
      two class tiles of the vocabulary head: the per-lane merge keeps the earlier tile on an equal max
      (vocab_head_combine_kernel, vocab_sample_combine_kernel).
  tie tree (tile nt-2, the last tile)
      adjacent tiles sit on adjacent combine lanes and meet in the tree merge of the same two combine kernels.
  tie lane (tile 0, tile 32), C >= 8200
      one combine lane merges tiles i and i + 32 in order.
  tie edge (C-9, C-1)
      a tie inside the last (padded) class group.
  near pair / quad / tile / lane
      two logits one fp32 ulp apart, the larger at the higher class: a merge that compares anything but the exact fp32 values
      picks the wrong one.  (The bias of the higher class carries the ulp.)  Labels cycle (higher, lower, higher): with C = 2
      a near pair is the only kind of the negative regime, and balanced labels would make every dW and db column cancel to
      about 1e-3 of its terms, where the relative budget measures nothing but the order of the sums.
  max first / mid / last
      a unique maximum with a lead of at least 14 (the sampling kernels' Gumbel noise cannot move it at t = 0.5), with labels at
      0, at C - 1 and inside the real part of a partial last tile (the label logit of vocab_head_gemm_kernel's kFwd epilogue,
      the ``c == y`` of the small heads' epilogues).
  const
      every logit equal: lse = l + log C, dlogits = (1/C - onehot) scale, arg-max 0.
  negative regime (bias about -1000, row max -990): a padded class must never become the max, the arg-max or part of the
      sum: padded classes become -inf in vocab_head_gemm_kernel's epilogue, the small heads' bias image is 0 for padded
      columns (head_fwd_tc_kernel, head_step_fwd_tc_kernel) and their epilogues guard every column with ``c < p.C``.
  spread regime (bias +-2000 at four classes): the max near +2000 in the last class tile with the rest of the row near 0, or
      in tile 0 with the -2000 classes later; labels at -2000 (NLL about 4000).  Partials merge with max-rescaled sums only
      here (the per-lane loops and the trees of vocab_head_combine_kernel and vocab_sample_combine_kernel).
Uncounted rows (length-0 rows and steps past a row's length) come from ``lengths`` (the ``counted`` rows of
vocab_head_gemm_kernel and head_step_fwd_tc_kernel, the length test of xent_steps_kernel); their labels are 10**6, which no
kernel may read.
"""
from __future__ import annotations

import dataclasses
import math
from typing import List, Optional, Tuple

import torch

import lstm_numerics as N

TILE = 256                     # classes per tile of the vocabulary head (csrc/head_vocab.cu BN)
UNREAD = 10 ** 6               # label at uncounted positions
TOP = 12                       # template value of the row max (ties, max kinds)
NEG_BIAS, NEG_TOP = -1000, 10  # negative regime: bias about -1000, max -990
NEG_ULP = 2.0 ** -14           # one fp32 ulp in [512, 1024)
SPREAD = 2000
REGIMES = ("ties", "negative", "spread")


@dataclasses.dataclass
class Kind:
    name: str
    values: torch.Tensor                 # [C] int64: the template added to the bias
    labels: Tuple[int, ...]              # label candidates, cycled over the rows of this kind
    pair: Optional[Tuple[int, int]] = None   # tie / near tie: (c1, c2), c1 < c2


@dataclasses.dataclass
class Case:
    name: str
    regime: str
    h: torch.Tensor                      # [T,B,H] fp64, integers
    W: torch.Tensor                      # [H,C] fp64, integers
    bias: torch.Tensor                   # [C] fp64
    labels: torch.Tensor                 # [B,T] int64, UNREAD at uncounted positions
    lengths: Optional[torch.Tensor]      # [B] int32 or None
    logits: torch.Tensor                 # [T,B,C] fp64: the exact logits
    kind_of: torch.Tensor                # [T,B] index into kinds
    kinds: List[Kind]

    @property
    def keep(self) -> torch.Tensor:      # [T,B] counted positions
        T, B = self.kind_of.shape
        k = N._keep(self.lengths, T, B, self.h.device)
        return torch.ones(T, B, dtype=torch.bool, device=self.h.device) if k is None else k.t()

    @property
    def lab(self) -> torch.Tensor:       # [T,B] labels, 0 at uncounted positions
        return torch.where(self.keep, self.labels.t(), 0)

    def describe(self) -> str:
        T, B, H = self.h.shape
        return f"{self.name} T={T} B={B} H={H} C={self.W.shape[1]}: " + ", ".join(k.name for k in self.kinds)


def _tie_pairs(C: int):
    nt = -(-C // TILE)
    last0 = TILE * (nt - 1)
    cand = [("tie pair", 4, 5), ("tie quad", 1, 3), ("tie thread", 2, 10), ("tie warp", 8, 40), ("tie tile", 6, 6 + TILE)]
    if nt >= 2:
        cand.append(("tie tree", TILE * (nt - 2) + 9, last0 + min(2, C - last0 - 1)))
    cand += [("tie lane", 7, 32 * TILE + 5), ("tie edge", C - 9, C - 1)]
    out, used = [], set()
    for name, a, b in cand:
        if 0 <= a < b < C and not ({a, b} & used):
            out.append((name, a, b))
            used |= {a, b}
    return out if out else [("tie pair", 0, 1)]


def _near_pairs(C: int):
    cand = [("near pair", 10, 11), ("near quad", 12, 14), ("near tile", 16, 16 + TILE), ("near lane", 17, 32 * TILE + 3)]
    out = [(n, a, b) for n, a, b in cand if b < C]
    return out if out else [("near pair", 0, 1)]


def _edge_labels(C: int, m: int):
    last0 = TILE * ((C - 1) // TILE)
    return tuple(dict.fromkeys((m, 0, C - 1, min(C - 1, last0 + (C - last0) // 2))))


def _kinds(regime: str, C: int, g: torch.Generator):
    """-> (bias [C] fp64, kinds).  Background values leave the row max a lead of 14 (ties), 2 (negative) or 16 (spread)."""
    def bg(lo, hi):
        return torch.randint(lo, hi + 1, (C,), generator=g)

    kinds = []
    if regime == "ties":
        bias = torch.randint(-2, 3, (C,), generator=g).double()
        special = set()
        for name, a, b in _tie_pairs(C):
            v = bg(-12, -4)
            v[a] = v[b] = TOP
            kinds.append(Kind(name, v, (a, b), (a, b)))
            special |= {a, b}
        for name, m in (("max first", 0), ("max mid", C // 2), ("max last", C - 1)):
            v = bg(-12, -4)
            v[m] = TOP
            kinds.append(Kind(name, v, _edge_labels(C, m)))
            special.add(m)
        bias[list(special)] = 0.0
        kinds.append(Kind("const", (5 - bias).long(), _edge_labels(C, C // 3)))
    elif regime == "negative":
        bias = NEG_BIAS + torch.randint(-2, 3, (C,), generator=g).double()
        near = _near_pairs(C)
        used = {c for _, a, b in near for c in (a, b)}
        tie = next(((n, a, b) for n, a, b in reversed(_tie_pairs(C)) if not ({a, b} & used)), None)
        for m in (0, C - 1):
            bias[m] = NEG_BIAS
        for name, a, b in near:
            v = bg(-10, 6)
            v[a] = v[b] = NEG_TOP
            kinds.append(Kind(name, v, (b, a, b), (a, b)))
            bias[a], bias[b] = NEG_BIAS, NEG_BIAS + NEG_ULP
        if tie is not None:
            name, a, b = tie
            v = bg(-10, 6)
            v[a] = v[b] = NEG_TOP
            kinds.append(Kind(name, v, (a, b), (a, b)))
            bias[a] = bias[b] = NEG_BIAS
        for name, m in (("max first", 0), ("max last", C - 1)):
            if m in used:
                continue
            v = bg(-10, 6)
            v[m] = NEG_TOP
            kinds.append(Kind(name, v, _edge_labels(C, m)))
    elif regime == "spread":
        assert C >= 15, "the spread regime needs four distinct classes"
        hi0, lo0, hi_l, lo_l = 2, 9, C - 3, C - 5
        bias = torch.randint(-2, 3, (C,), generator=g).double()
        bias[[hi0, hi_l]], bias[[lo0, lo_l]] = SPREAD, -SPREAD
        va, vb = bg(-4, 4), bg(-4, 4)
        va[hi_l], va[hi0], vb[hi0], vb[hi_l] = 8, -8, 8, -8
        kinds += [Kind("spread max last", va, (lo0, hi_l, 0)), Kind("spread max first", vb, (lo_l, hi0, C - 1))]
    else:
        raise ValueError(regime)
    return bias, kinds


def _split4(v: torch.Tensor) -> torch.Tensor:
    """[C] integers in [-16, 16] -> [4, C] integers in [-4, 4] summing to v."""
    q = torch.div(v, 4, rounding_mode="floor")
    rem = v - 4 * q
    return torch.stack([q + (rem > i).long() for i in range(4)])


def make_case(regime: str, T: int, B: int, H: int, C: int, lengths: bool = True, seed: int = 0, device="cpu") -> Case:
    """A case of ``regime`` (REGIMES) at h [T,B,H], W [H,C].  Row r = t·B + b takes kind r mod (number of kinds); its label cycles
    through the kind's candidates.  ``lengths``: per-row lengths in [0, T] with a length-0 row and a full row (T = 1: lengths 0
    or 1, a quarter of them 0), else every position counts."""
    g = torch.Generator().manual_seed(seed * 7919 + C * 31 + H + T * B)
    bias, kinds = _kinds(regime, C, g)
    P = len(kinds)
    G = H // P
    assert G >= 4, f"H = {H} is too small for {P} kinds"
    W = torch.zeros(H, C, dtype=torch.long)
    for p, k in enumerate(kinds):
        assert int(k.values.abs().max()) <= 16
        dims = [j * P + p for j in range(G)]
        main = [dims[j] for j in (0, G // 4, G // 2, 3 * G // 4)]
        W[main] = _split4(k.values)
        rest = [d for d in dims if d not in main]
        for d1, d2 in zip(rest[0::2], rest[1::2]):
            x = torch.randint(-4, 5, (C,), generator=g)
            W[d1], W[d2] = x, -x
    R = T * B
    kind_of = torch.arange(R) % P
    h = torch.zeros(R, H, dtype=torch.long)
    for p in range(P):
        h[kind_of == p, p:P * G:P] = 1
    if P * G < H:
        h[:, P * G:] = torch.randint(-2, 3, (R, H - P * G), generator=g)
    lab = torch.empty(R, dtype=torch.long)
    for p, k in enumerate(kinds):
        rows = (kind_of == p).nonzero().squeeze(1)
        cands = torch.tensor(k.labels)
        lab[rows] = cands[(rows // P) % len(k.labels)]
    ln = None
    if lengths:
        if T == 1:
            ln = (torch.rand(B, generator=g) >= 0.25).int()
            ln[0] = 0
            ln[-1] = 1
        else:
            ln = torch.randint(0, T + 1, (B,), generator=g, dtype=torch.int32)
            ln[0], ln[-1] = 0, T
            if B == 1:
                ln[0] = T - 1
    tmpl = torch.stack([k.values for k in kinds]).double()
    logits = (bias.view(1, C) + tmpl[kind_of]).view(T, B, C)
    labels = lab.view(T, B).t().contiguous()
    case = Case(f"{regime}", regime, h.double().view(T, B, H), W.double(), bias, labels, ln, logits, kind_of.view(T, B), kinds)
    if ln is not None:
        case.labels = torch.where(case.keep.t(), labels, UNREAD)
    return to(case, device)


def to(case: Case, device) -> Case:
    return dataclasses.replace(case, **{f.name: getattr(case, f.name).to(device) for f in dataclasses.fields(case)
                                        if isinstance(getattr(case, f.name), torch.Tensor)})


def small_head_path(dtype, H: int, C: int, per_step: bool):
    """The kernels the small heads select (csrc/head_wgmma.cu: ts_head_fwd_tc / ts_head_step_fwd, launch_bwd /
    launch_step_bwd) -> (NP of the tensor-core forward or None for the generic one, CP of the register backward or None for the
    per-output kernels)."""
    NP = 16
    while NP < C:
        NP *= 2
    smem = (H + 63) // 64 * NP * 128 + 4 * 128 * 64 * 2 + 1024 + 128 + NP * 4 + (64 if per_step else 0)
    tc = dtype == torch.bfloat16 and C <= 256 and smem <= 200 * 1024 and H % 8 == 0
    cp = None if C > 32 else (8 if C <= 8 else 16 if C <= 16 else 32)
    return (NP if tc else None), cp


STEP_BWD_ROWS = {8: 1024, 16: 512, 32: 192}    # step_bwd_rows<CP>


# ---- references ------------------------------------------------------------------------------------------------------------
def reference(case: Case, dloss: float, emulate: bool, vocab: bool):
    """The head's loss and gradients from the exact logits: fp64 (``emulate`` False) or fp32 at the kernels' rounding points
    (``vocab``: dlogits rounded to bf16 after the dloss / N scale and dh stored bf16, tests/test_gpu_next_token.py; otherwise
    fp32 dlogits and dh in h's dtype, which the caller rounds).  The last-state head is the case T = 1 without lengths.
    -> dict(loss, dh [T,B,H], dW, db, dlogits)."""
    dt = torch.float32 if emulate else torch.float64
    keep = case.keep.to(dt)
    lab = case.lab.unsqueeze(2)
    logp = torch.log_softmax(case.logits.to(dt), 2)
    n = keep.sum()
    loss = -(logp.gather(2, lab).squeeze(2) * keep).sum() / n
    d = (logp.exp() - torch.zeros_like(logp).scatter_(2, lab, 1.0)) * keep.unsqueeze(2)
    if vocab:
        d = d * (dloss / n)
        if emulate:
            d = d.bfloat16().to(dt)
    else:
        d = d / n * dloss
    T, B, H = case.h.shape
    h = case.h.to(dt)
    W = case.W.to(dt)
    dh = d @ W.t()
    if vocab and emulate:
        dh = dh.bfloat16().to(dt)
    dW = h.reshape(T * B, H).t() @ d.reshape(T * B, -1)
    return {"loss": loss, "dh": dh, "dW": dW, "db": d.sum((0, 1)), "dlogits": d}


def first_argmax(logits: torch.Tensor) -> torch.Tensor:
    """torch.argmax's first index (stated, not assumed: the smallest class among those at the max)."""
    mx = logits.amax(-1, keepdim=True)
    C = logits.shape[-1]
    idx = torch.arange(C, device=logits.device).expand_as(logits)
    return torch.where(logits == mx, idx, C).amin(-1)


# ---- assertions (the GPU tests call these; the negative controls must fail them) -------------------------------------------
def assert_counts(case: Case, correct, n) -> None:
    """``correct`` and N exactly: the rows whose first arg-max is the label, among the counted ones."""
    keep = case.keep
    want = int(((first_argmax(case.logits) == case.lab) & keep).sum())
    assert int(n) == int(keep.sum()), (case.name, int(n), int(keep.sum()))
    assert int(correct) == want, (case.name, "correct", int(correct), want)


def check_head(name: str, case: Case, got: dict, dloss: float, vocab: bool, floor: float, round_dh=None) -> float:
    """The budget of ``lstm_numerics.check_budget`` on loss, dh, dW and db (dlogits enter through the three gradients) and no
    gradient at uncounted positions -> the worst ratio.  ``round_dh``: rounds the emulated dh to the kernel's dh dtype."""
    f64 = reference(case, dloss, False, vocab)
    emu = reference(case, dloss, True, vocab)
    if round_dh is not None:
        emu["dh"] = round_dh(emu["dh"])
    worst = 0.0
    for k in ("loss", "dh", "dW", "db"):
        worst = max(worst, N.check_budget(f"{name} {k}", got[k], f64[k], emu[k], floor=floor))
    off = ~case.keep
    if bool(off.any()):
        assert float(got["dh"].reshape(case.h.shape)[off].abs().max()) == 0.0, f"{name}: gradient at uncounted positions"
    return worst


def lead(case: Case) -> torch.Tensor:
    """[T,B] how far the row max leads the largest logit outside the top pair (ties) or below the max (other kinds)."""
    l = case.logits
    top2 = l.topk(3, -1).values if l.shape[-1] >= 3 else torch.cat([l.topk(2, -1).values, l.new_full(l.shape[:-1] + (1,), -math.inf)], -1)
    tied = torch.tensor([k.pair is not None and k.name.startswith("tie") for k in case.kinds], device=l.device)[case.kind_of]
    return torch.where(tied, top2[..., 0] - top2[..., 2], top2[..., 0] - top2[..., 1])


def assert_tokens(case: Case, tokens, temperature: float) -> int:
    """Sampled tokens of a T = 1 case: the first arg-max at temperature 0; above it, on rows whose max leads by at least
    21 t (the Gumbel noise lies in [-2.85, 17.33]), the arg-max, or one of the two tied classes.  -> rows checked."""
    l = case.logits[0]
    t = tokens.long().view(-1).to(l.device)
    assert bool(((t >= 0) & (t < l.shape[1])).all()), "a token outside [0, C)"
    if temperature == 0:
        want = first_argmax(l)
        bad = (t != want).nonzero()
        assert bad.numel() == 0, (case.name, "greedy", [(int(r), int(t[r]), int(want[r])) for r in bad[:4, 0]])
        return l.shape[0]
    sure = lead(case)[0] >= 21 * temperature
    top = l.amax(1, keepdim=True)
    at_top = (l.gather(1, t.view(-1, 1)) == top).squeeze(1)
    bad = (sure & ~at_top).nonzero()
    assert bad.numel() == 0, (case.name, temperature, [(int(r), int(t[r])) for r in bad[:4, 0]])
    return int(sure.sum())


def check_logprob(name: str, case: Case, tokens, lp) -> float:
    """log p(token) under softmax(l) against fp64 within the budget of its fp32 evaluation."""
    l = case.logits[0]
    t = tokens.long().view(-1, 1).to(l.device)
    lp64 = torch.log_softmax(l, 1).gather(1, t).squeeze(1)
    lp32 = torch.log_softmax(l.float(), 1).gather(1, t).squeeze(1)
    return N.check_budget(f"{name} logprob", lp, lp64, lp32)


# ---- a model of the vocabulary head in torch, for the negative controls --------------------------------------------------------
def simulate(case: Case, dloss: float = 1.0, tie: str = "first", pad: Optional[float] = None, rescale: bool = True,
             mask: bool = True) -> dict:
    """The vocabulary head as its kernels compute it, in fp32 torch: per 256-class tile the max, sum exp(l - max) and arg-max,
    merged tile by tile in ascending order with max-rescaled sums, then loss, correct, N, bf16 dlogits and the gradients.
    Defects on request: ``tie='last'`` (the later class wins a tie), ``pad`` (padded classes enter with this logit instead of
    -inf), ``rescale=False`` (a new max does not rescale the running sum), ``mask=False`` (uncounted rows get dlogits too)."""
    T, B, C = case.logits.shape
    R = T * B
    l = case.logits.float().reshape(R, C)
    nt = -(-C // TILE)
    lp = torch.full((R, nt * TILE), -math.inf if pad is None else pad, dtype=torch.float32, device=l.device)
    lp[:, :C] = l
    tiles = lp.view(R, nt, TILE)
    tmax = tiles.amax(2)
    pos = torch.arange(TILE, device=l.device).expand_as(tiles)
    hit = tiles == tmax.unsqueeze(2)
    targ = (torch.where(hit, pos, TILE).amin(2) if tie == "first" else torch.where(hit, pos, -1).amax(2))
    targ = targ + TILE * torch.arange(nt, device=l.device)
    tse = torch.exp(tiles - tmax.unsqueeze(2)).sum(2)
    mx, se, arg = tmax[:, 0].clone(), tse[:, 0].clone(), targ[:, 0].clone()
    for i in range(1, nt):
        v, s, a = tmax[:, i], tse[:, i], targ[:, i]
        up = v > mx
        take = up | ((v == mx) & (tie == "last"))
        se = torch.where(up, (se * torch.exp(mx - v) if rescale else se) + s, se + s * torch.exp(v - mx))
        arg = torch.where(take, a, arg)
        mx = torch.maximum(mx, v)
    lse = mx + torch.log(se)
    keep = case.keep.reshape(R)
    y = case.lab.reshape(R)
    nll = (lse - l.gather(1, y.view(-1, 1)).squeeze(1)) * keep
    n = keep.sum()
    out = {"loss": nll.sum() / n, "correct": int(((arg == y) & keep).sum()), "n": int(n), "tokens": arg.view(T, B)}
    d = torch.exp(lp[:, :C] - lse.view(-1, 1)) - torch.zeros_like(l).scatter_(1, y.view(-1, 1), 1.0)
    if mask:
        d = d * keep.view(-1, 1)
    d = (d * (dloss / n)).bfloat16().float()
    H = case.h.shape[2]
    h = case.h.float().reshape(R, H)
    out.update(dh=(d @ case.W.float().t()).bfloat16().float().view(T, B, H), dW=h.t() @ d, db=d.sum(0))
    return out
