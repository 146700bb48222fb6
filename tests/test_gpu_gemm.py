"""The tensor-core GEMM (csrc/gemm2_wgmma.cu) and its dispatch (ops/cuda_gemm.matmul).

1. Exact: integer operands |a|, |b| <= 3 make every product exact and keep every partial sum of K <= 32768 terms below
   2^19, so the fp32 result is exact in any summation order.  fp32 output, the accumulate mode and the row sums must then
   equal the fp64 product bit for bit, and bf16 output its round-to-nearest-even.  Operands are views into NaN-filled
   buffers (pitch padding and trailing rows), outputs and row sums views into sentinel-filled buffers: a load past the
   logical extent poisons the result, a store outside [:M, :N] / [:M] changes the sentinel.
2. Random bf16 data at the training step's shapes: every element within the bound of fp32 accumulation of exact
   products, |C - C64| <= 2 K 2^-24 (|A| |B|) (+ the output rounding terms), and a negative control that the bound sees a
   lost k-block.
3. Bitwise identities of the schedule: the grid cap, the 2-CTA cluster, PDL, the stream, the dataflow gate and the
   reversed M walk change neither the template instantiation nor any tile's K order.
4. The ``done`` counters: one increment per 128-row block and column tile, nothing past the buffer; a short buffer is
   refused before launch.
5. ``matmul``'s choice between the tensor-core kernel and the CUDA-core ``gemm_generic``, on each side of every condition.
"""
import pytest
import torch

from lstm_tensorspark_b200.ops import cuda_gemm as G

gpu = pytest.mark.gpu

CONFIGS = [(1, 128), (1, 256), (2, 128), (2, 256)]                     # (CTAs per cluster, BN)
LAYOUTS = [(False, False), (False, True), (True, False), (True, True)]  # (A MN-major, B MN-major)
EXACT_SHAPES = [
    (8, 8, 8),            # one partial k-block; a 2-CTA cluster's peer lies wholly past M
    (128, 16, 64),        # the smallest shape matmul sends to the tensor cores
    (136, 24, 72),        # one row past a CTA tile, N below one 64-column box, a K tail of 8
    (264, 264, 136),      # one row past a 2-CTA tile, one column group past a 256 tile, a K tail
    (1000, 520, 264),     # ragged in every dimension
    (384, 1032, 4104),    # a long K with a tail, N 8 past a tile
    (4096, 4096, 512),    # 256+ tiles: several per cluster
]
SENT = -12288.0           # output sentinel, exact in bf16 and fp32
SENT_I = 0x5EAD           # counter sentinel


def _sid(s):
    return "x".join(map(str, s))


@pytest.fixture(scope="module")
def E():
    from lstm_tensorspark_b200.ops.cuda_ext import ext
    return ext()


@pytest.fixture(scope="module")
def dev():
    return torch.device("cuda", 0)


@pytest.fixture(scope="module")
def ints(dev):
    """ints(M, N, K): integer A [M, K], B [K, N] (bf16), bias [N] (fp32), their exact product A·B (fp64) and the row sums of
    A (fp64).  Each shape is drawn once for the module; the tensors are freed when the module's tests end."""
    cache = {}

    def get(M, N, K):
        if (M, N, K) not in cache:
            g = torch.Generator(device=dev).manual_seed(M * 1000003 + N * 1009 + K)
            A = torch.randint(-3, 4, (M, K), generator=g, device=dev).bfloat16()
            Bm = torch.randint(-3, 4, (K, N), generator=g, device=dev).bfloat16()
            bias = torch.randint(-3, 4, (N,), generator=g, device=dev).float()
            cache[(M, N, K)] = (A, Bm, bias, A.double() @ Bm.double(), A.double().sum(1))
        return cache[(M, N, K)]
    yield get
    cache.clear()
    torch.cuda.empty_cache()


# ----------------------------------------------------------------------------------------------------------------- helpers


def _storage(x, mn):
    """Storage of a logical [rows, K] operand: K-major [rows, K] or MN-major [K, rows]."""
    return x.t() if mn else x


def _nan_padded(s, pad=8, tail=8):
    """``s`` as a view into a larger bf16 buffer whose pitch padding (pad columns) and following tail rows are NaN."""
    buf = torch.full((s.shape[0] + tail, s.shape[1] + pad), float("nan"), dtype=torch.bfloat16, device=s.device)
    buf[:s.shape[0], :s.shape[1]] = s
    return buf[:s.shape[0], :s.shape[1]]


def _padded_out(M, N, dtype, dev, fill=None):
    """(buffer, [M, N] view at row 1, column 8 of it): everything outside the view is SENT."""
    buf = torch.full((M + 3, N + 24), SENT, dtype=dtype, device=dev)
    view = buf[1:1 + M, 8:8 + N]
    if fill is not None:
        view.copy_(fill)
    return buf, view


def _padded_vec(M, dev, fill=None):
    buf = torch.full((M + 12,), SENT, dtype=torch.float32, device=dev)
    view = buf[4:4 + M]
    if fill is not None:
        view.copy_(fill)
    return buf, view


def _assert_equal(got, exp, what):
    if torch.equal(got, exp):
        return
    bad = (got != exp) if got.dtype == exp.dtype else (got.double() != exp.double())
    bad |= torch.isnan(got)
    idx = bad.nonzero()
    first = tuple(int(i) for i in idx[0]) if len(idx) else None
    detail = f"got {got[first].item()} expected {exp[first].item()}" if first is not None else "shapes or dtypes differ"
    raise AssertionError(f"{what}: {len(idx)} of {got.numel()} elements differ; first at {first}: {detail}")


def _assert_outside_intact(buf, view_rows, view_cols, what):
    b = buf.clone()
    b[view_rows, view_cols] = SENT
    _assert_equal(b, torch.full_like(b, SENT), what + " (outside the output view)")


def _old(dev, shape, seed):
    g = torch.Generator(device=dev).manual_seed(seed)
    return torch.randint(-200, 201, shape, generator=g, device=dev).float()


def _exact_case(E, dev, M, N, K, Aop, Bop, bias, R, rs_ref, kw, tag):
    """Every output mode, with and without bias, against the exact product R (fp64) and the row sums rs_ref of A (None:
    no row sums).  ``kw``: layout, tile configuration and fold arguments."""
    rows, cols = slice(1, 1 + M), slice(8, 8 + N)
    old = _old(dev, (M, N), M + N + K)
    old_rs = _old(dev, (M,), M + 7)
    for with_bias in (False, True):
        b = bias if with_bias else None
        exp = R + bias.double() if with_bias else R
        t = f"{tag} bias={with_bias}"
        # bf16 output: the fp32 value is exact, its RNE rounding has one answer
        buf, C = _padded_out(M, N, torch.bfloat16, dev)
        E.gemm2(Aop, Bop, bias=b, out=C, **kw)
        _assert_equal(C, exp.to(torch.bfloat16), t + " bf16")
        _assert_outside_intact(buf, rows, cols, t + " bf16")
        # fp32 output over old content (no trace of it may stay), with row sums of A where there is no bias
        buf, C = _padded_out(M, N, torch.float32, dev, fill=old)
        rsbuf, rs = _padded_vec(M, dev, fill=old_rs) if not with_bias and rs_ref is not None else (None, None)
        E.gemm2(Aop, Bop, bias=b, out=C, out_fp32=True, rowsum=rs, **kw)
        _assert_equal(C, exp.float(), t + " fp32")
        _assert_outside_intact(buf, rows, cols, t + " fp32")
        if rs is not None:
            _assert_equal(rs, rs_ref.float(), t + " rowsum")
            _assert_equal(rsbuf[:4], torch.full_like(rsbuf[:4], SENT), t + " rowsum head")
            _assert_equal(rsbuf[4 + M:], torch.full_like(rsbuf[4 + M:], SENT), t + " rowsum tail")
        # fp32 accumulate: C = old + A·B (+ bias), rowsum_acc: rs = old + row sums
        buf, C = _padded_out(M, N, torch.float32, dev, fill=old)
        rsbuf, rs = _padded_vec(M, dev, fill=old_rs) if not with_bias and rs_ref is not None else (None, None)
        E.gemm2(Aop, Bop, bias=b, out=C, out_fp32=True, accumulate=True, rowsum=rs, rowsum_acc=True, **kw)
        _assert_equal(C, (old.double() + exp).float(), t + " fp32 accumulate")
        _assert_outside_intact(buf, rows, cols, t + " fp32 accumulate")
        if rs is not None:
            _assert_equal(rs, (old_rs.double() + rs_ref).float(), t + " rowsum accumulate")
            _assert_equal(rsbuf[:4], torch.full_like(rsbuf[:4], SENT), t + " rowsum accumulate head")
            _assert_equal(rsbuf[4 + M:], torch.full_like(rsbuf[4 + M:], SENT), t + " rowsum accumulate tail")


def _layout_case(E, dev, ints, shape, a_mn, b_mn, ctas, bn, max_ctas=0):
    M, N, K = shape
    A, Bm, bias, R, rs_ref = ints(M, N, K)
    Aop, Bop = _nan_padded(_storage(A, a_mn)), _nan_padded(_storage(Bm.t(), b_mn))
    kw = dict(a_mn=a_mn, b_mn=b_mn, ctas=ctas, bn=bn, max_ctas=max_ctas)
    _exact_case(E, dev, M, N, K, Aop, Bop, bias, R, rs_ref, kw, f"{shape} a_mn={a_mn} b_mn={b_mn} ctas={ctas} bn={bn} max_ctas={max_ctas}")


# -------------------------------------------------------------------------------------------------- 1. exact on integers
@gpu
@pytest.mark.parametrize("ctas,bn", CONFIGS)
@pytest.mark.parametrize("a_mn,b_mn", LAYOUTS)
@pytest.mark.parametrize("shape", EXACT_SHAPES, ids=_sid)
def test_gemm2_exact_on_integers(E, dev, ints, shape, a_mn, b_mn, ctas, bn):
    """Every layout, tile configuration and output mode, bit for bit, with poisoned padding and sentinel-guarded outputs."""
    _layout_case(E, dev, ints, shape, a_mn, b_mn, ctas, bn)


@gpu
@pytest.mark.parametrize("max_ctas", [1, 2, 3])
@pytest.mark.parametrize("ctas,bn", CONFIGS)
@pytest.mark.parametrize("a_mn,b_mn", LAYOUTS)
@pytest.mark.parametrize("shape", EXACT_SHAPES[-2:], ids=_sid)
def test_gemm2_exact_with_a_capped_grid(E, dev, ints, shape, a_mn, b_mn, ctas, bn, max_ctas):
    """One to three CTAs (one cluster with ctas = 2) walk every tile: the stage ring's phase wraps across many tiles."""
    _layout_case(E, dev, ints, shape, a_mn, b_mn, ctas, bn, max_ctas)


@gpu
@pytest.mark.parametrize("ctas,bn", CONFIGS)
@pytest.mark.parametrize("b_mn", [False, True])
@pytest.mark.parametrize("Bsz,T,F,N", [(128, 3, 128, 264), (256, 2, 192, 24)])
def test_gemm2_exact_folded_a(E, dev, Bsz, T, F, N, b_mn, ctas, bn):
    """K-major A read in place from a batch-major [Bsz, T, F] array (a pitched one) as the time-major X = [T·Bsz, F]."""
    M, K = T * Bsz, F
    g = torch.Generator(device=dev).manual_seed(Bsz + T + F)
    x_bm = torch.randint(-3, 4, (Bsz, T, F), generator=g, device=dev).bfloat16()
    X = x_bm.transpose(0, 1).reshape(M, K)
    store = _nan_padded(x_bm.reshape(Bsz, T * F))
    Bm = torch.randint(-3, 4, (K, N), generator=g, device=dev).bfloat16()
    bias = torch.randint(-3, 4, (N,), generator=g, device=dev).float()
    Bop = _nan_padded(_storage(Bm.t(), b_mn))
    kw = dict(b_mn=b_mn, ctas=ctas, bn=bn, a_fold=Bsz, fold_cols=F)
    _exact_case(E, dev, M, N, K, store, Bop, bias, X.double() @ Bm.double(), None, kw,            # (no row sums of a folded A)
                f"folded A {Bsz}x{T}x{F} N={N} b_mn={b_mn} ctas={ctas} bn={bn}")


@gpu
@pytest.mark.parametrize("ctas,bn", CONFIGS)
@pytest.mark.parametrize("a_mn", [False, True])
@pytest.mark.parametrize("Bsz,T,F,M", [(64, 3, 256, 136), (128, 2, 512, 264)])
def test_gemm2_exact_folded_b(E, dev, Bsz, T, F, M, a_mn, ctas, bn):
    """MN-major B read in place from a batch-major [Bsz, T, F] array (a pitched one) as X = [T·Bsz, F] (dW = dG^T X)."""
    K, N = T * Bsz, F
    g = torch.Generator(device=dev).manual_seed(Bsz + T + F + M)
    x_bm = torch.randint(-3, 4, (Bsz, T, F), generator=g, device=dev).bfloat16()
    X = x_bm.transpose(0, 1).reshape(K, N)
    store = _nan_padded(x_bm.reshape(Bsz, T * F))
    A = torch.randint(-3, 4, (M, K), generator=g, device=dev).bfloat16()
    bias = torch.randint(-3, 4, (N,), generator=g, device=dev).float()
    Aop = _nan_padded(_storage(A, a_mn))
    kw = dict(a_mn=a_mn, b_mn=True, ctas=ctas, bn=bn, b_fold=Bsz, fold_cols=F)
    _exact_case(E, dev, M, N, K, Aop, store, bias, A.double() @ X.double(), A.double().sum(1), kw,
                f"folded B {Bsz}x{T}x{F} M={M} a_mn={a_mn} ctas={ctas} bn={bn}")


# ------------------------------------------------------------------------------------------- 2. fp64 bound on random data
U = 2.0 ** -24
# name, (M, N, K), A MN-major, B MN-major, output ("bf16" | "fp32" | "acc"), bias, row sums, ctas, bn
RANDOM_CASES = [
    ("x-projection", (32768, 4096, 1024), False, False, "bf16", False, False, 2, 256),
    ("dX", (32768, 1024, 4096), False, True, "bf16", False, False, 1, 256),
    ("lstm-dW", (4096, 1024, 32768), True, True, "acc", False, True, 2, 256),
    ("vocab-dh", (4096, 1024, 32768), False, False, "bf16", False, False, 2, 256),
    ("vocab-dW", (1024, 32768, 4096), True, True, "acc", False, False, 2, 256),
    ("tail-1000x520x264", (1000, 520, 264), False, True, "fp32", True, True, 1, 128),
    ("tail-384x1032x4104", (384, 1032, 4104), True, False, "bf16", True, False, 2, 128),
]


def _random_problem(dev, M, N, K, seed):
    g = torch.Generator(device=dev).manual_seed(seed)
    A = torch.randn(M, K, generator=g, device=dev).bfloat16()
    Bm = torch.randn(K, N, generator=g, device=dev).bfloat16()
    bias = torch.randn(N, generator=g, device=dev)
    old = torch.randn(M, N, generator=g, device=dev) * 4
    old_rs = torch.randn(M, generator=g, device=dev) * 4
    return A, Bm, bias, old, old_rs


def _max_ratio(err, bound):
    """max(err / bound), where a NaN (a NaN output, or 0 / 0) counts as an infinite ratio: Python's max() and a
    tensor's NaN-propagating max would otherwise let a NaN pass a `<= 1` check or hide the other errors."""
    return float(torch.nan_to_num(err / bound, nan=float("inf"), posinf=float("inf")).max())


def _worst_ratio(A64, B64, C, K, bias=None, old=None, bf16=False, rows=4096):
    """max_ij |C - C64|_ij / bound_ij over every element, in row chunks (fp64 throughout):
         bound = 2 K 2^-24 (|A| |B|)  + 2^-24 (|C64| + |bias|) with bias  + 2^-24 |old| accumulating;  bf16: bound (1 + 2^-8) + 2^-8 |C64|
    where C64 is the exact result (A·B + bias + old).  K is the kernel's contraction length (the negative control passes a
    shortened A64 / B64 with the full K)."""
    worst = 0.0
    B64a = B64.abs()
    for r0 in range(0, A64.shape[0], rows):
        a = A64[r0:r0 + rows]
        ref = a @ B64
        bound = (2 * K * U) * (a.abs() @ B64a)
        if bias is not None:
            bound += U * (ref.abs() + bias.double().abs())
            ref += bias.double()
        if old is not None:
            o = old[r0:r0 + rows].double()
            bound += U * o.abs()
            ref += o
        if bf16:
            bound = bound * (1 + 2.0 ** -8) + 2.0 ** -8 * ref.abs()
        err = (C[r0:r0 + rows].double() - ref).abs()
        worst = max(worst, _max_ratio(err, bound))
        del a, ref, bound, err
    return worst


@gpu
@pytest.mark.parametrize("name,shape,a_mn,b_mn,out,with_bias,with_rowsum,ctas,bn", RANDOM_CASES, ids=[c[0] for c in RANDOM_CASES])
def test_gemm2_within_fp32_accumulation_bound(E, dev, name, shape, a_mn, b_mn, out, with_bias, with_rowsum, ctas, bn):
    """Normal bf16 operands at the shapes a training step issues: every element within the bound of fp32 accumulation."""
    M, N, K = shape
    A, Bm, bias, old, old_rs = _random_problem(dev, M, N, K, seed=sum(shape))
    Aop, Bop = _storage(A, a_mn).contiguous(), _storage(Bm.t(), b_mn).contiguous()
    b = bias if with_bias else None
    rs = old_rs.clone() if with_rowsum else None
    if out == "bf16":
        C = E.gemm2(Aop, Bop, bias=b, a_mn=a_mn, b_mn=b_mn, ctas=ctas, bn=bn)
    else:
        C = old.clone() if out == "acc" else torch.empty(M, N, device=dev)
        E.gemm2(Aop, Bop, bias=b, out=C, a_mn=a_mn, b_mn=b_mn, out_fp32=True, accumulate=out == "acc", ctas=ctas, bn=bn,
                rowsum=rs, rowsum_acc=out == "acc")
    del Aop, Bop
    A64, B64 = A.double(), Bm.double()
    del A, Bm
    r = _worst_ratio(A64, B64, C, K, bias=b, old=old if out == "acc" else None, bf16=out == "bf16")
    msg = f"\ngemm2 fp64 bound {name} {shape} out={out}: worst |C - C64| / bound = {r:.4f}"
    if rs is not None:
        rs_ref = A64.sum(1) + (old_rs.double() if out == "acc" else 0)
        rs_bound = 2 * K * U * A64.abs().sum(1) + (U * old_rs.double().abs() if out == "acc" else 0)
        r_rs = _max_ratio((rs.double() - rs_ref).abs(), rs_bound)
        msg += f", row sums {r_rs:.4f}"
        r = max(r, r_rs)
    print(msg)
    assert r <= 1.0, msg


@gpu
@pytest.mark.parametrize("out", ["fp32", "bf16"])
@pytest.mark.parametrize("shape", [(1000, 520, 264), (384, 1032, 4104)], ids=_sid)
def test_gemm2_bound_sees_a_lost_k_block(E, dev, shape, out):
    """Negative control: against a reference that drops the last 8 columns of K, the same bound must fail."""
    M, N, K = shape
    A, Bm, bias, _, _ = _random_problem(dev, M, N, K, seed=sum(shape) + 1)
    C = E.gemm2(A, Bm.t().contiguous(), bias=bias, out_fp32=out == "fp32")
    A64, B64 = A.double(), Bm.double()
    assert _worst_ratio(A64, B64, C, K, bias=bias, bf16=out == "bf16") <= 1.0
    r = _worst_ratio(A64[:, :K - 8], B64[:K - 8], C, K, bias=bias, bf16=out == "bf16")
    print(f"\ngemm2 fp64 bound negative control {shape} out={out}: ratio without the last 8 k = {r:.2f}")
    assert r > 1.0, r


def test_bound_ratio_fails_on_non_finite_output():
    """The section-2 check on the CPU: a NaN or infinite element of C makes the worst ratio infinite, wherever it lies
    and whatever the other elements hold."""
    g = torch.Generator().manual_seed(0)
    A64, B64 = torch.randn(40, 24, generator=g, dtype=torch.float64), torch.randn(24, 16, generator=g, dtype=torch.float64)
    C = (A64 @ B64).float()
    assert _worst_ratio(A64, B64, C, 24) <= 1.0
    for bad in (float("nan"), float("inf")):
        for where in ((0, 0), (39, 15), (17, 3)):
            Cb = C.clone()
            Cb[where] = bad
            assert _worst_ratio(A64, B64, Cb, 24, rows=16) == float("inf"), (bad, where)
    assert _max_ratio(torch.tensor([5.0, float("nan")]), torch.ones(2)) == float("inf")


# --------------------------------------------------------------------------------------- 3. bitwise schedule identities
def _gate(dev, M, rows_per_step=64):
    """Arrival counters that already satisfy every target the launch can set: [count, stride, base, per_step,
    rows_per_step, use_last] = [5, 3, 2, 4, 64, 1]; the counters sit at the last step's target or above it."""
    count, stride, base, per_step = 5, 3, 2, 4
    last = base + per_step * ((M - 1) // rows_per_step)
    gate = torch.zeros(count * stride, dtype=torch.int32, device=dev)
    gate[::stride] = last + torch.arange(count, dtype=torch.int32, device=dev)
    return gate, [count, stride, base, per_step, rows_per_step, 1]


def _blocks(M, N, ctas, bn):
    return -(-M // (128 * ctas)) * ctas * -(-N // bn)


@gpu
@pytest.mark.parametrize("bn", [128, 256])
@pytest.mark.parametrize("a_mn,b_mn", LAYOUTS)
def test_gemm2_schedule_identities(E, dev, a_mn, b_mn, bn):
    """Same instantiation, same K order per tile -> the same bits: repeat, grid cap, 1- vs 2-CTA clusters, PDL, an
    explicit stream, and the dataflow gate (already satisfied) with the M tiles walked forwards and backwards."""
    M, N, K = 1288, 1032, 1032
    A, Bm, bias, _, _ = _random_problem(dev, M, N, K, seed=5)
    Aop, Bop = _storage(A, a_mn).contiguous(), _storage(Bm.t(), b_mn).contiguous()
    for out in ("bf16", "fp32"):
        fp32 = out == "fp32"

        def run(ctas, **kw):
            C = torch.full((M, N), SENT, dtype=torch.float32 if fp32 else torch.bfloat16, device=dev)
            rs = torch.full((M,), SENT, device=dev) if fp32 else None
            E.gemm2(Aop, Bop, bias=bias, out=C, a_mn=a_mn, b_mn=b_mn, out_fp32=fp32, ctas=ctas, bn=bn, rowsum=rs, **kw)
            return C, rs

        def same(x, y, what):
            _assert_equal(x[0], y[0], f"{what} out={out} a_mn={a_mn} b_mn={b_mn} bn={bn}")
            if fp32:
                _assert_equal(x[1], y[1], f"{what} (row sums) out={out} a_mn={a_mn} b_mn={b_mn} bn={bn}")

        ref = run(1)
        for ctas in (1, 2):
            tag = f"ctas={ctas}"
            base = run(ctas)
            same(base, ref, "ctas=2 vs ctas=1")
            same(run(ctas), base, tag + " repeated call")
            for mc in (1, 3, 7):
                same(run(ctas, max_ctas=mc), base, f"{tag} max_ctas={mc}")
            same(run(ctas, pdl=True), base, tag + " pdl")
            s = torch.cuda.Stream(device=dev)
            s.wait_stream(torch.cuda.current_stream(dev))
            on_s = run(ctas, stream=s.cuda_stream)
            torch.cuda.current_stream(dev).wait_stream(s)
            same(on_s, base, tag + " explicit stream")
            for reverse_m in (0, 1):
                gate, cfg = _gate(dev, M)
                gate0 = gate.clone()
                err = torch.zeros(1, dtype=torch.int32, device=dev)
                done = torch.zeros(_blocks(M, N, ctas, bn), dtype=torch.int32, device=dev)
                gated = run(ctas, gate=gate, gate_cfg=cfg + [reverse_m], gate_err=err, done=done, max_ctas=3 * ctas)
                same(gated, base, f"{tag} gated reverse_m={reverse_m}")
                assert int(err.item()) == 0, (tag, reverse_m)
                assert torch.equal(gate, gate0)
                assert torch.equal(done, torch.ones_like(done)), (tag, reverse_m, done)


# ------------------------------------------------------------------------------------------------- 4. the done counters
@gpu
@pytest.mark.parametrize("ctas,bn", CONFIGS)
@pytest.mark.parametrize("shape", [(8, 8, 8), (136, 24, 72), (264, 264, 136), (1000, 520, 264)], ids=_sid)
def test_gemm2_done_counts_every_block_once(E, dev, ints, shape, ctas, bn):
    """``done[(row block) * tiles_n + column tile]`` goes up by exactly one for every block of the launch (a 2-CTA
    cluster's peer included where its rows lie past M), and nothing after the buffer changes."""
    M, N, K = shape
    A, Bm, bias, R, _ = ints(M, N, K)
    Bop = Bm.contiguous()
    n = _blocks(M, N, ctas, bn)
    for v in ("plain", "one cluster", "gated, M reversed"):
        g = torch.Generator(device=dev).manual_seed(n)
        buf = torch.full((n + 64,), SENT_I, dtype=torch.int32, device=dev)
        buf[:n] = torch.randint(0, 1000, (n,), generator=g, device=dev, dtype=torch.int32)
        before = buf.clone()
        kw = dict(max_ctas=1) if v == "one cluster" else {}
        if v.startswith("gated"):
            gate, cfg = _gate(dev, M)
            kw.update(gate=gate, gate_cfg=cfg + [1], gate_err=torch.zeros(1, dtype=torch.int32, device=dev))
        C = E.gemm2(A, Bop, bias=bias, b_mn=True, out_fp32=True, ctas=ctas, bn=bn, done=buf[:n], **kw)
        _assert_equal(C, (R + bias.double()).float(), f"{shape} ctas={ctas} bn={bn} {v}")
        assert torch.equal(buf[:n], before[:n] + 1), (shape, ctas, bn, v, (buf[:n] - before[:n]).tolist()[:32])
        assert torch.equal(buf[n:], before[n:]), (shape, ctas, bn, v)
        if "gate_err" in kw:
            assert int(kw["gate_err"].item()) == 0


@gpu
def test_gemm2_refuses_what_it_cannot_launch(E, dev, ints):
    """A ``done`` buffer shorter than the launch's blocks, an empty product and an unknown tile configuration raise
    before anything is launched: the output and the counters keep their contents."""
    for (M, N, K, ctas, bn) in [(8, 8, 8, 2, 256), (136, 24, 72, 2, 128), (1000, 520, 264, 1, 256), (264, 264, 136, 2, 256)]:
        A, Bm, bias, R, _ = ints(M, N, K)
        Bt = Bm.t().contiguous()
        n = _blocks(M, N, ctas, bn)
        peerless = -(-M // 128) * -(-N // bn)                  # ceil(M / 128) row blocks: no room for a peer past M
        for size in sorted({n - 1, peerless} - {n}):
            C = torch.full((M, N), SENT, device=dev)
            done = torch.full((size,), 7, dtype=torch.int32, device=dev)
            with pytest.raises(RuntimeError, match="done needs"):
                E.gemm2(A, Bt, out=C, out_fp32=True, ctas=ctas, bn=bn, done=done)
            torch.cuda.synchronize()
            assert torch.equal(C, torch.full_like(C, SENT)) and torch.equal(done, torch.full_like(done, 7)), (M, N, ctas, bn, size)
        done = torch.zeros(n, dtype=torch.int32, device=dev)
        C = E.gemm2(A, Bt, out_fp32=True, ctas=ctas, bn=bn, done=done)
        _assert_equal(C, R.float(), f"exact-size done {M}x{N}x{K}")
        assert torch.equal(done, torch.ones_like(done))
    A = torch.zeros(64, 64, dtype=torch.bfloat16, device=dev)
    with pytest.raises(RuntimeError, match="must be positive"):
        E.gemm2(A[:0], A)
    for ctas, bn in [(3, 256), (0, 128), (1, 192), (2, 64)]:
        with pytest.raises(RuntimeError, match="ctas must be 1 or 2 and bn 128 or 256"):
            E.gemm2(A, A, ctas=ctas, bn=bn)


# --------------------------------------------------------------------------------------------------- 5. matmul dispatch
def _ints(shape, seed, dtype=torch.bfloat16, dev="cuda"):
    g = torch.Generator(device=dev).manual_seed(seed)
    return torch.randint(-3, 4, shape, generator=g, device=dev).to(dtype)


def _pitched(rows, cols, pitch, offset=0, seed=0, dtype=torch.bfloat16):
    """A [rows, cols] integer view at column ``offset`` of a [rows, pitch] buffer."""
    buf = _ints((rows, pitch), seed, dtype)
    return buf[:, offset:offset + cols]


def _a_of(M, K, kind, seed=1):
    if kind == "kmajor":
        return _ints((M, K), seed)
    if kind == "mnmajor":
        return _ints((K, M), seed).t()
    if kind == "fp32":
        return _ints((M, K), seed, torch.float32)
    if kind == "pitch8":
        return _pitched(M, K, K + 8, seed=seed)
    if kind == "pitch4":
        return _pitched(M, K, K + 4, seed=seed)
    if kind == "base16":
        return _pitched(M, K, K + 16, offset=8, seed=seed)
    if kind == "base8":
        return _pitched(M, K, K + 16, offset=4, seed=seed)
    if kind == "mn-pitch8":
        return _pitched(K, M, M + 8, seed=seed).t()
    if kind == "mn-pitch4":
        return _pitched(K, M, M + 4, seed=seed).t()
    if kind == "strided":                          # neither K- nor MN-major: every other column
        return _pitched(M, 2 * K, 2 * K, seed=seed)[:, ::2]
    raise ValueError(kind)


# id, (M, N, K), A kind, B^T kind, out (None | (pitch, offset) of an fp32 / bf16 buffer), out dtype, accumulate, path
DISPATCH = [
    ("base", (128, 16, 64), "kmajor", "kmajor", None, torch.float32, False, "tc"),
    ("M=120", (120, 16, 64), "kmajor", "kmajor", None, torch.float32, False, "generic"),
    ("N=8", (128, 8, 64), "kmajor", "kmajor", None, torch.float32, False, "generic"),
    ("K=56", (128, 16, 56), "kmajor", "kmajor", None, torch.float32, False, "generic"),
    ("M=132", (132, 16, 64), "kmajor", "kmajor", None, torch.float32, False, "generic"),
    ("M=136", (136, 16, 64), "kmajor", "kmajor", None, torch.float32, False, "tc"),
    ("N=20", (128, 20, 64), "kmajor", "kmajor", None, torch.float32, False, "generic"),
    ("N=24", (128, 24, 64), "kmajor", "kmajor", None, torch.float32, False, "tc"),
    ("K=68", (128, 16, 68), "kmajor", "kmajor", None, torch.float32, False, "generic"),
    ("K=72", (128, 16, 72), "kmajor", "kmajor", None, torch.float32, False, "tc"),
    ("bf16-out", (136, 24, 72), "kmajor", "kmajor", None, torch.bfloat16, False, "tc"),
    ("a-mn", (136, 24, 72), "mnmajor", "kmajor", None, torch.float32, False, "tc"),
    ("b-mn", (136, 24, 72), "kmajor", "mnmajor", None, torch.bfloat16, False, "tc"),
    ("a-fp32", (136, 24, 72), "fp32", "kmajor", None, torch.float32, False, "generic"),
    ("a-pitch8", (136, 24, 72), "pitch8", "kmajor", None, torch.float32, False, "tc"),
    ("a-pitch4", (136, 24, 72), "pitch4", "kmajor", None, torch.float32, False, "generic"),
    ("b-mn-pitch8", (136, 24, 72), "kmajor", "mn-pitch8", None, torch.float32, False, "tc"),
    ("b-mn-pitch4", (136, 24, 72), "kmajor", "mn-pitch4", None, torch.float32, False, "generic"),
    ("a-base16", (136, 24, 72), "base16", "kmajor", None, torch.float32, False, "tc"),
    ("a-base8", (136, 24, 72), "base8", "kmajor", None, torch.float32, False, "generic"),
    ("b-base8", (136, 24, 72), "kmajor", "base8", None, torch.float32, False, "generic"),
    ("a-strided", (136, 24, 72), "strided", "kmajor", None, torch.float32, False, "generic"),
    ("b-strided", (136, 24, 72), "kmajor", "strided", None, torch.bfloat16, False, "generic"),
    ("out-pitch4", (136, 24, 72), "kmajor", "kmajor", (28, 0), torch.float32, False, "tc"),
    ("out-pitch2", (136, 24, 72), "kmajor", "kmajor", (26, 0), torch.float32, False, "generic"),
    ("out-base16", (136, 24, 72), "kmajor", "kmajor", (32, 4), torch.float32, False, "tc"),
    ("out-base8", (136, 24, 72), "kmajor", "kmajor", (32, 2), torch.float32, False, "generic"),
    ("acc-fp32", (136, 24, 72), "kmajor", "mnmajor", (32, 4), torch.float32, True, "tc"),
    ("acc-bf16", (136, 24, 72), "kmajor", "mnmajor", (32, 8), torch.bfloat16, True, "generic"),
    ("acc-fp32-generic", (120, 24, 72), "kmajor", "kmajor", (24, 0), torch.float32, True, "generic"),
]


@gpu
@pytest.mark.parametrize("name,shape,ak,bk,out,out_dtype,acc,path", DISPATCH, ids=[d[0] for d in DISPATCH])
def test_matmul_dispatch_boundaries(dev, name, shape, ak, bk, out, out_dtype, acc, path):
    """Each condition of _tc_ok, _major and the output checks, on both sides: the expected kernel, and the exact result."""
    M, N, K = shape
    a, b_t = _a_of(M, K, ak, seed=1), _a_of(N, K, bk, seed=2)
    bias = _ints((N,), 3, torch.float32)
    R = a.double() @ b_t.double().t() + bias.double()
    o = None
    if out is not None:
        pitch, off = out
        obuf = torch.full((M, pitch), SENT, dtype=out_dtype, device=dev)
        o = obuf[:, off:off + N]
        old = _ints((M, N), 4, torch.float32) * 10
        o.copy_(old)
        if acc:
            R = R + old.double()
    before = dict(G.STATS)
    res = G.matmul(a, b_t, out=o, accumulate=acc, out_dtype=out_dtype, bias=bias)
    other = "generic" if path == "tc" else "tc"
    assert G.STATS[path] == before[path] + 1 and G.STATS[other] == before[other], (name, path, before, G.STATS)
    got = o if o is not None else res
    assert got.dtype == out_dtype, (name, got.dtype)
    _assert_equal(got, R.to(out_dtype), name)
    if o is not None:
        outside = obuf.clone()
        outside[:, off:off + N] = SENT
        _assert_equal(outside, torch.full_like(outside, SENT), name + " (outside the output view)")


# --------------------------------------------------------------------------------------------------- _major (CPU only)
def test_major_classifies_views():
    """``_major``: K-major (unit contraction stride), MN-major (unit row stride, returned as its [K, rows] storage), or
    None; padded pitches and row slices keep their class, column steps and overlapping rows have none."""
    M, K = 12, 16
    x = torch.zeros(M, K)
    mn, s = G._major(x)
    assert mn is False and s is x
    xt = torch.zeros(K, M)
    mn, s = G._major(xt.t())
    assert mn is True and s.shape == (K, M) and s.stride() == (M, 1) and s.data_ptr() == xt.data_ptr()
    mn, s = G._major(x[3:9])                                                               # a row slice
    assert mn is False and s.shape == (6, K) and s.stride() == (K, 1)
    pitched = torch.zeros(M, K + 8)[:, :K]
    mn, s = G._major(pitched)
    assert mn is False and s.stride() == (K + 8, 1)
    pitched_t = torch.zeros(K, M + 8)[:, :M].t()
    mn, s = G._major(pitched_t)
    assert mn is True and s.shape == (K, M) and s.stride() == (M + 8, 1)
    mn, s = G._major(xt[:, 2:2 + 8].t())                                                   # a column slice of the storage
    assert mn is True and s.shape == (K, 8) and s.stride() == (M, 1)
    assert G._major(torch.zeros(M, 2 * K)[:, ::2]) is None                                 # contraction stride 2
    mn, s = G._major(torch.zeros(2 * K, M)[::2].t())                                       # every other storage row
    assert mn is True and s.stride() == (2 * M, 1)
    assert G._major(torch.zeros(K, 2 * M)[:, ::2].t()) is None                             # row stride 2
    assert G._major(torch.zeros(1, K).expand(M, K)) is None                                # every row the same memory
    assert G._major(torch.zeros(M * K).as_strided((M, K), (K // 2, 1))) is None            # rows overlap
    assert G._major(torch.zeros(M, K, 2)[..., 0]) is None                                  # both strides > 1
    assert G._major(torch.zeros(K)) is None and G._major(torch.zeros(2, M, K)) is None     # not 2-D
