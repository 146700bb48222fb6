"""Kernel tests (GPU, `pytest -m gpu`): every hand-written sm_90a kernel vs. the plain PyTorch fp32 reference of
the same op (ops/reference.py).  These run the CUDA path only — a missing extension is an error, not a skip."""
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def E():
    from lstm_tensorspark_b200.ops.cuda_ext import ext
    return ext()


@pytest.fixture(scope="module")
def dev():
    return torch.device("cuda", 0)


def _ref():
    from lstm_tensorspark_b200.ops import reference
    return reference


@pytest.mark.parametrize("dtype,tol", [(torch.float32, 1e-5), (torch.bfloat16, 2e-2)])
def test_pointwise_cell_fwd_bwd(E, dev, dtype, tol):
    ref = _ref()
    torch.manual_seed(0)
    B, H = 37, 24
    pre = torch.randn(B, 4 * H, device=dev).to(dtype)
    bias = torch.randn(4 * H, device=dev)
    c = torch.randn(B, H, device=dev)
    h, cn, act = E.lstm_pointwise_fwd(pre, bias, c)
    pr = (pre.float() + bias).requires_grad_(True)
    cr = c.clone().requires_grad_(True)
    i, f, g, o = ref.lstm_gates(pr)
    c_ref = f * cr + i * g
    h_ref = o * torch.tanh(c_ref)
    assert (h.float() - h_ref).abs().max() < tol and (cn - c_ref).abs().max() < tol
    dh = torch.randn(B, H, device=dev)
    dc = torch.randn(B, H, device=dev)
    (h_ref * dh + c_ref * dc).sum().backward()
    dpre, dcp = E.lstm_pointwise_bwd(dh.to(dtype), None, dc, act, c, cn)
    assert (dpre.float() - pr.grad).abs().max() < 10 * tol and (dcp - cr.grad).abs().max() < 10 * tol


@pytest.mark.parametrize("B,H,C,dtype", [(50, 96, 7, torch.bfloat16), (256, 1024, 10, torch.bfloat16), (300, 512, 40, torch.bfloat16),
                                         (130, 256, 200, torch.bfloat16), (50, 96, 7, torch.float32), (10, 16, 3, torch.float32),
                                         # backward in 32-row slabs with fp32 atomics (B > 640 at C <= 16, B > 256 at C <= 32)
                                         (1024, 1024, 10, torch.bfloat16), (257, 256, 32, torch.bfloat16),
                                         # the widest tensor-core head (NP = 256), and one class past each NP boundary
                                         (200, 64, 256, torch.bfloat16), (150, 128, 17, torch.bfloat16), (150, 128, 33, torch.bfloat16),
                                         (150, 128, 65, torch.bfloat16), (150, 128, 129, torch.bfloat16),
                                         # bf16 h the tensor-core kernel does not take (C > 256, H % 8 != 0): logits on CUDA cores
                                         (130, 64, 300, torch.bfloat16), (128, 100, 10, torch.bfloat16)])
def test_head_forward_and_backward_per_output_flags(E, dev, B, H, C, dtype):
    """Tensor-core head (bf16 h: TMA + wgmma, epilogue from the accumulator registers) / generic head (fp32 h, or shapes the
    tensor-core kernel does not take) vs the fp32 reference, and the fused backward kernel (dh, dW, db in one launch, overwrite and
    accumulate).  Both backward kernels take one flag per output: dW overwritten while db accumulates, and the reverse."""
    ref = _ref()
    torch.manual_seed(0)
    h = (torch.randn(B, H, device=dev) * 0.5).to(dtype)
    W = torch.randn(H, C, device=dev) * 0.1
    b = torch.randn(C, device=dev)
    y = torch.randint(0, C, (B,), device=dev)
    logits, dlog, loss, corr = E.head_fwd(h, W, b, y)
    tensor_cores = dtype == torch.bfloat16 and C <= 256 and H % 8 == 0
    Wr = W.bfloat16().float() if tensor_cores else W                     # the tensor-core path rounds W to bf16, the others do not
    hr = h.float().requires_grad_(True)
    Wq = Wr.clone().requires_grad_(True)
    bq = b.clone().requires_grad_(True)
    lr = hr @ Wq + bq
    lossr = ref.softmax_xent(lr, y)
    lossr.backward()
    assert (logits - lr).abs().max() < 2e-3
    assert abs(float(loss) / B - float(lossr)) < 1e-4
    assert int(corr) == int((lr.argmax(1) == y).sum())
    p = torch.softmax(lr.detach(), 1)
    p[torch.arange(B, device=dev), y] -= 1.0
    assert (dlog - p / B).abs().max() < 1e-5
    dW = torch.full((H, C), 7.0, device=dev)
    db = torch.full((C,), 7.0, device=dev)
    one = torch.ones(1, device=dev)
    dh = E.head_bwd(h.contiguous(), W, dlog, one, dW, db, False, False)      # overwrite: the 7s must be gone
    tol = 2e-2 if dtype == torch.bfloat16 else 1e-4
    assert (dW - h.float().t() @ dlog).abs().max() <= 1e-4 * max(1.0, float(dW.abs().max()))
    assert (db - dlog.sum(0)).abs().max() < 1e-5
    dh_ref = dlog @ W.t()
    assert (dh.float() - dh_ref).abs().max() <= tol * float(dh_ref.abs().max()) + 1e-7
    dW2, db2 = dW.clone(), db.clone()
    E.head_bwd(h.contiguous(), W, dlog, one, dW2, db2, True, True)           # accumulate
    assert (dW2 - 2 * dW).abs().max() <= 1e-4 * max(1.0, float(dW.abs().max())) and (db2 - 2 * db).abs().max() < 1e-5
    for bwd in (E.head_bwd, E.head_step_bwd):                                 # one flag per output: each overwrites or adds alone
        for acc_w, acc_b in ((False, True), (True, False)):
            dW3 = dW.clone() if acc_w else torch.full_like(dW, 7.0)
            db3 = db.clone() if acc_b else torch.full_like(db, 7.0)
            bwd(h.contiguous(), W, dlog, one, dW3, db3, acc_w, acc_b)
            assert (dW3 - (1 + acc_w) * dW).abs().max() <= 1e-4 * max(1.0, float(dW.abs().max())), (bwd, acc_w, acc_b)
            assert (db3 - (1 + acc_b) * db).abs().max() < 1e-5, (bwd, acc_w, acc_b)


@pytest.mark.parametrize("C", [10, 300])                  # the tensor-core head, and the CUDA-core logits + xent_rows
def test_head_edges_against_fp64(E, dev, C):
    """Integer-valued h and W, so the logits are exact in fp32 and the fp64 log_softmax is the reference: logits near +-80
    (the loss and dlogits stay finite), exact ties (``correct`` follows torch.argmax's first index), the label C - 1 in the
    padded last batch tile, and a dloss of 0.37 that scales dh, dW and db."""
    B, H = 200, 64
    g = torch.Generator().manual_seed(3)
    h = torch.randint(-1, 2, (B, H), generator=g).double()
    W = torch.randint(-3, 4, (H, C), generator=g).double()
    b = torch.zeros(C, dtype=torch.float64)
    b[0], b[1] = 80.0, -80.0
    W[0] = 0.0
    W[0, 3] = W[0, 7] = 4.0                               # classes 3 and 7 tie everywhere ...
    W[:, 7] = W[:, 3]
    b[7] = b[3]
    h[: B // 2, 0] = 40.0                                 # ... and win in the first half of the rows (+160)
    y = torch.randint(0, C, (B,), generator=g)
    y[: B // 4], y[B // 4: B // 2] = 3, 7
    y[B // 2: B // 2 + 8] = 1                             # labels at -80: a loss of about 160 per row
    y[-16:] = C - 1
    hd, Wd, bd, yd = h.to(dev, torch.bfloat16), W.float().to(dev), b.float().to(dev), y.to(dev)
    logits, dlog, loss, corr = E.head_fwd(hd, Wd, bd, yd)
    l64 = h @ W + b
    assert torch.equal(logits.double().cpu(), l64)
    logp = torch.log_softmax(l64, 1)
    nll = -logp.gather(1, y.view(-1, 1)).squeeze(1)
    assert torch.isfinite(loss).all() and torch.isfinite(dlog).all()
    assert abs(float(loss) - float(nll.sum())) <= 1e-5 * float(nll.sum())
    assert int(corr) == int((torch.argmax(l64, 1) == y).sum())
    assert int((torch.argmax(l64, 1)[: B // 2] == 3).sum()) == B // 2          # (the ties are real and argmax takes 3)
    d64 = (logp.exp() - torch.nn.functional.one_hot(y, C).double()) / B
    assert float((dlog.double().cpu() - d64).abs().max()) * B <= 1e-5
    dloss = 0.37
    dW = torch.full((H, C), 7.0, device=dev)
    db = torch.full((C,), 7.0, device=dev)
    dh = E.head_bwd(hd, Wd, dlog, torch.tensor([dloss], device=dev), dW, db, False, False)
    # the backward against fp64 products of the dlogits it is given: where the classes tie at logits near 160, fp32's
    # lse = max + log(sum) carries an absolute error of up to half an ulp of 160, so dlogits (checked above) sit up to
    # ~1e-5 relative from fp64, and dW[0, 3] = 0.37 x 40 x sum over 100 rows cancels to 0 in fp64 but not in that error
    dk = dlog.double().cpu()
    dh64, dW64, db64 = dloss * dk @ W.t(), dloss * h.t() @ dk, dloss * dk.sum(0)
    assert float((dh.double().cpu() - dh64).abs().max()) <= 2.0 ** -8 * float(dh64.abs().max())
    # fp32 sums of B terms that cancel: the worst-case bound (B + 2) u sum |terms|, element by element
    u = (B + 2) * 2.0 ** -24
    assert bool(((dW.double().cpu() - dW64).abs() <= u * dloss * (h.abs().t() @ dk.abs()) + 1e-30).all())
    assert bool(((db.double().cpu() - db64).abs() <= u * dloss * dk.abs().sum(0) + 1e-30).all())


N_HEADLINE = 1025 * 16384        # about the headline flat buffer (2 x 1024 LSTM + head): 16 grid-stride passes of the kernels


def _update_state(n, dev, seed):
    """fp32 p, m, v and a gradient with magnitudes from 1e-4 to 1; the last 64 elements (alignment padding) all zero."""
    gen = torch.Generator(device=dev).manual_seed(seed)
    scale = 10.0 ** (torch.rand(n, generator=gen, device=dev) * 4 - 4)
    p = torch.randn(n, generator=gen, device=dev) * 0.05
    g = torch.randn(n, generator=gen, device=dev) * scale
    m = torch.randn(n, generator=gen, device=dev) * scale * 0.3
    v = scale * scale * (0.5 + torch.rand(n, generator=gen, device=dev))
    for x in (p, g, m, v):
        x[-64:] = 0
    return p, g, m, v


def _flat_steps(E, dev, p, m, v, grads, kind, lr, t0=None, wd=0.0, gscale=1.0, wd_numel=-1):
    """One update per gradient of ``grads`` (in place on p, m, v), each against the fp64 update of the state before it
    (lstm_numerics.adam_update / sgd_update), element by element; the bf16 shadow bit for bit, the zero padding (the last 64
    elements) left at 0.  Adam: ``t0`` None = the host's lr_t of steps 1, 2, ...; else the bias correction from step_dev,
    preset to ``t0`` - 1 as a resumed run's.  -> the worst update ratio."""
    import lstm_numerics as N
    sh = torch.empty_like(p, dtype=torch.bfloat16)
    step_dev = None if t0 is None else torch.full((1,), t0 - 1, dtype=torch.int32, device=dev)
    worst = 0.0
    for k, g in enumerate(grads):
        p0, m0, v0 = p.clone(), m.clone(), v.clone()
        if kind == "sgd":
            E.flat_sgd(p, g, sh, lr, wd, gscale, wd_numel)
            ref = N.sgd_update(p0, g, lr, wd, gscale, wd_numel)
        elif t0 is None:
            t = k + 1
            lr_t = lr * (1 - 0.999 ** t) ** 0.5 / (1 - 0.9 ** t)
            E.flat_adam(p, g, m, v, sh, lr_t, 0.9, 0.999, 1e-8, wd, gscale, None, wd_numel)
            ref = N.adam_update(p0, m0, v0, g, None, lr_t, wd=wd, grad_scale=gscale, wd_numel=wd_numel)
        else:
            E.flat_adam(p, g, m, v, sh, lr, 0.9, 0.999, 1e-8, wd, gscale, step_dev, wd_numel)
            assert int(step_dev) == t0 + k
            ref = N.adam_update(p0, m0, v0, g, t0 + k, lr, wd=wd, grad_scale=gscale, wd_numel=wd_numel)
        worst = max(worst, N.check_update(f"step {k} p", p, ref.p, ref.bound_p))
        if kind == "adam":
            worst = max(worst, N.check_update(f"step {k} m", m, ref.m, ref.bound_m),
                        N.check_update(f"step {k} v", v, ref.v, ref.bound_v))
        N.check_shadow(f"step {k}", sh, p)
        assert not bool(p[-64:].any() or m[-64:].any() or v[-64:].any())
    return worst


def test_flat_adam_and_sgd(E, dev):
    """Three Adam steps with the host's lr_t and a gradient scale of 0.5 from zero moments, then SGD without and with weight
    decay over the first 4096 elements, against the fp64 update."""
    torch.manual_seed(0)
    n = 16384
    p = torch.randn(n, device=dev); g = torch.randn(n, device=dev)
    p[-64:] = 0; g[-64:] = 0
    m = torch.zeros(n, device=dev); v = torch.zeros(n, device=dev)
    _flat_steps(E, dev, p, m, v, [g] * 3, "adam", 1e-3, gscale=0.5)
    _flat_steps(E, dev, p, m, v, [g], "sgd", 0.1)
    _flat_steps(E, dev, p, m, v, [g], "sgd", 0.1, wd=0.5, wd_numel=4096)


@pytest.mark.parametrize("wd,gscale", [(0.0, 1.0), (0.1, 0.37)], ids=["plain", "wd-gscale"])
@pytest.mark.parametrize("kind,t0", [("adam", None), ("adam", 1), ("adam", 2), ("adam", 1000), ("adam", 100000), ("sgd", None)],
                         ids=["adam-host-lr_t", "adam-t1", "adam-t2", "adam-t1000", "adam-t100000", "sgd"])
@pytest.mark.parametrize("n", [16384, N_HEADLINE])
def test_flat_update_kernels_against_fp64(E, dev, n, kind, t0, wd, gscale):
    """Two consecutive updates over the flat buffer against the fp64 update: one grid-stride pass or about the headline's 16,
    Adam with the host's lr_t or its bias correction from step_dev (preset as a resumed run's), SGD, weight decay over
    [0, wd_numel) with wd_numel inside a grid-stride pass, a gradient scale."""
    p, g, m, v = _update_state(n, dev, seed=n % 1000 + (t0 or 0))
    g2 = g.roll(4096)                                                        # the second step's gradient
    g2[-64:] = 0
    wd_numel = (n * 3 // 4) // 64 * 64 + 20
    worst = _flat_steps(E, dev, p, m, v, [g, g2], kind, 0.05 if kind == "sgd" else 1e-3, t0, wd, gscale, wd_numel)
    print(f"\nflat {kind} n={n} t0={t0} wd={wd}: worst update ratio {worst:.3f}")


@pytest.mark.parametrize("ctas,bn", [(1, 128), (2, 256)])
@pytest.mark.parametrize("Bsz,T,F", [(128, 3, 128), (256, 5, 256), (384, 2, 512)])
def test_tcgen05_gemm2_folded_batch_major_operand(E, dev, ctas, bn, Bsz, T, F):
    """A batch-major [B,T,F] array read in place as the time-major matrix X = [T*B, F] (folded tensor map): X @ W^T (the
    x-projection) and dG^T @ X (the weight gradient of the first layer) against the same products over a transposed copy."""
    torch.manual_seed(1)
    x_bm = (torch.randn(Bsz, T, F, device=dev) * 0.5).bfloat16()
    X = x_bm.transpose(0, 1).reshape(T * Bsz, F)                      # time-major copy
    store = x_bm.view(Bsz, T * F)
    W = (torch.randn(520, F, device=dev) * 0.5).bfloat16()
    R = X.float() @ W.float().t()
    C = E.gemm2(store, W, out_fp32=True, ctas=ctas, bn=bn, a_fold=Bsz, fold_cols=F)
    assert C.shape == R.shape and (C - R).abs().max() / float(R.abs().max()) < 2e-3
    if F % bn:
        return                                                        # a folded B operand needs N % bn == 0
    dG = (torch.randn(T * Bsz, 384, device=dev) * 0.5).bfloat16()     # dW = dG^T @ X: A = dG^T (MN-major), B = X (MN-major, folded)
    R2 = dG.float().t() @ X.float()
    acc = torch.full((384, F), 2.0, device=dev)
    E.gemm2(dG, store, out=acc, a_mn=True, b_mn=True, accumulate=True, ctas=ctas, bn=bn, b_fold=Bsz, fold_cols=F)
    assert (acc - 2.0 - R2).abs().max() / float(R2.abs().max()) < 2e-3
    from lstm_tensorspark_b200.ops import cuda_gemm as G
    if G.folded_ok(x_bm):
        assert torch.equal(G.matmul(None, W, a_folded=x_bm), G.matmul(X, W))
        assert torch.equal(G.matmul(dG.t(), None, b_folded=x_bm, out_dtype=torch.float32), G.matmul(dG.t(), X.t(), out_dtype=torch.float32))


@pytest.mark.parametrize("M,N,K,dt", [(10, 64, 4, torch.float32), (33, 20, 48, torch.bfloat16), (150, 3, 16, torch.float32), (64, 4, 650, torch.bfloat16)])
def test_generic_gemm_and_dispatch(E, dev, M, N, K, dt):
    """CUDA-core GEMM for the shapes the tensor-core kernels cannot take (the reference's iris configuration)."""
    from lstm_tensorspark_b200.ops import cuda_gemm as G
    torch.manual_seed(0)
    a = torch.randn(M, K, device=dev).to(dt)
    b = torch.randn(K, N, device=dev).to(dt)
    R = a.float() @ b.float()
    tol = 1e-5 if dt == torch.float32 else 2e-2
    C = G.matmul(a, b.t(), out_dtype=torch.float32)
    assert (C - R).abs().max() <= 1e-5 * max(1.0, float(R.abs().max()))
    Ct = G.matmul(a.t().contiguous().t(), b.t().contiguous(), out_dtype=dt)           # other stride patterns
    assert (Ct.float() - R).abs().max() <= tol * max(1.0, float(R.abs().max()))
    acc = torch.ones(M, N, device=dev)
    G.matmul(a, b.t(), out=acc, accumulate=True)
    assert (acc - 1 - R).abs().max() <= 1e-5 * max(1.0, float(R.abs().max()))


def _seq_case(dev, T, B, H, D, tol, loss_on="seq"):
    from lstm_tensorspark_b200.ops import cuda_lstm
    ref = _ref()
    torch.manual_seed(1)
    params = [torch.randn(T, B, D, device=dev) * 0.5, torch.randn(B, H, device=dev) * 0.1, torch.randn(B, H, device=dev) * 0.1,
              torch.randn(4 * H, D, device=dev) / D ** 0.5, torch.randn(4 * H, H, device=dev) / H ** 0.5,
              torch.randn(4 * H, device=dev) * 0.1]
    pr = [p.bfloat16().float().requires_grad_(True) if i != 2 else p.clone().requires_grad_(True) for i, p in enumerate(params)]
    hs_r, hT_r, cT_r = ref.lstm_layer_sequence(*pr)
    wgt, w2, w3 = torch.randn_like(hs_r), torch.randn_like(hT_r), torch.randn_like(cT_r)

    def loss(hs, hT, cT):
        if loss_on == "last":            # only the final state is used downstream (top layer under the classifier): dh_seq is None
            return (hT.float() * w2).sum()
        if loss_on == "all":
            return (hs.float() * wgt).sum() + (hT.float() * w2).sum() + (cT.float() * w3).sum()
        return (hs.float() * wgt).sum()
    loss(hs_r, hT_r, cT_r).backward()
    pc = [p.clone().requires_grad_(True) for p in params]
    hs, hT, cT = cuda_lstm.lstm_layer_sequence(pc[0].bfloat16(), pc[1], pc[2], pc[3], pc[4], pc[5])
    loss(hs, hT, cT).backward()
    torch.cuda.synchronize()
    cuda_lstm.check_kernel_errors(dev)
    assert (hs.float() - hs_r).abs().max() < tol
    assert (cT - cT_r).abs().max() < tol
    def rel_l2(a, b):
        return float((a.float() - b.float()).norm() / (b.float().norm() + 1e-20))
    assert rel_l2(hs, hs_r) < 1e-2 and rel_l2(cT, cT_r) < 1e-2
    for a, b in zip(pc, pr):
        assert rel_l2(a.grad, b.grad) < 2e-2, (tuple(b.shape), rel_l2(a.grad, b.grad))


@pytest.mark.parametrize("T,B,H,D", [(1, 128, 64, 64), (1, 96, 128, 40), (2, 256, 256, 64), (3, 128, 64, 64), (5, 100, 128, 72),
                                     (4, 256, 256, 128), (8, 256, 1024, 1024), (3, 64, 2048, 256), (3, 64, 1280, 256)])
# last two: streamed-weights variant (the weight slice does not fit next to the ring; the backward runs in clusters of 2)
def test_persistent_tcgen05_lstm_sequence(dev, T, B, H, D):
    from lstm_tensorspark_b200.ops import cuda_lstm
    n0 = cuda_lstm.STATS["fast_fwd"], cuda_lstm.STATS["fast_bwd"]
    _seq_case(dev, T, B, H, D, tol=3e-2)
    assert cuda_lstm.STATS["fast_fwd"] == n0[0] + 1 and cuda_lstm.STATS["fast_bwd"] == n0[1] + 1   # the persistent kernels ran


def test_colsum_bf16(dev):
    from lstm_tensorspark_b200.ops.cuda_ext import ext
    for (R, C) in ((1000, 256), (32768, 4096), (7, 512)):
        x = (torch.randn(R, C, device=dev) * 0.3).bfloat16()
        ref = x.float().sum(0)
        got = ext().colsum_bf16(x)
        assert (got - ref).abs().max() <= 1e-3 * max(1.0, float(ref.abs().max()))


def test_transpose2d(dev):
    from lstm_tensorspark_b200.ops.cuda_ext import ext
    for (R, C) in ((4096, 1024), (1024, 4096), (100, 36), (65, 129)):
        x = torch.randn(R, C, device=dev).bfloat16()
        assert torch.equal(ext().transpose2d(x), x.t().contiguous())


def test_transpose01_rows(dev):
    from lstm_tensorspark_b200.ops.cuda_ext import ext
    for (B, T, D, dt) in ((7, 5, 24, torch.bfloat16), (64, 33, 1024, torch.bfloat16), (3, 4, 8, torch.float32)):
        x = torch.randn(B, T, D, device=dev).to(dt)
        y = ext().transpose01(x)
        assert y.shape == (T, B, D) and torch.equal(y, x.transpose(0, 1).contiguous())


@pytest.mark.parametrize("loss_on", ["last", "all"])
def test_persistent_lstm_final_state_gradients(dev, loss_on):
    _seq_case(dev, 6, 200, 256, 128, tol=3e-2, loss_on=loss_on)
    _seq_case(dev, 4, 20, 32, 16, tol=3e-2, loss_on=loss_on)          # generic path


def test_large_batch_runs_the_fast_path_in_chunks(dev):
    """B = 400, H = 1024 needs 4 batch tiles x 64 CTAs, more than an H100 holds even at two tiles per CTA: two chunks of the
    persistent kernels, not the generic path."""
    from lstm_tensorspark_b200.ops import cuda_lstm
    n0 = cuda_lstm.STATS["fast_fwd"], cuda_lstm.STATS["generic_fwd"]
    _seq_case(dev, 4, 400, 1024, 256, tol=3e-2, loss_on="all")
    assert cuda_lstm.STATS["fast_fwd"] == n0[0] + 2 and cuda_lstm.STATS["generic_fwd"] == n0[1]


@pytest.mark.parametrize("T,B,H,D", [(1, 10, 16, 4), (6, 33, 48, 20)])
def test_generic_shape_lstm_sequence(dev, T, B, H, D):
    from lstm_tensorspark_b200.ops import cuda_lstm
    n0 = cuda_lstm.STATS["generic_fwd"]
    _seq_case(dev, T, B, H, D, tol=3e-2)
    assert cuda_lstm.STATS["generic_fwd"] == n0 + 1


def test_single_step_cell_uses_the_persistent_kernels(dev):
    """The reference applies every layer for exactly ONE time step (fit_next on [B,D]); on the GPU that is the T = 1 case of
    the same persistent kernels."""
    from lstm_tensorspark_b200.ops import cuda_lstm, functional as F
    ref = _ref()
    torch.manual_seed(3)
    B, D, H = 128, 64, 128
    x = torch.randn(B, D, device=dev) * 0.5
    h = torch.randn(B, H, device=dev) * 0.1
    c = torch.randn(B, H, device=dev) * 0.1
    w_x = (torch.randn(4 * H, D, device=dev) / D ** 0.5).requires_grad_(True)
    w_h = (torch.randn(4 * H, H, device=dev) / H ** 0.5).requires_grad_(True)
    b = (torch.randn(4 * H, device=dev) * 0.1).requires_grad_(True)
    n0 = cuda_lstm.STATS["fast_fwd"]
    F.set_backend("cuda_ext")
    try:
        h1, c1 = F.lstm_cell_step(x.bfloat16(), h, c, w_x, w_h, b)
    finally:
        F.set_backend("auto")
    assert cuda_lstm.STATS["fast_fwd"] == n0 + 1
    hr, cr = ref.lstm_cell_step(x.bfloat16().float(), h, c, w_x.detach().bfloat16().float(), w_h.detach().bfloat16().float(), b.detach())
    assert (h1.float() - hr).abs().max() < 3e-2 and (c1.float() - cr).abs().max() < 3e-2
    (h1.float().sum() + c1.float().sum()).backward()
    assert w_x.grad is not None and w_h.grad is not None and torch.isfinite(w_h.grad).all()
    cuda_lstm.check_kernel_errors(dev)


def test_engine_step_trains_and_uses_kernels(dev):
    import __graft_entry__ as g
    g.smoke()


def test_fp32_iris_shape_on_gpu(dev):
    """Reference-shaped model (T=1, learned initial state, fp32) on the GPU path vs the CPU reference path."""
    from lstm_tensorspark_b200.config import Config
    from lstm_tensorspark_b200.models import SequenceClassifier
    from lstm_tensorspark_b200.ops import functional as F
    cfg = Config(hidden_units="16", in_features=4, batch_size=10)
    g = torch.Generator().manual_seed(0)
    m_cpu = SequenceClassifier(cfg, batch_size=10, generator=g); m_cpu.build_flat()
    g = torch.Generator().manual_seed(0)
    m_gpu = SequenceClassifier(cfg, batch_size=10, generator=g); m_gpu.to(dev); m_gpu.build_flat()
    x = torch.randn(10, 4); y = torch.randint(0, 3, (10,))
    l_cpu, _, _ = m_cpu(x, y); l_cpu.backward()
    l_gpu, _, _ = m_gpu(x.to(dev), y.to(dev)); l_gpu.backward()
    assert abs(float(l_cpu) - float(l_gpu)) < 1e-4
    assert (m_cpu.flat.grad - m_gpu.flat.grad.cpu()).abs().max() < 1e-4
