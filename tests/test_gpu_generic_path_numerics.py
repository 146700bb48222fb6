"""The generic LSTM path against fp64: the CUDA-core GEMM per time step (csrc/gemm_generic.cu) and the fused cell kernels
(csrc/lstm_pointwise.cu) that ops/cuda_lstm._LSTMSeqFn runs when ``fast_path_supported`` is false - every layer of a
``--dtype fp32`` model, and every bf16 layer with H % 64 != 0.

  a  the fp32 cell kernels' activations, element by element: within 2 ulp of the fp64 value rounded to fp32;
  b  the fp32 layer op against fp64 within the budget of the lstm_numerics.Fp32 arm (floor FLOOR_F32), per time step for
     h_seq and dx, per tensor for the rest;
  c  the bf16 layer op against fp64 within the budget of the lstm_numerics.Generic arm (floor FLOOR);
  d  an fp32 layer with T·B above the GEMM's former grid limit of 2,097,120 rows;
  e  whole ``--dtype fp32`` training steps (loss, every gradient of the flat buffer, the Adam update) against the fp64 model;
  f  whole bf16 training steps on the generic path.
Every case asserts the path it targets through cuda_lstm.STATS (and cuda_gemm.STATS["tc"] where the backward products move
onto the tensor cores); `-s` prints each case's worst budget ratio."""
import pytest
import torch

import lstm_numerics as N
import test_gpu_model_numerics as M

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
PER_STEP = ("h_seq", "dx")


@pytest.fixture(autouse=True)
def _fp32_matmuls(monkeypatch):
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)     # the reference arms' fp32 products stay fp32


def _stats():
    from lstm_tensorspark_b200.ops import cuda_gemm, cuda_lstm
    out = {k: cuda_lstm.STATS.get(k, 0) for k in ("fast_fwd", "fast_bwd", "generic_fwd", "generic_bwd", "batch_chunks")}
    out["tc"] = cuda_gemm.STATS["tc"]
    return out


# ---- a: the activations -------------------------------------------------------------------------------------------------------
def _ordered(x):
    """fp32 bit patterns as integers in the order of the values (-0 and +0 both 0): the ulp distance is a difference."""
    b = x.contiguous().view(torch.int32).long()
    return torch.where(b < 0, -(b & 0x7FFFFFFF), b)


def _check_ulp(name, got, want64, ulp=2, tiny=2.0 ** -126):
    """|got - fp32(want64)| <= ``ulp`` ulp, element by element; a result the kernel flushed to zero below ``tiny`` is allowed."""
    want = want64.float()
    d = (_ordered(got) - _ordered(want)).abs()
    flushed = (got == 0) & (want64.abs() < tiny)
    bad = (d > ulp) & ~flushed
    if bool(bad.any()):
        i = int(bad.nonzero()[0])
        raise AssertionError(f"{name}: {int(bad.sum())} of {got.numel()} values more than {ulp} ulp off; first: {float(got[i]):.9e} "
                             f"vs {float(want[i]):.9e} ({int(d[i])} ulp)")
    return int(torch.where(flushed, 0, d).max())


def _grid():
    """About 2^20 values over [-30, 30], and +-0, tiny, subnormal, huge and overflowing inputs."""
    dense = torch.linspace(-30.0, 30.0, (1 << 20) + 1, dtype=torch.float64).float()
    edges = [0.0, -0.0, 1e-45, -1e-45, 2.0 ** -126, -(2.0 ** -126), 1e-30, -1e-30, 1e-8, -1e-8, 2.0 ** -24, 0.5, -0.5, 9.0, -9.0,
             15.0, -15.0, 44.0, -44.0, 87.0, -87.0, 89.0, -89.0, 104.0, -104.0, 1e4, -1e4, 1e30, -1e30, 3.4e38, -3.4e38]
    return torch.cat([dense, torch.tensor(edges)]).to(DEV)


def test_fp32_forward_activations_within_2_ulp():
    """pre = x in every gate, zero bias and c_prev = 0: act holds sigmoid(x), sigmoid(x), tanh(x), sigmoid(x); c = i g and
    h = o tanh(c) are checked against the kernel's own i, g and o."""
    from lstm_tensorspark_b200.ops.cuda_ext import ext
    x = _grid()
    n = x.numel()
    pre = x.view(n, 1).expand(n, 4).contiguous()                  # B = n rows, H = 1
    h, c, act = ext().lstm_pointwise_fwd(pre, torch.zeros(4, device=DEV), torch.zeros(n, 1, device=DEV))
    torch.cuda.synchronize()
    x64 = x.double()
    worst = {}
    for k, name in ((0, "i"), (1, "f"), (3, "o")):
        worst[name] = _check_ulp(f"sigmoid ({name})", act[:, k], torch.sigmoid(x64))
    worst["g"] = _check_ulp("tanh (g)", act[:, 2], torch.tanh(x64))
    i, g, o = act[:, 0].double(), act[:, 2].double(), act[:, 3].double()
    worst["c"] = _check_ulp("c = i g", c[:, 0], i * g, ulp=1)
    worst["h"] = _check_ulp("h = o tanh(c)", h[:, 0], o * torch.tanh(c[:, 0].double()))
    print(f"\nfp32 activations: worst ulp " + ", ".join(f"{k} {v}" for k, v in worst.items()))


def test_fp32_backward_tanh_within_2_ulp():
    """The backward's tanh(c_new), read through dpre: with dh = 1, no dc, o = 1/2 the output gate's gradient is
    dh tanh(c) o (1 - o) = tanh(c) / 4, exact up to the tanh (and the flush to zero of a subnormal quarter)."""
    from lstm_tensorspark_b200.ops.cuda_ext import ext
    cn = _grid()
    n = cn.numel()
    act = torch.tensor([0.25, 0.75, 0.5, 0.5], device=DEV).repeat(n, 1)          # i, f, g, o
    dp, dc = ext().lstm_pointwise_bwd(None, torch.ones(n, 1, device=DEV), None, act, torch.zeros(n, 1, device=DEV), cn.view(n, 1))
    torch.cuda.synchronize()
    # (tanh(c) / 4 below 2^-126 is flushed to zero)
    worst = _check_ulp("tanh(c_new) in the backward", dp[:, 3] * 4, torch.tanh(cn.double()), tiny=2.0 ** -124)
    print(f"\nfp32 backward tanh: worst ulp {worst}")


# ---- b, c, d: the layer op ----------------------------------------------------------------------------------------------------
def _inputs(T, B, H, D, dtype, seed):
    """x, h0, W_x, W_h in ``dtype``'s values (bf16: bf16-representable; fp32: any fp32), fp32 c0 and bias; loss weights on h_seq
    and h_T that the op receives exactly, an fp32 one on c_T."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    rn = lambda *s: torch.randn(*s, generator=g, device=DEV)
    v = lambda t: t.to(dtype).float()
    params = [v(rn(T, B, D) * 0.5), v(rn(B, H) * 0.1), rn(B, H) * 0.1, v(rn(4 * H, D) / D ** 0.5), v(rn(4 * H, H) / H ** 0.5),
              rn(4 * H) * 0.1]
    return params, (v(rn(T, B, H)), v(rn(B, H)), rn(B, H))


def _lengths(T, B, seed):
    g = torch.Generator().manual_seed(seed)
    lengths = torch.randint(1, T + 1, (B,), generator=g, dtype=torch.int32)
    lengths[0], lengths[-1] = 1, T
    return lengths.to(DEV)


def _layer_case(case, T, B, H, D, dtype, lengths=None, reverse=False, dropout=0.0, weight_drop=0.0, loss="all", tc=None, seed=5):
    """The layer op (ops.cuda_lstm.lstm_layer_sequence) against fp64 within the budget of the generic path's arm.  ``dropout``:
    P of the output dropout (its mask and the incoming gradient's); ``weight_drop``: P of the mask on W_h.  ``loss``: "all" (h_seq,
    h_T and c_T) or "h_T" (no gradient into h_seq or c_T).  ``tc``: whether some backward product must run on the tensor cores."""
    from lstm_tensorspark_b200.ops import cuda_lstm
    from lstm_tensorspark_b200.ops import reference as ref
    from test_gpu_weight_drop import _masked_grad
    assert not cuda_lstm.fast_path_supported(B, H, dtype, DEV)
    params, (dh_seq, dh_T, dc_T) = _inputs(T, B, H, D, dtype, seed)
    if loss == "h_T":
        dh_seq = dc_T = None
    dspec = ref.DropoutSpec(dropout, (11, 3), 0, reverse, 7) if dropout else None
    wspec = ref.DropoutSpec(weight_drop, (11, 3), 0, reverse, 7, weight=True) if weight_drop else None
    x = params[0].to(dtype).requires_grad_(True)
    leaves = [p.clone().requires_grad_(True) for p in params[1:]]
    n0 = _stats()
    hs, hT, cT = cuda_lstm.lstm_layer_sequence(x, *leaves, lengths=lengths, reverse=reverse, dropout=dspec, weight_drop=wspec)
    obj = (hT.float() * dh_T).sum()
    if loss == "all":
        obj = obj + (hs.float() * dh_seq).sum() + (cT * dc_T).sum()
    obj.backward()
    torch.cuda.synchronize()
    delta = {k: v - n0[k] for k, v in _stats().items()}
    assert {k: v for k, v in delta.items() if k != "tc"} == {"fast_fwd": 0, "fast_bwd": 0, "generic_fwd": 1, "generic_bwd": 1,
                                                             "batch_chunks": 0}, delta
    if tc is not None:
        assert (delta["tc"] > 0) == tc, delta
    got = N.LayerOut(hs, hT, cT, x.grad, *[p.grad for p in leaves])
    arm = N.Fp32() if dtype == torch.float32 else N.Generic()
    floor = N.FLOOR_F32 if dtype == torch.float32 else N.FLOOR
    keep = N._keep(lengths, T, B, DEV)
    with torch.no_grad():
        arms = {}
        for name, dt, r in (("fp64", torch.float64, None), ("emu", torch.float32, arm)):
            x_, h0, c0, w_x, w_h, bias = [p.to(dt) for p in params]
            if wspec is not None:
                w_h = ref.weight_drop(params[4].to(dtype), wspec).to(dt)
            sc = N._drop_scale(N.Dropout(dropout, (11, 3), 7), 0, reverse, T, B, H, dt, DEV) if dropout else None
            fw = N._forward(x_, h0, c0, w_x, w_h, bias, keep, reverse, r, None)
            h_seq, h_T, c_T = N._state_out(fw, reverse)
            if sc is not None:
                h_seq = N._round(r, h_seq * sc)
            d = lambda t: None if t is None else t.to(dt)
            back = N._backward(fw, x_, w_x, w_h, d(dh_seq), d(dh_T), d(dc_T), keep, reverse, r, None, dh_scale=sc)
            out = N.LayerOut(h_seq, h_T, c_T, *back)
            if wspec is not None:
                out = out._replace(dw_h=_masked_grad(out.dw_h, wspec))
            arms[name] = out
        ratios = {n: N.check_budget(f"{case} {n}", getattr(got, n), getattr(arms["fp64"], n), getattr(arms["emu"], n),
                                    per_step=n in PER_STEP, floor=floor) for n in N.LayerOut._fields}
    print(f"\n{case}: worst budget ratio {max(ratios.values()):.3f} (" + ", ".join(f"{n} {r:.3f}" for n, r in ratios.items()) +
          f"); alpha {N.ALPHA}, floor {floor:.2e}")


F32 = torch.float32
BF16 = torch.bfloat16


def test_fp32_iris():
    """The reference's own iris configuration in fp32: one step, B = 10, H = 16, D = 4."""
    _layer_case("fp32 iris", 1, 10, 16, 4, F32)


def test_fp32_masked():
    _layer_case("fp32 masked", 64, 33, 48, 20, F32, lengths=_lengths(64, 33, 1))


def test_fp32_long_masked_reverse():
    """T = 256, B = 130 (a partial 32-row GEMM tile), masked reverse."""
    _layer_case("fp32 long masked reverse", 256, 130, 96, 40, F32, lengths=_lengths(256, 130, 2), reverse=True)


def test_fp32_dropout_reverse():
    _layer_case("fp32 dropout reverse", 128, 7, 200, 64, F32, dropout=0.3, reverse=True)


def test_fp32_weight_drop():
    _layer_case("fp32 weight drop", 64, 33, 48, 20, F32, weight_drop=0.5, lengths=_lengths(64, 33, 3))


@pytest.mark.parametrize("loss", ["h_T", "all"])
def test_fp32_loss_on(loss):
    """A loss on h_T alone (no gradient into h_seq or c_T arrives: dh_seq is None) and on all three outputs."""
    _layer_case(f"fp32 loss on {loss}", 96, 24, 40, 16, F32, loss=loss)


def test_bf16_generic_h48():
    """B = 33: the recurrence's products on gemm_generic; dW_h ([4H, T·B] x [T·B, H], all sides multiples of 8) on the tensor
    cores."""
    _layer_case("bf16 generic H=48", 64, 33, 48, 20, BF16, tc=True)


def test_bf16_generic_h100_masked():
    """H = 100 and D = 20: no side of a product with H or D in it is a multiple of 8, so every product runs on gemm_generic."""
    _layer_case("bf16 generic H=100", 128, 40, 100, 20, BF16, lengths=_lengths(128, 40, 4), tc=False)


def test_bf16_generic_h96_b256():
    """B = 256: the backward's dG W_h and the weight gradients run on the tensor-core GEMM, the forward on gemm_generic."""
    _layer_case("bf16 generic H=96 B=256", 128, 256, 96, 64, BF16, tc=True)


def test_bf16_generic_h200_b256_long_masked_reverse():
    _layer_case("bf16 generic H=200 B=256 masked reverse", 256, 256, 200, 64, BF16, lengths=_lengths(256, 256, 5), reverse=True,
                tc=True)


def test_bf16_generic_dropout_reverse():
    _layer_case("bf16 generic dropout reverse", 128, 33, 48, 20, BF16, dropout=0.3, reverse=True)


def test_bf16_generic_weight_drop():
    _layer_case("bf16 generic weight drop", 64, 256, 96, 64, BF16, weight_drop=0.5, lengths=_lengths(64, 256, 6), tc=True)


def test_fp32_beyond_the_old_grid_limit():
    """T = 2, B = 1,048,577: the gx and dx products have T·B = 2,097,154 rows, more 32-row GEMM tiles than grid y could hold."""
    _layer_case("fp32 T*B = 2097154", 2, 1048577, 16, 4, F32)


# ---- e, f: whole training steps -----------------------------------------------------------------------------------------------
GENERIC2 = {"generic_fwd": 2, "generic_bwd": 2}


@pytest.mark.parametrize("case,kw", [
    ("lengths", dict(lengths_seed=31)),
    ("bidirectional", dict(bidirectional=True, lengths_seed=41)),
    ("dropout", dict(dropout=0.2)),
    ("weight drop", dict(weight_drop=0.5)),
])
def test_fp32_training_steps(case, kw):
    """``--dtype fp32``, hidden 48,48, three Adam steps at lr 1e-3: the weights move off any bf16 grid, and the reference reads
    the fp32 master."""
    per = {k: v * (2 if kw.get("bidirectional") else 1) for k, v in GENERIC2.items()}
    M._model_case(f"fp32 steps {case}", "48,48", 32, 20, 12, per, dtype=torch.float32, learning_rate=1e-3, **kw)


def test_fp32_training_steps_attention_pooling():
    import test_gpu_pooling as P
    P._case("fp32 steps attention pooling", "attention", "48,48", 32, 20, 12, "generic_fwd", lengths_seed=51, A=24,
            dtype=torch.float32)


def test_bf16_generic_training_steps():
    """bf16, hidden 96,160 (neither a multiple of 64) with lengths: both layers on the generic path, the Generic arm."""
    M._model_case("bf16 generic steps", "96,160", 32, 64, 32, GENERIC2, lengths_seed=61, rounding=N.Generic())
