"""How the CUDA ops find a parameter's bf16 operand and where its gradient goes (``ops/params.py``), on CPU tensors registered
the way ``FlatParams`` registers its CUDA views: a fresh tensor returned to autograd, or the flat buffer's grad view written in
place (overwrite on the first write of a step, accumulate afterwards)."""
import gc

import pytest
import torch

from lstm_tensorspark_b200.models.flat import FlatParams
from lstm_tensorspark_b200.ops import params


@pytest.fixture(autouse=True)
def _registry(monkeypatch):
    monkeypatch.setattr(params, "_PARAMS", {})


def _registered(direct_bias: bool):
    """A flat buffer holding ``w [8,4]`` (direct) and ``b [4]`` (direct or not), both registered, grads at 7 before zero_grad."""
    w, b = torch.nn.Parameter(torch.randn(8, 4)), torch.nn.Parameter(torch.randn(4))
    flat = FlatParams([w], [b])
    shadow = flat.ensure_shadow()
    for p, o in zip(flat.params, flat.offsets):
        params.register_param(p.data_ptr(), shadow[o:o + p.numel()].view(p.shape), p.grad, owner=flat)
    flat.enable_direct_grads([w, b] if direct_bias else [w])
    flat.grad.fill_(7.0)
    flat.zero_grad()
    return flat, w, b


def test_unregistered_parameter_gets_a_fresh_tensor_returned_to_autograd():
    w = torch.randn(8, 4)
    out, acc, ret = params.grad_out(w.data_ptr(), (8, 4), w.device)
    assert out.shape == (8, 4) and out.dtype == torch.float32 and out.data_ptr() != w.data_ptr()
    assert acc is False and ret is out


def test_direct_parameter_overwrites_first_then_accumulates():
    flat, w, b = _registered(direct_bias=True)
    out, acc, ret = params.grad_out(w.data_ptr(), w.shape, w.device)
    assert out.data_ptr() == w.grad.data_ptr() and out.shape == w.shape
    assert acc is False and ret is None                  # first write of the step: the stale 7s need no memset
    assert float(w.grad.min()) == 7.0
    out2, acc2, ret2 = params.grad_out(w.data_ptr(), w.shape, w.device)
    assert out2.data_ptr() == out.data_ptr() and acc2 is True and ret2 is None
    _, acc_b, ret_b = params.grad_out(b.data_ptr(), b.shape, b.device)
    assert acc_b is False and ret_b is None              # each parameter has its own first write


def test_registered_parameter_that_is_not_direct_is_zeroed_on_demand_and_accumulated():
    flat, w, b = _registered(direct_bias=False)
    assert float(b.grad.abs().max()) == 0.0              # zero_grad zeroes what is not written directly
    b.grad.fill_(7.0)
    flat._stale.add(b.data_ptr())                        # a gradient from the last step, not yet zeroed
    out, acc, ret = params.grad_out(b.data_ptr(), b.shape, b.device)
    assert out.data_ptr() == b.grad.data_ptr() and acc is True and ret is None
    assert float(b.grad.abs().max()) == 0.0 and b.data_ptr() not in flat._stale
    b.grad.fill_(3.0)
    out, acc, ret = params.grad_out(b.data_ptr(), b.shape, b.device)
    assert acc is True and ret is None and float(b.grad.min()) == 3.0      # zeroed once, then accumulated into


def test_dead_owner_counts_as_unregistered():
    flat, w, b = _registered(direct_bias=True)
    addr = w.data_ptr()
    del flat
    gc.collect()
    out, acc, ret = params.grad_out(addr, w.shape, w.device)
    assert out.data_ptr() != w.grad.data_ptr() and acc is False and ret is out
    assert addr not in params._PARAMS                    # the stale entry is dropped: its address may be reused


def test_lowp_returns_the_shadow_only_for_a_matching_shape():
    flat, w, b = _registered(direct_bias=True)
    wb = params.lowp(w, torch.bfloat16)
    assert wb is params._PARAMS[w.data_ptr()][0] and wb.dtype == torch.bfloat16 and wb.shape == w.shape
    flat.shadow.zero_()                                  # the shadow is what is read, not a fresh cast of the fp32 weights
    assert float(wb.abs().max()) == 0.0 and float(params.lowp(w, torch.bfloat16).abs().max()) == 0.0
    flat_w = w.detach().view(-1)                         # the same address, another shape: a cast
    cast = params.lowp(flat_w, torch.bfloat16)
    assert cast.shape == flat_w.shape and torch.equal(cast, flat_w.bfloat16())
    assert torch.equal(params.lowp(w, torch.float32), w.detach())          # no shadow for other dtypes
    u = torch.randn(3, 5)
    assert torch.equal(params.lowp(u, torch.bfloat16), u.bfloat16())       # unregistered: a cast
