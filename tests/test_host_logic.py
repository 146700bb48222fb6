"""Host-side logic of the GPU path that does not need a GPU: lazy gradient zeroing, ownership of Adam slots under bucketed
two-shot allreduce, the wavefront GEMM's gate configuration, the generation-gated bucket queue and the release of parameters
to the gradient buckets."""
import types

import pytest
import torch

from lstm_tensorspark_b200.models.flat import FlatParams


def _flat():
    ps = [torch.nn.Parameter(torch.randn(8, 4)), torch.nn.Parameter(torch.randn(8, 8)), torch.nn.Parameter(torch.randn(8))]
    other = [torch.nn.Parameter(torch.randn(8, 3))]
    return FlatParams(ps, other), ps, other


def test_lazy_gradient_zeroing_protocol():
    flat, ps, other = _flat()
    flat.grad.fill_(7.0)
    flat.enable_direct_grads(ps)                       # w_x, w_h, bias are written by kernels; `other` goes through autograd
    flat.zero_grad()
    assert float(other[0].grad.abs().sum()) == 0.0     # autograd-accumulated parameters are really zeroed ...
    assert float(ps[0].grad.min()) == 7.0              # ... direct ones are only marked stale (no memset)
    a0 = ps[0].data_ptr()
    assert flat.take_sink(a0) is False                 # first write of the step: overwrite
    assert flat.take_sink(a0) is True                  # later writes: accumulate
    flat.ensure_zeroed(ps[1].data_ptr())               # a gradient about to be accumulated by autograd: zeroed on demand
    assert float(ps[1].grad.abs().sum()) == 0.0
    flat.finalize_grads()                              # parameters that got no gradient this step hold zeros afterwards
    assert float(ps[2].grad.abs().sum()) == 0.0 and not flat._stale
    assert float(ps[0].grad.min()) == 7.0              # (written by "the kernel": untouched)
    flat.zero_grad()
    assert flat.take_sink(a0) is False                 # next step starts over


def test_direct_set_follows_a_rebase():
    flat, ps, other = _flat()
    flat.enable_direct_grads(ps)
    old = set(flat._direct)
    flat.rebase(torch.zeros_like(flat.data), torch.zeros_like(flat.grad))
    assert flat._direct == {p.data_ptr() for p in ps} and flat._direct != old


def test_owned_ranges_of_bucketed_two_shot_adam():
    from lstm_tensorspark_b200.parallel.fused_comm import FusedComm
    n = 4 * 1000
    for world in (2, 3, 8):
        covered = torch.zeros(2 * n, dtype=torch.int32)
        for rank in range(world):
            fake = types.SimpleNamespace(rank=rank, world_size=world, _state_buckets=[(0, n, True), (n, 2 * n, False)])
            for lo, hi in FusedComm._owned_ranges(fake):
                assert lo % 4 == 0 and hi % 4 == 0
                covered[lo:hi] += 1
        assert bool((covered == 1).all())              # every Adam slot has exactly one owner (one-shot bucket: rank 0)


def test_weight_decay_cut_is_whole_float4s():
    """The update kernels choose the weight decay per float4, so ``FlatOptimizer.wd_numel`` is -1 or a multiple of 4; the
    cut the engine sets (``FlatParams.lstm_numel``) is a multiple of ``ALIGN``."""
    from lstm_tensorspark_b200.models.flat import ALIGN, FlatParams
    from lstm_tensorspark_b200.ops.optim import FlatOptimizer
    flat = FlatParams([torch.nn.Parameter(torch.zeros(10, 3))], [torch.nn.Parameter(torch.zeros(5))])
    assert flat.lstm_numel % ALIGN == 0 and ALIGN % 4 == 0
    opt = FlatOptimizer(flat, 0.1, "sgd", weight_decay=0.1)
    for ok in (-1, 0, 4, flat.lstm_numel):
        opt.wd_numel = ok
        assert opt.wd_numel == ok
    for bad in (-2, 2, 30):
        with pytest.raises(ValueError, match="wd_numel"):
            opt.wd_numel = bad
    assert opt.wd_numel == flat.lstm_numel


def test_wavefront_gate_configuration():
    from lstm_tensorspark_b200.ops import cuda_lstm as CL
    T, B, H = 128, 256, 1024
    v0 = (CL._wave_variant() & ~(3 << 16))             # one counter per operand k-block
    assert CL._gate_off(v0) == 512
    assert CL._gate_cfg(v0, 2, H // 64, 4, 4 * H // 64, 2, 1, B, False) == [32, 32, 8, 4, B, 1, 0]
    assert CL._gate_cfg(v0, 2, 4 * H // 64, 1, 4 * H // 64, T + 1, -1, B, True) == [128, 32, T + 1, -1, B, 0, 1]
    v1 = v0 | (1 << 16)                                # one counter per batch tile: every CTA of the tile arrives once per step
    assert CL._gate_off(v1) == 0
    assert CL._gate_cfg(v1, 2, H // 64, 4, 4 * H // 64, 2, 1, B, False) == [2, 1, 128, 64, B, 1, 0]
    assert CL._gate_cfg(v1, 2, 4 * H // 64, 1, 4 * H // 64, T + 1, -1, B, True) == [2, 1, 64 * (T + 1), -64, B, 0, 1]


def test_big_launch_queue_never_releases_a_dependent_of_its_own_producer():
    from lstm_tensorspark_b200.ops import params as P
    P._QUEUE.clear()
    fired = []
    P.big_launch_begin()                                # GEMM 1 is launched ...
    P.queue_after_big_launch(lambda: fired.append("bucket of GEMM 1"))      # ... and its bucket becomes ready
    P.after_big_launch()
    assert fired == []                                  # not under GEMM 1 itself (a dependent may start while its primary runs)
    P.big_launch_begin()                                # GEMM 2
    P.after_big_launch()
    assert fired == ["bucket of GEMM 1"]                # under the NEXT big kernel
    P.queue_after_big_launch(lambda: fired.append("last"))
    P.after_big_launch(flush=True)                      # end of backward: whatever is left goes in stream order
    assert fired[-1] == "last" and not P._QUEUE


def test_buckets_are_ready_once_released_and_in_plan_order():
    """``TrainEngine._backward_with_buckets`` over a scripted backward pass: a bucket is queued only once every parameter it
    needs is released - a sink taken (the gradient being written) is not enough - and only after the buckets ahead of it in
    the plan; the last bucket goes after backward."""
    from lstm_tensorspark_b200.engine import TrainEngine
    from lstm_tensorspark_b200.ops import params as P
    P._QUEUE.clear()
    flat, ps, other = _flat()
    flat.enable_direct_grads(ps + other)
    for p, o in zip(flat.params, flat.offsets):
        P.register_param(p.data_ptr(), p.detach().bfloat16(), flat.grad[o:o + p.numel()].view(p.shape), owner=flat)
    w_x, w_h, b = (p.data_ptr() for p in ps)
    head = other[0].data_ptr()
    plan = [{"lo": 0, "hi": 1, "need": {w_x}}, {"lo": 1, "hi": 2, "need": {w_h, b, head}}, {"lo": 2, "hi": 3, "need": {w_x}}]
    launched = []
    comm = types.SimpleNamespace(begin_grad_step=lambda flat, opt: None,
                                 launch_bucket=lambda lo, hi, **kw: launched.append(lo))

    def big_launch():
        P.big_launch_begin()
        P.after_big_launch()

    def backward():
        P.release(head)
        for addr in (w_h, b):
            P.grad_out(addr, (1,), "cpu")
        P.release(w_h, b)                               # bucket 1 is complete, but bucket 0 comes first
        big_launch()
        P.grad_out(w_x, (1,), "cpu")                    # bucket 0's gradient is being written: not released yet
        big_launch()
        assert launched == []
        P.release(w_x)                                  # buckets 0 and 1 queued, in plan order ...
        assert launched == []
        big_launch()                                    # ... behind the next big launch
        assert launched == [0, 1]

    eng = types.SimpleNamespace(flat=flat, comm=comm, _bucket_plan=plan, optimizer=None,
                                cfg=types.SimpleNamespace(grad_bucket_blocks=0))
    flat.zero_grad()
    TrainEngine._backward_with_buckets(eng, types.SimpleNamespace(backward=backward))
    assert launched == [0, 1, 2]
    assert P._LISTENER is None
    P.release(w_x)                                      # outside a backward pass: nobody listens
    assert launched == [0, 1, 2]


def test_a_countdown_releases_once_from_the_last_op():
    from lstm_tensorspark_b200.ops import params as P
    seen = []
    chunks = P.Countdown(3)
    with P.releases_to(lambda released: seen.append(sorted(released))):
        rels = [chunks.releaser() for _ in range(3)]    # the backward passes of three batch chunks, in autograd's order
        for rel in rels:
            rel(11)
            rel(12, 13)
    assert seen == [[11], [11, 12, 13]]


def test_device_shard_gathers_into_given_buffers():
    """`DeviceShard.next(out=...)` (the trainer hands it the captured graph's input buffers) yields the same batches as `next()`."""
    import numpy as np
    import torch
    from lstm_tensorspark_b200 import data as D
    rng = np.random.default_rng(0)
    x = rng.standard_normal((40, 3, 5)).astype(np.float32)
    y = rng.integers(0, 4, size=40).astype(np.int64)
    a = D.DeviceShard(x, y, 8, "cpu", dtype=torch.float32, shuffle=True, seed=3)
    b = D.DeviceShard(x, y, 8, "cpu", dtype=torch.float32, shuffle=True, seed=3)
    xb, yb = torch.empty(8, 3, 5), torch.empty(8, dtype=torch.int64)
    for _ in range(12):                                   # crosses two reshuffles
        xa, ya = a.next()
        xo, yo = b.next(out=(xb, yb))
        assert xo.data_ptr() == xb.data_ptr() and torch.equal(xa, xo) and torch.equal(ya, yo)
    wrong = (torch.empty(4, 3, 5), torch.empty(4, dtype=torch.int64))      # wrong batch size: falls back to fresh tensors
    xa, _ = a.next()
    xo, _ = b.next(out=wrong)
    assert torch.equal(xa, xo) and xo.data_ptr() != wrong[0].data_ptr()
