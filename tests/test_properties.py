"""Property tests (hypothesis) for the data layer and the flat parameter buffer - the invariants the reference's Spark
pipeline only held by accident (Q2, Q3) and the ones the fused allreduce relies on."""
import numpy as np
import pytest
import torch
from hypothesis import given, settings, strategies as st

from lstm_tensorspark_b200 import data as D


def _lines(n, f=3):
    return [",".join([f"{i}.{j}" for j in range(f)] + [str(i % 3)]) for i in range(n)]


@settings(max_examples=60, deadline=None)
@given(n=st.integers(1, 300), p=st.integers(1, 12), seed=st.integers(0, 10), policy=st.sampled_from(["drop", "spread"]))
def test_sharder_partitions_rows_without_duplicates(n, p, seed, policy):
    lines = _lines(n)
    if n // p == 0:
        with pytest.raises(ValueError):
            D.csv_to_partitions(lines, p, seed=seed, remainder=policy)
        return
    shards = D.csv_to_partitions(lines, p, seed=seed, remainder=policy)
    assert [k for k, _ in shards] == list(range(p))                      # exactly P keys: no (P+1)-th remainder shard (Q2)
    sizes = [len(rows) for _, rows in shards]
    assert min(sizes) >= n // p and max(sizes) - min(sizes) <= 1
    flat = [tuple(r) for _, rows in shards for r in rows]
    assert len(set(flat)) == len(flat)                                   # a row lands in at most one shard
    assert len(flat) == (n if policy == "spread" else (n // p) * p)
    again = D.csv_to_partitions(lines, p, seed=seed, remainder=policy)
    assert again == shards                                               # deterministic under a seed


@settings(max_examples=40, deadline=None)
@given(n=st.integers(1, 64), bs=st.integers(1, 70), passes=st.integers(1, 3))
def test_next_batch_yields_full_batches_and_every_row_once_per_pass(n, bs, passes):
    x = np.arange(n, dtype=np.float32).reshape(n, 1)
    y = np.arange(n, dtype=np.int64)
    if n < bs:
        with pytest.raises(ValueError):                                  # error, not the reference's infinite loop
            next(D.next_batch(x, y, bs))
        return
    it = D.next_batch(x, y, bs, shuffle=True, rng=np.random.default_rng(0))
    per_pass = n // bs
    for _ in range(passes):
        seen = []
        for _ in range(per_pass):
            bx, by = next(it)
            assert bx.shape == (bs, 1) and by.shape == (bs,)
            assert np.array_equal(bx[:, 0].astype(np.int64), by)         # rows and labels stay paired under the shuffle
            seen += by.tolist()
        assert len(set(seen)) == len(seen)                               # no row twice within a pass


@settings(max_examples=25, deadline=None)
@given(shapes=st.lists(st.tuples(st.integers(1, 40), st.integers(1, 9)), min_size=1, max_size=5))
def test_flat_params_layout_is_aligned_and_aliasing(shapes):
    from lstm_tensorspark_b200.models.flat import FlatParams, ALIGN
    params = [torch.nn.Parameter(torch.randn(*s)) for s in shapes]
    before = [p.detach().clone() for p in params]
    flat = FlatParams(params, [])
    assert flat.padded_numel % 4 == 0 and flat.padded_numel >= sum(p.numel() for p in params)
    off = 0
    for p, b in zip(params, before):
        assert torch.equal(p.detach(), b)                                # values survive the move into the flat buffer
        assert (p.data_ptr() - flat.data.data_ptr()) % (4 * ALIGN) == 0  # every segment starts on an ALIGN-element boundary
        assert p.data_ptr() >= flat.data.data_ptr() + 4 * off
        off += p.numel()
    flat.data.zero_()
    assert all(float(p.detach().abs().sum()) == 0.0 for p in params)     # parameters are views of the flat buffer


@settings(max_examples=40, deadline=None)
@given(depth=st.integers(2, 5), per_pass=st.integers(1, 6), bs=st.integers(1, 5), extra=st.integers(0, 3), stop=st.integers(0, 14),
       seed=st.integers(0, 5), shuffle=st.booleans())
def test_pinned_loader_matches_device_shard_and_resumes_anywhere(depth, per_pass, bs, extra, stop, seed, shuffle):
    """The pinned-host feed (prefetch depth d, in-place shuffles) hands out exactly the batches the device-resident gather draws
    from the same seed, and a loader restored from `state_dict()` taken after ANY number of batches continues the sequence."""
    n = bs * per_pass + min(extra, bs - 1)                       # rows beyond the last full batch are never served
    x = np.arange(n * 2, dtype=np.float32).reshape(n, 2)
    y = np.arange(n, dtype=np.int64)
    total = 15
    want = None
    if shuffle:                                                   # DeviceShard always permutes: the common reference sequence
        ds = D.DeviceShard(x, y, bs, "cpu", dtype=torch.float32, shuffle=True, seed=seed)
        want = [ds.next()[1].clone() for _ in range(total)]
    mk = lambda: D.PinnedHostLoader(x.copy(), y.copy(), bs, "cpu", shuffle=shuffle, seed=seed, depth=depth)
    a = mk()
    got = []
    for j in range(stop):
        xb, yb = a.next()
        assert np.array_equal(xb.numpy(), x[yb.numpy()])
        got.append(yb.clone())
    b = mk()
    b.load_state_dict(a.state_dict())
    for j in range(stop, total):
        xb, yb = b.next()
        assert np.array_equal(xb.numpy(), x[yb.numpy()])
        got.append(yb.clone())
    if want is None:
        want = [torch.arange(bs) + bs * (j % per_pass) for j in range(total)]
    for j in range(total):
        assert torch.equal(got[j], want[j]), (j, stop)
