"""Data layer: CSV reader, sharder, row parser, normaliser, batch iterators, synthetic sequences.

Parity targets (reference, read-only):
  * ``csv_to_partitions`` / ``text_to_rdd``  original src/rnn.py:104-138
  * ``process_batch``                         original src/rnn.py:141-158
  * ``next_batch``                            original src/rnn.py:161-177
  * ``min_max_normalizer``                    original src/rnn.py:95-101
  * standalone ``csv_to_batch`` / ``read_dataset_from_path``  original src/lstm-no-spark.py:90-112,254-258

Decisions where the reference is defective: Q2 (remainder shard hang) -> exactly P
shards of floor(N/P) rows, remainder dropped or spread; a shard smaller than the batch is an error, never
a hang.  Q10: labels are parsed to int64 up front.  Q3: ``batch_size == 0`` means the whole shard.
"""
from __future__ import annotations

import csv
import io
from typing import Iterable, Iterator, List, Optional, Sequence, Tuple

import numpy as np
import torch


# ------------------------------------------------------------------------------------------------
# CSV -> rows
# ------------------------------------------------------------------------------------------------
def read_lines(path: str) -> List[str]:
    with open(path, "r") as f:
        return f.read().splitlines()


def parse_csv_lines(lines: Iterable[str]) -> List[List[str]]:
    """Blank lines are dropped (reference: ``if len(d) > 0``, src/rnn.py:111-113)."""
    return [row for row in csv.reader(lines) if len(row) > 0]


def csv_to_batch(lines: Iterable[str]) -> List[List[str]]:
    """Standalone reader: no shuffle, no split (src/lstm-no-spark.py:90-112)."""
    return parse_csv_lines(lines)


def read_dataset_from_path(path: str) -> List[List[str]]:
    return csv_to_batch(read_lines(path))


def csv_to_partitions(lines: Iterable[str], num_partitions: int, shuffle: bool = True,
                      seed: Optional[int] = None, remainder: str = "drop") -> List[Tuple[int, List[List[str]]]]:
    """Shuffle the rows and cut them into exactly ``num_partitions`` keyed shards.

    The reference cuts chunks of ``floor(N/P)`` rows and lets the remainder become an extra
    (P+1)-th key (src/rnn.py:119-131), which then hangs ``next_batch`` (Q2).  Here every key
    ``0..P-1`` gets ``floor(N/P)`` rows; the ``N mod P`` left-over rows are dropped (``remainder="drop"``)
    or dealt round-robin to the first shards (``"spread"``).
    """
    if num_partitions < 1:
        raise ValueError("num_partitions must be >= 1")
    data = parse_csv_lines(lines)
    if shuffle:
        rng = np.random.default_rng(seed)
        perm = rng.permutation(len(data))
        data = [data[i] for i in perm]
    total = len(data)
    bs = total // num_partitions
    if bs == 0:
        raise ValueError(f"{total} rows cannot be split into {num_partitions} non-empty partitions")
    shards = [(k, data[k * bs:(k + 1) * bs]) for k in range(num_partitions)]
    if remainder == "spread":
        for j, row in enumerate(data[num_partitions * bs:]):
            shards[j % num_partitions][1].append(row)
    elif remainder != "drop":
        raise ValueError(f"unknown remainder policy {remainder!r}")
    return shards


def text_to_partitions(path: str, num_partitions: int, shuffle: bool = True, seed: Optional[int] = None,
                       remainder: str = "drop"):
    """File -> keyed shards (the role of ``text_to_rdd``, src/rnn.py:136-138)."""
    return csv_to_partitions(read_lines(path), num_partitions, shuffle=shuffle, seed=seed, remainder=remainder)


# ------------------------------------------------------------------------------------------------
# rows -> arrays
# ------------------------------------------------------------------------------------------------
def min_max_normalizer(x):
    """Global (whole-matrix) min-max scaling to [0, 1] — same semantics as src/rnn.py:95-101."""
    x = np.asarray(x, dtype=np.float64)
    mmax = np.amax(x)
    mmin = np.amin(x)
    rng = mmax - mmin
    if rng == 0:
        return np.zeros_like(x).tolist()
    d = 1.0 - ((mmax - x) / rng)
    return d.tolist()


def process_batch(train_xy: Sequence[Sequence[str]], normalize: bool = False,
                  seq_len: int = 1, in_features: Optional[int] = None) -> Tuple[np.ndarray, np.ndarray]:
    """Rows -> ``(x float32 [N, D] or [N, T, D], y int64 [N])``; label = last column."""
    xs, ys = [], []
    for row in train_xy:
        if len(row) <= 1:
            continue
        xs.append([float(v) for v in row[:-1]])
        ys.append(int(float(row[-1])))
    if not xs:
        raise ValueError("empty partition: no parsable rows")
    if normalize:
        xs = min_max_normalizer(xs)
    x = np.asarray(xs, dtype=np.float32)
    y = np.asarray(ys, dtype=np.int64)
    if seq_len > 1:
        if x.shape[1] % seq_len != 0:
            raise ValueError(f"row width {x.shape[1]} is not a multiple of seq_len={seq_len}")
        d = x.shape[1] // seq_len
        if in_features is not None and d != in_features:
            raise ValueError(f"row width {x.shape[1]} != seq_len*in_features = {seq_len}*{in_features}")
        x = x.reshape(x.shape[0], seq_len, d)
    elif in_features is not None and x.shape[1] != in_features:
        raise ValueError(f"row has {x.shape[1]} features, --in_features says {in_features}")
    return x, y


def resolve_batch_size(batch_size: int, shard_rows: int) -> int:
    """``--batch_size 0`` = whole shard (reference intent, src/rnn.py:193-199, Q3)."""
    bs = shard_rows if not batch_size else batch_size
    if bs > shard_rows:
        raise ValueError(f"shard has {shard_rows} rows but batch_size is {bs}: "
                         "reduce --batch_size or --partitions (the reference would spin forever here)")
    return bs


def next_batch(train_x, train_y, batch_size: int = 10, shuffle: bool = True,
               rng: Optional[np.random.Generator] = None) -> Iterator[Tuple[np.ndarray, np.ndarray]]:
    """Infinite generator of full batches; reshuffles every pass; the trailing partial batch is
    skipped (src/rnn.py:161-177)."""
    n = train_x.shape[0]
    total_iteration = n // batch_size
    if total_iteration == 0:
        raise ValueError(f"next_batch: {n} rows < batch_size {batch_size}")
    rng = rng if rng is not None else np.random.default_rng()
    while True:
        if shuffle:
            p = rng.permutation(n)
            train_x = train_x[p]
            train_y = train_y[p]
        for i in range(total_iteration):
            lo = i * batch_size
            yield train_x[lo:lo + batch_size], train_y[lo:lo + batch_size]


# ------------------------------------------------------------------------------------------------
# synthetic sequences (benchmark configs of BASELINE.json)
# ------------------------------------------------------------------------------------------------
def synthetic_sequences(n: int, seq_len: int, in_features: int, num_classes: int, seed: int = 0,
                        dtype=np.float32) -> Tuple[np.ndarray, np.ndarray]:
    """Class-dependent gaussian sequences (learnable, so loss curves are meaningful)."""
    rng = np.random.default_rng(seed)
    y = rng.integers(0, num_classes, size=n).astype(np.int64)
    centers = rng.standard_normal((num_classes, in_features)).astype(np.float32)
    if seq_len > 1:
        x = rng.standard_normal((n, seq_len, in_features), dtype=np.float32) * 0.5 + centers[y][:, None, :]
    else:
        x = rng.standard_normal((n, in_features), dtype=np.float32) * 0.5 + centers[y]
    return x.astype(dtype), y


# ------------------------------------------------------------------------------------------------
# loaders
# ------------------------------------------------------------------------------------------------
class DeviceShard:
    """Device-resident shard; a batch is an index gather on the device, no per-step H2D
    (replaces the per-step feed_dict copy, src/rnn.py:264-267)."""

    def __init__(self, x: np.ndarray, y: np.ndarray, batch_size: int, device, dtype=torch.float32,
                 shuffle: bool = True, seed: int = 0):
        self.x = torch.as_tensor(x).to(device=device, dtype=dtype)
        self.y = torch.as_tensor(y).to(device=device)
        self.n = self.x.shape[0]
        self.batch_size = resolve_batch_size(batch_size, self.n)
        self.per_epoch = self.n // self.batch_size
        self.shuffle = shuffle
        self.gen = torch.Generator(device="cpu")
        self.gen.manual_seed(seed)
        self._perm = None
        self._i = 0

    def _reshuffle(self):
        if self.shuffle:
            self._perm = torch.randperm(self.n, generator=self.gen).to(self.x.device)
        else:
            self._perm = torch.arange(self.n, device=self.x.device)
        self._i = 0

    def next(self, out=None) -> Tuple[torch.Tensor, torch.Tensor]:
        """``out = (x_buf, y_buf)``: gather the batch straight into these buffers (the input buffers of a captured CUDA graph:
        ``TrainEngine.graph_inputs()``) instead of into fresh tensors that then have to be copied there."""
        if self._perm is None or self._i >= self.per_epoch:
            self._reshuffle()
        lo = self._i * self.batch_size
        idx = self._perm[lo:lo + self.batch_size]
        self._i += 1
        if out is not None and out[0].shape[0] == idx.numel() and out[0].dtype == self.x.dtype:
            torch.index_select(self.x, 0, idx, out=out[0])
            torch.index_select(self.y, 0, idx, out=out[1])
            return out[0], out[1]
        return self.x.index_select(0, idx), self.y.index_select(0, idx)

    def state_dict(self):
        return {"gen": self.gen.get_state(), "i": self._i,
                "perm": None if self._perm is None else self._perm.cpu()}

    def load_state_dict(self, st):
        self.gen.set_state(st["gen"])
        self._i = st["i"]
        self._perm = None if st["perm"] is None else st["perm"].to(self.x.device)


class PinnedHostLoader:
    """Host-resident shard in PINNED memory: each ``next()`` issues the host->device copy of one contiguous batch
    (async, double-buffered device staging) and hands back device tensors — the end-to-end path of bench.py.
    Shuffling permutes the pinned copy once per pass (not per step), so a step is exactly one H2D DMA per tensor."""

    def __init__(self, x: np.ndarray, y: np.ndarray, batch_size: int, device, dtype=torch.float32,
                 shuffle: bool = True, seed: int = 0, depth: int = 2):
        """``depth``: device staging slots (the copy of a batch is enqueued ``depth - 1`` calls before it is handed out)."""
        assert depth >= 2
        self.device = torch.device(device)
        self.dtype = dtype
        self.depth = depth
        self.n = x.shape[0]
        self.batch_size = resolve_batch_size(batch_size, self.n)
        self.per_epoch = self.n // self.batch_size
        self.gen = torch.Generator(device="cpu")
        self.gen.manual_seed(seed)
        self.shuffle = shuffle
        cuda = self.device.type == "cuda"
        self.x_host = torch.as_tensor(x).to(dtype).contiguous()
        self.y_host = torch.as_tensor(y).contiguous()
        if cuda:
            self.x_host = self.x_host.pin_memory()
            self.y_host = self.y_host.pin_memory()
        shape_x = (self.batch_size,) + tuple(self.x_host.shape[1:])
        self.dev = [(torch.empty(shape_x, dtype=dtype, device=self.device),
                     torch.empty((self.batch_size,), dtype=torch.int64, device=self.device)) for _ in range(depth)]
        self._slot = 0
        self._pending = []
        self._copy_stream = None
        self.debug_skip_copy = False
        self._i = self.per_epoch if shuffle else 0
        # resume bookkeeping: `_order` = which original row sits in each row of the (in-place permuted) pinned arrays; per pass
        # the generator state and order from BEFORE that pass's shuffle (the last two passes: prefetched batches may already
        # belong to the next one); `_consumed` = (pass, batches handed out in it)
        self._order = torch.arange(self.n)
        self._pass = 0 if shuffle else 1
        self._pass_start = {}
        if not shuffle:
            self._pass_start[1] = (self.gen.get_state(), self._order.clone())
        self._consumed = (self._pass, 0)
        self.bytes_per_batch = self.dev[0][0].numel() * self.dev[0][0].element_size() + self.batch_size * 8

    def _reshuffle(self):
        # the async H2D copy of the last batch of the previous pass may not have run yet (the host is ahead of the GPU):
        # it must not read pinned memory that is being re-permuted underneath it
        if self._copy_stream is not None:
            self._copy_stream.synchronize()
        # a pass is ``original[randperm]`` - the same batches DeviceShard draws from the same seed - so the rows that are
        # already permuted in place have to be addressed through the inverse of the current order
        perm = torch.randperm(self.n, generator=self.gen)
        inv = torch.empty_like(self._order)
        inv[self._order] = torch.arange(self.n)
        idx = inv[perm]
        xs, ys = self.x_host[idx], self.y_host[idx]
        self.x_host.copy_(xs)
        self.y_host.copy_(ys)
        self._order = perm

    def _advance(self) -> int:
        if self._i >= self.per_epoch:
            self._pass += 1
            self._pass_start[self._pass] = (self.gen.get_state(), self._order.clone())
            self._pass_start.pop(self._pass - self.depth - 1, None)     # (a tiny shard can be prefetched several passes ahead)
            if self.shuffle:
                self._reshuffle()
            self._i = 0
        lo = self._i * self.batch_size
        self._i += 1
        return lo

    def state_dict(self):
        """Position of the NEXT batch to be handed out (prefetched-but-unconsumed batches are not counted), exact across a
        reshuffle: generator state and row order from before the shuffle of the pass that batch belongs to."""
        ps, k = self._consumed
        if k >= self.per_epoch or ps not in self._pass_start:      # the next batch opens a new pass
            if ps + 1 in self._pass_start:
                ps, k = ps + 1, 0
            else:                                                  # ... which has not been prefetched yet: current state is its start
                return {"gen": self.gen.get_state(), "order": self._order.clone(), "i": 0, "shuffle_first": self.shuffle, "pinned": True}
        gen, order = self._pass_start[ps]
        return {"gen": gen, "order": order.clone(), "i": k, "shuffle_first": self.shuffle, "pinned": True}

    def load_state_dict(self, st):
        """Call on a freshly constructed loader over the same arrays (rows in their original order)."""
        assert not self._pending and int(self._order[0]) == 0 and bool((self._order[1:] > self._order[:-1]).all())
        order = st["order"]
        self.x_host.copy_(self.x_host[order])
        self.y_host.copy_(self.y_host[order])
        self._order = order.clone()
        self.gen.set_state(st["gen"])
        self._pass = 0
        self._pass_start = {}
        self._i = self.per_epoch                     # the first _advance() opens pass 1: records its start, shuffles, ...
        self._advance()
        self._i = st["i"]                            # ... and the batches already consumed in it are skipped
        self._consumed = (self._pass, st["i"])

    def _issue(self):
        """Enqueue the H2D copy of the next batch on the copy stream into the free staging slot."""
        lo = self._advance()
        tag = (self._pass, self._i)                      # handing this batch out makes it the consumed position
        dx, dy = self.dev[self._slot]
        self._slot = (self._slot + 1) % self.depth
        if self.device.type != "cuda":
            dx.copy_(self.x_host[lo:lo + self.batch_size])
            dy.copy_(self.y_host[lo:lo + self.batch_size])
            return dx, dy, None, tag
        if self._copy_stream is None:
            self._copy_stream = torch.cuda.Stream(device=self.device)
        # the slot being overwritten was consumed by compute work already enqueued on the current stream
        self._copy_stream.wait_stream(torch.cuda.current_stream(self.device))
        with torch.cuda.stream(self._copy_stream):
            if not self.debug_skip_copy:                  # (bench diagnostics only: how much of a step is the DMA's interference?)
                dx.copy_(self.x_host[lo:lo + self.batch_size], non_blocking=True)
                dy.copy_(self.y_host[lo:lo + self.batch_size], non_blocking=True)
            ev = torch.cuda.Event()
            ev.record(self._copy_stream)
        return dx, dy, ev, tag

    def next(self) -> Tuple[torch.Tensor, torch.Tensor]:
        """Returns this step's batch (its H2D copy was enqueued one call earlier, so it overlaps the previous step's
        compute) and enqueues the copy of the following one.  Every step still moves its own inputs host->device."""
        while len(self._pending) < self.depth - 1:
            self._pending.append(self._issue())
        dx, dy, ev, self._consumed = self._pending.pop(0)
        if ev is not None:
            torch.cuda.current_stream(self.device).wait_event(ev)
        # refill: the slot this copy overwrites was handed out depth - 1 calls ago; the step that consumed it is enqueued
        self._pending.append(self._issue())
        return dx, dy
