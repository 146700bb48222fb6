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


def process_batch_ragged(train_xy: Sequence[Sequence[str]], seq_len: int, in_features: int,
                         normalize: bool = False) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """Variable-length rows -> ``(x float32 [N, seq_len, in_features], y int64 [N], lengths int32 [N])``.

    A row is ``k * in_features`` values followed by the label, ``1 <= k <= seq_len``; it is zero-padded on the right to
    ``seq_len`` steps and ``lengths = k``.  ``normalize``: global min-max over the real values only (padding excluded)."""
    if seq_len < 1 or in_features < 1:
        raise ValueError("variable-length rows need seq_len >= 1 and in_features >= 1")
    xs, ys, ls = [], [], []
    for n, row in enumerate(train_xy):
        if len(row) <= 1:
            continue
        width = len(row) - 1
        if width % in_features != 0 or not (1 <= width // in_features <= seq_len):
            raise ValueError(f"row {n}: {width} values is not a whole number of 1..{seq_len} steps of "
                             f"{in_features} features")
        xs.append([float(v) for v in row[:-1]])
        ys.append(int(float(row[-1])))
        ls.append(width // in_features)
    x = _pad_steps(xs, ls, seq_len, in_features, normalize)
    return x, np.asarray(ys, dtype=np.int64), np.asarray(ls, dtype=np.int32)


def _pad_steps(xs, ls, seq_len: int, in_features: int, normalize: bool) -> np.ndarray:
    """Rows of ``ls[i] * in_features`` values -> ``x float32 [N, seq_len, in_features]``, zero-padded on the right.
    ``normalize``: global min-max over the real values only (padding excluded)."""
    if not xs:
        raise ValueError("empty partition: no parsable rows")
    if normalize:
        flat = min_max_normalizer(np.concatenate([np.asarray(r, dtype=np.float64) for r in xs]))
        off = np.cumsum([0] + [len(r) for r in xs])
        xs = [flat[off[i]:off[i + 1]] for i in range(len(xs))]
    x = np.zeros((len(xs), seq_len, in_features), dtype=np.float32)
    for i, r in enumerate(xs):
        x[i, :ls[i]] = np.asarray(r, dtype=np.float32).reshape(ls[i], in_features)
    return x


def process_batch_per_step(train_xy: Sequence[Sequence[str]], seq_len: int, in_features: int, num_classes: int,
                           variable_length: bool = False, normalize: bool = False):
    """Rows with a label at every step (``--per_step_labels``) -> ``(x float32 [N, seq_len, in_features], y int64 [N, seq_len])``,
    plus ``lengths`` int32 [N] with ``variable_length``.

    A row is ``k * in_features`` values followed by ``k`` labels, the label of step t being the t-th of them; ``k = seq_len``, or
    ``1 <= k <= seq_len`` with ``variable_length`` (then zero-padded on the right to ``seq_len`` steps, padded labels 0 and never
    read).  A row that does not split this way, or a label outside ``[0, num_classes)``, is an error naming the row.
    ``normalize``: global min-max over the real feature values only."""
    if seq_len < 2 or in_features < 1:
        raise ValueError("per-step labels need seq_len >= 2 and in_features >= 1")
    xs, ys, ls = [], [], []
    for n, row in enumerate(train_xy):
        if len(row) <= 1:
            continue
        k, rem = divmod(len(row), in_features + 1)
        if rem or not (k == seq_len or (variable_length and 1 <= k <= seq_len)):
            want = f"1..{seq_len}" if variable_length else f"{seq_len}"
            raise ValueError(f"row {n}: {len(row)} fields is not {want} steps of {in_features} features followed by one "
                             "label per step")
        lab = [int(float(v)) for v in row[k * in_features:]]
        bad = [v for v in lab if not 0 <= v < num_classes]
        if bad:
            raise ValueError(f"row {n}: label {bad[0]} outside [0, {num_classes})")
        xs.append([float(v) for v in row[:k * in_features]])
        ys.append(lab)
        ls.append(k)
    x = _pad_steps(xs, ls, seq_len, in_features, normalize)
    y = np.zeros((len(xs), seq_len), dtype=np.int64)
    for i, lab in enumerate(ys):
        y[i, :ls[i]] = lab
    if variable_length:
        return x, y, np.asarray(ls, dtype=np.int32)
    return x, y


def process_tokens(train_xy: Sequence[Sequence[str]], seq_len: int, vocab_size: int, num_classes: int = 0,
                   variable_length: bool = False, per_step_labels: bool = False, next_token: bool = False):
    """Rows of token ids (``--vocab_size``) -> ``(x int32 [N, seq_len] ([N] when seq_len == 1), y int64 [N] or [N, seq_len])``,
    plus ``lengths`` int32 [N] with ``variable_length``.

    ``next_token`` (``--next_token``): a row is ``k`` ids and nothing else, ``k = seq_len + 1``, or ``2 <= k <= seq_len + 1`` with
    ``variable_length``; the input is ids ``0..k-2``, the label of step t is id ``t + 1`` and the length is ``k - 1``.

    A row is ``k`` ids followed by the label, or with ``per_step_labels`` by ``k`` labels; ``k = seq_len``, or
    ``1 <= k <= seq_len`` with ``variable_length`` (then padded on the right with id 0, label 0, never read).  A non-integer id,
    an id outside ``[0, vocab_size)``, a per-step label outside ``[0, num_classes)`` or a row that does not split this way is an
    error naming the row."""
    if seq_len < 1 or vocab_size < 1:
        raise ValueError("token rows need seq_len >= 1 and vocab_size >= 1")
    want = f"1..{seq_len}" if variable_length else f"{seq_len}"
    if next_token:
        if seq_len < 2:
            raise ValueError("next-token rows need seq_len >= 2")
        per_step_labels = True
        want = f"2..{seq_len + 1}" if variable_length else f"{seq_len + 1}"
    xs, ys, ls = [], [], []
    for n, row in enumerate(train_xy):
        if len(row) <= 1 and not next_token:
            continue
        if next_token:
            k, rem = len(row) - 1, 0                   # k steps: the last id is a label only
        elif per_step_labels:
            k, rem = divmod(len(row), 2)
        else:
            k, rem = len(row) - 1, 0
        if rem or not (k == seq_len or (variable_length and 1 <= k <= seq_len)):
            if next_token:
                raise ValueError(f"row {n}: {len(row)} fields is not {want} token ids (--next_token: every id but the last is "
                                 "an input, every id but the first a label)")
            raise ValueError(f"row {n}: {len(row)} fields is not {want} token ids followed by "
                             f"{'one label per step' if per_step_labels else 'the label'}")
        ids = []
        for v in row[:k + 1 if next_token else k]:
            s = str(v).strip()
            try:
                i = int(s)
            except ValueError:
                raise ValueError(f"row {n}: token id {s!r} is not an integer") from None
            if not 0 <= i < vocab_size:
                raise ValueError(f"row {n}: token id {i} outside [0, {vocab_size}) (--vocab_size {vocab_size})")
            ids.append(i)
        if next_token:
            ids, lab = ids[:-1], ids[1:]
        else:
            lab = [int(float(v)) for v in row[k:]]
        if per_step_labels and not next_token:
            bad = [v for v in lab if not 0 <= v < num_classes]
            if bad:
                raise ValueError(f"row {n}: label {bad[0]} outside [0, {num_classes})")
        xs.append(ids)
        ys.append(lab if per_step_labels else lab[0])
        ls.append(k)
    if not xs:
        raise ValueError("empty partition: no parsable rows")
    x = np.zeros((len(xs), seq_len), dtype=np.int32)
    y = np.zeros((len(xs), seq_len), dtype=np.int64) if per_step_labels else np.asarray(ys, dtype=np.int64)
    for i, r in enumerate(xs):
        x[i, :ls[i]] = r
        if per_step_labels:
            y[i, :ls[i]] = ys[i]
    if seq_len == 1:
        x = x[:, 0].copy()
    if variable_length:
        return x, y, np.asarray(ls, dtype=np.int32)
    return x, y


def parse_rows(rows: Sequence[Sequence[str]], cfg):
    """Rows -> ``(x, y, lengths)`` by the parser the flags of ``cfg`` select (``--vocab_size``, ``--per_step_labels``,
    ``--variable_length``); ``lengths`` is None unless ``cfg.variable_length``."""
    if cfg.vocab_size > 0:
        x, y, *lengths = process_tokens(rows, cfg.seq_len, cfg.vocab_size, cfg.num_classes,
                                        variable_length=cfg.variable_length, per_step_labels=cfg.per_step_labels,
                                        next_token=getattr(cfg, "next_token", False))
    elif cfg.per_step_labels:
        x, y, *lengths = process_batch_per_step(rows, cfg.seq_len, cfg.in_features, cfg.num_classes,
                                                variable_length=cfg.variable_length, normalize=cfg.normalize)
    elif cfg.variable_length:
        x, y, *lengths = process_batch_ragged(rows, cfg.seq_len, cfg.in_features, normalize=cfg.normalize)
    else:
        x, y, *lengths = process_batch(rows, normalize=cfg.normalize, seq_len=cfg.seq_len, in_features=cfg.in_features)
    return x, y, (lengths[0] if lengths else None)


def input_dtype(cfg) -> torch.dtype:
    """The dtype ``x`` goes to the device in: token ids stay int32 (4 B per position on the host -> device copy)."""
    return torch.int32 if cfg.vocab_size > 0 else torch.float32


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
# the generator key that draws a held-out set (``valid_of`` below) instead of a training set: same task, other samples
VALID_DRAWS = 0x76616C


def synthetic_sequences(n: int, seq_len: int, in_features: int, num_classes: int, seed: int = 0,
                        dtype=np.float32, variable_length: bool = False, valid_of: int = 0):
    """Class-dependent gaussian sequences (learnable, so loss curves are meaningful).  -> ``(x, y)``.

    ``valid_of = m > 0``: ``n`` held-out samples of the task ``m`` training samples were drawn from (the same class centres),
    labels and noise from a generator of their own.

    ``variable_length``: -> ``(x, y, lengths)``, the same ``x`` / ``y`` with per-sample lengths drawn uniformly from
    ``[max(1, seq_len // 4), seq_len]`` (int32) by a generator of their own, and the padded steps zeroed."""
    rng = np.random.default_rng(seed)
    y = rng.integers(0, num_classes, size=valid_of or n).astype(np.int64)
    centers = rng.standard_normal((num_classes, in_features)).astype(np.float32)
    if valid_of:
        rng = np.random.default_rng([seed, VALID_DRAWS])
        y = rng.integers(0, num_classes, size=n).astype(np.int64)
    if seq_len > 1:
        x = rng.standard_normal((n, seq_len, in_features), dtype=np.float32) * 0.5 + centers[y][:, None, :]
    else:
        x = rng.standard_normal((n, in_features), dtype=np.float32) * 0.5 + centers[y]
    if not variable_length:
        return x.astype(dtype), y
    if seq_len < 2:
        raise ValueError("variable-length sequences need seq_len >= 2")
    lengths = synthetic_lengths(n, seq_len, seed, valid=bool(valid_of))
    x[np.arange(seq_len)[None, :] >= lengths[:, None]] = 0.0
    return x.astype(dtype), y, lengths


def synthetic_per_step(n: int, seq_len: int, in_features: int, num_classes: int, seed: int = 0, dtype=np.float32,
                       variable_length: bool = False, valid_of: int = 0):
    """A learnable sequence-labelling task (``--per_step_labels``): every step has its own class, and its input is drawn around
    that class's centre.  -> ``(x [n, T, D], y int64 [n, T])``, plus ``lengths`` with ``variable_length`` (the lengths of
    ``synthetic_lengths``, padded steps zeroed and labelled 0).  Drawn by a generator of its own: the draws of
    ``synthetic_sequences`` are untouched."""
    if seq_len < 2:
        raise ValueError("per-step labels need seq_len >= 2")
    rng = np.random.default_rng([seed, 0x737465])
    centers = rng.standard_normal((num_classes, in_features)).astype(np.float32)
    if valid_of:                                       # held out: the same centres, other samples
        rng = np.random.default_rng([seed, 0x737465, VALID_DRAWS])
    y = rng.integers(0, num_classes, size=(n, seq_len)).astype(np.int64)
    x = rng.standard_normal((n, seq_len, in_features), dtype=np.float32) * 0.5 + centers[y]
    if not variable_length:
        return x.astype(dtype), y
    lengths = synthetic_lengths(n, seq_len, seed, valid=bool(valid_of))
    pad = np.arange(seq_len)[None, :] >= lengths[:, None]
    x[pad] = 0.0
    y[pad] = 0
    return x.astype(dtype), y, lengths


def synthetic_tokens(n: int, seq_len: int, vocab_size: int, num_classes: int, seed: int = 0, variable_length: bool = False,
                     per_step_labels: bool = False, p_class: float = 0.5, ids_per_class: int = 8, valid_of: int = 0):
    """A learnable token task (``--vocab_size``): every class owns ``ids_per_class`` indicative ids (distinct while the vocabulary
    allows); a step draws from its class's ids with probability ``p_class`` and from a Zipf(1.1) background over the whole
    vocabulary otherwise.  The class of a step is its sample's label, or with ``per_step_labels`` the step's own label.
    -> ``(x int32 [n, T] ([n] when T == 1), y int64 [n] or [n, T])``, plus ``lengths`` with ``variable_length`` (those of
    ``synthetic_lengths``; padded steps hold id 0 and label 0).  Drawn by a generator of its own: the draws of
    ``synthetic_sequences`` and ``synthetic_per_step`` are untouched."""
    if vocab_size < 1:
        raise ValueError("synthetic tokens need vocab_size >= 1")
    rng = np.random.default_rng([seed, 0x746F6B])
    own = rng.permutation(vocab_size)[:num_classes * ids_per_class] if vocab_size >= num_classes * ids_per_class \
        else rng.integers(0, vocab_size, size=num_classes * ids_per_class)
    own = own.reshape(num_classes, ids_per_class)
    if valid_of:                                       # held out: the same indicative ids, other samples
        rng = np.random.default_rng([seed, 0x746F6B, VALID_DRAWS])
    if per_step_labels:
        y = rng.integers(0, num_classes, size=(n, seq_len)).astype(np.int64)
        cls = y
    else:
        y = rng.integers(0, num_classes, size=n).astype(np.int64)
        cls = np.broadcast_to(y[:, None], (n, seq_len))
    pick = own[cls, rng.integers(0, ids_per_class, size=(n, seq_len))]
    background = (rng.zipf(1.1, size=(n, seq_len)) - 1) % vocab_size
    x = np.where(rng.random((n, seq_len)) < p_class, pick, background).astype(np.int32)
    lengths = None
    if variable_length:
        if seq_len < 2:
            raise ValueError("variable-length sequences need seq_len >= 2")
        lengths = synthetic_lengths(n, seq_len, seed, valid=bool(valid_of))
        pad = np.arange(seq_len)[None, :] >= lengths[:, None]
        x[pad] = 0
        if per_step_labels:
            y[pad] = 0
    if seq_len == 1:
        x = x[:, 0].copy()
        if per_step_labels:
            y = y[:, 0].copy()
    return (x, y) if lengths is None else (x, y, lengths)


NEXT_TOKEN_PROBS = (0.6, 0.2, 0.1, 0.1)
# entropy of a step of the chain below in nats: the loss a perfect model reaches (perplexity exp(1.0889) = 2.97)
NEXT_TOKEN_ENTROPY = -sum(p * float(np.log(p)) for p in NEXT_TOKEN_PROBS)


def next_token_chain(vocab_size: int, seed: int = 0) -> np.ndarray:
    """The successor table ``[V, 4]`` of the synthetic language (``synthetic_next_token``): id i is followed by
    ``succ[i, j]`` with probability ``NEXT_TOKEN_PROBS[j]``; the four successors of an id are distinct."""
    if vocab_size < 4:
        raise ValueError("the synthetic next-token chain needs vocab_size >= 4")
    rng = np.random.default_rng([seed, 0x6E7874])
    base = rng.integers(0, vocab_size, size=vocab_size)
    step = rng.integers(1, max(1, (vocab_size - 1) // 3) + 1, size=vocab_size)
    return ((base[:, None] + np.arange(4)[None, :] * step[:, None]) % vocab_size).astype(np.int64)


def synthetic_next_token(n: int, seq_len: int, vocab_size: int, seed: int = 0, variable_length: bool = False, valid_of: int = 0):
    """A learnable language (``--next_token``): a fixed sparse first-order Markov chain over the ids (``next_token_chain``), so
    the achievable loss is known in closed form (``NEXT_TOKEN_ENTROPY``).  ``n`` walks of ``seq_len + 1`` ids from a uniform
    start -> ``(x int32 [n, T] = ids 0..T-1, y int64 [n, T] = ids 1..T)``, plus ``lengths`` with ``variable_length`` (those of
    ``synthetic_lengths``; padded steps hold id 0 and label 0).  Drawn by a generator of its own: the draws of the other
    synthetic tasks are untouched."""
    if seq_len < 2:
        raise ValueError("next-token sequences need seq_len >= 2")
    succ = next_token_chain(vocab_size, seed)
    rng = np.random.default_rng([seed, 0x6E7874, 1] + ([VALID_DRAWS] if valid_of else []))   # held out: the same chain
    tok = np.empty((n, seq_len + 1), dtype=np.int64)
    tok[:, 0] = rng.integers(0, vocab_size, size=n)
    pick = rng.choice(4, size=(n, seq_len), p=NEXT_TOKEN_PROBS)
    for t in range(seq_len):
        tok[:, t + 1] = succ[tok[:, t], pick[:, t]]
    x, y = tok[:, :-1].astype(np.int32), tok[:, 1:].copy()
    if not variable_length:
        return x, y
    lengths = synthetic_lengths(n, seq_len, seed, valid=bool(valid_of))
    pad = np.arange(seq_len)[None, :] >= lengths[:, None]
    x[pad] = 0
    y[pad] = 0
    return x, y, lengths


def process_prompts(rows: Sequence[Sequence[str]], seq_len: int, vocab_size: int):
    """Prompts of ``--mode generate``: a row is ``k`` token ids, ``1 <= k <= seq_len`` -> ``(x int32 [N, seq_len]`` right-padded
    with id 0, ``lengths int32 [N])``.  A non-integer id, an id outside ``[0, vocab_size)`` or a row that is empty or longer than
    ``seq_len`` is an error naming the row."""
    xs = []
    for n, row in enumerate(rows):
        fields = [str(v).strip() for v in row]
        if not any(fields):
            raise ValueError(f"row {n}: an empty prompt (a prompt is 1..{seq_len} token ids)")
        if len(fields) > seq_len:
            raise ValueError(f"row {n}: a prompt of {len(fields)} token ids is longer than --seq_len {seq_len}")
        ids = []
        for s in fields:
            try:
                i = int(s)
            except ValueError:
                raise ValueError(f"row {n}: token id {s!r} is not an integer") from None
            if not 0 <= i < vocab_size:
                raise ValueError(f"row {n}: token id {i} outside [0, {vocab_size}) (--vocab_size {vocab_size})")
            ids.append(i)
        xs.append(ids)
    if not xs:
        raise ValueError("no prompts: the file has no rows")
    x = np.zeros((len(xs), seq_len), dtype=np.int32)
    for i, r in enumerate(xs):
        x[i, :len(r)] = r
    return x, np.asarray([len(r) for r in xs], dtype=np.int32)


def synthetic_prompts(n: int, seq_len: int, vocab_size: int, seed: int = 0):
    """``n`` prompts from the synthetic language: the first ``max(1, seq_len // 4)`` ids of the walks of
    ``synthetic_next_token`` -> ``(x int32 [n, k], lengths int32 [n])``."""
    k = max(1, seq_len // 4)
    x = synthetic_next_token(n, seq_len, vocab_size, seed=seed)[0][:, :k].copy()
    return x, np.full(n, k, dtype=np.int32)


def legal_fraction(prompts: np.ndarray, lengths: np.ndarray, generated: np.ndarray, succ: np.ndarray) -> float:
    """The share of the generated transitions - each prompt's last id to the first generated id, then generated id to generated
    id - that the chain ``succ [V, 4]`` (``next_token_chain``) allows."""
    prev = np.concatenate([prompts[np.arange(len(lengths)), lengths - 1][:, None], generated[:, :-1]], 1).astype(np.int64)
    ok = (succ[prev] == generated.astype(np.int64)[:, :, None]).any(2)
    return float(ok.mean())


# ------------------------------------------------------------------------------------------------
# one token stream (--stateful)
# ------------------------------------------------------------------------------------------------
def token_stream(rows: Sequence[Sequence[str]], vocab_size: int) -> np.ndarray:
    """``--stateful``: the ids of every row concatenated in file order -> int64 ``[n]``.  A row holds any number of ids, at least
    one.  A non-integer id or an id outside ``[0, vocab_size)`` is an error naming the row."""
    ids = []
    for n, row in enumerate(rows):
        fields = [str(v).strip() for v in row]
        if not any(fields):
            raise ValueError(f"row {n}: no token ids (--stateful: a row is one or more ids of the stream)")
        for s in fields:
            try:
                i = int(s)
            except ValueError:
                raise ValueError(f"row {n}: token id {s!r} is not an integer") from None
            if not 0 <= i < vocab_size:
                raise ValueError(f"row {n}: token id {i} outside [0, {vocab_size}) (--vocab_size {vocab_size})")
            ids.append(i)
    if not ids:
        raise ValueError("empty stream: the file has no token ids")
    return np.asarray(ids, dtype=np.int64)


def synthetic_stream(n: int, seq_len: int, vocab_size: int, seed: int = 0, valid: bool = False) -> np.ndarray:
    """``--stateful --synthetic n``: one walk of ``n * seq_len + 1`` ids of the chain of ``synthetic_next_token``
    (``next_token_chain``) from a uniform start -> int64.  Drawn by a generator of its own: the other synthetic tasks are
    untouched.  ``valid``: a held-out walk of the same chain, from a generator of its own."""
    succ = next_token_chain(vocab_size, seed)
    m = n * seq_len + 1
    rng = np.random.default_rng([seed, 0x6E7874, 2] + ([VALID_DRAWS] if valid else []))
    tok = np.empty(m, dtype=np.int64)
    tok[0] = rng.integers(0, vocab_size)
    pick = rng.choice(4, size=m - 1, p=NEXT_TOKEN_PROBS)
    for t in range(m - 1):
        tok[t + 1] = succ[tok[t], pick[t]]
    return tok


def split_stream(stream: np.ndarray, parts: int) -> List[np.ndarray]:
    """``--partitions N`` of one stream: ``N`` contiguous pieces of ``(n - 1) // N`` transitions each; consecutive pieces share
    one id (the last id of piece r is the first of piece r + 1), so no transition is lost.  The fewer than ``N`` transitions
    left at the end are dropped."""
    per = (len(stream) - 1) // parts
    if per < 1:
        raise ValueError(f"a stream of {len(stream)} ids cannot be split into {parts} partitions")
    return [stream[r * per:(r + 1) * per + 1] for r in range(parts)]


def stream_layout(stream: np.ndarray, batch_size: int, seq_len: int, tail: bool = False):
    """One shard's stream of ``n`` ids as ``B = batch_size`` parallel streams of ``L = (n - 1) // B`` positions: stream ``b`` has
    the inputs ``s[b L + p]`` and the labels ``s[b L + p + 1]``, ``0 <= p < L``.  Segment ``k`` is positions
    ``k T .. k T + T - 1`` of every stream (``T = seq_len``); there are ``K = L // T`` of them.  -> ``(x int32 [K B, T],
    y int64 [K B, T], tail_len)``, rows in (segment, stream) order, so batch ``k`` is rows ``k B .. k B + B - 1``.

    Training drops the ``L - K T < T`` positions left at the end of each stream (``tail_len = 0``).  ``tail``: they become one
    more segment, right-padded with id 0 and label 0, and ``tail_len = L - K T`` is its length in every row (0: none)."""
    n, B, T = len(stream), int(batch_size), int(seq_len)
    L = (n - 1) // B
    K = L // T
    if K == 0 and not (tail and L > 0):
        raise ValueError(f"a shard of {n} ids holds no segment of --batch_size {B} streams x --seq_len {T} positions: it needs "
                         f"at least {B * T + 1} ids")
    inp = stream[:B * L].reshape(B, L)
    lab = stream[1:B * L + 1].reshape(B, L)
    rest = L - K * T if tail else 0
    segs = K + (1 if rest else 0)
    x = np.zeros((B, segs * T), dtype=np.int32)
    y = np.zeros((B, segs * T), dtype=np.int64)
    x[:, :K * T + rest] = inp[:, :K * T + rest]
    y[:, :K * T + rest] = lab[:, :K * T + rest]
    x = x.reshape(B, segs, T).transpose(1, 0, 2).reshape(segs * B, T)
    y = y.reshape(B, segs, T).transpose(1, 0, 2).reshape(segs * B, T)
    return np.ascontiguousarray(x), np.ascontiguousarray(y), rest


def load_stream(cfg, n_synthetic: int = 0) -> np.ndarray:
    """The token stream of ``--stateful``: ``--synthetic n`` walks ``synthetic_stream``, otherwise the ids of ``--training_path``
    (``token_stream``)."""
    if cfg.synthetic:
        return synthetic_stream(n_synthetic or cfg.synthetic, cfg.seq_len, cfg.vocab_size, cfg.seed)
    return token_stream(read_dataset_from_path(cfg.training_path), cfg.vocab_size)


def synthetic_lengths(n: int, seq_len: int, seed: int = 0, valid: bool = False) -> np.ndarray:
    """Per-sample lengths, uniform in ``[max(1, seq_len // 4), seq_len]``, int32, from a generator seeded apart from the data's
    (``valid``: the lengths of a held-out set, from a generator of their own)."""
    rng = np.random.default_rng([seed, 0x6C656E] + ([VALID_DRAWS] if valid else []))
    return rng.integers(max(1, seq_len // 4), seq_len + 1, size=n).astype(np.int32)


def synthetic(cfg, n: int, seed: int, valid_of: int = 0):
    """``n`` synthetic samples of the task the flags of ``cfg`` select -> ``(x, y, lengths)``; ``lengths`` is None unless
    ``cfg.variable_length``.  ``valid_of = m > 0``: ``n`` held-out samples of the task ``synthetic(cfg, m, seed)`` draws from."""
    if getattr(cfg, "next_token", False):
        x, y, *lengths = synthetic_next_token(n, cfg.seq_len, cfg.vocab_size, seed=seed, variable_length=cfg.variable_length,
                                              valid_of=valid_of)
    elif cfg.vocab_size > 0:
        x, y, *lengths = synthetic_tokens(n, cfg.seq_len, cfg.vocab_size, cfg.num_classes, seed=seed,
                                          variable_length=cfg.variable_length, per_step_labels=cfg.per_step_labels,
                                          valid_of=valid_of)
    elif cfg.per_step_labels:
        x, y, *lengths = synthetic_per_step(n, cfg.seq_len, cfg.in_features, cfg.num_classes, seed=seed,
                                            variable_length=cfg.variable_length, valid_of=valid_of)
    else:
        x, y, *lengths = synthetic_sequences(n, cfg.seq_len, cfg.in_features, cfg.num_classes, seed=seed,
                                             variable_length=cfg.variable_length, valid_of=valid_of)
    return x, y, (lengths[0] if lengths else None)


def load_validation(cfg, n_train: int):
    """The held-out set of ``--valid_path`` / ``--valid_synthetic``, or None: a token stream with ``--stateful``, else
    ``(x, y, lengths)`` as ``parse_rows`` gives them.  ``--valid_synthetic`` draws from the task of the first training shard
    (``n_train`` samples of ``--synthetic`` at ``--seed``)."""
    if cfg.valid_synthetic:
        if cfg.stateful:
            return synthetic_stream(cfg.valid_synthetic, cfg.seq_len, cfg.vocab_size, cfg.seed, valid=True)
        return synthetic(cfg, cfg.valid_synthetic, cfg.seed, valid_of=max(1, n_train))
    if cfg.valid_path:
        rows = read_dataset_from_path(cfg.valid_path)
        return token_stream(rows, cfg.vocab_size) if cfg.stateful else parse_rows(rows, cfg)
    return None


# ------------------------------------------------------------------------------------------------
# loaders
# ------------------------------------------------------------------------------------------------
class DeviceShard:
    """Device-resident shard; a batch is an index gather on the device, no per-step H2D
    (replaces the per-step feed_dict copy, src/rnn.py:264-267)."""

    def __init__(self, x: np.ndarray, y: np.ndarray, batch_size: int, device, dtype=torch.float32,
                 shuffle: bool = True, seed: int = 0, lengths: Optional[np.ndarray] = None):
        """``lengths``: optional per-row sequence lengths; they follow their rows and ``next()`` returns them third."""
        self.x = torch.as_tensor(x).to(device=device, dtype=dtype)
        self.y = torch.as_tensor(y).to(device=device)
        self.lengths = None if lengths is None else torch.as_tensor(lengths).to(device=device, dtype=torch.int32)
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

    def next(self, out=None) -> Tuple[torch.Tensor, ...]:
        """-> ``(x, y)``, or ``(x, y, lengths)`` for a shard with lengths.  ``out = (x_buf, y_buf[, lengths_buf])``: gather the
        batch straight into these buffers (the input buffers of a captured CUDA graph: ``TrainEngine.graph_inputs()``)
        instead of into fresh tensors that then have to be copied there."""
        if self._perm is None or self._i >= self.per_epoch:
            self._reshuffle()
        lo = self._i * self.batch_size
        idx = self._perm[lo:lo + self.batch_size]
        self._i += 1
        out_l = out[2] if (out is not None and len(out) > 2) else None
        if out is not None and out[0].shape[0] == idx.numel() and out[0].dtype == self.x.dtype \
                and (self.lengths is None or out_l is not None):
            torch.index_select(self.x, 0, idx, out=out[0])
            torch.index_select(self.y, 0, idx, out=out[1])
            if self.lengths is None:
                return out[0], out[1]
            torch.index_select(self.lengths, 0, idx, out=out_l)
            return out[0], out[1], out_l
        if self.lengths is None:
            return self.x.index_select(0, idx), self.y.index_select(0, idx)
        return self.x.index_select(0, idx), self.y.index_select(0, idx), self.lengths.index_select(0, idx)

    def opened_pass(self) -> bool:
        """Was the batch ``next()`` handed out last the first of a pass over the shard?"""
        return self._i == 1

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
                 shuffle: bool = True, seed: int = 0, depth: int = 2, lengths: Optional[np.ndarray] = None):
        """``depth``: device staging slots (the copy of a batch is enqueued ``depth - 1`` calls before it is handed out).
        ``lengths``: optional per-row sequence lengths, permuted and copied with their rows; ``next()`` returns them third
        and every staging slot of ``dev`` is an ``(x, y, lengths)`` triple."""
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
        self.l_host = None if lengths is None else torch.as_tensor(lengths).to(torch.int32).contiguous()
        if cuda:
            self.x_host = self.x_host.pin_memory()
            self.y_host = self.y_host.pin_memory()
            if self.l_host is not None:
                self.l_host = self.l_host.pin_memory()
        shape_x = (self.batch_size,) + tuple(self.x_host.shape[1:])
        shape_y = (self.batch_size,) + tuple(self.y_host.shape[1:])          # [B], or [B,T] with a label per step
        self.dev = [(torch.empty(shape_x, dtype=dtype, device=self.device),
                     torch.empty(shape_y, dtype=torch.int64, device=self.device))
                    + (() if self.l_host is None else (torch.empty((self.batch_size,), dtype=torch.int32, device=self.device),))
                    for _ in range(depth)]
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
        self.bytes_per_batch = self.dev[0][0].numel() * self.dev[0][0].element_size() + self.dev[0][1].numel() * 8 \
            + (0 if self.l_host is None else self.batch_size * 4)

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
        if self.l_host is not None:
            self.l_host.copy_(self.l_host[idx])
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

    def opened_pass(self) -> bool:
        """Was the batch ``next()`` handed out last the first of a pass over the shard?"""
        return self._consumed[1] == 1

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
        if self.l_host is not None:
            self.l_host.copy_(self.l_host[order])
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
        slot = self.dev[self._slot]
        dx, dy = slot[0], slot[1]
        self._slot = (self._slot + 1) % self.depth
        if self.device.type != "cuda":
            dx.copy_(self.x_host[lo:lo + self.batch_size])
            dy.copy_(self.y_host[lo:lo + self.batch_size])
            if self.l_host is not None:
                slot[2].copy_(self.l_host[lo:lo + self.batch_size])
            return slot, None, tag
        if self._copy_stream is None:
            self._copy_stream = torch.cuda.Stream(device=self.device)
        # the slot being overwritten was consumed by compute work already enqueued on the current stream
        self._copy_stream.wait_stream(torch.cuda.current_stream(self.device))
        with torch.cuda.stream(self._copy_stream):
            if not self.debug_skip_copy:                  # (bench diagnostics only: how much of a step is the DMA's interference?)
                dx.copy_(self.x_host[lo:lo + self.batch_size], non_blocking=True)
                dy.copy_(self.y_host[lo:lo + self.batch_size], non_blocking=True)
                if self.l_host is not None:
                    slot[2].copy_(self.l_host[lo:lo + self.batch_size], non_blocking=True)
            ev = torch.cuda.Event()
            ev.record(self._copy_stream)
        return slot, ev, tag

    def next(self) -> Tuple[torch.Tensor, ...]:
        """Returns this step's batch - ``(x, y)``, or ``(x, y, lengths)`` with lengths - (its H2D copy was enqueued one call
        earlier, so it overlaps the previous step's compute) and enqueues the copy of the following one.  Every step still
        moves its own inputs host->device."""
        while len(self._pending) < self.depth - 1:
            self._pending.append(self._issue())
        slot, ev, self._consumed = self._pending.pop(0)
        if ev is not None:
            torch.cuda.current_stream(self.device).wait_event(ev)
        # refill: the slot this copy overwrites was handed out depth - 1 calls ago; the step that consumed it is enqueued
        self._pending.append(self._issue())
        return slot
