"""Rank launcher: ``--partitions N`` -> N processes, one per GPU (replaces SparkConf/SparkContext +
``local[N]`` executors, original src/rnn.py:355-363).  Honours a torchrun environment
(RANK / WORLD_SIZE / LOCAL_RANK / MASTER_*) when present; otherwise spawns the ranks itself on 127.0.0.1.

Failure detection: the parent polls its children; the first abnormal exit terminates the
remaining ranks and surfaces as ``RankFailure`` carrying every exit code — a dead peer is an error, not a hang.
"""
from __future__ import annotations

import io
import os
import socket
import sys
import time
import traceback
from typing import Callable, Dict, List, Optional

import torch
import torch.multiprocessing as mp


class RankFailure(RuntimeError):
    def __init__(self, exit_codes: Dict[int, Optional[int]]):
        self.exit_codes = exit_codes
        bad = {r: c for r, c in exit_codes.items() if c not in (0, None)}
        super().__init__(f"rank failure: exit codes {bad} (all: {exit_codes})")


def _free_port() -> int:
    with socket.socket(socket.AF_INET, socket.SOCK_STREAM) as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def in_torchrun() -> bool:
    return "RANK" in os.environ and "WORLD_SIZE" in os.environ


def _child(rank: int, world_size: int, port: int, fn: Callable, args: tuple, result_q):
    os.environ["RANK"] = str(rank)
    os.environ["LOCAL_RANK"] = str(rank)
    os.environ["WORLD_SIZE"] = str(world_size)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    try:
        out = fn(rank, world_size, *args)
        if result_q is not None:
            buf = io.BytesIO()
            torch.save(out, buf)                 # by value: fd-shared tensors die with the child
            result_q.put((rank, buf.getvalue()))
    except BaseException:
        traceback.print_exc()
        sys.stderr.flush()
        os._exit(1)


def launch(fn: Callable, world_size: int, args: tuple = (), poll_s: float = 0.2, timeout_s: Optional[float] = None,
           collect: bool = True) -> List:
    """Run ``fn(rank, world_size, *args)`` on every rank; returns the per-rank results ordered by rank."""
    if in_torchrun():
        rank = int(os.environ["RANK"])
        ws = int(os.environ["WORLD_SIZE"])
        return [fn(rank, ws, *args)]
    if world_size == 1:
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        os.environ.setdefault("MASTER_PORT", str(_free_port()))
        return [fn(0, 1, *args)]
    ctx = mp.get_context("spawn")
    port = _free_port()
    q = ctx.Queue() if collect else None
    procs = [ctx.Process(target=_child, args=(r, world_size, port, fn, args, q), daemon=False) for r in range(world_size)]
    for p in procs:
        p.start()
    results: Dict[int, object] = {}
    t0 = time.time()
    failed = False
    while True:
        if q is not None:
            while not q.empty():
                r, out = q.get()
                results[r] = torch.load(io.BytesIO(out), weights_only=False)
        codes = {r: p.exitcode for r, p in enumerate(procs)}
        if any(c not in (0, None) for c in codes.values()):
            failed = True
            break
        if all(c == 0 for c in codes.values()):
            break
        if timeout_s is not None and time.time() - t0 > timeout_s:
            failed = True
            break
        time.sleep(poll_s)
    if failed:
        time.sleep(0.5)
        for p in procs:
            if p.is_alive():
                p.terminate()
        for p in procs:
            p.join(5)
            if p.is_alive():
                p.kill()
        raise RankFailure({r: p.exitcode for r, p in enumerate(procs)})
    for p in procs:
        p.join()
    if q is not None:
        while not q.empty():
            r, out = q.get()
            results[r] = torch.load(io.BytesIO(out), weights_only=False)
    return [results.get(r) for r in range(world_size)]
