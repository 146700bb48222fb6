"""Cross-replica communication: the parameter average / gradient allreduce.

Reference: ``weights_rdd.reduceByKey(mean_weights).collect()`` — a Spark shuffle keyed by the 8 gate
names plus a driver-side collect (original src/rnn.py:393-407), run once per job; intended semantics =
element-wise mean over partitions (Q1).  Here one rank per GPU; three interchangeable back ends behind one
interface:

  * ``fused`` : hand-written sm_90a kernel doing the reduction over NVLink peer / NVLS multicast pointers
                with the update (average, SGD, Adam) fused in — the product path (parallel/fused_comm.py);
  * ``nccl``  : ``dist.all_reduce`` + separate update kernels — the baseline the fused path is measured against;
  * ``gloo``  : the same on CPU, used by the multi-process tests (our analogue of Spark ``local[N]``).
"""
from __future__ import annotations

import datetime
import os
from typing import Optional

import torch
import torch.distributed as dist

from ..models.flat import FlatParams


class Communicator:
    """world_size == 1 / base class: every collective is the identity."""
    name = "single"

    def __init__(self, rank: int = 0, world_size: int = 1):
        self.rank, self.world_size = rank, world_size

    # -- plumbing ---------------------------------------------------------------------------------
    def barrier(self):
        pass

    def broadcast_object(self, obj, src: int = 0):
        return obj

    def all_gather_object(self, obj):
        return [obj]

    def max_scalar(self, v: float) -> float:
        return v

    def adopt(self, flat: FlatParams):
        """Give the back end a chance to move the flat buffers into symmetric memory."""
        return flat

    # -- the hot path -------------------------------------------------------------------------------
    def average_params_(self, flat: FlatParams, scope: str = "lstm"):
        """w <- (sum_p w_p) / N over the chosen scope; result lands in every replica."""
        flat.refresh_shadow()

    def grad_step_(self, flat: FlatParams, optimizer):
        """g <- (sum_p g_p) / N then optimizer update (fused where the back end can)."""
        optimizer.step()

    def broadcast_params_(self, flat: FlatParams, src: int = 0):
        pass

    def optimizer_state(self, optimizer) -> dict:
        """Checkpointable optimizer state (complete on every rank)."""
        return optimizer.state_dict()

    def load_optimizer_state(self, optimizer, sd: dict):
        """Inverse of ``optimizer_state`` (the fused back end keeps only its own slice of Adam's m / v)."""
        optimizer.load_state_dict(sd)

    def allreduce_sum_(self, t: torch.Tensor) -> torch.Tensor:
        """Plain elementwise sum over ranks of a (CPU or device) tensor - job finalisation only, never on the step path."""
        return t

    def close(self):
        pass


class TorchDistComm(Communicator):
    """NCCL (GPU) / gloo (CPU) collectives + separate update — the baseline path."""

    def __init__(self, rank: int, world_size: int, backend: str, device: torch.device, timeout_s: float = 600.0):
        super().__init__(rank, world_size)
        self.name = backend
        self.backend = backend          # the torch.distributed backend (subclasses may change `name`)
        self.device = device
        if not dist.is_initialized():
            kw = {}
            if backend == "nccl":
                kw["device_id"] = device
            dist.init_process_group(backend=backend, rank=rank, world_size=world_size,
                                    timeout=datetime.timedelta(seconds=timeout_s), **kw)
        self.group = dist.group.WORLD

    def barrier(self):
        if self.backend == "nccl":
            dist.barrier(device_ids=[self.device.index])
        else:
            dist.barrier()

    def broadcast_object(self, obj, src: int = 0):
        box = [obj]
        dist.broadcast_object_list(box, src=src)
        return box[0]

    def all_gather_object(self, obj):
        out = [None] * self.world_size
        dist.all_gather_object(out, obj)
        return out

    def max_scalar(self, v: float) -> float:
        t = torch.tensor([v], dtype=torch.float64, device=self.device if self.backend == "nccl" else "cpu")
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return float(t.item())

    def average_params_(self, flat: FlatParams, scope: str = "lstm"):
        lo, hi = flat.segment(scope)
        seg = flat.data[lo:hi]
        dist.all_reduce(seg, op=dist.ReduceOp.SUM)
        seg.mul_(1.0 / self.world_size)
        flat.refresh_shadow()

    def grad_step_(self, flat: FlatParams, optimizer):
        dist.all_reduce(flat.grad, op=dist.ReduceOp.SUM)
        optimizer.step(grad_scale=1.0 / self.world_size)

    def broadcast_params_(self, flat: FlatParams, src: int = 0):
        dist.broadcast(flat.data, src=src)
        flat.refresh_shadow()

    def allreduce_sum_(self, t: torch.Tensor) -> torch.Tensor:
        buf = t.to(self.device) if self.backend == "nccl" else t.cpu()
        dist.all_reduce(buf, op=dist.ReduceOp.SUM)
        t.copy_(buf.to(t.device))
        return t

    def close(self):
        if dist.is_initialized():
            try:
                dist.destroy_process_group()
            except Exception:
                pass


def resolve_comm(kind: str, device: torch.device, clip_synced_grads: bool = False) -> str:
    """``auto``: the fused NVLink allreduce on GPUs, gloo on the CPU; nccl on GPUs when the gradient is clipped by the norm of
    the averaged gradient (the fused allreduce updates each gradient bucket before that norm is known)."""
    if kind != "auto":
        return kind
    if device.type != "cuda":
        return "gloo"
    return "nccl" if clip_synced_grads else "fused"


def make_communicator(kind: str, rank: int, world_size: int, device: torch.device, timeout_s: float = 600.0,
                      clip_synced_grads: bool = False) -> Communicator:
    if world_size == 1 and kind in ("auto", "gloo", "nccl"):
        return Communicator(0, 1)
    kind = resolve_comm(kind, device, clip_synced_grads)
    if kind == "gloo":
        return TorchDistComm(rank, world_size, "gloo", device, timeout_s)
    if kind == "nccl":
        return TorchDistComm(rank, world_size, "nccl", device, timeout_s)
    if kind == "fused":
        from .fused_comm import FusedComm
        return FusedComm(rank, world_size, device, timeout_s)
    raise ValueError(f"unknown comm back end {kind!r}")
