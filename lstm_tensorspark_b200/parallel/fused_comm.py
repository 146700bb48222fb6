"""``--comm fused``: the product path of the cross-replica sync.

The flat parameter / gradient / bf16-shadow buffers of every rank are carved out of ONE NVLink-symmetric
allocation (``torch.distributed._symmetric_memory``: cuMem VMM handles exchanged between ranks, plus an NVLS
multicast alias when the fabric supports it).  The sync itself is a single launch of
``csrc/fused_allreduce.cu`` per rank: reduction over peer / multicast pointers fused with the update
(average | SGD | Adam) and the bf16 shadow refresh.  NCCL is used only to bootstrap (store, rendezvous) and for
python-object broadcasts; no NCCL collective and no separate elementwise kernel runs on the sync path.

Replaces ``reduceByKey(mean_weights)`` + ``collect()`` (original src/rnn.py:393-407).
"""
from __future__ import annotations

import os
from typing import Optional

import torch
import torch.distributed as dist

from ..models.flat import FlatParams
from ..ops.cuda_ext import ext
from .comm import TorchDistComm

MODE_AVG, MODE_SGD, MODE_ADAM = 0, 1, 2
TWO_SHOT_BYTES = int(os.environ.get("LSTM_TS_AR_TWO_SHOT_BYTES", str(8 * 1024)))      # measured at 8 GPUs: two-shot wins from 16 KB up, ties below
AR_BLOCKS = int(os.environ.get("LSTM_TS_AR_BLOCKS", "64"))
AR_BLOCKS_P2P_LARGE = int(os.environ.get("LSTM_TS_AR_BLOCKS_P2P_LARGE", "128"))
AR_BLOCKS_LARGE = int(os.environ.get("LSTM_TS_AR_BLOCKS_LARGE", "64"))    # messages >= 32 MB (measured: 64 = 128 = 256 blocks, unroll irrelevant: sweep8c.log)


def _align(x: int, a: int = 4096) -> int:
    return (x + a - 1) // a * a


class SymmetricArena:
    """One symmetric allocation, sub-allocated at identical offsets on every rank."""

    def __init__(self, nbytes: int, device: torch.device, group):
        import torch.distributed._symmetric_memory as symm_mem
        self.buf = symm_mem.empty(nbytes, dtype=torch.uint8, device=device)
        self.buf.zero_()
        self.hdl = symm_mem.rendezvous(self.buf, group.group_name if hasattr(group, "group_name") else group)
        self.rank = self.hdl.rank
        self.world = self.hdl.world_size
        base = [int(p) for p in self.hdl.buffer_ptrs]
        delta = self.buf.data_ptr() - base[self.rank]
        self.base = [b + delta for b in base]
        mc = 0
        try:
            mc = int(self.hdl.multicast_ptr or 0)
        except Exception:                                   # noqa: BLE001
            mc = 0
        self.mc_base = (mc + delta) if mc else 0
        self.off = 0
        self.nbytes = nbytes

    def carve(self, numel: int, dtype: torch.dtype):
        nbytes = numel * torch.empty((), dtype=dtype).element_size()
        off = self.off
        assert off + nbytes <= self.nbytes, "symmetric arena exhausted"
        self.off = _align(off + nbytes)
        # NOT a view of self.buf: views share one autograd version counter, and an in-place update of the grad region
        # would then invalidate bf16-shadow views saved for backward.  set_() aliases the storage with its own counter.
        esize = torch.empty((), dtype=dtype).element_size()
        t = torch.empty(0, dtype=dtype, device=self.buf.device).set_(
            self.buf.untyped_storage(), (self.buf.storage_offset() + off) // esize, (numel,))
        return t, off

    def peers(self, off: int):
        return [b + off for b in self.base]

    def mc(self, off: int) -> int:
        return self.mc_base + off if self.mc_base else 0


class FusedComm(TorchDistComm):
    name = "fused"

    def __init__(self, rank: int, world_size: int, device: torch.device, timeout_s: float = 600.0):
        super().__init__(rank, world_size, "nccl", device, timeout_s)
        self.name = "fused"
        self.timeout_s = timeout_s
        self.arena: Optional[SymmetricArena] = None
        self.use_multicast = os.environ.get("LSTM_TS_AR_MULTICAST", "auto")
        self.blocks_override = 0          # tuning knob (bench/allreduce_sweep.py)
        self.launches = 0
        self._state_buckets = []          # (lo, hi, two_shot) buckets of the last fused Adam step: who owns which m / v slice
        self._gs = None

    # ------------------------------------------------------------------------------------------------
    def adopt(self, flat: FlatParams):
        E = ext()
        n = flat.padded_numel
        flag_words = E.ar_flag_words()
        total = 3 * _align(4 * n) + _align(2 * n) + _align(4 * flag_words) + 4096
        self.arena = SymmetricArena(total, self.device, dist.group.WORLD)
        A = self.arena
        self.data, self.off_data = A.carve(n, torch.float32)
        self.grad, self.off_grad = A.carve(n, torch.float32)
        self.stage, self.off_stage = A.carve(n, torch.float32)
        self.shadow, self.off_shadow = A.carve(n, torch.bfloat16)
        self.flags, self.off_flags = A.carve(flag_words, torch.int32)
        flat.rebase(self.data, self.grad)
        had_shadow = flat.shadow is not None
        flat.shadow = self.shadow
        flat.refresh_shadow()
        self.slots = E.ar_slots()
        self.epochs = torch.zeros(E.ar_max_blocks() * self.slots, dtype=torch.int32, device=self.device)
        self.err = torch.zeros(1, dtype=torch.int32, device=self.device)
        self.flat = flat
        torch.cuda.synchronize(self.device)
        dist.barrier(device_ids=[self.device.index])
        return flat

    def _ptr_table(self, off_in: int) -> torch.Tensor:
        A = self.arena
        rows = [A.peers(off_in), A.peers(self.off_data), A.peers(self.off_shadow), A.peers(self.off_flags)]
        return torch.tensor(rows, dtype=torch.int64)

    def _multicast_on(self) -> bool:
        if self.use_multicast in ("0", "off", "false"):
            return False
        return bool(self.arena.mc_base)

    def _launch(self, mode: int, off_in: int, n: int, lr: float = 0.0, b1: float = 0.0, b2: float = 0.0, eps: float = 0.0,
                wd: float = 0.0, m=None, v=None, force: Optional[str] = None, step_dev=None, elem_off: int = 0,
                wd_numel: int = -1, bump_step: bool = True, pdl: bool = False, blocks: int = 0, slot: int = 0):
        """One launch over elements [elem_off, elem_off + n) of the symmetric buffers (a gradient bucket or the whole message)."""
        E = ext()
        A = self.arena
        # the kernel moves float4s: a bucket starts on one, and its clipped weight-decay cut below stays a multiple of 4
        assert elem_off % 4 == 0, f"bucket offset {elem_off} is not a multiple of 4 elements"
        two_shot = (4 * n >= TWO_SHOT_BYTES) if force is None else (force == "two_shot")
        # NVLS (in-switch reduction) pays from 3 ranks up; with 2 ranks the peer-pointer kernel is faster stand-alone (measured:
        # measured) - but it needs 122 registers, so a bucket that has to squeeze onto the SMs a
        # GEMM leaves idle (pdl) keeps the 32-register multimem variant
        mc = self._multicast_on() and two_shot and (self.world_size > 2 or pdl or self.use_multicast in ("1", "on", "force"))
        if mode == MODE_AVG and not two_shot:
            off_in_eff = self.off_stage        # one-shot average stages w first
        else:
            off_in_eff = off_in
        e4, e2 = 4 * elem_off, 2 * elem_off
        mb = E.ar_max_blocks()
        slot = slot % self.slots                       # independent barrier state per slot (kernels of two buckets may overlap)
        fl = 4 * slot * (E.ar_flag_words() // self.slots)
        rows = [[p + e4 for p in A.peers(off_in_eff)], [p + e4 for p in A.peers(self.off_data)],
                [p + e2 for p in A.peers(self.off_shadow)], [p + fl for p in A.peers(self.off_flags)]]
        ptrs = torch.tensor(rows, dtype=torch.int64)
        if m is not None and elem_off:
            m, v = m[elem_off:elem_off + n], v[elem_off:elem_off + n]
        elif m is not None and m.numel() != n:
            m, v = m[:n], v[:n]
        if wd_numel >= 0:
            wd_numel = max(0, min(n, wd_numel - elem_off))
        # grid: the NVLS kernel is switch-bound (64 = 128 = 256 CTAs); the peer-pointer kernel is bound by bytes in
        # flight per SM - 128 CTAs from 4 MB up (2 GPUs, 1 GB: 2.00 ms vs 2.57 ms with 64; NCCL 2.20 ms)
        nblk = blocks or self.blocks_override or ((AR_BLOCKS_P2P_LARGE if 4 * n >= (4 << 20) else AR_BLOCKS) if not mc
                                                  else (AR_BLOCKS_LARGE if 4 * n >= (32 << 20) else AR_BLOCKS))
        E.fused_allreduce(ptrs, (A.mc(off_in_eff) + e4) if mc else 0, (A.mc(self.off_data) + e4) if mc else 0,
                          (A.mc(self.off_shadow) + e2) if mc else 0, m, v, self.epochs[slot * mb:(slot + 1) * mb], self.err, n, self.rank, self.world_size,
                          mode, two_shot, mc, nblk, lr, b1, b2, eps, wd, float(self.timeout_s), step_dev, wd_numel, bump_step, pdl)
        self.launches += 1
        return two_shot

    # ------------------------------------------------------------------------------------------------
    def average_params_(self, flat: FlatParams, scope: str = "lstm", force: Optional[str] = None):
        lo, hi = flat.segment(scope)
        assert lo == 0
        self._launch(MODE_AVG, self.off_data, hi, force=force)

    def grad_step_(self, flat: FlatParams, optimizer, force: Optional[str] = None):
        """Whole-message gradient sync + update in one launch (no overlap)."""
        self.begin_grad_step(flat, optimizer)
        self.launch_bucket(0, flat.padded_numel, force=force)

    # -- bucketed gradient sync: a bucket's allreduce + update is launched as soon as its gradients are final ----------
    def begin_grad_step(self, flat: FlatParams, optimizer):
        optimizer.step_count += 1
        if optimizer.kind == "adam" and optimizer.step_dev is not None:
            ext().ar_bump_step(optimizer.step_dev)          # here, not inside a bucket launch (see csrc/fused_allreduce.cu)
        self._gs = {"opt": optimizer, "bump": False, "buckets": []}
        if optimizer.kind == "adam":
            self._state_buckets = self._gs["buckets"]       # filled as the step's buckets launch; complete between steps

    def launch_bucket(self, lo: int, hi: int, pdl: bool = False, force: Optional[str] = None, blocks: int = 0):
        gs = self._gs
        opt = gs["opt"]
        n = hi - lo
        if opt.kind == "adam":
            two = self._launch(MODE_ADAM, self.off_grad, n, opt.lr, opt.beta1, opt.beta2, opt.eps, opt.weight_decay, opt.m, opt.v,
                               force=force, step_dev=opt.step_dev, elem_off=lo, wd_numel=opt.wd_numel, bump_step=gs["bump"],
                               pdl=pdl, blocks=blocks, slot=len(gs["buckets"]))
        else:
            two = self._launch(MODE_SGD, self.off_grad, n, opt.lr, wd=opt.weight_decay, force=force, elem_off=lo,
                               wd_numel=opt.wd_numel, pdl=pdl, blocks=blocks, slot=len(gs["buckets"]))
        gs["bump"] = False
        gs["buckets"].append((lo, hi, bool(two)))

    def _owned_ranges(self):
        """Element ranges of the flat buffer whose Adam slots THIS rank maintains: a two-shot bucket is split like the kernel
        splits it (ceil(n4 / world) float4 per rank, csrc/fused_allreduce.cu); a one-shot bucket is updated identically by every
        rank (rank 0 contributes it)."""
        out = []
        for lo, hi, two in self._state_buckets:
            if not two:
                if self.rank == 0:
                    out.append((lo, hi))
                continue
            n4 = (hi - lo) // 4
            per = (n4 + self.world_size - 1) // self.world_size
            a = min(per * self.rank, n4)
            b = min(a + per, n4)
            out.append((lo + 4 * a, lo + 4 * b))
        return out

    def optimizer_state(self, optimizer) -> dict:
        """The two-shot fused gradient step keeps Adam's (m, v) for 1/N of every bucket on each rank (the slice it reduces
        and updates).  A checkpoint holds the FULL state: every rank contributes exactly its owned slices (everything else
        masked to zero, whatever it holds) and a sum reassembles it.  Any other mode (parameter averaging: every rank runs
        its own full optimizer) returns the local state."""
        sd = optimizer.state_dict()
        if self._state_buckets and optimizer.kind == "adam" and self.world_size > 1:
            for k in ("m", "v"):
                src = getattr(optimizer, k)
                full = torch.zeros_like(src)
                for lo, hi in self._owned_ranges():
                    full[lo:hi] = src[lo:hi]
                dist.all_reduce(full, op=dist.ReduceOp.SUM)
                sd[k] = full.cpu()
        return sd

    def load_optimizer_state(self, optimizer, sd: dict):
        optimizer.load_state_dict(sd)          # full m / v everywhere; the two-shot step only ever reads the owned slice

    def check_errors(self):
        if int(self.err.item()) != 0:
            raise RuntimeError("fused allreduce: cross-GPU barrier timed out (a peer rank is dead or stalled)")

    def close(self):
        try:
            if self.arena is not None:
                torch.cuda.synchronize(self.device)
                self.check_errors()
        finally:
            super().close()
