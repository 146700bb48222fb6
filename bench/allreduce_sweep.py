#!/usr/bin/env python
"""BASELINE.json config 5: parameter-average allreduce bandwidth sweep, 1 KB - 1 GB, fused kernel vs NCCL.

    torchrun --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port 29533 bench/allreduce_sweep.py

For every message size: our fused kernel (one-shot / two-shot, peer-pointer / NVLS multicast) doing the in-place
fp32 average + bf16 shadow refresh, against ``dist.all_reduce`` + the separate scale kernel the NCCL path needs.
Device-timed with CUDA events, max over ranks.  Reports algorithm bandwidth S/t and bus bandwidth 2(N-1)/N * S/t
against the 450 GB/s/dir NVLink 4 nominal of an H100 (not measured here).
"""
from __future__ import annotations

import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch
import torch.distributed as dist


def time_ms(fn, iters, warm, dev, world):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize(dev)
    dist.barrier(device_ids=[dev.index])
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize(dev)
    t = torch.tensor([e0.elapsed_time(e1) / iters], dtype=torch.float64, device=dev)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item())


def main():
    rank = int(os.environ.get("RANK", "0")); world = int(os.environ.get("WORLD_SIZE", "1"))
    local = int(os.environ.get("LOCAL_RANK", str(rank)))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    from lstm_tensorspark_b200.models.flat import FlatParams
    from lstm_tensorspark_b200.parallel.fused_comm import FusedComm
    max_bytes = int(os.environ.get("SWEEP_MAX_BYTES", str(1 << 30)))
    tune = os.environ.get("SWEEP_TUNE", "0") == "1"          # also sweep grid size / unroll of the NVLS kernel
    comm = FusedComm(rank, world, dev, 120)
    p = torch.nn.Parameter(torch.zeros(max_bytes // 4, device=dev))
    flat = FlatParams([p], [])
    comm.adopt(flat)
    rows = []
    size = 1024
    nccl_buf = torch.zeros(max_bytes // 4, device=dev)
    while size <= max_bytes:
        n = size // 4
        n = max(1024 // 4, (n + 3) // 4 * 4)
        iters = 200 if size <= (1 << 20) else (50 if size <= (1 << 26) else 10)
        rec = {"bytes": n * 4, "world": world}
        variants = [("auto", None, "auto", 0, False), ("one_shot", "one_shot", "0", 0, False), ("two_shot_p2p", "two_shot", "0", 0, False)]
        if comm.arena.mc_base:
            variants.append(("two_shot_nvls", "two_shot", "force", 0, False))
        if tune and size >= (1 << 22):
            variants += [("p2p_b128", "two_shot", "0", 128, False), ("p2p_b132", "two_shot", "0", 132, False), ("p2p_b256", "two_shot", "0", 256, False)]
        if comm.arena.mc_base:
            if tune and size >= (1 << 22):
                variants += [("nvls_b64", "two_shot", "auto", 64, False), ("nvls_b128", "two_shot", "auto", 128, False),
                             ("nvls_b256", "two_shot", "auto", 256, False)]
        for name, force, mc, blocks, unroll in variants:
            if force == "one_shot" and size > (1 << 26):
                continue
            comm.use_multicast = mc
            comm.blocks_override = blocks

            def fn():
                comm._launch(0, comm.off_data, n, force=force)
            ms = time_ms(fn, iters, 5, dev, world)
            rec[name + "_us"] = ms * 1e3
            rec[name + "_busbw_GBs"] = 2 * (world - 1) / world * n * 4 / (ms / 1e3) / 1e9
        seg = nccl_buf[:n]

        def fn_nccl():
            dist.all_reduce(seg)
            seg.mul_(1.0 / world)
        ms = time_ms(fn_nccl, iters, 5, dev, world)
        rec["nccl_us"] = ms * 1e3
        rec["nccl_busbw_GBs"] = 2 * (world - 1) / world * n * 4 / (ms / 1e3) / 1e9
        rows.append(rec)
        if rank == 0:
            print(json.dumps(rec), flush=True)
        size *= 4
    comm.check_errors()
    if rank == 0:
        os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
        with open(os.path.join(ROOT, "gpurun_out", f"allreduce_sweep_n{world}.json"), "w") as f:
            json.dump(rows, f, indent=1)
    comm.close()


if __name__ == "__main__":
    main()
