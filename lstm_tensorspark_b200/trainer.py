"""Per-replica trainer + job driver.

Parity targets (reference, read-only):
  * ``train_rnn(partition, net_settings, FLAGS, train_optimizer)``   original src/rnn.py:180-297
  * standalone ``train_rnn(dataset, net_settings, train_optimizer)`` original src/lstm-no-spark.py:153-251
  * driver ``main``                                                    original src/rnn.py:339-411

One implementation serves both entry points.  Differences by design: the cross-replica mean
is exact and is written back into every replica and to ``--output_path`` (Q1, Q12); one run timestamp is
shared by all ranks; a real resume path exists (Q4); replicas start from identical seeded weights unless
``--independent_init`` (Q9).
"""
from __future__ import annotations

import json
import math
import os
import sys
import time
from typing import Callable, Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import data as D
from .config import Config
from .models.classifier import SequenceClassifier
from .models.recurrent.lstm import clear_weight_decay_collection
from .ops import functional as F
from .ops.loss import report_accuracy, report_loss
from .ops.optim import FlatOptimizer, nonmono_trigger
from .parallel.comm import Communicator, make_communicator
from .utils import checkpoint as ckpt
from .utils import metrics as M

try:
    from tqdm import trange
except Exception:                                    # pragma: no cover
    trange = None


def resolve_device(cfg: Config, rank: int) -> torch.device:
    if cfg.device == "cpu" or (cfg.device == "auto" and not torch.cuda.is_available()):
        return torch.device("cpu")
    n = torch.cuda.device_count()
    if n == 0:
        raise RuntimeError("--device cuda requested but no GPU is visible")
    local = int(os.environ.get("LOCAL_RANK", rank))
    if local >= n:
        raise RuntimeError(f"rank {rank} needs GPU {local}, only {n} visible (run_job maps partitions beyond the GPU count "
                           "round-robin onto the visible ones; a torchrun world larger than the box is an error)")
    torch.cuda.set_device(local)
    return torch.device("cuda", local)


def resolve_dtype(cfg: Config, device: torch.device) -> torch.dtype:
    if cfg.dtype == "auto":
        return torch.bfloat16 if device.type == "cuda" else torch.float32
    return {"fp32": torch.float32, "float32": torch.float32, "bf16": torch.bfloat16, "bfloat16": torch.bfloat16}[cfg.dtype]


def compute_max_steps(cfg: Config, batch_size: int, per_epoch: int) -> int:
    if cfg.max_steps:
        return cfg.max_steps
    if cfg.steps_mode == "compat":
        return cfg.epochs * (batch_size if batch_size else 1)      # src/rnn.py:256 (sic), Q5
    return cfg.epochs * per_epoch


class ReplicaResult(dict):
    pass


def _check_device_errors(device: torch.device, comm) -> None:
    """Failure surfacing: the persistent LSTM kernels and the fused allreduce bound every in-kernel wait and
    raise a sticky device flag instead of hanging; turn it into a Python error at the sync points we have anyway."""
    if device.type != "cuda":
        return
    from .ops import cuda_lstm
    cuda_lstm.check_kernel_errors(device)
    if hasattr(comm, "check_errors"):
        comm.check_errors()


def score_rows(model, xs: torch.Tensor, ys: torch.Tensor, ls: Optional[torch.Tensor], bs: int) -> Tuple[float, float, int]:
    """Loss and accuracy of the rows ``xs`` / ``ys`` (per-sample lengths ``ls`` or None) with ``model`` in eval mode, in batches of
    ``bs`` rows: the full batches (static shapes for the kernels), then the tail as the last ``bs`` rows, counting only the ones
    not seen yet; --per_step_labels weighs each batch by its number of counted positions.  -> (loss, accuracy, count)."""
    n = xs.shape[0]
    windows = [(lo, 0) for lo in range(0, n - bs + 1, bs)] + ([(n - bs, bs - n % bs)] if n % bs else [])
    loss_sum, correct, count = 0.0, 0, 0
    for lo, first in windows:
        loss, ok, cnt = model.score(xs[lo:lo + bs], ys[lo:lo + bs], None if ls is None else ls[lo:lo + bs], first)
        loss_sum += float(loss) * int(cnt); correct += int(ok); count += int(cnt)
    return loss_sum / count, correct / count, count


def score_stream(model, xs: torch.Tensor, ys: torch.Tensor, B: int, tail: int, dtype: torch.dtype,
                 cache: Optional[F.CacheHistory] = None) -> Tuple[float, ...]:
    """--stateful: loss and accuracy of a stream laid out by ``data.stream_layout(..., tail=True)`` as ``B`` parallel streams,
    with ``model`` in eval mode, the state carried from segment to segment from zero (``tail``: the length of the last, short
    segment in every row, 0 = none).  Uses the model's own state buffers only.  -> (loss, accuracy, positions).

    ``cache``: score with the continuous cache pointer (``SequenceClassifier.score``); the history is reset here, so it holds
    this stream only.  -> (the mixture's loss, accuracy, positions, the model's own loss over the same positions)."""
    device = xs.device
    segs = xs.shape[0] // B
    tail_lengths = torch.full((B,), tail, dtype=torch.int32, device=device) if tail else None
    state = model.rnn.zero_state(B, dtype, device)
    if cache is not None:
        cache.reset()
    loss_sum, model_sum, correct, count = 0.0, 0.0, 0, 0
    for k in range(segs):
        lengths = tail_lengths if (tail and k == segs - 1) else None
        out = model.score(xs[k * B:(k + 1) * B], ys[k * B:(k + 1) * B], lengths, state=state,
                          **({} if cache is None else {"cache": cache}))
        loss, ok, cnt = out[:3]
        state = model.rnn.final_state()
        loss_sum += float(loss) * int(cnt); correct += int(ok); count += int(cnt)
        if cache is not None:
            model_sum += float(out[3]) * int(cnt)
    if cache is not None:
        return loss_sum / count, correct / count, count, model_sum / count
    return loss_sum / count, correct / count, count


def validation_scorer(valid, cfg: Config, batch_size: int, device: torch.device, dtype: torch.dtype):
    """The held-out set ``valid`` (``data.load_validation``) copied to the device once -> ``score(model) -> (loss, accuracy,
    count)`` in batches of ``batch_size`` (``score_rows`` / ``score_stream``), or None without a set."""
    if valid is None:
        return None
    if cfg.stateful:
        x, y, tail = D.stream_layout(valid, batch_size, cfg.seq_len, tail=True)
        xs = torch.as_tensor(x).to(device=device, dtype=D.input_dtype(cfg))
        ys = torch.as_tensor(y).to(device)
        return lambda model: score_stream(model, xs, ys, batch_size, tail, dtype)
    x, y, lengths = valid
    if x.shape[0] < batch_size:
        raise ValueError(f"the validation set has {x.shape[0]} samples, fewer than the batch size {batch_size} it is scored in")
    xs = torch.as_tensor(x).to(device=device, dtype=D.input_dtype(cfg))
    ys = torch.as_tensor(y).to(device)
    ls = None if lengths is None else torch.as_tensor(lengths).to(device=device, dtype=torch.int32)
    return lambda model: score_rows(model, xs, ys, ls, batch_size)


def train_rnn(partition, cfg: Config, rank: int = 0, world_size: int = 1, comm: Optional[Communicator] = None,
              train_optimizer: Optional[Callable] = None, standalone: bool = False,
              run_stamp: Optional[str] = None, defer_average: bool = False, valid=None) -> Optional[ReplicaResult]:
    """Train one replica on one shard.  ``partition`` = ``(key, rows)`` (distributed) or a list of rows
    (standalone) or ``(key, (x ndarray, y ndarray))`` for pre-parsed / synthetic data.  ``valid``: the held-out set
    (``data.load_validation``), scored at every evaluation step, or None."""
    comm = comm or Communicator(0, 1)
    prefix_name = "lstm_no_spark" if standalone else "spark_lstm"
    tag = "RNN-LSTM"

    if partition is None or (isinstance(partition, (list, tuple)) and len(partition) == 0):
        print(f"{tag} - ZERO SIZE")
        return None
    if standalone and not (isinstance(partition, tuple) and len(partition) == 2 and isinstance(partition[0], int)):
        partition_key, rows = 0, partition
    else:
        partition_key, rows = partition
    if not cfg.quiet:
        print(f"LSTM - Partition: {partition_key}")

    device = resolve_device(cfg, rank)
    dtype = resolve_dtype(cfg, device)
    F.set_backend(cfg.backend if cfg.backend != "auto" else "auto")

    if cfg.stateful:
        # one token stream (a piece of it with --partitions) as --batch_size parallel streams, in (segment, stream) order
        stream = rows if isinstance(rows, np.ndarray) else D.token_stream(rows, cfg.vocab_size)
        train_x, train_y, _ = D.stream_layout(stream, cfg.batch_size, cfg.seq_len)
        train_lengths = None
    elif isinstance(rows, tuple):
        train_x, train_y = rows[0], rows[1]
        train_lengths = rows[2] if len(rows) > 2 else None
    else:
        train_x, train_y, train_lengths = D.parse_rows(rows, cfg)
    batch_size = D.resolve_batch_size(cfg.batch_size, train_x.shape[0])

    # ---- model + optimizer + sync = one TrainEngine (the same object bench.py drives) ----------------------
    from .engine import TrainEngine
    eng = TrainEngine(cfg, rank, world_size, comm, batch_size=batch_size, device=device, dtype=dtype,
                      train_optimizer=train_optimizer, partition_key=partition_key)
    model, optimizer = eng.model, eng.optimizer

    # ---- run directory -----------------------------------------------------------------
    current_exec = run_stamp or str(time.time())
    model_save_dir = os.path.join(cfg.checkpoint_path, current_exec) if standalone else \
        os.path.join(cfg.checkpoint_path, current_exec, str(partition_key))
    saver = ckpt.Saver(model_save_dir, prefix_name)
    saver.write_params_settings(cfg.params_str())
    sink = M.SummarySink(os.path.join(model_save_dir, "train"))
    jlog = M.JsonLog(cfg.json_log)

    x_dtype = D.input_dtype(cfg)
    shuffle = not cfg.stateful                 # the stream layout is served in order: batch k continues the streams of batch k-1
    if cfg.data_residency == "host":
        # the reference's feed (src/rnn.py:264-267: every batch travels host -> device), as an asynchronous DMA pipeline
        loader = D.PinnedHostLoader(train_x, train_y, batch_size, device, dtype=x_dtype, shuffle=shuffle,
                                    seed=cfg.seed + 17 * (rank + 1), depth=3, lengths=train_lengths)
    else:
        loader = D.DeviceShard(train_x, train_y, batch_size, device, dtype=x_dtype, shuffle=shuffle,
                               seed=cfg.seed + 17 * (rank + 1), lengths=train_lengths)
    start_step = 0
    if cfg.resume or cfg.use_pretrained_model:
        src = cfg.resume or ckpt.find_latest_run(cfg.checkpoint_path, None if standalone else str(partition_key))
        if src and os.path.isdir(src):
            if not standalone and ckpt.latest_checkpoint(src) is None and os.path.isdir(os.path.join(src, str(partition_key))):
                src = os.path.join(src, str(partition_key))        # --resume <run dir>: every rank picks its own partition
            src = ckpt.latest_checkpoint(src)
        if src:
            variables, meta, opt_state = ckpt.load(src)
            model.check_compatible(variables, ckpt.recorded_settings(meta), f"checkpoint {src}")
            check_stateful(opt_state, meta, cfg, f"checkpoint {src}")
            model.load_reference_state_dict(variables, strict=False)
            eng.flat.refresh_shadow()
            if opt_state is not None:
                comm.load_optimizer_state(optimizer, opt_state["optimizer"])
                eng.set_dropout_step(optimizer.step_count)       # the masks continue where the interrupted run's would have
                if opt_state.get("loader") is not None:
                    st = opt_state["loader"]
                    if bool(st.get("pinned")) == isinstance(loader, D.PinnedHostLoader):
                        loader.load_state_dict(st)                   # continue the data order, do not replay it
                        if cfg.stateful and opt_state.get("state") is not None:
                            eng.load_carried_state(opt_state["state"])   # ... and every stream from where it stopped
                    else:
                        sys.stderr.write(f"{tag} - checkpoint was written with another --data_residency: data order starts over\n")
            start_step = int(meta.get("global_step", -1)) + 1
            if not cfg.quiet:
                print(f"{tag} - restored {src} (resuming at step {start_step})")
        # every rank must resume at the same step (per-step collectives would otherwise mismatch): fail loudly if not
        if world_size > 1:
            hi_s, lo_s = comm.max_scalar(float(start_step)), -comm.max_scalar(-float(start_step))
            if hi_s != lo_s:
                raise RuntimeError(f"{tag} - ranks disagree on the resume step (min {int(lo_s)}, max {int(hi_s)}): "
                                   "a checkpoint is missing or stale on some rank")

    max_steps = compute_max_steps(cfg, batch_size, loader.per_epoch)
    score_valid = validation_scorer(valid, cfg, batch_size, device, dtype)
    averages = optimizer.ax is not None

    use_bar = (trange is not None) and (rank == 0) and not cfg.quiet
    total_steps = trange(start_step, max_steps) if use_bar else range(start_step, max_steps)

    prof = None
    if cfg.trace and rank == 0:
        acts = [torch.profiler.ProfilerActivity.CPU]
        if device.type == "cuda":
            acts.append(torch.profiler.ProfilerActivity.CUDA)
        prof = torch.profiler.profile(activities=acts)
        prof.__enter__()

    fault = None
    if cfg.fault_inject:
        fr, fs = cfg.fault_inject.split(":")
        fault = (int(fr), int(fs))

    bar_loss = M.LaggedScalar(device)
    timer = M.DeviceTimer(device)
    start = time.time()
    timer.start()
    t_acc, t_loss = 0.0, 0.0
    samples = 0
    for step in total_steps:
        if fault is not None and fault == (rank, step):
            sys.stderr.write(f"{tag} - fault injected on rank {rank} at step {step}\n")
            sys.stderr.flush()
            os._exit(17)
        # with a captured step the batch is gathered straight into the graph's input buffers (no second copy)
        gi = eng.graph_inputs() if isinstance(loader, D.DeviceShard) else None
        batch = loader.next(out=gi) if gi is not None else loader.next()
        train_input, train_labels = batch[0], batch[1]
        batch_lengths = batch[2] if len(batch) > 2 else None      # variable-length samples: int32 [B]

        with M.nvtx_range("step", cfg.nvtx):
            if cfg.cuda_graph and device.type == "cuda" and eng._graph is None and step == start_step + 3:
                # static shapes: replay the captured step from here on (host feed: one graph per staging slot, no extra copy)
                eng.capture(train_input, train_labels, bind=list(loader.dev) if isinstance(loader, D.PinnedHostLoader) else (),
                            lengths=batch_lengths)
            loss = eng.step(train_input, train_labels, batch_lengths, reset=cfg.stateful and loader.opened_pass())
        samples += batch_size

        with M.nvtx_range("param_avg", cfg.nvtx):
            eng.maybe_average()

        is_eval = (step % cfg.evaluate_every == 0) or (step + 1) == max_steps
        if is_eval:
            t_loss = float(loss.detach().float().item())
            g_norm = float(eng.grad_norm().item()) if cfg.clip_grad_norm > 0 else None
            ar_tar = eng.activation_penalties()
            ar_tar = None if ar_tar is None else [float(v) for v in ar_tar.tolist()]
        elif use_bar:
            t_loss = bar_loss.push(loss)         # CUDA: the previous step's loss, read back asynchronously (no host sync)
        if use_bar:
            total_steps.set_description("Loss: {:.4f} - t_acc {:.3f}".format(t_loss, t_acc))

        if is_eval:
            _check_device_errors(device, comm)       # sticky in-kernel timeout flags (dead peer / stalled grid barrier)
            val = None
            if score_valid is not None:
                with M.nvtx_range("validate", cfg.nvtx), torch.no_grad(), eng.averaged_weights():
                    model.eval()                                     # no dropout, raw W_h; the average once there is one
                    try:
                        val = score_valid(model)
                    finally:
                        model.train()
                if cfg.optimizer == "ntasgd":
                    fire = nonmono_trigger(optimizer.nonmono_history, val[0], cfg.nonmono, optimizer.averaging)
                    if world_size > 1:                               # every replica switches at the same step
                        fire = comm.max_scalar(1.0 if fire else 0.0) > 0
                    optimizer.nonmono_history.append(val[0])
                    if fire:
                        optimizer.start_averaging()
                        if rank == 0 and not cfg.quiet:
                            print(f"{tag} - NT-ASGD: validation loss {val[0]:.6f} did not improve on the best before the last "
                                  f"{cfg.nonmono} validations: averaging the weights from step {step + 1} on")
            with M.nvtx_range("eval_ckpt", cfg.nvtx):
                saver.save(model.reference_state_dict(), global_step=step,
                           extra={"rank": rank, "world_size": world_size, "partition_key": partition_key,
                                  "loss": t_loss, "config": cfg.__dict__},
                           opt_state={"optimizer": comm.optimizer_state(optimizer), "loader": loader.state_dict(),
                                      "stateful": cfg.stateful, "batch_size": batch_size,
                                      "state": None if not cfg.stateful else
                                      [(h.detach().cpu().clone(), c.detach().cpu().clone()) for h, c in eng.carried_state()]})
                model.eval()                                         # no dropout while scoring
                with torch.no_grad(), M.capture(sink):
                    # same batch, from the initial state (src/rnn.py:276-279); --stateful: from the state it was trained from
                    xent, ok, n = model.score(train_input, train_labels, batch_lengths, state=eng.state_prev)
                    e_loss = report_loss(xent)
                    e_acc = report_accuracy(ok.float() / n.float())
                model.train()
                t_loss, t_acc = float(e_loss.item()), float(e_acc.item())
                extra = {}
                if g_norm is not None:                               # the pre-clip norm of this step's gradient
                    sink.add("grad_norm", g_norm)
                    extra["grad_norm"] = g_norm
                if ar_tar is not None:                               # this step's unweighted AR and TAR
                    for k, v in zip(("ar", "tar"), ar_tar):
                        sink.add(k, v)
                        extra[k] = v
                if cfg.next_token:
                    extra["perplexity"] = math.exp(t_loss)
                    sink.add("perplexity", extra["perplexity"])
                if val is not None:                                  # the held-out set, scored before this checkpoint
                    extra.update(val_loss=val[0], val_accuracy=val[1])
                    if cfg.next_token:
                        extra["val_perplexity"] = math.exp(val[0]) if val[0] < 700 else float("inf")
                if averages:
                    extra.update(averaging=int(optimizer.averaging), averaged_steps=optimizer.averaged_steps)
                for k in ("val_loss", "val_accuracy", "val_perplexity", "averaging", "averaged_steps"):
                    if k in extra:
                        sink.add(k, extra[k])
                sink.flush(step)
                jlog.write(step=step, loss=t_loss, acc=t_acc, rank=rank, **extra)
            if use_bar:
                ppl = " - ppl {:.2f}".format(extra["perplexity"]) if cfg.next_token else ""
                total_steps.set_description("Loss: {:.4f} - t_acc {:.3f}".format(t_loss, t_acc) + ppl)

    # ---- the cross-replica average (src/rnn.py:393-407) ------------------------------------------------
    with M.nvtx_range("final_param_avg", cfg.nvtx):
        averaged = eng.finish_averaging()       # asgd / ntasgd: the average is the model that is averaged and exported
        if not defer_average:                   # oversubscribed ranks average all their replicas at once (_rank_main)
            eng.maybe_average(force=True)
    device_ms = timer.stop_ms()
    end_time = time.time() - start
    n_steps = max(1, max_steps - start_step)
    if not cfg.quiet:
        print("{} - Partition: {} - Time: {}s".format(tag, partition_key, end_time))
    if prof is not None:
        prof.__exit__(None, None, None)
        prof.export_chrome_trace(cfg.trace)

    records = [(k, [[t.detach().float().cpu().clone() for t in layer] if isinstance(layer, list)
                    else layer.detach().float().cpu().clone() for layer in v])
               for k, v in model.rnn.map_data_by_key()]
    result = ReplicaResult(partition_key=partition_key, rank=rank, records=records, averaged=averaged,
                           variables=model.reference_state_dict(), loss=t_loss, acc=t_acc, steps=n_steps,
                           seconds=end_time, device_ms=device_ms, samples=samples, model_save_dir=model_save_dir)
    if defer_average:
        lo, hi = eng.flat.segment(cfg.average_scope)
        result["flat_scope"] = eng.flat.data[lo:hi].detach().float().cpu().clone()
        result["batch_size"] = batch_size
    jlog.write(event="done", rank=rank, seconds=end_time, device_ms=device_ms, samples_per_s=samples / max(end_time, 1e-9))
    sink.close()
    jlog.close()
    return result


# ====================================================================================================
# job driver
# ====================================================================================================
def _rank_main(rank: int, world_size: int, cfg: Config, shards, standalone: bool, valid=None):
    device = resolve_device(cfg, rank)
    comm = make_communicator(cfg.comm, rank, world_size, device, cfg.timeout_s, clip_synced_grads=cfg.clips_synced_grads())
    try:
        stamp = comm.broadcast_object(str(time.time()), src=0)
        mine = list(shards[rank::world_size]) if shards is not None else [None]
        if len(shards or []) <= world_size:
            shard = shards[rank] if shards is not None else None
            res = train_rnn(shard, cfg, rank, world_size, comm, standalone=standalone, run_stamp=stamp, valid=valid)
        else:
            res = _train_oversubscribed(mine, len(shards), cfg, rank, world_size, comm, stamp, valid)
        comm.barrier()
        if res is not None and rank != 0:
            # only rank 0's records are needed by the driver (all replicas hold the same average)
            res = ReplicaResult({k: v for k, v in res.items() if k not in ("records", "variables")})
        return res
    finally:
        comm.close()


def _train_oversubscribed(mine, n_partitions: int, cfg: Config, rank: int, world_size: int, comm, stamp: str, valid=None):
    """More partitions than workers (the reference runs ``--partitions`` tasks on ``local[workers]`` executor threads,
    original src/rnn.py:355-358: each worker takes its tasks in turn).  Every partition is still its own replica
    with its own checkpoint directory; a rank trains its partitions one after the other and the one-shot average at the
    end of the job (src/rnn.py:393-407) runs over ALL partitions: local sum -> cross-rank sum -> / partitions."""
    results = []
    for shard in mine:
        results.append(train_rnn(shard, cfg, rank, 1, None, standalone=False, run_stamp=stamp, defer_average=True, valid=valid))
    results = [r for r in results if r is not None]
    if not results:
        return None
    total = torch.zeros_like(results[0]["flat_scope"])
    for r in results:
        total += r["flat_scope"]
    count = torch.tensor([float(len(results))], dtype=torch.float64)
    if world_size > 1:
        comm.allreduce_sum_(total)
        comm.allreduce_sum_(count)
    mean = total / float(count.item())
    # rebuild the exported records from the averaged flat segment (everything outside the scope: this rank's first replica)
    r0 = results[0]
    model = SequenceClassifier(cfg, batch_size=r0["batch_size"], device="cpu")
    model.load_reference_state_dict(r0["variables"], strict=False)
    flat = model.build_flat()
    lo, hi = flat.segment(cfg.average_scope)
    with torch.no_grad():
        flat.data[lo:hi].copy_(mean)
    records = [(k, [[t.detach().float().cpu().clone() for t in layer] if isinstance(layer, list)
                    else layer.detach().float().cpu().clone() for layer in v]) for k, v in model.rnn.map_data_by_key()]
    out = ReplicaResult({k: v for k, v in r0.items() if k not in ("flat_scope",)})
    out.update(records=records, variables=model.reference_state_dict(), partitions_trained=[r["partition_key"] for r in results],
               seconds=sum(r["seconds"] for r in results), samples=sum(r["samples"] for r in results))
    return out


def resolve_workers(cfg: Config, standalone: bool) -> int:
    """Concurrent ranks for ``--partitions`` replicas: one per GPU while GPUs last (Q14), round-robin beyond that."""
    if standalone:
        return 1
    cap = cfg.max_workers
    if cap <= 0:
        on_gpu = cfg.device == "cuda" or (cfg.device == "auto" and torch.cuda.is_available())
        cap = max(1, torch.cuda.device_count()) if on_gpu else cfg.partitions
    return max(1, min(cfg.partitions, cap))


def check_stateful(opt_state: Optional[dict], meta: dict, cfg: Config, what: str) -> None:
    """Resuming training: raise unless the checkpoint was written with this run's ``--stateful`` (recorded in its optimizer-state
    file, else in its flags; nothing recorded counts as off).  The variables are the same either way, but the data order and
    the carried state are not."""
    saved = bool(opt_state.get("stateful")) if opt_state is not None and "stateful" in opt_state else \
        bool(ckpt.recorded_settings(meta).get("stateful"))
    if saved != bool(cfg.stateful):
        raise ValueError(f"{what} was written {'with' if saved else 'without'} --stateful, this run is "
                         f"{'with' if cfg.stateful else 'without'} it: {'add' if saved else 'drop'} --stateful to resume it "
                         "(--mode eval scores it either way)")


def load_shards(cfg: Config, world_size: int, standalone: bool):
    if cfg.stateful:
        # one stream; --partitions: contiguous pieces of it, consecutive pieces sharing one id
        stream = D.load_stream(cfg)
        return [(0, stream)] if standalone else list(enumerate(D.split_stream(stream, world_size)))
    if cfg.synthetic:
        return [(r, D.synthetic(cfg, cfg.synthetic // world_size, cfg.seed + r)) for r in range(world_size)]
    if standalone:
        return [(0, D.read_dataset_from_path(cfg.training_path))]
    return D.text_to_partitions(cfg.training_path, world_size, shuffle=True, seed=cfg.seed, remainder=cfg.remainder)


def _averaged_variables(cfg: Config, variables, ax: torch.Tensor, batch_size: int):
    """The variables (reference names) of the model whose flat buffer is ``ax``: ``variables`` laid out as training laid them
    out (at its ``batch_size``), with every value taken from ``ax``."""
    model = SequenceClassifier(cfg, batch_size=batch_size, device="cpu")
    model.load_reference_state_dict(variables, strict=False)
    flat = model.build_flat()
    if flat.data.numel() != ax.numel():
        raise ValueError(f"the checkpoint's weight average holds {ax.numel()} values, the model it belongs to {flat.data.numel()}: "
                         "give the flags it was trained with")
    with torch.no_grad():
        flat.data.copy_(ax)
    return model.reference_state_dict()


def _find_trained_model(cfg: Config, standalone: bool):
    """--resume <file | dir>, else <output_path>/averaged_model.pt (distributed job), else the latest checkpoint under
    --checkpoint_path.  -> (variables in the reference's names, description, the flags the file records
    (``utils.checkpoint.recorded_settings``), "averaged" | "raw").  A training checkpoint whose optimizer state holds a weight
    average (--optimizer asgd / ntasgd, averaging on, k >= 1) gives the average's variables, as training evaluates it."""
    src = cfg.resume
    if not src and not standalone and cfg.output_path and os.path.isfile(os.path.join(cfg.output_path, "averaged_model.pt")):
        src = os.path.join(cfg.output_path, "averaged_model.pt")
    if not src:
        src = ckpt.find_latest_run(cfg.checkpoint_path, None if standalone else "0")
    if src and os.path.isdir(src) and os.path.isfile(os.path.join(src, "averaged_model.pt")):
        src = os.path.join(src, "averaged_model.pt")
    if src and os.path.isfile(src) and src.endswith(".pt"):
        blob = torch.load(src, map_location="cpu", weights_only=False)
        meta = blob.get("meta") or {}
        return blob["variables"], src, ckpt.recorded_settings(meta), meta.get("weights", "raw")
    if src and os.path.isdir(src):
        if ckpt.latest_checkpoint(src) is None and os.path.isdir(os.path.join(src, "0")):
            src = os.path.join(src, "0")
        last = ckpt.latest_checkpoint(src)
        if last:
            variables, meta, opt_state = ckpt.load(last)
            sd = (opt_state or {}).get("optimizer") or {}
            if sd.get("ax") is not None and int(sd.get("on", 0)) and int(sd.get("k", 0)) >= 1:
                variables = _averaged_variables(cfg, variables, sd["ax"], int(opt_state.get("batch_size") or cfg.batch_size))
                return variables, last, ckpt.recorded_settings(meta), "averaged"
            return variables, last, ckpt.recorded_settings(meta), "raw"
    raise FileNotFoundError(f"--mode {cfg.mode}: no trained model found (give --resume <averaged_model.pt | checkpoint dir>)")


def _load_trained_model(cfg: Config, found, batch_size: int, device: torch.device, dtype: torch.dtype):
    """A TrainEngine in eval mode holding the model ``_find_trained_model`` found (``found``), after the compatibility checks
    (``SequenceClassifier.check_compatible``).  The reference's trainable initial state is one row PER BATCH ROW
    ([batch_size, H], src/models/recurrent/lstm.py:24-33): at another batch size every row starts from the mean learned row."""
    from .engine import TrainEngine
    variables, src, settings, _weights = found
    eng = TrainEngine(cfg, 0, 1, Communicator(0, 1), batch_size=batch_size, device=device, dtype=dtype)
    eng.model.eval()                                    # no dropout
    shapes = {k: tuple(v.shape) for k, v in eng.model.named_reference_variables()}
    variables = dict(variables)
    eng.model.check_compatible(variables, settings, f"model {src}")   # before the row averaging below, which must never touch the table
    for k, v in list(variables.items()):
        want = shapes.get(k)
        if k != "Embedding/weights" and want is not None and tuple(v.shape) != want and v.dim() == 2 and len(want) == 2 and v.shape[1] == want[1]:
            variables[k] = v.float().mean(0, keepdim=True).expand(want).contiguous()
    eng.model.load_reference_state_dict(variables, strict=False)
    eng.flat.refresh_shadow()
    return eng


def evaluate_job(cfg: Config, standalone: bool = False) -> Dict:
    """``--mode eval``: score a trained model on ``--training_path`` (or ``--synthetic``) - loss and accuracy over the whole
    file in batches of ``--batch_size``, forward kernels only, one device.  Not in the reference (its ``--mode`` flag knows
    only ``train`` and the averaged model is thrown away, src/rnn.py:371,407-408); it closes the train -> average -> use loop."""
    found = _find_trained_model(cfg, standalone)
    src = found[1]
    if cfg.stateful:
        return _evaluate_stream(cfg, found)
    x, y, lengths = D.synthetic(cfg, cfg.synthetic, cfg.seed) if cfg.synthetic else \
        D.parse_rows(D.read_dataset_from_path(cfg.training_path), cfg)
    device = resolve_device(cfg, 0)
    dtype = resolve_dtype(cfg, device)
    F.set_backend(cfg.backend if cfg.backend != "auto" else "auto")
    n = x.shape[0]
    bs = D.resolve_batch_size(cfg.batch_size if cfg.batch_size and cfg.batch_size <= n else 0, n)
    eng = _load_trained_model(cfg, found, bs, device, dtype)
    xs = torch.as_tensor(x).to(device=device, dtype=D.input_dtype(cfg))
    ys = torch.as_tensor(y).to(device)
    ls = None if lengths is None else torch.as_tensor(lengths).to(device=device, dtype=torch.int32)
    start = time.time()
    loss, accuracy, count = score_rows(eng.model, xs, ys, ls, bs)
    out = {"mode": "eval", "model": src, "samples": n}
    if eng.model.per_step:
        out["positions"] = count
    out.update(loss=loss, accuracy=accuracy, seconds=time.time() - start, weights=found[3])
    if cfg.next_token:
        out["perplexity"] = math.exp(out["loss"])
    if not cfg.quiet:
        positions = "{positions} positions, " if eng.model.per_step else ""
        print(("RNN-LSTM - eval: model {model}, {samples} samples, " + positions +
               "loss {loss:.6f}, accuracy {accuracy:.4f}" + (", perplexity {perplexity:.4f}" if cfg.next_token else "")).format(**out))
    if cfg.json_log:
        jl = M.JsonLog(cfg.json_log); jl.write(**out); jl.close()
    return out


def _evaluate_stream(cfg: Config, found) -> Dict:
    """``--mode eval --stateful``: the perplexity of the whole stream (``--training_path`` or ``--synthetic``) cut into
    ``--batch_size`` streams (``data.stream_layout``), the state carried from segment to segment from zero.  The positions left
    after the last full segment run as one more segment with that length in every row, so every position is scored."""
    src = found[1]
    stream = D.load_stream(cfg)
    B, T = cfg.batch_size, cfg.seq_len
    x, y, tail = D.stream_layout(stream, B, T, tail=True)
    device = resolve_device(cfg, 0)
    dtype = resolve_dtype(cfg, device)
    F.set_backend(cfg.backend if cfg.backend != "auto" else "auto")
    eng = _load_trained_model(cfg, found, B, device, dtype)
    model = eng.model
    xs = torch.as_tensor(x).to(device=device, dtype=D.input_dtype(cfg))
    ys = torch.as_tensor(y).to(device)
    cache = None
    if cfg.cache_window > 0:
        H = cfg.hidden_list()[-1] * (2 if cfg.bidirectional else 1)
        cache = F.CacheHistory(cfg.cache_window, cfg.cache_theta, cfg.cache_lambda, B, T, H, eng.dtype, device)
    start = time.time()
    scored = score_stream(model, xs, ys, B, tail, eng.dtype, cache=cache)
    loss, accuracy, count = scored[:3]
    out = {"mode": "eval", "model": src, "stream": int(len(stream)), "streams": B, "positions": count,
           "loss": loss, "accuracy": accuracy, "seconds": time.time() - start, "weights": found[3]}
    out["perplexity"] = math.exp(out["loss"])
    line = ("RNN-LSTM - eval: model {model}, a stream of {stream} ids in {streams} streams, {positions} positions, "
            "loss {loss:.6f}, accuracy {accuracy:.4f}, perplexity {perplexity:.4f}")
    if cache is not None:
        out.update(loss_model=scored[3], perplexity_model=math.exp(scored[3]), cache_window=cfg.cache_window,
                   cache_theta=cfg.cache_theta, cache_lambda=cfg.cache_lambda)
        line += (" with the cache pointer (window {cache_window}, theta {cache_theta:g}, lambda {cache_lambda:g}); the model "
                 "alone: loss {loss_model:.6f}, perplexity {perplexity_model:.4f}")
    if not cfg.quiet:
        print(line.format(**out))
    if cfg.json_log:
        jl = M.JsonLog(cfg.json_log); jl.write(**out); jl.close()
    return out


def generate_job(cfg: Config, standalone: bool = False) -> Dict:
    """``--mode generate``: continue prompts with a trained ``--next_token`` model, found as ``--mode eval`` finds it, on one
    device in batches of ``--batch_size`` (a short last batch is filled with copies of its first prompt, whose output is dropped,
    so every batch has the shape the decode graph was captured at).  Prompts are the rows of ``--training_path`` (1..seq_len ids
    each) or, with ``--synthetic n``, the starts of n walks of the synthetic chain; ``--max_new_tokens`` ids are drawn per prompt
    at ``--temperature`` (filtered by ``--top_k`` / ``--top_p``) with noise seeded by ``--seed``; prompt i draws the noise of counter row i, so a prompt's continuation
    does not depend on ``--batch_size`` and a prompt repeated k times gives k independent samples.  Writes ``<output_path>/generated.csv`` (one line of ids per prompt, in
    prompt order) and reports tokens/s, the mean log-probability per token and, with ``--synthetic``, the share of generated
    transitions the chain allows."""
    found = _find_trained_model(cfg, standalone)
    src = found[1]
    if cfg.synthetic:
        prompts, lengths = D.synthetic_prompts(cfg.synthetic, cfg.seq_len, cfg.vocab_size, cfg.seed)
    else:
        prompts, lengths = D.process_prompts(D.read_dataset_from_path(cfg.training_path), cfg.seq_len, cfg.vocab_size)
    device = resolve_device(cfg, 0)
    dtype = resolve_dtype(cfg, device)
    F.set_backend(cfg.backend if cfg.backend != "auto" else "auto")
    n, N = prompts.shape[0], cfg.max_new_tokens
    bs = min(cfg.batch_size, n) if cfg.batch_size else n
    eng = _load_trained_model(cfg, found, bs, device, dtype)
    outs, lps = [], []
    start = time.time()
    for lo in range(0, n, bs):
        rows = min(bs, n - lo)
        idx = np.concatenate([np.arange(lo, lo + rows), np.full(bs - rows, lo)])     # the short tail: masked copies of row lo
        width = int(lengths[idx].max())
        x = torch.as_tensor(prompts[idx, :width]).to(device=device, dtype=torch.int32)
        ls = torch.as_tensor(lengths[idx]).to(device=device, dtype=torch.int32)
        tok, lp = eng.model.generate(x, ls, N, cfg.temperature, cfg.seed, row0=lo,        # prompt lo + b: its own noise
                                     top_k=cfg.top_k, top_p=cfg.top_p)
        outs.append(tok[:rows])
        lps.append(lp[:rows])
    tokens = torch.cat(outs).cpu().numpy()                 # the one wait for the device
    logprob = torch.cat(lps).double().cpu().numpy()
    seconds = time.time() - start
    _check_device_errors(device, None)
    os.makedirs(cfg.output_path or ".", exist_ok=True)
    path = os.path.join(cfg.output_path or ".", "generated.csv")
    with open(path, "w") as f:
        f.writelines(",".join(str(int(v)) for v in row) + "\n" for row in tokens)
    out = {"mode": "generate", "model": src, "weights": found[3], "prompts": n, "tokens": int(tokens.size), "seconds": seconds,
           "tokens_per_s": tokens.size / max(seconds, 1e-9), "mean_logprob": float(logprob.mean()), "temperature": cfg.temperature,
           "top_k": cfg.top_k, "top_p": cfg.top_p, "output": path}
    if cfg.synthetic:
        out["legal_fraction"] = D.legal_fraction(prompts, lengths, tokens, D.next_token_chain(cfg.vocab_size, cfg.seed))
    if not cfg.quiet:
        print(("RNN-LSTM - generate: model {model}, {prompts} prompts, {tokens} tokens in {seconds:.3f}s ({tokens_per_s:.1f} "
               "tokens/s) at temperature {temperature:g}, top_k {top_k}, top_p {top_p:g}, mean log-probability {mean_logprob:.4f} "
               "per token" +
               (", legal_fraction {legal_fraction:.4f}" if cfg.synthetic else "") + ", wrote {output}").format(**out))
    if cfg.json_log:
        jl = M.JsonLog(cfg.json_log); jl.write(**out); jl.close()
    return out


def run_job(cfg: Config, standalone: bool = False) -> Dict:
    """``main`` of both entry points: shard -> N replicas -> average -> output."""
    if cfg.mode == "eval":
        return evaluate_job(cfg, standalone)
    if cfg.mode == "generate":
        return generate_job(cfg, standalone)
    from .parallel.launch import launch, in_torchrun
    world_size = resolve_workers(cfg, standalone)
    if in_torchrun():
        world_size = int(os.environ["WORLD_SIZE"])
    n_shards = 1 if standalone else max(cfg.partitions, world_size)
    if n_shards > world_size:
        if cfg.sync_mode == "grad_allreduce" or (cfg.sync_mode == "param_avg" and cfg.sync_every):
            raise ValueError(f"--partitions {cfg.partitions} > {world_size} workers needs the one-shot parameter average "
                             "(--sync_mode param_avg --sync_every 0): replicas that take turns cannot sync every step")
        if cfg.optimizer == "ntasgd":
            raise ValueError(f"--optimizer ntasgd with --partitions {cfg.partitions} > {world_size} workers: replicas that take "
                             "turns cannot decide together when averaging starts (use --optimizer asgd, or one worker per partition)")
        sys.stderr.write(f"RNN-LSTM - warning: {n_shards} partitions on {world_size} workers: each worker trains its "
                         "partitions in turn (round-robin), the final average runs over all partitions\n")
    if not cfg.quiet:
        print("Total workers: ", f"[{world_size}]")
    shards = load_shards(cfg, n_shards, standalone)
    # the held-out set: every rank scores the same one (--valid_synthetic: of the first shard's task)
    valid = D.load_validation(cfg, cfg.synthetic // n_shards if cfg.synthetic else 0)
    start = time.time()
    results = launch(_rank_main, world_size, args=(cfg, shards, standalone, valid))
    total = time.time() - start
    res0 = next((r for r in results if r is not None and "records" in r), None)
    if res0 is not None and cfg.output_path:
        ckpt.save_averaged_model(cfg.output_path, res0["records"], res0["variables"],
                                 {"world_size": world_size, "sync_mode": cfg.sync_mode, "average_scope": cfg.average_scope,
                                  "hidden_units": cfg.hidden_units, "pooling": cfg.pooling,
                                  "attention_units": cfg.attention_units, "vocab_size": cfg.vocab_size,
                                  "next_token": cfg.next_token, "stateful": cfg.stateful,
                                  "tie_embeddings": cfg.tie_embeddings, "seconds": total,
                                  "weights": "averaged" if cfg.optimizer in ("asgd", "ntasgd") and res0.get("averaged") else "raw"})
    if not cfg.quiet:
        print("RNN-LSTM - Total Processing Time {}s".format(total))
    return {"results": results, "seconds": total, "world_size": world_size, "partitions": n_shards}
