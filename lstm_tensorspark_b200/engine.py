"""TrainEngine: the public "one training step" API (model + flat buffers + optimizer + cross-replica sync).

This is what ``bench.py``, ``__graft_entry__.smoke`` and the per-replica trainer call:

    eng = TrainEngine(cfg, rank, world_size, comm, batch_size=B)
    loss = eng.step(x, y)            # forward, backward, (fused allreduce +) optimizer update
    loss = eng.step(x, y, lengths)   # variable-length batch: int32 [B] per-sample lengths, x right-padded
    norm = eng.grad_norm()           # --clip_grad_norm: the last step's gradient norm before clipping (None without)
    ar_tar = eng.activation_penalties()  # --activation_reg / --temporal_activation_reg: the last step's (AR, TAR) (None without)
    loss = eng.step(x, y, reset=k == 0)  # --stateful: batch k of a pass continues every stream from the state batch k-1 ended in
    with eng.averaged_weights(): ...     # --optimizer asgd / ntasgd: score the average of the iterates, then train on
    eng.finish_averaging()               # end of training: the average becomes the weights, before the replica average / export

One step replaces the reference's ``sess.run([train_op, loss], feed_dict=...)`` (original src/rnn.py:264-267):
H2D feed, forward, backward, 14·L+2 ApplyAdam launches, D2H loss.  With ``cuda_graph=True`` the whole step is
captured once and replayed (launch-bound inner loops belong in CUDA graphs, not in a tracing compiler).
"""
from __future__ import annotations

import contextlib
from typing import Optional

import torch

from .config import FUSED_CLIP_ERROR, Config
from .models.classifier import SequenceClassifier
from .models.recurrent.lstm import clear_weight_decay_collection, weight_decay_collection
from .ops import functional as F
from .ops import params
from .ops.optim import FlatOptimizer
from .parallel.comm import Communicator


import os as _os

_BUCKET_PDL = _os.environ.get("LSTM_TS_BUCKET_PDL", "1") == "1"      # 0: buckets in plain stream order (no overlap) - for A/B timing


class TrainEngine:
    def __init__(self, cfg: Config, rank: int = 0, world_size: int = 1, comm: Optional[Communicator] = None,
                 batch_size: Optional[int] = None, device: Optional[torch.device] = None,
                 dtype: Optional[torch.dtype] = None, train_optimizer=None, partition_key: Optional[int] = None):
        self.cfg = cfg
        self.rank, self.world_size = rank, world_size
        self.comm = comm or Communicator(0, 1)
        if device is None:
            device = torch.device("cuda", torch.cuda.current_device()) if (cfg.device != "cpu" and torch.cuda.is_available()) \
                else torch.device("cpu")
        self.device = device
        if dtype is None:
            dtype = torch.bfloat16 if (device.type == "cuda" and cfg.dtype in ("auto", "bf16", "bfloat16")) else torch.float32
        self.dtype = dtype
        F.set_backend(cfg.backend)
        if cfg.deterministic and device.type == "cuda":
            from .ops import cuda_lstm
            cuda_lstm.SEQ_VARIANT = (cuda_lstm.SEQ_VARIANT & ~(7 << 12)) | (3 << 12)     # in-order operand stream
        clear_weight_decay_collection()
        seed = cfg.seed + (1000003 * (rank + 1) if cfg.independent_init else 0)
        gen = torch.Generator(device="cpu")
        gen.manual_seed(seed)
        self.model = SequenceClassifier(cfg, batch_size=batch_size, device="cpu", generator=gen)
        self.model.to(device)
        self.flat = self.model.build_flat()
        self.comm.adopt(self.flat)
        self.model.set_compute_dtype(dtype)
        if train_optimizer is not None:
            self.optimizer = train_optimizer(cfg.learning_rate)(self.flat)
        else:
            self.optimizer = FlatOptimizer(self.flat, cfg.learning_rate, cfg.optimizer, weight_decay=0.0)
        # K12: the optional L2 term of create_variable (original src/models/recurrent/lstm.py:9-11) is folded into the
        # update kernel (g + wd * w over the LSTM weight / bias segment) instead of an autograd term over 67 MB of weights;
        # variables outside that segment that asked for decay (learned initial states) keep the autograd term
        self.optimizer.weight_decay = float(cfg.weight_decay or 0.0)
        self.optimizer.wd_numel = self.flat.lstm_numel
        seg_ids = {id(p) for p in self.model.rnn.averaged_parameters()}
        self._wd_in_kernel = [(v, fn, wd) for (v, fn, wd) in weight_decay_collection() if id(v) in seg_ids]
        self._wd_autograd = [(v, fn, wd) for (v, fn, wd) in weight_decay_collection() if id(v) not in seg_ids]
        self.sync_grads = cfg.sync_mode == "grad_allreduce" and world_size > 1
        self.optimizer.clip_norm = float(cfg.clip_grad_norm or 0.0)
        if self.optimizer.clip_norm > 0 and self.sync_grads and getattr(self.comm, "name", "") == "fused":
            raise ValueError(FUSED_CLIP_ERROR)
        self._bucket_plan = self._make_bucket_plan() if (self.sync_grads and hasattr(self.comm, "launch_bucket")
                                                         and cfg.grad_buckets) else None
        self._graph = None
        self._static = None
        self._bound = {}                        # (x ptr, y ptr, lengths ptr, shape) -> (graph captured on those buffers, its loss)
        self._bound_keepalive = []
        self.steps_done = 0
        self._averaging_finished = False
        # every dropout (between layers, output, input, embedding rows, weight drop): the masks are keyed on (seed, partition)
        # and on the number of training steps this engine has completed - a counter of its own, device-resident on the GPU (a
        # captured graph advances it; the optimizer's step_dev is bumped before backward by the fused allreduce and never by
        # SGD), a host int on the CPU
        rnn = self.model.rnn
        self._dropout_on = rnn.draws_masks
        rnn.dropout_key = (cfg.seed & 0xFFFFFFFF, rank if partition_key is None else int(partition_key))
        rnn.dropout_step = torch.zeros(1, dtype=torch.int32, device=device) if device.type == "cuda" else 0
        # --stateful: static buffers per layer (h in the compute dtype, as the kernels store it; c fp32).  `state` is what the next
        # step starts from, `state_prev` what the last step started from; a captured graph reads and writes these same buffers
        self.stateful = bool(getattr(cfg, "stateful", False))
        self.state = self.state_prev = None
        if self.stateful:
            bs = cfg.batch_size if batch_size is None else batch_size
            self.state = rnn.zero_state(bs, dtype, device)
            self.state_prev = rnn.zero_state(bs, dtype, device)
        # --activation_reg / --temporal_activation_reg: the coefficients, and a static [2] buffer of the last step's (AR, TAR)
        self.act_reg = (float(getattr(cfg, "activation_reg", 0.0)), float(getattr(cfg, "temporal_activation_reg", 0.0)))
        self._act_pen = torch.zeros(2, dtype=torch.float32, device=device) if any(self.act_reg) else None

    # ---------------------------------------------------------------------------------------------------
    def _make_bucket_plan(self):
        """Gradient buckets in the order backward finishes them: [top layer (+ head)], ..., [layer 0].  A bucket = a
        contiguous element range of the flat buffer + the parameters that must have been released before it may be synced.
        (Reference counterpart: the one-shot reduceByKey over all weights, original src/rnn.py:393-407 - here the sync
        of the upper layers hides under the backward recurrence of the layers below.)  Bidirectional: every direction of a layer
        is a layer here (flat order: forward, reverse per depth; backward finishes the reverse direction first)."""
        flat = self.flat
        if not flat._direct:
            return None
        off = {id(p): o for p, o in zip(flat.params, flat.offsets)}
        layers = self.model.rnn.directions()
        others = [p for p in flat.params[len(self.model.rnn.averaged_parameters()):]]
        others_direct = all(p.data_ptr() in flat._direct for p in others)
        # --vocab_size: the table's gradient is the last one backward writes (after layer 0's), and it is the last parameter of
        # the flat buffer - a bucket of its own, so the top layer's bucket does not wait for the whole backward pass
        table = None if self.model.embedding is None else self.model.embedding.weights
        top_others = [p for p in others if p is not table]
        end = [off[id(l.w_x)] for l in layers[1:]] + [flat.lstm_numel]        # end of each layer's segment
        plan = []
        for li in reversed(range(len(layers))):
            l = layers[li]
            # [w_h, bias] is released with the layer's bias gradient, [w_x] already with its weight-gradient GEMM (or with the dX
            # GEMM when there is one): two buckets per layer, each launched under the GEMM / recurrence kernel that follows it
            lo_x, lo_h, hi = off[id(l.w_x)], off[id(l.w_h)], end[li]
            need_h = [l.w_h, l.bias]
            if li == len(layers) - 1 and others_direct:
                # head weights / bias (and the attention weights) follow the last layer in the flat buffer
                hi = flat.padded_numel if table is None else off[id(table)]
                need_h = need_h + top_others
            plan.append({"lo": lo_x, "hi": lo_h, "need": {l.w_x.data_ptr()}})
            plan.append({"lo": lo_h, "hi": hi, "need": {p.data_ptr() for p in need_h}})
        if table is not None and others_direct:
            plan.append({"lo": off[id(table)], "hi": flat.padded_numel, "need": {table.data_ptr()}})
        if not others_direct:
            plan.append({"lo": flat.lstm_numel, "hi": flat.padded_numel, "need": None})    # autograd-accumulated: only final at the end
        return plan

    def _backward_with_buckets(self, loss: torch.Tensor):
        flat, comm, plan = self.flat, self.comm, self._bucket_plan
        comm.begin_grad_step(flat, self.optimizer)
        state = {"next": 0}

        def ready(released):
            # queue every leading bucket whose parameters have all been released; it is launched (PDL) right after the next big
            # backward kernel (weight-gradient GEMM / lower layer's recurrence), i.e. it runs next to that kernel
            while state["next"] < len(plan) - 1:
                b = plan[state["next"]]
                if b["need"] is None or not b["need"] <= released:
                    break
                params.queue_after_big_launch(lambda b=b: comm.launch_bucket(b["lo"], b["hi"], pdl=_BUCKET_PDL, blocks=self.cfg.grad_bucket_blocks))
                state["next"] += 1

        with params.releases_to(ready):
            loss.backward()
        flat.finalize_grads()
        params.after_big_launch(flush=True)                 # queued, but no big kernel followed (generic path / last layer)
        for b in plan[state["next"]:]:
            comm.launch_bucket(b["lo"], b["hi"])
        if getattr(self.optimizer, "ax", None) is not None:
            self.optimizer.average_()                       # asgd / ntasgd: the buckets updated p; every rank averages all of it

    def _step_eager(self, x: torch.Tensor, y: torch.Tensor, lengths: Optional[torch.Tensor] = None) -> torch.Tensor:
        if self.stateful:
            with torch.no_grad():
                for (h, c), (hp, cp) in zip(self.state, self.state_prev):
                    hp.copy_(h)
                    cp.copy_(c)
        self.flat.zero_grad()
        loss, _logits, _correct = self.model(x, y, lengths, state=self.state_prev)
        if self._wd_autograd:
            loss = loss + torch.stack([fn(v) * wd for (v, fn, wd) in self._wd_autograd]).sum()
        train_loss = loss
        if self._act_pen is not None:          # AR / TAR weigh into what backward runs on, not into the reported loss
            pen = self.model.rnn.activation_penalties
            with torch.no_grad():
                self._act_pen.copy_(pen)
            train_loss = loss + self.act_reg[0] * pen[0] + self.act_reg[1] * pen[1]
        l2 = None
        if self._wd_in_kernel:                 # reported total loss includes the L2 value (of the weights this step used); its
            with torch.no_grad():              # gradient is applied by the update kernel
                l2 = torch.stack([fn(v) * wd for (v, fn, wd) in self._wd_in_kernel]).sum()
        if self._bucket_plan:
            self._backward_with_buckets(train_loss)  # backward + per-bucket fused allreduce / update, overlapped with backward
        else:
            train_loss.backward()
            self.flat.finalize_grads()
            if self.sync_grads:
                self.comm.grad_step_(self.flat, self.optimizer)
            else:
                self.optimizer.step()
        if l2 is not None:
            loss = loss.detach() + l2
        if self._dropout_on:
            self._bump_dropout_step()
        if self.stateful:
            with torch.no_grad():
                for (h, c), (hT, cT) in zip(self.state, self.model.rnn.final_state()):
                    h.copy_(hT)
                    c.copy_(cT)
        return loss.detach()

    def _bump_dropout_step(self):
        rnn = self.model.rnn
        if isinstance(rnn.dropout_step, torch.Tensor):
            from .ops.cuda_ext import ext
            ext().ar_bump_step(rnn.dropout_step)          # a one-thread kernel: inside a captured step it runs on every replay
        else:
            rnn.dropout_step += 1

    def set_dropout_step(self, n: int):
        """Steps completed, for the dropout masks (a resumed run draws the masks the uninterrupted run would have)."""
        rnn = self.model.rnn
        if isinstance(rnn.dropout_step, torch.Tensor):
            rnn.dropout_step.fill_(int(n))
        else:
            rnn.dropout_step = int(n)

    def step(self, x: torch.Tensor, y: torch.Tensor, lengths: Optional[torch.Tensor] = None, reset: bool = False) -> torch.Tensor:
        """One full training step on this replica; returns the (detached, device) loss.  ``lengths``: optional int32 ``[B]``
        per-sample sequence lengths of a right-padded ``x`` (a captured graph must have been captured with lengths too).

        ``--stateful``: the step copies ``state`` into ``state_prev``, runs forward and backward from ``state_prev`` (a constant:
        no gradient crosses the segment boundary) and after the update writes the final states into ``state``.  ``reset``: the
        batch opens a new pass over the streams; ``state`` is zeroed first (one ``zero_()`` outside any graph, so a captured
        step stays valid across passes)."""
        self.steps_done += 1
        if reset and self.stateful:
            for h, c in self.state:
                h.zero_()
                c.zero_()
        if self._graph is None:
            return self._step_eager(x, y, lengths)
        if (lengths is None) != (self._static[2] is None):
            raise ValueError("the captured step was captured " + ("with" if lengths is None else "without") + " lengths")
        bound = self._bound.get((x.data_ptr(), y.data_ptr(), 0 if lengths is None else lengths.data_ptr(), tuple(x.shape)))
        if bound is not None:                   # the batch already sits in a buffer a graph was captured on: no staging copy
            g, sloss = bound
        else:
            sx, sy, sl, sloss = self._static
            if x.data_ptr() != sx.data_ptr():       # (a loader may have gathered the batch straight into graph_inputs())
                sx.copy_(x, non_blocking=True)
            if y.data_ptr() != sy.data_ptr():
                sy.copy_(y, non_blocking=True)
            if lengths is not None and lengths.data_ptr() != sl.data_ptr():
                sl.copy_(lengths, non_blocking=True)
            g = self._graph
        g.replay()
        self.optimizer.step_count += 1          # host mirror; the kernels use the device-resident counter
        return sloss

    def grad_norm(self) -> Optional[torch.Tensor]:
        """``--clip_grad_norm``: the global norm of the last step's gradient before clipping (a 0-dim fp32 tensor on the
        engine's device; read it without a host sync until you need the value), else None."""
        if self.optimizer.clip_norm <= 0:
            return None
        return self.optimizer.clip_out[0].clone()

    def activation_penalties(self) -> Optional[torch.Tensor]:
        """``--activation_reg`` / ``--temporal_activation_reg``: the unweighted ``(AR, TAR)`` of the last training step, a device
        fp32 ``[2]`` tensor (the static buffer every step, and every replay of a captured one, rewrites; copy it to keep it), else
        None."""
        return self._act_pen

    def carried_state(self):
        """``--stateful``: ``[(h [B,H], c [B,H]) per layer]``, the buffers the next step starts from (None without the flag)."""
        return self.state

    def load_carried_state(self, state) -> None:
        """Put a saved carried state (``carried_state()`` of an earlier run, on any device) into the buffers."""
        with torch.no_grad():
            for (h, c), (h1, c1) in zip(self.state, state):
                h.copy_(h1)
                c.copy_(c1)

    def graph_inputs(self):
        """(x, y, lengths) input buffers of the captured graph (lengths None when captured without), or None: a loader that
        assembles batches on the device can write them here directly (``DeviceShard.next(out=...)``) and ``step()`` then skips
        its staging copy."""
        return None if self._graph is None else self._static[:3]

    def maybe_average(self, force: bool = False):
        """Parameter-average sync point (reference semantics: once, at the end; or every ``sync_every`` steps)."""
        cfg = self.cfg
        if self.world_size <= 1 or cfg.sync_mode != "param_avg":
            return
        if force or (cfg.sync_every and self.steps_done % cfg.sync_every == 0):
            self.comm.average_params_(self.flat, cfg.average_scope)

    @contextlib.contextmanager
    def averaged_weights(self):
        """``--optimizer asgd / ntasgd``: inside the block the model holds the average of the iterates (``ax``), once averaging
        is on and has averaged at least one update; the raw weights are back, bit for bit, when it exits.  A no-op otherwise."""
        opt = self.optimizer
        swap = opt.ax is not None and opt.has_average()
        if swap:
            opt.swap_average()
        try:
            yield swap
        finally:
            if swap:
                opt.swap_average()

    def finish_averaging(self) -> bool:
        """End of training with ``--optimizer asgd / ntasgd``: put the average into the weights (once; the raw last iterate
        goes to ``ax``), so the replica average, the export and the returned variables are those of the averaged model.  -> whether
        it swapped."""
        opt = self.optimizer
        if opt.ax is None or not opt.has_average() or self._averaging_finished:
            return False
        opt.swap_average()
        self._averaging_finished = True
        return True

    # ---------------------------------------------------------------------------------------------------
    def capture(self, x: torch.Tensor, y: torch.Tensor, warmup: int = 3, bind=(), lengths: Optional[torch.Tensor] = None):
        """Capture fwd+bwd+update into one CUDA graph (static shapes).  Adam's bias correction is derived in-kernel from
        a device-resident step counter, so replays are exact.

        ``bind``: ``(x, y)`` pairs of LONG-LIVED device buffers that batches will be handed over in (the two staging slots of
        ``PinnedHostLoader``, fixed slices of a device-resident shard).  One more graph is captured directly on each of them,
        and ``step()`` replays it when it is given exactly that buffer - the 67 MB copy into the graph's own input buffer
        (27 us of a 4 ms step) disappears.  Any other tensor still goes through the staging copy.

        ``lengths`` (int32 ``[B]``): variable-length batches - a third static graph input; ``bind`` then takes
        ``(x, y, lengths)`` triples."""
        assert self.device.type == "cuda"
        sx, sy = x.clone(), y.clone()
        sl = None if lengths is None else lengths.clone()
        # warm-up / capture run real updates: snapshot the training state and put it back, so capturing is not
        # `warmup` uncounted optimizer steps on one batch and the host / device Adam step counters stay equal
        opt = self.optimizer
        snap = {"data": self.flat.data.clone(), "step_count": opt.step_count,
                "m": None if opt.m is None else opt.m.clone(), "v": None if opt.v is None else opt.v.clone(),
                "step_dev": None if opt.step_dev is None else opt.step_dev.clone(),
                "ax": None if opt.ax is None else opt.ax.clone(), "avg": None if opt.avg is None else opt.avg.clone(),
                "dropout_step": self.model.rnn.dropout_step.clone(),
                "state": None if not self.stateful else [(h.clone(), c.clone()) for h, c in self.state + self.state_prev]}
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            for _ in range(warmup):
                self._step_eager(sx, sy, sl)
        torch.cuda.current_stream().wait_stream(s)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            sloss = self._step_eager(sx, sy, sl)
        bound = {}
        for b in bind:
            bx, by, bl = (tuple(b) + (None,))[:3]
            assert bx.shape == sx.shape and bx.dtype == sx.dtype and by.shape == sy.shape and bx.is_contiguous() and by.is_contiguous()
            assert (bl is None) == (sl is None) and (bl is None or (bl.shape == sl.shape and bl.dtype == sl.dtype and bl.is_contiguous()))
            gb = torch.cuda.CUDAGraph()
            with torch.cuda.graph(gb):
                lb = self._step_eager(bx, by, bl)
            bound[(bx.data_ptr(), by.data_ptr(), 0 if bl is None else bl.data_ptr(), tuple(bx.shape))] = (gb, lb)
            self._bound_keepalive.append((bx, by, bl))      # the graphs hold raw pointers into these buffers
        with torch.no_grad():
            self.flat.data.copy_(snap["data"])
            self.flat.refresh_shadow()
            if snap["m"] is not None:
                opt.m.copy_(snap["m"]); opt.v.copy_(snap["v"])
            if snap["step_dev"] is not None:
                opt.step_dev.copy_(snap["step_dev"])
            if snap["ax"] is not None:                      # capturing does not advance the average either
                opt.ax.copy_(snap["ax"]); opt.avg.copy_(snap["avg"])
            self.model.rnn.dropout_step.copy_(snap["dropout_step"])
            if snap["state"] is not None:                   # capturing does not advance the carry
                for (h, c), (h1, c1) in zip(self.state + self.state_prev, snap["state"]):
                    h.copy_(h1)
                    c.copy_(c1)
            opt.step_count = snap["step_count"]
        self._graph, self._static, self._bound = g, (sx, sy, sl, sloss), bound
        return g

    @torch.no_grad()
    def evaluate(self, x: torch.Tensor, y: torch.Tensor, lengths: Optional[torch.Tensor] = None):
        """Loss and accuracy of a batch with the model in eval mode (no dropout); ``--per_step_labels``: over the counted
        positions of ``y [B,T]``.  ``--stateful``: from ``state_prev``, the state the last step's batch was trained from."""
        was_training = self.model.training
        self.model.eval()
        try:
            loss, correct, count = self.model.score(x, y, lengths, state=self.state_prev)
        finally:
            self.model.train(was_training)
        return loss, correct.float() / count.float()
