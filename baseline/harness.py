"""Stand-in for "the reference's own NCCL(+cuBLAS) build" (BASELINE.md §2).

The reference (TensorFlow-1.0 + PySpark, original src/rnn.py) has no GPU/NCCL code path and cannot run in this
image, so the bar our kernels are measured against is built here from stock library parts only — none of this
framework's models, kernels or engine:

    torch.nn.LSTM (cuDNN persistent RNN kernels, cuBLAS GEMMs), bf16 autocast over fp32 master weights
    torch.nn.Linear head + F.cross_entropy
    torch.optim.Adam(fused=True)
    DistributedDataParallel -> NCCL all_reduce of the gradients every step (bucketed, overlapped)

Same model shape, same schedule (per-step gradient allreduce), same synthetic data shapes as bench.py's own arm.

Two variants, both timed by ``bench.py`` (the better one is the bar):
  * ``stock``: what the docs tell a user to write - fp32 module, ``torch.autocast(bf16)``, ``batch_first=True``, eager launches;
  * ``tuned``: what a careful user ends up with - bf16 module weights (no per-step re-cast of 16.8 M weights) with fp32 master
    copies + fused Adam on the masters, time-major input (no transposes around cuDNN), bf16 gradient buckets in DDP, and the
    whole step captured in a CUDA graph when there is one rank.
"""
from __future__ import annotations

import numpy as np
import torch
import torch.distributed as dist
import torch.nn as nn
import torch.nn.functional as F


class CudnnLSTMClassifier(nn.Module):
    def __init__(self, hidden, in_features, num_classes, time_major=False, bidirectional=False, dropout=0.0, per_step=False,
                 pooling="last", attention_units=128, vocab_size=0):
        super().__init__()
        self.per_step = per_step
        self.pooling = pooling
        assert len(set(hidden)) == 1, "nn.LSTM stacks equal-width layers"
        self.time_major = time_major
        self.bidirectional = bidirectional
        self.lstm = nn.LSTM(in_features, hidden[0], num_layers=len(hidden), batch_first=not time_major, bidirectional=bidirectional,
                            dropout=dropout)
        self.head = nn.Linear(hidden[-1] * (2 if bidirectional else 1), num_classes)
        if pooling == "attention":                      # u_t = tanh(W_a h_t + b_a), e_t = u_t . v
            self.att = nn.Linear(hidden[-1] * (2 if bidirectional else 1), attention_units)
            self.context = nn.Parameter(torch.randn(attention_units) / attention_units ** 0.5)
        # vocab_size > 0: token ids [B,T] (time-major [T,B]) through nn.Embedding(V, in_features) in front of the stack
        self.embed = nn.Embedding(vocab_size, in_features) if vocab_size > 0 else None

    def pool(self, out, lengths=None):
        """``--pooling mean | max | attention`` over the outputs ``out`` (time-major [T,B,H] or batch-major [B,T,H]) at each row's
        steps t < lengths[b] (every step without lengths)."""
        seq = out if self.time_major else out.transpose(0, 1)            # [T,B,H]
        T = seq.shape[0]
        keep = torch.ones(T, seq.shape[1], dtype=torch.bool, device=seq.device) if lengths is None else \
            torch.arange(T, device=seq.device).view(T, 1) < lengths.view(1, -1)
        hm = seq.masked_fill(~keep.unsqueeze(2), 0)
        if self.pooling == "mean":
            return hm.sum(0) / keep.sum(0, keepdim=True).t().to(hm.dtype)
        if self.pooling == "max":
            return seq.masked_fill(~keep.unsqueeze(2), float("-inf")).max(0).values
        e = (torch.tanh(self.att(hm)) @ self.context.to(hm.dtype)).masked_fill(~keep, float("-inf"))
        return (torch.softmax(e.float(), 0).to(hm.dtype).unsqueeze(2) * hm).sum(0)

    def forward(self, x, lengths=None):
        if self.embed is not None:
            x = self.embed(x)
        out, (h_n, _) = self.lstm(x)
        if self.per_step:                               # nn.Linear over every output: logits [B,T,C] (time-major: [T,B,C])
            return self.head(out)
        if self.pooling != "last":
            return self.head(self.pool(out, lengths))
        if self.bidirectional:                          # [forward final | reverse final (after time 0)], as the framework's model
            return self.head(torch.cat([h_n[-2], h_n[-1]], 1))
        return self.head(out[-1] if self.time_major else out[:, -1, :])


class BaselineRunner:
    def __init__(self, hidden, in_features, num_classes, batch, seq_len, rank, world, device, optimizer="adam", lr=1e-3,
                 variant="stock", bidirectional=False, dropout=0.0, per_step=False, pooling="last", vocab_size=0):
        """``per_step``: sequence labelling - labels ``[B,T]``, the head over every output and the mean cross-entropy over all
        ``T·B`` positions (default: classify the final state, labels ``[B]``).  ``pooling``: classify the mean / max / attention
        pooling of the top layer's outputs (``nn.LSTM`` + masked pool + ``nn.Linear``); a step then takes ``lengths``.
        ``vocab_size`` > 0: a step takes int token ids ``[B,T]`` read through ``nn.Embedding(vocab_size, in_features)``."""
        self.rank, self.world, self.device = rank, world, device
        self.B, self.T, self.D, self.C = batch, seq_len, in_features, num_classes
        self.variant = variant
        self.per_step = per_step
        self.tuned = variant == "tuned"
        self.graph = None
        self.bound = {}
        self.bind_inputs = True
        torch.manual_seed(0)
        if world > 1 and not dist.is_initialized():
            dist.init_process_group("nccl", rank=rank, world_size=world, device_id=device)
        model = CudnnLSTMClassifier(hidden, in_features, num_classes, time_major=self.tuned, bidirectional=bidirectional,
                                    dropout=dropout, per_step=per_step, pooling=pooling, vocab_size=vocab_size).to(device)
        if self.tuned:
            model = model.to(torch.bfloat16)
            model.lstm.flatten_parameters()
        self.model = nn.parallel.DistributedDataParallel(model, device_ids=[device.index], gradient_as_bucket_view=True) if world > 1 else model
        self.params = [p for p in self.model.parameters()]
        if self.tuned:                                   # fp32 master weights: the optimizer never sees the bf16 copies
            self.masters = [p.detach().float().clone().requires_grad_(True) for p in self.params]
            for m in self.masters:
                m.grad = torch.zeros_like(m)
            opt_params = self.masters
        else:
            opt_params = self.params
        if optimizer == "adam":
            self.opt = torch.optim.Adam(opt_params, lr=lr, fused=True, capturable=self.tuned and world == 1)
        else:
            self.opt = torch.optim.SGD(opt_params, lr=lr)

    def _step_stock(self, x, y):
        self.opt.zero_grad(set_to_none=True)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            logits = self.model(x)
        if self.per_step:
            loss = F.cross_entropy(logits.float().reshape(-1, self.C), y.reshape(-1))
        else:
            loss = F.cross_entropy(logits.float(), y)
        loss.backward()
        self.opt.step()
        return loss.detach()

    def _step_tuned(self, x, y):
        """x arrives batch-major [B,T,D] like in every arm; the time-major view is a stride permutation (cuDNN takes it)."""
        for p in self.params:
            p.grad = None
        logits = self.model(x.transpose(0, 1))
        if self.per_step:                                # time-major logits [T,B,C] against labels [B,T]
            loss = F.cross_entropy(logits.float().reshape(-1, self.C), y.t().reshape(-1))
        else:
            loss = F.cross_entropy(logits.float(), y)
        loss.backward()
        with torch.no_grad():
            torch._foreach_copy_([m.grad for m in self.masters], [p.grad for p in self.params])  # bf16 grads -> fp32
        self.opt.step()
        with torch.no_grad():
            torch._foreach_copy_(self.params, self.masters)                                      # fp32 masters -> bf16 weights
        return loss.detach()

    def train_step(self, x, y):
        if self.graph is not None:
            bound = self.bound.get((x.data_ptr(), y.data_ptr()))
            if bound is not None:                    # a graph captured directly on this buffer (same input binding as the framework's arm)
                bound[0].replay()
                return bound[1]
            sx, sy, sloss = self.static
            sx.copy_(x, non_blocking=True)
            sy.copy_(y, non_blocking=True)
            self.graph.replay()
            return sloss
        return self._step_tuned(x, y) if self.tuned else self._step_stock(x, y)

    def capture(self, x, y, warmup=3, bind=()):
        """CUDA-graph the whole step (single rank: NCCL buckets inside a capture are not worth the fragility for a baseline).
        ``bind``: long-lived (x, y) buffers that get a graph of their own (no staging copy when a step is handed one of them)."""
        self.bound = {}
        if self.world > 1:
            return False
        try:
            sx, sy = x.clone(), y.clone()
            s = torch.cuda.Stream()
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                for _ in range(warmup):
                    self.train_step(sx, sy)
            torch.cuda.current_stream().wait_stream(s)
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                sloss = self.train_step(sx, sy)
            bound = {}
            for bx, by in bind:
                gb = torch.cuda.CUDAGraph()
                with torch.cuda.graph(gb):
                    lb = self.train_step(bx, by)
                bound[(bx.data_ptr(), by.data_ptr())] = (gb, lb)
            self.graph, self.static, self.bound = g, (sx, sy, sloss), bound
            return True
        except Exception as e:                           # noqa: BLE001
            self.graph = None
            self.capture_error = repr(e)[:200]
            torch.cuda.synchronize()
            return False

    def make_steps(self):
        B, T, D, C = self.B, self.T, self.D, self.C
        rng = np.random.default_rng(1234 + self.rank)
        nb = 4
        xs = rng.standard_normal((nb * B, T, D), dtype=np.float32)
        ys = rng.integers(0, C, size=(nb * B, T) if self.per_step else nb * B).astype(np.int64)
        dev_x = torch.as_tensor(xs).to(self.device, dtype=torch.bfloat16)
        dev_y = torch.as_tensor(ys).to(self.device)
        host_x = torch.as_tensor(xs).to(torch.bfloat16).pin_memory()
        host_y = torch.as_tensor(ys).pin_memory()
        stage = [(torch.empty(B, T, D, dtype=torch.bfloat16, device=self.device),
                  torch.empty((B, T) if self.per_step else (B,), dtype=torch.int64, device=self.device)) for _ in range(2)]
        loss_host = torch.empty(2, dtype=torch.float32, pin_memory=True)
        loss_evt = [torch.cuda.Event(), torch.cuda.Event()]
        it = {"i": 0, "slot": 0, "pending": None, "k": 0, "last": float("nan")}
        copy_stream = torch.cuda.Stream(device=self.device)

        def issue():
            """double-buffered prefetch on a copy stream (what a careful PyTorch user does with pinned memory)"""
            i = it["i"] % nb
            it["i"] += 1
            sx, sy = stage[it["slot"]]
            it["slot"] ^= 1
            copy_stream.wait_stream(torch.cuda.current_stream(self.device))
            with torch.cuda.stream(copy_stream):
                sx.copy_(host_x[i * B:(i + 1) * B], non_blocking=True)
                sy.copy_(host_y[i * B:(i + 1) * B], non_blocking=True)
                ev = torch.cuda.Event()
                ev.record(copy_stream)
            return sx, sy, ev

        def step_dev():
            i = it["i"] % nb
            it["i"] += 1
            return self.train_step(dev_x[i * B:(i + 1) * B], dev_y[i * B:(i + 1) * B])

        def step_e2e():
            if it["pending"] is None:
                it["pending"] = issue()
            sx, sy, ev = it["pending"]
            torch.cuda.current_stream(self.device).wait_event(ev)
            it["pending"] = issue()
            loss = self.train_step(sx, sy)
            k = it["k"]                              # same asynchronous, one-step-late loss read-back as the framework's arm
            loss_host[k & 1].copy_(loss.float(), non_blocking=True)
            loss_evt[k & 1].record()
            if k > 0:
                loss_evt[(k - 1) & 1].synchronize()
                it["last"] = float(loss_host[(k - 1) & 1])
            it["k"] = k + 1
            return loss_host

        graphed = False
        if self.tuned:
            graphed = self.capture(dev_x[:B], dev_y[:B], bind=[(dev_x[i * B:(i + 1) * B], dev_y[i * B:(i + 1) * B]) for i in range(nb)] + stage
                                   if self.bind_inputs else ())
        h2d = B * T * D * 2 + B * (T if self.per_step else 1) * 8
        return step_dev, step_e2e, h2d, 4, 0, {"lstm": "cudnn", "comm": "nccl-ddp" if self.world > 1 else "none",
                                              "variant": self.variant, "cuda_graph": graphed}
