"""Flag system shared by both entry points (``rnn.py`` and ``lstm-no-spark.py``).

Parity targets (reference, read-only):
  * distributed CLI  : original src/rnn.py:306-336   (argparse, ``parse_known_args``)
  * standalone flags : original src/lstm-no-spark.py:9-38 (``tf.app.flags`` + ``params_str`` dump)
  * ``net_settings``  : original src/rnn.py:376-389

One dataclass, one parser.  Every reference flag keeps its name, type and default; the Spark-only flags
(``--master``, ``--spark_exec_memory``) are accepted and ignored.  New flags are additive.
"""
from __future__ import annotations

import argparse
import dataclasses
import warnings
from dataclasses import dataclass, field
from typing import List, Optional, Sequence


@dataclass
class Config:
    # ---- reference flags (rnn.py:310-334) -------------------------------------------------------
    master: str = "local"               # accepted for CLI compatibility, unused (no Spark)
    spark_exec_memory: str = "4g"       # accepted for CLI compatibility, unused
    partitions: int = 4                 # number of data shards / replicas (one rank per GPU while GPUs last)
    epochs: int = 1
    hidden_units: str = "128,256"
    batch_size: int = 10                # 0 => whole shard in one batch (reference intent, Q3)
    num_classes: int = 3
    in_features: int = 4
    learning_rate: float = 1e-3
    evaluate_every: int = 10
    training_path: str = "train"
    labels_path: str = "train_labels"   # parsed, never read (as in the reference)
    output_path: str = "output_path"    # averaged model is written here (Q12)
    mode: str = "train"
    checkpoint_path: str = "train_dir"
    # ---- additive flags -------------------------------------------------------------------------
    use_pretrained_model: bool = False  # the flag the reference reads but never defines (Q4)
    resume: str = ""                    # explicit checkpoint dir/prefix to resume from
    seq_len: int = 1                    # time steps per sample (reference == 1)
    variable_length: bool = False       # samples of 1..seq_len steps: a CSV row is k*in_features values + label (zero-padded to
                                        # seq_len); --synthetic draws lengths in [seq_len//4, seq_len].  The final state is each
                                        # sample's state after its own last step (padded steps hold the state)
    bidirectional: bool = False         # every layer also runs a reverse-time LSTM; layer l+1 and the classifier read
                                        # [forward | reverse] (2 H wide), as nn.LSTM(bidirectional=True) on a packed sequence
    dropout: float = 0.0                # nn.LSTM(dropout=P): in training, the output sequence of every layer but the last is
                                        # multiplied by a Bernoulli(1-P) mask / (1-P) before the next layer reads it
    dtype: str = "auto"                 # auto: bf16 on cuda, fp32 on cpu
    device: str = "auto"                # auto | cpu | cuda
    backend: str = "auto"               # auto | cuda_ext (hand-written sm_90a kernels) | torch
    optimizer: str = "adam"             # adam (TF formulation) | sgd
    sync_mode: str = "param_avg"        # param_avg (reference) | grad_allreduce | none
    sync_every: int = 0                 # 0 => once at the end of training (reference); N => every N steps
    average_scope: str = "lstm"         # lstm (reference: map_data_by_key set) | all
    comm: str = "auto"                  # auto | fused (in-kernel NVLink allreduce) | nccl | gloo
    steps_mode: str = "compat"          # compat: max_steps = epochs*batch_size (Q5) | epochs: epochs*batches/epoch
    max_steps: int = 0                  # explicit override of the step count
    seed: int = 0
    independent_init: bool = False      # reference behaviour: every replica draws its own init (Q9)
    learn_initial_state: Optional[bool] = None  # None: True when seq_len == 1 (reference, Q7)
    init: str = "truncated_normal"      # truncated_normal (std 1, reference Q8) | scaled (1/sqrt(fan_in))
    init_std: float = 1.0
    normalize: bool = False             # global min-max normalisation (Q11)
    weight_decay: float = 0.0           # L2 term of create_variable (never enabled in the reference)
    synthetic: int = 0                  # >0: use N synthetic sequences instead of a CSV
    remainder: str = "drop"             # drop | spread : rows beyond floor(N/P)*P (Q2)
    cuda_graph: bool = False
    data_residency: str = "device"      # device: the shard lives in HBM, a batch is an on-device gather (no per-step H2D) |
                                        # host: the shard stays in pinned host memory and every batch is copied host->device by an
                                        # asynchronous, triple-buffered DMA (the reference's per-step feed, src/rnn.py:264-267; shards > HBM)
    trace: str = ""                     # path for a torch.profiler chrome trace
    nvtx: bool = False
    json_log: str = ""                  # machine readable metrics file
    max_workers: int = 0                # ranks that run concurrently (Spark's local[N]); 0 = min(partitions, visible GPUs) on
                                        # CUDA, = partitions on the CPU.  partitions > workers: a rank trains its partitions in turn
    deterministic: bool = False         # bit-reproducible runs: the recurrence kernels consume operand blocks in index order (not
                                        # arrival order), so fp32 accumulation order is fixed (a few % slower)
    grad_buckets: bool = True           # fused comm, grad_allreduce: per-layer buckets synced under the lower layers' backward
    grad_bucket_blocks: int = 64        # CTAs of an overlapped bucket launch (it runs on the SMs the recurrence leaves idle)
    fault_inject: str = ""              # "rank:step" => that rank exits abnormally at that step (test hook)
    timeout_s: float = 600.0
    quiet: bool = False

    # ------------------------------------------------------------------------------------------
    def hidden_list(self) -> List[int]:
        vals = [int(h) for h in str(self.hidden_units).split(",") if str(h).strip()]
        if not vals or any(v <= 0 for v in vals):
            raise ValueError(f"--hidden_units must be a comma list of positive ints, got {self.hidden_units!r}")
        return vals

    def resolved_learn_initial_state(self) -> bool:
        if self.learn_initial_state is None:
            return self.seq_len == 1
        return bool(self.learn_initial_state)

    def net_settings(self, batch_size: Optional[int] = None) -> List[dict]:
        """The model-config object handed to ``RNN`` (reference: src/rnn.py:376-389)."""
        bs = self.batch_size if batch_size is None else batch_size
        hidden = self.hidden_list()
        settings = []
        for i, h in enumerate(hidden):
            settings.append({
                "layer_name": f"LSTMLayer{i}",
                "dim_size": self.in_features if i == 0 else (2 if self.bidirectional else 1) * hidden[i - 1],
                "num_hidden": h,
                "batch_size": bs,
                "normalize": True,      # present in the reference dict, never read there either
            })
        return settings

    def params_str(self) -> str:
        """``KEY = value`` per flag, sorted, upper-cased (reference: src/lstm-no-spark.py:33-37)."""
        items = sorted(dataclasses.asdict(self).items())
        return "".join(f"{k.upper()} = {v}\n" for k, v in items)

    def validate(self) -> "Config":
        self.hidden_list()
        if self.partitions < 1:
            raise ValueError("--partitions must be >= 1")
        if self.batch_size < 0:
            raise ValueError("--batch_size must be >= 0 (0 = whole shard)")
        if self.seq_len < 1:
            raise ValueError("--seq_len must be >= 1")
        if self.variable_length and self.seq_len < 2:
            raise ValueError("--variable_length needs --seq_len >= 2 (the longest sample's number of steps)")
        if self.bidirectional and self.seq_len < 2:
            raise ValueError("--bidirectional needs --seq_len >= 2 (the reverse direction runs over a whole sequence)")
        if not 0.0 <= self.dropout < 1.0:
            raise ValueError(f"--dropout must satisfy 0 <= P < 1, got {self.dropout}")
        if self.dropout > 0 and len(self.hidden_list()) == 1:
            warnings.warn(f"--dropout {self.dropout} has no effect with one layer: dropout applies between stacked layers "
                          "(it drops the output of every layer but the last)")
        if self.sync_mode not in ("param_avg", "grad_allreduce", "none"):
            raise ValueError(f"unknown --sync_mode {self.sync_mode}")
        if self.optimizer not in ("adam", "sgd"):
            raise ValueError(f"unknown --optimizer {self.optimizer}")
        if self.average_scope not in ("lstm", "all"):
            raise ValueError(f"unknown --average_scope {self.average_scope}")
        if self.steps_mode not in ("compat", "epochs"):
            raise ValueError(f"unknown --steps_mode {self.steps_mode}")
        if self.data_residency not in ("device", "host"):
            raise ValueError(f"unknown --data_residency {self.data_residency}")
        if self.remainder not in ("drop", "spread"):
            raise ValueError(f"unknown --remainder {self.remainder}")
        if self.mode not in ("train", "eval"):
            raise ValueError("--mode is train (the only one the reference implements, src/rnn.py:371) or eval (score a trained "
                             "model: --resume <averaged_model.pt | checkpoint dir>, default = what the last training run left)")
        return self


def _str2bool(v) -> bool:
    if isinstance(v, bool):
        return v
    s = str(v).strip().lower()
    if s in ("1", "true", "t", "yes", "y", "on"):
        return True
    if s in ("0", "false", "f", "no", "n", "off", ""):
        return False
    raise argparse.ArgumentTypeError(f"expected a boolean, got {v!r}")


_HELP = {
    "master": "Host or master node location (accepted for compatibility; ranks replace Spark workers)",
    "spark_exec_memory": "Spark executor memory (accepted for compatibility; unused)",
    "partitions": "Number of distributed partitions (= ranks, one per GPU)",
    "epochs": "Number of epochs",
    "hidden_units": "List of hidden units per layer (separated by comma)",
    "batch_size": "Mini batch size (0 = whole shard)",
    "num_classes": "Number of classes in dataset",
    "in_features": "Number of input features",
    "learning_rate": "Learning rate",
    "evaluate_every": "Numbers of steps for each evaluation",
    "training_path": "Path to training set",
    "labels_path": "Path to training_labels",
    "output_path": "Path for store network state",
    "mode": "Execution mode",
    "checkpoint_path": "Directory where to save network model and logs",
}


def build_parser(standalone: bool = False) -> argparse.ArgumentParser:
    desc = "RNN-LSTM on H100 (standalone)" if standalone else "RNN-LSTM on H100 (one rank per partition)"
    p = argparse.ArgumentParser(description=desc)
    defaults = Config()
    for f in dataclasses.fields(Config):
        if standalone and f.name in ("master", "spark_exec_memory", "partitions"):
            continue
        default = getattr(defaults, f.name)
        if standalone and f.name == "epochs":
            default = 5                                   # src/lstm-no-spark.py:12
        helptxt = _HELP.get(f.name, f.name.replace("_", " "))
        if f.type in ("bool", bool) or isinstance(default, bool) or f.name == "learn_initial_state":
            p.add_argument(f"--{f.name}", nargs="?", const=True, default=default, type=_str2bool, help=helptxt)
        else:
            p.add_argument(f"--{f.name}", default=default, type=type(default), help=helptxt)
    return p


def parse_args(argv: Optional[Sequence[str]] = None, standalone: bool = False) -> Config:
    """``parse_known_args`` like the reference (src/rnn.py:336): unknown arguments are ignored."""
    parser = build_parser(standalone)
    ns, _unknown = parser.parse_known_args(list(argv) if argv is not None else None)
    kw = vars(ns)
    if standalone:
        kw.setdefault("partitions", 1)
        kw["partitions"] = 1
    cfg = Config(**kw)
    return cfg.validate()
