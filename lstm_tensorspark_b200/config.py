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
import math
import warnings
from dataclasses import dataclass, field
from typing import List, Optional, Sequence


FUSED_CLIP_ERROR = ("--clip_grad_norm with --sync_mode grad_allreduce needs the norm of the averaged gradient before any update, "
                    "which --comm fused does not compute (it updates each gradient bucket as soon as it is reduced): use --comm nccl")


ATTENTION_UNITS_DEFAULT = 128
NUM_CLASSES_DEFAULT = 3
MAX_NEW_TOKENS_DEFAULT = 32
TEMPERATURE_DEFAULT = 1.0


@dataclass
class Config:
    # ---- reference flags (rnn.py:310-334) -------------------------------------------------------
    master: str = "local"               # accepted for CLI compatibility, unused (no Spark)
    spark_exec_memory: str = "4g"       # accepted for CLI compatibility, unused
    partitions: int = 4                 # number of data shards / replicas (one rank per GPU while GPUs last)
    epochs: int = 1
    hidden_units: str = "128,256"
    batch_size: int = 10                # 0 => whole shard in one batch (reference intent, Q3)
    num_classes: int = NUM_CLASSES_DEFAULT
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
    weight_drop: float = 0.0            # AWD-LSTM weight drop: in training, every layer direction's recurrent weights W_h are
                                        # multiplied by a Bernoulli(1-P) mask / (1-P) drawn once per step (DropConnect)
    output_dropout: float = 0.0         # in training, the top layer's output sequence is dropped before the head / pooling reads it
    input_dropout: float = 0.0          # in training, the embedding output x_t is dropped before the first layer (--vocab_size)
    embedding_dropout: float = 0.0      # in training, whole rows of the embedding table are dropped for the lookup, one mask per step
    locked_dropout: bool = False        # --dropout / --output_dropout / --input_dropout draw one mask per sequence and training step,
                                        # shared by every time step (AWD-LSTM's LockedDropout), not a new mask per step
    activation_reg: float = 0.0         # AWD-LSTM's AR: training adds ALPHA * mean(out^2) of the top layer's output as the head reads it
    temporal_activation_reg: float = 0.0  # AWD-LSTM's TAR: training adds BETA * mean((h_t - h_{t-1})^2) of its raw output
    per_step_labels: bool = False       # sequence labelling: a label at every time step ([B,T]), the head scores the top layer's
                                        # output at each step (nn.LSTM -> nn.Linear -> cross_entropy over the real positions); a CSV
                                        # row is k*in_features values followed by k labels
    pooling: str = "last"               # what the classifier reads: last (the top layer's state after each sample's last step) |
                                        # mean | max | attention over the top layer's outputs at the sample's real steps
    attention_units: int = ATTENTION_UNITS_DEFAULT  # A of --pooling attention: u_t = tanh(h_t W_a + b_a) [A], score u_t . v
    vocab_size: int = 0                 # V > 0: the input is int token ids [B,T] (one step: [B]) and the first layer reads
                                        # x_t = Embedding[tok_t], a learned [V, in_features] table (nn.Embedding); a CSV row is k ids
                                        # followed by the label (--per_step_labels: by k labels).  0 = float features
    next_token: bool = False            # language modelling (needs --vocab_size V): the label of step t is the token of step t + 1.
                                        # Turns on --per_step_labels and sets --num_classes to V; a CSV row is seq_len + 1 ids
    stateful: bool = False              # --next_token on one token stream cut into --batch_size parallel streams: consecutive
                                        # batches continue each stream and start from the state the previous batch ended in,
                                        # detached (truncated backpropagation through time); --mode eval scores the whole stream
    tie_embeddings: bool = False        # --next_token with --in_features == the last --hidden_units: the softmax reads the embedding
                                        # table as its weights, logits = h Embedding^T + bias (Press & Wolf 2017), no Dense1/weights
    max_new_tokens: int = MAX_NEW_TOKENS_DEFAULT  # --mode generate: tokens sampled after each prompt
    temperature: float = TEMPERATURE_DEFAULT      # --mode generate: sample from softmax(logits / temperature); 0 = greedy
    top_k: int = 0                      # --mode generate: sample from the k most likely classes only (ties at the k-th kept); 0 = off
    top_p: float = 1.0                  # --mode generate: then from the smallest top set of tempered mass >= P (nucleus); 1 = off
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
    clip_grad_norm: float = 0.0         # >0: clip the gradient by its global norm to this value before the update (0 = off)
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

    def __post_init__(self):
        # --next_token implies the label layout and the class count (validate() reports the combinations it refuses)
        if self.next_token and self.vocab_size > 0:
            self.per_step_labels = True
            if self.num_classes == NUM_CLASSES_DEFAULT:
                self.num_classes = self.vocab_size

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

    def clips_synced_grads(self) -> bool:
        """Gradient clipping on the averaged gradient of several replicas (``--sync_mode grad_allreduce``)."""
        return self.clip_grad_norm > 0 and self.sync_mode == "grad_allreduce" and self.partitions > 1

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
        if self.stateful:
            if not self.next_token:
                raise ValueError("--stateful needs --next_token: it carries the state along one token stream, whose labels are "
                                 "the ids that follow")
            if self.variable_length:
                raise ValueError("--stateful does not combine with --variable_length: the stream is cut into segments of "
                                 "exactly --seq_len positions and has no padding")
            if self.learn_initial_state:
                raise ValueError("--stateful does not combine with --learn_initial_state true: a pass starts from the zero state "
                                 "and every later segment from the state the previous one ended in")
            if self.pooling != "last":
                raise ValueError(f"--stateful does not combine with --pooling {self.pooling}: every step's output is scored")
            if self.batch_size < 1:
                raise ValueError("--stateful needs --batch_size B >= 1: the stream is cut into B parallel streams")
        if self.tie_embeddings:
            if not self.next_token:
                raise ValueError("--tie_embeddings needs --next_token: the softmax can share the embedding table only when its "
                                 "classes are the vocabulary")
            if self.in_features != self.hidden_list()[-1]:
                raise ValueError(f"--tie_embeddings needs --in_features (the embedding width, {self.in_features}) equal to the last "
                                 f"--hidden_units ({self.hidden_list()[-1]}): the softmax reads the table's rows as its weights")
        if self.next_token:
            if self.vocab_size <= 0:
                raise ValueError("--next_token needs --vocab_size V > 0: it predicts the next token id out of the V of the vocabulary")
            if self.seq_len < 2:
                raise ValueError("--next_token needs --seq_len >= 2 (a row is seq_len + 1 token ids: seq_len inputs, each labelled "
                                 "with the id that follows it)")
            if self.num_classes != self.vocab_size:
                raise ValueError(f"--next_token sets --num_classes to --vocab_size ({self.vocab_size}), got --num_classes "
                                 f"{self.num_classes}: drop --num_classes")
            if self.pooling != "last":
                raise ValueError(f"--next_token does not combine with --pooling {self.pooling}: every step's output is scored, "
                                 "there is nothing to pool")
            if self.bidirectional:
                raise ValueError("--next_token does not combine with --bidirectional: a reverse layer sees the token it is asked to "
                                 "predict")
            self.per_step_labels = True
        if self.variable_length and self.seq_len < 2:
            raise ValueError("--variable_length needs --seq_len >= 2 (the longest sample's number of steps)")
        if self.bidirectional and self.seq_len < 2:
            raise ValueError("--bidirectional needs --seq_len >= 2 (the reverse direction runs over a whole sequence)")
        if self.per_step_labels and self.seq_len < 2:
            raise ValueError("--per_step_labels needs --seq_len >= 2 (one label per time step of a sequence; the one-step [B,D] "
                             "path classifies the last state only)")
        if self.pooling not in ("last", "mean", "max", "attention"):
            raise ValueError(f"unknown --pooling {self.pooling!r}: one of last, mean, max, attention")
        if self.attention_units < 1:
            raise ValueError(f"--attention_units must be >= 1, got {self.attention_units}")
        if self.pooling != "last" and self.seq_len < 2:
            raise ValueError(f"--pooling {self.pooling} needs --seq_len >= 2 (it pools the top layer's outputs over the time steps "
                             "of a sequence)")
        if self.pooling != "last" and self.per_step_labels:
            raise ValueError(f"--pooling {self.pooling} does not combine with --per_step_labels: per-step labels score every "
                             "step's output, there is nothing to pool (use --pooling last)")
        if self.attention_units != ATTENTION_UNITS_DEFAULT and self.pooling != "attention":
            warnings.warn(f"--attention_units {self.attention_units} has no effect without --pooling attention")
        if self.vocab_size < 0:
            raise ValueError(f"--vocab_size must be >= 0 (0 = float features), got {self.vocab_size}")
        if self.vocab_size > 0 and self.normalize:
            raise ValueError("--normalize does not combine with --vocab_size: token ids are not feature values to scale")
        if not 0.0 <= self.dropout < 1.0:
            raise ValueError(f"--dropout must satisfy 0 <= P < 1, got {self.dropout}")
        if self.dropout > 0 and len(self.hidden_list()) == 1:
            warnings.warn(f"--dropout {self.dropout} has no effect with one layer: dropout applies between stacked layers "
                          "(it drops the output of every layer but the last)")
        if not 0.0 <= self.weight_drop < 1.0:
            raise ValueError(f"--weight_drop must satisfy 0 <= P < 1, got {self.weight_drop}")
        for flag in ("output_dropout", "input_dropout", "embedding_dropout"):
            p = getattr(self, flag)
            if not 0.0 <= p < 1.0:
                raise ValueError(f"--{flag} must satisfy 0 <= P < 1, got {p}")
            if p > 0 and flag != "output_dropout" and self.vocab_size <= 0:
                raise ValueError(f"--{flag} needs --vocab_size > 0: it drops the token embedding, and float features have none")
        if self.output_dropout > 0 and self.pooling == "last" and not self.per_step_labels:
            raise ValueError("--output_dropout needs a head that reads the top layer's output sequence (--per_step_labels, "
                             "--next_token or --pooling mean | max | attention): with --pooling last the head reads only the "
                             "final state, and there is no sequence to drop")
        for flag in ("activation_reg", "temporal_activation_reg"):
            c = getattr(self, flag)
            if not (math.isfinite(c) and c >= 0):
                raise ValueError(f"--{flag} must be a finite number >= 0 (0 = off), got {c}")
            if c > 0 and self.pooling == "last" and not self.per_step_labels:
                raise ValueError(f"--{flag} needs a head that reads the top layer's output sequence (--per_step_labels, "
                                 "--next_token or --pooling mean | max | attention): with --pooling last the head reads only the "
                                 "final state, and there is no sequence to regularise")
        if self.locked_dropout and not (self.dropout > 0 or self.output_dropout > 0 or self.input_dropout > 0):
            warnings.warn("--locked_dropout has no effect without --dropout, --output_dropout or --input_dropout > 0: it shares "
                          "their masks across time steps")
        if self.sync_mode not in ("param_avg", "grad_allreduce", "none"):
            raise ValueError(f"unknown --sync_mode {self.sync_mode}")
        if not (math.isfinite(self.clip_grad_norm) and self.clip_grad_norm >= 0):
            raise ValueError(f"--clip_grad_norm must be a finite number >= 0 (0 = off), got {self.clip_grad_norm}")
        if self.clips_synced_grads() and self.comm == "fused":
            raise ValueError(FUSED_CLIP_ERROR)
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
        if self.mode not in ("train", "eval", "generate"):
            raise ValueError("--mode is train (the only one the reference implements, src/rnn.py:371), eval (score a trained "
                             "model: --resume <averaged_model.pt | checkpoint dir>, default = what the last training run left) or "
                             "generate (continue prompts with a --next_token model, found the same way)")
        if self.max_new_tokens < 1:
            raise ValueError(f"--max_new_tokens must be >= 1, got {self.max_new_tokens}")
        if not (math.isfinite(self.temperature) and self.temperature >= 0):
            raise ValueError(f"--temperature must be a finite number >= 0 (0 = greedy), got {self.temperature}")
        if self.top_k < 0:
            raise ValueError(f"--top_k must be an integer >= 0 (0 = off), got {self.top_k}")
        if not (math.isfinite(self.top_p) and 0 < self.top_p <= 1):
            raise ValueError(f"--top_p must be a number in (0, 1] (1 = off), got {self.top_p}")
        if self.mode == "generate" and not self.next_token:
            raise ValueError("--mode generate needs --next_token (and the --vocab_size the model was trained with): it continues "
                             "token sequences with a next-token language model")
        for flag, default in (("max_new_tokens", MAX_NEW_TOKENS_DEFAULT), ("temperature", TEMPERATURE_DEFAULT), ("top_k", 0),
                              ("top_p", 1.0)):
            if getattr(self, flag) != default and self.mode != "generate":
                warnings.warn(f"--{flag} {getattr(self, flag)} has no effect without --mode generate")
        if self.mode == "generate" and self.temperature == 0:
            for flag, default in (("top_k", 0), ("top_p", 1.0)):
                if getattr(self, flag) != default:
                    warnings.warn(f"--{flag} {getattr(self, flag)} has no effect with --temperature 0: greedy decoding takes the "
                                  "arg-max, which every filter keeps")
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
    "mode": "Execution mode: train, eval (score a trained model) or generate (continue the prompts of --training_path, or of "
            "--synthetic walks, with a --next_token model; writes <output_path>/generated.csv)",
    "max_new_tokens": "--mode generate: tokens to sample after each prompt (>= 1)",
    "temperature": "--mode generate: sample from softmax(logits / temperature) by Gumbel-max with noise seeded by --seed; 0 = "
                   "greedy (the arg-max)",
    "top_k": "--mode generate: sample only from the K classes with the largest logits (every class tied with the K-th is kept); "
             "0 = off.  No effect at --temperature 0",
    "top_p": "--mode generate: nucleus sampling, after --top_k: sample only from the classes with the largest logits whose "
             "share of softmax(logits / temperature) first reaches P (ties at the cut are kept); 1 = off.  The reported "
             "log-probabilities stay under the full softmax",
    "checkpoint_path": "Directory where to save network model and logs",
    "clip_grad_norm": "Clip the gradient by its global L2 norm to this value before the update, as "
                      "torch.nn.utils.clip_grad_norm_ (0 = off); the norm includes the --weight_decay term and, with "
                      "--sync_mode grad_allreduce, is that of the averaged gradient (--comm nccl or gloo)",
    "pooling": "What the classifier reads: last (the top layer's final state, default), or mean / max / attention pooling of "
               "the top layer's outputs over each sample's real steps",
    "attention_units": "Units A of --pooling attention (score = tanh(h_t W_a + b_a) . v)",
    "vocab_size": "Read token ids through a learned embedding table of V rows and --in_features columns (nn.Embedding in front "
                  "of the first layer); a CSV row is k ids followed by the label (or by k labels with --per_step_labels). "
                  "0 = float features",
    "next_token": "Train a next-token language model on --vocab_size V token ids: the label of step t is the id of step t + 1 "
                  "(turns on --per_step_labels, sets --num_classes to V); a CSV row is seq_len + 1 ids, or 2..seq_len + 1 with "
                  "--variable_length; evaluations also report perplexity = exp(loss)",
    "stateful": "With --next_token: read --training_path (or --synthetic) as one token stream cut into --batch_size parallel "
                "streams; each batch continues every stream by --seq_len positions from the state the previous batch ended in, "
                "with gradients stopped there (truncated backpropagation through time); --mode eval reports the perplexity of the "
                "whole stream",
    "tie_embeddings": "With --next_token and --in_features equal to the last --hidden_units: the softmax reuses the embedding "
                      "table as its weights (logits = h Embedding^T + Dense1/bias; weight tying, Press & Wolf 2017), so the model "
                      "has no Dense1/weights and the table's gradient is the sum of both uses",
    "weight_drop": "Weight drop (DropConnect on the recurrent weights, AWD-LSTM): in training, every layer's hidden-to-hidden "
                   "matrix W_h (both directions, one-layer models too) is multiplied by a Bernoulli(1 - P) mask scaled by "
                   "1 / (1 - P), one mask per training step shared by every time step and batch row; evaluation and generation "
                   "use the raw weights.  0 = off",
    "output_dropout": "In training, drop the top layer's output sequence (both directions) with probability P before the head "
                      "or the pooling reads it (AWD-LSTM's dropout); needs --per_step_labels, --next_token or --pooling mean | "
                      "max | attention.  0 = off",
    "input_dropout": "In training, drop the embedding output x_t = Embedding[tok_t] with probability P before the first layer "
                     "reads it (AWD-LSTM's dropouti); needs --vocab_size > 0.  0 = off",
    "embedding_dropout": "In training, drop whole rows of the embedding table with probability P for the lookup, one mask over "
                         "the V ids per training step, kept rows scaled by 1 / (1 - P) (AWD-LSTM's dropoute); needs --vocab_size "
                         "> 0.  With --tie_embeddings the softmax still reads the raw table.  0 = off",
    "locked_dropout": "Locked (variational) dropout: --dropout, --output_dropout and --input_dropout draw one mask per sequence "
                      "and training step, shared by every time step (AWD-LSTM's LockedDropout; Gal & Ghahramani 2016), instead "
                      "of a new mask at every step",
    "activation_reg": "AWD-LSTM's activation regularisation (AR): in training, the loss backward runs on gains ALPHA times the "
                      "mean square of the top layer's output as the head reads it (after --output_dropout) over the real "
                      "positions; the reported loss stays the cross-entropy, and AR is logged as `ar`.  Needs --per_step_labels, "
                      "--next_token or --pooling mean | max | attention.  0 = off",
    "temporal_activation_reg": "AWD-LSTM's temporal activation regularisation (TAR): in training, the loss backward runs on gains "
                               "BETA times the mean square of h_t - h_{t-1} of the top layer's raw output (before dropout) over "
                               "the real steps t >= 1 of each sequence; logged as `tar`.  Same head rule as --activation_reg.  0 = off",
    "per_step_labels": "Label every time step (sequence labelling): labels [B,T], loss and accuracy over the real positions; "
                       "a CSV row is k*in_features values followed by k labels",
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
