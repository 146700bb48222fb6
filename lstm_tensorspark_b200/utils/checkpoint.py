"""Checkpoint writer / reader with the reference's directory layout and variable names.

Reference mechanism: ``tf.train.Saver(tf.trainable_variables())`` (default ``max_to_keep=5``), saved every
``evaluate_every`` steps and on the last step into ``<checkpoint_path>/<unix-time>/<partition_key>/`` with
prefix ``spark_lstm`` (standalone: ``<checkpoint_path>/<unix-time>/``, prefix ``lstm_no_spark``), next to a
``params_settings`` text file and a ``train/`` events dir (original src/rnn.py:230,234-250,273-274;
original src/lstm-no-spark.py:182-202,230).

Layout reproduced here:
    <dir>/params_settings
    <dir>/checkpoint                       TF-style index: model_checkpoint_path + all_model_checkpoint_paths
    <dir>/<prefix>-<step>.index            json: variable name -> shape/dtype (human readable)
    <dir>/<prefix>-<step>.data-00000-of-00001   torch-serialised {name: tensor} keyed by the reference names
    <dir>/<prefix>-<step>.meta             json: step, flags, and (new) optimizer / RNG / data-iterator state file
    <dir>/train/                           TensorBoard events
The binary Saver-V2 bundle cannot be produced without TensorFlow; names + layout are the contract.
New vs reference: optimizer slots, step counter and loader state ARE saved (``.opt`` file) so ``--resume`` /
``--use_pretrained_model`` really resumes (the reference's restore branch is dead code, Q4).
"""
from __future__ import annotations

import glob
import json
import os
import re
from typing import Dict, List, Optional, Tuple

import torch

DATA_SUFFIX = ".data-00000-of-00001"


class Saver:
    def __init__(self, directory: str, prefix: str, max_to_keep: int = 5):
        self.dir = directory
        self.prefix = prefix
        self.max_to_keep = max_to_keep
        self.kept: List[str] = []
        os.makedirs(directory, exist_ok=True)

    # -----------------------------------------------------------------------------------------
    def write_params_settings(self, text: str):
        with open(os.path.join(self.dir, "params_settings"), "w+") as f:
            f.write(text)

    def _write_index_file(self):
        with open(os.path.join(self.dir, "checkpoint"), "w") as f:
            if self.kept:
                f.write(f'model_checkpoint_path: "{self.kept[-1]}"\n')
            for k in self.kept:
                f.write(f'all_model_checkpoint_paths: "{k}"\n')

    def save(self, variables: Dict[str, torch.Tensor], global_step: int, extra: Optional[dict] = None,
             opt_state: Optional[dict] = None) -> str:
        name = f"{self.prefix}-{global_step}"
        base = os.path.join(self.dir, name)
        torch.save(variables, base + DATA_SUFFIX)
        with open(base + ".index", "w") as f:
            json.dump({k: {"shape": list(v.shape), "dtype": str(v.dtype)} for k, v in variables.items()}, f, indent=1)
        meta = {"global_step": global_step, "prefix": self.prefix, "format": "torch", "has_opt_state": opt_state is not None}
        meta.update(extra or {})
        with open(base + ".meta", "w") as f:
            json.dump(meta, f, indent=1, default=str)
        if opt_state is not None:
            torch.save(opt_state, base + ".opt")
        if name in self.kept:
            self.kept.remove(name)
        self.kept.append(name)
        while len(self.kept) > self.max_to_keep:
            old = self.kept.pop(0)
            for p in glob.glob(os.path.join(self.dir, old + ".*")):
                os.remove(p)
        self._write_index_file()
        return base


def latest_checkpoint(directory: str) -> Optional[str]:
    """Parse the TF-style ``checkpoint`` index; returns the path prefix or None."""
    idx = os.path.join(directory, "checkpoint")
    if not os.path.isfile(idx):
        return None
    with open(idx) as f:
        for line in f:
            m = re.match(r'model_checkpoint_path:\s*"(.*)"', line.strip())
            if m:
                return os.path.join(directory, m.group(1))
    return None


def find_latest_run(checkpoint_path: str, rank_key: Optional[str]) -> Optional[str]:
    """Newest ``<checkpoint_path>/<ts>[/<rank_key>]`` that contains a checkpoint."""
    if not os.path.isdir(checkpoint_path):
        return None
    runs = []
    for d in os.listdir(checkpoint_path):
        try:
            ts = float(d)
        except ValueError:
            continue
        runs.append((ts, d))
    for _, d in sorted(runs, reverse=True):
        cand = os.path.join(checkpoint_path, d) if rank_key is None else os.path.join(checkpoint_path, d, rank_key)
        if latest_checkpoint(cand):
            return cand
    return None


def load(prefix_path: str) -> Tuple[Dict[str, torch.Tensor], dict, Optional[dict]]:
    variables = torch.load(prefix_path + DATA_SUFFIX, map_location="cpu", weights_only=False)
    with open(prefix_path + ".meta") as f:
        meta = json.load(f)
    opt = None
    if os.path.isfile(prefix_path + ".opt"):
        opt = torch.load(prefix_path + ".opt", map_location="cpu", weights_only=False)
    return variables, meta, opt


def recorded_settings(meta: dict) -> dict:
    """The flags a model file recorded: a training checkpoint keeps them under ``meta["config"]``, ``averaged_model.pt`` keeps
    the ones it records (``pooling``, ``vocab_size``, ``next_token``, ...) at the top level of its meta."""
    return meta.get("config") or meta


def save_averaged_model(output_path: str, records, variables: Dict[str, torch.Tensor], meta: dict):
    """Write the cross-replica average to ``--output_path`` (the reference computes it and throws it away,
    src/rnn.py:407-408, Q12).  ``records`` = the 8 keyed ``map_data_by_key`` entries."""
    os.makedirs(output_path, exist_ok=True)
    rec = {k: [[t.detach().cpu().clone() for t in layer] if isinstance(layer, (list, tuple)) else layer.detach().cpu().clone()
               for layer in v] for k, v in records}
    torch.save({"records": rec, "variables": variables, "meta": meta}, os.path.join(output_path, "averaged_model.pt"))
    with open(os.path.join(output_path, "averaged_model.json"), "w") as f:
        json.dump({"keys": [k for k, _ in records], **meta}, f, indent=1, default=str)
