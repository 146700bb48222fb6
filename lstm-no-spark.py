#!/usr/bin/env python
"""Standalone entry point (world_size = 1, CPU-capable): the counterpart of
original src/lstm-no-spark.py:261-288."""
import sys

from lstm_tensorspark_b200.config import parse_args
from lstm_tensorspark_b200.trainer import run_job


def main(argv):
    cfg = parse_args(argv[1:], standalone=True)
    print("Parameters:")
    print(cfg.params_str())
    run_job(cfg, standalone=True)


if __name__ == "__main__":
    main(sys.argv)
