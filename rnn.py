#!/usr/bin/env python
"""Distributed entry point: ``python rnn.py --training_path dataset/iris.data --partitions 4 ...``
(replaces ``spark-submit rnn.py ...`` of the reference, original src/rnn.py:339-414, README.md:40).
One rank per partition / GPU; also runs under torchrun."""
import sys

from lstm_tensorspark_b200.config import parse_args
from lstm_tensorspark_b200.trainer import run_job


def main(argv):
    cfg = parse_args(argv[1:], standalone=False)
    if not cfg.quiet:
        print("Parameters:")
        print(cfg.params_str())
    run_job(cfg, standalone=False)


if __name__ == "__main__":
    main(sys.argv)
