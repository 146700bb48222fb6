"""lstm_tensorspark_b200 — a Blackwell-native distributed LSTM trainer with the capabilities, CLI and
checkpoint layout of EmanuelOverflow/LSTM-TensorSpark."""
__version__ = "0.1.0"

from .config import Config, parse_args          # noqa: F401

import os as _os

# Kernels of the layer wavefront wait for each other on the device; lazy module loading could serialise the first launches
# behind running kernels.  Only effective when set before the CUDA context exists (ops/cuda_lstm.py also warms the kernels up).
_os.environ.setdefault("CUDA_MODULE_LOADING", "EAGER")
