"""mqdet_b200 — H100-native (sm_90a) implementation of MQ-Det's multi-modal query forward pass.

Host code is Python/PyTorch plumbing over hand-written CUDA kernels behind a C ABI (include/mqdet_b200.h,
mqdet_b200/csrc).  The module tree mirrors the slice of ``maskrcnn_benchmark.modeling`` on the hot path
(SURVEY.md §8b) with the reference's class names, constructor arguments, parameter names and forward signatures.
"""
from . import _lib, ops  # noqa: F401

__all__ = ["_lib", "ops"]
