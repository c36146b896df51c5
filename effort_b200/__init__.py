"""effort_b200 -- H100-native (sm_90a) implementation of kolinko/effort's bucketMul hot path.

Only what the path needs lives here: csrc/ (CUDA kernels + the C-ABI of include/effort_b200.h) and the
host-side mirror of the reference's operator interface (ops.py).  Importing the package does not touch
CUDA; the first operator call loads libeffort_b200.so and raises if it is missing (no CPU fallback).
"""
from ._lib import EffortError, lib_path, load  # noqa: F401

__all__ = ["EffortError", "lib_path", "load"]
