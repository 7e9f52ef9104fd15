"""scail_b200 — Hopper-native (sm_90a) implementation of the SCAIL-14B denoising hot path.

Host code is Python/PyTorch (device memory, streams, torch.distributed); every per-step op is a
hand-written CUDA kernel in libscail_b200.so reached through the C ABI in include/scail_b200.h.
There is no CPU fallback: ops raise if the library or a CUDA device is missing.
"""
from . import _lib  # noqa: F401

__all__ = ["_lib"]
