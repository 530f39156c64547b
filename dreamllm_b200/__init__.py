"""dreamllm_b200 — H100-native (sm_90a) implementation of DreamLLM's data-parallel hot path.

Host side is Python/PyTorch (device memory, streams, torch.distributed); all arithmetic on the path runs in
hand-written CUDA behind the C ABI declared in include/dreamllm_sm100.h (libdreamllm_sm100.so).
"""
from . import _lib  # noqa: F401

__all__ = ["_lib"]
