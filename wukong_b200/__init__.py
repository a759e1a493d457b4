"""wukong_b200 — H100-native (sm_90a) graph-exploration engine behind Wukong's query/plan surface.

The product is native: CUDA kernels + a C ABI (include/wukong_b200.h) in libwukong_b200.so and a
C++ host layer (reference-surface mirror, store builder, data generators) in libwukong_host.so.
This Python package is only a ctypes veneer used by the tests and bench.py.  There is NO CPU
fallback: every compute entry point fails loudly if the CUDA library or a GPU is missing.
"""
from . import capi  # noqa: F401

__all__ = ["capi"]
