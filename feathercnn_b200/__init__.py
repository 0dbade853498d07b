"""feathercnn_b200 — H100-native (sm_90a) CNN inference backend behind FeatherCNN's API.

The product is the native code: ``csrc/`` (hand-written CUDA kernels + the C ABI of ``include/fcuda.h``) and
``host/`` (C++ ``feather::Net``).  This Python package is a thin ctypes binding used by tests and bench.py;
importing it does not load the native libraries until the first call, and any call fails loudly if they are
missing (no CPU / PyTorch fallback).
"""
__all__ = ["booster", "net", "tools"]
