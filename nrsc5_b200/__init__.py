"""nrsc5_b200 — H100-native NRSC-5 FM physical-layer receive engine.

The product is `libnrsc5_b200.so` (hand-written sm_90a CUDA behind the C ABI
in include/nrsc5_b200.h).  This package is the thin Python host-side mirror of
that ABI (ctypes), plus the synthetic-capture generator used by bench/tests.
"""
from .engine import Engine, EngineError, lib_path, load_library  # noqa: F401
