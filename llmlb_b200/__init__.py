"""llmlb_b200 — H100-native in-process inference backend behind llmlb's endpoint boundary.

csrc/      CUDA kernels (sm_90a) + engine + C ABI  -> libllmlb_b200.so
ffi.py     ctypes binding of include/llmlb_b200.h
host/      gateway-side hot path (router, registry, SSE accounting) above the C ABI
"""
__all__ = ["ffi", "build"]
