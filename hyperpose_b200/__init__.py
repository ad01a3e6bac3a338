"""hyperpose_b200 -- H100-native replacement of HyperPose's inference hot path.

The product is `libhyperpose_b200.so` (CUDA, sm_90a) behind the C ABI of
`include/hyperpose_b200.h`; `capi` is its ctypes binding, `synthetic` the seeded input
generators used by tests and bench.  Nothing here imports `oracle/`.
"""
__all__ = ["capi", "synthetic", "build"]
