"""x265_b200 -- H100-native (sm_90a) block-primitive engine behind x265's EncoderPrimitives table.

The product is libx265cu.so (C ABI in include/x265_b200.h).  This package is the thin Python host
mirror used by tests and bench.py: it loads the library with ctypes and exposes the per-call table
and the batched API on numpy arrays / raw device pointers.  There is no CPU fallback: importing
works without a GPU (so the build can be checked), but every compute entry point raises without CUDA.
"""
from .lib import Lib, load, DeviceBuffer, CudaUnavailable, Analyser  # noqa: F401
