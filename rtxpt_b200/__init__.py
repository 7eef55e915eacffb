"""rtxpt_b200 — CUDA-native (H100, sm_90a) wavefront path tracer behind RTXPT's PathTrace boundary.

The product is the C-ABI shared library built from rtxpt_b200/csrc (include/rtxpt_b200.h); this Python package only holds the
ctypes mirror of that ABI, the scene-table builder and the synthetic scenes used by tests and bench.py."""
from . import structs
