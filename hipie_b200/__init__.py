"""hipie_b200 — H100-native (sm_90a) implementation of HIPIE's inference hot path.

Host side mirrors the reference's detectron2 / HIPIE operator interfaces; all hot ops go through the
C-ABI shared library `libhipie_b200.so` (include/hipie_b200.h).  There is no CPU fallback: calling an
op without the built library or without a CUDA device raises.
"""
__version__ = "0.1.0"
