"""mnc_b200 -- H100-native implementation of the MNC (Multi-task Network Cascades) inference
hot path: sm_90a CUDA kernels behind a C-ABI (include/mnc_b200.h), with a host-side mirror of
the reference's Python layer / lib API (mnc_b200/lib)."""
__version__ = "0.1.0"
