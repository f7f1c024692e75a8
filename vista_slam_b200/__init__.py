"""H100-native (sm_90a) implementation of ViSTA-SLAM's STA frontend forward pass.

Only the hot path lives here: hand-written CUDA kernels behind a C ABI (csrc/, include/sta_b200.h)
and the host-side mirror of the reference module surface (sta_model/).
"""
__all__ = ["build", "_lib"]
