"""iggt_official_b200 -- Hopper-native (H100, sm_90a) implementation of the IGGT multi-view inference hot path.

Public surface mirrors the reference (`iggt.models.vggt.IGGT` / `VGGT`, `forward(images, query_points=None)`,
same `state_dict` layout); the math runs in hand-written CUDA kernels behind the C ABI in include/iggt_b200.h.
"""
__version__ = "0.1.0"
