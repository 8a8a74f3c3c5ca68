"""detectandtrack_b200 — H100 (sm_90a) hot path behind the DetectAndTrack
cfg / model-builder / tools surface.  Host code is Python mirroring the
reference's module names (core/, modeling/, ops/, utils/); the arithmetic runs in
hand-written CUDA through the C ABI in include/dt_b200.h (``_lib``).  There is
no CPU fallback: every op raises if libdt_b200.so or a CUDA device is missing.
"""
__version__ = '0.1.0'
