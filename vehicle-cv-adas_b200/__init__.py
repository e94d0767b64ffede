"""adas_b200 -- H100-native (sm_90a) per-frame ADAS inference path with the reference's
Python API surface (YoloDetector / UltrafastLaneDetectorV2 / BYTETracker, coreEngine protocol).

Host code is Python; all arithmetic on the hot path runs in hand-written CUDA kernels inside
libadas_b200.so (C ABI in include/adas_b200.h, bound in _capi.py).  There is no CPU fallback.
"""
__version__ = "0.1.0"
