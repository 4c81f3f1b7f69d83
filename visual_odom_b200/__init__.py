"""vo-b200: H100-native (sm_90a) implementation of the visual_odom hot path -- FAST corners, the four-way
pyramidal LK ring of circularMatching(), stereo triangulation and the PnP/RANSAC pose solve -- behind a C-ABI
(include/vo_b200.h, visual_odom_b200/libvo_b200.so).  `capi` is the ctypes binding; there is no CPU fallback:
`capi.load_library()` raises when the library has not been built and `capi.Context` raises without an H100."""
__all__ = ["capi", "synth", "dist", "build"]
