"""ezrt_b200 -- H100-native (sm_90a CUDA) drop-in for EzRT's path-tracing hot path.

Host mirror of the reference's main()/display() (P5/main.cpp) on top of the C ABI in
include/ezrt.h.  The package holds only what the path needs: csrc/ (CUDA kernels, C ABI,
host scene pipeline), api.py (ctypes mirror), scenes.py (synthetic benchmark scenes),
dist.py (image-tile partition across GPUs + the single framebuffer gather).
"""
from .api import *  # noqa: F401,F403
from .api import (Material, RenderConfig, Scene, TriangleList, camera_orbit, hdr_cache, hdr_load,  # noqa: F401
                  transform_matrix)
