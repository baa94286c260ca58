"""nersemble_b200 -- H100-native (sm_90a) render hot path for NeRSemble.

Python host code mirroring the reference's nerfstudio plugin surface
(src/nersemble/nerfstudio/**) over a C-ABI CUDA library (libnsb.so, include/nsb.h).
There is NO CPU fallback: every op raises if the CUDA library or a GPU is missing.
"""
__version__ = "0.1.0"
