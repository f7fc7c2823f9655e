"""Host-side helpers of the H100 Gaussian-splat rasterizer (scene synthesis, raw `_C` call helpers, multi-GPU slabs).

The drop-in API itself lives in the sibling package ``diff_gaussian_rasterization`` (same import name as the
reference's extension); the C ABI is ``librgs_b200.so`` in this directory (``include/rgs_b200.h``).
"""
import os as _os

PACKAGE_DIR = _os.path.dirname(_os.path.abspath(__file__))
LIB_PATH = _os.path.join(PACKAGE_DIR, "librgs_b200.so")
