"""H100-native shading pass of MomentsInGraphics/vulkan_renderer behind the reference's C host surface.

The product is libvkr_b200.so (hand-written sm_90a CUDA + C++ host code, C-ABI in include/vkr_b200.h; the names predate the port to H100).
This Python package is a thin ctypes mirror for tests and benchmarks. Importing it loads the library
and verifies that every symbol of the header is exported; it raises if the library was not built.
(VKR_B200_NO_AUTOLOAD=1 in the environment skips that: bench.py's reference arm, which only needs the
synthetic data sets of synth.py, runs without the product library in its process.)
"""
import os

from . import api
from .api import load_library

_lib = None if os.environ.get("VKR_B200_NO_AUTOLOAD") == "1" else load_library()

from .frame import Frame  # noqa: E402

__all__ = ["api", "load_library", "Frame"]
