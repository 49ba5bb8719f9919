"""cube_slam_b200 -- H100-native (sm_90a) front end for CubeSLAM's per-frame cuboid proposal path.

The product is the C-ABI shared library cube_slam_b200/lib/libcubeslam_b200.so (include/cube_slam_b200.h).
This package holds the CUDA sources (csrc/), the in-tree build (build.py) and a thin host-side mirror of
the reference's C++ interface for this path (detect_3d_cuboid.py, line_lbd.py).
"""
from . import _lib  # noqa: F401
from ._lib import CUBOID_DTYPE  # noqa: F401
from .detect_3d_cuboid import (Context, CubeSlamError, cuboid, cuboid_draw_edges, cuboid_measurement, default_params, detect_3d_cuboid,  # noqa: F401
                               plot_image_with_cuboid)
from .line_lbd import BinaryDescriptorMatcher, LSDDetector, line_lbd_detect  # noqa: F401

__all__ = ["BinaryDescriptorMatcher", "Context", "LSDDetector", "CubeSlamError", "cuboid", "cuboid_draw_edges", "cuboid_measurement", "default_params", "detect_3d_cuboid", "line_lbd_detect",
           "plot_image_with_cuboid"]
