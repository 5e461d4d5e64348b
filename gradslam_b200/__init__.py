"""gradslam_b200 — a Hopper (sm_90a) engine for gradslam's PointFusion / ICPSLAM inner loop.

Drop-in for the hot path of gradslam/gradslam: `RGBDImages`, `Pointclouds`, `PointFusion`, `ICPSLAM`, the
odometry providers and the `fusionutils` / `icputils` functions keep the reference's names, arguments and
error behaviour; the arithmetic runs in hand-written CUDA kernels behind the C ABI of include/gsx.h.
"""
from .version import __version__
from .structures import *  # noqa: F401,F403  (Pointclouds, RGBDImages, structutils helpers - as gradslam/__init__.py)
from .structures import (BilateralFilter, Pointclouds, RGBDImages, RenderedViews, bilateral_filter_depth,
                         pointclouds_from_rgbdimages, render_pointclouds)
from .geometry import *  # noqa: F401,F403  (project_points, inverse_intrinsics, se3_exp, ... at the top level)
from . import geometry, ingest, odometry, slam
from .slam import ICPSLAM, PointFusion
