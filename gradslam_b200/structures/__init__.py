"""Containers of the hot path: batched RGB-D frames and capacity-backed surfel maps."""
from .pointclouds import Pointclouds
from .rgbdimages import RGBDImages
from . import structutils
from .structutils import list_to_padded, padded_to_list
from .utils import RenderedViews, pointclouds_from_rgbdimages, render_pointclouds

__all__ = ["Pointclouds", "RGBDImages", "pointclouds_from_rgbdimages", "render_pointclouds", "RenderedViews", "structutils",
           "list_to_padded", "padded_to_list"]
