"""gradICP odometry provider (mirror of gradslam/odometry/gradicp.py:11-122)."""
from typing import Union

import torch

from ..structures.pointclouds import Pointclouds
from .base import OdometryProvider
from .icp import _check_provide_args, _provide
from .icputils import _check_huber_delta

__all__ = ["GradICPOdometryProvider"]


class GradICPOdometryProvider(OdometryProvider):
    def __init__(self, numiters: int = 20, damp: float = 1e-8, dist_thresh: Union[float, int, None] = None,
                 lambda_max: Union[float, int] = 2.0, B: Union[float, int] = 1.0, B2: Union[float, int] = 1.0,
                 nu: Union[float, int] = 200.0, *, huber_delta: Union[float, int, None] = None):
        """huber_delta (extension, metres, None = off): Huber-weighted point-to-plane residuals, as in
        ICPOdometryProvider, inside the gradLM loop."""
        _check_huber_delta(huber_delta)
        for name, v in (("lambda_max", lambda_max), ("B", B), ("B2", B2), ("nu", nu)):
            if not isinstance(v, (float, int)):
                raise TypeError("Expected {} to be of type float or int; got {}".format(name, type(v)))
        self.numiters = numiters
        self.damp = damp
        self.dist_thresh = dist_thresh
        self.huber_delta = huber_delta
        self.lambda_max = lambda_max
        self.B = B
        self.B2 = B2
        self.nu = nu

    def provide(self, maps_pointclouds: Pointclouds, frames_pointclouds: Pointclouds) -> torch.Tensor:
        """Transforms (B,1,4,4) aligning each frame cloud to its map cloud with the gradLM solver."""
        _check_provide_args(maps_pointclouds, frames_pointclouds, "GradICPOdometryProvider")
        return _provide(self, maps_pointclouds, frames_pointclouds, 1)
