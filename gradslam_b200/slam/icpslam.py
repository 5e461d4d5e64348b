"""ICPSLAM: point-based SLAM driver — localise each live frame, then aggregate it into the map.

Host-side mirror of gradslam.slam.ICPSLAM (gradslam/slam/icpslam.py:16-264): same constructor keywords and
defaults, `forward(frames) -> (Pointclouds, poses[B,L,4,4])`, `step(pointclouds, live_frame, prev_frame,
inplace)`.  The per-frame work runs in the sm_90a kernels of libgsx; with `odom='gt'` a whole sequence is
one C call (gsx_pointfusion_sequence_gt) with no host synchronisation between frames.
"""
import warnings
from typing import Optional, Union

import torch
import torch.nn as nn

from ..structures.pointclouds import Pointclouds
from ..structures.rgbdimages import RGBDImages
from .fusionutils import update_map_aggregate

__all__ = ["ICPSLAM"]


def _compose_canonical(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """a · b for rigid (..., 4, 4) transforms in the canonical order of the fused step's k_pose_compose: every entry is
    (a_i0 b_0j + a_i1 b_1j) + a_i2 b_2j (+ a_i3 in the last column), each product and sum rounded on its own.  A
    matmul may fuse or reorder these (cuBLAS does, at some batch sizes), so the differentiable step composes with
    separate elementwise ops and returns the fused step's poses bit for bit.  The bottom row is [0, 0, 0, 1]."""
    p = [a[..., :3, k:k + 1] * b[..., k:k + 1, :] for k in range(3)]
    top = (p[0] + p[1]) + p[2]
    top = torch.cat([top[..., :3], top[..., 3:] + a[..., :3, 3:]], -1)
    bottom = torch.tensor([0.0, 0.0, 0.0, 1.0], dtype=a.dtype, device=a.device).expand(*a.shape[:-2], 1, 4)
    return torch.cat([top, bottom], -2)


def _normalize_device(device):
    """torch.device with an explicit index for CUDA (the engine's default device is CUDA, not CPU)."""
    device = torch.device(device)
    if device.type == "cuda" and device.index is None:
        device = torch.device("cuda", torch.cuda.current_device() if torch.cuda.is_available() else 0)
    return device


class ICPSLAM(nn.Module):
    def __init__(self, *, odom: str = "gradicp", dsratio: int = 4, numiters: int = 20, damp: float = 1e-8,
                 dist_thresh: Union[float, int, None] = None, lambda_max: Union[float, int] = 2.0,
                 B: Union[float, int] = 1.0, B2: Union[float, int] = 1.0, nu: Union[float, int] = 200.0,
                 association: str = "nn", device: Union[torch.device, str, None] = None):
        """association (extension): how the ICP odometry pairs live points with the map.  'nn' (default, the
        reference's) = exact 1-NN between the lattice-thinned live cloud and the lattice-active map points; 'projective'
        = each live point with the map row visible at the pixel it projects to in the map rendered from the previous
        pose (Keller et al.'s PointFusion, KinectFusion).  The two give different poses.  No effect with odom='gt'."""
        super().__init__()
        if not isinstance(association, str):
            raise TypeError("Expected association to be of type str. Got {0}.".format(type(association)))
        if association not in ("nn", "projective"):
            raise ValueError("association must be 'nn' or 'projective'. Got {!r}.".format(association))
        if odom not in ["gt", "icp", "gradicp"]:
            msg = "odometry method ({}) not supported for PointFusion. ".format(odom)
            msg += "Currently supported odometry modules for PointFusion are: 'gt', 'icp', 'gradicp'"
            raise ValueError(msg)
        odomprov = None
        if odom == "icp":
            from ..odometry.icp import ICPOdometryProvider

            odomprov = ICPOdometryProvider(numiters, damp, dist_thresh)
        elif odom == "gradicp":
            from ..odometry.gradicp import GradICPOdometryProvider

            odomprov = GradICPOdometryProvider(numiters, damp, dist_thresh, lambda_max, B, B2, nu)
        self.odom = odom
        self.odomprov = odomprov
        self.dsratio = dsratio
        self.association = association
        self.device = _normalize_device(device if device is not None else "cuda")

    # ------------------------------------------------------------------ sequence driver
    def forward(self, frames: RGBDImages, out: Optional[Pointclouds] = None):
        """Builds the maps from a (B, L) batch of sequences.  Returns (Pointclouds, poses (B,L,4,4)).
        out (extension): EMPTY maps with pre-allocated row storage that receive the result in place - e.g. this rank's
        block of a job-wide store, `parallel.GatheredMaps(...).local`.  Give it room for L*H*W rows per sequence: a map
        that outgrows its storage is re-allocated elsewhere (step loop) or reports the overflow (sequence call)."""
        if not isinstance(frames, RGBDImages):
            raise TypeError("Expected frames to be of type gradslam.RGBDImages. Got {0}.".format(type(frames)))
        batch_size, seq_len = frames.shape[:2]
        self._check_out(out, batch_size)
        pointclouds = out if out is not None else Pointclouds(device=self.device)
        fast = self._forward_sequence(frames, out=out)
        if fast is not None:
            return fast
        recovered_poses = torch.empty(batch_size, seq_len, 4, 4, device=self.device)
        prev_frame = None
        for s in range(seq_len):
            live_frame = frames[:, s].to(self.device)
            if s == 0 and live_frame.poses is None:
                live_frame.poses = torch.eye(4, dtype=torch.float, device=self.device).view(1, 1, 4, 4).repeat(
                    batch_size, 1, 1, 1)
            pointclouds, live_frame.poses = self.step(pointclouds, live_frame, prev_frame, inplace=True)
            prev_frame = live_frame if self.odom != "gt" else None
            recovered_poses[:, s] = live_frame.poses[:, 0]
        return pointclouds, recovered_poses

    def _check_out(self, out, batch_size):
        if out is None:
            return
        if not isinstance(out, Pointclouds):
            raise TypeError("Expected out to be of type gradslam.Pointclouds. Got {0}.".format(type(out)))
        if out.device != self.device or not out.has_points or len(out) != batch_size:
            raise ValueError("out must hold %d pre-allocated maps on %s" % (batch_size, self.device))
        if any(out._host_counts()):
            raise ValueError("out must be empty (the maps are built from scratch)")

    def _forward_sequence(self, frames, out=None):
        """Hook for single-call whole-sequence drivers (PointFusion with odom='gt'); None = use the step loop."""
        return None

    def step(self, pointclouds: Pointclouds, live_frame: RGBDImages, prev_frame: Optional[RGBDImages] = None,
             inplace: bool = False):
        """One SLAM step on `live_frame` (sequence length 1).  Returns (Pointclouds, poses (B,1,4,4))."""
        if not isinstance(live_frame, RGBDImages):
            raise TypeError("Expected live_frame to be of type gradslam.RGBDImages. Got {0}.".format(type(live_frame)))
        live_frame.poses = self._localize(pointclouds, live_frame, prev_frame)
        pointclouds = self._map(pointclouds, live_frame, inplace)
        return pointclouds, live_frame.poses

    def _localize(self, pointclouds: Pointclouds, live_frame: RGBDImages, prev_frame: RGBDImages):
        if not isinstance(pointclouds, Pointclouds):
            raise TypeError("Expected pointclouds to be of type gradslam.Pointclouds. Got {0}.".format(
                type(pointclouds)))
        if not isinstance(live_frame, RGBDImages):
            raise TypeError("Expected live_frame to be of type gradslam.RGBDImages. Got {0}.".format(type(live_frame)))
        if not isinstance(prev_frame, (RGBDImages, type(None))):
            raise TypeError("Expected prev_frame to be of type gradslam.RGBDImages or None. Got {0}.".format(
                type(prev_frame)))
        if prev_frame is not None:
            if self.odom == "gt":
                warnings.warn("`prev_frame` is not used when using `odom='gt'` (should be None)")
            elif not prev_frame.has_poses:
                raise ValueError("`prev_frame` should have poses, but did not.")
        if prev_frame is None and pointclouds.has_points and self.odom != "gt":
            warnings.warn("`prev_frame` was None despite `{}` odometry method. Using `live_frame` poses.".format(
                self.odom))
        if prev_frame is None or self.odom == "gt":
            if not live_frame.has_poses:
                raise ValueError("`live_frame` must have poses when `prev_frame` is None or `odom='gt'`.")
            return live_frame.poses

        from ..odometry.icputils import _wants_grad, downsample_pointclouds, downsample_rgbdimages, localize_against_map

        live_frame.poses = prev_frame.poses
        wants_grad = _wants_grad(live_frame.depth_image, prev_frame.poses, *pointclouds._grad_tensors())
        if self.association == "projective":
            from ..odometry.icputils import localize_projective, localize_projective_taped

            if not pointclouds.has_normals:
                raise ValueError("projective ICP association needs a map with normals")
            fn = localize_projective_taped if wants_grad else localize_projective
            return fn(pointclouds, live_frame, prev_frame, self.dsratio, self.odomprov)
        if wants_grad:
            # differentiable mode (reference op order, slam/icpslam.py:238-247): the K1 maps carry their hand-written
            # backward, the association kernels are index-only, the ICP algebra is taped.
            from .fusionutils import find_active_map_points

            frames_pc = downsample_rgbdimages(live_frame, self.dsratio)
            pc2im_bnhw = find_active_map_points(pointclouds, prev_frame)
            maps_pc = downsample_pointclouds(pointclouds, pc2im_bnhw, self.dsratio)
            transform = self.odomprov.provide(maps_pc, frames_pc)
            return _compose_canonical(transform.squeeze(1), prev_frame.poses.squeeze(1)).unsqueeze(1)
        # source / target gathering, the ICP loop and the final T_icp · prev_pose all happen in one C call
        return localize_against_map(pointclouds, live_frame, prev_frame, self.dsratio, self.odomprov)

    def _map(self, pointclouds: Pointclouds, live_frame: RGBDImages, inplace: bool = False):
        return update_map_aggregate(pointclouds, live_frame, inplace)
