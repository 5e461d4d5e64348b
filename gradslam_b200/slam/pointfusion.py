"""PointFusion: ICPSLAM whose mapping step is confidence-weighted surfel fusion.

Host-side mirror of gradslam.slam.PointFusion (gradslam/slam/pointfusion.py:16-112): same keywords and
defaults (dist_th=0.05, angle_th=20, sigma=0.6), `dot_th = cos(angle_th)`.
"""
import math
import warnings
from typing import Optional, Union

import torch

from .. import _C
from ..structures.pointclouds import Pointclouds
from ..structures.rgbdimages import RGBDImages
from ..structures.pointclouds import _PruneHistory
from .fusionutils import _check_free_space_margin, _prune_scratch, fuse_and_prune, prune_unstable, update_map_fusion
from .icpslam import ICPSLAM

__all__ = ["PointFusion"]


class _SequenceWorkspace:
    """Scratch of gsx_pointfusion_sequence_gt (two frame workspaces used alternately), per (device, stream, B, H, W)."""

    _cache = {}

    def __init__(self, device, B, H, W):
        self.buf = torch.zeros(_C.lib().gsx_pointfusion_sequence_workspace_bytes(B, H, W), dtype=torch.uint8,
                               device=device)

    @classmethod
    def get(cls, device, B, H, W):
        key = (str(device), torch.cuda.current_stream(device).cuda_stream, B, H, W)
        if key not in cls._cache:
            cls._cache[key] = cls(device, B, H, W)
        return cls._cache[key]


class PointFusion(ICPSLAM):
    def __init__(self, *, odom: str = "gradicp", dist_th: Union[float, int] = 0.05,
                 angle_th: Union[float, int] = 20, sigma: Union[float, int] = 0.6, dsratio: int = 4,
                 numiters: int = 20, damp: float = 1e-8, dist_thresh: Union[float, int, None] = None,
                 lambda_max: Union[float, int] = 2.0, B: Union[float, int] = 1.0, B2: Union[float, int] = 1.0,
                 nu: Union[float, int] = 200.0, association: str = "nn",
                 device: Union[torch.device, str, None] = None, stable_confidence: Union[float, int, None] = None,
                 max_unstable_age: Optional[int] = None, free_space_margin: Union[float, int, None] = None):
        """stable_confidence, max_unstable_age (extension, give both or neither): after every map update, remove the
        surfels whose confidence is still below `stable_confidence` `max_unstable_age` frames after they were created
        (Keller et al. 2013, section 4.3).  Confidence is the map's `features_padded` value - gradslam's alpha,
        clamp(exp(-|v|^2 / 2 sigma^2), 1e-7, 1.01) of the camera-frame vertex, summed over merges - so a good threshold
        depends on the scene's depth range and on sigma; there is no universal default.  max_unstable_age = 0 tests each
        surfel in the frame that creates it.  Default: nothing is removed (gradslam's behaviour).

        free_space_margin (extension, metres >= 0, inf allowed; needs stable_confidence and max_unstable_age): in the same
        step, also remove the free-space violations of Keller et al. 2013, section 4.3 - wherever the live frame merged
        a pixel into a surfel that is stable after the merge, every surfel projecting to that pixel more than the margin
        (camera z) in front of it.  The paper finds "in front" on a 4x4-supersampled index map; here it is the merged
        pixel itself, at image resolution.  Default None: no such removal."""
        for name, val, kinds in (("stable_confidence", stable_confidence, (float, int)),
                                 ("max_unstable_age", max_unstable_age, (int,))):
            if val is not None and (isinstance(val, bool) or not isinstance(val, kinds)):
                raise TypeError("{} must be of type {}; but was of type {}.".format(
                    name, " or ".join(k.__name__ for k in kinds), type(val)))
        if (stable_confidence is None) != (max_unstable_age is None):
            raise ValueError("give both stable_confidence and max_unstable_age, or neither")
        if stable_confidence is not None and not stable_confidence >= 0:
            raise ValueError("stable_confidence ({}) must be >= 0".format(stable_confidence))
        if max_unstable_age is not None and max_unstable_age < 0:
            raise ValueError("max_unstable_age ({}) must be >= 0".format(max_unstable_age))
        if free_space_margin is not None:
            _check_free_space_margin(free_space_margin)
            if stable_confidence is None:
                raise ValueError("free_space_margin needs stable_confidence and max_unstable_age")
        super().__init__(odom=odom, dsratio=dsratio, numiters=numiters, damp=damp, dist_thresh=dist_thresh,
                         lambda_max=lambda_max, B=B, B2=B2, nu=nu, association=association, device=device)
        if not isinstance(dist_th, (float, int)):
            raise TypeError("Distance threshold must be of type float or int; but was of type {}.".format(
                type(dist_th)))
        if not isinstance(angle_th, (float, int)):
            raise TypeError("Angle threshold must be of type float or int; but was of type {}.".format(
                type(angle_th)))
        if dist_th < 0:
            warnings.warn("Distance threshold ({}) should be non-negative.".format(dist_th))
        if not ((0 <= angle_th) and (angle_th <= 90)):
            warnings.warn("Angle threshold ({}) should be non-negative and <=90.".format(angle_th))
        self.dist_th = dist_th
        self.dot_th = math.cos((angle_th * math.pi) / 180)
        self.sigma = sigma
        self.stable_confidence = stable_confidence
        self.max_unstable_age = max_unstable_age
        self.free_space_margin = free_space_margin

    def _map(self, pointclouds: Pointclouds, live_frame: RGBDImages, inplace: bool = False):
        if self.stable_confidence is not None and isinstance(pointclouds, Pointclouds):
            if pointclouds._prune is not None and pointclouds._prune.t_max != self.max_unstable_age:
                raise ValueError("max_unstable_age ({}) differs from the one this map was pruned with ({})".format(
                    self.max_unstable_age, pointclouds._prune.t_max))
        if self.free_space_margin is not None:
            return fuse_and_prune(pointclouds, live_frame, self.dist_th, self.dot_th, self.sigma, self.stable_confidence,
                                  self.max_unstable_age, self.free_space_margin, inplace)
        pointclouds = update_map_fusion(pointclouds, live_frame, self.dist_th, self.dot_th, self.sigma, inplace)
        if self.stable_confidence is not None:
            prune_unstable(pointclouds, self.stable_confidence, self.max_unstable_age)
        return pointclouds

    def forward(self, frames, out=None):
        """As ICPSLAM.forward; additionally accepts a `gradslam_b200.ingest.RawRGBD` batch (uint8 colour + uint16 depth)
        when odom='gt': the raw frames are uploaded and converted on the device, overlapped with the fusion."""
        from ..ingest import RawRGBD

        if isinstance(frames, RawRGBD):
            if self.odom != "gt" or frames.poses is None:
                raise ValueError("RawRGBD input is supported for odom='gt' with poses; convert with "
                                 "ingest.rgbdimages_from_raw for the other odometry modes")
            self._check_out(out, frames.shape[0])
            return self._forward_sequence(frames, raw=True, out=out)
        return super().forward(frames, out)

    def _forward_sequence(self, frames, chunk: int = 4, raw: bool = False, out=None):
        """odom='gt': the whole (B, L) sequence runs as C calls chaining K1 -> K2/K3 -> K4 per frame with no
        host synchronisation.  Frames that live in HOST memory are uploaded `chunk` frames at a time on a side
        stream, so the copy of chunk i+1 overlaps the fusion of chunk i (pin the host tensors for this)."""
        if self.odom != "gt" or frames.poses is None or torch.is_tensor(self.sigma):
            return None
        dev = self.device
        if raw:
            B, L, H, W = frames.shape
            src_depth, src_rgb = frames.depths, frames.colors
            if src_depth.device == dev:  # already uploaded: convert in one go
                from ..ingest import raw_to_float

                rgb_f, depth_f = raw_to_float(src_rgb, src_depth, frames.scaling_factor, frames.normalize_color)
                return self._forward_sequence(RGBDImages(rgb_f, depth_f, frames.intrinsics.to(dev),
                                                         frames.poses.to(dev)), out=out)
            on_device = False
        else:
            if torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in (
                    frames.depth_image, frames.rgb_image, frames.poses, frames.intrinsics)):
                return None  # differentiable mode goes through the per-frame step loop
            if frames.channels_first:
                frames = frames.to_channels_last()
            B, L, H, W = frames.shape
            src_depth, src_rgb = frames.depth_image, frames.rgb_image
            on_device = src_depth.device == dev
        P = H * W
        K = frames.intrinsics.to(dev).contiguous()
        poses = frames.poses.to(dev).contiguous()
        if on_device:
            depth, rgb = src_depth.contiguous(), src_rgb.contiguous()
            chunk = L
        else:
            depth = torch.empty((B, L, H, W, 1), dtype=torch.float32, device=dev)
            rgb = torch.empty((B, L, H, W, 3), dtype=torch.float32, device=dev)
            copy_stream = torch.cuda.Stream(device=dev)
            if raw:  # staging buffers for the 5-byte pixels; converted chunk by chunk on the compute stream
                raw_depth = torch.empty((B, L, H, W), dtype=src_depth.dtype, device=dev)
                raw_rgb = torch.empty((B, L, H, W, 3), dtype=torch.uint8, device=dev)
        for t, name in ((depth, "depth_image"), (rgb, "rgb_image"), (K, "intrinsics"), (poses, "poses")):
            _C.require_cuda(t, name)
        if out is not None:  # caller-provided storage (validated by forward: empty, B maps, this device)
            if not (out.has_normals and out.has_colors and out._has_cc):
                raise ValueError("out must have normals, colours and a confidence count per point for map fusion")
            pc = out
            pc._cur = 0
        else:
            pc = Pointclouds(device=dev)
            pc._allocate(B, L * P, 1, zero=False)
        ws = _SequenceWorkspace.get(dev, B, H, W)
        if self.stable_confidence is not None:  # a fresh map: frame s of the call is pruned step s
            pc._prune = hist = _PruneHistory.fresh(B, self.max_unstable_age, dev)
            prune_scratch = _prune_scratch(B, pc.capacity, dev)
            if self.free_space_margin is not None:
                fs_scratch = torch.empty(_C.lib().gsx_fusion_free_space_scratch_bytes(B, H, W, pc.capacity),
                                         dtype=torch.uint8, device=dev)
        main = torch.cuda.current_stream(dev)
        ready = []
        if not on_device:
            copy_stream.wait_stream(main)  # the fresh buffers must exist before the copies start
            with torch.cuda.stream(copy_stream):
                for s0 in range(0, L, chunk):
                    s1 = min(L, s0 + chunk)
                    dst_d, dst_c = (raw_depth, raw_rgb) if raw else (depth, rgb)
                    for b in range(B):  # per-element slices are contiguous: true async DMA from pinned memory
                        dst_d[b, s0:s1].copy_(src_depth[b, s0:s1], non_blocking=True)
                        dst_c[b, s0:s1].copy_(src_rgb[b, s0:s1], non_blocking=True)
                    ev = torch.cuda.Event()
                    ev.record(copy_stream)
                    ready.append(ev)
        for i, s0 in enumerate(range(0, L, chunk)):
            s1 = min(L, s0 + chunk)
            if ready:
                main.wait_event(ready[i])
            if raw:  # u8 / u16 -> float32 for this chunk (per element: the chunk is contiguous inside an element)
                for b in range(B):
                    _C.launch("gsx_ingest_raw", raw_rgb[b, s0:s1], raw_depth[b, s0:s1], (s1 - s0) * P,
                              frames.scaling_factor, 1 if frames.normalize_color else 0, rgb[b, s0:s1], depth[b, s0:s1])
            if self.stable_confidence is None:
                _C.launch("gsx_pointfusion_sequence_gt", pc._geo, pc._col, pc._counts_dev, pc.capacity,
                          min(s0 * P, pc.capacity), depth, rgb, K, poses, B, L, s0, s1, H, W, float(self.dist_th),
                          float(self.dot_th), float(self.sigma), ws.buf, pc._overflow_flag())
            elif self.free_space_margin is not None:
                _C.launch("gsx_pointfusion_sequence_gt_prune_free_space", pc._geo, pc._col, pc._counts_dev, pc.capacity,
                          min(s0 * P, pc.capacity), depth, rgb, K, poses, B, L, s0, s1, H, W, float(self.dist_th),
                          float(self.dot_th), float(self.sigma), ws.buf, hist.ring, self.max_unstable_age,
                          float(self.stable_confidence), prune_scratch, prune_scratch.numel(),
                          float(self.free_space_margin), fs_scratch, fs_scratch.numel(), pc._overflow_flag())
            else:
                _C.launch("gsx_pointfusion_sequence_gt_prune", pc._geo, pc._col, pc._counts_dev, pc.capacity,
                          min(s0 * P, pc.capacity), depth, rgb, K, poses, B, L, s0, s1, H, W, float(self.dist_th),
                          float(self.dot_th), float(self.sigma), ws.buf, hist.ring, self.max_unstable_age,
                          float(self.stable_confidence), prune_scratch, prune_scratch.numel(), pc._overflow_flag())
        if not on_device:
            for t in ((raw_depth, raw_rgb) if raw else (depth, rgb)):
                t.record_stream(copy_stream)
        pc._cur = L & 1
        pc._counts_host = None
        pc._bound = pc.capacity
        pc._list_cache = {}
        pc._tail_dirty = pc._uninit
        if self.stable_confidence is not None:  # rows past the pruned sizes hold stale values
            hist.step = L
            pc._uninit = pc._tail_dirty = True
        return pc, poses.clone()
