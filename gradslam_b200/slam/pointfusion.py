"""PointFusion: ICPSLAM whose mapping step is confidence-weighted surfel fusion.

Host-side mirror of gradslam.slam.PointFusion (gradslam/slam/pointfusion.py:16-112): same keywords and
defaults (dist_th=0.05, angle_th=20, sigma=0.6), `dot_th = cos(angle_th)`.
"""
import math
import warnings
from typing import Optional, Union

import torch

from .. import _C
from ..structures.pointclouds import EMBED_DTYPES, Pointclouds
from ..structures.rgbdimages import BilateralFilter, RGBDImages
from ..structures.pointclouds import _PruneHistory
from .fusionutils import (_check_free_space_margin, _check_history, _check_merge_overlapping, _prune_scratch,
                          fuse_and_prune, prune_unstable, update_map_fusion)
from .icpslam import ICPSLAM

__all__ = ["PointFusion"]


class _SequenceWorkspace:
    """Scratch of gsx_pointfusion_sequence_gt (one frame workspace and a block of frame headers, re-armed by every
    call), per (device, stream, B, H, W)."""

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
                 max_unstable_age: Optional[int] = None, free_space_margin: Union[float, int, None] = None,
                 surfel_radii: bool = False, merge_overlapping: bool = False, target_splat_px: int = 0,
                 photometric_weight: Union[float, int] = 0.0, depth_filter: Optional[BilateralFilter] = None,
                 depth_filter_tracking_only: bool = False, huber_delta: Union[float, int, None] = None,
                 photometric_huber_delta: Union[float, int, None] = None):
        """huber_delta, photometric_huber_delta (extension, None = off): Huber-weighted tracking residuals, as in
        ICPSLAM.

        stable_confidence, max_unstable_age (extension, give both or neither): after every map update, remove the
        surfels whose confidence is still below `stable_confidence` `max_unstable_age` frames after they were created
        (Keller et al. 2013, section 4.3).  Confidence is the map's `features_padded` value - gradslam's alpha,
        clamp(exp(-|v|^2 / 2 sigma^2), 1e-7, 1.01) of the camera-frame vertex, summed over merges - so a good threshold
        depends on the scene's depth range and on sigma; there is no universal default.  max_unstable_age = 0 tests each
        surfel in the frame that creates it.  Default: nothing is removed (gradslam's behaviour).

        free_space_margin (extension, metres >= 0, inf allowed; needs stable_confidence and max_unstable_age): in the same
        step, also remove the free-space violations of Keller et al. 2013, section 4.3 - wherever the live frame merged
        a pixel into a surfel that is stable after the merge, every surfel projecting to that pixel more than the margin
        (camera z) in front of it.  The paper finds "in front" on a 4x4-supersampled index map; here it is the merged
        pixel itself, at image resolution.  Default None: no such removal.

        surfel_radii (extension, default False): every fused surfel also gets a radius (`radii_padded`), as
        fusionutils.update_map_fusion(surfel_radii=True) gives it, in the whole-sequence call, the step API, the
        differentiable mode and with pruning.  Nothing else in the map changes.

        merge_overlapping (extension, default False; needs surfel_radii=True, stable_confidence and max_unstable_age): in
        every pruned step, also merge overlapping surfels (Keller et al. 2013, section 4.3, the third rule), as
        fusionutils.fuse_and_prune(merge_overlapping=True) does: a surfel that projects to a pixel the live frame merged
        into a stable surfel, with a similar normal (dot > cos(angle_th)) and a disk that overlaps the stable surfel's,
        is folded into it (confidence-weighted mean) and removed; one per pixel, the closest.  Without
        free_space_margin no free-space violation is removed.  stable_confidence=0 makes the age rule a no-op (every
        surfel is stable), so merging can run alone; the stable surfels are then every surfel the frame merged into.

        target_splat_px (extension, default 0; > 0 needs association='projective' and surfel_radii=True): track against
        the map rendered with its surfels as oriented disks, see ICPSLAM.

        photometric_weight (extension, default 0; > 0 needs association='projective'): joint geometric and photometric
        tracking against the map's colours, see ICPSLAM.

        Frames with embeddings (RGBDImages(embeddings=...)) give maps with per-surfel embeddings, merged with the
        colours' weights, on every path; the pruning options (stable_confidence, free_space_margin, merge_overlapping)
        refuse them with ValueError.  With RGBDImages(..., upsample_embeddings=True) the embedding image may be coarser
        than the depth and is upsampled bilinearly where it is fused; the whole-sequence call then uploads only the
        coarse images.

        depth_filter, depth_filter_tracking_only (extension; default None, False): bilateral filtering of the live depth
        for the tracking and the fusion, or for the tracking alone, see ICPSLAM.  The whole-sequence call (odom='gt')
        filters the frames on the device as they arrive - all at once when they are already there, else each uploaded
        (and, for RawRGBD, converted) chunk - and fuses the filtered depth; with depth_filter_tracking_only it filters
        nothing, since there is no tracking."""
        if not isinstance(surfel_radii, bool):
            raise TypeError("surfel_radii must be of type bool; but was of type {}.".format(type(surfel_radii)))
        _check_merge_overlapping(merge_overlapping, surfel_radii)
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
        if merge_overlapping and stable_confidence is None:
            raise ValueError("merge_overlapping needs stable_confidence and max_unstable_age (stable_confidence=0 makes "
                             "the age rule a no-op)")
        super().__init__(odom=odom, dsratio=dsratio, numiters=numiters, damp=damp, dist_thresh=dist_thresh,
                         lambda_max=lambda_max, B=B, B2=B2, nu=nu, association=association, device=device,
                         target_splat_px=target_splat_px, photometric_weight=photometric_weight,
                         depth_filter=depth_filter, depth_filter_tracking_only=depth_filter_tracking_only,
                         huber_delta=huber_delta, photometric_huber_delta=photometric_huber_delta)
        if target_splat_px > 0 and not surfel_radii:
            raise ValueError("target_splat_px > 0 needs surfel_radii=True (a map without radii has no disks)")
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
        self.surfel_radii = surfel_radii
        self.merge_overlapping = merge_overlapping

    def _refuse_pruned_embeddings(self, frames):
        if frames.embeddings is not None and self.stable_confidence is not None:
            raise ValueError("PointFusion's pruning options (stable_confidence, free_space_margin, merge_overlapping) "
                             "are not supported on frames with embeddings")

    def _map(self, pointclouds: Pointclouds, live_frame: RGBDImages, inplace: bool = False):
        self._refuse_pruned_embeddings(live_frame)
        if self.stable_confidence is not None and isinstance(pointclouds, Pointclouds):
            _check_history(pointclouds, self.max_unstable_age)
        if self.free_space_margin is not None or self.merge_overlapping:
            margin = math.inf if self.free_space_margin is None else self.free_space_margin
            return fuse_and_prune(pointclouds, live_frame, self.dist_th, self.dot_th, self.sigma, self.stable_confidence,
                                  self.max_unstable_age, margin, inplace, surfel_radii=self.surfel_radii,
                                  merge_overlapping=self.merge_overlapping)
        pointclouds = update_map_fusion(pointclouds, live_frame, self.dist_th, self.dot_th, self.sigma, inplace,
                                        surfel_radii=self.surfel_radii)
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
        if isinstance(frames, RGBDImages):
            self._refuse_pruned_embeddings(frames)
        return super().forward(frames, out)

    def _forward_sequence(self, frames, chunk: int = 4, raw: bool = False, out=None):
        """odom='gt': the whole (B, L) sequence runs as C calls chaining K2/K3 -> K4 per frame with no
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
                    frames.depth_image, frames.rgb_image, frames.poses, frames.intrinsics, frames.embeddings)):
                return None  # differentiable mode goes through the per-frame step loop
            if frames.channels_first:
                frames = frames.to_channels_last()
            B, L, H, W = frames.shape
            src_depth, src_rgb = frames.depth_image, frames.rgb_image
            on_device = src_depth.device == dev
        src_emb = None if raw else frames.embeddings
        P = H * W
        K = frames.intrinsics.to(dev).contiguous()
        poses = frames.poses.to(dev).contiguous()
        if on_device:
            depth, rgb = src_depth.contiguous(), src_rgb.contiguous()
            emb = None if src_emb is None else src_emb.contiguous()
            chunk = L
        else:
            depth = torch.empty((B, L, H, W, 1), dtype=torch.float32, device=dev)
            rgb = torch.empty((B, L, H, W, 3), dtype=torch.float32, device=dev)
            emb = None if src_emb is None else torch.empty(src_emb.shape, dtype=src_emb.dtype, device=dev)
            copy_stream = torch.cuda.Stream(device=dev)
            if raw:  # staging buffers for the 5-byte pixels; converted chunk by chunk on the compute stream
                raw_depth = torch.empty((B, L, H, W), dtype=src_depth.dtype, device=dev)
                raw_rgb = torch.empty((B, L, H, W, 3), dtype=torch.uint8, device=dev)
        for t, name in ((depth, "depth_image"), (rgb, "rgb_image"), (K, "intrinsics"), (poses, "poses")):
            _C.require_cuda(t, name)
        if out is not None:  # caller-provided storage (validated by forward: empty, B maps, this device)
            if not (out.has_normals and out.has_colors and out._has_cc):
                raise ValueError("out must have normals, colours and a confidence count per point for map fusion")
            if out.has_embeddings != (emb is not None) or (emb is not None and (
                    out._emb.shape[2], out._emb.dtype) != (emb.shape[-1], emb.dtype)):
                raise ValueError("out must have embeddings of the frames' dimension and dtype exactly when the frames "
                                 "have embeddings")
            pc = out
            pc._cur = 0
        else:
            pc = Pointclouds(device=dev)
            pc._allocate(B, L * P, 1, zero=False)
            if emb is not None:  # L*H*W rows of D channels per element: see INTEGRATION.md for a smaller `out`
                pc._alloc_embeddings(emb.shape[-1], emb.dtype)
        ws = _SequenceWorkspace.get(dev, B, H, W)
        prune = (None, 0, 0.0, None, 0)  # ring, t_max, c_stable, scratch, its bytes: pruning off
        free_space = (0.0, None, 0)  # margin, scratch, its bytes: the age rule alone
        merge = (None, 0)  # merge scratch, its bytes: no merging
        if self.stable_confidence is not None:  # a fresh map: frame s of the call is pruned step s
            pc._prune = hist = _PruneHistory.fresh(B, self.max_unstable_age, dev)
            scratch = _prune_scratch(B, pc.capacity, dev)
            prune = (hist.ring, self.max_unstable_age, float(self.stable_confidence), scratch, scratch.numel())
            if self.free_space_margin is not None or self.merge_overlapping:
                fs_scratch = torch.empty(_C.lib().gsx_fusion_free_space_scratch_bytes(B, H, W, pc.capacity),
                                         dtype=torch.uint8, device=dev)
                margin = math.inf if self.free_space_margin is None else float(self.free_space_margin)
                free_space = (margin, fs_scratch, fs_scratch.numel())
            if self.merge_overlapping:
                ms = torch.empty(_C.lib().gsx_fusion_merge_scratch_bytes(B, H, W, pc.capacity), dtype=torch.uint8,
                                 device=dev)
                merge = (ms, ms.numel())
        # the depth the driver fuses: the frames' own, or its bilateral filter in a second buffer
        filt = self.depth_filter if not self.depth_filter_tracking_only else None
        fused_depth = depth if filt is None else torch.empty_like(depth)
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
                        if emb is not None:
                            emb[b, s0:s1].copy_(src_emb[b, s0:s1], non_blocking=True)
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
            if filt is not None:  # the whole (B, L) at once, or this chunk of every element
                for src, dst, n in ([(depth, fused_depth, B * L)] if on_device else
                                    [(depth[b, s0:s1], fused_depth[b, s0:s1], s1 - s0) for b in range(B)]):
                    _C.launch("gsx_depth_bilateral", src, dst, None, n, H, W, filt.radius, filt.sigma_space,
                              filt.sigma_range)
            if emb is None:
                _C.launch("gsx_pointfusion_sequence_gt_merge", pc._geo, pc._col, pc._counts_dev, pc.capacity,
                          min(s0 * P, pc.capacity), fused_depth, rgb, K, poses, B, L, s0, s1, H, W, float(self.dist_th),
                          float(self.dot_th), float(self.sigma), ws.buf, *prune, *free_space, pc._overflow_flag(),
                          1 if self.surfel_radii else 0, *merge)
            else:
                if i == 0:
                    assoc = torch.empty((B, P), dtype=torch.int32, device=dev)
                    rec = torch.empty((B, P, 2), dtype=torch.float32, device=dev)
                args = (pc._geo, pc._col, pc._counts_dev, pc.capacity, min(s0 * P, pc.capacity), fused_depth, rgb, K,
                        poses, B, L, s0, s1, H, W, float(self.dist_th), float(self.dot_th), float(self.sigma), ws.buf,
                        pc._overflow_flag(), 1 if self.surfel_radii else 0, pc._emb, emb)
                if frames.upsample_embeddings:  # (B, L, h, w, D) coarse images, sampled by the upsampled KE
                    _C.launch("gsx_pointfusion_sequence_gt_emb_upsampled", *args, emb.shape[2], emb.shape[3],
                              emb.shape[-1], EMBED_DTYPES[emb.dtype], assoc, rec)
                else:
                    _C.launch("gsx_pointfusion_sequence_gt_emb", *args, emb.shape[-1], EMBED_DTYPES[emb.dtype], assoc,
                              rec)
        if not on_device:
            for t in ((raw_depth, raw_rgb) if raw else (depth, rgb)):
                t.record_stream(copy_stream)
            if emb is not None:
                emb.record_stream(copy_stream)
        pc._cur = L & 1
        pc._counts_host = None
        pc._bound = pc.capacity
        pc._list_cache = {}
        pc._tail_dirty = pc._uninit
        if self.stable_confidence is not None:  # rows past the pruned sizes hold stale values
            hist.step = L
            pc._uninit = pc._tail_dirty = True
        return pc, poses.clone()
