"""Frame -> cloud conversion (mirror of gradslam/structures/utils.py:7-57) and its inverse, cloud -> frames."""
import math
from typing import NamedTuple, Optional

import torch

from .. import _C
from .pointclouds import Pointclouds
from .rgbdimages import RGBDImages

__all__ = ["pointclouds_from_rgbdimages", "render_pointclouds", "RenderedViews"]


def pointclouds_from_rgbdimages(rgbdimages: RGBDImages, *, global_coordinates: bool = True,
                                filter_missing_depths: bool = True) -> Pointclouds:
    """Converts a sequence-length-1 RGBDImages batch into Pointclouds (points, normals, colors).

    With `filter_missing_depths` the valid pixels of every element are compacted in row-major order by the
    stable-append kernel (the same K4 kernel PointFusion uses, run with no matches)."""
    if not isinstance(rgbdimages, RGBDImages):
        raise TypeError("Expected rgbdimages to be of type gradslam.RGBDImages. Got {0}.".format(type(rgbdimages)))
    if not rgbdimages.shape[1] == 1:
        raise ValueError("Expected rgbdimages to have sequence length of 1. Got {0}.".format(rgbdimages.shape[1]))
    B = rgbdimages.shape[0]
    rgbdimages = rgbdimages.to_channels_last()
    if filter_missing_depths:
        from ..slam.fusionutils import _append_valid_pixels

        return _append_valid_pixels(Pointclouds(device=rgbdimages.device), rgbdimages, global_coordinates)
    vmap = rgbdimages.global_vertex_map if global_coordinates else rgbdimages.vertex_map
    nmap = rgbdimages.global_normal_map if global_coordinates else rgbdimages.normal_map
    return Pointclouds(points=vmap.reshape(B, -1, 3).contiguous(), normals=nmap.reshape(B, -1, 3).contiguous(),
                       colors=rgbdimages.rgb_image.reshape(B, -1, 3).contiguous())


class RenderedViews(NamedTuple):
    """Images of a map seen from L cameras per element, channels last.  Uncovered pixels: index -1, zeros elsewhere."""
    depth: torch.Tensor                 # (B, L, H, W, 1) camera-frame z of the visible row
    rgb: Optional[torch.Tensor]         # (B, L, H, W, 3), None for a map without colours
    normals: Optional[torch.Tensor]     # (B, L, H, W, 3) in the camera frame, None for a map without normals
    confidence: Optional[torch.Tensor]  # (B, L, H, W, 1) confidence count, None without that feature
    index: torch.Tensor                 # (B, L, H, W) int64 map row of the pixel, or -1


def _render(geo, col, counts, bound, K, poses, H, W, want_normals, want_conf, splat=0):
    """gsx_render_splats on dense CUDA tensors -> (depth, rgb, normals, confidence, index); splat = max_splat_px."""
    B, L = poses.shape[:2]
    dev = poses.device
    cap = 0 if geo is None else geo.shape[1]
    img = lambda c: torch.empty((B, L, H, W, c), dtype=torch.float32, device=dev)
    index = torch.empty((B, L, H, W), dtype=torch.int64, device=dev)
    depth, rgb = img(1), None if col is None else img(3)
    normals, conf = img(3) if want_normals else None, img(1) if want_conf else None
    _C.launch("gsx_render_splats", geo, col, counts, cap, bound, K, 16, poses, L * 16, B, L, H, W, index, depth, rgb,
              normals, conf, splat)
    return depth, rgb, normals, conf, index


class _RenderFn(torch.autograd.Function):
    """gsx_render_splats as one differentiable op over (geometry rows, colour rows, poses, intrinsics); backward =
    gsx_render_splats_bwd at the forward's index, or gsx_render_splats_bwd_intrinsics when the intrinsics require grad
    (the association and the footprint carry no gradient, the radius none either)."""

    @staticmethod
    def forward(ctx, pack, geo, col, poses, intrinsics):
        counts, bound, H, W, want_normals, want_conf, splat = pack
        K = intrinsics.detach().contiguous()
        outs = _render(geo.detach(), None if col is None else col.detach(), counts, bound, K, poses.detach(), H, W,
                       want_normals, want_conf, splat)
        ctx.mark_non_differentiable(outs[4])
        ctx.set_materialize_grads(False)
        ctx.save_for_backward(geo, poses, outs[4])
        ctx.pack = (counts, K, H, W, splat)
        ctx.K_shape = intrinsics.shape
        return outs

    @staticmethod
    def backward(ctx, g_depth, g_rgb, g_normals, g_conf, _g_index):
        geo, poses, index = ctx.saved_tensors
        counts, K, H, W, splat = ctx.pack
        _, need_geo, need_col, need_pose, need_K = ctx.needs_input_grad
        B, L = poses.shape[:2]
        dev, cap = geo.device, geo.shape[1]
        d_geo = torch.empty_like(geo) if need_geo else None
        d_col = torch.empty((B, cap, 4), dtype=torch.float32, device=dev) if need_col else None
        d_poses = torch.empty((B, L, 4, 4), dtype=torch.float32, device=dev) if need_pose else None
        scratch = None
        if need_pose:
            scratch = torch.empty(_C.lib().gsx_render_views_bwd_scratch_bytes(B, L, H, W), dtype=torch.uint8,
                                  device=dev)
        gs = [None if g is None else g.contiguous() for g in (g_depth, g_rgb, g_normals, g_conf)]
        if need_K:
            g_K = torch.zeros((B, 4, 4), dtype=torch.float32, device=dev)
            scratch = torch.empty(_C.lib().gsx_render_splats_bwd_intrinsics_scratch_bytes(B, L, H, W),
                                  dtype=torch.uint8, device=dev)
            _C.launch("gsx_render_splats_bwd_intrinsics", geo.detach(), counts, cap, K, 16, poses.detach(), L * 16,
                      index, B, L, H, W, *gs, d_geo, d_col, d_poses, g_K, scratch, scratch.numel(), splat)
            return None, d_geo, d_col, d_poses, g_K.view(ctx.K_shape)
        _C.launch("gsx_render_splats_bwd", geo.detach(), counts, cap, K, 16, poses.detach(), L * 16, index, B, L, H, W,
                  *gs, d_geo, d_col, d_poses, scratch, 0 if scratch is None else scratch.numel(), splat)
        return None, d_geo, d_col, d_poses, None


def _render_blend(geo, col, counts, bound, K, poses, H, W, want_normals, use_conf, band, splat):
    """gsx_render_blend on dense CUDA tensors -> (depth, rgb, normals, weight, index, front depth)."""
    B, L = poses.shape[:2]
    dev = poses.device
    cap = geo.shape[1]
    img = lambda c: torch.empty((B, L, H, W, c), dtype=torch.float32, device=dev)
    index = torch.empty((B, L, H, W), dtype=torch.int64, device=dev)
    front, weight, depth = torch.empty((B, L, H, W), dtype=torch.float32, device=dev), img(1), img(1)
    rgb, normals = None if col is None else img(3), img(3) if want_normals else None
    scratch = torch.empty(_C.lib().gsx_render_blend_scratch_bytes(B, L, H, W, bound, splat), dtype=torch.uint8,
                          device=dev)
    _C.launch("gsx_render_blend", geo, col, counts, cap, bound, K, 16, poses, L * 16, B, L, H, W, int(use_conf), band,
              splat, index, front, weight, depth, rgb, normals, scratch, scratch.numel())
    return depth, rgb, normals, weight, index, front


class _RenderBlendFn(torch.autograd.Function):
    """gsx_render_blend as one differentiable op over (geometry rows, colour rows, poses); backward =
    gsx_render_blend_bwd: through the blend weights to the rows' positions, normals, radii and confidence counts, to
    their colours and to the poses.  Which rows cover a pixel, and the front depth, carry no gradient."""

    @staticmethod
    def forward(ctx, pack, geo, col, poses):
        counts, bound, H, W, want_normals, use_conf, band, splat, K = pack
        depth, rgb, normals, weight, index, front = _render_blend(
            geo.detach(), None if col is None else col.detach(), counts, bound, K, poses.detach(), H, W, want_normals,
            use_conf, band, splat)
        ctx.mark_non_differentiable(index)
        ctx.set_materialize_grads(False)
        ctx.save_for_backward(geo, col, poses, front, weight, depth, rgb, normals)
        ctx.pack = pack
        return depth, rgb, normals, weight, index

    @staticmethod
    def backward(ctx, g_depth, g_rgb, g_normals, g_weight, _g_index):
        geo, col, poses, front, weight, depth, rgb, normals = ctx.saved_tensors
        counts, bound, H, W, _, use_conf, band, splat, K = ctx.pack
        _, need_geo, need_col, need_pose = ctx.needs_input_grad
        B, L = poses.shape[:2]
        dev, cap = geo.device, geo.shape[1]
        d_geo = torch.empty_like(geo) if need_geo else None
        d_col = torch.empty((B, cap, 4), dtype=torch.float32, device=dev) if need_col else None
        d_poses = torch.empty((B, L, 4, 4), dtype=torch.float32, device=dev) if need_pose else None
        scratch = None
        if need_pose:
            scratch = torch.empty(_C.lib().gsx_render_blend_bwd_scratch_bytes(B, L, bound), dtype=torch.uint8,
                                  device=dev)
        gs = [None if g is None else g.contiguous() for g in (g_depth, g_rgb, g_normals, g_weight)]
        _C.launch("gsx_render_blend_bwd", geo.detach(), None if col is None else col.detach(), counts, cap, bound, K,
                  16, poses.detach(), L * 16, B, L, H, W, int(use_conf), band, splat, front, weight, depth, rgb,
                  normals, *gs, d_geo, d_col, d_poses, scratch, 0 if scratch is None else scratch.numel())
        return None, d_geo, d_col, d_poses


def _blend_band(blend_band):
    """None, or blend_band as a float >= 0 (+inf allowed)."""
    if blend_band is None:
        return None
    if isinstance(blend_band, bool) or not isinstance(blend_band, (int, float)):
        raise TypeError("Expected blend_band to be None or a number. Got {}.".format(type(blend_band)))
    band = float(blend_band)
    if math.isnan(band) or band < 0:
        raise ValueError("Expected blend_band >= 0 (metres, inf allowed). Got {}.".format(blend_band))
    return band


def _camera(t, name, B):
    if not torch.is_tensor(t):
        raise TypeError("Expected {} to be of type torch.Tensor. Got {}.".format(name, type(t)))
    if t.ndim != 4 or tuple(t.shape[-2:]) != (4, 4):
        raise ValueError("Expected {} to have shape (B, L, 4, 4). Got {}.".format(name, tuple(t.shape)))
    if B is not None and t.shape[0] != B:
        raise ValueError("Expected equal batch sizes for {} and poses. Got {} and {}.".format(name, t.shape[0], B))


MAX_SPLAT_PX = 16  # GSX_MAX_SPLAT_PX (include/gsx.h)


def render_pointclouds(pointclouds: Pointclouds, intrinsics: torch.Tensor, poses: torch.Tensor, height: int,
                       width: int, max_splat_px: int = 0, blend_band: Optional[float] = None) -> RenderedViews:
    """Renders every map of the batch from L cameras: a map row covers the one pixel it projects to (the projection of
    find_active_map_points) and each pixel shows the covering row with the smallest camera-frame depth, ties to the
    lowest row index.

    intrinsics (B, 1, 4, 4) as in RGBDImages; poses (B, L, 4, 4) camera-to-world.  `RGBDImages(out.rgb, out.depth,
    intrinsics, poses)` turns the result into frames.  Differentiable w.r.t. the map rows (points, normals, colours,
    confidence counts), the poses and the intrinsics, at the fixed pixel assignment.  Only a disk pixel's depth depends on
    the intrinsics' values (through its ray, max_splat_px >= 1), so with max_splat_px = 0 their gradient is zero.  No
    host synchronisation.

    max_splat_px (extension, 0 .. 16, default 0 = the one-pixel rule above for every row): a row with a surfel radius
    (`radii_padded` > 0, PointFusion(surfel_radii=True)) and a non-zero normal is drawn as an oriented disk: every pixel
    within max_splat_px pixels of its projected centre whose ray meets the disk shows it, at the depth where the ray
    meets the disk's plane.  Rows without a radius keep the one-pixel rule.  The footprint carries no gradient, and
    the radius none either.  Cost grows with (2 max_splat_px + 1)^2 per disk row and view.

    blend_band (extension, default None = the z-buffer above): a float >= 0 in metres (inf allowed) blends.  Each pixel
    then shows the normalised, weighted mean of the rows that cover it (the coverage above, at max_splat_px) at a depth
    no more than blend_band behind the front surface, the depth the z-buffer shows.  A disk row weighs
    c (1 - s^2 / r^2), with s its in-plane distance from the ray's hit to its centre and r its radius; any other row
    weighs c; c is the confidence count, or 1 for a map without one.  depth, rgb and normals (camera frame, not
    renormalised) are the weighted means, confidence is the sum of the weights, and index is the z-buffer's.  Gradients
    reach every contributing row's position, normal, radius, confidence count and colour, and the poses, through the
    weights as well as the values.  Intrinsics that require grad are refused (no d/dK through the blend)."""
    if not isinstance(pointclouds, Pointclouds):
        raise TypeError("Expected pointclouds to be of type gradslam.Pointclouds. Got {0}.".format(type(pointclouds)))
    for name, v in (("height", height), ("width", width)):
        if not isinstance(v, int) or isinstance(v, bool):
            raise TypeError("Expected {} to be of type int. Got {}.".format(name, type(v)))
        if v < 1:
            raise ValueError("Expected {} >= 1. Got {}.".format(name, v))
    if not isinstance(max_splat_px, int) or isinstance(max_splat_px, bool):
        raise TypeError("Expected max_splat_px to be of type int. Got {}.".format(type(max_splat_px)))
    if not 0 <= max_splat_px <= MAX_SPLAT_PX:
        raise ValueError("Expected 0 <= max_splat_px <= {}. Got {}.".format(MAX_SPLAT_PX, max_splat_px))
    band = _blend_band(blend_band)
    _camera(poses, "poses", None)
    B = poses.shape[0]
    _camera(intrinsics, "intrinsics", B)
    if intrinsics.shape[1] != 1:
        raise ValueError("Expected intrinsics to have shape (B, 1, 4, 4). Got {}.".format(tuple(intrinsics.shape)))
    if band is not None and torch.is_grad_enabled() and intrinsics.requires_grad:
        raise ValueError("render_pointclouds: blend_band has no gradient w.r.t. the intrinsics; detach them")
    if pointclouds.has_points and len(pointclouds) != B:
        raise ValueError("Expected equal batch sizes for pointclouds and poses. Got {0} and {1}.".format(
            len(pointclouds), B))
    if pointclouds.has_points and pointclouds._col is not None and pointclouds._col.shape[:2] != pointclouds._geo.shape[:2]:
        # the kernels address both row stores with one capacity
        raise ValueError("pointclouds: colour rows {} do not match the geometry rows {}".format(
            tuple(pointclouds._col.shape), tuple(pointclouds._geo.shape)))
    _C.require_cuda(poses, "poses")
    _C.require_cuda(intrinsics, "intrinsics")
    dev = poses.device
    if intrinsics.device != dev:
        raise ValueError("intrinsics ({}) and poses ({}) must be on the same device".format(intrinsics.device, dev))
    K = intrinsics.detach().contiguous()
    if not pointclouds.has_points:  # nothing to project: every pixel uncovered
        d, _, _, _, idx = _render(None, None, None, 0, K, poses.detach().contiguous(), height, width, False, False)
        return RenderedViews(d, None, None, None, idx)
    _C.require_cuda(pointclouds._geo, "pointclouds (geometry rows)")
    if pointclouds.device != dev:
        raise ValueError("pointclouds ({}) and poses ({}) must be on the same device".format(pointclouds.device, dev))
    geo, col = pointclouds._geo.contiguous(), None if pointclouds._col is None else pointclouds._col.contiguous()
    counts = pointclouds._counts_dev[pointclouds._cur]
    want = (pointclouds.has_normals, pointclouds._has_cc)
    poses_c = poses.contiguous()
    from ..odometry.icputils import _wants_grad

    if band is not None:
        pack = (counts.clone(), pointclouds._bound, height, width, pointclouds.has_normals, pointclouds._has_cc, band,
                max_splat_px, K)
        if _wants_grad(geo, col, poses_c):
            depth, rgb, normals, weight, index = _RenderBlendFn.apply(pack, geo, col, poses_c)
        else:
            depth, rgb, normals, weight, index, _ = _render_blend(
                geo.detach(), None if col is None else col.detach(), counts, pointclouds._bound, K, poses_c.detach(),
                height, width, *pack[4:8])
        return RenderedViews(depth, rgb, normals, weight if pointclouds._has_cc else None, index)
    if _wants_grad(geo, col, poses_c, intrinsics):
        outs = _RenderFn.apply((counts.clone(), pointclouds._bound, height, width) + want + (max_splat_px,), geo, col,
                               poses_c, intrinsics)
    else:
        outs = _render(geo.detach(), None if col is None else col.detach(), counts, pointclouds._bound, K,
                       poses_c.detach(), height, width, *want, max_splat_px)
    return RenderedViews(*outs)
