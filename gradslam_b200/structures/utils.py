"""Frame -> cloud conversion (mirror of gradslam/structures/utils.py:7-57) and its inverse, cloud -> frames."""
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


def _render(geo, col, counts, bound, K, poses, H, W, want_normals, want_conf):
    """gsx_render_views on dense CUDA tensors -> (depth, rgb, normals, confidence, index)."""
    B, L = poses.shape[:2]
    dev = poses.device
    cap = 0 if geo is None else geo.shape[1]
    img = lambda c: torch.empty((B, L, H, W, c), dtype=torch.float32, device=dev)
    index = torch.empty((B, L, H, W), dtype=torch.int64, device=dev)
    depth, rgb = img(1), None if col is None else img(3)
    normals, conf = img(3) if want_normals else None, img(1) if want_conf else None
    _C.launch("gsx_render_views", geo, col, counts, cap, bound, K, 16, poses, L * 16, B, L, H, W, index, depth, rgb,
              normals, conf)
    return depth, rgb, normals, conf, index


class _RenderFn(torch.autograd.Function):
    """gsx_render_views as one differentiable op over (geometry rows, colour rows, poses); backward =
    gsx_render_views_bwd at the forward's index (the association carries no gradient)."""

    @staticmethod
    def forward(ctx, pack, geo, col, poses):
        counts, bound, K, H, W, want_normals, want_conf = pack
        outs = _render(geo.detach(), None if col is None else col.detach(), counts, bound, K, poses.detach(), H, W,
                       want_normals, want_conf)
        ctx.mark_non_differentiable(outs[4])
        ctx.set_materialize_grads(False)
        ctx.save_for_backward(geo, poses, outs[4])
        ctx.pack = (counts, K, H, W)
        return outs

    @staticmethod
    def backward(ctx, g_depth, g_rgb, g_normals, g_conf, _g_index):
        geo, poses, index = ctx.saved_tensors
        counts, K, H, W = ctx.pack
        _, need_geo, need_col, need_pose = ctx.needs_input_grad
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
        _C.launch("gsx_render_views_bwd", geo.detach(), counts, cap, K, 16, poses.detach(), L * 16, index, B, L, H, W, *gs,
                  d_geo, d_col, d_poses, scratch, 0 if scratch is None else scratch.numel())
        return None, d_geo, d_col, d_poses


def _camera(t, name, B):
    if not torch.is_tensor(t):
        raise TypeError("Expected {} to be of type torch.Tensor. Got {}.".format(name, type(t)))
    if t.ndim != 4 or tuple(t.shape[-2:]) != (4, 4):
        raise ValueError("Expected {} to have shape (B, L, 4, 4). Got {}.".format(name, tuple(t.shape)))
    if B is not None and t.shape[0] != B:
        raise ValueError("Expected equal batch sizes for {} and poses. Got {} and {}.".format(name, t.shape[0], B))


def render_pointclouds(pointclouds: Pointclouds, intrinsics: torch.Tensor, poses: torch.Tensor, height: int,
                       width: int) -> RenderedViews:
    """Renders every map of the batch from L cameras: a map row covers the one pixel it projects to (the projection of
    find_active_map_points) and each pixel shows the covering row with the smallest camera-frame depth, ties to the
    lowest row index.

    intrinsics (B, 1, 4, 4) as in RGBDImages; poses (B, L, 4, 4) camera-to-world.  `RGBDImages(out.rgb, out.depth,
    intrinsics, poses)` turns the result into frames.  Differentiable w.r.t. the map rows (points, normals, colours,
    confidence counts) and the poses, at the fixed pixel assignment; not w.r.t. the intrinsics.  No host
    synchronisation."""
    if not isinstance(pointclouds, Pointclouds):
        raise TypeError("Expected pointclouds to be of type gradslam.Pointclouds. Got {0}.".format(type(pointclouds)))
    for name, v in (("height", height), ("width", width)):
        if not isinstance(v, int) or isinstance(v, bool):
            raise TypeError("Expected {} to be of type int. Got {}.".format(name, type(v)))
        if v < 1:
            raise ValueError("Expected {} >= 1. Got {}.".format(name, v))
    _camera(poses, "poses", None)
    B = poses.shape[0]
    _camera(intrinsics, "intrinsics", B)
    if intrinsics.shape[1] != 1:
        raise ValueError("Expected intrinsics to have shape (B, 1, 4, 4). Got {}.".format(tuple(intrinsics.shape)))
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

    if _wants_grad(geo, col, poses_c):
        outs = _RenderFn.apply((counts.clone(), pointclouds._bound, K, height, width) + want, geo, col, poses_c)
    else:
        outs = _render(geo.detach(), None if col is None else col.detach(), counts, pointclouds._bound, K,
                       poses_c.detach(), height, width, *want)
    return RenderedViews(*outs)
