"""Dataset output contract -> device ingest (SURVEY.md §8f.2).

gradslam's loaders (gradslam/datasets/icl.py:393-533, tum.py, scannet.py) read 8-bit colour and 16-bit depth from disk,
convert them to float32 on the HOST (colour as float(u8), optionally / 255; depth as u16 / scaling_factor) and only then
ship 16 bytes per pixel to the device.  Here the raw 5 bytes per pixel are uploaded (pinned memory, asynchronous) and the
same conversion runs on the device (csrc/gsx_ingest.cu), bit-identical to the host-side one.  The image resize the
loaders can also do is not covered: pass frames at their final size (and `scale_intrinsics` if they were resized).
"""
from typing import Optional, Union

import torch

from . import _C
from .structures.rgbdimages import RGBDImages

__all__ = ["scale_intrinsics", "relative_poses", "raw_to_float", "rgbdimages_from_raw", "RawRGBD"]


def scale_intrinsics(intrinsics: torch.Tensor, h_ratio: Union[float, int], w_ratio: Union[float, int]) -> torch.Tensor:
    """Intrinsics of frames resized by (h_ratio, w_ratio) (mirror of gradslam/datasets/datautils.py:73-122)."""
    if not torch.is_tensor(intrinsics):
        raise TypeError("Unsupported input intrinsics type {}".format(type(intrinsics)))
    if not (intrinsics.shape[-2:] == (3, 3) or intrinsics.shape[-2:] == (4, 4)):
        raise ValueError("intrinsics must have shape (*, 3, 3) or (*, 4, 4), but had shape {} instead".format(
            intrinsics.shape))
    if intrinsics.is_cuda:  # on the device, next to the raw-frame conversion (csrc/gsx_ingest.cu); same float32 products
        K = intrinsics.to(torch.float).contiguous()
        out = torch.empty_like(K)
        n = K.numel() // (K.shape[-1] * K.shape[-1])
        _C.launch("gsx_ingest_calibration", K, n, K.shape[-1], float(h_ratio), float(w_ratio), out, None, 0, 0, None,
                  None)
        return out
    out = intrinsics.to(torch.float).clone()
    out[..., 0, 0] *= w_ratio
    out[..., 1, 1] *= h_ratio
    out[..., 0, 2] *= w_ratio
    out[..., 1, 2] *= h_ratio
    return out


def relative_poses(poses: torch.Tensor) -> torch.Tensor:
    """Poses (B, L, 4, 4) or (L, 4, 4) made relative to the first frame of each sequence, as the reference's loaders
    deliver them (gradslam/datasets/icl.py:515-533: relative_transformation(T_0, T_s) with a general inverse of T_0).
    Runs on the device (csrc/gsx_ingest.cu); CUDA float32 input."""
    if not torch.is_tensor(poses):
        raise TypeError("Input poses type is not a torch.Tensor. Got {}".format(type(poses)))
    if poses.dim() not in (3, 4) or poses.shape[-2:] != (4, 4):
        raise ValueError("poses must have shape (B, L, 4, 4) or (L, 4, 4). Got {}".format(tuple(poses.shape)))
    _C.require_cuda(poses, "poses")
    p = poses.contiguous()
    B, L = (1, p.shape[0]) if p.dim() == 3 else p.shape[:2]
    out = torch.empty_like(p)
    flag = torch.zeros(1, dtype=torch.int32, device=p.device)
    _C.launch("gsx_ingest_calibration", None, 0, 4, 1.0, 1.0, None, p, B, L, out, flag)
    return out


def _check_raw(colors, depths):
    if not (torch.is_tensor(colors) and colors.dtype == torch.uint8 and colors.shape[-1] == 3):
        raise TypeError("colors must be a uint8 tensor (..., H, W, 3)")
    if not (torch.is_tensor(depths) and depths.dtype in (torch.uint16, torch.int16)):
        raise TypeError("depths must be a uint16 tensor (..., H, W) or (..., H, W, 1) (int16 storage of the same bits is accepted)")
    if depths.dim() == colors.dim() and depths.shape[-1] == 1:
        depths = depths[..., 0]
    if tuple(depths.shape) != tuple(colors.shape[:-1]):
        raise ValueError("colors {} and depths {} do not describe the same frames".format(tuple(colors.shape), tuple(depths.shape)))
    return colors, depths


def raw_to_float(colors_u8: torch.Tensor, depths_u16: torch.Tensor, scaling_factor: float = 5000.0,
                 normalize_color: bool = False, out_rgb: Optional[torch.Tensor] = None,
                 out_depth: Optional[torch.Tensor] = None):
    """Device-side conversion of CUDA uint8 colour (...,H,W,3) / uint16 depth (...,H,W) to float32 (…,3) / (…,1)."""
    colors_u8, depths_u16 = _check_raw(colors_u8, depths_u16)
    if not colors_u8.is_cuda or not depths_u16.is_cuda:
        raise RuntimeError("gradslam_b200: raw_to_float needs CUDA tensors; there is no CPU path")
    colors_u8, depths_u16 = colors_u8.contiguous(), depths_u16.contiguous()
    dev = colors_u8.device
    rgb = out_rgb if out_rgb is not None else torch.empty(colors_u8.shape, dtype=torch.float32, device=dev)
    depth = out_depth if out_depth is not None else torch.empty((*depths_u16.shape, 1), dtype=torch.float32, device=dev)
    _C.launch("gsx_ingest_raw", colors_u8, depths_u16, depths_u16.numel(), float(scaling_factor),
              1 if normalize_color else 0, rgb, depth)
    return rgb, depth


class RawRGBD(object):
    """A (B, L) batch of sequences in dataset-native form: uint8 colour (B,L,H,W,3), uint16 depth (B,L,H,W), float32
    intrinsics (B,1,4,4) and poses (B,L,4,4), on the host (pin the image tensors) or on the device.
    `PointFusion(odom='gt')(raw)` uploads and converts chunk by chunk, overlapped with the fusion."""

    def __init__(self, colors_u8, depths_u16, intrinsics, poses, scaling_factor: float = 5000.0,
                 normalize_color: bool = False):
        self.colors, self.depths = _check_raw(colors_u8, depths_u16)
        if self.colors.dim() != 5:
            raise ValueError("colors must have shape (B, L, H, W, 3)")
        self.intrinsics, self.poses = intrinsics, poses
        self.scaling_factor, self.normalize_color = float(scaling_factor), bool(normalize_color)
        self.shape = tuple(self.colors.shape[:4])


def rgbdimages_from_raw(colors_u8, depths_u16, intrinsics, poses=None, *, scaling_factor: float = 5000.0,
                        normalize_color: bool = False, device: Union[torch.device, str] = "cuda",
                        resized_from=None, relative_to_first: bool = False) -> RGBDImages:
    """Uploads raw frames (B,L,H,W,3) uint8 / (B,L,H,W) uint16 and returns the float32 RGBDImages the reference's loaders
    would have produced (same bits), resident on `device`.  resized_from=(H_orig, W_orig): the frames were resized from
    that size, so the intrinsics are scaled accordingly; relative_to_first: absolute poses (as stored on disk) are made
    relative to the first frame of each sequence (both on the device, as the loaders do on the host)."""
    colors_u8, depths_u16 = _check_raw(colors_u8, depths_u16)
    dev = torch.device(device)
    rgb, depth = raw_to_float(colors_u8.to(dev, non_blocking=True), depths_u16.to(dev, non_blocking=True),
                              scaling_factor, normalize_color)
    K = intrinsics.to(dev)
    if resized_from is not None:
        H, W = colors_u8.shape[-3], colors_u8.shape[-2]
        K = scale_intrinsics(K, H / float(resized_from[0]), W / float(resized_from[1]))
    P = None if poses is None else poses.to(dev)
    if P is not None and relative_to_first:
        P = relative_poses(P.to(torch.float32))
    return RGBDImages(rgb, depth, K, P)
