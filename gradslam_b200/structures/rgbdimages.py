"""RGBDImages: batched RGB-D sequence container with lazily computed vertex / normal maps.

Host-side mirror of gradslam.RGBDImages (gradslam/structures/rgbdimages.py:13-915): same constructor,
properties, indexing and error behaviour.  The four cached maps are produced by ONE hand-written sm_90a
kernel (gsx_backproject_normals_fwd) instead of the reference's einsum / slice / cross / norm chain
(rgbdimages.py:643-762).  Containers may hold tensors on any device, but computing a map requires CUDA
tensors: there is no CPU compute path.
"""
from typing import Optional, Union

import torch

from .. import _C

__all__ = ["RGBDImages"]


def _frame_base(t: torch.Tensor, inner: int):
    """(B,L,H,W,C) tensor -> (tensor, batch stride) such that element (b,l) starts at b*bstride + l*inner."""
    B, L = t.shape[:2]
    ok = t.stride(-1) == 1 if t.shape[-1] > 1 else True
    exp = 1
    for d in range(t.dim() - 1, 1, -1):  # dims H,W,C must be dense
        if t.shape[d] != 1 and t.stride(d) != exp:
            ok = False
        exp *= t.shape[d]
    if L > 1 and t.stride(1) != inner:
        ok = False
    if not ok:
        t = t.contiguous()
    bstride = t.stride(0) if B > 1 else L * inner
    return t, bstride


class _BackprojectFn(torch.autograd.Function):
    """depth, intrinsics, poses -> (vertex, normal, gvertex, gnormal); all channels-last.
    forward = gsx_backproject_normals_fwd, backward = gsx_backproject_normals_bwd (d/d depth, d/d poses)."""

    @staticmethod
    def forward(ctx, depth, intrinsics, poses, want):
        B, L, H, W, _ = depth.shape
        _C.require_cuda(depth, "depth_image")
        _C.require_cuda(intrinsics, "intrinsics")
        d, d_bs = _frame_base(depth.detach(), H * W)
        K = intrinsics.detach().contiguous()
        P = None
        if poses is not None:
            _C.require_cuda(poses, "poses")
            P = poses.detach().contiguous()
        outs = [torch.empty((B, L, H, W, 3), dtype=torch.float32, device=depth.device) if w else None for w in want]
        _C.launch("gsx_backproject_normals_fwd", d, d_bs, K, 16, P, L * 16, B, L, H, W, *outs)
        ctx.saved = (d, d_bs, K, P, (B, L, H, W))
        ctx.need_pose = poses is not None and poses.requires_grad
        return tuple(outs)

    @staticmethod
    def backward(ctx, g_v, g_n, g_gv, g_gn):
        d, d_bs, K, P, (B, L, H, W) = ctx.saved
        dev = d.device
        gs = [None if g is None else g.contiguous() for g in (g_v, g_n, g_gv, g_gn)]
        g_depth = torch.empty((B, L, H, W, 1), dtype=torch.float32, device=dev)
        g_poses = torch.empty((B, L, 4, 4), dtype=torch.float32, device=dev) if ctx.need_pose else None
        nbytes = _C.lib().gsx_backproject_normals_bwd_scratch_bytes(B, L, H, W)
        scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev) if ctx.need_pose else None
        _C.launch("gsx_backproject_normals_bwd", d, d_bs, K, 16, P, L * 16, B, L, H, W, *gs, g_depth, g_poses, scratch,
                  nbytes if ctx.need_pose else 0)
        return g_depth, None, g_poses, None


def backproject(depth, intrinsics, poses, want=(True, True, True, True)):
    """Runs K1.  depth (B,L,H,W,1) channels-last.  Returns a 4-tuple (entries not wanted are None)."""
    return _BackprojectFn.apply(depth, intrinsics, poses, tuple(bool(w) for w in want))


class RGBDImages(object):
    _INTERNAL_TENSORS = [
        "_rgb_image", "_depth_image", "_intrinsics", "_poses", "_pixel_pos",
        "_vertex_map", "_normal_map", "_global_vertex_map", "_global_normal_map",
    ]

    def __init__(self, rgb_image: torch.Tensor, depth_image: torch.Tensor, intrinsics: torch.Tensor,
                 poses: Optional[torch.Tensor] = None, channels_first: bool = False,
                 device: Union[torch.device, str, None] = None, *, pixel_pos: Optional[torch.Tensor] = None):
        super().__init__()
        for name, val, opt in (("rgb_image", rgb_image, False), ("depth_image", depth_image, False),
                               ("intrinsics", intrinsics, False), ("poses", poses, True),
                               ("pixel_pos", pixel_pos, True)):
            if not (torch.is_tensor(val) or (opt and val is None)):
                kind = "tensor or None" if opt else "tensor"
                raise TypeError("Expected {} to be of type {}; got {}".format(name, kind, type(val)))
        if not isinstance(channels_first, bool):
            raise TypeError("Expected channels_first to be of type bool; got {}".format(type(channels_first)))
        self._channels_first = channels_first

        if rgb_image.ndim != 5:
            raise ValueError("rgb_image should have ndim=5, but had ndim={}".format(rgb_image.ndim))
        if depth_image.ndim != 5:
            raise ValueError("depth_image should have ndim=5, but had ndim={}".format(depth_image.ndim))
        if intrinsics.ndim != 4:
            raise ValueError("intrinsics should have ndim=4, but had ndim={}".format(intrinsics.ndim))
        if poses is not None and poses.ndim != 4:
            raise ValueError("poses should have ndim=4, but had ndim={}".format(poses.ndim))

        cdim = self.cdim
        self._rgb_image_shape = rgb_image.shape
        self._depth_shape = tuple(v if i != cdim else 1 for i, v in enumerate(rgb_image.shape))
        self._depth_image_shape = self._depth_shape
        self._intrinsics_shape = (rgb_image.shape[0], 1, 4, 4)
        self._poses_shape = (*rgb_image.shape[:2], 4, 4)
        self._pixel_pos_shape = (*rgb_image.shape[:cdim], *rgb_image.shape[cdim + 1:], 3)

        if rgb_image.shape[cdim] != 3:
            raise ValueError("Expected rgb_image to have 3 channels on dimension {0}. Got {1} instead".format(
                cdim, rgb_image.shape[cdim]))
        if depth_image.shape != self._depth_shape:
            raise ValueError("Expected depth_image to have shape {0}. Got {1} instead".format(
                self._depth_shape, depth_image.shape))
        if intrinsics.shape != self._intrinsics_shape:
            raise ValueError("Expected intrinsics to have shape {0}. Got {1} instead".format(
                self._intrinsics_shape, intrinsics.shape))
        if poses is not None and poses.shape != self._poses_shape:
            raise ValueError("Expected poses to have shape {0}. Got {1} instead".format(self._poses_shape, poses.shape))
        if pixel_pos is not None and pixel_pos.shape != self._pixel_pos_shape:
            raise ValueError("Expected pixel_pos to have shape {0}. Got {1} instead".format(
                self._pixel_pos_shape, pixel_pos.shape))

        devices = set(x.device for x in (rgb_image, depth_image, intrinsics, poses, pixel_pos) if x is not None)
        if len(devices) != 1:
            raise ValueError("All inputs must be on same device, but got more than 1 device: {}".format(devices))

        self._rgb_image = rgb_image if device is None else rgb_image.to(device)
        self.device = self._rgb_image.device
        self._depth_image = depth_image.to(self.device)
        self._intrinsics = intrinsics.to(self.device)
        self._poses = poses.to(self.device) if poses is not None else None
        self._pixel_pos = pixel_pos.to(self.device) if pixel_pos is not None else None

        self._vertex_map = None
        self._global_vertex_map = None
        self._normal_map = None
        self._global_normal_map = None
        self._valid_depth_mask = None

        self._B, self._L = self._rgb_image.shape[:2]
        self.h = self._rgb_image.shape[3] if channels_first else self._rgb_image.shape[2]
        self.w = self._rgb_image.shape[4] if channels_first else self._rgb_image.shape[3]
        self.shape = (self._B, self._L, self.h, self.w)

    # ------------------------------------------------------------------ indexing / protocol
    def __getitem__(self, index):
        """Selects batch / sequence ranges; tensors are views, cached maps are sliced too (rgbdimages.py:185-236)."""
        if not isinstance(index, (tuple, int)):
            raise IndexError(index)
        if isinstance(index, int):
            sl = (slice(index, index + 1), slice(None, None))
        else:
            if len(index) > 2:
                raise IndexError("Only batch and sequences can be indexed")
            sl = tuple(slice(x, x + 1) if isinstance(x, int) else x for x in index)
            if len(sl) == 1:
                sl = (sl[0], slice(None, None))
        new_rgb = self._rgb_image[sl[0], sl[1]]
        if new_rgb.shape[0] == 0:
            raise IndexError("Incorrect indexing at dimension 0, make sure range is within 0 and {0}".format(self._B))
        if new_rgb.shape[1] == 0:
            raise IndexError("Incorrect indexing at dimension 1, make sure range is within 0 and {0}".format(self._L))
        other = RGBDImages(new_rgb, self._depth_image[sl[0], sl[1]], self._intrinsics[sl[0], :],
                           channels_first=self.channels_first)
        for k in self._INTERNAL_TENSORS:
            if k in ("_rgb_image", "_depth_image", "_intrinsics"):
                continue
            v = getattr(self, k)
            if torch.is_tensor(v):
                setattr(other, k, v[sl[0], sl[1]])
        return other

    def __len__(self):
        return self._B

    # ------------------------------------------------------------------ plain properties
    @property
    def channels_first(self):
        return self._channels_first

    @property
    def cdim(self):
        return 2 if self.channels_first else 4

    @property
    def rgb_image(self):
        return self._rgb_image

    @property
    def depth_image(self):
        return self._depth_image

    @property
    def intrinsics(self):
        return self._intrinsics

    @property
    def poses(self):
        return self._poses

    @property
    def pixel_pos(self):
        return self._pixel_pos

    @property
    def has_poses(self):
        return self._poses is not None

    @property
    def valid_depth_mask(self):
        if self._valid_depth_mask is None:
            self._valid_depth_mask = self._depth_image > 0
        return self._valid_depth_mask

    # ------------------------------------------------------------------ lazily computed maps (K1)
    def _compute_maps(self, local: bool, glob: bool):
        """One K1 launch fills every map that is missing among the requested group(s)."""
        need = [local and self._vertex_map is None, local and self._normal_map is None,
                glob and self._global_vertex_map is None, glob and self._global_normal_map is None]
        if not any(need):
            return
        depth = self._depth_image if not self.channels_first else self._depth_image.permute(0, 1, 3, 4, 2)
        outs = backproject(depth, self._intrinsics, self._poses, need)
        names = ("_vertex_map", "_normal_map", "_global_vertex_map", "_global_normal_map")
        for name, o in zip(names, outs):
            if o is not None:
                setattr(self, name, o.permute(0, 1, 4, 2, 3).contiguous() if self.channels_first else o)

    @property
    def vertex_map(self):
        if self._vertex_map is None:
            self._compute_maps(True, False)
        return self._vertex_map

    @property
    def normal_map(self):
        if self._normal_map is None:
            self._compute_maps(True, False)
        return self._normal_map

    @property
    def global_vertex_map(self):
        if self._global_vertex_map is None:
            self._compute_maps(False, True)
        return self._global_vertex_map

    @property
    def global_normal_map(self):
        if self._global_normal_map is None:
            self._compute_maps(False, True)
        return self._global_normal_map

    # ------------------------------------------------------------------ setters (cache invalidation as rgbdimages.py:399-463)
    @staticmethod
    def _assert_shape(value, shape):
        if not torch.is_tensor(value):
            raise TypeError("value must be torch.Tensor. Got {}".format(type(value)))
        if value.shape != shape:
            raise ValueError("Expected value to have shape {0}. Got {1} instead".format(shape, value.shape))

    def _drop_maps(self, local=True):
        if local:
            self._vertex_map = None
            self._normal_map = None
        self._global_vertex_map = None
        self._global_normal_map = None

    @rgb_image.setter
    def rgb_image(self, value):
        if value is not None:
            self._assert_shape(value, self._rgb_image_shape)
        self._rgb_image = value

    @depth_image.setter
    def depth_image(self, value):
        if value is not None:
            self._assert_shape(value, self._depth_image_shape)
        self._depth_image = value
        self._valid_depth_mask = None
        self._drop_maps()

    @intrinsics.setter
    def intrinsics(self, value):
        if value is not None:
            self._assert_shape(value, self._intrinsics_shape)
        self._intrinsics = value
        self._drop_maps()

    @poses.setter
    def poses(self, value):
        if value is not None:
            self._assert_shape(value, self._poses_shape)
        self._poses = value
        self._drop_maps(local=False)

    # ------------------------------------------------------------------ copies / device moves
    def clone(self):
        other = RGBDImages(self._rgb_image.clone(), self._depth_image.clone(), self._intrinsics.clone(),
                           channels_first=self.channels_first)
        for k in self._INTERNAL_TENSORS:
            if k in ("_rgb_image", "_depth_image", "_intrinsics"):
                continue
            v = getattr(self, k)
            if torch.is_tensor(v):
                setattr(other, k, v.clone())
        return other

    def detach(self):
        other = self.clone()
        for k in self._INTERNAL_TENSORS:
            v = getattr(self, k)
            if torch.is_tensor(v):
                setattr(other, k, v.detach())
        return other

    def to(self, device: Union[torch.device, str], copy: bool = False):
        device = torch.empty(0, device=device).device
        if not copy and self.device == device:
            return self
        other = self.clone()
        other.device = device
        for k in self._INTERNAL_TENSORS:
            v = getattr(self, k)
            if torch.is_tensor(v):
                setattr(other, k, v.to(device))
        other._valid_depth_mask = None
        return other

    def cpu(self):
        return self.to(torch.device("cpu"))

    def cuda(self):
        return self.to(torch.device("cuda"))

    # ------------------------------------------------------------------ layout
    def to_channels_last(self, copy: bool = False):
        if not (copy or self.channels_first):
            return self
        return self.clone().to_channels_last_()

    def to_channels_first(self, copy: bool = False):
        if not copy and self.channels_first:
            return self
        return self.clone().to_channels_first_()

    def _permute_all(self, order):
        for k in ("_rgb_image", "_depth_image", "_vertex_map", "_global_vertex_map", "_normal_map",
                  "_global_normal_map"):
            v = getattr(self, k)
            if v is not None:
                setattr(self, k, v.permute(*order).contiguous())
        self._valid_depth_mask = None
        self._rgb_image_shape = tuple(self._rgb_image.shape)
        self._depth_image_shape = tuple(self._depth_image.shape)
        self._depth_shape = self._depth_image_shape

    def to_channels_last_(self):
        if not self.channels_first:
            return self
        self._permute_all((0, 1, 3, 4, 2))
        self._channels_first = False
        return self

    def to_channels_first_(self):
        if self.channels_first:
            return self
        self._permute_all((0, 1, 4, 2, 3))
        self._channels_first = True
        return self
