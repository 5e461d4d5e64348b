"""RGBDImages: batched RGB-D sequence container with lazily computed vertex / normal maps.

Host-side mirror of gradslam.RGBDImages (gradslam/structures/rgbdimages.py:13-915): same constructor,
properties, indexing and error behaviour.  The four cached maps are produced by ONE hand-written sm_90a
kernel (gsx_backproject_normals_fwd) instead of the reference's einsum / slice / cross / norm chain
(rgbdimages.py:643-762).  Containers may hold tensors on any device, but computing a map requires CUDA
tensors: there is no CPU compute path.
"""
import math
from dataclasses import dataclass
from typing import Optional, Union

import numpy as np
import torch

from .. import _C

__all__ = ["RGBDImages", "BilateralFilter", "bilateral_filter_depth"]


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
    forward = gsx_backproject_normals_fwd, backward = gsx_backproject_normals_bwd (d/d depth, d/d poses), or
    gsx_backproject_normals_bwd_intrinsics when the intrinsics require grad (also d/d fx, cx, fy, cy)."""

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
        ctx.K_shape = intrinsics.shape
        return tuple(outs)

    @staticmethod
    def backward(ctx, g_v, g_n, g_gv, g_gn):
        d, d_bs, K, P, (B, L, H, W) = ctx.saved
        dev = d.device
        gs = [None if g is None else g.contiguous() for g in (g_v, g_n, g_gv, g_gn)]
        g_depth = torch.empty((B, L, H, W, 1), dtype=torch.float32, device=dev)
        g_poses = torch.empty((B, L, 4, 4), dtype=torch.float32, device=dev) if ctx.need_pose else None
        if ctx.needs_input_grad[1]:
            g_K = torch.zeros((B, 4, 4), dtype=torch.float32, device=dev)  # (B*L == 0 launches nothing)
            nbytes = _C.lib().gsx_backproject_normals_bwd_intrinsics_scratch_bytes(B, L, H, W)
            scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
            _C.launch("gsx_backproject_normals_bwd_intrinsics", d, d_bs, K, 16, P, L * 16, B, L, H, W, *gs, g_depth,
                      g_poses, g_K, scratch, nbytes)
            return g_depth, g_K.view(ctx.K_shape), g_poses, None
        nbytes = _C.lib().gsx_backproject_normals_bwd_scratch_bytes(B, L, H, W)
        scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev) if ctx.need_pose else None
        _C.launch("gsx_backproject_normals_bwd", d, d_bs, K, 16, P, L * 16, B, L, H, W, *gs, g_depth, g_poses, scratch,
                  nbytes if ctx.need_pose else 0)
        return g_depth, None, g_poses, None


def backproject(depth, intrinsics, poses, want=(True, True, True, True)):
    """Runs K1.  depth (B,L,H,W,1) channels-last.  Returns a 4-tuple (entries not wanted are None)."""
    return _BackprojectFn.apply(depth, intrinsics, poses, tuple(bool(w) for w in want))


_MAX_FILTER_RADIUS = 7


@dataclass(frozen=True)
class BilateralFilter:
    """Edge-preserving bilateral filter of input depth (KinectFusion, Newcombe et al. 2011), as gsx_depth_bilateral
    computes it: each valid pixel (0 < d < inf) becomes the mean of the valid depths in its (2 radius + 1)^2 window,
    weighted by exp(-(du^2 + dv^2) / (2 sigma_space^2) - (d_q - d_p)^2 / (2 sigma_range^2)); invalid pixels (holes,
    NaN, inf) stay as they are.  radius: pixels, 1 .. 7; sigma_space: pixels; sigma_range: metres (depth units).
    A depth step much larger than sigma_range keeps both sides apart."""

    radius: int
    sigma_space: float
    sigma_range: float

    def __post_init__(self):
        if isinstance(self.radius, bool) or not isinstance(self.radius, int):
            raise TypeError("BilateralFilter.radius must be an int; got {}".format(type(self.radius)))
        if not 1 <= self.radius <= _MAX_FILTER_RADIUS:
            raise ValueError("BilateralFilter.radius must be in 1..{}; got {}".format(_MAX_FILTER_RADIUS, self.radius))
        for name in ("sigma_space", "sigma_range"):
            v = getattr(self, name)
            if isinstance(v, bool) or not isinstance(v, (float, int)):
                raise TypeError("BilateralFilter.{} must be a float; got {}".format(name, type(v)))
            ok = math.isfinite(float(v)) and v > 0
            if ok:  # the kernel takes c = 1/(2 sigma^2) rounded once to float32: finite and non-zero there too
                two_var = 2.0 * float(v) * float(v)
                with np.errstate(over="ignore", under="ignore"):
                    c = np.float32(1.0 / two_var) if two_var > 0 else np.float32(np.inf)
                ok = bool(np.isfinite(c) and c > 0)
            if not ok:
                raise ValueError("BilateralFilter.{} must be finite and > 0 with 1/(2 sigma^2) a finite positive "
                                 "float32; got {}".format(name, v))
            object.__setattr__(self, name, float(v))


def _depth_layout(depth):
    """(B,L,H,W,1) channels-last or (B,L,1,H,W) channels-first -> (n images, H, W); the two hold the same bytes."""
    if depth.dim() != 5 or not (depth.shape[-1] == 1 or depth.shape[2] == 1):
        raise ValueError("depth must be (B,L,H,W,1) or (B,L,1,H,W); got shape {}".format(tuple(depth.shape)))
    B, L = depth.shape[:2]
    H, W = (depth.shape[2], depth.shape[3]) if depth.shape[-1] == 1 else (depth.shape[3], depth.shape[4])
    return B * L, H, W


class _BilateralFn(torch.autograd.Function):
    """depth -> filtered depth.  forward = gsx_depth_bilateral, backward = gsx_depth_bilateral_bwd (it needs the
    forward's per-pixel weight sums, which are kept only when depth requires grad)."""

    @staticmethod
    def forward(ctx, depth, f):
        _C.require_cuda(depth, "depth")
        n, H, W = _depth_layout(depth)
        d = depth.detach().contiguous()
        out = torch.empty_like(d, memory_format=torch.contiguous_format)
        den = torch.empty_like(d, memory_format=torch.contiguous_format) if ctx.needs_input_grad[0] else None
        if n * H * W > 0:
            _C.launch("gsx_depth_bilateral", d, out, den, n, H, W, f.radius, f.sigma_space, f.sigma_range)
        if den is not None:
            ctx.save_for_backward(d, out, den)
        ctx.f, ctx.dims = f, (n, H, W)
        return out

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, g_out):
        d, out, den = ctx.saved_tensors
        f, (n, H, W) = ctx.f, ctx.dims
        g_depth = torch.empty_like(d)
        if n * H * W > 0:
                _C.launch("gsx_depth_bilateral_bwd", d, out, den, g_out.contiguous(), g_depth, n, H, W, f.radius,
                      f.sigma_space, f.sigma_range)
        return g_depth, None


def bilateral_filter_depth(depth: torch.Tensor, f: BilateralFilter) -> torch.Tensor:
    """Bilateral filter (`f`) of a CUDA float32 depth tensor, (B,L,H,W,1) channels-last or (B,L,1,H,W) channels-first;
    returns a new tensor of the same shape.  Differentiable w.r.t. depth (exact, deterministic backward)."""
    if not isinstance(f, BilateralFilter):
        raise TypeError("Expected f to be of type BilateralFilter. Got {}.".format(type(f)))
    return _BilateralFn.apply(depth, f)


_EMBED_DTYPES = (torch.float32, torch.float16, torch.bfloat16)


def _check_embedding_image(e, rgb_shape, cdim):
    """(B, L, H, W, D) channels-last (cdim 4) or (B, L, D, H, W) channels-first (cdim 2) beside rgb of rgb_shape."""
    if not torch.is_tensor(e):
        raise TypeError("Expected embeddings to be of type tensor or None; got {}".format(type(e)))
    if e.dtype not in _EMBED_DTYPES:
        raise TypeError("embeddings must be float32, float16 or bfloat16; got {}".format(e.dtype))
    if e.ndim != 5:
        raise ValueError("embeddings should have ndim=5, but had ndim={}".format(e.ndim))
    D = e.shape[cdim]
    exp = tuple(v if i != cdim else D for i, v in enumerate(rgb_shape))
    if D < 1 or tuple(e.shape) != exp:
        raise ValueError("Expected embeddings to have shape {0} with D >= 1 ({1}). Got {2} instead".format(
            tuple("D" if i == cdim else v for i, v in enumerate(exp)),
            "(B, L, D, H, W)" if cdim == 2 else "(B, L, H, W, D)", tuple(e.shape)))


def _check_coarse_embedding_image(e, rgb_shape, cdim):
    """(B, L, h, w, D) channels-last (cdim 4) or (B, L, D, h, w) channels-first (cdim 2), 1 <= h <= H, 1 <= w <= W, an
    embedding image that the fused map update upsamples bilinearly to the (H, W) of rgb_shape."""
    if not torch.is_tensor(e):
        raise TypeError("Expected embeddings to be of type tensor or None; got {}".format(type(e)))
    if e.dtype not in _EMBED_DTYPES:
        raise TypeError("embeddings must be float32, float16 or bfloat16; got {}".format(e.dtype))
    if e.ndim != 5:
        raise ValueError("embeddings should have ndim=5, but had ndim={}".format(e.ndim))
    sp = (2, 3) if cdim == 4 else (3, 4)  # (h, w) dimensions of e
    D, (h, w) = e.shape[cdim], (e.shape[sp[0]], e.shape[sp[1]])
    H, W = rgb_shape[sp[0]], rgb_shape[sp[1]]
    if tuple(e.shape[:2]) != tuple(rgb_shape[:2]) or D < 1 or not (1 <= h <= H and 1 <= w <= W):
        raise ValueError("Expected upsampled embeddings to have shape {0} with D >= 1, 1 <= h <= {1} and 1 <= w <= {2}. "
                         "Got {3} instead".format("(B, L, D, h, w)" if cdim == 2 else "(B, L, h, w, D)", H, W,
                                                  tuple(e.shape)))


class RGBDImages(object):
    _INTERNAL_TENSORS = [
        "_rgb_image", "_depth_image", "_intrinsics", "_poses", "_pixel_pos",
        "_vertex_map", "_normal_map", "_global_vertex_map", "_global_normal_map", "_embeddings",
    ]

    def __init__(self, rgb_image: torch.Tensor, depth_image: torch.Tensor, intrinsics: torch.Tensor,
                 poses: Optional[torch.Tensor] = None, channels_first: bool = False,
                 device: Union[torch.device, str, None] = None, *, pixel_pos: Optional[torch.Tensor] = None,
                 embeddings: Optional[torch.Tensor] = None, upsample_embeddings: bool = False):
        """embeddings (extension): a per-pixel embedding image at the depth's resolution, (B, L, H, W, D) or, with
        channels_first, (B, L, D, H, W), D >= 1, in float32, float16 or bfloat16, on the frames' device.  The fused map
        update keeps a confidence-weighted mean of it per surfel (Pointclouds.embeddings_padded).
        upsample_embeddings (extension, default False): the embedding image is coarser than the depth, (B, L, h, w, D)
        or (B, L, D, h, w) with 1 <= h <= H and 1 <= w <= W (a CLIP or DINO feature grid), and the map update samples
        it bilinearly at each pixel it fuses, as F.interpolate(e, (H, W), mode='bilinear', align_corners=False) would,
        without forming the full-resolution image."""
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
        if not isinstance(upsample_embeddings, bool):
            raise TypeError("Expected upsample_embeddings to be of type bool; got {}".format(type(upsample_embeddings)))
        if upsample_embeddings:
            if embeddings is None:
                raise ValueError("upsample_embeddings=True needs an embedding image (embeddings=...)")
            _check_coarse_embedding_image(embeddings, rgb_image.shape, cdim)
        elif embeddings is not None:
            _check_embedding_image(embeddings, rgb_image.shape, cdim)

        devices = set(x.device for x in (rgb_image, depth_image, intrinsics, poses, pixel_pos, embeddings)
                      if x is not None)
        if len(devices) != 1:
            raise ValueError("All inputs must be on same device, but got more than 1 device: {}".format(devices))

        self._rgb_image = rgb_image if device is None else rgb_image.to(device)
        self.device = self._rgb_image.device
        self._depth_image = depth_image.to(self.device)
        self._intrinsics = intrinsics.to(self.device)
        self._poses = poses.to(self.device) if poses is not None else None
        self._pixel_pos = pixel_pos.to(self.device) if pixel_pos is not None else None
        self._embeddings = embeddings.to(self.device) if embeddings is not None else None
        self._upsample_embeddings = upsample_embeddings

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
        other._upsample_embeddings = self._upsample_embeddings
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
    def embeddings(self):
        """The per-pixel embedding image (B, L, H, W, D) ((B, L, D, H, W) channels-first), or None; with
        upsample_embeddings, the coarse (B, L, h, w, D) image."""
        return self._embeddings

    @property
    def upsample_embeddings(self):
        """True when the embedding image is coarser than the depth and is upsampled bilinearly where it is fused."""
        return self._upsample_embeddings

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

    # ------------------------------------------------------------------ depth filtering
    def bilateral_filtered(self, f: BilateralFilter):
        """A new RGBDImages whose depth is bilateral_filter_depth(depth_image, f), with the same rgb, intrinsics,
        poses and pixel positions (not copies).  Differentiable w.r.t. the depth."""
        if self.channels_first:  # (filtered as channels-last: a (B,L,1,H,1) shape alone does not say which it is)
            depth = bilateral_filter_depth(self._depth_image.permute(0, 1, 3, 4, 2), f).permute(0, 1, 4, 2, 3)
        else:
            depth = bilateral_filter_depth(self._depth_image, f)
        return RGBDImages(self._rgb_image, depth, self._intrinsics, self._poses, channels_first=self.channels_first,
                          pixel_pos=self._pixel_pos, embeddings=self._embeddings,
                          upsample_embeddings=self._upsample_embeddings)

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
        other._upsample_embeddings = self._upsample_embeddings
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
                  "_global_normal_map", "_embeddings"):
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
