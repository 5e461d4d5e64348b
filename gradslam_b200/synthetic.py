"""Deterministic synthetic RGB-D sequences (SURVEY.md §8d): a camera moving inside an axis-aligned
box room, depth by analytic ray/box intersection, so frames are mutually consistent and ICP sees at
least three non-parallel planes.  Everything is float32, channels-last, generated on the CPU from a
seeded `torch.Generator` so the same tensors come out on every machine.

This is input generation for tests and bench.py — it is not part of the hot path.
"""
import math

import numpy as np
import torch

ROOM_HALF_EXTENTS = (2.0, 1.5, 3.0)  # metres; camera 0 sits at the room centre (+ 2 mm * b in x)


def intrinsics(H, W):
    fx = 525.0 * W / 640.0
    K = np.eye(4, dtype=np.float64)
    K[0, 0] = fx
    K[1, 1] = fx
    K[0, 2] = (W - 1) / 2.0
    K[1, 2] = (H - 1) / 2.0
    return K


def _room_from_cam(s, b, motion_scale=1.0, yaw0=0.0):
    """Camera-to-room transform of frame s, element b: yaw yaw0 + 0.01*s rad, t = (0.01 s + 0.002 b, 0.005 s, 0.008 s)."""
    a = yaw0 + 0.01 * s * motion_scale
    T = np.eye(4, dtype=np.float64)
    T[0, 0], T[0, 2] = math.cos(a), math.sin(a)
    T[2, 0], T[2, 2] = -math.sin(a), math.cos(a)
    T[:3, 3] = (0.01 * s * motion_scale + 0.002 * b, 0.005 * s * motion_scale, 0.008 * s * motion_scale)
    return T


def _camera_rays(H, W):
    """(H,W,3) camera-frame ray directions of intrinsics(H, W) with unit z, so a ray's parameter is its z-depth."""
    K = intrinsics(H, W)
    fx, fy, cx, cy = K[0, 0], K[1, 1], K[0, 2], K[1, 2]
    return np.stack(
        np.broadcast_arrays((np.arange(W)[None, :] - cx) / fx, (np.arange(H)[:, None] - cy) / fy, np.ones((H, W))), -1
    )


def _wall_exit(T, dirs):
    """(H,W,3) ray parameter at which each ray of the camera T (camera-to-room) leaves the room through the pair of walls
    normal to room axis 0, 1, 2; the depth is the minimum over the axes."""
    d_room = dirs @ T[:3, :3].T
    o = T[:3, 3]
    half = np.asarray(ROOM_HALF_EXTENTS)
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.where(d_room > 0, (half - o) / d_room, np.where(d_room < 0, (-half - o) / d_room, np.inf))


def make_sequence(B, L, H, W, seed=0, hole_fraction=0.02, motion_scale=1.0, pin_memory=False,
                  yaw0=0.0):
    """Returns (rgb (B,L,H,W,3), depth (B,L,H,W,1), intrinsics (B,1,4,4), poses (B,L,4,4)), all float32 CPU.

    poses are camera-to-world with frame 0 of every element at identity (world = camera 0).

    yaw0 turns the first camera about the vertical axis.  With yaw0 = 0 (SURVEY.md's scene) the 62-degree
    horizontal field of view only sees the far wall, so point-to-plane ICP observes 3 of the 6 degrees of
    freedom and drifts (the reference drifts identically); yaw0 ~ 0.6 looks into a corner (two walls + floor /
    ceiling) and makes ICP well conditioned."""
    gen = torch.Generator().manual_seed(int(seed))
    dirs = _camera_rays(H, W)
    depth = torch.empty((B, L, H, W, 1), dtype=torch.float32, pin_memory=pin_memory)
    poses = torch.empty((B, L, 4, 4), dtype=torch.float32)
    for b in range(B):
        T0_inv = np.linalg.inv(_room_from_cam(0, b, motion_scale, yaw0))
        for s in range(L):
            T = _room_from_cam(s, b, motion_scale, yaw0)
            depth[b, s, :, :, 0] = torch.from_numpy(_wall_exit(T, dirs).min(-1).astype(np.float32))
            poses[b, s] = torch.from_numpy((T0_inv @ T).astype(np.float32))
    if hole_fraction > 0:
        holes = torch.rand((B, L, H, W, 1), generator=gen) < hole_fraction
        depth[holes] = 0.0
    rgb = torch.empty((B, L, H, W, 3), dtype=torch.float32, pin_memory=pin_memory)
    torch.rand((B, L, H, W, 3), generator=gen, out=rgb)
    Kt = torch.from_numpy(intrinsics(H, W).astype(np.float32)).view(1, 1, 4, 4).repeat(B, 1, 1, 1)
    return rgb, depth, Kt, poses


# wall texture of make_textured_sequence: channel c at in-wall coordinates (a, b) (metres) is
# 0.5 + 0.4 sin(2 pi a / la_c + pa_c) sin(2 pi b / lb_c + pb_c)
TEXTURE_WAVELENGTHS = ((0.30, 0.45), (0.40, 0.25), (0.55, 0.35))
TEXTURE_PHASES = ((0.3, 1.1), (2.0, 0.4), (1.3, 2.6))


def make_textured_sequence(B, L, H, W, seed=0, hole_fraction=0.02, motion_scale=1.0, yaw0=0.0):
    """make_sequence(B, L, H, W, seed, ...) with a painted room: the same depth, holes, poses and intrinsics, but the
    colour of a pixel is a smooth function of the room-frame point its ray meets (products of sinusoids of the two
    in-wall coordinates, TEXTURE_WAVELENGTHS / TEXTURE_PHASES), so a surface point has the same colour in every frame.
    Hole pixels are coloured as if they had depth.  Everything is deterministic; seed only drives make_sequence's holes."""
    for name, v in (("B", B), ("L", L), ("H", H), ("W", W)):
        if isinstance(v, bool) or not isinstance(v, int):
            raise TypeError("{} must be an int; got {}".format(name, type(v)))
        if v < 1:
            raise ValueError("{} must be >= 1; got {}".format(name, v))
    if not math.isfinite(float(yaw0)) or not math.isfinite(float(motion_scale)):
        raise ValueError("yaw0 and motion_scale must be finite")
    _, depth, Kt, poses = make_sequence(B, L, H, W, seed=seed, hole_fraction=hole_fraction, motion_scale=motion_scale,
                                        yaw0=yaw0)
    dirs = _camera_rays(H, W)
    rgb = torch.empty((B, L, H, W, 3), dtype=torch.float32)
    for b in range(B):
        for s in range(L):
            T = _room_from_cam(s, b, motion_scale, yaw0)
            t_exit = _wall_exit(T, dirs)
            axis = t_exit.argmin(-1)  # the wall the ray meets
            p = T[:3, 3] + t_exit.min(-1)[..., None] * (dirs @ T[:3, :3].T)  # room-frame surface point
            a = np.where(axis == 0, p[..., 1], p[..., 0])
            c = np.where(axis == 2, p[..., 1], p[..., 2])
            col = [0.5 + 0.4 * np.sin(2 * math.pi * a / la + pa) * np.sin(2 * math.pi * c / lb + pb)
                   for (la, lb), (pa, pb) in zip(TEXTURE_WAVELENGTHS, TEXTURE_PHASES)]
            rgb[b, s] = torch.from_numpy(np.stack(col, -1).astype(np.float32))
    return rgb, depth, Kt, poses


# the box of make_dynamic_sequence, in room coordinates (metres): in front of the far wall (z = 3), in view of camera 0
DYNAMIC_BOX_CENTER = (0.0, 0.0, 2.0)
DYNAMIC_BOX_HALF_EXTENTS = (0.5, 0.5, 0.25)


def make_dynamic_sequence(B, L, H, W, k0, k1, seed=0, hole_fraction=0.02, motion_scale=1.0, pin_memory=False, yaw0=0.0,
                          box_center=DYNAMIC_BOX_CENTER, box_half_extents=DYNAMIC_BOX_HALF_EXTENTS):
    """make_sequence's room with an axis-aligned box that is there only in frames [k0, k1): a scene that changes.
    Same return values, cameras, colours and holes as make_sequence(B, L, H, W, seed, ...); in frames [k0, k1) a valid
    pixel whose ray meets the box first sees the box instead of the wall."""
    rgb, depth, Kt, poses = make_sequence(B, L, H, W, seed=seed, hole_fraction=hole_fraction,
                                          motion_scale=motion_scale, pin_memory=pin_memory, yaw0=yaw0)
    K = intrinsics(H, W)
    dirs = np.stack(
        np.broadcast_arrays((np.arange(W)[None, :] - K[0, 2]) / K[0, 0], (np.arange(H)[:, None] - K[1, 2]) / K[1, 1],
                            np.ones((H, W))), -1)
    lo = np.asarray(box_center) - np.asarray(box_half_extents)
    hi = np.asarray(box_center) + np.asarray(box_half_extents)
    for b in range(B):
        for s in range(max(k0, 0), min(k1, L)):
            T = _room_from_cam(s, b, motion_scale, yaw0)
            d_room = dirs @ T[:3, :3].T
            o = T[:3, 3]
            with np.errstate(divide="ignore", invalid="ignore"):  # slab test; a ray parallel to a slab gives +-inf
                t1, t2 = (lo - o) / d_room, (hi - o) / d_room
                t_in = np.nan_to_num(np.minimum(t1, t2), nan=-np.inf).max(-1)
                t_out = np.nan_to_num(np.maximum(t1, t2), nan=np.inf).min(-1)
            t_box = torch.from_numpy(np.where((t_out >= t_in) & (t_in > 0), t_in, np.inf).astype(np.float32))
            d = depth[b, s, :, :, 0]
            depth[b, s, :, :, 0] = torch.where((d > 0) & (t_box < d), t_box, d)
    return rgb, depth, Kt, poses


def add_depth_noise(depth, seed, a=0.0012, b=0.0019, z0=0.4):
    """depth (any shape, float32, CPU) plus the axial noise of a Kinect v1 (Nguyen, Izadi and Lovell 2012): independent
    zero-mean Gaussian noise of sigma(z) = a + b (z - z0)^2 metres per pixel, from a torch.Generator seeded with `seed`.
    Holes (depth 0) stay 0, and a noisy depth is clamped to at least a tenth of the clean one, so no valid pixel becomes
    a hole.  Real sensors' noise is spatially correlated and quantised: independent noise is the harsher case."""
    gen = torch.Generator().manual_seed(int(seed))
    noise = torch.randn(depth.shape, generator=gen, dtype=torch.float32)
    d64 = depth.double()
    sigma = a + b * (d64 - z0) ** 2
    noisy = torch.maximum(d64 + sigma * noise.double(), 0.1 * d64)
    return torch.where(depth > 0, noisy, d64).to(torch.float32)


def punch_lattice_holes(depth, row_step=5, col_step=7):
    """Zeroes depth (..., H, W, 1) on a sparse lattice (rows 2, 2+row_step, ...; columns 3, 3+col_step, ...).  No two
    holes touch, not even diagonally, so no valid pixel has BOTH its right and its lower neighbour missing: at such
    pixels the normal is the normalised rounding residue of a cancelling cross product (see gsx_common.cuh cross_ref) and
    its derivative is ~1e7 - fine for parity fixtures, useless for checking gradient FORMULAS against autograd."""
    depth = depth.clone()
    depth[..., 2::row_step, 3::col_step, :] = 0.0
    return depth
