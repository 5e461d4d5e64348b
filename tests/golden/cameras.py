"""Seeded inputs in which every batch element has its own camera (shared by make_golden_cameras.py, which freezes the
reference's outputs for them, and by the CPU / GPU tests, which rebuild the same inputs).

make_sequence gives every element the same intrinsics and, bit for bit, the same poses, so a kernel that read element
0's camera for every element would pass on it.  Here each element has its own fx != fy, an off-centre principal point,
optionally a skew K[0,1] and a 4th column K[0:2,3] (back-projection ignores both, as the reference's inverse_intrinsics
does; projection uses all twelve entries), its own yaw, yaw rate and direction of motion, and elements 1.. start at a
pose that is not the identity.  Depth is cast through each element's own camera into the box room of synthetic.py.
Depends on gradslam_b200.synthetic only."""
import math

import numpy as np
import torch

from gradslam_b200.synthetic import ROOM_HALF_EXTENTS, punch_lattice_holes


class CameraShape(tuple):
    """The (B, L, H, W) of a parametrized GPU test whose inputs come from camera_inputs instead of make_sequence."""


def camera_intrinsics(B, H, W, skew=0.0):
    """float64 (B, 4, 4): element b has fx = f (1 + 0.06 b), fy = 0.93 fx, a principal point 1.5 + b pixels off
    centre, and with skew != 0 K[0,1] = skew (b + 1), K[0,3] = 0.3 + 0.2 b, K[1,3] = -0.25 - 0.15 b."""
    K = np.tile(np.eye(4), (B, 1, 1))
    for b in range(B):
        fx = 525.0 * W / 640.0 * (1.0 + 0.06 * b)
        K[b, 0, 0] = fx
        K[b, 1, 1] = 0.93 * fx
        K[b, 0, 2] = (W - 1) / 2.0 + (1.5 + b) * (-1) ** b
        K[b, 1, 2] = (H - 1) / 2.0 - 0.5 * (1.5 + b)
        if skew:
            K[b, 0, 1] = skew * (b + 1)
            K[b, 0, 3] = 0.3 + 0.2 * b
            K[b, 1, 3] = -0.25 - 0.15 * b
    return K


def room_from_cam(b, s):
    """float64 camera-to-room transform of element b at frame s.  Elements alternate between the two far corners
    (yaw +-(0.6 + 0.05 b), like synthetic.py's yaw0 = 0.6) and turn at their own rate; each translates along its own
    direction (synthetic.py's (1, 0.5, 0.8) cm per frame, turned by 1.3 b rad about the vertical, scaled by 1 + 0.25 b)
    from its own start point."""
    sign = (-1) ** b
    a = sign * (0.6 + 0.05 * b) + 0.01 * (1.0 + 0.5 * b) * s * sign
    phi = 1.3 * b
    v = np.array([0.01 * math.cos(phi) + 0.008 * math.sin(phi), 0.005, -0.01 * math.sin(phi) + 0.008 * math.cos(phi)])
    T = np.eye(4)
    T[0, 0], T[0, 2] = math.cos(a), math.sin(a)
    T[2, 0], T[2, 2] = -math.sin(a), math.cos(a)
    T[:3, 3] = np.array([0.05 * b, -0.03 * b, -0.04 * b]) + s * (1.0 + 0.25 * b) * v
    return T


def camera_poses(B, L):
    """float64 (B, L, 4, 4) camera-to-world poses: element 0 relative to its first frame (identity at s = 0), the other
    elements in room coordinates (their first pose is not the identity)."""
    poses = np.empty((B, L, 4, 4))
    for b in range(B):
        to_world = np.linalg.inv(room_from_cam(b, 0)) if b == 0 else np.eye(4)
        for s in range(L):
            poses[b, s] = to_world @ room_from_cam(b, s)
    return poses


def camera_inputs(B, L, H, W, seed, skew=0.0, lattice_holes=False):
    """Returns (rgb (B,L,H,W,3), depth (B,L,H,W,1), intrinsics (B,1,4,4), poses (B,L,4,4)), all float32 CPU, like
    make_sequence.  2 % random depth holes, or with lattice_holes=True none but punch_lattice_holes' lattice (for
    gradient checks)."""
    gen = torch.Generator().manual_seed(int(seed))
    K = camera_intrinsics(B, H, W, skew)
    half = np.asarray(ROOM_HALF_EXTENTS)
    depth = torch.empty((B, L, H, W, 1), dtype=torch.float32)
    for b in range(B):
        fx, fy, cx, cy = K[b, 0, 0], K[b, 1, 1], K[b, 0, 2], K[b, 1, 2]
        dirs = np.stack(np.broadcast_arrays((np.arange(W)[None, :] - cx) / fx, (np.arange(H)[:, None] - cy) / fy,
                                            np.ones((H, W))), -1)  # unit z: the ray parameter is the z-depth
        for s in range(L):
            T = room_from_cam(b, s)
            d_room = dirs @ T[:3, :3].T
            o = T[:3, 3]
            with np.errstate(divide="ignore", invalid="ignore"):
                t_exit = np.where(d_room > 0, (half - o) / d_room, np.where(d_room < 0, (-half - o) / d_room, np.inf))
            depth[b, s, :, :, 0] = torch.from_numpy(t_exit.min(-1).astype(np.float32))
    if lattice_holes:
        depth = punch_lattice_holes(depth)
    else:
        depth[torch.rand((B, L, H, W, 1), generator=gen) < 0.02] = 0.0
    rgb = torch.rand((B, L, H, W, 3), generator=gen)
    Kt = torch.from_numpy(K.astype(np.float32)).view(B, 1, 4, 4)
    return rgb, depth, Kt, torch.from_numpy(camera_poses(B, L).astype(np.float32))


# Reference runs frozen by make_golden_cameras.py: (name, class, B, L, H, W, seed, camera_inputs kwargs, slam kwargs)
CAMERA_CASES = [
    ("cam_pf_gt", "PointFusion", 3, 4, 48, 64, 51, dict(), dict(odom="gt")),
    ("cam_pf_gt_skew", "PointFusion", 3, 4, 48, 64, 51, dict(skew=0.75), dict(odom="gt")),
    ("cam_pf_icp", "PointFusion", 3, 3, 48, 64, 52, dict(), dict(odom="icp", numiters=8, dsratio=2)),
    ("cam_pf_gradicp", "PointFusion", 3, 3, 48, 64, 53, dict(), dict(odom="gradicp", numiters=8, dsratio=2)),
    ("cam_icpslam_gradicp", "ICPSLAM", 3, 3, 48, 64, 54, dict(), dict(odom="gradicp", numiters=5, dsratio=2)),
]
# every SAMPLE_STRIDE-th row of each frozen map is stored (with float64 sums of all rows)
SAMPLE_STRIDE = 53  # (as fullsize.py samples the full-size run)
# the three correspondence tables of one fusion step (frames 0 and 1 fused, tables of frame 2), skew and 4th column set
TABLES_CASE = dict(B=3, L=3, H=48, W=64, seed=55, skew=0.75)


def frozen_table(ref, name):
    """Table `name` (active, similar or unique) of ref_cameras.npz as the int64 (rows, 4) tensor the reference returned:
    the file holds active and unique column-major as int32, and similar as its mask over the active rows."""
    if name == "similar":
        return frozen_table(ref, "active")[torch.from_numpy(ref["tables/similar_mask"])]
    return torch.from_numpy(ref["tables/" + name].T.astype(np.int64))
