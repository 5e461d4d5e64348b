"""CPU oracle of surfel radii (PointFusion with surfel_radii=True), built on gsx_oracle's fusion step, which it leaves
as it is: the radius column is carried beside the oracle's SurfelMap, per element a float32 (N_b, 1) tensor.

    pixel radius    s = 0.5 (k00 + k11), r0 = (sqrt(2) d) s, r = 2 r0 where 2|n_z| <= 1, else r0 / |n_z|
                    (d the pixel's depth, n its camera-frame normal, k00 / k11 the diagonal of inverse_intrinsics)
    append          the new row's radius is r
    merge           ((c0 r_row) + (alpha r)) inv with the merge's c0, alpha and inv; a row of radius 0 takes r
    prune           the radius goes with its row (prune_oracle / free_space_oracle's kept indices)

Every operation is a separate float32 torch op, rounded on its own, as the kernels compute it."""
import math

import torch

import free_space_oracle as fo
import gsx_oracle as oracle
import prune_oracle as po

F32 = torch.float32
SQRT2_F = torch.tensor(math.sqrt(2.0), dtype=F32)  # sqrt(2) rounded to float32


def surfel_radius(d, nz, k00, k11):
    """Radius of the surfel a pixel of depth d and camera-frame normal z component nz creates (broadcasting)."""
    s = 0.5 * (k00 + k11)
    r0 = (SQRT2_F * d) * s
    a = nz.abs()
    return torch.where(2.0 * a <= 1.0, 2.0 * r0, r0 / a)


def merge_radius(r_row, r, c0, alpha):
    """A merged row's radius: the merge's confidence-weighted mean, or r where the row has none (0)."""
    tot = c0 + alpha
    inv = 1 / torch.where(tot == 0, torch.ones_like(tot), tot)
    return torch.where(r_row == 0, r, ((c0 * r_row) + (alpha * r)) * inv)


def radius_image(depth, maps, K):
    """float32 (B,H,W) radius of every pixel of frame 0 of depth (B,1,H,W,1); maps = frame_maps(depth, K, ...)."""
    Kinv = oracle.inverse_intrinsics(K)  # (B,1,4,4)
    B = depth.shape[0]
    k00 = Kinv[:, 0, 0, 0].view(B, 1, 1)
    k11 = Kinv[:, 0, 1, 1].view(B, 1, 1)
    return surfel_radius(depth[:, 0, ..., 0], maps["normal"][:, 0, ..., 2], k00, k11)


def fuse_radii(smap, radii, maps, depth, K, pc2im, sigma):
    """The radii of oracle.fuse_with_map(smap, maps, rgb, pc2im, sigma): radii = smap's (None for an empty map)."""
    r_pix = radius_image(depth, maps, K)
    alpha = oracle.get_alpha(maps["vertex"][:, 0], sigma)[..., 0]
    valid = maps["valid"][:, 0]
    B = valid.shape[0]
    out = [r.clone() for r in radii] if smap.has_points else [torch.zeros((0, 1), dtype=F32) for _ in range(B)]
    new_mask = torch.ones_like(valid)
    if smap.has_points and pc2im.shape[0] != 0:
        b, n, h, w = pc2im.unbind(1)
        for i in range(B):
            sel = b == i
            ni, hi, wi = n[sel], h[sel], w[sel]
            out[i][ni, 0] = merge_radius(out[i][ni, 0], r_pix[i, hi, wi], smap.ccounts[i][ni, 0], alpha[i, hi, wi])
        new_mask[b, h, w] = False
    new_mask = new_mask & valid
    return [torch.cat([out[i], r_pix[i][new_mask[i]].unsqueeze(1)], 0) for i in range(B)]


def run_pointfusion(rgb, depth, K, poses, *, c_stable=None, t_max=None, margin=None, dist_th=0.05, angle_th=20.0,
                    sigma=0.6):
    """free_space_oracle.run_pointfusion with odom='gt' (c_stable None: no pruning; margin None: the age rule alone),
    with the radii.  Returns (PrunedMap, radii: per element float32 (N_b, 1))."""
    L = depth.shape[1]
    dot_th = math.cos(angle_th * math.pi / 180)
    pm = po.PrunedMap()
    radii = None
    K4 = K[:, 0]
    for s in range(L):
        d, c, pose = depth[:, s:s + 1], rgb[:, s:s + 1], poses[:, s]
        maps = oracle.frame_maps(d, K, pose.unsqueeze(1))
        table = oracle.find_correspondences(pm.smap, maps, pose, K4, dist_th, dot_th)
        radii = fuse_radii(pm.smap, radii, maps, d, K, table, sigma)
        pm.smap = oracle.fuse_with_map(pm.smap, maps, c, table, sigma)
        if c_stable is not None:
            extra = None
            if margin is not None:
                bound = fo.bound_image(pm.smap, table, pose, K4, depth.shape[2], depth.shape[3], c_stable)
                extra = fo.violators(pm.smap, bound, pose, K4, margin)
            keeps = fo.prune_step(pm, c_stable, t_max, extra)
            if keeps is not None:
                radii = [r[k] for r, k in zip(radii, keeps)]
    return pm, radii
