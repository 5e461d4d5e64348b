"""CPU oracle of the projective ICP against the disk-splat render of the map (ICPSLAM / PointFusion(target_splat_px=M),
gsx_icp_localize_projective, gsx_icp_projective_targets at M >= 1).  Test infrastructure only; built on
projective_oracle (association and loop), splat_oracle (the disk render) and radii_oracle (fusion with radii), with the
oracle's canonical arithmetic.

For M >= 1 and element b with prev = the previous camera-to-world pose:
    index       splat_oracle.splat_index of the map seen from prev at M (R1d's z-buffer, keys, ties and fill)
    depth       splat_oracle.splat_values(...).depth at that index: t, where the pixel's ray meets the plane of the disk
                row that won it; the row's camera z for a one-pixel row
    tgt_p       at a pixel a disk row (radius > 0, normal != 0) won, gsx_oracle.frame_maps(depth, K, prev)["gvertex"],
                the K1 global vertex of t; the winning row's point at any other covered pixel; zeros where uncovered
    tgt_n       the winning row's normal, zeros where uncovered
M = 0 is projective_oracle.target_images.  Everything is differentiable torch (the index carries no gradient), so
autograd through it defines the gradients of the differentiable mode."""
import math

import torch

import gsx_oracle as oracle
import projective_oracle as po
import radii_oracle as ro
import splat_oracle as so


def padded_radii(radii, N):
    """Per-element (N_b, 1) radii -> float32 (B, N, 1), zero-padded."""
    out = torch.zeros(len(radii), N, 1)
    for b, r in enumerate(radii):
        out[b, :r.shape[0]] = r
    return out


def target_images(smap, radii, prev_pose, K, H, W, M):
    """smap: gsx_oracle.SurfelMap with normals; radii: per element (N_b, 1); prev_pose (B,4,4); K (B,4,4)
    -> (idx (B,H*W) int64, tgt_p, tgt_n (B,H*W,3))."""
    if M == 0 or not smap.has_points or sum(smap.counts()) == 0:
        return po.target_images(smap, prev_pose, K, H, W)
    B = prev_pose.shape[0]
    pts, nrm, col, cc = smap.padded()
    rp = padded_radii(radii, pts.shape[1])
    index = so.splat_index(pts.detach(), nrm.detach(), rp, smap.counts(), prev_pose.detach().unsqueeze(1), K, H, W, M)
    depth = so.splat_values(pts, nrm, col, cc, rp, prev_pose.unsqueeze(1), K, index).depth  # (B,1,H,W,1)
    surface = oracle.frame_maps(depth, K.unsqueeze(1), prev_pose.unsqueeze(1))["gvertex"].reshape(B, H * W, 3)
    idx = index.view(B, H * W)
    rows = idx.clamp(min=0)

    def gather(t):  # (one zero row appended, as projective_oracle does)
        t = torch.cat([t, t.new_zeros(B, 1, t.shape[-1])], 1)
        g = torch.gather(t, 1, rows.unsqueeze(-1).expand(B, H * W, t.shape[-1]))
        return torch.where((idx >= 0).unsqueeze(-1), g, torch.zeros_like(g))

    disk = torch.cat([so.is_disk(nrm.detach(), rp), torch.zeros((B, 1), dtype=torch.bool)], 1)
    won = torch.gather(disk, 1, rows) & (idx >= 0)
    return idx, torch.where(won.unsqueeze(-1), surface, gather(pts)), gather(nrm)


def odometry_projective(smap, radii, live_maps_at_prev_pose, prev_pose, K, H, W, odom, ds, icp_kwargs, M):
    """projective_oracle.odometry_projective with the target images of target_images(..., M)."""
    kw = dict(icp_kwargs)
    dth = kw.pop("dist_thresh", None)
    f_pts, _ = oracle.downsample_frame(live_maps_at_prev_pose, ds)
    idx, tgt_p, tgt_n = target_images(smap, radii, prev_pose, K, H, W, M)
    Ts = []
    for b in range(prev_pose.shape[0]):
        sl = slice(b, b + 1)
        assoc = lambda s, sl=sl: po.associate(s.unsqueeze(0), prev_pose[sl], K[sl], H, W, idx[sl], tgt_p[sl], dth)[1][0]
        Ts.append(po.icp(f_pts[b], tgt_p[b], tgt_n[b], assoc, odom, **kw))
    return oracle.rigid_compose(torch.stack(Ts), prev_pose)


def run_pointfusion(rgb, depth, K, poses=None, *, M, odom="gradicp", dist_th=0.05, angle_th=20.0, sigma=0.6, dsratio=4,
                    numiters=20, damp=1e-8, dist_thresh=None, lambda_max=2.0, B=1.0, B2=1.0, nu=200.0):
    """PointFusion(odom, association='projective', surfel_radii=True, target_splat_px=M): frame 0 takes poses[:, 0] (the
    identity if poses is None).  Returns (gsx_oracle.SlamResult(SurfelMap, poses (B,L,4,4)), radii per element)."""
    Bn, L, H, W, _ = depth.shape
    dot_th = math.cos(angle_th * math.pi / 180)
    kw = dict(numiters=numiters, damp=damp, dist_thresh=dist_thresh)
    if odom == "gradicp":
        kw.update(lambda_max=lambda_max, B=B, B2=B2, nu=nu)
    smap, radii = oracle.SurfelMap(), None
    out_poses = torch.empty(Bn, L, 4, 4)
    K4 = K[:, 0]
    prev_pose = None
    for s in range(L):
        d, c = depth[:, s:s + 1], rgb[:, s:s + 1]
        if s == 0:
            pose = torch.eye(4).repeat(Bn, 1, 1) if poses is None else poses[:, 0]
        else:
            at_prev = oracle.frame_maps(d, K, prev_pose.unsqueeze(1))
            pose = odometry_projective(smap, radii, at_prev, prev_pose, K4, H, W, odom, dsratio, kw, M)
        maps = oracle.frame_maps(d, K, pose.unsqueeze(1))
        table = oracle.find_correspondences(smap, maps, pose, K4, dist_th, dot_th)
        radii = ro.fuse_radii(smap, radii, maps, d, K, table, sigma)
        smap = oracle.fuse_with_map(smap, maps, c, table, sigma)
        prev_pose = pose
        out_poses[:, s] = pose
    return oracle.SlamResult(smap, out_poses), radii
