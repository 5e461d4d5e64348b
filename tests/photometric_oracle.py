"""CPU oracle of the joint geometric and photometric projective ICP (ICPSLAM / PointFusion(photometric_weight=w),
gsx_icp_localize_projective, gsx_icp_projective_targets at w > 0).  Test infrastructure only; built on projective_oracle
(association and loop) and projective_splat_oracle (target images at M >= 1), with the oracle's canonical arithmetic.

    intensity       I(r, g, b) = (0.299 r + 0.587 g) + 0.114 b, float32, every product and sum rounded on its own
    model image     I_m (B, H*W): the intensity of the colour of the row that wins the pixel in the index image of the
                    geometric targets (R1 for M = 0, R1d for M >= 1); 0 where uncovered (an uncovered pixel has none)
    valid pixel     j = (h, w) off the image border, covered, and its four neighbours covered; there
                    g_u = 0.5 (I_m[h,w+1] - I_m[h,w-1]), g_v = 0.5 (I_m[h+1,w] - I_m[h-1,w])
    source          I_s: the intensity of the live colour at each source point's lattice pixel
    row             for a source point s associated with a valid pixel j (the geometric association, dist_thresh
                    included): q = T_prev^-1 s, (u, v, den) as project() computes them with k = the first three rows of
                    the 4x4 K; du/dq_i = (k[i] - u k[8+i]) / den, dv/dq_i = (k[4+i] - v k[8+i]) / den;
                    c_cam = g_u du/dq + g_v dv/dq, c = R_prev c_cam; A_p = [c, s x c], r_p = I_s - I_m[j]
    sums            the geometric 28 sums plus w (A_p[p] A_p[q]), w (A_p[p] r_p), w (r_p r_p): rᵀr is the joint energy
With w = 0 every function here is projective_oracle's / projective_splat_oracle's.  Everything is differentiable torch
(the index and the association carry no gradient), so autograd through it defines the differentiable mode's gradients."""
import math

import torch

import gsx_oracle as oracle
import projective_oracle as po
import projective_splat_oracle as pso
import radii_oracle as ro

F32 = torch.float32
_WR, _WG, _WB, _HALF = (torch.tensor(x, dtype=F32) for x in (0.299, 0.587, 0.114, 0.5))


def intensity(rgb):
    """(..., 3) float32 colours -> (...) intensities."""
    return (_WR * rgb[..., 0] + _WG * rgb[..., 1]) + _WB * rgb[..., 2]


def model_intensity(colors_padded, idx):
    """colors_padded (B, N, 3), idx (B, H*W) int64 (-1 = uncovered) -> I_m (B, H*W), 0 where uncovered."""
    B, P = idx.shape
    col = torch.cat([colors_padded, colors_padded.new_zeros(B, 1, 3)], 1)
    I = intensity(torch.gather(col, 1, idx.clamp(min=0).unsqueeze(-1).expand(B, P, 3)))
    return torch.where(idx >= 0, I, torch.zeros_like(I))


def stencil(I_m, idx, H, W):
    """-> (valid (B, H*W) bool, g_u, g_v (B, H*W), zero off the valid pixels)."""
    B = idx.shape[0]
    cov = (idx >= 0).view(B, H, W)
    I = I_m.view(B, H, W)
    pad = lambda t: torch.nn.functional.pad(t, (1, 1, 1, 1))
    inner = (cov[:, 1:-1, 1:-1] & cov[:, 1:-1, 2:] & cov[:, 1:-1, :-2] & cov[:, 2:, 1:-1] & cov[:, :-2, 1:-1])
    valid = pad(inner.to(F32)) > 0
    gu = torch.where(valid, pad(_HALF * (I[:, 1:-1, 2:] - I[:, 1:-1, :-2])), torch.zeros((), dtype=F32))
    gv = torch.where(valid, pad(_HALF * (I[:, 2:, 1:-1] - I[:, :-2, 1:-1])), torch.zeros((), dtype=F32))
    return valid.view(B, H * W), gu.view(B, H * W), gv.view(B, H * W)


def photometric_rows(s, I_s, j, valid, gu, gv, I_m, prev_pose, K):
    """One element: source s (Ns, 3) world frame, I_s (Ns,), pixel j (Ns,) int64 of the geometric association;
    valid / gu / gv / I_m (H*W,); prev_pose, K (4, 4) -> (A_p (n, 6), r_p (n, 1)) of the points with a photometric row,
    in source order."""
    keep = j >= 0
    keep = keep & valid[j.clamp(min=0)]
    s, I_s, jj = s[keep], I_s[keep], j[keep]
    q = oracle.rigid_apply(oracle.rigid_inverse(prev_pose), s)
    x, y, z = q[:, 0], q[:, 1], q[:, 2]
    row = lambda i: ((K[i, 0] * x + K[i, 1] * y) + K[i, 2] * z) + K[i, 3]
    hx, hy, hz = row(0), row(1), row(2)
    den = torch.where(hz != 0, hz, torch.ones_like(hz))
    u, v = hx / den, hy / den
    g_u, g_v = gu[jj], gv[jj]
    cc = [g_u * ((K[0, i] - u * K[2, i]) / den) + g_v * ((K[1, i] - v * K[2, i]) / den) for i in range(3)]
    R = prev_pose[:3, :3]
    cx, cy, cz = (oracle._dot3(R[r, 0], R[r, 1], R[r, 2], cc[0], cc[1], cc[2]) for r in range(3))
    sx, sy, sz = s[:, 0], s[:, 1], s[:, 2]
    A = torch.stack([cx, cy, cz, cz * sy - cy * sz, cx * sz - cz * sx, cy * sx - cx * sy], 1)
    return A, (I_s - I_m[jj]).unsqueeze(1)


def _normal_equations(A, b, Ap, rp, w):
    """(AᵀA + w A_pᵀA_p, Aᵀb + w A_pᵀr_p, bᵀb + w r_pᵀr_p)."""
    w = torch.tensor(w, dtype=F32)
    return (A.t() @ A + w * (Ap.t() @ Ap), A.t() @ b + w * (Ap.t() @ rp),
            torch.dot(b[:, 0], b[:, 0]) + w * torch.dot(rp[:, 0], rp[:, 0]))


def icp(src, tgt_p, tgt_n, assoc, photo, w, odom, numiters=20, damp=1e-8, lambda_max=2.0, B=1.0, B2=1.0,
        nu=200.0):
    """projective_oracle.icp on the joint energy: assoc(src (Ns,3)) -> j (Ns,); photo(src, j) -> (A_p, r_p)."""
    damp = torch.tensor(damp, dtype=F32)
    lambda_min = 1 / lambda_max

    def system(s):
        j = assoc(s)
        A, b = po._rows(s, tgt_p, tgt_n, j)
        return _normal_equations(A, b, *photo(s, j), w)

    T = torch.eye(4)
    src = oracle.rigid_apply(T, src)
    for _ in range(numiters):
        AtA, Atb, err = system(src)
        xi = torch.inverse(AtA + torch.eye(6) * damp) @ Atb
        dT = oracle.se3_exp(xi)
        one = oracle.rigid_apply(dT, src)
        new_err = system(one)[2]
        if odom == "icp":
            if new_err < err:
                src = one
                damp = damp / 2
                T = oracle.mat4_mul(dT, T)
            else:
                damp = damp * 2
        else:
            diff = (new_err - err).clamp(-70.0, 70.0)
            damp = damp * (lambda_min + (lambda_max - lambda_min) / (1 + torch.exp(-B * diff)))
            sig = 1 / ((1 + torch.exp(-B2 * diff)) ** (1 / nu))
            dT = oracle.se3_exp(sig * xi)
            src = oracle.rigid_apply(dT, src)
            T = oracle.mat4_mul(dT, T)
    return T


def target_images(smap, radii, prev_pose, K, H, W, M):
    """-> (idx, tgt_p, tgt_n, I_m) of the map seen from prev_pose; M = 0 needs no radii."""
    idx, tgt_p, tgt_n = pso.target_images(smap, radii, prev_pose, K, H, W, M)
    if not smap.has_points or sum(smap.counts()) == 0:
        return idx, tgt_p, tgt_n, torch.zeros(idx.shape, dtype=F32)
    return idx, tgt_p, tgt_n, model_intensity(smap.padded()[2], idx)


def source_intensity(live_rgb, live_maps_at_prev_pose, ds):
    """live_rgb (B,1,H,W,3) -> per element the intensities of the source points (downsample_frame's order)."""
    m = live_maps_at_prev_pose["valid"][:, 0, ::ds, ::ds]
    I = intensity(live_rgb[:, 0, ::ds, ::ds])
    return [I[b][m[b]] for b in range(I.shape[0])]


def odometry(smap, radii, live_maps_at_prev_pose, live_rgb, prev_pose, K, H, W, odom, ds, icp_kwargs, M, w):
    """ICPSLAM._localize with association='projective', target_splat_px=M, photometric_weight=w -> (B,4,4)."""
    if w == 0:
        return pso.odometry_projective(smap, radii, live_maps_at_prev_pose, prev_pose, K, H, W, odom, ds, icp_kwargs, M)
    kw = dict(icp_kwargs)
    dth = kw.pop("dist_thresh", None)
    f_pts, _ = oracle.downsample_frame(live_maps_at_prev_pose, ds)
    I_s = source_intensity(live_rgb, live_maps_at_prev_pose, ds)
    idx, tgt_p, tgt_n, I_m = target_images(smap, radii, prev_pose, K, H, W, M)
    valid, gu, gv = stencil(I_m, idx, H, W)
    Ts = []
    for b in range(prev_pose.shape[0]):
        sl = slice(b, b + 1)
        assoc = lambda s, sl=sl: po.associate(s.unsqueeze(0), prev_pose[sl], K[sl], H, W, idx[sl], tgt_p[sl], dth)[1][0]
        photo = lambda s, j, b=b, Is=I_s[b]: photometric_rows(s, Is, j, valid[b], gu[b], gv[b], I_m[b], prev_pose[b],
                                                              K[b])
        Ts.append(icp(f_pts[b], tgt_p[b], tgt_n[b], assoc, photo, w, odom, **kw))
    return oracle.rigid_compose(torch.stack(Ts), prev_pose)


def run_slam(rgb, depth, K, poses=None, *, w, M=0, mode="pointfusion", odom="gradicp", dist_th=0.05, angle_th=20.0,
             sigma=0.6, dsratio=4, numiters=20, damp=1e-8, dist_thresh=None, lambda_max=2.0, B=1.0, B2=1.0, nu=200.0):
    """PointFusion(odom, association='projective', surfel_radii=True, target_splat_px=M, photometric_weight=w) (mode
    'pointfusion') or ICPSLAM(...) (mode 'icpslam', M = 0); frame 0 takes poses[:, 0] (the identity if poses is None).
    Returns gsx_oracle.SlamResult(SurfelMap, poses (B,L,4,4))."""
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
            pose = odometry(smap, radii, at_prev, c, prev_pose, K4, H, W, odom, dsratio, kw, M, w)
        maps = oracle.frame_maps(d, K, pose.unsqueeze(1))
        if mode == "pointfusion":
            table = oracle.find_correspondences(smap, maps, pose, K4, dist_th, dot_th)
            radii = ro.fuse_radii(smap, radii, maps, d, K, table, sigma)
            smap = oracle.fuse_with_map(smap, maps, c, table, sigma)
        else:
            smap = oracle.update_map_aggregate(smap, maps, c)
        prev_pose = pose
        out_poses[:, s] = pose
    return oracle.SlamResult(smap, out_poses)


def translation_error(poses, gt):
    """Worst element's final translation error (metres): max_b |t_b(L-1) - t_gt,b(L-1)|."""
    return float((poses[:, -1, :3, 3].double() - gt[:, -1, :3, 3].double()).norm(dim=-1).max())
