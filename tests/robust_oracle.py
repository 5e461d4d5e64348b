"""CPU oracle of the Huber-weighted tracking energy (ICPSLAM / PointFusion(huber_delta=, photometric_huber_delta=), the
*_robust entry points of libgsx).  Test infrastructure only; built on gsx_oracle (1-NN), projective_oracle,
projective_splat_oracle and photometric_oracle with the oracle's canonical arithmetic.

For a residual r and a scale delta > 0, with a = |r|:
    inside, a <= delta (equality is inside)   weight 1: the row adds A_p A_q, A_p r and r r, the unweighted products
    outside                                   h = delta / a; the row adds h (A_p A_q), h (A_p r) and
                                              rho = delta ((a + a) - delta) in slot 27
    photometric (weight w, scale delta_p)     inside w (A_p A_q), w (A_p r_p), w (r_p r_p); outside (w h_p) (A_p A_q),
                                              (w h_p) (A_p r_p), w rho_p
    loop                                      the unchanged LM / gradLM loop of iteratively reweighted least squares:
                                              err and new_err are slot 27, the Huber energy sum rho
delta = +inf takes the inside branch on every row, and every function here is then its unweighted oracle's bit for bit.
Everything is differentiable torch with torch.where branches (the association carries no gradient), so float64
autograd through it defines the gradient of the differentiable mode, with the inside branch's derivative at a = delta."""
import math

import torch

import gsx_oracle as oracle
import photometric_oracle as pho
import projective_oracle as po
import radii_oracle as ro

F32 = torch.float32


def weights(r, delta, inside=None):
    """r (n,) residuals -> (inside (n,) bool, h (n,): 1 inside, delta / |r| outside, rho (n,): r r inside, delta ((a + a)
    - delta) outside).  Safe for autograd: the branch a row does not take gets no gradient and no NaN.  inside: the
    rows' branch decisions when they are given (a float64 evaluation on the float32 kernels' branches), else a <= delta."""
    d = torch.as_tensor(delta, dtype=r.dtype)
    a = r.abs()
    if inside is None:
        inside = a <= d
    one = torch.ones_like(a)
    a_out = torch.where(inside, one, a)  # (inside rows never divide)
    h = torch.where(inside, one, d / a_out)
    rho = torch.where(inside, r * r, torch.where(inside, one, d * ((a_out + a_out) - d)))
    return inside, h, rho


def row_products(A, r, delta, w=None, inside=None):
    """The 28 products every row adds, as the kernels write them (row_products<true>, and add_weighted_products<true>
    when w is given): A (n,6), r (n,) -> (n,28) in the kernels' order (21 upper-triangular A_p A_q, 6 A_p r, slot 27).
    inside: optional branch decisions (weights)."""
    inside, h, rho = weights(r, delta, inside)
    iu = torch.triu_indices(6, 6)
    pq = A[:, iu[0]] * A[:, iu[1]]
    pr = A * r.unsqueeze(1)
    if w is None:
        c = h.unsqueeze(1)
        return torch.cat([torch.where(inside.unsqueeze(1), pq, c * pq), torch.where(inside.unsqueeze(1), pr, c * pr),
                          rho.unsqueeze(1)], 1)
    w = torch.as_tensor(w, dtype=A.dtype)
    c = (w * h).unsqueeze(1)
    return torch.cat([torch.where(inside.unsqueeze(1), w * pq, c * pq), torch.where(inside.unsqueeze(1), w * pr, c * pr),
                      (w * rho).unsqueeze(1)], 1)


def system(A, b, delta, Ap=None, rp=None, w=0.0, delta_p=math.inf):
    """(AᵀCA + w A_pᵀC_pA_p, AᵀCb + w A_pᵀC_pr_p, sum rho + w sum rho_p) with C = diag(h): the robust normal equations of
    one element.  At delta = delta_p = +inf, exactly gsx_oracle.solve_linear_system's / photometric_oracle's sums."""
    inside, h, rho = weights(b[:, 0], delta)
    c = h.unsqueeze(1)
    b_in = torch.where(inside, b[:, 0], torch.zeros_like(b[:, 0]))
    AtA, Atb = A.t() @ (c * A), A.t() @ (c * b)
    err = torch.dot(b_in, b_in) + torch.where(inside, torch.zeros_like(rho), rho).sum()
    if Ap is None:
        return AtA, Atb, err
    w = torch.tensor(w, dtype=F32)
    inp, hp, rhop = weights(rp[:, 0], delta_p)
    cp = hp.unsqueeze(1)
    rp_in = torch.where(inp, rp[:, 0], torch.zeros_like(rp[:, 0]))
    return (AtA + w * (Ap.t() @ (cp * Ap)), Atb + w * (Ap.t() @ (cp * rp)),
            err + w * (torch.dot(rp_in, rp_in) + torch.where(inp, torch.zeros_like(rhop), rhop).sum()))


def icp(src, sys_fn, odom, numiters=20, damp=1e-8, lambda_max=2.0, B=1.0, B2=1.0, nu=200.0):
    """The LM (odom='icp') or gradLM ('gradicp') loop of one element from the identity, on sys_fn(src (Ns,3)) ->
    (AᵀA, Aᵀb, err): gsx_oracle.point_to_plane_icp / _gradicp and photometric_oracle.icp with the robust system."""
    damp = torch.tensor(damp, dtype=F32)
    lambda_min = 1 / lambda_max
    T = torch.eye(4)
    src = oracle.rigid_apply(T, src)
    for _ in range(numiters):
        AtA, Atb, err = sys_fn(src)
        xi = torch.inverse(AtA + torch.eye(6) * damp) @ Atb
        dT = oracle.se3_exp(xi)
        one = oracle.rigid_apply(dT, src)
        new_err = sys_fn(one)[2]
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


def _split(icp_kwargs):
    kw = dict(icp_kwargs)
    return kw.pop("dist_thresh", None), kw


def odometry_nn(smap, live_maps_at_prev_pose, prev_pose, K, H, W, odom, ds, icp_kwargs, delta):
    """gsx_oracle.odometry (the 1-NN association) with Huber-weighted rows -> (B,4,4)."""
    dth, kw = _split(icp_kwargs)
    f_pts, _ = oracle.downsample_frame(live_maps_at_prev_pose, ds)
    table = oracle.find_active_map_points(smap, prev_pose, K, H, W)
    m_pts, m_nrm = oracle.downsample_map(smap, table, ds)
    Ts = []
    for b in range(smap.B):
        def sys_fn(s, b=b):
            A, r, _ = oracle.gauss_newton_solve(s, m_pts[b], m_nrm[b], dth)
            return system(A, r, delta)
        Ts.append(icp(f_pts[b], sys_fn, odom, **kw))
    return oracle.rigid_compose(torch.stack(Ts), prev_pose)


def odometry_projective(smap, radii, live_maps_at_prev_pose, live_rgb, prev_pose, K, H, W, odom, ds, icp_kwargs, M, w,
                        delta, delta_p):
    """photometric_oracle.odometry (projective association, target_splat_px=M, photometric_weight=w) with Huber-weighted
    rows -> (B,4,4)."""
    dth, kw = _split(icp_kwargs)
    f_pts, _ = oracle.downsample_frame(live_maps_at_prev_pose, ds)
    idx, tgt_p, tgt_n, I_m = pho.target_images(smap, radii, prev_pose, K, H, W, M)
    if w:
        I_s = pho.source_intensity(live_rgb, live_maps_at_prev_pose, ds)
        valid, gu, gv = pho.stencil(I_m, idx, H, W)
    Ts = []
    for b in range(prev_pose.shape[0]):
        sl = slice(b, b + 1)
        assoc = lambda s, sl=sl: po.associate(s.unsqueeze(0), prev_pose[sl], K[sl], H, W, idx[sl], tgt_p[sl], dth)[1][0]

        def sys_fn(s, b=b, assoc=assoc):
            j = assoc(s)
            A, r = po._rows(s, tgt_p[b], tgt_n[b], j)
            if not w:
                return system(A, r, delta)
            Ap, rp = pho.photometric_rows(s, I_s[b], j, valid[b], gu[b], gv[b], I_m[b], prev_pose[b], K[b])
            return system(A, r, delta, Ap, rp, w, delta_p)
        Ts.append(icp(f_pts[b], sys_fn, odom, **kw))
    return oracle.rigid_compose(torch.stack(Ts), prev_pose)


def run_slam(rgb, depth, K, poses=None, *, association="nn", delta=math.inf, delta_p=math.inf, w=0.0, M=0,
             mode="pointfusion", odom="gradicp", dist_th=0.05, angle_th=20.0, sigma=0.6, dsratio=4, numiters=20,
             damp=1e-8, dist_thresh=None, lambda_max=2.0, B=1.0, B2=1.0, nu=200.0):
    """PointFusion (mode 'pointfusion') or ICPSLAM ('icpslam') with odom 'icp' / 'gradicp' and Huber-weighted tracking;
    association 'nn' is gsx_oracle.run_slam's, 'projective' photometric_oracle.run_slam's (surfel radii, target_splat_px
    = M, photometric_weight = w).  delta / delta_p = +inf (the defaults) are the unweighted runs.  Frame 0 takes
    poses[:, 0] (the identity if poses is None).  Returns gsx_oracle.SlamResult(SurfelMap, poses (B,L,4,4))."""
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
            if association == "nn":
                pose = odometry_nn(smap, at_prev, prev_pose, K4, H, W, odom, dsratio, kw, delta)
            else:
                pose = odometry_projective(smap, radii, at_prev, c, prev_pose, K4, H, W, odom, dsratio, kw, M, w, delta,
                                           delta_p)
        maps = oracle.frame_maps(d, K, pose.unsqueeze(1))
        if mode == "pointfusion":
            table = oracle.find_correspondences(smap, maps, pose, K4, dist_th, dot_th)
            if association == "projective":
                radii = ro.fuse_radii(smap, radii, maps, d, K, table, sigma)
            smap = oracle.fuse_with_map(smap, maps, c, table, sigma)
        else:
            smap = oracle.update_map_aggregate(smap, maps, c)
        prev_pose = pose
        out_poses[:, s] = pose
    return oracle.SlamResult(smap, out_poses)


def worst_translation_error(poses, gt, first):
    """max over elements and frames >= first of |t - t_gt| (metres)."""
    return float((poses[:, first:, :3, 3].double() - gt[:, first:, :3, 3].double()).norm(dim=-1).max())
