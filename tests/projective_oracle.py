"""CPU oracle of the projective frame-to-model ICP (gsx_icp_localize_projective, ICPSLAM(association='projective')).
Test infrastructure only; built on render_oracle.render_index and gsx_oracle.project_map with the oracle's canonical
arithmetic, so the association is bit-exact against the CUDA path and the poses agree to rounding.

For element b with prev = the previous camera-to-world pose and K the intrinsics:
    target images   idx (B, H*W): render_index's row of every pixel (smallest camera z, ties to the lowest n) or -1;
                    tgt_p / tgt_n (B, H*W, 3): that row's world-frame point and normal, zeros where uncovered
    source          the live frame's global vertex map at prev on the ds lattice, valid pixels in row-major order
    association     s -> pixel j = h*W + w of project_map(s) (frustum (-1e-3, W-0.999) x (-1e-3, H-0.999), z > 0,
                    round half to even, clamp) iff in the frustum, idx[j] >= 0 and, with dist_thresh, d2 < dist_thresh
                    where d2 = (dx*dx + dy*dy) + dz*dz, d = s - tgt_p[j]
    loop            gsx_oracle's point-to-plane rows, damped solve, se3_exp and LM / gradLM update, then T_icp · prev
Everything is differentiable torch (the association carries no gradient), so autograd through it is the gradient
definition of the differentiable mode."""
import math

import torch

import gsx_oracle as oracle
import render_oracle

F32 = torch.float32


def target_images(smap, prev_pose, K, H, W):
    """smap: gsx_oracle.SurfelMap; prev_pose (B,4,4); K (B,4,4) -> (idx (B,H*W) int64, tgt_p, tgt_n (B,H*W,3))."""
    B = prev_pose.shape[0]
    rows = oracle.SurfelMap([p.detach() for p in smap.points]) if smap.has_points else smap  # (the index has no gradient)
    idx = render_oracle.render_index(rows, prev_pose.detach().unsqueeze(1), K, H, W).view(B, H * W)
    pts, nrm, _, _ = smap.padded()

    def gather(t):  # (one zero row appended: an element without rows still gathers)
        t = torch.cat([t, t.new_zeros(B, 1, 3)], 1)
        g = torch.gather(t, 1, idx.clamp(min=0).unsqueeze(-1).expand(B, H * W, 3))
        return torch.where((idx >= 0).unsqueeze(-1), g, torch.zeros_like(g))

    return idx, gather(pts), gather(nrm)


def associate(src, prev_pose, K, H, W, idx, tgt_p, dist_thresh=None):
    """src (B,Ns,3) world frame -> (d2 (B,Ns): +inf unless a row covers the pixel s projects to, j (B,Ns) int64 or -1)."""
    B, Ns, _ = src.shape
    u, v, z = oracle.project_map(src, prev_pose, K)
    lo = torch.tensor(-1e-3, dtype=F32)
    inframe = ((u > lo) & (u < torch.tensor(W - 0.999, dtype=F32)) & (v > lo)
               & (v < torch.tensor(H - 0.999, dtype=F32)) & (z > 0))
    j = v.round().long().clamp(0, H - 1) * W + u.round().long().clamp(0, W - 1)
    ok = inframe & (torch.gather(idx, 1, j) >= 0)
    p = torch.gather(tgt_p, 1, j.unsqueeze(-1).expand(B, Ns, 3))
    d = src - p
    d2 = torch.where(ok, (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2],
                     torch.full_like(u, float("inf")))
    if dist_thresh is not None:
        ok = ok & (d2 < torch.tensor(dist_thresh, dtype=F32))
    return d2, torch.where(ok, j, torch.full_like(j, -1))


def _rows(src, tgt_p, tgt_n, j):
    """Point-to-plane rows of the associated source points (gsx_oracle.gauss_newton_solve after its 1-NN)."""
    keep = j >= 0
    s, p, n = src[keep], tgt_p[j[keep]], tgt_n[j[keep]]
    sx, sy, sz = s[:, 0:1], s[:, 1:2], s[:, 2:3]
    nx, ny, nz = n[:, 0:1], n[:, 1:2], n[:, 2:3]
    A = torch.cat([nx, ny, nz, nz * sy - ny * sz, nx * sz - nz * sx, ny * sx - nx * sy], 1)
    b = nx * (p[:, 0:1] - sx) + ny * (p[:, 1:2] - sy) + nz * (p[:, 2:3] - sz)
    return A, b


def icp(src, tgt_p, tgt_n, assoc, odom, numiters=20, damp=1e-8, lambda_max=2.0, B=1.0, B2=1.0, nu=200.0):
    """The LM (odom='icp', gsx_oracle.point_to_plane_icp) or gradLM ('gradicp', point_to_plane_gradicp) loop of one
    element with the association `assoc(src (Ns,3)) -> j (Ns,)`, from the identity.  -> T (4,4)."""
    damp = torch.tensor(damp, dtype=F32)
    lambda_min = 1 / lambda_max
    T = torch.eye(4)
    src = oracle.rigid_apply(T, src)
    for _ in range(numiters):
        A, b = _rows(src, tgt_p, tgt_n, assoc(src))
        xi = oracle.solve_linear_system(A, b, damp)
        dT = oracle.se3_exp(xi)
        err = torch.dot(b[:, 0], b[:, 0])
        one = oracle.rigid_apply(dT, src)
        _, b1 = _rows(one, tgt_p, tgt_n, assoc(one))
        new_err = torch.dot(b1[:, 0], b1[:, 0])
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


def odometry_projective(smap, live_maps_at_prev_pose, prev_pose, K, H, W, odom, ds, icp_kwargs):
    """ICPSLAM._localize with association='projective' -> new pose (B,4,4) = T_icp · prev_pose.  icp_kwargs: numiters,
    damp, dist_thresh and, for gradicp, lambda_max / B / B2 / nu."""
    kw = dict(icp_kwargs)
    dth = kw.pop("dist_thresh", None)
    f_pts, _ = oracle.downsample_frame(live_maps_at_prev_pose, ds)
    idx, tgt_p, tgt_n = target_images(smap, prev_pose, K, H, W)
    Ts = []
    for b in range(prev_pose.shape[0]):
        sl = slice(b, b + 1)
        assoc = lambda s, sl=sl: associate(s.unsqueeze(0), prev_pose[sl], K[sl], H, W, idx[sl], tgt_p[sl], dth)[1][0]
        Ts.append(icp(f_pts[b], tgt_p[b], tgt_n[b], assoc, odom, **kw))
    return oracle.rigid_compose(torch.stack(Ts), prev_pose)


def run_slam(rgb, depth, K, poses=None, *, mode="pointfusion", odom="gradicp", dist_th=0.05, angle_th=20.0, sigma=0.6,
             dsratio=4, numiters=20, damp=1e-8, dist_thresh=None, lambda_max=2.0, B=1.0, B2=1.0, nu=200.0):
    """gsx_oracle.run_slam with projective ICP odometry (odom 'icp' or 'gradicp'); frame 0 takes poses[:, 0] (the
    identity if poses is None).  Returns gsx_oracle.SlamResult(SurfelMap, poses (B,L,4,4))."""
    Bn, L, H, W, _ = depth.shape
    dot_th = math.cos(angle_th * math.pi / 180)
    kw = dict(numiters=numiters, damp=damp, dist_thresh=dist_thresh)
    if odom == "gradicp":
        kw.update(lambda_max=lambda_max, B=B, B2=B2, nu=nu)
    smap = oracle.SurfelMap()
    out_poses = torch.empty(Bn, L, 4, 4)
    K4 = K[:, 0]
    prev_pose = None
    for s in range(L):
        d, c = depth[:, s:s + 1], rgb[:, s:s + 1]
        if s == 0:
            pose = torch.eye(4).repeat(Bn, 1, 1) if poses is None else poses[:, 0]
        else:
            at_prev = oracle.frame_maps(d, K, prev_pose.unsqueeze(1))
            pose = odometry_projective(smap, at_prev, prev_pose, K4, H, W, odom, dsratio, kw)
        maps = oracle.frame_maps(d, K, pose.unsqueeze(1))
        if mode == "pointfusion":
            smap = oracle.update_map_fusion(smap, maps, c, pose, K4, dist_th, dot_th, sigma)
        else:
            smap = oracle.update_map_aggregate(smap, maps, c)
        prev_pose = pose
        out_poses[:, s] = pose
    return oracle.SlamResult(smap, out_poses)


def small_case(H, W):
    """Three elements: 0 sees through a unit camera at the identity (u = x / z exactly), so rows and source points sit on
    the frustum bounds, on half-pixel ties and share a camera z; 1 has a rotated camera with skew and a 4th K column;
    2 has an empty map.  Inputs of the CPU and GPU association tests; returns (SurfelMap, row lists, src (3,Ns,3),
    prev poses (3,4,4), K (3,4,4))."""
    g = torch.Generator().manual_seed(3)
    K = torch.eye(4).repeat(3, 1, 1)
    K[1, 0, 0], K[1, 1, 1], K[1, 0, 2], K[1, 1, 2] = 3.0, 2.8, 3.6, 2.4
    K[1, 0, 1], K[1, 0, 3], K[1, 1, 3] = 0.2, 0.35, -0.3
    pose = torch.eye(4).repeat(3, 1, 1)
    pose[1] = oracle.se3_exp(torch.tensor([0.1, -0.05, 0.2, 0.05, -0.1, 0.08]))
    # element 0: pixels on a grid, two rows per pixel at the same z (tie -> lower n), rows behind the camera
    xs, ys = torch.meshgrid(torch.arange(W, dtype=torch.float32), torch.arange(H, dtype=torch.float32), indexing="xy")
    grid = torch.stack([xs.reshape(-1), ys.reshape(-1), torch.ones(H * W)], -1)
    keep = torch.rand(H * W, generator=g) < 0.7  # some pixels uncovered
    rows0 = torch.cat([grid[keep], grid[keep] + torch.tensor([0.2, -0.2, 0.0]), grid[:5] * torch.tensor([1, 1, -1.0]),
                       torch.tensor([[-1e-3, 1.0, 1.0], [W - 0.999, 1.0, 1.0], [2.0, H - 0.999, 1.0],
                                     [W - 1.0009, 1.0, 1.0], [3.0, -0.0009, 1.0]])], 0)
    # element 1: random rows in front of the rotated camera
    q = torch.rand(60, 3, generator=g) * torch.tensor([2.0, 2.0, 1.0]) + torch.tensor([-1.0, -1.0, 0.8])
    rows1 = oracle.rigid_apply(pose[1], q)
    rows1 = torch.cat([rows1, rows1[:10]], 0)  # exact duplicates: tie in z, lower n wins
    maps = [rows0, rows1, torch.empty(0, 3)]
    # sources: near the rows, on half-pixel ties, on the frustum bounds, behind the camera
    s0 = torch.cat([grid + 0.01 * torch.randn(H * W, 3, generator=g),
                    torch.tensor([[2.5, 1.5, 1.0], [3.5, 2.5, 1.0], [1.5, 0.5, 1.0], [-1e-3, 2.0, 1.0],
                                  [W - 0.999, 2.0, 1.0], [W - 1.0009, 2.0, 1.0], [1.0, -0.0009, 1.0], [1.0, 2.0, -1.0],
                                  [1.0, 2.0, 0.0]])], 0)
    s1 = oracle.rigid_apply(pose[1], q[:40] + 0.02 * torch.randn(40, 3, generator=g))
    n = s0.shape[0]
    src = torch.zeros(3, n, 3)
    src[0] = s0
    src[1, :40] = s1
    src[2] = s0
    normals = [torch.nn.functional.normalize(torch.randn(m.shape[0], 3, generator=g), dim=1) for m in maps]
    smap = oracle.SurfelMap(maps, normals, [torch.zeros_like(m) for m in maps], [torch.ones(m.shape[0], 1) for m in maps])
    return smap, maps, src, pose, K
