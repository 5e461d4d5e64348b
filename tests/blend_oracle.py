"""CPU oracle of the blended splat render (render_pointclouds(blend_band=eps), gsx_render_blend).

Coverage, the front depth and the band are decisions, taken in float32 with the arithmetic of the disk-splat oracle
(tests/splat_oracle.py), which the CUDA path equals bit for bit:

    covers     a disk row (radius > 0, non-zero normal, max_splat_px = M >= 1) covers pixel p when p is in its +-M box
               and the ray meets the disk, at plane depth t_n(p); s2_n(p) = (ex ex + ey ey) + ez ez with
               e = t d - q, the quantity the disk test compares with r^2.  Any other row, or every row at M = 0,
               covers the one pixel find_active_map_points gives it, at its camera z, with s2 = 0.
    front      z_f(p) = the depth render_pointclouds(max_splat_px=M) shows at p; index = its index image.
    band       row n contributes to p when it covers p and t_n(p) <= float32(float64(z_f(p)) + eps).

The values are one differentiable torch statement (float64 in the tests), so that autograd of it is the gradient
reference:

    w_n = c_n (1 - s2_n / r_n^2) for a disk row, c_n otherwise (c_n = the confidence count, or 1 without one)
    W = sum w_n;  depth = sum w_n t_n / W;  rgb = sum w_n col_n / W;  normals = sum w_n (R^T n_n) / W;  confidence = W
    and zeros (no gradient) where W = 0."""
from collections import namedtuple

import torch

import gsx_oracle as oracle
import splat_oracle as so

F32 = torch.float32

Blended = namedtuple("Blended", "depth rgb normals confidence index")
# Contributors: flat pixel slot ((b L + l) H + h) W + w, element b, view l, pixel h, w, row n, whether a disk
Contributors = namedtuple("Contributors", "slot b l h w n disk")


def front(points, normals, radii, counts, poses, K, H, W, M):
    """(index (B,L,H,W), z_f (B,L,H,W) float32) of render_pointclouds(max_splat_px=M), from float32 rows."""
    r = radii if M > 0 else torch.zeros_like(radii)  # M = 0: R1, one pixel for every row
    index = so.splat_index(points, normals, r, counts, poses, K, H, W, max(M, 0))
    zf = so.splat_values(points, normals, None, None, r, poses, K, index).depth[..., 0]
    return index, zf


def contributors(points, normals, radii, counts, poses, K, H, W, M, band):
    """The (pixel, row) pairs that contribute, decided in float32; and the index image and z_f."""
    B, L = poses.shape[:2]
    N = points.shape[1]
    index, zf = front(points, normals, radii, counts, poses, K, H, W, M)
    lim = (zf.double() + band).to(F32).view(-1)  # the band's limit, one float32 rounding
    live = torch.arange(N).view(1, N) < torch.tensor(counts).view(B, 1)
    disk = (so.is_disk(normals, radii) & live) if M > 0 else torch.zeros((B, N), dtype=torch.bool)
    Kinv = oracle.inverse_intrinsics(K)
    k00, k02 = Kinv[:, 0, 0].view(B, 1), Kinv[:, 0, 2].view(B, 1)
    k11, k12 = Kinv[:, 1, 1].view(B, 1), Kinv[:, 1, 2].view(B, 1)
    ones = torch.ones((), dtype=F32)
    out = []
    # one-pixel rows: the association of find_active_map_points, at the camera z
    pt_lists = [points[b, :counts[b]][~disk[b, :counts[b]]] for b in range(B)]
    rowmap = torch.zeros((B, max(N, 1)), dtype=torch.int64)
    for b in range(B):
        r = torch.nonzero(~disk[b, :counts[b]]).flatten()
        rowmap[b, :r.numel()] = r
    pmap = oracle.SurfelMap(pt_lists)
    for l in range(L):
        if sum(x.shape[0] for x in pt_lists) > 0:
            table = oracle.find_active_map_points(pmap, poses[:, l], K, H, W)
            if table.shape[0]:
                _, _, z = oracle.project_map(pmap.padded()[0], poses[:, l], K)
                b, j, h, w = table.unbind(1)
                slot = ((b * L + l) * H + h) * W + w
                keep = z[b, j] <= lim[slot]
                out.append((slot[keep], b[keep], torch.full_like(b[keep], l), h[keep], w[keep], rowmap[b, j][keep],
                            torch.zeros_like(keep[keep])))
        if M == 0:
            continue
        q, m = so._camera(points, normals, poses[:, l])
        u, v, _ = oracle.project_map(points, poses[:, l], K)
        cu = u.clamp(-M - 2, W + M + 1).round().long()
        cv = v.clamp(-M - 2, H + M + 1).round().long()
        mq = so._dot3(m, q)
        rr = radii[..., 0] * radii[..., 0]
        for dh in range(-M, M + 1):
            for dw in range(-M, M + 1):
                h, w = cv + dh, cu + dw
                inside = disk & (q[..., 2] > 0) & (h >= 0) & (h < H) & (w >= 0) & (w < W)
                dx = k00 * w.to(F32) + k02
                dy = k11 * h.to(F32) + k12
                md = oracle._dot3(m[..., 0], m[..., 1], m[..., 2], dx, dy, ones)
                t = mq / torch.where(md == 0, ones, md)
                ex, ey, ez = t * dx - q[..., 0], t * dy - q[..., 1], t * ones - q[..., 2]
                e2 = (ex * ex + ey * ey) + ez * ez
                cov = inside & (md != 0) & (t > 0) & (e2 <= rr)
                b, n = torch.nonzero(cov).unbind(1)
                if b.numel() == 0:
                    continue
                slot = ((b * L + l) * H + h[b, n]) * W + w[b, n]
                keep = t[b, n] <= lim[slot]
                out.append((slot[keep], b[keep], torch.full_like(b[keep], l), h[b, n][keep], w[b, n][keep], n[keep],
                            torch.ones_like(keep[keep])))
    if not out:
        e = torch.zeros(0, dtype=torch.int64)
        return Contributors(e, e, e, e, e, e, torch.zeros(0, dtype=torch.bool)), index, zf
    cols = [torch.cat([o[k] for o in out]) for k in range(7)]
    return Contributors(*cols), index, zf


def blend_values(points, normals, colors, ccounts, radii, poses, K, con, index):
    """Outputs from the contributors `con`: differentiable w.r.t. points, normals, colors, ccounts (None: weight 1),
    radii and poses, in their dtype.  K only gives the rays."""
    B, L, H, W = index.shape
    dt = points.dtype
    b, l, n = con.b, con.l, con.n
    Tinv = oracle.rigid_inverse(poses)  # (B,L,4,4)
    R, t0 = Tinv[b, l, :3, :3], Tinv[b, l, :3, 3]
    q = torch.einsum("kij,kj->ki", R, points[b, n]) + t0
    m = torch.einsum("kij,kj->ki", R, normals[b, n])
    Kinv = oracle.inverse_intrinsics(K.to(F32)).to(dt)
    ray = torch.stack([Kinv[b, 0, 0] * con.w.to(dt) + Kinv[b, 0, 2], Kinv[b, 1, 1] * con.h.to(dt) + Kinv[b, 1, 2],
                       torch.ones(b.shape, dtype=dt)], -1)
    md = (m * ray).sum(-1)
    disk = con.disk
    t_disk = (m * q).sum(-1) / torch.where(disk, md, torch.ones_like(md))
    t = torch.where(disk, t_disk, q[:, 2])
    e = t.unsqueeze(-1) * ray - q
    r = radii[b, n, 0]
    s2 = (e * e).sum(-1)
    c = torch.ones(b.shape, dtype=dt) if ccounts is None else ccounts[b, n, 0]
    wgt = torch.where(disk, c * (1 - s2 / torch.where(disk, r * r, torch.ones_like(r))), c)
    P = B * L * H * W

    def total(x):  # (k, C) -> (P, C)
        return torch.zeros((P, x.shape[1]), dtype=dt).index_add(0, con.slot, x)

    Wsum = total(wgt.unsqueeze(-1))
    nz = Wsum != 0
    den = torch.where(nz, Wsum, torch.ones_like(Wsum))

    def mean(x, C):
        return torch.where(nz, total(wgt.unsqueeze(-1) * x) / den, torch.zeros((P, C), dtype=dt)).view(B, L, H, W, C)

    depth = mean(t.unsqueeze(-1), 1)
    rgb = None if colors is None else mean(colors[b, n], 3)
    nrm = mean(m, 3)
    conf = None if ccounts is None else Wsum.view(B, L, H, W, 1)
    return Blended(depth, rgb, nrm, conf, index)


def blend_views(points, normals, colors, ccounts, radii, counts, poses, K, H, W, M, band):
    """The full blended render from padded rows (B,N,3) / (B,N,1): decisions from the rows rounded to float32 (they
    are float32 on the GPU), values in the inputs' dtype."""
    f = lambda t: t.to(F32)
    con, index, _ = contributors(f(points), f(normals), f(radii), counts, f(poses), K, H, W, M, band)
    return blend_values(points, normals, colors, ccounts, radii, poses, K, con, index)


def min_disk_cosine(normals, radii, poses, K, con, shape):
    """float64 (B,L,H,W): the smallest |cos| between a pixel's ray and the normal of a disk row contributing to it
    (1 where none does)."""
    B, L, H, W = shape
    b, l, n = con.b, con.l, con.n
    R = poses[b, l, :3, :3].double()
    m = torch.einsum("kji,kj->ki", R, normals[b, n].double())
    Kinv = oracle.inverse_intrinsics(K).double()
    d = torch.stack([Kinv[b, 0, 0] * con.w.double() + Kinv[b, 0, 2], Kinv[b, 1, 1] * con.h.double() + Kinv[b, 1, 2],
                     torch.ones(b.shape, dtype=torch.float64)], -1)
    cos = ((m * d).sum(-1) / (m.norm(dim=-1) * d.norm(dim=-1)).clamp_min(1e-300)).abs()
    cos = torch.where(con.disk, cos, torch.ones_like(cos))
    out = torch.ones(B * L * H * W, dtype=torch.float64).scatter_reduce(0, con.slot, cos, reduce="amin")
    return out.view(B, L, H, W)

