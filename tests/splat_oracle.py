"""CPU oracle of the disk-splat render (render_pointclouds(max_splat_px >= 1), gsx_render_splats), built on the oracle's
projection (gsx_oracle.project_map, rigid_apply, inverse_intrinsics) and render_oracle's one-pixel rule.

    disk row    radius r > 0 and a non-zero normal n; q = T^-1 p, m = R^T n; skipped unless q.z > 0
    box         (2 M + 1)^2 pixels around round-half-even(u, v) of project_map, clipped to the image
    covered     d = K^-1 (w, h, 1): m.d != 0, t = (m.q) / (m.d) > 0 and |t d - q|^2 <= r^2
    key         (bits(t) << 32) | n per covered pixel, as render_oracle's (bits(z) << 32) | n for the other rows

`splat_values` evaluates the outputs at a FIXED index with differentiable torch ops (any float dtype): depth = t for a
pixel won by a disk row, z of T^-1 p otherwise; normals R^T n, colour and confidence the row's."""
import torch

import gsx_oracle as oracle
import render_oracle
from render_oracle import Rendered

F32 = torch.float32


def is_disk(normals, radii):
    """bool (B,N): rows drawn as disks."""
    return (radii[..., 0] > 0) & (normals != 0).any(-1)


def _dot3(a, b):
    return oracle._dot3(a[..., 0], a[..., 1], a[..., 2], b[..., 0], b[..., 1], b[..., 2])


def _camera(points, normals, pose):
    """q = T^-1 p and m = R^T n for poses (B,4,4) and rows (B,N,3)."""
    Tinv = oracle.rigid_inverse(pose)
    q = oracle.rigid_apply(Tinv, points)
    r = lambda i, j: Tinv[:, i, j].unsqueeze(-1)
    m = torch.stack([oracle._dot3(r(i, 0), r(i, 1), r(i, 2), normals[..., 0], normals[..., 1], normals[..., 2])
                     for i in range(3)], -1)
    return q, m


def splat_index(points, normals, radii, counts, poses, K, H, W, M):
    """points / normals (B,N,3), radii (B,N,1) padded float32, counts [N_b]; poses (B,L,4,4); K (B,4,4) -> (B,L,H,W)."""
    B, L = poses.shape[:2]
    N = points.shape[1]
    empty = torch.iinfo(torch.int64).max
    keys = torch.full((B * L * H * W,), empty, dtype=torch.int64)
    live = torch.arange(N).view(1, N) < torch.tensor(counts).view(B, 1)
    disk = is_disk(normals, radii) & live
    Kinv = oracle.inverse_intrinsics(K)
    k00, k02 = Kinv[:, 0, 0].view(B, 1), Kinv[:, 0, 2].view(B, 1)
    k11, k12 = Kinv[:, 1, 1].view(B, 1), Kinv[:, 1, 2].view(B, 1)
    ones = torch.ones((), dtype=F32)
    # one-pixel rows: render_oracle's rule on a map of the non-disk rows
    pt_lists = [points[b, :counts[b]][~disk[b, :counts[b]]] for b in range(B)]
    rowmap = torch.zeros((B, max(N, 1)), dtype=torch.int64)  # row of the one-pixel map -> row of the map
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
                n = rowmap[b, j]
                zbits = z[b, j].contiguous().view(torch.int32).to(torch.int64)
                keys.scatter_reduce_(0, ((b * L + l) * H + h) * W + w, (zbits << 32) | n, reduce="amin",
                                     include_self=True)
        # disk rows
        q, m = _camera(points, normals, poses[:, l])
        u, v, _ = oracle.project_map(points, poses[:, l], K)
        cu = u.clamp(-M - 2, W + M + 1).round().long()
        cv = v.clamp(-M - 2, H + M + 1).round().long()
        mq = _dot3(m, q)
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
                tbits = t[b, n].contiguous().view(torch.int32).to(torch.int64)
                slot = ((b * L + l) * H + h[b, n]) * W + w[b, n]
                keys.scatter_reduce_(0, slot, (tbits << 32) | n, reduce="amin", include_self=True)
    index = torch.where(keys == empty, torch.full_like(keys, -1), keys & 0xFFFFFFFF)
    return index.view(B, L, H, W)


def splat_values(points, normals, colors, ccounts, radii, poses, K, index):
    """Outputs at a fixed index (differentiable w.r.t. points, normals, colors, ccounts and poses; any float dtype).
    radii / K only decide which rows are disks and the pixels' rays."""
    B, L, H, W = index.shape
    out = render_oracle.render_values(points, normals, colors, ccounts, poses, index)
    n = index.clamp(min=0).view(B, L * H * W)
    disk = torch.cat([is_disk(normals.detach(), radii), torch.zeros((B, 1), dtype=torch.bool)], 1)
    won = torch.gather(disk, 1, n).view(B, L, H, W) & (index >= 0)
    dt = points.dtype
    Kinv = oracle.inverse_intrinsics(K.to(F32)).to(dt)
    hh = torch.arange(H, dtype=F32).view(1, 1, H, 1).to(dt)
    ww = torch.arange(W, dtype=F32).view(1, 1, 1, W).to(dt)
    dx = Kinv[:, 0, 0].view(B, 1, 1, 1) * ww + Kinv[:, 0, 2].view(B, 1, 1, 1)
    dy = Kinv[:, 1, 1].view(B, 1, 1, 1) * hh + Kinv[:, 1, 2].view(B, 1, 1, 1)
    dx, dy = dx.expand(B, L, H, W), dy.expand(B, L, H, W)

    def gather(t):  # (one zero row appended, as render_oracle does)
        t = torch.cat([t, t.new_zeros(B, 1, 3)], 1)
        return torch.gather(t, 1, n.unsqueeze(-1).expand(B, L * H * W, 3)).view(B, L, H * W, 3)

    Tinv = oracle.rigid_inverse(poses)  # (B,L,4,4)
    q = oracle.rigid_apply(Tinv, gather(points)).view(B, L, H, W, 3)
    r = lambda i, j: Tinv[..., i, j].view(B, L, 1, 1)
    nm = gather(normals).view(B, L, H, W, 3)
    m = torch.stack([oracle._dot3(r(i, 0), r(i, 1), r(i, 2), nm[..., 0], nm[..., 1], nm[..., 2]) for i in range(3)], -1)
    md = oracle._dot3(m[..., 0], m[..., 1], m[..., 2], dx, dy, torch.ones_like(dx))
    t = _dot3(m, q) / torch.where(won, md, torch.ones_like(md))
    depth = torch.where(won.unsqueeze(-1), t.unsqueeze(-1), out.depth)
    return Rendered(depth, out.rgb, out.normals, out.confidence, index)


def disk_ray_cosine(normals, radii, poses, K, index):
    """float64 (B,L,H,W): cos of the angle between a pixel's ray and the normal of the disk row that won it (1 where a
    one-pixel row or nothing won it)."""
    B, L, H, W = index.shape
    n = index.clamp(min=0).view(B, L * H * W)
    disk = torch.cat([is_disk(normals, radii), torch.zeros((B, 1), dtype=torch.bool)], 1)
    won = torch.gather(disk, 1, n).view(B, L, H, W) & (index >= 0)
    nm = torch.gather(torch.cat([normals, normals.new_zeros(B, 1, 3)], 1).double(), 1,
                      n.unsqueeze(-1).expand(B, L * H * W, 3)).view(B, L, H, W, 3)
    R = poses[..., :3, :3].double()  # m = R^T n
    m = torch.einsum("blji,blhwj->blhwi", R, nm)
    Kinv = oracle.inverse_intrinsics(K).double()
    ww = torch.arange(W, dtype=torch.float64).view(1, 1, 1, W)
    hh = torch.arange(H, dtype=torch.float64).view(1, 1, H, 1)
    d = torch.stack([(Kinv[:, 0, 0].view(B, 1, 1, 1) * ww + Kinv[:, 0, 2].view(B, 1, 1, 1)).expand(B, L, H, W),
                     (Kinv[:, 1, 1].view(B, 1, 1, 1) * hh + Kinv[:, 1, 2].view(B, 1, 1, 1)).expand(B, L, H, W),
                     torch.ones(B, L, H, W, dtype=torch.float64)], -1)
    cos = (m * d).sum(-1) / (m.norm(dim=-1) * d.norm(dim=-1)).clamp_min(1e-300)
    return torch.where(won, cos, torch.ones_like(cos))


def splat_views(points, normals, colors, ccounts, radii, counts, poses, K, H, W, M):
    """The full disk render: index, then the values."""
    index = splat_index(points, normals, radii, counts, poses, K, H, W, M)
    return splat_values(points, normals, colors, ccounts, radii, poses, K, index)
