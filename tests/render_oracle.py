"""CPU oracle of gsx_render_views / render_pointclouds, built on the oracle's association (gsx_oracle.project_map and
find_active_map_points) and its canonical arithmetic, so the CUDA path must equal it bit for bit.

    index   per pixel, the table row [b, n, h, w] of find_active_map_points with the smallest key
            (bits(z) << 32) | n  (scatter_reduce 'amin'; z > 0, so the float bits order like the values), or -1
    depth   z of T^-1 p (project_map's z)        normals   R^T n       rgb / confidence   the row's colour / ccount

`render_values` evaluates the outputs at a FIXED index with differentiable torch ops (any float dtype), which is the
backward's definition: the association carries no gradient."""
from collections import namedtuple

import torch

import gsx_oracle as oracle

Rendered = namedtuple("Rendered", "depth rgb normals confidence index")


def render_index(smap, poses, K, H, W):
    """smap: gsx_oracle.SurfelMap; poses (B,L,4,4) camera-to-world; K (B,4,4) -> int64 (B,L,H,W)."""
    B, L = poses.shape[:2]
    empty = torch.iinfo(torch.int64).max
    keys = torch.full((B * L * H * W,), empty, dtype=torch.int64)
    if smap.has_points:
        pts = smap.padded()[0]
        for l in range(L):
            table = oracle.find_active_map_points(smap, poses[:, l], K, H, W)
            if table.shape[0] == 0:
                continue
            _, _, z = oracle.project_map(pts, poses[:, l], K)
            b, n, h, w = table.unbind(1)
            zbits = z[b, n].contiguous().view(torch.int32).to(torch.int64)
            slot = ((b * L + l) * H + h) * W + w
            keys.scatter_reduce_(0, slot, (zbits << 32) | n, reduce="amin", include_self=True)
    index = torch.where(keys == empty, torch.full_like(keys, -1), keys & 0xFFFFFFFF)
    return index.view(B, L, H, W)


def render_values(points, normals, colors, ccounts, poses, index):
    """Outputs at a fixed index.  points / normals / colors (B,N,3), ccounts (B,N,1) padded (normals / colors /
    ccounts may be None); poses (B,L,4,4); index (B,L,H,W) -> Rendered."""
    B, L, H, W = index.shape
    covered = (index >= 0).view(B, L, H * W, 1)
    n = index.clamp(min=0).view(B, L * H * W)

    def gather(t):  # (one zero row appended: a map of no rows still gathers for its uncovered pixels)
        t = torch.cat([t, t.new_zeros(B, 1, t.shape[-1])], 1)
        return torch.gather(t, 1, n.unsqueeze(-1).expand(B, L * H * W, t.shape[-1])).view(B, L, H * W, t.shape[-1])

    def masked(t, c):
        return torch.where(covered, t, torch.zeros_like(t)).view(B, L, H, W, c)

    Tinv = oracle.rigid_inverse(poses)  # (B,L,4,4)
    q = oracle.rigid_apply(Tinv, gather(points))
    depth = masked(q[..., 2:3], 1)
    nrm = None
    if normals is not None:
        m = gather(normals)
        r = lambda i, j: Tinv[..., i, j].unsqueeze(-1)
        nrm = masked(torch.stack([oracle._dot3(r(i, 0), r(i, 1), r(i, 2), m[..., 0], m[..., 1], m[..., 2])
                                  for i in range(3)], -1), 3)
    rgb = None if colors is None else masked(gather(colors), 3)
    conf = None if ccounts is None else masked(gather(ccounts), 1)
    return Rendered(depth, rgb, nrm, conf, index)


def render_views(smap, poses, K, H, W):
    """The full render of a SurfelMap: index, then the gathers."""
    index = render_index(smap, poses, K, H, W)
    if not smap.has_points:
        return Rendered(torch.zeros(index.shape + (1,)), None, None, None, index)
    pts, nrm, col, cc = smap.padded()
    return render_values(pts, nrm, col, cc, poses, index)
