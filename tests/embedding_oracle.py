"""CPU oracle of per-surfel embeddings (RGBDImages(embeddings=...) fused by PointFusion / ICPSLAM).

gsx_oracle.fuse_with_map and update_map_aggregate restated with a list of per-element (N_b, D) embeddings beside the
colours.  With the association the oracle computes, per pixel:

    merged into row n     c0 = the row's confidence before the merge, alpha = the pixel's confidence weight,
                          tot = c0 + alpha, inv = 1 / (tot == 0 ? 1 : tot),
                          E[n, d] = ((c0 * E[n, d]) + (alpha * e[pix, d])) * inv     (the colour merge's expression)
    appended as row n     E[n] = e[pix]
    untouched rows        keep their embedding bit for bit

Every operation is a separate float32 torch op, as the kernels compute it.  A float16 / bfloat16 map is read by an
exact upcast and each merged value is rounded once to the storage dtype: the map's stored values are rounded after
every frame.  With e := rgb (D = 3, float32) the embeddings equal the colours bit for bit."""
import math

import torch

import gsx_oracle as oracle

F32 = torch.float32


def fuse_with_map(smap, emb, maps, rgb, e, pc2im, sigma):
    """gsx_oracle.fuse_with_map with embeddings: emb = smap's (list of (N_b, D), None for an empty map), e (B,1,H,W,D).
    Returns (new SurfelMap, new embeddings list)."""
    gv, gn, col, ef = maps["gvertex"][:, 0], maps["gnormal"][:, 0], rgb[:, 0], e[:, 0]
    alpha = oracle.get_alpha(maps["vertex"][:, 0], sigma)  # (B,H,W,1)
    valid = maps["valid"][:, 0]
    B = gv.shape[0]
    out = smap.clone()
    out_e = [x.clone() for x in emb] if smap.has_points else [ef.new_zeros((0, ef.shape[-1])) for _ in range(B)]
    new_mask = torch.ones_like(valid)
    if smap.has_points and pc2im.shape[0] != 0:
        b, n, h, w = pc2im.unbind(1)
        for i in range(B):
            sel = b == i
            ni, hi, wi = n[sel], h[sel], w[sel]
            cc = out.ccounts[i][ni]
            a = alpha[i, hi, wi]
            tot = cc + a
            inv = 1 / torch.where(tot == 0, torch.ones_like(tot), tot)
            out.points[i][ni] = ((cc * out.points[i][ni]) + (a * gv[i, hi, wi])) * inv
            out.normals[i][ni] = ((cc * out.normals[i][ni]) + (a * gn[i, hi, wi])) * inv
            out.colors[i][ni] = ((cc * out.colors[i][ni]) + (a * col[i, hi, wi])) * inv
            merged = ((cc * out_e[i][ni].to(F32)) + (a * ef[i, hi, wi].to(F32))) * inv
            out_e[i][ni] = merged.to(out_e[i].dtype)
            out.ccounts[i][ni] = tot
        new_mask[b, h, w] = False
    new_mask = new_mask & valid
    fresh = oracle.SurfelMap(
        [gv[i][new_mask[i]] for i in range(B)],
        [gn[i][new_mask[i]] for i in range(B)],
        [col[i][new_mask[i]] for i in range(B)],
        [alpha[i][new_mask[i]] for i in range(B)],
    )
    return out.append(fresh), [torch.cat([out_e[i], ef[i][new_mask[i]]], 0) for i in range(B)]


def update_map_aggregate(smap, emb, maps, rgb, e):
    """gsx_oracle.update_map_aggregate with embeddings: every valid pixel is appended with its embedding."""
    valid = maps["valid"][:, 0]
    B = valid.shape[0]
    ef = e[:, 0]
    fresh = [ef[i][valid[i]] for i in range(B)]
    emb = fresh if emb is None else [torch.cat([x, y], 0) for x, y in zip(emb, fresh)]
    return oracle.update_map_aggregate(smap, maps, rgb), emb


def run_pointfusion(rgb, depth, K, poses, emb, *, dist_th=0.05, angle_th=20.0, sigma=0.6):
    """PointFusion with odom='gt' over (B, L) frames with embeddings emb (B,L,H,W,D).  Returns (SurfelMap, embeddings)."""
    dot_th = math.cos(angle_th * math.pi / 180)
    smap, out = oracle.SurfelMap(), None
    for s in range(depth.shape[1]):
        pose = poses[:, s]
        maps = oracle.frame_maps(depth[:, s:s + 1], K, pose.unsqueeze(1))
        table = oracle.find_correspondences(smap, maps, pose, K[:, 0], dist_th, dot_th)
        smap, out = fuse_with_map(smap, out, maps, rgb[:, s:s + 1], emb[:, s:s + 1], table, sigma)
    return smap, out


def run_aggregate(rgb, depth, K, poses, emb):
    """ICPSLAM with odom='gt' (every valid pixel appended) with embeddings.  Returns (SurfelMap, embeddings)."""
    smap, out = oracle.SurfelMap(), None
    for s in range(depth.shape[1]):
        maps = oracle.frame_maps(depth[:, s:s + 1], K, poses[:, s:s + 1])
        smap, out = update_map_aggregate(smap, out, maps, rgb[:, s:s + 1], emb[:, s:s + 1])
    return smap, out


def random_embeddings(B, L, H, W, D, dtype=F32, seed=0):
    """Deterministic embedding images (B, L, H, W, D) in [-1, 1) of the given storage dtype."""
    g = torch.Generator().manual_seed(seed)
    return (torch.rand((B, L, H, W, D), generator=g, dtype=F32) * 2 - 1).to(dtype)
