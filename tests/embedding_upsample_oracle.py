"""CPU oracle of embedding images coarser than the depth (RGBDImages(..., embeddings=e, upsample_embeddings=True)).

The fused map update samples the coarse (h, w) image bilinearly at each pixel of the (H, W) depth, as
F.interpolate(e, (H, W), mode='bilinear', align_corners=False) does.  Along x (y likewise with h, H):

    scale = (float)w / (float)W
    sx = scale * (u + 0.5f) - 0.5f,  0 where that is below 0
    x0 = (int)sx,  x1 = x0 + (x0 < w - 1 ? 1 : 0)
    lx1 = sx - x0,  lx0 = 1 - lx1

    f = ly0 * (lx0 * e[y0,x0] + lx1 * e[y0,x1]) + ly1 * (lx0 * e[y1,x0] + lx1 * e[y1,x1])

in float32, each operation a separate op, in that order; half-precision taps are upcast exactly and f is not rounded to
the storage type.  f then enters the embedding merge of tests/embedding_oracle.py with its rounding: merged
((c0 * E) + (alpha * f)) * inv, appended f.  At h = H, w = W, f is e itself (finite e).

The backward is the adjoint: d e[t] is the sum over fine pixels p, in row-major order, of w_k(p) * d f(p) for every tap k
of p (in the order 00, 01, 10, 11) that lands on texel t, w_00 = ly0 * lx0 and so on; a tap that lands on the same
texel twice at the clamped border counts twice."""
import torch

import embedding_oracle as eo

F32 = torch.float32


def taps(n, m):
    """Fine indices 0..n-1 of an axis upsampled from m coarse samples -> (i0, i1) int64 and (l0, l1) float32 (n,)."""
    scale = torch.tensor(m, dtype=F32) / torch.tensor(n, dtype=F32)
    s = scale * (torch.arange(n, dtype=F32) + 0.5) - 0.5
    s = torch.where(s < 0, torch.zeros_like(s), s)
    i0 = s.to(torch.int64)
    i1 = i0 + (i0 < m - 1).to(torch.int64)
    l1 = s - i0.to(F32)
    l0 = 1 - l1
    return i0, i1, l0, l1


def upsample(e, H, W):
    """(..., h, w, D) channels-last embedding image of any float dtype -> (..., H, W, D) float32 samples f."""
    h, w = e.shape[-3], e.shape[-2]
    y0, y1, ly0, ly1 = taps(H, h)
    x0, x1, lx0, lx1 = taps(W, w)
    ef = e.to(F32)
    ly0, ly1 = ly0.view(H, 1, 1), ly1.view(H, 1, 1)
    lx0, lx1 = lx0.view(1, W, 1), lx1.view(1, W, 1)

    def tap(yi, xi):
        return ef[..., yi, :, :][..., xi, :]

    return ly0 * (lx0 * tap(y0, x0) + lx1 * tap(y0, x1)) + ly1 * (lx0 * tap(y1, x0) + lx1 * tap(y1, x1))


def upsample_adjoint(df, h, w):
    """The adjoint of upsample: df (B, H, W, D) float32 -> d e (B, h, w, D), summed per texel over the pixels in
    row-major order and, per pixel, over its taps in the order 00, 01, 10, 11."""
    B, H, W, D = df.shape
    y0, y1, ly0, ly1 = taps(H, h)
    x0, x1, lx0, lx1 = taps(W, w)
    ys = torch.stack([y0, y0, y1, y1], 1)  # (H, 4): tap k's row
    xs = torch.stack([x0, x1, x0, x1], 1)  # (W, 4)
    wy = torch.stack([ly0, ly0, ly1, ly1], 1)
    wx = torch.stack([lx0, lx1, lx0, lx1], 1)
    t = (ys.view(H, 1, 4) * w + xs.view(1, W, 4)).reshape(-1)  # (H*W*4,) texel of (pixel, tap), pixel-major
    wk = (wy.view(H, 1, 4) * wx.view(1, W, 4)).reshape(-1)  # w_k(p)
    out = torch.zeros((B, h * w, D), dtype=F32)
    for b in range(B):
        src = wk.view(-1, 1) * df[b].reshape(H * W, 1, D).expand(H * W, 4, D).reshape(-1, D)
        out[b].index_add_(0, t, src)  # sequential over the index list on the CPU: pixel-major, tap-minor
    return out.view(B, h, w, D)


def merge_backward(assoc, c0, alpha, E, e, g, H, W):
    """Backward of the upsampled merge for one frame, float32 (the GPU kernels' statement): assoc (B, P) as K4 writes
    it (appended rows at or past N), c0 / alpha (B, P) of the merged pixels, E (B, N, D) the map's N rows of embeddings
    before the merge, e (B, h, w, D) the coarse image, g (B, cap_out, D) the upstream gradient.  Returns (d E (B, N, D):
    g c0 inv for merged rows, g for the others; d e; d c0; d alpha)."""
    B, P = assoc.shape
    h, w, D = e.shape[1], e.shape[2], e.shape[3]
    f = upsample(e, H, W).reshape(B, P, D)
    dE = g[:, :E.shape[1]].clone()
    df = torch.zeros((B, P, D), dtype=F32)
    dc0 = torch.zeros((B, P), dtype=F32)
    dal = torch.zeros((B, P), dtype=F32)
    for b in range(B):
        a = assoc[b]
        m = (a < 0).nonzero().flatten()
        n = -a[m].long() - 1
        cb, ab = c0[b, m].view(-1, 1), alpha[b, m].view(-1, 1)
        tot = cb + ab
        inv = 1 / torch.where(tot == 0, torch.ones_like(tot), tot)
        dinv = torch.where(tot == 0, torch.zeros_like(inv), -(inv * inv))
        gm, Em, fm = g[b, n], E[b, n], f[b, m]
        num = cb * Em + ab * fm
        dE[b, n] = gm * cb * inv
        df[b, m] = gm * ab * inv
        dc0[b, m] = (gm * (Em * inv + num * dinv)).sum(1)
        dal[b, m] = (gm * (fm * inv + num * dinv)).sum(1)
        ap = (a > 0).nonzero().flatten()
        df[b, ap] = g[b, a[ap].long() - 1]
    return dE, upsample_adjoint(df.view(B, H, W, D), h, w), dc0, dal


def _stored(emb, dtype):
    return [x.to(dtype) for x in emb]


def run_pointfusion(rgb, depth, K, poses, e, **kw):
    """PointFusion with odom='gt' over (B, L) frames with coarse embedding images e (B, L, h, w, D).  Returns
    (SurfelMap, embeddings list of e's dtype)."""
    import gsx_oracle as oracle

    H, W = depth.shape[2], depth.shape[3]
    dist_th, sigma = kw.get("dist_th", 0.05), kw.get("sigma", 0.6)
    dot_th = eo.math.cos(kw.get("angle_th", 20.0) * eo.math.pi / 180)
    smap, out = oracle.SurfelMap(), None
    for s in range(depth.shape[1]):
        pose = poses[:, s]
        maps = oracle.frame_maps(depth[:, s:s + 1], K, pose.unsqueeze(1))
        table = oracle.find_correspondences(smap, maps, pose, K[:, 0], dist_th, dot_th)
        smap, out = eo.fuse_with_map(smap, out, maps, rgb[:, s:s + 1], upsample(e[:, s:s + 1], H, W), table, sigma)
        out = _stored(out, e.dtype)  # merged rows are rounded already; appended rows take f rounded once
    return smap, out


def run_aggregate(rgb, depth, K, poses, e):
    """ICPSLAM with odom='gt' (every valid pixel appended with its sample f) with coarse embedding images."""
    H, W = depth.shape[2], depth.shape[3]
    smap, emb = eo.run_aggregate(rgb, depth, K, poses, upsample(e, H, W))
    return smap, _stored(emb, e.dtype)
