"""Blended splats (render_pointclouds(blend_band=eps), gsx_render_blend) on the GPU: the forward against
tests/blend_oracle.py on ragged maps with a camera per element, past one 32-view chunk and on a fused 640x480 map; the
index image bit for bit R1d's; two runs bit for bit equal; gradients against float64 autograd of the oracle; a loss on
the blended depth reaching rows behind the front and the radii, which the z-buffer render does not; and blend_band=None
unchanged."""
import math

import pytest
import torch

import blend_oracle as bo
import splat_oracle as so
from test_gpu_render_splat import _case, _padded

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _pc(gs, smap, radii, colors=True, features=True, grad=False):
    """Pointclouds on the GPU; with grad, the leaves (points, normals, colours, ccounts, radii) are returned too."""
    leaves = [[t.to(DEV).requires_grad_(grad) for t in lst]
              for lst in (smap.points, smap.normals, smap.colors, smap.ccounts, radii)]
    pc = gs.Pointclouds(points=leaves[0], normals=leaves[1], colors=leaves[2] if colors else None,
                        features=leaves[3] if features else None)
    pc.radii_list = leaves[4]
    return pc, leaves


def _assert_close(got, want, name, atol=2e-5):
    g, w = got.detach().cpu().double(), want.detach().double()
    scale = max(w.abs().max().item(), 1.0)
    torch.testing.assert_close(g, w, rtol=1e-4, atol=atol * scale, msg=name)


def _check_forward(out, want, colors, features):
    # A disk's weight c (1 - s2/r^2) is good to about c 2.4e-7 |q| / r in float32 (e = t d - q cancels): 1e-4 relative
    # at r = 0.005, and up to a few 1e-4 absolute in a mean whose contributors differ by O(1) (normals, or depths
    # with a wide band) when every contributor sits near its rim.
    assert torch.equal(out.index.cpu(), want.index)
    _assert_close(out.depth, want.depth, "depth", atol=1e-3)
    _assert_close(out.normals, want.normals, "normals", atol=1e-3)
    if colors:
        _assert_close(out.rgb, want.rgb, "rgb", atol=1e-3)
    else:
        assert out.rgb is None
    if features:
        _assert_close(out.confidence, want.confidence, "confidence", atol=2e-4)
    else:
        assert out.confidence is None


@pytest.mark.parametrize("M", [0, 1, 4, 16])
@pytest.mark.parametrize("band", [0.0, 0.02, math.inf])
def test_forward_matches_the_oracle(M, band):
    import gradslam_b200 as gs

    H, W = 48, 64
    smap, radii, K, poses = _case(4, seed=M)
    pc, _ = _pc(gs, smap, radii)
    Kd, Pd = K.view(3, 1, 4, 4).to(DEV), poses.to(DEV)
    out = gs.render_pointclouds(pc, Kd, Pd, H, W, max_splat_px=M, blend_band=band)
    pts, nrm, col, cc, rp = _padded(smap, radii)
    want = bo.blend_views(pts.double(), nrm.double(), col.double(), cc.double(), rp, smap.counts(), poses.double(), K,
                          H, W, M, band)
    _check_forward(out, want, True, True)
    assert torch.equal(out.index, gs.render_pointclouds(pc, Kd, Pd, H, W, max_splat_px=M).index)
    con, _, _ = bo.contributors(pts, nrm, rp, smap.counts(), poses, K, H, W, M, band)
    covered = int((out.index >= 0).sum())
    if band > 0:  # pixels with more than one contributor
        assert int((torch.bincount(con.slot) > 1).sum()) > covered // (50 if M else 1000)


@pytest.mark.parametrize("colors,features,with_radii", [(False, True, True), (True, False, True),
                                                        (False, False, False)])
def test_forward_without_colours_confidence_or_radii_past_one_view_chunk(colors, features, with_radii):
    import gradslam_b200 as gs

    H, W, M, band, L = 48, 64, 2, 0.05, 40
    smap, radii, K, poses = _case(L, seed=5)
    if not with_radii:
        radii = [torch.zeros_like(r) for r in radii]
    pc, _ = _pc(gs, smap, radii, colors=colors, features=features)
    out = gs.render_pointclouds(pc, K.view(3, 1, 4, 4).to(DEV), poses.to(DEV), H, W, max_splat_px=M, blend_band=band)
    pts, nrm, col, cc, rp = _padded(smap, radii)
    want = bo.blend_views(pts.double(), nrm.double(), col.double() if colors else None,
                          cc.double() if features else None, rp, smap.counts(), poses.double(), K, H, W, M, band)
    _check_forward(out, want, colors, features)


def test_fused_640x480_map_matches_the_oracle():
    import gradslam_b200 as gs
    from gradslam_b200.synthetic import make_sequence

    H, W, M, band = 480, 640, 4, 0.02
    rgb, depth, K, poses = make_sequence(1, 3, H, W, seed=3)
    frames = gs.RGBDImages(rgb.to(DEV), depth.to(DEV), K.to(DEV), poses.to(DEV))
    pc = gs.PointFusion(odom="gt", device=DEV, surfel_radii=True)(frames)[0]
    view = poses[:, 1:2].clone()
    view[:, 0, 0, 3] += 0.01
    out = gs.render_pointclouds(pc, K.to(DEV), view.to(DEV), H, W, max_splat_px=M, blend_band=band)
    n = pc._host_counts()
    pts, nrm, col = pc.points_padded.cpu(), pc.normals_padded.cpu(), pc.colors_padded.cpu()
    cc, rp = pc.features_padded.cpu(), pc.radii_padded.cpu()
    want = bo.blend_views(pts.double(), nrm.double(), col.double(), cc.double(), rp, n, view.double(), K[:, 0], H, W, M,
                          band)
    # A contributor whose ray meets its disk within about 1e-6 r^2 of the rim has a float32 weight 1 - s2/r^2 of large
    # relative error; fused confidence counts span orders of magnitude, so such a row can hold a sizeable share of a
    # pixel's W.  Allow one pixel in a thousand to differ by more than the tolerance.
    assert torch.equal(out.index.cpu(), want.index)
    covered = int((want.index >= 0).sum())
    for name in ("depth", "rgb", "normals", "confidence"):
        g, w = getattr(out, name).cpu().double(), getattr(want, name)
        off = ((g - w).abs() > 1e-3 * max(w.abs().max().item(), 1e-30) + 1e-4 * w.abs()).any(-1)
        assert int(off.sum()) <= covered // 1000, (name, int(off.sum()))
    assert int((out.index >= 0).sum()) > H * W // 2


def _loss(out, ups):
    return sum((o * u.to(DEV)).sum() for o, u in zip((out.depth, out.normals, out.rgb, out.confidence), ups))


def _backward(gs, smap, radii, K, poses, H, W, M, band, ups):
    pc, leaves = _pc(gs, smap, radii, grad=True)
    P = poses.to(DEV).requires_grad_(True)
    out = gs.render_pointclouds(pc, K.view(3, 1, 4, 4).to(DEV), P, H, W, max_splat_px=M, blend_band=band)
    _loss(out, ups).backward()
    return out, leaves, P


@pytest.mark.parametrize("M,band", [(3, 0.02), (1, math.inf), (0, 0.05)])
def test_backward_against_float64_autograd_and_deterministic(M, band):
    import gradslam_b200 as gs

    H, W = 48, 64
    smap, radii, K, poses = _case(4, seed=2)
    pts, nrm, col, cc, rp = _padded(smap, radii)
    con, index, _ = bo.contributors(pts, nrm, rp, smap.counts(), poses, K, H, W, M, band)
    ref_leaves = [t.double().requires_grad_(True) for t in (pts, nrm, col, cc, rp, poses)]
    ref = bo.blend_values(*ref_leaves[:5], ref_leaves[5], K, con, index)
    g = torch.Generator().manual_seed(4)
    ups = [torch.randn(3, 4, H, W, c, generator=g) for c in (1, 3, 3, 1)]
    # Pixels whose upstream gradient stays zero, where float32 cannot be matched by any float64 reference: a disk met
    # at a grazing angle (|cos| < 0.1: t = (m.q)/(m.d) with a cancelling m.d), and a total weight below 0.01 (every
    # contributor at its rim, where 1 - s2/r^2 cancels).
    bad = (bo.min_disk_cosine(nrm, rp, poses, K, con, index.shape) < 0.1) | (ref.confidence[..., 0].detach() < 1e-2)
    bad &= index >= 0
    assert int(bad.sum()) < int((index >= 0).sum()) // 10
    ups = [torch.where(bad.unsqueeze(-1), torch.zeros_like(u), u) for u in ups]
    out, leaves, P = _backward(gs, smap, radii, K, poses, H, W, M, band, ups)
    assert torch.equal(out.index.cpu(), index)
    sum((o * u.double()).sum() for o, u in zip((ref.depth, ref.normals, ref.rgb, ref.confidence), ups)).backward()
    for k in range(5):
        for b, leaf in enumerate(leaves[k]):
            n = leaf.shape[0]
            if n == 0:
                continue
            want = ref_leaves[k].grad[b, :n]
            got = leaf.grad.cpu().double()
            torch.testing.assert_close(got, want, rtol=1e-3, atol=1e-4 * max(want.abs().max().item(), 1.0),
                                       msg="leaf %d element %d" % (k, b))
    gp = ref_leaves[5].grad
    torch.testing.assert_close(P.grad.cpu().double(), gp, rtol=1e-3, atol=1e-4 * gp.abs().max().item())
    if M > 0:
        assert float(leaves[4][0].grad.abs().sum()) > 0
    # two runs: equal bits, forward and backward
    out2, leaves2, P2 = _backward(gs, smap, radii, K, poses, H, W, M, band, ups)
    for name in ("index", "depth", "rgb", "normals", "confidence"):
        assert torch.equal(getattr(out, name), getattr(out2, name)), name
    for k in range(5):
        for a, b in zip(leaves[k], leaves2[k]):
            if a.shape[0]:
                assert torch.equal(a.grad, b.grad)
    assert torch.equal(P.grad, P2.grad)


def test_blended_depth_reaches_rows_behind_the_front_and_radii_unlike_the_z_buffer():
    import gradslam_b200 as gs

    H, W, M, band = 48, 64, 3, 0.05
    smap, radii, K, poses = _case(4, seed=7)
    pts, nrm, col, cc, rp = _padded(smap, radii)
    con, index, _ = bo.contributors(pts, nrm, rp, smap.counts(), poses, K, H, W, M, band)
    front = set(zip(torch.arange(3).view(3, 1).expand(3, 4 * H * W)[index.view(3, -1) >= 0].tolist(),
                    index.view(3, -1)[index.view(3, -1) >= 0].tolist()))
    behind = sorted(set(zip(con.b.tolist(), con.n.tolist())) - front)
    assert len(behind) > 20

    def grads(blend):
        pc, leaves = _pc(gs, smap, radii, grad=True)
        out = gs.render_pointclouds(pc, K.view(3, 1, 4, 4).to(DEV), poses.to(DEV), H, W, max_splat_px=M,
                                    blend_band=band if blend else None)
        out.depth.sum().backward()
        return leaves

    blended, hard = grads(True), grads(False)
    for leaves, nonzero in ((blended, True), (hard, False)):
        moved = [bool(leaves[0][b].grad[n].abs().sum() > 0) for b, n in behind]
        assert (sum(moved) > len(behind) // 2) if nonzero else not any(moved)
        radii_grad = sum(float(r.grad.abs().sum()) for r in leaves[4] if r.grad is not None)
        assert (radii_grad > 0) == nonzero


def test_no_blend_band_renders_as_before():
    import gradslam_b200 as gs

    H, W, M = 48, 64, 2
    smap, radii, K, poses = _case(4, seed=3)
    pc, _ = _pc(gs, smap, radii)
    Kd, Pd = K.view(3, 1, 4, 4).to(DEV), poses.to(DEV)
    out = gs.render_pointclouds(pc, Kd, Pd, H, W, max_splat_px=M, blend_band=None)
    pts, nrm, col, cc, rp = _padded(smap, radii)
    want = so.splat_views(pts, nrm, col, cc, rp, smap.counts(), poses, K, H, W, M)
    for name in ("index", "depth", "rgb", "normals", "confidence"):
        assert torch.equal(getattr(out, name).cpu(), getattr(want, name)), name
