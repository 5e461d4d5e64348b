"""Disk-splat rendering (render_pointclouds(max_splat_px >= 1), R1d): bit for bit against tests/splat_oracle.py on ragged
maps with a camera per element, mixed zero and non-zero radii and more than 32 views; today's output at max_splat_px = 0
and on maps without radii; the backward against float64 autograd of the oracle at the fixed index, deterministic; and
the holes of a one-frame plane filled."""
import pytest
import torch

import splat_oracle as so
from test_gpu_render import _ragged_map

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _radii(smap, seed):
    """Per element (N_b, 1): half the rows without a radius, the others 0.005 .. 0.05 (about 0.3 .. 3 pixels)."""
    g = torch.Generator().manual_seed(seed)
    out = []
    for p in smap.points:
        r = torch.rand(p.shape[0], 1, generator=g) * 0.045 + 0.005
        r[torch.rand(p.shape[0], generator=g) < 0.5] = 0.0
        out.append(r)
    return out


def _case(L, seed=0, H=48, W=64):
    smap, K, poses = _ragged_map(H, W, seed=seed)
    K = K.clone()
    for b in range(3):  # a camera per element
        K[b, 0, 0] *= 1.0 + 0.07 * b
        K[b, 1, 1] *= 1.0 - 0.05 * b
        K[b, 0, 2] += 1.5 * b
    if L != poses.shape[1]:
        poses = torch.stack([torch.stack([poses[b, l % 4] for l in range(L)]) for b in range(3)])
        poses[:, :, 0, 3] += torch.arange(L, dtype=torch.float32).view(1, L) * 0.003
    return smap, _radii(smap, seed + 1), K, poses


def _padded(smap, radii):
    pts, nrm, col, cc = smap.padded()
    N = pts.shape[1]
    rp = torch.zeros(len(radii), N, 1)
    for b, r in enumerate(radii):
        rp[b, :r.shape[0]] = r
    return pts, nrm, col, cc, rp


def _pointclouds(gs, smap, radii):
    dev = lambda lst: [t.to(DEV) for t in lst]
    pc = gs.Pointclouds(points=dev(smap.points), normals=dev(smap.normals), colors=dev(smap.colors),
                        features=dev(smap.ccounts))
    pc.radii_list = dev(radii)
    return pc


def _assert_equal(got, want):
    for name in ("index", "depth", "rgb", "normals", "confidence"):
        assert torch.equal(getattr(got, name).cpu(), getattr(want, name)), name


@pytest.mark.parametrize("L,M", [(4, 3), (35, 2)], ids=["4_views", "35_views"])
def test_disk_render_matches_the_oracle_bit_for_bit(L, M):
    import gradslam_b200 as gs

    H, W = 48, 64
    smap, radii, K, poses = _case(L)
    pc = _pointclouds(gs, smap, radii)
    out = gs.render_pointclouds(pc, K.view(3, 1, 4, 4).to(DEV), poses.to(DEV), H, W, max_splat_px=M)
    pts, nrm, col, cc, rp = _padded(smap, radii)
    want = so.splat_views(pts, nrm, col, cc, rp, smap.counts(), poses, K, H, W, M)
    _assert_equal(out, want)
    idx = out.index.cpu()
    disk = so.is_disk(nrm, rp)
    won_by_disk = torch.gather(torch.cat([disk, torch.zeros(3, 1, dtype=torch.bool)], 1), 1,
                               idx.clamp(min=0).view(3, -1)).view(idx.shape) & (idx >= 0)
    assert int(won_by_disk.sum()) > 1000 and int(((idx >= 0) & ~won_by_disk).sum()) > 100  # both kinds visible
    # disks cover more than points
    point = gs.render_pointclouds(pc, K.view(3, 1, 4, 4).to(DEV), poses.to(DEV), H, W)
    assert int((out.index >= 0).sum()) > int((point.index >= 0).sum())


def test_zero_max_splat_px_and_maps_without_radii_render_as_before():
    import gradslam_b200 as gs
    import render_oracle

    H, W = 48, 64
    smap, radii, K, poses = _case(4, seed=3)
    Kd, Pd = K.view(3, 1, 4, 4).to(DEV), poses.to(DEV)
    before = render_oracle.render_views(smap, poses, K, H, W)
    with_radii = _pointclouds(gs, smap, radii)
    _assert_equal(gs.render_pointclouds(with_radii, Kd, Pd, H, W, max_splat_px=0), before)
    plain = _pointclouds(gs, smap, [torch.zeros_like(r) for r in radii])
    for M in (1, 4, 16):
        _assert_equal(gs.render_pointclouds(plain, Kd, Pd, H, W, max_splat_px=M), before)


def _backward(gs, smap, radii, K, poses, H, W, M, ups):
    leaves = [[t.to(DEV).requires_grad_(True) for t in lst]
              for lst in (smap.points, smap.normals, smap.colors, smap.ccounts)]
    P = poses.to(DEV).requires_grad_(True)
    pc = gs.Pointclouds(points=leaves[0], normals=leaves[1], colors=leaves[2], features=leaves[3])
    pc.radii_list = [r.to(DEV) for r in radii]
    out = gs.render_pointclouds(pc, K.view(3, 1, 4, 4).to(DEV), P, H, W, max_splat_px=M)
    loss = sum((o * u.to(DEV)).sum() for o, u in zip((out.depth, out.normals, out.rgb, out.confidence), ups))
    loss.backward()
    return out, leaves, P


def test_backward_against_float64_autograd_and_deterministic():
    import gradslam_b200 as gs

    H, W, M = 48, 64, 3
    smap, radii, K, poses = _case(4, seed=2)
    g = torch.Generator().manual_seed(4)
    ups = [torch.randn(3, 4, H, W, c, generator=g) for c in (1, 3, 3, 1)]
    pts, nrm, col, cc, rp = _padded(smap, radii)
    index = so.splat_index(pts, nrm, rp, smap.counts(), poses, K, H, W, M)
    # pixels where a disk meets the ray at a grazing angle (|cos| < 0.1) take no upstream gradient: there dt/dq =
    # m / (m.d) is ill-conditioned in float32 (m.d is a cancelling sum) and no float64 reference can be matched
    graze = so.disk_ray_cosine(nrm, rp, poses, K, index).abs() < 0.1
    ups = [torch.where(graze.unsqueeze(-1), torch.zeros_like(u), u) for u in ups]
    out, leaves, P = _backward(gs, smap, radii, K, poses, H, W, M, ups)
    assert torch.equal(out.index.cpu(), index)
    assert 0 < int(graze.sum()) < int((index >= 0).sum()) // 20
    ref_leaves = [t.double().requires_grad_(True) for t in (pts, nrm, col, cc)] + [poses.double().requires_grad_(True)]
    ref = so.splat_values(*ref_leaves[:4], rp, ref_leaves[4], K, index)
    sum((o * u.double()).sum() for o, u in zip((ref.depth, ref.normals, ref.rgb, ref.confidence), ups)).backward()
    for k in range(4):
        for b, leaf in enumerate(leaves[k]):
            n = leaf.shape[0]
            if n == 0:
                continue
            want = ref_leaves[k].grad[b, :n]
            got = leaf.grad.cpu().double()
            torch.testing.assert_close(got, want, rtol=1e-4, atol=1e-5 * max(want.abs().max().item(), 1.0))
    gp = ref_leaves[4].grad
    torch.testing.assert_close(P.grad.cpu().double(), gp, rtol=1e-3, atol=1e-4 * gp.abs().max().item())
    # a disk row that wins several pixels of one view
    disk = so.is_disk(nrm, rp)
    e, pix = (index[:, 0] >= 0).reshape(3, -1).nonzero().unbind(1)
    rows = index[:, 0].reshape(3, -1)[e, pix]
    assert bool(disk[e, rows].any()) and len(set(zip(e.tolist(), rows.tolist()))) < rows.numel()
    # two runs: bitwise-equal gradients
    _, leaves2, P2 = _backward(gs, smap, radii, K, poses, H, W, M, ups)
    for k in range(4):
        for a, b in zip(leaves[k], leaves2[k]):
            if a.shape[0]:  # (the empty element's leaves take no gradient)
                assert torch.equal(a.grad, b.grad)
    assert torch.equal(P.grad, P2.grad)


def test_disks_fill_the_holes_of_a_one_frame_plane():
    """A fronto-parallel wall fused from one frame with isolated one-pixel depth holes, rendered from that camera: the
    holes stay empty with one pixel per row and are covered with disks."""
    import gradslam_b200 as gs
    from gradslam_b200.synthetic import intrinsics as synth_intrinsics

    H, W = 48, 64
    K = torch.from_numpy(synth_intrinsics(H, W)).float().view(1, 1, 4, 4)
    depth = torch.full((1, 1, H, W, 1), 2.0)
    holes = torch.zeros(H, W, dtype=torch.bool)
    holes[3:H - 3:5, 4:W - 3:6] = True  # isolated pixels, away from the border
    depth[0, 0, holes] = 0.0
    rgb = torch.rand(1, 1, H, W, 3, generator=torch.Generator().manual_seed(0))
    frames = gs.RGBDImages(rgb.to(DEV), depth.to(DEV), K.to(DEV), torch.eye(4).view(1, 1, 4, 4).to(DEV))
    pc = gs.PointFusion(odom="gt", device=DEV, surfel_radii=True)(frames)[0]
    Kd, Pd = K.to(DEV), torch.eye(4).view(1, 1, 4, 4).to(DEV)
    point = gs.render_pointclouds(pc, Kd, Pd, H, W).index[0, 0].cpu()
    assert torch.equal(point < 0, holes)
    disk = gs.render_pointclouds(pc, Kd, Pd, H, W, max_splat_px=2)
    assert bool((disk.index >= 0).all()) and bool((disk.depth > 0).all())
