"""render_pointclouds / gsx_render_views (R1 z-buffer, R2 resolve, R3 backward) on the GPU: bit-for-bit parity with the
render oracle (tests/render_oracle.py), agreement with the fusion step's association, a fuse-then-render round trip,
the benchmark's map, gradients against float64 autograd, and determinism."""
import math

import pytest
import torch

import gsx_oracle as oracle
import render_oracle
from gradslam_b200.synthetic import intrinsics as synth_intrinsics, make_sequence, punch_lattice_holes

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _yaw_pose(yaw, t):
    c, s = math.cos(yaw), math.sin(yaw)
    T = torch.eye(4, dtype=torch.float64)
    T[:3, :3] = torch.tensor([[c, 0.0, s], [0.0, 1.0, 0.0], [-s, 0.0, c]], dtype=torch.float64)
    T[:3, 3] = torch.tensor(t, dtype=torch.float64)
    return T.float()


def _ragged_map(H, W, seed=0):
    """B = 3 maps: element 0 with exact duplicates (ties), rows around z = 0 and rows straddling the image border;
    element 1 empty; element 2 a plain cloud.  Returns (SurfelMap, K (B,4,4), poses (B,4,4,4))."""
    g = torch.Generator().manual_seed(seed)
    K = torch.from_numpy(synth_intrinsics(H, W)).float()
    fx, cx, cy = K[0, 0].item(), K[0, 2].item(), K[1, 2].item()
    z = torch.rand(3000, generator=g) * 2.0 + 0.5
    u, v = torch.rand(3000, generator=g) * (W + 8) - 4, torch.rand(3000, generator=g) * (H + 8) - 4  # past the border
    p0 = torch.stack([(u - cx) / fx * z, (v - cy) / fx * z, z], 1)
    near = torch.rand(200, 3, generator=g) * torch.tensor([0.2, 0.2, 0.02]) - torch.tensor([0.1, 0.1, 0.01])  # z ~ 0
    p0 = torch.cat([p0, near, p0[:300], p0[100:150]], 0)  # duplicates: the lower index must win
    p2 = torch.randn(800, 3, generator=g) * torch.tensor([0.6, 0.4, 0.3]) + torch.tensor([0.0, 0.0, 2.0])
    pts = [p0, torch.zeros(0, 3), p2]
    unit = lambda p: torch.nn.functional.normalize(torch.randn(p.shape[0], 3, generator=g), dim=1)
    smap = oracle.SurfelMap(pts, [unit(p) for p in pts], [torch.rand(p.shape[0], 3, generator=g) for p in pts],
                            [torch.randint(1, 20, (p.shape[0], 1), generator=g).float() for p in pts])
    poses = torch.stack([torch.stack([_yaw_pose(0.03 * l * (b + 1), (0.02 * l, -0.01 * l, 0.03 * l)) for l in range(4)])
                         for b in range(3)])
    return smap, K.repeat(3, 1, 1), poses


def _gpu_pointclouds(gs, smap, colors=True, features=True):
    dev = lambda lst: None if lst is None else [t.to(DEV) for t in lst]
    return gs.Pointclouds(points=dev(smap.points), normals=dev(smap.normals),
                          colors=dev(smap.colors) if colors else None, features=dev(smap.ccounts) if features else None)


def _assert_equal_render(got, want):
    for name in ("index", "depth", "rgb", "normals", "confidence"):
        g, w = getattr(got, name), getattr(want, name)
        assert torch.equal(g.cpu(), w), name


def test_parity_with_the_oracle_bit_for_bit():
    import gradslam_b200 as gs

    H, W = 48, 64
    smap, K, poses = _ragged_map(H, W)
    pc = _gpu_pointclouds(gs, smap)
    out = gs.render_pointclouds(pc, K.view(3, 1, 4, 4).to(DEV), poses.to(DEV), H, W)
    want = render_oracle.render_views(smap, poses, K, H, W)
    _assert_equal_render(out, want)
    assert (out.index[1] == -1).all() and (out.index[0] >= 0).sum() > 1000 and (out.index[2] >= 0).sum() > 300
    assert out.depth.shape == (3, 4, H, W, 1) and out.rgb.shape == (3, 4, H, W, 3) and out.index.dtype == torch.int64


def _canonical_z(pts, pose):
    """z of T^-1 p with the canonical rounding (each product and sum rounded, left to right), elementwise on the GPU."""
    R, t = pose[:3, :3], pose[:3, 3]
    tz = ((-R[0, 2]) * t[0] + (-R[1, 2]) * t[1]) + (-R[2, 2]) * t[2]
    return ((R[0, 2] * pts[:, 0] + R[1, 2] * pts[:, 1]) + R[2, 2] * pts[:, 2]) + tz


def test_index_agrees_with_find_active_map_points():
    """Per pixel, index = the minimum-(z, n) row among the rows fusionutils.find_active_map_points assigns to it."""
    import gradslam_b200 as gs
    from gradslam_b200.slam import fusionutils

    H, W = 48, 64
    smap, K, poses = _ragged_map(H, W, seed=1)
    pc = _gpu_pointclouds(gs, smap)
    Kd, Pd = K.view(3, 1, 4, 4).to(DEV), poses.to(DEV)
    out = gs.render_pointclouds(pc, Kd, Pd, H, W)
    B, L = 3, 4
    pts = pc.points_padded
    for l in range(L):
        frame = gs.RGBDImages(torch.zeros(B, 1, H, W, 3, device=DEV), torch.ones(B, 1, H, W, 1, device=DEV), Kd,
                              Pd[:, l:l + 1])
        table = fusionutils.find_active_map_points(pc, frame)
        b, n, h, w = table.unbind(1)
        z = torch.stack([_canonical_z(pts[e], Pd[e, l]) for e in range(B)])[b, n]
        keys = torch.full((B * H * W,), torch.iinfo(torch.int64).max, dtype=torch.int64, device=DEV)
        keys.scatter_reduce_(0, (b * H + h) * W + w, (z.view(torch.int32).to(torch.int64) << 32) | n, reduce="amin")
        want = torch.where(keys == torch.iinfo(torch.int64).max, torch.full_like(keys, -1), keys & 0xFFFFFFFF)
        assert torch.equal(out.index[:, l].reshape(-1), want), l


def test_fuse_then_render_round_trip():
    import gradslam_b200 as gs

    B, H, W = 8, 480, 640
    rgb, depth, K, poses = make_sequence(B, 1, H, W, seed=0)
    frames = gs.RGBDImages(rgb.to(DEV), depth.to(DEV), K.to(DEV), poses.to(DEV))
    pc, _ = gs.PointFusion(odom="gt", device=DEV)(frames)
    out = gs.render_pointclouds(pc, K.to(DEV), poses.to(DEV), H, W)
    valid = depth.to(DEV)[..., 0] > 0  # (B,1,H,W)
    assert torch.equal(out.index >= 0, valid)
    rows = torch.cumsum(valid.reshape(B, -1).to(torch.int64), 1).reshape(valid.shape) - 1  # appended in row-major order
    assert torch.equal(out.index[valid], rows[valid])
    assert torch.equal(out.rgb[valid], frames.rgb_image[valid])
    d = frames.depth_image
    torch.testing.assert_close(out.depth[valid], d[valid], rtol=1e-5, atol=0)
    torch.testing.assert_close(out.normals[valid], frames.normal_map[valid], rtol=0, atol=1e-5)
    assert (out.depth[~valid] == 0).all() and (out.rgb[~valid] == 0).all()
    # a render is a frame batch the rest of the API accepts
    again = gs.RGBDImages(out.rgb, out.depth, K.to(DEV), poses.to(DEV))
    assert again.shape == (B, 1, H, W)


def test_bench_map_matches_the_oracle():
    """The benchmark's map (B = 8, 32 frames, 640x480, seed 0: ~1.1 M rows per element, many grid-stride passes of R1)
    rendered from poses 0, 15 and 31; elements 0 and 7 against the oracle, bit for bit."""
    import gradslam_b200 as gs

    B, L, H, W = 8, 32, 480, 640
    rgb, depth, K, poses = make_sequence(B, L, H, W, seed=0)
    pc, _ = gs.PointFusion(odom="gt", device=DEV)(gs.RGBDImages(rgb.to(DEV), depth.to(DEV), K.to(DEV), poses.to(DEV)))
    views = poses[:, [0, 15, 31]]
    out = gs.render_pointclouds(pc, K.to(DEV), views.to(DEV), H, W)
    assert min(pc.num_points_per_pointcloud.tolist()) > 600000
    for b in (0, 7):
        smap = oracle.SurfelMap([pc.points_list[b].cpu()], [pc.normals_list[b].cpu()], [pc.colors_list[b].cpu()],
                                [pc.features_list[b].cpu()])
        want = render_oracle.render_views(smap, views[b:b + 1], K[b:b + 1, 0], H, W)
        got = render_oracle.Rendered(*(t[b:b + 1] for t in (out.depth, out.rgb, out.normals, out.confidence,
                                                            out.index)))
        _assert_equal_render(got, want)


def test_backward_against_float64_autograd():
    import gradslam_b200 as gs

    H, W = 48, 64
    smap, K, poses = _ragged_map(H, W, seed=2)
    # rows behind every camera: never visible
    smap.points[2] = torch.cat([smap.points[2], torch.tensor([[0.0, 0.0, -2.0], [0.3, 0.1, -1.0]])])
    for lst, row in ((smap.normals, [0.0, 0.0, 1.0]), (smap.colors, [0.5, 0.5, 0.5]), (smap.ccounts, [3.0])):
        lst[2] = torch.cat([lst[2], torch.tensor([row, row])])
    leaves = [[t.to(DEV).requires_grad_(True) for t in lst]
              for lst in (smap.points, smap.normals, smap.colors, smap.ccounts)]
    P = poses.to(DEV).requires_grad_(True)
    pc = gs.Pointclouds(points=leaves[0], normals=leaves[1], colors=leaves[2], features=leaves[3])
    out = gs.render_pointclouds(pc, K.view(3, 1, 4, 4).to(DEV), P, H, W)
    g = torch.Generator().manual_seed(4)
    ups = [torch.randn(3, 4, H, W, c, generator=g) for c in (1, 3, 3, 1)]
    loss = sum((o * u.to(DEV)).sum() for o, u in zip((out.depth, out.normals, out.rgb, out.confidence), ups))
    loss.backward()

    index = out.index.cpu()
    assert torch.equal(index, render_oracle.render_index(smap, poses, K, H, W))
    ref_leaves = [t.double().requires_grad_(True) for t in smap.padded()] + [poses.double().requires_grad_(True)]
    ref = render_oracle.render_values(*ref_leaves, index)
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
    assert (P.grad[..., 3, :] == 0).all()
    # a row that wins pixels in several views, and the never-visible rows' gradients exactly zero
    wins = torch.zeros(3, 4000, dtype=torch.int64)
    for l in range(4):
        e, pix = (index[:, l] >= 0).reshape(3, -1).nonzero().unbind(1)
        wins[e, index[:, l].reshape(3, -1)[e, pix]] += 1
    assert (wins > 1).any()
    assert (leaves[0][2].grad[-2:] == 0).all() and (leaves[2][2].grad[-2:] == 0).all()
    # padding rows of the packed store get zero
    pc2 = _gpu_pointclouds(gs, smap)
    geo = pc2._geo.detach().clone().requires_grad_(True)
    pc2._geo = geo
    out2 = gs.render_pointclouds(pc2, K.view(3, 1, 4, 4).to(DEV), poses.to(DEV), H, W)
    (out2.depth.sum() + out2.normals.sum() + out2.confidence.sum()).backward()
    counts = pc2.num_points_per_pointcloud.tolist()
    assert counts[1] == 0
    for b, c in enumerate(counts):
        assert (geo.grad[b, c:] == 0).all()
    assert (geo.grad[..., 7] == 0).all() and geo.grad[0, :counts[0]].abs().sum() > 0
    # the formula the kernels implement, checked numerically (float64 gradcheck) at the index of a tiny render
    Hs, Ws = 6, 8
    Ks = torch.from_numpy(synth_intrinsics(Hs, Ws)).float().repeat(3, 1, 1)
    tiny = oracle.SurfelMap(*([t[:20] for t in lst] for lst in (smap.points, smap.normals, smap.colors, smap.ccounts)))
    idx = gs.render_pointclouds(_gpu_pointclouds(gs, tiny), Ks.view(3, 1, 4, 4).to(DEV), poses.to(DEV), Hs, Ws).index
    idx = idx.cpu()
    assert (idx >= 0).sum() > 10

    def f(*xs):
        o = render_oracle.render_values(*xs, idx)
        return o.depth, o.normals, o.rgb, o.confidence

    small = [t.double().requires_grad_(True) for t in tiny.padded()] + [poses.double().requires_grad_(True)]
    assert torch.autograd.gradcheck(f, tuple(small), eps=1e-6, atol=1e-6, fast_mode=True)


def test_gradients_through_differentiable_fusion():
    """Differentiable PointFusion(odom='gt') (K1 and K4 backward), then a render from pose 1: d loss / d(input depth,
    colours) against the oracle's autograd of the same chain (the tolerance of test_gpu_backward.py)."""
    import gradslam_b200 as gs

    B, L, H, W = 2, 3, 48, 64
    rgb, depth, K, poses = make_sequence(B, L, H, W, seed=41, yaw0=0.6, hole_fraction=0.0)
    depth = punch_lattice_holes(depth)
    target = depth[:, 1:2] * 1.01

    d_ref, c_ref = depth.clone().requires_grad_(True), rgb.clone().requires_grad_(True)
    ref_map = oracle.run_slam(c_ref, d_ref, K, poses, odom="gt").map
    ref = render_oracle.render_views(ref_map, poses[:, 1:2], K[:, 0], H, W)
    (((ref.depth - target) ** 2).sum() + ref.rgb.sum()).backward()

    d_gpu, c_gpu = depth.to(DEV).requires_grad_(True), rgb.to(DEV).requires_grad_(True)
    pc, _ = gs.PointFusion(odom="gt", device=DEV)(gs.RGBDImages(c_gpu, d_gpu, K.to(DEV), poses.to(DEV)))
    out = gs.render_pointclouds(pc, K.to(DEV), poses[:, 1:2].to(DEV), H, W)
    assert torch.equal(out.index.cpu(), ref.index)
    (((out.depth - target.to(DEV)) ** 2).sum() + out.rgb.sum()).backward()
    for got, want in ((d_gpu.grad.cpu(), d_ref.grad), (c_gpu.grad.cpu(), c_ref.grad)):
        assert torch.isfinite(got).all()
        scale = want.abs().max().item()
        assert scale > 0
        torch.testing.assert_close(got, want, rtol=1e-3, atol=1e-4 * scale)


def test_determinism_and_mode_equality():
    import gradslam_b200 as gs

    H, W = 48, 64
    smap, K, poses = _ragged_map(H, W, seed=3)
    Kd, Pd = K.view(3, 1, 4, 4).to(DEV), poses.to(DEV)
    pc = _gpu_pointclouds(gs, smap)
    a = gs.render_pointclouds(pc, Kd, Pd, H, W)
    b = gs.render_pointclouds(pc, Kd, Pd, H, W)
    for x, y in zip(a, b):
        assert torch.equal(x, y)
    # the autograd path runs the same forward kernels
    Pg = Pd.clone().requires_grad_(True)
    c = gs.render_pointclouds(pc, Kd, Pg, H, W)
    assert c.depth.requires_grad and not c.index.requires_grad
    for x, y in zip(a, c):
        assert torch.equal(x, y.detach())
    # a map without colours or confidence: depth only, same depth and index
    d = gs.render_pointclouds(_gpu_pointclouds(gs, smap, colors=False, features=False), Kd, Pd, H, W)
    assert d.rgb is None and d.confidence is None
    assert torch.equal(d.depth, a.depth) and torch.equal(d.index, a.index) and torch.equal(d.normals, a.normals)
    # an empty map: every pixel uncovered
    e = gs.render_pointclouds(gs.Pointclouds(device=DEV), Kd, Pd, H, W)
    assert (e.index == -1).all() and (e.depth == 0).all() and e.rgb is None
