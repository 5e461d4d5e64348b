"""The bilateral depth filter on the GPU (gsx_depth_bilateral / gsx_depth_bilateral_bwd, bilateral_filter_depth and the
depth_filter keywords of PointFusion / ICPSLAM): the forward is bit-identical to the float32 statement of
tests/bilateral_oracle.py, the backward matches autograd of its float64 statement, and the SLAM drivers filter exactly
what they are documented to filter."""
import math

import numpy as np
import pytest
import torch

import bilateral_oracle as bo
import gradslam_b200 as gs
from gradslam_b200.synthetic import add_depth_noise, make_sequence

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _bits(t):
    return np.ascontiguousarray(t, dtype=np.float32).view(np.uint32)


def _assert_forward_exact(depth, f):
    """depth: (B,L,H,W,1) CPU float32.  The GPU filter equals the float32 statement bit for bit (NaN included)."""
    B, L, H, W, _ = depth.shape
    got = gs.bilateral_filter_depth(depth.to(DEV), f).cpu()
    want, _ = bo.bilateral_f32(depth.numpy().reshape(B * L, H, W), f.radius, f.sigma_space, f.sigma_range)
    assert got.shape == depth.shape
    assert np.array_equal(_bits(got.numpy()).ravel(), _bits(want).ravel())
    return got


def _with_bad_pixels(depth, seed):
    g = torch.Generator().manual_seed(seed)
    d = depth.clone()
    u = torch.rand(d.shape, generator=g)
    d[u < 0.03] = 0.0
    d[(u >= 0.03) & (u < 0.04)] = float("nan")
    d[(u >= 0.04) & (u < 0.05)] = float("inf")
    d[(u >= 0.05) & (u < 0.06)] = -1.0
    return d


@pytest.mark.parametrize("radius", range(1, 8))
def test_forward_matches_oracle_bit_for_bit_at_every_radius(radius):
    _, depth, _, _ = make_sequence(2, 2, 37, 45, seed=radius, yaw0=0.6)  # H, W not multiples of the 32 x 8 tile
    noisy = _with_bad_pixels(add_depth_noise(depth, seed=radius), radius)
    f = gs.BilateralFilter(radius, 0.7 * radius, 0.04)
    _assert_forward_exact(noisy, f)


# images smaller than the 32 x 8 tile, one-pixel and two-pixel wide, a tile and one row or column
SMALL_AND_ODD = [(1, 1, 1, 1, 3), (2, 3, 5, 7, 7), (1, 2, 3, 40, 4), (3, 1, 33, 2, 2), (1, 1, 9, 33, 1)]


@pytest.mark.parametrize("B,L,H,W,radius", SMALL_AND_ODD)
def test_forward_on_small_and_odd_images(B, L, H, W, radius):
    g = torch.Generator().manual_seed(H * 100 + W)
    depth = 2.0 + 0.05 * torch.randn((B, L, H, W, 1), generator=g)  # a different image per element
    _assert_forward_exact(_with_bad_pixels(depth, W), gs.BilateralFilter(radius, 1.5, 0.05))


def test_forward_at_full_size():
    _, depth, _, _ = make_sequence(8, 2, 480, 640, seed=4, yaw0=0.6)
    _assert_forward_exact(add_depth_noise(depth, seed=4), gs.BilateralFilter(3, 2.0, 0.05))


def test_forward_past_one_grid_dimension_of_images():
    n = 70_000  # > 65 535 images in one launch
    g = torch.Generator().manual_seed(9)
    depth = (1.0 + torch.rand((n, 1, 2, 3, 1), generator=g)) * (torch.rand((n, 1, 2, 3, 1), generator=g) > 0.1)
    _assert_forward_exact(depth, gs.BilateralFilter(1, 1.0, 0.1))


def test_channels_first_layout_and_rgbdimages():
    rgb, depth, K, poses = make_sequence(2, 2, 24, 32, seed=5)
    f = gs.BilateralFilter(2, 1.5, 0.03)
    want = gs.bilateral_filter_depth(depth.to(DEV), f)
    cf = gs.bilateral_filter_depth(depth.permute(0, 1, 4, 2, 3).contiguous().to(DEV), f)
    assert cf.shape == (2, 2, 1, 24, 32) and torch.equal(cf.permute(0, 1, 3, 4, 2), want)
    fr = gs.RGBDImages(rgb.to(DEV), depth.to(DEV), K.to(DEV), poses.to(DEV))
    ff = fr.bilateral_filtered(f)
    assert torch.equal(ff.depth_image, want)
    assert ff.rgb_image is fr.rgb_image and ff.intrinsics is fr.intrinsics and ff.poses is fr.poses
    frc = fr.to_channels_first()
    ffc = frc.bilateral_filtered(f)
    assert ffc.channels_first and torch.equal(ffc.depth_image.permute(0, 1, 3, 4, 2), want)


# ------------------------------------------------------------------------------------------------------------ backward
def _gpu_backward(depth, f, g_out):
    """d(sum(g_out * filtered))/d(depth) on the GPU, twice: the two calls agree bit for bit.  depth, g_out (B,L,H,W,1)
    CPU float32; returns the gradient as an (n, H, W) CPU tensor."""
    B, L, H, W, _ = depth.shape
    grads = []
    for _ in range(2):
        d = depth.to(DEV).requires_grad_(True)
        gs.bilateral_filter_depth(d, f).backward(g_out.to(DEV))
        grads.append(d.grad.cpu())
    assert torch.equal(grads[0].view(torch.int32), grads[1].view(torch.int32))
    return grads[0].view(B * L, H, W)


def _assert_backward_close_to_autograd(depth, f, g_out):
    B, L, H, W, _ = depth.shape
    got = _gpu_backward(depth, f, g_out)
    d2 = depth.numpy().reshape(B * L, H, W)
    x = torch.from_numpy(d2.astype(np.float64)).requires_grad_(True)
    keep = bo.keep_masks(d2, f.radius, f.sigma_space, f.sigma_range)
    want, = torch.autograd.grad(bo.bilateral_f64(x, f.radius, f.sigma_space, f.sigma_range, keep)[0], x,
                                g_out.double().view(B * L, H, W))
    _, mag = bo.bilateral_bwd_formula(d2, g_out.numpy().reshape(B * L, H, W), f.radius, f.sigma_space, f.sigma_range)
    err = np.abs(got.double().numpy() - want.numpy())
    assert np.all(err <= 1e-4 * mag + 1e-30), float((err / mag).max())


def _assert_backward_close_to_formula(depth, f, g_out):
    """Against bilateral_bwd_formula (float64 numpy) where autograd of bilateral_f64 would not fit in memory."""
    B, L, H, W, _ = depth.shape
    got = _gpu_backward(depth, f, g_out)
    want, mag = bo.bilateral_bwd_formula(depth.numpy().reshape(B * L, H, W), g_out.numpy().reshape(B * L, H, W),
                                         f.radius, f.sigma_space, f.sigma_range)
    err = np.abs(got.double().numpy() - want)
    assert np.all(err <= 1e-4 * mag + 1e-30), float((err / mag).max())


@pytest.mark.parametrize("radius,H,W", [(1, 9, 11), (2, 23, 35), (3, 37, 45), (4, 17, 66), (5, 30, 33), (6, 20, 70),
                                        (7, 41, 39)])
def test_backward_matches_float64_autograd_and_is_deterministic(radius, H, W):
    """Every instantiation of k_depth_bilateral_bwd<R>, on images that are not a whole number of tiles."""
    _, depth, _, _ = make_sequence(2, 1, H, W, seed=radius, yaw0=0.6)
    depth = _with_bad_pixels(add_depth_noise(depth, seed=radius), radius + 1)
    f = gs.BilateralFilter(radius, 0.8 * radius, 0.05)
    g_out = torch.randn(depth.shape, generator=torch.Generator().manual_seed(2))
    _assert_backward_close_to_autograd(depth, f, g_out)


@pytest.mark.parametrize("B,L,H,W,radius", SMALL_AND_ODD)
def test_backward_on_small_and_odd_images(B, L, H, W, radius):
    g = torch.Generator().manual_seed(H * 100 + W + 1)
    depth = 2.0 + 0.05 * torch.randn((B, L, H, W, 1), generator=g)
    g_out = torch.randn(depth.shape, generator=g)
    _assert_backward_close_to_autograd(_with_bad_pixels(depth, W), gs.BilateralFilter(radius, 1.5, 0.05), g_out)


def test_backward_past_one_grid_dimension_of_images():
    """70 000 images > 65 535: the images past gridDim.z come from the kernel's image-stride loop."""
    n = 70_000
    g = torch.Generator().manual_seed(10)
    depth = (1.0 + 0.05 * torch.rand((n, 1, 2, 3, 1), generator=g)) * (torch.rand((n, 1, 2, 3, 1), generator=g) > 0.1)
    g_out = torch.randn(depth.shape, generator=g)
    _assert_backward_close_to_formula(depth, gs.BilateralFilter(1, 1.0, 0.1), g_out)


def test_backward_at_full_size():
    _, depth, _, _ = make_sequence(8, 2, 480, 640, seed=4, yaw0=0.6)
    depth = _with_bad_pixels(add_depth_noise(depth, seed=4), 5)
    g_out = torch.randn(depth.shape, generator=torch.Generator().manual_seed(3))
    _assert_backward_close_to_formula(depth, gs.BilateralFilter(3, 2.0, 0.05), g_out)


def test_no_grad_call_keeps_no_weight_sums():
    d = torch.full((1, 1, 8, 8, 1), 2.0, device=DEV)
    out = gs.bilateral_filter_depth(d, gs.BilateralFilter(2, 1.0, 0.1))
    assert out.grad_fn is None


# ------------------------------------------------------------------------------------------------------------ drivers
def _assert_same_maps(a, b):
    assert a.num_points_per_pointcloud.tolist() == b.num_points_per_pointcloud.tolist()
    for attr in ("points_list", "normals_list", "colors_list", "features_list"):
        for x, y in zip(getattr(a, attr), getattr(b, attr)):
            assert torch.equal(x, y), attr


def _frames(rgb, depth, K, poses):
    return gs.RGBDImages(rgb.to(DEV), depth.to(DEV), K.to(DEV), poses.to(DEV))


F = gs.BilateralFilter(3, 2.0, 0.05)
PRUNE = dict(stable_confidence=1.0, max_unstable_age=2, free_space_margin=0.05, surfel_radii=True,
             merge_overlapping=True)


@pytest.mark.parametrize("opts", [{}, PRUNE], ids=["plain", "prune_radii_merge"])
@pytest.mark.parametrize("source", ["device", "pinned", "raw"])
def test_sequence_call_equals_fusing_the_filtered_frames(source, opts):
    from gradslam_b200 import ingest

    B, L, H, W = 2, 6, 48, 64
    rgb, depth, K, poses = make_sequence(B, L, H, W, seed=7, yaw0=0.6)
    depth = add_depth_noise(depth, seed=7)
    if source == "raw":
        col = (rgb.numpy() * 255.0).astype(np.uint8)
        dep = np.round(depth.numpy()[..., 0] * 5000.0).astype(np.uint16)
        frames = ingest.RawRGBD(torch.from_numpy(col).pin_memory(), torch.from_numpy(dep).pin_memory(), K, poses)
        rgb, depth = ingest.raw_to_float(torch.from_numpy(col).to(DEV), torch.from_numpy(dep).to(DEV), 5000.0, False)
        rgb, depth = rgb.cpu(), depth.cpu()
    elif source == "pinned":
        frames = gs.RGBDImages(rgb.pin_memory(), depth.pin_memory(), K, poses)
    else:
        frames = _frames(rgb, depth, K, poses)
    pc, p = gs.PointFusion(odom="gt", device=DEV, depth_filter=F, **opts)(frames)
    ref = _frames(rgb, gs.bilateral_filter_depth(depth.to(DEV), F).cpu(), K, poses)
    pc_ref, p_ref = gs.PointFusion(odom="gt", device=DEV, **opts)(ref)
    _assert_same_maps(pc, pc_ref)
    assert torch.equal(p, p_ref)
    # the filter changed the map
    pc_raw, _ = gs.PointFusion(odom="gt", device=DEV, **opts)(_frames(rgb, depth, K, poses))
    assert pc_raw.num_points_per_pointcloud.tolist() != pc.num_points_per_pointcloud.tolist()


def _step_loop(slam, frames):
    pc = gs.Pointclouds(device=DEV)
    for s in range(frames.shape[1]):
        pc, _ = slam.step(pc, frames[:, s], None, inplace=True)
    return pc


def test_step_loop_equals_fusing_the_filtered_frames():
    rgb, depth, K, poses = make_sequence(2, 4, 48, 64, seed=8, yaw0=0.6)
    depth = add_depth_noise(depth, seed=8)
    pc = _step_loop(gs.PointFusion(odom="gt", device=DEV, depth_filter=F, **PRUNE), _frames(rgb, depth, K, poses))
    ref = _frames(rgb, gs.bilateral_filter_depth(depth.to(DEV), F).cpu(), K, poses)
    _assert_same_maps(pc, _step_loop(gs.PointFusion(odom="gt", device=DEV, **PRUNE), ref))


def test_tracking_only_with_ground_truth_poses_filters_nothing():
    rgb, depth, K, poses = make_sequence(2, 4, 48, 64, seed=9, yaw0=0.6)
    depth = add_depth_noise(depth, seed=9)
    fr = _frames(rgb, depth, K, poses)
    pc, p = gs.PointFusion(odom="gt", device=DEV, depth_filter=F, depth_filter_tracking_only=True)(fr)
    pc_ref, p_ref = gs.PointFusion(odom="gt", device=DEV)(fr)
    _assert_same_maps(pc, pc_ref)
    assert torch.equal(p, p_ref)
    pc = _step_loop(gs.PointFusion(odom="gt", device=DEV, depth_filter=F, depth_filter_tracking_only=True), fr)
    _assert_same_maps(pc, _step_loop(gs.PointFusion(odom="gt", device=DEV), fr))


@pytest.mark.parametrize("association", ["nn", "projective"])
@pytest.mark.parametrize("odom", ["icp", "gradicp"])
def test_tracking_only_tracks_the_filtered_frame_and_fuses_the_raw_one(odom, association):
    rgb, depth, K, poses = make_sequence(2, 3, 48, 64, seed=10, yaw0=0.6)
    depth = add_depth_noise(depth, seed=10)
    fr = _frames(rgb, depth, K, poses)
    kw = dict(odom=odom, association=association, numiters=5, device=DEV)
    pc, p = gs.PointFusion(depth_filter=F, depth_filter_tracking_only=True, **kw)(fr)
    # by hand: localise the filtered frame, fuse the raw one
    slam = gs.PointFusion(**kw)
    pc_ref, prev, want = gs.Pointclouds(device=DEV), None, []
    for s in range(fr.shape[1]):
        live = fr[:, s]
        track = live if prev is None else live.bilateral_filtered(F)
        live.poses = slam._localize(pc_ref, track, prev)
        pc_ref = slam._map(pc_ref, live, True)
        prev = live
        want.append(live.poses[:, 0])
    assert torch.equal(p, torch.stack(want, 1))
    _assert_same_maps(pc, pc_ref)
    # and it is not the unfiltered run
    _, p_raw = gs.PointFusion(**kw)(fr)
    assert not torch.equal(p, p_raw)


@pytest.mark.parametrize("odom", ["gt", "gradicp"])
def test_differentiable_mode_puts_the_filter_on_the_tape(odom):
    B, L, H, W = 2, 3, 24, 32
    rgb, depth, K, poses = make_sequence(B, L, H, W, seed=11, yaw0=0.6)
    depth = add_depth_noise(depth, seed=11)
    kw = dict(odom=odom, numiters=3, device=DEV)
    if odom == "gt":
        with torch.no_grad():
            pc_fused, p_fused = gs.PointFusion(depth_filter=F, **kw)(_frames(rgb, depth, K, poses))

    def loss(pc, p):
        g = torch.Generator().manual_seed(1)
        terms = [(t * torch.randn(t.shape, generator=g).to(DEV)).sum()
                 for b in range(B) for t in (pc.points_list[b], pc.normals_list[b], pc.features_list[b])]
        return sum(terms) + (p * torch.randn(p.shape, generator=g).to(DEV)).sum()

    d = depth.to(DEV).requires_grad_(True)
    pc, p = gs.PointFusion(depth_filter=F, **kw)(gs.RGBDImages(rgb.to(DEV), d, K.to(DEV), poses.to(DEV)))
    if odom == "gt":  # the taped step loop and the whole-sequence call fuse the same maps
        _assert_same_maps(pc, pc_fused)
        assert torch.equal(p, p_fused)
    loss(pc, p).backward()
    # the hand-composed chain: the driver's gradient w.r.t. a filtered leaf, pushed through the filter's backward
    d_raw = depth.to(DEV).requires_grad_(True)
    filtered = gs.bilateral_filter_depth(d_raw, F)
    leaf = filtered.detach().requires_grad_(True)
    pc2, p2 = gs.PointFusion(**kw)(gs.RGBDImages(rgb.to(DEV), leaf, K.to(DEV), poses.to(DEV)))
    loss(pc2, p2).backward()
    want, = torch.autograd.grad(filtered, d_raw, leaf.grad)
    assert torch.equal(d.grad, want)
    assert bool(d.grad.abs().sum() > 0)


# ------------------------------------------------------------------------------------------------- effect on noisy input
def _dot(a, b):  # in one fixed order on the CPU, so GPU and oracle normals give the same decisions
    return (a[..., 0] * b[..., 0] + a[..., 1] * b[..., 1]) + a[..., 2] * b[..., 2]


def test_filter_on_noisy_input_matches_oracle_and_helps():
    """Oracle figures (CPU, float32 statement then the fusion oracle) for this scene: 7916 / 7881 fused rows and 64.6 %
    of live normals within 20 degrees of the clean ones on raw noisy depth; 6637 / 6531 rows and 79.7 % filtered."""
    import gsx_oracle as oracle

    B, L, H, W = 2, 4, 48, 64
    rgb, depth, K, poses = make_sequence(B, L, H, W, seed=3, yaw0=0.6)
    noisy = add_depth_noise(depth, seed=11)
    f = gs.BilateralFilter(3, 2.0, 0.05)
    dot_th = math.cos(20 * math.pi / 180)
    clean = gs.RGBDImages(rgb.to(DEV), depth.to(DEV), K.to(DEV)).normal_map.cpu()
    clean_ref = oracle.frame_maps(depth, K)["normal"]
    res = {}
    for name, filt in (("raw", None), ("filtered", f)):
        pc, _ = gs.PointFusion(odom="gt", device=DEV, depth_filter=filt)(_frames(rgb, noisy, K, poses))
        fr = gs.RGBDImages(rgb.to(DEV), noisy.to(DEV), K.to(DEV))
        live = fr.normal_map if filt is None else fr.bilateral_filtered(filt).normal_map
        valid = (depth[..., 0] > 0) & (noisy[..., 0] > 0)
        share = float((_dot(live.cpu(), clean)[valid] > dot_th).double().mean())
        d_ref = noisy if filt is None else torch.from_numpy(
            bo.bilateral_f32(noisy.numpy().reshape(-1, H, W), 3, 2.0, 0.05)[0].reshape(noisy.shape))
        ref = oracle.run_slam(rgb, d_ref, K, poses, odom="gt")
        share_ref = float((_dot(oracle.frame_maps(d_ref, K)["normal"], clean_ref)[valid] > dot_th).double().mean())
        assert pc.num_points_per_pointcloud.tolist() == ref.map.counts()
        assert share == share_ref
        res[name] = (sum(ref.map.counts()), share)
    assert res["filtered"][0] < res["raw"][0] and res["filtered"][1] > res["raw"][1]
