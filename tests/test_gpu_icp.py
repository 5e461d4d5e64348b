"""GPU parity for the ICP path (K5 exact 1-NN, K6 normal equations, K7 solve / se3_exp / LM-gradLM update) against
the CPU oracle.  Index work (nn association) is bit-exact; poses are compared at north_star's 1e-4."""
import math

import pytest
import torch

import gsx_oracle as oracle
from cameras import camera_inputs
from gradslam_b200.synthetic import make_sequence

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _cloud(seed, H=48, W=64):
    rgb, depth, K, poses = make_sequence(1, 1, H, W, seed=seed, hole_fraction=0.0)
    m = oracle.frame_maps(depth, K, poses)
    return m["gvertex"][0, 0].reshape(-1, 3).contiguous(), m["gnormal"][0, 0].reshape(-1, 3).contiguous()


def test_knn1_bit_exact_with_ties():
    from gradslam_b200.odometry import icputils

    g = torch.Generator().manual_seed(0)
    src = torch.rand(1, 3000, 3, generator=g)
    tgt = torch.rand(1, 2500, 3, generator=g)
    tgt[0, 1200:1300] = tgt[0, 100:200]  # exact duplicates: the lower index must win
    src[0, :50] = tgt[0, 1200:1250]
    d2, idx = icputils.knn1(src.to(DEV), tgt.to(DEV))
    rd2, ridx = oracle.knn1(src[0], tgt[0])
    assert torch.equal(idx[0].cpu(), ridx)
    assert torch.equal(d2[0].cpu(), rd2)
    assert (idx[0, :50].cpu() == torch.arange(100, 150)).all()


def test_gauss_newton_rows_match_oracle():
    from gradslam_b200.odometry import icputils

    tgt, tgt_n = _cloud(5)
    T = oracle.se3_exp(torch.tensor([0.02, -0.01, 0.015, 0.03, -0.02, 0.01]))
    src = oracle.rigid_apply(T, tgt)
    for th in (None, 0.002):
        A, b, idx = icputils.gauss_newton_solve(src[None].to(DEV), tgt[None].to(DEV), tgt_n[None].to(DEV), th)
        rA, rb, ridx = oracle.gauss_newton_solve(src, tgt, tgt_n, th)
        assert torch.equal(idx.cpu(), ridx)
        torch.testing.assert_close(A.cpu(), rA, rtol=1e-6, atol=1e-7)
        torch.testing.assert_close(b.cpu(), rb, rtol=1e-5, atol=1e-7)


@pytest.mark.parametrize("mode", ["icp", "gradicp"])
@pytest.mark.parametrize("dist_thresh", [None, 0.01])
def test_icp_functions_match_oracle(mode, dist_thresh):
    from gradslam_b200.odometry import icputils

    tgt, tgt_n = _cloud(5)
    T_true = oracle.se3_exp(torch.tensor([0.02, -0.01, 0.015, 0.03, -0.02, 0.01]))
    src = oracle.rigid_apply(T_true, tgt)
    T0 = torch.eye(4)
    if mode == "icp":
        T, idx = icputils.point_to_plane_ICP(src[None].to(DEV), tgt[None].to(DEV), tgt_n[None].to(DEV), T0.to(DEV),
                                             numiters=12, dist_thresh=dist_thresh)
        rT, ridx = oracle.point_to_plane_icp(src, tgt, tgt_n, T0, numiters=12, dist_thresh=dist_thresh)
    else:
        T, idx = icputils.point_to_plane_gradICP(src[None].to(DEV), tgt[None].to(DEV), tgt_n[None].to(DEV),
                                                 T0.to(DEV), numiters=12, dist_thresh=dist_thresh)
        rT, ridx = oracle.point_to_plane_gradicp(src, tgt, tgt_n, T0, numiters=12, dist_thresh=dist_thresh)
    # north_star tolerance on poses: 1e-4
    torch.testing.assert_close(T.cpu(), rT, rtol=0, atol=1e-4)
    assert T.cpu()[3].tolist() == [0, 0, 0, 1]
    # the last association agrees except where the 1e-6-level pose difference moves a point across a tie
    assert idx.shape == ridx.shape and (idx.cpu() == ridx).float().mean() > 0.99


def test_long_gradicp_run_tracks_oracle():
    """40 gradLM iterations (the reference's tests use 30-100): the pose stays within 1e-4 of the oracle's and the
    alignment error does not grow."""
    from gradslam_b200.odometry import icputils

    tgt, tgt_n = _cloud(6, 60, 80)
    T_true = oracle.se3_exp(torch.tensor([0.01, 0.006, -0.004, 0.01, -0.008, 0.006]))
    src = oracle.rigid_apply(T_true, tgt)
    T, _ = icputils.point_to_plane_gradICP(src[None].to(DEV), tgt[None].to(DEV), tgt_n[None].to(DEV),
                                           torch.eye(4, device=DEV), numiters=40)
    rT, _ = oracle.point_to_plane_gradicp(src, tgt, tgt_n, torch.eye(4), numiters=40)
    torch.testing.assert_close(T.cpu(), rT, rtol=0, atol=1e-4)
    err0 = (T_true - torch.eye(4)).abs().max().item()
    assert (T.cpu() @ T_true - torch.eye(4)).abs().max().item() <= err0 + 1e-5


@pytest.mark.parametrize("mode", [0, 1])
def test_icp_align_takes_non_dense_clouds(mode):
    """Clouds that are every other row of larger tensors (each copied to a dense temporary for the call) give the
    transform and association of the dense clouds, bit for bit."""
    from gradslam_b200.odometry import icputils

    tgt, tgt_n = _cloud(5)
    src = oracle.rigid_apply(oracle.se3_exp(torch.tensor([0.02, -0.01, 0.015, 0.03, -0.02, 0.01])), tgt)
    g = torch.Generator().manual_seed(3)
    dense, strided = [], []
    for t in (src, tgt, tgt_n):
        big = torch.randn(1, 2 * t.shape[0], 3, generator=g)  # the rows in between are noise
        big[0, ::2] = t
        dense.append(t[None].to(DEV))
        strided.append(big.to(DEV)[:, ::2])
        assert not strided[-1].is_contiguous()
    cs, ct = icputils._counts(src.shape[0], 1, DEV), icputils._counts(tgt.shape[0], 1, DEV)
    T, idx = icputils.icp_align(dense[0], cs, dense[1], dense[2], ct, None, mode, 10, 1e-8, None, want_idx=True)
    T_s, idx_s = icputils.icp_align(strided[0], cs, strided[1], strided[2], ct, None, mode, 10, 1e-8, None,
                                    want_idx=True)
    assert torch.equal(T_s, T)
    assert torch.equal(idx_s, idx)


def test_providers_ragged_batch_match_oracle():
    import gradslam_b200 as gs

    clouds = [_cloud(7, 40, 56), _cloud(8, 48, 64)]
    Ts = [oracle.se3_exp(torch.tensor(v)) for v in ([0.02, 0.0, 0.01, 0.02, 0.01, -0.01], [-0.01, 0.02, 0.0, -0.02, 0.0, 0.02])]
    srcs = [oracle.rigid_apply(T, c[0])[:-37 * i or None] for i, (T, c) in enumerate(zip(Ts, clouds))]  # ragged
    maps_pc = gs.Pointclouds([c[0].to(DEV) for c in clouds], [c[1].to(DEV) for c in clouds])
    frames_pc = gs.Pointclouds([s.to(DEV) for s in srcs])
    for prov, fn in ((gs.odometry.ICPOdometryProvider(numiters=8), oracle.point_to_plane_icp),
                     (gs.odometry.GradICPOdometryProvider(numiters=8), oracle.point_to_plane_gradicp)):
        T = prov.provide(maps_pc, frames_pc)
        assert T.shape == (2, 1, 4, 4)
        for b in range(2):
            rT, _ = fn(srcs[b], clouds[b][0], clouds[b][1], torch.eye(4), numiters=8)
            torch.testing.assert_close(T[b, 0].cpu(), rT, rtol=0, atol=1e-4)
    with pytest.raises(TypeError):
        gs.odometry.ICPOdometryProvider().provide(3, frames_pc)
    with pytest.raises(ValueError):
        gs.odometry.ICPOdometryProvider().provide(gs.Pointclouds([c[0].to(DEV) for c in clouds]), frames_pc)


def _nn_dist(a, b):
    return oracle.knn1(a, b)[0].sqrt()


ICP_CASES = [("PointFusion", "gradicp", False), ("PointFusion", "icp", False), ("ICPSLAM", "gradicp", False),
             ("PointFusion", "gradicp", True), ("PointFusion", "icp", True), ("ICPSLAM", "icp", True)]


@pytest.mark.parametrize("cls,odom,cameras", ICP_CASES,
                         ids=["%s-%s%s" % (c, o, "-cameras" if cam else "") for c, o, cam in ICP_CASES])
def test_slam_with_icp_odometry_matches_oracle(cls, odom, cameras):
    """cameras: B=3, a camera per element (tests/golden/cameras.py) with skew and 4th intrinsics column."""
    import gradslam_b200 as gs

    if cameras:
        B, L, H, W = 3, 3, 48, 64
        rgb, depth, K, poses = camera_inputs(B, L, H, W, 2, skew=0.75)
    else:
        B, L, H, W = 2, 3, 64, 64
        rgb, depth, K, poses = make_sequence(B, L, H, W, seed=2)
    slam = getattr(gs, cls)(odom=odom, numiters=10, device=DEV)
    frames = gs.RGBDImages(rgb.to(DEV), depth.to(DEV), K.to(DEV), poses.to(DEV))
    pc, rec = slam(frames)
    ref = oracle.run_slam(rgb, depth, K, poses, mode="pointfusion" if cls == "PointFusion" else "aggregate", odom=odom,
                          numiters=10)
    # north_star: 1e-4 on poses, 1e-3 on fused point coordinates
    torch.testing.assert_close(rec.cpu(), ref.poses, rtol=0, atol=1e-4)
    got = pc.num_points_per_pointcloud.tolist()
    for b in range(B):
        # a pose difference of ~1e-6 can flip a borderline match, so sizes may differ by a handful of points
        assert abs(got[b] - ref.map.counts()[b]) <= max(3, ref.map.counts()[b] // 500), (got, ref.map.counts())
        mine = pc.points_list[b].cpu()
        if got[b] == ref.map.counts()[b]:
            torch.testing.assert_close(mine, ref.map.points[b], rtol=0, atol=1e-3)
        else:  # set comparison: every point has a counterpart within 1e-3
            assert _nn_dist(mine, ref.map.points[b]).quantile(0.999) < 1e-3
            assert _nn_dist(ref.map.points[b], mine).quantile(0.999) < 1e-3


@pytest.mark.parametrize("nt", [5000, 60000])
def test_knn1_grid_path_is_exact(nt):
    """Targets larger than 4096 points go through the uniform-grid search: identical (distance, index) to the
    brute-force oracle, including duplicated targets, far-away queries (full-scan fallback) and queries outside the
    target bounding box."""
    from gradslam_b200.odometry import icputils

    g = torch.Generator().manual_seed(1)
    # targets on three planes of a box (surface-like), plus duplicates
    a = torch.rand(nt, 3, generator=g)
    face = torch.randint(0, 3, (nt,), generator=g)
    a[torch.arange(nt), face] = 0.0
    tgt = a * torch.tensor([4.0, 3.0, 6.0])
    tgt[nt // 2: nt // 2 + 200] = tgt[:200]
    src = tgt[torch.randint(0, nt, (3000,), generator=g)] + 0.01 * torch.randn(3000, 3, generator=g)
    src[:100] = tgt[nt // 2: nt // 2 + 100]                      # exact hits on duplicated points -> lower index
    src[100:150] += 50.0                                          # far outside the grid
    src[150:200] = torch.rand(50, 3, generator=g) * torch.tensor([4.0, 3.0, 6.0]) + 1.0  # inside the box, off-surface
    d2, idx = icputils.knn1(src[None].to(DEV), tgt[None].to(DEV))
    rd2, ridx = oracle.knn1(src, tgt)
    assert torch.equal(idx[0].cpu(), ridx)
    assert torch.equal(d2[0].cpu(), rd2)
    assert (idx[0, :100].cpu() == torch.arange(100)).all()


def test_slam_with_dense_icp_uses_grid_and_matches_oracle():
    """dsratio=1 makes the ICP clouds larger than 4096 points, so the localisation runs on the grid search."""
    import gradslam_b200 as gs

    B, L, H, W = 1, 3, 64, 80
    rgb, depth, K, poses = make_sequence(B, L, H, W, seed=13)
    slam = gs.PointFusion(odom="gradicp", numiters=6, dsratio=1, device=DEV)
    pc, rec = slam(gs.RGBDImages(rgb.to(DEV), depth.to(DEV), K.to(DEV), poses.to(DEV)))
    ref = oracle.run_slam(rgb, depth, K, poses, odom="gradicp", numiters=6, dsratio=1)
    torch.testing.assert_close(rec.cpu(), ref.poses, rtol=0, atol=1e-4)
    assert abs(pc.num_points_per_pointcloud.tolist()[0] - ref.map.counts()[0]) <= 12
