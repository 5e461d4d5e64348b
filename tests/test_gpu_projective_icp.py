"""GPU parity of the projective ICP odometry (gsx_icp_localize_projective, gsx_icp_project_associate,
ICPSLAM / PointFusion(association='projective')) against the CPU oracle of tests/projective_oracle.py: the association
bit for bit, poses at the ICP tests' 1e-4, maps at 1e-3, gradients at the tolerances of test_gpu_backward.py."""
import pytest
import torch

import gsx_oracle as oracle
import projective_oracle as po
from cameras import camera_inputs
from gradslam_b200.synthetic import make_sequence, punch_lattice_holes

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _frames(rgb, depth, K, poses):
    import gradslam_b200 as gs

    return gs.RGBDImages(rgb.to(DEV), depth.to(DEV), K.to(DEV), poses.to(DEV))


def _fused_map(frames):
    import gradslam_b200 as gs

    pc, _ = gs.PointFusion(odom="gt", device=DEV)(frames)
    return pc


def _oracle_map(pc, elems=None):
    elems = range(len(pc)) if elems is None else elems
    return oracle.SurfelMap([pc.points_list[b].cpu() for b in elems], [pc.normals_list[b].cpu() for b in elems])


def _icp_kwargs(odom, numiters, dist_thresh):
    kw = dict(numiters=numiters, damp=1e-8, dist_thresh=dist_thresh)
    if odom == "gradicp":
        kw.update(lambda_max=2.0, B=1.0, B2=1.0, nu=200.0)
    return kw


@pytest.mark.parametrize("dist_thresh", [None, 0.0004])
def test_project_associate_bit_exact_on_corner_cases(dist_thresh):
    """Half-pixel ties, rows and points on the frustum bounds, z ties, uncovered pixels, an empty map, a camera per
    element with skew and a 4th intrinsics column (projective_oracle.small_case)."""
    from gradslam_b200.odometry.icputils import project_associate

    H, W = 6, 8
    smap, _, src, pose, K = po.small_case(H, W)
    idx, tgt_p, _ = po.target_images(smap, pose, K, H, W)
    want_d2, want_j = po.associate(src, pose, K, H, W, idx, tgt_p, dist_thresh)
    counts = torch.full((3,), src.shape[1], dtype=torch.int32, device=DEV)
    d2, j = project_associate(src.to(DEV), counts, tgt_p.to(DEV), idx.to(DEV), pose.to(DEV), K.to(DEV), H, W,
                              dist_thresh)
    assert torch.equal(j.cpu(), want_j)
    assert torch.equal(d2.cpu(), want_d2)
    assert (want_j[0] >= 0).any() and (want_j[1] >= 0).any()


@pytest.mark.parametrize("dist_thresh", [None, 0.001])
def test_project_associate_bit_exact_on_fused_maps_with_cameras(dist_thresh):
    """Maps fused from camera_inputs (a camera per element, skew, 4th column); the index image of the render equals the
    oracle's, and the association of the next frame's lattice points equals the oracle's bit for bit."""
    import gradslam_b200 as gs
    from gradslam_b200.odometry.icputils import project_associate

    B, L, H, W = 3, 3, 45, 62
    rgb, depth, K, poses = camera_inputs(B, L, H, W, 62, skew=0.75)
    pc = _fused_map(_frames(rgb, depth, K, poses)[:, :2])
    smap = _oracle_map(pc)
    idx, tgt_p, _ = po.target_images(smap, poses[:, 1], K[:, 0], H, W)
    rendered = gs.render_pointclouds(pc, K.to(DEV), poses[:, 1:2].to(DEV), H, W)
    assert torch.equal(rendered.index.view(B, H * W).cpu(), idx)
    pts, _ = oracle.downsample_frame(oracle.frame_maps(depth[:, 2:3], K, poses[:, 1:2]), 2)
    ns = max(p.shape[0] for p in pts)
    src = torch.zeros(B, ns, 3)
    for b, p in enumerate(pts):
        src[b, : p.shape[0]] = p
    counts = torch.tensor([p.shape[0] for p in pts], dtype=torch.int32, device=DEV)
    want_d2, want_j = po.associate(src, poses[:, 1], K[:, 0], H, W, idx, tgt_p, dist_thresh)
    d2, j = project_associate(src.to(DEV), counts, tgt_p.to(DEV), idx.to(DEV), poses[:, 1].to(DEV), K[:, 0].to(DEV),
                              H, W, dist_thresh)
    for b, p in enumerate(pts):
        n = p.shape[0]
        assert torch.equal(j[b, :n].cpu(), want_j[b, :n])
        assert torch.equal(d2[b, :n].cpu(), want_d2[b, :n])
        assert (j[b, n:] == -1).all()
        if dist_thresh is None:
            assert (want_j[b, :n] >= 0).sum() > n // 2
    if dist_thresh is not None:  # the threshold rejects some covered pairs
        assert ((want_j < 0) & torch.isfinite(want_d2)).any()


@pytest.mark.parametrize("ds", [1, 2, 4])
@pytest.mark.parametrize("dist_thresh", [None, 0.01])
@pytest.mark.parametrize("odom", ["icp", "gradicp"])
def test_localize_projective_matches_oracle_and_taped_path(odom, dist_thresh, ds):
    """The fused call against the oracle (H*W = 2790, not a multiple of 256; W % 4 = 2; a camera per element), and the
    differentiable mode (live depth requiring grad) against the fused call, bit for bit."""
    import gradslam_b200 as gs

    B, L, H, W = 3, 3, 45, 62
    rgb, depth, K, poses = camera_inputs(B, L, H, W, 61, skew=0.75)
    frames = _frames(rgb, depth, K, poses)
    pc = _fused_map(frames[:, :2])
    slam = gs.PointFusion(odom=odom, association="projective", numiters=10, dsratio=ds, dist_thresh=dist_thresh,
                          device=DEV)
    got = slam._localize(pc, frames[:, 2], frames[:, 1])
    at_prev = oracle.frame_maps(depth[:, 2:3], K, poses[:, 1:2])
    want = po.odometry_projective(_oracle_map(pc), at_prev, poses[:, 1], K[:, 0], H, W, odom, ds,
                                  _icp_kwargs(odom, 10, dist_thresh))
    torch.testing.assert_close(got[:, 0].cpu(), want, rtol=0, atol=1e-4)
    assert not torch.equal(got[:, 0].cpu(), poses[:, 1])  # it moved
    d_req = depth[:, 2:3].to(DEV).requires_grad_(True)
    live = gs.RGBDImages(rgb[:, 2:3].to(DEV), d_req, K.to(DEV), poses[:, 2:3].to(DEV))
    taped = slam._localize(pc, live, frames[:, 1])
    assert taped.requires_grad
    assert torch.equal(taped.detach(), got)


SLAM_CASES = [("PointFusion", "icp"), ("PointFusion", "gradicp"), ("ICPSLAM", "gradicp")]


@pytest.mark.parametrize("cls,odom", SLAM_CASES, ids=["%s-%s" % c for c in SLAM_CASES])
def test_slam_with_projective_odometry_matches_oracle(cls, odom):
    import gradslam_b200 as gs

    B, L, H, W = 3, 4, 48, 64
    rgb, depth, K, poses = camera_inputs(B, L, H, W, 63, skew=0.75)
    slam = getattr(gs, cls)(odom=odom, association="projective", numiters=10, dsratio=2, device=DEV)
    pc, rec = slam(_frames(rgb, depth, K, poses))
    ref = po.run_slam(rgb, depth, K, poses, mode="pointfusion" if cls == "PointFusion" else "aggregate", odom=odom,
                      numiters=10, dsratio=2)
    torch.testing.assert_close(rec.cpu(), ref.poses, rtol=0, atol=1e-4)
    assert pc.num_points_per_pointcloud.tolist() == ref.map.counts()
    for b in range(B):
        torch.testing.assert_close(pc.points_list[b].cpu(), ref.map.points[b], rtol=0, atol=1e-3)


@pytest.mark.parametrize("odom", ["icp", "gradicp"])
def test_empty_map_no_depth_and_camera_turned_away_keep_the_previous_pose(odom):
    """Element 1 has an empty map, element 2 a live frame without valid depth, element 3's previous camera is turned
    half a circle so the map lies behind it: each keeps its previous pose exactly, fused and taped."""
    import gradslam_b200 as gs

    B, L, H, W = 4, 3, 40, 52
    rgb, depth, K, poses = camera_inputs(B, L, H, W, 64, skew=0.75)
    depth[1, :2] = 0.0
    depth[2, 2] = 0.0
    frames = _frames(rgb, depth, K, poses)
    pc = _fused_map(frames[:, :2])
    assert pc.num_points_per_pointcloud.tolist()[1] == 0
    prev_poses = poses[:, 1].clone()
    prev_poses[3] = prev_poses[3] @ torch.diag(torch.tensor([-1.0, 1.0, -1.0, 1.0]))
    prev = gs.RGBDImages(rgb[:, 1:2].to(DEV), depth[:, 1:2].to(DEV), K.to(DEV), prev_poses[:, None].to(DEV))
    slam = gs.PointFusion(odom=odom, association="projective", numiters=10, dsratio=2, device=DEV)
    got = slam._localize(pc, frames[:, 2], prev)[:, 0].cpu()
    assert torch.equal(got[1:], prev_poses[1:])
    assert not torch.equal(got[0], prev_poses[0])
    d_req = depth[:, 2:3].to(DEV).requires_grad_(True)
    live = gs.RGBDImages(rgb[:, 2:3].to(DEV), d_req, K.to(DEV), poses[:, 2:3].to(DEV))
    taped = slam._localize(pc, live, prev)[:, 0].detach().cpu()
    assert torch.equal(taped, got)


def test_benchmark_inputs_match_oracle():
    """The benchmark's ICP leg at 640x480, B=8: the last frame localised against the map of the first seven; elements 0
    and 7 against the oracle.  dsratio=1 (307 k source points per element) runs at that size."""
    import gradslam_b200 as gs

    B, L, H, W = 8, 8, 480, 640
    rgb, depth, K, poses = make_sequence(B, L, H, W, seed=100, yaw0=0.6)
    frames = _frames(rgb, depth, K, poses)
    pc = _fused_map(frames[:, : L - 1])
    slam = gs.PointFusion(odom="gradicp", association="projective", device=DEV)
    got = slam._localize(pc, frames[:, L - 1], frames[:, L - 2])[:, 0].cpu()
    elems = [0, 7]
    at_prev = oracle.frame_maps(depth[elems][:, L - 1:L], K[elems], poses[elems][:, L - 2:L - 1])
    want = po.odometry_projective(_oracle_map(pc, elems), at_prev, poses[elems][:, L - 2], K[elems][:, 0], H, W,
                                  "gradicp", 4, _icp_kwargs("gradicp", 20, None))
    torch.testing.assert_close(got[elems], want, rtol=0, atol=1e-4)
    dense = gs.PointFusion(odom="gradicp", association="projective", dsratio=1, device=DEV)
    got1 = dense._localize(pc, frames[:, L - 1], frames[:, L - 2])[:, 0].cpu()
    assert torch.isfinite(got1).all()
    assert (got1 - poses[:, L - 1]).abs().max() < 0.02


def test_differentiable_mode_gradients_match_oracle_autograd():
    """d(pose)/d(live depth), d(pose)/d(previous pose) and d(pose)/d(map points, normals) of ICPSLAM's projective
    gradICP step against autograd of the oracle, on lattice-hole depth (see test_gpu_backward.make_sequence)."""
    import gradslam_b200 as gs

    B, H, W = 1, 32, 40
    rgb, depth, K, poses = make_sequence(B, 2, H, W, seed=33, yaw0=0.6, hole_fraction=0.0)
    depth = punch_lattice_holes(depth)
    m0 = oracle.frame_maps(depth[:, :1], K, poses[:, :1])
    valid = m0["valid"][0, 0]
    P0, N0 = m0["gvertex"][0, 0][valid], m0["gnormal"][0, 0][valid]
    w = torch.randn(4, 4, generator=torch.Generator().manual_seed(2))

    p_ref, n_ref = P0.clone().requires_grad_(True), N0.clone().requires_grad_(True)
    prev_ref = poses[:, 0].clone().requires_grad_(True)
    d_ref = depth[:, 1:2].clone().requires_grad_(True)
    at_prev = oracle.frame_maps(d_ref, K, prev_ref.unsqueeze(1))
    ref = po.odometry_projective(oracle.SurfelMap([p_ref], [n_ref]), at_prev, prev_ref, K[:, 0], H, W, "gradicp", 2,
                                 _icp_kwargs("gradicp", 3, None))
    (ref[0] * w).sum().backward()

    p_g, n_g = P0.to(DEV).requires_grad_(True), N0.to(DEV).requires_grad_(True)
    pc = gs.Pointclouds(points=p_g[None], normals=n_g[None])
    prev_g = poses[:, 0:1].to(DEV).requires_grad_(True)
    d_g = depth[:, 1:2].to(DEV).requires_grad_(True)
    live = gs.RGBDImages(rgb[:, 1:2].to(DEV), d_g, K.to(DEV), poses[:, 1:2].to(DEV))
    prev = gs.RGBDImages(rgb[:, 0:1].to(DEV), depth[:, 0:1].to(DEV), K.to(DEV), prev_g)
    slam = gs.ICPSLAM(odom="gradicp", association="projective", numiters=3, dsratio=2, device=DEV)
    out = slam._localize(pc, live, prev)
    torch.testing.assert_close(out[:, 0].detach().cpu(), ref.detach(), rtol=0, atol=1e-4)
    (out[0, 0] * w.to(DEV)).sum().backward()
    for got, want in ((d_g.grad, d_ref.grad), (prev_g.grad[:, 0, :3], prev_ref.grad[:, :3]), (p_g.grad, p_ref.grad),
                      (n_g.grad, n_ref.grad)):
        got = got.cpu()
        assert torch.isfinite(got).all() and want.abs().max() > 0
        scale = want.abs().max().item()
        torch.testing.assert_close(got, want, rtol=5e-2, atol=5e-3 * scale)
