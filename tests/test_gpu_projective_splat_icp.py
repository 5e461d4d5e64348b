"""GPU parity of the projective ICP against the disk-splat render (ICPSLAM / PointFusion(target_splat_px=M),
gsx_icp_localize_projective and gsx_icp_projective_targets at max_splat_px = M) with tests/projective_splat_oracle.py:
the target images bit for bit, poses at the ICP tests' 1e-4, maps at 1e-3, gradients at the tolerances of
test_gpu_projective_icp.py."""
import math

import pytest
import torch

import gsx_oracle as oracle
import projective_oracle as po
import projective_splat_oracle as pso
import radii_oracle as ro
from cameras import camera_inputs
from gradslam_b200.synthetic import make_sequence, punch_lattice_holes
from test_gpu_projective_icp import _frames, _icp_kwargs, _oracle_map

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _radii_map(frames):
    import gradslam_b200 as gs

    pc, _ = gs.PointFusion(odom="gt", surfel_radii=True, device=DEV)(frames)
    return pc


def _radii(pc, elems=None):
    elems = range(len(pc)) if elems is None else elems
    return [pc.radii_list[b].cpu() for b in elems]


def _targets(pc, K, prev, H, W, M):
    from gradslam_b200.odometry.icputils import projective_targets

    return [t.cpu() for t in projective_targets(pc, K.to(DEV), prev.to(DEV), H, W, target_splat_px=M)]


def _assert_targets(got, want):
    for name, g, w in zip(("index", "tgt_p", "tgt_n"), got, want):
        assert torch.equal(g, w), name


def _won_by_disk(idx, radii):
    """bool (B, H*W): pixels a row with a radius won."""
    out = torch.zeros_like(idx, dtype=torch.bool)
    for b, r in enumerate(radii):
        cov = idx[b] >= 0
        out[b, cov] = r[idx[b, cov], 0] > 0
    return out


@pytest.mark.parametrize("M", [1, 3])
def test_targets_bit_exact_on_the_corner_cases(M):
    """projective_oracle.small_case (ties, frustum bounds, rows behind the camera, skew and a 4th K column, an empty
    element) with radii on most rows."""
    import gradslam_b200 as gs

    H, W = 6, 8
    smap, maps, _, pose, K = po.small_case(H, W)
    g = torch.Generator().manual_seed(5)
    radii = [torch.where(torch.rand(m.shape[0], 1, generator=g) < 0.3, 0.0, 0.2 + torch.rand(m.shape[0], 1, generator=g))
             for m in maps]
    pc = gs.Pointclouds(points=[m.to(DEV) for m in maps], normals=[n.to(DEV) for n in smap.normals])
    pc.radii_list = [r.to(DEV) for r in radii]
    got = _targets(pc, K, pose, H, W, M)
    want = pso.target_images(smap, radii, pose, K, H, W, M)
    _assert_targets(got, want)
    assert bool(_won_by_disk(want[0], radii)[:2].any(-1).all())
    _assert_targets(_targets(pc, K, pose, H, W, 0), po.target_images(smap, pose, K, H, W))


@pytest.mark.parametrize("M", [1, 3])
def test_targets_bit_exact_on_fused_maps_and_equal_to_k1_at_disk_pixels(M):
    """Maps fused with radii from camera_inputs (a camera per element, skew, 4th column); at the pixels a disk won the
    target point is RGBDImages(splat depth, ..., prev).global_vertex_map bit for bit."""
    import gradslam_b200 as gs

    B, L, H, W = 3, 3, 45, 62
    rgb, depth, K, poses = camera_inputs(B, L, H, W, 62, skew=0.75)
    pc = _radii_map(_frames(rgb, depth, K, poses)[:, :2])
    radii = _radii(pc)
    got = _targets(pc, K[:, 0], poses[:, 1], H, W, M)
    _assert_targets(got, pso.target_images(_oracle_map(pc), radii, poses[:, 1], K[:, 0], H, W, M))
    disk = _won_by_disk(got[0], radii)
    assert int(disk.sum()) > 1000
    splat = gs.render_pointclouds(pc, K.to(DEV), poses[:, 1:2].to(DEV), H, W, max_splat_px=M)
    assert torch.equal(splat.index.view(B, H * W).cpu(), got[0])
    k1 = gs.RGBDImages(torch.zeros(B, 1, H, W, 3, device=DEV), splat.depth, K.to(DEV), poses[:, 1:2].to(DEV))
    k1 = k1.global_vertex_map.reshape(B, H * W, 3).cpu()
    assert torch.equal(got[1][disk], k1[disk])


def test_splat_targets_cover_the_lattice_holes():
    """Lattice-hole depth: the one-pixel targets leave the holes empty, disks cover them, both bit for bit."""
    B, L, H, W = 2, 2, 40, 52
    rgb, depth, K, poses = make_sequence(B, L, H, W, seed=21, yaw0=0.6, hole_fraction=0.0)
    depth = punch_lattice_holes(depth)
    pc = _radii_map(_frames(rgb, depth, K, poses)[:, :1])
    smap, radii = _oracle_map(pc), _radii(pc)
    idx = {}
    for M in (0, 1, 2):
        got = _targets(pc, K[:, 0], poses[:, 0], H, W, M)
        _assert_targets(got, pso.target_images(smap, radii, poses[:, 0], K[:, 0], H, W, M))
        idx[M] = got[0]
    for M in (1, 2):
        assert int(((idx[M] >= 0) & (idx[0] < 0)).sum()) > 20
        assert int(((idx[M] < 0) & (idx[0] >= 0)).sum()) == 0


@pytest.mark.parametrize("ds", [1, 2, 4])
@pytest.mark.parametrize("dist_thresh", [None, 0.01])
@pytest.mark.parametrize("odom", ["icp", "gradicp"])
def test_localize_matches_oracle_and_taped_path(odom, dist_thresh, ds):
    """The fused call at M = 3 against the oracle (H*W = 2790, a camera per element), and the differentiable mode (live
    depth requiring grad) against the fused call, bit for bit."""
    import gradslam_b200 as gs

    B, L, H, W = 3, 3, 45, 62
    rgb, depth, K, poses = camera_inputs(B, L, H, W, 61, skew=0.75)
    frames = _frames(rgb, depth, K, poses)
    pc = _radii_map(frames[:, :2])
    slam = gs.PointFusion(odom=odom, association="projective", numiters=10, dsratio=ds, dist_thresh=dist_thresh,
                          surfel_radii=True, target_splat_px=3, device=DEV)
    got = slam._localize(pc, frames[:, 2], frames[:, 1])
    at_prev = oracle.frame_maps(depth[:, 2:3], K, poses[:, 1:2])
    want = pso.odometry_projective(_oracle_map(pc), _radii(pc), at_prev, poses[:, 1], K[:, 0], H, W, odom, ds,
                                   _icp_kwargs(odom, 10, dist_thresh), 3)
    torch.testing.assert_close(got[:, 0].cpu(), want, rtol=0, atol=1e-4)
    assert not torch.equal(got[:, 0].cpu(), poses[:, 1])
    d_req = depth[:, 2:3].to(DEV).requires_grad_(True)
    live = gs.RGBDImages(rgb[:, 2:3].to(DEV), d_req, K.to(DEV), poses[:, 2:3].to(DEV))
    taped = slam._localize(pc, live, frames[:, 1])
    assert taped.requires_grad
    assert torch.equal(taped.detach(), got)


@pytest.mark.parametrize("odom", ["icp", "gradicp"])
def test_empty_map_no_depth_and_camera_turned_away_keep_the_previous_pose(odom):
    import gradslam_b200 as gs

    B, L, H, W = 4, 3, 40, 52
    rgb, depth, K, poses = camera_inputs(B, L, H, W, 64, skew=0.75)
    depth[1, :2] = 0.0
    depth[2, 2] = 0.0
    frames = _frames(rgb, depth, K, poses)
    pc = _radii_map(frames[:, :2])
    assert pc.num_points_per_pointcloud.tolist()[1] == 0
    prev_poses = poses[:, 1].clone()
    prev_poses[3] = prev_poses[3] @ torch.diag(torch.tensor([-1.0, 1.0, -1.0, 1.0]))
    prev = gs.RGBDImages(rgb[:, 1:2].to(DEV), depth[:, 1:2].to(DEV), K.to(DEV), prev_poses[:, None].to(DEV))
    slam = gs.PointFusion(odom=odom, association="projective", numiters=10, dsratio=2, surfel_radii=True,
                          target_splat_px=3, device=DEV)
    got = slam._localize(pc, frames[:, 2], prev)[:, 0].cpu()
    assert torch.equal(got[1:], prev_poses[1:])
    assert not torch.equal(got[0], prev_poses[0])
    d_req = depth[:, 2:3].to(DEV).requires_grad_(True)
    live = gs.RGBDImages(rgb[:, 2:3].to(DEV), d_req, K.to(DEV), poses[:, 2:3].to(DEV))
    taped = slam._localize(pc, live, prev)[:, 0].detach().cpu()
    assert torch.equal(taped, got)


def test_maps_without_radii_give_the_point_poses():
    """M > 0 on a map without radii gives the M = 0 poses bit for bit, fused and taped."""
    import gradslam_b200 as gs

    B, L, H, W = 3, 3, 45, 62
    rgb, depth, K, poses = camera_inputs(B, L, H, W, 65, skew=0.75)
    frames = _frames(rgb, depth, K, poses)
    pc, _ = gs.PointFusion(odom="gt", device=DEV)(frames[:, :2])
    run = lambda M: gs.ICPSLAM(odom="gradicp", association="projective", numiters=10, dsratio=2, target_splat_px=M,
                               device=DEV)._localize(pc, frames[:, 2], frames[:, 1])
    base = run(0)
    assert torch.equal(run(3), base) and torch.equal(run(16), base)
    d_req = depth[:, 2:3].to(DEV).requires_grad_(True)
    live = gs.RGBDImages(rgb[:, 2:3].to(DEV), d_req, K.to(DEV), poses[:, 2:3].to(DEV))
    taped = gs.ICPSLAM(odom="gradicp", association="projective", numiters=10, dsratio=2, target_splat_px=3,
                       device=DEV)._localize(pc, live, frames[:, 1])
    assert torch.equal(taped.detach(), base)


def test_icpslam_run_with_splat_targets_matches_oracle():
    """An aggregation map has no radii: a whole ICPSLAM run at M = 3 is the one-pixel run."""
    import gradslam_b200 as gs

    B, L, H, W = 3, 4, 48, 64
    rgb, depth, K, poses = make_sequence(B, L, H, W, seed=8, yaw0=0.6)
    slam = gs.ICPSLAM(odom="gradicp", association="projective", numiters=10, dsratio=2, target_splat_px=3, device=DEV)
    pc, rec = slam(_frames(rgb, depth, K, poses))
    ref = po.run_slam(rgb, depth, K, poses, mode="aggregate", odom="gradicp", numiters=10, dsratio=2)
    torch.testing.assert_close(rec.cpu(), ref.poses, rtol=0, atol=1e-4)
    assert pc.num_points_per_pointcloud.tolist() == ref.map.counts()
    for b in range(B):
        torch.testing.assert_close(pc.points_list[b].cpu(), ref.map.points[b], rtol=0, atol=1e-3)


def _full_oracle_map(pc):
    if not pc.has_points:
        return oracle.SurfelMap(), None
    cpu = lambda lst: [t.cpu() for t in lst]
    return (oracle.SurfelMap(cpu(pc.points_list), cpu(pc.normals_list), cpu(pc.colors_list), cpu(pc.features_list)),
            cpu(pc.radii_list))


@pytest.mark.parametrize("odom", ["icp", "gradicp"])
def test_pointfusion_run_with_splat_targets_matches_oracle_step_by_step(odom):
    """PointFusion(surfel_radii=True, target_splat_px=3) over four frames, checked per step against the oracle from the
    GPU's own map: the pose at 1e-4, then the fused map (sizes exact, points and radii at 1e-3); forward() gives the
    same poses.  A whole run is not compared with a whole oracle run: with splat targets a change of 1e-7 in one pose
    moves later poses by up to 1e-3 (the merges that flip move the disks), so rounding alone would decide the result."""
    import gradslam_b200 as gs

    B, L, H, W = 3, 4, 48, 64
    rgb, depth, K, poses = make_sequence(B, L, H, W, seed=8, yaw0=0.6)
    frames = _frames(rgb, depth, K, poses)
    slam = gs.PointFusion(odom=odom, association="projective", numiters=10, dsratio=2, surfel_radii=True,
                          target_splat_px=3, device=DEV)
    pc, prev, got = gs.Pointclouds(device=DEV), None, []
    for s in range(L):
        smap, radii = _full_oracle_map(pc)
        live = frames[:, s]
        pc, pose = slam.step(pc, live, prev)
        pose = pose[:, 0].cpu()
        got.append(pose)
        d = depth[:, s:s + 1]
        if s > 0:
            at_prev = oracle.frame_maps(d, K, prev.poses.cpu())
            want = pso.odometry_projective(smap, radii, at_prev, prev.poses[:, 0].cpu(), K[:, 0], H, W, odom, 2,
                                           _icp_kwargs(odom, 10, None), 3)
            torch.testing.assert_close(pose, want, rtol=0, atol=1e-4)
        maps = oracle.frame_maps(d, K, pose.unsqueeze(1))
        table = oracle.find_correspondences(smap, maps, pose, K[:, 0], 0.05, slam.dot_th)
        want_radii = ro.fuse_radii(smap, radii, maps, d, K, table, 0.6)
        want_map = oracle.fuse_with_map(smap, maps, rgb[:, s:s + 1], table, 0.6)
        assert pc.num_points_per_pointcloud.tolist() == want_map.counts()
        for b in range(B):
            torch.testing.assert_close(pc.points_list[b].cpu(), want_map.points[b], rtol=0, atol=1e-3)
            torch.testing.assert_close(pc.radii_list[b].cpu(), want_radii[b], rtol=0, atol=1e-3)
        prev = live
    assert (torch.stack(got, 1) - poses).abs().max() < 0.02  # it tracks
    _, rec = slam(frames)
    assert torch.equal(rec.cpu(), torch.stack(got, 1))


def test_benchmark_inputs_match_oracle():
    """640x480, B = 8: the last frame localised against the radii map of the first seven at M = 3; elements 0 and 7
    against the oracle."""
    import gradslam_b200 as gs

    B, L, H, W = 8, 8, 480, 640
    rgb, depth, K, poses = make_sequence(B, L, H, W, seed=100, yaw0=0.6)
    frames = _frames(rgb, depth, K, poses)
    pc = _radii_map(frames[:, : L - 1])
    slam = gs.PointFusion(odom="gradicp", association="projective", surfel_radii=True, target_splat_px=3, device=DEV)
    got = slam._localize(pc, frames[:, L - 1], frames[:, L - 2])[:, 0].cpu()
    elems = [0, 7]
    at_prev = oracle.frame_maps(depth[elems][:, L - 1:L], K[elems], poses[elems][:, L - 2:L - 1])
    want = pso.odometry_projective(_oracle_map(pc, elems), _radii(pc, elems), at_prev, poses[elems][:, L - 2],
                                   K[elems][:, 0], H, W, "gradicp", 4, _icp_kwargs("gradicp", 20, None), 3)
    torch.testing.assert_close(got[elems], want, rtol=0, atol=1e-4)


def test_differentiable_mode_gradients_match_oracle_autograd():
    """d(pose)/d(live depth, previous pose, map points, normals) of the projective gradICP step at M = 3 on a map with
    radii, against autograd of the oracle, on lattice-hole depth."""
    import gradslam_b200 as gs

    B, H, W = 1, 32, 40
    rgb, depth, K, poses = make_sequence(B, 2, H, W, seed=33, yaw0=0.6, hole_fraction=0.0)
    depth = punch_lattice_holes(depth)
    m0 = oracle.frame_maps(depth[:, :1], K, poses[:, :1])
    valid = m0["valid"][0, 0]
    P0, N0 = m0["gvertex"][0, 0][valid], m0["gnormal"][0, 0][valid]
    R0 = ro.radius_image(depth[:, :1], m0, K)[0][valid].unsqueeze(1)
    w = torch.randn(4, 4, generator=torch.Generator().manual_seed(2))

    p_ref, n_ref = P0.clone().requires_grad_(True), N0.clone().requires_grad_(True)
    prev_ref = poses[:, 0].clone().requires_grad_(True)
    d_ref = depth[:, 1:2].clone().requires_grad_(True)
    at_prev = oracle.frame_maps(d_ref, K, prev_ref.unsqueeze(1))
    ref = pso.odometry_projective(oracle.SurfelMap([p_ref], [n_ref]), [R0], at_prev, prev_ref, K[:, 0], H, W,
                                  "gradicp", 2, _icp_kwargs("gradicp", 3, None), 3)
    (ref[0] * w).sum().backward()

    p_g, n_g = P0.to(DEV).requires_grad_(True), N0.to(DEV).requires_grad_(True)
    pc = gs.Pointclouds(points=p_g[None], normals=n_g[None])
    pc.radii_list = [R0.to(DEV)]
    prev_g = poses[:, 0:1].to(DEV).requires_grad_(True)
    d_g = depth[:, 1:2].to(DEV).requires_grad_(True)
    live = gs.RGBDImages(rgb[:, 1:2].to(DEV), d_g, K.to(DEV), poses[:, 1:2].to(DEV))
    prev = gs.RGBDImages(rgb[:, 0:1].to(DEV), depth[:, 0:1].to(DEV), K.to(DEV), prev_g)
    slam = gs.ICPSLAM(odom="gradicp", association="projective", numiters=3, dsratio=2, target_splat_px=3, device=DEV)
    out = slam._localize(pc, live, prev)
    torch.testing.assert_close(out[:, 0].detach().cpu(), ref.detach(), rtol=0, atol=1e-4)
    (out[0, 0] * w.to(DEV)).sum().backward()
    for got, want in ((d_g.grad, d_ref.grad), (prev_g.grad[:, 0, :3], prev_ref.grad[:, :3]), (p_g.grad, p_ref.grad),
                      (n_g.grad, n_ref.grad)):
        got = got.cpu()
        assert torch.isfinite(got).all() and want.abs().max() > 0
        scale = want.abs().max().item()
        torch.testing.assert_close(got, want, rtol=5e-2, atol=5e-3 * scale)


def test_projective_entry_points_refuse_a_bad_max_splat_px_without_a_launch():
    from gradslam_b200 import _C

    bufs = [torch.full((256,), -7.25, device=DEV) for _ in range(8)]
    geo, counts, depth, K, prev, out, ws, tgt = bufs
    index = torch.full((64,), -7, dtype=torch.int64, device=DEV)
    for bad in (-1, 17):
        with pytest.raises(RuntimeError, match="max_splat_px"):
            _C.launch("gsx_icp_localize_projective", geo, counts, 4, 4, depth, 16, K, 16, prev, 16, 1, 4, 4, 1, 1, 1,
                      1e-8, 0, 0.0, 2.0, 1.0, 1.0, 200.0, out, 16, ws, 1024, bad, None, None, 0, 0.0, math.inf,
                      math.inf)
        with pytest.raises(RuntimeError, match="max_splat_px"):
            _C.launch("gsx_icp_projective_targets", geo, None, counts, 4, 4, K, 16, prev, 16, 1, 4, 4, bad, index, tgt,
                      tgt, None)
    torch.cuda.synchronize()
    for t in bufs:
        assert torch.equal(t, torch.full((256,), -7.25, device=DEV))
    assert torch.equal(index, torch.full((64,), -7, dtype=torch.int64, device=DEV))
