"""GPU parity of the joint geometric and photometric projective ICP (ICPSLAM / PointFusion(photometric_weight=w),
gsx_icp_localize_projective, gsx_icp_projective_targets at w > 0) with tests/photometric_oracle.py: the model image and
the association bit for bit, poses at the ICP tests' 1e-4, w = 0 and a black scene bit for bit against the geometric
call; the differentiable mode's poses equal the fused call's and its gradients match autograd of the oracle."""
import math

import pytest
import torch

import gsx_oracle as oracle
import photometric_oracle as ph
from cameras import camera_inputs
from gradslam_b200.synthetic import make_sequence, make_textured_sequence
from test_gpu_projective_icp import _frames, _icp_kwargs
from test_photometric_oracle import W_TRACK

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
# Pose tolerance against the oracle where the joint sums run over thousands of points (ds = 1 at 90x120, 640x480): the
# photometric rows reach |c| ~ 50 per metre, so float32 sums in the kernel's fixed order and the oracle's matmul order
# part by up to ~2e-4 in translation after gradICP's iterations (measured on an H100: 1.7e-4 and 1.9e-4).  Elsewhere 1e-4.
ATOL_MANY_POINTS = 5e-4


def _map(frames, radii=True):
    import gradslam_b200 as gs

    pc, _ = gs.PointFusion(odom="gt", surfel_radii=radii, device=DEV)(frames)
    return pc


def _oracle(pc, elems=None):
    """-> (SurfelMap with colours, radii per element) of the device map."""
    elems = range(len(pc)) if elems is None else elems
    cpu = lambda lst: None if lst is None else [lst[b].cpu() for b in elems]
    return (oracle.SurfelMap(cpu(pc.points_list), cpu(pc.normals_list), cpu(pc.colors_list), cpu(pc.features_list)),
            cpu(pc.radii_list))


@pytest.mark.parametrize("M", [0, 3])
def test_model_image_and_association_bit_exact(M):
    from gradslam_b200.odometry.icputils import projective_intensity

    B, L, H, W = 3, 3, 45, 62
    rgb, depth, K, poses = camera_inputs(B, L, H, W, 71, skew=0.75)
    pc = _map(_frames(rgb, depth, K, poses)[:, :2])
    idx, I_m = (t.cpu() for t in projective_intensity(pc, K[:, 0].to(DEV), poses[:, 1].to(DEV), H, W, M))
    smap, radii = _oracle(pc)
    w_idx, _, _, w_Im = ph.target_images(smap, radii, poses[:, 1], K[:, 0], H, W, M)
    assert torch.equal(idx, w_idx)
    assert torch.equal(I_m, w_Im)
    assert int((idx >= 0).sum()) > 1000


@pytest.mark.parametrize("ds", [1, 2, 4])
@pytest.mark.parametrize("dist_thresh", [None, 0.01])
@pytest.mark.parametrize("odom", ["icp", "gradicp"])
def test_localize_matches_oracle(odom, dist_thresh, ds):
    import gradslam_b200 as gs

    B, L, H, W = 3, 3, 90, 120  # (the texture's shortest wavelength spans ~10 pixels: its gradients are resolved)
    rgb, depth, K, poses = make_textured_sequence(B, L, H, W, seed=3, yaw0=0.3)
    frames = _frames(rgb, depth, K, poses)
    pc = _map(frames[:, :2])
    for M in (0, 3):
        slam = gs.PointFusion(odom=odom, association="projective", numiters=10, dsratio=ds, dist_thresh=dist_thresh,
                              surfel_radii=True, target_splat_px=M, photometric_weight=W_TRACK, device=DEV)
        got = slam._localize(pc, frames[:, 2], frames[:, 1])[:, 0].cpu()
        at_prev = oracle.frame_maps(depth[:, 2:3], K, poses[:, 1:2])
        smap, radii = _oracle(pc)
        want = ph.odometry(smap, radii, at_prev, rgb[:, 2:3], poses[:, 1], K[:, 0], H, W, odom, ds,
                           _icp_kwargs(odom, 10, dist_thresh), M, W_TRACK)
        torch.testing.assert_close(got, want, rtol=0, atol=1e-4 if ds > 1 else ATOL_MANY_POINTS)
        geo = gs.PointFusion(odom=odom, association="projective", numiters=10, dsratio=ds, dist_thresh=dist_thresh,
                             surfel_radii=True, target_splat_px=M, device=DEV)._localize(pc, frames[:, 2], frames[:, 1])
        assert not torch.equal(got, geo[:, 0].cpu())


def test_colours_at_zero_weight_and_a_black_scene_give_the_geometric_poses():
    """gsx_icp_localize_projective with colours at w = 0 is its geometric call bit for bit; so is w > 0 on a scene whose
    colours are all 0 (every photometric row and residual is 0)."""
    import gradslam_b200 as gs
    from gradslam_b200.odometry.icputils import localize_projective

    B, L, H, W = 3, 3, 45, 62
    rgb, depth, K, poses = camera_inputs(B, L, H, W, 72, skew=0.75)
    for colours in (rgb, torch.zeros_like(rgb)):
        frames = _frames(colours, depth, K, poses)
        pc = _map(frames[:, :2])
        for M in (0, 3):
            odom = gs.ICPSLAM(odom="gradicp", association="projective", numiters=10, dsratio=2).odomprov
            live = frames[:, 2]
            base = localize_projective(pc, live, frames[:, 1], 2, odom, M)
            for w in ((0.0, 0.5) if colours is not rgb else (0.0,)):
                from gradslam_b200 import _C
                from gradslam_b200.odometry.icputils import _ProjectiveWorkspace

                out = torch.empty_like(base)
                ws = _ProjectiveWorkspace.get(DEV, B, H, W, 2, True)
                _C.launch("gsx_icp_localize_projective", pc._geo, pc._counts_dev[pc._cur], pc.capacity, pc._bound,
                          live.depth_image.contiguous(), H * W, K.to(DEV).contiguous(), 16,
                          poses[:, 1:2].to(DEV).contiguous(), 16, B, H, W, 2, 1, 10, 1e-8, 0, 0.0, 2.0, 1.0, 1.0, 200.0,
                          out, 16, ws, ws.numel(), M, pc._col, live.rgb_image.contiguous(), H * W * 3, w,
                          math.inf, math.inf)
                assert torch.equal(out, base), (M, w)


@pytest.mark.parametrize("odom", ["icp", "gradicp"])
def test_empty_map_no_depth_and_camera_turned_away_keep_the_previous_pose(odom):
    import gradslam_b200 as gs

    B, L, H, W = 4, 3, 40, 52
    rgb, depth, K, poses = make_textured_sequence(B, L, H, W, seed=4, yaw0=0.6)
    depth[1, :2] = 0.0
    depth[2, 2] = 0.0
    frames = _frames(rgb, depth, K, poses)
    pc = _map(frames[:, :2])
    assert pc.num_points_per_pointcloud.tolist()[1] == 0
    prev_poses = poses[:, 1].clone()
    prev_poses[3] = prev_poses[3] @ torch.diag(torch.tensor([-1.0, 1.0, -1.0, 1.0]))
    prev = gs.RGBDImages(rgb[:, 1:2].to(DEV), depth[:, 1:2].to(DEV), K.to(DEV), prev_poses[:, None].to(DEV))
    slam = gs.PointFusion(odom=odom, association="projective", numiters=10, dsratio=2, surfel_radii=True,
                          photometric_weight=W_TRACK, device=DEV)
    got = slam._localize(pc, frames[:, 2], prev)[:, 0].cpu()
    assert torch.equal(got[1:], prev_poses[1:])
    assert not torch.equal(got[0], prev_poses[0])


@pytest.mark.parametrize("odom", ["icp", "gradicp"])
def test_pointfusion_and_icpslam_runs_match_oracle_step_by_step(odom):
    """Per step, from the device's own map, against the oracle at 1e-4; forward() gives the same poses."""
    import gradslam_b200 as gs

    B, L, H, W = 2, 4, 48, 64
    rgb, depth, K, poses = make_textured_sequence(B, L, H, W, seed=8, yaw0=0.0)
    frames = _frames(rgb, depth, K, poses)
    for cls in (gs.PointFusion, gs.ICPSLAM):
        extra = dict(surfel_radii=True) if cls is gs.PointFusion else {}
        slam = cls(odom=odom, association="projective", numiters=10, dsratio=2, photometric_weight=W_TRACK,
                   device=DEV, **extra)
        pc, prev, got = gs.Pointclouds(device=DEV), None, []
        for s in range(L):
            smap = _oracle(pc)[0] if pc.has_points else oracle.SurfelMap()
            live = frames[:, s]
            pc, pose = slam.step(pc, live, prev)
            pose = pose[:, 0].cpu()
            got.append(pose)
            if s > 0:
                at_prev = oracle.frame_maps(depth[:, s:s + 1], K, prev.poses.cpu())
                want = ph.odometry(smap, None, at_prev, rgb[:, s:s + 1], prev.poses[:, 0].cpu(), K[:, 0], H, W, odom,
                                   2, _icp_kwargs(odom, 10, None), 0, W_TRACK)
                torch.testing.assert_close(pose, want, rtol=0, atol=1e-4)
            prev = live
        _, rec = slam(frames)
        assert torch.equal(rec.cpu(), torch.stack(got, 1))


@pytest.mark.parametrize("odom", ["icp", "gradicp"])
def test_joint_tracking_halves_the_far_wall_drift_on_the_device(odom):
    """The accuracy gain of test_photometric_oracle at the same size and weight, with the device's PointFusion."""
    import gradslam_b200 as gs

    rgb, depth, K, poses = make_textured_sequence(1, 8, 120, 160, seed=0, yaw0=0.0)
    frames = _frames(rgb, depth, K, poses)
    err = {}
    for w in (0.0, W_TRACK):
        _, rec = gs.PointFusion(odom=odom, association="projective", surfel_radii=True, photometric_weight=w,
                                device=DEV)(frames)
        err[w] = ph.translation_error(rec.cpu(), poses)
    assert err[W_TRACK] <= 0.5 * err[0.0], err


def test_benchmark_inputs_match_oracle():
    """640x480, B = 8, make_sequence's random colours: the last frame against the map of the first seven at M = 0;
    elements 0 and 7 against the oracle.  (Fresh noise in every frame makes the photometric term ill conditioned: at
    M = 3 the device and the oracle part by 1e-3, rounding order alone; the textured tests cover M = 3.)"""
    import gradslam_b200 as gs

    B, L, H, W = 8, 8, 480, 640
    rgb, depth, K, poses = make_sequence(B, L, H, W, seed=100, yaw0=0.6)
    frames = _frames(rgb, depth, K, poses)
    pc = _map(frames[:, : L - 1])
    elems = [0, 7]
    smap, radii = _oracle(pc, elems)
    at_prev = oracle.frame_maps(depth[elems][:, L - 1:L], K[elems], poses[elems][:, L - 2:L - 1])
    for M in (0,):
        slam = gs.PointFusion(odom="gradicp", association="projective", surfel_radii=True, target_splat_px=M,
                              photometric_weight=W_TRACK, device=DEV)
        got = slam._localize(pc, frames[:, L - 1], frames[:, L - 2])[:, 0].cpu()
        want = ph.odometry(smap, radii, at_prev, rgb[elems][:, L - 1:L], poses[elems][:, L - 2], K[elems][:, 0], H, W,
                           "gradicp", 4, _icp_kwargs("gradicp", 20, None), M, W_TRACK)
        torch.testing.assert_close(got[elems], want, rtol=0, atol=ATOL_MANY_POINTS)


@pytest.mark.parametrize("M", [0, 3])
@pytest.mark.parametrize("odom", ["icp", "gradicp"])
def test_taped_poses_equal_the_fused_poses(odom, M):
    """The differentiable mode (live depth and rgb requiring grad) gives the fused call's poses bit for bit."""
    import gradslam_b200 as gs

    B, L, H, W = 3, 3, 90, 120
    rgb, depth, K, poses = make_textured_sequence(B, L, H, W, seed=5, yaw0=0.3)
    frames = _frames(rgb, depth, K, poses)
    pc = _map(frames[:, :2])
    for ds, dth in ((1, None), (2, 0.01), (4, None)):
        slam = gs.PointFusion(odom=odom, association="projective", numiters=10, dsratio=ds, dist_thresh=dth,
                              surfel_radii=True, target_splat_px=M, photometric_weight=W_TRACK, device=DEV)
        fused = slam._localize(pc, frames[:, 2], frames[:, 1])
        live = gs.RGBDImages(rgb[:, 2:3].to(DEV).requires_grad_(True), depth[:, 2:3].to(DEV).requires_grad_(True),
                             K.to(DEV), poses[:, 2:3].to(DEV))
        taped = slam._localize(pc, live, frames[:, 1])
        assert taped.requires_grad
        assert torch.equal(taped.detach(), fused), (ds, dth)


@pytest.mark.parametrize("M", [0, 3])
def test_differentiable_mode_gradients_match_oracle_autograd(M):
    """d(pose)/d(live depth, live rgb, map points, normals, colours, previous pose) of the joint gradICP step against
    autograd of the oracle, on lattice-hole depth of the textured scene."""
    import gradslam_b200 as gs
    import radii_oracle as ro
    from gradslam_b200.synthetic import punch_lattice_holes

    B, H, W = 1, 32, 40
    rgb, depth, K, poses = make_textured_sequence(B, 2, H, W, seed=33, yaw0=0.6, hole_fraction=0.0)
    depth = punch_lattice_holes(depth)
    m0 = oracle.frame_maps(depth[:, :1], K, poses[:, :1])
    valid = m0["valid"][0, 0]
    P0, N0, C0 = m0["gvertex"][0, 0][valid], m0["gnormal"][0, 0][valid], rgb[0, 0][valid]
    R0 = ro.radius_image(depth[:, :1], m0, K)[0][valid].unsqueeze(1)
    wts = torch.randn(4, 4, generator=torch.Generator().manual_seed(2))

    p_ref, n_ref, c_ref = (t.clone().requires_grad_(True) for t in (P0, N0, C0))
    prev_ref = poses[:, 0].clone().requires_grad_(True)
    d_ref, rgb_ref = depth[:, 1:2].clone().requires_grad_(True), rgb[:, 1:2].clone().requires_grad_(True)
    at_prev = oracle.frame_maps(d_ref, K, prev_ref.unsqueeze(1))
    ref = ph.odometry(oracle.SurfelMap([p_ref], [n_ref], [c_ref]), [R0], at_prev, rgb_ref, prev_ref, K[:, 0], H, W,
                      "gradicp", 2, _icp_kwargs("gradicp", 3, None), M, W_TRACK)
    (ref[0] * wts).sum().backward()

    p_g, n_g, c_g = (t.to(DEV).requires_grad_(True) for t in (P0, N0, C0))
    pc = gs.Pointclouds(points=p_g[None], normals=n_g[None], colors=c_g[None])
    pc.radii_list = [R0.to(DEV)]
    prev_g = poses[:, 0:1].to(DEV).requires_grad_(True)
    d_g, rgb_g = depth[:, 1:2].to(DEV).requires_grad_(True), rgb[:, 1:2].to(DEV).requires_grad_(True)
    live = gs.RGBDImages(rgb_g, d_g, K.to(DEV), poses[:, 1:2].to(DEV))
    prev = gs.RGBDImages(rgb[:, 0:1].to(DEV), depth[:, 0:1].to(DEV), K.to(DEV), prev_g)
    slam = gs.ICPSLAM(odom="gradicp", association="projective", numiters=3, dsratio=2, target_splat_px=M,
                      photometric_weight=W_TRACK, device=DEV)
    out = slam._localize(pc, live, prev)
    torch.testing.assert_close(out[:, 0].detach().cpu(), ref.detach(), rtol=0, atol=1e-4)
    (out[0, 0] * wts.to(DEV)).sum().backward()
    for name, got, want in (("depth", d_g.grad, d_ref.grad), ("rgb", rgb_g.grad, rgb_ref.grad),
                            ("prev", prev_g.grad[:, 0, :3], prev_ref.grad[:, :3]), ("points", p_g.grad, p_ref.grad),
                            ("normals", n_g.grad, n_ref.grad), ("colours", c_g.grad, c_ref.grad)):
        got = got.cpu()
        assert torch.isfinite(got).all() and want.abs().max() > 0, name
        scale = want.abs().max().item()
        torch.testing.assert_close(got, want, rtol=5e-2, atol=5e-3 * scale, msg=name)


def test_projective_entry_points_refuse_bad_weights_and_null_colours_without_a_launch():
    from gradslam_b200 import _C

    bufs = [torch.full((256,), -7.25, device=DEV) for _ in range(8)]
    geo, counts, depth, K, prev, out, ws, col = bufs
    index = torch.full((64,), -7, dtype=torch.int64, device=DEV)
    call = lambda w, c, r: _C.launch("gsx_icp_localize_projective", geo, counts, 4, 4, depth, 16, K, 16, prev, 16, 1,
                                     4, 4, 1, 1, 1, 1e-8, 0, 0.0, 2.0, 1.0, 1.0, 200.0, out, 16, ws, 1024, 0, c, r, 48,
                                     w, math.inf, math.inf)
    for bad in (-0.5, float("nan"), float("inf")):
        with pytest.raises(RuntimeError, match="photometric_weight"):
            call(bad, col, col)
    for c, r in ((None, col), (col, None)):
        with pytest.raises(RuntimeError, match="colour"):
            call(0.5, c, r)
    with pytest.raises(RuntimeError, match="null"):
        _C.launch("gsx_icp_projective_targets", geo, None, counts, 4, 4, K, 16, prev, 16, 1, 4, 4, 0, index, col, col,
                  col)
    torch.cuda.synchronize()
    for t in bufs:
        assert torch.equal(t, torch.full((256,), -7.25, device=DEV))
    assert torch.equal(index, torch.full((64,), -7, dtype=torch.int64, device=DEV))
