"""Removal of free-space violations (PointFusion's free_space_margin, fusionutils.fuse_and_prune) against the oracle of
tests/free_space_oracle.py, bit for bit: the whole-sequence call and the step API on the dynamic scene for several
t_max and margins (ring entries included), a camera per element, an all-invalid frame, an element whose map stays
empty and a camera turned away from the map, batch groups, split and host-fed calls, continuation through step(),
640x480, margin = inf against the age rule's entry points, ICP odometry, the differentiable mode and its gradients, and
the box leaving the GPU's own map."""
import math

import pytest
import torch

import gsx_oracle as oracle
import free_space_oracle as fo
import prune_oracle as po
from cameras import camera_inputs
from gradslam_b200.synthetic import DYNAMIC_BOX_CENTER, DYNAMIC_BOX_HALF_EXTENTS, make_dynamic_sequence

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _frames(gs, rgb, depth, K, poses):
    return gs.RGBDImages(rgb.to(DEV), depth.to(DEV), K.to(DEV), poses.to(DEV))


def _turn_away(poses, b, s):
    """Element b's camera at frame s turned by pi about its vertical axis: the map is behind it."""
    R = torch.tensor([[-1.0, 0.0, 0.0, 0.0], [0.0, 1.0, 0.0, 0.0], [0.0, 0.0, -1.0, 0.0], [0.0, 0.0, 0.0, 1.0]])
    poses[b, s] = poses[b, s] @ R


_inputs = {}


def _scene(kind, B=3, L=10, H=48, W=64):
    key = (kind, B, L, H, W)
    if key not in _inputs:
        if kind == "cameras":
            rgb, depth, K, poses = camera_inputs(B, L, H, W, 17, skew=0.75)
        else:
            k0, k1 = (1, 3) if L <= 6 else (2, 5)
            rgb, depth, K, poses = make_dynamic_sequence(B, L, H, W, k0, k1, seed=5)
            if kind == "edge":
                depth[:, L // 2] = 0.0  # an all-invalid frame
                depth[1] = 0.0          # element 1's map stays empty
                _turn_away(poses, 2, L // 2 + 1)
        c = po.confidence_quantile(oracle.run_slam(rgb, depth, K, poses, odom="gt").map, 0.3)
        _inputs[key] = (rgb, depth, K, poses, c)
    return _inputs[key]


_refs = {}


def _ref(kind, t_max, margin, **shape):
    key = (kind, t_max, margin, tuple(sorted(shape.items())))
    if key not in _refs:
        rgb, depth, K, poses, c = _scene(kind, **shape)
        _refs[key] = po_map = fo.run_pointfusion(rgb, depth, K, poses, c_stable=c, t_max=t_max, margin=margin)[0]
        if margin is not None and margin < math.inf and rgb.shape[2] <= 48:  # the rule removes rows here
            age = po.run_pointfusion(rgb, depth, K, poses, c_stable=c, t_max=t_max)[0]
            assert sum(po_map.counts()) < sum(age.counts())
    return _refs[key]


def _assert_matches(pc, smap):
    assert [int(c) for c in pc.num_points_per_pointcloud.tolist()] == smap.counts()
    for b in range(len(smap.counts())):
        assert torch.equal(pc.points_list[b].detach().cpu(), smap.points[b]), b
        assert torch.equal(pc.normals_list[b].detach().cpu(), smap.normals[b]), b
        assert torch.equal(pc.colors_list[b].detach().cpu(), smap.colors[b]), b
        assert torch.equal(pc.features_list[b].detach().cpu(), smap.ccounts[b]), b


def _assert_ring(pc, pm, t_max):
    """Rows are in creation order, so ring(k) = the number of rows created at or before step k."""
    h = pc._prune
    ring = h.ring.cpu()
    for k in range(max(h.step - 1 - t_max, 0), h.step):
        for b in range(len(pm.counts())):
            want = int((pm.created[b] <= k).sum()) if pm.created is not None else 0
            assert int(ring[k % (t_max + 2), b]) == want, (k, b)


def _slam(gs, c, t_max, margin, **kw):
    return gs.PointFusion(odom="gt", device=DEV, stable_confidence=c, max_unstable_age=t_max, free_space_margin=margin,
                          **kw)


def _steps(slam, frames, L, pc=None, s_begin=0, inplace=True):
    import gradslam_b200 as gs

    pc = gs.Pointclouds(device=DEV) if pc is None else pc
    for s in range(s_begin, L):
        pc, _ = slam.step(pc, frames[:, s], None, inplace=inplace)
    return pc


@pytest.mark.parametrize("t_max,margin", [(0, 0.1), (1, 0.0), (1, 0.1), (3, 0.0), (3, 0.1), (100, 0.05)])
def test_sequence_and_steps_match_oracle(t_max, margin):
    import gradslam_b200 as gs

    rgb, depth, K, poses, c = _scene("dynamic")
    pm = _ref("dynamic", t_max, margin)
    frames = _frames(gs, rgb, depth, K, poses)
    slam = _slam(gs, c, t_max, margin)
    whole, _ = slam(frames)
    _assert_matches(whole, pm.smap)
    _assert_ring(whole, pm, t_max)
    stepped = _steps(slam, frames, depth.shape[1])
    _assert_matches(stepped, pm.smap)
    _assert_ring(stepped, pm, t_max)


@pytest.mark.parametrize("kind", ["cameras", "edge"])
def test_cameras_and_edge_cases_match_oracle(kind):
    """A camera per element (intrinsics, skew, poses); an all-invalid frame, an element whose map stays empty and a
    camera turned away from the map."""
    import gradslam_b200 as gs

    rgb, depth, K, poses, c = _scene(kind)
    pm = _ref(kind, 1, 0.0)
    frames = _frames(gs, rgb, depth, K, poses)
    slam = _slam(gs, c, 1, 0.0)
    _assert_matches(slam(frames)[0], pm.smap)
    _assert_matches(_steps(slam, frames, depth.shape[1]), pm.smap)
    if kind == "edge":
        assert pm.counts()[1] == 0


@pytest.mark.parametrize("groups", [1, 2, 3, 4])
def test_batch_groups_match_oracle(groups, monkeypatch):
    import gradslam_b200 as gs
    from gradslam_b200 import _C

    monkeypatch.setenv("GSX_SEQ_GROUPS", str(groups))
    assert _C.lib().gsx_pointfusion_sequence_groups(5) == groups
    rgb, depth, K, poses, c = _scene("dynamic", B=5, L=7)
    pm = _ref("dynamic", 1, 0.0, B=5, L=7)
    whole, _ = _slam(gs, c, 1, 0.0)(_frames(gs, rgb, depth, K, poses))
    _assert_matches(whole, pm.smap)


def test_split_and_host_fed_calls_equal_one_device_call():
    """Pinned host frames go in calls of four frames: the second call starts at frame 4 and continues the ring."""
    import gradslam_b200 as gs

    rgb, depth, K, poses, c = _scene("dynamic")
    pm = _ref("dynamic", 3, 0.0)
    slam = _slam(gs, c, 3, 0.0)
    dev_pc, _ = slam(_frames(gs, rgb, depth, K, poses))
    host = gs.RGBDImages(rgb.pin_memory(), depth.pin_memory(), K.pin_memory(), poses.pin_memory())
    host_pc, _ = slam(host)
    _assert_matches(dev_pc, pm.smap)
    _assert_matches(host_pc, pm.smap)
    assert torch.equal(dev_pc._prune.ring, host_pc._prune.ring)


@pytest.mark.parametrize("inplace", [True, False])
def test_forward_then_steps_continue_the_history(inplace):
    import gradslam_b200 as gs

    rgb, depth, K, poses, c = _scene("dynamic")
    L = depth.shape[1]
    pm = _ref("dynamic", 1, 0.1)
    frames = _frames(gs, rgb, depth, K, poses)
    slam = _slam(gs, c, 1, 0.1)
    half, _ = slam(frames[:, : L // 2])
    out = _steps(slam, frames, L, pc=half, s_begin=L // 2, inplace=inplace)
    _assert_matches(out, pm.smap)
    if not inplace:  # the first half is untouched, history included
        assert half._prune.step == L // 2
        first, _ = fo.run_pointfusion(rgb[:, : L // 2], depth[:, : L // 2], K, poses[:, : L // 2], c_stable=c, t_max=1,
                                      margin=0.1)
        _assert_matches(half, first.smap)


def test_full_size_match_oracle():
    """640x480, B = 2: hundreds of 512-row tiles per element, violators far below the window."""
    import gradslam_b200 as gs

    shape = dict(B=2, L=5, H=480, W=640)
    rgb, depth, K, poses, c = _scene("dynamic", **shape)
    pm = _ref("dynamic", 1, 0.05, **shape)
    frames = _frames(gs, rgb, depth, K, poses)
    slam = _slam(gs, c, 1, 0.05)
    _assert_matches(slam(frames)[0], pm.smap)
    _assert_matches(_steps(slam, frames, 5), pm.smap)


def test_infinite_margin_equals_the_age_rule_entry_points():
    """margin = inf: the free-space rule of gsx_pointfusion_sequence_gt and gsx_fusion_prune gives exactly what their
    age rule alone gives, ring included."""
    import gradslam_b200 as gs

    rgb, depth, K, poses, c = _scene("dynamic")
    frames = _frames(gs, rgb, depth, K, poses)
    L = depth.shape[1]
    for run in (lambda s: s(frames)[0], lambda s: _steps(s, frames, L)):
        a, b = run(_slam(gs, c, 3, math.inf)), run(_slam(gs, c, 3, None))
        assert torch.equal(a.num_points_per_pointcloud, b.num_points_per_pointcloud)
        for key in ("points", "normals", "colors", "features"):
            for x, y in zip(getattr(a, key + "_list"), getattr(b, key + "_list")):
                assert torch.equal(x, y), key
        assert torch.equal(a._prune.ring, b._prune.ring) and a._prune.step == b._prune.step


@pytest.mark.parametrize("odom", ["icp", "gradicp"])
@pytest.mark.parametrize("association", ["nn", "projective"])
def test_icp_odometry_with_free_space(odom, association):
    import gradslam_b200 as gs

    B, L, H, W = 2, 6, 48, 64
    rgb, depth, K, poses = make_dynamic_sequence(B, L, H, W, 1, 3, seed=9, yaw0=0.6)
    icp = dict(numiters=20, dsratio=4) if association == "nn" else dict(numiters=10, dsratio=2)
    c = po.confidence_quantile(oracle.run_slam(rgb, depth, K, poses, odom="gt").map, 0.3)
    pm, ref_poses = fo.run_pointfusion(rgb, depth, K, poses, c_stable=c, t_max=1, margin=0.0, odom=odom,
                                       association=association, **icp)
    slam = gs.PointFusion(odom=odom, association=association, device=DEV, stable_confidence=c, max_unstable_age=1,
                          free_space_margin=0.0, **icp)
    pc, got_poses = slam(_frames(gs, rgb, depth, K, poses))
    torch.testing.assert_close(got_poses.cpu(), ref_poses, rtol=0, atol=1e-4)
    # bit for bit against the oracle fused and pruned at the recovered poses (a decision may flip under a pose 1e-6 away)
    _assert_matches(pc, fo.run_pointfusion(rgb, depth, K, got_poses.cpu(), c_stable=c, t_max=1, margin=0.0)[0].smap)


def test_differentiable_mode_values_and_gradients_match_oracle():
    """With depth and colours that require grad: the map equals the no-grad call bit for bit, and d(map)/d(depth,
    colours) matches the oracle's autograd, where the removal is an index_select."""
    import gradslam_b200 as gs

    B, L, H, W, t_max, margin = 2, 5, 24, 32, 1, 0.0
    rgb, depth, K, poses = make_dynamic_sequence(B, L, H, W, 1, 3, seed=41, yaw0=0.3)
    c = po.confidence_quantile(oracle.run_slam(rgb, depth, K, poses, odom="gt").map, 0.3)
    d_ref, c_ref = depth.clone().requires_grad_(True), rgb.clone().requires_grad_(True)
    pm, _ = fo.run_pointfusion(c_ref, d_ref, K, poses, c_stable=c, t_max=t_max, margin=margin)
    age, _ = po.run_pointfusion(rgb, depth, K, poses, c_stable=c, t_max=t_max)
    assert sum(pm.counts()) < sum(age.counts())
    counts = pm.counts()
    g = torch.Generator().manual_seed(5)
    ws = [[torch.randn(n, k, generator=g) for k in (3, 3, 1)] for n in counts]
    sum((t * w).sum() for b in range(B) for t, w in zip((pm.smap.points[b], pm.smap.colors[b], pm.smap.ccounts[b]),
                                                          ws[b])).backward()

    d_gpu, c_gpu = depth.clone().to(DEV).requires_grad_(True), rgb.clone().to(DEV).requires_grad_(True)
    slam = _slam(gs, c, t_max, margin)
    pc, _ = slam(gs.RGBDImages(c_gpu, d_gpu, K.to(DEV), poses.to(DEV)))
    with torch.no_grad():
        ng, _ = slam(_frames(gs, rgb, depth, K, poses))
    _assert_matches(ng, oracle.SurfelMap(*([x.detach() for x in lst] for lst in (
        pm.smap.points, pm.smap.normals, pm.smap.colors, pm.smap.ccounts))))
    assert [int(n) for n in pc.num_points_per_pointcloud.tolist()] == counts
    for b in range(B):
        for key in ("points", "normals", "colors", "features"):
            assert torch.equal(getattr(pc, key + "_list")[b].detach(), getattr(ng, key + "_list")[b]), (b, key)
    sum((t * w.to(DEV)).sum() for b in range(B) for t, w in zip((pc.points_list[b], pc.colors_list[b],
                                                                 pc.features_list[b]), ws[b])).backward()
    for got, want in ((d_gpu.grad.cpu(), d_ref.grad), (c_gpu.grad.cpu(), c_ref.grad)):
        assert torch.isfinite(got).all()
        torch.testing.assert_close(got, want, rtol=1e-3, atol=1e-4 * want.abs().max().item())


def test_box_leaves_the_gpu_map():
    import gradslam_b200 as gs

    rgb, depth, K, poses, c = _scene("dynamic")
    frames = _frames(gs, rgb, depth, K, poses)
    with_rule, _ = _slam(gs, c, 1, 0.1)(frames)
    without, _ = _slam(gs, c, 1, None)(frames)

    def in_box(pc):
        m = oracle.SurfelMap([p.cpu() for p in pc.points_list])
        return fo.rows_in_box(m, DYNAMIC_BOX_CENTER, DYNAMIC_BOX_HALF_EXTENTS, pad=0.02)

    assert in_box(with_rule) == [0, 0, 0]
    assert min(in_box(without)) > 500
