"""Surfel radii on the GPU (PointFusion(surfel_radii=True)): all eight geometry slots and the colour rows bit for bit
against the CPU oracle (tests/radii_oracle.py) on the whole-sequence driver in 1..4 batch groups and on the step API,
with a camera per element and past the 64-frame header block, with the age and free-space rules; slots 0-6 and the
colours equal a run without radii; the differentiable mode's radii and their (zero) gradient."""
import math

import pytest
import torch

import radii_oracle as ro
from cameras import camera_inputs
from gradslam_b200.synthetic import make_dynamic_sequence, make_sequence

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
DIST_TH, SIGMA = 0.05, 0.6
DOT_TH = math.cos(20 * math.pi / 180)
L = 70  # past one 64-frame block of frame headers

_cache = {}


def _cached(key, make):
    if key not in _cache:
        _cache[key] = make()
    return _cache[key]


def _frames(gs, rgb, depth, K, poses):
    return gs.RGBDImages(rgb.to(DEV), depth.to(DEV), K.to(DEV), poses.to(DEV))


def _assert_matches(pc, smap, radii):
    assert [int(c) for c in pc.num_points_per_pointcloud.tolist()] == smap.counts()
    for b in range(len(smap.counts())):
        assert torch.equal(pc.points_list[b].detach().cpu(), smap.points[b]), b
        assert torch.equal(pc.normals_list[b].detach().cpu(), smap.normals[b]), b
        assert torch.equal(pc.colors_list[b].detach().cpu(), smap.colors[b]), b
        assert torch.equal(pc.features_list[b].detach().cpu(), smap.ccounts[b]), b
        assert torch.equal(pc.radii_list[b].detach().cpu(), radii[b]), b
        assert bool((radii[b] > 0).all())


def _assert_same_but_radii(a, b):
    """slots 0-6 of the geometry rows and the colour rows equal; b has no radii."""
    ca, cb = a._host_counts(), b._host_counts()
    assert ca == cb
    for i, n in enumerate(ca):
        assert torch.equal(a._geo[i, :n, :7], b._geo[i, :n, :7]), i
        assert torch.equal(a._col[i, :n], b._col[i, :n]), i
        assert bool((b._geo[i, :n, 7] == 0).all()), i
        assert bool((a._geo[i, :n, 7] > 0).all()), i


def _steps(slam, frames):
    import gradslam_b200 as gs

    pc = gs.Pointclouds(device=DEV)
    for s in range(frames.shape[1]):
        pc, _ = slam.step(pc, frames[:, s], None, inplace=True)
    return pc


def _camera_case():
    """B = 5 elements, each with its own intrinsics and trajectory, 70 frames, and the oracle's map and radii."""
    def make():
        rgb, depth, K, poses = camera_inputs(5, L, 24, 32, seed=61)
        pm, radii = ro.run_pointfusion(rgb, depth, K, poses)
        return rgb, depth, K, poses, pm, radii

    return _cached("camera", make)


@pytest.mark.parametrize("groups", [1, 2, 3, 4])
def test_whole_sequence_with_radii_matches_oracle_in_batch_groups(groups, monkeypatch):
    import gradslam_b200 as gs

    monkeypatch.setenv("GSX_SEQ_GROUPS", str(groups))
    rgb, depth, K, poses, pm, radii = _camera_case()
    assert len(set(K[:, 0, 0, 0].tolist())) == 5  # a camera per element
    frames = _frames(gs, rgb, depth, K, poses)
    pc, _ = gs.PointFusion(odom="gt", device=DEV, surfel_radii=True)(frames)
    _assert_matches(pc, pm.smap, radii)
    off, _ = gs.PointFusion(odom="gt", device=DEV)(frames)
    _assert_same_but_radii(pc, off)


def test_step_api_with_radii_matches_oracle_and_the_run_without():
    import gradslam_b200 as gs

    rgb, depth, K, poses, pm, radii = _camera_case()
    frames = _frames(gs, rgb, depth, K, poses)
    pc = _steps(gs.PointFusion(odom="gt", device=DEV, surfel_radii=True), frames)
    _assert_matches(pc, pm.smap, radii)
    _assert_same_but_radii(pc, _steps(gs.PointFusion(odom="gt", device=DEV), frames))


def test_update_map_fusion_and_fuse_with_map_take_the_option():
    """The fusionutils calls that end in K4: update_map_fusion, and fuse_with_map on the reference's correspondence
    table, give the sequence's radii frame by frame."""
    import gradslam_b200 as gs
    from gradslam_b200.slam import fusionutils as fu

    rgb, depth, K, poses = make_sequence(2, 4, 24, 32, seed=62)
    _, radii = ro.run_pointfusion(rgb, depth, K, poses)
    frames = _frames(gs, rgb, depth, K, poses)
    a, b = gs.Pointclouds(device=DEV), gs.Pointclouds(device=DEV)
    for s in range(4):
        a = fu.update_map_fusion(a, frames[:, s], DIST_TH, DOT_TH, SIGMA, surfel_radii=True)
        table = fu.find_correspondences(b, frames[:, s], DIST_TH, DOT_TH) if b.has_points else \
            torch.empty((0, 4), dtype=torch.int64, device=DEV)
        b = fu.fuse_with_map(b, frames[:, s], table, SIGMA, surfel_radii=True)
    for pc in (a, b):
        for i in range(2):
            assert torch.equal(pc.radii_list[i].cpu(), radii[i]), i
    with pytest.raises(TypeError, match="surfel_radii"):
        fu.update_map_fusion(a, frames[:, 0], DIST_TH, DOT_TH, SIGMA, surfel_radii=1)


@pytest.mark.parametrize("kind", ["age", "free_space"])
def test_pruned_runs_with_radii_match_oracle(kind):
    """The age rule alone, and with the free-space rule: pruning moves whole rows, radius included, on the sequence
    driver and on the step API (fuse_and_prune)."""
    import gradslam_b200 as gs

    def make():
        if kind == "age":
            rgb, depth, K, poses = make_sequence(3, L, 48, 64, seed=7)
            margin = None
        else:
            rgb, depth, K, poses = make_dynamic_sequence(3, L, 48, 64, seed=5, k0=30, k1=44,
                                                         box_center=(1.5, 0.4, 1.35), box_half_extents=(0.2, 0.2, 0.2))
            margin = 0.05
        pm0, _ = ro.run_pointfusion(rgb, depth, K, poses)
        c = float(torch.quantile(torch.cat([x[:, 0] for x in pm0.smap.ccounts]).double(), 0.4, interpolation="lower"))
        pm, radii = ro.run_pointfusion(rgb, depth, K, poses, c_stable=c, t_max=3, margin=margin)
        assert sum(pm.smap.counts()) < sum(pm0.smap.counts())
        return rgb, depth, K, poses, c, margin, pm, radii

    rgb, depth, K, poses, c, margin, pm, radii = _cached(("pruned", kind), make)
    frames = _frames(gs, rgb, depth, K, poses)
    kw = dict(odom="gt", device=DEV, stable_confidence=c, max_unstable_age=3, free_space_margin=margin)
    slam = gs.PointFusion(surfel_radii=True, **kw)
    whole, _ = slam(frames)
    _assert_matches(whole, pm.smap, radii)
    _assert_matches(_steps(slam, frames), pm.smap, radii)
    off, _ = gs.PointFusion(**kw)(frames)
    _assert_same_but_radii(whole, off)


def test_differentiable_mode_gives_the_fused_radii_and_no_gradient_through_them():
    import gradslam_b200 as gs

    rgb, depth, K, poses = make_sequence(2, 3, 24, 32, seed=63)
    fused = _steps(gs.PointFusion(odom="gt", device=DEV, surfel_radii=True), _frames(gs, rgb, depth, K, poses))
    grads = {}
    for radii in (True, False):
        d = depth.to(DEV).requires_grad_(True)
        frames = gs.RGBDImages(rgb.to(DEV), d, K.to(DEV), poses.to(DEV))
        pc = _steps(gs.PointFusion(odom="gt", device=DEV, surfel_radii=radii), frames)
        assert pc.points_padded.requires_grad
        if radii:
            assert pc.radii_padded.requires_grad
            for i in range(2):
                assert torch.equal(pc.radii_list[i].detach(), fused.radii_list[i]), i
            g, = torch.autograd.grad(pc.radii_padded.sum(), d, allow_unused=True)
            assert g is None or bool((g == 0).all())
        grads[radii], = torch.autograd.grad(pc.points_padded.sum() + pc.features_padded.sum(), d)
    assert torch.equal(grads[True], grads[False])
