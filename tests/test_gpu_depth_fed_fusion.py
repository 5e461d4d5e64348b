"""Oracle parity of the depth-fed fusion path, where K1r stores nothing per pixel and K2 / K4 re-evaluate each pixel's
world vertex, world normal and confidence weight from its depth stencil.  The cases aim at what that re-evaluation can
get wrong: the camera of the right element (a camera per element, skew and 4th intrinsics column), the last column and
row, which take their neighbour's difference (W % 4 != 0, (H - 1) % 8 == 0, H or W = 2), holes on a lattice and pixels
whose right and lower neighbours are both holes (the normal is the cross product's rounding residue there), several K2
grid-stride passes, batch groups, chunked host-fed calls, and the differentiable mode, which packs caller-supplied maps
instead and must give the same maps.  Every case runs the whole-sequence call and the per-frame step API."""
import pytest
import torch

import gsx_oracle as oracle
from cameras import camera_inputs
from gradslam_b200.synthetic import make_sequence, punch_lattice_holes

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _partners(n):
    """Index of the pixel each pixel along an axis of length n takes its difference with: the next one, the previous
    one for the last."""
    i = torch.arange(n)
    return torch.where(i < n - 1, i + 1, i - 1)


def _punch_corner_holes(depth):
    """Zeroes both difference partners (right / left in the last column, lower / upper in the last row) of a lattice of
    pixels that includes the last row and column, so that the cancelling cross product is reached everywhere."""
    depth = depth.clone()
    H, W = depth.shape[2], depth.shape[3]
    pw, ph = _partners(W), _partners(H)
    for h in list(range(1, H - 1, 6)) + [H - 1]:
        for w in list(range(2, W - 1, 9)) + [W - 1]:
            depth[:, :, h, int(pw[w])] = 0.0
            depth[:, :, int(ph[h]), w] = 0.0
    return depth


def _inputs(B, L, H, W, kind, seed=7):
    if kind == "cameras":
        return camera_inputs(B, L, H, W, seed, skew=0.75)
    if kind == "camera_lattice":
        return camera_inputs(B, L, H, W, seed, skew=0.75, lattice_holes=True)
    rgb, depth, K, poses = make_sequence(B, L, H, W, seed=seed)
    if kind == "lattice":
        depth = punch_lattice_holes(depth)
    elif kind == "corner_holes":
        depth = _punch_corner_holes(depth)
    return rgb, depth, K, poses


_ref_cache = {}


def _case(B, L, H, W, kind):
    key = (B, L, H, W, kind)
    if key not in _ref_cache:
        rgb, depth, K, poses = _inputs(B, L, H, W, kind)
        _ref_cache[key] = (rgb, depth, K, poses, oracle.run_slam(rgb, depth, K, poses, odom="gt").map)
    return _ref_cache[key]


def _frames(gs, rgb, depth, K, poses):
    return gs.RGBDImages(rgb.to(DEV), depth.to(DEV), K.to(DEV), poses.to(DEV))


def _assert_matches_oracle(pc, ref_map):
    assert [int(c) for c in pc.num_points_per_pointcloud.tolist()] == ref_map.counts()
    for b in range(len(ref_map.counts())):
        assert torch.equal(pc.points_list[b].detach().cpu(), ref_map.points[b]), b
        assert torch.equal(pc.normals_list[b].detach().cpu(), ref_map.normals[b]), b
        assert torch.equal(pc.colors_list[b].detach().cpu(), ref_map.colors[b]), b
        assert torch.equal(pc.features_list[b].detach().cpu(), ref_map.ccounts[b]), b


def _sequence_and_steps(gs, frames, L):
    slam = gs.PointFusion(odom="gt", device=DEV)
    whole, _ = slam(frames)
    pc = gs.Pointclouds(device=DEV)
    for s in range(L):
        pc, _ = slam.step(pc, frames[:, s], None, inplace=True)
    return whole, pc


SHAPES = [
    ((3, 4, 48, 64), "cameras"),
    ((3, 3, 48, 64), "camera_lattice"),
    ((2, 3, 33, 47), "corner_holes"),   # W % 4 != 0, odd H * W
    ((2, 3, 41, 64), "corner_holes"),   # (H - 1) % 8 == 0
    ((2, 3, 41, 47), "lattice"),
    ((2, 3, 2, 40), "random"),          # H = 2: every row takes the other row's difference
    ((2, 3, 36, 2), "random"),          # W = 2
    ((2, 3, 2, 2), "random"),
]


@pytest.mark.parametrize("shape,kind", SHAPES, ids=["x".join(map(str, s)) + "-" + k for s, k in SHAPES])
def test_depth_fed_fusion_matches_oracle(shape, kind):
    import gradslam_b200 as gs

    B, L, H, W = shape
    rgb, depth, K, poses, ref = _case(B, L, H, W, kind)
    whole, steps = _sequence_and_steps(gs, _frames(gs, rgb, depth, K, poses), L)
    _assert_matches_oracle(whole, ref)
    _assert_matches_oracle(steps, ref)


def test_corner_holes_reach_the_residue_case():
    """The corner-hole inputs really contain valid pixels whose right and lower neighbours are both holes, also in the
    last column and the last row."""
    for H, W in ((33, 47), (41, 64)):
        d = _inputs(2, 3, H, W, "corner_holes")[1][..., 0] > 0
        both = d & ~d[:, :, :, _partners(W)] & ~d[:, :, _partners(H), :]
        assert both.any()
        assert both[..., :, W - 1].any() and both[..., H - 1, :].any()


@pytest.fixture
def k2_grid_cap():
    from gradslam_b200 import _C

    yield _C.lib().gsx_debug_set_k2_grid_cap
    _C.lib().gsx_debug_set_k2_grid_cap(0)


def test_k2_several_passes_match_oracle(k2_grid_cap):
    import gradslam_b200 as gs

    B, L, H, W = 3, 4, 48, 64
    rgb, depth, K, poses, ref = _case(B, L, H, W, "cameras")
    frames = _frames(gs, rgb, depth, K, poses)
    for cap in (1, 3, 7):
        k2_grid_cap(cap)
        whole, steps = _sequence_and_steps(gs, frames, L)
        _assert_matches_oracle(whole, ref)
        _assert_matches_oracle(steps, ref)


@pytest.mark.parametrize("groups", [1, 2, 3, 4])
def test_batch_groups_match_oracle(groups, monkeypatch):
    """Each group's K1r of frame s+1 runs beside K2 / K4 of frame s with the other workspace half, so the header of
    each half must point at its own frame's depth."""
    import gradslam_b200 as gs
    from gradslam_b200 import _C

    monkeypatch.setenv("GSX_SEQ_GROUPS", str(groups))
    assert _C.lib().gsx_pointfusion_sequence_groups(5) == groups
    rgb, depth, K, poses, ref = _case(5, 5, 48, 64, "cameras")
    whole, steps = _sequence_and_steps(gs, _frames(gs, rgb, depth, K, poses), 5)
    _assert_matches_oracle(whole, ref)
    _assert_matches_oracle(steps, ref)


def test_host_fed_chunked_calls_match_oracle():
    """Pinned host frames are uploaded four frames at a time: L = 6 makes two sequence calls, the second starting at
    frame 4 into the buffer the copies are still filling."""
    import gradslam_b200 as gs

    rgb, depth, K, poses, ref = _case(3, 6, 48, 64, "cameras")
    host = gs.RGBDImages(rgb.pin_memory(), depth.pin_memory(), K.pin_memory(), poses.pin_memory())
    assert not host.depth_image.is_cuda
    pc, out_poses = gs.PointFusion(odom="gt", device=DEV)(host)
    _assert_matches_oracle(pc, ref)
    assert torch.equal(out_poses.cpu(), poses)


def test_differentiable_mode_equals_no_grad_and_oracle():
    """With a depth that requires grad the frame records are packed from the materialised maps (the per-pixel
    records K1r still writes in that mode); the maps equal the no-grad call's and the oracle's, and a gradient flows."""
    import gradslam_b200 as gs

    B, L, H, W = 3, 3, 48, 64
    rgb, depth, K, poses, ref = _case(B, L, H, W, "camera_lattice")
    no_grad, _ = gs.PointFusion(odom="gt", device=DEV)(_frames(gs, rgb, depth, K, poses))
    d = depth.to(DEV).requires_grad_(True)
    frames = gs.RGBDImages(rgb.to(DEV), d, K.to(DEV), poses.to(DEV))
    pc, _ = gs.PointFusion(odom="gt", device=DEV)(frames)
    _assert_matches_oracle(pc, ref)
    counts = [int(c) for c in pc.num_points_per_pointcloud.tolist()]
    assert counts == [int(c) for c in no_grad.num_points_per_pointcloud.tolist()]
    for b, n in enumerate(counts):
        assert torch.equal(pc._geo[b, :n].detach(), no_grad._geo[b, :n]), b
        assert torch.equal(pc._col[b, :n].detach(), no_grad._col[b, :n]), b
    pc.points_padded.sum().backward()
    assert d.grad is not None and torch.isfinite(d.grad).all()
