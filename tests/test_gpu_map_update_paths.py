"""The argument errors of the fused map update and of pruning (update_map_fusion, fuse_and_prune, prune_unstable), in the
in-place mode and in the differentiable mode that inputs requiring grad select: both modes reject the same inputs with
the same exception, and a max_unstable_age mismatch leaves the map, its sizes and its pruning history untouched."""
import pytest
import torch

from gradslam_b200.synthetic import make_sequence

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
DIST_TH, DOT_TH, SIGMA, C_STABLE, MARGIN = 0.05, 0.94, 0.6, 0.5, 0.05


def _frames(grad, poses=True):
    import gradslam_b200 as gs

    rgb, depth, K, P = make_sequence(2, 2, 24, 32, seed=3)
    rgb, depth = rgb.to(DEV).requires_grad_(grad), depth.to(DEV).requires_grad_(grad)
    return gs.RGBDImages(rgb, depth, K.to(DEV), P.to(DEV) if poses else None)


def _map(frames, features="one"):
    """A fused map of frame 0 (it requires grad when the frames do); features "none" / "two": the same rows rebuilt
    without features, or with two feature channels."""
    import gradslam_b200 as gs
    from gradslam_b200.slam import fusionutils as fu

    pc = fu.update_map_fusion(gs.Pointclouds(device=DEV), frames[:, 0], DIST_TH, DOT_TH, SIGMA)
    if features == "one":
        return pc
    f = pc.features_padded
    return gs.Pointclouds(pc.points_padded, pc.normals_padded, pc.colors_padded,
                          None if features == "none" else torch.cat([f, f], -1))


def _update(pc, frames, t_max=1, inplace=False):
    from gradslam_b200.slam import fusionutils as fu

    return fu.update_map_fusion(pc, frames[:, 1], DIST_TH, DOT_TH, SIGMA, inplace=inplace)


def _fuse_and_prune(pc, frames, t_max=1, inplace=False):
    from gradslam_b200.slam import fusionutils as fu

    return fu.fuse_and_prune(pc, frames[:, 1], DIST_TH, DOT_TH, SIGMA, C_STABLE, t_max, MARGIN, inplace=inplace)


def _prune(pc, frames, t_max=1, inplace=True):
    from gradslam_b200.slam import fusionutils as fu

    return fu.prune_unstable(pc, C_STABLE, t_max)


@pytest.mark.parametrize("grad", [False, True])
@pytest.mark.parametrize("op", [_update, _fuse_and_prune])
def test_frame_without_poses(op, grad):
    import gradslam_b200 as gs

    with pytest.raises(ValueError, match="rgbdimages must have poses for map fusion"):
        op(gs.Pointclouds(device=DEV), _frames(grad, poses=False))


@pytest.mark.parametrize("grad", [False, True])
@pytest.mark.parametrize("op,features,message", [
    (_update, "none", "Pointclouds must have features for map fusion"),
    (_update, "two", "features must be a single confidence count per point for map fusion"),
    (_fuse_and_prune, "none", "pruning needs maps with colours and a confidence count per point"),
    (_fuse_and_prune, "two", "pruning needs maps with colours and a confidence count per point"),
    (_prune, "none", "pruning needs maps with colours and a confidence count per point"),
    (_prune, "two", "pruning needs maps with colours and a confidence count per point"),
])
def test_map_without_one_confidence_channel(op, features, message, grad):
    frames = _frames(grad)
    pc = _map(frames, features)
    assert any(t.requires_grad for t in pc._grad_tensors()) == grad
    with pytest.raises(ValueError, match=message):
        op(pc, frames)


@pytest.mark.parametrize("grad", [False, True])
@pytest.mark.parametrize("op,inplace", [(_fuse_and_prune, False), (_fuse_and_prune, True), (_prune, True)])
def test_max_unstable_age_mismatch_leaves_the_map_untouched(op, inplace, grad):
    frames = _frames(grad)
    pc = _map(frames)
    pc = op(pc, frames, t_max=1, inplace=True)  # the map's first pruned step: history with max_unstable_age 1
    assert pc._prune is not None and pc._prune.t_max == 1 and pc._prune.step == 1
    counts = pc.num_points_per_pointcloud.clone()
    ring = pc._prune.ring.clone()
    rows = [getattr(pc, k + "_padded").detach().clone() for k in ("points", "normals", "colors", "features")]
    with pytest.raises(ValueError, match=r"max_unstable_age \(2\) differs from the one this map was pruned with \(1\)"):
        op(pc, frames, t_max=2, inplace=inplace)
    assert torch.equal(pc.num_points_per_pointcloud, counts)
    assert torch.equal(pc._prune.ring, ring) and pc._prune.step == 1
    for k, want in zip(("points", "normals", "colors", "features"), rows):
        assert torch.equal(getattr(pc, k + "_padded").detach(), want), k
