"""Argument checks of per-surfel embeddings, all raised on the host before any CUDA call: RGBDImages' and Pointclouds'
shape, D, dtype, device and layout errors; the refusal of pruning, exchange and mismatched maps; half precision in the
differentiable mode."""
import math

import pytest
import torch

import gradslam_b200 as gs
from gradslam_b200.slam import fusionutils as fu


def _frames(B=2, L=1, H=4, W=5, emb=None, channels_first=False):
    if channels_first:
        rgb, depth = torch.rand(B, L, 3, H, W), torch.rand(B, L, 1, H, W)
    else:
        rgb, depth = torch.rand(B, L, H, W, 3), torch.rand(B, L, H, W, 1)
    K = torch.eye(4).repeat(B, 1, 1, 1)
    poses = torch.eye(4).repeat(B, L, 1, 1)
    return gs.RGBDImages(rgb, depth, K, poses, channels_first=channels_first, embeddings=emb)


def test_rgbdimages_accepts_both_layouts_and_carries_the_image():
    e = torch.rand(2, 3, 4, 5, 7)
    f = _frames(L=3, emb=e)
    assert f.embeddings is e
    assert f[:, 1].embeddings.shape == (2, 1, 4, 5, 7)
    assert torch.equal(f.clone().embeddings, e) and f.clone().embeddings is not e
    assert torch.equal(f.detach().embeddings, e)
    cf = f.to_channels_first()
    assert cf.embeddings.shape == (2, 3, 7, 4, 5)
    assert torch.equal(cf.to_channels_last().embeddings, e)
    g = _frames(L=3, emb=torch.rand(2, 3, 7, 4, 5, dtype=torch.float16), channels_first=True)
    assert g.embeddings.shape == (2, 3, 7, 4, 5) and g.embeddings.dtype == torch.float16
    assert _frames(emb=torch.rand(2, 1, 4, 5, 1, dtype=torch.bfloat16)).embeddings.shape[-1] == 1


@pytest.mark.parametrize("bad, err", [
    (torch.rand(2, 1, 4, 5), ValueError),  # ndim
    (torch.rand(2, 1, 4, 6, 3), ValueError),  # W
    (torch.rand(1, 1, 4, 5, 3), ValueError),  # B
    (torch.rand(2, 1, 4, 5, 0), ValueError),  # D = 0
    (torch.rand(2, 1, 3, 4, 5), ValueError),  # channels-first layout on channels-last frames
    (torch.rand(2, 1, 4, 5, 3, dtype=torch.float64), TypeError),
    (torch.zeros(2, 1, 4, 5, 3, dtype=torch.int32), TypeError),
    ([[0.0]], TypeError),
])
def test_rgbdimages_refuses_bad_embeddings(bad, err):
    with pytest.raises(err):
        _frames(emb=bad)


def test_rgbdimages_refuses_channels_last_embeddings_on_channels_first_frames():
    with pytest.raises(ValueError):
        _frames(emb=torch.rand(2, 1, 4, 5, 3), channels_first=True)


def test_rgbdimages_refuses_embeddings_on_another_device():
    with pytest.raises(ValueError, match="same device"):
        _frames(emb=torch.rand(2, 1, 4, 5, 3, device="meta"))


def test_bilateral_filtered_frames_keep_the_embeddings():
    e = torch.rand(2, 1, 4, 5, 3)
    f = _frames(emb=e)
    # (the filter itself needs CUDA; the container keeps the image through the constructor it uses)
    kept = gs.RGBDImages(f.rgb_image, f.depth_image, f.intrinsics, f.poses, embeddings=f.embeddings)
    assert kept.embeddings is e


def test_pointclouds_embeddings_from_lists_and_tensors():
    pts = [torch.rand(3, 3), torch.rand(5, 3)]
    emb = [torch.rand(3, 4, dtype=torch.float16), torch.rand(5, 4, dtype=torch.float16)]
    pc = gs.Pointclouds(pts, embeddings=emb)
    assert pc.has_embeddings and pc.embedding_dim == 4
    assert pc.embeddings_padded.shape == (2, 5, 4) and pc.embeddings_padded.dtype == torch.float16
    assert torch.equal(pc.embeddings_list[1], emb[1])
    assert bool((pc.embeddings_padded[0, 3:] == 0).all())
    assert torch.equal(pc[1].embeddings_list[0], emb[1])
    c = pc.clone()
    assert torch.equal(c.embeddings_list[0], emb[0]) and c._emb is not pc._emb
    pc.reserve(50)
    assert pc._emb.shape == (2, 50, 4) and torch.equal(pc.embeddings_list[1], emb[1])
    pc.append_points(gs.Pointclouds(pts, embeddings=emb))
    assert torch.equal(pc.embeddings_list[0], torch.cat([emb[0], emb[0]]))
    t = gs.Pointclouds(torch.rand(2, 3, 3), embeddings=torch.rand(2, 3, 2))
    assert t.embedding_dim == 2 and not gs.Pointclouds(pts).has_embeddings
    assert gs.Pointclouds(pts).embedding_dim == 0 and gs.Pointclouds(pts).embeddings_padded is None


def test_pointclouds_embedding_setters_are_out_of_place():
    pc = gs.Pointclouds(torch.rand(2, 3, 3), embeddings=torch.rand(2, 3, 2))
    old = pc._emb
    new = torch.rand(2, 3, 6, dtype=torch.bfloat16)
    pc.embeddings_padded = new
    assert pc._emb is not old and pc.embedding_dim == 6 and torch.equal(pc.embeddings_padded, new)
    lst = [torch.rand(3, 1), torch.rand(3, 1)]
    pc.embeddings_list = lst
    assert pc.embedding_dim == 1 and torch.equal(pc.embeddings_list[1], lst[1])


@pytest.mark.parametrize("kw, err", [
    (dict(embeddings=[torch.rand(3, 4)]), ValueError),  # one list entry for two clouds
    (dict(embeddings=[torch.rand(3, 4), torch.rand(4, 4)]), ValueError),  # count
    (dict(embeddings=[torch.rand(3, 4), torch.rand(5, 2)]), ValueError),  # D differs
    (dict(embeddings=[torch.rand(3, 4), torch.rand(5, 4, dtype=torch.float16)]), ValueError),  # dtype differs
    (dict(embeddings=[torch.rand(3, 0), torch.rand(5, 0)]), ValueError),  # D = 0
    (dict(embeddings=[torch.rand(3, 4).double(), torch.rand(5, 4).double()]), TypeError),
    (dict(embeddings=torch.rand(2, 5, 4)), TypeError),  # a tensor beside a list of points
])
def test_pointclouds_refuses_bad_embeddings(kw, err):
    with pytest.raises(err):
        gs.Pointclouds([torch.rand(3, 3), torch.rand(5, 3)], **kw)


def test_pointclouds_refuses_bad_tensor_embeddings_and_mismatched_appends():
    with pytest.raises(ValueError):
        gs.Pointclouds(torch.rand(2, 3, 3), embeddings=torch.rand(2, 4, 2))
    with pytest.raises(TypeError):  # as normals / colours without points
        gs.Pointclouds(embeddings=torch.rand(2, 4, 2))
    a = gs.Pointclouds([torch.rand(3, 3)], embeddings=[torch.rand(3, 2)])
    for other in (gs.Pointclouds([torch.rand(3, 3)]), gs.Pointclouds([torch.rand(3, 3)], embeddings=[torch.rand(3, 5)])):
        with pytest.raises(ValueError, match="embeddings"):
            a.append_points(other)


def _map_with(emb):
    pts = [torch.rand(3, 3), torch.rand(3, 3)]
    return gs.Pointclouds(pts, normals=[torch.rand(3, 3)] * 2, colors=[torch.rand(3, 3)] * 2,
                          features=[torch.rand(3, 1)] * 2, embeddings=emb)


@pytest.mark.parametrize("map_emb, frame_emb", [
    ([torch.rand(3, 4)] * 2, None),  # the map has embeddings, the frame none
    (None, torch.rand(2, 1, 4, 5, 4)),  # the other way round
    ([torch.rand(3, 4)] * 2, torch.rand(2, 1, 4, 5, 3)),  # D differs
    ([torch.rand(3, 4)] * 2, torch.rand(2, 1, 4, 5, 4, dtype=torch.float16)),  # dtype differs
])
def test_map_updates_refuse_mismatched_embeddings(map_emb, frame_emb):
    pc, f = _map_with(map_emb), _frames(emb=frame_emb)
    table = torch.empty((0, 4), dtype=torch.int64)
    for call in (lambda: fu.update_map_fusion(pc, f, 0.05, 0.9, 0.6),
                 lambda: fu.fuse_with_map(pc, f, table, 0.6)):
        with pytest.raises(ValueError, match="embeddings"):
            call()


def test_aggregate_refuses_mismatched_embeddings():
    pts = gs.Pointclouds([torch.rand(3, 3)] * 2, normals=[torch.rand(3, 3)] * 2, colors=[torch.rand(3, 3)] * 2,
                         embeddings=[torch.rand(3, 4)] * 2)
    with pytest.raises(ValueError, match="embeddings"):
        fu.update_map_aggregate(pts, _frames())


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_half_embeddings_refuse_the_differentiable_mode(dtype):
    f = _frames(emb=torch.rand(2, 1, 4, 5, 3, dtype=dtype).requires_grad_(True))
    with pytest.raises(TypeError, match="float32"):
        fu.update_map_fusion(gs.Pointclouds(), f, 0.05, 0.9, 0.6)
    g = _frames(emb=torch.rand(2, 1, 4, 5, 3, dtype=dtype))
    g.depth_image.requires_grad_(True)
    with pytest.raises(TypeError, match="float32"):
        fu.update_map_aggregate(gs.Pointclouds(), g)


def test_pruning_and_exchange_refuse_embeddings():
    pc = _map_with([torch.rand(3, 4)] * 2)
    with pytest.raises(ValueError, match="embeddings"):
        fu.prune_unstable(pc, 0.5, 3)
    with pytest.raises(ValueError, match="embeddings"):
        fu.fuse_and_prune(pc, _frames(emb=torch.rand(2, 1, 4, 5, 4)), 0.05, 0.9, 0.6, 0.5, 3, math.inf)
    with pytest.raises(ValueError, match="embeddings"):
        fu.fuse_and_prune(gs.Pointclouds(), _frames(emb=torch.rand(2, 1, 4, 5, 4)), 0.05, 0.9, 0.6, 0.5, 3, 0.1)
    from gradslam_b200 import parallel

    with pytest.raises(ValueError, match="embeddings"):
        parallel.gather_maps_begin(pc)


@pytest.mark.parametrize("kw", [dict(stable_confidence=0.5, max_unstable_age=3),
                                dict(stable_confidence=0.5, max_unstable_age=3, free_space_margin=0.1),
                                dict(stable_confidence=0.0, max_unstable_age=3, surfel_radii=True,
                                     merge_overlapping=True)])
def test_pointfusion_pruning_options_refuse_frames_with_embeddings(kw):
    slam = gs.PointFusion(odom="gt", device="cpu", **kw)
    f = _frames(L=2, emb=torch.rand(2, 2, 4, 5, 3))
    with pytest.raises(ValueError, match="embeddings"):
        slam(f)
    with pytest.raises(ValueError, match="embeddings"):
        slam.step(gs.Pointclouds(), f[:, 0])
