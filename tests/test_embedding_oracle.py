"""The embedding oracle (tests/embedding_oracle.py) on the CPU: it leaves gsx_oracle's map as it is, fuses e := rgb into
the colours bit for bit, and rounds a half-precision map after every frame."""
import pytest
import torch

import embedding_oracle as eo
import gsx_oracle as oracle
from gradslam_b200.synthetic import make_sequence


@pytest.fixture(scope="module")
def seq():
    return make_sequence(2, 4, 24, 32, seed=71)


def _same_map(a, b):
    assert a.counts() == b.counts()
    for x, y in ((a.points, b.points), (a.normals, b.normals), (a.colors, b.colors), (a.ccounts, b.ccounts)):
        assert (x is None) == (y is None)
        for i in range(0 if x is None else len(x)):
            assert torch.equal(x[i], y[i])


def test_restated_oracle_keeps_the_map_bit_for_bit(seq):
    rgb, depth, K, poses = seq
    smap, emb = eo.run_pointfusion(rgb, depth, K, poses, eo.random_embeddings(2, 4, 24, 32, 5, seed=1))
    _same_map(smap, oracle.run_slam(rgb, depth, K, poses, odom="gt").map)
    assert [int(e.shape[0]) for e in emb] == smap.counts()
    assert all(e.shape[1] == 5 and e.dtype == torch.float32 for e in emb)
    assert sum(smap.counts()) < int((depth > 0).sum())  # the frames do merge into earlier surfels


def test_rgb_as_embedding_equals_the_colours(seq):
    rgb, depth, K, poses = seq
    smap, emb = eo.run_pointfusion(rgb, depth, K, poses, rgb.clone())
    for i in range(2):
        assert torch.equal(emb[i], smap.colors[i])
    agg, emb = eo.run_aggregate(rgb, depth, K, poses, rgb.clone())
    _same_map(agg, oracle.run_slam(rgb, depth, K, poses, odom="gt", mode="aggregate").map)
    for i in range(2):
        assert torch.equal(emb[i], agg.colors[i])


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_half_map_is_rounded_after_every_frame(seq, dtype):
    """A half map equals a float32 map whose values are rounded to the storage dtype after every frame; rounding only
    at the end gives another map."""
    rgb, depth, K, poses = seq
    e = eo.random_embeddings(2, 4, 24, 32, 3, dtype=dtype, seed=2)
    _, half = eo.run_pointfusion(rgb, depth, K, poses, e)
    smap, per_frame, at_end = oracle.SurfelMap(), None, None
    for s in range(4):
        pose = poses[:, s]
        maps = oracle.frame_maps(depth[:, s:s + 1], K, pose.unsqueeze(1))
        table = oracle.find_correspondences(smap, maps, pose, K[:, 0], 0.05, eo.math.cos(20 * eo.math.pi / 180))
        ef = e[:, s:s + 1].float()
        _, per_frame = eo.fuse_with_map(smap, per_frame, maps, rgb[:, s:s + 1], ef, table, 0.6)
        per_frame = [x.to(dtype).float() for x in per_frame]
        smap, at_end = eo.fuse_with_map(smap, at_end, maps, rgb[:, s:s + 1], ef, table, 0.6)
    for i in range(2):
        assert half[i].dtype == dtype
        assert torch.equal(half[i], per_frame[i].to(dtype))
    assert any(not torch.equal(half[i], at_end[i].to(dtype)) for i in range(2))
