"""CPU checks of the free-space-violation oracle (tests/free_space_oracle.py): PointFusion's free_space_margin keyword
errors, the rule's limit (margin = inf is the age rule alone), a hand-built case at the margin's edge, agreement of
the positional ring update with the creation-step formulation, and the dynamic scene's box leaving the map."""
import math

import pytest
import torch

import gsx_oracle as oracle
import free_space_oracle as fo
import prune_oracle as po
import gradslam_b200 as gs
from gradslam_b200.synthetic import DYNAMIC_BOX_CENTER, DYNAMIC_BOX_HALF_EXTENTS, intrinsics, make_dynamic_sequence

F32 = torch.float32


@pytest.mark.parametrize("kw,exc", [
    (dict(free_space_margin=0.1), ValueError),  # without the age rule's keywords
    (dict(stable_confidence=1.0, max_unstable_age=2, free_space_margin="0.1"), TypeError),
    (dict(stable_confidence=1.0, max_unstable_age=2, free_space_margin=True), TypeError),
    (dict(stable_confidence=1.0, max_unstable_age=2, free_space_margin=-0.01), ValueError),
    (dict(stable_confidence=1.0, max_unstable_age=2, free_space_margin=math.nan), ValueError),
    (dict(stable_confidence=1.0, max_unstable_age=2, free_space_margin=-math.inf), ValueError),
])
def test_keyword_errors(kw, exc):
    with pytest.raises(exc):
        gs.PointFusion(odom="gt", device="cpu", **kw)


def test_keyword_accepted_and_off_by_default():
    assert gs.PointFusion(odom="gt", device="cpu").free_space_margin is None
    for m in (0, 0.05, math.inf):
        slam = gs.PointFusion(odom="gt", device="cpu", stable_confidence=1e-6, max_unstable_age=2, free_space_margin=m)
        assert slam.free_space_margin == m
    with pytest.raises(TypeError):
        gs.ICPSLAM(odom="gt", device="cpu", free_space_margin=0.1)


_inputs = {}


def _dynamic(B=2, L=10, H=48, W=64, k0=2, k1=5, seed=5):
    key = (B, L, H, W, k0, k1, seed)
    if key not in _inputs:
        _inputs[key] = make_dynamic_sequence(B, L, H, W, k0, k1, seed=seed)
    return _inputs[key]


def _assert_same_map(a, b):
    assert a.counts() == b.counts()
    for x, y in ((a.points, b.points), (a.normals, b.normals), (a.colors, b.colors), (a.ccounts, b.ccounts)):
        for u, v in zip(x, y):
            assert torch.equal(u, v)


@pytest.mark.parametrize("t_max", [0, 1, 3])
def test_infinite_margin_equals_the_age_rule(t_max):
    rgb, depth, K, poses = _dynamic()
    c = po.confidence_quantile(oracle.run_slam(rgb, depth, K, poses, odom="gt").map, 0.3)
    want, _ = po.run_pointfusion(rgb, depth, K, poses, c_stable=c, t_max=t_max)
    got, _ = fo.run_pointfusion(rgb, depth, K, poses, c_stable=c, t_max=t_max, margin=math.inf)
    _assert_same_map(got.smap, want.smap)
    assert all(torch.equal(x, y) for x, y in zip(got.created, want.created))


def test_hand_built_margin_edge():
    """Camera at the world origin; every row on the optical axis projects to the same pixel.  A stable wall row at z = 3
    is merged there; with margin 0.5 the bound is 2.5: a row at exactly 2.5 is kept, the float just below it and a box
    row at 1.5 are removed, a row behind the wall is kept.  An unstable merged row gives no bound; an unmerged pixel
    neither."""
    H, W = 48, 64
    K = torch.from_numpy(intrinsics(H, W).astype("float32")).unsqueeze(0)
    pose = torch.eye(4).unsqueeze(0)
    z = [3.0, 1.5, 2.5, float(torch.nextafter(torch.tensor(2.5), torch.tensor(0.0))), 3.5]
    pts = torch.tensor([[0.0, 0.0, v] for v in z], dtype=F32)
    cc = torch.tensor([[2.0], [5.0], [0.1], [0.1], [0.1]], dtype=F32)
    smap = oracle.SurfelMap([pts], [pts.clone()], [pts.clone()], [cc])
    u, v, _ = oracle.project_map(pts.unsqueeze(0), pose, K)
    h, w = int(v[0, 0].round()), int(u[0, 0].round())
    table = torch.tensor([[0, 0, h, w]])
    bound = fo.bound_image(smap, table, pose, K, H, W, 1.0)
    assert float(bound[0, h, w]) == 3.0 and int(torch.isfinite(bound).sum()) == 1
    assert fo.violators(smap, bound, pose, K, 0.5)[0].tolist() == [False, True, False, True, False]
    assert fo.violators(smap, bound, pose, K, math.inf)[0].tolist() == [False] * 5
    assert int(torch.isfinite(fo.bound_image(smap, table, pose, K, H, W, 2.5)).sum()) == 0  # wall not stable
    pm = po.PrunedMap(smap)
    keep = fo.prune_step(pm, 1.0, 5, fo.violators(smap, bound, pose, K, 0.5))  # (no row is old enough for the age rule)
    assert keep[0].tolist() == [0, 2, 4]  # the box row is stable, but in front
    assert pm.smap.points[0][:, 2].tolist() == [3.0, 2.5, 3.5]


def _random_run(seed, t_max, steps=12, Bn=3):
    """Random appends, merges, thresholds and violators inside, below and above the age window: the positional ring
    update equals the creation-step formulation."""
    g = torch.Generator().manual_seed(seed)
    base = oracle.SurfelMap([torch.rand(int(torch.randint(0, 5, (1,), generator=g)), 3, generator=g) for _ in range(Bn)],
                            None, None, None)
    base.normals = [p.clone() for p in base.points]
    base.colors = [p.clone() for p in base.points]
    base.ccounts = [torch.rand(p.shape[0], 1, generator=g) for p in base.points]
    pm, ring_map, ring = po.PrunedMap(base.clone()), base.clone(), fo.PositionalRingPruner(Bn, t_max)
    where = set()
    for _ in range(steps):
        merges = [torch.rand(p.shape[0], 1, generator=g) * (torch.rand(p.shape[0], 1, generator=g) < 0.3)
                  for p in pm.smap.points]
        new = [torch.rand(int(torch.randint(0, 6, (1,), generator=g)), 3, generator=g) for _ in range(Bn)]
        new_cc = [torch.rand(p.shape[0], 1, generator=g) for p in new]
        for m in (pm.smap, ring_map):
            for b in range(Bn):
                m.ccounts[b] = m.ccounts[b] + merges[b]
            m.append(oracle.SurfelMap([p.clone() for p in new], [p.clone() for p in new], [p.clone() for p in new],
                                      [c.clone() for c in new_cc]))
        extra = [torch.rand(p.shape[0], generator=g) < 0.15 for p in pm.smap.points]
        s = pm.step
        for b in range(Bn):  # where the violators lie relative to this step's window (creation step s - t_max)
            if pm.created is not None and extra[b].any():
                cr = torch.cat([pm.created[b], torch.full((extra[b].numel() - pm.created[b].numel(),), s)])[extra[b]]
                where |= {"below" if x < s - t_max else "inside" if x == s - t_max else "above" for x in cr.tolist()}
        c_stable = float(torch.rand(1, generator=g)) * 1.5
        fo.prune_step(pm, c_stable, t_max, extra)
        ring(ring_map, c_stable, extra)
        _assert_same_map(pm.smap, ring_map)
    return where


@pytest.mark.parametrize("t_max", [0, 1, 2, 5])
def test_positional_ring_and_creation_formulations_agree(t_max):
    where = set()
    for seed in range(6):
        where |= _random_run(seed, t_max)
    assert {"below", "inside"} <= where and (t_max == 0 or "above" in where)  # (t_max = 0: the window is the newest)


def test_dynamic_scene_box_leaves_the_map():
    """The box is there in frames [2, 5); after it has left and the wall behind it has been merged while stable again,
    the map holds no row inside the box's volume.  Without the rule the box's rows stay for good."""
    rgb, depth, K, poses = _dynamic()
    c = po.confidence_quantile(oracle.run_slam(rgb, depth, K, poses, odom="gt").map, 0.3)
    without, _ = po.run_pointfusion(rgb, depth, K, poses, c_stable=c, t_max=1)
    assert min(fo.rows_in_box(without.smap, DYNAMIC_BOX_CENTER, DYNAMIC_BOX_HALF_EXTENTS, pad=0.02)) > 500
    pm, _ = fo.run_pointfusion(rgb, depth, K, poses, c_stable=c, t_max=1, margin=0.1)
    assert fo.rows_in_box(pm.smap, DYNAMIC_BOX_CENTER, DYNAMIC_BOX_HALF_EXTENTS, pad=0.02) == [0, 0]
    # while the box is in view its rows are kept: nothing stable lies behind them along a merged ray
    mid, _ = fo.run_pointfusion(rgb[:, :5], depth[:, :5], K, poses[:, :5], c_stable=c, t_max=1, margin=0.1)
    assert min(fo.rows_in_box(mid.smap, DYNAMIC_BOX_CENTER, DYNAMIC_BOX_HALF_EXTENTS, pad=0.02)) > 500
