"""The oracle of the merging of overlapping surfels (tests/merge_oracle.py) on hand-built maps with exact expected values:
the absorption, the boundaries of the normal and overlap tests, the winner among several candidates (a tie on d2
included), merge targets, rows the age or free-space rule removes, an unstable absorber and zero radii; the positional
ring update against creation-step stamps on a synthetic sequence; and the keyword errors of PointFusion and
fuse_and_prune.  No GPU needed."""
import math

import numpy as np
import pytest
import torch

import free_space_oracle as fo
import gsx_oracle as oracle
import merge_oracle as mo
import prune_oracle as po

F32 = torch.float32
H = W = 4
POSE = torch.eye(4).unsqueeze(0)
K = torch.tensor([[[1.0, 0.0, 1.0, 0.0], [0.0, 1.0, 1.0, 0.0], [0.0, 0.0, 1.0, 0.0], [0.0, 0.0, 0.0, 1.0]]])
DOT_TH = math.cos(20 * math.pi / 180)
DOWN = (0.0, 0.0, -1.0)


def _map(rows):
    """rows: (point, normal, colour, ccount, radius); z = 1 puts (x, y) at pixel (round(y + 1), round(x + 1))."""
    t = lambda i, k: [torch.tensor([r[i] for r in rows], dtype=F32).view(len(rows), k)]
    smap = oracle.SurfelMap(t(0, 3), t(1, 3), t(2, 3), t(3, 1))
    return smap, t(4, 1)


def _pairs(rows, table, c_stable=0.5, dot_th=DOT_TH, removed=None):
    smap, radii = _map(rows)
    table = torch.tensor(table, dtype=torch.int64).view(-1, 4)
    removed = [torch.zeros(len(rows), dtype=torch.bool)] if removed is None else [torch.tensor(removed)]
    return mo.merge_pairs(smap, radii, table, POSE, K, H, W, c_stable, dot_th, removed)[0].tolist()


M = ((0.0, 0.0, 1.0), DOWN, (0.5, 0.25, 0.0), 1.0, 0.25)  # the stable row pixel (1, 1) merged into
AT_11 = [[0, 0, 1, 1]]


def test_hand_built_absorption_has_exact_values():
    rows = [M, ((0.125, 0.0, 1.0), DOWN, (0.25, 0.5, 1.0), 1.0, 0.125)]
    smap, radii = _map(rows)
    pairs = mo.merge_pairs(smap, radii, torch.tensor(AT_11), POSE, K, H, W, 0.5, DOT_TH,
                           [torch.zeros(2, dtype=torch.bool)])
    assert pairs[0].tolist() == [[0, 1]]
    out, r = mo.absorb(smap, radii, pairs)
    assert out.points[0][0].tolist() == [0.0625, 0.0, 1.0]
    assert out.normals[0][0].tolist() == [0.0, 0.0, -1.0]
    assert out.colors[0][0].tolist() == [0.375, 0.375, 0.5]
    assert out.ccounts[0][0].tolist() == [2.0]
    assert r[0][0].tolist() == [0.1875]
    assert out.points[0][1].tolist() == [0.125, 0.0, 1.0]  # removed by the pruned step, not by the absorption


def test_unequal_confidences_use_the_fusion_operand_order():
    rows = [((0.0, 0.0, 1.0), DOWN, (0.5, 0.25, 0.0), 3.0, 0.25), ((0.1, 0.0, 1.0), DOWN, (0.3, 0.7, 0.9), 0.7, 0.2)]
    smap, radii = _map(rows)
    out, r = mo.absorb(smap, radii, [torch.tensor([[0, 1]])])
    cm, cn = torch.tensor(3.0, dtype=F32), torch.tensor(0.7, dtype=F32)
    inv = 1 / (cm + cn)
    want = ((cm * smap.points[0][0]) + (cn * smap.points[0][1])) * inv
    assert torch.equal(out.points[0][0], want)
    assert torch.equal(r[0][0], ((cm * radii[0][0]) + (cn * radii[0][1])) * inv)
    assert torch.equal(out.ccounts[0][0], (cm + cn).view(1))


def test_normal_dot_exactly_at_the_threshold_is_not_similar():
    n = (0.0, 0.6, -0.8)
    rows = [M, ((0.125, 0.0, 1.0), n, (0.0, 0.0, 0.0), 1.0, 0.125)]
    dot = float(torch.tensor(0.8, dtype=F32))  # (0 * 0 + 0 * 0.6) + (-1)(-0.8) in float32
    assert _pairs(rows, AT_11, dot_th=dot) == []
    assert _pairs(rows, AT_11, dot_th=float(np.nextafter(np.float32(dot), np.float32(0)))) == [[0, 1]]


def test_d2_exactly_at_the_squared_radius_sum_overlaps():
    rows = [((0.0, 0.0, 1.0), DOWN, (0.0, 0.0, 0.0), 1.0, 0.125), ((0.25, 0.0, 1.0), DOWN, (0.0, 0.0, 0.0), 1.0, 0.125)]
    assert _pairs(rows, AT_11) == [[0, 1]]  # d2 = 0.0625 = (0.125 + 0.125)^2
    farther = float(np.nextafter(np.float32(0.25), np.float32(1)))  # d2 = 0.0625 + 2^-25 > 0.0625
    rows[1] = ((farther, 0.0, 1.0),) + rows[1][1:]
    assert _pairs(rows, AT_11) == []


def test_several_candidates_smallest_d2_then_smallest_row():
    rows = [M,
            ((0.25, 0.0, 1.0), DOWN, (0.0, 0.0, 0.0), 1.0, 0.25),     # d2 = 0.0625
            ((-0.125, 0.0, 1.0), DOWN, (0.0, 0.0, 0.0), 1.0, 0.25),   # d2 = 0.015625, the lower index of the tie
            ((0.125, 0.0, 1.0), DOWN, (0.0, 0.0, 0.0), 1.0, 0.25),    # d2 = 0.015625
            ((0.0, 0.0, 1.0), (1.0, 0.0, 0.0), (0.0, 0.0, 0.0), 1.0, 0.25)]  # d2 = 0, normal too different
    assert _pairs(rows, AT_11) == [[0, 2]]


def test_a_merge_target_is_no_candidate():
    rows = [M, ((0.125, 0.0, 1.0), DOWN, (0.0, 0.0, 0.0), 1.0, 0.25), ((0.25, 0.0, 1.0), DOWN, (0.0, 0.0, 0.0), 1.0, 0.25)]
    assert _pairs(rows, AT_11) == [[0, 1]]
    # row 1 is what pixel (3, 3) merged into: the farther row 2 is absorbed instead
    assert _pairs(rows, AT_11 + [[0, 1, 3, 3]]) == [[0, 2]]


def test_a_candidate_the_age_rule_removes_is_no_candidate():
    rows = [M, ((0.125, 0.0, 1.0), DOWN, (0.0, 0.0, 0.0), 0.25, 0.25), ((0.25, 0.0, 1.0), DOWN, (0.0, 0.0, 0.0), 1.0, 0.25)]
    smap, _ = _map(rows)
    pm = po.PrunedMap(smap)
    pm.created, pm.step = [torch.tensor([0, 1, 1])], 2  # step 2, t_max 1: the rows created at step 1 are tested
    age = mo.age_removals(pm, 0.5, 1)
    assert age[0].tolist() == [False, True, False]
    assert _pairs(rows, AT_11, removed=age[0].tolist()) == [[0, 2]]
    assert _pairs(rows, AT_11) == [[0, 1]]


def test_an_unstable_absorber_absorbs_nothing():
    rows = [M, ((0.125, 0.0, 1.0), DOWN, (0.0, 0.0, 0.0), 1.0, 0.25)]
    assert _pairs(rows, AT_11, c_stable=1.0) == [[0, 1]]  # ccount 1.0 >= 1.0: stable
    assert _pairs(rows, AT_11, c_stable=1.5) == []


def test_an_absorber_the_free_space_rule_removes_absorbs_nothing():
    rows = [M, ((0.125, 0.0, 1.0), DOWN, (0.0, 0.0, 0.0), 1.0, 0.25)]
    assert _pairs(rows, AT_11, removed=[True, False]) == []
    assert _pairs(rows, AT_11, removed=[False, True]) == []


@pytest.mark.parametrize("which", [0, 1])
def test_a_zero_radius_never_overlaps(which):
    rows = [list(M), [(0.0, 0.0, 1.0), DOWN, (0.0, 0.0, 0.0), 1.0, 0.25]]
    rows[which][4] = 0.0
    assert _pairs([tuple(r) for r in rows], AT_11) == []


@pytest.mark.parametrize("t_max,margin", [(0, None), (2, None), (2, 0.05)])
def test_positional_ring_matches_creation_steps(t_max, margin):
    """The ring the kernel keeps, replayed on the same removals (absorbed rows anywhere in the map), equals the row
    counts the creation-step stamps give."""
    from gradslam_b200.synthetic import make_dynamic_sequence

    rgb, depth, K4, poses = make_dynamic_sequence(2, 6, 24, 32, 1, 3, seed=3)
    c = po.confidence_quantile(oracle.run_slam(rgb, depth, K4, poses, odom="gt").map, 0.25)
    ring = fo.PositionalRingPruner(2, t_max)
    pm, radii, _, absorbed = mo.run_pointfusion(rgb, depth, K4, poses, c_stable=c, t_max=t_max, margin=margin,
                                                ring=ring)
    assert min(absorbed) > 0
    for k in range(max(pm.step - 1 - t_max, 0), pm.step):
        for b in range(2):
            assert ring.at(k, b) == int((pm.created[b] <= k).sum()), (k, b)
    assert [r.shape[0] for r in radii] == pm.counts()


def test_merge_off_is_the_radii_oracle():
    import radii_oracle as ro
    from gradslam_b200.synthetic import make_sequence

    rgb, depth, K4, poses = make_sequence(2, 5, 24, 32, seed=4)
    pm, radii, _, absorbed = mo.run_pointfusion(rgb, depth, K4, poses, c_stable=0.0, t_max=2, margin=0.05,
                                                merge=False)
    ref, ref_radii = ro.run_pointfusion(rgb, depth, K4, poses, c_stable=0.0, t_max=2, margin=0.05)
    assert absorbed == [0, 0] and pm.counts() == ref.counts()
    for b in range(2):
        assert torch.equal(pm.smap.points[b], ref.smap.points[b]) and torch.equal(radii[b], ref_radii[b])


def _frame():
    import gradslam_b200 as gs

    rgb = torch.zeros(1, 1, 4, 4, 3)
    depth = torch.ones(1, 1, 4, 4, 1)
    return gs.RGBDImages(rgb, depth, torch.eye(4).view(1, 1, 4, 4), torch.eye(4).view(1, 1, 4, 4))


@pytest.mark.parametrize("kw,exc", [
    (dict(merge_overlapping=1, surfel_radii=True, stable_confidence=0, max_unstable_age=1), TypeError),
    (dict(merge_overlapping="yes", surfel_radii=True, stable_confidence=0, max_unstable_age=1), TypeError),
    (dict(merge_overlapping=True, stable_confidence=0, max_unstable_age=1), ValueError),
    (dict(merge_overlapping=True, surfel_radii=True), ValueError),
])
def test_pointfusion_keyword_errors(kw, exc):
    import gradslam_b200 as gs

    with pytest.raises(exc, match="merge_overlapping"):
        gs.PointFusion(odom="gt", device="cpu", **kw)


def test_pointfusion_keyword_accepted_and_off_by_default():
    import gradslam_b200 as gs

    assert gs.PointFusion(odom="gt", device="cpu").merge_overlapping is False
    slam = gs.PointFusion(odom="gt", device="cpu", surfel_radii=True, stable_confidence=0, max_unstable_age=0,
                          merge_overlapping=True)
    assert slam.merge_overlapping is True and slam.free_space_margin is None


@pytest.mark.parametrize("kw,exc", [(dict(merge_overlapping=1, surfel_radii=True), TypeError),
                                    (dict(merge_overlapping=True), ValueError)])
def test_fuse_and_prune_keyword_errors(kw, exc):
    import gradslam_b200 as gs
    from gradslam_b200.slam import fusionutils as fu

    with pytest.raises(exc, match="merge_overlapping"):
        fu.fuse_and_prune(gs.Pointclouds(), _frame(), 0.05, DOT_TH, 0.6, 0.0, 1, math.inf, **kw)
