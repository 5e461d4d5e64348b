"""CPU checks of the unstable-surfel removal oracle (tests/prune_oracle.py): the rule's limits, a known-answer case, and
agreement of its creation-step formulation with the ring formulation the CUDA path uses."""
import math

import pytest
import torch

import gsx_oracle as oracle
import prune_oracle as po
from gradslam_b200.synthetic import make_sequence

B, L, H, W = 2, 6, 24, 32


def _inputs(empty_element=None):
    rgb, depth, K, poses = make_sequence(B, L, H, W, seed=3)
    if empty_element is not None:
        depth[empty_element] = 0.0
    return rgb, depth, K, poses


def _assert_same_map(a, b):
    assert a.counts() == b.counts()
    for x, y in ((a.points, b.points), (a.normals, b.normals), (a.colors, b.colors), (a.ccounts, b.ccounts)):
        for u, v in zip(x, y):
            assert torch.equal(u, v)


def test_zero_threshold_removes_nothing():
    rgb, depth, K, poses = _inputs()
    ref = oracle.run_slam(rgb, depth, K, poses, odom="gt").map
    for t_max in (0, 2):
        pm, _ = po.run_pointfusion(rgb, depth, K, poses, c_stable=0.0, t_max=t_max)
        _assert_same_map(pm.smap, ref)


@pytest.mark.parametrize("t_max", [0, 1, 3])
def test_infinite_threshold_keeps_only_the_last_t_max_steps(t_max):
    rgb, depth, K, poses = _inputs()
    pm, _ = po.run_pointfusion(rgb, depth, K, poses, c_stable=math.inf, t_max=t_max)
    last = L - 1
    for b in range(B):
        created = pm.created[b]
        assert bool(((created > last - t_max) & (created <= last)).all())
        assert torch.equal(created, torch.sort(created, stable=True).values)  # in order
        if t_max == 0:
            assert created.numel() == 0
        else:
            assert set(created.tolist()) <= set(range(last - t_max + 1, last + 1))


def _hand_map(cc):
    n = len(cc)
    pts = [torch.arange(3 * n, dtype=torch.float32).view(n, 3)]
    return oracle.SurfelMap(pts, [p.clone() for p in pts], [p.clone() for p in pts],
                            [torch.tensor(cc, dtype=torch.float32).view(n, 1)])


def _append(smap, cc, start):
    other = _hand_map(cc)
    other.points[0] += start
    smap.append(other)


def test_known_answer_merges_around_the_age_test():
    """t_max = 2, c_stable = 1: rows a, b, c are created at step 0 with confidence 0.3.  a is merged to 1.1 at step 1,
    just before its test at step 2, and is kept; c reaches 1.1 only at step 3, after its test, and is gone by then; b is
    never merged and is removed.  The rows of steps 1 and 2 are untouched at step 2."""
    pm = po.PrunedMap(_hand_map([0.3, 0.3, 0.3]))
    assert po.prune_step(pm, 1.0, 2)[0].tolist() == [0, 1, 2]           # step 0
    pm.smap.ccounts[0][0] += 0.8                                         # merge into a
    _append(pm.smap, [0.2], 100)
    assert po.prune_step(pm, 1.0, 2)[0].tolist() == [0, 1, 2, 3]        # step 1
    _append(pm.smap, [0.1, 2.0], 200)
    assert po.prune_step(pm, 1.0, 2)[0].tolist() == [0, 3, 4, 5]        # step 2: b and c removed
    assert pm.created[0].tolist() == [0, 1, 2, 2]
    assert pm.smap.ccounts[0][:, 0].tolist() == pytest.approx([1.1, 0.2, 0.1, 2.0])
    assert po.prune_step(pm, 1.0, 2)[0].tolist() == [0, 2, 3]           # step 3: the 0.2 row of step 1 removed
    assert pm.created[0].tolist() == [0, 2, 2]


def test_t_max_zero_tests_rows_in_the_step_that_creates_them():
    pm = po.PrunedMap(_hand_map([0.5, 1.5, 0.9]))
    assert po.prune_step(pm, 1.0, 0)[0].tolist() == [1]
    _append(pm.smap, [2.0, 0.1], 10)
    pm.smap.ccounts[0][0] -= 1.0  # an old row below the threshold is not tested again
    assert po.prune_step(pm, 1.0, 0)[0].tolist() == [0, 1]


def test_empty_element_and_rows_appended_between_steps():
    rgb, depth, K, poses = _inputs(empty_element=1)
    ref = oracle.run_slam(rgb, depth, K, poses, odom="gt").map
    c = po.confidence_quantile(oracle.SurfelMap([ref.points[0]], None, None, [ref.ccounts[0]]), 0.5)
    pm, _ = po.run_pointfusion(rgb[:, :3], depth[:, :3], K, poses[:, :3], c_stable=c, t_max=1)
    assert pm.counts()[1] == 0
    # out of view, so never merged; confidence below the threshold
    extra = oracle.SurfelMap([torch.rand(5, 3) - 100.0, torch.rand(0, 3)], [torch.rand(5, 3), torch.rand(0, 3)],
                             [torch.rand(5, 3), torch.rand(0, 3)], [torch.full((5, 1), 1e-9), torch.zeros(0, 1)])
    pm.smap.append(extra)
    pm, _ = po.run_pointfusion(rgb[:, :4], depth[:, :4], K, poses[:, :4], c_stable=c, t_max=1, pm=pm, s_begin=3)
    rows = [i for i, p in enumerate(pm.smap.points[0]) if any(torch.equal(p, q) for q in extra.points[0])]
    assert len(rows) == 5 and pm.created[0][rows].tolist() == [3] * 5  # stamped at the next pruned step
    pm, _ = po.run_pointfusion(rgb, depth, K, poses, c_stable=c, t_max=1, pm=pm, s_begin=4)
    assert pm.counts()[1] == 0
    assert not any(torch.equal(p, q) for p in pm.smap.points[0] for q in extra.points[0])  # removed at step 4


def _random_run(seed, t_max, steps=12, Bn=3):
    """Random appends, merges and thresholds: the ring formulation equals the creation-step formulation."""
    g = torch.Generator().manual_seed(seed)
    base = oracle.SurfelMap([torch.rand(int(torch.randint(0, 5, (1,), generator=g)), 3, generator=g) for _ in range(Bn)],
                            None, None, None)
    base.normals = [p.clone() for p in base.points]
    base.colors = [p.clone() for p in base.points]
    base.ccounts = [torch.rand(p.shape[0], 1, generator=g) for p in base.points]
    pm, ring_map, ring = po.PrunedMap(base.clone()), base.clone(), po.RingPruner(Bn, t_max)
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
        c_stable = float(torch.rand(1, generator=g)) * 1.5
        po.prune_step(pm, c_stable, t_max)
        ring(ring_map, c_stable)
        _assert_same_map(pm.smap, ring_map)


@pytest.mark.parametrize("t_max", [0, 1, 2, 5])
def test_ring_and_creation_formulations_agree(t_max):
    for seed in range(6):
        _random_run(seed, t_max)
