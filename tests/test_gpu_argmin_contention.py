"""Oracle parity of the per-pixel arg-min when many map rows compete for the same pixels.  A pixel's slot holds only the
index of the row that currently wins it; a candidate that finds the slot taken recomputes the stored row's key
(1/(cc+1e-20), squared ray distance, index) from the row and the pixel's frame vertex.  The map built here puts four
rows on each of a lattice of ~300 pixels, the rows of a pixel one lattice size apart in index, so that they meet in
different grid-stride passes of K2 and after its deferred settle:
  * exact duplicates (same position, normal and confidence): the lowest index decides;
  * equal confidence at different distances along the pixel's ray: the nearest, stored last, wins;
  * a higher confidence farther away: it beats a nearer row of lower confidence, and the nearer of two such rows wins.
One fusion step from depth, one through the differentiable mode (frame maps packed by K1r), and the table API's
find_best_unique_correspondences are compared with the oracle bit for bit."""
import math

import pytest
import torch

import gsx_oracle as oracle
from gradslam_b200.synthetic import make_sequence

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
DOT_TH = math.cos(20 * math.pi / 180)
DIST_TH, SIGMA = 0.05, 0.6
B, H, W = 2, 48, 64
STEP = 3  # lattice of contested pixels
# (offset along the ray, confidence) of the four rows of a pixel, per kind; the winner is row 0 (duplicates) or row 3
KINDS = {
    "duplicates": [(0.0, 0.5)] * 4,
    "equal_cc": [(0.02, 0.5), (0.03, 0.5), (0.01, 0.5), (0.005, 0.5)],
    "higher_cc_farther": [(0.001, 0.3), (0.03, 0.9), (0.002, 0.3), (0.01, 0.9)],
}
WINNER = {"duplicates": 0, "equal_cc": 3, "higher_cc_farther": 3}


def _scene():
    """Frame, its oracle maps, the contested map (rows as CPU tensors) and, per element, {pixel: (kind, rows)}."""
    rgb, depth, K, poses = make_sequence(B, 1, H, W, seed=5)
    maps = oracle.frame_maps(depth, K, poses)
    gv, gn = maps["gvertex"][:, 0], maps["gnormal"][:, 0]
    kinds = list(KINDS)
    per_b, expect = [], []
    for b in range(B):
        centre = poses[b, 0, :3, 3]
        pixels = [(h, w) for h in range(1, H - 1, STEP) for w in range(1, W - 1, STEP)
                  if depth[b, 0, h, w, 0] > 0 and float(gn[b, h, w].norm()) > 0.5]
        G = len(pixels)
        pts, nrm, cc = torch.zeros(4 * G, 3), torch.zeros(4 * G, 3), torch.zeros(4 * G, 1)
        want = {}
        for g, (h, w) in enumerate(pixels):
            kind = kinds[g % len(kinds)]
            ray = gv[b, h, w] - centre
            ray = ray / ray.norm()
            for k, (t, c) in enumerate(KINDS[kind]):
                n = k * G + g  # the rows of one pixel are G apart
                pts[n] = gv[b, h, w] + t * ray
                nrm[n] = gn[b, h, w]
                cc[n] = c
            want[(h, w)] = (kind, WINNER[kind] * G + g)
        per_b.append((pts, nrm, cc))
        expect.append(want)
    N = min(p[0].shape[0] for p in per_b)
    g = torch.Generator().manual_seed(0)
    cols = torch.rand(B, N, 3, generator=g)
    pts = torch.stack([p[0][:N] for p in per_b])
    nrm = torch.stack([p[1][:N] for p in per_b])
    cc = torch.stack([p[2][:N] for p in per_b])
    # rows cut off by the common size N no longer compete: drop their pixels from the expectation
    for b in range(B):
        G = per_b[b][0].shape[0] // 4
        expect[b] = {px: kw for px, kw in expect[b].items() if all(k * G + kw[1] % G < N for k in range(4))}
    return (rgb, depth, K, poses), maps, (pts, nrm, cols, cc), expect


@pytest.fixture(scope="module")
def scene():
    return _scene()


def _smap(rows):
    pts, nrm, cols, cc = rows
    return oracle.SurfelMap([p.clone() for p in pts], [n.clone() for n in nrm], [c.clone() for c in cols],
                            [c.clone() for c in cc])


def _pc(gs, rows):
    pts, nrm, cols, cc = rows
    return gs.Pointclouds(points=pts.to(DEV), normals=nrm.to(DEV), colors=cols.to(DEV), features=cc.to(DEV))


def _assert_maps_equal(pc, ref):
    assert [int(c) for c in pc.num_points_per_pointcloud.tolist()] == ref.counts()
    for b in range(B):
        assert torch.equal(pc.points_list[b].detach().cpu(), ref.points[b]), b
        assert torch.equal(pc.normals_list[b].detach().cpu(), ref.normals[b]), b
        assert torch.equal(pc.colors_list[b].detach().cpu(), ref.colors[b]), b
        assert torch.equal(pc.features_list[b].detach().cpu(), ref.ccounts[b]), b


@pytest.fixture
def k2_grid_cap():
    from gradslam_b200 import _C

    yield _C.lib().gsx_debug_set_k2_grid_cap
    _C.lib().gsx_debug_set_k2_grid_cap(0)


def test_oracle_winners_are_the_constructed_ones(scene):
    """The scene does what it claims: every contested pixel has its four rows as live candidates, and the oracle picks
    the row the construction intends."""
    (rgb, depth, K, poses), maps, rows, expect = scene
    smap = _smap(rows)
    gv, gn = maps["gvertex"][:, 0], maps["gnormal"][:, 0]
    active = oracle.find_active_map_points(smap, poses[:, 0], K[:, 0], H, W)
    similar, _ = oracle.find_similar_map_points(smap, gv, gn, active, DIST_TH, DOT_TH)
    unique = oracle.find_best_unique_correspondences(smap, gv, similar)
    for b in range(B):
        assert len(expect[b]) > 100
        live = similar[similar[:, 0] == b]
        per_pixel = torch.bincount(live[:, 2] * W + live[:, 3], minlength=H * W)
        won = {(int(r[2]), int(r[3])): int(r[1]) for r in unique[unique[:, 0] == b]}
        for (h, w), (kind, n) in expect[b].items():
            assert int(per_pixel[h * W + w]) == 4, (b, h, w, kind)
            assert won[(h, w)] == n, (b, h, w, kind)


@pytest.mark.parametrize("cap", [0, 1, 3])
@pytest.mark.parametrize("packed", [False, True], ids=["depth_fed", "packed_maps"])
def test_contested_fusion_step_matches_oracle(scene, k2_grid_cap, cap, packed):
    """cap: K2's CTAs in all (0: the default grid).  packed: depth requires grad, so the step runs the differentiable
    mode, whose frame records K1r packs from the materialised maps."""
    import gradslam_b200 as gs
    from gradslam_b200.slam import fusionutils as fu

    (rgb, depth, K, poses), maps, rows, _ = scene
    ref = oracle.update_map_fusion(_smap(rows), maps, rgb, poses[:, 0], K[:, 0], DIST_TH, DOT_TH, SIGMA)
    k2_grid_cap(cap)
    d = depth.to(DEV).requires_grad_(packed)
    frame = gs.RGBDImages(rgb.to(DEV), d, K.to(DEV), poses.to(DEV))
    pc = fu.update_map_fusion(_pc(gs, rows), frame, DIST_TH, DOT_TH, SIGMA, inplace=False)
    _assert_maps_equal(pc, ref)


def test_contested_best_unique_correspondences_match_oracle(scene):
    import gradslam_b200 as gs
    from gradslam_b200.slam import fusionutils as fu

    (rgb, depth, K, poses), maps, rows, _ = scene
    smap = _smap(rows)
    gv, gn = maps["gvertex"][:, 0], maps["gnormal"][:, 0]
    r_similar, _ = oracle.find_similar_map_points(
        smap, gv, gn, oracle.find_active_map_points(smap, poses[:, 0], K[:, 0], H, W), DIST_TH, DOT_TH)
    frame = gs.RGBDImages(rgb.to(DEV), depth.to(DEV), K.to(DEV), poses.to(DEV))
    pc = _pc(gs, rows)
    similar, _ = fu.find_similar_map_points(pc, frame, fu.find_active_map_points(pc, frame), DIST_TH, DOT_TH)
    assert torch.equal(similar.cpu(), r_similar)
    # the candidates in reverse order as well: the winner is then claimed first or last
    for table in (similar, similar.flip(0)):
        got = fu.find_best_unique_correspondences(pc, frame, table)
        assert torch.equal(got.cpu(), oracle.find_best_unique_correspondences(smap, gv, r_similar))
