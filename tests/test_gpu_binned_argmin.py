"""Oracle parity of the binned per-pixel arg-min.  K2 appends every live candidate to the bin of the K4 tile that owns
its pixel; K4 takes the minimum of (key_hi, n) in shared memory and combines it with the pixel's arg-min slot, which
holds the candidates that found their bin full (and the winners gsx_records_from_table stores).  The bin capacity is
capped at 0 (every candidate goes to the slot), 1 and 3 (nearly every tile overflows, so both halves meet in K4's
combine) and left at the built-in value; every result is compared with the CPU oracle bit for bit."""
import math

import pytest
import torch

import gsx_oracle as oracle
from gradslam_b200.synthetic import make_sequence

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
DOT_TH = math.cos(20 * math.pi / 180)
DIST_TH, SIGMA = 0.05, 0.6
CAPS = [0, 1, 3, None]  # None: the built-in capacity
CAP_IDS = ["cap0", "cap1", "cap3", "shipped"]

_ref_cache = {}


@pytest.fixture
def bin_cap():
    from gradslam_b200 import _C

    def set_cap(c):
        _C.lib().gsx_debug_set_bin_capacity(-1 if c is None else c)

    yield set_cap
    _C.lib().gsx_debug_set_bin_capacity(-1)


def _frames(gs, rgb, depth, K, poses):
    return gs.RGBDImages(rgb.to(DEV), depth.to(DEV), K.to(DEV), poses.to(DEV))


def _assert_element_matches(pc, b, ref_map, rb):
    assert int(pc.num_points_per_pointcloud[b]) == ref_map.counts()[rb]
    assert torch.equal(pc.points_list[b].detach().cpu(), ref_map.points[rb]), b
    assert torch.equal(pc.normals_list[b].detach().cpu(), ref_map.normals[rb]), b
    assert torch.equal(pc.colors_list[b].detach().cpu(), ref_map.colors[rb]), b
    assert torch.equal(pc.features_list[b].detach().cpu(), ref_map.ccounts[rb]), b


def _assert_matches_oracle(pc, ref_map):
    assert [int(c) for c in pc.num_points_per_pointcloud.tolist()] == ref_map.counts()
    for b in range(len(ref_map.counts())):
        _assert_element_matches(pc, b, ref_map, b)


def _ref(key, make):
    if key not in _ref_cache:
        _ref_cache[key] = make()
    return _ref_cache[key]


# ---------------------------------------------------------------------------------------------- the bench's inputs
L_BENCH = 4


def _bench_inputs():
    """The bench configuration (B=8, 640x480, seed 0), its first L_BENCH frames, and the oracle's maps of elements 0
    and 7 (batch elements are independent, so the oracle runs on those two alone)."""
    rgb, depth, K, poses = make_sequence(8, L_BENCH, 480, 640, seed=0)
    sel = torch.tensor([0, 7])
    ref = oracle.run_slam(rgb[sel], depth[sel], K[sel], poses[sel], odom="gt").map
    return rgb, depth, K, poses, ref


@pytest.mark.parametrize("cap", CAPS, ids=CAP_IDS)
def test_bench_elements_match_oracle(cap, bin_cap):
    """Elements 0 and 7 of the bench's batch after L_BENCH frames, whole-sequence call and step loop."""
    import gradslam_b200 as gs

    rgb, depth, K, poses, ref = _ref("bench", _bench_inputs)
    bin_cap(cap)
    frames = _frames(gs, rgb, depth, K, poses)
    slam = gs.PointFusion(odom="gt", device=DEV)
    pc, _ = slam(frames)
    for rb, b in enumerate((0, 7)):
        _assert_element_matches(pc, b, ref, rb)
    pc = gs.Pointclouds(device=DEV)
    for s in range(L_BENCH):
        pc, _ = slam.step(pc, frames[:, s], None, inplace=True)
    for rb, b in enumerate((0, 7)):
        _assert_element_matches(pc, b, ref, rb)


# ---------------------------------------------------------------------------------------------- sequence driver
@pytest.mark.parametrize("cap", CAPS, ids=CAP_IDS)
@pytest.mark.parametrize("groups", [1, 2, 3, 4])
def test_batch_groups_match_oracle(groups, cap, bin_cap, monkeypatch):
    """B=5 in 1..4 concurrent batch groups: each group's bins and counts start at its first element."""
    import gradslam_b200 as gs
    from gradslam_b200 import _C

    monkeypatch.setenv("GSX_SEQ_GROUPS", str(groups))
    assert _C.lib().gsx_pointfusion_sequence_groups(5) == groups

    def make():
        rgb, depth, K, poses = make_sequence(5, 5, 48, 64, seed=0)
        return rgb, depth, K, poses, oracle.run_slam(rgb, depth, K, poses, odom="gt").map

    rgb, depth, K, poses, ref = _ref("groups", make)
    bin_cap(cap)
    pc, _ = gs.PointFusion(odom="gt", device=DEV)(_frames(gs, rgb, depth, K, poses))
    _assert_matches_oracle(pc, ref)


# ---------------------------------------------------------------------------------------------- partial last tile
@pytest.mark.parametrize("cap", CAPS, ids=CAP_IDS)
@pytest.mark.parametrize("shape", [(2, 4, 41, 64), (3, 3, 33, 47)])
def test_partial_last_tile_matches_oracle(shape, cap, bin_cap):
    """H*W = 2624 and 1551: the last K4 tile of every element is partial."""
    import gradslam_b200 as gs

    B, L, H, W = shape
    assert (H * W) % 512 != 0

    def make():
        rgb, depth, K, poses = make_sequence(B, L, H, W, seed=3)
        return rgb, depth, K, poses, oracle.run_slam(rgb, depth, K, poses, odom="gt").map

    rgb, depth, K, poses, ref = _ref(("partial",) + shape, make)
    bin_cap(cap)
    frames = _frames(gs, rgb, depth, K, poses)
    slam = gs.PointFusion(odom="gt", device=DEV)
    pc, _ = slam(frames)
    _assert_matches_oracle(pc, ref)
    pc = gs.Pointclouds(device=DEV)
    for s in range(L):
        pc, _ = slam.step(pc, frames[:, s], None, inplace=True)
    _assert_matches_oracle(pc, ref)


# ---------------------------------------------------------------------------------------------- differentiable mode
@pytest.mark.parametrize("cap", CAPS, ids=CAP_IDS)
def test_differentiable_steps_match_oracle(cap, bin_cap):
    """depth requires grad: every step runs the differentiable mode, whose frame maps K1r packs into records."""
    import gradslam_b200 as gs

    B, L, H, W = 2, 3, 48, 64

    def make():
        rgb, depth, K, poses = make_sequence(B, L, H, W, seed=4)
        return rgb, depth, K, poses, oracle.run_slam(rgb, depth, K, poses, odom="gt").map

    rgb, depth, K, poses, ref = _ref("diff", make)
    bin_cap(cap)
    frames = gs.RGBDImages(rgb.to(DEV), depth.to(DEV).requires_grad_(True), K.to(DEV), poses.to(DEV))
    slam = gs.PointFusion(odom="gt", device=DEV)
    pc = gs.Pointclouds(device=DEV)
    for s in range(L):
        pc, _ = slam.step(pc, frames[:, s], None)
    _assert_matches_oracle(pc, ref)


# ---------------------------------------------------------------------------------------------- contention
# Four rows on each of a lattice of pixels, the rows of a pixel G apart in index (G = number of contested pixels), so
# that with small bins some of a pixel's candidates are binned and the others go to the arg-min slot.
C_B, C_H, C_W, STEP = 2, 48, 64, 3
KINDS = {
    "duplicates": [(0.0, 0.5)] * 4,  # the lowest index decides
    "equal_cc": [(0.02, 0.5), (0.03, 0.5), (0.01, 0.5), (0.005, 0.5)],  # the nearest, stored last, wins
    "higher_cc_farther": [(0.001, 0.3), (0.03, 0.9), (0.002, 0.3), (0.01, 0.9)],  # confidence first, then distance
    "tied_keys_reversed": [(0.01, 0.5), (0.0, 0.7), (0.0, 0.7), (0.01, 0.5)],  # two equal keys: the lower n wins
}


def _contention_scene():
    rgb, depth, K, poses = make_sequence(C_B, 1, C_H, C_W, seed=5)
    maps = oracle.frame_maps(depth, K, poses)
    gv, gn = maps["gvertex"][:, 0], maps["gnormal"][:, 0]
    kinds = list(KINDS)
    per_b = []
    for b in range(C_B):
        centre = poses[b, 0, :3, 3]
        pixels = [(h, w) for h in range(1, C_H - 1, STEP) for w in range(1, C_W - 1, STEP)
                  if depth[b, 0, h, w, 0] > 0 and float(gn[b, h, w].norm()) > 0.5]
        G = len(pixels)
        pts, nrm, cc = torch.zeros(4 * G, 3), torch.zeros(4 * G, 3), torch.zeros(4 * G, 1)
        for g, (h, w) in enumerate(pixels):
            ray = gv[b, h, w] - centre
            ray = ray / ray.norm()
            for k, (t, c) in enumerate(KINDS[kinds[g % len(kinds)]]):
                pts[k * G + g] = gv[b, h, w] + t * ray
                nrm[k * G + g] = gn[b, h, w]
                cc[k * G + g] = c
        per_b.append((pts, nrm, cc))
    N = min(p[0].shape[0] for p in per_b)
    cols = torch.rand(C_B, N, 3, generator=torch.Generator().manual_seed(0))
    rows = tuple(torch.stack([p[i][:N] for p in per_b]) for i in range(3))
    return (rgb, depth, K, poses), maps, (rows[0], rows[1], cols, rows[2])


def _smap(rows):
    pts, nrm, cols, cc = rows
    return oracle.SurfelMap([p.clone() for p in pts], [n.clone() for n in nrm], [c.clone() for c in cols],
                            [c.clone() for c in cc])


def _pc(gs, rows):
    pts, nrm, cols, cc = rows
    return gs.Pointclouds(points=pts.to(DEV), normals=nrm.to(DEV), colors=cols.to(DEV), features=cc.to(DEV))


def test_contention_scene_has_contested_pixels():
    (rgb, depth, K, poses), maps, rows = _ref("contention", _contention_scene)
    smap = _smap(rows)
    gv, gn = maps["gvertex"][:, 0], maps["gnormal"][:, 0]
    active = oracle.find_active_map_points(smap, poses[:, 0], K[:, 0], C_H, C_W)
    similar, _ = oracle.find_similar_map_points(smap, gv, gn, active, DIST_TH, DOT_TH)
    for b in range(C_B):
        live = similar[similar[:, 0] == b]
        per_pixel = torch.bincount(live[:, 2] * C_W + live[:, 3], minlength=C_H * C_W)
        assert int((per_pixel == 4).sum()) > 100


@pytest.mark.parametrize("cap", CAPS, ids=CAP_IDS)
@pytest.mark.parametrize("packed", [False, True], ids=["depth_fed", "packed_maps"])
def test_contested_step_matches_oracle(cap, packed, bin_cap):
    """One fusion step on the contested map (step API), from depth and through the differentiable mode."""
    import gradslam_b200 as gs
    from gradslam_b200.slam import fusionutils as fu

    (rgb, depth, K, poses), maps, rows = _ref("contention", _contention_scene)
    ref = oracle.update_map_fusion(_smap(rows), maps, rgb, poses[:, 0], K[:, 0], DIST_TH, DOT_TH, SIGMA)
    bin_cap(cap)
    frame = gs.RGBDImages(rgb.to(DEV), depth.to(DEV).requires_grad_(packed), K.to(DEV), poses.to(DEV))
    pc = fu.update_map_fusion(_pc(gs, rows), frame, DIST_TH, DOT_TH, SIGMA, inplace=False)
    _assert_matches_oracle(pc, ref)


@pytest.mark.parametrize("cap", CAPS, ids=CAP_IDS)
def test_contested_table_api_matches_oracle(cap, bin_cap):
    """find_correspondences + fuse_with_map: the winners reach K4 through the arg-min slots only (the bins are empty),
    and fusing a second frame right after on the same workspace finds no stale bin records."""
    import gradslam_b200 as gs
    from gradslam_b200.slam import fusionutils as fu

    (rgb, depth, K, poses), maps, rows = _ref("contention", _contention_scene)
    smap = _smap(rows)
    gv = maps["gvertex"][:, 0]
    table = oracle.find_correspondences(smap, maps, poses[:, 0], K[:, 0], DIST_TH, DOT_TH)
    ref = oracle.fuse_with_map(smap, maps, rgb, table, SIGMA)
    bin_cap(cap)
    frame = gs.RGBDImages(rgb.to(DEV), depth.to(DEV), K.to(DEV), poses.to(DEV))
    pc = _pc(gs, rows)
    got = fu.find_correspondences(pc, frame, DIST_TH, DOT_TH)
    assert torch.equal(got.cpu(), oracle.find_best_unique_correspondences(smap, gv, oracle.find_similar_map_points(
        smap, gv, maps["gnormal"][:, 0], oracle.find_active_map_points(smap, poses[:, 0], K[:, 0], C_H, C_W),
        DIST_TH, DOT_TH)[0]))
    fused = fu.fuse_with_map(pc, frame, got, SIGMA)
    _assert_matches_oracle(fused, ref)
    # the fused step (bins filled) followed by the table path on the same workspace
    stepped = fu.update_map_fusion(_pc(gs, rows), frame, DIST_TH, DOT_TH, SIGMA)
    _assert_matches_oracle(stepped, oracle.update_map_fusion(_smap(rows), maps, rgb, poses[:, 0], K[:, 0], DIST_TH,
                                                             DOT_TH, SIGMA))
    _assert_matches_oracle(fu.fuse_with_map(pc, frame, got, SIGMA), ref)
