"""PointFusion(odom='gt') on 133-frame sequences, bit for bit against the CPU oracle: past the 64-frame block of frame
headers the whole-sequence driver keeps.

gsx_pointfusion_sequence_gt holds the headers of kSeqFrames = 64 frames (frame s reads slot s % 64) and rewrites a
block of slots when a call starts and at every 64-aligned frame; K4's scan tile and epoch come from a ticket that counts
on through the call; the arg-min slots and candidate-bin counts carry from one frame to the next; the prune ring has
t_max + 2 rows.  133 frames wrap the header ring twice.  Every input here has frame s >= 64 at another pose than frame
s - 64, so a frame that fused with a stale header would use the wrong depth and camera and differ from the oracle.
The whole-sequence call in 1..4 batch groups, the step API, pinned host frames in calls that start inside a block and
cross into the next, bin overflow that stops and resumes after frame 64, pruning and free-space removal, and the
profiling path bench.py times."""
import math

import pytest
import torch

import free_space_oracle as fo
import gsx_oracle as oracle
import prune_oracle as po
from gradslam_b200.synthetic import make_dynamic_sequence, make_sequence

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
DIST_TH, SIGMA = 0.05, 0.6
DOT_TH = math.cos(20 * math.pi / 180)
L = 133  # two header blocks and 5 frames
BLOCK = 64  # kSeqFrames
TILE = 512  # pixels of a K4 tile: 48 x 64 is 6 tiles, 41 x 64 ends in a partial one
BIN_CAP = 1024  # kBinCap: gsx_debug_set_bin_capacity takes a smaller capacity
# the camera walks forward through the first block, back from frame 100 to 64, and on from 101: K2's candidate count per
# tile falls as well as rises after frame 64, and no frame comes back 64 positions later
ORDER = list(range(BLOCK)) + list(range(100, BLOCK - 1, -1)) + list(range(101, L))

_cache = {}


def _cached(key, make):
    if key not in _cache:
        _cache[key] = make()
    return _cache[key]


def _assert_headers_differ(poses):
    """Every frame s >= 64 has another pose than frame s - 64, in every element: a stale header is a wrong camera."""
    d = (poses[:, BLOCK:] - poses[:, :-BLOCK]).abs().flatten(2).amax(2)
    assert d.shape[1] == poses.shape[1] - BLOCK > 0
    assert float(d.min()) > 0.1, float(d.min())


def _frames(gs, rgb, depth, K, poses):
    return gs.RGBDImages(rgb.to(DEV), depth.to(DEV), K.to(DEV), poses.to(DEV))


def _host(gs, rgb, depth, K, poses):
    return gs.RGBDImages(rgb.pin_memory(), depth.pin_memory(), K.pin_memory(), poses.pin_memory())


def _assert_matches(pc, smap):
    assert [int(c) for c in pc.num_points_per_pointcloud.tolist()] == smap.counts()
    for b in range(len(smap.counts())):
        assert torch.equal(pc.points_list[b].detach().cpu(), smap.points[b]), b
        assert torch.equal(pc.normals_list[b].detach().cpu(), smap.normals[b]), b
        assert torch.equal(pc.colors_list[b].detach().cpu(), smap.colors[b]), b
        assert torch.equal(pc.features_list[b].detach().cpu(), smap.ccounts[b]), b


def _steps(slam, frames, pc=None, s_begin=0):
    import gradslam_b200 as gs

    pc = gs.Pointclouds(device=DEV) if pc is None else pc
    for s in range(s_begin, frames.shape[1]):
        pc, _ = slam.step(pc, frames[:, s], None, inplace=True)
    return pc


def _walk(rgb, depth, K, poses):
    """oracle.run_slam(..., odom='gt') frame by frame (update_map_fusion spelled out).  Returns the map and, per frame,
    the map size before it, the merged and new rows (summed over elements) and K2's candidates per (element, K4 tile)."""
    B, n, H, W, _ = depth.shape
    T = (H * W + TILE - 1) // TILE
    smap = oracle.SurfelMap()
    counters, cand = [], torch.zeros(n, B, T, dtype=torch.int64)
    for s in range(n):
        maps = oracle.frame_maps(depth[:, s:s + 1], K, poses[:, s:s + 1])
        gv, gn = maps["gvertex"][:, 0], maps["gnormal"][:, 0]
        t = oracle.find_active_map_points(smap, poses[:, s], K[:, 0], H, W)
        t, _ = oracle.find_similar_map_points(smap, gv, gn, t, DIST_TH, DOT_TH)
        for b in range(B):
            rows = t[t[:, 0] == b]
            cand[s, b] = torch.bincount((rows[:, 2] * W + rows[:, 3]) // TILE, minlength=T)
        unique = oracle.find_best_unique_correspondences(smap, gv, t)
        before = sum(smap.counts()) if smap.has_points else 0
        smap = oracle.fuse_with_map(smap, maps, rgb[:, s:s + 1], unique, SIGMA)
        counters.append({"map_points": before, "merged": int(unique.shape[0]), "new": sum(smap.counts()) - before})
    return smap, counters, cand


def _sequence(B, H, W, seed):
    """make_sequence inputs and the oracle's map."""
    def make():
        rgb, depth, K, poses = make_sequence(B, L, H, W, seed=seed)
        return rgb, depth, K, poses, oracle.run_slam(rgb, depth, K, poses, odom="gt").map

    return _cached(("sequence", B, H, W, seed), make)


# ------------------------------------------------------------------ 1. whole sequence, device-resident
@pytest.mark.parametrize("groups", [1, 2, 3, 4])
def test_whole_sequence_in_batch_groups_matches_oracle(groups, monkeypatch):
    """B = 5 in 1..4 groups: each group rewrites its own elements' header slots at frames 64 and 128."""
    import gradslam_b200 as gs
    from gradslam_b200 import _C

    monkeypatch.setenv("GSX_SEQ_GROUPS", str(groups))
    assert _C.lib().gsx_pointfusion_sequence_groups(5) == groups
    rgb, depth, K, poses, ref = _sequence(5, 48, 64, seed=31)
    _assert_headers_differ(poses)
    pc, _ = gs.PointFusion(odom="gt", device=DEV)(_frames(gs, rgb, depth, K, poses))
    _assert_matches(pc, ref)


@pytest.mark.parametrize("B,H,W", [(5, 48, 64), (2, 41, 64)], ids=["full_tiles", "partial_last_tile"])
def test_whole_sequence_and_step_loop_match_oracle(B, H, W):
    import gradslam_b200 as gs

    rgb, depth, K, poses, ref = _sequence(B, H, W, seed=31)
    _assert_headers_differ(poses)
    frames = _frames(gs, rgb, depth, K, poses)
    slam = gs.PointFusion(odom="gt", device=DEV)
    _assert_matches(slam(frames)[0], ref)
    _assert_matches(_steps(slam, frames), ref)


# ------------------------------------------------------------------ 2. host-fed calls across a block boundary
@pytest.mark.parametrize("chunk", [4, 61, 64, 65])
def test_host_fed_calls_across_block_boundaries_match_oracle(chunk):
    """Pinned host frames in calls of `chunk` frames.  61: calls [0, 61), [61, 122) and [122, 133); the second writes
    slots 61-63 at its start and slots 0-57 at frame 64, the third slots 58-63 and then 0-4.  65: a call [65, 130) that
    starts one frame into the second block and crosses into the third.  64: every call starts on a block."""
    import gradslam_b200 as gs

    rgb, depth, K, poses, ref = _sequence(5, 48, 64, seed=31)
    _assert_headers_differ(poses)
    slam = gs.PointFusion(odom="gt", device=DEV)
    dev_pc, _ = slam(_frames(gs, rgb, depth, K, poses))
    host_pc, _ = slam._forward_sequence(_host(gs, rgb, depth, K, poses), chunk=chunk)
    _assert_matches(host_pc, ref)
    _assert_matches(dev_pc, ref)


# ------------------------------------------------------------------ 3. bin overflow that stops and resumes after 64
def _overflow_scene():
    """make_sequence in ORDER, the oracle's map, and a bin capacity at which some tile overflows at a frame s >= 64,
    not at s + 1, and again later: the slots its overflow used are read again after the header ring wrapped."""
    def make():
        rgb, depth, K, poses = make_sequence(3, L, 48, 64, seed=33)
        rgb, depth, poses = rgb[:, ORDER].contiguous(), depth[:, ORDER].contiguous(), poses[:, ORDER].contiguous()
        ref, _, cand = _walk(rgb, depth, K, poses)
        for cap in sorted(set(cand[BLOCK:].flatten().tolist())):
            if cap >= BIN_CAP:
                break
            over = cand > cap
            if any(bool((over[s] & ~over[s + 1] & over[s + 2:].any(0)).any()) for s in range(BLOCK, L - 2)):
                return rgb, depth, K, poses, ref, cap
        pytest.fail("no bin capacity below %d gives an overflow that stops and resumes after frame %d" % (BIN_CAP,
                                                                                                           BLOCK))

    return _cached("overflow", make)


@pytest.fixture
def bin_cap():
    from gradslam_b200 import _C

    yield lambda c: _C.lib().gsx_debug_set_bin_capacity(c)
    _C.lib().gsx_debug_set_bin_capacity(-1)


@pytest.mark.parametrize("groups,chunk", [(1, None), (3, None), (None, 61)],
                         ids=["groups1", "groups3", "host_chunk61"])
def test_overflow_that_stops_and_resumes_after_the_first_block_matches_oracle(groups, chunk, bin_cap, monkeypatch):
    import gradslam_b200 as gs

    rgb, depth, K, poses, ref, cap = _overflow_scene()
    _assert_headers_differ(poses)
    bin_cap(cap)
    slam = gs.PointFusion(odom="gt", device=DEV)
    if chunk is None:
        monkeypatch.setenv("GSX_SEQ_GROUPS", str(groups))
        pc, _ = slam(_frames(gs, rgb, depth, K, poses))
    else:
        pc, _ = slam._forward_sequence(_host(gs, rgb, depth, K, poses), chunk=chunk)
    _assert_matches(pc, ref)


# ------------------------------------------------------------------ 4. pruning and free space over the long run
# make_sequence's room with a box in frames [70, 84), filling most of the view of those cameras, in front of the wall
# they see: its stable surfels are free-space violations once the box is gone and the wall merges again
BOX = dict(k0=70, k1=84, box_center=(1.5, 0.4, 1.35), box_half_extents=(0.2, 0.2, 0.2))


def _pruned_inputs(kind):
    """Inputs, the threshold (a quantile of the unpruned oracle map's confidences, as tests/test_gpu_prune.py picks it)
    and the free-space margin (None: the age rule alone)."""
    def make():
        if kind == "age":
            rgb, depth, K, poses = make_sequence(3, L, 48, 64, seed=7)
            q, margin = 0.5, None
        else:
            rgb, depth, K, poses = make_dynamic_sequence(3, L, 48, 64, seed=5, **BOX)
            q, margin = 0.3, 0.05
        c = po.confidence_quantile(oracle.run_slam(rgb, depth, K, poses, odom="gt").map, q)
        return rgb, depth, K, poses, c, margin

    return _cached(("pruned_inputs", kind), make)


def _pruned(kind, t_max):
    """_pruned_inputs and the oracle's pruned map."""
    def make():
        rgb, depth, K, poses, c, margin = _pruned_inputs(kind)
        pm, _ = fo.run_pointfusion(rgb, depth, K, poses, c_stable=c, t_max=t_max, margin=margin)
        assert any(bool((cr <= L - 1 - t_max).any()) for cr in pm.created)  # rows old enough to be tested are kept
        if margin is not None:  # the free-space rule removes rows the age rule keeps
            assert sum(pm.counts()) < sum(po.run_pointfusion(rgb, depth, K, poses, c_stable=c, t_max=t_max)[0].counts())
        return rgb, depth, K, poses, c, margin, pm

    return _cached(("pruned", kind, t_max), make)


def _assert_ring(pc, pm, t_max):
    """Rows are in creation order, so ring(k) = the number of rows created at or before step k."""
    h = pc._prune
    ring = h.ring.cpu()
    assert ring.shape[0] == t_max + 2
    for k in range(max(h.step - 1 - t_max, 0), h.step):
        for b in range(len(pm.counts())):
            assert int(ring[k % (t_max + 2), b]) == int((pm.created[b] <= k).sum()), (k, b)


@pytest.mark.parametrize("kind,t_max", [("age", 3), ("age", 70), ("free_space", 3)])
def test_pruned_whole_and_host_fed_calls_match_oracle(kind, t_max):
    """t_max = 70: the prune ring (72 rows) is longer than the header ring.  The host-fed calls of 61 frames continue
    the ring across calls."""
    import gradslam_b200 as gs

    rgb, depth, K, poses, c, margin, pm = _pruned(kind, t_max)
    _assert_headers_differ(poses)
    slam = gs.PointFusion(odom="gt", device=DEV, stable_confidence=c, max_unstable_age=t_max, free_space_margin=margin)
    whole, _ = slam(_frames(gs, rgb, depth, K, poses))
    host, _ = slam._forward_sequence(_host(gs, rgb, depth, K, poses), chunk=61)
    for pc in (whole, host):
        _assert_matches(pc, pm.smap)
        assert pc._prune.step == L
        _assert_ring(pc, pm, t_max)
    assert torch.equal(whole._prune.ring, host._prune.ring)


@pytest.mark.parametrize("kind,t_max", [("age", 3), ("age", 70), ("free_space", 3)])
def test_pruned_forward_then_steps_match_oracle(kind, t_max):
    """forward() over frames [0, 70), then step() to frame 133: the history step counts on from the call."""
    import gradslam_b200 as gs

    rgb, depth, K, poses, c, margin, pm = _pruned(kind, t_max)
    _assert_headers_differ(poses)
    frames = _frames(gs, rgb, depth, K, poses)
    slam = gs.PointFusion(odom="gt", device=DEV, stable_confidence=c, max_unstable_age=t_max, free_space_margin=margin)
    first, _ = slam(frames[:, :70])
    assert first._prune.step == 70
    pc = _steps(slam, frames, pc=first, s_begin=70)
    assert pc._prune.step == L
    _assert_matches(pc, pm.smap)
    _assert_ring(pc, pm, t_max)


# ------------------------------------------------------------------ 5. the profiling path
def test_profiling_path_counters_and_then_step_api_match_oracle():
    """profiling.profile_pointfusion_gt runs the driver's launches from Python on the step API's workspace: its
    per-frame counters equal the oracle's.  The step API then re-arms that workspace, whose ticket has counted to
    70 * T, and its map equals the oracle's."""
    import gradslam_b200 as gs
    from gradslam_b200 import profiling

    n = 70
    rgb, depth, K, poses = make_sequence(2, n, 48, 64, seed=35)
    _assert_headers_differ(poses)
    ref, counters, _ = _walk(rgb, depth, K, poses)
    frames = _frames(gs, rgb, depth, K, poses)
    _, got = profiling.profile_pointfusion_gt(frames.depth_image.contiguous(), frames.rgb_image.contiguous(),
                                              frames.intrinsics.contiguous(), frames.poses.contiguous(), DIST_TH,
                                              DOT_TH, SIGMA)
    assert len(got) == n
    for s, (g, want) in enumerate(zip(got, counters)):
        assert g["frame"] == s
        assert {k: g[k] for k in want} == want, s
    _assert_matches(_steps(gs.PointFusion(odom="gt", device=DEV), frames), ref)
