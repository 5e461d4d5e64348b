"""The per-pixel arg-min slots of the fusion workspace are zero whenever a frame's K2 starts.  K4 keeps that so: it reads
and clears only the slots of tiles whose candidate bin overflowed, or of an element whose slots gsx_records_from_table
filled.  The sequence driver zeroes the re-arm state once per call and runs no K1r; the per-frame step API's K1r clears
what a frame abandoned before its K4 left behind.  Every map is compared with the CPU oracle bit for bit."""
import math

import pytest
import torch

import gsx_oracle as oracle
from gradslam_b200.synthetic import make_sequence

DEV = "cuda:0"
DIST_TH, SIGMA = 0.05, 0.6
DOT_TH = math.cos(20 * math.pi / 180)
B, L, H, W = 5, 6, 48, 64
TILE = 512  # pixels of a K4 tile
# The camera steps back and forth through the synthetic sequence, so that a tile's candidate count falls as well as
# rises from frame to frame (along the sequence's own order it only grows).
ORDER = [0, 3, 1, 5, 2, 4]
CAPS = list(range(256, 576, 8))
SMALL_CAP = 2

_cache = {}


def _scene(H=H, W=W):
    """The inputs, the oracle's map after each prefix of frames, and the number of K2 candidates per (frame, element,
    K4 tile)."""
    if (H, W) not in _cache:
        rgb, depth, K, poses = make_sequence(B, L, H, W, seed=21)
        rgb, depth, poses = rgb[:, ORDER].contiguous(), depth[:, ORDER].contiguous(), poses[:, ORDER].contiguous()
        maps = [None] + [oracle.run_slam(rgb[:, :s], depth[:, :s], K, poses[:, :s], odom="gt").map
                         for s in range(1, L + 1)]
        T = (H * W + TILE - 1) // TILE
        counts = torch.zeros(L, B, T, dtype=torch.int64)
        for s in range(1, L):
            fm = oracle.frame_maps(depth[:, s:s + 1], K, poses[:, s:s + 1])
            active = oracle.find_active_map_points(maps[s], poses[:, s], K[:, 0], H, W)
            similar, _ = oracle.find_similar_map_points(maps[s], fm["gvertex"][:, 0], fm["gnormal"][:, 0], active,
                                                        DIST_TH, DOT_TH)
            for b in range(B):
                rows = similar[similar[:, 0] == b]
                counts[s, b] = torch.bincount((rows[:, 2] * W + rows[:, 3]) // TILE, minlength=T)
        _cache[(H, W)] = (rgb, depth, K, poses, maps, counts)
    return _cache[(H, W)]


def _mixed_cap(counts):
    """A bin capacity at which some tile overflows in a frame and not in the next one, and overflows again later: a
    slot its overflow left behind would be read by that later frame."""
    for cap in CAPS:
        over = counts > cap
        for s in range(1, L - 2):
            if bool((over[s] & ~over[s + 1] & over[s + 2:].any(0)).any()):
                return cap
    pytest.fail("no capacity in [%d, %d] gives an overflow that stops and resumes" % (CAPS[0], CAPS[-1]))


@pytest.fixture
def bin_cap():
    from gradslam_b200 import _C

    yield lambda c: _C.lib().gsx_debug_set_bin_capacity(c)
    _C.lib().gsx_debug_set_bin_capacity(-1)


def _frames(gs, rgb, depth, K, poses):
    return gs.RGBDImages(rgb.to(DEV), depth.to(DEV), K.to(DEV), poses.to(DEV))


def _assert_matches(pc, ref):
    assert [int(c) for c in pc.num_points_per_pointcloud.tolist()] == ref.counts()
    for b in range(B):
        assert torch.equal(pc.points_list[b].detach().cpu(), ref.points[b]), b
        assert torch.equal(pc.normals_list[b].detach().cpu(), ref.normals[b]), b
        assert torch.equal(pc.colors_list[b].detach().cpu(), ref.colors[b]), b
        assert torch.equal(pc.features_list[b].detach().cpu(), ref.ccounts[b]), b


@pytest.mark.gpu
@pytest.mark.parametrize("groups", [1, 2, 3, 4])
def test_overflow_that_stops_and_resumes_matches_oracle(groups, bin_cap, monkeypatch):
    """Whole-sequence call in 1..4 batch groups, and the same frames from pinned host memory, which the driver takes in
    two calls (frames [0, 4) and [4, 6), the second with s_begin = 4)."""
    import gradslam_b200 as gs

    monkeypatch.setenv("GSX_SEQ_GROUPS", str(groups))
    rgb, depth, K, poses, maps, counts = _scene()
    bin_cap(_mixed_cap(counts))
    slam = gs.PointFusion(odom="gt", device=DEV)
    pc, _ = slam(_frames(gs, rgb, depth, K, poses))
    _assert_matches(pc, maps[L])
    host = gs.RGBDImages(rgb.pin_memory(), depth.pin_memory(), K.pin_memory(), poses.pin_memory())
    pc, _ = slam(host)
    _assert_matches(pc, maps[L])


def _abandon(gs, pc, frame, table=None):
    """K1r and the association of `frame` (K2, or the rows of `table`), without its K4."""
    from gradslam_b200.slam import fusionutils as fu

    frame = frame.to_channels_last()
    fu._prepare_map(pc, frame, True)
    ws = fu._Workspace.get(pc.device, B, frame.shape[2], frame.shape[3])
    fu._launch_frame_records(ws, frame, SIGMA, pc.device)
    if table is None:
        fu._launch_association(ws, pc, frame, dist_th=DIST_TH, dot_th=DOT_TH)
    else:
        fu._launch_association(ws, pc, frame, table=table)


@pytest.mark.gpu
@pytest.mark.parametrize("hw", [(48, 64), (41, 64)], ids=["full_tiles", "partial_last_tile"])
@pytest.mark.parametrize("path", ["k2_overflow", "table"])
def test_step_after_abandoned_frame_matches_oracle(path, hw, bin_cap):
    """Frame s + 1 stops after K2 with overflowing bins, or after gsx_records_from_table, and then frame s is stepped on
    the same workspace.  The abandoned slots hold the rows that frame s + 1's pixels chose, which are not frame s's
    winners: unless K1r clears them, frame s's overflowing candidates are compared with them and K4 merges into them.
    The bin capacity is small throughout, so frame s overflows too and K4 reads its tiles' slots.  41 x 64 pixels end
    in a partial K4 tile, which is also a partial K1r block."""
    import gradslam_b200 as gs
    from gradslam_b200.slam import fusionutils as fu

    h, w = hw
    rgb, depth, K, poses, maps, counts = _scene(h, w)
    over = (counts > SMALL_CAP).flatten(1).any(1)
    s = next(f for f in range(1, L - 1) if over[f] and over[f + 1])  # frames s and s + 1 both overflow
    bin_cap(SMALL_CAP)
    frames = _frames(gs, rgb, depth, K, poses)
    slam = gs.PointFusion(odom="gt", device=DEV)
    pc = gs.Pointclouds(device=DEV)
    for f in range(s):
        pc, _ = slam.step(pc, frames[:, f], None, inplace=True)
    if path == "k2_overflow":
        _abandon(gs, pc, frames[:, s + 1])
    else:
        _abandon(gs, pc, frames[:, s + 1], table=fu.find_correspondences(pc, frames[:, s + 1], DIST_TH, DOT_TH))
    pc, _ = slam.step(pc, frames[:, s], None, inplace=True)
    _assert_matches(pc, maps[s + 1])


@pytest.mark.gpu
def test_fresh_call_after_failed_call_matches_oracle(bin_cap):
    """The error path with overflowing bins: a sequence call fails at an injected frame, and a fresh call on the same
    cached workspace equals the oracle.  The failure falls between frames, after K4 has restored every enqueued frame's
    state, so this does not exercise the per-call re-arm (the next test does)."""
    import gradslam_b200 as gs
    from gradslam_b200 import _C

    rgb, depth, K, poses, maps, counts = _scene()
    bin_cap(_mixed_cap(counts))
    frames = _frames(gs, rgb, depth, K, poses)
    slam = gs.PointFusion(odom="gt", device=DEV)
    _C.lib().gsx_debug_fail_at_frame(L - 2)
    with pytest.raises(RuntimeError, match="injected failure"):
        slam(frames)
    torch.cuda.synchronize()
    pc, _ = slam(frames)
    _assert_matches(pc, maps[L])


@pytest.mark.gpu
def test_sequence_call_after_dirty_workspace_matches_oracle(bin_cap):
    """A K2 with overflowing bins runs on the sequence driver's workspace and no K4 follows, leaving slots and bin
    counts dirty.  The next sequence call re-arms the workspace itself and equals the oracle; without the re-arm its
    first K4 would read the stale counts, bins and slots and merge into rows of the previous map."""
    import gradslam_b200 as gs
    from gradslam_b200 import _C
    from gradslam_b200.slam.pointfusion import _SequenceWorkspace

    rgb, depth, K, poses, maps, counts = _scene()
    bin_cap(SMALL_CAP)
    frames = _frames(gs, rgb, depth, K, poses)
    slam = gs.PointFusion(odom="gt", device=DEV)
    pc, _ = slam(frames)
    ws = _SequenceWorkspace.get(DEV, B, H, W)
    s = L - 1
    d = depth.to(DEV)[:, s].contiguous()
    pose = poses.to(DEV)[:, s].contiguous()
    Kd = K.to(DEV).contiguous()
    _C.launch("gsx_fusion_sequence_frame", d, H * W, Kd, 16, pose, 16, B, H, W, SIGMA, 0, ws.buf)
    _C.launch("gsx_fusion_project_select", pc._geo, pc._counts_dev[pc._cur], pc.capacity, pc.capacity, pose, 16, Kd,
              16, B, H, W, float(DIST_TH), float(DOT_TH), ws.buf)
    torch.cuda.synchronize()
    again, _ = slam(frames)
    _assert_matches(again, maps[L])


def test_sequence_workspace_is_one_frame_workspace():
    """The sequence driver needs one fusion workspace plus the frame headers of a block of frames (under 1 MB)."""
    from gradslam_b200 import _C

    lib = _C.lib()
    one = lib.gsx_fusion_workspace_bytes(8, 480, 640)
    seq = lib.gsx_pointfusion_sequence_workspace_bytes(8, 480, 640)
    assert one <= seq < one + (1 << 20)
    assert seq < 90_000_000
