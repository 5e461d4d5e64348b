"""Removal of unstable surfels (PointFusion's stable_confidence / max_unstable_age) against the creation-step oracle of
tests/prune_oracle.py, bit for bit: the whole-sequence call and the step API, a camera per element, batch groups, split
and host-fed calls, continuation through step(), an all-invalid frame, K4's capacity overflow, the in-place compaction
across many tiles, ICP odometry, the differentiable mode and its backward kernel, and the argument errors."""
import math

import pytest
import torch

import gsx_oracle as oracle
import prune_oracle as po
from cameras import camera_inputs
from gradslam_b200.synthetic import make_sequence

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _frames(gs, rgb, depth, K, poses):
    return gs.RGBDImages(rgb.to(DEV), depth.to(DEV), K.to(DEV), poses.to(DEV))


_cache = {}


def _case(B, L, H, W, kind="random", t_max=1, q=0.5, seed=7):
    """Inputs, a threshold at quantile q of the unpruned oracle map's confidences, and the pruned oracle map."""
    key = (B, L, H, W, kind, t_max, q, seed)
    if key not in _cache:
        if kind == "cameras":
            rgb, depth, K, poses = camera_inputs(B, L, H, W, seed, skew=0.75)
        else:
            rgb, depth, K, poses = make_sequence(B, L, H, W, seed=seed)
            if kind == "invalid_frame":
                depth[:, L // 2] = 0.0
        full = oracle.run_slam(rgb, depth, K, poses, odom="gt").map
        c = po.confidence_quantile(full, q)
        pm, _ = po.run_pointfusion(rgb, depth, K, poses, c_stable=c, t_max=t_max)
        assert sum(pm.counts()) < sum(full.counts())  # some rows are removed ...
        assert any(bool((cr <= L - 1 - t_max).any()) for cr in pm.created)  # ... and some tested rows are kept
        _cache[key] = (rgb, depth, K, poses, c, pm)
    return _cache[key]


def _assert_matches(pc, smap, n=None):
    assert [int(c) for c in pc.num_points_per_pointcloud.tolist()] == smap.counts()
    for b in range(len(smap.counts())):
        assert torch.equal(pc.points_list[b].detach().cpu(), smap.points[b]), b
        assert torch.equal(pc.normals_list[b].detach().cpu(), smap.normals[b]), b
        assert torch.equal(pc.colors_list[b].detach().cpu(), smap.colors[b]), b
        assert torch.equal(pc.features_list[b].detach().cpu(), smap.ccounts[b]), b


def _slam(gs, c, t_max, **kw):
    return gs.PointFusion(odom="gt", device=DEV, stable_confidence=c, max_unstable_age=t_max, **kw)


def _steps(slam, frames, L, pc=None, s_begin=0, inplace=True):
    import gradslam_b200 as gs

    pc = gs.Pointclouds(device=DEV) if pc is None else pc
    for s in range(s_begin, L):
        pc, _ = slam.step(pc, frames[:, s], None, inplace=inplace)
    return pc


@pytest.mark.parametrize("t_max", [0, 1, 3])
def test_sequence_and_steps_match_oracle(t_max):
    import gradslam_b200 as gs

    rgb, depth, K, poses, c, pm = _case(3, 6, 48, 64, t_max=t_max)
    frames = _frames(gs, rgb, depth, K, poses)
    slam = _slam(gs, c, t_max)
    whole, _ = slam(frames)
    _assert_matches(whole, pm.smap)
    assert whole._prune.step == 6
    _assert_matches(_steps(slam, frames, 6), pm.smap)


@pytest.mark.parametrize("kind", ["cameras", "invalid_frame"])
def test_camera_per_element_and_all_invalid_frame_match_oracle(kind):
    import gradslam_b200 as gs

    rgb, depth, K, poses, c, pm = _case(3, 6, 48, 64, kind=kind, t_max=1)
    frames = _frames(gs, rgb, depth, K, poses)
    slam = _slam(gs, c, 1)
    _assert_matches(slam(frames)[0], pm.smap)
    _assert_matches(_steps(slam, frames, 6), pm.smap)


@pytest.mark.parametrize("groups", [1, 2, 3, 4])
def test_batch_groups_match_oracle(groups, monkeypatch):
    """Each group prunes its own elements on its own stream, with its own ring column."""
    import gradslam_b200 as gs
    from gradslam_b200 import _C

    monkeypatch.setenv("GSX_SEQ_GROUPS", str(groups))
    assert _C.lib().gsx_pointfusion_sequence_groups(5) == groups
    rgb, depth, K, poses, c, pm = _case(5, 5, 48, 64, kind="cameras", t_max=1)
    whole, _ = _slam(gs, c, 1)(_frames(gs, rgb, depth, K, poses))
    _assert_matches(whole, pm.smap)


def test_split_and_host_fed_calls_equal_one_device_call():
    """Pinned host frames go in calls of four frames: the second call starts at frame 4 and continues the ring."""
    import gradslam_b200 as gs

    rgb, depth, K, poses, c, pm = _case(3, 7, 48, 64, t_max=3)
    slam = _slam(gs, c, 3)
    dev_pc, _ = slam(_frames(gs, rgb, depth, K, poses))
    host = gs.RGBDImages(rgb.pin_memory(), depth.pin_memory(), K.pin_memory(), poses.pin_memory())
    host_pc, _ = slam(host)
    _assert_matches(dev_pc, pm.smap)
    _assert_matches(host_pc, pm.smap)
    assert torch.equal(dev_pc._prune.ring, host_pc._prune.ring)


@pytest.mark.parametrize("inplace", [True, False])
def test_forward_then_steps_continue_the_history(inplace):
    import gradslam_b200 as gs

    rgb, depth, K, poses, c, pm = _case(3, 6, 48, 64, t_max=1)
    frames = _frames(gs, rgb, depth, K, poses)
    slam = _slam(gs, c, 1)
    half, _ = slam(frames[:, :3])
    out = _steps(slam, frames, 6, pc=half, s_begin=3, inplace=inplace)
    _assert_matches(out, pm.smap)
    if not inplace:  # the first half is untouched, history included
        assert half._prune.step == 3
        _assert_matches(half, po.run_pointfusion(rgb[:, :3], depth[:, :3], K, poses[:, :3], c_stable=c, t_max=1)[0].smap)


def test_t_max_mismatch_raises_before_any_launch():
    import gradslam_b200 as gs

    rgb, depth, K, poses, c, pm = _case(3, 6, 48, 64, t_max=1)
    frames = _frames(gs, rgb, depth, K, poses)
    pc, _ = _slam(gs, c, 1)(frames[:, :2])
    ring = pc._prune.ring.clone()
    counts = pc.num_points_per_pointcloud.clone()
    with pytest.raises(ValueError, match="max_unstable_age"):
        _slam(gs, c, 2).step(pc, frames[:, 2], None, inplace=True)
    assert torch.equal(pc._prune.ring, ring) and pc._prune.step == 2
    assert torch.equal(pc.num_points_per_pointcloud, counts)


def test_merge_overflow_keeps_the_oracle_prefix():
    """Storage too small for the last element's last frame: K4 clamps that element to the capacity and raises the flag;
    the prune then removes the window's rows (all below the capacity) and the element's rows equal the oracle's first
    rows.  The other elements equal the oracle."""
    import gradslam_b200 as gs

    B, L, H, W, t_max = 3, 3, 48, 64, 1
    rgb, depth, K, poses = make_sequence(B, L, H, W, seed=4)
    poses[B - 1, L - 1, :3, 3] += 5.0  # the last frame of the last element sees nothing of its map: all appended
    c = po.confidence_quantile(oracle.run_slam(rgb, depth, K, poses, odom="gt").map, 0.5)
    peak = [0] * B  # largest size of each element right after a K4, before the last frame
    pm = po.PrunedMap()
    for s in range(L):
        pm, _ = po.run_pointfusion(rgb[:, :s + 1], depth[:, :s + 1], K, poses[:, :s + 1], pm=pm, s_begin=s)
        if s < L - 1:
            peak = [max(p, n) for p, n in zip(peak, pm.counts())]
        else:
            peak[:B - 1] = [max(p, n) for p, n in zip(peak[:B - 1], pm.counts()[:B - 1])]
            before_last = pm.counts()[B - 1]
        po.prune_step(pm, c, t_max)
    low = max(peak)
    cap = (low + before_last) // 2
    assert low < cap < before_last
    geo = torch.empty((B, cap, 8), dtype=torch.float32, device=DEV)
    col = torch.empty((B, cap, 4), dtype=torch.float32, device=DEV)
    out = gs.Pointclouds()
    out._attach(geo, col)
    pc, _ = _slam(gs, c, t_max)(_frames(gs, rgb, depth, K, poses), out=out)
    counts = [int(n) for n in pc.num_points_per_pointcloud.tolist()]
    with pytest.raises(RuntimeError, match="capacity exceeded"):
        pc.points_list
    assert counts[:B - 1] == pm.counts()[:B - 1] and counts[B - 1] < pm.counts()[B - 1]
    for b in range(B):
        n = counts[b]
        assert torch.equal(geo[b, :n, 0:3].cpu(), pm.smap.points[b][:n]), b
        assert torch.equal(geo[b, :n, 3:6].cpu(), pm.smap.normals[b][:n]), b
        assert torch.equal(geo[b, :n, 6:7].cpu(), pm.smap.ccounts[b][:n]), b
        assert torch.equal(col[b, :n, 0:3].cpu(), pm.smap.colors[b][:n]), b


_big = {}


def _big_case(t_max):
    """640x480 inputs, the unpruned oracle map, and a threshold that removes some but not all of the first 512 rows of
    the first window (the rows of step 0, tested at step t_max; nothing is removed before, so they are rows 0..511)."""
    if not _big:
        B, L, H, W = 2, 6, 480, 640
        rgb, depth, K, poses = make_sequence(B, L, H, W, seed=11)
        pm, _ = po.run_pointfusion(rgb[:, :t_max + 1], depth[:, :t_max + 1], K, poses[:, :t_max + 1])
        first = pm.smap.ccounts[0][:512, 0]
        c = po.confidence_quantile(pm.smap, 0.5)
        if not bool((first < c).any()) or bool((first < c).all()):
            c = float(first.double().median())
        assert bool((first < c).any()) and not bool((first < c).all())
        pm, _ = po.run_pointfusion(rgb, depth, K, poses, pm=pm, s_begin=t_max + 1)
        _big.update(inputs=(rgb, depth, K, poses), full=pm.smap, c=c)
    return _big["inputs"], _big["full"], _big["c"]


@pytest.mark.parametrize("which", ["some", "none", "all"])
def test_in_place_compaction_across_many_tiles(which):
    """640x480: a window holds ~10^5 rows per element, hundreds of 512-row tiles.  'some': a threshold that removes rows
    in the window's first tile, so every later tile moves its rows across tile boundaries; 'none' removes nothing (no
    row is stored); 'all' removes every tested row."""
    import gradslam_b200 as gs

    t_max = 2
    (rgb, depth, K, poses), full, c_some = _big_case(t_max)
    c = {"some": c_some, "none": 0.0, "all": math.inf}[which]
    ref = full if which == "none" else po.run_pointfusion(rgb, depth, K, poses, c_stable=c, t_max=t_max)[0].smap
    frames = _frames(gs, rgb, depth, K, poses)
    slam = _slam(gs, c, t_max)
    _assert_matches(slam(frames)[0], ref)
    _assert_matches(_steps(slam, frames, depth.shape[1]), ref)


@pytest.mark.parametrize("odom", ["icp", "gradicp"])
@pytest.mark.parametrize("association", ["nn", "projective"])
def test_icp_odometry_with_pruning(odom, association):
    import gradslam_b200 as gs

    # (the projective association is a z-buffer decision: the inputs and ICP settings of the unpruned projective SLAM
    # test, tests/test_gpu_projective_icp.py, where the poses stay within the tolerance of the oracle's)
    B, L, H, W = (2, 4, 48, 64) if association == "nn" else (3, 4, 48, 64)
    if association == "nn":
        rgb, depth, K, poses = make_sequence(B, L, H, W, seed=9)
        icp = dict(numiters=20, dsratio=4)
    else:
        rgb, depth, K, poses = camera_inputs(B, L, H, W, 63, skew=0.75)
        icp = dict(numiters=10, dsratio=2)
    c = po.confidence_quantile(oracle.run_slam(rgb, depth, K, poses, odom="gt").map, 0.5)
    pm, ref_poses = po.run_pointfusion(rgb, depth, K, poses, c_stable=c, t_max=1, odom=odom, association=association,
                                       **icp)
    slam = gs.PointFusion(odom=odom, association=association, device=DEV, stable_confidence=c, max_unstable_age=1,
                          **icp)
    pc, got_poses = slam(_frames(gs, rgb, depth, K, poses))
    torch.testing.assert_close(got_poses.cpu(), ref_poses, rtol=0, atol=1e-4)
    # the map, bit for bit, against the oracle fused and pruned at the recovered poses: a merge decision may flip under a
    # pose 1e-6 away (one row of projective-icp lands 4.8e-3 from the oracle-ICP map's), so exactness is checked there
    _assert_matches(pc, po.run_pointfusion(rgb, depth, K, got_poses.cpu(), c_stable=c, t_max=1)[0].smap)
    if association == "nn":
        assert [int(n) for n in pc.num_points_per_pointcloud.tolist()] == pm.counts()
        for b in range(B):
            torch.testing.assert_close(pc.points_list[b].cpu(), pm.smap.points[b], rtol=0, atol=1e-3)
            torch.testing.assert_close(pc.features_list[b].cpu(), pm.smap.ccounts[b], rtol=0, atol=1e-3)


def test_differentiable_mode_values_and_gradients_match_oracle():
    """With depth and colours that require grad: the map equals the no-grad call bit for bit, and d(map)/d(depth,
    colours) matches the oracle's autograd, where the removal is an index_select."""
    import gradslam_b200 as gs

    B, L, H, W, t_max = 2, 3, 24, 32, 1
    rgb, depth, K, poses = make_sequence(B, L, H, W, seed=41, yaw0=0.6)
    c = po.confidence_quantile(oracle.run_slam(rgb, depth, K, poses, odom="gt").map, 0.5)
    d_ref, c_ref = depth.clone().requires_grad_(True), rgb.clone().requires_grad_(True)
    pm, _ = po.run_pointfusion(c_ref, d_ref, K, poses, c_stable=c, t_max=t_max)
    counts = pm.counts()
    g = torch.Generator().manual_seed(5)
    ws = [[torch.randn(n, k, generator=g) for k in (3, 3, 1)] for n in counts]
    sum((t * w).sum() for b in range(B) for t, w in zip((pm.smap.points[b], pm.smap.colors[b], pm.smap.ccounts[b]),
                                                          ws[b])).backward()

    d_gpu, c_gpu = depth.clone().to(DEV).requires_grad_(True), rgb.clone().to(DEV).requires_grad_(True)
    slam = _slam(gs, c, t_max)
    pc, _ = slam(gs.RGBDImages(c_gpu, d_gpu, K.to(DEV), poses.to(DEV)))
    with torch.no_grad():
        ng, _ = slam(_frames(gs, rgb, depth, K, poses))
    _assert_matches(ng, oracle.SurfelMap(*([x.detach() for x in lst] for lst in (
        pm.smap.points, pm.smap.normals, pm.smap.colors, pm.smap.ccounts))))
    assert [int(n) for n in pc.num_points_per_pointcloud.tolist()] == counts
    for b in range(B):
        for key in ("points", "normals", "colors", "features"):
            assert torch.equal(getattr(pc, key + "_list")[b].detach(), getattr(ng, key + "_list")[b]), (b, key)
    sum((t * w.to(DEV)).sum() for b in range(B) for t, w in zip((pc.points_list[b], pc.colors_list[b],
                                                                 pc.features_list[b]), ws[b])).backward()
    for got, want in ((d_gpu.grad.cpu(), d_ref.grad), (c_gpu.grad.cpu(), c_ref.grad)):
        assert torch.isfinite(got).all()
        torch.testing.assert_close(got, want, rtol=1e-3, atol=1e-4 * want.abs().max().item())


def test_differentiable_prune_wrt_previous_map():
    """prune_unstable on a map that requires grad: d(pruned map)/d(previous rows) is the gather keep_map describes."""
    import gradslam_b200 as gs
    from gradslam_b200.slam import fusionutils as fu

    B, H, W = 2, 20, 28
    rgb, depth, K, poses = make_sequence(B, 1, H, W, seed=43)
    with torch.no_grad():
        base = fu.update_map_fusion(gs.Pointclouds(device=DEV), _frames(gs, rgb, depth, K, poses)[:, 0], 0.05, 0.94, 0.6)
    n0 = base.num_points_per_pointcloud.tolist()
    leaves = {k: getattr(base, k + "_padded").clone().requires_grad_(True) for k in ("points", "normals", "colors",
                                                                                     "features")}
    pc = gs.Pointclouds(leaves["points"], leaves["normals"], leaves["colors"], leaves["features"])
    pc._set_counts(n0)
    c = float(leaves["features"].detach()[0, : n0[0]].median())
    fu.prune_unstable(pc, c, 0)  # a map without history: every row is in the window
    n1 = pc.num_points_per_pointcloud.tolist()
    assert 0 < n1[0] < n0[0]
    g = torch.Generator().manual_seed(3)
    wts = {k: torch.randn(B, max(n1), ch, generator=g).to(DEV) for k, ch in (("points", 3), ("normals", 3),
                                                                              ("colors", 3), ("features", 1))}
    mask = pc.nonpad_mask.unsqueeze(-1)
    sum((getattr(pc, k + "_padded") * wts[k] * mask).sum() for k in wts).backward()
    for b in range(B):
        keep = torch.nonzero(leaves["features"].detach()[b, : n0[b], 0] >= torch.tensor(c, dtype=torch.float32,
                                                                                         device=DEV)).flatten()
        for k in leaves:
            want = torch.zeros_like(leaves[k][b])
            want[keep] = wts[k][b, : keep.numel()]
            assert torch.equal(leaves[k].grad[b], want), (b, k)


@pytest.mark.parametrize("B,cap", [(3, 70001), (2, 5 * 512 + 17)])
def test_backward_kernel_matches_float64_gather(B, cap):
    """gsx_fusion_prune_unstable_bwd against float64 autograd of the gather, at large and ragged sizes, with one element
    whose window is empty (rows before the window pass through)."""
    from gradslam_b200 import _C
    from gradslam_b200.slam.fusionutils import _prune_scratch

    g = torch.Generator().manual_seed(B)
    counts = [cap - 5, cap // 3, 0][:B]
    geo = torch.rand(B, cap, 8, generator=g)
    geo[..., 7] = 0
    geo[:, ::7, 6] = 0.5  # confidence equal to the threshold: kept
    col = torch.rand(B, cap, 4, generator=g)
    col[..., 3] = 0
    t_max, step = 1, 2  # window [ring(0), ring(1))
    ring = torch.zeros(t_max + 2, B, dtype=torch.int32)
    ring[0] = torch.tensor([counts[0] // 4, counts[1], 0][:B], dtype=torch.int32)  # element 1: empty window
    ring[1] = torch.tensor(counts, dtype=torch.int32)
    geo_d, col_d, ring_d = geo.to(DEV), col.to(DEV), ring.to(DEV)
    cnt = torch.tensor(counts, dtype=torch.int32, device=DEV)
    keep_map = torch.arange(cap, dtype=torch.int32, device=DEV).repeat(B, 1)
    scratch = _prune_scratch(B, cap, DEV)
    _C.launch("gsx_fusion_prune_unstable", geo_d, col_d, cnt, cap, ring_d, t_max + 2, step, t_max, 0.5, B, keep_map,
              scratch, scratch.numel())
    g_geo, g_col = torch.randn(B, cap, 8, generator=g), torch.randn(B, cap, 4, generator=g)
    d_geo = torch.empty(B, cap, 8, device=DEV)
    d_col = torch.empty(B, cap, 4, device=DEV)
    cin = torch.tensor(counts, dtype=torch.int32, device=DEV)
    _C.launch("gsx_fusion_prune_unstable_bwd", keep_map, cin, cap, g_geo.to(DEV), g_col.to(DEV), cap, B, d_geo, d_col)
    for b in range(B):
        x64 = torch.cat([geo[b], col[b]], 1).double().requires_grad_(True)
        n = torch.arange(cap)
        ws = int(ring[0, b])
        keep = torch.nonzero((n < counts[b]) & ~((n >= ws) & (n < counts[b]) & (geo[b, :, 6] < 0.5))).flatten()
        assert int(cnt[b]) == keep.numel()
        y = x64.index_select(0, keep)
        up = torch.cat([g_geo[b], g_col[b]], 1).double()
        up[:, 7] = 0
        up[:, 11] = 0
        (y * up[: keep.numel()]).sum().backward()
        torch.testing.assert_close(torch.cat([d_geo[b], d_col[b]], 1).cpu().double(), x64.grad, rtol=0, atol=0)
        assert torch.equal(geo_d[b, : keep.numel()].cpu(), geo[b, keep])
        assert torch.equal(col_d[b, : keep.numel()].cpu(), col[b, keep])
