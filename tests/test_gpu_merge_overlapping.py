"""Merging of overlapping surfels (PointFusion(merge_overlapping=True), fusionutils.fuse_and_prune) against the oracle of
tests/merge_oracle.py, bit for bit in every geometry slot, the colours, the counts and the ring: the whole-sequence call
and the step API for t_max 0 and 4 with and without a free-space margin, a camera per element, batch groups 1-4, split
and host-fed calls that continue the ring, continuation through step(), 640x480, ICP odometry, and the differentiable
mode's values and gradients end to end and, over every channel, as an op against float64 autograd of the absorption.
Every case checks that the oracle absorbed rows."""
import pytest
import torch

import gsx_oracle as oracle
import merge_oracle as mo
import prune_oracle as po
from cameras import camera_inputs
from gradslam_b200.synthetic import make_dynamic_sequence

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _frames(gs, rgb, depth, K, poses):
    return gs.RGBDImages(rgb.to(DEV), depth.to(DEV), K.to(DEV), poses.to(DEV))


_inputs = {}


def _scene(kind, B=3, L=10, H=48, W=64):
    key = (kind, B, L, H, W)
    if key not in _inputs:
        if kind == "cameras":
            rgb, depth, K, poses = camera_inputs(B, L, H, W, 23, skew=0.75)
        else:
            rgb, depth, K, poses = make_dynamic_sequence(B, L, H, W, 2, 5, seed=5)
        c = po.confidence_quantile(oracle.run_slam(rgb, depth, K, poses, odom="gt").map, 0.25)
        _inputs[key] = (rgb, depth, K, poses, c)
    return _inputs[key]


_refs = {}


def _ref(kind, t_max, margin, **shape):
    key = (kind, t_max, margin, tuple(sorted(shape.items())))
    if key not in _refs:
        rgb, depth, K, poses, c = _scene(kind, **shape)
        pm, radii, _, absorbed = mo.run_pointfusion(rgb, depth, K, poses, c_stable=c, t_max=t_max, margin=margin)
        assert min(absorbed) > 0, absorbed
        _refs[key] = (pm, radii)
    return _refs[key]


def _assert_matches(pc, pm, radii):
    smap = pm.smap
    assert [int(c) for c in pc.num_points_per_pointcloud.tolist()] == smap.counts()
    for b in range(len(smap.counts())):
        assert torch.equal(pc.points_list[b].detach().cpu(), smap.points[b]), b
        assert torch.equal(pc.normals_list[b].detach().cpu(), smap.normals[b]), b
        assert torch.equal(pc.colors_list[b].detach().cpu(), smap.colors[b]), b
        assert torch.equal(pc.features_list[b].detach().cpu(), smap.ccounts[b]), b
        assert torch.equal(pc.radii_list[b].detach().cpu(), radii[b]), b


def _assert_ring(pc, pm, t_max):
    """Rows are in creation order, so ring(k) = the number of rows created at or before step k."""
    h = pc._prune
    ring = h.ring.cpu()
    assert h.step == pm.step
    for k in range(max(h.step - 1 - t_max, 0), h.step):
        for b in range(len(pm.counts())):
            assert int(ring[k % (t_max + 2), b]) == int((pm.created[b] <= k).sum()), (k, b)


def _slam(gs, c, t_max, margin, **kw):
    return gs.PointFusion(odom="gt", device=DEV, stable_confidence=c, max_unstable_age=t_max, free_space_margin=margin,
                          surfel_radii=True, merge_overlapping=True, **kw)


def _steps(slam, frames, L, pc=None, s_begin=0, inplace=True):
    import gradslam_b200 as gs

    pc = gs.Pointclouds(device=DEV) if pc is None else pc
    for s in range(s_begin, L):
        pc, _ = slam.step(pc, frames[:, s], None, inplace=inplace)
    return pc


@pytest.mark.parametrize("t_max,margin", [(0, None), (0, 0.05), (4, None), (4, 0.05)])
def test_sequence_and_steps_match_oracle(t_max, margin):
    import gradslam_b200 as gs

    rgb, depth, K, poses, c = _scene("dynamic")
    pm, radii = _ref("dynamic", t_max, margin)
    frames = _frames(gs, rgb, depth, K, poses)
    slam = _slam(gs, c, t_max, margin)
    whole, _ = slam(frames)
    _assert_matches(whole, pm, radii)
    _assert_ring(whole, pm, t_max)
    stepped = _steps(slam, frames, depth.shape[1])
    _assert_matches(stepped, pm, radii)
    _assert_ring(stepped, pm, t_max)


def test_a_camera_per_element_matches_oracle():
    import gradslam_b200 as gs

    rgb, depth, K, poses, c = _scene("cameras")
    assert len(set(K[:, 0, 0, 0].tolist())) == 3
    pm, radii = _ref("cameras", 4, 0.05)
    frames = _frames(gs, rgb, depth, K, poses)
    slam = _slam(gs, c, 4, 0.05)
    _assert_matches(slam(frames)[0], pm, radii)
    _assert_matches(_steps(slam, frames, depth.shape[1]), pm, radii)


@pytest.mark.parametrize("groups", [1, 2, 3, 4])
def test_batch_groups_match_oracle(groups, monkeypatch):
    import gradslam_b200 as gs
    from gradslam_b200 import _C

    monkeypatch.setenv("GSX_SEQ_GROUPS", str(groups))
    assert _C.lib().gsx_pointfusion_sequence_groups(5) == groups
    rgb, depth, K, poses, c = _scene("dynamic", B=5, L=7)
    pm, radii = _ref("dynamic", 4, 0.05, B=5, L=7)
    whole, _ = _slam(gs, c, 4, 0.05)(_frames(gs, rgb, depth, K, poses))
    _assert_matches(whole, pm, radii)
    _assert_ring(whole, pm, 4)


def test_split_host_fed_calls_continue_the_ring():
    """Pinned host frames go in calls of four frames: later calls start at frames 4 and 8 and continue the ring."""
    import gradslam_b200 as gs

    rgb, depth, K, poses, c = _scene("dynamic")
    pm, radii = _ref("dynamic", 4, None)
    host = gs.RGBDImages(rgb.pin_memory(), depth.pin_memory(), K.pin_memory(), poses.pin_memory())
    pc, _ = _slam(gs, c, 4, None)(host)
    _assert_matches(pc, pm, radii)
    _assert_ring(pc, pm, 4)


@pytest.mark.parametrize("inplace", [True, False])
def test_forward_then_steps_continue_the_history(inplace):
    import gradslam_b200 as gs

    rgb, depth, K, poses, c = _scene("dynamic")
    L = depth.shape[1]
    pm, radii = _ref("dynamic", 4, 0.05)
    frames = _frames(gs, rgb, depth, K, poses)
    slam = _slam(gs, c, 4, 0.05)
    half, _ = slam(frames[:, : L // 2])
    out = _steps(slam, frames, L, pc=half, s_begin=L // 2, inplace=inplace)
    _assert_matches(out, pm, radii)
    _assert_ring(out, pm, 4)


def test_full_size_matches_oracle():
    """640x480, B = 2: absorbed rows far below the age window, hundreds of compaction tiles per element."""
    import gradslam_b200 as gs

    shape = dict(B=2, L=4, H=480, W=640)
    rgb, depth, K, poses, c = _scene("dynamic", **shape)
    pm, radii = _ref("dynamic", 1, 0.05, **shape)
    frames = _frames(gs, rgb, depth, K, poses)
    slam = _slam(gs, c, 1, 0.05)
    _assert_matches(slam(frames)[0], pm, radii)
    _assert_matches(_steps(slam, frames, 4), pm, radii)


def test_merge_off_keeps_every_other_entry_point():
    """merge_overlapping=False through the new entry points is the free-space run with radii, ring included."""
    import gradslam_b200 as gs

    rgb, depth, K, poses, c = _scene("dynamic")
    frames = _frames(gs, rgb, depth, K, poses)
    kw = dict(odom="gt", device=DEV, stable_confidence=c, max_unstable_age=4, free_space_margin=0.05, surfel_radii=True)
    a, _ = gs.PointFusion(**kw)(frames)
    b, _ = gs.PointFusion(merge_overlapping=False, **kw)(frames)
    m, _ = gs.PointFusion(merge_overlapping=True, **kw)(frames)
    for key in ("points", "normals", "colors", "features", "radii"):
        for x, y in zip(getattr(a, key + "_list"), getattr(b, key + "_list")):
            assert torch.equal(x, y), key
    assert torch.equal(a._prune.ring, b._prune.ring)
    assert int(m.num_points_per_pointcloud.sum()) < int(a.num_points_per_pointcloud.sum())


@pytest.mark.parametrize("odom,association", [("icp", "nn"), ("gradicp", "projective")])
def test_icp_odometry_with_merging(odom, association):
    import gradslam_b200 as gs

    B, L, H, W = 2, 6, 48, 64
    rgb, depth, K, poses = make_dynamic_sequence(B, L, H, W, 1, 3, seed=9, yaw0=0.6)
    icp = dict(numiters=20, dsratio=4) if association == "nn" else dict(numiters=10, dsratio=2)
    c = po.confidence_quantile(oracle.run_slam(rgb, depth, K, poses, odom="gt").map, 0.25)
    slam = gs.PointFusion(odom=odom, association=association, device=DEV, stable_confidence=c, max_unstable_age=1,
                          free_space_margin=0.0, surfel_radii=True, merge_overlapping=True, **icp)
    pc, got_poses = slam(_frames(gs, rgb, depth, K, poses))
    # bit for bit against the oracle fused and pruned at the recovered poses (a decision may flip under a pose 1e-6 away)
    pm, radii, _, absorbed = mo.run_pointfusion(rgb, depth, K, got_poses.cpu(), c_stable=c, t_max=1, margin=0.0)
    assert min(absorbed) > 0
    _assert_matches(pc, pm, radii)


def test_differentiable_mode_values_and_gradients_match_oracle():
    """With depth and colours that require grad: the map equals the oracle's bit for bit, d(map)/d(depth, colours)
    matches the oracle's autograd (where the absorption is separate float32 ops), and two runs give the same bytes."""
    import gradslam_b200 as gs

    B, L, H, W, t_max, margin = 2, 5, 24, 32, 1, 0.0
    rgb, depth, K, poses = make_dynamic_sequence(B, L, H, W, 1, 3, seed=41, yaw0=0.3)
    c = po.confidence_quantile(oracle.run_slam(rgb, depth, K, poses, odom="gt").map, 0.25)
    d_ref, c_ref = depth.clone().requires_grad_(True), rgb.clone().requires_grad_(True)
    pm, radii, _, absorbed = mo.run_pointfusion(c_ref, d_ref, K, poses, c_stable=c, t_max=t_max, margin=margin)
    assert min(absorbed) > 0
    counts = pm.counts()
    g = torch.Generator().manual_seed(5)
    ws = [[torch.randn(n, k, generator=g) for k in (3, 3, 1)] for n in counts]
    sum((t * w).sum() for b in range(B) for t, w in zip((pm.smap.points[b], pm.smap.colors[b], pm.smap.ccounts[b]),
                                                          ws[b])).backward()

    grads = []
    for _ in range(2):
        d_gpu, c_gpu = depth.clone().to(DEV).requires_grad_(True), rgb.clone().to(DEV).requires_grad_(True)
        pc, _ = _slam(gs, c, t_max, margin)(gs.RGBDImages(c_gpu, d_gpu, K.to(DEV), poses.to(DEV)))
        _assert_matches(pc, po.PrunedMap(oracle.SurfelMap(*([x.detach() for x in lst] for lst in (
            pm.smap.points, pm.smap.normals, pm.smap.colors, pm.smap.ccounts)))), radii)
        sum((t * w.to(DEV)).sum() for b in range(B) for t, w in zip((pc.points_list[b], pc.colors_list[b],
                                                                     pc.features_list[b]), ws[b])).backward()
        grads.append((d_gpu.grad.cpu(), c_gpu.grad.cpu()))
    for x, y in zip(*grads):
        assert torch.equal(x, y)
    for got, want in zip(grads[0], (d_ref.grad, c_ref.grad)):
        assert torch.isfinite(got).all()
        torch.testing.assert_close(got, want, rtol=1e-3, atol=1e-4 * want.abs().max().item())


def test_prune_merge_op_gradient_matches_float64_absorb_and_gather():
    """The pruned step with merging as an op on map rows that require grad: over every channel (position, normal,
    colour, confidence), d(loss)/d(rows) of gsx_fusion_prune_merge_bwd against float64 autograd of
    merge_oracle.absorb on the GPU's pairs followed by the keep_map gather; the forward rows equal the same absorption
    in float32 bit for bit."""
    import gradslam_b200 as gs
    from gradslam_b200.slam import fusionutils as fu

    rgb, depth, K, poses, c = _scene("dynamic")
    L = depth.shape[1]
    frames = _frames(gs, rgb, depth, K, poses)
    slam = _slam(gs, c, 4, 0.05)
    pc = _steps(slam, frames, L - 1)
    live = frames[:, L - 1]
    got = []
    fu._fuse(pc, live, slam.sigma, slam.dist_th, slam.dot_th, assoc_out=got, radii=True)
    lc = live.to_channels_last()
    free_space = (got[0], lc.intrinsics.contiguous(), lc.poses.contiguous(), depth.shape[2], depth.shape[3], 0.05)
    counts_in = [int(x) for x in pc._counts_dev[pc._cur].tolist()]
    geo0, col0 = pc._geo.detach().clone(), pc._col.detach().clone()
    pc._geo, pc._col = geo0.clone().requires_grad_(True), col0.clone().requires_grad_(True)
    leaves = (pc._geo, pc._col)
    fu._prune(pc, c, 4, free_space, slam.dot_th)
    keep_map, _, pairs, _, _ = pc._geo.grad_fn.saved
    assert pairs.shape[0] > 0
    B, cap = geo0.shape[0], geo0.shape[1]
    counts_out = [int(x) for x in pc._counts_dev[pc._cur].tolist()]
    gen = torch.Generator().manual_seed(11)
    up_geo, up_col = torch.randn(B, cap, 8, generator=gen), torch.randn(B, cap, 4, generator=gen)
    up_geo[..., 7] = 0
    up_col[..., 3] = 0
    for b in range(B):
        up_geo[b, counts_out[b]:] = 0
        up_col[b, counts_out[b]:] = 0
    ((pc._geo * up_geo.to(DEV)).sum() + (pc._col * up_col.to(DEV)).sum()).backward()
    d_geo, d_col = leaves[0].grad.cpu(), leaves[1].grad.cpu()
    pairs, keep_map = pairs.cpu().long(), keep_map.cpu().long()
    out_geo, out_col = pc._geo.detach().cpu(), pc._col.detach().cpu()
    normal_grads = 0
    for b in range(B):
        n_in = counts_in[b]
        pb = pairs[pairs[:, 0] == b][:, 1:]
        keep = keep_map[b, :n_in]
        kept = torch.nonzero(keep >= 0).flatten()
        assert keep[kept].tolist() == list(range(counts_out[b]))
        for dtype in (torch.float32, torch.float64):
            x = geo0[b, :n_in].cpu().to(dtype).requires_grad_(True)
            y = col0[b, :n_in].cpu().to(dtype).requires_grad_(True)
            smap = oracle.SurfelMap([x[:, 0:3]], [x[:, 3:6]], [y[:, 0:3]], [x[:, 6:7]])
            new, radii = mo.absorb(smap, [x[:, 7:8].detach()], [pb])
            rows = torch.cat([new.points[0], new.normals[0], new.ccounts[0], radii[0]], 1)[kept]
            cols = new.colors[0][kept]
            if dtype == torch.float32:  # the forward, bit for bit
                assert torch.equal(rows, out_geo[b, : counts_out[b]]), b
                assert torch.equal(cols, out_col[b, : counts_out[b], :3]), b
                continue
            ((rows * up_geo[b, : counts_out[b]].double()).sum() +
             (cols * up_col[b, : counts_out[b], :3].double()).sum()).backward()
            # float32 against float64: the confidence slot sums terms of size |G| |x_m - x_n| / c with c ~ 1e-6
            torch.testing.assert_close(d_geo[b, :n_in].double(), x.grad, rtol=1e-4, atol=1e-5 * x.grad.abs().max())
            torch.testing.assert_close(d_col[b, :n_in].double(), y.grad, rtol=1e-4, atol=1e-5 * y.grad.abs().max())
            assert bool((d_geo[b, n_in:] == 0).all()) and bool((d_col[b, :, 3] == 0).all())
            normal_grads += int((x.grad[pb[:, 0], 3:6] != 0).any(1).sum())
    assert normal_grads > 0
