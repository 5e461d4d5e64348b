"""Batched kernels with a camera of its own per batch element (tests/golden/cameras.py: per-element fx != fy, principal
point, skew K[0,1] and 4th column K[0:2,3], trajectory), where an element that read another element's camera gives
different bits: the three correspondence tables, ICP localisation (the fused gathers of gsx_icp_localize against the
differentiable path's K1 + find_active_map_points + downsampling), and the renderer past one 32-view chunk."""
import math
import os

import numpy as np
import pytest
import torch

import gsx_oracle as oracle
import render_oracle
from cameras import TABLES_CASE, camera_inputs, camera_intrinsics, frozen_table
from test_gpu_render import _canonical_z

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
GOLD = os.path.join(os.path.dirname(__file__), "golden")
DOT_TH = math.cos(20 * math.pi / 180)


def test_tables_with_per_element_cameras_match_oracle_and_frozen_reference():
    """find_active_map_points / find_similar_map_points / find_best_unique_correspondences of one fusion step, B=3,
    with skew and the 4th column set: bit for bit against the oracle and the tables frozen from the reference."""
    import gradslam_b200 as gs
    from gradslam_b200.slam import fusionutils as fu

    c = TABLES_CASE
    B, H, W = c["B"], c["H"], c["W"]
    rgb, depth, K, poses = camera_inputs(B, c["L"], H, W, c["seed"], skew=c["skew"])
    frames = gs.RGBDImages(rgb.to(DEV), depth.to(DEV), K.to(DEV), poses.to(DEV))
    pc = gs.Pointclouds(device=DEV)
    smap = oracle.SurfelMap()
    for s in range(2):
        pc = fu.update_map_fusion(pc, frames[:, s], 0.05, DOT_TH, 0.6, inplace=True)
        m = oracle.frame_maps(depth[:, s:s + 1], K, poses[:, s:s + 1])
        smap = oracle.update_map_fusion(smap, m, rgb[:, s:s + 1], poses[:, s], K[:, 0], 0.05, DOT_TH, 0.6)
    assert pc.num_points_per_pointcloud.tolist() == smap.counts()
    live = frames[:, 2]
    maps = oracle.frame_maps(depth[:, 2:3], K, poses[:, 2:3])
    gv, gn = maps["gvertex"][:, 0], maps["gnormal"][:, 0]
    active = fu.find_active_map_points(pc, live).cpu()
    r_active = oracle.find_active_map_points(smap, poses[:, 2], K[:, 0], H, W)
    assert torch.equal(active, r_active)
    assert torch.equal(torch.unique(active[:, 0]), torch.arange(B))
    similar, mask = fu.find_similar_map_points(pc, live, active.to(DEV), 0.05, DOT_TH)
    r_similar, r_mask = oracle.find_similar_map_points(smap, gv, gn, r_active, 0.05, DOT_TH)
    assert torch.equal(similar.cpu(), r_similar) and torch.equal(mask.cpu(), r_mask)
    unique = fu.find_best_unique_correspondences(pc, live, similar).cpu()
    assert torch.equal(unique, oracle.find_best_unique_correspondences(smap, gv, r_similar))
    ref = np.load(os.path.join(GOLD, "ref_cameras.npz"))
    for name, t in (("active", active), ("similar", similar.cpu()), ("unique", unique)):
        assert torch.equal(t, frozen_table(ref, name)), name


@pytest.mark.parametrize("odom", ["icp", "gradicp"])
def test_icp_localisation_fused_equals_differentiable_path(odom):
    """ICPSLAM, B=3, a camera per element: the fused call (k_icp_gather_src / k_icp_gather_tgt gather the ICP clouds)
    and the differentiable path (K1 + find_active_map_points + downsample_*) recover bit-identical poses, both within
    1e-4 of the oracle."""
    import gradslam_b200 as gs

    B, L, H, W = 3, 3, 48, 64
    rgb, depth, K, poses = camera_inputs(B, L, H, W, 71, skew=0.75)
    slam = gs.ICPSLAM(odom=odom, numiters=5, dsratio=2, device=DEV)
    with torch.no_grad():
        _, fused = slam(gs.RGBDImages(rgb.to(DEV), depth.to(DEV), K.to(DEV), poses.to(DEV)))
    d = depth.to(DEV).requires_grad_(True)
    _, diff = slam(gs.RGBDImages(rgb.to(DEV), d, K.to(DEV), poses.to(DEV)))
    assert diff.requires_grad
    assert torch.equal(diff.detach(), fused), (diff.detach() - fused).abs().max().item()
    ref = oracle.run_slam(rgb, depth, K, poses, mode="aggregate", odom=odom, numiters=5, dsratio=2)
    torch.testing.assert_close(fused.cpu(), ref.poses, rtol=0, atol=1e-4)
    assert (fused.cpu() - poses).abs().max() > 1e-3  # the poses are recovered, not copied from the input


# ---------------------------------------------------------------------------------------------- renderer, L > 32 views
VIEWS_PER_CTA = 32     # kViews in gsx_render.cu
R1_CTA_CAP = 132 * 8   # kNumSMs * kRenderCtasPerSM
_render_cache = {}


def _fused_map_and_views(L):
    """A map fused on the GPU from camera_inputs(3, 2, 240, 320) (~10^5 rows per element), rendered at 48x64 through
    each element's skewed K from L views near its two frames, each view its own pose."""
    import gradslam_b200 as gs

    if "map" not in _render_cache:
        rgb, depth, K, poses = camera_inputs(3, 2, 240, 320, 61)
        pc, _ = gs.PointFusion(odom="gt", device=DEV)(gs.RGBDImages(rgb.to(DEV), depth.to(DEV), K.to(DEV),
                                                                    poses.to(DEV)))
        _render_cache["map"] = (pc, poses)
    pc, poses = _render_cache["map"]
    views = torch.empty(3, L, 4, 4, dtype=torch.float64)
    for b in range(3):
        for l in range(L):
            a = 0.002 * l - 0.06
            turn = torch.eye(4, dtype=torch.float64)
            turn[0, 0], turn[0, 2], turn[2, 0], turn[2, 2] = math.cos(a), math.sin(a), -math.sin(a), math.cos(a)
            turn[:3, 3] = torch.tensor([0.001 * l, -0.0005 * l, 0.0])
            views[b, l] = poses[b, l % 2].double() @ turn
    K = torch.from_numpy(camera_intrinsics(3, 48, 64, skew=0.75)).float().view(3, 1, 4, 4)
    return pc, K, views.float()


def _oracle_map(pc):
    return oracle.SurfelMap([p.detach().cpu() for p in pc.points_list], [n.detach().cpu() for n in pc.normals_list],
                            [c.detach().cpu() for c in pc.colors_list], [f.detach().cpu() for f in pc.features_list])


def _assert_r1_strides_in_every_chunk(pc, L):
    chunks = -(-L // VIEWS_PER_CTA)
    rows_per_pass = -(-R1_CTA_CAP // (3 * chunks)) * 256
    assert min(pc.num_points_per_pointcloud.tolist()) > rows_per_pass, "R1 would not grid-stride"


@pytest.mark.parametrize("L", [33, 70])
def test_render_past_one_view_chunk_matches_oracle(L):
    """B=3, L=33 (one partial second chunk) and L=70 (three chunks): every output bit for bit, and per view of chunks
    1 and 2 the index equals the minimum-(z, n) row of fusionutils.find_active_map_points."""
    import gradslam_b200 as gs
    from gradslam_b200.slam import fusionutils

    H, W = 48, 64
    pc, K, views = _fused_map_and_views(L)
    _assert_r1_strides_in_every_chunk(pc, L)
    Kd, Pd = K.to(DEV), views.to(DEV)
    out = gs.render_pointclouds(pc, Kd, Pd, H, W)
    want = render_oracle.render_views(_oracle_map(pc), views, K[:, 0], H, W)
    for name in ("index", "depth", "rgb", "normals", "confidence"):
        assert torch.equal(getattr(out, name).cpu(), getattr(want, name)), name
    assert ((out.index[:, VIEWS_PER_CTA:] >= 0).flatten(2).sum(2) > H * W // 2).all()
    pts = pc.points_padded
    for l in range(VIEWS_PER_CTA, L):
        frame = gs.RGBDImages(torch.zeros(3, 1, H, W, 3, device=DEV), torch.ones(3, 1, H, W, 1, device=DEV), Kd,
                              Pd[:, l:l + 1])
        b, n, h, w = fusionutils.find_active_map_points(pc, frame).unbind(1)
        z = torch.stack([_canonical_z(pts[e], Pd[e, l]) for e in range(3)])[b, n]
        keys = torch.full((3 * H * W,), torch.iinfo(torch.int64).max, dtype=torch.int64, device=DEV)
        keys.scatter_reduce_(0, (b * H + h) * W + w, (z.view(torch.int32).to(torch.int64) << 32) | n, reduce="amin")
        index = torch.where(keys == torch.iinfo(torch.int64).max, torch.full_like(keys, -1), keys & 0xFFFFFFFF)
        assert torch.equal(out.index[:, l].reshape(-1), index), l


def test_render_backward_across_view_chunks_against_float64_autograd():
    """L=70: d/d(rows) sums a row's pixels over views of different chunks; d/d(poses) of views >= 32 is nonzero and
    matches float64 autograd at the kernel's index."""
    import gradslam_b200 as gs

    H, W, L = 48, 64, 70
    pc0, K, views = _fused_map_and_views(L)
    smap = _oracle_map(pc0)
    leaves = [[t.to(DEV).requires_grad_(True) for t in lst]
              for lst in (smap.points, smap.normals, smap.colors, smap.ccounts)]
    P = views.to(DEV).requires_grad_(True)
    pc = gs.Pointclouds(points=leaves[0], normals=leaves[1], colors=leaves[2], features=leaves[3])
    out = gs.render_pointclouds(pc, K.to(DEV), P, H, W)
    g = torch.Generator().manual_seed(8)
    ups = [torch.randn(3, L, H, W, c, generator=g) for c in (1, 3, 3, 1)]
    sum((o * u.to(DEV)).sum() for o, u in zip((out.depth, out.normals, out.rgb, out.confidence), ups)).backward()

    index = out.index.cpu()
    ref_leaves = [t.double().requires_grad_(True) for t in smap.padded()] + [views.double().requires_grad_(True)]
    ref = render_oracle.render_values(*ref_leaves, index)
    sum((o * u.double()).sum() for o, u in zip((ref.depth, ref.normals, ref.rgb, ref.confidence), ups)).backward()
    for k in range(4):
        for b, leaf in enumerate(leaves[k]):
            want = ref_leaves[k].grad[b, :leaf.shape[0]]
            torch.testing.assert_close(leaf.grad.cpu().double(), want, rtol=1e-4,
                                       atol=1e-5 * max(want.abs().max().item(), 1.0))
    gp = ref_leaves[4].grad
    torch.testing.assert_close(P.grad.cpu().double(), gp, rtol=1e-3, atol=1e-4 * gp.abs().max().item())
    assert (P.grad[:, VIEWS_PER_CTA:, :3].abs().amax(dim=(2, 3)) > 0).all()
    assert (P.grad[..., 3, :] == 0).all()
    # rows that win pixels in views of two different chunks
    N = max(smap.counts())
    won = torch.zeros(3, 3, N + 1, dtype=torch.bool)  # (chunk, element, row); row N collects the uncovered pixels
    for l in range(L):
        won[l // VIEWS_PER_CTA].scatter_(1, torch.where(index[:, l] >= 0, index[:, l], N).reshape(3, -1), True)
    won = won[..., :N]
    assert ((won[0] & won[1]) | (won[0] & won[2]) | (won[1] & won[2])).any()
