"""Per-surfel embeddings on the GPU: the step API, the whole-sequence call, ICPSLAM aggregation and the differentiable
mode against the CPU oracle (tests/embedding_oracle.py) bit for bit; e := rgb equals the colours on every path; the rest
of the map and the poses equal a run without embeddings; gradients against float64 autograd; the Pointclouds store
through reallocation, copies, indexing and download."""
import math

import pytest
import torch

import embedding_oracle as eo
from cameras import camera_inputs
from gradslam_b200.synthetic import make_sequence

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
DIST_TH, SIGMA = 0.05, 0.6
DOT_TH = math.cos(20 * math.pi / 180)


def _frames(gs, rgb, depth, K, poses, emb=None):
    return gs.RGBDImages(rgb.to(DEV), depth.to(DEV), K.to(DEV), poses.to(DEV),
                         embeddings=None if emb is None else emb.to(DEV))


def _steps(slam, frames, pc=None):
    import gradslam_b200 as gs

    pc = gs.Pointclouds(device=DEV) if pc is None else pc
    prev = None
    for s in range(frames.shape[1]):
        live = frames[:, s]
        pc, live.poses = slam.step(pc, live, prev, inplace=True)
        prev = live if slam.odom != "gt" else None
    return pc


def _assert_emb(pc, emb):
    assert [int(c) for c in pc.num_points_per_pointcloud.tolist()] == [int(e.shape[0]) for e in emb]
    for b, e in enumerate(emb):
        got = pc.embeddings_list[b].detach().cpu()
        assert got.dtype == e.dtype
        assert torch.equal(got, e), b


def _assert_same_map(a, b):
    """geometry, colours and counts of two maps bit for bit (b may lack embeddings)"""
    ca, cb = a._host_counts(), b._host_counts()
    assert ca == cb
    for i, n in enumerate(ca):
        assert torch.equal(a._geo[i, :n].detach(), b._geo[i, :n].detach()), i
        assert torch.equal(a._col[i, :n].detach(), b._col[i, :n].detach()), i


def _assert_emb_is_colour(pc):
    assert pc.embedding_dim == 3
    for b in range(len(pc)):
        assert torch.equal(pc.embeddings_list[b].detach(), pc.colors_list[b].detach()), b


_cache = {}


def _camera_case(H, W, L=3):
    key = (H, W, L)
    if key not in _cache:
        rgb, depth, K, poses = camera_inputs(2, L, H, W, seed=81)
        depth[1, :, : H // 3] = 0  # ragged: element 1 sees a third fewer pixels
        _cache[key] = (rgb, depth, K, poses)
    return _cache[key]


@pytest.mark.parametrize("D", [1, 3, 5, 64, 512])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16])
def test_step_api_matches_oracle(D, dtype):
    import gradslam_b200 as gs

    rgb, depth, K, poses = _camera_case(48, 64)
    e = eo.random_embeddings(2, 3, 48, 64, D, dtype=dtype, seed=D)
    smap, ref = eo.run_pointfusion(rgb, depth, K, poses, e)
    slam = gs.PointFusion(odom="gt", device=DEV)
    pc = _steps(slam, _frames(gs, rgb, depth, K, poses, e))
    _assert_emb(pc, ref)
    assert pc._host_counts()[0] != pc._host_counts()[1]
    _assert_same_map(pc, _steps(slam, _frames(gs, rgb, depth, K, poses)))


def test_step_api_matches_oracle_at_640x480():
    import gradslam_b200 as gs

    rgb, depth, K, poses = _camera_case(480, 640, L=2)
    e = eo.random_embeddings(2, 2, 480, 640, 16, dtype=torch.float16, seed=3)
    _, ref = eo.run_pointfusion(rgb, depth, K, poses, e)
    _assert_emb(_steps(gs.PointFusion(odom="gt", device=DEV), _frames(gs, rgb, depth, K, poses, e)), ref)


@pytest.mark.parametrize("groups", [1, 2, 3, 4])
def test_sequence_call_rgb_as_embedding_in_batch_groups(groups, monkeypatch):
    import gradslam_b200 as gs

    monkeypatch.setenv("GSX_SEQ_GROUPS", str(groups))
    rgb, depth, K, poses = make_sequence(4, 4, 24, 32, seed=82)
    slam = gs.PointFusion(odom="gt", device=DEV)
    pc, _ = slam(_frames(gs, rgb, depth, K, poses, rgb))
    _assert_emb_is_colour(pc)
    _assert_same_map(pc, slam(_frames(gs, rgb, depth, K, poses))[0])


@pytest.mark.parametrize("radii", [False, True])
def test_sequence_call_equals_step_loop_device_and_pinned(radii):
    import gradslam_b200 as gs

    rgb, depth, K, poses = _camera_case(48, 64)
    e = eo.random_embeddings(2, 3, 48, 64, 24, dtype=torch.bfloat16, seed=4)
    slam = gs.PointFusion(odom="gt", device=DEV, surfel_radii=radii)
    steps = _steps(slam, _frames(gs, rgb, depth, K, poses, e))
    _, ref = eo.run_pointfusion(rgb, depth, K, poses, e)
    _assert_emb(steps, ref)
    dev_pc, _ = slam(_frames(gs, rgb, depth, K, poses, e))
    pinned = gs.RGBDImages(rgb.pin_memory(), depth.pin_memory(), K.pin_memory(), poses.pin_memory(),
                           embeddings=e.pin_memory())
    host_pc, _ = slam(pinned)
    for pc in (dev_pc, host_pc):
        _assert_emb(pc, ref)
        _assert_same_map(pc, steps)
    rgb_pc, _ = slam(_frames(gs, rgb, depth, K, poses, rgb))
    _assert_emb_is_colour(rgb_pc)
    _assert_same_map(rgb_pc, steps)


def test_sequence_call_past_one_header_block():
    import gradslam_b200 as gs

    rgb, depth, K, poses = make_sequence(2, 70, 16, 24, seed=83)
    slam = gs.PointFusion(odom="gt", device=DEV)
    pc, _ = slam(_frames(gs, rgb, depth, K, poses, rgb))
    _assert_emb_is_colour(pc)
    _assert_same_map(pc, slam(_frames(gs, rgb, depth, K, poses))[0])


def test_sequence_call_out_too_small_reports_overflow_and_stays_in_capacity():
    import gradslam_b200 as gs

    rgb, depth, K, poses = make_sequence(1, 3, 24, 32, seed=84)
    cap = 600
    out = gs.Pointclouds(device=DEV)
    out._allocate(1, cap, 1)
    # one element: the first `cap` rows of a longer allocation are a dense store, and the rows past it must stay as they are
    backing = torch.full((1, cap + 64, 8), 7.0, device=DEV)
    out._emb = backing[:, :cap]
    slam = gs.PointFusion(odom="gt", device=DEV)
    e = eo.random_embeddings(1, 3, 24, 32, 8, seed=5)
    pc, _ = slam(_frames(gs, rgb, depth, K, poses, e), out=out)
    torch.cuda.synchronize()
    assert int(pc._overflow.item()) == 1
    assert pc._emb.data_ptr() == backing.data_ptr()
    assert bool((backing[:, cap:] == 7.0).all())
    assert bool((backing[:, :cap] != 7.0).all())
    with pytest.raises(RuntimeError, match="capacity exceeded"):
        pc._host_counts()


def test_icpslam_aggregation_and_tracking_ignore_embeddings():
    import gradslam_b200 as gs

    rgb, depth, K, poses = make_sequence(2, 3, 24, 32, seed=85)
    e = eo.random_embeddings(2, 3, 24, 32, 6, seed=6)
    agg = gs.ICPSLAM(odom="gt", device=DEV)
    pc, _ = agg(_frames(gs, rgb, depth, K, poses, rgb))
    _assert_emb_is_colour(pc)
    pc, _ = agg(_frames(gs, rgb, depth, K, poses, e))
    _assert_emb(pc, eo.run_aggregate(rgb, depth, K, poses, e)[1])
    for odom in ("icp", "gradicp"):
        for cls in (gs.ICPSLAM, gs.PointFusion):
            slam = cls(odom=odom, device=DEV, dsratio=2, numiters=3)
            a, pa = slam(_frames(gs, rgb, depth, K, poses, rgb))
            b, pb = slam(_frames(gs, rgb, depth, K, poses))
            assert torch.equal(pa, pb), (odom, cls)
            _assert_same_map(a, b)
            _assert_emb_is_colour(a)


def test_update_map_fusion_and_fuse_with_map_carry_embeddings():
    import gradslam_b200 as gs
    from gradslam_b200.slam import fusionutils as fu

    rgb, depth, K, poses = make_sequence(2, 3, 24, 32, seed=86)
    frames = _frames(gs, rgb, depth, K, poses, rgb)
    a, b = gs.Pointclouds(device=DEV), gs.Pointclouds(device=DEV)
    for s in range(3):
        a = fu.update_map_fusion(a, frames[:, s], DIST_TH, DOT_TH, SIGMA)
        table = fu.find_correspondences(b, frames[:, s], DIST_TH, DOT_TH) if b.has_points else \
            torch.empty((0, 4), dtype=torch.int64, device=DEV)
        b = fu.fuse_with_map(b, frames[:, s], table, SIGMA)
    _assert_emb_is_colour(a)
    _assert_emb_is_colour(b)
    with pytest.raises(ValueError, match="embeddings"):
        fu.update_map_fusion(a, _frames(gs, rgb, depth, K, poses)[:, 0], DIST_TH, DOT_TH, SIGMA)


def test_store_survives_reserve_copies_indexing_and_download():
    import gradslam_b200 as gs
    from gradslam_b200.slam import fusionutils as fu

    rgb, depth, K, poses = make_sequence(2, 4, 24, 32, seed=87)
    e = eo.random_embeddings(2, 4, 24, 32, 5, dtype=torch.float16, seed=7)
    frames = _frames(gs, rgb, depth, K, poses, e)
    pc = gs.Pointclouds(device=DEV)
    caps = set()
    for s in range(4):  # the step loop grows the store (reserve) several times
        pc = fu.update_map_fusion(pc, frames[:, s], DIST_TH, DOT_TH, SIGMA, inplace=True)
        caps.add(pc.capacity)
    assert len(caps) > 1
    ref = eo.run_pointfusion(rgb, depth, K, poses, e)[1]
    _assert_emb(pc, ref)
    _assert_emb(pc.clone(), ref)
    _assert_emb(pc.detach(), ref)
    _assert_emb(pc.to("cpu"), ref)
    _assert_emb(pc[1], ref[1:])
    d = pc.download()
    torch.cuda.synchronize()
    _assert_emb(d, ref)
    both = pc.clone().append_points(pc)
    _assert_emb(both, [torch.cat([r, r], 0) for r in ref])


def _diff_case():
    """A map of two frames with embeddings, then a third frame in the differentiable mode."""
    import gradslam_b200 as gs
    from gradslam_b200.slam import fusionutils as fu

    rgb, depth, K, poses = camera_inputs(2, 3, 24, 32, seed=88, lattice_holes=True)
    e = eo.random_embeddings(2, 3, 24, 32, 7, seed=8)
    frames = _frames(gs, rgb, depth, K, poses, e)
    pc = gs.Pointclouds(device=DEV)
    for s in range(2):
        pc = fu.update_map_fusion(pc, frames[:, s], DIST_TH, DOT_TH, SIGMA, inplace=True)
    return rgb, depth, K, poses, e, pc


def test_differentiable_forward_equals_fused_path():
    import gradslam_b200 as gs
    from gradslam_b200.slam import fusionutils as fu

    rgb, depth, K, poses = make_sequence(2, 3, 24, 32, seed=89)
    for emb in (rgb, eo.random_embeddings(2, 3, 24, 32, 4, seed=9)):
        fused, diff = gs.Pointclouds(device=DEV), gs.Pointclouds(device=DEV)
        for s in range(3):
            sl = slice(s, s + 1)
            fused = fu.update_map_fusion(fused, _frames(gs, rgb[:, sl], depth[:, sl], K, poses[:, sl], emb[:, sl]),
                                         DIST_TH, DOT_TH, SIGMA)
            f = gs.RGBDImages(rgb[:, sl].to(DEV), depth[:, sl].to(DEV), K.to(DEV), poses[:, sl].to(DEV),
                              embeddings=emb[:, sl].to(DEV).requires_grad_(True))
            diff = fu.update_map_fusion(diff, f, DIST_TH, DOT_TH, SIGMA)
        assert diff._emb.requires_grad
        _assert_same_map(diff, fused)
        _assert_emb(diff, [x.cpu() for x in fused.embeddings_list])
        if emb is rgb:
            _assert_emb_is_colour(diff)


def _reference_grads(pc_geo, pc_emb, counts_in, assoc, depth, K, e, w, count_out):
    """float64 autograd of the oracle statement with the association fixed: the loss sum(w * E_out) over the rows."""
    B, H, W = depth.shape[0], depth.shape[2], depth.shape[3]
    P = H * W
    c0 = pc_geo[..., 6].double().clone().requires_grad_(True)
    E = pc_emb.double().clone().requires_grad_(True)
    d = depth[:, 0, ..., 0].double().clone().requires_grad_(True)
    ed = e[:, 0].double().reshape(B, P, -1).clone().requires_grad_(True)
    Kd = K[:, 0].double()
    fx, fy, cx, cy = Kd[:, 0, 0], Kd[:, 1, 1], Kd[:, 0, 2], Kd[:, 1, 2]
    u = torch.arange(W, dtype=torch.float64).view(1, 1, W)
    v = torch.arange(H, dtype=torch.float64).view(1, H, 1)
    x = (u / (fx + 1e-6).view(B, 1, 1) - (cx / (fx + 1e-6)).view(B, 1, 1)) * d
    y = (v / (fy + 1e-6).view(B, 1, 1) - (cy / (fy + 1e-6)).view(B, 1, 1)) * d
    sq = (x * x + y * y + d * d).reshape(B, P)
    alpha = torch.clamp(torch.exp(-sq / (2 * SIGMA ** 2)), 1e-7, 1.01)
    loss = 0
    for b in range(B):
        out = torch.cat([E[b, : counts_in[b]], E.new_zeros((count_out[b] - counts_in[b], E.shape[2]))], 0)
        a = assoc[b]
        m = (a < 0).nonzero().flatten()
        n = -a[m].long() - 1
        cb, ab = c0[b, n].unsqueeze(1), alpha[b, m].unsqueeze(1)
        out[n] = (cb * E[b, n] + ab * ed[b, m]) / (cb + ab)
        ap = (a > 0).nonzero().flatten()
        out[a[ap].long() - 1] = ed[b, ap]
        loss = loss + (w[b, : count_out[b]].double() * out).sum()
    loss.backward()
    return E.grad, c0.grad, d.grad, ed.grad


def test_gradients_match_float64_autograd_of_the_oracle_statement():
    import gradslam_b200 as gs
    from gradslam_b200.slam import fusionutils as fu

    rgb, depth, K, poses, e, pc = _diff_case()
    counts_in = pc._host_counts()
    geo0, emb0 = pc._geo.detach().clone(), pc._emb.detach().clone()
    pc._geo.requires_grad_(True)
    pc._emb.requires_grad_(True)
    geo_leaf, emb_leaf = pc._geo, pc._emb
    d = depth[:, 2:3].to(DEV).requires_grad_(True)
    ef = e[:, 2:3].to(DEV).requires_grad_(True)
    frame = gs.RGBDImages(rgb[:, 2:3].to(DEV), d, K.to(DEV), poses[:, 2:3].to(DEV), embeddings=ef)
    got = []
    out = fu._fuse(pc, frame, SIGMA, DIST_TH, DOT_TH, assoc_out=got)
    count_out = out._host_counts()
    w = torch.randn(out._emb.shape, generator=torch.Generator().manual_seed(10)).to(DEV)
    (out._emb * w).sum().backward()
    rE, rc0, rd, re = _reference_grads(geo0.cpu(), emb0.cpu(), counts_in, got[0].cpu(), depth[:, 2:3], K,
                                       e[:, 2:3], w.cpu(), count_out)
    tol = dict(rtol=1e-4, atol=1e-5)
    torch.testing.assert_close(emb_leaf.grad.cpu().double(), rE, **tol)
    torch.testing.assert_close(geo_leaf.grad[..., 6].cpu().double(), rc0, **tol)
    torch.testing.assert_close(ef.grad.cpu().double().reshape(re.shape), re, **tol)
    torch.testing.assert_close(d.grad[:, 0, ..., 0].cpu().double(), rd, **tol)
    assert float(rc0.abs().sum()) > 0 and float(rd.abs().sum()) > 0


def test_gradients_of_a_loss_without_embeddings_are_unchanged():
    import gradslam_b200 as gs
    from gradslam_b200.slam import fusionutils as fu

    rgb, depth, K, poses, e, pc = _diff_case()
    grads = []
    for with_emb in (True, False):
        m = pc.clone()
        if not with_emb:
            m._emb = None
        m._geo.requires_grad_(True)
        geo_leaf = m._geo
        d = depth[:, 2:3].to(DEV).requires_grad_(True)
        frame = gs.RGBDImages(rgb[:, 2:3].to(DEV), d, K.to(DEV), poses[:, 2:3].to(DEV),
                              embeddings=e[:, 2:3].to(DEV) if with_emb else None)
        out = fu.update_map_fusion(m, frame, DIST_TH, DOT_TH, SIGMA)
        (out.points_padded.sum() + (out.colors_padded * 0.5).sum() + out.features_padded.sum()).backward()
        grads.append((d.grad, geo_leaf.grad))
    assert torch.equal(grads[0][0], grads[1][0])
    assert torch.equal(grads[0][1], grads[1][1])
