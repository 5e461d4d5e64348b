"""Embedding images coarser than the depth on the GPU (RGBDImages(..., upsample_embeddings=True)): the step API, the
whole-sequence call, ICPSLAM aggregation and the differentiable mode against the CPU oracle
(tests/embedding_upsample_oracle.py) bit for bit; the upsampled path against the full-resolution path fed with the
oracle's samples; the rest of the map and the poses against a run without embeddings; gradients w.r.t. the coarse
image against float64 autograd, and their determinism."""
import math

import pytest
import torch
import torch.nn.functional as F

import embedding_oracle as eo
import embedding_upsample_oracle as uo
from cameras import camera_inputs
from gradslam_b200.synthetic import make_sequence

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
DIST_TH, SIGMA = 0.05, 0.6
DOT_TH = math.cos(20 * math.pi / 180)


def _frames(gs, rgb, depth, K, poses, emb=None, up=True):
    return gs.RGBDImages(rgb.to(DEV), depth.to(DEV), K.to(DEV), poses.to(DEV),
                         embeddings=None if emb is None else emb.to(DEV), upsample_embeddings=up and emb is not None)


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


_cache = {}


def _camera_case(H, W, L=3):
    key = (H, W, L)
    if key not in _cache:
        rgb, depth, K, poses = camera_inputs(2, L, H, W, seed=91)
        depth[1, :, : H // 3] = 0  # ragged: element 1 sees a third fewer pixels
        _cache[key] = (rgb, depth, K, poses)
    return _cache[key]


@pytest.mark.parametrize("D", [1, 3, 5, 64, 512])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16])
def test_step_api_matches_oracle(D, dtype):
    import gradslam_b200 as gs

    rgb, depth, K, poses = _camera_case(48, 64)
    e = eo.random_embeddings(2, 3, 7, 10, D, dtype=dtype, seed=D)  # non-integer ratios
    smap, ref = uo.run_pointfusion(rgb, depth, K, poses, e)
    slam = gs.PointFusion(odom="gt", device=DEV)
    pc = _steps(slam, _frames(gs, rgb, depth, K, poses, e))
    _assert_emb(pc, ref)
    assert pc._host_counts()[0] != pc._host_counts()[1]
    _assert_same_map(pc, _steps(slam, _frames(gs, rgb, depth, K, poses)))


def test_step_api_matches_oracle_at_640x480_from_a_stride_8_image():
    import gradslam_b200 as gs

    rgb, depth, K, poses = _camera_case(480, 640, L=2)
    e = eo.random_embeddings(2, 2, 60, 80, 64, dtype=torch.float16, seed=3)
    _, ref = uo.run_pointfusion(rgb, depth, K, poses, e)
    _assert_emb(_steps(gs.PointFusion(odom="gt", device=DEV), _frames(gs, rgb, depth, K, poses, e)), ref)


@pytest.mark.parametrize("hw", [(3, 4), (1, 32), (24, 1), (17, 23)])
def test_float32_equals_the_full_resolution_path_fed_with_the_samples(hw):
    import gradslam_b200 as gs

    rgb, depth, K, poses = make_sequence(2, 3, 24, 32, seed=92)
    e = eo.random_embeddings(2, 3, hw[0], hw[1], 8, seed=11)
    slam = gs.PointFusion(odom="gt", device=DEV)
    up = _steps(slam, _frames(gs, rgb, depth, K, poses, e))
    full = _steps(slam, _frames(gs, rgb, depth, K, poses, uo.upsample(e, 24, 32), up=False))
    _assert_emb(up, [x.cpu() for x in full.embeddings_list])
    seq, _ = slam(_frames(gs, rgb, depth, K, poses, e))
    _assert_emb(seq, [x.cpu() for x in full.embeddings_list])


def test_image_at_the_depth_size_equals_the_full_resolution_path():
    import gradslam_b200 as gs

    rgb, depth, K, poses = make_sequence(2, 3, 24, 32, seed=93)
    e = eo.random_embeddings(2, 3, 24, 32, 16, seed=12)
    slam = gs.PointFusion(odom="gt", device=DEV)
    for run in (lambda f: _steps(slam, f), lambda f: slam(f)[0]):
        up = run(_frames(gs, rgb, depth, K, poses, e))
        full = run(_frames(gs, rgb, depth, K, poses, e, up=False))
        for a, b in zip(up.embeddings_list, full.embeddings_list):
            assert torch.equal(a, b)


@pytest.mark.parametrize("groups", [1, 2, 3, 4])
def test_sequence_call_equals_step_loop_in_batch_groups(groups, monkeypatch):
    import gradslam_b200 as gs

    monkeypatch.setenv("GSX_SEQ_GROUPS", str(groups))
    rgb, depth, K, poses = make_sequence(4, 4, 24, 32, seed=94)
    e = eo.random_embeddings(4, 4, 3, 4, 16, dtype=torch.float16, seed=13)
    slam = gs.PointFusion(odom="gt", device=DEV)
    pc, _ = slam(_frames(gs, rgb, depth, K, poses, e))
    steps = _steps(slam, _frames(gs, rgb, depth, K, poses, e))
    _assert_emb(pc, [x.cpu() for x in steps.embeddings_list])
    _assert_same_map(pc, slam(_frames(gs, rgb, depth, K, poses))[0])


@pytest.mark.parametrize("radii", [False, True])
def test_sequence_call_equals_step_loop_device_and_pinned(radii):
    import gradslam_b200 as gs

    rgb, depth, K, poses = _camera_case(48, 64)
    e = eo.random_embeddings(2, 3, 6, 8, 24, dtype=torch.bfloat16, seed=14)
    slam = gs.PointFusion(odom="gt", device=DEV, surfel_radii=radii)
    steps = _steps(slam, _frames(gs, rgb, depth, K, poses, e))
    _, ref = uo.run_pointfusion(rgb, depth, K, poses, e)
    _assert_emb(steps, ref)
    dev_pc, _ = slam(_frames(gs, rgb, depth, K, poses, e))
    pinned = gs.RGBDImages(rgb.pin_memory(), depth.pin_memory(), K.pin_memory(), poses.pin_memory(),
                           embeddings=e.pin_memory(), upsample_embeddings=True)
    host_pc, _ = slam(pinned)
    cf = gs.RGBDImages(rgb.permute(0, 1, 4, 2, 3).to(DEV), depth.permute(0, 1, 4, 2, 3).to(DEV), K.to(DEV),
                       poses.to(DEV), channels_first=True, embeddings=e.permute(0, 1, 4, 2, 3).to(DEV),
                       upsample_embeddings=True)
    cf_pc, _ = slam(cf)
    for pc in (dev_pc, host_pc, cf_pc):
        _assert_emb(pc, ref)
        _assert_same_map(pc, steps)


def test_sequence_call_past_one_header_block():
    import gradslam_b200 as gs

    rgb, depth, K, poses = make_sequence(2, 70, 16, 24, seed=95)
    e = eo.random_embeddings(2, 70, 2, 3, 4, seed=15)
    slam = gs.PointFusion(odom="gt", device=DEV)
    pc, _ = slam(_frames(gs, rgb, depth, K, poses, e))
    _assert_emb(pc, uo.run_pointfusion(rgb, depth, K, poses, e)[1])
    _assert_same_map(pc, slam(_frames(gs, rgb, depth, K, poses))[0])


def test_sequence_call_out_too_small_reports_overflow_and_stays_in_capacity():
    import gradslam_b200 as gs

    rgb, depth, K, poses = make_sequence(1, 3, 24, 32, seed=96)
    cap = 600
    out = gs.Pointclouds(device=DEV)
    out._allocate(1, cap, 1)
    backing = torch.full((1, cap + 64, 8), 7.0, device=DEV)
    out._emb = backing[:, :cap]
    slam = gs.PointFusion(odom="gt", device=DEV)
    e = eo.random_embeddings(1, 3, 3, 4, 8, seed=16)
    pc, _ = slam(_frames(gs, rgb, depth, K, poses, e), out=out)
    torch.cuda.synchronize()
    assert int(pc._overflow.item()) == 1
    assert pc._emb.data_ptr() == backing.data_ptr()
    assert bool((backing[:, cap:] == 7.0).all())
    assert bool((backing[:, :cap] != 7.0).all())
    with pytest.raises(RuntimeError, match="capacity exceeded"):
        pc._host_counts()


def test_icpslam_aggregation_appends_the_samples_and_tracking_ignores_them():
    import gradslam_b200 as gs

    rgb, depth, K, poses = make_sequence(2, 3, 24, 32, seed=97)
    e = eo.random_embeddings(2, 3, 5, 7, 6, dtype=torch.float16, seed=17)
    pc, _ = gs.ICPSLAM(odom="gt", device=DEV)(_frames(gs, rgb, depth, K, poses, e))
    _assert_emb(pc, uo.run_aggregate(rgb, depth, K, poses, e)[1])
    e = e.float()  # (gradICP may run the map update in the differentiable mode, which is float32 only)
    for odom in ("icp", "gradicp"):
        for cls in (gs.ICPSLAM, gs.PointFusion):
            slam = cls(odom=odom, device=DEV, dsratio=2, numiters=3)
            a, pa = slam(_frames(gs, rgb, depth, K, poses, e))
            b, pb = slam(_frames(gs, rgb, depth, K, poses))
            assert torch.equal(pa, pb), (odom, cls)
            _assert_same_map(a, b)
            assert a.embedding_dim == 6


def test_update_map_fusion_and_fuse_with_map_carry_coarse_images():
    import gradslam_b200 as gs
    from gradslam_b200.slam import fusionutils as fu

    rgb, depth, K, poses = make_sequence(2, 3, 24, 32, seed=98)
    e = eo.random_embeddings(2, 3, 3, 4, 5, seed=18)
    frames = _frames(gs, rgb, depth, K, poses, e)
    a, b = gs.Pointclouds(device=DEV), gs.Pointclouds(device=DEV)
    for s in range(3):
        a = fu.update_map_fusion(a, frames[:, s], DIST_TH, DOT_TH, SIGMA)
        table = fu.find_correspondences(b, frames[:, s], DIST_TH, DOT_TH) if b.has_points else \
            torch.empty((0, 4), dtype=torch.int64, device=DEV)
        b = fu.fuse_with_map(b, frames[:, s], table, SIGMA)
    ref = uo.run_pointfusion(rgb, depth, K, poses, e)[1]
    _assert_emb(a, ref)
    _assert_emb(b, ref)
    # a map from coarse frames takes full-resolution frames of the same D and dtype, and the other way round
    full = _frames(gs, rgb, depth, K, poses, uo.upsample(e, 24, 32), up=False)
    mixed = fu.update_map_fusion(a, full[:, 0], DIST_TH, DOT_TH, SIGMA)
    assert mixed.embedding_dim == 5
    fu.update_map_fusion(mixed, frames[:, 1], DIST_TH, DOT_TH, SIGMA)


def test_differentiable_forward_equals_fused_path():
    import gradslam_b200 as gs
    from gradslam_b200.slam import fusionutils as fu

    rgb, depth, K, poses = make_sequence(2, 3, 24, 32, seed=99)
    e = eo.random_embeddings(2, 3, 4, 5, 4, seed=19)
    fused, diff = gs.Pointclouds(device=DEV), gs.Pointclouds(device=DEV)
    for s in range(3):
        sl = slice(s, s + 1)
        fused = fu.update_map_fusion(fused, _frames(gs, rgb[:, sl], depth[:, sl], K, poses[:, sl], e[:, sl]),
                                     DIST_TH, DOT_TH, SIGMA)
        f = gs.RGBDImages(rgb[:, sl].to(DEV), depth[:, sl].to(DEV), K.to(DEV), poses[:, sl].to(DEV),
                          embeddings=e[:, sl].to(DEV).requires_grad_(True), upsample_embeddings=True)
        diff = fu.update_map_fusion(diff, f, DIST_TH, DOT_TH, SIGMA)
    assert diff._emb.requires_grad
    _assert_same_map(diff, fused)
    _assert_emb(diff, [x.cpu() for x in fused.embeddings_list])


def _reference_grads(pc_geo, pc_emb, counts_in, assoc, depth, K, e, w, count_out):
    """float64 autograd of the oracle statement with the association fixed: bilinear upsampling of the coarse image e
    (B, 1, h, w, D), then the merge; the loss sum(w * E_out) over the rows.  Also returns, per merged row, the
    magnitude of d c0's terms, sum_d |w_d| (|E_d| / tot + |c0 E_d + alpha f_d| / tot^2): d c0 = sum_d w_d (E_d / tot
    - num_d / tot^2) cancels where c0 >> alpha, and float32 evaluation errs by a few ulp of that magnitude."""
    B, H, W = depth.shape[0], depth.shape[2], depth.shape[3]
    P = H * W
    c0 = pc_geo[..., 6].double().clone().requires_grad_(True)
    E = pc_emb.double().clone().requires_grad_(True)
    d = depth[:, 0, ..., 0].double().clone().requires_grad_(True)
    ec = e[:, 0].double().clone().requires_grad_(True)
    ed = F.interpolate(ec.permute(0, 3, 1, 2), (H, W), mode="bilinear", align_corners=False)
    ed = ed.permute(0, 2, 3, 1).reshape(B, P, -1)
    Kd = K[:, 0].double()
    fx, fy, cx, cy = Kd[:, 0, 0], Kd[:, 1, 1], Kd[:, 0, 2], Kd[:, 1, 2]
    u = torch.arange(W, dtype=torch.float64).view(1, 1, W)
    v = torch.arange(H, dtype=torch.float64).view(1, H, 1)
    x = (u / (fx + 1e-6).view(B, 1, 1) - (cx / (fx + 1e-6)).view(B, 1, 1)) * d
    y = (v / (fy + 1e-6).view(B, 1, 1) - (cy / (fy + 1e-6)).view(B, 1, 1)) * d
    sq = (x * x + y * y + d * d).reshape(B, P)
    alpha = torch.clamp(torch.exp(-sq / (2 * SIGMA ** 2)), 1e-7, 1.01)
    loss = 0
    mag = torch.zeros(c0.shape, dtype=torch.float64)
    for b in range(B):
        out = torch.cat([E[b, : counts_in[b]], E.new_zeros((count_out[b] - counts_in[b], E.shape[2]))], 0)
        a = assoc[b]
        m = (a < 0).nonzero().flatten()
        n = -a[m].long() - 1
        cb, ab = c0[b, n].unsqueeze(1), alpha[b, m].unsqueeze(1)
        out[n] = (cb * E[b, n] + ab * ed[b, m]) / (cb + ab)
        with torch.no_grad():
            tot = cb + ab
            mag[b, n] = (w[b, n].double().abs() * (E[b, n].abs() / tot + (cb * E[b, n] + ab * ed[b, m]).abs() /
                                                      (tot * tot))).sum(1)
        ap = (a > 0).nonzero().flatten()
        out[a[ap].long() - 1] = ed[b, ap]
        loss = loss + (w[b, : count_out[b]].double() * out).sum()
    loss.backward()
    return E.grad, c0.grad, d.grad, ec.grad, mag


@pytest.mark.parametrize("D, hw", [(7, (5, 7)), (8, (6, 8)), (8, (1, 32))])
def test_gradients_match_float64_autograd_and_are_deterministic(D, hw):
    """D = 7: the scalar gather; D = 8: 16-byte chunks"""
    import gradslam_b200 as gs
    from gradslam_b200.slam import fusionutils as fu

    rgb, depth, K, poses = camera_inputs(2, 3, 24, 32, seed=100, lattice_holes=True)
    e = eo.random_embeddings(2, 3, hw[0], hw[1], D, seed=20)
    frames = _frames(gs, rgb, depth, K, poses, e)
    base = gs.Pointclouds(device=DEV)
    for s in range(2):
        base = fu.update_map_fusion(base, frames[:, s], DIST_TH, DOT_TH, SIGMA, inplace=True)
    counts_in = base._host_counts()
    runs = []
    for _ in range(2):
        pc = base.clone()
        geo0, emb0 = pc._geo.detach().clone(), pc._emb.detach().clone()
        pc._geo.requires_grad_(True)
        pc._emb.requires_grad_(True)
        geo_leaf, emb_leaf = pc._geo, pc._emb
        d = depth[:, 2:3].to(DEV).requires_grad_(True)
        ef = e[:, 2:3].to(DEV).requires_grad_(True)
        frame = gs.RGBDImages(rgb[:, 2:3].to(DEV), d, K.to(DEV), poses[:, 2:3].to(DEV), embeddings=ef,
                              upsample_embeddings=True)
        got = []
        out = fu._fuse(pc, frame, SIGMA, DIST_TH, DOT_TH, assoc_out=got)
        count_out = out._host_counts()
        w = torch.randn(out._emb.shape, generator=torch.Generator().manual_seed(21)).to(DEV)
        (out._emb * w).sum().backward()
        assert ef.grad.shape == ef.shape
        runs.append((emb_leaf.grad, geo_leaf.grad, ef.grad, d.grad, got[0], w, count_out))
    for a, b in zip(runs[0][:5], runs[1][:5]):
        assert torch.equal(a, b)
    gE, ggeo, ge, gd, assoc, w, count_out = runs[0]
    rE, rc0, rd, re, mag = _reference_grads(geo0.cpu(), emb0.cpu(), counts_in, assoc.cpu(), depth[:, 2:3], K,
                                            e[:, 2:3], w.cpu(), count_out)
    tol = dict(rtol=1e-4, atol=1e-5)
    torch.testing.assert_close(gE.cpu().double(), rE, **tol)
    err = (ggeo[..., 6].cpu().double() - rc0).abs()
    bound = 1e-5 + 1e-4 * rc0.abs() + 64 * torch.finfo(torch.float32).eps * mag
    assert bool((err <= bound).all()), float((err / bound).max())
    torch.testing.assert_close(ge[:, 0].cpu().double(), re, **tol)
    torch.testing.assert_close(gd[:, 0, ..., 0].cpu().double(), rd, **tol)
    assert float(rc0.abs().sum()) > 0 and float(rd.abs().sum()) > 0 and float(re.abs().sum()) > 0


def test_embedding_op_backward_against_the_oracle_statement():
    """gsx_embed_merge_bwd_upsampled on a hand-made record against uo.merge_backward, including degenerate merges,
    a one-texel-wide image and g = None"""
    import gradslam_b200 as gs

    g = torch.Generator().manual_seed(22)
    B, H, W, N, cap = 2, 20, 28, 30, 90
    for h, w, D in ((4, 5, 12), (1, 28, 3), (20, 1, 8)):
        P = H * W
        E = torch.randn((B, N, D), generator=g)
        e = torch.randn((B, h, w, D), generator=g)
        rec = torch.rand((B, P, 2), generator=g)
        rec[0, :7] = 0.0
        gr = torch.randn((B, cap, D), generator=g)
        assoc = torch.zeros((B, P), dtype=torch.int32)
        for b in range(B):
            pix = torch.randperm(P, generator=g)[:N + 50]
            assoc[b, pix[:N]] = -(torch.arange(N, dtype=torch.int32) + 1)
            assoc[b, pix[N:]] = torch.arange(N, N + 50, dtype=torch.int32) + 1
        counts_in = torch.full((B,), N, dtype=torch.int32)
        dE_ref, de_ref, dc0_ref, dal_ref = uo.merge_backward(assoc, rec[..., 0], rec[..., 1], E, e, gr, H, W)
        t = [x.to(DEV) for x in (assoc, rec, counts_in, E, e, gr)]
        outs = []
        for _ in range(2):
            dE, de = torch.empty_like(t[3]), torch.empty_like(t[4])
            dw = torch.empty((2, B, P), device=DEV)
            gs._C.launch("gsx_embed_merge_bwd_upsampled", t[0], t[1], t[2], t[3], N, t[4], t[5], cap, B, H, W, h, w, D,
                         dE, de, dw[0], dw[1])
            outs.append((dE, de, dw))
        assert all(torch.equal(a, b) for a, b in zip(outs[0], outs[1]))
        dE, de, dw = (x.cpu() for x in outs[0])
        torch.testing.assert_close(dE, dE_ref, rtol=1e-5, atol=1e-5)
        torch.testing.assert_close(de, de_ref, rtol=1e-5, atol=1e-5)
        torch.testing.assert_close(dw[0], dc0_ref, rtol=1e-5, atol=1e-5)
        torch.testing.assert_close(dw[1], dal_ref, rtol=1e-5, atol=1e-5)
        de0 = torch.full_like(t[4], 5.0)
        dw0 = torch.empty((2, B, P), device=DEV)
        gs._C.launch("gsx_embed_merge_bwd_upsampled", t[0], t[1], t[2], t[3], N, t[4], None, cap, B, H, W, h, w, D,
                     torch.empty_like(t[3]), de0, dw0[0], dw0[1])
        assert bool((de0 == 0).all())
