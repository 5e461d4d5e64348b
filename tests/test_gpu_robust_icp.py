"""GPU checks of the Huber-weighted tracking (huber_delta / photometric_huber_delta of the ICP entry points) against
tests/robust_oracle.py: fused poses at the ICP tests' tolerances for both associations, the Huber kernels at a scale no
residual reaches equal to the unweighted ones bit for bit, taped poses equal to fused ones, the ops' gradients against
float64 autograd on both sides of delta, the differentiable mode against autograd of the oracle, and the gain on a
scene with an object that appears."""
import math

import pytest
import torch

import gsx_oracle as oracle
import robust_oracle as ro
from cameras import camera_inputs
from gradslam_b200.synthetic import make_dynamic_sequence, make_textured_sequence
from test_gpu_photometric_icp import ATOL_MANY_POINTS, _map, _oracle
from test_gpu_projective_icp import _frames, _icp_kwargs
from test_photometric_oracle import W_TRACK

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
INF = math.inf
FLT_MAX = 3.4028234663852886e38  # the largest finite float32: a scale no residual reaches, so the Huber kernels run


def _inputs(textured):
    """B = 3 with a camera per element (or the textured scene), ragged source counts; element 1 has no live depth."""
    B, L, H, W = 3, 3, 90, 120
    if textured:
        rgb, depth, K, poses = make_textured_sequence(B, L, H, W, seed=3, yaw0=0.3)
    else:
        rgb, depth, K, poses = camera_inputs(B, L, H, W, 17, skew=0.5)
    depth[1, 2] = 0.0
    return rgb, depth, K, poses, H, W


@pytest.mark.parametrize("ds", [1, 4])
@pytest.mark.parametrize("odom", ["icp", "gradicp"])
def test_fused_nn_poses_match_oracle(odom, ds):
    import gradslam_b200 as gs

    rgb, depth, K, poses, H, W = _inputs(False)
    frames = _frames(rgb, depth, K, poses)
    pc = _map(frames[:, :2], radii=False)
    smap, _ = _oracle(pc)
    at_prev = oracle.frame_maps(depth[:, 2:3], K, poses[:, 1:2])
    for delta in (0.005, 0.02):
        slam = gs.ICPSLAM(odom=odom, numiters=10, dsratio=ds, huber_delta=delta, device=DEV)
        got = slam._localize(pc, frames[:, 2], frames[:, 1])[:, 0].cpu()
        want = ro.odometry_nn(smap, at_prev, poses[:, 1], K[:, 0], H, W, odom, ds, _icp_kwargs(odom, 10, None), delta)
        torch.testing.assert_close(got, want, rtol=0, atol=1e-4 if ds > 1 else ATOL_MANY_POINTS)
        assert torch.equal(got[1], poses[1, 1])
        plain = gs.ICPSLAM(odom=odom, numiters=10, dsratio=ds, device=DEV)._localize(pc, frames[:, 2], frames[:, 1])
        assert not torch.equal(got, plain[:, 0].cpu())


@pytest.mark.parametrize("ds", [1, 2])
@pytest.mark.parametrize("w", [0.0, W_TRACK])
@pytest.mark.parametrize("odom", ["icp", "gradicp"])
def test_fused_projective_poses_match_oracle(odom, w, ds):
    import gradslam_b200 as gs

    rgb, depth, K, poses, H, W = _inputs(w > 0)
    frames = _frames(rgb, depth, K, poses)
    pc = _map(frames[:, :2])
    smap, radii = _oracle(pc)
    at_prev = oracle.frame_maps(depth[:, 2:3], K, poses[:, 1:2])
    scales = [(0.005, None), (0.02, None)] + ([(0.02, 0.01), (None, 0.01)] if w else [])
    for M in (0, 3):
        for delta, delta_p in scales:
            slam = gs.PointFusion(odom=odom, association="projective", numiters=10, dsratio=ds, surfel_radii=True,
                                  target_splat_px=M, photometric_weight=w, huber_delta=delta,
                                  photometric_huber_delta=delta_p, device=DEV)
            got = slam._localize(pc, frames[:, 2], frames[:, 1])[:, 0].cpu()
            want = ro.odometry_projective(smap, radii, at_prev, rgb[:, 2:3], poses[:, 1], K[:, 0], H, W, odom, ds,
                                          _icp_kwargs(odom, 10, None), M, w, INF if delta is None else delta,
                                          INF if delta_p is None else delta_p)
            # (gradICP with weighted photometric rows drifts past 1e-4 on rounding order alone at ds = 2 too:
            # 3.9e-4 measured on an H100; the unweighted photometric term's ds = 1 tolerance covers it)
            tol = 1e-4 if ds > 1 and not (w and odom == "gradicp") else ATOL_MANY_POINTS
            torch.testing.assert_close(got, want, rtol=0, atol=tol)
            assert torch.equal(got[1], poses[1, 1])


def test_every_robust_entry_point_at_infinity_is_its_counterpart_bit_for_bit():
    """A finite scale runs the Huber-weighted kernels (+inf runs the unweighted ones); at FLT_MAX every row is inside
    it, so they must give the unweighted outputs bit for bit."""
    from gradslam_b200.odometry import GradICPOdometryProvider
    from gradslam_b200.odometry.icputils import (_JointNormalEqBatchedFn, _NormalEqBatchedFn, downsample_rgbdimages,
                                                 icp_align, localize_against_map, localize_projective,
                                                 project_associate, projective_targets)

    rgb, depth, K, poses, H, W = _inputs(True)
    frames = _frames(rgb, depth, K, poses)
    pc = _map(frames[:, :2])
    prov = GradICPOdometryProvider(10, 1e-8, None)
    robust = GradICPOdometryProvider(10, 1e-8, None)
    robust.huber_delta = FLT_MAX
    for ds in (1, 4):
        assert torch.equal(localize_against_map(pc, frames[:, 2], frames[:, 1], ds, robust),
                           localize_against_map(pc, frames[:, 2], frames[:, 1], ds, prov))
        for M in (0, 3):
            for w in (0.0, W_TRACK):
                want = localize_projective(pc, frames[:, 2], frames[:, 1], ds, prov, M, w)
                got = localize_projective(pc, frames[:, 2], frames[:, 1], ds, robust, M, w,
                                          FLT_MAX if w else None)
                assert torch.equal(got, want), (ds, M, w)
    # icp_align on ragged clouds
    g = torch.Generator().manual_seed(5)
    src = torch.randn(3, 700, 3, generator=g).to(DEV)
    tgt = (src + 0.01 * torch.randn(3, 700, 3, generator=g).to(DEV))
    tn = torch.nn.functional.normalize(torch.randn(3, 700, 3, generator=g), dim=-1).to(DEV)
    cs, ct = (torch.tensor(c, dtype=torch.int32, device=DEV) for c in ([700, 0, 350], [500, 700, 1]))
    for mode in (0, 1):
        a = icp_align(src, cs, tgt, tn, ct, None, mode, 8, 1e-8, None, want_idx=True)
        b = icp_align(src, cs, tgt, tn, ct, None, mode, 8, 1e-8, None, want_idx=True, huber_delta=FLT_MAX)
        rows = torch.arange(700, device=DEV) < cs.unsqueeze(1)  # (rows beyond a source size are not written)
        assert torch.equal(a[0], b[0]) and torch.equal(a[1][rows], b[1][rows])
    # the two ops, forward and backward (d/dK included)
    idx = torch.where(torch.rand(3, 700, generator=g).to(DEV) < 0.8,
                      torch.randint(0, 700, (3, 700), generator=g).to(DEV), torch.full((3, 700), -1, device=DEV))
    gs_ = torch.randn(3, 28, generator=g).to(DEV)
    outs = []
    for h in ((), (FLT_MAX,)):
        x = [t.clone().requires_grad_(True) for t in (src, tgt, tn)]
        s = _NormalEqBatchedFn.apply(*x, idx, cs, *h)
        (s * gs_).sum().backward()
        outs.append([s.detach()] + [t.grad for t in x])
    _same(*outs, scattered=(2, 3))
    K4 = K[:, 0].to(DEV)
    prev = poses[:, 1].to(DEV)
    index, tp, tnn = projective_targets(pc, K4, prev, H, W)
    live_pc = downsample_rgbdimages(frames[:, 2], 2)
    s_pts, s_col = live_pc.points_padded.contiguous(), live_pc.colors_padded.contiguous()
    counts = live_pc._counts_dev[live_pc._cur]
    jdx = project_associate(s_pts, counts, tp, index, prev, K4, H, W)[1]
    mcol = torch.gather(torch.cat([pc.colors_padded, pc.colors_padded.new_zeros(3, 1, 3)], 1), 1,
                        index.clamp(min=0).unsqueeze(-1).expand(3, H * W, 3)) * (index >= 0).unsqueeze(-1)
    gj = torch.randn(3, 28, generator=g).to(DEV)
    outs = []
    for h in ((), ((FLT_MAX, FLT_MAX),)):
        x = [t.clone().requires_grad_(True) for t in (s_pts, s_col, tp, tnn, mcol, prev, K4)]
        s = _JointNormalEqBatchedFn.apply(*x[:6], jdx, index, counts, x[6], W_TRACK, H, W, *h)
        (s * gj).sum().backward()
        outs.append([s.detach()] + [t.grad for t in x])
    _same(*outs, scattered=(3, 4, 5))


def _same(a, b, scattered):
    """Bit for bit, except the target gradients the Python side scatters with index_add_, whose float atomics add in
    no fixed order: those to float32 rounding."""
    for i, (u, v) in enumerate(zip(a, b)):
        if i in scattered:
            torch.testing.assert_close(u, v)
        else:
            assert torch.equal(u, v), i


@pytest.mark.parametrize("odom", ["icp", "gradicp"])
def test_taped_poses_equal_the_fused_poses(odom):
    import gradslam_b200 as gs

    rgb, depth, K, poses, H, W = _inputs(True)
    frames = _frames(rgb, depth, K, poses)
    pc = _map(frames[:, :2])
    live = gs.RGBDImages(rgb[:, 2:3].to(DEV).requires_grad_(True), depth[:, 2:3].to(DEV).requires_grad_(True),
                         K.to(DEV), poses[:, 2:3].to(DEV))
    cases = [dict(huber_delta=0.01), dict(association="projective", target_splat_px=3, huber_delta=0.01)]
    cases += [dict(association="projective", target_splat_px=M, photometric_weight=W_TRACK, huber_delta=0.02,
                   photometric_huber_delta=0.01) for M in (0, 3)]
    for kw in cases:
        for ds in (1, 4):
            slam = gs.PointFusion(odom=odom, numiters=10, dsratio=ds, surfel_radii=True, device=DEV, **kw)
            fused = slam._localize(pc, frames[:, 2], frames[:, 1])
            taped = slam._localize(pc, live, frames[:, 1])
            assert taped.requires_grad
            assert torch.equal(taped.detach(), fused), (kw, ds)


def test_normal_eq_op_gradients_match_float64_autograd():
    """The geometric op's sums and backward against float64 autograd of robust_oracle.row_products, ragged batch with
    rows on both sides of delta."""
    from gradslam_b200.odometry.icputils import _NormalEqBatchedFn

    g = torch.Generator().manual_seed(11)
    B, N, delta = 3, 3000, 0.05
    src = torch.randn(B, N, 3, generator=g)
    tgt = src + 0.08 * torch.randn(B, N, 3, generator=g)
    tn = torch.nn.functional.normalize(torch.randn(B, N, 3, generator=g), dim=-1)
    idx = torch.randint(0, N, (B, N), generator=g)
    idx[torch.rand(B, N, generator=g) < 0.1] = -1
    counts = torch.tensor([N, 0, 1777], dtype=torch.int32)
    gs_ = torch.randn(B, 28, generator=g)
    x = [t.to(DEV).requires_grad_(True) for t in (src, tgt, tn)]
    sums = _NormalEqBatchedFn.apply(*x, idx.to(DEV), counts.to(DEV), delta)
    (sums * gs_.to(DEV)).sum().backward()
    for b in range(B):
        keep = (idx[b] >= 0) & (torch.arange(N) < counts[b])
        s = src[b].double().requires_grad_(True)
        p = tgt[b].double().requires_grad_(True)
        n = tn[b].double().requires_grad_(True)
        j = idx[b][keep]
        ss, pp, nn_ = s[keep], p[j], n[j]
        A = torch.stack([nn_[:, 0], nn_[:, 1], nn_[:, 2], nn_[:, 2] * ss[:, 1] - nn_[:, 1] * ss[:, 2],
                         nn_[:, 0] * ss[:, 2] - nn_[:, 2] * ss[:, 0], nn_[:, 1] * ss[:, 0] - nn_[:, 0] * ss[:, 1]], 1)
        r = (nn_ * (pp - ss)).sum(1)
        want = ro.row_products(A, r, delta).sum(0)
        if b != 1:
            assert (r.abs() > delta).any() and (r.abs() <= delta).any()
        (want * gs_[b].double()).sum().backward()
        torch.testing.assert_close(sums[b].detach().cpu().double(), want.detach(), rtol=1e-4, atol=1e-3)
        for got, ref in ((x[0].grad[b], s.grad), (x[1].grad[b], p.grad), (x[2].grad[b], n.grad)):
            torch.testing.assert_close(got.cpu().double(), ref, rtol=1e-3, atol=1e-3 * max(1.0, ref.abs().max().item()))


@pytest.mark.parametrize("assoc", ["nn", "projective"])
def test_differentiable_mode_gradients_match_oracle_autograd(assoc):
    """d(pose)/d(live depth) (and d/dK, through the joint op, with the photometric term) of
    ICPSLAM(odom='gradicp', huber_delta=...) against autograd of the oracle, on lattice-hole depth."""
    import gradslam_b200 as gs
    from gradslam_b200.synthetic import punch_lattice_holes

    B, H, W = 1, 32, 40
    rgb, depth, K, poses = make_textured_sequence(B, 2, H, W, seed=33, yaw0=0.6, hole_fraction=0.0)
    depth = punch_lattice_holes(depth)
    m0 = oracle.frame_maps(depth[:, :1], K, poses[:, :1])
    valid = m0["valid"][0, 0]
    P0, N0, C0 = m0["gvertex"][0, 0][valid], m0["gnormal"][0, 0][valid], rgb[0, 0][valid]
    wts = torch.randn(4, 4, generator=torch.Generator().manual_seed(2))
    w = W_TRACK if assoc == "projective" else 0.0
    delta, delta_p = 0.003, 0.02

    d_ref = depth[:, 1:2].clone().requires_grad_(True)
    K_ref = K.clone().requires_grad_(True)
    at_prev = oracle.frame_maps(d_ref, K_ref, poses[:, :1])
    smap = oracle.SurfelMap([P0], [N0], [C0])
    kw = _icp_kwargs("gradicp", 3, None)
    if assoc == "nn":
        ref = ro.odometry_nn(smap, at_prev, poses[:, 0], K_ref[:, 0], H, W, "gradicp", 2, kw, delta)
    else:
        ref = ro.odometry_projective(smap, None, at_prev, rgb[:, 1:2], poses[:, 0], K_ref[:, 0], H, W, "gradicp", 2, kw,
                                     0, w, delta, delta_p)
    (ref[0] * wts).sum().backward()

    pc = gs.Pointclouds(points=P0[None].to(DEV), normals=N0[None].to(DEV), colors=C0[None].to(DEV))
    d_g = depth[:, 1:2].to(DEV).requires_grad_(True)
    K_g = K.to(DEV).requires_grad_(True)
    live = gs.RGBDImages(rgb[:, 1:2].to(DEV), d_g, K_g, poses[:, 1:2].to(DEV))
    prev = gs.RGBDImages(rgb[:, 0:1].to(DEV), depth[:, 0:1].to(DEV), K_g, poses[:, 0:1].to(DEV))
    extra = dict(association="projective", photometric_weight=w, photometric_huber_delta=delta_p) if w else {}
    slam = gs.ICPSLAM(odom="gradicp", numiters=3, dsratio=2, huber_delta=delta, device=DEV, **extra)
    out = slam._localize(pc, live, prev)
    torch.testing.assert_close(out[:, 0].detach().cpu(), ref.detach(), rtol=0, atol=1e-4)
    (out[0, 0] * wts.to(DEV)).sum().backward()
    for name, got, want in (("depth", d_g.grad, d_ref.grad), ("K", K_g.grad, K_ref.grad)):
        got = got.cpu()
        assert torch.isfinite(got).all() and want.abs().max() > 0, name
        torch.testing.assert_close(got, want, rtol=5e-2, atol=5e-3 * want.abs().max().item(), msg=name)


@pytest.mark.parametrize("cls", ["PointFusion", "ICPSLAM"])
def test_dynamic_scene_accuracy_on_the_device(cls):
    """make_dynamic_sequence: a box appears at frame 3.  Step by step, projective gradICP at dsratio 2: huber_delta =
    0.02 m cuts the worst translation error from frame 3 on at least tenfold."""
    import gradslam_b200 as gs

    rgb, depth, K, poses = make_dynamic_sequence(1, 8, 48, 64, 3, 8, yaw0=0.6)
    frames = _frames(rgb, depth, K, poses)
    err = {}
    for delta in (None, 0.02):
        extra = dict(surfel_radii=True) if cls == "PointFusion" else {}
        slam = getattr(gs, cls)(odom="gradicp", association="projective", dsratio=2, huber_delta=delta, device=DEV,
                                **extra)
        pc, prev, got = gs.Pointclouds(device=DEV), None, []
        for s in range(frames.shape[1]):
            pc, pose = slam.step(pc, frames[:, s], prev)
            got.append(pose[:, 0].cpu())
            prev = frames[:, s]
        err[delta] = ro.worst_translation_error(torch.stack(got, 1), poses, 3)
    assert err[0.02] * 10 <= err[None], err
