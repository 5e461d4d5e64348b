"""The benchmark's pose-gradient configuration (BASELINE.json config 3: ICPSLAM(odom='gradicp'), 10 Gauss-Newton
iterations, dsratio 4, 640x480, B=8, L=2) with gradients: the differentiable forward against the fused no-grad call,
and d(poses)/d(depth, input poses) against PyTorch autograd of the oracle.

At this size the backward reaches what the small gradient tests never do: 1200 K1 pose-partial tiles per image, a
~19 k-point ICP target on the grid 1-NN path with the grid reused through the taped chain, ~75 reduction blocks per
element in the normal-equation and rigid-transform backward, and the look-back compaction over B x map bound flags."""
import os

import pytest
import torch

import gsx_oracle as oracle
from gradslam_b200.synthetic import make_sequence, punch_lattice_holes

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
B, L, H, W = 8, 2, 480, 640
SLAM_KW = dict(odom="gradicp", numiters=10, dsratio=4)


def _frames(gs, rgb, depth, K, poses):
    return gs.RGBDImages(rgb.to(DEV), depth, K.to(DEV), poses)


def test_config3_differentiable_poses_equal_fused_path():
    """bench.py's exact inputs (2 % random holes): all gradients finite, map sizes equal to the no-grad call's, and the
    recovered poses BIT-identical to the fused path's (gsx_icp_localize: gather, ICP loop and k_pose_compose in one
    call) - DESIGN.md section 1."""
    import gradslam_b200 as gs

    rgb, depth, K, poses = make_sequence(B, L, H, W, seed=0, yaw0=0.6)
    slam = gs.ICPSLAM(device=DEV, **SLAM_KW)
    d = depth.to(DEV).requires_grad_(True)
    p = poses.to(DEV).requires_grad_(True)
    pc, rec = slam(_frames(gs, rgb, d, K, p))
    rec.sum().backward()
    assert torch.isfinite(d.grad).all() and torch.isfinite(p.grad).all()
    assert d.grad.abs().max() > 0 and p.grad.abs().max() > 0
    with torch.no_grad():
        pc_f, rec_f = slam(_frames(gs, rgb, depth.to(DEV), K, poses.to(DEV)))
    assert pc.num_points_per_pointcloud.tolist() == pc_f.num_points_per_pointcloud.tolist()
    diff = (rec.detach() - rec_f).abs().max().item()
    assert torch.equal(rec.detach(), rec_f), "differentiable vs fused poses differ by up to %g" % diff


def _grad_stats(got, want):
    """(max |got - want| / max |want|, relative L2 error, fraction of elements outside rtol 5e-2 / atol 5e-3 max)."""
    got, want = got.double(), want.double()
    scale = want.abs().max().item()
    err = (got - want).abs()
    outside = (err > 5e-2 * want.abs() + 5e-3 * scale).double().mean().item()
    return err.max().item() / scale, (err.norm() / want.norm()).item(), outside


def test_config3_pose_gradients_match_oracle_autograd():
    """d(loss)/d(depth of both frames, input poses) for loss = sum(w * recovered pose of frame 1), against the oracle's
    autograd (oracle.run_slam, CPU float32 canonical order).  Lattice holes instead of random ones: no pixel has a
    degenerate normal (see tests/test_gpu_backward.py::make_sequence).  The GPU runs the whole batch of 8; the oracle
    runs elements 0 and 7 (GSX_FULLSIZE_ALL=1: all eight).  Frame 1's input pose never enters the computation (ICP
    replaces it), so its gradient is exactly zero on both sides; the bottom row of every pose gradient is zero.

    Bounds: the small-size test's elementwise tolerance (rtol 5e-2, atol 5e-3 of the largest gradient) on every element.
    Measured on one H100 80GB HBM3 (400 W), elements 0 / 7: the largest error is 2.5e-5 / 4.5e-5 of the largest
    gradient for depth[:, 0], 1.2e-6 / 1.1e-6 for depth[:, 1] and 6.1e-7 / 1.4e-6 for poses[:, 0]. The largest
    relative L2 error is 5.2e-5, and no element is outside the bound. No 1-NN association flipped, so no relative-L2
    or outlier-fraction bound is needed."""
    import gradslam_b200 as gs

    rgb, depth, K, poses = make_sequence(B, L, H, W, seed=0, yaw0=0.6, hole_fraction=0.0)
    depth = punch_lattice_holes(depth)
    w = torch.randn(B, 4, 4, generator=torch.Generator().manual_seed(8))
    checked = list(range(B)) if os.environ.get("GSX_FULLSIZE_ALL") == "1" else [0, B - 1]

    d_gpu = depth.to(DEV).requires_grad_(True)
    p_gpu = poses.to(DEV).requires_grad_(True)
    _, rec = gs.ICPSLAM(device=DEV, **SLAM_KW)(_frames(gs, rgb, d_gpu, K, p_gpu))
    (rec[:, 1] * w.to(DEV)).sum().backward()

    d_ref = depth[checked].clone().requires_grad_(True)
    p_ref = poses[checked].clone().requires_grad_(True)
    ref = oracle.run_slam(rgb[checked], d_ref, K[checked], p_ref, mode="aggregate", **SLAM_KW)
    (ref.poses[:, 1] * w[checked]).sum().backward()
    torch.testing.assert_close(rec.detach()[checked].cpu(), ref.poses.detach(), rtol=0, atol=1e-4)

    g_d, g_p = d_gpu.grad.cpu(), p_gpu.grad.cpu()
    assert torch.isfinite(g_d).all() and torch.isfinite(g_p).all()
    assert g_p[:, :, 3, :].abs().max() == 0
    assert g_p[:, 1].abs().max() == 0 and p_ref.grad[:, 1].abs().max() == 0
    for i, b in enumerate(checked):
        pairs = [("depth[%d, 0]" % b, g_d[b, 0], d_ref.grad[i, 0]), ("depth[%d, 1]" % b, g_d[b, 1], d_ref.grad[i, 1]),
                 ("poses[%d, 0]" % b, g_p[b, 0, :3], p_ref.grad[i, 0, :3])]
        for name, got, want in pairs:
            assert want.abs().max() > 0, name
            stats = "%s: max err %.3g of max, rel L2 %.3g, outside %.3g" % ((name,) + _grad_stats(got, want))
            torch.testing.assert_close(got, want, rtol=5e-2, atol=5e-3 * want.abs().max().item(),
                                       msg=lambda m, s=stats: s + "\n" + m)
            print(stats)
