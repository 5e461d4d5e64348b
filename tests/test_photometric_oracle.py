"""CPU checks of the photometric term's oracle (tests/photometric_oracle.py), of make_textured_sequence and of the
photometric_weight keyword's argument checks.  No GPU."""
import math

import pytest
import torch

import gsx_oracle as oracle
import photometric_oracle as ph
import projective_oracle as po
from gradslam_b200 import ICPSLAM, PointFusion
from gradslam_b200.synthetic import make_sequence, make_textured_sequence

# the weight of the tracking checks here and on the device (DESIGN.md section 4): colours in [0, 1]
W_TRACK = 0.1


def _camera(skew):
    K = torch.eye(4)
    K[0, 0], K[1, 1], K[0, 2], K[1, 2] = 30.0, 28.0, 15.5, 11.5
    if skew:
        K[0, 1], K[0, 3], K[1, 3] = 0.7, 0.35, -0.3
    return K


@pytest.mark.parametrize("skew", [False, True])
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_row_is_the_derivative_of_a_linear_ramp(skew, seed):
    """I_m linear in the pixel (dyadic slopes: the central differences are exact): c is the float64 gradient of the
    continuous I(pi(q(s))) with respect to s, and A_p = [c, s x c] is minus the derivative of r_p = I_s - I(pi(q(s)))
    under s -> s + v + omega x s."""
    g = torch.Generator().manual_seed(seed)
    H, W = 24, 32
    K = _camera(skew)
    prev = oracle.se3_exp(0.2 * torch.randn(6, generator=g))
    au, av, a0 = 0.25, -0.125, 0.5
    hh, ww = torch.meshgrid(torch.arange(H, dtype=torch.float32), torch.arange(W, dtype=torch.float32), indexing="ij")
    I_m = (au * ww + av * hh + a0).reshape(1, H * W)
    idx = torch.arange(H * W).view(1, H * W)
    valid, gu, gv = ph.stencil(I_m, idx, H, W)
    assert torch.equal(gu.view(H, W)[1:-1, 1:-1], torch.full((H - 2, W - 2), au))
    assert torch.equal(gv.view(H, W)[1:-1, 1:-1], torch.full((H - 2, W - 2), av))
    # points in front of the camera that project inside the border
    uv = torch.rand(40, 2, generator=g) * torch.tensor([W - 6.0, H - 6.0]) + 3.0
    z = 1.0 + torch.rand(40, generator=g)
    q = torch.stack([(uv[:, 0] - 15.5) / 30.0 * z, (uv[:, 1] - 11.5) / 28.0 * z, z], 1)
    s = oracle.rigid_apply(prev, q)
    _, j = po.associate(s.unsqueeze(0), prev.unsqueeze(0), K.unsqueeze(0), H, W, idx, torch.zeros(1, H * W, 3))
    j = j[0]
    assert (j >= 0).all()
    I_s = torch.rand(40, generator=g)
    A, r = ph.photometric_rows(s, I_s, j, valid[0], gu[0], gv[0], I_m[0], prev, K)
    assert A.shape == (40, 6)
    assert torch.equal(r[:, 0], I_s - I_m[0, j])

    Kd, Td = K.double(), prev.double()

    def ramp(x):  # continuous I(pi(q(x))), x (N,3) float64 world frame
        qq = (x - Td[:3, 3]) @ Td[:3, :3]
        h = qq @ Kd[:3, :3].t() + Kd[:3, 3]
        return au * h[:, 0] / h[:, 2] + av * h[:, 1] / h[:, 2] + a0

    sd = s.double().requires_grad_(True)
    c_ref, = torch.autograd.grad(ramp(sd).sum(), sd)
    torch.testing.assert_close(A[:, :3].double(), c_ref, rtol=1e-4, atol=1e-5)
    xi = torch.zeros(6, dtype=torch.float64, requires_grad=True)
    moved = s.double() + xi[:3] + torch.cross(xi[3:].expand(40, 3), s.double(), dim=1)
    rows = []
    for i in range(40):
        rows.append(torch.autograd.grad(I_s[i].double() - ramp(moved)[i], xi, retain_graph=True)[0])
    torch.testing.assert_close(A.double(), -torch.stack(rows), rtol=1e-4, atol=1e-5)


def test_rows_only_at_photometrically_valid_pixels():
    """A pixel on the border, or with an uncovered neighbour, has no photometric row; its geometric row stays."""
    H, W = 6, 7
    idx = torch.arange(H * W).view(1, H * W).clone()
    idx[0, 2 * W + 4] = -1  # uncovers (2,4): (2,3), (2,5), (1,4), (3,4) lose their row, (2,4) has none
    I_m = ph.model_intensity(torch.rand(1, H * W, 3), idx)
    assert I_m[0, 2 * W + 4] == 0
    valid, _, _ = ph.stencil(I_m, idx, H, W)
    v = valid.view(H, W)
    want = torch.zeros(H, W, dtype=torch.bool)
    want[1:-1, 1:-1] = True
    for h, w in ((2, 4), (2, 3), (2, 5), (1, 4), (3, 4)):
        want[h, w] = False
    assert torch.equal(v, want)


def test_intensity_is_rounded_per_operation():
    rgb = torch.rand(1000, 3, generator=torch.Generator().manual_seed(5))
    r, g, b = rgb.unbind(-1)
    t = lambda x: torch.tensor(x, dtype=torch.float32)
    assert torch.equal(ph.intensity(rgb), (t(0.299) * r + t(0.587) * g) + t(0.114) * b)


@pytest.mark.parametrize("odom", ["icp", "gradicp"])
def test_zero_weight_is_the_geometric_oracle(odom):
    rgb, depth, K, poses = make_textured_sequence(2, 3, 24, 32, seed=1, yaw0=0.6)
    want = po.run_slam(rgb, depth, K, poses, mode="icpslam", odom=odom, dsratio=2)
    got = ph.run_slam(rgb, depth, K, poses, w=0.0, mode="icpslam", odom=odom, dsratio=2)
    assert torch.equal(got.poses, want.poses)


@pytest.mark.parametrize("odom", ["icp", "gradicp"])
def test_joint_tracking_at_least_halves_the_far_wall_drift(odom):
    """yaw0 = 0: only the far wall is in view, so point-to-plane ICP cannot see sliding along it; the wall's texture
    can.  Over 8 frames at 120 x 160 the joint energy at W_TRACK must at least halve the final translation error."""
    rgb, depth, K, poses = make_textured_sequence(1, 8, 120, 160, seed=0, yaw0=0.0)
    geo = ph.translation_error(ph.run_slam(rgb, depth, K, poses, w=0.0, odom=odom).poses, poses)
    joint = ph.translation_error(ph.run_slam(rgb, depth, K, poses, w=W_TRACK, odom=odom).poses, poses)
    assert joint <= 0.5 * geo, (geo, joint)


def test_textured_sequence_keeps_make_sequence_geometry():
    a = make_textured_sequence(2, 3, 12, 16, seed=3, yaw0=0.6)
    b = make_textured_sequence(2, 3, 12, 16, seed=3, yaw0=0.6)
    ref = make_sequence(2, 3, 12, 16, seed=3, yaw0=0.6)
    for x, y in zip(a, b):
        assert torch.equal(x, y)
    for i in (1, 2, 3):  # depth (holes included), intrinsics, poses
        assert torch.equal(a[i], ref[i])
    assert a[0].min() >= 0.1 - 1e-6 and a[0].max() <= 0.9 + 1e-6


def test_textured_sequence_colour_follows_the_surface():
    """A room point keeps its colour across frames: the pixel of frame 1 that sees frame 0's centre surface point has
    (to interpolation) frame 0's centre colour."""
    H, W = 240, 320
    rgb, depth, K, poses = make_textured_sequence(1, 2, H, W, seed=0, hole_fraction=0.0)
    Kd, h, w = K[0, 0].double(), H // 2, W // 2
    d = depth[0, 0, h, w, 0].double()
    p0 = torch.stack([(w - Kd[0, 2]) / Kd[0, 0] * d, (h - Kd[1, 2]) / Kd[1, 1] * d, d, torch.ones((), dtype=torch.float64)])
    q1 = torch.linalg.inv(poses[0, 1].double()) @ p0
    u, v = Kd[0, 0] * q1[0] / q1[2] + Kd[0, 2], Kd[1, 1] * q1[1] / q1[2] + Kd[1, 2]
    u0, v0 = int(u.floor()), int(v.floor())
    fu, fv = float(u - u0), float(v - v0)
    c = rgb[0, 1].double()
    interp = ((1 - fu) * (1 - fv) * c[v0, u0] + fu * (1 - fv) * c[v0, u0 + 1] + (1 - fu) * fv * c[v0 + 1, u0]
              + fu * fv * c[v0 + 1, u0 + 1])
    torch.testing.assert_close(interp, rgb[0, 0, h, w].double(), atol=0.02, rtol=0)


@pytest.mark.parametrize("bad", [dict(B=0), dict(L=0), dict(H=-1), dict(W=2.5), dict(B=True), dict(yaw0=math.nan),
                                 dict(motion_scale=math.inf)])
def test_textured_sequence_rejects_bad_arguments(bad):
    args = dict(B=1, L=2, H=8, W=8)
    args.update(bad)
    with pytest.raises((TypeError, ValueError)):
        make_textured_sequence(args.pop("B"), args.pop("L"), args.pop("H"), args.pop("W"), **args)


@pytest.mark.parametrize("cls", [ICPSLAM, PointFusion])
@pytest.mark.parametrize("w,exc", [("0.1", TypeError), (True, TypeError), (None, TypeError), (-0.1, ValueError),
                                   (math.nan, ValueError), (math.inf, ValueError),
                                   (10 ** 400, ValueError), (1e39, ValueError)])
def test_photometric_weight_argument_checks(cls, w, exc):
    with pytest.raises(exc):
        cls(odom="gradicp", association="projective", photometric_weight=w, device="cpu")


@pytest.mark.parametrize("cls", [ICPSLAM, PointFusion])
def test_photometric_weight_needs_projective_association(cls):
    with pytest.raises(ValueError, match="projective"):
        cls(odom="icp", association="nn", photometric_weight=0.5, device="cpu")
    assert cls(odom="icp", association="nn", photometric_weight=0, device="cpu").photometric_weight == 0.0
    m = cls(odom="icp", association="projective", photometric_weight=2, device="cpu", target_splat_px=0)
    assert m.photometric_weight == 2.0
