"""CPU checks of the splat-target oracle (tests/projective_splat_oracle.py) and of the `target_splat_px` keyword."""
import math

import pytest
import torch

import gsx_oracle as oracle
import projective_oracle as po
import projective_splat_oracle as pso

H, W = 21, 21


def _camera():
    """K with fx = fy = 100 and the principal point at the centre pixel, and a previous pose that is not the identity."""
    K = torch.eye(4).view(1, 4, 4).clone()
    K[0, 0, 0], K[0, 1, 1] = 100.0, 100.0
    K[0, 0, 2] = K[0, 1, 2] = 10.0
    pose = oracle.se3_exp(torch.tensor([0.03, -0.02, 0.05, 0.1, -0.05, 0.2])).view(1, 4, 4)
    return K, pose


def _map(rows_cam, normals_cam, radii, pose):
    """A one-element SurfelMap of rows given in the previous camera's frame."""
    R, t = pose[0, :3, :3], pose[0, :3, 3]
    pts = rows_cam @ R.T + t
    nrm = normals_cam @ R.T
    return oracle.SurfelMap([pts], [nrm]), [torch.tensor(radii, dtype=torch.float32).view(-1, 1)]


def test_zero_splat_px_and_maps_without_radii_are_the_point_targets():
    smap, _, _, pose, K = po.small_case(6, 8)
    radii = [torch.full((p.shape[0], 1), 0.3) for p in smap.points]
    want = po.target_images(smap, pose, K, 6, 8)
    for got in (pso.target_images(smap, radii, pose, K, 6, 8, 0),
                pso.target_images(smap, [torch.zeros_like(r) for r in radii], pose, K, 6, 8, 3)):
        for g, w in zip(got, want):
            assert torch.equal(g, w)
    # with radii the disks cover more pixels
    idx3 = pso.target_images(smap, radii, pose, K, 6, 8, 3)[0]
    assert int((idx3 >= 0).sum()) > int((want[0] >= 0).sum())


def test_oblique_disk_takes_the_surface_point_of_each_pixel():
    """A disk of radius 4 pixels at depth 1, tilted 50 degrees about the camera's y axis: every pixel it wins gets the
    point where the pixel's ray meets the disk's plane, prev · (t K^-1 (w, h, 1)), computed here in float64."""
    K, pose = _camera()
    a = math.radians(50)
    n_cam = torch.tensor([[math.sin(a), 0.0, -math.cos(a)]])
    smap, radii = _map(torch.tensor([[0.0, 0.0, 1.0]]), n_cam, [0.04], pose)
    idx, tgt_p, tgt_n = pso.target_images(smap, radii, pose, K, H, W, 6)
    won = (idx[0] == 0).nonzero().flatten()
    assert 10 < won.numel() < 60
    q, m = torch.tensor([0.0, 0.0, 1.0], dtype=torch.float64), n_cam[0].double()
    R, c = pose[0, :3, :3].double(), pose[0, :3, 3].double()
    for j in won.tolist():
        h, w = divmod(j, W)
        d = torch.tensor([(w - 10) / 100.0, (h - 10) / 100.0, 1.0], dtype=torch.float64)
        t = torch.dot(m, q) / torch.dot(m, d)
        x = R @ (t * d) + c
        torch.testing.assert_close(tgt_p[0, j].double(), x, rtol=0, atol=2e-6)
        assert float((t * d - q).norm()) <= 0.04 + 1e-6  # on the disk
    assert torch.equal(tgt_n[0, won], smap.normals[0].expand(won.numel(), 3))
    # the centre row's own point only where the ray passes through it
    assert not torch.equal(tgt_p[0, won], smap.points[0].expand(won.numel(), 3))


def test_one_pixel_rows_keep_their_position_and_win_only_by_depth():
    """A fronto-parallel disk of radius 5.25 pixels at depth 2 with two rows without a radius inside its footprint: the
    one in front (depth 1.9) wins its pixel and keeps its position; the one behind (depth 2.1) loses it to the disk."""
    K, pose = _camera()
    rows = torch.tensor([[0.0, 0.0, 2.0], [0.02, 0.0, 1.9], [-0.042, 0.0, 2.1]])
    normals = torch.tensor([[0.0, 0.0, -1.0]] * 3)
    smap, radii = _map(rows, normals, [0.105, 0.0, 0.0], pose)
    idx, tgt_p, _ = pso.target_images(smap, radii, pose, K, H, W, 4)
    front, behind = 10 * W + 11, 10 * W + 8  # u = 100 * x / z + 10
    assert int(idx[0, front]) == 1 and torch.equal(tgt_p[0, front], smap.points[0][1])
    assert int(idx[0, behind]) == 0
    assert int((idx[0] == 0).sum()) == 76  # the 9 x 9 box less its 4 corners (5.25 pixels) and the front row's pixel
    # with M = 0 every row covers its one pixel
    idx0 = pso.target_images(smap, radii, pose, K, H, W, 0)[0]
    assert sorted(idx0[0][idx0[0] >= 0].tolist()) == [0, 1, 2]


@pytest.mark.parametrize("cls", ["ICPSLAM", "PointFusion"])
def test_target_splat_px_argument_errors(cls):
    import gradslam_b200 as gs

    kw = dict(surfel_radii=True) if cls == "PointFusion" else {}
    make = lambda **k: getattr(gs, cls)(odom="icp", association="projective", **kw, **k)
    for bad in (1.0, True, "3", None):
        with pytest.raises(TypeError, match="target_splat_px"):
            make(target_splat_px=bad)
    for bad in (-1, 17):
        with pytest.raises(ValueError, match="target_splat_px"):
            make(target_splat_px=bad)
    with pytest.raises(ValueError, match="association"):
        getattr(gs, cls)(odom="icp", target_splat_px=2, **kw)
    with pytest.raises(TypeError):
        getattr(gs, cls)("icp", "projective")  # keyword-only
    for m in (0, 1, 16):
        assert make(target_splat_px=m).target_splat_px == m
    assert getattr(gs, cls)(odom="gt").target_splat_px == 0
    assert getattr(gs, cls)(odom="gt", association="projective", target_splat_px=3, **kw).target_splat_px == 3


def test_pointfusion_refuses_splat_targets_without_radii():
    import gradslam_b200 as gs

    with pytest.raises(ValueError, match="surfel_radii"):
        gs.PointFusion(odom="gradicp", association="projective", target_splat_px=3)
    assert gs.PointFusion(odom="gradicp", association="projective", target_splat_px=0).target_splat_px == 0


def test_projective_entry_points_refuse_a_bad_max_splat_px_before_any_cuda_call():
    from gradslam_b200 import _C

    lib = _C.lib()
    bufs = [torch.full((256,), -7.25) for _ in range(9)]
    geo, counts, depth, K, prev, out, ws, index, tgt = (t.data_ptr() for t in bufs)
    for bad in (-1, 17):
        rc = lib.gsx_icp_localize_projective(geo, counts, 4, 4, depth, 16, K, 16, prev, 16, 1, 4, 4, 1, 1, 1, 1e-8, 0,
                                             0.0, 2.0, 1.0, 1.0, 200.0, out, 16, ws, 1 << 20, bad, None, None, 0, 0.0,
                                             math.inf, math.inf, None)
        assert rc != 0 and b"max_splat_px" in lib.gsx_last_error()
        rc = lib.gsx_icp_projective_targets(geo, None, counts, 4, 4, K, 16, prev, 16, 1, 4, 4, bad, index, tgt, tgt,
                                            None, None)
        assert rc != 0 and b"max_splat_px" in lib.gsx_last_error()
    for t in bufs:
        assert torch.equal(t, torch.full((256,), -7.25))
