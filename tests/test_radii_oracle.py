"""Surfel radii on the CPU: the radius and merge rules on hand-computed cases, the oracle's radii over a fused sequence,
the Pointclouds views, and the argument checks of the radii entry points (run before any CUDA call)."""
import math

import numpy as np
import pytest
import torch

import gsx_oracle as oracle
import radii_oracle as ro
from gradslam_b200.synthetic import make_sequence

F32 = torch.float32


def _f(x):
    return torch.tensor(x, dtype=F32)


def _k(f):
    """K^-1's diagonal entry for focal length f, as inverse_intrinsics rounds it."""
    return 1.0 / (_f(f) + 1e-6)


@pytest.mark.parametrize("fx,fy,d", [(525.0, 525.0, 1.0), (60.15625, 55.9453125, 2.7), (480.0, 500.0, 0.35)])
def test_fronto_parallel_plane_gives_sqrt2_d_over_f(fx, fy, d):
    k00, k11 = _k(fx), _k(fy)
    s = np.float32(0.5) * (np.float32(k00) + np.float32(k11))
    want = (np.float32(math.sqrt(2.0)) * np.float32(d)) * s
    for nz in (1.0, -1.0):
        r = ro.surfel_radius(_f(d), _f(nz), k00, k11)
        assert r.dtype == F32 and float(r) == float(want)
    assert math.isclose(float(want), math.sqrt(2.0) * d * 0.5 * (1 / fx + 1 / fy), rel_tol=1e-6)


def test_tilt_sixty_degrees_sits_on_the_branch_point_and_steeper_tilts_take_the_cap():
    k, d = _k(525.0), _f(1.5)
    r0 = ro.surfel_radius(d, _f(1.0), k, k)
    # cos 60 deg = 0.5 exactly: the cap's branch, and r0 / 0.5 is the same value
    assert float(ro.surfel_radius(d, _f(0.5), k, k)) == float(2.0 * r0) == float(r0 / 0.5)
    for deg in (61.0, 75.0, 89.9, 90.0):
        nz = _f(math.cos(math.radians(deg)))
        assert float(ro.surfel_radius(d, nz, k, k)) == float(2.0 * r0), deg
    assert float(ro.surfel_radius(d, _f(0.0), k, k)) == float(2.0 * r0)  # zero normal
    assert float(ro.surfel_radius(d, _f(-0.0), k, k)) == float(2.0 * r0)
    for deg in (10.0, 45.0, 59.0):  # below the cap: r0 / |n_z|
        nz = _f(math.cos(math.radians(deg)))
        assert float(ro.surfel_radius(d, nz, k, k)) == float(r0 / nz), deg
        assert float(ro.surfel_radius(d, -nz, k, k)) == float(r0 / nz), deg
    # just below the branch point |n_z| > 0.5 divides
    nz = torch.nextafter(_f(0.5), _f(1.0))
    assert float(ro.surfel_radius(d, nz, k, k)) == float(r0 / nz) < float(2.0 * r0)


def test_merge_rule_and_adoption_of_a_zero_radius():
    c0, alpha = _f([2.0, 0.75, 3.0, 0.0]), _f([1.0, 0.25, 0.5, 0.0])
    r_row, r = _f([3.0, 0.0, 0.01, 0.2]), _f([6.0, 0.5, 0.04, 0.3])
    got = ro.merge_radius(r_row, r, c0, alpha)
    tot = c0 + alpha
    inv = 1 / torch.where(tot == 0, torch.ones_like(tot), tot)
    assert float(got[0]) == 4.0  # (2 * 3 + 1 * 6) / 3
    assert float(got[1]) == 0.5  # a row without a radius takes the pixel's
    assert float(got[2]) == float(((c0[2] * r_row[2]) + (alpha[2] * r[2])) * inv[2])
    assert float(got[3]) == 0.0  # c0 + alpha == 0: inv = 1, the weighted sum is 0


def test_oracle_radii_follow_the_map_over_a_sequence():
    """The radii column has one entry per row, the first frame's radii are the pixel radii of its valid pixels in
    row-major order, every radius is positive, and the other columns are those of the oracle without radii."""
    rgb, depth, K, poses = make_sequence(2, 5, 24, 32, seed=11)
    pm, radii = ro.run_pointfusion(rgb, depth, K, poses)
    ref = oracle.run_slam(rgb, depth, K, poses, odom="gt").map
    assert pm.smap.counts() == ref.counts()
    for b in range(2):
        for got, want in ((pm.smap.points, ref.points), (pm.smap.normals, ref.normals),
                          (pm.smap.colors, ref.colors), (pm.smap.ccounts, ref.ccounts)):
            assert torch.equal(got[b], want[b])
        assert radii[b].shape == (ref.counts()[b], 1) and radii[b].dtype == F32
        assert bool((radii[b] > 0).all())
    maps = oracle.frame_maps(depth[:, :1], K, poses[:, :1])
    r_pix = ro.radius_image(depth[:, :1], maps, K)
    first, r_first = ro.run_pointfusion(rgb[:, :1], depth[:, :1], K, poses[:, :1])
    for b in range(2):
        assert torch.equal(r_first[b][:, 0], r_pix[b][maps["valid"][b, 0]])
    # a merged row's radius moved: some rows of the first frame were merged later and differ from their first value
    n0 = first.smap.counts()
    assert any(not torch.equal(radii[b][:n0[b]], r_first[b]) for b in range(2))


def test_pruned_oracle_radii_follow_the_kept_rows():
    rgb, depth, K, poses = make_sequence(2, 6, 24, 32, seed=12)
    pm0, r0 = ro.run_pointfusion(rgb, depth, K, poses)
    c = float(torch.quantile(torch.cat([x[:, 0] for x in pm0.smap.ccounts]).double(), 0.5, interpolation="lower"))
    pm, radii = ro.run_pointfusion(rgb, depth, K, poses, c_stable=c, t_max=2)
    assert sum(pm.smap.counts()) < sum(pm0.smap.counts())
    for b in range(2):
        assert radii[b].shape == (pm.smap.counts()[b], 1)
        assert bool((radii[b] > 0).all())


# ------------------------------------------------------------------ Pointclouds views
def test_pointclouds_radii_views_and_setter():
    import gradslam_b200 as gs

    pts = torch.rand(2, 5, 3)
    pc = gs.Pointclouds(points=pts, normals=torch.rand(2, 5, 3), features=torch.rand(2, 5, 1), device="cpu")
    assert pc.radii_padded.shape == (2, 5, 1) and bool((pc.radii_padded == 0).all())  # construction leaves 0
    assert pc.radii_padded.data_ptr() == pc._geo.data_ptr() + 7 * 4  # a strided view of slot 7
    held = pc.radii_padded
    r = torch.rand(2, 5, 1)
    pc.radii_padded = r
    assert torch.equal(pc.radii_padded, r) and bool((held == 0).all())  # written out of place
    assert torch.equal(pc.points_padded, pts)
    lst = [torch.full((5, 1), 0.25), torch.full((5, 1), 0.5)]
    pc.radii_list = lst
    assert [torch.equal(a, b) for a, b in zip(pc.radii_list, lst)] == [True, True]
    with pytest.raises(ValueError):
        pc.radii_padded = torch.rand(2, 5, 3)
    with pytest.raises(ValueError):
        pc.radii_list = [torch.rand(5, 2), torch.rand(5, 2)]


def test_surfel_radii_option_must_be_a_bool():
    import gradslam_b200 as gs

    with pytest.raises(TypeError, match="surfel_radii"):
        gs.PointFusion(odom="gt", surfel_radii=1)
    assert gs.PointFusion(odom="gt", surfel_radii=True).surfel_radii is True


# ------------------------------------------------------------------ C entry points
def _bufs(n):
    bufs = [torch.full((256,), -7.25) for _ in range(n)]
    assert all(t.data_ptr() % 16 == 0 for t in bufs)
    return bufs


@pytest.mark.parametrize("radii", [-1, 2, 7])
def test_merge_append_radii_refuses_bad_arguments_before_any_cuda_call(radii):
    from gradslam_b200 import _C

    lib = _C.lib()
    bufs = _bufs(7)
    geo, col, cin, cout, rgb, ws, flag = (t.data_ptr() for t in bufs)
    rc = lib.gsx_fusion_merge_append_radii(geo, col, 1, cin, cout, 16, rgb, 0, 1, 4, 4, ws, flag, None, radii, None)
    assert rc != 0 and b"surfel_radii" in lib.gsx_last_error()
    # also with an empty batch, which is otherwise a no-op
    rc = lib.gsx_fusion_merge_append_radii(None, None, 1, None, None, 16, None, 0, 0, 4, 4, None, None, None, radii,
                                           None)
    assert rc != 0 and b"surfel_radii" in lib.gsx_last_error()
    assert lib.gsx_fusion_merge_append_radii(None, None, 1, None, None, 16, None, 0, 0, 4, 4, None, None, None, 1,
                                             None) == 0
    rc = lib.gsx_fusion_merge_append_radii(None, col, 1, cin, cout, 16, rgb, 0, 1, 4, 4, ws, flag, None, 1, None)
    assert rc != 0 and b"null map pointer" in lib.gsx_last_error()
    rc = lib.gsx_fusion_merge_append_radii(geo, col, 1, cin, cin, 16, rgb, 0, 1, 4, 4, ws, flag, None, 1, None)
    assert rc != 0 and b"must not alias" in lib.gsx_last_error()
    for t in bufs:
        assert torch.equal(t, torch.full((256,), -7.25))


def test_sequence_radii_refuses_bad_arguments_before_any_cuda_call():
    from gradslam_b200 import _C

    lib = _C.lib()
    bufs = _bufs(9)
    geo, col, counts, depth, rgb, K, poses, ws, flag = (t.data_ptr() for t in bufs)

    def call(radii, s_begin=0, s_end=2, L=2, geo=geo):
        return lib.gsx_pointfusion_sequence_gt_radii(geo, col, counts, 16, 0, depth, rgb, K, poses, 1, L, s_begin,
                                                     s_end, 4, 4, 0.05, 0.94, 0.6, ws, None, 0, 0.0, None, 0, 0.0,
                                                     None, 0, flag, radii, None)

    for radii in (-1, 2):
        assert call(radii) != 0 and b"surfel_radii" in lib.gsx_last_error()
        assert call(radii, s_begin=1, s_end=1) != 0  # an empty frame range is checked too
    assert call(1, s_begin=2, s_end=1) != 0 and b"bad frame range" in lib.gsx_last_error()
    assert call(1, geo=None) != 0 and b"null map" in lib.gsx_last_error()
    assert call(1, s_begin=1, s_end=1) == 0  # nothing to do
    for t in bufs:
        assert torch.equal(t, torch.full((256,), -7.25))


# ------------------------------------------------------------------ disk-splat oracle
def _plane_case(r, M, normal=(0.0, 0.0, -1.0)):
    import splat_oracle as so

    K = torch.eye(4).view(1, 4, 4).clone()
    K[0, 0, 0] = K[0, 1, 1] = 100.0
    K[0, 0, 2] = K[0, 1, 2] = 10.0
    pts = torch.tensor([[[0.0, 0.0, 1.0]]])
    nrm = torch.tensor([[normal]])
    radii = torch.tensor([[[r]]])
    poses = torch.eye(4).view(1, 1, 4, 4)
    return so.splat_views(pts, nrm, pts.clone(), torch.ones(1, 1, 1), radii, [1], poses, K, 21, 21, M)


def test_splat_oracle_on_a_hand_built_plane():
    """A fronto-parallel disk of radius 2.5 pixels at depth 1 on the optical axis covers the 21 pixels within 2.5 pixels
    of the centre, all at depth exactly 1; the box clips it to 3 x 3 at max_splat_px = 1; a row without a radius or
    without a normal covers the centre pixel only; a disk behind the camera nothing."""
    out = _plane_case(0.025, 4)
    hh, ww = torch.meshgrid(torch.arange(21), torch.arange(21), indexing="ij")
    want = ((hh - 10) ** 2 + (ww - 10) ** 2) <= 6.25
    assert torch.equal(out.index[0, 0] == 0, want) and int(want.sum()) == 21
    assert bool((out.depth[0, 0][want] == 1.0).all()) and bool((out.depth[0, 0][~want] == 0).all())
    assert torch.equal(out.normals[0, 0][want], torch.tensor([0.0, 0.0, -1.0]).expand(21, 3))
    clipped = _plane_case(0.025, 1)
    assert int((clipped.index >= 0).sum()) == 9 and bool((clipped.index[0, 0, 9:12, 9:12] == 0).all())
    for r, normal in ((0.0, (0.0, 0.0, -1.0)), (0.025, (0.0, 0.0, 0.0))):
        one = _plane_case(r, 4, normal)
        assert int((one.index >= 0).sum()) == 1 and int(one.index[0, 0, 10, 10]) == 0
    # a 60-degree tilt about the y axis: the disk's footprint is an ellipse narrowed along w
    tilted = _plane_case(0.025, 4, (math.sin(math.radians(60)), 0.0, -0.5))
    cov = tilted.index[0, 0] == 0
    assert int(cov[10].sum()) < int(cov[:, 10].sum()) == 5
    # the depth of a covered pixel off the centre is where its ray meets the tilted plane
    w = 11
    d = (w - 10) / 100.0
    t = 1.0 / (1.0 - math.tan(math.radians(60)) * d)
    assert math.isclose(float(tilted.depth[0, 0, 10, w]), t, rel_tol=1e-5)


def test_render_pointclouds_refuses_a_bad_max_splat_px():
    import gradslam_b200 as gs

    pc = gs.Pointclouds(points=torch.rand(1, 4, 3))
    K, poses = torch.eye(4).view(1, 1, 4, 4), torch.eye(4).view(1, 1, 4, 4)
    for bad, err in ((-1, ValueError), (17, ValueError), (2.0, TypeError), (True, TypeError)):
        with pytest.raises(err, match="max_splat_px"):
            gs.render_pointclouds(pc, K, poses, 8, 8, max_splat_px=bad)


def test_splat_entry_points_refuse_a_bad_max_splat_px_before_any_cuda_call():
    from gradslam_b200 import _C

    lib = _C.lib()
    bufs = _bufs(4)
    K, poses, index, scratch = (t.data_ptr() for t in bufs)
    for bad in (-1, 17):
        rc = lib.gsx_render_splats(None, None, None, 0, 0, K, 0, poses, 16, 1, 1, 4, 4, index, None, None, None, None,
                                   bad, None)
        assert rc != 0 and b"max_splat_px" in lib.gsx_last_error()
        rc = lib.gsx_render_splats_bwd(None, None, 0, K, 0, poses, 16, index, 1, 1, 4, 4, None, None, None, None, None,
                                       None, None, scratch, 1024, bad, None)
        assert rc != 0 and b"max_splat_px" in lib.gsx_last_error()
    for t in bufs:
        assert torch.equal(t, torch.full((256,), -7.25))
