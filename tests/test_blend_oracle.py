"""The blended splat render on the CPU: the oracle against the disk-splat and one-pixel oracles where only the front row
can contribute, a hand-built two-disk case with known weights, and the argument checks of render_pointclouds and of
the C entry points (run before any CUDA call)."""
import math

import pytest
import torch

import blend_oracle as bo
import render_oracle
import splat_oracle as so

F64 = torch.float64


def _map(seed, B=2, N=300, H=24, W=32):
    """Random ragged maps in front of a camera per element, about half the rows with radii of 0.3 .. 3 pixels."""
    g = torch.Generator().manual_seed(seed)
    K = torch.eye(4).repeat(B, 1, 1)
    for b in range(B):
        K[b, 0, 0], K[b, 1, 1] = 30.0 + 3 * b, 29.0 - 2 * b
        K[b, 0, 2], K[b, 1, 2] = W / 2 - 0.5 + b, H / 2 - 0.5
    z = torch.rand(B, N, generator=g) * 2.0 + 0.5
    u, v = torch.rand(B, N, generator=g) * (W + 4) - 2, torch.rand(B, N, generator=g) * (H + 4) - 2
    pts = torch.stack([(u - K[:, 0, 2:3]) / K[:, 0, 0:1] * z, (v - K[:, 1, 2:3]) / K[:, 1, 1:2] * z, z], -1)
    nrm = torch.nn.functional.normalize(torch.randn(B, N, 3, generator=g) + torch.tensor([0.0, 0.0, -2.0]), dim=-1)
    col = torch.rand(B, N, 3, generator=g)
    cc = torch.randint(1, 20, (B, N, 1), generator=g).float()
    radii = torch.rand(B, N, 1, generator=g) * 0.09 + 0.01
    radii[torch.rand(B, N, generator=g) < 0.5] = 0.0
    counts = [N, N - 70][:B]
    for b, c in enumerate(counts):
        pts[b, c:], nrm[b, c:], col[b, c:], cc[b, c:], radii[b, c:] = 0, 0, 0, 0, 0
    poses = torch.eye(4).repeat(B, 2, 1, 1)
    poses[:, 1, 0, 3] = 0.03
    return pts, nrm, col, cc, radii, counts, poses, K


@pytest.mark.parametrize("M", [0, 1, 3])
def test_zero_band_on_distinct_depths_is_the_z_buffer(M):
    H, W = 24, 32
    pts, nrm, col, cc, radii, counts, poses, K = _map(1, H=H, W=W)
    con, index, _ = bo.contributors(pts, nrm, radii, counts, poses, K, H, W, M, 0.0)
    # distinct depths: exactly one contributor, the front row, per covered pixel
    assert torch.equal(torch.bincount(con.slot, minlength=index.numel()), (index >= 0).view(-1).long())
    assert int(con.disk.sum()) > (100 if M else -1) and int((~con.disk).sum()) > 50
    d = lambda t: t.to(F64)
    got = bo.blend_values(d(pts), d(nrm), d(col), d(cc), radii, d(poses), K, con, index)
    if M == 0:
        smap_want = render_oracle.render_values(d(pts), d(nrm), d(col), d(cc), d(poses), index)
    else:
        smap_want = so.splat_values(d(pts), d(nrm), d(col), d(cc), radii, d(poses), K, index)
    for name in ("depth", "rgb", "normals"):
        torch.testing.assert_close(getattr(got, name), getattr(smap_want, name), rtol=1e-12, atol=1e-12)
    # the blended confidence is the front row's weight: c (1 - s2/r^2) <= c
    assert bool((got.confidence <= smap_want.confidence + 1e-12).all())


def _two_disks(band, c=(2.0, 3.0)):
    K = torch.eye(4).view(1, 4, 4).clone()
    K[0, 0, 0] = K[0, 1, 1] = 100.0
    K[0, 0, 2] = K[0, 1, 2] = 10.0
    pts = torch.tensor([[[0.0, 0.0, 1.0], [0.0, 0.0, 1.01]]])
    nrm = torch.tensor([[[0.0, 0.0, -1.0], [0.0, 0.0, -1.0]]])
    col = torch.tensor([[[1.0, 0.0, 0.0], [0.0, 1.0, 0.0]]])
    cc = torch.tensor([[[c[0]], [c[1]]]])
    radii = torch.tensor([[[0.025], [0.025]]])
    poses = torch.eye(4).view(1, 1, 4, 4)
    return bo.blend_views(*(t.double() for t in (pts, nrm, col, cc)), radii, [2], poses.double(), K, 21, 21, 4, band)


def test_two_fronto_parallel_disks_have_known_weights():
    out = _two_disks(0.02)
    assert int(out.index[0, 0, 10, 10]) == 0
    # the centre pixel: both disks at s = 0 (up to K^-1's rounding), weights c
    torch.testing.assert_close(out.confidence[0, 0, 10, 10, 0], torch.tensor(5.0, dtype=F64), rtol=1e-6, atol=0)
    torch.testing.assert_close(out.depth[0, 0, 10, 10, 0], torch.tensor((2 * 1.0 + 3 * 1.01) / 5, dtype=F64),
                               rtol=1e-6, atol=0)
    torch.testing.assert_close(out.rgb[0, 0, 10, 10], torch.tensor([0.4, 0.6, 0.0], dtype=F64), rtol=1e-5, atol=1e-6)
    # one pixel right: the ray (0.01, 0, 1) meets disk 0 at s = 0.01 and disk 1 at s = 0.0101
    w0, w1 = 2 * (1 - 0.01 ** 2 / 0.025 ** 2), 3 * (1 - 0.0101 ** 2 / 0.025 ** 2)
    torch.testing.assert_close(out.confidence[0, 0, 10, 11, 0], torch.tensor(w0 + w1, dtype=F64), rtol=1e-5, atol=0)
    torch.testing.assert_close(out.depth[0, 0, 10, 11, 0], torch.tensor((w0 * 1.0 + w1 * 1.01) / (w0 + w1),
                                                                         dtype=F64), rtol=1e-6, atol=0)
    torch.testing.assert_close(out.normals[0, 0, 10, 11], torch.tensor([0.0, 0.0, -1.0], dtype=F64))
    # a band narrower than the gap: the front disk alone, at its weight
    near = _two_disks(0.005)
    torch.testing.assert_close(near.depth[0, 0, 10, 11, 0], torch.tensor(1.0, dtype=F64), rtol=1e-6, atol=0)
    torch.testing.assert_close(near.confidence[0, 0, 10, 11, 0], torch.tensor(w0, dtype=F64), rtol=1e-5, atol=0)
    # zero confidence on both: W = 0, and the pixel shows zeros while the index keeps the front row
    zero = _two_disks(math.inf, c=(0.0, 0.0))
    assert int(zero.index[0, 0, 10, 10]) == 0
    assert bool((zero.depth == 0).all()) and bool((zero.rgb == 0).all()) and bool((zero.confidence == 0).all())


def test_render_pointclouds_refuses_a_bad_blend_band_and_intrinsics_that_require_grad():
    import gradslam_b200 as gs

    pc = gs.Pointclouds(points=torch.rand(1, 4, 3))
    K, poses = torch.eye(4).view(1, 1, 4, 4), torch.eye(4).view(1, 1, 4, 4)
    for bad, err in ((-0.1, ValueError), (float("nan"), ValueError), (-math.inf, ValueError), (True, TypeError),
                     ("0.1", TypeError), (torch.tensor(0.1), TypeError), ([0.1], TypeError)):
        with pytest.raises(err, match="blend_band"):
            gs.render_pointclouds(pc, K, poses, 8, 8, blend_band=bad)
    with pytest.raises(ValueError, match="intrinsics"):
        gs.render_pointclouds(pc, K.clone().requires_grad_(True), poses, 8, 8, max_splat_px=2, blend_band=0.01)


def _bufs(n):
    bufs = [torch.full((4096,), -7.25) for _ in range(n)]
    assert all(t.data_ptr() % 16 == 0 for t in bufs)
    return bufs


def test_blend_entry_points_refuse_bad_arguments_before_any_cuda_call():
    from gradslam_b200 import _C

    lib = _C.lib()
    bufs = _bufs(12)
    geo, col, counts, K, poses, index, front, weight, depth, rgb, nrm, scratch = (t.data_ptr() for t in bufs)
    need = lib.gsx_render_blend_scratch_bytes(1, 1, 4, 4, 8, 1)
    assert need > 0 and lib.gsx_render_blend_scratch_bytes(1, 1, 4, 4, 8, 17) == -1

    def fwd(B=1, L=1, H=4, W=4, M=1, band=0.01, geo=geo, index=index, weight=weight, scratch=scratch, nbytes=need,
            cap=16, max_count=8):
        return lib.gsx_render_blend(geo, col, counts, cap, max_count, K, 16, poses, 16, B, L, H, W, 1, band, M, index,
                                    front, weight, depth, rgb, nrm, scratch, nbytes, None)

    def bwd(B=1, M=1, band=0.01, fr=front, nbytes=4096 * 4, g_depth=None):
        return lib.gsx_render_blend_bwd(geo, col, counts, 16, 8, K, 16, poses, 16, B, 1, 4, 4, 1, band, M, fr, weight,
                                        None, None, None, g_depth, None, None, None, geo, col, depth, scratch, nbytes,
                                        None)

    refused = [(lambda: fwd(B=0), b"bad extents"), (lambda: fwd(H=-1), b"bad extents"),
               (lambda: fwd(M=-1), b"max_splat_px"), (lambda: fwd(M=17), b"max_splat_px"),
               (lambda: fwd(band=-1.0), b"blend_band"), (lambda: fwd(band=math.nan), b"blend_band"),
               (lambda: fwd(geo=None), b"null map pointer"), (lambda: fwd(index=None), b"null pointer"),
               (lambda: fwd(weight=None), b"null pointer"), (lambda: fwd(scratch=None), b"scratch too small"),
               (lambda: fwd(nbytes=need - 1), b"scratch too small"), (lambda: fwd(max_count=17), b"max_count"),
               (lambda: fwd(L=40000, H=300, W=300), b"overflows"),
               (lambda: bwd(B=0), b"bad extents"), (lambda: bwd(M=17), b"max_splat_px"),
               (lambda: bwd(band=math.nan), b"blend_band"), (lambda: bwd(fr=None), b"null pointer"),
               (lambda: bwd(nbytes=0), b"scratch too small"), (lambda: bwd(g_depth=depth), b"g_depth without")]
    for call, msg in refused:
        rc = call()
        assert rc != 0 and msg in lib.gsx_last_error(), (msg, lib.gsx_last_error())
    for t in bufs:
        assert torch.equal(t, torch.full((4096,), -7.25))
