"""The upsampling oracle (tests/embedding_upsample_oracle.py) on the CPU: its samples against F.interpolate(bilinear,
align_corners=False) at integer and non-integer ratios, one-texel axes and the identity; its backward against float64
autograd of F.interpolate followed by the merge; the PointFusion oracle on coarse images against the full-resolution
oracle fed with the upsampled image."""
import pytest
import torch
import torch.nn.functional as F

import embedding_oracle as eo
import embedding_upsample_oracle as uo
from gradslam_b200.synthetic import make_sequence


def _interpolate(e, H, W, dtype=torch.float32):
    """F.interpolate of a (B, h, w, D) image in `dtype`, back in channels-last layout"""
    x = e.to(dtype).permute(0, 3, 1, 2)
    return F.interpolate(x, (H, W), mode="bilinear", align_corners=False).permute(0, 2, 3, 1)


@pytest.mark.parametrize("h, w, H, W", [
    (60, 80, 480, 640),  # stride 8
    (30, 40, 480, 640),  # stride 16
    (35, 46, 480, 640),  # non-integer ratios
    (5, 7, 23, 31),  # odd sizes
    (1, 9, 17, 29),  # one texel row
    (6, 1, 19, 13),  # one texel column
    (1, 1, 5, 6),
    (13, 17, 14, 17),  # nearly the depth's size
])
def test_samples_match_f_interpolate(h, w, H, W):
    g = torch.Generator().manual_seed(h * 100 + w)
    e = torch.rand((2, h, w, 3), generator=g) * 2 - 1
    got = uo.upsample(e, H, W)
    ref = _interpolate(e, H, W)
    assert got.shape == (2, H, W, 3) and got.dtype == torch.float32
    # A few ulp of the values (|e| < 1; F.interpolate may weight the taps in another order).  At a non-integer ratio
    # the float32 source coordinate sx itself is rounded, by up to an ulp of max(h, w) in either computation, which
    # moves the sample by that much times the spread of the taps (< 2).
    eps = torch.finfo(torch.float32).eps
    integer = H % h == 0 and W % w == 0
    atol = 4 * eps + (0 if integer else 2 * 2 * eps * max(h, w))
    torch.testing.assert_close(got, ref, rtol=0, atol=atol)
    torch.testing.assert_close(got.double(), _interpolate(e, H, W, torch.float64), rtol=0, atol=atol)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16])
def test_full_resolution_image_is_returned_as_is(dtype):
    e = (torch.rand((2, 9, 11, 5), generator=torch.Generator().manual_seed(1)) * 2 - 1).to(dtype)
    f = uo.upsample(e, 9, 11)
    assert f.dtype == torch.float32
    assert torch.equal(f, e.float())


def test_half_taps_are_upcast_exactly_and_the_sample_is_not_rounded():
    e = (torch.rand((1, 3, 4, 2), generator=torch.Generator().manual_seed(2)) * 2 - 1).to(torch.float16)
    f = uo.upsample(e, 7, 9)
    assert torch.equal(f, uo.upsample(e.float(), 7, 9))
    assert not torch.equal(f, f.half().float())


def test_taps_are_monotone_and_clamped():
    for n, m in ((480, 60), (480, 35), (17, 1), (13, 13), (31, 7)):
        i0, i1, l0, l1 = uo.taps(n, m)
        assert bool((i0[1:] >= i0[:-1]).all())
        assert int(i0.min()) == 0 and int(i1.max()) <= m - 1
        assert bool(((l0 >= 0) & (l0 <= 1) & (l1 >= 0) & (l1 <= 1)).all())


@pytest.mark.parametrize("h, w, H, W", [(3, 4, 24, 32), (5, 7, 23, 31), (1, 4, 9, 16), (6, 6, 6, 6)])
def test_backward_matches_float64_autograd_of_interpolate_and_merge(h, w, H, W):
    g = torch.Generator().manual_seed(h * 10 + w)
    B, D, N, cap = 2, 6, 15, 40  # N rows before the merge, cap after
    P = H * W
    E = torch.randn((B, N, D), generator=g)
    e = torch.randn((B, h, w, D), generator=g)
    c0 = torch.rand((B, P), generator=g) * 3
    alpha = torch.rand((B, P), generator=g)
    alpha[0, :5] = 0.0
    c0[0, :5] = 0.0  # degenerate merges (tot = 0)
    gr = torch.randn((B, cap, D), generator=g)
    assoc = torch.zeros((B, P), dtype=torch.int32)
    for b in range(B):  # merged into rows 0..14, appended as rows 15..34, the other pixels untouched
        pix = torch.randperm(P, generator=g)[:35]
        assoc[b, pix[:15]] = -(torch.arange(15, dtype=torch.int32) + 1)
        assoc[b, pix[15:]] = torch.arange(15, 35, dtype=torch.int32) + 1
    dE, de, dc0, dal = uo.merge_backward(assoc, c0, alpha, E, e, gr, H, W)

    Ed, ed = E.double().requires_grad_(True), e.double().requires_grad_(True)
    cd, ad = c0.double().requires_grad_(True), alpha.double().requires_grad_(True)
    f = _interpolate(ed, H, W, torch.float64).reshape(B, P, D)
    loss = 0
    for b in range(B):
        out = torch.cat([Ed[b], Ed.new_zeros((cap - N, D))], 0)
        a = assoc[b]
        m = (a < 0).nonzero().flatten()
        n = -a[m].long() - 1
        cb, ab = cd[b, m].unsqueeze(1), ad[b, m].unsqueeze(1)
        tot = cb + ab
        out[n] = (cb * Ed[b, n] + ab * f[b, m]) / torch.where(tot == 0, torch.ones_like(tot), tot)
        ap = (a > 0).nonzero().flatten()
        out[a[ap].long() - 1] = f[b, ap]
        loss = loss + (gr[b].double() * out).sum()
    loss.backward()
    tol = dict(rtol=1e-5, atol=1e-5)
    torch.testing.assert_close(dE.double(), Ed.grad, **tol)
    torch.testing.assert_close(de.double(), ed.grad, **tol)
    torch.testing.assert_close(dc0.double(), cd.grad, **tol)
    torch.testing.assert_close(dal.double(), ad.grad, **tol)
    assert float(de.abs().sum()) > 0


def test_adjoint_counts_a_clamped_tap_twice():
    # w = 1: both x taps land on texel 0, so each pixel adds lx0 * df + lx1 * df = df (up to rounding)
    df = torch.rand((1, 4, 5, 2), generator=torch.Generator().manual_seed(3))
    de = uo.upsample_adjoint(df, 4, 1)
    torch.testing.assert_close(de, df.sum(2, keepdim=True), rtol=1e-6, atol=1e-6)


@pytest.fixture(scope="module")
def seq():
    return make_sequence(2, 3, 24, 32, seed=72)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16])
def test_pointfusion_on_coarse_images_is_the_merge_of_the_samples(seq, dtype):
    """float32: the full-resolution oracle fed with the upsampled image; half: each appended sample rounded once and
    each merge rounded once per frame, as the full-resolution oracle rounds."""
    rgb, depth, K, poses = seq
    e = (torch.rand((2, 3, 3, 4, 5), generator=torch.Generator().manual_seed(4)) * 2 - 1).to(dtype)
    smap, got = uo.run_pointfusion(rgb, depth, K, poses, e)
    assert [int(x.shape[0]) for x in got] == smap.counts() and all(x.dtype == dtype for x in got)
    if dtype == torch.float32:
        _, ref = eo.run_pointfusion(rgb, depth, K, poses, uo.upsample(e, 24, 32))
        for a, b in zip(got, ref):
            assert torch.equal(a, b)
    full = eo.run_pointfusion(rgb, depth, K, poses, e.float().repeat_interleave(8, 2).repeat_interleave(8, 3))[1]
    assert any(not torch.equal(a.float(), b) for a, b in zip(got, full))  # (the sample is not a nearest lookup)
    agg, got = uo.run_aggregate(rgb, depth, K, poses, e)
    f = uo.upsample(e, 24, 32)
    for b in range(2):
        assert torch.equal(got[b], f[b][depth[b, ..., 0] > 0].to(dtype))
