"""CPU checks of the bilateral depth filter's oracle (tests/bilateral_oracle.py): the float32 and float64 statements
agree, autograd of the float64 statement is the written-out backward, invalid pixels pass through, and a depth step
much larger than sigma_range survives the filter."""
import numpy as np
import pytest
import torch

import bilateral_oracle as bo
from gradslam_b200.synthetic import add_depth_noise, make_sequence


def _scene(n=2, H=13, W=17, seed=0):
    rng = np.random.default_rng(seed)
    return (2.0 + 0.3 * rng.standard_normal((n, H, W)) * 0.1 + np.linspace(0, 0.2, W)).astype(np.float32)


@pytest.mark.parametrize("radius,ss,sr", [(1, 1.0, 0.05), (3, 2.0, 0.05), (7, 4.5, 0.1)])
def test_float32_and_float64_statements_agree(radius, ss, sr):
    d = _scene()
    d[0, 3, 4] = 0.0
    out32, den32 = bo.bilateral_f32(d, radius, ss, sr)
    out64, den64 = bo.bilateral_f64(torch.from_numpy(d.astype(np.float64)), radius, ss, sr)
    ulp = np.spacing(np.abs(out64.numpy()).astype(np.float32))
    # a float32 sum over the window's 2r+1 rows of 2r+1 terms: a few ulps per row
    assert np.all(np.abs(out32 - out64.numpy()) <= 2 * (2 * radius + 1) * ulp)
    np.testing.assert_allclose(den32, den64.numpy(), rtol=1e-5)


@pytest.mark.parametrize("radius", [1, 2, 3])
def test_autograd_of_the_float64_statement_is_the_written_out_backward(radius):
    d = _scene(n=2, H=7, W=9, seed=radius)
    d[0, 2, 3] = 0.0
    d[1, 0, 0] = np.nan
    d[1, 4, 5] = np.inf
    ss, sr = 1.5, 0.04
    keep = bo.keep_masks(d, radius, ss, sr)
    x = torch.from_numpy(d.astype(np.float64)).requires_grad_(True)
    fn = lambda t: bo.bilateral_f64(t, radius, ss, sr, keep)[0]  # noqa: E731
    g = torch.from_numpy(np.random.default_rng(7).standard_normal(d.shape))
    auto, = torch.autograd.grad(fn(x), x, g)
    formula, mag = bo.bilateral_bwd_formula(d, g.numpy(), radius, ss, sr)
    np.testing.assert_allclose(auto.numpy(), formula, rtol=1e-10, atol=1e-12 * mag.max())
    # the float64 statement's own derivative, by finite differences, on the valid pixels (the masks held fixed)
    fin = torch.from_numpy(np.where(np.isfinite(d) & (d > 0), d, 1.0).astype(np.float64)).requires_grad_(True)
    keep_fin = bo.keep_masks(fin.detach().numpy().astype(np.float32), radius, ss, sr)
    assert torch.autograd.gradcheck(lambda t: bo.bilateral_f64(t, radius, ss, sr, keep_fin)[0], (fin,), eps=1e-7,
                                    atol=1e-5, rtol=1e-4)


def test_invalid_centres_pass_through_and_invalid_neighbours_are_ignored():
    d = np.full((1, 5, 5), 2.0, dtype=np.float32)
    bad = [(0, 0, 0.0), (1, 1, -1.0), (2, 2, np.nan), (3, 3, np.inf)]
    for y, x, v in bad:
        d[0, y, x] = v
    out, den = bo.bilateral_f32(d, 2, 2.0, 0.05)
    for y, x, v in bad:
        assert np.array_equal(out[0, y, x], np.float32(v), equal_nan=True)
        assert den[0, y, x] == 0
    valid = (d > 0) & np.isfinite(d)
    np.testing.assert_allclose(out[valid], 2.0, rtol=2e-6)  # only the constant valid depth was averaged
    # a pixel whose whole window is invalid keeps its depth (its own weight is 1)
    lone = np.zeros((1, 3, 3), dtype=np.float32)
    lone[0, 1, 1] = 1.25
    out, den = bo.bilateral_f32(lone, 1, 1.0, 0.05)
    assert out[0, 1, 1] == np.float32(1.25) and den[0, 1, 1] == 1


def test_a_depth_step_much_larger_than_sigma_range_is_preserved():
    d = np.full((1, 16, 16), 1.5, dtype=np.float32)
    d[:, :, 8:] = 3.0  # a 1.5 m step; sigma_range 3 cm
    out, _ = bo.bilateral_f32(d, 5, 3.0, 0.03)
    np.testing.assert_allclose(out, d, rtol=2e-6)  # no pair across the step is kept: each side averages itself


def test_the_filter_reduces_noise_on_a_plane():
    depth = torch.full((1, 1, 48, 64, 1), 2.5)
    noisy = add_depth_noise(depth, seed=3)[0, :, :, :, 0].numpy()
    out, _ = bo.bilateral_f32(noisy, 3, 2.0, 0.05)
    assert np.median(np.abs(out - 2.5)) < 0.5 * np.median(np.abs(noisy - 2.5))


def test_add_depth_noise_is_seeded_and_keeps_holes():
    _, depth, _, _ = make_sequence(1, 2, 24, 32, seed=1)
    a, b = add_depth_noise(depth, seed=5), add_depth_noise(depth, seed=5)
    assert torch.equal(a, b) and not torch.equal(a, add_depth_noise(depth, seed=6))
    assert a.dtype == torch.float32 and a.shape == depth.shape
    assert torch.equal(a == 0, depth == 0) and bool((a >= 0).all())
    z = depth[depth > 0].double()
    sigma = 0.0012 + 0.0019 * (z - 0.4) ** 2
    r = (a[depth > 0].double() - z) / sigma
    assert abs(float(r.mean())) < 0.05 and abs(float(r.std()) - 1.0) < 0.05
