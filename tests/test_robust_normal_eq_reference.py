"""CPU checks of the Huber scales of the float64 joint normal-equation reference (tests/joint_normal_eq_reference.py):
at +inf it is the unweighted reference bit for bit, in float32 its per-row products are robust_oracle's, both branches
carry rows at the median scales, its bounds and per-row terms are consistent, and a residual exactly on the scale takes
the inside branch, decided on the float32 residual.  No GPU."""
import math

import numpy as np
import pytest
import torch

import gsx_oracle as oracle
import joint_normal_eq_reference as jr
import photometric_oracle as ph
import projective_oracle as po
import robust_oracle as ro
from cameras import camera_intrinsics

W_TRACK = 0.1
INF = math.inf
H, W = 60, 80


def _case(n=3000, seed=0, skew=0.75):
    K = torch.from_numpy(camera_intrinsics(2, H, W, skew=skew)[1])
    prev = oracle.se3_exp(torch.tensor([0.1, -0.05, 0.2, 0.15, -0.2, 0.1])).double()
    return jr.synthetic_element(H, W, n, K, prev, seed)


def _medians(x, idx, index):
    """The float32 medians of |r| and |r_p|: scales with rows on both sides."""
    r, rp, _ = jr.float32_residuals(*(x[k] for k in jr.NAMES[:5]), idx, index, H, W)
    return float(r.abs().median()), float(rp.abs().median())


def _scale_cases(x, idx, index):
    d, dp = _medians(x, idx, index)
    return [(d, INF), (INF, dp), (d, dp)]


def _same(a, b):
    if isinstance(a, dict):
        assert a.keys() == b.keys()
        for k in a:
            _same(a[k], b[k])
    else:
        assert torch.equal(a, b)


def test_infinite_scales_are_the_unweighted_reference_bit_for_bit():
    """Explicit +inf, and a scale past the largest float32 (it rounds to +inf as the kernels' float parameter does),
    give the default reference: sums, bounds, gradients and per-row terms."""
    x, idx, index = _case(n=800, seed=1)
    g = torch.randn(28, generator=torch.Generator().manual_seed(1))
    want = jr.reference(x, idx, index, H, W, W_TRACK, 4, g)
    for d, dp in ((INF, INF), (1e39, INF), (INF, 1e39), (1e39, 1e39)):
        _same(jr.reference(x, idx, index, H, W, W_TRACK, 4, g, delta=d, delta_p=dp), want)
    # the largest finite float32 keeps every row inside: the robust statement, summed row by row, is the same sums
    fm = float(np.finfo(np.float32).max)
    got = jr.reference(x, idx, index, H, W, W_TRACK, 4, g, delta=fm, delta_p=fm)
    torch.testing.assert_close(got["sums"], want["sums"], rtol=1e-12, atol=0)
    for k in jr.NAMES:
        torch.testing.assert_close(got["grad"][k], want["grad"][k], rtol=1e-10, atol=1e-12)
        assert (got["grad_bound"][k] >= want["grad_bound"][k]).all()  # (R_B_ROBUST > R_B)
    torch.testing.assert_close(got["sum_bound"], want["sum_bound"], rtol=1e-12, atol=0)


@pytest.mark.parametrize("case", [0, 1, 2])
def test_float32_pair_rows_are_robust_oracle_row_products(case):
    """In float32 the pair values are robust_oracle.row_products(A, r, delta) plus row_products(A_p, r_p, delta_p, w)
    bit for bit, and magnitudes and running errors are at least |value|."""
    x, idx, index = _case(seed=2)
    d, dp = _scale_cases(x, idx, index)[case]
    mx = {k: v.abs() for k, v in x.items()}
    vals, mags, errs, (A, r), (Ap, rp), vj = jr._pair_rows(x, mx, idx, index, H, W, W_TRACK, delta=d, delta_p=dp)
    A_ref, b_ref = po._rows(x["src"], x["tgt"], x["tgt_n"], idx)
    I_m = ph.intensity(x["model_col"])
    valid, gu, gv = ph.stencil(I_m.unsqueeze(0), index.unsqueeze(0), H, W)
    Ap_ref, rp_ref = ph.photometric_rows(x["src"], ph.intensity(x["src_col"]), idx, valid[0], gu[0], gv[0], I_m,
                                         x["prev"], x["K"])
    want = ro.row_products(A_ref, b_ref[:, 0], d)
    want[vj] = want[vj] + ro.row_products(Ap_ref, rp_ref[:, 0], dp, w=W_TRACK)
    assert torch.equal(vals.t(), want)
    assert (mags >= vals.abs()).all() and (errs >= vals.abs()).all()
    # and the scales change the products of the rows outside them
    plain = jr._pair_rows(x, mx, idx, index, H, W, W_TRACK)[0]
    out = torch.zeros(vals.shape[1], dtype=torch.bool)
    if not math.isinf(d):
        out |= b_ref[:, 0].abs() > d
    if not math.isinf(dp):
        out[vj] |= rp_ref[:, 0].abs() > dp
    assert out.any() and not out.all()
    assert torch.equal(vals[:, ~out], plain[:, ~out])
    assert not torch.equal(vals[27, out], plain[27, out])


def test_both_branches_carry_rows_at_the_median_scales():
    x, idx, index = _case()
    d, dp = _medians(x, idx, index)
    assert 0.003 < d < 0.015 and 0.05 < dp < 0.5, (d, dp)
    r, rp, vj = jr.float32_residuals(*(x[k] for k in jr.NAMES[:5]), idx, index, H, W)
    assert rp.numel() > 500
    for res, s in ((r, d), (rp, dp)):
        share = float((res.abs() > s).double().mean())
        assert 0.45 < share < 0.55, share
    plain = jr.joint_sums(*(x[k].double() for k in jr.NAMES), idx, index, H, W, W_TRACK)
    for dd, ddp in _scale_cases(x, idx, index):
        got = jr.joint_sums(*(x[k].double() for k in jr.NAMES), idx, index, H, W, W_TRACK, dd, ddp)
        assert ((got - plain).abs() > 1e-9 * plain.abs()).all(), (dd, ddp)


@pytest.mark.parametrize("case", [0, 1, 2])
def test_robust_per_row_terms_sum_to_the_gradient_and_bounds_cover_the_values(case):
    x, idx, index = _case(seed=6)
    d, dp = _scale_cases(x, idx, index)[case]
    g = torch.randn(28, generator=torch.Generator().manual_seed(1))
    ref = jr.reference(x, idx, index, H, W, W_TRACK, jr.blocks_of(idx.numel()), g, delta=d, delta_p=dp)
    for name in ("prev", "K"):
        terms = ref["row_terms"][name].sum(0).view(3, 4)
        torch.testing.assert_close(terms, ref["grad"][name][:3], rtol=1e-12, atol=1e-12 * terms.abs().max().item())
        assert (ref["grad"][name][3] == 0).all() and (ref["grad_bound"][name][3] == 0).all()
    assert ref["grad"]["K"][0, 1] != 0 and (ref["grad"]["K"][:3, 3] != 0).all()
    for name in jr.NAMES:
        grad, bound = ref["grad"][name], ref["grad_bound"][name]
        assert ((grad == 0) | (bound > 0)).all(), name
        assert (bound >= jr.R_B_ROBUST * jr.U32 * grad.abs() * (1 - 1e-9)).all(), name
    assert (ref["sum_bound"] >= 14 * jr.U32 * ref["sums"].abs() * (1 - 1e-9)).all()
    # a float32 evaluation of the robust sums (at most `rows` additions per term) lies within the bound
    got = jr.joint_sums(*(x[k] for k in jr.NAMES), idx, index, H, W, W_TRACK, d, dp)
    assert got.dtype == torch.float32
    rows = int((idx >= 0).sum())
    ok, ratio = jr.within(got.double(), ref["sums"], jr.U32 * (ref["row_err"] + rows * ref["row_abs"]))
    assert ok and np.isfinite(ratio), ratio


def _single_row(x, idx, index, photometric, sign):
    """An element with one associated row k: a row with a photometric row when `photometric`, with sign(r_k) (or
    sign(r_p,k)) = sign and, for the geometric residual, |r_k| in float64 above its float32 value, so that a float64
    decision would put the row outside a scale equal to the float32 |r_k|.  -> (idx with only k, k, float32 |r_k|)."""
    r, rp, vj = jr.float32_residuals(*(x[k] for k in jr.NAMES[:5]), idx, index, H, W)
    rows = torch.nonzero(idx >= 0)[:, 0]
    _, b64 = po._rows(x["src"].double(), x["tgt"].double(), x["tgt_n"].double(), idx)
    if photometric:
        res = torch.zeros_like(r)
        res[vj] = rp
        ok = vj & (torch.sign(res) == sign) & (res.abs() > 0.01)
    else:
        res = r
        ok = (torch.sign(r) == sign) & (b64[:, 0].abs() > r.double().abs())
    k = int(torch.nonzero(ok)[0, 0])
    one = torch.full_like(idx, -1)
    one[rows[k]] = idx[rows[k]]
    return one, int(rows[k]), float(res[k].abs())


@pytest.mark.parametrize("sign", [1.0, -1.0])
@pytest.mark.parametrize("photometric", [False, True])
def test_a_residual_on_the_scale_takes_the_inside_branch(photometric, sign):
    """delta = float32 |r_k|: the reference's sums and gradients are the unweighted ones (the inside branch and its
    derivative, decided on the float32 residual even where the float64 one lies above it); delta = nextafter(|r_k|, 0)
    is outside: continuous sums, different gradients."""
    x, idx, index = _case(n=600, seed=7)
    one, k, a = _single_row(x, idx, index, photometric, sign)
    g = torch.randn(28, generator=torch.Generator().manual_seed(3))
    below = float(np.nextafter(np.float32(a), np.float32(0)))
    scale = lambda s: (INF, s) if photometric else (s, INF)
    plain = jr.reference(x, one, index, H, W, W_TRACK, 1, g)
    tie = jr.reference(x, one, index, H, W, W_TRACK, 1, g, *scale(a))
    out = jr.reference(x, one, index, H, W, W_TRACK, 1, g, *scale(below))
    torch.testing.assert_close(tie["sums"], plain["sums"], rtol=1e-14, atol=0)
    torch.testing.assert_close(out["sums"], plain["sums"], rtol=1e-4, atol=1e-12)  # (continuous at the scale)
    name = "src_col" if photometric else "src"
    for n in jr.NAMES:
        torch.testing.assert_close(tie["grad"][n], plain["grad"][n], rtol=1e-12, atol=1e-15)
    d = (out["grad"][name][k] - plain["grad"][name][k]).abs().max()
    assert d > 1e-3 * plain["grad"][name][k].abs().max(), d
    # the outside branch is robust_oracle's at that scale, differentiated in float64
    s = x["src"].double().clone().requires_grad_(True)
    sc = x["src_col"].double().clone().requires_grad_(True)
    if photometric:
        I_m = ph.intensity(x["model_col"].double())
        valid, gu, gv = ph.stencil(I_m.unsqueeze(0), index.unsqueeze(0), H, W)
        Ap, rp = ph.photometric_rows(s, ph.intensity(sc), one, valid[0], gu[0], gv[0], I_m, x["prev"].double(),
                                     x["K"].double())
        rows = ro.row_products(Ap, rp[:, 0], below, w=float(np.float32(W_TRACK)), inside=torch.tensor([False]))
        A, b = po._rows(s, x["tgt"].double(), x["tgt_n"].double(), one)
        rows = rows + ro.row_products(A, b[:, 0], INF)
        want = torch.autograd.grad((rows.sum(0) * g.double()).sum(), sc)[0]
    else:
        A, b = po._rows(s, x["tgt"].double(), x["tgt_n"].double(), one)
        rows = ro.row_products(A, b[:, 0], below, inside=torch.tensor([False]))
        want = torch.autograd.grad((rows.sum(0) * g.double()).sum(), s)[0]
        assert bool(b[0, 0].abs() > a)  # (the float64 residual lies above the scale: a float64 decision is outside)
    torch.testing.assert_close(out["grad"][name][k], want[k], rtol=1e-10, atol=1e-14)
