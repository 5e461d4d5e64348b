"""CPU checks of the float64 reference of the joint normal-equation op (tests/joint_normal_eq_reference.py): in float32
it is photometric_oracle's statement, w = 0 is the geometric one, its pair arithmetic restates the same expressions,
and its bounds and per-row terms are consistent.  No GPU."""
import numpy as np
import pytest
import torch

import gsx_oracle as oracle
import joint_normal_eq_reference as jr
import photometric_oracle as ph
import projective_oracle as po
from cameras import camera_intrinsics

W_TRACK = 0.1


def _case(H=12, W=16, n=300, seed=0, skew=0.75):
    K = torch.from_numpy(camera_intrinsics(2, H, W, skew=skew)[1])
    prev = oracle.se3_exp(torch.tensor([0.1, -0.05, 0.2, 0.15, -0.2, 0.1])).double()
    return jr.synthetic_element(H, W, n, K, prev, seed)


def _upper(AtA, Atb, bb):
    iu = torch.triu_indices(6, 6)
    return torch.cat([AtA[iu[0], iu[1]], Atb[:, 0], bb.view(1)])


@pytest.mark.parametrize("seed", [0, 1])
def test_float32_reference_is_the_photometric_oracle(seed):
    """The model colour image gathered from map rows at the index image (uncovered pixels 0): the sums equal
    photometric_oracle's system at that association (model_intensity, stencil, photometric_rows) bit for bit."""
    x, idx, index = _case(seed=seed)
    H, W = 12, 16
    g = torch.Generator().manual_seed(seed)
    rows = torch.rand(H * W, 3, generator=g)
    x["model_col"] = torch.where((index >= 0).unsqueeze(1), rows[index.clamp(min=0)], torch.zeros(()))
    got = jr.joint_sums(*(x[k] for k in jr.NAMES), idx, index, H, W, W_TRACK)
    assert got.dtype == torch.float32
    I_m = ph.model_intensity(rows.unsqueeze(0), index.unsqueeze(0))
    valid, gu, gv = ph.stencil(I_m, index.unsqueeze(0), H, W)
    A, b = po._rows(x["src"], x["tgt"], x["tgt_n"], idx)
    Ap, rp = ph.photometric_rows(x["src"], ph.intensity(x["src_col"]), idx, valid[0], gu[0], gv[0], I_m[0], x["prev"],
                                 x["K"])
    assert Ap.shape[0] > 20 and Ap.shape[0] < A.shape[0]  # (some rows have a photometric row, not all)
    assert torch.equal(got, _upper(*ph._normal_equations(A, b, Ap, rp, W_TRACK)))


def test_zero_weight_is_the_geometric_system():
    x, idx, index = _case(seed=3)
    got = jr.joint_sums(*(x[k] for k in jr.NAMES), idx, index, 12, 16, 0.0)
    A, b = po._rows(x["src"], x["tgt"], x["tgt_n"], idx)
    assert torch.equal(got, _upper(A.t() @ A, A.t() @ b, torch.dot(b[:, 0], b[:, 0])))


@pytest.mark.parametrize("H,W", [(2, 9), (7, 2)])
def test_no_interior_pixel_gives_the_geometric_sums(H, W):
    x, idx, index = _case(H, W, n=40, seed=4)
    geo = jr.joint_sums(*(x[k] for k in jr.NAMES), idx, index, H, W, 0.0)
    assert torch.equal(jr.joint_sums(*(x[k] for k in jr.NAMES), idx, index, H, W, 0.5), geo)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_pair_arithmetic_restates_the_rows_bit_for_bit(dtype):
    """The values of the bound's pair evaluation are po._rows' and ph.photometric_rows' in the same dtype."""
    H, W = 12, 16
    x, idx, index = _case(seed=5)
    x = {k: v.to(dtype) for k, v in x.items()}
    mx = {k: v.abs() for k, v in x.items()}
    vals, mags, errs, (A, r), (Ap, rp), vj = jr._pair_rows(x, mx, idx, index, H, W, W_TRACK)
    A_ref, b_ref = po._rows(x["src"], x["tgt"], x["tgt_n"], idx)
    assert torch.equal(torch.stack([a.v for a in A], 1), A_ref) and torch.equal(r.v, b_ref[:, 0])
    I_m = ph.intensity(x["model_col"])
    valid, gu, gv = ph.stencil(I_m.unsqueeze(0), index.unsqueeze(0), H, W)
    Ap_ref, rp_ref = ph.photometric_rows(x["src"], ph.intensity(x["src_col"]), idx, valid[0], gu[0], gv[0], I_m,
                                         x["prev"], x["K"])
    assert torch.equal(torch.stack([a.v for a in Ap], 1), Ap_ref) and torch.equal(rp.v, rp_ref[:, 0])
    assert int(vj.sum()) == Ap_ref.shape[0] > 0
    assert (mags >= vals.abs()).all() and (errs >= vals.abs()).all()


def test_per_row_terms_sum_to_the_gradient_and_bounds_cover_the_values():
    H, W = 12, 16
    x, idx, index = _case(seed=6)
    g = torch.randn(28, generator=torch.Generator().manual_seed(1))
    ref = jr.reference(x, idx, index, H, W, W_TRACK, jr.blocks_of(idx.numel()), g)
    for name in ("prev", "K"):
        terms = ref["row_terms"][name].sum(0).view(3, 4)
        torch.testing.assert_close(terms, ref["grad"][name][:3], rtol=1e-12, atol=1e-12 * terms.abs().max().item())
        assert (ref["grad"][name][3] == 0).all() and (ref["grad_bound"][name][3] == 0).all()
    # skew and the 4th column of K get a gradient; every gradient has a positive bound where it is not 0
    assert ref["grad"]["K"][0, 1] != 0 and (ref["grad"]["K"][:3, 3] != 0).all()
    for name in jr.NAMES:
        grad, bound = ref["grad"][name], ref["grad_bound"][name]
        assert ((grad == 0) | (bound > 0)).all(), name
        # a bound is a small multiple of u times a magnitude that is at least |value|
        assert (bound >= jr.R_B * jr.U32 * grad.abs() * (1 - 1e-9)).all(), name
    assert (ref["sum_bound"] >= 14 * jr.U32 * ref["sums"].abs() * (1 - 1e-9)).all()
    # a float32 evaluation of the same sums (matmul order: at most `rows` additions per term) lies within the bound
    got = jr.joint_sums(*(x[k] for k in jr.NAMES), idx, index, H, W, W_TRACK).double()
    rows = int((idx >= 0).sum())
    bound = jr.U32 * (ref["row_err"] + rows * ref["row_abs"])
    ok, ratio = jr.within(got, ref["sums"], bound)
    assert ok, ratio
    assert np.isfinite(ratio)
