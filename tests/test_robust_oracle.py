"""CPU checks of the Huber-weighted tracking oracle (tests/robust_oracle.py): +inf is the unweighted oracles bit for bit,
hand-computed rows on both sides of delta and at it, the written-out backward against float64 autograd, and the gain on
a scene with an object that appears.  No GPU."""
import math

import pytest
import torch

import gsx_oracle as oracle
import photometric_oracle as ph
import projective_oracle as po
import robust_oracle as ro
from gradslam_b200.synthetic import make_dynamic_sequence, make_sequence, make_textured_sequence

INF = math.inf


@pytest.mark.parametrize("odom", ["icp", "gradicp"])
@pytest.mark.parametrize("mode", ["pointfusion", "icpslam"])
def test_infinite_delta_is_the_1nn_oracle_bit_for_bit(odom, mode):
    rgb, depth, K, poses = make_sequence(2, 3, 24, 32, seed=1, yaw0=0.6)
    want = oracle.run_slam(rgb, depth, K, poses, mode="pointfusion" if mode == "pointfusion" else "aggregate",
                           odom=odom, dsratio=2)
    got = ro.run_slam(rgb, depth, K, poses, association="nn", mode=mode, odom=odom, dsratio=2)
    assert torch.equal(got.poses, want.poses)


@pytest.mark.parametrize("odom", ["icp", "gradicp"])
def test_infinite_delta_is_the_projective_oracle_bit_for_bit(odom):
    rgb, depth, K, poses = make_sequence(2, 3, 24, 32, seed=2, yaw0=0.6)
    want = po.run_slam(rgb, depth, K, poses, mode="pointfusion", odom=odom, dsratio=2)
    got = ro.run_slam(rgb, depth, K, poses, association="projective", odom=odom, dsratio=2)
    assert torch.equal(got.poses, want.poses)


@pytest.mark.parametrize("odom", ["icp", "gradicp"])
@pytest.mark.parametrize("M", [0, 3])
def test_infinite_delta_is_the_photometric_oracle_bit_for_bit(odom, M):
    rgb, depth, K, poses = make_textured_sequence(2, 3, 24, 32, seed=1, yaw0=0.6)
    want = ph.run_slam(rgb, depth, K, poses, w=0.1, M=M, odom=odom, dsratio=2)
    got = ro.run_slam(rgb, depth, K, poses, association="projective", w=0.1, M=M, odom=odom, dsratio=2)
    assert torch.equal(got.poses, want.poses)


def _f(x):
    return torch.tensor(x, dtype=torch.float32)


def test_hand_computed_rows_inside_outside_and_at_delta():
    A = torch.tensor([[1.0, 0.0, 0.0, 0.5, -2.0, 0.25]] * 4)
    r = torch.tensor([0.25, -0.5, 2.0, -4.0])  # delta = 0.5: inside, at delta (inside), outside (h = 1/4, 1/8)
    rows = ro.row_products(A, r, 0.5)
    iu = torch.triu_indices(6, 6)
    pq = A[0, iu[0]] * A[0, iu[1]]
    torch.testing.assert_close(rows[0], torch.cat([pq, A[0] * 0.25, _f([0.0625])]), rtol=0, atol=0)
    torch.testing.assert_close(rows[1], torch.cat([pq, A[0] * -0.5, _f([0.25])]), rtol=0, atol=0)
    # outside: h (A_p A_q), h (A_p r) = delta sgn(r) A_p, rho = delta ((a + a) - delta)
    torch.testing.assert_close(rows[2], torch.cat([0.25 * pq, 0.5 * A[0], _f([0.5 * (4.0 - 0.5)])]), rtol=0, atol=0)
    torch.testing.assert_close(rows[3], torch.cat([0.125 * pq, -0.5 * A[0], _f([0.5 * (8.0 - 0.5)])]), rtol=0, atol=0)
    # photometric: inside w (A A), outside (w h) (A A), w rho; +inf weighs every row 1
    w = 0.5
    rows_p = ro.row_products(A, r, 0.5, w=w)
    torch.testing.assert_close(rows_p[2], torch.cat([(w * 0.25) * pq, (w * 0.25) * (A[0] * 2.0), _f([w * 1.75])]))
    torch.testing.assert_close(rows_p[0], w * ro.row_products(A, r, INF)[0], rtol=0, atol=0)
    plain = torch.cat([A[:, iu[0]] * A[:, iu[1]], A * r.unsqueeze(1), (r * r).unsqueeze(1)], 1)
    assert torch.equal(ro.row_products(A, r, INF), plain)
    # the sums of system() are the rows' sums
    AtA, Atb, err = ro.system(A, r.unsqueeze(1), 0.5)
    s = rows.sum(0)
    torch.testing.assert_close(AtA[iu[0], iu[1]], s[:21])
    torch.testing.assert_close(Atb[:, 0], s[21:27])
    torch.testing.assert_close(err, s[27])


def written_out_backward(A, r, delta, G, g_r, g_rr):
    """d(sum_k g_k products_k)/dA and /dr of row_products written out: G (6,6) upper, g_r (6,), g_rr."""
    a = r.abs()
    out = a > delta
    h = torch.where(out, delta / torch.where(out, a, torch.ones_like(a)), torch.ones_like(a))
    Gs = G + G.t()  # d(sum_{p<=q} G_pq A_p A_q)/dA_p = sum_q (G + G^T)_pq A_q
    dA = h.unsqueeze(1) * (A @ Gs.t() + g_r.unsqueeze(0) * r.unsqueeze(1))
    Q = ((A @ G) * A).sum(1)
    dr_in = (A * g_r).sum(1) + 2 * g_rr * r
    dr_out = -(h / r) * Q + 2 * g_rr * h * r  # h r = delta sgn(r) is constant
    return dA, torch.where(out, dr_out, dr_in)


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_float64_autograd_equals_the_written_out_backward(seed):
    g = torch.Generator().manual_seed(seed)
    n, delta = 64, 0.3
    A = torch.randn(n, 6, generator=g, dtype=torch.float64, requires_grad=True)
    r = (torch.randn(n, generator=g, dtype=torch.float64) * 0.6)
    r[:4] = torch.tensor([0.3, -0.3, 0.29, -0.31], dtype=torch.float64)  # at delta (inside) and either side of it
    r.requires_grad_(True)
    coeff = torch.randn(28, generator=g, dtype=torch.float64)
    (ro.row_products(A, r, delta).sum(0) * coeff).sum().backward()
    iu = torch.triu_indices(6, 6)
    G = torch.zeros(6, 6, dtype=torch.float64)
    G[iu[0], iu[1]] = coeff[:21]
    dA, dr = written_out_backward(A.detach(), r.detach(), delta, G, coeff[21:27], coeff[27])
    torch.testing.assert_close(A.grad, dA)
    torch.testing.assert_close(r.grad, dr)
    assert (r.detach().abs() > delta).any() and (r.detach().abs() <= delta).any()


@pytest.mark.parametrize("association", ["projective", "nn"])
def test_huber_keeps_gradicp_on_track_when_a_box_appears(association):
    """make_dynamic_sequence: a box appears in front of the wall at frame 3.  PointFusion with gradICP, dsratio=2, no
    dist_thresh: delta = 0.02 m cuts the worst translation error from frame 3 on at least tenfold (DESIGN.md section 4:
    963 -> 41 mm projective, 909 -> 31 mm 1-NN)."""
    rgb, depth, K, poses = make_dynamic_sequence(1, 8, 48, 64, 3, 8, yaw0=0.6)
    plain = ro.run_slam(rgb, depth, K, poses, association=association, odom="gradicp", dsratio=2)
    robust = ro.run_slam(rgb, depth, K, poses, association=association, odom="gradicp", dsratio=2, delta=0.02)
    e_plain = ro.worst_translation_error(plain.poses, poses, 3)
    e_robust = ro.worst_translation_error(robust.poses, poses, 3)
    assert e_robust * 10 <= e_plain, (e_plain, e_robust)
