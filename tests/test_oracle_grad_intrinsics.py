"""Pins the CPU oracle's autograd d/dK (oracle/gsx_oracle.py, torch ops on the intrinsics) against the gradient of the
unmodified reference w.r.t. its camera intrinsics, frozen by tests/golden/make_golden_grad_intrinsics.py.  The CUDA
backward kernels are compared with the oracle's autograd on the GPU (tests/test_gpu_intrinsics_grad.py), so this closes
the chain reference -> oracle -> kernels for d/dK.  CPU only."""
import os

import numpy as np
import pytest
import torch

import gsx_oracle as oracle
from gradslam_b200.synthetic import make_sequence

GOLD = os.path.join(os.path.dirname(__file__), "golden")
# the entries of the 4x4 K the reference's inverse_intrinsics reads: fx, cx, fy, cy
READ = [(0, 0), (0, 2), (1, 1), (1, 2)]


@pytest.fixture(scope="module")
def ref():
    return np.load(os.path.join(GOLD, "ref_grad_intrinsics.npz"))


def _check(got, want, rtol):
    want = torch.from_numpy(np.asarray(want))
    assert got.shape == want.shape
    assert torch.isfinite(got).all()
    mask = torch.zeros(4, 4, dtype=torch.bool)
    for i, j in READ:
        mask[i, j] = True
    assert (got[..., ~mask] == 0).all() and (want[..., ~mask] == 0).all()
    torch.testing.assert_close(got[..., mask], want[..., mask], rtol=rtol, atol=rtol * want.abs().max().item())


def test_oracle_pointfusion_intrinsics_gradient_matches_reference(ref):
    torch.set_num_threads(1)
    rgb, depth, K, poses = make_sequence(1, 2, 24, 32, seed=41, yaw0=0.6)
    Kg = K.clone().requires_grad_(True)
    res = oracle.run_slam(rgb, depth, Kg, poses, odom="gt")
    n = res.map.counts()[0]
    assert n == int(ref["pf_gt/count"][0])
    g = torch.Generator().manual_seed(5)
    wp, wc, wf = torch.randn(n, 3, generator=g), torch.randn(n, 3, generator=g), torch.randn(n, 1, generator=g)
    ((res.map.points[0] * wp).sum() + (res.map.colors[0] * wc).sum() + (res.map.ccounts[0] * wf).sum()).backward()
    _check(Kg.grad, ref["pf_gt/d_K"], 1e-3)


def test_oracle_icpslam_intrinsics_gradient_matches_reference(ref):
    torch.set_num_threads(1)
    rgb, depth, K, poses = make_sequence(1, 2, 32, 40, seed=17, yaw0=0.6)
    Kg = K.clone().requires_grad_(True)
    res = oracle.run_slam(rgb, depth, Kg, poses, mode="aggregate", odom="gradicp", numiters=3, dsratio=2)
    torch.testing.assert_close(res.poses.detach(), torch.from_numpy(ref["icpslam/poses"]), rtol=0, atol=1e-5)
    w = torch.randn(res.poses.shape, generator=torch.Generator().manual_seed(9))
    (res.poses * w).sum().backward()
    _check(Kg.grad, ref["icpslam/d_K"], 5e-3)
