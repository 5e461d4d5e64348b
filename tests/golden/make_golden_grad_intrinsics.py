"""Freezes the gradient of the UNMODIFIED gradslam reference w.r.t. the camera INTRINSICS (PyTorch autograd through
projutils.inverse_intrinsics and the vertex-map op chain) as fixtures (run in the build container only):

    python tests/golden/make_golden_grad_intrinsics.py     ->  tests/golden/ref_grad_intrinsics.npz

These vectors pin the oracle's autograd d/dK (tests/test_oracle_grad_intrinsics.py), which in turn is what the CUDA
backward kernels are compared with on the GPU (tests/test_gpu_intrinsics_grad.py).  Inputs are NOT stored: the tests
regenerate them from the recorded seeds.  The loss weights are those of make_golden_grad.py's cases of the same name.

Cases (all float32, CPU; K is (B,1,4,4) and only fx, cx, fy, cy get a gradient):
  pf_gt       PointFusion(odom='gt'), B=1, L=2, 24x32: d(sum w.map points/colours/ccounts) / dK
  icpslam     ICPSLAM(odom='gradicp', numiters=3, dsratio=2), B=1, L=2, 32x40: d(sum w.poses) / dK
"""
import os
import sys
import warnings

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, HERE)
sys.path.insert(0, ROOT)
warnings.simplefilter("ignore")

from ref_loader import load_reference  # noqa: E402

load_reference()
from gradslam.slam.icpslam import ICPSLAM  # noqa: E402
from gradslam.slam.pointfusion import PointFusion  # noqa: E402
from gradslam.structures.rgbdimages import RGBDImages  # noqa: E402

from gradslam_b200.synthetic import make_sequence  # noqa: E402

GRAD_CASES = {
    "pf_gt": dict(B=1, L=2, H=24, W=32, seed=41, wseed=5),
    "icpslam": dict(B=1, L=2, H=32, W=40, seed=17, wseed=9, numiters=3, dsratio=2),
}


def main():
    torch.manual_seed(0)
    torch.set_num_threads(1)  # reduction order of the reference's ATen sums must not depend on the pool
    out = {}

    c = GRAD_CASES["pf_gt"]
    rgb, depth, K, poses = make_sequence(c["B"], c["L"], c["H"], c["W"], seed=c["seed"], yaw0=0.6)
    Kg = K.clone().requires_grad_(True)
    pc, _ = PointFusion(odom="gt")(RGBDImages(rgb, depth, Kg, poses))
    n = int(pc.num_points_per_pointcloud[0])
    g = torch.Generator().manual_seed(c["wseed"])
    wp, wc, wf = torch.randn(n, 3, generator=g), torch.randn(n, 3, generator=g), torch.randn(n, 1, generator=g)
    ((pc.points_list[0] * wp).sum() + (pc.colors_list[0] * wc).sum() + (pc.features_list[0] * wf).sum()).backward()
    out["pf_gt/count"] = np.array([n])
    out["pf_gt/d_K"] = Kg.grad.numpy()
    print("pf_gt: n=%d dK\n%s" % (n, Kg.grad[0, 0]))

    c = GRAD_CASES["icpslam"]
    rgb, depth, K, poses = make_sequence(c["B"], c["L"], c["H"], c["W"], seed=c["seed"], yaw0=0.6)
    Kg = K.clone().requires_grad_(True)
    _, rec = ICPSLAM(odom="gradicp", numiters=c["numiters"], dsratio=c["dsratio"])(RGBDImages(rgb, depth, Kg, poses))
    w = torch.randn(rec.shape, generator=torch.Generator().manual_seed(c["wseed"]))
    (rec * w).sum().backward()
    out["icpslam/poses"] = rec.detach().numpy()
    out["icpslam/d_K"] = Kg.grad.numpy()
    print("icpslam: dK\n%s" % Kg.grad[0, 0])

    np.savez_compressed(os.path.join(HERE, "ref_grad_intrinsics.npz"), **out)
    print("wrote ref_grad_intrinsics.npz (%d arrays)" % len(out))


if __name__ == "__main__":
    main()
