"""Freezes outputs of the UNMODIFIED gradslam reference on inputs where every batch element has its own camera
(tests/golden/cameras.py; run in the build container only):

    python tests/golden/make_golden_cameras.py     ->  tests/golden/ref_cameras.npz

Same mechanism as make_golden.py (reference imported from /root/reference through ref_loader.py).  Cases: PointFusion
with ground-truth odometry with and without skew / 4th intrinsics column, PointFusion with ICP and gradICP odometry,
ICPSLAM with gradICP, and the three correspondence tables of one fusion step.  Inputs are NOT stored: the tests
regenerate them from the recorded seeds.  Maps are stored as their sizes, float64 sums and absolute sums of every
attribute per element, and every SAMPLE_STRIDE-th row (cameras.py), which keeps the file small; poses in full; the
active and unique tables in full (column-major int32, which compresses ~3x better), the similar table as its mask over
the active rows (cameras.frozen_table reads them back); about 100 KiB in all.  The archive is written with fixed member
timestamps, so a rerun reproduces it byte for byte.
"""
import io
import os
import sys
import warnings
import zipfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, HERE)
sys.path.insert(0, ROOT)
warnings.simplefilter("ignore")

from ref_loader import load_reference  # noqa: E402

load_reference()
from gradslam.slam import fusionutils as ref_fu  # noqa: E402
from gradslam.slam.icpslam import ICPSLAM  # noqa: E402
from gradslam.slam.pointfusion import PointFusion  # noqa: E402
from gradslam.structures.pointclouds import Pointclouds  # noqa: E402
from gradslam.structures.rgbdimages import RGBDImages  # noqa: E402

from cameras import CAMERA_CASES, SAMPLE_STRIDE, TABLES_CASE, camera_inputs  # noqa: E402


def save_npz(path, arrays):
    """np.savez_compressed without the wall-clock timestamps it gives the archive members."""
    with zipfile.ZipFile(path, "w", zipfile.ZIP_DEFLATED) as zf:
        for key, value in arrays.items():
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.ascontiguousarray(value), allow_pickle=False)
            info = zipfile.ZipInfo(key + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
            info.compress_type = zipfile.ZIP_DEFLATED
            zf.writestr(info, buf.getvalue())


def pack_map_summary(prefix, pc, out):
    """Sizes, then per attribute: float64 column sums and absolute sums (B, C) over each element's rows, and rows 0, S,
    2S, ... of every element, concatenated in element order."""
    out[prefix + "/counts"] = np.array([int(c) for c in pc.num_points_per_pointcloud], dtype=np.int64)
    attrs = [("points", pc.points_list), ("normals", pc.normals_list), ("colors", pc.colors_list)]
    if pc.has_features:
        attrs.append(("ccounts", pc.features_list))
    for name, lst in attrs:
        arrays = [t.numpy() for t in lst]
        out["%s/%s/sum" % (prefix, name)] = np.stack([a.astype(np.float64).sum(0) for a in arrays])
        out["%s/%s/abs_sum" % (prefix, name)] = np.stack([np.abs(a.astype(np.float64)).sum(0) for a in arrays])
        out["%s/%s/sample" % (prefix, name)] = np.concatenate([a[::SAMPLE_STRIDE] for a in arrays])


def main():
    out = {}
    for name, cls, B, L, H, W, seed, cam_kw, kw in CAMERA_CASES:
        rgb, depth, K, poses = camera_inputs(B, L, H, W, seed, **cam_kw)
        slam = (PointFusion if cls == "PointFusion" else ICPSLAM)(**kw)
        pc, rec = slam(RGBDImages(rgb, depth, K, poses))
        pack_map_summary(name, pc, out)
        out[name + "/poses"] = rec.numpy()
        print(name, out[name + "/counts"], "max |pose - gt| %.2e" % (rec - poses).abs().max().item())

    c = TABLES_CASE
    rgb, depth, K, poses = camera_inputs(c["B"], c["L"], c["H"], c["W"], c["seed"], skew=c["skew"])
    frames = RGBDImages(rgb, depth, K, poses)
    slam = PointFusion(odom="gt")
    pc = Pointclouds()
    for s in range(2):
        pc, _ = slam.step(pc, frames[:, s], None, inplace=True)
    live = frames[:, 2]
    t_active = ref_fu.find_active_map_points(pc, live)
    t_similar, mask = ref_fu.find_similar_map_points(pc, live, t_active, slam.dist_th, slam.dot_th)
    t_unique = ref_fu.find_best_unique_correspondences(pc, live, t_similar)
    out["tables/active"] = np.ascontiguousarray(t_active.numpy().T.astype(np.int32))
    assert torch.equal(t_similar, t_active[mask])  # (the similar table is the active table's masked rows)
    out["tables/similar_mask"] = mask.numpy()
    out["tables/unique"] = np.ascontiguousarray(t_unique.numpy().T.astype(np.int32))
    pack_map_summary("tables/map_before", pc, out)
    print("tables", t_active.shape, t_similar.shape, t_unique.shape)

    path = os.path.join(HERE, "ref_cameras.npz")
    save_npz(path, out)
    print("ref_cameras.npz", os.path.getsize(path) // 1024, "KiB")


if __name__ == "__main__":
    main()
