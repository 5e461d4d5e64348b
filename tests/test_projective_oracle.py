"""CPU checks of the projective ICP oracle (tests/projective_oracle.py) and of the `association` keyword."""
import numpy as np
import pytest
import torch

import gsx_oracle as oracle
import projective_oracle as po
from gradslam_b200.synthetic import make_sequence

H, W = 6, 8


def _brute_force(src, maps, prev_pose, K, dist_thresh):
    """The definition point by point: every row's pixel and camera z by project_map, the pixel's winner by a scan over
    the rows (smallest z, then lowest n), then each source point's pixel, frustum test, cover test and distance."""
    B, Ns, _ = src.shape
    j_out = np.full((B, Ns), -1, dtype=np.int64)
    for b in range(B):
        pb, Kb = prev_pose[b:b + 1], K[b:b + 1]
        pts = maps[b]
        winner = {}
        if pts.shape[0]:
            u, v, z = (t[0].numpy() for t in oracle.project_map(pts.unsqueeze(0), pb, Kb))
            for n in range(pts.shape[0]):
                if not (u[n] > np.float32(-1e-3) and u[n] < np.float32(W - 0.999) and v[n] > np.float32(-1e-3)
                        and v[n] < np.float32(H - 0.999) and z[n] > 0):
                    continue
                pix = min(max(int(round(float(v[n]))), 0), H - 1) * W + min(max(int(round(float(u[n]))), 0), W - 1)
                if pix not in winner or (z[n], n) < (z[winner[pix]], winner[pix]):
                    winner[pix] = n
        u, v, z = (t[0].numpy() for t in oracle.project_map(src[b:b + 1], pb, Kb))
        for i in range(Ns):
            if not (u[i] > np.float32(-1e-3) and u[i] < np.float32(W - 0.999) and v[i] > np.float32(-1e-3)
                    and v[i] < np.float32(H - 0.999) and z[i] > 0):
                continue
            pix = min(max(int(round(float(v[i]))), 0), H - 1) * W + min(max(int(round(float(u[i]))), 0), W - 1)
            if pix not in winner:
                continue
            s, p = src[b, i].numpy(), pts[winner[pix]].numpy()
            d = s - p
            d2 = np.float32(np.float32(d[0] * d[0]) + np.float32(d[1] * d[1])) + np.float32(d[2] * d[2])
            if dist_thresh is None or d2 < np.float32(dist_thresh):
                j_out[b, i] = pix
    return torch.from_numpy(j_out)


@pytest.mark.parametrize("dist_thresh", [None, 0.0004])
def test_association_equals_brute_force(dist_thresh):
    smap, maps, src, pose, K = po.small_case(H, W)
    idx, tgt_p, tgt_n = po.target_images(smap, pose, K, H, W)
    d2, j = po.associate(src, pose, K, H, W, idx, tgt_p, dist_thresh)
    want = _brute_force(src, maps, pose, K, dist_thresh)
    assert torch.equal(j, want)
    assert (j[2] == -1).all() and torch.isinf(d2[2]).all()  # the empty map
    assert (j[0] >= 0).any() and (j[1] >= 0).any() and (j[0] == -1).any()
    # uncovered pixels hold zeros; covered ones the winning row
    b, p = torch.nonzero(idx >= 0, as_tuple=True)
    assert torch.equal(tgt_p[b, p], torch.stack([maps[bb][n] for bb, n in zip(b.tolist(), idx[b, p].tolist())]))
    assert (tgt_p[idx < 0] == 0).all() and (tgt_n[idx < 0] == 0).all()


def test_association_corner_cases():
    """Half-pixel ties round to even, bounds are strict, z <= 0 never associates."""
    smap, maps, src, pose, K = po.small_case(H, W)
    idx, tgt_p, _ = po.target_images(smap, pose, K, H, W)
    idx_all = torch.arange(H * W).repeat(3, 1)  # every pixel covered
    _, j = po.associate(src[:1], pose[:1], K[:1], H, W, idx_all[:1], tgt_p[:1])
    tail = j[0, H * W:].tolist()
    assert tail[:3] == [2 * W + 2, 2 * W + 4, 0 * W + 2]  # (u, v) = (2.5, 1.5) -> (2, 2); (3.5, 2.5) -> (4, 2); (1.5, 0.5)
    assert tail[3] == -1 and tail[4] == -1 and tail[5] == 2 * W + W - 1 and tail[6] == 1
    assert tail[7] == -1 and tail[8] == -1


def test_taped_loop_with_nn_association_equals_the_oracle_loops():
    """The restated loop, given the 1-NN association, is gsx_oracle's point_to_plane_icp / gradicp bit for bit."""
    _, depth, K, poses = make_sequence(1, 2, 24, 32, seed=4, yaw0=0.6)
    m0 = oracle.frame_maps(depth[:, :1], K, poses[:, :1])
    m1 = oracle.frame_maps(depth[:, 1:], K, poses[:, :1])
    tgt, tgt_n = (m0[k][0, 0][m0["valid"][0, 0]] for k in ("gvertex", "gnormal"))
    src = m1["gvertex"][0, 0][m1["valid"][0, 0]][::3]
    assoc = lambda s: oracle.knn1(s, tgt)[1]
    for odom, fn in (("icp", oracle.point_to_plane_icp), ("gradicp", oracle.point_to_plane_gradicp)):
        T = po.icp(src, tgt, tgt_n, assoc, odom, numiters=5)
        T_ref, _ = fn(src, tgt, tgt_n, torch.eye(4), numiters=5)
        assert torch.equal(T, T_ref)


# max |pose - ground truth| over 5 frames of the oracle's projective PointFusion on make_sequence(1, 5, 48, 64, seed=7,
# yaw0=0.6), numiters=10, dsratio=2, measured on the CPU: icp 1.43e-2, gradicp 1.24e-2 (the 1-NN oracle: 1.21e-2 for
# both).  Holding the first pose would be 4 cm off by frame 4.
TRACKING_BOUND = 2e-2


@pytest.mark.parametrize("odom", ["icp", "gradicp"])
def test_oracle_tracks_ground_truth(odom):
    rgb, depth, K, poses = make_sequence(1, 5, 48, 64, seed=7, yaw0=0.6)
    res = po.run_slam(rgb, depth, K, poses, odom=odom, numiters=10, dsratio=2)
    err = (res.poses - poses).abs().max().item()
    assert err < TRACKING_BOUND, err


@pytest.mark.parametrize("cls", ["ICPSLAM", "PointFusion"])
def test_association_argument_errors(cls):
    import gradslam_b200 as gs

    with pytest.raises(TypeError):
        getattr(gs, cls)(odom="icp", association=1)
    with pytest.raises(TypeError):
        getattr(gs, cls)(odom="icp", association=None)
    with pytest.raises(ValueError):
        getattr(gs, cls)(odom="icp", association="knn")
    with pytest.raises(TypeError):
        getattr(gs, cls)("icp")  # keyword-only
    for a in ("nn", "projective"):
        assert getattr(gs, cls)(odom="gt", association=a).association == a
