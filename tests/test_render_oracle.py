"""CPU checks of the map renderer's definition (tests/render_oracle.py) and of the argument checks of its C entry points
(gsx_render_views*, no GPU needed: they reject bad arguments before any CUDA call)."""
import ctypes
import math

import numpy as np
import torch

import gsx_oracle as oracle
import render_oracle

F32 = torch.float32


def _pose(yaw, t):
    c, s = math.cos(yaw), math.sin(yaw)
    T = torch.eye(4, dtype=torch.float64)
    T[:3, :3] = torch.tensor([[c, 0.0, s], [0.0, 1.0, 0.0], [-s, 0.0, c]], dtype=torch.float64)
    T[:3, 3] = torch.tensor(t, dtype=torch.float64)
    return T.float()


def _next(x, toward):
    return float(np.nextafter(np.float32(x), np.float32(toward)))


def _edge_map_and_cameras(H=4, W=5):
    """Element 0: rows placed against the identity camera with K = I (u = x / z exactly); element 1: empty;
    element 2: a random cloud in front of the camera."""
    lo, hi = np.float32(-1e-3), np.float32(W - 0.999)
    rows0 = [
        (1.0, 1.0, 2.0),              # 0: pixel (1,1), z = 2
        (1.0, 1.0, 1.0),              # 1: same pixel, nearer: wins
        (3.0, 2.0, 1.0),              # 2: tie with row 5 (identical): the lower index wins
        (2.0, 1.0, -1.0),             # 3: behind the camera
        (0.0, 0.0, 0.0),              # 4: z == 0
        (3.0, 2.0, 1.0),              # 5: duplicate of row 2
        (float(hi), 0.0, 1.0),        # 6: u exactly on the right bound: out
        (_next(hi, 0), 0.0, 1.0),     # 7: just inside: pixel w = 4
        (float(lo), 3.0, 1.0),        # 8: u exactly on the left bound: out
        (_next(lo, 1), 3.0, 1.0),     # 9: just inside: pixel w = 0
        (2.0, _next(H - 0.999, 0), 1.0),  # 10: v just inside the lower bound: pixel h = 3
        (2.5, 0.5, 1.0),              # 11: round half to even: pixel (0, 2)
    ]
    p0 = torch.tensor(rows0, dtype=F32)
    g = torch.Generator().manual_seed(3)
    p2 = torch.randn(40, 3, generator=g) * 0.5 + torch.tensor([0.0, 0.0, 3.0])
    pts = [p0, torch.zeros(0, 3), p2]
    unit = lambda p: torch.nn.functional.normalize(torch.randn(p.shape[0], 3, generator=g), dim=1)
    smap = oracle.SurfelMap(pts, [unit(p) for p in pts], [torch.rand(p.shape[0], 3, generator=g) for p in pts],
                            [torch.randint(1, 9, (p.shape[0], 1), generator=g).float() for p in pts])
    K = torch.eye(4).repeat(3, 1, 1)
    K[2, 0, 0], K[2, 1, 1], K[2, 0, 2], K[2, 1, 2] = 4.0, 4.0, 2.0, 1.5
    poses = torch.stack([torch.stack([torch.eye(4), _pose(0.1, (0.05, -0.02, 0.1))]) for _ in range(3)])
    return smap, poses, K, H, W


def _brute_force(smap, poses, K, H, W):
    """Per pixel, the minimum (z, n) over the map rows whose projection lands on it, row by row in Python."""
    B, L = poses.shape[:2]
    index = torch.full((B, L, H, W), -1, dtype=torch.int64)
    for b in range(B):
        pts = smap.points[b]
        for l in range(L):
            best = {}
            for n in range(pts.shape[0]):
                u, v, z = oracle.project_map(pts[n].view(1, 1, 3), poses[b, l].view(1, 4, 4), K[b].view(1, 4, 4))
                u, v, z = u.item(), v.item(), z.item()
                if not (u > np.float32(-1e-3) and u < np.float32(W - 0.999) and v > np.float32(-1e-3)
                        and v < np.float32(H - 0.999) and z > 0):
                    continue
                h, w = min(max(int(np.rint(v)), 0), H - 1), min(max(int(np.rint(u)), 0), W - 1)
                if (h, w) not in best or (z, n) < best[(h, w)]:
                    best[(h, w)] = (z, n)
            for (h, w), (z, n) in best.items():
                index[b, l, h, w] = n
    return index


def test_oracle_index_equals_brute_force_with_ties_bounds_and_an_empty_element():
    smap, poses, K, H, W = _edge_map_and_cameras()
    out = render_oracle.render_views(smap, poses, K, H, W)
    assert torch.equal(out.index, _brute_force(smap, poses, K, H, W))
    idx = out.index[0, 0]
    assert idx[1, 1] == 1 and idx[2, 3] == 2 and idx[0, 4] == 7 and idx[3, 0] == 9 and idx[3, 2] == 10
    assert idx[0, 2] == 11
    assert not {3, 4, 5, 6, 8} & set(out.index[0].flatten().tolist())
    assert (out.index[1] == -1).all() and (out.depth[1] == 0).all() and (out.rgb[1] == 0).all()
    assert (out.index[2] >= 0).sum() > 10


def test_oracle_values_are_the_winning_rows():
    smap, poses, K, H, W = _edge_map_and_cameras()
    out = render_oracle.render_views(smap, poses, K, H, W)
    for b, l, h, w in (out.index >= 0).nonzero().tolist():
        n = int(out.index[b, l, h, w])
        _, _, z = oracle.project_map(smap.points[b][n].view(1, 1, 3), poses[b, l].view(1, 4, 4), K[b].view(1, 4, 4))
        assert out.depth[b, l, h, w, 0] == z.item()
        assert torch.equal(out.rgb[b, l, h, w], smap.colors[b][n])
        assert torch.equal(out.confidence[b, l, h, w], smap.ccounts[b][n])
        R = poses[b, l, :3, :3].double()
        torch.testing.assert_close(out.normals[b, l, h, w].double(), R.t() @ smap.normals[b][n].double(),
                                   rtol=0, atol=1e-6)
    unc = out.index < 0
    assert (out.depth[unc] == 0).all() and (out.normals[unc] == 0).all() and (out.confidence[unc] == 0).all()


def _closed_form_grads(pts, nrm, poses, index, g_depth, g_nrm, g_rgb, g_conf):
    """The backward the kernels implement, written out in float64: per row, a sum over the pixels it won; per pose,
    dL/dR = (p - t) g_q^T + n g_n^T and dL/dt = -R g_q with g_q = (0, 0, g_depth)."""
    B, N = pts.shape[:2]
    L = poses.shape[1]
    d_geo = torch.zeros(B, N, 7, dtype=torch.float64)
    d_col = torch.zeros(B, N, 3, dtype=torch.float64)
    d_pose = torch.zeros(B, L, 4, 4, dtype=torch.float64)
    for b, l, h, w in (index >= 0).nonzero().tolist():
        n = int(index[b, l, h, w])
        R, t = poses[b, l, :3, :3], poses[b, l, :3, 3]
        gq = torch.tensor([0.0, 0.0, float(g_depth[b, l, h, w, 0])], dtype=torch.float64)
        gn = g_nrm[b, l, h, w]
        d_geo[b, n, 0:3] += R @ gq
        d_geo[b, n, 3:6] += R @ gn
        d_geo[b, n, 6] += g_conf[b, l, h, w, 0]
        d_col[b, n] += g_rgb[b, l, h, w]
        d_pose[b, l, :3, :3] += torch.outer(pts[b, n] - t, gq) + torch.outer(nrm[b, n], gn)
        d_pose[b, l, :3, 3] -= R @ gq
    return d_geo, d_col, d_pose


def test_oracle_backward_equals_float64_autograd_and_the_closed_form():
    smap, poses, K, H, W = _edge_map_and_cameras()
    index = render_oracle.render_index(smap, poses, K, H, W)
    pts, nrm, col, cc = (t.double() for t in smap.padded())
    g = torch.Generator().manual_seed(11)
    B, L = poses.shape[:2]
    ups = [torch.randn(B, L, H, W, c, generator=g, dtype=torch.float64) for c in (1, 3, 3, 1)]

    def grads(dtype):
        leaves = [t.to(dtype).clone().requires_grad_(True) for t in (pts, nrm, col, cc, poses.double())]
        out = render_oracle.render_values(*leaves, index)
        loss = sum((o * u.to(dtype)).sum() for o, u in zip((out.depth, out.normals, out.rgb, out.confidence), ups))
        loss.backward()
        return [x.grad.double() for x in leaves]

    g64, g32 = grads(torch.float64), grads(torch.float32)
    for a, b in zip(g32, g64):
        torch.testing.assert_close(a, b, rtol=1e-5, atol=1e-5)
    d_geo, d_col, d_pose = _closed_form_grads(pts, nrm, poses.double(), index, ups[0], ups[1], ups[2], ups[3])
    torch.testing.assert_close(g64[0], d_geo[..., 0:3])
    torch.testing.assert_close(g64[1], d_geo[..., 3:6])
    torch.testing.assert_close(g64[2], d_col)
    torch.testing.assert_close(g64[3], d_geo[..., 6:7])
    torch.testing.assert_close(g64[4], d_pose)
    # rows that win no pixel get exactly zero
    won = torch.zeros(pts.shape[:2], dtype=torch.bool)
    for b, l, h, w in (index >= 0).nonzero().tolist():
        won[b, int(index[b, l, h, w])] = True
    assert (g64[0][~won] == 0).all() and (g64[2][~won] == 0).all()


def test_oracle_formula_gradcheck():
    smap, poses, K, H, W = _edge_map_and_cameras()
    index = render_oracle.render_index(smap, poses, K, H, W)
    pts, nrm, col, cc = (t.double().requires_grad_(True) for t in smap.padded())
    P = poses.double().requires_grad_(True)

    def f(p, n, c, k, T):
        o = render_oracle.render_values(p, n, c, k, T, index)
        return o.depth, o.normals, o.rgb, o.confidence

    assert torch.autograd.gradcheck(f, (pts, nrm, col, cc, P), eps=1e-6, atol=1e-6)


# ---- C entry points: argument checks before any CUDA call --------------------------------------------------------
def _lib():
    from gradslam_b200 import _C

    return _C.lib()


def _err(lib):
    return lib.gsx_last_error()


def test_render_entry_points_reject_bad_arguments_without_a_gpu():
    lib = _lib()
    p = ctypes.c_void_p(256)  # never dereferenced: every call below fails its argument checks first
    fwd = lambda *a: lib.gsx_render_views(*a)
    # args: geo, col, counts, cap, max_count, K, K_bstride, poses, pose_bstride, B, L, H, W, index, depth, rgb, n, conf, s
    base = [p, p, p, 10, 10, p, 16, p, 16, 2, 3, 4, 5, p, p, p, p, p, None]
    cases = {
        "null index": {13: None},
        "null poses": {7: None},
        "null intrinsics": {5: None},
        "null map": {0: None},
        "null counts": {2: None},
        "rgb without colours": {1: None},
        "H = 0": {11: 0},
        "W < 0": {12: -3},
        "L = 0": {10: 0},
        "B = 0": {9: 0},
        "L*H*W overflow": {10: 2, 11: 40000, 12: 40000},
        "too many views": {9: 300, 10: 300},
        "max_count > capacity": {4: 11},
        "negative max_count": {4: -1},
        "misaligned rows": {0: ctypes.c_void_p(260)},
    }
    for what, change in cases.items():
        args = list(base)
        for i, v in change.items():
            args[i] = v
        rc = fwd(*args)
        assert rc != 0, what
        assert b"gsx_render_views" in _err(lib), what

    assert lib.gsx_render_views_bwd_scratch_bytes(8, 32, 480, 640) >= 8 * 32 * 1200 * 12 * 4
    assert lib.gsx_render_views_bwd_scratch_bytes(0, 1, 1, 1) < 0
    # args: geo, counts, cap, K, K_bstride, poses, pose_bstride, index, B, L, H, W, g x4, d_geo, d_col, d_poses,
    #       scratch, scratch_bytes, stream
    bbase = [p, p, 10, p, 16, p, 16, p, 2, 3, 4, 5, p, p, p, p, p, p, p, p, 1 << 20, None]
    bcases = {
        "null index": {7: None},
        "null poses": {5: None},
        "null map": {0: None},
        "null counts": {1: None},
        "scratch too small": {20: 16},
        "null scratch": {19: None},
        "H = 0": {10: 0},
        "L*H*W overflow": {9: 2, 10: 40000, 11: 40000},
        "negative capacity": {2: -1},
    }
    for what, change in bcases.items():
        args = list(bbase)
        for i, v in change.items():
            args[i] = v
        rc = lib.gsx_render_views_bwd(*args)
        assert rc != 0, what
        assert b"gsx_render_views_bwd" in _err(lib), what


def test_render_pointclouds_rejects_bad_arguments_without_a_gpu():
    import pytest

    import gradslam_b200 as gs

    pc = gs.Pointclouds(points=[torch.zeros(4, 3), torch.zeros(2, 3)])
    K, poses = torch.eye(4).repeat(2, 1, 1, 1), torch.eye(4).repeat(2, 3, 1, 1)
    with pytest.raises(TypeError):
        gs.render_pointclouds(poses, K, poses, 4, 5)
    with pytest.raises(ValueError):
        gs.render_pointclouds(pc, K, poses, 0, 5)
    with pytest.raises(ValueError):
        gs.render_pointclouds(pc, K, poses, 4, -1)
    with pytest.raises(ValueError):  # not 4x4
        gs.render_pointclouds(pc, K, poses[..., :3, :], 4, 5)
    with pytest.raises(ValueError):
        gs.render_pointclouds(pc, K[..., :3, :3], poses, 4, 5)
    with pytest.raises(ValueError):  # batch sizes
        gs.render_pointclouds(pc, K[:1], poses, 4, 5)
    with pytest.raises(ValueError):
        gs.render_pointclouds(pc, K.repeat(2, 1, 1, 1), poses.repeat(2, 1, 1, 1), 4, 5)
    with pytest.raises(RuntimeError, match="CUDA"):  # the engine has no CPU path
        gs.render_pointclouds(pc, K, poses, 4, 5)
    assert gs.structures.render_pointclouds is gs.render_pointclouds


def test_render_pointclouds_rejects_row_stores_of_different_capacities():
    import pytest

    import gradslam_b200 as gs

    pc = gs.Pointclouds(points=[torch.zeros(4, 3)], colors=[torch.zeros(4, 3)])
    pc._col = pc._col[:, :2]
    with pytest.raises(ValueError, match="colour rows"):
        gs.render_pointclouds(pc, torch.eye(4).view(1, 1, 4, 4), torch.eye(4).view(1, 1, 4, 4), 4, 5)
