"""Oracle parity for kernel branches the shape-by-shape parity tests do not reach: K2's grid-stride loop over several
passes, the plain K1r kernel next to the TMA one (with partial tiles), K4's colour staging from a misaligned base, the
batch groups of the sequence driver, host-fed frames, K4's capacity guard, the grid 1-NN on batched, ragged and
degenerate clouds, and long ICPSLAM runs whose ICP target outgrows any per-pixel bound."""
import pytest
import torch

import gsx_oracle as oracle
from cameras import CameraShape, camera_inputs
from gradslam_b200.synthetic import make_sequence

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
K2_BLOCK = 256  # threads per K2 CTA (kBlock in gsx_common.cuh)
SENTINEL = 0x7FC0DEAD  # a NaN bit pattern no kernel writes

_ref_cache = {}


def _inputs_and_ref(B, L, H, W, seed=0, cameras=False):
    """Seeded inputs and the oracle's PointFusion(odom='gt') run on them (cached: several tests share a shape).
    cameras=True: a camera per element (tests/golden/cameras.py), skew and 4th intrinsics column set."""
    key = (B, L, H, W, seed, cameras)
    if key not in _ref_cache:
        if cameras:
            rgb, depth, K, poses = camera_inputs(B, L, H, W, seed, skew=0.75)
        else:
            rgb, depth, K, poses = make_sequence(B, L, H, W, seed=seed)
        _ref_cache[key] = (rgb, depth, K, poses, oracle.run_slam(rgb, depth, K, poses, odom="gt").map)
    return _ref_cache[key]


def _frames(gs, rgb, depth, K, poses):
    return gs.RGBDImages(rgb.to(DEV), depth.to(DEV), K.to(DEV), poses.to(DEV))


def _assert_matches_oracle(pc, ref_map):
    assert [int(c) for c in pc.num_points_per_pointcloud.tolist()] == ref_map.counts()
    for b in range(len(ref_map.counts())):
        assert torch.equal(pc.points_list[b].cpu(), ref_map.points[b]), b
        assert torch.equal(pc.normals_list[b].cpu(), ref_map.normals[b]), b
        assert torch.equal(pc.colors_list[b].cpu(), ref_map.colors[b]), b
        assert torch.equal(pc.features_list[b].cpu(), ref_map.ccounts[b]), b


def _assert_same_rows(a, b):
    """Two device maps hold the same sizes and the same packed rows, bit for bit."""
    counts = [int(c) for c in a.num_points_per_pointcloud.tolist()]
    assert counts == [int(c) for c in b.num_points_per_pointcloud.tolist()]
    for i, n in enumerate(counts):
        assert torch.equal(a._geo[i, :n], b._geo[i, :n]), i
        assert torch.equal(a._col[i, :n], b._col[i, :n]), i


# ---------------------------------------------------------------------------------------------- K2 grid-stride passes
@pytest.fixture
def k2_grid_cap():
    from gradslam_b200 import _C

    yield _C.lib().gsx_debug_set_k2_grid_cap
    _C.lib().gsx_debug_set_k2_grid_cap(0)


@pytest.mark.parametrize("shape", [(2, 4, 48, 64), (3, 3, 64, 64), (1, 5, 120, 160),
                                   pytest.param(CameraShape((3, 4, 48, 64)), id="cameras")])
def test_k2_multi_pass_grid_stride_matches_oracle(shape, k2_grid_cap):
    """K2 capped to 1, 3 or 7 CTAs in all (3 and 7 do not divide B): every thread walks several map rows, prefetching
    the next row and settling each 128-bit CAS one iteration late across passes.  Whole-sequence call and step loop."""
    import gradslam_b200 as gs

    B, L, H, W = shape
    rgb, depth, K, poses, ref = _inputs_and_ref(B, L, H, W, cameras=isinstance(shape, CameraShape))
    frames = _frames(gs, rgb, depth, K, poses)
    # every frame after the first projects at least the first frame's valid pixels
    min_rows = int((depth[:, 0, ..., 0] > 0).flatten(1).sum(1).min())
    for cap in (1, 3, 7):
        k2_grid_cap(cap)
        ctas = max(1, -(-cap // B))  # CTAs per element (launch_project_select)
        assert min_rows > 2 * ctas * K2_BLOCK, "K2 would not take three passes"
        slam = gs.PointFusion(odom="gt", device=DEV)
        pc, _ = slam(frames)
        _assert_matches_oracle(pc, ref)
        pc = gs.Pointclouds(device=DEV)
        for s in range(L):
            pc, _ = slam.step(pc, frames[:, s], None, inplace=True)
        _assert_matches_oracle(pc, ref)


# ---------------------------------------------------------------------------------------------- K1r and K4 layouts
def _k1r_uses_tma(H, W):
    """depth_tensor_map() in gsx_fusion.cu for a dense (B, L, H, W) depth tensor: every frame base is 16-byte aligned
    iff W % 4 == 0; a last column / row that starts a tile of its own rules TMA out."""
    return W % 4 == 0 and (W - 1) % 32 != 0 and (H - 1) % 8 != 0


@pytest.mark.parametrize("shape,branch", [((2, 3, 41, 64), "plain: (H-1) % 8 == 0"),
                                          ((2, 3, 33, 47), "plain: W % 4 != 0, misaligned K4 colours"),
                                          ((2, 3, 42, 100), "tma: partial tiles in both dimensions"),
                                          ((3, 3, 42, 100), "tma: partial tiles, a camera per element")])
def test_frame_record_layouts_match_oracle(shape, branch, monkeypatch):
    import gradslam_b200 as gs

    B, L, H, W = shape
    tma = branch.startswith("tma")
    assert _k1r_uses_tma(H, W) == tma
    if tma:
        assert H % 8 != 0 and W % 32 != 0
    if "misaligned" in branch:
        # frame (b, s) starts (b*L + s) * H*W * 3 floats into the colour tensor: odd H*W puts odd frames off 16 bytes
        assert (H * W) % 2 == 1 and B * L > 1
    rgb, depth, K, poses, ref = _inputs_and_ref(B, L, H, W, cameras="camera per element" in branch)
    pc, _ = gs.PointFusion(odom="gt", device=DEV)(_frames(gs, rgb, depth, K, poses))
    _assert_matches_oracle(pc, ref)
    if tma:  # the plain kernel on the same shape gives the same bits
        monkeypatch.setenv("GSX_NO_TMA", "1")
        plain, _ = gs.PointFusion(odom="gt", device=DEV)(_frames(gs, rgb, depth, K, poses))
        _assert_same_rows(plain, pc)


# ---------------------------------------------------------------------------------------------- sequence driver
@pytest.mark.parametrize("groups", [1, 2, 3, 4])
def test_batch_groups_match_oracle(groups, monkeypatch):
    """B=5 split into 1..4 groups (G=3: sizes 1, 2, 2; G=4: 1, 1, 1, 2); L=5 alternates the two workspace halves
    more than once.  With a camera per element, a group that read its first element's camera (or element 0's) fails."""
    import gradslam_b200 as gs
    from gradslam_b200 import _C

    monkeypatch.setenv("GSX_SEQ_GROUPS", str(groups))
    assert _C.lib().gsx_pointfusion_sequence_groups(5) == groups
    for cameras in (False, True):
        rgb, depth, K, poses, ref = _inputs_and_ref(5, 5, 48, 64, cameras=cameras)
        pc, out_poses = gs.PointFusion(odom="gt", device=DEV)(_frames(gs, rgb, depth, K, poses))
        _assert_matches_oracle(pc, ref)
        assert torch.equal(out_poses.cpu(), poses)


def test_host_fed_frames_equal_device_resident():
    """Pinned host frames are uploaded 4 frames at a time, so L=5 makes a second sequence call with s_begin = 4.  On
    the synthetic inputs and with a camera per element."""
    import gradslam_b200 as gs

    slam = gs.PointFusion(odom="gt", device=DEV)
    for cameras in (False, True):
        rgb, depth, K, poses, ref = _inputs_and_ref(5, 5, 48, 64, cameras=cameras)
        dev_pc, _ = slam(_frames(gs, rgb, depth, K, poses))
        host = gs.RGBDImages(rgb.pin_memory(), depth.pin_memory(), K.pin_memory(), poses.pin_memory())
        assert not host.depth_image.is_cuda
        host_pc, host_poses = slam(host)
        _assert_same_rows(host_pc, dev_pc)
        _assert_matches_oracle(host_pc, ref)
        assert torch.equal(host_poses.cpu(), poses)


def test_merge_capacity_overflow_clamps_only_the_overflowing_element():
    """Caller-provided storage too small for one element's last frame: K4 drops that element's surplus rows, clamps its
    size to the capacity and raises the flag; the other elements and the memory behind the storage are untouched."""
    import gradslam_b200 as gs

    B, L, H, W = 3, 3, 48, 64
    rgb, depth, K, poses = make_sequence(B, L, H, W, seed=4)
    poses[B - 1, L - 1, :3, 3] += 5.0  # the last frame of the last element sees nothing of its map: all appended
    ref = oracle.run_slam(rgb, depth, K, poses, odom="gt").map
    before = oracle.run_slam(rgb[:, :L - 1], depth[:, :L - 1], K, poses[:, :L - 1], odom="gt").map
    final = ref.counts()
    low = max(max(final[:B - 1]), before.counts()[B - 1])
    cap = (low + final[B - 1]) // 2
    assert low < cap < final[B - 1]
    geo = torch.empty((B + 1, cap, 8), dtype=torch.float32, device=DEV)
    col = torch.empty((B + 1, cap, 4), dtype=torch.float32, device=DEV)
    geo[B].view(torch.int32).fill_(SENTINEL)
    col[B].view(torch.int32).fill_(SENTINEL)
    out = gs.Pointclouds()
    out._attach(geo[:B], col[:B])
    pc, _ = gs.PointFusion(odom="gt", device=DEV)(_frames(gs, rgb, depth, K, poses), out=out)
    counts = [int(c) for c in pc.num_points_per_pointcloud.tolist()]  # device sizes, no overflow check
    with pytest.raises(RuntimeError, match="capacity exceeded"):
        pc.points_list
    assert counts == final[:B - 1] + [cap]
    for b in range(B):
        n = counts[b]
        assert torch.equal(geo[b, :n, 0:3].cpu(), ref.points[b][:n]), b
        assert torch.equal(geo[b, :n, 3:6].cpu(), ref.normals[b][:n]), b
        assert torch.equal(geo[b, :n, 6:7].cpu(), ref.ccounts[b][:n]), b
        assert torch.equal(col[b, :n, 0:3].cpu(), ref.colors[b][:n]), b
    assert (geo[B].view(torch.int32) == SENTINEL).all()
    assert (col[B].view(torch.int32) == SENTINEL).all()


# ---------------------------------------------------------------------------------------------- grid 1-NN
def _target(kind, n, g):
    if kind == "surface":  # three faces of a box
        a = torch.rand(n, 3, generator=g)
        a[torch.arange(n), torch.randint(0, 3, (n,), generator=g)] = 0.0
        return a * torch.tensor([4.0, 3.0, 6.0])
    if kind == "planar":  # one grid axis of one cell
        a = torch.rand(n, 3, generator=g) * torch.tensor([5.0, 2.0, 0.0])
        return a + torch.tensor([0.0, 0.0, 1.5])
    if kind == "collinear":
        return torch.rand(n, 1, generator=g) * torch.tensor([[1.0, -2.0, 0.5]]) + torch.tensor([0.3, 0.2, 0.1])
    if kind == "identical":
        return torch.tensor([[0.25, -1.5, 2.0]]).repeat(n, 1)
    if kind == "clusters":  # 100 units apart: the rings run out and queries between them scan everything
        a = torch.rand(n, 3, generator=g) * 0.5
        a[n // 2:] += 100.0
        return a
    raise KeyError(kind)


def _cell_boundary_queries(tgt, m, g):
    """Points whose coordinates lie exactly on cell faces of the search grid that k_grid_bbox builds for `tgt`."""
    lo, hi = tgt.min(0).values, tgt.max(0).values
    ext = torch.clamp((hi - lo).max(), min=1e-6)
    c = ext / 64.0  # (float32 as in the kernel: kGridMaxDim = 64)
    k = torch.randint(0, 65, (m, 3), generator=g).to(torch.float32)
    return lo + k * c


@pytest.mark.parametrize("kind", ["surface", "planar", "collinear", "identical", "clusters"])
def test_knn1_grid_batched_ragged_and_degenerate(kind):
    """B=3 padded clouds, target sizes {60000, 3000, 0} (the stride puts every element on the grid path), ragged source
    sizes; queries near the target, on cell faces, and far away.  (idx, d2) per element equal the brute-force oracle;
    an empty target gives idx -1 and d2 +inf, as the padding rows do."""
    from gradslam_b200.odometry import icputils

    g = torch.Generator().manual_seed(11)
    nt, ns = [60000, 3000, 0], [2500, 1700, 900]
    Nt, Ns = max(nt), max(ns)
    tgt = torch.zeros(3, Nt, 3)
    src = torch.zeros(3, Ns, 3)
    for b in range(3):
        t = _target(kind, max(nt[b], 1), g)[:nt[b]]
        tgt[b, :nt[b]] = t
        base = t if nt[b] else _target(kind, 100, g)
        q = base[torch.randint(0, base.shape[0], (ns[b],), generator=g)] + 0.01 * torch.randn(ns[b], 3, generator=g)
        q[: ns[b] // 4] = _cell_boundary_queries(base, ns[b] // 4, g)
        q[ns[b] // 4: ns[b] // 4 + 40] += 30.0 * torch.randn(40, 3, generator=g)
        src[b, :ns[b]] = q
    d2, idx = icputils.knn1(src.to(DEV), tgt.to(DEV), torch.tensor(ns, dtype=torch.int32, device=DEV),
                            torch.tensor(nt, dtype=torch.int32, device=DEV))
    d2, idx = d2.cpu(), idx.cpu()
    for b in range(3):
        if nt[b]:
            rd2, ridx = oracle.knn1(src[b, :ns[b]], tgt[b, :nt[b]])
            assert torch.equal(idx[b, :ns[b]], ridx), b
            assert torch.equal(d2[b, :ns[b]], rd2), b
        else:
            assert (idx[b, :ns[b]] == -1).all()
            assert torch.isposinf(d2[b, :ns[b]]).all()
        assert (idx[b, ns[b]:] == -1).all() and torch.isposinf(d2[b, ns[b]:]).all()


# ---------------------------------------------------------------------------------------------- ICP localisation
def test_batched_icp_on_grid_path_matches_oracle():
    """PointFusion with gradICP, dsratio 2 at 120x160: lattice targets of several thousand points for two elements at
    once, searched through the grid."""
    import gradslam_b200 as gs

    B, L, H, W = 2, 3, 120, 160
    rgb, depth, K, poses = make_sequence(B, L, H, W, seed=3, yaw0=0.6)
    slam = gs.PointFusion(odom="gradicp", numiters=10, dsratio=2, device=DEV)
    pc, rec = slam(_frames(gs, rgb, depth, K, poses))
    ref = oracle.run_slam(rgb, depth, K, poses, odom="gradicp", numiters=10, dsratio=2)
    torch.testing.assert_close(rec.cpu(), ref.poses, rtol=0, atol=1e-4)
    got = pc.num_points_per_pointcloud.tolist()
    for b in range(B):
        # a pose difference of ~1e-6 can flip a borderline match, so sizes may differ by a handful of points
        assert abs(got[b] - ref.map.counts()[b]) <= max(3, ref.map.counts()[b] // 500), (got, ref.map.counts())


@pytest.mark.parametrize("odom", ["icp", "gradicp"])
def test_long_icpslam_static_camera_matches_oracle(odom):
    """ICPSLAM appends every valid pixel of every frame, so a camera that dwells piles up one more map point per
    lattice pixel per frame: after 40 frames the lattice-active ICP target holds ~40 points per lattice pixel.  The
    target buffer must hold all of them (no dropped target rows, no overflow reported against the map)."""
    import gradslam_b200 as gs

    B, L, H, W = 1, 40, 32, 40
    rgb, depth, K, poses = make_sequence(B, L, H, W, seed=0, motion_scale=0.0, yaw0=0.6)
    slam = gs.ICPSLAM(odom=odom, numiters=3, dsratio=4, device=DEV)
    pc, rec = slam(_frames(gs, rgb, depth, K, poses))
    ref = oracle.run_slam(rgb, depth, K, poses, mode="aggregate", odom=odom, numiters=3, dsratio=4)
    assert [len(p) for p in pc.points_list] == ref.map.counts()  # (reads the sizes through the overflow check)
    torch.testing.assert_close(rec.cpu(), ref.poses, rtol=0, atol=1e-4)
