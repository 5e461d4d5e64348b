"""Host-side mirror logic on CPU tensors: containers, validation, error behaviour (reference conventions:
TypeError for wrong types, ValueError for wrong shapes, raised before any compute)."""
import math

import pytest
import torch

import gradslam_b200 as gs
from gradslam_b200.geometry import geometryutils, projutils, se3utils
from gradslam_b200.slam import fusionutils


def _clouds():
    pts = [torch.rand(3, 3), torch.rand(5, 3)]
    return gs.Pointclouds(pts, [p.clone() for p in pts], [p.clone() for p in pts], [torch.rand(3, 1), torch.rand(5, 1)]), pts


def test_pointclouds_list_padded_views():
    pc, pts = _clouds()
    assert len(pc) == 2 and pc.has_points and pc.has_normals and pc.has_colors and pc.has_features
    assert pc.points_padded.shape == (2, 5, 3)
    assert torch.equal(pc.points_list[0], pts[0]) and torch.equal(pc.points_list[1], pts[1])
    assert pc.points_padded[0, 3:].abs().sum() == 0  # zero padding
    assert pc.nonpad_mask.tolist() == [[True] * 3 + [False] * 2, [True] * 5]
    assert pc.num_points_per_pointcloud.tolist() == [3, 5]
    assert pc.num_features == 1


def test_pointclouds_from_padded_and_empty():
    t = torch.rand(2, 4, 3)
    pc = gs.Pointclouds(t)
    assert pc.points_padded.shape == (2, 4, 3) and pc.equisized
    empty = gs.Pointclouds()
    assert not empty.has_points and len(empty) == 0
    with pytest.raises(IndexError):
        empty[0]
    with pytest.raises(TypeError):
        gs.Pointclouds(3)
    with pytest.raises(ValueError):
        gs.Pointclouds([])
    with pytest.raises(ValueError):
        gs.Pointclouds([torch.rand(3, 2)])
    with pytest.raises(ValueError):
        gs.Pointclouds(torch.rand(2, 4, 3), normals=torch.rand(2, 5, 3))
    with pytest.raises(TypeError):
        gs.Pointclouds([torch.rand(3, 3)], normals=torch.rand(1, 3, 3))


def test_pointclouds_append_clone_index():
    pc, pts = _clouds()
    other, pts2 = _clouds()
    before = pc.clone()
    pc.append_points(other)
    assert pc.num_points_per_pointcloud.tolist() == [6, 10]
    assert torch.equal(pc.points_list[0], torch.cat([pts[0], pts2[0]]))
    assert torch.equal(pc.points_list[1], torch.cat([pts[1], pts2[1]]))
    assert before.num_points_per_pointcloud.tolist() == [3, 5]  # clone is deep
    assert pc.points_padded[0, 6:].abs().sum() == 0
    sub = pc[1]
    assert len(sub) == 1 and sub.points_list[0].shape == (10, 3)
    sub = pc[[0, 1]]
    assert len(sub) == 2
    e = gs.Pointclouds()
    e.append_points(other)
    assert e.num_points_per_pointcloud.tolist() == [3, 5]
    with pytest.raises(TypeError):
        pc.append_points(torch.rand(3))
    with pytest.raises(ValueError):
        pc.append_points(gs.Pointclouds([torch.rand(2, 3)]))  # batch size mismatch
    with pytest.raises(ValueError):
        pc.append_points(gs.Pointclouds([torch.rand(2, 3), torch.rand(2, 3)]))  # missing normals


def test_pointclouds_rigid_ops_and_projection():
    pc, pts = _clouds()
    T = torch.eye(4)
    T[:3, 3] = torch.tensor([1.0, 2.0, 3.0])
    moved = pc.transform(T)
    torch.testing.assert_close(moved.points_list[1], pts[1] + T[:3, 3])
    assert moved.points_padded[0, 3:].abs().sum() == 0  # padding is not offset
    assert torch.equal(pc.points_list[1], pts[1])  # out of place
    R = torch.tensor([[0.0, -1, 0], [1, 0, 0], [0, 0, 1]])
    rot = pc.rotate(R)
    torch.testing.assert_close(rot.points_list[0], pts[0] @ R.t())
    torch.testing.assert_close(rot.normals_list[0], pts[0] @ R.t())
    torch.testing.assert_close((pc + 1.0).points_list[0], pts[0] + 1.0)
    torch.testing.assert_close((pc * 2.0).points_list[0], pts[0] * 2.0)
    K = torch.eye(4)
    K[0, 0] = K[1, 1] = 100.0
    K[0, 2], K[1, 2] = 32.0, 24.0
    proj = pc.pinhole_projection(K)
    want = torch.stack([100 * pts[0][:, 0] / pts[0][:, 2] + 32, 100 * pts[0][:, 1] / pts[0][:, 2] + 24,
                        torch.ones(3)], -1)
    torch.testing.assert_close(proj.points_list[0], want, rtol=1e-5, atol=1e-5)
    with pytest.raises(ValueError):
        pc.transform(torch.eye(3))
    with pytest.raises(TypeError):
        pc.rotate_(3)


def test_pointclouds_setters():
    pc, _ = _clouds()
    new = torch.rand(2, 5, 3)
    pc.points_padded = new
    assert torch.equal(pc.points_padded, new)
    with pytest.raises(ValueError):
        pc.points_padded = torch.rand(2, 6, 3)
    pc.features_padded = torch.rand(2, 5, 4)
    assert pc.num_features == 4


def test_rgbdimages_validation_and_slicing():
    rgb, depth = torch.rand(2, 3, 8, 10, 3), torch.rand(2, 3, 8, 10, 1)
    K, poses = torch.eye(4).repeat(2, 1, 1, 1), torch.eye(4).repeat(2, 3, 1, 1)
    fr = gs.RGBDImages(rgb, depth, K, poses)
    assert fr.shape == (2, 3, 8, 10) and len(fr) == 2 and not fr.channels_first and fr.cdim == 4
    sub = fr[:, 1]
    assert sub.shape == (2, 1, 8, 10) and sub.poses.shape == (2, 1, 4, 4)
    assert sub.depth_image.data_ptr() == depth[:, 1:2].data_ptr()  # a view, not a copy
    assert fr[1, 0:2].shape == (1, 2, 8, 10)
    assert torch.equal(fr.valid_depth_mask, depth > 0)
    with pytest.raises(TypeError):
        gs.RGBDImages(3, depth, K)
    with pytest.raises(ValueError):
        gs.RGBDImages(rgb[0], depth, K)
    with pytest.raises(ValueError):
        gs.RGBDImages(rgb, depth[..., :0], K)
    with pytest.raises(ValueError):
        gs.RGBDImages(rgb, depth, torch.eye(4).repeat(2, 2, 1, 1))
    with pytest.raises(IndexError):
        fr[5]
    with pytest.raises(IndexError):
        fr[0, 0, 0]
    cf = fr.to_channels_first()
    assert cf.channels_first and cf.rgb_image.shape == (2, 3, 3, 8, 10) and cf.depth_image.shape == (2, 3, 1, 8, 10)
    assert torch.equal(cf.to_channels_last().rgb_image, rgb)
    fr.poses = poses * 2  # setter validates shape
    with pytest.raises(ValueError):
        fr.poses = torch.eye(4)
    with pytest.raises(RuntimeError, match="CUDA"):
        fr.vertex_map  # compute needs CUDA tensors: no CPU path


def test_geometry_helpers():
    K = torch.eye(4)
    K[0, 0], K[1, 1], K[0, 2], K[1, 2] = 120.3, -120.0, 79.875, 59.875
    torch.testing.assert_close(projutils.inverse_intrinsics(K) @ K, torch.eye(4), rtol=1e-5, atol=1e-5)
    p = torch.tensor([[1.0, 2.0, 4.0], [0.0, 0.0, 0.0]])
    uv = projutils.project_points(p, K)
    torch.testing.assert_close(uv[0], torch.tensor([120.3 * 0.25 + 79.875, -120.0 * 0.5 + 59.875]))
    assert uv[1].tolist() == [0.0, 0.0]  # z == 0 divides by 1
    assert projutils.homogenize_points(p).shape == (2, 4)
    torch.testing.assert_close(projutils.unhomogenize_points(torch.tensor([[2.0, 4.0, 2.0]])), torch.tensor([[1.0, 2.0]]))
    back = projutils.unproject_points(torch.tensor([[1.0, 1.0]]), torch.eye(3), torch.tensor([2.0]))
    torch.testing.assert_close(back, torch.tensor([[2.0, 2.0, 2.0]]))
    with pytest.raises(TypeError):
        projutils.project_points(3, K)
    with pytest.raises(ValueError):
        projutils.inverse_intrinsics(torch.eye(5))
    T = se3utils.se3_exp(torch.tensor([0.1, 0.2, 0.3, 0.0, 0.0, math.pi / 2]))
    torch.testing.assert_close(T[:3, :3], torch.tensor([[0.0, -1, 0], [1, 0, 0], [0, 0, 1]]), rtol=1e-6, atol=1e-6)
    Tinv = geometryutils.inverse_transformation(T)
    torch.testing.assert_close(geometryutils.compose_transformations(T, Tinv), torch.eye(4), rtol=1e-6, atol=1e-6)
    torch.testing.assert_close(geometryutils.relative_transformation(T, T), torch.eye(4), rtol=1e-5, atol=1e-6)
    cloud = torch.rand(7, 3)
    torch.testing.assert_close(geometryutils.transform_pointcloud(cloud, T), cloud @ T[:3, :3].t() + T[:3, 3])
    g = geometryutils.create_meshgrid(3, 4, normalized_coords=False)
    assert g.shape == (1, 3, 4, 2) and g[0, 2, 3].tolist() == [2.0, 3.0]


def test_fusionutils_small_helpers_and_errors():
    pts = torch.tensor([[-1.0, 0.0, 1.0], [0.0, 0.0, 0.0]])
    a = fusionutils.get_alpha(pts, 0.6)
    torch.testing.assert_close(a, torch.tensor([6.2177e-02, 1.0]), rtol=1e-3, atol=1e-6)
    assert fusionutils.are_points_close(pts, pts + 0.01, 0.05).all()
    assert not fusionutils.are_points_close(pts, pts + 1.0, 0.05).any()
    n = torch.tensor([[0.0, 0.0, 1.0]])
    assert fusionutils.are_normals_similar(n, n, 0.9).all()
    with pytest.warns(RuntimeWarning):
        fusionutils.are_normals_similar(n * 2, n * 2, 0.9)
    with pytest.raises(TypeError):
        fusionutils.get_alpha(3, 0.6)
    with pytest.raises(ValueError):
        fusionutils.get_alpha(torch.rand(4, 2), 0.6)
    with pytest.raises(TypeError):
        fusionutils.update_map_fusion(3, None, 0.05, 0.9, 0.6)
    pc = gs.Pointclouds()
    with pytest.raises(TypeError):
        fusionutils.update_map_fusion(pc, 3, 0.05, 0.9, 0.6)
    rgb, depth = torch.rand(1, 2, 8, 8, 3), torch.rand(1, 2, 8, 8, 1)
    fr = gs.RGBDImages(rgb, depth, torch.eye(4).view(1, 1, 4, 4), torch.eye(4).repeat(1, 2, 1, 1))
    with pytest.raises(ValueError):  # sequence length must be 1
        fusionutils.update_map_fusion(pc, fr, 0.05, 0.9, 0.6)


def test_slam_constructors_and_defaults():
    slam = gs.PointFusion(odom="gt")
    assert slam.dist_th == 0.05 and slam.sigma == 0.6 and slam.dsratio == 4
    assert abs(slam.dot_th - math.cos(math.radians(20))) < 1e-12
    with pytest.raises(ValueError):
        gs.PointFusion(odom="nope")
    with pytest.raises(TypeError):
        gs.PointFusion(odom="gt", dist_th="x")
    with pytest.warns(UserWarning):
        gs.PointFusion(odom="gt", angle_th=120)
    with pytest.raises(TypeError):
        slam(3)
    assert gs.ICPSLAM(odom="gt").odomprov is None


def test_structutils_list_padded_round_trip():
    """gradslam/structures/structutils.py:47-124: padding sizes, pad value, equisized stacking, cutting back, errors."""
    import pytest
    import torch

    from gradslam_b200.structures import list_to_padded, padded_to_list, structutils

    g = torch.Generator().manual_seed(0)
    items = [torch.rand(n, 3, generator=g) for n in (4, 0, 7)]
    padded = list_to_padded(items, pad_value=-1.0)
    assert padded.shape == (3, 7, 3)
    assert torch.equal(padded[0, :4], items[0]) and (padded[0, 4:] == -1).all() and (padded[1] == -1).all()
    assert list_to_padded(items, (9, 5)).shape == (3, 9, 5)
    with pytest.raises(ValueError):
        list_to_padded(items, (9,))
    with pytest.raises(ValueError):
        list_to_padded([torch.rand(2, 3, 1)], (4, 4))
    same = [torch.rand(5, 3, generator=g) for _ in range(2)]
    assert torch.equal(list_to_padded(same, equisized=True), torch.stack(same))
    back = padded_to_list(padded, [4, 0, 7])
    assert all(torch.equal(a, b) for a, b in zip(back, items))
    assert padded_to_list(padded, [(2, 2), (0, 3), (7, 1)])[2].shape == (7, 1)
    assert len(structutils.padded_to_list(padded)) == 3
    with pytest.raises(ValueError):
        padded_to_list(padded[0])
    with pytest.raises(ValueError):
        padded_to_list(padded, [1, 2])
    with pytest.raises(ValueError):
        padded_to_list(padded, [(1, 2, 3)] * 3)


def test_top_level_namespace_mirrors_the_reference():
    """gradslam/__init__.py re-exports the geometry and structures names at the top level."""
    import gradslam_b200 as gs

    for name in ("project_points", "unproject_points", "inverse_intrinsics", "homogenize_points", "unhomogenize_points",
                 "Pointclouds", "RGBDImages", "list_to_padded", "padded_to_list", "ICPSLAM", "PointFusion"):
        assert hasattr(gs, name), name
    assert gs.slam.update_map_fusion is gs.slam.fusionutils.update_map_fusion


def test_visualisation_export_host_side():
    """Pointclouds.open3d / .plotly (pointclouds.py:1239-1383): array preparation, colour ranges, sub-sampling, and the
    viewer objects built through stub modules (neither package is installed in the build image)."""
    import sys
    import types

    import numpy as np
    import pytest
    import torch

    from gradslam_b200.structures import Pointclouds
    from gradslam_b200.structures.export import cloud_arrays

    g = torch.Generator().manual_seed(0)
    pts = [torch.rand(50, 3, generator=g), torch.rand(20, 3, generator=g)]
    nrm = [torch.rand(50, 3, generator=g), torch.rand(20, 3, generator=g)]
    col = [torch.rand(50, 3, generator=g) * 255, torch.rand(20, 3, generator=g)]  # one 0..255 cloud, one 0..1 cloud
    pc = Pointclouds(pts, nrm, col)
    p, c, n = cloud_arrays(pc, 0, include_normals=True)
    assert p.shape == (50, 3) and np.array_equal(p, pts[0].numpy()) and np.array_equal(n, nrm[0].numpy())
    np.testing.assert_allclose(c, (col[0] / 255).clamp(0, 1).numpy())
    _, c1, n1 = cloud_arrays(pc, 1, color_range=255.0)
    np.testing.assert_allclose(c1, (col[1] * 255).clamp(0, 255).numpy())
    assert n1 is None
    torch.manual_seed(3)
    p_sub, c_sub, _ = cloud_arrays(pc, 0, max_num_points=10)
    assert p_sub.shape == (10, 3) and c_sub.shape == (10, 3)
    rows = {tuple(r) for r in pts[0].numpy().round(6).tolist()}
    assert all(tuple(r) in rows for r in p_sub.round(6).tolist())
    with pytest.raises(TypeError):
        cloud_arrays(pc, 0.0)
    with pytest.raises(TypeError):
        pc.plotly("0")

    # missing packages fail at the call with a clear message
    for name in ("open3d", "plotly", "plotly.graph_objects"):
        sys.modules.pop(name, None)
    import importlib.util
    if importlib.util.find_spec("open3d") is None:
        with pytest.raises(ImportError, match="open3d"):
            pc.open3d(0)
    if importlib.util.find_spec("plotly") is None:
        with pytest.raises(ImportError, match="plotly"):
            pc.plotly(0)

    # stub viewers: check what is handed over
    class _Obj:
        def __init__(self, **kw):
            self.__dict__.update(kw)

        def update_layout(self, **kw):
            self.layout = kw

    go = types.ModuleType("plotly.graph_objects")
    go.Scatter3d = lambda **kw: _Obj(**kw)
    go.Figure = lambda data: _Obj(data=data)
    plotly = types.ModuleType("plotly")
    plotly.graph_objects = go
    o3d = types.ModuleType("open3d")
    o3d.geometry = types.SimpleNamespace(PointCloud=lambda: _Obj())
    o3d.utility = types.SimpleNamespace(Vector3dVector=lambda a: np.asarray(a))
    sys.modules.update({"plotly": plotly, "plotly.graph_objects": go, "open3d": o3d})
    try:
        fig = pc.plotly(1, point_size=3)
        sc = fig.data[0]
        assert sc.mode == "markers" and sc.marker["size"] == 3 and sc.marker["color"].dtype == np.uint8
        assert np.array_equal(sc.x, pts[1].numpy()[:, 0]) and fig.layout["showlegend"] is False
        assert pc.plotly(1, include_colors=False, as_figure=False).marker == {"size": 2}
        pcd = pc.open3d(0, include_normals=True)
        assert pcd.points.shape == (50, 3) and pcd.normals.shape == (50, 3) and pcd.colors.max() <= 1.0
        assert not hasattr(pc.open3d(0, include_colors=False), "colors")
    finally:
        for name in ("plotly", "plotly.graph_objects", "open3d"):
            sys.modules.pop(name, None)


def test_downsample_pointclouds_known_answer():
    """The reference's hand-built case (tests/odometry/test_icputils.py:800-867) restated as data: rows whose pixel lies
    on the ds lattice survive, in table order; attributes follow; missing attributes stay missing."""
    import torch

    from gradslam_b200.odometry.icputils import downsample_pointclouds
    from gradslam_b200.structures import Pointclouds

    pts = torch.tensor([[5.0, 5, 5], [3, 3, 3], [1, 2, 3], [3, 2, 1], [1, 0, 1], [0, 0, 0]]).unsqueeze(0)
    table = torch.tensor([[0, 0, 0, 0], [0, 1, 4, 2], [0, 2, 3, 1], [0, 3, 0, 3], [0, 4, 3, 3], [0, 5, 3, 6]])
    ds = downsample_pointclouds(Pointclouds(pts, -pts, 2 * pts), table, 3)
    want = torch.tensor([[5.0, 5, 5], [3, 2, 1], [1, 0, 1], [0, 0, 0]]).unsqueeze(0)
    assert torch.equal(ds.points_padded, want) and torch.equal(ds.normals_padded, -want)
    assert torch.equal(ds.colors_padded, 2 * want)
    ds2 = downsample_pointclouds(Pointclouds(pts), table, 2)
    assert torch.equal(ds2.points_padded, torch.tensor([[5.0, 5, 5], [3, 3, 3]]).unsqueeze(0))
    assert ds2.normals_padded is None and ds2.colors_padded is None


def test_batched_downsample_pointclouds_matches_per_element_indexing():
    """downsample_pointclouds selects all elements at once; the result must equal the reference's per-element boolean
    indexing (icputils.py:604-617), including an empty element, an unsorted table and zero padding."""
    import torch

    import gradslam_b200 as gs
    from gradslam_b200.odometry.icputils import downsample_pointclouds

    g = torch.Generator().manual_seed(5)
    sizes = [40, 0, 65]
    mk = lambda c: [torch.rand(n, c, generator=g) for n in sizes]
    pc = gs.Pointclouds(mk(3), mk(3), mk(3))
    rows = []
    for b, n in enumerate(sizes):
        for i in range(n):
            if torch.rand((), generator=g) < 0.6:
                rows.append([b, i, int(torch.randint(0, 12, (), generator=g)), int(torch.randint(0, 12, (), generator=g))])
    table = torch.tensor(rows)
    table = table[torch.randperm(table.shape[0], generator=g)]  # element blocks interleaved
    ds = 3
    out = downsample_pointclouds(pc, table, ds)
    kept = table[(table[:, 2] % ds == 0) & (table[:, 3] % ds == 0)]
    for b in range(len(sizes)):
        sel = kept[kept[:, 0] == b][:, 1]
        for name in ("points_list", "normals_list", "colors_list"):
            assert torch.equal(getattr(out, name)[b], getattr(pc, name)[b][sel]), (name, b)
        n = int(out.num_points_per_pointcloud[b])
        assert n == sel.numel() and float(out.points_padded[b, n:].abs().sum()) == 0.0
    # no row survives
    empty = downsample_pointclouds(pc, table[:0], ds)
    assert empty.num_points_per_pointcloud.tolist() == [0, 0, 0]


def test_compact_rows_is_stable_and_differentiable():
    import torch

    from gradslam_b200.odometry.icputils import _compact_rows

    g = torch.Generator().manual_seed(2)
    mask = torch.rand(5, 37, generator=g) < 0.35
    mask[3] = False
    v = torch.rand(5, 37, 3, generator=g, requires_grad=True)
    (out,), counts = _compact_rows(mask, [v])
    assert counts == mask.sum(1).tolist() and out.shape == (5, max(counts), 3)
    for b in range(5):
        assert torch.equal(out[b, : counts[b]], v[b][mask[b]])
        assert float(out[b, counts[b]:].detach().abs().sum()) == 0.0
    out.sum().backward()
    assert torch.equal(v.grad, mask.unsqueeze(-1).expand(-1, -1, 3).float())


def test_exchange_mode_selection(monkeypatch):
    from gradslam_b200 import parallel

    monkeypatch.delenv("GSX_MAP_EXCHANGE", raising=False)
    assert parallel._exchange_mode("cpu", 2) == "all_gather"  # gloo tests
    assert parallel._exchange_mode("cuda:0", 2) == "peer"
    assert parallel._exchange_mode("cuda:0", 4) == "all_gather"
    assert parallel._exchange_mode("cuda:0", 8) == "all_gather"
    monkeypatch.setenv("GSX_MAP_EXCHANGE", "p2p")
    assert parallel._exchange_mode("cuda:0", 8) == "p2p"
    monkeypatch.setenv("GSX_MAP_EXCHANGE", "bogus")
    import pytest

    with pytest.raises(ValueError):
        parallel._exchange_mode("cuda:0", 2)


def test_bind_host_to_gpu_is_harmless_without_a_gpu():
    import os

    from gradslam_b200 import parallel

    before = os.sched_getaffinity(0)
    assert parallel.bind_host_to_gpu("cuda:0") is None or os.sched_getaffinity(0) <= before
    os.sched_setaffinity(0, before)


def test_differentiable_pose_composition_uses_canonical_order():
    """ICPSLAM's differentiable step composes T_icp · prev pose with separately rounded products and sums in the
    order of the fused step's k_pose_compose (the oracle's rigid_compose), so both steps return the same bits."""
    import gsx_oracle as oracle
    from gradslam_b200.slam.icpslam import _compose_canonical

    g = torch.Generator().manual_seed(0)
    A = torch.stack([oracle.se3_exp(torch.randn(6, generator=g)) for _ in range(64)]).requires_grad_(True)
    P = torch.stack([oracle.se3_exp(torch.randn(6, generator=g)) for _ in range(64)]).requires_grad_(True)
    out = _compose_canonical(A, P)
    assert torch.equal(out.detach(), oracle.rigid_compose(A.detach(), P.detach()))
    w = torch.randn(64, 4, 4, generator=g)
    (out * w).sum().backward()
    A2, P2 = A.detach().double().requires_grad_(True), P.detach().double().requires_grad_(True)
    ((A2[:, :3, :3] @ P2[:, :3, :] + torch.cat([torch.zeros(64, 3, 3, dtype=torch.float64), A2[:, :3, 3:]], -1))
     * w[:, :3].double()).sum().backward()
    torch.testing.assert_close(A.grad.double(), A2.grad, rtol=1e-6, atol=1e-6)
    torch.testing.assert_close(P.grad.double(), P2.grad, rtol=1e-6, atol=1e-6)
