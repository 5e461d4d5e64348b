"""GPU parity: CUDA hot path (through the C ABI) vs the CPU oracle on identical seeded inputs."""
import pytest
import torch

import gsx_oracle as oracle
from cameras import CameraShape, camera_inputs
from gradslam_b200.synthetic import make_sequence

pytestmark = pytest.mark.gpu


def _dev():
    return torch.device("cuda:0")


def _frames(gs, rgb, depth, K, poses, dev):
    return gs.RGBDImages(rgb.to(dev), depth.to(dev), K.to(dev), None if poses is None else poses.to(dev))


@pytest.mark.parametrize("shape", [(2, 3, 48, 64), (1, 2, 120, 160), (3, 1, 33, 47),
                                   pytest.param(CameraShape((3, 4, 48, 64)), id="cameras")])
def test_frame_maps_bit_exact(shape):
    """K1 against oracle.frame_maps: all four maps identical to the last bit (canonical arithmetic).  With a camera per
    element (skew and 4th column set, which back-projection ignores)."""
    import gradslam_b200 as gs

    B, L, H, W = shape
    if isinstance(shape, CameraShape):
        rgb, depth, K, poses = camera_inputs(B, L, H, W, seed=3, skew=0.75)
    else:
        rgb, depth, K, poses = make_sequence(B, L, H, W, seed=3)
    fr = _frames(gs, rgb, depth, K, poses, _dev())
    ref = oracle.frame_maps(depth, K, poses)
    for name, got in (("vertex", fr.vertex_map), ("normal", fr.normal_map), ("gvertex", fr.global_vertex_map),
                      ("gnormal", fr.global_normal_map)):
        assert torch.equal(got.cpu(), ref[name]), name
    # without poses the global maps are the local maps
    fr2 = _frames(gs, rgb, depth, K, None, _dev())
    assert torch.equal(fr2.global_vertex_map.cpu(), ref["vertex"])
    assert torch.equal(fr2.global_normal_map.cpu(), ref["normal"])


def _compare_maps(pc, ref_map, exact_structure=True):
    got = [int(c) for c in pc.num_points_per_pointcloud.tolist()]
    assert got == ref_map.counts()
    for b in range(len(got)):
        # every operation of the fusion step is canonical IEEE arithmetic on both sides (the exp of the confidence
        # weight is taken in double and rounded once), so the maps are bit-identical
        assert torch.equal(pc.points_list[b].cpu(), ref_map.points[b])
        assert torch.equal(pc.normals_list[b].cpu(), ref_map.normals[b])
        assert torch.equal(pc.colors_list[b].cpu(), ref_map.colors[b])
        assert torch.equal(pc.features_list[b].cpu(), ref_map.ccounts[b])


@pytest.mark.parametrize("shape", [(2, 4, 48, 64), (1, 5, 120, 160), (3, 3, 64, 64),
                                   pytest.param(CameraShape((3, 4, 48, 64)), id="cameras")])
def test_pointfusion_gt_sequence_matches_oracle(shape):
    import gradslam_b200 as gs

    B, L, H, W = shape
    if isinstance(shape, CameraShape):
        rgb, depth, K, poses = camera_inputs(B, L, H, W, seed=0, skew=0.75)
    else:
        rgb, depth, K, poses = make_sequence(B, L, H, W, seed=0)
    slam = gs.PointFusion(odom="gt", device=_dev())
    pc, out_poses = slam(_frames(gs, rgb, depth, K, poses, _dev()))
    ref = oracle.run_slam(rgb, depth, K, poses, odom="gt")
    _compare_maps(pc, ref.map)
    assert torch.equal(out_poses.cpu(), poses)


def test_step_api_equals_sequence_call():
    """slam.step() frame by frame (per-frame C calls) == slam(frames) (single C call), on the synthetic inputs and with
    a camera per element."""
    import gradslam_b200 as gs

    B, L, H, W = 2, 4, 48, 64
    dev = _dev()
    slam = gs.PointFusion(odom="gt", device=dev)
    for rgb, depth, K, poses in (make_sequence(B, L, H, W, seed=5), camera_inputs(3, L, H, W, seed=5, skew=0.75)):
        B = rgb.shape[0]
        frames = _frames(gs, rgb, depth, K, poses, dev)
        pc_seq, _ = slam(frames)
        pc = gs.Pointclouds(device=dev)
        for s in range(L):
            pc, _ = slam.step(pc, frames[:, s], None, inplace=True)
        assert pc.num_points_per_pointcloud.tolist() == pc_seq.num_points_per_pointcloud.tolist()
        for b in range(B):
            assert torch.equal(pc.points_list[b], pc_seq.points_list[b])
            assert torch.equal(pc.features_list[b], pc_seq.features_list[b])
            assert torch.equal(pc.colors_list[b], pc_seq.colors_list[b])
    # not-inplace step leaves the input map untouched
    before = [p.clone() for p in pc.points_list]
    pc2, _ = slam.step(pc, frames[:, 0], None, inplace=False)
    for b in range(B):
        assert torch.equal(pc.points_list[b], before[b])
    assert pc2 is not pc


def test_ragged_and_empty_inputs():
    """All-invalid depth for one element (its map stays empty), tiny images, single frame."""
    import gradslam_b200 as gs

    B, L, H, W = 2, 3, 16, 24
    rgb, depth, K, poses = make_sequence(B, L, H, W, seed=7)
    depth[1] = 0.0  # element 1 never sees a valid depth
    slam = gs.PointFusion(odom="gt", device=_dev())
    pc, _ = slam(_frames(gs, rgb, depth, K, poses, _dev()))
    ref = oracle.run_slam(rgb, depth, K, poses, odom="gt")
    assert ref.map.counts()[1] == 0
    _compare_maps(pc, ref.map)


def test_cpu_tensors_are_refused():
    import gradslam_b200 as gs

    rgb, depth, K, poses = make_sequence(1, 1, 16, 16, seed=0)
    fr = gs.RGBDImages(rgb, depth, K, poses)
    with pytest.raises(RuntimeError, match="CUDA"):
        fr.vertex_map


def test_materialised_maps_path_equals_fused_path():
    """update_map_fusion with frame maps already cached on the RGBDImages (K1 output gathered by K2/K4) gives the
    same bits as the default path where K2/K4 sample the depth image on the fly."""
    import gradslam_b200 as gs
    from gradslam_b200.slam import fusionutils

    B, L, H, W = 2, 3, 40, 56
    rgb, depth, K, poses = make_sequence(B, L, H, W, seed=9)
    dev = _dev()
    frames = _frames(gs, rgb, depth, K, poses, dev)
    slam = gs.PointFusion(odom="gt", device=dev)
    pc_a, pc_b = gs.Pointclouds(device=dev), gs.Pointclouds(device=dev)
    for s in range(L):
        fa, fb = frames[:, s], frames[:, s]
        fb.global_vertex_map, fb.global_normal_map  # materialise (K1) -> non-fused kernels
        pc_a = fusionutils.update_map_fusion(pc_a, fa, slam.dist_th, slam.dot_th, slam.sigma, inplace=True)
        pc_b = fusionutils.update_map_fusion(pc_b, fb, slam.dist_th, slam.dot_th, slam.sigma, inplace=True)
    assert pc_a.num_points_per_pointcloud.tolist() == pc_b.num_points_per_pointcloud.tolist()
    for b in range(B):
        for attr in ("points_list", "normals_list", "colors_list", "features_list"):
            assert torch.equal(getattr(pc_a, attr)[b], getattr(pc_b, attr)[b]), attr


def test_update_map_aggregate_matches_oracle():
    """ICPSLAM mapping step (append every valid pixel) == oracle.update_map_aggregate, bit for bit."""
    import gradslam_b200 as gs
    from gradslam_b200.slam import fusionutils

    B, L, H, W = 2, 3, 32, 48
    rgb, depth, K, poses = make_sequence(B, L, H, W, seed=12)
    dev = _dev()
    frames = _frames(gs, rgb, depth, K, poses, dev)
    pc = gs.Pointclouds(device=dev)
    smap = oracle.SurfelMap()
    for s in range(L):
        pc = fusionutils.update_map_aggregate(pc, frames[:, s], inplace=True)
        smap = oracle.update_map_aggregate(smap, oracle.frame_maps(depth[:, s:s + 1], K, poses[:, s:s + 1]), rgb[:, s:s + 1])
    assert pc.num_points_per_pointcloud.tolist() == smap.counts()
    assert not pc.has_features
    for b in range(B):
        assert torch.equal(pc.points_list[b].cpu(), smap.points[b])
        assert torch.equal(pc.normals_list[b].cpu(), smap.normals[b])
        assert torch.equal(pc.colors_list[b].cpu(), smap.colors[b])


def test_update_map_fusion_threshold_monotonicity():
    """The reference's property test (tests/slam/test_fusionutils.py:1138-1176): looser thresholds merge more and
    append less; with impossible thresholds every valid pixel is appended."""
    import gradslam_b200 as gs
    from gradslam_b200.slam import fusionutils as fu

    rgb, depth, K, poses = make_sequence(2, 2, 40, 56, seed=17)
    dev = _dev()
    frames = _frames(gs, rgb, depth, K, poses, dev)
    base = fu.update_map_fusion(gs.Pointclouds(device=dev), frames[:, 0], 0.05, 0.94, 0.6)
    n0 = base.num_points_per_pointcloud
    valid1 = (depth[:, 1, ..., 0] > 0).flatten(1).sum(1)
    strict = fu.update_map_fusion(base, frames[:, 1], 0.0, 1.0, 0.6)       # nothing can match
    loose = fu.update_map_fusion(base, frames[:, 1], 0.05, 0.94, 0.6)
    looser = fu.update_map_fusion(base, frames[:, 1], 0.2, 0.5, 0.6)
    assert (strict.num_points_per_pointcloud.cpu() == n0.cpu() + valid1).all()
    assert (looser.num_points_per_pointcloud <= loose.num_points_per_pointcloud).all()
    assert (loose.num_points_per_pointcloud <= strict.num_points_per_pointcloud).all()
    assert (base.num_points_per_pointcloud == n0).all()  # inputs untouched


def test_sliced_sequence_with_cached_maps():
    """Maps computed once on the whole (B, L) RGBDImages and then sliced per frame are strided views; the fusion must
    give the same bits as the on-the-fly path."""
    import gradslam_b200 as gs

    B, L, H, W = 2, 3, 32, 40
    rgb, depth, K, poses = make_sequence(B, L, H, W, seed=23)
    dev = _dev()
    frames = _frames(gs, rgb, depth, K, poses, dev)
    frames.global_vertex_map, frames.global_normal_map  # K1 over the full sequence; slices below are views
    slam = gs.PointFusion(odom="gt", device=dev)
    pc = gs.Pointclouds(device=dev)
    for s in range(L):
        live = frames[:, s]
        assert not live.global_vertex_map.is_contiguous() or B == 1
        pc, _ = slam.step(pc, live, None, inplace=True)
    ref, _ = slam(_frames(gs, rgb, depth, K, poses, dev))
    assert pc.num_points_per_pointcloud.tolist() == ref.num_points_per_pointcloud.tolist()
    for b in range(B):
        assert torch.equal(pc.points_list[b], ref.points_list[b])
        assert torch.equal(pc.normals_list[b], ref.normals_list[b])
        assert torch.equal(pc.features_list[b], ref.features_list[b])


def test_sequence_driver_error_path_joins_streams_and_poisons_nothing():
    """A launch failure in the middle of gsx_pointfusion_sequence_gt (injected at frame 2 of 4, after the batch-group
    streams were forked and two frames were enqueued): the call returns the error as a RuntimeError, the internal streams
    are joined to the caller's stream (a synchronize returns, nothing is left running unordered), and the next call on
    the same cached workspace produces the bit-identical, correct map - no epoch / record state survives a failed call."""
    import gradslam_b200 as gs
    from gradslam_b200 import _C

    B, L, H, W = 4, 4, 48, 64
    rgb, depth, K, poses = make_sequence(B, L, H, W, seed=12)
    frames = _frames(gs, rgb, depth, K, poses, _dev())
    slam = gs.PointFusion(odom="gt", device=_dev())
    good, _ = slam(frames)
    _C.lib().gsx_debug_fail_at_frame(2)
    with pytest.raises(RuntimeError, match="injected failure at frame 2"):
        slam(frames)
    torch.cuda.synchronize()
    again, _ = slam(frames)
    assert again.num_points_per_pointcloud.tolist() == good.num_points_per_pointcloud.tolist()
    for b in range(B):
        assert torch.equal(again.points_list[b], good.points_list[b])
        assert torch.equal(again.features_list[b], good.features_list[b])
    # and the per-frame path on the same workspace is unaffected as well
    ref = oracle.run_slam(rgb, depth, K, poses, odom="gt")
    _compare_maps(again, ref.map)


def test_packed_store_views_and_input_validation():
    """The public tensors are strided views of the packed rows (no copies), and tensors whose pointers reach a kernel
    are validated: a CPU map or a float64 colour image raises instead of being reinterpreted."""
    import gradslam_b200 as gs
    from gradslam_b200.slam import fusionutils as fu

    rgb, depth, K, poses = make_sequence(2, 2, 32, 40, seed=2)
    frames = _frames(gs, rgb, depth, K, poses, _dev())
    pc = fu.update_map_fusion(gs.Pointclouds(device=_dev()), frames[:, 0], 0.05, 0.94, 0.6)
    assert pc._geo.shape[-1] == 8 and pc._col.shape[-1] == 4
    assert pc.points_padded.data_ptr() == pc._geo.data_ptr()
    assert pc.normals_padded.data_ptr() == pc._geo.data_ptr() + 12
    assert pc.features_padded.data_ptr() == pc._geo.data_ptr() + 24
    assert pc.colors_padded.data_ptr() == pc._col.data_ptr()
    assert pc.points_padded.stride() == (pc.capacity * 8, 8, 1)
    assert (pc._geo[..., 7] == 0).all() and (pc._col[..., 3] == 0).all()
    # float64 inputs are cast to float32 rows on construction
    p64 = torch.rand(1, 5, 3, dtype=torch.float64, device=_dev())
    assert gs.Pointclouds(p64, p64, p64, p64[..., :1]).points_padded.dtype == torch.float32
    # a CPU map with CUDA frames, and a float64 colour image, raise
    cpu_map = gs.Pointclouds(torch.rand(2, 4, 3), torch.rand(2, 4, 3), torch.rand(2, 4, 3), torch.rand(2, 4, 1))
    with pytest.raises((RuntimeError, ValueError)):
        fu.update_map_fusion(cpu_map, frames[:, 1], 0.05, 0.94, 0.6)
    bad = gs.RGBDImages(rgb.double().to(_dev()), depth.to(_dev()), K.to(_dev()), poses.to(_dev()))
    with pytest.raises(TypeError):
        fu.update_map_fusion(pc, bad[:, 1], 0.05, 0.94, 0.6)
    with pytest.raises(ValueError, match="both have or not have features"):
        fu.update_map_aggregate(pc, frames[:, 1])
