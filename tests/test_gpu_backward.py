"""Backward of K1 (depth -> vertex / normal / global maps) against PyTorch autograd of a plain fp32 torch
implementation of the same op chain (gradslam/structures/rgbdimages.py:643-762)."""
import pytest
import torch

from cameras import CameraShape, camera_inputs
from gradslam_b200.synthetic import make_sequence as _make_sequence, punch_lattice_holes

pytestmark = pytest.mark.gpu


def make_sequence(*args, **kw):
    """Inputs for checking gradient FORMULAS: sparse lattice holes instead of random ones, so that no pixel's normal is
    the normalised residue of a cancelling cross product (derivative ~1e7; both the kernels and the reference produce
    it, but no tolerance survives it).  Parity on the random-hole distribution is pinned by the golden fixtures
    (tests/golden/ref_grad.npz is recorded from the reference on random holes)."""
    kw.setdefault("hole_fraction", 0.0)
    rgb, depth, K, poses = _make_sequence(*args, **kw)
    return rgb, punch_lattice_holes(depth), K, poses
DEV = "cuda:0"


def _torch_maps(depth, K, poses):
    """Differentiable fp32 torch reference (einsum-free, same formulas).  depth (B,L,H,W,1)."""
    B, L, H, W, _ = depth.shape
    fx, fy, cx, cy = K[:, 0, 0, 0] + 1e-6, K[:, 0, 1, 1] + 1e-6, K[:, 0, 0, 2], K[:, 0, 1, 2]
    u = torch.arange(W, dtype=torch.float32, device=depth.device).view(1, 1, 1, W)
    v = torch.arange(H, dtype=torch.float32, device=depth.device).view(1, 1, H, 1)
    d = depth[..., 0]
    vf = (d > 0).float()
    x = ((u - cx.view(B, 1, 1, 1)) / fx.view(B, 1, 1, 1)) * d * vf
    y = ((v - cy.view(B, 1, 1, 1)) / fy.view(B, 1, 1, 1)) * d * vf
    vert = torch.stack([x.expand(B, L, H, W), y.expand(B, L, H, W), d * vf], -1)
    dh = torch.zeros_like(vert)
    dv = torch.zeros_like(vert)
    dh[..., :, :-1, :] = vert[..., :, 1:, :] - vert[..., :, :-1, :]
    dv[..., :-1, :, :] = vert[..., 1:, :, :] - vert[..., :-1, :, :]
    dh = torch.cat([dh[..., :, :-1, :], dh[..., :, -2:-1, :]], dim=-2)
    dv = torch.cat([dv[..., :-1, :, :], dv[..., -2:-1, :, :]], dim=-3)
    c = torch.cross(dh, dv, dim=-1)
    nrm = torch.linalg.norm(c, dim=-1, keepdim=True)
    n = c / torch.where(nrm == 0, torch.ones_like(nrm), nrm) * vf.unsqueeze(-1)
    R, t = poses[..., :3, :3], poses[..., :3, 3]
    gv = (torch.einsum("blij,blhwj->blhwi", R, vert) + t.view(B, L, 1, 1, 3)) * vf.unsqueeze(-1)
    gn = torch.einsum("blij,blhwj->blhwi", R, n)
    return vert, n, gv, gn


@pytest.mark.parametrize("shape", [(2, 2, 24, 40), (1, 1, 17, 23),
                                   pytest.param(CameraShape((3, 2, 24, 40)), id="cameras")])
def test_backproject_backward_matches_autograd(shape):
    """With a camera per element, d/d pose of each element is checked against its own camera's chain."""
    import gradslam_b200 as gs

    B, L, H, W = shape
    if isinstance(shape, CameraShape):
        rgb, depth, K, poses = camera_inputs(B, L, H, W, 21, skew=0.75, lattice_holes=True)
    else:
        rgb, depth, K, poses = make_sequence(B, L, H, W, seed=21)
    g = torch.Generator().manual_seed(3)
    ups = [torch.randn(B, L, H, W, 3, generator=g).to(DEV) for _ in range(4)]
    # engine
    d1 = depth.to(DEV).requires_grad_(True)
    p1 = poses.to(DEV).requires_grad_(True)
    fr = gs.RGBDImages(rgb.to(DEV), d1, K.to(DEV), p1)
    outs = (fr.vertex_map, fr.normal_map, fr.global_vertex_map, fr.global_normal_map)
    loss = sum((o * w).sum() for o, w in zip(outs, ups))
    loss.backward()
    # torch reference
    d2 = depth.to(DEV).requires_grad_(True)
    p2 = poses.to(DEV).requires_grad_(True)
    refs = _torch_maps(d2, K.to(DEV), p2)
    for o, r in zip(outs, refs):
        torch.testing.assert_close(o.detach(), r.detach(), rtol=1e-4, atol=1e-5)
    sum((o * w).sum() for o, w in zip(refs, ups)).backward()
    scale = d2.grad.abs().max().item()
    torch.testing.assert_close(d1.grad, d2.grad, rtol=1e-3, atol=1e-4 * scale)
    pscale = p2.grad.abs().max().item()
    torch.testing.assert_close(p1.grad[..., :3, :], p2.grad[..., :3, :], rtol=1e-3, atol=1e-4 * pscale)
    assert p1.grad[..., 3, :].abs().max() == 0


def test_backward_only_global_maps_and_no_pose_grad():
    import gradslam_b200 as gs

    rgb, depth, K, poses = make_sequence(1, 2, 20, 28, seed=22)
    d1 = depth.to(DEV).requires_grad_(True)
    fr = gs.RGBDImages(rgb.to(DEV), d1, K.to(DEV), poses.to(DEV))
    w = torch.randn(1, 2, 20, 28, 3, device=DEV)
    (fr.global_vertex_map * w).sum().backward()
    d2 = depth.to(DEV).requires_grad_(True)
    refs = _torch_maps(d2, K.to(DEV), poses.to(DEV))
    (refs[2] * w).sum().backward()
    torch.testing.assert_close(d1.grad, d2.grad, rtol=1e-3, atol=1e-5)


def test_gradicp_function_gradients_match_oracle_autograd():
    """point_to_plane_gradICP in differentiable mode (CUDA 1-NN + taped algebra): d(T)/d(src) equals the gradient
    PyTorch's tape gives for the oracle restatement of the reference (icputils.py:370-545)."""
    import gsx_oracle as oracle
    from gradslam_b200.odometry import icputils

    rgb, depth, K, poses = make_sequence(1, 1, 40, 56, seed=31, hole_fraction=0.0, yaw0=0.6)
    m = oracle.frame_maps(depth, K, poses)
    tgt = m["gvertex"][0, 0].reshape(-1, 3).contiguous()
    tgt_n = m["gnormal"][0, 0].reshape(-1, 3).contiguous()
    T_true = oracle.se3_exp(torch.tensor([0.01, -0.005, 0.008, 0.01, -0.01, 0.005]))
    src0 = oracle.rigid_apply(T_true, tgt)
    w = torch.randn(4, 4, generator=torch.Generator().manual_seed(1))
    # oracle (CPU autograd)
    s_ref = src0.clone().requires_grad_(True)
    T_ref, _ = oracle.point_to_plane_gradicp(s_ref, tgt, tgt_n, torch.eye(4), numiters=4)
    (T_ref * w).sum().backward()
    # engine, differentiable mode
    s_gpu = src0.clone().to(DEV).requires_grad_(True)
    T_gpu, _ = icputils.point_to_plane_gradICP(s_gpu[None], tgt[None].to(DEV), tgt_n[None].to(DEV),
                                               torch.eye(4, device=DEV), numiters=4)
    (T_gpu * w.to(DEV)).sum().backward()
    torch.testing.assert_close(T_gpu.detach().cpu(), T_ref.detach(), rtol=0, atol=1e-4)
    scale = s_ref.grad.abs().max().item()
    torch.testing.assert_close(s_gpu.grad.cpu(), s_ref.grad, rtol=2e-2, atol=2e-3 * scale)
    # the fused (non-differentiable) loop gives the same forward value
    T_fused, _ = icputils.point_to_plane_gradICP(src0[None].to(DEV), tgt[None].to(DEV), tgt_n[None].to(DEV),
                                                 torch.eye(4, device=DEV), numiters=4)
    torch.testing.assert_close(T_fused.cpu(), T_gpu.detach().cpu(), rtol=0, atol=1e-4)


def test_icpslam_pose_gradient_wrt_live_depth():
    """Config-3 style check at small size: ICPSLAM(odom='gradicp'), L=2; gradient of the recovered pose of frame 1
    w.r.t. the depth of frame 1 (through the K1 backward kernel and the taped gradLM) vs the oracle's autograd."""
    import gradslam_b200 as gs
    import gsx_oracle as oracle

    B, L, H, W = 1, 2, 32, 40
    rgb, depth, K, poses = make_sequence(B, L, H, W, seed=33, yaw0=0.6)
    w = torch.randn(4, 4, generator=torch.Generator().manual_seed(2))
    d_ref = depth.clone().requires_grad_(True)
    ref = oracle.run_slam(rgb, d_ref, K, poses, mode="aggregate", odom="gradicp", numiters=3, dsratio=2)
    (ref.poses[0, 1] * w).sum().backward()
    d_gpu = depth.clone().to(DEV).requires_grad_(True)
    slam = gs.ICPSLAM(odom="gradicp", numiters=3, dsratio=2, device=DEV)
    pc, rec = slam(gs.RGBDImages(rgb.to(DEV), d_gpu, K.to(DEV), poses.to(DEV)))
    torch.testing.assert_close(rec.detach().cpu(), ref.poses.detach(), rtol=0, atol=1e-4)
    (rec[0, 1] * w.to(DEV)).sum().backward()
    # frame 1 (the live frame) AND frame 0 (whose pixels became the map the ICP aligns to)
    for s in (1, 0):
        g_ref, g_gpu = d_ref.grad[:, s], d_gpu.grad[:, s].cpu()
        assert torch.isfinite(g_gpu).all() and g_ref.abs().max() > 0
        scale = g_ref.abs().max().item()
        torch.testing.assert_close(g_gpu, g_ref, rtol=5e-2, atol=5e-3 * scale)


@pytest.mark.parametrize("B,L,cameras", [(1, 2, False), (2, 3, False), (3, 3, True)], ids=["1-2", "2-3", "cameras"])
def test_pointfusion_map_gradients_match_oracle_autograd(B, L, cameras):
    """PointFusion(odom='gt') in differentiable mode: d(fused map)/d(depth, colours) through the K1 backward kernel and
    the K4 backward kernel (gsx_fusion_merge_append_bwd), against PyTorch autograd of the oracle restatement
    (fusionutils.py:580-722).  L=3 chains a merge into rows that were themselves merged one frame earlier.  cameras:
    a camera per element (tests/golden/cameras.py) with skew and 4th intrinsics column."""
    import gradslam_b200 as gs
    import gsx_oracle as oracle

    H, W = 24, 32
    if cameras:
        rgb, depth, K, poses = camera_inputs(B, L, H, W, 41, skew=0.75, lattice_holes=True)
    else:
        rgb, depth, K, poses = make_sequence(B, L, H, W, seed=41, yaw0=0.6)
    d_ref, c_ref = depth.clone().requires_grad_(True), rgb.clone().requires_grad_(True)
    ref = oracle.run_slam(c_ref, d_ref, K, poses, odom="gt")
    g = torch.Generator().manual_seed(5)
    counts = ref.map.counts()
    # (normals are left out of the loss: the oracle's autograd of |cross| is NaN at zero-length normals; the normal
    # channel of the K4 backward is covered by test_merge_append_op_gradients_wrt_previous_map, K1's by the tests above)
    ws = [[torch.randn(n, c, generator=g) for c in (3, 3, 1)] for n in counts]
    loss = 0
    for b in range(B):
        for t, w in zip((ref.map.points[b], ref.map.colors[b], ref.map.ccounts[b]), ws[b]):
            loss = loss + (t * w).sum()
    loss.backward()

    d_gpu, c_gpu = depth.clone().to(DEV).requires_grad_(True), rgb.clone().to(DEV).requires_grad_(True)
    slam = gs.PointFusion(odom="gt", device=DEV)
    pc, _ = slam(gs.RGBDImages(c_gpu, d_gpu, K.to(DEV), poses.to(DEV)))
    assert pc.num_points_per_pointcloud.tolist() == counts
    loss = 0
    for b in range(B):
        torch.testing.assert_close(pc.points_list[b].detach().cpu(), ref.map.points[b].detach(), rtol=1e-5, atol=1e-6)
        for t, w in zip((pc.points_list[b], pc.colors_list[b], pc.features_list[b]), ws[b]):
            loss = loss + (t * w.to(DEV)).sum()
    loss.backward()
    for got, want in ((d_gpu.grad.cpu(), d_ref.grad), (c_gpu.grad.cpu(), c_ref.grad)):
        assert torch.isfinite(got).all()
        scale = want.abs().max().item()
        torch.testing.assert_close(got, want, rtol=1e-3, atol=1e-4 * scale)
    # the same call without gradients takes the fused in-place kernels and gives the same map, bit for bit
    with torch.no_grad():
        pc2, _ = slam(gs.RGBDImages(rgb.to(DEV), depth.to(DEV), K.to(DEV), poses.to(DEV)))
    assert pc2.num_points_per_pointcloud.tolist() == counts
    for b in range(B):
        assert torch.equal(pc2.points_list[b], pc.points_list[b].detach())
        assert torch.equal(pc2.normals_list[b], pc.normals_list[b].detach())
        assert torch.equal(pc2.colors_list[b], pc.colors_list[b].detach())
        assert torch.equal(pc2.features_list[b], pc.features_list[b].detach())


def test_merge_append_op_gradients_wrt_previous_map():
    """update_map_fusion with a map that requires grad: d(updated map)/d(previous map rows) through
    gsx_fusion_merge_append_bwd (matched rows are scaled by c/(c+alpha), their confidence collects the quotient-rule
    terms, untouched rows pass through), against float64 autograd of the same formulas on the kernel's association."""
    import gradslam_b200 as gs
    from gradslam_b200.slam import fusionutils as fu

    B, H, W = 2, 20, 28
    rgb, depth, K, poses = make_sequence(B, 2, H, W, seed=43, yaw0=0.6)
    frames = gs.RGBDImages(rgb.to(DEV), depth.to(DEV), K.to(DEV), poses.to(DEV))
    with torch.no_grad():
        base = fu.update_map_fusion(gs.Pointclouds(device=DEV), frames[:, 0], 0.05, 0.94, 0.6)
        table = fu.find_correspondences(base, frames[:, 1], 0.05, 0.94)
    assert table.shape[0] > 0
    n0 = base.num_points_per_pointcloud.tolist()
    leaves = {k: getattr(base, k + "_padded").clone().requires_grad_(True)
              for k in ("points", "normals", "colors", "features")}
    pc = gs.Pointclouds(leaves["points"], leaves["normals"], leaves["colors"], leaves["features"])
    pc._set_counts(n0)
    out = fu.update_map_fusion(pc, frames[:, 1], 0.05, 0.94, 0.6)
    n1 = out.num_points_per_pointcloud.tolist()
    g = torch.Generator().manual_seed(3)
    wts = {k: torch.randn(B, max(n1), c, generator=g).to(DEV) for k, c in (("points", 3), ("normals", 3), ("colors", 3),
                                                                              ("features", 1))}
    mask = out.nonpad_mask.unsqueeze(-1)
    sum((getattr(out, k + "_padded") * wts[k] * mask).sum() for k in wts).backward()

    # float64 reference on the same association (fusionutils.py:654-699)
    f1 = frames[:, 1]
    ref = {k: v.detach().double().requires_grad_(True) for k, v in leaves.items()}
    b, n, h, w = table.unbind(1)
    alpha = fu.get_alpha(f1.vertex_map[:, 0].double(), 0.6, dim=-1, keepdim=True)[b, h, w]
    cc = ref["features"][b, n]
    tot = cc + alpha
    new = {}
    for k, fmap in (("points", f1.global_vertex_map), ("normals", f1.global_normal_map), ("colors", f1.rgb_image)):
        new[k] = ref[k].index_put((b, n), (cc * ref[k][b, n] + alpha * fmap[:, 0].double()[b, h, w]) / tot)
    new["features"] = ref["features"].index_put((b, n), tot)
    live = (torch.arange(max(n0), device=DEV).view(1, -1) < torch.tensor(n0, device=DEV).view(-1, 1)).unsqueeze(-1)
    sum((new[k] * wts[k][:, :max(n0)].double() * live).sum() for k in new).backward()
    for k in leaves:
        got, want = leaves[k].grad.double() * live, ref[k].grad
        torch.testing.assert_close(got, want, rtol=1e-4, atol=1e-5 * want.abs().max().item())


def _lm_reference_functions():
    import importlib.util
    import os
    spec = importlib.util.spec_from_file_location(
        "icp_diff_ref", os.path.join(os.path.dirname(os.path.abspath(__file__)), "test_icp_diff_host.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_solve_update_transform_ops_forward_and_backward():
    """K7 ops on the device (gsx_icp_solve_*, gsx_icp_update_*, gsx_rigid_transform_*) against float64 autograd of the
    reference formulas (solve_linear_system icputils.py:22-90, se3_exp se3utils.py:77-115, gates icputils.py:519-543,
    transform_pointcloud geometryutils.py:737-794)."""
    from gradslam_b200.odometry import icputils as iu
    refm = _lm_reference_functions()
    g = torch.Generator().manual_seed(11)
    A = torch.randn(300, 6, dtype=torch.float64, generator=g)
    bb = torch.randn(300, dtype=torch.float64, generator=g) * 0.05
    M = A.t() @ A
    tri = torch.triu_indices(6, 6)
    sums64 = torch.cat([M[tri[0], tri[1]], A.t() @ bb, (bb * bb).sum().view(1)])
    damp64 = torch.tensor([1e-3], dtype=torch.float64)
    wo = torch.randn(22, dtype=torch.float64, generator=g)
    # solve
    s_ref, d_ref = sums64.clone().requires_grad_(True), damp64.clone().requires_grad_(True)
    o_ref = refm._solve(torch.cat([s_ref, d_ref]))
    (o_ref * wo).sum().backward()
    s_gpu, d_gpu = sums64.float().to(DEV).requires_grad_(True), damp64.float().to(DEV).requires_grad_(True)
    xi, dT = iu._SolveFn.apply(s_gpu, d_gpu)
    torch.testing.assert_close(torch.cat([xi, dT.reshape(-1)]).detach().cpu().double(), o_ref.detach(), rtol=0, atol=2e-6)
    ((xi * wo[:6].float().to(DEV)).sum() + (dT.reshape(-1) * wo[6:].float().to(DEV)).sum()).backward()
    for got, want in ((s_gpu.grad, s_ref.grad), (d_gpu.grad, d_ref.grad)):
        torch.testing.assert_close(got.cpu().double(), want, rtol=1e-3, atol=2e-4 * s_ref.grad.abs().max().item())
    # update, both modes and both branches
    for mode, err, nerr in ((1, 0.5, 0.3), (1, 0.3, 0.5), (0, 0.5, 0.3), (0, 0.3, 0.5)):
        xi64 = torch.randn(6, dtype=torch.float64, generator=g) * 0.05
        T64 = refm._se3_exp(torch.randn(6, dtype=torch.float64, generator=g) * 0.3)
        inp = torch.cat([xi64, torch.tensor([err, nerr, 1e-3], dtype=torch.float64), T64.reshape(-1)]).requires_grad_(True)
        wu = torch.randn(33, dtype=torch.float64, generator=g)
        o_ref = refm._update(inp, mode, 2.0, 1.0, 1.0, 200.0)
        (o_ref * wu).sum().backward()
        leaf = [t.float().to(DEV).requires_grad_(True) for t in (xi64, torch.tensor(err), torch.tensor(nerr),
                                                                  torch.tensor([1e-3]), T64)]
        dmp, dTa, Tn = iu._UpdateFn.apply(*leaf, mode, 2.0, 1.0, 1.0, 200.0)
        got = torch.cat([dmp.reshape(-1), dTa.reshape(-1), Tn.reshape(-1)])
        torch.testing.assert_close(got.detach().cpu().double(), o_ref.detach(), rtol=0, atol=2e-6)
        (got * wu.float().to(DEV)).sum().backward()
        g_got = torch.cat([t.grad.reshape(-1) for t in leaf]).cpu().double()
        torch.testing.assert_close(g_got, inp.grad, rtol=1e-4, atol=2e-5)
    # rigid transform
    P64 = torch.randn(1000, 3, dtype=torch.float64, generator=g)
    T64 = refm._se3_exp(torch.randn(6, dtype=torch.float64, generator=g) * 0.5)
    wp = torch.randn(1000, 3, dtype=torch.float64, generator=g)
    p_ref, t_ref = P64.clone().requires_grad_(True), T64.clone().requires_grad_(True)
    ((p_ref @ t_ref[:3, :3].t() + t_ref[:3, 3]) * wp).sum().backward()
    p_gpu, t_gpu = P64.float().to(DEV).requires_grad_(True), T64.float().to(DEV).requires_grad_(True)
    out = iu._RigidTransformFn.apply(p_gpu, t_gpu)
    torch.testing.assert_close(out.detach().cpu().double(), (P64 @ T64[:3, :3].t() + T64[:3, 3]), rtol=0, atol=1e-5)
    (out * wp.float().to(DEV)).sum().backward()
    torch.testing.assert_close(p_gpu.grad.cpu().double(), p_ref.grad, rtol=1e-4, atol=1e-5)
    torch.testing.assert_close(t_gpu.grad.cpu().double(), t_ref.grad, rtol=1e-4, atol=1e-3)


def test_icp_lm_function_gradients_match_oracle_autograd():
    """point_to_plane_ICP (LM accept / reject, icputils.py:235-367) in differentiable mode against the oracle's tape."""
    import gsx_oracle as oracle
    from gradslam_b200.odometry.icputils import point_to_plane_ICP

    rgb, depth, K, poses = make_sequence(1, 1, 40, 56, seed=29, hole_fraction=0.0, yaw0=0.6)
    m = oracle.frame_maps(depth, K, poses)
    tgt = m["gvertex"][0, 0].reshape(-1, 3).contiguous()
    tgt_n = m["gnormal"][0, 0].reshape(-1, 3).contiguous()
    T_true = oracle.se3_exp(torch.tensor([0.01, -0.005, 0.008, 0.01, -0.01, 0.005]))
    src0 = oracle.rigid_apply(T_true, tgt)
    s_ref = src0.clone().requires_grad_(True)
    T_ref, _ = oracle.point_to_plane_icp(s_ref, tgt, tgt_n, torch.eye(4), numiters=4)
    wT = torch.randn(4, 4, generator=torch.Generator().manual_seed(2))
    (T_ref * wT).sum().backward()
    s_gpu = src0.clone().to(DEV).requires_grad_(True)
    T_gpu, _ = point_to_plane_ICP(s_gpu.unsqueeze(0), tgt.to(DEV).unsqueeze(0), tgt_n.to(DEV).unsqueeze(0),
                                  torch.eye(4, device=DEV), numiters=4)
    torch.testing.assert_close(T_gpu.detach().cpu(), T_ref.detach(), rtol=0, atol=1e-4)
    (T_gpu * wT.to(DEV)).sum().backward()
    scale = s_ref.grad.abs().max().item()
    torch.testing.assert_close(s_gpu.grad.cpu(), s_ref.grad, rtol=2e-2, atol=2e-3 * scale)


def test_normal_equation_op_forward_and_backward():
    """K6 as an op: the 28 sums and their hand-written backward against a plain torch construction of A, b
    (icputils.py:210-230) and PyTorch autograd, including filtered rows (idx = -1) and shared targets."""
    from gradslam_b200.odometry.icputils import _NormalEqFn

    g = torch.Generator().manual_seed(7)
    ns, nt = 700, 300
    src = torch.randn(ns, 3, generator=g)
    tgt = torch.randn(nt, 3, generator=g)
    tn = torch.nn.functional.normalize(torch.randn(nt, 3, generator=g), dim=1)
    idx = torch.randint(0, nt, (ns,), generator=g)
    idx[::7] = -1
    w = torch.randn(28, generator=g)

    def ref(s, p, n):
        keep = idx >= 0
        s, pp, nn = s[keep], p[idx[keep]], n[idx[keep]]
        sx, sy, sz = s[:, 0:1], s[:, 1:2], s[:, 2:3]
        nx, ny, nz = nn[:, 0:1], nn[:, 1:2], nn[:, 2:3]
        A = torch.cat([nx, ny, nz, nz * sy - ny * sz, nx * sz - nz * sx, ny * sx - nx * sy], 1)
        b = nx * (pp[:, 0:1] - sx) + ny * (pp[:, 1:2] - sy) + nz * (pp[:, 2:3] - sz)
        AtA, Atb = A.t() @ A, A.t() @ b
        iu = torch.triu_indices(6, 6)
        return torch.cat([AtA[iu[0], iu[1]], Atb[:, 0], (b * b).sum().view(1)])

    a = [t.clone().double().requires_grad_(True) for t in (src, tgt, tn)]
    want = ref(*a)
    (want * w.double()).sum().backward()
    b_ = [t.clone().to(DEV).requires_grad_(True) for t in (src, tgt, tn)]
    got = _NormalEqFn.apply(b_[0], b_[1], b_[2], idx.to(DEV))
    torch.testing.assert_close(got.cpu().double(), want.detach(), rtol=1e-4, atol=1e-3)
    (got * w.to(DEV)).sum().backward()
    for x, y in zip(b_, a):
        scale = y.grad.abs().max().item()
        torch.testing.assert_close(x.grad.cpu().double(), y.grad, rtol=1e-3, atol=1e-4 * scale)


def test_batched_differentiable_icp_equals_per_element_chain():
    """The batched op chain (one set of autograd ops for all elements, ragged sizes) against the per-element chain of
    round 1: transforms bit-identical, association identical, gradients w.r.t. the source clouds, the target clouds and
    the target normals equal to float32 rounding; and the providers use it (ICPSLAM-style call with B=3)."""
    import gradslam_b200 as gs
    from gradslam_b200.odometry import icputils as iu
    from gradslam_b200.odometry.gradicp import GradICPOdometryProvider

    g = torch.Generator().manual_seed(5)
    Bn, sizes_s, sizes_t = 3, [700, 512, 655], [900, 1024, 640]
    Ns, Nt = max(sizes_s), max(sizes_t)
    rgb, depth, K, poses = make_sequence(1, 1, 40, 56, seed=7, hole_fraction=0.0, yaw0=0.6)
    fr = gs.RGBDImages(rgb.to(DEV), depth.to(DEV), K.to(DEV), poses.to(DEV))
    base_p = fr.global_vertex_map[0, 0].reshape(-1, 3)
    base_n = fr.global_normal_map[0, 0].reshape(-1, 3)
    T_true = [torch.tensor([[1, 0, 0, 0.01 * (b + 1)], [0, 1, 0, -0.005], [0, 0, 1, 0.004 * b], [0, 0, 0, 1.0]],
                           device=DEV) for b in range(Bn)]
    src = torch.zeros(Bn, Ns, 3, device=DEV)
    tgt = torch.zeros(Bn, Nt, 3, device=DEV)
    tgt_n = torch.zeros(Bn, Nt, 3, device=DEV)
    for b in range(Bn):
        pick_t = torch.randperm(base_p.shape[0], generator=g)[: sizes_t[b]].to(DEV)
        pick_s = torch.randperm(base_p.shape[0], generator=g)[: sizes_s[b]].to(DEV)
        tgt[b, : sizes_t[b]] = base_p[pick_t]
        tgt_n[b, : sizes_t[b]] = base_n[pick_t]
        src[b, : sizes_s[b]] = base_p[pick_s] @ T_true[b][:3, :3].t() + T_true[b][:3, 3]
    cs = torch.tensor(sizes_s, dtype=torch.int32, device=DEV)
    ct = torch.tensor(sizes_t, dtype=torch.int32, device=DEV)
    w = torch.randn(Bn, 4, 4, generator=g).to(DEV)
    leaves = [t.clone().requires_grad_(True) for t in (src, tgt, tgt_n)]
    T_b, idx_b = iu._taped_icp_batched(leaves[0], cs, leaves[1], leaves[2], ct, None, 1, 4, 1e-8, None)
    (T_b * w).sum().backward()
    for b in range(Bn):
        l1 = [src[b:b + 1, : sizes_s[b]].clone().requires_grad_(True), tgt[b:b + 1, : sizes_t[b]].clone().requires_grad_(True),
              tgt_n[b:b + 1, : sizes_t[b]].clone().requires_grad_(True)]
        T_1, idx_1 = iu._taped_icp(l1[0], l1[1], l1[2], None, 1, 4, 1e-8, None)
        (T_1 * w[b]).sum().backward()
        assert torch.equal(T_1, T_b[b])
        assert torch.equal(idx_1, idx_b[b, : sizes_s[b]][idx_b[b, : sizes_s[b]] >= 0])
        for got, want, n in ((leaves[0].grad[b], l1[0].grad[0], sizes_s[b]), (leaves[1].grad[b], l1[1].grad[0], sizes_t[b]),
                             (leaves[2].grad[b], l1[2].grad[0], sizes_t[b])):
            scale = want.abs().max().item()
            torch.testing.assert_close(got[:n], want, rtol=1e-4, atol=1e-5 * scale)
            assert got[n:].numel() == 0 or got[n:].abs().max() == 0  # padding rows carry no gradient
    # the providers run the batched chain when a gradient is requested
    maps = gs.Pointclouds([tgt[b, : sizes_t[b]] for b in range(Bn)], [tgt_n[b, : sizes_t[b]] for b in range(Bn)])
    s_req = [src[b, : sizes_s[b]].clone().requires_grad_(True) for b in range(Bn)]
    out = GradICPOdometryProvider(numiters=4).provide(maps, gs.Pointclouds(s_req))
    assert out.shape == (Bn, 1, 4, 4) and torch.equal(out[:, 0], T_b.detach())
    (out[:, 0] * w).sum().backward()
    for b in range(Bn):
        scale = leaves[0].grad[b].abs().max().item()
        torch.testing.assert_close(s_req[b].grad, leaves[0].grad[b, : sizes_s[b]], rtol=1e-4, atol=1e-5 * scale)


# ------------------------------------------------------------------------------------------ large shapes and edges
U32 = 2.0 ** -24  # unit roundoff of float32


def _k1_reference_grads(depth, K, poses, ups, which):
    """float64 autograd of _torch_maps: d(sum(ups[i] * map i for i in which))/d(depth, poses)."""
    d = depth.detach().double().requires_grad_(True)
    p = None if poses is None else poses.detach().double().requires_grad_(True)
    refs = _torch_maps(d, K.double(), p if p is not None else torch.eye(4, dtype=torch.float64, device=d.device)
                       .expand(depth.shape[0], depth.shape[1], 4, 4))
    sum((refs[i] * ups[i].double()).sum() for i in which).backward()
    return d.grad, (None if p is None else p.grad)


@pytest.mark.parametrize("B,L,H,W,holes", [(2, 2, 480, 640, "zero"), (1, 3, 37, 45, "negative"),
                                           (2, 1, 2, 9, "zero"), (1, 2, 11, 2, "negative"), (1, 1, 2, 2, "zero")])
def test_k1_backward_large_and_minimal_shapes(B, L, H, W, holes):
    """K1 backward against float64 autograd: 480x640 with B*L = 4 (1200 tiles of pose partials per image reduced by
    k_pose_grad_reduce), H*W not a multiple of the 256-pixel tile, and H or W = 2 (the border stencil terms coincide:
    the first row / column is also the one before the last).  Holes are zeros or negative depths (both invalid)."""
    from gradslam_b200.structures.rgbdimages import backproject

    rgb, depth, K, poses = make_sequence(B, L, max(H, 8), max(W, 8), seed=51 + H)
    depth = depth[:, :, :H, :W].clone()
    depth[:, :, 0, 0] = 0.0  # (no pixel has this one as its right or lower neighbour: no degenerate normal)
    if holes == "negative":
        depth = torch.where(depth > 0, depth, -0.5 - depth)
        assert (depth < 0).any()
    g = torch.Generator().manual_seed(H * W)
    ups = [torch.randn(B, L, H, W, 3, generator=g).to(DEV) for _ in range(4)]
    d1 = depth.to(DEV).requires_grad_(True)
    p1 = poses.to(DEV).requires_grad_(True)
    outs = backproject(d1, K.to(DEV), p1)
    sum((o * u).sum() for o, u in zip(outs, ups)).backward()
    gd, gp = _k1_reference_grads(depth.to(DEV), K.to(DEV), poses.to(DEV), ups, range(4))
    torch.testing.assert_close(d1.grad.double(), gd, rtol=1e-3, atol=1e-4 * gd.abs().max().item())
    torch.testing.assert_close(p1.grad[..., :3, :].double(), gp[..., :3, :], rtol=1e-3,
                               atol=1e-4 * gp.abs().max().item())
    assert p1.grad[..., 3, :].abs().max() == 0
    assert d1.grad[depth.to(DEV) <= 0].abs().max() == 0


@pytest.mark.parametrize("which", [0, 1, 2, 3])
def test_k1_backward_single_upstream_map(which):
    """Only one of the four maps reaches the loss: the other three upstream pointers are null in the kernel."""
    from gradslam_b200.structures.rgbdimages import backproject

    B, L, H, W = 1, 2, 29, 35
    rgb, depth, K, poses = make_sequence(B, L, H, W, seed=61)
    ups = [torch.randn(B, L, H, W, 3, generator=torch.Generator().manual_seed(i)).to(DEV) for i in range(4)]
    d1 = depth.to(DEV).requires_grad_(True)
    p1 = poses.to(DEV).requires_grad_(True)
    outs = backproject(d1, K.to(DEV), p1)
    (outs[which] * ups[which]).sum().backward()
    gd, gp = _k1_reference_grads(depth.to(DEV), K.to(DEV), poses.to(DEV), ups, [which])
    torch.testing.assert_close(d1.grad.double(), gd, rtol=1e-3, atol=1e-4 * gd.abs().max().item())
    if which < 2:  # the local maps do not depend on the pose
        assert p1.grad is None or p1.grad.abs().max() == 0
    else:
        torch.testing.assert_close(p1.grad[..., :3, :].double(), gp[..., :3, :], rtol=1e-3,
                                   atol=1e-4 * gp.abs().max().item())


def test_k1_backward_without_poses_and_strided_depth_view():
    """poses=None with a global-vertex upstream (world frame == camera frame), and the depth of frame s passed as the
    view frames[:, s] of a (B, L) tensor: its element stride is L*H*W, not the dense H*W."""
    import gradslam_b200 as gs

    B, L, H, W = 2, 3, 23, 31
    rgb, depth, K, poses = make_sequence(B, L, H, W, seed=62)
    ups = [torch.randn(B, 1, H, W, 3, generator=torch.Generator().manual_seed(i)).to(DEV) for i in range(4)]
    d_all = depth.to(DEV).requires_grad_(True)
    fr = gs.RGBDImages(rgb.to(DEV), d_all, K.to(DEV))[:, 1]
    assert fr.depth_image.stride(0) == L * H * W
    (fr.global_vertex_map * ups[2]).sum().backward()
    gd, _ = _k1_reference_grads(depth[:, 1:2].to(DEV), K.to(DEV), None, ups, [2])
    torch.testing.assert_close(d_all.grad[:, 1:2].double(), gd, rtol=1e-3, atol=1e-4 * gd.abs().max().item())
    assert d_all.grad[:, 0].abs().max() == 0 and d_all.grad[:, 2].abs().max() == 0
    # and with poses, through the same view: pose gradient of that frame only
    d_all.grad = None
    p_all = poses.to(DEV).requires_grad_(True)
    fr = gs.RGBDImages(rgb.to(DEV), d_all, K.to(DEV), p_all)[:, 1]
    (fr.global_normal_map * ups[3]).sum().backward()
    gd, gp = _k1_reference_grads(depth[:, 1:2].to(DEV), K.to(DEV), poses[:, 1:2].to(DEV), ups, [3])
    torch.testing.assert_close(d_all.grad[:, 1:2].double(), gd, rtol=1e-3, atol=1e-4 * gd.abs().max().item())
    torch.testing.assert_close(p_all.grad[:, 1:2, :3].double(), gp[..., :3, :], rtol=1e-3,
                               atol=1e-4 * gp.abs().max().item())
    assert p_all.grad[:, 0].abs().max() == 0 and p_all.grad[:, 2].abs().max() == 0


def test_k1_backward_zero_cross_product_pixel():
    """A valid pixel whose right AND lower neighbours are missing: dh = dv = -v.  At pixel (0,0) with the principal
    point at (0,0), v = (0, 0, d) exactly, so every product of the cross product has a zero factor and c = 0 in any
    rounding (checked with the FMA-contracted arithmetic of cross_ref).  The kernel takes its nrm == 0 branch (the
    normal is c itself, d n / d c = I); float64 autograd of the reference formula does the same."""
    from gradslam_b200.structures.rgbdimages import backproject

    B, L, H, W = 1, 1, 6, 8
    rgb, depth, K, poses = make_sequence(B, L, H, W, seed=63)
    K = K.clone()
    K[..., 0, 2] = 0.0
    K[..., 1, 2] = 0.0
    depth = depth.clone()
    depth[0, 0, 0, 0] = 1.25
    depth[0, 0, 0, 1] = 0.0
    depth[0, 0, 1, 0] = 0.0
    ups = [torch.randn(B, L, H, W, 3, generator=torch.Generator().manual_seed(i)).to(DEV) for i in range(4)]
    d1 = depth.to(DEV).requires_grad_(True)
    p1 = poses.to(DEV).requires_grad_(True)
    outs = backproject(d1, K.to(DEV), p1)
    v = outs[0].detach()[0, 0].cpu()
    c, nrm = oracle_cross(v[0, 1] - v[0, 0], v[1, 0] - v[0, 0])
    assert torch.equal(c, torch.zeros(3)) and nrm.item() == 0.0
    assert torch.equal(outs[1].detach()[0, 0, 0, 0].cpu(), torch.zeros(3))
    sum((o * u).sum() for o, u in zip(outs, ups)).backward()
    gd, gp = _k1_reference_grads(depth.to(DEV), K.to(DEV), poses.to(DEV), ups, range(4))
    assert d1.grad[0, 0, 0, 0].abs().item() > 0
    torch.testing.assert_close(d1.grad.double(), gd, rtol=1e-3, atol=1e-4 * gd.abs().max().item())
    torch.testing.assert_close(p1.grad[..., :3, :].double(), gp[..., :3, :], rtol=1e-3,
                               atol=1e-4 * gp.abs().max().item())


def oracle_cross(a, b):
    import gsx_oracle as oracle
    c, n = oracle.cross_norm_fma(a.view(1, 3).float(), b.view(1, 3).float())
    return c.view(3), n.view(-1)


def _normal_eq_reference(s, p, n, idx):
    """The 28 sums in float64 and, for the error bound, the same sums of absolute values."""
    keep = idx >= 0
    s, pp, nn = s[keep], p[idx[keep]], n[idx[keep]]
    sx, sy, sz = s[:, 0:1], s[:, 1:2], s[:, 2:3]
    nx, ny, nz = nn[:, 0:1], nn[:, 1:2], nn[:, 2:3]
    A = torch.cat([nx, ny, nz, nz * sy - ny * sz, nx * sz - nz * sx, ny * sx - nx * sy], 1)
    b = nx * (pp[:, 0:1] - sx) + ny * (pp[:, 1:2] - sy) + nz * (pp[:, 2:3] - sz)
    iu = torch.triu_indices(6, 6)
    sums = torch.cat([(A.t() @ A)[iu[0], iu[1]], (A.t() @ b)[:, 0], (b * b).sum().view(1)])
    Aa, ba = A.abs(), b.abs()
    mags = torch.cat([(Aa.t() @ Aa)[iu[0], iu[1]], (Aa.t() @ ba)[:, 0], (ba * ba).sum().view(1)])
    return sums, mags


def _sum_bound(mags, n_terms):
    """Error bound of a float32 sum of n_terms products whose factors carry a few roundings each: every term passes
    through at most n_terms additions (any order), plus 8 roundings for the factors; |error| <= (n + 8) u sum|term|."""
    return (n_terms + 8) * U32 * mags + 1e-30


def test_normal_equation_op_large_sizes_and_batched_ragged():
    """K6 as an op at ns = 2^17 + 37 (513 reduction blocks, a partial last block): the 28 sums within the float32
    summation bound of float64, the backward against float64 autograd; then the batched op on ragged elements (a
    zero-size element, an element whose rows are all filtered) equal per element, bit for bit, to the unbatched op."""
    from gradslam_b200.odometry.icputils import _NormalEqBatchedFn, _NormalEqFn

    g = torch.Generator().manual_seed(71)
    ns, nt = (1 << 17) + 37, 5000
    src = torch.randn(ns, 3, generator=g)
    tgt = torch.randn(nt, 3, generator=g)
    tn = torch.nn.functional.normalize(torch.randn(nt, 3, generator=g), dim=1)
    idx = torch.randint(0, nt, (ns,), generator=g)
    idx[::5] = -1
    w = torch.randn(28, generator=g)
    a = [t.clone().double().requires_grad_(True) for t in (src, tgt, tn)]
    want, mags = _normal_eq_reference(*a, idx)
    (want * w.double()).sum().backward()
    b_ = [t.clone().to(DEV).requires_grad_(True) for t in (src, tgt, tn)]
    got = _NormalEqFn.apply(b_[0], b_[1], b_[2], idx.to(DEV))
    err = (got.detach().cpu().double() - want.detach()).abs()
    assert (err <= _sum_bound(mags.detach(), ns)).all(), (err / mags.detach()).max()
    # a sum that dropped blocks would miss ~(1 - kept/513) of every entry: far outside the bound
    assert (want.detach().abs() > 10 * _sum_bound(mags.detach(), ns))[:21].any()
    (got * w.to(DEV)).sum().backward()
    for x, y in zip(b_, a):
        torch.testing.assert_close(x.grad.cpu().double(), y.grad, rtol=1e-3, atol=1e-4 * y.grad.abs().max().item())

    # batched, ragged: sizes 3000, 0, 2^15 + 5 (all filtered), 70001
    sizes = [3000, 0, (1 << 15) + 5, 70001]
    Bn, Ns = len(sizes), max(sizes)
    srcb = torch.zeros(Bn, Ns, 3)
    idxb = torch.full((Bn, Ns), -1, dtype=torch.int64)
    tgtb = torch.randn(Bn, nt, 3, generator=g)
    tnb = torch.nn.functional.normalize(torch.randn(Bn, nt, 3, generator=g), dim=2)
    for e, n in enumerate(sizes):
        srcb[e, :n] = torch.randn(n, 3, generator=g)
        if e != 2:
            idxb[e, :n] = torch.randint(0, nt, (n,), generator=g)
    counts = torch.tensor(sizes, dtype=torch.int32, device=DEV)
    wb = torch.randn(Bn, 28, generator=g).to(DEV)
    lb = [t.to(DEV).requires_grad_(True) for t in (srcb, tgtb, tnb)]
    sums_b = _NormalEqBatchedFn.apply(lb[0], lb[1], lb[2], idxb.to(DEV), counts)
    (sums_b * wb).sum().backward()
    assert torch.equal(sums_b[1].detach(), torch.zeros(28, device=DEV))
    assert torch.equal(sums_b[2].detach(), torch.zeros(28, device=DEV))
    for e, n in enumerate(sizes):
        if n == 0:
            assert lb[0].grad[e].abs().max() == 0 and lb[1].grad[e].abs().max() == 0
            continue
        l1 = [lb[0].detach()[e, :n].clone().requires_grad_(True), lb[1].detach()[e].clone().requires_grad_(True),
              lb[2].detach()[e].clone().requires_grad_(True)]
        s1 = _NormalEqFn.apply(l1[0], l1[1], l1[2], idxb[e, :n].to(DEV))
        assert torch.equal(s1.detach(), sums_b[e].detach()), e
        (s1 * wb[e]).sum().backward()
        assert torch.equal(l1[0].grad, lb[0].grad[e, :n]), e
        assert lb[0].grad[e, n:].numel() == 0 or lb[0].grad[e, n:].abs().max() == 0
        torch.testing.assert_close(l1[1].grad, lb[1].grad[e], rtol=1e-5, atol=1e-6 * l1[1].grad.abs().max().item() + 1e-30)
        torch.testing.assert_close(l1[2].grad, lb[2].grad[e], rtol=1e-5, atol=1e-6 * l1[2].grad.abs().max().item() + 1e-30)
        if e == 2:
            assert lb[0].grad[e].abs().max() == 0 and lb[1].grad[e].abs().max() == 0
        else:
            ref, mg = _normal_eq_reference(srcb[e, :n].double(), tgtb[e].double(), tnb[e].double(), idxb[e, :n])
            assert ((sums_b[e].detach().cpu().double() - ref).abs() <= _sum_bound(mg, n)).all(), e


def test_rigid_transform_backward_large_empty_and_batched():
    """d/dT of the rigid transform (k_rigid_bwd partials + k_rigid_bwd_reduce) at n = 2^20 + 3 (4097 blocks) within the
    float32 summation bound of float64; n = 0 gives an exactly zero g_T; in a batched call a zero-count element gets a
    zero g_T and its padding rows zero gradient."""
    from gradslam_b200.odometry import icputils as iu
    refm = _lm_reference_functions()

    g = torch.Generator().manual_seed(81)
    n = (1 << 20) + 3
    P64 = torch.randn(n, 3, dtype=torch.float64, generator=g)
    T64 = refm._se3_exp(torch.randn(6, dtype=torch.float64, generator=g) * 0.5)
    G64 = torch.randn(n, 3, dtype=torch.float64, generator=g)
    P32, G32 = P64.float(), G64.float()
    p_gpu, t_gpu = P32.to(DEV).requires_grad_(True), T64.float().to(DEV).requires_grad_(True)
    out = iu._RigidTransformFn.apply(p_gpu, t_gpu)
    (out * G32.to(DEV)).sum().backward()
    Pd, Gd = P32.double(), G32.double()  # the float32 inputs, summed exactly in float64
    ph = torch.cat([Pd, torch.ones(n, 1, dtype=torch.float64)], 1)
    want = Gd.t() @ ph
    mags = Gd.abs().t() @ ph.abs()
    got = t_gpu.grad.cpu().double()
    nblk = -(-n // 256)
    bound = (5 + 8 + nblk + 1) * U32 * mags  # shuffle tree, 8 warps, the blocks in order, the product
    assert ((got[:3] - want).abs() <= bound).all(), ((got[:3] - want).abs() / mags).max()
    assert got[3].abs().max() == 0
    torch.testing.assert_close(p_gpu.grad.cpu().double(), Gd @ T64[:3, :3].float().double(), rtol=0, atol=1e-5)

    # n = 0
    p0 = torch.zeros(0, 3, device=DEV, requires_grad=True)
    t0 = T64.float().to(DEV).requires_grad_(True)
    iu._RigidTransformFn.apply(p0, t0).sum().backward()
    assert torch.equal(t0.grad, torch.zeros(4, 4, device=DEV))

    # batched with a zero-count element
    sizes = [700, 0, 1500]
    Bn, N = len(sizes), max(sizes)
    Pb = torch.randn(Bn, N, 3, generator=g)
    Tb = torch.stack([refm._se3_exp(torch.randn(6, dtype=torch.float64, generator=g) * 0.5).float() for _ in sizes])
    Gb = torch.randn(Bn, N, 3, generator=g)
    pb, tb = Pb.to(DEV).requires_grad_(True), Tb.to(DEV).requires_grad_(True)
    counts = torch.tensor(sizes, dtype=torch.int32, device=DEV)
    ob = iu._RigidTransformBatchedFn.apply(pb, tb, counts)
    (ob * Gb.to(DEV)).sum().backward()
    for e, m in enumerate(sizes):
        assert ob[e, m:].abs().max() == 0 if m < N else True
        assert pb.grad[e, m:].numel() == 0 or pb.grad[e, m:].abs().max() == 0
        ph = torch.cat([Pb[e, :m].double(), torch.ones(m, 1, dtype=torch.float64)], 1)
        want = Gb[e, :m].double().t() @ ph
        bound = (5 + 8 + -(-m // 256) + 1) * U32 * (Gb[e, :m].double().abs().t() @ ph.abs())
        assert ((tb.grad[e, :3].cpu().double() - want).abs() <= bound).all(), e
        assert tb.grad[e, 3].abs().max() == 0
    assert torch.equal(tb.grad[1], torch.zeros(4, 4, device=DEV))


def test_batched_differentiable_icp_on_the_grid_path():
    """B = 3 ragged targets of 20 k - 60 k points (the grid 1-NN, kGridThreshold = 4096), the grid built by the first
    association and reused by the other 2 * numiters - 1 through target_cache: _taped_icp_batched equals the per-element
    chain AND the fused icp_align bit for bit, its gradients equal the per-element chain's, and for one element they
    match the oracle's autograd (the tolerance of test_gradicp_function_gradients_match_oracle_autograd)."""
    import gsx_oracle as oracle
    import gradslam_b200 as gs
    from gradslam_b200.odometry import icputils as iu

    g = torch.Generator().manual_seed(91)
    rgb, depth, K, poses = make_sequence(1, 1, 240, 320, seed=92, yaw0=0.6)
    fr = gs.RGBDImages(rgb.to(DEV), depth.to(DEV), K.to(DEV), poses.to(DEV))
    valid = (depth[0, 0, ..., 0] > 0).reshape(-1).to(DEV)
    base_p = fr.global_vertex_map[0, 0].reshape(-1, 3)[valid]
    base_n = fr.global_normal_map[0, 0].reshape(-1, 3)[valid]
    sizes_t, sizes_s = [20000, 60000, 41234], [5000, 3000, 7001]
    Bn, Nt, Ns, numiters = 3, max(sizes_t), max(sizes_s), 4
    src = torch.zeros(Bn, Ns, 3, device=DEV)
    tgt = torch.zeros(Bn, Nt, 3, device=DEV)
    tgt_n = torch.zeros(Bn, Nt, 3, device=DEV)
    for b in range(Bn):
        T = oracle.se3_exp(torch.tensor([0.01 * (b + 1), -0.005, 0.004 * b, 0.01, -0.008 * b, 0.005])).to(DEV)
        pick_t = torch.randperm(base_p.shape[0], generator=g)[: sizes_t[b]].to(DEV)
        pick_s = torch.randperm(base_p.shape[0], generator=g)[: sizes_s[b]].to(DEV)
        tgt[b, : sizes_t[b]] = base_p[pick_t]
        tgt_n[b, : sizes_t[b]] = base_n[pick_t]
        src[b, : sizes_s[b]] = base_p[pick_s] @ T[:3, :3].t() + T[:3, 3]
    cs = torch.tensor(sizes_s, dtype=torch.int32, device=DEV)
    ct = torch.tensor(sizes_t, dtype=torch.int32, device=DEV)
    w = torch.randn(Bn, 4, 4, generator=g).to(DEV)
    leaves = [t.clone().requires_grad_(True) for t in (src, tgt, tgt_n)]
    T_b, idx_b = iu._taped_icp_batched(leaves[0], cs, leaves[1], leaves[2], ct, None, 1, numiters, 1e-8, None)
    (T_b * w).sum().backward()
    T_f, _ = iu.icp_align(src, cs, tgt, tgt_n, ct, None, 1, numiters, 1e-8, None)
    assert torch.equal(T_f, T_b.detach())
    for b in range(Bn):
        ns, nt = sizes_s[b], sizes_t[b]
        l1 = [src[b:b + 1, :ns].clone().requires_grad_(True), tgt[b:b + 1, :nt].clone().requires_grad_(True),
              tgt_n[b:b + 1, :nt].clone().requires_grad_(True)]
        T_1, idx_1 = iu._taped_icp(l1[0], l1[1], l1[2], None, 1, numiters, 1e-8, None)
        (T_1 * w[b]).sum().backward()
        assert torch.equal(T_1, T_b[b])
        assert torch.equal(idx_1, idx_b[b, :ns][idx_b[b, :ns] >= 0])
        for got, want, n in ((leaves[0].grad[b], l1[0].grad[0], ns), (leaves[1].grad[b], l1[1].grad[0], nt),
                             (leaves[2].grad[b], l1[2].grad[0], nt)):
            torch.testing.assert_close(got[:n], want, rtol=1e-4, atol=1e-5 * want.abs().max().item())
            assert got[n:].numel() == 0 or got[n:].abs().max() == 0
    # element 0 against the oracle's tape
    s_ref = src[0, : sizes_s[0]].cpu().clone().requires_grad_(True)
    T_ref, _ = oracle.point_to_plane_gradicp(s_ref, tgt[0, : sizes_t[0]].cpu(), tgt_n[0, : sizes_t[0]].cpu(),
                                             torch.eye(4), numiters=numiters)
    (T_ref * w[0].cpu()).sum().backward()
    torch.testing.assert_close(T_b[0].detach().cpu(), T_ref.detach(), rtol=0, atol=1e-4)
    scale = s_ref.grad.abs().max().item()
    torch.testing.assert_close(leaves[0].grad[0, : sizes_s[0]].cpu(), s_ref.grad, rtol=2e-2, atol=2e-3 * scale)


def test_aggregate_backward_full_size():
    """update_map_aggregate with gradients (K4 backward with with_ccounts = 0, as in ICPSLAM) at 480x640, B = 2: the
    previous map's rows pass their gradient through, every appended row carries its pixel's gradient back to K1; against
    float64 autograd of the same formulas (rows appended in row-major pixel order)."""
    import gradslam_b200 as gs
    from gradslam_b200.slam import fusionutils as fu

    B, H, W = 2, 480, 640
    rgb, depth, K, poses = make_sequence(B, 2, H, W, seed=101, yaw0=0.6)
    with torch.no_grad():
        base = fu.update_map_aggregate(gs.Pointclouds(device=DEV),
                                       gs.RGBDImages(rgb[:, :1].to(DEV), depth[:, :1].to(DEV), K.to(DEV),
                                                     poses[:, :1].to(DEV)))
    n0 = base.num_points_per_pointcloud.tolist()
    leaves = {k: getattr(base, k + "_padded").clone().requires_grad_(True) for k in ("points", "normals", "colors")}
    pc = gs.Pointclouds(leaves["points"], leaves["normals"], leaves["colors"])
    pc._set_counts(n0)
    d1 = depth[:, 1:2].to(DEV).requires_grad_(True)
    c1 = rgb[:, 1:2].to(DEV).requires_grad_(True)
    out = fu.update_map_aggregate(pc, gs.RGBDImages(c1, d1, K.to(DEV), poses[:, 1:2].to(DEV)))
    n1 = out.num_points_per_pointcloud.tolist()
    valid = depth[:, 1, ..., 0] > 0
    assert [n1[b] - n0[b] for b in range(B)] == valid.flatten(1).sum(1).tolist()
    g = torch.Generator().manual_seed(102)
    wts = {k: torch.randn(B, max(n1), 3, generator=g).to(DEV) for k in ("points", "normals", "colors")}
    mask = out.nonpad_mask.unsqueeze(-1)
    sum((getattr(out, k + "_padded") * wts[k] * mask).sum() for k in wts).backward()

    d64 = depth[:, 1:2].to(DEV).double().requires_grad_(True)
    _, _, gv, gn = _torch_maps(d64, K.to(DEV).double(), poses[:, 1:2].to(DEV).double())
    c64 = rgb[:, 1:2].to(DEV).double().requires_grad_(True)
    loss = 0
    for b in range(B):
        m = valid[b].to(DEV)
        for k, t in (("points", gv), ("normals", gn), ("colors", c64)):
            loss = loss + (t[b, 0][m] * wts[k][b, n0[b]:n1[b]].double()).sum()
    loss.backward()
    torch.testing.assert_close(d1.grad.double(), d64.grad, rtol=1e-3, atol=1e-4 * d64.grad.abs().max().item())
    torch.testing.assert_close(c1.grad.double(), c64.grad, rtol=0, atol=0)
    for k in leaves:
        for b in range(B):
            assert torch.equal(leaves[k].grad[b, : n0[b]], wts[k][b, : n0[b]])


def test_confidence_clamp_backward():
    """alpha = clamp(exp(-|v|^2 / 2 sigma^2), 1e-7, 1.01): with a small sigma a known set of pixels has exp below 1e-7.
    Fusing one frame into an empty map appends every valid pixel with confidence alpha, so d(sum w * confidence)/d depth
    is w * d alpha / d depth per pixel: exactly zero where the clamp is active (as torch.clamp's autograd gives), and the
    float64 derivative of the formula elsewhere."""
    import math

    import gradslam_b200 as gs
    from gradslam_b200.slam import fusionutils as fu

    B, H, W = 1, 40, 56
    rgb, depth, K, poses = make_sequence(B, 1, H, W, seed=111, yaw0=0.6)
    d64 = depth.to(DEV).double().requires_grad_(True)
    v = _torch_maps(d64, K.to(DEV).double(), poses.to(DEV).double())[0][0, 0]
    sq = (v * v).sum(-1)
    valid = depth[0, 0, ..., 0].to(DEV) > 0
    sigma = (sq[valid].median().sqrt() / math.sqrt(2 * 16.5)).item()  # about half of the pixels clamp
    e = torch.exp(-sq / (2 * sigma * sigma))
    clamped = valid & (e < 0.5e-7)
    free = valid & (e > 2e-7)
    assert clamped.sum() > 100 and free.sum() > 100
    wts = torch.randn(H * W, generator=torch.Generator().manual_seed(112)).to(DEV)
    (torch.clamp(e, 1e-7, 1.01)[valid] * wts[: int(valid.sum())].double()).sum().backward()

    d1 = depth.to(DEV).requires_grad_(True)
    pc = fu.update_map_fusion(gs.Pointclouds(device=DEV), gs.RGBDImages(rgb.to(DEV), d1, K.to(DEV), poses.to(DEV)),
                              0.05, 0.94, sigma)
    n = int(valid.sum())
    assert pc.num_points_per_pointcloud.tolist() == [n]
    (pc.features_list[0][:, 0] * wts[:n]).sum().backward()
    g = d1.grad[0, 0, ..., 0]
    assert g[clamped].abs().max() == 0
    assert (g[free] != 0).all()
    want = d64.grad[0, 0, ..., 0]
    torch.testing.assert_close(g[free].double(), want[free], rtol=1e-4, atol=1e-6 * want.abs().max().item())
