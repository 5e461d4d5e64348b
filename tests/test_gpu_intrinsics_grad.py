"""d(loss)/d(intrinsics) of K1's backward (gsx_backproject_normals_bwd_intrinsics) and of the differentiable PointFusion
and ICPSLAM paths that reach K through it, against PyTorch autograd of the CPU oracle (oracle/gsx_oracle.py) and the
reference's frozen d/dK (tests/golden/ref_grad_intrinsics.npz).

d/dK sums a term over every pixel of every frame, and the terms of d/dcx have both signs, so the tolerances scale with
sum |per-pixel term|, evaluated in float64 from the upstream map gradients K1's backward actually received."""
import os

import numpy as np
import pytest
import torch

import gsx_oracle as oracle
import projective_oracle as po
from cameras import camera_inputs
from gradslam_b200.synthetic import make_sequence as _make_sequence, punch_lattice_holes

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
GOLD = os.path.join(os.path.dirname(__file__), "golden")
READ = [(0, 0), (0, 2), (1, 1), (1, 2)]  # fx, cx, fy, cy: the entries K1 reads


def make_sequence(*args, **kw):
    """Lattice holes instead of random ones (see tests/test_gpu_backward.py): no normal is the residue of a cancelling
    cross product, whose derivative no tolerance survives."""
    kw.setdefault("hole_fraction", 0.0)
    rgb, depth, K, poses = _make_sequence(*args, **kw)
    return rgb, punch_lattice_holes(depth), K, poses


def _maps64(depth, k, poses):
    """K1's maps in float64 with a K^-1 entry PER PIXEL (k: four (B,L,H,W) tensors k00, k02, k11, k12), so that autograd
    w.r.t. k gives each pixel's own term.  depth (B,L,H,W), poses (B,L,4,4) or None."""
    B, L, H, W = depth.shape
    u = torch.arange(W, dtype=torch.float64, device=depth.device).view(1, 1, 1, W)
    v = torch.arange(H, dtype=torch.float64, device=depth.device).view(1, 1, H, 1)
    vf = (depth > 0).double()
    vert = torch.stack([(k[0] * u + k[1]) * depth * vf, (k[2] * v + k[3]) * depth * vf, depth * vf], -1)
    dh = vert[..., :, 1:, :] - vert[..., :, :-1, :]
    dv = vert[..., 1:, :, :] - vert[..., :-1, :, :]
    dh = torch.cat([dh, dh[..., :, -1:, :]], -2)
    dv = torch.cat([dv, dv[..., -1:, :, :]], -3)
    c = torch.cross(dh, dv, dim=-1)
    nrm = torch.linalg.norm(c, dim=-1, keepdim=True)
    n = c / torch.where(nrm == 0, torch.ones_like(nrm), nrm) * vf.unsqueeze(-1)
    if poses is None:
        return vert, n, vert, n
    R, t = poses[..., :3, :3], poses[..., :3, 3]
    gv = (torch.einsum("blij,blhwj->blhwi", R, vert) + t[:, :, None, None, :]) * vf.unsqueeze(-1)
    gn = torch.einsum("blij,blhwj->blhwi", R, n)
    return vert, n, gv, gn


def _term_scale(depth, K, poses, ups):
    """(B,4,4): sum over pixels and frames of |each pixel's term| of d/dK, in float64, for upstream gradients ups (four
    (B,L,H,W,3) tensors or None) of the four maps."""
    depth, K = depth.double(), K.double().reshape(-1, 4, 4)
    poses = None if poses is None else poses.double()
    B, L, H, W = depth.shape
    ex, ey, cx, cy = K[:, 0, 0] + 1e-6, K[:, 1, 1] + 1e-6, K[:, 0, 2], K[:, 1, 2]
    kb = [1 / ex, -cx / ex, 1 / ey, -cy / ey]
    k = [x.view(B, 1, 1, 1).expand(B, L, H, W).clone().requires_grad_(True) for x in kb]
    maps = _maps64(depth, k, poses)
    loss = sum((m * g.double()).sum() for m, g in zip(maps, ups) if g is not None)
    t = [x.abs().sum((1, 2, 3)) for x in torch.autograd.grad(loss, k, allow_unused=True, materialize_grads=True)]
    s = torch.zeros(B, 4, 4, dtype=torch.float64, device=depth.device)
    s[:, 0, 0] = (t[1] * cx.abs() + t[0]) / ex ** 2
    s[:, 0, 2] = t[1] / ex
    s[:, 1, 1] = (t[3] * cy.abs() + t[2]) / ey ** 2
    s[:, 1, 2] = t[3] / ey
    return s


@pytest.fixture
def k1_calls(monkeypatch):
    """Records (depth (B,L,H,W), K, poses, upstream gradients) of every K1 backward call."""
    from gradslam_b200.structures import rgbdimages

    calls = []
    orig = rgbdimages._BackprojectFn.backward

    def backward(ctx, *g):
        d, d_bs, K, P, (B, L, H, W) = ctx.saved
        depth = torch.as_strided(d, (B, L, H, W), (d_bs, H * W, W, 1)).clone()
        calls.append((depth, K.clone(), None if P is None else P.clone(),
                      [None if x is None else x.detach().clone() for x in g]))
        return orig(ctx, *g)

    monkeypatch.setattr(rgbdimages._BackprojectFn, "backward", staticmethod(backward))
    return calls


def _scale_of(calls, B):
    s = torch.zeros(B, 4, 4, dtype=torch.float64)
    for depth, K, P, ups in calls:
        s += _term_scale(depth, K, P, ups).cpu()
    return s


def _check(got, want, scale, rel):
    """got, want (B,1,4,4); scale (B,4,4).  Entries K1 never reads are exactly 0.  Where the terms of an axis cancel
    exactly (a normal that does not depend on fy), float32 leaves rounding residue of the other axis's size: fx and fy
    (cx and cy) share a unit, so each entry's tolerance is at least 1e-2 of its partner's."""
    got = got.detach().cpu().reshape(-1, 4, 4)
    want = want.detach().cpu().reshape(-1, 4, 4).to(got.dtype)
    assert torch.isfinite(got).all()
    mask = torch.zeros(4, 4, dtype=torch.bool)
    for i, j in READ:
        mask[i, j] = True
    assert (got[:, ~mask] == 0).all()
    err = (got - want).abs().double()
    partner = torch.zeros_like(scale)
    for (i, j), (p, q) in zip(READ, [(1, 1), (1, 2), (0, 0), (0, 2)]):
        partner[:, i, j] = scale[:, p, q]
    tol = rel * (scale + 1e-2 * partner) + 1e-30
    assert (err[:, mask] <= tol[:, mask]).all(), (got, want, scale)


# ----------------------------------------------------------------------------------------------------- K1 backward
@pytest.mark.parametrize("which", ["all", "vertex", "normal", "gvertex", "gnormal"])
@pytest.mark.parametrize("shape", [(2, 2, 24, 40), (1, 1, 17, 23), (1, 3, 2, 2), "cameras"])
def test_k1_intrinsics_gradient_matches_oracle_autograd(shape, which):
    """Every upstream map alone and all four, holes, the last row and column (17x23 and 2x2 are all edge), L > 1
    sharing one K, B > 1 with a camera per element (skew and a 4th column, which K1 never reads)."""
    import gradslam_b200 as gs

    if shape == "cameras":
        B, L, H, W = 3, 2, 24, 40
        rgb, depth, K, poses = camera_inputs(B, L, H, W, 21, skew=0.75, lattice_holes=True)
    else:
        B, L, H, W = shape
        rgb, depth, K, poses = make_sequence(B, L, H, W, seed=21)
    g = torch.Generator().manual_seed(3)
    names = ["vertex", "normal", "gvertex", "gnormal"]
    ups = [torch.randn(B, L, H, W, 3, generator=g) if which in ("all", n) else None for n in names]

    K_ref = K.clone().requires_grad_(True)
    m = oracle.frame_maps(depth, K_ref, poses)
    sum((m[n] * u).sum() for n, u in zip(names, ups) if u is not None).backward()

    K_gpu = K.to(DEV).requires_grad_(True)
    fr = gs.RGBDImages(rgb.to(DEV), depth.to(DEV), K_gpu, poses.to(DEV))
    outs = (fr.vertex_map, fr.normal_map, fr.global_vertex_map, fr.global_normal_map)
    sum((o * u.to(DEV)).sum() for o, u in zip(outs, ups) if u is not None).backward()

    assert K_gpu.grad.shape == K.shape
    scale = _term_scale(depth[..., 0], K, poses, ups)
    assert (scale[:, 0, 0] > 0).all() and (scale[:, 1, 1] > 0).all()
    _check(K_gpu.grad, K_ref.grad, scale, 1e-4)


def test_k1_depth_and_pose_gradients_unchanged_when_intrinsics_require_grad():
    """The kWantK instantiation computes g_depth and g_poses with the same arithmetic: bit for bit."""
    import gradslam_b200 as gs

    B, L, H, W = 2, 2, 48, 64
    rgb, depth, K, poses = make_sequence(B, L, H, W, seed=23)
    g = torch.Generator().manual_seed(4)
    ups = [torch.randn(B, L, H, W, 3, generator=g).to(DEV) for _ in range(4)]
    grads = []
    for k_grad in (False, True):
        d = depth.to(DEV).requires_grad_(True)
        p = poses.to(DEV).requires_grad_(True)
        k = K.to(DEV).requires_grad_(k_grad)
        fr = gs.RGBDImages(rgb.to(DEV), d, k, p)
        outs = (fr.vertex_map, fr.normal_map, fr.global_vertex_map, fr.global_normal_map)
        sum((o * u).sum() for o, u in zip(outs, ups)).backward()
        assert (k.grad is not None) == k_grad
        grads.append((d.grad, p.grad))
    assert torch.equal(grads[0][0], grads[1][0]) and torch.equal(grads[0][1], grads[1][1])


def test_k1_intrinsics_gradient_with_only_k_requiring_grad_and_no_poses():
    import gradslam_b200 as gs

    rgb, depth, K, _ = make_sequence(2, 1, 20, 28, seed=24)
    w = torch.randn(2, 1, 20, 28, 3, generator=torch.Generator().manual_seed(6))
    K_ref = K.clone().requires_grad_(True)
    (oracle.frame_maps(depth, K_ref)["vertex"] * w).sum().backward()
    K_gpu = K.to(DEV).requires_grad_(True)
    (gs.RGBDImages(rgb.to(DEV), depth.to(DEV), K_gpu).vertex_map * w.to(DEV)).sum().backward()
    _check(K_gpu.grad, K_ref.grad, _term_scale(depth[..., 0], K, None, [w, None, None, None]), 1e-4)


# ------------------------------------------------------------------------------------------ PointFusion and ICPSLAM
@pytest.mark.parametrize("B,L,cameras", [(1, 2, False), (2, 3, False), (3, 2, True)], ids=["1-2", "2-3", "cameras"])
def test_pointfusion_intrinsics_gradient_matches_oracle_autograd(B, L, cameras, k1_calls):
    import gradslam_b200 as gs

    H, W = 24, 32
    if cameras:
        rgb, depth, K, poses = camera_inputs(B, L, H, W, 41, skew=0.75, lattice_holes=True)
    else:
        rgb, depth, K, poses = make_sequence(B, L, H, W, seed=41, yaw0=0.6)
    K_ref = K.clone().requires_grad_(True)
    ref = oracle.run_slam(rgb, depth, K_ref, poses, odom="gt")
    counts = ref.map.counts()
    g = torch.Generator().manual_seed(5)
    ws = [[torch.randn(n, c, generator=g) for c in (3, 3, 1)] for n in counts]
    sum((t * w).sum() for b in range(B)
        for t, w in zip((ref.map.points[b], ref.map.colors[b], ref.map.ccounts[b]), ws[b])).backward()

    K_gpu = K.to(DEV).requires_grad_(True)
    pc, _ = gs.PointFusion(odom="gt", device=DEV)(gs.RGBDImages(rgb.to(DEV), depth.to(DEV), K_gpu, poses.to(DEV)))
    assert pc.num_points_per_pointcloud.tolist() == counts
    sum((t * w.to(DEV)).sum() for b in range(B)
        for t, w in zip((pc.points_list[b], pc.colors_list[b], pc.features_list[b]), ws[b])).backward()
    _check(K_gpu.grad, K_ref.grad, _scale_of(k1_calls, B), 1e-4)

    # only K requires grad: the map equals the fused no-grad run bit for bit
    with torch.no_grad():
        pc2, _ = gs.PointFusion(odom="gt", device=DEV)(gs.RGBDImages(rgb.to(DEV), depth.to(DEV), K.to(DEV),
                                                                     poses.to(DEV)))
    for b in range(B):
        assert torch.equal(pc2.points_list[b], pc.points_list[b].detach())
        assert torch.equal(pc2.normals_list[b], pc.normals_list[b].detach())
        assert torch.equal(pc2.features_list[b], pc.features_list[b].detach())


@pytest.mark.parametrize("association", ["nn", "projective"])
@pytest.mark.parametrize("odom", ["icp", "gradicp"])
def test_icpslam_intrinsics_gradient_matches_oracle_autograd(odom, association, k1_calls):
    """d(poses)/dK through the live points (K1) and the aggregated map, with only K requiring grad; the poses and the
    map equal the fused no-grad run bit for bit."""
    import gradslam_b200 as gs

    B, L, H, W = 1, 3, 32, 40
    rgb, depth, K, poses = make_sequence(B, L, H, W, seed=33, yaw0=0.6)
    w = torch.randn(B, L, 4, 4, generator=torch.Generator().manual_seed(2))
    K_ref = K.clone().requires_grad_(True)
    run = oracle.run_slam if association == "nn" else po.run_slam
    ref = run(rgb, depth, K_ref, poses, mode="aggregate", odom=odom, numiters=3, dsratio=2)
    (ref.poses * w).sum().backward()

    K_gpu = K.to(DEV).requires_grad_(True)
    slam = gs.ICPSLAM(odom=odom, association=association, numiters=3, dsratio=2, device=DEV)
    pc, rec = slam(gs.RGBDImages(rgb.to(DEV), depth.to(DEV), K_gpu, poses.to(DEV)))
    assert rec.requires_grad
    torch.testing.assert_close(rec.detach().cpu(), ref.poses.detach(), rtol=0, atol=1e-4)
    (rec * w.to(DEV)).sum().backward()
    assert K_ref.grad[0, 0, 0, 0] != 0
    _check(K_gpu.grad, K_ref.grad, _scale_of(k1_calls, B), 5e-3)

    with torch.no_grad():
        pc2, rec2 = slam(gs.RGBDImages(rgb.to(DEV), depth.to(DEV), K.to(DEV), poses.to(DEV)))
    assert torch.equal(rec2, rec.detach())
    assert torch.equal(pc2.points_list[0], pc.points_list[0].detach())


def test_icpslam_intrinsics_gradient_matches_reference_fixture():
    """The reference's own d/dK (random holes, as recorded) - the case of tests/golden/make_golden_grad_intrinsics.py."""
    import gradslam_b200 as gs

    ref = np.load(os.path.join(GOLD, "ref_grad_intrinsics.npz"))
    rgb, depth, K, poses = _make_sequence(1, 2, 32, 40, seed=17, yaw0=0.6)
    K_gpu = K.to(DEV).requires_grad_(True)
    _, rec = gs.ICPSLAM(odom="gradicp", numiters=3, dsratio=2, device=DEV)(
        gs.RGBDImages(rgb.to(DEV), depth.to(DEV), K_gpu, poses.to(DEV)))
    torch.testing.assert_close(rec.detach().cpu(), torch.from_numpy(ref["icpslam/poses"]), rtol=0, atol=1e-4)
    w = torch.randn(rec.shape, generator=torch.Generator().manual_seed(9))
    (rec * w.to(DEV)).sum().backward()
    want = torch.from_numpy(ref["icpslam/d_K"])
    torch.testing.assert_close(K_gpu.grad.cpu(), want, rtol=5e-2, atol=5e-2 * want.abs().max().item())


def test_pointfusion_intrinsics_gradient_matches_reference_fixture():
    import gradslam_b200 as gs

    ref = np.load(os.path.join(GOLD, "ref_grad_intrinsics.npz"))
    rgb, depth, K, poses = _make_sequence(1, 2, 24, 32, seed=41, yaw0=0.6)
    K_gpu = K.to(DEV).requires_grad_(True)
    pc, _ = gs.PointFusion(odom="gt", device=DEV)(gs.RGBDImages(rgb.to(DEV), depth.to(DEV), K_gpu, poses.to(DEV)))
    n = int(pc.num_points_per_pointcloud[0])
    assert n == int(ref["pf_gt/count"][0])
    g = torch.Generator().manual_seed(5)
    wp, wc, wf = torch.randn(n, 3, generator=g), torch.randn(n, 3, generator=g), torch.randn(n, 1, generator=g)
    ((pc.points_list[0] * wp.to(DEV)).sum() + (pc.colors_list[0] * wc.to(DEV)).sum()
     + (pc.features_list[0] * wf.to(DEV)).sum()).backward()
    want = torch.from_numpy(ref["pf_gt/d_K"])
    torch.testing.assert_close(K_gpu.grad.cpu(), want, rtol=1e-3, atol=1e-3 * want.abs().max().item())


def test_icpslam_depth_gradient_unchanged_when_intrinsics_require_grad():
    import gradslam_b200 as gs

    rgb, depth, K, poses = make_sequence(1, 2, 32, 40, seed=33, yaw0=0.6)
    w = torch.randn(1, 2, 4, 4, generator=torch.Generator().manual_seed(2)).to(DEV)
    grads = []
    for k_grad in (False, True):
        d = depth.to(DEV).requires_grad_(True)
        k = K.to(DEV).requires_grad_(k_grad)
        _, rec = gs.ICPSLAM(odom="gradicp", numiters=3, dsratio=2, device=DEV)(
            gs.RGBDImages(rgb.to(DEV), d, k, poses.to(DEV)))
        (rec * w).sum().backward()
        grads.append((rec.detach(), d.grad))
    assert torch.equal(grads[0][0], grads[1][0]) and torch.equal(grads[0][1], grads[1][1])


# ------------------------------------------------------------------------- renderer (R3d) and projective ICP
def _splat_term_scale(pts, nrm, rp, poses, K, index, g_depth):
    """(B,4,4) float64: sum over the disk pixels of |each pixel's term| of d/dK, g t m / (m.d) (w, 1, h, 1)."""
    import splat_oracle as so

    pts, nrm, poses, K, g = pts.double(), nrm.double(), poses.double(), K.double().reshape(-1, 4, 4), g_depth.double()
    B, L, H, W = index.shape
    n = index.clamp(min=0).view(B, L * H * W)
    disk = torch.cat([so.is_disk(nrm, rp), torch.zeros((B, 1), dtype=torch.bool)], 1)
    won = (torch.gather(disk, 1, n).view(B, L, H, W) & (index >= 0)).double()
    gather = lambda t: torch.gather(torch.cat([t, t.new_zeros(B, 1, 3)], 1), 1,
                                    n.unsqueeze(-1).expand(B, L * H * W, 3)).view(B, L, H, W, 3)
    Tinv = torch.linalg.inv(poses)
    R, t = Tinv[..., :3, :3].view(B, L, 1, 1, 3, 3), Tinv[..., :3, 3].view(B, L, 1, 1, 3)
    q = (R @ gather(pts).unsqueeze(-1)).squeeze(-1) + t
    m = (R @ gather(nrm).unsqueeze(-1)).squeeze(-1)
    ex, ey, cx, cy = K[:, 0, 0] + 1e-6, K[:, 1, 1] + 1e-6, K[:, 0, 2], K[:, 1, 2]
    u = torch.arange(W, dtype=torch.float64).view(1, 1, 1, W)
    v = torch.arange(H, dtype=torch.float64).view(1, 1, H, 1)
    rx, ry = (u - cx.view(B, 1, 1, 1)) / ex.view(B, 1, 1, 1), (v - cy.view(B, 1, 1, 1)) / ey.view(B, 1, 1, 1)
    md = m[..., 0] * rx + m[..., 1] * ry + m[..., 2]
    md = torch.where(won > 0, md, torch.ones_like(md))
    tt = (m * q).sum(-1) / md
    tx, ty = (g[..., 0] * tt * m[..., 0] / md * won).abs(), (g[..., 0] * tt * m[..., 1] / md * won).abs()
    S = [(tx * u).sum((1, 2, 3)), tx.sum((1, 2, 3)), (ty * v).sum((1, 2, 3)), ty.sum((1, 2, 3))]
    s = torch.zeros(B, 4, 4, dtype=torch.float64)
    s[:, 0, 0] = (S[1] * cx.abs() + S[0]) / ex ** 2
    s[:, 0, 2] = S[1] / ex
    s[:, 1, 1] = (S[3] * cy.abs() + S[2]) / ey ** 2
    s[:, 1, 2] = S[3] / ey
    return s


@pytest.mark.parametrize("M", [0, 3])
def test_render_intrinsics_gradient_matches_oracle_autograd(M):
    """render_pointclouds d/dK: a disk pixel's depth through its ray (M >= 1); one-pixel rows give exactly 0 (M = 0).
    A camera per element, L = 4 views sharing it."""
    import gradslam_b200 as gs
    import splat_oracle as so
    from test_gpu_render_splat import _case, _padded, _pointclouds

    H, W = 48, 64
    smap, radii, K, poses = _case(4, seed=2)
    pts, nrm, col, cc, rp = _padded(smap, radii)
    index = so.splat_index(pts, nrm, rp, smap.counts(), poses, K, H, W, M)
    g = torch.Generator().manual_seed(4)
    ups = [torch.randn(3, 4, H, W, c, generator=g) for c in (1, 3, 3, 1)]
    if M:  # grazing rays: dt/dd = -t m/(m.d) is ill-conditioned in float32 there (see test_gpu_render_splat.py)
        graze = so.disk_ray_cosine(nrm, rp, poses, K, index).abs() < 0.1
        ups = [torch.where(graze.unsqueeze(-1), torch.zeros_like(u), u) for u in ups]

    K_ref = K.clone().requires_grad_(True)
    ref = so.splat_values(pts.double(), nrm.double(), col.double(), cc.double(), rp, poses.double(), K_ref, index)
    sum((o * u.double()).sum() for o, u in zip((ref.depth, ref.rgb, ref.normals, ref.confidence), ups)).backward()

    K_gpu = K.view(-1, 1, 4, 4).to(DEV).requires_grad_(True)
    out = gs.render_pointclouds(_pointclouds(gs, smap, radii), K_gpu, poses.to(DEV), H, W, max_splat_px=M)
    if M:  # (splat_index is the disk rule; at M = 0 the engine draws one pixel per row)
        assert torch.equal(out.index.cpu(), index)
    sum((o * u.to(DEV)).sum() for o, u in zip((out.depth, out.rgb, out.normals, out.confidence), ups)).backward()
    assert K_gpu.grad.shape == (3, 1, 4, 4)
    if M == 0:
        assert (K_gpu.grad == 0).all()  # (the oracle's splat_values treats every disk row as a disk at any M)
        return
    scale = _splat_term_scale(pts, nrm, rp, poses, K, index, ups[0])
    assert scale[:, 0, 0].sum() > 0  # (an element whose pixels no disk won gets exactly 0)
    _check(K_gpu.grad, K_ref.grad, scale, 1e-4)


@pytest.mark.parametrize("M,w", [(0, 0.0), (3, 0.0), (0, 0.1), (3, 0.1)])
def test_projective_localisation_intrinsics_gradient_matches_oracle_autograd(M, w):
    """d(pose)/dK of the taped projective gradICP step: the live points (K1), the splatted targets' disk depths and
    surface points (R3d, K1) and the photometric row (every entry of K's first three rows), against autograd of the
    oracle; the other gradients are unchanged bit for bit when K also requires grad."""
    import gradslam_b200 as gs
    import photometric_oracle as ph
    import radii_oracle as ro
    from gradslam_b200.synthetic import make_textured_sequence
    from test_gpu_projective_icp import _icp_kwargs

    B, H, W = 1, 32, 40
    rgb, depth, K, poses = make_textured_sequence(B, 2, H, W, seed=33, yaw0=0.6, hole_fraction=0.0)
    depth = punch_lattice_holes(depth)
    m0 = oracle.frame_maps(depth[:, :1], K, poses[:, :1])
    valid = m0["valid"][0, 0]
    P0, N0, C0 = m0["gvertex"][0, 0][valid], m0["gnormal"][0, 0][valid], rgb[0, 0][valid]
    R0 = ro.radius_image(depth[:, :1], m0, K)[0][valid].unsqueeze(1)
    wts = torch.randn(4, 4, generator=torch.Generator().manual_seed(2))

    K_ref = K.clone().requires_grad_(True)
    at_prev = oracle.frame_maps(depth[:, 1:2], K_ref, poses[:, :1])
    ref = ph.odometry(oracle.SurfelMap([P0], [N0], [C0]), [R0], at_prev, rgb[:, 1:2], poses[:, 0], K_ref[:, 0], H, W,
                      "gradicp", 2, _icp_kwargs("gradicp", 3, None), M, w)
    (ref[0] * wts).sum().backward()

    slam = gs.ICPSLAM(odom="gradicp", association="projective", numiters=3, dsratio=2, target_splat_px=M,
                      photometric_weight=w, device=DEV)

    def run(k_grad, d_grad):
        pc = gs.Pointclouds(points=P0[None].to(DEV), normals=N0[None].to(DEV), colors=C0[None].to(DEV))
        pc.radii_list = [R0.to(DEV)]
        k = K.to(DEV).requires_grad_(k_grad)
        d = depth[:, 1:2].to(DEV).requires_grad_(d_grad)
        prev_p = poses[:, 0:1].to(DEV).requires_grad_(d_grad)
        live = gs.RGBDImages(rgb[:, 1:2].to(DEV), d, k, poses[:, 1:2].to(DEV))
        prev = gs.RGBDImages(rgb[:, 0:1].to(DEV), depth[:, 0:1].to(DEV), k, prev_p)
        out = slam._localize(pc, live, prev)
        if out.requires_grad:
            (out[0, 0] * wts.to(DEV)).sum().backward()
        return out.detach(), k.grad, d.grad, prev_p.grad

    out, g_K, _, _ = run(True, False)
    torch.testing.assert_close(out[:, 0].cpu(), ref.detach(), rtol=0, atol=1e-4)
    want = K_ref.grad
    assert (g_K[..., 3, :] == 0).all()
    if w == 0:  # K's skew and 4th column are read by the photometric row only
        assert (g_K[..., 0, 1] == 0).all() and (g_K[..., :3, 3] == 0).all()
    assert torch.isfinite(g_K).all() and want.abs().max() > 0
    torch.testing.assert_close(g_K.cpu(), want, rtol=5e-2, atol=5e-3 * want.abs().max().item())
    # only K requires grad: the taped poses equal the fused call's bit for bit
    fused, _, _, _ = run(False, False)
    assert torch.equal(out, fused)
    # d/d depth and d/d previous pose do not change when K also requires grad
    _, _, gd0, gp0 = run(False, True)
    _, _, gd1, gp1 = run(True, True)
    assert torch.equal(gd0, gd1) and torch.equal(gp0, gp1)
