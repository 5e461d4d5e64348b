"""The Huber-weighted normal-equation ops (huber= of _JointNormalEqBatchedFn: k_icp_joint_linearize_idx<true>,
k_icp_joint_linearize_bwd<kWantK, true>; huber_delta of _NormalEqBatchedFn: k_icp_linearize_idx<true>,
k_icp_linearize_bwd<true>) called directly, against the float64 reference of tests/joint_normal_eq_reference.py at
finite scales within its derived float32 bounds: hundreds of blocks, a ragged batch with a camera per element,
residuals exactly on the scale and one float32 step inside it, the identities, determinism, the benchmark's size, and
the differentiable mode end to end against autograd of robust_oracle.  The scales are the float32 medians of the
residuals, so both branches carry rows.  Each bound check prints its largest error-to-bound ratio."""
import math

import numpy as np
import pytest
import torch

import gsx_oracle as oracle
import joint_normal_eq_reference as jr
import robust_oracle as ro
from cameras import camera_inputs
from test_gpu_joint_normal_eq import GRADS, PER_ROW, SIZES, W_TRACK, _check, _elements, _far_outside, _run

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
INF = math.inf


def _residuals(x, idx, index, H, W):
    return jr.float32_residuals(*(x[k] for k in jr.NAMES[:5]), idx, index, H, W)


def _medians(x, idx, index, H, W):
    r, rp, _ = _residuals(x, idx, index, H, W)
    return float(r.abs().median()), float(rp.abs().median())


def _cases(d, dp):
    return [(d, INF), (INF, dp), (d, dp)]


def _geometric(els, g, delta):
    """_NormalEqBatchedFn at delta on the geometric inputs of elements (x, idx, index) -> (sums, g_src, g_tgt, g_tgt_n)
    on the CPU."""
    from gradslam_b200.odometry.icputils import _NormalEqBatchedFn

    sizes = [int(e[1].numel()) for e in els]
    Ns = max(sizes)
    src = torch.zeros(len(els), Ns, 3)
    idx = torch.full((len(els), Ns), -1, dtype=torch.int64)
    for b, (x, i, _) in enumerate(els):
        src[b, :i.numel()], idx[b, :i.numel()] = x["src"], i
    leaves = [t.to(DEV).requires_grad_(True) for t in
              (src, torch.stack([e[0]["tgt"] for e in els]), torch.stack([e[0]["tgt_n"] for e in els]))]
    sums = _NormalEqBatchedFn.apply(*leaves, idx.to(DEV), torch.tensor(sizes, dtype=torch.int32, device=DEV), delta)
    (sums * g.to(DEV)).sum().backward()
    return [sums.detach().cpu()] + [t.grad.cpu() for t in leaves]


# ------------------------------------------------------------------------------------------------------ a. many blocks
def test_many_blocks_robust_sums_and_gradients_within_float64_bounds():
    """ns = 2^17 + 37 rows (513 blocks, a partial last block) into 240 x 320 images with holes, at the median scales:
    half of the geometric and half of the photometric rows lie outside them."""
    H, W, ns = 240, 320, (1 << 17) + 37
    els = _elements([ns], H, W, seed=21)
    x, idx, index = els[0]
    r, rp, _ = _residuals(x, idx, index, H, W)
    d, dp = _medians(x, idx, index, H, W)
    assert float((r.abs() > d).double().mean()) >= 0.25 and float((rp.abs() > dp).double().mean()) >= 0.25
    g = torch.randn(1, 28, generator=torch.Generator().manual_seed(21))
    blocks = jr.blocks_of(ns)
    assert blocks == 513
    plain = jr.joint_sums(*(x[k].double() for k in jr.NAMES), idx, index, H, W, W_TRACK)
    for huber in _cases(d, dp):
        got = _run(els, H, W, W_TRACK, g, huber=huber)
        ref = jr.reference(x, idx, index, H, W, W_TRACK, blocks, g[0], *huber)
        _check(got, 0, ref, f"many-blocks-{huber}")
        # the bounds have teeth: the unweighted sums lie far outside them
        assert _far_outside(plain, ref), huber
    # the geometric op at delta on the same rows lies within the w = 0 reference's bounds
    ref = jr.reference(x, idx, index, H, W, 0.0, blocks, g[0], d, INF)
    sums, g_src, g_tgt, g_tn = _geometric(els, g, d)
    ratios = {}
    for name, got in (("sums", sums[0]), ("src", g_src[0]), ("tgt", g_tgt[0]), ("tgt_n", g_tn[0])):
        want, bound = (ref["sums"], ref["sum_bound"]) if name == "sums" else (ref["grad"][name], ref["grad_bound"][name])
        ok, ratios[name] = jr.within(got, want, bound)
        assert ok, (name, ratios)
    print("ERROR/BOUND", "many-blocks-geometric-op", {k: round(v, 4) for k, v in ratios.items()})


# ----------------------------------------------------------------------------- b. batched, ragged, a camera per element
def test_batched_ragged_robust_equals_each_element_alone_and_the_reference():
    H, W = 60, 80
    els = _elements(SIZES, H, W, seed=22, all_filtered=(2,))
    g = torch.randn(len(SIZES), 28, generator=torch.Generator().manual_seed(22))
    d, dp = _medians(*els[3], H, W)
    blocks = jr.blocks_of(max(SIZES))
    zero = lambda t: bool((t == 0).all())
    for huber in _cases(d, dp):
        got = _run(els, H, W, W_TRACK, g, pad_value=7.5, huber=huber)  # (padding rows hold garbage)
        for e, n in enumerate(SIZES):
            if n == 0 or e == 2:  # the empty and the all-filtered element: exactly zero sums and gradients
                assert zero(got["sums"][e]) and all(zero(got[k][e]) for k in GRADS), (huber, e)
                continue
            for k in PER_ROW:
                assert zero(got[k][e, n:]), (huber, e, k)
            one = _run([els[e]], H, W, W_TRACK, g[e:e + 1], huber=huber)
            assert torch.equal(one["sums"][0], got["sums"][e]), (huber, e)
            for k in PER_ROW:
                assert torch.equal(one[k][0], got[k][e, :n]), (huber, e, k)
            for k in ("prev", "K"):
                assert torch.equal(one[k][0], got[k][e]), (huber, e, k)
            for k in ("tgt", "tgt_n", "model_col"):  # index_add_: atomics in no fixed order
                torch.testing.assert_close(one[k][0], got[k][e], rtol=1e-5, atol=1e-6 * one[k][0].abs().max().item(),
                                           msg=f"{huber} {e} {k}")
        for e in (0, 3):
            x, idx, index = els[e]
            _check(got, e, jr.reference(x, idx, index, H, W, W_TRACK, blocks, g[e], *huber), f"ragged-{e}-{huber}")


# ------------------------------------------------------------------------------------ c. residuals exactly on the scale
def _bits(t):
    return [hex(v) for v in torch.as_tensor(t, dtype=torch.float32).reshape(-1).view(torch.int32).tolist()]


@pytest.mark.parametrize("sign", [1.0, -1.0])
@pytest.mark.parametrize("photometric", [False, True])
def test_a_residual_on_the_scale_is_inside_and_one_step_below_is_outside(photometric, sign):
    """An element with one associated row k.  delta (or delta_p) = float32 |r_k|: the op is the unweighted op bit for
    bit, sums and every gradient.  One float32 step below: the sums are the reference's float32 products of the
    outside branch bit for bit (slot 27 delta ((a + a) - delta), or w (delta_p ((a_p + a_p) - delta_p)), which rounds
    to the unweighted r r there: (a - u)(a + u) = a^2 - u^2), the weighted slots differ from the unweighted ones (h is
    1 - 2^-24 or 1 - 2^-23; a product may round back), and the gradients, whose outside branch differs from the inside
    one well beyond rounding, lie within the bounds.  The photometric case zeroes the target normal at the row's pixel,
    so that its geometric row adds exact zeros."""
    H, W = 60, 80
    (x, idx, index), = _elements([600], H, W, seed=23)
    r, rp, vj = _residuals(x, idx, index, H, W)
    rows = torch.nonzero(idx >= 0)[:, 0]
    res = torch.zeros_like(r)
    res[vj] = rp
    if photometric:
        ok = vj & (torch.sign(res) == sign) & (res.abs() > 0.01)
    else:
        res = r
        ok = ~vj & (torch.sign(r) == sign) & (r.abs() > 1e-4)
    k = int(torch.nonzero(ok)[0, 0])
    row, a = int(rows[k]), float(res[k].abs())
    one = torch.full_like(idx, -1)
    one[row] = idx[row]
    if photometric:
        x = dict(x, tgt_n=x["tgt_n"].clone())
        x["tgt_n"][idx[row]] = 0.0
    els = [(x, one, index)]
    below = float(np.nextafter(np.float32(a), np.float32(0)))
    scale = (lambda s: (INF, s)) if photometric else (lambda s: (s, INF))
    g = torch.randn(1, 28, generator=torch.Generator().manual_seed(23))
    plain, tie, out = (_run(els, H, W, W_TRACK, g, huber=h) for h in ((INF, INF), scale(a), scale(below)))
    mx = {n: v.abs() for n, v in x.items()}
    products = lambda h: jr._pair_rows(x, mx, one, index, H, W, W_TRACK, delta=h[0], delta_p=h[1])[0][:, 0]
    msg = dict(residual=_bits(res[k]), scale=_bits(a), plain=_bits(plain["sums"][0][27]), tie=_bits(tie["sums"][0][27]))
    assert torch.equal(plain["sums"][0], products((INF, INF))), msg
    assert torch.equal(tie["sums"][0], plain["sums"][0]), msg
    for name in GRADS:
        assert torch.equal(tie[name], plain[name]), (name, msg)
    assert torch.equal(out["sums"][0], products(scale(below))), msg
    nz = plain["sums"][0][:27] != 0
    assert int(nz.sum()) >= 20 and int(((out["sums"][0][:27] != plain["sums"][0][:27]) & nz).sum()) >= int(nz.sum()) - 2
    ref = jr.reference(x, one, index, H, W, W_TRACK, jr.blocks_of(600), g[0], *scale(below))
    _check(out, 0, ref, f"on-the-scale-{'photometric' if photometric else 'geometric'}-{sign:+.0f}")
    name = "src_col" if photometric else "src"
    assert not torch.equal(out[name], plain[name])


# ------------------------------------------------------------------------------------------------------- d. identities
def test_zero_weight_robust_is_the_geometric_op_and_photometric_gradients_vanish():
    H, W = 45, 62
    els = _elements([5000, 777, 2], H, W, seed=24)
    g = torch.randn(3, 28, generator=torch.Generator().manual_seed(24))
    d, dp = _medians(*els[0], H, W)
    got = _run(els, H, W, 0.0, g, huber=(d, dp))
    sums, g_src, _, _ = _geometric(els, g, d)
    assert torch.equal(got["sums"], sums)
    assert torch.equal(got["src"], g_src)
    for k in ("src_col", "model_col", "prev", "K"):
        assert bool((got[k] == 0).all()), k
    # and the scale changes the geometric sums
    assert not torch.equal(_geometric(els, g, INF)[0][:2], sums[:2])


def test_intrinsics_instantiation_leaves_the_robust_gradients_unchanged():
    H, W = 48, 64
    els = _elements([4000, 2500], H, W, seed=25)
    g = torch.randn(2, 28, generator=torch.Generator().manual_seed(25))
    huber = _medians(*els[0], H, W)
    with_k = _run(els, H, W, W_TRACK, g, k_grad=True, huber=huber)
    without = _run(els, H, W, W_TRACK, g, k_grad=False, huber=huber)
    assert without["K"] is None
    assert torch.equal(with_k["sums"], without["sums"])
    for k in ("src", "src_col", "prev"):
        assert torch.equal(with_k[k], without[k]), k
    for k in ("tgt", "tgt_n", "model_col"):
        torch.testing.assert_close(with_k[k], without[k], rtol=1e-5, atol=1e-6 * with_k[k].abs().max().item())
    assert bool((with_k["K"][:, 3] == 0).all())
    assert bool((with_k["K"][:, 0, 1] != 0).all()) and bool((with_k["K"][:, :3, 3] != 0).all())


# ---------------------------------------------------------------------------------------------------- e. determinism
def test_robust_backwards_are_deterministic():
    """Two launches of each backward at finite scales give every output bit for bit (fixed-order reductions)."""
    from gradslam_b200 import _C

    H, W = 60, 80
    els = _elements([70001, 3000], H, W, seed=26)
    d, dp = _medians(*els[0], H, W)
    B, Ns = 2, 70001
    src = torch.zeros(B, Ns, 3)
    col = torch.zeros(B, Ns, 3)
    idx = torch.full((B, Ns), -1, dtype=torch.int64)
    for b, (x, i, _) in enumerate(els):
        src[b, :i.numel()], col[b, :i.numel()], idx[b, :i.numel()] = x["src"], x["src_col"], i
    dv = lambda t: t.contiguous().to(DEV)
    stack = lambda k: dv(torch.stack([e[0][k] for e in els]))
    counts = torch.tensor([70001, 3000], dtype=torch.int32, device=DEV)
    g = dv(torch.randn(B, 28, generator=torch.Generator().manual_seed(26)))
    args = (dv(src), counts, Ns, dv(col), stack("tgt"), stack("tgt_n"), stack("model_col"),
            dv(torch.stack([e[2] for e in els])), B, H, W, dv(idx), stack("prev"), stack("K"), W_TRACK, g)
    nbytes = _C.lib().gsx_icp_joint_normal_eq_batched_bwd_scratch_bytes(B, Ns)
    P = H * W
    runs = {"joint": [], "geometric": []}
    for _ in range(2):
        o = [torch.full((B, Ns, 3), float("nan"), device=DEV) for _ in range(4)]
        o += [torch.full((B, Ns, 5, 3), float("nan"), device=DEV), torch.full((B, 4, 4), float("nan"), device=DEV),
              torch.full((B, 4, 4), float("nan"), device=DEV)]
        scratch = torch.empty(nbytes, dtype=torch.uint8, device=DEV)
        _C.launch("gsx_icp_joint_normal_eq_batched_bwd", *args, *o, scratch, nbytes, d, dp)
        runs["joint"].append([t.cpu() for t in o])
        o = [torch.full((B, Ns, 3), float("nan"), device=DEV) for _ in range(3)]
        _C.launch("gsx_icp_normal_eq_batched_bwd", dv(src), counts, Ns, stack("tgt"), stack("tgt_n"), P, B, dv(idx), g,
                  *o, d)
        runs["geometric"].append([t.cpu() for t in o])
    for name, (a, b) in runs.items():
        for u, v in zip(a, b):
            assert bool(torch.isfinite(u).all()), name
            assert torch.equal(u.view(torch.int32), v.view(torch.int32)), name


# ------------------------------------------------------------------------------------------------ f. benchmark size
@pytest.fixture
def robust_joint_calls(monkeypatch):
    """Keeps the inputs of the last forward call of _JointNormalEqBatchedFn, its Huber scales included."""
    from gradslam_b200.odometry import icputils

    last = {}
    orig = icputils._JointNormalEqBatchedFn.forward

    def forward(ctx, src, src_col, tgt, tgt_n, model_col, prev, idx, index, src_counts, K, w, H, W,
                huber=(math.inf, math.inf)):
        last.clear()
        last.update(src=src.detach().clone(), src_col=src_col.detach().clone(), tgt=tgt.detach().clone(),
                    tgt_n=tgt_n.detach().clone(), model_col=model_col.detach().clone(), prev=prev.detach().clone(),
                    idx=idx.clone(), index=index.clone(), counts=src_counts.clone(), K=K.detach().clone(), w=w, H=H,
                    W=W, huber=tuple(float(d) for d in huber))
        return orig(ctx, src, src_col, tgt, tgt_n, model_col, prev, idx, index, src_counts, K, w, H, W, huber)

    monkeypatch.setattr(icputils._JointNormalEqBatchedFn, "forward", staticmethod(forward))
    return last


@pytest.mark.parametrize("M", [0, 3])
def test_benchmark_size_robust_taped_poses_equal_fused_and_the_op_matches_the_reference(M, robust_joint_calls):
    """B = 8, 640 x 480, ds = 1, the textured scene at W_TRACK with huber_delta = 0.02 and photometric_huber_delta =
    0.05: the differentiable mode's poses equal the fused call's bit for bit, and the last joint op it ran, re-run on
    its recorded inputs at its scales and at the medians of its residuals, matches the reference for elements 0 and 7."""
    import gradslam_b200 as gs
    from gradslam_b200.synthetic import make_textured_sequence

    B, L, H, W = 8, 3, 480, 640
    rgb, depth, K, poses = make_textured_sequence(B, L, H, W, seed=5, yaw0=0.3)
    frames = gs.RGBDImages(rgb.to(DEV), depth.to(DEV), K.to(DEV), poses.to(DEV))
    pc, _ = gs.PointFusion(odom="gt", surfel_radii=True, device=DEV)(frames[:, :2])
    slam = gs.PointFusion(odom="gradicp", association="projective", dsratio=1, surfel_radii=True, target_splat_px=M,
                          photometric_weight=W_TRACK, huber_delta=0.02, photometric_huber_delta=0.05, device=DEV)
    fused = slam._localize(pc, frames[:, 2], frames[:, 1])
    live = gs.RGBDImages(rgb[:, 2:3].to(DEV).requires_grad_(True), depth[:, 2:3].to(DEV).requires_grad_(True),
                         K.to(DEV), poses[:, 2:3].to(DEV))
    taped = slam._localize(pc, live, frames[:, 1])
    assert taped.requires_grad
    assert torch.equal(taped.detach(), fused)

    rec = dict(robust_joint_calls)
    assert jr.scales(*rec["huber"]) == jr.scales(0.02, 0.05)
    counts = rec["counts"].cpu().tolist()
    assert min(counts) > 1100 * jr.BLOCK
    Ns = rec["src"].shape[1]
    els = []
    for b in range(B):
        n = counts[b]
        x = {"src": rec["src"][b, :n], "src_col": rec["src_col"][b, :n], "tgt": rec["tgt"][b], "tgt_n": rec["tgt_n"][b],
             "model_col": rec["model_col"][b], "prev": rec["prev"].reshape(B, 4, 4)[b],
             "K": rec["K"].reshape(B, 4, 4)[b]}
        els.append(({k: v.float().cpu() for k, v in x.items()}, rec["idx"][b, :n].cpu(), rec["index"][b].cpu()))
    res = [_residuals(*e, H, W) for e in els]
    medians = (float(torch.cat([r[0] for r in res]).abs().median()), float(torch.cat([r[1] for r in res]).abs().median()))
    g = torch.randn(B, 28, generator=torch.Generator().manual_seed(27))
    for what, huber in (("recorded", rec["huber"]), ("medians", medians)):
        got = _run(els, H, W, rec["w"], g, ns=Ns, huber=huber)
        for b in (0, 7):
            x, idx, index = els[b]
            assert int((idx >= 0).sum()) > 100_000
            r, rp, _ = res[b]
            print("OUTSIDE", what, huber, b, float((r.abs() > huber[0]).double().mean()),
                  float((rp.abs() > huber[1]).double().mean()))
            ref = jr.reference(x, idx, index, H, W, rec["w"], jr.blocks_of(Ns), g[b], *huber)
            _check(got, b, ref, f"benchmark-M{M}-{what}-element-{b}")


# ------------------------------------------------------------------------------------------- g. end to end, batched
def _slam_map(rgb, depth, K, poses):
    """Each element's frame 0 as its map: (oracle.SurfelMap, gs.Pointclouds)."""
    import gradslam_b200 as gs

    m0 = oracle.frame_maps(depth[:, :1], K, poses[:, :1])
    B = depth.shape[0]
    valid = [m0["valid"][b, 0] for b in range(B)]
    P = [m0["gvertex"][b, 0][valid[b]] for b in range(B)]
    N = [m0["gnormal"][b, 0][valid[b]] for b in range(B)]
    C = [rgb[b, 0][valid[b]] for b in range(B)]
    pc = gs.Pointclouds(points=[p.to(DEV) for p in P], normals=[n.to(DEV) for n in N], colors=[c.to(DEV) for c in C])
    return oracle.SurfelMap(P, N, C), pc


def _taped(pc, rgb, depth, K, poses, delta, extra):
    """ICPSLAM(odom='gradicp', huber_delta=delta) from frame 0 to frame 1 -> (poses (B,1,4,4), d_g leaf, K_g leaf)."""
    import gradslam_b200 as gs

    d_g = depth[:, 1:2].to(DEV).requires_grad_(True)
    K_g = K.to(DEV).requires_grad_(True)
    live = gs.RGBDImages(rgb[:, 1:2].to(DEV), d_g, K_g, poses[:, 1:2].to(DEV))
    prev = gs.RGBDImages(rgb[:, 0:1].to(DEV), depth[:, 0:1].to(DEV), K_g, poses[:, 0:1].to(DEV))
    slam = gs.ICPSLAM(odom="gradicp", numiters=3, dsratio=2, huber_delta=delta, device=DEV, **extra)
    return slam._localize(pc, live, prev), d_g, K_g


@pytest.mark.parametrize("assoc", ["nn", "projective"])
def test_batched_differentiable_mode_gradients_match_oracle_autograd(assoc):
    """B = 3 with a camera per element, element 1 without live depth: d(pose)/d(live depth) and d/dK of
    ICPSLAM(odom='gradicp', huber_delta=...) against autograd of robust_oracle; the empty element keeps its previous
    pose with zero gradient, and each element's gradients are its B = 1 call's to float32 rounding."""
    from test_gpu_projective_icp import _icp_kwargs

    B, H, W = 3, 32, 40
    rgb, depth, K, poses = camera_inputs(B, 2, H, W, 31, skew=0.5, lattice_holes=True)
    depth[1, 1] = 0.0
    w = W_TRACK if assoc == "projective" else 0.0
    delta, delta_p = 0.003, 0.02
    extra = dict(association="projective", photometric_weight=w, photometric_huber_delta=delta_p) if w else {}
    wts = torch.randn(B, 4, 4, generator=torch.Generator().manual_seed(28))

    smap, pc = _slam_map(rgb, depth, K, poses)
    d_ref = depth[:, 1:2].clone().requires_grad_(True)
    K_ref = K.clone().requires_grad_(True)
    at_prev = oracle.frame_maps(d_ref, K_ref, poses[:, :1])
    kw = _icp_kwargs("gradicp", 3, None)
    if assoc == "nn":
        ref = ro.odometry_nn(smap, at_prev, poses[:, 0], K_ref[:, 0], H, W, "gradicp", 2, kw, delta)
    else:
        ref = ro.odometry_projective(smap, None, at_prev, rgb[:, 1:2], poses[:, 0], K_ref[:, 0], H, W, "gradicp", 2,
                                     kw, 0, w, delta, delta_p)
    (ref * wts).sum().backward()

    out, d_g, K_g = _taped(pc, rgb, depth, K, poses, delta, extra)
    torch.testing.assert_close(out[:, 0].detach().cpu(), ref.detach(), rtol=0, atol=1e-4)
    assert torch.equal(out[1, 0].detach().cpu(), poses[1, 0])
    (out[:, 0] * wts.to(DEV)).sum().backward()
    got = {"depth": d_g.grad.cpu(), "K": K_g.grad.cpu()}
    want = {"depth": d_ref.grad, "K": K_ref.grad}
    assert bool((got["depth"][1] == 0).all()) and bool((got["K"][1] == 0).all())
    for name in ("depth", "K"):
        assert torch.isfinite(got[name]).all(), name
        for b in (0, 2):
            assert want[name][b].abs().max() > 0, (name, b)
            torch.testing.assert_close(got[name][b], want[name][b], rtol=5e-2, atol=5e-3 * want[name][b].abs().max().item(),
                                       msg=f"{name} {b}")
    # each element alone
    for b in (0, 2):
        sl = slice(b, b + 1)
        _, pc_b = _slam_map(rgb[sl], depth[sl], K[sl], poses[sl])
        out_b, d_b, K_b = _taped(pc_b, rgb[sl], depth[sl], K[sl], poses[sl], delta, extra)
        torch.testing.assert_close(out_b.detach(), out[sl].detach(), rtol=0, atol=1e-6)
        (out_b[:, 0] * wts[sl].to(DEV)).sum().backward()
        for name, one in (("depth", d_b.grad.cpu()[0]), ("K", K_b.grad.cpu()[0])):
            torch.testing.assert_close(got[name][b], one, rtol=1e-4, atol=1e-5 * one.abs().max().item(),
                                       msg=f"alone {name} {b}")
