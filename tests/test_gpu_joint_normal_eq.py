"""The joint geometric and photometric normal-equation op (_JointNormalEqBatchedFn: k_icp_joint_linearize_idx,
k_icp_joint_linearize_bwd<kWantK>, the fixed-order block reductions) called directly, against the float64 reference of
tests/joint_normal_eq_reference.py within its derived float32 bounds: hundreds of blocks, a ragged batch with a camera
per element, the image border and holes, the identities of w = 0 and of images without an interior pixel, and the
benchmark's size.  Each bound check prints its largest error-to-bound ratio."""
import math

import pytest
import torch

import gsx_oracle as oracle
import joint_normal_eq_reference as jr
from cameras import camera_intrinsics

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
W_TRACK = 0.1  # (test_photometric_oracle.W_TRACK)
GRADS = ("src", "src_col", "tgt", "tgt_n", "model_col", "prev", "K")
PER_ROW = ("src", "src_col")  # written per row by the kernel; the others are scattered (index_add_) or reduced


def _cameras(B, H, W, seed):
    """A camera per element: camera_intrinsics with skew and a 4th column, and a non-identity previous pose."""
    K = torch.from_numpy(camera_intrinsics(B, H, W, skew=0.75))
    g = torch.Generator().manual_seed(seed)
    prev = torch.stack([oracle.se3_exp((0.3 * torch.randn(6, generator=g)).float()).double() for _ in range(B)])
    return K, prev


def _elements(sizes, H, W, seed, all_filtered=()):
    K, prev = _cameras(len(sizes), H, W, seed)
    els = []
    for e, n in enumerate(sizes):
        x, idx, index = jr.synthetic_element(H, W, n, K[e], prev[e], seed * 100 + e)
        if e in all_filtered:
            idx[:] = -1
        els.append((x, idx, index))
    return els


def _run(els, H, W, w, g, k_grad=True, ns=None, pad_value=0.0, huber=(math.inf, math.inf)):
    """The op on a padded batch of elements (x, idx, index) with upstream gradient g (B, 28) at the Huber scales
    huber = (huber_delta, photometric_huber_delta).  Padding rows hold pad_value and idx -1.  -> dict of CPU tensors:
    "sums" (B, 28) and the gradient of every input."""
    from gradslam_b200.odometry.icputils import _JointNormalEqBatchedFn

    B = len(els)
    sizes = [int(e[1].numel()) for e in els]
    Ns = max(1, max(sizes)) if ns is None else ns
    src = torch.full((B, Ns, 3), pad_value)
    src_col = torch.full((B, Ns, 3), pad_value)
    idx = torch.full((B, Ns), -1, dtype=torch.int64)
    for b, ((x, i, _), n) in enumerate(zip(els, sizes)):
        src[b, :n], src_col[b, :n], idx[b, :n] = x["src"], x["src_col"], i
    stack = lambda k: torch.stack([e[0][k] for e in els])
    leaves = {"src": src, "src_col": src_col, "tgt": stack("tgt"), "tgt_n": stack("tgt_n"),
              "model_col": stack("model_col"), "prev": stack("prev"), "K": stack("K")}
    leaves = {k: v.to(DEV).requires_grad_(k != "K" or k_grad) for k, v in leaves.items()}
    index = torch.stack([e[2] for e in els]).to(DEV)
    counts = torch.tensor(sizes, dtype=torch.int32, device=DEV)
    sums = _JointNormalEqBatchedFn.apply(leaves["src"], leaves["src_col"], leaves["tgt"], leaves["tgt_n"],
                                         leaves["model_col"], leaves["prev"], idx.to(DEV), index, counts, leaves["K"],
                                         w, H, W, huber)
    (sums * g.to(DEV)).sum().backward()
    out = {"sums": sums.detach().cpu()}
    for k, v in leaves.items():
        out[k] = None if v.grad is None else v.grad.cpu()
    return out


def _check(got, b, ref, what):
    """Element b of the op's outputs within the reference's bounds; prints the largest error-to-bound ratios."""
    ratios = {}
    ok, ratios["sums"] = jr.within(got["sums"][b], ref["sums"], ref["sum_bound"])
    assert ok, (what, "sums", ratios)
    for name in GRADS:
        g = got[name][b]
        if name in PER_ROW:
            g = g[:ref["grad"][name].shape[0]]
        ok, ratios[name] = jr.within(g, ref["grad"][name], ref["grad_bound"][name])
        assert ok, (what, name, ratios)
    print("ERROR/BOUND", what, {k: round(v, 4) for k, v in ratios.items()})
    return ratios


def _far_outside(want, ref, bound_key="sum_bound", value_key="sums", factor=10.0):
    return float(((want - ref[value_key]).abs() / (ref[bound_key] + 1e-300)).max()) > factor


# ------------------------------------------------------------------------------------------------------ a. many blocks
def test_many_blocks_sums_and_gradients_within_float64_bounds():
    """ns = 2^17 + 37 rows: 513 blocks, a partial last block, into 240 x 320 target images with holes; the associated
    pixels include every covered pixel of the two outer rows and columns of each side and pixels next to holes."""
    H, W, ns = 240, 320, (1 << 17) + 37
    (x, idx, index), = _elements([ns], H, W, seed=11)
    assert 0.15 < float((idx < 0).double().mean()) < 0.25
    g = torch.randn(1, 28, generator=torch.Generator().manual_seed(1))
    got = _run([(x, idx, index)], H, W, W_TRACK, g)
    blocks = jr.blocks_of(ns)
    assert blocks == 513
    ref = jr.reference(x, idx, index, H, W, W_TRACK, blocks, g[0])
    _check(got, 0, ref, "many-blocks")
    # the bounds have teeth: without the last block's 37 rows the reference lies far outside them
    cut = idx.clone()
    cut[(ns // jr.BLOCK) * jr.BLOCK:] = -1
    ref_cut = jr.reference(x, cut, index, H, W, W_TRACK, blocks, g[0])
    assert _far_outside(ref_cut["sums"], ref, factor=4.0)


# ----------------------------------------------------------------------------- b. batched, ragged, a camera per element
SIZES = [3000, 0, (1 << 15) + 5, 70001, 1]


def test_batched_ragged_equals_each_element_alone_and_the_reference():
    H, W = 60, 80
    els = _elements(SIZES, H, W, seed=12, all_filtered=(2,))
    g = torch.randn(len(SIZES), 28, generator=torch.Generator().manual_seed(2))
    got = _run(els, H, W, W_TRACK, g, pad_value=7.5)  # (padding rows hold garbage the kernels must not read)
    zero = lambda t: bool((t == 0).all())
    for e, n in enumerate(SIZES):
        if n == 0 or e == 2:  # the empty and the all-filtered element: exactly zero sums and gradients
            assert zero(got["sums"][e]), e
            assert all(zero(got[k][e]) for k in GRADS), e
            continue
        for k in PER_ROW:  # padding rows: zero gradients
            assert zero(got[k][e, n:]), (e, k)
        one = _run([els[e]], H, W, W_TRACK, g[e:e + 1])
        assert torch.equal(one["sums"][0], got["sums"][e]), e
        for k in PER_ROW:
            assert torch.equal(one[k][0], got[k][e, :n]), (e, k)
        for k in ("prev", "K"):
            assert torch.equal(one[k][0], got[k][e]), (e, k)
        for k in ("tgt", "tgt_n", "model_col"):  # index_add_: atomics in no fixed order
            torch.testing.assert_close(one[k][0], got[k][e], rtol=1e-5, atol=1e-6 * one[k][0].abs().max().item(),
                                       msg=f"{e} {k}")
    blocks = jr.blocks_of(max(SIZES))
    for e, other in ((0, 1), (3, 4)):
        x, idx, index = els[e]
        ref = jr.reference(x, idx, index, H, W, W_TRACK, blocks, g[e])
        _check(got, e, ref, f"ragged-element-{e}")
        # the neighbouring element's camera (intrinsics and previous pose) gives sums far outside the bounds
        xo = dict(x, K=els[other][0]["K"], prev=els[other][0]["prev"])
        assert _far_outside(jr.joint_sums(*(xo[k].double() for k in jr.NAMES), idx, index, H, W, W_TRACK), ref), e


# ------------------------------------------------------------------------------------------------------- c. identities
def test_zero_weight_is_the_geometric_op_and_photometric_gradients_vanish():
    from gradslam_b200.odometry.icputils import _NormalEqBatchedFn

    H, W = 45, 62
    els = _elements([5000, 777, 2], H, W, seed=13)
    g = torch.randn(3, 28, generator=torch.Generator().manual_seed(3))
    got = _run(els, H, W, 0.0, g)
    Ns = 5000
    src = torch.zeros(3, Ns, 3)
    idx = torch.full((3, Ns), -1, dtype=torch.int64)
    for b, (x, i, _) in enumerate(els):
        src[b, :i.numel()], idx[b, :i.numel()] = x["src"], i
    s = src.to(DEV).requires_grad_(True)
    geo = _NormalEqBatchedFn.apply(s, torch.stack([e[0]["tgt"] for e in els]).to(DEV),
                                   torch.stack([e[0]["tgt_n"] for e in els]).to(DEV), idx.to(DEV),
                                   torch.tensor([5000, 777, 2], dtype=torch.int32, device=DEV))
    (geo * g.to(DEV)).sum().backward()
    assert torch.equal(got["sums"], geo.detach().cpu())
    assert torch.equal(got["src"], s.grad.cpu())
    for k in ("src_col", "model_col", "prev", "K"):
        assert bool((got[k] == 0).all()), k
    # and w > 0 changes the sums of the elements with photometric rows
    assert not torch.equal(_run(els, H, W, W_TRACK, g)["sums"][:2], got["sums"][:2])


@pytest.mark.parametrize("H,W", [(2, 50), (40, 2), (1, 64), (64, 1)])
def test_images_without_an_interior_pixel_give_the_geometric_sums(H, W):
    els = _elements([400, 1000], H, W, seed=14)
    g = torch.randn(2, 28, generator=torch.Generator().manual_seed(4))
    geo = _run(els, H, W, 0.0, g)
    for w in (W_TRACK, 3.0):
        got = _run(els, H, W, w, g)
        assert torch.equal(got["sums"], geo["sums"]), w
        for k in ("src", "prev", "K", "src_col", "model_col"):
            assert torch.equal(got[k], geo[k]), (w, k)


def test_intrinsics_instantiation_leaves_the_other_gradients_unchanged():
    H, W = 48, 64
    els = _elements([4000, 2500], H, W, seed=15)
    g = torch.randn(2, 28, generator=torch.Generator().manual_seed(5))
    with_k, without = _run(els, H, W, W_TRACK, g, k_grad=True), _run(els, H, W, W_TRACK, g, k_grad=False)
    assert without["K"] is None
    assert torch.equal(with_k["sums"], without["sums"])
    for k in ("src", "src_col", "prev"):
        assert torch.equal(with_k[k], without[k]), k
    for k in ("tgt", "tgt_n", "model_col"):
        torch.testing.assert_close(with_k[k], without[k], rtol=1e-5, atol=1e-6 * with_k[k].abs().max().item())
    assert bool((with_k["K"][:, 3] == 0).all())
    assert bool((with_k["K"][:, 0, 1] != 0).all()) and bool((with_k["K"][:, :3, 3] != 0).all())


def test_joint_backward_is_deterministic():
    """Two launches of the backward give every per-row output and the reduced pose and intrinsics gradients bit for
    bit (the fixed-order reductions: no atomics)."""
    from gradslam_b200 import _C

    H, W = 60, 80
    els = _elements([70001, 3000], H, W, seed=16)
    B, Ns = 2, 70001
    src = torch.zeros(B, Ns, 3)
    col = torch.zeros(B, Ns, 3)
    idx = torch.full((B, Ns), -1, dtype=torch.int64)
    for b, (x, i, _) in enumerate(els):
        src[b, :i.numel()], col[b, :i.numel()], idx[b, :i.numel()] = x["src"], x["src_col"], i
    d = lambda t: t.contiguous().to(DEV)
    stack = lambda k: d(torch.stack([e[0][k] for e in els]))
    args = (d(src), torch.tensor([70001, 3000], dtype=torch.int32, device=DEV), Ns, d(col), stack("tgt"),
            stack("tgt_n"), stack("model_col"), d(torch.stack([e[2] for e in els])), B, H, W, d(idx), stack("prev"),
            stack("K"), W_TRACK, d(torch.randn(B, 28, generator=torch.Generator().manual_seed(6))))
    nbytes = _C.lib().gsx_icp_joint_normal_eq_batched_bwd_scratch_bytes(B, Ns)
    outs = []
    for _ in range(2):
        o = [torch.full((B, Ns, 3), float("nan"), device=DEV) for _ in range(4)]
        o += [torch.full((B, Ns, 5, 3), float("nan"), device=DEV), torch.full((B, 4, 4), float("nan"), device=DEV),
              torch.full((B, 4, 4), float("nan"), device=DEV)]
        scratch = torch.empty(nbytes, dtype=torch.uint8, device=DEV)
        _C.launch("gsx_icp_joint_normal_eq_batched_bwd", *args, *o, scratch, nbytes, math.inf, math.inf)
        outs.append([t.cpu() for t in o])
    for a, b in zip(*outs):
        assert bool(torch.isfinite(a).all())
        assert torch.equal(a.view(torch.int32), b.view(torch.int32))


# ------------------------------------------------------------------------------------------------ d. benchmark size
@pytest.fixture
def joint_calls(monkeypatch):
    """Keeps the inputs of the last forward call of _JointNormalEqBatchedFn."""
    from gradslam_b200.odometry import icputils

    last = {}
    orig = icputils._JointNormalEqBatchedFn.forward

    def forward(ctx, src, src_col, tgt, tgt_n, model_col, prev, idx, index, src_counts, K, w, H, W,
                huber=(math.inf, math.inf)):
        last.clear()
        last.update(src=src.detach().clone(), src_col=src_col.detach().clone(), tgt=tgt.detach().clone(),
                    tgt_n=tgt_n.detach().clone(), model_col=model_col.detach().clone(), prev=prev.detach().clone(),
                    idx=idx.clone(), index=index.clone(), counts=src_counts.clone(), K=K.detach().clone(), w=w, H=H,
                    W=W)
        return orig(ctx, src, src_col, tgt, tgt_n, model_col, prev, idx, index, src_counts, K, w, H, W, huber)

    monkeypatch.setattr(icputils._JointNormalEqBatchedFn, "forward", staticmethod(forward))
    return last


@pytest.mark.parametrize("M", [0, 3])
def test_benchmark_size_taped_poses_equal_fused_and_the_op_matches_the_reference(M, joint_calls):
    """B = 8, 640 x 480, ds = 1 (about 1,200 blocks per element), the textured scene at W_TRACK: the differentiable
    mode's poses equal the fused call's bit for bit, and the last joint op it ran, re-run on its recorded inputs,
    matches the reference for elements 0 and 7."""
    import gradslam_b200 as gs
    from gradslam_b200.synthetic import make_textured_sequence

    B, L, H, W = 8, 3, 480, 640
    rgb, depth, K, poses = make_textured_sequence(B, L, H, W, seed=5, yaw0=0.3)
    frames = gs.RGBDImages(rgb.to(DEV), depth.to(DEV), K.to(DEV), poses.to(DEV))
    pc, _ = gs.PointFusion(odom="gt", surfel_radii=True, device=DEV)(frames[:, :2])
    slam = gs.PointFusion(odom="gradicp", association="projective", dsratio=1, surfel_radii=True, target_splat_px=M,
                          photometric_weight=W_TRACK, device=DEV)
    fused = slam._localize(pc, frames[:, 2], frames[:, 1])
    live = gs.RGBDImages(rgb[:, 2:3].to(DEV).requires_grad_(True), depth[:, 2:3].to(DEV).requires_grad_(True),
                         K.to(DEV), poses[:, 2:3].to(DEV))
    taped = slam._localize(pc, live, frames[:, 1])
    assert taped.requires_grad
    assert torch.equal(taped.detach(), fused)

    rec = dict(joint_calls)
    counts = rec["counts"].cpu().tolist()
    assert min(counts) > 1100 * jr.BLOCK  # (about 1,200 blocks per element)
    Ns = rec["src"].shape[1]
    els = []
    for b in range(B):
        n = counts[b]
        x = {"src": rec["src"][b, :n], "src_col": rec["src_col"][b, :n], "tgt": rec["tgt"][b], "tgt_n": rec["tgt_n"][b],
             "model_col": rec["model_col"][b], "prev": rec["prev"].reshape(B, 4, 4)[b],
             "K": rec["K"].reshape(B, 4, 4)[b]}
        els.append(({k: v.float().cpu() for k, v in x.items()}, rec["idx"][b, :n].cpu(), rec["index"][b].cpu()))
    g = torch.randn(B, 28, generator=torch.Generator().manual_seed(7))
    got = _run(els, H, W, rec["w"], g, ns=Ns)
    for b in (0, 7):
        x, idx, index = els[b]
        assert int((idx >= 0).sum()) > 100_000
        ref = jr.reference(x, idx, index, H, W, rec["w"], jr.blocks_of(Ns), g[b])
        _check(got, b, ref, f"benchmark-M{M}-element-{b}")
