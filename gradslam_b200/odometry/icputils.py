"""Point-to-plane ICP building blocks.

Host-side mirror of gradslam/odometry/icputils.py (same names, arguments, errors).  The association
(`chamferdist.knn_points` in the reference), the row build, the normal-equation reduction, the damped solve,
the SE(3) exponential and the LM / gradLM update all run in csrc/gsx_icp.cu; nothing here loops over points.
"""
import ctypes
import math
from typing import Optional, Union

import torch

from .. import _C
from ..structures.pointclouds import Pointclouds
from ..structures.rgbdimages import RGBDImages, _frame_base

__all__ = ["solve_linear_system", "gauss_newton_solve", "point_to_plane_ICP", "point_to_plane_gradICP",
           "downsample_pointclouds", "downsample_rgbdimages"]


def _need_tensor(x, name):
    if not torch.is_tensor(x):
        raise TypeError("Expected {} to be of type torch.Tensor. Got {}.".format(name, type(x)))


def solve_linear_system(A: torch.Tensor, b: torch.Tensor, damp: Union[float, torch.Tensor] = 1e-8):
    """x = (A^T A + damp I)^-1 A^T b — the normal equations, not the system itself (icputils.py:22-90)."""
    _need_tensor(A, "A")
    _need_tensor(b, "b")
    if not (isinstance(damp, float) or torch.is_tensor(damp)):
        raise TypeError("Expected damp to be of type float or torch.Tensor. Got {0}.".format(type(damp)))
    if torch.is_tensor(damp) and damp.ndim != 0:
        raise ValueError("Expected torch.Tensor damp to have ndim=0 (scalar). Got {0}.".format(damp.ndim))
    if A.ndim != 2:
        raise ValueError("A should have ndim=2, but had ndim={}".format(A.ndim))
    if b.ndim != 2:
        raise ValueError("b should have ndim=2, but had ndim={}".format(b.ndim))
    if b.shape[1] != 1:
        raise ValueError("b.shape[1] should 1, but was {0}".format(b.shape[1]))
    if A.shape[0] != b.shape[0]:
        raise ValueError("A.shape[0] and b.shape[0] should be equal ({0} != {1})".format(A.shape[0], b.shape[0]))
    damp = damp if torch.is_tensor(damp) else torch.tensor(damp, dtype=A.dtype, device=A.device)
    At = A.transpose(0, 1)
    normal = At @ A + torch.eye(A.shape[1], dtype=A.dtype, device=A.device) * damp
    return torch.inverse(normal) @ (At @ b)


def _check_clouds(src_pc, tgt_pc, tgt_normals, dist_thresh):
    _need_tensor(src_pc, "src_pc")
    _need_tensor(tgt_pc, "tgt_pc")
    _need_tensor(tgt_normals, "tgt_normals")
    if not (isinstance(dist_thresh, (float, int)) or dist_thresh is None):
        raise TypeError("Expected dist_thresh to be of type float or int. Got {0}.".format(type(dist_thresh)))
    for name, t in (("src_pc", src_pc), ("tgt_pc", tgt_pc), ("tgt_normals", tgt_normals)):
        if t.ndim != 3:
            raise ValueError("{} should have ndim=3, but had ndim={}".format(name, t.ndim))
    for name, t in (("src_pc", src_pc), ("tgt_pc", tgt_pc), ("tgt_normals", tgt_normals)):
        if t.shape[0] != 1:
            raise ValueError("{}.shape[0] should be 1, but was {} instead".format(name, t.shape[0]))
    if tgt_pc.shape[1] != tgt_normals.shape[1]:
        raise ValueError("tgt_pc.shape[1] and tgt_normals.shape[1] must be equal. Got {0}!={1}".format(
            tgt_pc.shape[1], tgt_normals.shape[1]))
    for name, t in (("src_pc", src_pc), ("tgt_pc", tgt_pc), ("tgt_normals", tgt_normals)):
        if t.shape[2] != 3:
            raise ValueError("{}.shape[2] should be 3, but was {} instead".format(name, t.shape[2]))


def _check_huber_delta(delta, name="huber_delta"):
    """A Huber scale of the robust tracking energy: None (off) or a real number (not a bool), finite and > 0 that stays
    > 0 and finite as the float32 the kernels take."""
    if delta is None:
        return
    if isinstance(delta, bool) or not isinstance(delta, (float, int)):
        raise TypeError("Expected {} to be None or of type float or int. Got {}.".format(name, type(delta)))
    try:
        d = float(delta)
    except OverflowError:  # an int beyond float range
        d = math.inf
    if not (math.isfinite(d) and d > 0 and math.isfinite(ctypes.c_float(d).value) and ctypes.c_float(d).value > 0):
        raise ValueError("Expected a finite float32 {} > 0 (or None). Got {}.".format(name, delta))


def _counts(n, B, device):
    return torch.full((B,), n, dtype=torch.int32, device=device)


def knn1(src: torch.Tensor, tgt: torch.Tensor, src_counts=None, tgt_counts=None, target_cache: Optional[dict] = None):
    """Exact 1-NN of every row of src (B,Ns,3) in tgt (B,Nt,3) (padded clouds: optional int32 sizes (B,); rows beyond a
    source size get idx -1).  Returns (squared distances (B,Ns), idx int64 (B,Ns)); ties resolve to the lowest target
    index.  CUDA kernel k_icp_knn_linearize.
    target_cache: a dict the caller keeps while it queries the SAME, unmodified target repeatedly (the ICP loop): the
    search grid of the target is then built by the first call only."""
    _C.require_cuda(src, "src")
    _C.require_cuda(tgt, "tgt")
    src = src.contiguous()
    B, Ns, _ = src.shape
    Nt = tgt.shape[1]
    key = (tgt.data_ptr(), tuple(tgt.shape), tuple(tgt.stride()), tgt._version, Ns)
    hit = target_cache is not None and target_cache.get("key") == key
    if hit:
        tgt_c, scratch, nt_t = target_cache["tgt"], target_cache["scratch"], target_cache["nt"]
    else:
        tgt_c = tgt.contiguous()
        scratch = torch.empty(_C.lib().gsx_knn1_scratch_bytes(B, Ns, Nt), dtype=torch.uint8, device=src.device)
        nt_t = _counts(Nt, B, src.device) if tgt_counts is None else tgt_counts
        if target_cache is not None:
            target_cache.update(key=key, tgt=tgt_c, scratch=scratch, nt=nt_t)
    # (the kernel writes the rows below each source size; the padding rows keep -1 / inf)
    idx = torch.full((B, Ns), -1, dtype=torch.int64, device=src.device)
    d2 = torch.full((B, Ns), float("inf"), dtype=torch.float32, device=src.device)
    ns_t = _counts(Ns, B, src.device) if src_counts is None else src_counts
    _C.launch("gsx_knn1", src, ns_t, Ns, tgt_c, nt_t, Nt, B, idx, d2, scratch, scratch.numel(), 0 if hit else 1)
    return d2, idx


def gauss_newton_solve(src_pc: torch.Tensor, tgt_pc: torch.Tensor, tgt_normals: torch.Tensor,
                       dist_thresh: Union[float, int, None] = None):
    """Point-to-plane rows for one Gauss-Newton step: A (Nsf,6), b (Nsf,1), nn indices (Nsf,) (icputils.py:93-232).
    The association is the CUDA exact 1-NN; the row algebra below is differentiable torch (as in the reference)."""
    _check_clouds(src_pc, tgt_pc, tgt_normals, dist_thresh)
    src_pc, tgt_pc, tgt_normals = src_pc.contiguous(), tgt_pc.contiguous(), tgt_normals.contiguous()
    d2, idx = knn1(src_pc.detach(), tgt_pc.detach())
    keep = torch.ones_like(d2[0], dtype=torch.bool) if dist_thresh is None else d2[0] < dist_thresh
    idx = idx[0][keep]
    s = src_pc[0][keep]
    p = tgt_pc[0].index_select(0, idx)
    n = tgt_normals[0].index_select(0, idx)
    sx, sy, sz = s[:, 0:1], s[:, 1:2], s[:, 2:3]
    nx, ny, nz = n[:, 0:1], n[:, 1:2], n[:, 2:3]
    A = torch.cat([nx, ny, nz, nz * sy - ny * sz, nx * sz - nz * sx, ny * sx - nx * sy], 1)
    b = nx * (p[:, 0:1] - sx) + ny * (p[:, 1:2] - sy) + nz * (p[:, 2:3] - sz)
    return A, b, idx


def _check_icp_args(src_pc, tgt_pc, tgt_normals, initial_transform, numiters):
    _need_tensor(src_pc, "src_pc")
    _need_tensor(tgt_pc, "tgt_pc")
    _need_tensor(tgt_normals, "tgt_normals")
    if not (torch.is_tensor(initial_transform) or initial_transform is None):
        raise TypeError("Expected initial_transform to be of type torch.Tensor. Got {0}.".format(
            type(initial_transform)))
    if not isinstance(numiters, int):
        raise TypeError("Expected numiters to be of type int. Got {0}.".format(type(numiters)))
    if initial_transform is not None:
        if initial_transform.ndim != 2:
            raise ValueError("Expected initial_transform.ndim to be 2. Got {0}.".format(initial_transform.ndim))
        if not (initial_transform.shape[0] == 4 and initial_transform.shape[1] == 4):
            raise ValueError("Expected initial_transform.shape to be (4, 4). Got {0}.".format(initial_transform.shape))


def icp_align(src, src_counts, tgt, tgt_normals, tgt_counts, T0, mode, numiters, damp, dist_thresh, lambda_max=2.0,
              B=1.0, B2=1.0, nu=200.0, want_idx=False, huber_delta=None):
    """Batched ICP (mode 0) / gradICP (mode 1) on padded clouds (Bn, N, 3) with int32 sizes.  One C call; with
    huber_delta the Huber-weighted rows of gsx_icp_align."""
    for name, t in (("src", src), ("tgt", tgt), ("tgt_normals", tgt_normals)):
        _C.require_cuda(t, name)
    Bn, Ns, _ = src.shape
    Nt = tgt.shape[1]
    dev = src.device
    out = torch.empty((Bn, 4, 4), dtype=torch.float32, device=dev)
    idx = torch.empty((Bn, Ns), dtype=torch.int64, device=dev) if want_idx else None
    nbytes = _C.lib().gsx_icp_align_scratch_bytes(Bn, Ns, Nt)
    scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    T0c = None if T0 is None else T0.to(dev).float().contiguous()
    args = (src.contiguous(), src_counts, Ns, tgt.contiguous(), tgt_normals.contiguous(), tgt_counts, Nt, Bn, T0c,
            int(mode), int(numiters), float(damp), 0 if dist_thresh is None else 1,
            0.0 if dist_thresh is None else float(dist_thresh), float(lambda_max), float(B), float(B2), float(nu), out,
            idx, scratch, nbytes, _huber_scale(huber_delta))
    _C.launch("gsx_icp_align", *args)
    return out, idx


def _wants_grad(*tensors):
    return torch.is_grad_enabled() and any(torch.is_tensor(t) and t.requires_grad for t in tensors)


class _NormalEqFn(torch.autograd.Function):
    """(src (Ns,3), tgt (Nt,3), tgt_normals (Nt,3), nn_idx (Ns,) int64) -> the 28 sums of the point-to-plane normal
    equations.  forward = gsx_icp_normal_eq_fwd, backward = gsx_icp_normal_eq_bwd (hand-written kernels)."""

    @staticmethod
    def forward(ctx, src, tgt, tgt_n, idx):
        src_c, tgt_c, tn_c, idx_c = src.detach().contiguous(), tgt.detach().contiguous(), tgt_n.detach().contiguous(), \
            idx.contiguous()
        for name, t in (("src", src_c), ("tgt", tgt_c), ("tgt_normals", tn_c)):
            _C.require_cuda(t, name)
        ns, dev = src_c.shape[0], src_c.device
        sums = torch.empty(28, dtype=torch.float32, device=dev)
        nbytes = _C.lib().gsx_icp_normal_eq_scratch_bytes(ns)
        scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        _C.launch("gsx_icp_normal_eq_fwd", src_c, ns, tgt_c, tn_c, idx_c, sums, scratch, nbytes)
        ctx.saved = (src_c, tgt_c, tn_c, idx_c)
        return sums

    @staticmethod
    def backward(ctx, g):
        src_c, tgt_c, tn_c, idx_c = ctx.saved
        ns = src_c.shape[0]
        g = g.contiguous().float()
        g_src = torch.empty_like(src_c)
        rows_p, rows_n = torch.empty_like(src_c), torch.empty_like(src_c)
        _C.launch("gsx_icp_normal_eq_bwd", src_c, ns, tgt_c, tn_c, idx_c, g, g_src, rows_p, rows_n)
        safe = idx_c.clamp(min=0)  # rows with idx < 0 carry zero gradients
        g_tgt = torch.zeros_like(tgt_c).index_add_(0, safe, rows_p)
        g_tn = torch.zeros_like(tn_c).index_add_(0, safe, rows_n)
        return g_src, g_tgt, g_tn, None


class _SolveFn(torch.autograd.Function):
    """(28 sums, damp) -> (xi (6,), dT (4,4)): damped 6x6 solve + se3_exp in one kernel (K7a).
    forward = gsx_icp_solve_fwd, backward = gsx_icp_solve_bwd (dual numbers, one lane per input)."""

    @staticmethod
    def forward(ctx, sums, damp):
        s, d = sums.detach().contiguous().float(), damp.detach().reshape(1).contiguous().float()
        _C.require_cuda(s, "sums")
        dev = s.device
        xi = torch.empty(6, dtype=torch.float32, device=dev)
        dT = torch.empty((4, 4), dtype=torch.float32, device=dev)
        _C.launch("gsx_icp_solve_fwd", s, d, 1, xi, dT)
        ctx.saved = (s, d, damp.shape)
        return xi, dT

    @staticmethod
    def backward(ctx, g_xi, g_dT):
        s, d, damp_shape = ctx.saved
        g_xi = None if g_xi is None else g_xi.contiguous().float()
        g_dT = None if g_dT is None else g_dT.contiguous().float()
        g_s, g_d = torch.empty_like(s), torch.empty_like(d)
        _C.launch("gsx_icp_solve_bwd", s, d, 1, g_xi, g_dT, g_s, g_d)
        return g_s, g_d.view(damp_shape)


class _UpdateFn(torch.autograd.Function):
    """(xi, err, new_err, damp, T) -> (new damp, applied step (4,4), step @ T): LM accept / reject (mode 0) or the
    gradLM gates (mode 1), the applied se3_exp and the pose accumulation in one kernel (K7b).
    forward = gsx_icp_update_fwd, backward = gsx_icp_update_bwd."""

    @staticmethod
    def forward(ctx, xi, err, new_err, damp, T, mode, lambda_max, B, B2, nu):
        dev = xi.device
        ins = [t.detach().reshape(n).contiguous().float() for t, n in ((xi, 6), (err, 1), (new_err, 1), (damp, 1),
                                                                       (T, 16))]
        _C.require_cuda(ins[0], "xi")
        damp_out = torch.empty(1, dtype=torch.float32, device=dev)
        dT = torch.empty((4, 4), dtype=torch.float32, device=dev)
        Tn = torch.empty((4, 4), dtype=torch.float32, device=dev)
        par = (int(mode), float(lambda_max), float(B), float(B2), float(nu))
        _C.launch("gsx_icp_update_fwd", *ins, 1, *par, damp_out, dT, Tn)
        ctx.saved = (ins, par, (xi.shape, err.shape, new_err.shape, damp.shape, T.shape))
        return damp_out.view(damp.shape), dT, Tn

    @staticmethod
    def backward(ctx, g_damp, g_dT, g_T):
        ins, par, shapes = ctx.saved
        gs = [None if g is None else g.contiguous().float() for g in (g_damp, g_dT, g_T)]
        outs = [torch.empty_like(t) for t in ins]
        _C.launch("gsx_icp_update_bwd", *ins, 1, *par, *gs, *outs)
        return tuple(o.view(sh) for o, sh in zip(outs, shapes)) + (None,) * 5


class _RigidTransformFn(torch.autograd.Function):
    """(points (N,3), T (4,4)) -> R p + t (transform_pointcloud, geometryutils.py:737-794).
    forward = gsx_rigid_transform_fwd, backward = gsx_rigid_transform_bwd (deterministic reduction for d/dT)."""

    @staticmethod
    def forward(ctx, points, T):
        p, Tc = points.detach().contiguous().float(), T.detach().contiguous().float()
        _C.require_cuda(p, "points")
        out = torch.empty_like(p)
        _C.launch("gsx_rigid_transform_fwd", p, p.shape[0], Tc, out)
        ctx.saved = (p, Tc)
        return out

    @staticmethod
    def backward(ctx, g):
        p, Tc = ctx.saved
        dev, n = p.device, p.shape[0]
        g = g.contiguous().float()
        g_p, g_T = torch.empty_like(p), torch.empty_like(Tc)
        nbytes = _C.lib().gsx_rigid_transform_bwd_scratch_bytes(n)
        scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        _C.launch("gsx_rigid_transform_bwd", p, n, Tc, g, g_p, g_T, scratch, nbytes)
        return g_p, g_T


# ------------------------------------------------------------------------------------------------ batched variants
# The same four ops for a padded batch (B, N, 3) with int32 sizes: ONE op chain records the differentiable ICP of all
# batch elements (the reference's providers, and round 1 here, ran one chain per element: odometry/icp.py:84-97).  Every
# kernel takes the batch index from blockIdx.y; values per element are bit-identical to the per-element ops (padding rows
# contribute exact zeros to the fixed-order sums).
class _NormalEqBatchedFn(torch.autograd.Function):
    """gsx_icp_normal_eq_batched_fwd / _bwd; huber_delta: the float32 Huber scale of the rows (+inf = unweighted)."""

    @staticmethod
    def forward(ctx, src, tgt, tgt_n, idx, src_counts, huber_delta=math.inf):
        src_c, tgt_c, tn_c = (t.detach().contiguous().float() for t in (src, tgt, tgt_n))
        idx_c = idx.contiguous()
        _C.require_cuda(src_c, "src")
        Bn, Ns, _ = src_c.shape
        Nt, dev = tgt_c.shape[1], src_c.device
        sums = torch.empty((Bn, 28), dtype=torch.float32, device=dev)
        nbytes = Bn * _C.lib().gsx_icp_normal_eq_scratch_bytes(Ns)
        scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        _C.launch("gsx_icp_normal_eq_batched_fwd", src_c, src_counts, Ns, tgt_c, tn_c, Nt, Bn, idx_c, sums, scratch,
                  nbytes, float(huber_delta))
        ctx.saved = (src_c, tgt_c, tn_c, idx_c, src_counts)
        ctx.huber_delta = float(huber_delta)
        return sums

    @staticmethod
    def backward(ctx, g):
        src_c, tgt_c, tn_c, idx_c, src_counts = ctx.saved
        Bn, Ns, _ = src_c.shape
        Nt, dev = tgt_c.shape[1], src_c.device
        g = g.contiguous().float()
        g_src = torch.empty_like(src_c)
        rows_p, rows_n = torch.empty_like(src_c), torch.empty_like(src_c)
        _C.launch("gsx_icp_normal_eq_batched_bwd", src_c, src_counts, Ns, tgt_c, tn_c, Nt, Bn, idx_c, g, g_src, rows_p,
                  rows_n, ctx.huber_delta)
        # rows with idx < 0 carry zero gradients; scatter the per-source-row target gradients with the association
        flat = (idx_c.clamp(min=0) + torch.arange(Bn, device=dev).view(Bn, 1) * Nt).view(-1)
        g_tgt = torch.zeros((Bn * Nt, 3), dtype=torch.float32, device=dev).index_add_(0, flat, rows_p.view(-1, 3))
        g_tn = torch.zeros((Bn * Nt, 3), dtype=torch.float32, device=dev).index_add_(0, flat, rows_n.view(-1, 3))
        return g_src, g_tgt.view(Bn, Nt, 3), g_tn.view(Bn, Nt, 3), None, None, None


class _SolveBatchedFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, sums, damp):
        s, d = sums.detach().contiguous().float(), damp.detach().contiguous().float()
        _C.require_cuda(s, "sums")
        Bn, dev = s.shape[0], s.device
        xi = torch.empty((Bn, 6), dtype=torch.float32, device=dev)
        dT = torch.empty((Bn, 4, 4), dtype=torch.float32, device=dev)
        _C.launch("gsx_icp_solve_fwd", s, d, Bn, xi, dT)
        ctx.saved = (s, d)
        return xi, dT

    @staticmethod
    def backward(ctx, g_xi, g_dT):
        s, d = ctx.saved
        g_xi = None if g_xi is None else g_xi.contiguous().float()
        g_dT = None if g_dT is None else g_dT.contiguous().float()
        g_s, g_d = torch.empty_like(s), torch.empty_like(d)
        _C.launch("gsx_icp_solve_bwd", s, d, s.shape[0], g_xi, g_dT, g_s, g_d)
        return g_s, g_d


class _UpdateBatchedFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, xi, err, new_err, damp, T, mode, lambda_max, B, B2, nu):
        dev = xi.device
        ins = [t.detach().contiguous().float() for t in (xi, err, new_err, damp, T)]
        _C.require_cuda(ins[0], "xi")
        Bn = ins[0].shape[0]
        damp_out = torch.empty(Bn, dtype=torch.float32, device=dev)
        dT = torch.empty((Bn, 4, 4), dtype=torch.float32, device=dev)
        Tn = torch.empty((Bn, 4, 4), dtype=torch.float32, device=dev)
        par = (int(mode), float(lambda_max), float(B), float(B2), float(nu))
        _C.launch("gsx_icp_update_fwd", *ins, Bn, *par, damp_out, dT, Tn)
        ctx.saved = (ins, par)
        return damp_out, dT, Tn

    @staticmethod
    def backward(ctx, g_damp, g_dT, g_T):
        ins, par = ctx.saved
        gs = [None if g is None else g.contiguous().float() for g in (g_damp, g_dT, g_T)]
        outs = [torch.empty_like(t) for t in ins]
        _C.launch("gsx_icp_update_bwd", *ins, ins[0].shape[0], *par, *gs, *outs)
        return tuple(outs) + (None,) * 5


class _RigidTransformBatchedFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, points, T, counts):
        p, Tc = points.detach().contiguous().float(), T.detach().contiguous().float()
        _C.require_cuda(p, "points")
        out = torch.empty_like(p)
        _C.launch("gsx_rigid_transform_batched_fwd", p, counts, p.shape[1], p.shape[0], Tc, out)
        ctx.saved = (p, Tc, counts)
        return out

    @staticmethod
    def backward(ctx, g):
        p, Tc, counts = ctx.saved
        dev = p.device
        Bn, n = p.shape[0], p.shape[1]
        g = g.contiguous().float()
        g_p, g_T = torch.empty_like(p), torch.empty_like(Tc)
        nbytes = Bn * _C.lib().gsx_rigid_transform_bwd_scratch_bytes(n)
        scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        _C.launch("gsx_rigid_transform_batched_bwd", p, counts, n, Bn, Tc, g, g_p, g_T, scratch, nbytes)
        return g_p, g_T, None


class _JointNormalEqBatchedFn(torch.autograd.Function):
    """The joint geometric + photometric normal equations of the projective ICP at a given association (idx (B,Ns) pixel
    or -1): (src, src_col (B,Ns,3), tgt, tgt_n, model_col (B,H*W,3), prev (B,4,4)) -> (B,28).  forward =
    gsx_icp_joint_normal_eq_batched_fwd, backward = gsx_icp_joint_normal_eq_batched_bwd, with d/dK when K requires grad
    (the photometric row reads K's first three rows); the gradients of the model colours come per source row for the
    five stencil pixels and are scattered here.  huber: (huber_delta, photometric_huber_delta) as float32 scales
    (+inf = that residual unweighted)."""

    @staticmethod
    def forward(ctx, src, src_col, tgt, tgt_n, model_col, prev, idx, index, src_counts, K, w, H, W,
                huber=(math.inf, math.inf)):
        ins = [t.detach().contiguous().float() for t in (src, src_col, tgt, tgt_n, model_col, prev)]
        _C.require_cuda(ins[0], "src")
        Bn, Ns = ins[0].shape[:2]
        idx_c, index_c, K_c = idx.contiguous(), index.contiguous(), K.detach().contiguous()
        sums = torch.empty((Bn, 28), dtype=torch.float32, device=src.device)
        nbytes = Bn * _C.lib().gsx_icp_normal_eq_scratch_bytes(Ns)
        scratch = torch.empty(nbytes, dtype=torch.uint8, device=src.device)
        huber = tuple(float(d) for d in huber)
        _C.launch("gsx_icp_joint_normal_eq_batched_fwd", ins[0], src_counts, Ns, ins[1], ins[2], ins[3], ins[4],
                  index_c, Bn, int(H), int(W), idx_c, ins[5], K_c, float(w), sums, scratch, nbytes, *huber)
        ctx.saved = (ins, idx_c, index_c, src_counts, K_c, float(w), int(H), int(W), prev.shape)
        ctx.huber = huber
        ctx.K_shape = K.shape
        return sums

    @staticmethod
    def backward(ctx, g):
        (src, src_col, tgt, tgt_n, model_col, prev), idx, index, src_counts, K, w, H, W, prev_shape = ctx.saved
        Bn, Ns = src.shape[:2]
        P, dev = H * W, src.device
        g = g.contiguous().float()
        g_src, g_col, rows_p, rows_n = (torch.empty_like(src) for _ in range(4))
        rows_st = torch.empty((Bn, Ns, 5, 3), dtype=torch.float32, device=dev)
        g_prev = torch.empty((Bn, 4, 4), dtype=torch.float32, device=dev)
        g_K = torch.zeros((Bn, 4, 4), dtype=torch.float32, device=dev) if ctx.needs_input_grad[9] else None
        nbytes = _C.lib().gsx_icp_joint_normal_eq_batched_bwd_scratch_bytes(Bn, Ns)
        scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        _C.launch("gsx_icp_joint_normal_eq_batched_bwd", src, src_counts, Ns, src_col, tgt, tgt_n, model_col, index, Bn,
                  H, W, idx, prev, K, w, g, g_src, g_col, rows_p, rows_n, rows_st, g_prev, g_K, scratch, nbytes,
                  *ctx.huber)
        g_K = None if g_K is None else g_K.view(ctx.K_shape)
        base = torch.arange(Bn, device=dev).view(Bn, 1) * P
        flat = (idx.clamp(min=0) + base).view(-1)  # rows with idx < 0 carry zero gradients
        g_tgt = torch.zeros((Bn * P, 3), dtype=torch.float32, device=dev).index_add_(0, flat, rows_p.view(-1, 3))
        g_tn = torch.zeros((Bn * P, 3), dtype=torch.float32, device=dev).index_add_(0, flat, rows_n.view(-1, 3))
        offs = torch.tensor([0, -1, 1, -W, W], device=dev)
        st = ((idx.clamp(min=0).unsqueeze(-1) + offs).clamp(0, P - 1) + base.unsqueeze(-1)).view(-1)
        g_model = torch.zeros((Bn * P, 3), dtype=torch.float32, device=dev).index_add_(0, st, rows_st.view(-1, 3))
        return (g_src, g_col, g_tgt.view(Bn, P, 3), g_tn.view(Bn, P, 3), g_model.view(Bn, P, 3),
                g_prev.view(prev_shape), None, None, None, g_K, None, None, None, None)


def _normal_equations_batched(src, src_counts, tgt, tgt_n, tgt_counts, dist_thresh, target_cache=None, associate=None,
                              normal_eq=None, huber_delta=None):
    if normal_eq is not None:  # (the projective association with the photometric term)
        idx = associate(src.detach())
        return normal_eq(src, tgt, tgt_n, idx), idx
    if associate is None:
        d2, idx = knn1(src.detach(), tgt.detach(), src_counts, tgt_counts, target_cache)
        if dist_thresh is not None:
            idx = torch.where(d2 < dist_thresh, idx, torch.full_like(idx, -1))
    else:
        idx = associate(src.detach())
    return _NormalEqBatchedFn.apply(src, tgt, tgt_n, idx, src_counts, _huber_scale(huber_delta)), idx


def _taped_icp_batched(src, src_counts, tgt, tgt_n, tgt_counts, T0, mode, numiters, damp, dist_thresh, lambda_max=2.0,
                       B=1.0, B2=1.0, nu=200.0, associate=None, normal_eq=None, huber_delta=None):
    """The differentiable ICP / gradICP loop of `_taped_icp` for a padded batch: src (Bn,Ns,3), tgt / tgt_n (Bn,Nt,3),
    int32 sizes (Bn,).  One chain of batched ops for all elements; returns (T (Bn,4,4), last nn idx (Bn,Ns), -1 = none).
    Per element the values are bit-identical to the per-element chain and to the fused no-grad loop.
    associate: None = exact 1-NN in tgt (thresholded by dist_thresh); otherwise a function of the current source
    (Bn,Ns,3), detached, returning the int64 target row per source row (-1 = none) - the projective association.
    normal_eq: None = _NormalEqBatchedFn; otherwise a function (src, tgt, tgt_n, idx) -> (Bn,28) sums (the joint op of
    the photometric term, which then carries its own Huber scales).
    huber_delta: None = unweighted rows; else the Huber-weighted normal-equation op at that scale (the rows of
    gsx_icp_align), so the loop minimises the Huber energy as the fused loop does."""
    dev = src.device
    Bn, Ns = src.shape[0], src.shape[1]
    # No valid source (or target) point in any element gives a padded width of 0, which the kernels reject.  One zero
    # padding row (the sizes stay 0) makes every element an empty element of a ragged batch, as the fused loop sees it.
    pad = lambda t: torch.cat([t, t.new_zeros(Bn, 1, 3)], 1) if t.shape[1] == 0 else t
    src, tgt, tgt_n = pad(src), pad(tgt), pad(tgt_n)
    dampt = torch.full((Bn,), float(damp), dtype=torch.float32, device=dev)
    T = (torch.eye(4, dtype=torch.float32, device=dev).repeat(Bn, 1, 1) if T0 is None
         else T0.to(torch.float32).expand(Bn, 4, 4).contiguous())
    tgt, tgt_n = tgt.contiguous(), tgt_n.contiguous()  # once (strided views of packed map rows), not per iteration
    cur = _RigidTransformBatchedFn.apply(src, T, src_counts)
    idx = None
    grid = {}  # the target's search grid: built by the first of the 2 * numiters associations
    for _ in range(numiters):
        sums, idx = _normal_equations_batched(cur, src_counts, tgt, tgt_n, tgt_counts, dist_thresh, grid, associate,
                                              normal_eq, huber_delta)
        xi, dT = _SolveBatchedFn.apply(sums, dampt)
        one_step = _RigidTransformBatchedFn.apply(cur, dT, src_counts)
        sums_next, _ = _normal_equations_batched(one_step, src_counts, tgt, tgt_n, tgt_counts, dist_thresh, grid,
                                                 associate, normal_eq, huber_delta)
        dampt, dT_applied, T = _UpdateBatchedFn.apply(xi, sums[:, 27], sums_next[:, 27], dampt, T, mode, lambda_max, B,
                                                      B2, nu)
        cur = _RigidTransformBatchedFn.apply(cur, dT_applied, src_counts)
    return T, (None if idx is None else idx[:, :Ns])


def _normal_equations(src, tgt, tgt_n, dist_thresh):
    """Association (CUDA exact 1-NN, index-only) + the differentiable normal-equation op.  src (Ns,3) -> 28 sums."""
    d2, idx = knn1(src.detach().unsqueeze(0), tgt.detach().unsqueeze(0))
    idx = idx[0]
    if dist_thresh is not None:
        idx = torch.where(d2[0] < dist_thresh, idx, torch.full_like(idx, -1))
    return _NormalEqFn.apply(src, tgt, tgt_n, idx), idx


def _taped_icp(src_pc, tgt_pc, tgt_normals, initial_transform, mode, numiters, damp, dist_thresh, lambda_max=2.0,
               B=1.0, B2=1.0, nu=200.0):
    """Differentiable variant used when an input requires grad: the same loop as the fused kernel sequence, as a chain
    of autograd ops that each have a hand-written forward AND backward kernel -
    rigid transform (`_RigidTransformFn`), 1-NN association (index-only, no gradient, as in the reference), normal
    equations (`_NormalEqFn`), damped solve + se3_exp (`_SolveFn`), LM / gradLM update (`_UpdateFn`).  PyTorch only
    records the tape; no ATen arithmetic runs between the ops and there is no host synchronisation
    (icputils.py:235-545)."""
    dtype, device = torch.float32, src_pc.device
    damp = torch.tensor([float(damp)], dtype=dtype, device=device)
    T = torch.eye(4, dtype=dtype, device=device) if initial_transform is None else initial_transform.to(dtype)
    src = _RigidTransformFn.apply(src_pc[0], T)
    tgt, tgt_n = tgt_pc[0], tgt_normals[0]
    idx = None
    for _ in range(numiters):
        sums, idx = _normal_equations(src, tgt, tgt_n, dist_thresh)
        xi, dT = _SolveFn.apply(sums, damp)
        one_step = _RigidTransformFn.apply(src, dT)
        sums_next, _ = _normal_equations(one_step, tgt, tgt_n, dist_thresh)
        damp, dT_applied, T = _UpdateFn.apply(xi, sums[27], sums_next[27], damp, T, mode, lambda_max, B, B2, nu)
        src = _RigidTransformFn.apply(src, dT_applied)
    return T, idx[idx >= 0]


def _single(src_pc, tgt_pc, tgt_normals, initial_transform, mode, numiters, damp, dist_thresh, **kw):
    if _wants_grad(src_pc, tgt_pc, tgt_normals, initial_transform):
        return _taped_icp(src_pc, tgt_pc, tgt_normals, initial_transform, mode, numiters, damp, dist_thresh, **kw)
    dev = src_pc.device
    T0 = None if initial_transform is None else initial_transform.view(1, 4, 4)
    T, idx = icp_align(src_pc.contiguous(), _counts(src_pc.shape[1], 1, dev), tgt_pc.contiguous(),
                       tgt_normals.contiguous(), _counts(tgt_pc.shape[1], 1, dev), T0, mode, numiters, damp,
                       dist_thresh, want_idx=True, **kw)
    idx = idx[0]
    return T[0], idx[idx >= 0]


def point_to_plane_ICP(src_pc: torch.Tensor, tgt_pc: torch.Tensor, tgt_normals: torch.Tensor,
                       initial_transform: Optional[torch.Tensor] = None, numiters: int = 20, damp: float = 1e-8,
                       dist_thresh: Union[float, int, None] = None):
    """Rigid transform aligning src to tgt with point-to-plane LM (icputils.py:235-367).  Returns (T (4,4), nn idx)."""
    _check_icp_args(src_pc, tgt_pc, tgt_normals, initial_transform, numiters)
    return _single(src_pc, tgt_pc, tgt_normals, initial_transform, 0, numiters, damp, dist_thresh)


def point_to_plane_gradICP(src_pc: torch.Tensor, tgt_pc: torch.Tensor, tgt_normals: torch.Tensor,
                           initial_transform: Optional[torch.Tensor] = None, numiters: int = 20, damp: float = 1e-8,
                           dist_thresh: Union[float, int, None] = None, lambda_max: Union[float, int] = 2.0,
                           B: Union[float, int] = 1.0, B2: Union[float, int] = 1.0, nu: Union[float, int] = 200.0):
    """Same with the gradLM solver (icputils.py:370-545)."""
    _check_icp_args(src_pc, tgt_pc, tgt_normals, initial_transform, numiters)
    for name, v in (("lambda_max", lambda_max), ("B", B), ("B2", B2), ("nu", nu)):
        if not isinstance(v, (float, int)):
            raise TypeError("Expected {} to be of type float or int; got {}".format(name, type(v)))
    return _single(src_pc, tgt_pc, tgt_normals, initial_transform, 1, numiters, damp, dist_thresh,
                   lambda_max=lambda_max, B=B, B2=B2, nu=nu)


def downsample_pointclouds(pointclouds: Pointclouds, pc2im_bnhw: torch.Tensor, ds_ratio: int) -> Pointclouds:
    """Keeps the active map points whose pixel lies on the ds lattice (icputils.py:548-620)."""
    if not isinstance(pointclouds, Pointclouds):
        raise TypeError("Expected pointclouds to be of type gradslam.Pointclouds. Got {0}.".format(type(pointclouds)))
    if not torch.is_tensor(pc2im_bnhw):
        raise TypeError("Expected pc2im_bnhw to be of type torch.Tensor. Got {0}.".format(type(pc2im_bnhw)))
    if not isinstance(ds_ratio, int):
        raise TypeError("Expected ds_ratio to be of type int. Got {0}.".format(type(ds_ratio)))
    if pc2im_bnhw.ndim != 2:
        raise ValueError("Expected pc2im_bnhw to have ndim=2. Got {0}.".format(pc2im_bnhw.ndim))
    if pc2im_bnhw.shape[1] != 4:
        raise ValueError("pc2im_bnhw.shape[1] must be 4, but was {0}.".format(pc2im_bnhw.shape[1]))
    B = len(pointclouds)
    dev = pc2im_bnhw.device
    t = pc2im_bnhw[(pc2im_bnhw[:, 2] % ds_ratio == 0) & (pc2im_bnhw[:, 3] % ds_ratio == 0)]
    # all elements at once (the reference loops over b, icputils.py:604-617): element b keeps its rows in table order
    order = torch.sort(t[:, 0], stable=True).indices
    b_of, n_of = t[order, 0], t[order, 1]
    counts_t = torch.bincount(b_of, minlength=B)[:B]
    counts = [int(c) for c in counts_t.tolist()]  # (the one host synchronisation: the ragged sizes)
    nmax = max(counts) if counts else 0
    starts = torch.cumsum(counts_t, 0) - counts_t
    pos = torch.arange(b_of.numel(), device=dev) - starts[b_of]
    idx = torch.zeros((B, nmax), dtype=torch.int64, device=dev)
    idx[b_of, pos] = n_of
    keep = (torch.arange(nmax, device=dev).unsqueeze(0) < counts_t.unsqueeze(1)).unsqueeze(-1)

    def pick(padded):
        if padded is None:
            return None
        g = torch.gather(padded, 1, idx.unsqueeze(-1).expand(-1, -1, padded.shape[-1]))
        return torch.where(keep, g, torch.zeros((), dtype=g.dtype, device=g.device))

    out = Pointclouds(points=pick(pointclouds.points_padded), normals=pick(pointclouds.normals_padded),
                      colors=pick(pointclouds.colors_padded))
    out._set_counts(counts)
    return out


def _compact_rows(mask: torch.Tensor, values):
    """mask (B, n) bool, values: tensors (B, n, C).  Per element the selected rows, in their original order, moved to
    the front of a (B, max count, C) tensor, zeros behind them; returns (tensors, sizes as a host list)."""
    B, n = mask.shape
    counts_t = mask.sum(1)
    counts = [int(c) for c in counts_t.tolist()]  # (the one host synchronisation: the ragged sizes)
    nmax = max(counts) if counts else 0
    order = torch.sort((~mask).to(torch.uint8), dim=1, stable=True).indices[:, :nmax]  # selected rows first, in order
    keep = (torch.arange(nmax, device=mask.device).unsqueeze(0) < counts_t.unsqueeze(1)).unsqueeze(-1)
    outs = []
    for v in values:
        g = torch.gather(v, 1, order.unsqueeze(-1).expand(-1, -1, v.shape[-1]))
        outs.append(torch.where(keep, g, torch.zeros((), dtype=g.dtype, device=g.device)))
    return outs, counts


def downsample_rgbdimages(rgbdimages: RGBDImages, ds_ratio: int) -> Pointclouds:
    """Strided subsample of the global maps + valid mask -> Pointclouds (icputils.py:623-669)."""
    if not isinstance(rgbdimages, RGBDImages):
        raise TypeError("Expected rgbdimages to be of type gradslam.RGBDImages. Got {0}.".format(type(rgbdimages)))
    if not isinstance(ds_ratio, int):
        raise TypeError("Expected ds_ratio to be of type int. Got {0}.".format(type(ds_ratio)))
    if rgbdimages.shape[1] != 1:
        raise ValueError("Sequence length of rgbdimages must be 1, but was {0}.".format(rgbdimages.shape[1]))
    fr = rgbdimages.to_channels_last()
    B = len(fr)
    mask = fr.valid_depth_mask.squeeze(-1)[:, 0, ::ds_ratio, ::ds_ratio].reshape(B, -1)
    sub = lambda m: m[:, 0, ::ds_ratio, ::ds_ratio].reshape(B, -1, m.shape[-1])
    # all elements at once (the reference indexes element by element, icputils.py:655-667)
    (pts, nrm, col), counts = _compact_rows(mask, [sub(fr.global_vertex_map), sub(fr.global_normal_map),
                                                    sub(fr.rgb_image)])
    out = Pointclouds(points=pts, normals=nrm, colors=col)
    out._set_counts(counts)
    return out


# --------------------------------------------------------------------------------------------- fused localisation
class _IcpWorkspace:
    _cache = {}

    def __init__(self, device, B, H, W, ds, capacity):
        n = _C.lib().gsx_icp_workspace_bytes(B, H, W, ds, capacity)
        self.buf = torch.zeros(n, dtype=torch.uint8, device=device)
        self.capacity = capacity
        self.epoch = 0

    @classmethod
    def get(cls, device, B, H, W, ds, capacity):
        key = (str(device), B, H, W, ds)
        ws = cls._cache.get(key)
        if ws is None or ws.capacity < capacity:
            ws = cls(device, B, H, W, ds, capacity)
            cls._cache[key] = ws
        return ws

    def next_epoch(self):
        self.epoch += 1
        if self.epoch >= (1 << 30) - 1:
            self.buf.zero_()
            self.epoch = 1
        return self.epoch


class _IcpTargetScratch:
    """Target clouds (points, normals, search grid) of localize_against_map, cached per (device, B) and grown by
    doubling: calls are stream-ordered, so one buffer serves every call on the device."""
    _cache = {}

    @classmethod
    def get(cls, device, B, tgt_capacity):
        key = (str(device), B)
        buf = cls._cache.get(key)
        need = _C.lib().gsx_icp_tgt_scratch_bytes(B, tgt_capacity)
        if buf is None or buf.numel() < need:
            grown = _C.lib().gsx_icp_tgt_scratch_bytes(B, min(2 * tgt_capacity, 1 << 29))
            buf = torch.empty(max(need, grown), dtype=torch.uint8, device=device)
            cls._cache[key] = buf
        return buf


def localize_against_map(pointclouds, live_frame, prev_frame, dsratio, odomprov):
    """ICPSLAM._localize for odom in {icp, gradicp} (slam/icpslam.py:238-247) as ONE C call: gathers the source
    (live frame on the ds lattice at the previous pose) and target (lattice-active map points) clouds, runs the
    batched ICP loop and returns the new poses (B,1,4,4) = T_icp · prev pose.  No host synchronisation."""
    live = live_frame.to_channels_last()
    B, _, H, W = live.shape
    dev = pointclouds.device
    _C.require_cuda(live.depth_image, "depth_image")
    depth, d_bs = _frame_base(live.depth_image, H * W)
    K = live.intrinsics.contiguous()
    prev = prev_frame.poses.contiguous()
    _C.require_cuda(pointclouds._geo, "pointclouds (geometry rows)")
    geo = pointclouds._geo.contiguous()
    ws = _IcpWorkspace.get(dev, B, H, W, dsratio, pointclouds.capacity)
    # target capacity: the lattice-active map points are a subset of the map, so the map's host-side size bound holds
    # every target.  No per-pixel bound would do: ICPSLAM's aggregate map gains a point on every lattice pixel of every
    # frame, so a camera that dwells piles up one more point per lattice pixel per frame.
    bound = max(1, pointclouds._bound)
    tgt = _IcpTargetScratch.get(dev, B, bound)
    out = torch.empty((B, 1, 4, 4), dtype=torch.float32, device=dev)
    mode = 1 if hasattr(odomprov, "lambda_max") else 0
    dth = odomprov.dist_thresh
    args = (geo, pointclouds._counts_dev[pointclouds._cur], pointclouds.capacity, pointclouds._bound, depth, d_bs, K, 16,
            prev, 16, B, H, W, int(dsratio), mode, int(odomprov.numiters), float(odomprov.damp),
            0 if dth is None else 1, 0.0 if dth is None else float(dth), float(getattr(odomprov, "lambda_max", 2.0)),
            float(getattr(odomprov, "B", 1.0)), float(getattr(odomprov, "B2", 1.0)),
            float(getattr(odomprov, "nu", 200.0)), tgt, bound, out, 16, ws.buf, ws.capacity, ws.next_epoch(),
            pointclouds._overflow_flag(), _huber_scale(getattr(odomprov, "huber_delta", None)))
    _C.launch("gsx_icp_localize", *args)
    return out


# ------------------------------------------------------------------------------------ projective association
def project_associate(src, src_counts, tgt_points, tgt_index, prev_poses, K, H, W, dist_thresh=None):
    """Projective association of a padded source batch src (B,Ns,3) (world frame, int32 sizes (B,)) with target images
    rendered from prev_poses (B,4,4) with intrinsics K (B,4,4): tgt_points (B,H*W,3), tgt_index (B,H*W) int64 (-1 =
    uncovered).  Returns (squared distances (B,Ns), pixel index int64 (B,Ns), -1 = none); rows beyond a source size get
    -1 / inf.  CUDA kernel k_icp_project_associate, the association of gsx_icp_localize_projective."""
    _C.require_cuda(src, "src")
    src = src.contiguous()
    Bn, Ns, _ = src.shape
    idx = torch.full((Bn, Ns), -1, dtype=torch.int64, device=src.device)
    d2 = torch.full((Bn, Ns), float("inf"), dtype=torch.float32, device=src.device)
    _C.launch("gsx_icp_project_associate", src, src_counts, Ns, tgt_points.contiguous(), tgt_index.contiguous(),
              prev_poses.contiguous(), 16, K.contiguous(), 16, Bn, int(H), int(W), 0 if dist_thresh is None else 1,
              0.0 if dist_thresh is None else float(dist_thresh), idx, d2)
    return d2, idx


class _ProjectiveWorkspace:
    """Workspace of gsx_icp_localize_projective per (device, B, H, W, ds, photometric): nothing in it outlives a call,
    so one buffer serves every stream-ordered call with that shape."""
    _cache = {}

    @classmethod
    def get(cls, device, B, H, W, ds, photometric):
        key = (str(device), B, H, W, ds, bool(photometric))
        buf = cls._cache.get(key)
        if buf is None:
            buf = torch.empty(_C.lib().gsx_icp_projective_workspace_bytes(B, H, W, ds, int(bool(photometric))),
                              dtype=torch.uint8, device=device)
            cls._cache[key] = buf
        return buf


def _solver_params(odomprov):
    return (1 if hasattr(odomprov, "lambda_max") else 0, float(getattr(odomprov, "lambda_max", 2.0)),
            float(getattr(odomprov, "B", 1.0)), float(getattr(odomprov, "B2", 1.0)), float(getattr(odomprov, "nu", 200.0)))


def projective_targets(pointclouds, K, prev_poses, H, W, target_splat_px=0):
    """The target images of the projective ICP, the map's predicted vertex and normal maps seen from prev_poses (B,4,4)
    with intrinsics K (B,4,4): (index (B,H*W) int64, -1 = uncovered; points, normals (B,H*W,3) world frame, zeros where
    uncovered).  target_splat_px >= 1 renders the surfels with radii as disks (render_pointclouds(max_splat_px)) and a
    disk's point is the surface point the pixel sees.  Forward only (gsx_icp_projective_targets)."""
    _C.require_cuda(K, "K")
    _C.require_cuda(prev_poses, "prev_poses")
    B = prev_poses.numel() // 16
    dev = prev_poses.device
    index = torch.empty((B, H * W), dtype=torch.int64, device=dev)
    tgt_p = torch.empty((B, H * W, 3), dtype=torch.float32, device=dev)
    tgt_n = torch.empty_like(tgt_p)
    geo, counts, cap, bound = None, None, 0, 0
    if pointclouds.has_points:
        _C.require_cuda(pointclouds._geo, "pointclouds (geometry rows)")
        geo, counts = pointclouds._geo.detach().contiguous(), pointclouds._counts_dev[pointclouds._cur]
        cap, bound = pointclouds.capacity, pointclouds._bound
    _C.launch("gsx_icp_projective_targets", geo, None, counts, cap, bound, K.detach().contiguous(), 16,
              prev_poses.detach().contiguous(), 16, B, int(H), int(W), int(target_splat_px), index, tgt_p, tgt_n, None)
    return index, tgt_p, tgt_n


def projective_intensity(pointclouds, K, prev_poses, H, W, target_splat_px=0):
    """The model image of the photometric term: (index (B,H*W) int64 as projective_targets gives it, I_m (B,H*W) the
    intensity (0.299 r + 0.587 g) + 0.114 b of the colour of each pixel's winning row, 0 where uncovered).  Forward only
    (gsx_icp_projective_targets)."""
    _C.require_cuda(K, "K")
    _C.require_cuda(prev_poses, "prev_poses")
    B = prev_poses.numel() // 16
    dev = prev_poses.device
    index = torch.empty((B, H * W), dtype=torch.int64, device=dev)
    tgt_p = torch.empty((B, H * W, 3), dtype=torch.float32, device=dev)
    tgt_n, I_m = torch.empty_like(tgt_p), torch.empty((B, H * W), dtype=torch.float32, device=dev)
    geo, col, counts, cap, bound = None, None, None, 0, 0
    if pointclouds.has_points:
        if not pointclouds.has_colors:
            raise ValueError("the photometric term needs a map with colours")
        _C.require_cuda(pointclouds._geo, "pointclouds (geometry rows)")
        geo, col = pointclouds._geo.detach().contiguous(), pointclouds._col.detach().contiguous()
        counts, cap, bound = pointclouds._counts_dev[pointclouds._cur], pointclouds.capacity, pointclouds._bound
    _C.launch("gsx_icp_projective_targets", geo, col, counts, cap, bound, K.detach().contiguous(), 16,
              prev_poses.detach().contiguous(), 16, B, int(H), int(W), int(target_splat_px), index, tgt_p, tgt_n, I_m)
    return index, I_m


def localize_projective(pointclouds, live_frame, prev_frame, dsratio, odomprov, target_splat_px=0,
                        photometric_weight=0.0, photometric_huber_delta=None):
    """ICPSLAM._localize with association='projective' as ONE C call (gsx_icp_localize_projective): the source
    is the live frame on the ds lattice at the previous pose, the target is the map rendered from the previous pose at
    full resolution (surfels with radii as disks when target_splat_px >= 1, see projective_targets), each source point
    is associated with the pixel it projects to.  Returns the new poses (B,1,4,4) = T_icp · prev pose.  No host
    synchronisation.  photometric_weight w > 0 adds the photometric term (the live frame's and the map's colours);
    w = 0 is the geometric call.  With odomprov.huber_delta or photometric_huber_delta set, the residuals are
    Huber-weighted at those scales."""
    live = live_frame.to_channels_last()
    B, _, H, W = live.shape
    dev = pointclouds.device
    _C.require_cuda(live.depth_image, "depth_image")
    _C.require_cuda(pointclouds._geo, "pointclouds (geometry rows)")
    depth, d_bs = _frame_base(live.depth_image, H * W)
    K = live.intrinsics.contiguous()
    prev = prev_frame.poses.contiguous()
    out = torch.empty((B, 1, 4, 4), dtype=torch.float32, device=dev)
    mode, lambda_max, Bp, B2p, nu = _solver_params(odomprov)
    dth = odomprov.dist_thresh
    args = (pointclouds._geo.contiguous(), pointclouds._counts_dev[pointclouds._cur], pointclouds.capacity,
            pointclouds._bound, depth, d_bs, K, 16, prev, 16, B, H, W, int(dsratio), mode, int(odomprov.numiters),
            float(odomprov.damp), 0 if dth is None else 1, 0.0 if dth is None else float(dth), lambda_max, Bp, B2p, nu,
            out, 16)
    rgb, rgb_bs, col = None, 0, None
    if photometric_weight:
        if not pointclouds.has_colors or live.rgb_image is None:
            raise ValueError("photometric_weight > 0 needs a map with colours and a live frame with rgb_image")
        _C.require_cuda(live.rgb_image, "rgb_image")
        rgb, rgb_bs = _frame_base(live.rgb_image, H * W * 3)
        col = pointclouds._col.contiguous()
    ws = _ProjectiveWorkspace.get(dev, B, H, W, int(dsratio), photometric_weight > 0)
    _C.launch("gsx_icp_localize_projective", *args, ws, ws.numel(), int(target_splat_px), col, rgb, rgb_bs,
              float(photometric_weight), _huber_scale(getattr(odomprov, "huber_delta", None)),
              _huber_scale(photometric_huber_delta))
    return out


def _huber_scale(delta):
    """The float32 Huber scale the C entry points take: +inf (None) leaves the residual unweighted."""
    return math.inf if delta is None else float(delta)


def localize_projective_taped(pointclouds, live_frame, prev_frame, dsratio, odomprov, target_splat_px=0,
                              photometric_weight=0.0, photometric_huber_delta=None):
    """The differentiable counterpart of `localize_projective`, bit-identical poses: the index image comes from
    gsx_render_views, the target images are gathers of the map rows at that index (so the gradient reaches the rows that
    won a pixel, each at most one), and the batched ICP chain runs with the projective association.  With
    target_splat_px >= 1 the index and depth come from render_pointclouds(max_splat_px=target_splat_px), and at a pixel
    a disk row won the target point is the K1 global vertex of that depth from the previous pose (the gradient reaches
    the live depth, the previous pose and the winning rows' positions and normals; the radius gets none).
    photometric_weight w > 0 adds the photometric term through _JointNormalEqBatchedFn: the model colour image is the
    gather of the map's colours at the index image (the gradient reaches the colours of the winning rows), the source
    colours are the live rgb on the lattice, and the previous pose gets the gradient of q = T_prev^-1 s and R_prev too.
    The gradient w.r.t. the intrinsics reaches the poses through the live points (K1), the disk depths of the splatted
    targets and their surface points (R3d, K1) and the photometric row; the index image and the association use K only
    to choose pixels and carry none.  odomprov.huber_delta and photometric_huber_delta weigh the residuals as
    localize_projective does, through the Huber-weighted ops, so the poses stay the fused call's bit for bit.
    live_frame.poses must be the previous poses.  Returns (B,1,4,4)."""
    from ..slam.icpslam import _compose_canonical
    from ..structures.rgbdimages import RGBDImages
    from ..structures.utils import render_pointclouds

    frames_pc = downsample_rgbdimages(live_frame, dsratio)
    live = live_frame.to_channels_last()
    B, _, H, W = live.shape
    dev = pointclouds.device
    Kg = live.intrinsics  # values: carries d/dK
    K = Kg.detach().contiguous()  # pixel choices only
    prev = prev_frame.poses
    prev_d = prev.detach().contiguous()
    if target_splat_px:
        splat = render_pointclouds(pointclouds, Kg, prev, H, W, max_splat_px=target_splat_px)
        index = splat.index.view(B, H * W)
    else:
        index = torch.empty((B, H * W), dtype=torch.int64, device=dev)
        _C.launch("gsx_render_views", pointclouds._geo.detach().contiguous(), None,
                  pointclouds._counts_dev[pointclouds._cur], pointclouds.capacity, pointclouds._bound, K, 16, prev_d, 16,
                  B, 1, H, W, index, None, None, None, None)
    covered = (index >= 0).unsqueeze(-1)
    rows = index.clamp(min=0).unsqueeze(-1).expand(B, H * W, 3)

    def target(padded):  # (one zero row appended: an element, or a batch, of empty maps still gathers)
        padded = torch.cat([padded, padded.new_zeros(B, 1, 3)], 1)
        return torch.where(covered, torch.gather(padded, 1, rows), torch.zeros((), dtype=padded.dtype, device=dev))

    tgt_p, tgt_n = target(pointclouds.points_padded), target(pointclouds.normals_padded)
    if target_splat_px:
        # the pixels a disk row (radius > 0, normal != 0) won, decided on the detached rows: no gradient
        radii = pointclouds.radii_padded.detach()[..., 0]
        radius = torch.gather(torch.cat([radii, radii.new_zeros(B, 1)], 1), 1, index.clamp(min=0))
        disk = covered[..., 0] & (radius > 0) & (tgt_n.detach() != 0).any(-1)
        surface = RGBDImages(splat.depth.new_zeros(B, 1, H, W, 3), splat.depth, Kg, prev).global_vertex_map
        tgt_p = torch.where(disk.unsqueeze(-1), surface.reshape(B, H * W, 3), tgt_p)
    src_counts = frames_pc._counts_dev[frames_pc._cur]
    dth = odomprov.dist_thresh
    tgt_p_d = tgt_p.detach().contiguous()
    assoc = lambda cur: project_associate(cur, src_counts, tgt_p_d, index, prev_d.view(B, 4, 4), K, H, W, dth)[1]
    mode, lambda_max, Bp, B2p, nu = _solver_params(odomprov)
    normal_eq = None
    huber = getattr(odomprov, "huber_delta", None)
    scales = (_huber_scale(huber), _huber_scale(photometric_huber_delta))
    if photometric_weight:
        if not pointclouds.has_colors or live.rgb_image is None:
            raise ValueError("photometric_weight > 0 needs a map with colours and a live frame with rgb_image")
        model_col = target(pointclouds.colors_padded)
        src_col = frames_pc.colors_padded
        if src_col.shape[1] == 0:  # _taped_icp_batched pads an empty source with one zero row; so do its colours
            src_col = src_col.new_zeros(B, 1, 3)
        prev_v = prev.reshape(B, 4, 4)
        normal_eq = lambda cur, t_p, t_n, idx: _JointNormalEqBatchedFn.apply(
            cur, src_col, t_p, t_n, model_col, prev_v, idx, index, src_counts, Kg, photometric_weight, H, W, scales)
    T, _ = _taped_icp_batched(frames_pc.points_padded, src_counts, tgt_p, tgt_n, None, None, mode, odomprov.numiters,
                              odomprov.damp, dth, lambda_max, Bp, B2p, nu, associate=assoc, normal_eq=normal_eq,
                              huber_delta=huber)
    return _compose_canonical(T, prev.squeeze(1)).unsqueeze(1)
