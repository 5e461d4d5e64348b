"""Float64 reference of the joint geometric and photometric normal-equation op (_JointNormalEqBatchedFn,
gsx_icp_joint_normal_eq_batched_fwd / _bwd, d/dK included, include/gsx.h) for one batch element, with error bounds
for the float32 kernels.  Test infrastructure only.

The statement is photometric_oracle's (tests/photometric_oracle.py) at a GIVEN association: the geometric row of every
row i with idx[i] >= 0 (projective_oracle._rows) and, where the associated pixel is photometrically valid
(photometric_oracle.stencil on the index image, the model image being the intensity of the model colours), the
photometric row (photometric_oracle.photometric_rows), both with their float32 constants (0.299f, 0.587f, 0.114f, 0.5f,
the float32 weight w).  `joint_sums` evaluates it in the inputs' dtype and autograd through it is the reference of the
backward; from float32 inputs promoted to float64 it is the reference of the kernels.

Error bounds.  `_pair_rows` evaluates the same expressions once more in (value, magnitude, running error)
arithmetic.  The running error e bounds, to first order in u = 2^-24, |float32 result - exact| / u of every
intermediate (Wilkinson's running error analysis, one rounding per operation, the float32 inputs and constants exact):
e(a +- b) = e_a + e_b + |a +- b|, e(a b) = e_a |b| + |a| e_b + |a b|, e(a / b) = (e_a + |a/b| e_b) / |b| + |a/b|.  The
per-row products of the 28 sums carry their row's e (the photometric product is added to the geometric one in the
accumulator, which e includes); the kernels then reduce the rows with a 5-level warp butterfly, 8 warps in order and
the blocks in order, 13 + blocks additions per row, each erring by at most u times the sum of |terms| below it:

    |sums_kernel - sums| <= u (sum_rows e + (13 + blocks) sum_rows |term|)          (`sum_bound`).

A plain magnitude bound (d u times the expression evaluated with |.| and sums of absolute values: m(a +- b) = m_a + m_b,
m(a b) = m_a m_b, m(a / b) = (m_a + |a/b| m_b) / |b|, d = the rounding depth, R_F = 80 for these products) holds too,
but the photometric row cancels inside itself (I(j+1) - I(j-1), k_2 - u, R c, s x c): its magnitude is 15-80 times its
value, its products' 200-6000 times, and a bound that loose cannot see the rows of a whole block go missing.  The
magnitudes serve the backward:

The backward is a sum over paths of products of local partials.  Differentiating the pair arithmetic's magnitudes with
respect to the input magnitudes gives, for each input, the sum over paths of the products of the partials' magnitudes
(d(m_a m_b)/d m_a = m_b >= |b|, and the quotient's partials are |1/b| and |a/b^2|): the magnitude of the backward.
The kernels evaluate those partials with dual numbers.  The derivative part of a product a b is a' b + a b', so if
every operand's derivative has depth <= 2 d + c the product's has <= 2 (d_a + d_b + 1) + c, and likewise for sums; a
quotient (a' - q b') / b by the denominator den (depth D = 8) adds at most 2 D + 2 more.  The photometric row A_p
(depth R_A = 39) passes through three such quotients, so its derivative has depth <= 2 R_A + 3 (2 D + 2) = 132.  The
adjoint weight dL/dA_p = w (g r + sum_q g A_q) has depth R_A + 9 (a product, 7 additions, the weight); it multiplies
the derivative (+1), six such products are added (+5), and the chain to the pose, the colours or the stencil pixels
adds at most 3: every per-row gradient term has depth <= R_B = 132 + 48 + 9 = 189 (the geometric row's are shallower).
The per-row outputs (g_src, g_src_col) err by at most R_B u m', the scattered ones (g_tgt, g_tgt_n, g_model_col, summed
by index_add_ in any order over at most c rows per pixel) by (R_B + c) u m', and g_prev, g_K (each row's term reduced
like the sums, depth 13 + blocks) by (13 + blocks) u sum_rows |term| + R_B u m', where the per-row terms come from
per-row leaf copies of prev and K (as tests/test_gpu_intrinsics_grad.py's _term_scale does for K1).

Huber scales (delta, delta_p: the op's huber=(huber_delta, photometric_huber_delta), robust_oracle's weights).  The
kernels get the scales as float32 (`scales` rounds them the same way) and decide each row's branch on its float32
residual, r or r_p, evaluated in their operation order: `float32_residuals` restates it bit for bit (the library builds
with -fmad=false).  A row inside its scale (|r| <= delta, equality inside) adds the unweighted products; outside, with
a = |r| and h = delta / a, the geometric row adds h (A_p A_q), h (A_p r), delta ((a + a) - delta) and the photometric
row (w h_p) (A_p A_q), (w h_p) (A_p r_p), w (delta_p ((a_p + a_p) - delta_p)) with w h_p = w (delta_p / a_p).  The
float64 values and autograd are evaluated on the float32 branch, so at a tie the inside branch's derivative applies.
The pair arithmetic adds |.| (exact: e and m unchanged) and states those expressions in the same order; the sum bound
follows as above.  The backward of an outside row (huber_adjoint) adds depth: r_p has depth 4 (the intensities 3, the
difference 1), h_p = delta_p / a_p 5 (delta_p exact), w h_p 6.  The A_p adjoint (w h_p) v, v = g r_p + sum_q g A_q
of depth R_A + 8, gets depth R_A + 8 + 6 + 1 = R_A + 15 instead of R_A + 9: every A_p path gains 6 levels,
R_B_ROBUST = R_B + 6.  The r_p adjoint w (-(h_p / r_p) Q + 2 g_27 (h_p r_p)), Q the sum of 21 products g (A_p A_q)
(depth 2 R_A + 2 + 21), has depth 2 R_A + 36, and the colours' chain adds 2: 2 R_A + 38 = 116 < R_B.  The geometric
row's A and r have depth <= 4, so its adjoints stay far below.  R_B_ROBUST applies only when a scale is finite."""
import math

import torch

import photometric_oracle as ph
import projective_oracle as po
import robust_oracle as ro

U32 = 2.0 ** -24
BLOCK = 256  # rows per block of the kernels (kIcpBlock)
R_F = 80  # the products of the sums
R_A, D = 39, 8  # the photometric row A_p, the projection's denominator
R_B = (2 * R_A + 3 * (2 * D + 2)) + (R_A + 9) + 9
R_H = 6  # w h_p = w (delta_p / |r_p|) of an outside photometric row
R_B_ROBUST = (2 * R_A + 3 * (2 * D + 2)) + (R_A + 8 + R_H + 1) + 9
NAMES = ("src", "src_col", "tgt", "tgt_n", "model_col", "prev", "K")
_IU = torch.triu_indices(6, 6)


def blocks_of(ns_stride):
    """Reduction blocks of a call whose padded row count is ns_stride."""
    return max(1, math.ceil(ns_stride / BLOCK))


def scales(delta, delta_p):
    """The Huber scales as the kernels get them: float32 (+inf stays +inf)."""
    return tuple(float(torch.tensor(float(d), dtype=torch.float32)) for d in (delta, delta_p))


def float32_residuals(src, src_col, tgt, tgt_n, model_col, idx, index, H, W):
    """The residuals the kernels decide the Huber branches on, in float32 with their operation order: r (rows with
    idx >= 0, source order), r_p (those of them with a photometric row) and vj (which rows have one)."""
    f = lambda t: t.detach().float()
    _, b = po._rows(f(src), f(tgt), f(tgt_n), idx)
    I_m = ph.intensity(f(model_col))
    valid = ph.stencil(I_m.unsqueeze(0), index.unsqueeze(0), H, W)[0][0]
    keep = idx >= 0
    j = idx[keep]
    vj = valid[j]
    return b[:, 0], ph.intensity(f(src_col)[keep][vj]) - I_m[j[vj]], vj


def joint_sums(src, src_col, tgt, tgt_n, model_col, prev, K, idx, index, H, W, w, delta=math.inf, delta_p=math.inf):
    """One element: src, src_col (n, 3) its rows (i < count); tgt, tgt_n, model_col (H*W, 3); prev, K (4, 4);
    idx (n,) int64 associated pixel or -1, only covered pixels; index (H*W,) int64, -1 = uncovered.  -> (28,) in the
    inputs' dtype: the upper triangle of A^T A + w A_p^T A_p row by row, A^T b + w A_p^T r_p, b^T b + w r_p^T r_p;
    with a finite Huber scale delta / delta_p, the rows' Huber-weighted products summed (module docstring)."""
    A, b = po._rows(src, tgt, tgt_n, idx)
    I_m = ph.intensity(model_col)
    valid, gu, gv = ph.stencil(I_m.unsqueeze(0), index.unsqueeze(0), H, W)
    Ap, rp = ph.photometric_rows(src, ph.intensity(src_col), idx, valid[0], gu[0], gv[0], I_m, prev, K)
    delta, delta_p = scales(delta, delta_p)
    if math.isinf(delta) and math.isinf(delta_p):
        AtA, Atb, bb = ph._normal_equations(A, b, Ap, rp, w)
        return torch.cat([AtA[_IU[0], _IU[1]], Atb[:, 0], bb.view(1)])
    r32, rp32, _ = float32_residuals(src, src_col, tgt, tgt_n, model_col, idx, index, H, W)
    geo = ro.row_products(A, b[:, 0], delta, inside=r32.abs() <= delta)
    pho = ro.row_products(Ap, rp[:, 0], delta_p, w=torch.tensor(w, dtype=torch.float32).to(A.dtype),
                          inside=rp32.abs() <= delta_p)
    return geo.sum(0) + pho.sum(0)


class _P:
    """(value, magnitude, running error) arithmetic; see the module docstring."""
    __slots__ = ("v", "m", "e")

    def __init__(self, v, m, e=None):
        self.v, self.m = v, m
        self.e = torch.zeros_like(v.detach()) if e is None else e

    def __add__(a, b):
        v = a.v + b.v
        return _P(v, a.m + b.m, a.e + b.e + v.detach().abs())

    def __sub__(a, b):
        v = a.v - b.v
        return _P(v, a.m + b.m, a.e + b.e + v.detach().abs())

    def __mul__(a, b):
        v = a.v * b.v
        av, bv = a.v.detach().abs(), b.v.detach().abs()
        return _P(v, a.m * b.m, a.e * bv + av * b.e + v.detach().abs())

    def __truediv__(a, b):
        q = a.v / b.v
        qa, bv = q.detach().abs(), b.v.detach().abs()
        return _P(q, (a.m + qa * b.m) / bv, (a.e + qa * b.e) / bv + qa)

    def __neg__(a):
        return _P(-a.v, a.m, a.e)

    def __abs__(a):
        return _P(a.v.abs(), a.m, a.e)


def _where(mask, a, b):
    """Row by row: pair a where mask, else pair b."""
    return _P(torch.where(mask, a.v, b.v), torch.where(mask, a.m, b.m), torch.where(mask, a.e, b.e))


def _huber_pairs(prods, r, wt, delta, inside):
    """The 28 products of rows with residual pair r, as pairs: inside rows keep prods (their unweighted products, times
    wt for the photometric row when wt is given); outside ones get h (A_p A_q), h (A_p r), delta ((a + a) - delta), h =
    delta / a, or with wt (wt h) (..) and wt (delta ((a + a) - delta)), wt h = wt (delta / a).  prods: (products A_p A_q
    and A_p r (27 pairs, unweighted), the 28 inside pairs)."""
    raw, kept = prods
    if math.isinf(delta):
        return kept
    a = abs(r)
    one = _const(1.0, r.v)
    a_out = _where(inside, one, a)  # (inside rows never divide)
    d = _const(delta, r.v)
    h = d / a_out
    rho = d * ((a_out + a_out) - d)
    if wt is not None:
        h, rho = wt * h, wt * rho
    return [_where(inside, k, o) for k, o in zip(kept, [h * p for p in raw] + [rho])]


def _const(x, like):
    c = torch.tensor(x, dtype=torch.float32).to(like.dtype)  # the kernels' float32 constant
    return _P(c, c.abs())


def _intensity(c):
    """c: three pairs -> (0.299 r + 0.587 g) + 0.114 b."""
    wr, wg, wb = (_const(x, c[0].v) for x in (0.299, 0.587, 0.114))
    return (wr * c[0] + wg * c[1]) + wb * c[2]


def _pair_rows(x, mx, idx, index, H, W, w, prev_rows=None, K_rows=None, delta=math.inf, delta_p=math.inf):
    """The 28 per-row products in pair arithmetic, (28, n_rows) values and magnitudes, for the rows with idx >= 0.
    x: dict NAMES -> float tensors (values); mx: the same -> magnitudes (leaves of the backward's magnitude);
    prev_rows / K_rows: optional (n_rows, 12) per-row copies of the first three rows of prev and K used for the values
    (leaves of the per-row terms).  Values are bit-identical to po._rows / ph.photometric_rows in the same dtype.
    delta, delta_p: Huber scales (the branches are the float32 residuals')."""
    delta, delta_p = scales(delta, delta_p)
    keep = idx >= 0
    j = idx[keep]
    n = int(j.numel())
    P = lambda name, rows: _P(x[name][rows], mx[name][rows])
    s, s_col = P("src", keep), P("src_col", keep)
    comp = lambda p, c: _P(p.v[:, c], p.m[:, c])
    sx, sy, sz = (comp(s, c) for c in range(3))
    tp, tn = P("tgt", j), P("tgt_n", j)
    nx, ny, nz = (comp(tn, c) for c in range(3))
    px, py, pz = (comp(tp, c) for c in range(3))
    A = [nx, ny, nz, nz * sy - ny * sz, nx * sz - nz * sx, ny * sx - nx * sy]
    r = (nx * (px - sx) + ny * (py - sy)) + nz * (pz - sz)
    raw = [A[p] * A[q] for p in range(6) for q in range(p, 6)] + [A[p] * r for p in range(6)]
    geo = raw + [r * r]
    if not (math.isinf(delta) and math.isinf(delta_p)):
        r32, rp32, _ = float32_residuals(*(x[k] for k in ("src", "src_col", "tgt", "tgt_n", "model_col")), idx, index,
                                         H, W)
        geo = _huber_pairs((raw, geo), r, None, delta, r32.abs() <= delta)

    # photometric rows: the stencil's validity and g_u, g_v at j (values of the model colours, any dtype)
    I_m = ph.intensity(x["model_col"])
    valid = ph.stencil(I_m.unsqueeze(0), index.unsqueeze(0), H, W)[0][0]
    vj = valid[j]
    jv = j[vj]
    mc = lambda off: [comp(P("model_col", jv + off), c) for c in range(3)]
    half = _const(0.5, x["src"])
    gu = half * (_intensity(mc(1)) - _intensity(mc(-1)))
    gv = half * (_intensity(mc(W)) - _intensity(mc(-W)))
    sub = lambda p: _P(p.v[vj], p.m[vj])
    rp = _intensity([sub(comp(s_col, c)) for c in range(3)]) - _intensity(mc(0))
    sx, sy, sz = sub(sx), sub(sy), sub(sz)

    def entries(name, rows):  # the first three rows of a 4x4, as 12 pairs per photometric row
        if rows is not None:
            v = rows[vj]
        else:
            v = x[name][:3].reshape(1, 12).expand(int(vj.sum()), 12)
        m = mx[name][:3].reshape(1, 12).expand(v.shape[0], 12)
        return [_P(v[:, e], m[:, e]) for e in range(12)]

    T, k = entries("prev", prev_rows), entries("K", K_rows)
    R = [T[4 * a + b] for a in range(3) for b in range(3)]  # R[a][b] at 3 a + b
    t = [T[3], T[7], T[11]]
    ri = [R[3 * b + a] for a in range(3) for b in range(3)]  # T^-1 rotation R^T
    ti = [((-R[0 + i]) * t[0] + (-R[3 + i]) * t[1]) + (-R[6 + i]) * t[2] for i in range(3)]
    qx, qy, qz = (((ri[3 * a] * sx + ri[3 * a + 1] * sy) + ri[3 * a + 2] * sz) + ti[a] for a in range(3))
    hx, hy, hz = (((k[4 * a] * qx + k[4 * a + 1] * qy) + k[4 * a + 2] * qz) + k[4 * a + 3] for a in range(3))
    one = _const(1.0, hz.v)
    den = _P(torch.where(hz.v != 0, hz.v, one.v), torch.where(hz.v != 0, hz.m, one.m), torch.where(hz.v != 0, hz.e, one.e))
    u, v = hx / den, hy / den
    cc = [gu * ((k[i] - u * k[8 + i]) / den) + gv * ((k[4 + i] - v * k[8 + i]) / den) for i in range(3)]
    cx, cy, cz = (((R[3 * a] * cc[0] + R[3 * a + 1] * cc[1]) + R[3 * a + 2] * cc[2]) for a in range(3))
    Ap = [cx, cy, cz, cz * sy - cy * sz, cx * sz - cz * sx, cy * sx - cx * sy]
    wt = _const(w, x["src"])
    raw = [Ap[p] * Ap[q] for p in range(6) for q in range(p, 6)] + [Ap[p] * rp for p in range(6)]
    pho = [wt * p for p in raw] + [wt * (rp * rp)]
    if not math.isinf(delta_p):
        pho = _huber_pairs((raw, pho), rp, wt, delta_p, rp32.abs() <= delta_p)

    def scatter(p):  # the photometric products at the rows that have them, 0 elsewhere
        z = lambda t: torch.zeros(n, dtype=t.dtype).masked_scatter(vj, t)
        return _P(z(p.v), z(p.m), z(p.e))

    out = [g + scatter(p) for g, p in zip(geo, pho)]
    stack = lambda f: torch.stack([f(o) for o in out])
    return stack(lambda o: o.v), stack(lambda o: o.m), stack(lambda o: o.e), (A, r), (Ap, rp), vj


def reference(inputs, idx, index, H, W, w, blocks, g=None, delta=math.inf, delta_p=math.inf):
    """inputs: dict NAMES -> one element's float32 tensors (CPU; src, src_col cut at the element's count);
    idx (n,), index (H*W,) int64; blocks: reduction blocks of the call (blocks_of(ns_stride)); g: optional (28,)
    upstream gradient; delta, delta_p: the Huber scales of the call.  -> dict: "sums" (28,) float64, "sum_bound" (28,);
    with g also "grad" and "grad_bound", dicts NAMES -> float64 tensors of the inputs' shapes (the bottom rows of prev
    and K get 0 and bound 0)."""
    delta, delta_p = scales(delta, delta_p)
    R = R_B if math.isinf(delta) and math.isinf(delta_p) else R_B_ROBUST
    x = {k: v.detach().double().clone().requires_grad_(True) for k, v in inputs.items()}
    sums = joint_sums(*(x[k] for k in NAMES), idx, index, H, W, w, delta, delta_p)
    out = {"sums": sums.detach()}
    mx = {k: v.detach().abs().requires_grad_(True) for k, v in x.items()}
    rows = int((idx >= 0).sum())
    xd = {k: v.detach() for k, v in x.items()}
    prev_rows = x["prev"].detach()[:3].reshape(1, 12).expand(rows, 12).clone().requires_grad_(True)
    K_rows = x["K"].detach()[:3].reshape(1, 12).expand(rows, 12).clone().requires_grad_(True)
    vals, mags, errs, *_ = _pair_rows(xd, mx, idx, index, H, W, w, prev_rows, K_rows, delta, delta_p)
    out["row_err"], out["row_abs"] = errs.sum(1).detach(), vals.detach().abs().sum(1)
    out["sum_bound"] = U32 * (out["row_err"] + (13 + blocks) * out["row_abs"])
    if g is None:
        return out
    g = g.detach().double()
    grads = torch.autograd.grad((sums * g).sum(), [x[k] for k in NAMES], allow_unused=True, materialize_grads=True)
    out["grad"] = dict(zip(NAMES, grads))
    # the per-row terms of g_prev and g_K, and the magnitude of every gradient
    vj_any = prev_rows.shape[0] > 0
    terms = (torch.autograd.grad((vals * g.view(28, 1)).sum(), [prev_rows, K_rows], allow_unused=True,
                                 materialize_grads=True) if vj_any else (prev_rows, K_rows))
    gm = torch.autograd.grad((mags * g.abs().view(28, 1)).sum(), [mx[k] for k in NAMES], allow_unused=True,
                             materialize_grads=True)
    gm = dict(zip(NAMES, gm))
    # rows summed into one pixel of the scattered gradients: the associated pixel, and the five stencil pixels
    P = H * W
    j = idx[idx >= 0]
    per_pixel = torch.bincount(j, minlength=P).max().item() if j.numel() else 0
    st = (j.unsqueeze(1) + torch.tensor([0, -1, 1, -W, W])).clamp(0, P - 1).reshape(-1)
    per_stencil = torch.bincount(st, minlength=P).max().item() if st.numel() else 0
    bound = {"src": R * U32 * gm["src"], "src_col": R * U32 * gm["src_col"],
             "tgt": (R + per_pixel) * U32 * gm["tgt"], "tgt_n": (R + per_pixel) * U32 * gm["tgt_n"],
             "model_col": (R + per_stencil) * U32 * gm["model_col"]}
    for name, term in (("prev", terms[0]), ("K", terms[1])):
        b = torch.zeros(4, 4, dtype=torch.float64)
        b[:3] = ((13 + blocks) * U32 * term.detach().abs().sum(0)).view(3, 4)
        bound[name] = b + R * U32 * gm[name]
        bound[name][3] = 0.0
    out["grad_bound"] = {k: v.detach() for k, v in bound.items()}
    out["row_terms"] = {"prev": terms[0].detach(), "K": terms[1].detach()}
    return out


def synthetic_element(H, W, n_rows, K, prev, seed, unassociated=0.2, holes=0.08):
    """Inputs of one element of the op: target images of a surface 0.5-5 m in front of the camera prev (camera to
    world), an index image with holes (a `holes` share of pixels uncovered: zero target point, normal and colour), and
    n_rows world-frame source points near the targets of covered pixels, a share `unassociated` of them with idx = -1.
    The first rows visit every covered pixel of the two outer rows and columns of each side, so the border and its
    inner neighbours are associated.  K, prev: (4,4) float64.  -> (dict NAMES -> float32 tensors, idx (n_rows,),
    index (H*W,))."""
    g = torch.Generator().manual_seed(seed)
    P = H * W
    index = torch.arange(P, dtype=torch.int64)
    index[torch.rand(P, generator=g) < holes] = -1
    cov = index >= 0
    hh, ww = torch.meshgrid(torch.arange(H, dtype=torch.float64), torch.arange(W, dtype=torch.float64), indexing="ij")
    z = 0.5 + 4.5 * torch.rand(H, W, generator=g, dtype=torch.float64)
    Kd, T = K.double(), prev.double()
    y = (hh - Kd[1, 2]) / Kd[1, 1] * z
    x = (ww - Kd[0, 2] - Kd[0, 1] * y / z) / Kd[0, 0] * z
    cam = torch.stack([x, y, z], -1).view(P, 3)
    tgt = cam @ T[:3, :3].t() + T[:3, 3]
    nrm = torch.nn.functional.normalize(torch.randn(P, 3, generator=g, dtype=torch.float64) * 0.3
                                        + torch.tensor([0.0, 0.0, -1.0], dtype=torch.float64), dim=1) @ T[:3, :3].t()
    col = torch.rand(P, 3, generator=g, dtype=torch.float64)
    zero = lambda t: torch.where(cov.unsqueeze(1), t, torch.zeros_like(t))
    tgt, nrm, col = zero(tgt), zero(nrm), zero(col)
    h_all, w_all = torch.arange(P) // W, torch.arange(P) % W
    edge = ((h_all < 2) | (h_all >= H - 2) | (w_all < 2) | (w_all >= W - 2)) & cov
    covered = torch.nonzero(cov)[:, 0]
    idx = covered[torch.randint(0, covered.numel(), (n_rows,), generator=g)]
    first = torch.nonzero(edge)[:, 0][:n_rows]
    idx[:first.numel()] = first
    src = cam[idx] @ T[:3, :3].t() + T[:3, 3] + 0.01 * torch.randn(n_rows, 3, generator=g, dtype=torch.float64)
    off = torch.rand(n_rows, generator=g) < unassociated
    off[:first.numel()] = False
    idx[off] = -1
    inputs = {"src": src, "src_col": torch.rand(n_rows, 3, generator=g, dtype=torch.float64), "tgt": tgt,
              "tgt_n": nrm, "model_col": col, "prev": T, "K": Kd}
    return {k: v.float() for k, v in inputs.items()}, idx, index


def within(got, want, bound):
    """-> (ok, largest error-to-bound ratio) of float tensors of one shape; entries with bound 0 must be exact."""
    err = (got.detach().cpu().double() - want.detach().cpu().double()).abs()
    ok = bool((err <= bound).all())
    pos = bound > 0
    ratio = float((err[pos] / bound[pos]).max()) if pos.any() else 0.0
    return ok, ratio
