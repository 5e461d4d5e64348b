"""CPU statements of the bilateral depth filter of gsx_filter.cu (include/gsx.h gsx_depth_bilateral).

* `exp32` and `bilateral_f32`: the float32 statement in numpy, operation for operation as the kernel computes it (every
  product and sum rounded to float32 on its own, no FMA) - the bit-exact target of the forward.
* `bilateral_f64`: the same filter in float64 torch, differentiable - the target of the backward.  The pairs it skips
  are the float32 statement's, so both differentiate the same function.
* `bilateral_bwd_formula`: the backward written out on its own (include/gsx.h), with the float64 sum of the absolute
  values of its terms for scaling tolerances.
Depth is an (n, H, W) stack of images.  A pixel is valid iff 0 < d < inf.
"""
import numpy as np
import torch

F32 = np.float32
LOG2E, LN2_HI, LN2_LO = F32("1.44269502"), F32("0.693145751953125"), F32("1.42860677e-06")
# 1/7!, 1/6!, ..., 1/2!, 1, 1: the Horner coefficients of gsx_exp32.cuh
POLY = tuple(F32(c) for c in ("1.98412698e-04", "1.38888889e-03", "8.33333377e-03", "4.16666679e-02",
                              "1.66666672e-01", "0.5", "1.0", "1.0"))
X_MIN = F32(-17.0)
MAX_RADIUS = 7


def exp32(x):
    """gsx::exp32 on a float32 array (stated on [-17, 0])."""
    x = np.asarray(x, dtype=F32)
    with np.errstate(invalid="ignore", over="ignore"):  # (outside [-17, 0] the value is not defined, only computed)
        k = np.rint(x * LOG2E)
        r = (x - k * LN2_HI) - k * LN2_LO
        p = POLY[0] * r + POLY[1]
        for c in POLY[2:]:
            p *= r
            p += c
        scale = ((k.astype(np.int32) + np.int32(127)).view(np.uint32) << np.uint32(23)).view(F32)
    p *= scale
    return p


def constants(sigma_space, sigma_range):
    """c_s, c_r: 1/(2 sigma^2) in float64, rounded once to float32."""
    return F32(1.0 / (2.0 * sigma_space * sigma_space)), F32(1.0 / (2.0 * sigma_range * sigma_range))


def _valid(a):
    return (a > 0) & (a < np.inf)


def _windows(d, radius):
    """(dv, du, neighbour image) in window order; out-of-image neighbours read 0 (invalid)."""
    n, H, W = d.shape
    r = radius
    pad = np.zeros((n, H + 2 * r, W + 2 * r), dtype=d.dtype)
    pad[:, r:r + H, r:r + W] = d
    for dv in range(-r, r + 1):
        for du in range(-r, r + 1):
            yield dv, du, pad[:, r + dv:r + dv + H, r + du:r + du + W]


def _pairs_f32(d, radius, c_s, c_r):
    """(dv, du, q, ok, x, keep) per window offset, in float32 as the kernel computes them."""
    with np.errstate(invalid="ignore", over="ignore"):
        for dv, du, q in _windows(d, radius):
            ok = _valid(q)
            dl = q - d
            x = -(F32(du * du + dv * dv) * c_s + (dl * dl) * c_r)
            yield dv, du, q, ok, x, ok & (x >= X_MIN)


def bilateral_f32(depth, radius, sigma_space, sigma_range):
    """The kernel's forward: (out, den) float32 (n, H, W); den = 0 at invalid centres."""
    d = np.ascontiguousarray(depth, dtype=F32)
    c_s, c_r = constants(sigma_space, sigma_range)
    num = np.zeros_like(d)
    den = np.zeros_like(d)
    for _, _, q, ok, x, keep in _pairs_f32(d, radius, c_s, c_r):
        w = np.where(keep, exp32(x), F32(0))
        num = num + w * np.where(ok, q, F32(0))
        den = den + w
    vp = _valid(d)
    with np.errstate(invalid="ignore", divide="ignore"):
        out = np.where(vp, num / den, d)
    return out, np.where(vp, den, F32(0))


def keep_masks(depth, radius, sigma_space, sigma_range):
    """The float32 statement's kept pairs, one (n, H, W) mask per window offset (window order)."""
    d = np.ascontiguousarray(depth, dtype=F32)
    c_s, c_r = constants(sigma_space, sigma_range)
    return [keep for *_, keep in _pairs_f32(d, radius, c_s, c_r)]


def bilateral_f64(depth, radius, sigma_space, sigma_range, keep=None):
    """The filter in float64 torch (differentiable w.r.t. depth, an (n, H, W) float64 tensor) on the float32 statement's
    pairs (`keep`, from keep_masks; computed from depth when None).  Returns (out, den)."""
    if keep is None:
        keep = keep_masks(depth.detach().cpu().numpy(), radius, sigma_space, sigma_range)
    c_s, c_r = (float(c) for c in constants(sigma_space, sigma_range))
    vp = (depth > 0) & (depth < float("inf"))
    d = torch.where(vp, depth, torch.zeros_like(depth))  # no NaN / inf reaches a derivative
    n, H, W = d.shape
    r = radius
    pad = torch.nn.functional.pad(d, (r, r, r, r))
    num = torch.zeros_like(d)
    den = torch.zeros_like(d)
    i = 0
    for dv in range(-r, r + 1):
        for du in range(-r, r + 1):
            q = pad[:, r + dv:r + dv + H, r + du:r + du + W]
            k = torch.from_numpy(keep[i]).to(d.device)
            w = torch.where(k, torch.exp(-((du * du + dv * dv) * c_s + (q - d) ** 2 * c_r)), torch.zeros_like(d))
            num = num + w * q
            den = den + w
            i += 1
    out = torch.where(vp, num / torch.where(vp, den, torch.ones_like(den)), depth)
    return out, torch.where(vp, den, torch.zeros_like(den))


def bilateral_bwd_formula(depth, g_out, radius, sigma_space, sigma_range):
    """g_depth of the written-out backward (include/gsx.h) in float64 numpy, and the float64 sum of the absolute values
    of its terms (each product split into its factors' magnitudes) at every pixel."""
    d32 = np.ascontiguousarray(depth, dtype=F32)
    keep = keep_masks(d32, radius, sigma_space, sigma_range)
    with torch.no_grad():
        out, den = (t.numpy() for t in bilateral_f64(torch.from_numpy(d32.astype(np.float64)), radius, sigma_space,
                                                     sigma_range, keep))
    c_s, c_r = (float(c) for c in constants(sigma_space, sigma_range))
    vp = _valid(d32)
    d = np.where(vp, d32.astype(np.float64), 0.0)
    out = np.where(vp, out, 0.0)  # (an invalid pixel's terms are all masked: keep NaN out of the products)
    g = np.asarray(g_out, dtype=np.float64)
    W_safe = np.where(vp, den, 1.0)
    self_sum = np.zeros_like(d)
    self_mag = np.zeros_like(d)
    cross = np.zeros_like(d)
    cross_mag = np.zeros_like(d)
    for (dv, du, ds), (_, _, os_), (_, _, Ws), (_, _, gs), k in zip(
            _windows(d, radius), _windows(out, radius), _windows(W_safe, radius), _windows(g, radius), keep):
        if dv == 0 and du == 0:
            continue
        w = np.where(k, np.exp(-((du * du + dv * dv) * c_s + (ds - d) ** 2 * c_r)), 0.0)
        self_sum += w * (ds - d) * (ds - out)
        self_mag += w * np.abs(ds - d) * np.abs(ds - out)
        with np.errstate(invalid="ignore", divide="ignore"):
            f = np.where(k, gs * (w / Ws), 0.0)
        cross += f * (1.0 - 2.0 * c_r * (d - os_) * (d - ds))
        cross_mag += np.abs(f) * (1.0 + 2.0 * c_r * np.abs(d - os_) * np.abs(d - ds))
    gq = np.where(vp, g * (1.0 + 2.0 * c_r * self_sum) / W_safe + cross, g)
    mag = np.where(vp, np.abs(g) * (1.0 + 2.0 * c_r * self_mag) / W_safe + cross_mag, np.abs(g))
    return gq, mag
