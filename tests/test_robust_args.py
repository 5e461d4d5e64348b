"""Argument checks of the Huber-weighted tracking (CPU only): the huber_delta / photometric_huber_delta keywords of the
providers and SLAM drivers, and the scales of the ICP C entry points, which refuse a bad scale or inconsistent colour
pointers before any CUDA call."""
import math

import pytest

import gradslam_b200 as gs
from gradslam_b200 import _C
from gradslam_b200.odometry import GradICPOdometryProvider, ICPOdometryProvider

BAD_TYPE = [True, "0.1", [0.1], 1j]
BAD_VALUE = [0.0, -0.1, -1, math.nan, math.inf, -math.inf, 1e39, 10 ** 400, 1e-50]


@pytest.mark.parametrize("cls", [ICPOdometryProvider, GradICPOdometryProvider])
def test_providers_validate_huber_delta(cls):
    assert cls(huber_delta=0.02).huber_delta == 0.02
    assert cls(huber_delta=1).huber_delta == 1
    assert cls().huber_delta is None
    for bad in BAD_TYPE:
        with pytest.raises(TypeError):
            cls(huber_delta=bad)
    for bad in BAD_VALUE:
        with pytest.raises(ValueError):
            cls(huber_delta=bad)
    with pytest.raises(TypeError):  # keyword-only
        cls(20, 1e-8, None, 0.02) if cls is ICPOdometryProvider else cls(20, 1e-8, None, 2.0, 1.0, 1.0, 200.0, 0.02)


@pytest.mark.parametrize("cls", [gs.ICPSLAM, gs.PointFusion])
def test_drivers_validate_both_scales(cls):
    s = cls(odom="gradicp", huber_delta=0.02, device="cpu")
    assert s.odomprov.huber_delta == 0.02
    s = cls(odom="icp", association="projective", photometric_weight=0.1, huber_delta=0.05,
            photometric_huber_delta=0.1, device="cpu")
    assert s.odomprov.huber_delta == 0.05 and s.photometric_huber_delta == 0.1
    assert cls(odom="gt", huber_delta=0.02, device="cpu").odomprov is None  # (no tracking: no effect)
    for name in ("huber_delta", "photometric_huber_delta"):
        for bad in BAD_TYPE:
            with pytest.raises(TypeError, match=name):
                cls(odom="gradicp", association="projective", photometric_weight=0.1, device="cpu", **{name: bad})
        for bad in BAD_VALUE:
            with pytest.raises(ValueError, match=name):
                cls(odom="gradicp", association="projective", photometric_weight=0.1, device="cpu", **{name: bad})
    with pytest.raises(ValueError, match="photometric_weight > 0"):
        cls(odom="gradicp", association="projective", photometric_huber_delta=0.1, device="cpu")
    with pytest.raises(ValueError, match="photometric_weight > 0"):
        cls(odom="gradicp", photometric_huber_delta=0.1, device="cpu")


# fake device addresses: none is dereferenced, every refusal comes before a launch
P = [4096 * (i + 1) for i in range(32)]
GOOD = [0.02, math.inf]
BAD_SCALES = [0.0, -0.5, math.nan, -math.inf]


def _align(delta):
    return _C.lib().gsx_icp_align(P[0], P[1], 16, P[2], P[3], P[4], 16, 1, None, 1, 2, 1e-8, 0, 0.0, 2.0, 1.0, 1.0,
                                  200.0, P[5], None, P[6], 1 << 20, delta, None)


def _localize(delta):
    return _C.lib().gsx_icp_localize(P[0], P[1], 64, 64, P[2], 16, P[3], 16, P[4], 16, 1, 4, 4, 1, 1, 2, 1e-8, 0, 0.0,
                                     2.0, 1.0, 1.0, 200.0, P[5], 64, P[6], 16, P[7], 64, 1, None, delta, None)


def _projective(delta, delta_p, w=0.1, col=P[8], rgb=P[9]):
    return _C.lib().gsx_icp_localize_projective(P[0], P[1], 64, 64, P[2], 16, P[3], 16, P[4], 16, 1, 4, 4, 1, 1, 2,
                                                1e-8, 0, 0.0, 2.0, 1.0, 1.0, 200.0, P[5], 16, P[6], 1 << 20, 0, col,
                                                rgb, 48, w, delta, delta_p, None)


def _normal_eq(delta):
    fwd = _C.lib().gsx_icp_normal_eq_batched_fwd(P[0], P[1], 16, P[2], P[3], 16, 1, P[4], P[5], P[6], 1 << 20, delta,
                                                 None)
    bwd = _C.lib().gsx_icp_normal_eq_batched_bwd(P[0], P[1], 16, P[2], P[3], 16, 1, P[4], P[5], P[6], P[7], P[8], delta,
                                                 None)
    return fwd, bwd


def _joint(delta, delta_p, w=0.1):
    fwd = _C.lib().gsx_icp_joint_normal_eq_batched_fwd(P[0], P[1], 16, P[2], P[3], P[4], P[5], P[6], 1, 4, 4, P[7],
                                                       P[8], P[9], w, P[10], P[11], 1 << 20, delta, delta_p, None)
    bwd = _C.lib().gsx_icp_joint_normal_eq_batched_bwd(P[0], P[1], 16, P[2], P[3], P[4], P[5], P[6], 1, 4, 4, P[7],
                                                       P[8], P[9], w, P[10], P[11], P[12], P[13], P[14], P[15], P[16],
                                                       None, P[17], 1 << 20, delta, delta_p, None)
    return fwd, bwd


def _error():
    return _C.lib().gsx_last_error().decode()


@pytest.mark.parametrize("bad", BAD_SCALES)
def test_icp_entry_points_refuse_a_bad_scale(bad):
    assert _align(bad) != 0 and "huber_delta" in _error()
    assert _localize(bad) != 0 and "huber_delta" in _error()
    for d, dp in ((bad, 0.1), (0.1, bad)):
        assert _projective(d, dp) != 0 and "huber_delta" in _error()
        for rc in _joint(d, dp):
            assert rc != 0 and "huber_delta" in _error()
    for rc in _normal_eq(bad):
        assert rc != 0 and "huber_delta" in _error()


def test_projective_entry_points_refuse_inconsistent_photometric_arguments():
    for col, rgb in ((None, P[9]), (P[8], None)):
        assert _projective(0.02, 0.1, col=col, rgb=rgb) != 0 and "colour" in _error()
    assert _projective(0.02, 0.1, w=0.0, col=None, rgb=None) != 0 and "photometric_weight > 0" in _error()
    for w in (-0.5, math.nan, math.inf):
        assert _projective(0.02, math.inf, w=w) != 0 and "photometric_weight" in _error()
        for rc in _joint(0.02, math.inf, w=w):
            assert rc != 0 and "photometric_weight" in _error()
    # null pointers of the joint op are refused before the scales are used
    fwd = _C.lib().gsx_icp_joint_normal_eq_batched_fwd(None, P[1], 16, P[2], P[3], P[4], P[5], P[6], 1, 4, 4, P[7],
                                                       P[8], P[9], 0.1, P[10], P[11], 1 << 20, 0.1, 0.1, None)
    assert fwd != 0 and "null" in _error()
