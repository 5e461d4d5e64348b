"""Argument checks of the bilateral depth filter (CPU only): gsx_depth_bilateral / gsx_depth_bilateral_bwd refuse bad
arguments before any CUDA call, and BilateralFilter and the SLAM drivers' keywords validate theirs."""
import ctypes

import pytest
import torch

import gradslam_b200 as gs
from gradslam_b200 import _C

OK = dict(n=2, H=8, W=8, radius=3, ss=2.0, sr=0.05)


def _fwd(depth=16, out=4096, den=None, n=2, H=8, W=8, radius=3, ss=2.0, sr=0.05):
    return _C.lib().gsx_depth_bilateral(depth, out, den, n, H, W, radius, ss, sr, None)


def _bwd(ptrs=(16, 4096, 8192, 12288, 16384), n=2, H=8, W=8, radius=3, ss=2.0, sr=0.05):
    return _C.lib().gsx_depth_bilateral_bwd(*ptrs, n, H, W, radius, ss, sr, None)


BAD = [dict(n=-1), dict(H=0), dict(W=0), dict(H=-3), dict(radius=0), dict(radius=8), dict(ss=0.0), dict(sr=-1.0),
       dict(ss=float("nan")), dict(sr=float("inf")), dict(ss=1e-30), dict(sr=1e30)]


@pytest.mark.parametrize("bad", BAD, ids=[",".join("%s=%s" % kv for kv in b.items()) for b in BAD])
def test_forward_and_backward_refuse_bad_extents_radius_and_sigmas(bad):
    # the pointers are never dereferenced: every refusal comes before a launch
    assert _fwd(**bad) != 0
    assert b"gsx_depth_bilateral" in _C.lib().gsx_last_error()
    assert _bwd(**bad) != 0
    assert b"gsx_depth_bilateral_bwd" in _C.lib().gsx_last_error()


def test_null_pointers_are_refused():
    assert _fwd(depth=None) != 0 and b"null" in _C.lib().gsx_last_error()
    assert _fwd(out=None) != 0 and b"null" in _C.lib().gsx_last_error()
    for i in range(5):
        ptrs = [16, 4096, 8192, 12288, 16384]
        ptrs[i] = None
        assert _bwd(tuple(ptrs)) != 0 and b"null" in _C.lib().gsx_last_error()


def test_overlapping_buffers_are_refused():
    nbytes = 2 * 8 * 8 * 4
    assert _fwd(depth=1024, out=1024 + nbytes - 4) != 0 and b"overlap" in _C.lib().gsx_last_error()
    assert _fwd(depth=1024 + 4, out=1024) != 0
    assert _fwd(depth=1024, out=1024) != 0
    assert _fwd(depth=1024, out=1024 + nbytes, den=1024 + 8) != 0  # den over depth
    assert _fwd(depth=1024, out=1024 + nbytes, den=1024 + nbytes + 8) != 0  # den over out
    assert _bwd((16, 4096, 8192, 12288, 12288 + 4)) != 0 and b"overlap" in _C.lib().gsx_last_error()
    assert _bwd((16, 4096, 8192, 12288, 16)) != 0


def test_no_images_is_a_no_op():
    assert _fwd(n=0) == 0
    assert _bwd(n=0) == 0


def test_bilateral_filter_validates_its_fields():
    f = gs.BilateralFilter(3, 2, 0.05)
    assert (f.radius, f.sigma_space, f.sigma_range) == (3, 2.0, 0.05) and isinstance(f.sigma_space, float)
    with pytest.raises(AttributeError):
        f.radius = 2  # frozen
    for args in ((0, 1.0, 0.1), (8, 1.0, 0.1), (2, 0.0, 0.1), (2, 1.0, -0.1), (2, float("nan"), 0.1),
                 (2, 1.0, float("inf")), (2, 1e-30, 0.1), (2, 1.0, 1e30)):
        with pytest.raises(ValueError):
            gs.BilateralFilter(*args)
    for args in ((2.0, 1.0, 0.1), (True, 1.0, 0.1), (2, "1", 0.1), (2, 1.0, None)):
        with pytest.raises(TypeError):
            gs.BilateralFilter(*args)


def test_filter_needs_a_cuda_tensor_and_a_depth_shape():
    f = gs.BilateralFilter(2, 1.5, 0.03)
    with pytest.raises(RuntimeError, match="CUDA"):
        gs.bilateral_filter_depth(torch.ones(1, 1, 4, 4, 1), f)
    with pytest.raises(TypeError):
        gs.bilateral_filter_depth(torch.ones(1, 1, 4, 4, 1), (2, 1.5, 0.03))


def test_slam_keywords_are_validated():
    f = gs.BilateralFilter(2, 1.5, 0.03)
    for cls in (gs.ICPSLAM, gs.PointFusion):
        m = cls(odom="icp", depth_filter=f, depth_filter_tracking_only=True, device="cpu")
        assert m.depth_filter is f and m.depth_filter_tracking_only is True
        m = cls(odom="gt", device="cpu")
        assert m.depth_filter is None and m.depth_filter_tracking_only is False
        with pytest.raises(TypeError):
            cls(odom="gt", depth_filter=(2, 1.5, 0.03), device="cpu")
        with pytest.raises(TypeError):
            cls(odom="gt", depth_filter=f, depth_filter_tracking_only=1, device="cpu")


def test_abi_signature_widths():
    # the image count is int64: 8 x 10 000 frames of a sequence are more images than one grid dimension holds
    assert _C.SIGNATURES["gsx_depth_bilateral"][1][3] is ctypes.c_int64
    assert _C.SIGNATURES["gsx_depth_bilateral_bwd"][1][5] is ctypes.c_int64
