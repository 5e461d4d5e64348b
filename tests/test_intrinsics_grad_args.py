"""Argument checks of gsx_backproject_normals_bwd_intrinsics and its scratch size: they run before any launch, so they
are testable without a GPU."""
import ctypes
import math

import pytest

from gradslam_b200 import _C

FAKE = 256  # a non-null, 16-byte aligned pointer value that is never dereferenced: every call below is refused first


def _call(**kw):
    a = dict(depth=FAKE, intrinsics=FAKE, g_depth=FAKE, poses=None, g_poses=None, g_K=FAKE, scratch=FAKE,
             scratch_bytes=_C.lib().gsx_backproject_normals_bwd_intrinsics_scratch_bytes(2, 3, 8, 8), B=2, L=3, H=8, W=8)
    a.update(kw)
    return _C.lib().gsx_backproject_normals_bwd_intrinsics(
        a["depth"], 64, a["intrinsics"], 16, a["poses"], 48, a["B"], a["L"], a["H"], a["W"], None, None, None, None,
        a["g_depth"], a["g_poses"], a["g_K"], a["scratch"], a["scratch_bytes"], None)


def test_scratch_size_holds_the_pose_and_the_intrinsics_partials():
    lib = _C.lib()
    for B, L, H, W in [(1, 1, 2, 2), (8, 2, 480, 640), (3, 5, 17, 23)]:
        tiles = (H * W + 255) // 256
        n = lib.gsx_backproject_normals_bwd_intrinsics_scratch_bytes(B, L, H, W)
        assert n >= B * L * tiles * (12 + 4) * 4
        assert n >= lib.gsx_backproject_normals_bwd_scratch_bytes(B, L, H, W)
    assert lib.gsx_backproject_normals_bwd_intrinsics_scratch_bytes(1, 1, 1, 4) < 0
    assert lib.gsx_backproject_normals_bwd_intrinsics_scratch_bytes(-1, 1, 4, 4) < 0


@pytest.mark.parametrize("field", ["depth", "intrinsics", "g_depth"])
def test_refuses_null_pointers(field):
    assert _call(**{field: None}) != 0
    assert b"null pointer" in _C.lib().gsx_last_error()


@pytest.mark.parametrize("kw", [dict(scratch=None), dict(scratch_bytes=0),
                                dict(scratch_bytes=_C.lib().gsx_backproject_normals_bwd_scratch_bytes(2, 3, 8, 8))],
                         ids=["null", "zero", "pose_only_size"])
def test_refuses_a_scratch_too_small_for_the_intrinsics_partials(kw):
    """The scratch of the pose-only backward is not enough once g_intrinsics is requested."""
    assert _call(**kw) != 0
    assert b"scratch too small" in _C.lib().gsx_last_error()


def test_refuses_bad_extents():
    assert _call(H=1) != 0
    assert _call(B=70000, L=1) != 0


def test_render_and_joint_backward_entry_points_refuse_bad_intrinsics_arguments():
    lib = _C.lib()
    n = lib.gsx_render_splats_bwd_intrinsics_scratch_bytes(2, 3, 8, 8)
    assert n >= lib.gsx_render_views_bwd_scratch_bytes(2, 3, 8, 8) + 2 * 3 * 1 * 4 * 4
    assert lib.gsx_render_splats_bwd_intrinsics_scratch_bytes(0, 1, 8, 8) < 0
    call = lambda K, scratch, nbytes, M: lib.gsx_render_splats_bwd_intrinsics(
        FAKE, FAKE, 16, K, 16, FAKE, 48, FAKE, 2, 3, 8, 8, FAKE, None, None, None, None, None, None, FAKE, scratch,
        nbytes, M, None)
    assert call(None, FAKE, n, 2) != 0 and b"null pointer" in lib.gsx_last_error()
    for scratch, nbytes in ((None, n), (FAKE, n - 1)):
        assert call(FAKE, scratch, nbytes, 2) != 0 and b"scratch too small" in lib.gsx_last_error()
    assert call(FAKE, FAKE, n, 17) != 0 and b"max_splat_px" in lib.gsx_last_error()
    m = lib.gsx_icp_joint_normal_eq_batched_bwd_scratch_bytes(2, 300)
    assert m >= 2 * 2 * 12 * 4 * 2
    jcall = lambda g_prev, nbytes: lib.gsx_icp_joint_normal_eq_batched_bwd(
        FAKE, FAKE, 300, FAKE, FAKE, FAKE, FAKE, FAKE, 2, 8, 8, FAKE, FAKE, FAKE, ctypes.c_float(0.1), FAKE, FAKE, FAKE,
        FAKE, FAKE, FAKE, g_prev, FAKE, FAKE, nbytes, math.inf, math.inf, None)
    assert jcall(None, m) != 0 and b"null pointer" in lib.gsx_last_error()
    assert jcall(FAKE, m - 1) != 0 and b"scratch too small" in lib.gsx_last_error()
