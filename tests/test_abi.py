"""The C-ABI library loads and exports exactly the symbols include/gsx.h declares (no compute calls: CPU only)."""
import ctypes
import os
import re

import pytest
import torch

from gradslam_b200 import _C

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _header():
    text = open(os.path.join(ROOT, "include", "gsx.h")).read()
    return re.sub(r"/\*.*?\*/", "", text, flags=re.S)


def _declared():
    return set(re.findall(r"\b(gsx_[a-z0-9_]+)\s*\(", _header()))


def test_header_and_binding_list_the_same_symbols():
    assert _declared() == set(_C.SIGNATURES)


def test_binding_matches_every_prototype_parameter_by_parameter():
    """A scalar bound with the wrong width (int for int64_t) would silently truncate a size: every prototype's return
    type and parameter kinds must be the ones SIGNATURES declares."""
    text = "\n".join(l for l in _header().splitlines() if not l.lstrip().startswith("#"))
    scalar = {"int": ctypes.c_int, "int64_t": ctypes.c_int64, "float": ctypes.c_float, "double": ctypes.c_double,
              "uint32_t": ctypes.c_uint32}
    result = {**scalar, "void": None, "const char *": ctypes.c_char_p}
    protos = re.findall(r"((?:const\s+)?[A-Za-z_]\w*\s*\**)\s*\b(gsx_\w+)\s*\(([^)]*)\)\s*;", text)
    assert {name for _, name, _ in protos} == set(_C.SIGNATURES)
    for ret, name, params in protos:
        want_args = []
        for p in params.split(","):
            p = p.strip()
            if p == "void":
                continue
            want_args.append(ctypes.c_void_p if "*" in p else scalar[" ".join(p.split()[:-1])])
        res, args = _C.SIGNATURES[name]
        assert res is result[" ".join(ret.replace("*", " *").split())], name
        assert args == want_args, name


@pytest.mark.parametrize("position", [0, 3])
def test_launch_refuses_a_cpu_tensor_before_calling_the_library(position, monkeypatch):
    calls = []
    monkeypatch.setitem(_C._entries, (_C.lib(), "gsx_icp_solve_fwd"), lambda *a: calls.append(a) or 0)
    args = [None, None, 1, None, None]
    args[position] = torch.zeros(28)
    with pytest.raises(RuntimeError, match=r"gsx_icp_solve_fwd takes CUDA tensors.*argument %d is on cpu" % position):
        _C.launch("gsx_icp_solve_fwd", *args)
    assert calls == []


def test_library_exports_every_declared_symbol():
    assert os.path.exists(_C.LIB_PATH), "libgsx.so was not built"
    handle = ctypes.CDLL(_C.LIB_PATH)
    for name in sorted(_declared()):
        assert hasattr(handle, name), name


def test_host_only_entry_points():
    lib = _C.lib()
    assert lib.gsx_version() == 200
    n = lib.gsx_fusion_workspace_bytes(8, 480, 640)
    assert n >= 8 * 480 * 640 * 16
    assert 0 < lib.gsx_fusion_workspace_stats_offset(8, 480, 640) < n
    # argument validation happens before any launch, so it is testable without a GPU
    rc = lib.gsx_backproject_normals_fwd(None, 0, None, 0, None, 0, 1, 1, 4, 4, None, None, None, None, None)
    assert rc != 0 and b"null" in lib.gsx_last_error()


@pytest.mark.parametrize("H,W,s_begin,frames", [(2, 2, 0, 1 << 30), (480, 640, 5, 1_789_570)],
                         ids=["one_tile", "600_tiles"])
def test_sequence_call_refuses_more_scan_epochs_than_a_state_word_holds(H, W, s_begin, frames):
    """K4's scan epoch is ticket / tiles + 1 and the ticket counts on through a call: gsx_pointfusion_sequence_gt refuses
    a call of (s_end - s_begin) * tiles >= 2^30 before any CUDA call, and leaves every buffer as it was.
    1 789 570 frames of 600 tiles is the first frame count past the bound (1 789 569 * 600 < 2^30)."""
    tiles = (H * W + 511) // 512
    assert frames * tiles >= 1 << 30 > (frames - 1) * tiles
    bufs = [torch.full((256,), -7.25) for _ in range(9)]  # geometry, colours, counts, depth, rgb, K, poses, ws, flag
    assert all(t.data_ptr() % 16 == 0 for t in bufs)
    geo, col, counts, depth, rgb, K, poses, ws, flag = (t.data_ptr() for t in bufs)
    s_end = s_begin + frames
    rc = _C.lib().gsx_pointfusion_sequence_gt(geo, col, counts, 16, 0, depth, rgb, K, poses, 1, s_end, s_begin, s_end,
                                              H, W, 0.05, 0.94, 0.6, ws, None, 0, 0.0, None, 0, 0.0, None, 0, flag,
                                              None)
    assert rc != 0
    assert b"split the call" in _C.lib().gsx_last_error()
    for t in bufs:
        assert torch.equal(t, torch.full((256,), -7.25))


def test_no_oracle_import_in_product_package():
    """The product never routes through the oracle (or any CPU fallback)."""
    pkg = os.path.join(ROOT, "gradslam_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith(".py"):
                src = open(os.path.join(dirpath, f)).read()
                assert "gsx_oracle" not in src and "import oracle" not in src, os.path.join(dirpath, f)


def test_peer_entry_points_check_their_arguments_without_a_gpu():
    """gsx_peer_*: argument validation happens before any CUDA call, so it is testable here."""
    import ctypes

    from gradslam_b200 import _C

    lib = _C.lib()
    buf = (ctypes.c_ubyte * 64)()
    off = ctypes.c_int64(0)
    assert lib.gsx_peer_export(None, buf, ctypes.byref(off), None) != 0
    assert b"gsx_peer_export" in lib.gsx_last_error()
    out = ctypes.c_void_p()
    assert lib.gsx_peer_open(None, 0, ctypes.byref(out)) != 0
    assert lib.gsx_peer_open(buf, -1, ctypes.byref(out)) != 0
    # a block wider than a pitch would overlap the next block
    assert lib.gsx_peer_copy_rows(ctypes.c_void_p(16), 32, ctypes.c_void_p(16), 64, 48, 2, None) != 0
    assert b"gsx_peer_copy_rows" in lib.gsx_last_error()
    # nothing to move is not an error (and touches no pointer)
    assert lib.gsx_peer_copy_rows(None, 32, None, 32, 0, 4, None) == 0
    assert lib.gsx_peer_close_all() == 0
