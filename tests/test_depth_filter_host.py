"""Exhaustive CPU check of exp32, the float32 exponential of the bilateral depth filter (gradslam_b200/csrc/
gsx_exp32.cuh): the header is compiled for the host with -ffp-contract=off (no FMA, as the library's -fmad=false) and
evaluated for EVERY float32 argument in [-17, 0].  Each result must equal the numpy statement of tests/
bilateral_oracle.py bit for bit, and lie within kExp32MaxUlps of float32(exp(float64 x)); exp32(+-0) = 1."""
import ctypes
import multiprocessing
import os
import subprocess
from concurrent.futures import ProcessPoolExecutor

import numpy as np
import pytest

import bilateral_oracle as bo

HERE = os.path.dirname(os.path.abspath(__file__))
CHUNK = 1 << 22


SO = os.path.join(HERE, "_build", "depth_filter_host.so")


def _load():
    lib = ctypes.CDLL(SO)
    lib.exp32_fill.argtypes = [ctypes.c_uint32, ctypes.c_uint32, ctypes.c_void_p]
    lib.exp32_max_ulps.restype = ctypes.c_int
    return lib


@pytest.fixture(scope="module")
def lib():
    os.makedirs(os.path.dirname(SO), exist_ok=True)
    src = os.path.join(HERE, "host", "depth_filter_host.cpp")
    subprocess.run(["g++", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-o", SO, src], check=True)
    return _load()


def _check_chunk(lo_hi):
    lo, hi = lo_hi
    return _check_range(_load(), lo, hi)


def _check_range(lib, lo, hi):
    """bit patterns [lo, hi): (mismatches against the numpy statement, max ulps against float32(exp(float64)))"""
    n = hi - lo
    got = np.empty(n, dtype=np.float32)
    lib.exp32_fill(lo, n, got.ctypes.data)
    x = (np.arange(n, dtype=np.uint32) + np.uint32(lo)).view(np.float32)
    want = bo.exp32(x)
    ref = np.exp(x.astype(np.float64)).astype(np.float32)
    ulps = np.abs(got.view(np.int32).astype(np.int64) - ref.view(np.int32))
    return int(np.count_nonzero(got.view(np.uint32) != want.view(np.uint32))), int(ulps.max())


def test_every_float32_argument_in_minus_17_to_0(lib):
    # negative floats: bit patterns grow with magnitude, from -0 (0x80000000) to -17; 1.1 G arguments
    lo, hi = int(np.float32(-0.0).view(np.uint32)), int(np.float32(-17.0).view(np.uint32)) + 1
    chunks = [(s, min(s + CHUNK, hi)) for s in range(lo, hi, CHUNK)]
    # numpy's float32 passes are serial: one process per core (spawned - the test process runs threads)
    with ProcessPoolExecutor(max_workers=min(8, os.cpu_count() or 1),
                             mp_context=multiprocessing.get_context("spawn")) as pool:
        res = list(pool.map(_check_chunk, chunks))
    assert sum(r[0] for r in res) == 0
    assert max(r[1] for r in res) <= lib.exp32_max_ulps() == 1


def test_zero_and_the_range_ends(lib):
    got = np.empty(1, dtype=np.float32)
    for z in (0.0, -0.0):
        lib.exp32_fill(int(np.float32(z).view(np.uint32)), 1, got.ctypes.data)
        assert got[0] == np.float32(1.0)
        assert bo.exp32(np.float32(z)) == np.float32(1.0)
    assert _check_range(lib, int(np.float32(0.0).view(np.uint32)), 1) == (0, 0)
