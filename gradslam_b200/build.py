"""Builds gradslam_b200/_lib/libgsx.so in-tree with nvcc for sm_90a (cross-compiles without a GPU)."""
import glob
import os
import subprocess
import sys

_HERE = os.path.dirname(os.path.abspath(__file__))
SRC_DIR = os.path.join(_HERE, "csrc")
OUT = os.path.join(_HERE, "_lib", "libgsx.so")

# -fmad=false: the kernels' decisions must be bit-identical to the CPU oracle (no FMA contraction).
# Where an FMA is wanted (the float64 polynomial of gsx_exp.cuh, the dual-number refinements) it is written as fma().
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-fmad=false", "-std=c++17",
              "--shared", "-Xcompiler", "-fPIC"]


def sources():
    return sorted(glob.glob(os.path.join(SRC_DIR, "*.cu")))


def needs_build():
    if not os.path.exists(OUT):
        return True
    deps = sources() + glob.glob(os.path.join(SRC_DIR, "*.cuh")) + [os.path.join(_HERE, "..", "include", "gsx.h")]
    return any(os.path.getmtime(d) > os.path.getmtime(OUT) for d in deps)


def build(force=False, verbose=False):
    if not force and not needs_build():
        return OUT
    os.makedirs(os.path.dirname(OUT), exist_ok=True)
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    cmd = [nvcc] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-o", OUT] + sources()
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        sys.stderr.write(res.stdout + res.stderr)
        raise RuntimeError("nvcc failed building libgsx.so")
    if verbose:
        print(res.stderr)
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
