"""In-tree build of libacb200.so (hand-written sm_90a CUDA + C++ host) with nvcc."""
import os
import shutil
import subprocess
from pathlib import Path

HERE = Path(__file__).resolve().parent
CSRC = HERE / "csrc"
LIB = HERE / "libacb200.so"
SOURCES = ["acb_build.cpp", "acb_kernels.cu", "acb_prefilter.cu", "acb_comm.cu", "acb_api.cu"]
HEADERS = ["acb_build.hpp", "acb_plan.hpp", "acb_fingerprint.cuh", "acb_comm.hpp", "acb_device.cuh", "acb_ptx.cuh", "../../include/acb200.h", "../../include/acb200_debug.h"]
GENCODE = ["-gencode", "arch=compute_90a,code=sm_90a"]  # H100 (Hopper)
NVCC_FLAGS = [
    *GENCODE, "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC,-O3,-Wall", "-shared", "--expt-relaxed-constexpr",
]


def find_nvcc():
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and Path(cand).exists():
            return cand
    raise RuntimeError("nvcc not found")


def needs_build():
    if not LIB.exists():
        return True
    t = LIB.stat().st_mtime
    # this script counts as a source: a library built with other flags (another architecture) is stale
    return any((CSRC / s).stat().st_mtime > t for s in SOURCES + HEADERS + ["../build.py"])


def build_library(force=False, verbose=False):
    if not force and not needs_build():
        return LIB
    cmd = [find_nvcc(), *NVCC_FLAGS, *[str(CSRC / s) for s in SOURCES], "-o", str(LIB)]
    if verbose:
        cmd.insert(1, "-Xptxas=-v")
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("nvcc failed:\n" + r.stdout + r.stderr)
    if verbose:
        print(r.stdout + r.stderr)
    return LIB


if __name__ == "__main__":
    import sys
    print(build_library(force=True, verbose="-v" in sys.argv))
