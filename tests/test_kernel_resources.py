"""Occupancy assumptions of the kernels, checked at compile time (`nvcc -Xptxas -v`, no GPU needed):
the narrow prefilter geometry runs 1 024 threads per CTA (at most 64 registers per thread), the
wide geometry relies on two 512-thread CTAs per SM (again 64), and nothing may spill."""
import re
import shutil
import subprocess
import tempfile
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
CSRC = ROOT / "aho-corasick_b200" / "csrc"


def ptxas_info(source):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not Path(nvcc).exists():
        pytest.skip("nvcc not available")
    with tempfile.TemporaryDirectory() as tmp:
        r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v",
                            "-c", str(CSRC / source), "-o", str(Path(tmp) / "o.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    out = {}
    name = None
    for line in r.stderr.splitlines():
        m = re.search(r"Compiling entry function '(\S+)'", line)
        if m:
            name = m.group(1)
            out[name] = {}
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and name:
            out[name]["spill"] = int(m.group(1)) + int(m.group(2))
        m = re.search(r"Used (\d+) registers", line)
        if m and name:
            out[name]["regs"] = int(m.group(1))
    return out


def test_prefilter_kernel_register_budget():
    info = {k: v for k, v in ptxas_info("acb_prefilter.cu").items() if "prefilter_kernel" in k}
    assert len(info) == 48   # [mode][masked][static / per-CTA / global tiles] x {stride 1, dense, stride 2 narrow, wide}
    for name, v in info.items():
        assert v["spill"] == 0, name
        # 65 536 registers per SM: 1 024 threads (narrow) or 2 x 512 threads (wide) => 64 per thread
        assert v["regs"] <= 64, (name, v["regs"])


def test_walk_and_helper_kernels_do_not_spill():
    for name, v in ptxas_info("acb_kernels.cu").items():
        if "acb" in name:
            assert v["spill"] == 0, name
