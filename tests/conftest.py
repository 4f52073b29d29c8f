import os
import subprocess
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))
if str(ROOT / "tests") not in sys.path:
    sys.path.insert(0, str(ROOT / "tests"))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: test needs a CUDA device (run on an H100)")
    # The oracle is test infrastructure: build it on demand (gcc only, ~1 s).
    so = ROOT / "oracle" / "libac_oracle.so"
    src = ROOT / "oracle" / "ac_oracle.c"
    if not so.exists() or so.stat().st_mtime < src.stat().st_mtime:
        subprocess.check_call(["make", "-C", str(ROOT / "oracle")], stdout=subprocess.DEVNULL)


def _has_cuda():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


def pytest_collection_modifyitems(config, items):
    if _has_cuda():
        return
    if os.environ.get("ACB_EMULATE") == "1":
        # dry run against the product's kernel sources compiled for the CPU (tests/emu/): "device"
        # pointers are host pointers, one CTA at a time, CUDA threads as fibers.  Tests that need
        # torch.cuda still fail -- select with -k
        import ctypes
        sys.path.insert(0, str(ROOT / "tests" / "emu"))
        import build_emu
        import aho_corasick_b200 as ab
        from aho_corasick_b200 import packed
        lib = ctypes.CDLL(str(build_emu.build(asan=os.environ.get("ACB_EMU_ASAN") == "1")))
        ab._declare(lib)
        packed._declare(lib)
        ab._lib = lib
        packed._lib = lib
        return
    if os.environ.get("ACB_FAKE_DEVICE") == "1":
        # dry run of the GPU test programs against the CPU oracle (tests/fake_device.py); tests that
        # need device-resident haystacks still fail -- select with -k
        import fake_device
        fake_device.install()
        return
    skip = pytest.mark.skip(reason="no CUDA device in this container")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)
