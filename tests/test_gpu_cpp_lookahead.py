"""tests/cpp/test_lookahead.cpp (acb200::Candidates and lookahead() of include/acb200.hpp) on the GPU; and, without a
GPU, the same program linked against the dry-run library of tests/emu/.  The executables go to the test's temporary
directory: the repository tree may be read-only."""
import subprocess
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
CPP = ROOT / "tests" / "cpp"


def _build_and_run(exe, libdir, libname):
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-Werror", "-I", str(ROOT / "include"),
                           str(CPP / "test_lookahead.cpp"), "-o", str(exe), "-L", str(libdir), f"-l{libname}",
                           f"-Wl,-rpath,{libdir}"])
    r = subprocess.run([str(exe)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "all checks passed" in r.stdout, r.stdout + r.stderr


@pytest.mark.gpu
def test_cpp_lookahead_runs(tmp_path):
    _build_and_run(tmp_path / "test_lookahead", ROOT / "aho-corasick_b200", "acb200")


def test_cpp_lookahead_on_the_dry_run_library(tmp_path):
    sys.path.insert(0, str(ROOT / "tests" / "emu"))
    import build_emu
    lib = build_emu.build()
    _build_and_run(tmp_path / "test_lookahead_emu", lib.parent, "acb200_emu")
