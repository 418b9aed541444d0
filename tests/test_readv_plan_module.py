"""The read planners (curvine_b200/csrc/host/readv_plan.{h,cc}) build with a plain C++ compiler: only include/ and csrc/host on the include
path, no CUDA header among the dependencies, no warning.  They are geometry and validation over a FileBlocks, so they stay testable and
reviewable apart from the device reader.  Host only: nothing here touches a GPU."""
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOST = os.path.join(ROOT, "curvine_b200", "csrc", "host")
SRC = os.path.join(HOST, "readv_plan.cc")


def _gxx(*args, tmp_path):
    gxx = shutil.which("g++")
    if gxx is None:
        pytest.skip("g++ is not installed")
    cmd = [gxx, "-std=c++17", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), "-I", HOST, *args]
    return subprocess.run(cmd, cwd=tmp_path, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)


def test_readv_plan_compiles_without_cuda_and_without_warnings(tmp_path):
    r = _gxx("-c", SRC, "-o", str(tmp_path / "readv_plan.o"), tmp_path=tmp_path)
    assert r.returncode == 0, r.stdout
    assert r.stdout == "", r.stdout
    deps = _gxx("-M", SRC, tmp_path=tmp_path)
    assert deps.returncode == 0, deps.stdout
    headers = deps.stdout.replace("\\\n", " ").split()[1:]
    assert SRC in headers and os.path.join(HOST, "readv_plan.h") in headers, headers
    # the repository's own prefix is left out: only what a header is called, and where else it comes from, may not name CUDA
    named = [os.path.relpath(h, ROOT) if h.startswith(ROOT + os.sep) else h for h in headers]
    assert not [h for h in named if "cuda" in h.lower()], named
