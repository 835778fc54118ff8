"""Build glue (SURVEY 2*, reference CMakeLists.txt:1-30): the CMake target `rwkv_cuda` produces
build/librwkv_cuda.a, and the reference's own examples/storygen CMake project - copied into a scratch tree
at test time, unmodified - finds this engine through it (examples/storygen/CMakeLists.txt:35). No GPU needed
(nvcc cross-compiles); the second half needs /root/reference."""
import os
import shutil
import subprocess

import pytest

from util import ROOT

REF = "/root/reference"


def _run(cmd, **kw):
    r = subprocess.run(cmd, capture_output=True, text=True, **kw)
    assert r.returncode == 0, " ".join(cmd) + "\n" + r.stdout[-3000:] + r.stderr[-3000:]
    return r.stdout


@pytest.fixture(scope="module")
def static_lib(tmp_path_factory):
    if not shutil.which("cmake") or not (shutil.which("nvcc") or os.path.exists("/usr/local/cuda/bin/nvcc")):
        pytest.skip("cmake / nvcc not available")
    b = tmp_path_factory.mktemp("cmake_build")
    gen = ["-G", "Ninja"] if shutil.which("ninja") else []
    _run(["cmake", "-S", ROOT, "-B", str(b)] + gen)
    _run(["cmake", "--build", str(b), "-j", "8"])
    lib = os.path.join(str(b), "librwkv_cuda.a")
    assert os.path.exists(lib)
    return lib


def test_static_library_exports_both_surfaces(static_lib):
    nm = _run(["nm", "-C", "--defined-only", static_lib])
    for sym in ("rwkv_b200_load", "rwkv_b200_forward", "cuda_rwkv_parralel(", "setState(", "getOutput(", "freeTensors(", "load(std::"):
        assert sym in nm, sym
    assert "sm_90a" in subprocess.run(["cuobjdump", "-lelf", static_lib], capture_output=True, text=True).stdout


def test_reference_storygen_cmake_project_links(static_lib, tmp_path):
    src = os.path.join(REF, "examples", "storygen")
    if not os.path.exists(os.path.join(src, "CMakeLists.txt")):
        pytest.skip("/root/reference not present")
    tree = tmp_path / "tree"
    (tree / "examples").mkdir(parents=True)
    shutil.copytree(src, tree / "examples" / "storygen")          # the reference's project files, unmodified, scratch only
    os.symlink(os.path.join(ROOT, "include"), tree / "include")  # ../../include          (storygen CMakeLists.txt:20)
    (tree / "build").mkdir()
    os.symlink(static_lib, tree / "build" / "librwkv_cuda.a")    # ../../build/librwkv_cuda.a (CMakeLists.txt:35)
    b = tmp_path / "sg_build"
    gen = ["-G", "Ninja"] if shutil.which("ninja") else []
    _run(["cmake", "-S", str(tree / "examples" / "storygen"), "-B", str(b), "-DCMAKE_CUDA_ARCHITECTURES=90a"] + gen)
    _run(["cmake", "--build", str(b), "-j", "8"])
    exe = b / "storygen"
    assert exe.exists()
    # without a model file the program explains itself and stops (storygen.cpp:19-22)
    r = subprocess.run([str(exe)], cwd=str(b), capture_output=True, text=True, input="", timeout=60)
    assert "No model file found" in r.stderr or "Failed to load tokenizer" in r.stderr
