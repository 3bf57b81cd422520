"""ls::Buffer (laser_slam_b200/csrc/ls_buffer.cuh), the owner of every device and pinned array of the library, compiled by
a plain host compiler against cudart (tests/compile/buffer_check.cpp)."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CUDA = os.environ.get("CUDA_HOME", "/usr/local/cuda")


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("buffer") / "buffer_check")
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    lib = os.path.join(CUDA, "lib64")
    r = subprocess.run([cxx, "-std=c++17", "-O1", "-Wall", "-Werror", "-I", os.path.join(ROOT, "laser_slam_b200", "csrc"),
                        "-I", os.path.join(CUDA, "include"), os.path.join(ROOT, "tests", "compile", "buffer_check.cpp"),
                        "-o", out, "-L", lib, "-lcudart", f"-Wl,-rpath,{lib}"], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    return out


def test_failed_reserve_leaves_an_empty_buffer_and_no_error(exe):
    """Without a device every allocation fails: the buffer is null with capacity 0, the error is returned and
    cudaGetLastError() is clean afterwards; moved-from buffers are empty and destroying both is safe."""
    r = subprocess.run([exe, "nogpu"], capture_output=True, text=True)
    if "gpu present" in r.stdout:
        pytest.skip("a GPU is present: allocations succeed (test_buffer_on_the_device)")
    assert r.returncode == 0 and "ok" in r.stdout, r.stdout + r.stderr


@pytest.mark.gpu
def test_buffer_on_the_device(exe):
    """Growth, no change when need <= capacity, the pinned variant, moves, and a 2^50-byte request refused without
    allocating: the buffer is empty and no error is left behind."""
    r = subprocess.run([exe, "gpu"], capture_output=True, text=True)
    assert r.returncode == 0 and "ok" in r.stdout, r.stdout + r.stderr
