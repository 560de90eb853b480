"""mm_devbuf (mashmap_b200/csrc/mm_devbuf.h), the owning device array of the host code: after a failed reserve the
array is empty and the runtime's pending error is cleared, so a context that returned MM_ENOMEM stays usable."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CUDA_HOME = os.environ.get("CUDA_HOME", "/usr/local/cuda")


@pytest.fixture(scope="module")
def devbuf_check(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("devbuf") / "devbuf_check")
    lib = os.path.join(CUDA_HOME, "lib64")
    cmd = ["g++", "-std=c++17", "-O1", "-Wall", "-Werror", "-I", os.path.join(ROOT, "mashmap_b200", "csrc"),
           "-I", os.path.join(CUDA_HOME, "include"), os.path.join(ROOT, "tests", "devbuf_check.cpp"), "-o", exe,
           "-L", lib, "-lcudart", f"-Wl,-rpath,{lib}"]
    p = subprocess.run(cmd, capture_output=True, text=True)
    assert p.returncode == 0, p.stderr
    return exe


def test_failed_reserve_without_device_leaves_empty_array(devbuf_check):
    p = subprocess.run([devbuf_check, "nodevice"], capture_output=True, text=True)
    if p.returncode == 77:
        pytest.skip("a CUDA device is present: test_failed_reserve_on_gpu covers it")
    assert p.returncode == 0, p.stdout + p.stderr


@pytest.mark.gpu
def test_failed_reserve_on_gpu(devbuf_check):
    p = subprocess.run([devbuf_check, "gpu"], capture_output=True, text=True)
    assert p.returncode == 0 and "ok" in p.stdout, p.stdout + p.stderr
