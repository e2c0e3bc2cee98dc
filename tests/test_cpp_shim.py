"""The header-only C++ shim (include/cloudini_b200/cloudini.hpp) mirrors the reference's Cloudini:: API on the C ABI."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# The executables are built into the test's temporary directory, never into the source tree (which may be read-only).


def _run_env(tmp_path):
    """The executables link against cloudini_b200/lib; when the suite is re-run against another build of the library
    (CLDN_B200_LIB: a tuning variant, or the cusim emulation under tests/test_cusim_kernels.py) that build is put first
    on the loader path under the linked name."""
    alt = os.environ.get("CLDN_B200_LIB")
    if not alt:
        return None
    os.makedirs(tmp_path / "lib", exist_ok=True)
    link = tmp_path / "lib" / "libcloudini_b200.so"
    if not link.exists():
        os.symlink(os.path.abspath(alt), link)
    return dict(os.environ, LD_LIBRARY_PATH=str(tmp_path / "lib"))


def _compile(lib_built, out_dir):
    exe = os.path.join(str(out_dir), "shim_roundtrip")
    cmd = ["g++", "-std=c++17", "-O1", "-I" + os.path.join(ROOT, "include"), os.path.join(ROOT, "tests", "cpp", "shim_roundtrip.cpp"),
           "-L" + os.path.dirname(lib_built), "-lcloudini_b200", "-Wl,-rpath," + os.path.dirname(lib_built), "-o", exe]
    subprocess.check_call(cmd)
    return exe


def test_shim_compiles_and_links(lib_built, tmp_path):
    assert os.path.exists(_compile(lib_built, tmp_path))


@pytest.mark.gpu
def test_shim_roundtrip_on_gpu(lib_built, tmp_path):
    exe = _compile(lib_built, tmp_path)
    out = subprocess.run([exe], capture_output=True, text=True, timeout=120, env=_run_env(tmp_path))
    assert out.returncode == 0, out.stdout + out.stderr
    assert "shim_roundtrip: ok" in out.stdout


# ---- cloudini_ros shim (include/cloudini_b200/ros_msg_utils.hpp) -------------------------------------------------------
def _compile_ros(lib_built, out_dir):
    exe = os.path.join(str(out_dir), "ros_shim_convert")
    cmd = ["g++", "-std=c++17", "-O1", "-I" + os.path.join(ROOT, "include"), os.path.join(ROOT, "tests", "cpp", "ros_shim_convert.cpp"),
           "-L" + os.path.dirname(lib_built), "-lcloudini_b200", "-Wl,-rpath," + os.path.dirname(lib_built), "-o", exe]
    subprocess.check_call(cmd)
    return exe


def test_ros_shim_compiles_and_links(lib_built, tmp_path):
    assert os.path.exists(_compile_ros(lib_built, tmp_path))


# (the GPU run of this executable lives at the end of tests/test_gpu_ros.py: it needs the N3 kernels, which have not
# had a hardware run yet, and this file sorts first)
