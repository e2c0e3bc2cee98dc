"""Builds libcloudini_b200.so (sm_90a) in-tree with nvcc. No torch extension machinery: the product is a plain
C-ABI shared library (include/cloudini_b200.h)."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB_DIR = os.path.join(HERE, "lib")
LIB = os.path.join(LIB_DIR, "libcloudini_b200.so")
SOURCES = ["cldn_host.cpp", "cldn_ros.cpp", "cldn_encode.cu", "cldn_decode.cu", "cldn_decode_tiles.cu", "cldn_sections.cu", "cldn_preproc.cu", "cldn_lz4.cu", "cldn_zstd.cu",
           "cldn_zstd_enc.cu", "cldn_blobs_async.cu", "cldn_api.cu"]
HEADERS = ["cldn_plan.h", "cldn_kernels.h", "cldn_device.cuh", "cldn_stage2.cuh", "cldn_decode_fast.cuh", "cldn_encode_fast.cuh", "cldn_encode_points.cuh", "../../include/cloudini_b200.h", "../../include/cloudini_b200_ros.h"]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC,-fvisibility=default", "-Xptxas=-v",
]


def _nvcc():
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if cand and (os.path.sep not in cand or os.path.exists(cand)):
            return cand
    return "nvcc"


def needs_build():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    return any(os.path.getmtime(os.path.join(CSRC, f)) > t for f in SOURCES + HEADERS)


def build(force=False, verbose=False):
    """Compile every translation unit for sm_90a and link the shared library. Returns the library path."""
    if not force and not needs_build():
        return LIB
    os.makedirs(LIB_DIR, exist_ok=True)
    obj_dir = os.path.join(HERE, "build")
    os.makedirs(obj_dir, exist_ok=True)
    nvcc = _nvcc()
    procs = []
    for src in SOURCES:
        obj = os.path.join(obj_dir, os.path.splitext(src)[0] + ".o")
        cmd = [nvcc, *NVCC_FLAGS, "-x", "cu", "-c", os.path.join(CSRC, src), "-o", obj]
        procs.append((src, obj, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    objs = []
    for src, obj, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            sys.stderr.write(out)
            raise RuntimeError(f"nvcc failed on {src}")
        if verbose:
            sys.stderr.write(out)
        objs.append(obj)
    cmd = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-shared", "-o", LIB, *objs, "-lcudart", "-ldl"]
    subprocess.check_call(cmd)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
