"""Kernel logic without a GPU: the `-m gpu` parity suite re-run against tests/cusim (TEST INFRASTRUCTURE ONLY).

tests/cusim compiles the *unmodified* CUDA sources of cloudini_b200/csrc with g++ against a shim of <cuda_runtime.h>
that emulates the CUDA execution model on the CPU (CTA threads = fibers, exact __syncthreads / warp-collective
semantics, CTAs dispatched in order on several OS threads so the decoupled look-backs really run concurrently). It is
not a fallback of the product — cloudini_b200/lib never contains it and bench.py / smoke() refuse it — and it proves
nothing about performance; it lets this CPU-only container catch indexing / scan / packing / protocol bugs before the
H100 run, which stays the parity gate. Every parity test of tests/test_gpu_parity.py runs unchanged, each
thread-resume order (forward, reverse, shuffled) must give identical bytes.
"""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "cusim"))


@pytest.fixture(scope="module")
def cusim_lib(lib_built):
    import platform
    if platform.machine() != "x86_64":
        pytest.skip("cusim's context switch is x86-64 only")
    import build_cusim
    return build_cusim.build()


def _run_gpu_suite(cusim_lib, extra_env, selection):
    env = dict(os.environ, CLDN_B200_LIB=cusim_lib, CLDN_B200_ALLOW_EMULATION="tests-only", **extra_env)
    cmd = [sys.executable, "-m", "pytest", "-x", "-q", "-m", "gpu", "-p", "no:cacheprovider", *selection]
    r = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=1500)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-2000:]
    return r.stdout


def test_parity_suite_under_emulation(cusim_lib):
    out = _run_gpu_suite(cusim_lib, {"CLDN_B200_FUZZ": "1", "CLDN_B200_FUZZ_SEEDS": "60"}, ["tests/test_gpu_parity.py", "tests/test_gpu_fast_paths.py", "tests/test_gpu_stage2_device.py", "tests/test_gpu_ros.py",
                                    "tests/test_gpu_zz_legacy_kernels.py", "tests/test_cpp_shim.py", "tests/test_gpu_concurrency.py"])
    assert " passed" in out and "failed" not in out


@pytest.mark.parametrize("order,workers", [("rev", "8"), ("rand", "3"), ("fwd", "1")])
def test_thread_order_and_cta_concurrency_do_not_matter(cusim_lib, order, workers):
    # (the "rand" run also delays every CTA start at random: CUSIM_JITTER)
    # reverse / shuffled resume order inside a CTA, 1..8 OS threads running CTAs: same bytes (look-backs, persistent
    # chunk claims and the in-kernel chunk walk are the protocols this exercises)
    sel = ["tests/test_gpu_parity.py", "tests/test_gpu_ros.py", "tests/test_gpu_zz_legacy_kernels.py", "-k",
           "float_clouds_sizes or adversarial or int_min or decode_modes or batch or c3_padded or v5_ or lossless or padded_and_unaligned or viz_ or raw_fields or gorilla_field or long_run"]
    env = {"CUSIM_ORDER": order, "CUSIM_WORKERS": workers}
    if order == "rand":
        env["CUSIM_JITTER"] = "1"
    _run_gpu_suite(cusim_lib, env, sel)


def test_product_entry_points_refuse_the_emulation(cusim_lib):
    # bench.py and smoke() must never report numbers / parity from the emulated library
    env = dict(os.environ, CLDN_B200_LIB=cusim_lib)
    env.pop("CLDN_B200_ALLOW_EMULATION", None)
    r = subprocess.run([sys.executable, "-c", "import cloudini_b200 as cb; cb.lib()"], cwd=ROOT, env=env, capture_output=True, text=True, timeout=120)
    assert r.returncode != 0 and "cusim test emulation" in r.stderr          # the package itself refuses it without the test flag
    env["CLDN_B200_ALLOW_EMULATION"] = "tests-only"                           # ... and bench / smoke refuse it even with the flag
    r = subprocess.run([sys.executable, "bench.py", "--steps", "1", "--warmup", "1"], cwd=ROOT, env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode != 0 and "cusim" in (r.stdout + r.stderr)
    r = subprocess.run([sys.executable, "-c", "import __graft_entry__ as g; g.smoke()"], cwd=ROOT, env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode != 0 and "cusim" in (r.stdout + r.stderr)


@pytest.mark.skipif(not os.environ.get("CLDN_CUSIM_ASAN"), reason="opt-in (CLDN_CUSIM_ASAN=1, ~10 min): the parity suite under an AddressSanitizer build of the emulation")
def test_no_out_of_bounds_access_under_asan(lib_built):
    # memcheck without a GPU: "device" memory is the instrumented heap, dynamic shared memory is allocated to the exact
    # size a launch asks for, so a kernel that reads or writes out of bounds is a reported error
    import build_cusim
    lib = build_cusim.build(asan=True)
    libasan = subprocess.check_output(["gcc", "-print-file-name=libasan.so"], text=True).strip()
    libstdcxx = subprocess.check_output(["gcc", "-print-file-name=libstdc++.so.6"], text=True).strip()
    env = dict(os.environ, CLDN_B200_LIB=lib, CLDN_B200_ALLOW_EMULATION="tests-only", LD_PRELOAD=f"{libasan} {libstdcxx}", ASAN_OPTIONS="detect_leaks=0", CLDN_B200_FUZZ="1",
               CLDN_B200_FUZZ_SEEDS="40")
    cmd = [sys.executable, "-m", "pytest", "-x", "-q", "-m", "gpu", "-p", "no:cacheprovider", "-k", "not c2_full_size",
           "tests/test_gpu_parity.py", "tests/test_gpu_ros.py", "tests/test_gpu_zz_legacy_kernels.py"]
    r = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=3000)
    assert r.returncode == 0 and "AddressSanitizer" not in (r.stdout + r.stderr), r.stdout[-3000:] + r.stderr[-3000:]


def test_racecheck_under_thread_sanitizer(lib_built):
    # racecheck without a GPU: every CUDA thread is a ThreadSanitizer fiber (switches carry no synchronisation), barriers and
    # __syncwarp publish their happens-before edges, so an unsynchronised pair of accesses to shared or global memory is a
    # report. The detector is checked against its own controls first, then every kernel family runs in strict mode (a
    # shuffle is NOT a memory fence, as the CUDA model defines it).
    import platform
    if platform.machine() != "x86_64":
        pytest.skip("cusim's context switch is x86-64 only")
    import build_cusim
    try:
        exe = build_cusim.build_racecheck()
    except subprocess.CalledProcessError as e:   # g++ without -fsanitize=thread support; a source the emulation cannot
        pytest.skip(f"ThreadSanitizer toolchain unavailable: {e}")   # rewrite (RuntimeError) is a FAILURE, not a skip

    def warnings(args, strict=False):
        env = dict(os.environ, TSAN_OPTIONS="halt_on_error=0 report_signal_unsafe=0", CUSIM_WORKERS="4")
        env.pop("LD_PRELOAD", None)
        if strict:
            env["CUSIM_TSAN_STRICT"] = "1"
        r = subprocess.run([exe, *args], env=env, capture_output=True, text=True, timeout=900)
        return (r.stdout + r.stderr).count("WARNING: ThreadSanitizer"), r

    probe, r = warnings(["--control-fixed"])
    if "FATAL: ThreadSanitizer" in r.stderr:
        pytest.skip("ThreadSanitizer cannot run in this environment: " + r.stderr[-200:])
    assert probe == 0
    assert warnings(["--control-racy"])[0] > 0                       # missing __syncthreads is seen
    assert warnings(["--control-shfl"])[0] == 0                      # shuffle as fence (lenient model)
    assert warnings(["--control-shfl"], strict=True)[0] > 0          # ... and not a fence in the strict model
    n, r = warnings([], strict=True)
    assert r.returncode == 0 and "racecheck_main: done" in r.stdout, r.stdout[-2000:] + r.stderr[-2000:]
    assert n == 0, r.stderr[-4000:]


def test_emulation_enforces_the_dynamic_shared_memory_launch_rule(tmp_path):
    # a launch with more than 48 KB of dynamic shared memory and no cudaFuncSetAttribute fails on the GPU with
    # cudaErrorInvalidValue; the emulation must not be more forgiving (tests/cusim/selftest_smem_rule.cpp)
    import platform
    if platform.machine() != "x86_64":
        pytest.skip("cusim's context switch is x86-64 only")
    here = os.path.join(ROOT, "tests", "cusim")
    exe = str(tmp_path / "smem_rule")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-pthread", "-w", "-I", here, os.path.join(here, "selftest_smem_rule.cpp"),
                           os.path.join(here, "cusim.cpp"), "-o", exe, "-ldl"])
    r = subprocess.run([exe], capture_output=True, text=True, timeout=60)
    assert r.returncode == 0, r.stdout + r.stderr
    r = subprocess.run([exe], env=dict(os.environ, CUSIM_SMEM_MONOTONIC="1"), capture_output=True, text=True, timeout=60)
    assert r.returncode == 0, r.stdout + r.stderr


def test_dynamic_shared_memory_limits_are_only_ever_raised(cusim_lib):
    # cudaFuncAttributeMaxDynamicSharedMemorySize is one value per kernel for the whole process. A launch site that set what
    # its own launch needs could lower it between another thread's set and that thread's launch, which then fails with
    # cudaErrorInvalidValue. Under CUSIM_SMEM_MONOTONIC=1 every lowering call fails, so a lowering call site is found with
    # one thread: e.g. viz preprocessing at step 16 and then at step 12 (32,800 -> 24,608 bytes for viz_compact_kernel).
    out = _run_gpu_suite(cusim_lib, {"CUSIM_SMEM_MONOTONIC": "1"},
                         ["tests/test_gpu_parity.py", "tests/test_gpu_ros.py", "tests/test_gpu_fast_paths.py", "tests/test_gpu_concurrency.py"])
    assert " passed" in out and "failed" not in out


def test_persistent_encoder_needs_no_co_resident_grid(cusim_lib):
    # The XYZI encoder launches an occupancy-sized persistent grid (2 SMs x 3 CTAs here) while the emulation runs only 2 CTAs
    # at a time, and the batch has many more tiles than the grid. A kernel whose CTAs waited for tiles of CTAs that have not
    # started would stall here until the timeout; the encoder takes its tiles in order from a ticket counter instead.
    env = dict(os.environ, CLDN_B200_LIB=cusim_lib, CLDN_B200_ALLOW_EMULATION="tests-only", CUSIM_WORKERS="2", CUSIM_SMS="2")
    code = r"""
import numpy as np, cloudini_b200 as cb
from cloudini_b200 import synth
from oracle.client import best_oracle
oracle = best_oracle()
n = 3 * 1024 * 6 + 517                                  # 19 full tiles and a partial one per frame
info, _ = synth.cloud_c2(n, seed=1)
clouds = [synth.cloud_c2(n, seed=10 + k)[1] for k in range(4)]
clouds[1].view(np.float32)[4 * 5000 + 1] = np.nan         # one tile of the exact path
enc = cb.PointcloudEncoder(info)
outs = [np.zeros(cb.MaxCompressedSize(info, n, True), dtype=np.uint8) for _ in clouds]
sizes = enc.encode_batch_host(clouds, outs)
for c, o, s in zip(clouds, outs, sizes):
    assert bytes(o[:s]) == oracle.encode(info, c), "differs from the oracle"
print("encoded", sum(sizes))
"""
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, env=env, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "encoded" in r.stdout, r.stdout[-2000:] + r.stderr[-3000:]


def test_concurrent_handles_under_thread_sanitizer(lib_built, tmp_path):
    # tests/cusim/threads_racecheck_main.cpp: four host threads, each with its own encoder, decoder and preprocessor for its
    # own layout, through every API; the library's host code is instrumented, so a data race on process-wide state (the
    # launch counter, lazily initialised statics, the shared memory limits, the stage-2 loader) is a report. Kernel races are
    # the job of test_racecheck_under_thread_sanitizer: the lenient model here.
    import platform
    if platform.machine() != "x86_64":
        pytest.skip("cusim's context switch is x86-64 only")
    import build_cusim
    from cloudini_b200.build import SOURCES
    try:
        build_cusim.build_racecheck()   # the instrumented kernels and C ABI (objects next to its own driver)
    except subprocess.CalledProcessError as e:
        pytest.skip(f"ThreadSanitizer toolchain unavailable: {e}")
    here = os.path.join(ROOT, "tests", "cusim")
    objs = [os.path.join(build_cusim.OUT_DIR, os.path.splitext(s)[0] + "_tsan.o") for s in SOURCES + ["cusim.cpp"]]
    drv, exe = str(tmp_path / "threads_main.o"), str(tmp_path / "threads_racecheck")
    subprocess.check_call(["g++", "-std=c++17", "-O0", "-g", "-fPIC", "-pthread", "-w", "-fsanitize=thread", "-I", here, "-I",
                           os.path.join(ROOT, "include"), "-x", "c++", "-c", os.path.join(here, "threads_racecheck_main.cpp"), "-o", drv])
    subprocess.check_call(["g++", "-fsanitize=thread", "-pthread", "-o", exe, drv, *objs, "-ldl"])
    env = dict(os.environ, TSAN_OPTIONS="halt_on_error=0 report_signal_unsafe=0", CUSIM_WORKERS="2")
    env.pop("LD_PRELOAD", None)
    env.pop("CUSIM_TSAN_STRICT", None)
    r = subprocess.run([exe], env=env, capture_output=True, text=True, timeout=1500)
    if "FATAL: ThreadSanitizer" in r.stderr:
        pytest.skip("ThreadSanitizer cannot run in this environment: " + r.stderr[-200:])
    assert r.returncode == 0 and "threads_racecheck: done" in r.stdout, r.stdout[-2000:] + r.stderr[-3000:]
    assert "WARNING: ThreadSanitizer" not in r.stderr, r.stderr[-6000:]
    # the control: a plain counter every job bumps is reported (the emulation's own locks do not order the host threads)
    r = subprocess.run([exe, "--control-racy"], env=env, capture_output=True, text=True, timeout=1500)
    assert "WARNING: ThreadSanitizer" in r.stderr and "g_control_counter" in r.stderr, r.stdout[-2000:] + r.stderr[-3000:]


def test_host_code_never_dereferences_device_memory(cusim_lib, tmp_path):
    # "device" memory is host memory in the emulation, so a host-side `*device_ptr` (a segmentation fault on the GPU box)
    # would pass unnoticed. CUSIM_HOSTCHECK=1 maps every cudaMalloc region inaccessible except while a kernel runs or a
    # cudaMemcpy / cudaMemset is in progress; the detector is checked against its own control first.
    here = os.path.join(ROOT, "tests", "cusim")
    exe = str(tmp_path / "hostcheck")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-pthread", "-w", "-I", here, os.path.join(here, "selftest_hostcheck.cpp"),
                           os.path.join(here, "cusim.cpp"), "-o", exe, "-ldl"])
    env = dict(os.environ, CUSIM_HOSTCHECK="1")
    assert subprocess.run([exe], env=env, capture_output=True, text=True, timeout=60).returncode == 0
    r = subprocess.run([exe, "--touch"], env=env, capture_output=True, text=True, timeout=60)
    assert r.returncode != 0 and "touched device memory" in r.stderr
    # CUSIM_ASYNC=1: a cudaMemcpyAsync(DeviceToHost) result arrives when the host synchronises with the stream (or an
    # event behind the copy), not before — reading it early yields 0xEE here, stale data on the GPU box
    r = subprocess.run([exe, "--async"], env=dict(env, CUSIM_ASYNC="1"), capture_output=True, text=True, timeout=60)
    assert r.returncode == 0, r.stdout + r.stderr
    out = _run_gpu_suite(cusim_lib, {"CUSIM_HOSTCHECK": "1", "CUSIM_ASYNC": "1"}, ["tests/test_gpu_parity.py", "tests/test_gpu_ros.py", "tests/test_gpu_zz_legacy_kernels.py"])
    assert " passed" in out and "failed" not in out
