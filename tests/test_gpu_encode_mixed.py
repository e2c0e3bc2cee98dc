"""cldn_b200_encode_mixed_blobs (MixedEncoder): batches of clouds of any mix of layouts, compressions and dims.

Blob f must be byte-identical to cldn_b200_encoder_create(&infos[f]) + that frame's cldn_b200_encode_blobs, which for
NONE (and host-blob LZ4 / ZSTD) is the reference's PointcloudEncoder(infos[f]).encode(cloud_f). Every frame gets the
status and message that single-layout path gives it alone; a refused frame's output is not written.
"""
import ctypes as C
import os
import subprocess
import sys
import threading

import numpy as np
import pytest

import cloudini_b200 as cb

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_gpu_encode_blobs import (EMULATED, PAD_BYTE, SHUFFLED_LANES, _Buf, _device_u64, _encode_blobs, _launches,  # noqa: E402
                                   _layout, _src, _with_dims)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NONE, LZ4, ZSTD = cb.CompressionOption.NONE, cb.CompressionOption.LZ4, cb.CompressionOption.ZSTD
HOST, DEVICE, DEVICE_POINTS = cb.MEM_HOST, cb.MEM_DEVICE, cb.MEM_DEVICE_POINTS
MEMS = [HOST, DEVICE_POINTS, DEVICE]
MEM_IDS = ["host", "device_points", "device"]
MILLION = 70_000 if EMULATED else 1_000_000
MIX = ["xyzi", "xyz", "c3", "xyzirt", "lossless", "gorilla"]


def _dims(info, cloud):
    n = cloud.size // info.point_step if info.point_step else 0
    return (n, 1) if info.width == 0 and info.height == 0 else (info.width, info.height)


def _cap(info, cloud):
    n = cloud.size // info.point_step
    return cb.MaxCompressedSize(_with_dims(info, *_dims(info, cloud)), n, True)


def _frame(name, n, seed, version, comp, dims=False):
    info, cloud = _layout(name, n, seed, version)
    info.compression_opt = comp
    info.width, info.height = (n, 1) if dims else (0, 0)
    return info, cloud


def _mixed_frames(seed, comps, sizes=None):
    """Frames interleaving every layout of MIX, wire versions 3..5 and the compressions `comps`."""
    sizes = sizes or [0, 1, 40_000, MILLION, 32_769, 5_000, 32_768, 70_001, 3]
    frames = []
    for k in range(2 * len(MIX) + 1):
        frames.append(_frame(MIX[k % len(MIX)], sizes[k % len(sizes)], seed + k, 3 + k % 3, comps[k % len(comps)], dims=k % 4 == 1))
    return frames


def _run(me, frames, mem, caps=None, want_sizes=True):
    """encode_mixed_blobs on guarded buffers: (rc, message, statuses, frame errors, blobs, guards intact, untouched)."""
    n = len(frames)
    m = max(n, 1)
    caps = caps or [_cap(i, c) for i, c in frames]
    ins = [_src(c, mem != HOST) for _, c in frames]
    outs = [_Buf(cap, mem == DEVICE) for cap in caps]
    status, written = (C.c_int32 * m)(), (C.c_size_t * m)()
    rc = cb.lib().cldn_b200_encode_mixed_blobs(me._h, n, (cb._CInfo * m)(*[cb._to_c(i) for i, _ in frames]),
                                               (C.c_void_p * m)(*[b.ptr for b in ins]), (C.c_size_t * m)(*[c.size for _, c in frames]),
                                               (C.c_void_p * m)(*[o.ptr for o in outs]), (C.c_size_t * m)(*caps), mem, status,
                                               written if want_sizes else None)
    msg = cb.lib().cldn_b200_last_error().decode() if rc else ""
    if not want_sizes:
        me.sync()
        written = _device_u64(me.sizes_device_ptr(), n)
    bodies = [o.body() for o in outs]
    blobs = [bodies[f][:written[f]].tobytes() if status[f] == 0 else None for f in range(n)]
    guards = all(o.guards_intact() for o in outs) and all(i.guards_intact() for i in ins)
    return rc, msg, list(status), [me.frame_error(f) for f in range(n)], blobs, guards, [bool((b == PAD_BYTE).all()) for b in bodies]


def _alone(info, cloud, mem, stage2=False, cap=None):
    """(status, message, blob) of cldn_b200_encoder_create(&info) + encode_blobs of this frame alone."""
    c = cb._to_c(info)
    h = C.c_void_p()
    rc = cb.lib().cldn_b200_encoder_create(C.byref(c), -1, None, C.byref(h))
    if rc:
        return rc, cb.lib().cldn_b200_last_error().decode(), None
    enc = cb.PointcloudEncoder.__new__(cb.PointcloudEncoder)
    enc._h, enc._info = h, info
    if stage2:
        enc.set_stage2_on_device(True)
    n = cloud.size // info.point_step if info.point_step else 0
    w, hh = _dims(info, cloud)
    # DEVICE_POINTS blobs are the host blobs (cloudini_b200.h, cldn_mem_t)
    rc, msg, blobs, _, _ = _encode_blobs(enc, [cloud], mem == DEVICE, caps=[cap] if cap else [_cap(info, cloud) if n * info.point_step == cloud.size else 64],
                                         dims=[(w, hh)])
    enc.close()
    return rc, msg[len("frame 0: "):] if msg.startswith("frame 0: ") else msg, blobs[0] if blobs else None


def _device_stage2(info, mem, stage2):
    return info.compression_opt != NONE and (stage2 or (mem == DEVICE and info.compression_opt == LZ4))


def _same_blob(a, b, lossy_order):
    """Byte equality; where the emulation's shuffled lanes reorder the device LZ4 / ZSTD coders' matches, equal points."""
    if not lossy_order:
        return a == b
    d = cb.PointcloudDecoder().decode_blobs([a, b])
    return d[0][0] == d[1][0] == 0 and np.array_equal(d[0][2], d[1][2])


# ---- 1. the oracle, frame by frame -------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("mem", MEMS, ids=MEM_IDS)
def test_blobs_equal_the_oracle_frame_by_frame(oracle, mem):
    comps = [NONE, LZ4] if mem == DEVICE else [NONE, LZ4, ZSTD]
    frames = _mixed_frames(10 + mem, comps)
    me = cb.MixedEncoder()
    rc, msg, status, _, blobs, guards, _ = _run(me, frames, mem)
    assert rc == 0 and status == [0] * len(frames), msg
    assert guards, "a byte outside a frame's buffer changed"
    reference = oracle.kind.startswith("reference")
    for f, ((info, cloud), blob) in enumerate(zip(frames, blobs)):
        if info.compression_opt == NONE or (reference and mem != DEVICE):
            assert blob == oracle.encode(_with_dims(info, *_dims(info, cloud)), cloud), (f, info.version, info.compression_opt)
        else:   # device LZ4 is this library's coder; without the compiled reference, LZ4 / ZSTD against the single call
            st, m, want = _alone(info, cloud, mem)
            assert st == 0, m
            assert _same_blob(blob, want, SHUFFLED_LANES and _device_stage2(info, mem, False)), f


# ---- 2. the single-layout call -----------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("stage2", [False, True], ids=["library", "stage2_on_device"])
@pytest.mark.parametrize("mem", MEMS, ids=MEM_IDS)
def test_blobs_equal_the_single_layout_call(mem, stage2):
    comps = [NONE, LZ4, ZSTD] if stage2 or mem != DEVICE else [NONE, LZ4]
    frames = _mixed_frames(20 + mem, comps, [0, 1, 9_000, 32_769, 40_000, 2])
    me = cb.MixedEncoder()
    me.set_stage2_on_device(stage2)
    rc, msg, status, _, blobs, guards, _ = _run(me, frames, mem)
    assert rc == 0 and guards, msg
    for f, (info, cloud) in enumerate(frames):
        st, m, want = _alone(info, cloud, mem, stage2)
        assert st == 0, m
        assert _same_blob(blobs[f], want, SHUFFLED_LANES and _device_stage2(info, mem, stage2)), (f, info.compression_opt)


# ---- 3. a status per frame ---------------------------------------------------------------------------------------------
def _bad(kind, seed):
    """(info, cloud, capacity) of a frame the encoder refuses."""
    info, cloud = _frame("xyzi", 3000, seed, 5, NONE)
    cap = _cap(info, cloud)
    if kind == "short":
        cap -= 1
    elif kind == "17_bytes":
        cloud, cap = cloud[:17], 4096
    elif kind == "dims":
        info.width, info.height = 1000, 2
    elif kind == "offset":
        info.fields = [cb.PointField(f.name, f.offset + (20 if k == 3 else 0), f.type, f.resolution) for k, f in enumerate(info.fields)]
        cap = 1 << 16
    elif kind == "zstd_device":
        info.compression_opt = ZSTD
    return info, cloud, cap


@pytest.mark.gpu
@pytest.mark.parametrize("mem", MEMS, ids=MEM_IDS)
def test_statuses_per_frame(mem):
    kinds = ["short", "17_bytes", "dims", "offset"] + (["zstd_device"] if mem == DEVICE else [])
    good = _mixed_frames(30, [NONE, LZ4], [5_000, 0, 40_000, 1, 33_000])[:7]
    want_good = [_alone(i, c, mem)[2] for i, c in good]
    me = cb.MixedEncoder()
    for kind in kinds:
        for pos in (0, 3, len(good)):
            bi, bc, bcap = _bad(kind, pos)
            frames = good[:pos] + [(bi, bc)] + good[pos:]
            caps = [_cap(i, c) for i, c in good[:pos]] + [bcap] + [_cap(i, c) for i, c in good[pos:]]
            rc, msg, status, errors, blobs, guards, untouched = _run(me, frames, mem, caps)
            st, m, _ = _alone(bi, bc, mem, cap=bcap)
            assert st != 0 and status[pos] == st and errors[pos] == m, (kind, pos, status[pos], errors[pos], st, m)
            assert rc == st and msg == f"frame {pos}: {m}", (kind, msg)
            assert untouched[pos] and guards, kind
            got = blobs[:pos] + blobs[pos + 1:]
            assert all(s == 0 for k, s in enumerate(status) if k != pos)
            for f, (b, w) in enumerate(zip(got, want_good)):
                assert _same_blob(b, w, SHUFFLED_LANES and mem == DEVICE and good[f][0].compression_opt == LZ4), (kind, pos, f)
    # two bad frames: the lowest one is named
    b1, b2 = _bad("dims", 1), _bad("short", 2)
    frames = [good[0], (b1[0], b1[1]), good[1], (b2[0], b2[1])]
    rc, msg, status, errors, _, _, untouched = _run(me, frames, mem, [_cap(*good[0]), b1[2], _cap(*good[1]), b2[2]])
    assert status[0] == status[2] == 0 and status[1] == -1 and status[3] == -2
    assert rc == -1 and msg == f"frame 1: {errors[1]}" and untouched[1] and untouched[3]


# ---- 4. launches and ordering ------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_launches_are_the_groups_encode_batch_plus_one_and_sizes_can_stay_on_the_device():
    groups = [("xyzi", NONE), ("c3", NONE), ("xyzi", LZ4), ("xyzirt", NONE)]
    sizes = [1, 40_000, 0, 32_769]
    frames = []
    for k in range(2 * len(groups)):   # interleaved: every group's frames are apart in the call
        name, comp = groups[k % len(groups)]
        frames.append(_frame(name, sizes[k // len(groups) * 2 + k % 2], 40 + k, 5, comp))
    ins = [_src(c, True) for _, c in frames]
    caps = [_cap(i, c) for i, c in frames]
    outs = [_Buf(c, True) for c in caps]
    me = cb.MixedEncoder()
    args = ([b.ptr for b in ins], [c.size for _, c in frames], [i for i, _ in frames], [o.ptr for o in outs], caps)
    me.encode_blobs_device(*args)   # warm: layouts planned, buffers grown
    mixed = _launches(lambda: me.encode_blobs_device(*args))
    per_group = 0
    for k, (name, comp) in enumerate(groups):
        idx = list(range(k, len(frames), len(groups)))
        enc = cb.PointcloudEncoder(frames[k][0])
        batch = enc.make_device_batch([args[0][f] for f in idx], [args[1][f] for f in idx], [args[3][f] for f in idx], [caps[f] for f in idx])
        enc.encode_batch_device(batch, want_sizes=True)
        per_group += _launches(lambda: enc.encode_batch_device(batch, write_header=True, want_sizes=True))
    assert mixed == per_group + 1, (mixed, per_group)
    status, sizes_sync = me.encode_blobs_device(*args)
    assert status == [0] * len(frames)
    assert me.encode_blobs_device(*args, want_sizes=False) == ([0] * len(frames), None)
    me.sync()
    assert _device_u64(me.sizes_device_ptr(), len(frames)) == sizes_sync


@pytest.mark.gpu
@pytest.mark.skipif(EMULATED, reason="the emulation runs every launch to its end before returning")
def test_without_sizes_the_call_returns_before_its_work_is_done():
    import torch
    s = torch.cuda.Stream()
    frames = [_frame(MIX[k % 4], MILLION, 50 + k, 5, NONE) for k in range(8)]
    ins = [_src(c, True) for _, c in frames]
    caps = [_cap(i, c) for i, c in frames]
    outs = [_Buf(c, True) for c in caps]
    me = cb.MixedEncoder(stream=s.cuda_stream)
    args = ([b.ptr for b in ins], [c.size for _, c in frames], [i for i, _ in frames], [o.ptr for o in outs], caps)
    _, sizes = me.encode_blobs_device(*args)
    me.encode_blobs_device(*args, want_sizes=False)
    busy = not s.query()
    me.sync()
    assert busy, "the asynchronous call waited for its kernels"
    assert _device_u64(me.sizes_device_ptr(), len(frames)) == sizes


# ---- 5. the layout cache -----------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("mem", [HOST, DEVICE], ids=["host", "device"])
def test_more_layouts_than_the_cache_holds(mem):
    layouts = []
    for k in range(48):   # 3 x the 16 layouts the handle keeps
        info, _ = _frame(MIX[k % len(MIX)], 1, 60, 3 + k % 3, [NONE, LZ4][k // 24])
        info.fields = [cb.PointField(f.name, f.offset, f.type, f.resolution * (1 + k / 64) if f.resolution else None) for f in info.fields]
        layouts.append((MIX[k % len(MIX)], info))
    me = cb.MixedEncoder()
    for rnd in range(2):
        for b in range(0, len(layouts), 6):
            frames = []
            for k, (name, info) in enumerate(layouts[b:b + 6]):
                cloud = _layout(name, [3000, 0, 33_000][(k + rnd) % 3], 70 + b + k, info.version)[1]
                frames.append((cb.EncodingInfo(**{**info.__dict__, "fields": list(info.fields)}), cloud))
            rc, msg, status, _, blobs, guards, _ = _run(me, frames, mem)
            assert rc == 0 and guards, msg
            for f, (info, cloud) in enumerate(frames):
                assert _same_blob(blobs[f], _alone(info, cloud, mem)[2], SHUFFLED_LANES and _device_stage2(info, mem, False)), (rnd, b, f)
            assert me.cached_layouts() <= 16 + 6


# ---- 6. round trip -----------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("mem", MEMS, ids=MEM_IDS)
def test_round_trip_through_decode_blobs(oracle, mem):
    frames = _mixed_frames(80, [NONE, LZ4] + ([ZSTD] if mem != DEVICE else []), [3000, 0, 40_000, 1, 32_769])
    rc, msg, _, _, blobs, _, _ = _run(cb.MixedEncoder(), frames, mem)
    assert rc == 0, msg
    for f, ((st, dinfo, out), (info, cloud)) in enumerate(zip(cb.PointcloudDecoder().decode_blobs(blobs), frames)):
        assert st == 0 and dinfo.width * dinfo.height * info.point_step == cloud.size, f
        pts, back = cloud.reshape(-1, info.point_step), out.reshape(-1, info.point_step)
        for fld in info.fields:
            size = cb.SizeOf(fld.type)
            a, b = pts[:, fld.offset:fld.offset + size], back[:, fld.offset:fld.offset + size]
            floats = fld.type in (cb.FieldType.FLOAT32, cb.FieldType.FLOAT64)
            if info.encoding_opt != cb.EncodingOptions.LOSSY or fld.resolution is None or not floats:
                assert np.array_equal(a, b), (f, fld.name)   # lossless fields: bit-exact
                continue
            dt = np.float32 if fld.type == cb.FieldType.FLOAT32 else np.float64
            x, y = np.ascontiguousarray(a).view(dt).ravel().astype(np.float64), np.ascontiguousarray(b).view(dt).ravel().astype(np.float64)
            finite = np.isfinite(x)
            assert np.array_equal(np.isnan(x), np.isnan(y)), (f, fld.name)
            assert np.all(np.abs(x[finite] - y[finite]) <= fld.resolution * 0.5 * (1 + 1e-3) + np.abs(x[finite]) * 1e-6), (f, fld.name)
        want = np.zeros(cloud.size, dtype=np.uint8)
        oracle.decode(blobs[f], want)
        assert np.array_equal(out, want), f


# ---- 7. threads and caller streams -------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_two_handles_on_two_threads_on_caller_streams():
    n = 8_000 if EMULATED else 80_000
    jobs = [_mixed_frames(90 + t, [NONE, LZ4], [n, 1, n // 2 + t, 0, 32_769]) for t in range(2)]

    def work(t):
        stream = 0
        if not EMULATED:
            import torch
            s = torch.cuda.Stream()
            stream = s.cuda_stream
        me = cb.MixedEncoder(stream=stream)
        out = []
        for _ in range(3):
            for mem in (DEVICE, HOST):
                rc, msg, _, _, blobs, guards, _ = _run(me, jobs[t], mem)
                assert rc == 0 and guards, msg
                out.append(blobs)
        me.close()
        return out

    alone = [work(t) for t in range(2)]
    got, errors = [None, None], []

    def run(t):
        try:
            got[t] = work(t)
        except BaseException as e:  # noqa: BLE001 -- reported below
            errors.append(e)

    threads = [threading.Thread(target=run, args=(t,)) for t in range(2)]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    assert not errors, errors
    if SHUFFLED_LANES:
        return   # the device LZ4 coder's bytes follow the shuffled lane order; tests 1-2 compare its points
    assert got == alone


@pytest.mark.gpu
def test_python_api():
    me = cb.MixedEncoder()
    frames = [_frame("xyzi", 100, 1, 5, NONE), _frame("c3", 0, 2, 4, LZ4), (_frame("xyz", 10, 3, 3, NONE)[0], np.zeros(17, dtype=np.uint8))]
    res = me.encode_blobs([c for _, c in frames], [i for i, _ in frames])
    assert [r[0] for r in res] == [0, 0, -1] and res[2][1] is None
    assert me.frame_error(2) == "Input cloud_data size is not a multiple of point_step" and me.frame_error(0) == ""
    assert res[0][1] == _alone(*frames[0], HOST)[2]
    ins = [_src(c, True) for _, c in frames[:2]]
    got = me.encode_blobs_from_device([b.ptr for b in ins], [c.size for _, c in frames[:2]], [i for i, _ in frames[:2]])
    assert got == res[:2]
    assert me.encode_blobs([], []) == []


# ---- 8. the same file under the CPU emulation --------------------------------------------------------------------------
@pytest.mark.skipif(EMULATED, reason="already running under the emulation")
@pytest.mark.parametrize("order,workers", [("fwd", "1"), ("fwd", "8"), ("rand", "1"), ("rand", "8")])
def test_this_file_under_emulation(lib_built, order, workers):
    from test_cusim_kernels import _run_gpu_suite
    import platform
    if platform.machine() != "x86_64":
        pytest.skip("cusim's context switch is x86-64 only")
    sys.path.insert(0, os.path.join(ROOT, "tests", "cusim"))
    import build_cusim
    env = {"CUSIM_ORDER": order, "CUSIM_WORKERS": workers}
    if order == "rand":
        env["CUSIM_JITTER"] = "1"
    out = _run_gpu_suite(build_cusim.build(), env, ["tests/test_gpu_encode_mixed.py"])
    assert " passed" in out and "failed" not in out


@pytest.mark.skipif(EMULATED, reason="already running under the emulation")
def test_encode_mixed_blobs_under_thread_sanitizer(lib_built, tmp_path):
    # tests/cusim/encode_mixed_racecheck_main.cpp: one device-blob and one host-blob batch of three layouts, every CUDA
    # thread a ThreadSanitizer fiber (strict model: a shuffle is no fence)
    import platform
    if platform.machine() != "x86_64":
        pytest.skip("cusim's context switch is x86-64 only")
    here = os.path.join(ROOT, "tests", "cusim")
    sys.path.insert(0, here)
    import build_cusim
    from cloudini_b200.build import SOURCES
    try:
        build_cusim.build_racecheck()
    except subprocess.CalledProcessError as e:
        pytest.skip(f"ThreadSanitizer toolchain unavailable: {e}")
    objs = [os.path.join(build_cusim.OUT_DIR, os.path.splitext(s)[0] + "_tsan.o") for s in SOURCES + ["cusim.cpp"]]
    drv, exe = str(tmp_path / "encode_mixed_main.o"), str(tmp_path / "encode_mixed_racecheck")
    subprocess.check_call(["g++", "-std=c++17", "-O0", "-g", "-fPIC", "-pthread", "-w", "-fsanitize=thread", "-I", here, "-I",
                           os.path.join(ROOT, "include"), "-x", "c++", "-c", os.path.join(here, "encode_mixed_racecheck_main.cpp"), "-o", drv])
    subprocess.check_call(["g++", "-fsanitize=thread", "-pthread", "-o", exe, drv, *objs, "-ldl"])
    env = dict(os.environ, TSAN_OPTIONS="halt_on_error=0 report_signal_unsafe=0", CUSIM_WORKERS="4", CUSIM_TSAN_STRICT="1")
    env.pop("LD_PRELOAD", None)
    r = subprocess.run([exe], env=env, capture_output=True, text=True, timeout=1500)
    if "FATAL: ThreadSanitizer" in r.stderr:
        pytest.skip("ThreadSanitizer cannot run in this environment: " + r.stderr[-200:])
    assert r.returncode == 0 and "encode_mixed_racecheck: done" in r.stdout, r.stdout[-2000:] + r.stderr[-3000:]
    assert "WARNING: ThreadSanitizer" not in r.stderr, r.stderr[-4000:]
