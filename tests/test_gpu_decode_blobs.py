"""cldn_b200_decode_blobs: complete blobs of any layout, size, wire version and compression in one call, with a status
per frame.

Every frame must give what DecodeHeader + cldn_b200_decode give that blob alone: the same status and message when it
fails, the oracle's points when it decodes. Outputs sit between guard bytes and their padding is pre-filled, so a write
outside a frame's own buffer or into its padding is seen. Blobs come from this library's encoder; the expected points
are the oracle's decode (the compiled reference where it exists; the C port otherwise, which has no stage 2, so LZ4 /
ZSTD frames are then compared with the single-blob decode).
"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import cloudini_b200 as cb
from cloudini_b200 import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMULATED = bool(os.environ.get("CLDN_B200_LIB"))   # tests/cusim: the same checks on smaller inputs
GUARD = 64
G_BYTE, PAD_BYTE = 0xA7, 0x5A
NONE, LZ4, ZSTD = cb.CompressionOption.NONE, cb.CompressionOption.LZ4, cb.CompressionOption.ZSTD


class _Buf:
    """`cap` bytes between two guards of GUARD bytes, host (numpy) or device (torch on the GPU, numpy under cusim)."""

    def __init__(self, cap, device, fill=PAD_BYTE, src=None):
        a = np.full(GUARD + cap + GUARD, G_BYTE, dtype=np.uint8)
        a[GUARD:GUARD + cap] = fill if src is None else np.frombuffer(src, dtype=np.uint8)
        self.cap, self.device = cap, device
        if device and not EMULATED:
            import torch
            self.t = torch.from_numpy(a).cuda()
            torch.cuda.synchronize()
            self.base = self.t.data_ptr()
        else:
            self.t = a
            self.base = a.ctypes.data
        self.ptr = self.base + GUARD

    def all(self):
        return self.t.cpu().numpy() if self.device and not EMULATED else self.t

    def body(self):
        return self.all()[GUARD:GUARD + self.cap]

    def guards_intact(self):
        a = self.all()
        return bool((a[:GUARD] == G_BYTE).all() and (a[GUARD + self.cap:] == G_BYTE).all())


def _info_of(blob):
    try:
        info, _ = cb.DecodeHeader(blob)
        return info
    except RuntimeError:
        return None


def _need(blob):
    info = _info_of(blob)
    n = info.width * info.height * info.point_step if info else 0
    return n if n < (1 << 31) else 0


def _alone(blob, cap, device):
    """(status, message, output) of DecodeHeader + cldn_b200_decode on this blob alone."""
    L = cb.lib()
    raw = np.frombuffer(blob, dtype=np.uint8) if len(blob) else np.zeros(1, dtype=np.uint8)
    c, used = cb._CInfo(), C.c_size_t(0)
    rc = L.cldn_b200_decode_header(raw.ctypes.data, len(blob), C.byref(c), C.byref(used))
    if rc:
        return rc, L.cldn_b200_last_error().decode(), None
    src = _Buf(max(len(blob), 1), device, src=bytes(blob) + b"\0" * (len(blob) == 0))
    out = _Buf(cap, device)
    dec = cb.PointcloudDecoder()
    rc = L.cldn_b200_decode(dec._h, C.byref(c), src.ptr + used.value, len(blob) - used.value, out.ptr, cap, 1 if device else 0)
    msg = L.cldn_b200_last_error().decode() if rc else ""
    dec.close()
    return rc, msg, out.body().copy()


def _want(oracle, blob, cap, device):
    info = _info_of(blob)
    if info.compression_opt != NONE and oracle.kind == "port":
        return _alone(blob, cap, device)[2]
    out = np.full(cap, PAD_BYTE, dtype=np.uint8)
    oracle.decode(blob, out[:info.width * info.height * info.point_step])
    return out


def _decode_blobs(blobs, caps, device):
    """Runs decode_blobs on guarded buffers. Returns (statuses, messages, infos, outputs, guards intact, return code)."""
    dec = cb.PointcloudDecoder()
    ins = [_Buf(max(len(b), 1), device, src=bytes(b) + b"\0" * (len(b) == 0)) for b in blobs]
    outs = [_Buf(c, device) for c in caps]
    n = len(blobs)
    m = max(n, 1)
    status = (C.c_int32 * m)()
    decoded = (C.c_size_t * m)()
    rc = cb.lib().cldn_b200_decode_blobs(dec._h, n, (C.c_void_p * m)(*[b.ptr for b in ins]), (C.c_size_t * m)(*[len(b) for b in blobs]),
                                         (C.c_void_p * m)(*[o.ptr for o in outs]), (C.c_size_t * m)(*caps), 1 if device else 0, status, decoded)
    top = cb.lib().cldn_b200_last_error().decode() if rc else ""
    msgs = [dec.frame_error(f) for f in range(n)]
    st = [int(status[f]) for f in range(n)]
    for f in range(n):
        want = _need(blobs[f]) if st[f] == 0 else 0
        assert decoded[f] == want, (f, decoded[f], want)
    first_bad = next((f for f in range(n) if st[f] != 0), None)
    assert rc == (0 if first_bad is None else st[first_bad])
    if first_bad is not None:
        assert top == f"frame {first_bad}: {msgs[first_bad]}"
    guards = all(o.guards_intact() for o in outs) and all(i.guards_intact() for i in ins)
    dec.close()
    return st, msgs, [o.body().copy() for o in outs], guards


def _check_batch(oracle, blobs, device, caps=None, check_messages=True):
    caps = caps or [_need(b) for b in blobs]
    st, msgs, outs, guards = _decode_blobs(blobs, caps, device)
    assert guards, "a byte outside a frame's buffer changed"
    for f, b in enumerate(blobs):
        a_st, a_msg, a_out = _alone(b, caps[f], device)
        assert st[f] == a_st, (f, st[f], a_st, msgs[f], a_msg)
        if st[f] == 0:
            assert msgs[f] == ""
            assert np.array_equal(outs[f], _want(oracle, b, caps[f], device)), f"frame {f} differs from the oracle"
        elif check_messages:
            assert msgs[f] == a_msg, (f, msgs[f], a_msg)
    return st


def _encode(info, cloud, compression=NONE, version=None):
    info.compression_opt = compression
    if version is not None:
        info.version = version
    info.width, info.height = cloud.size // info.point_step, 1
    return cb.PointcloudEncoder(info).encode(cloud)


def _xyzi(n, seed):
    return synth.cloud_c2(n, seed=seed)


# ---- 1. varying sizes, one layout ------------------------------------------------------------------------------------
def _sizes(seed):
    rng = np.random.default_rng(seed)
    fixed = [0, 1, 32767, 32768, 32769]
    if EMULATED:
        return fixed + [int(x) for x in rng.integers(0, 70_000, 3)]
    return fixed + [int(x) for x in rng.integers(0, 300_000, 64 - len(fixed))]


@pytest.mark.gpu
@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
def test_varying_sizes_one_layout_round_trip_from_encode_batch(oracle, device):
    sizes = _sizes(11)
    info = synth.info_xyzi(1)
    info.compression_opt = NONE
    clouds = [_xyzi(n, seed=200 + k)[1] if n else np.zeros(0, dtype=np.uint8) for k, n in enumerate(sizes)]
    # encode_batch: one launch for every frame; each payload is put behind the header that states its own size
    enc = cb.PointcloudEncoder(info)
    d_in = [_Buf(max(c.size, 1), True, src=c.tobytes() + b"\0" * (c.size == 0)) for c in clouds]
    caps = [cb.MaxCompressedSize(info, c.size // 16, False) for c in clouds]
    d_out = [_Buf(cap, True) for cap in caps]
    written = enc.encode_batch_device(enc.make_device_batch([b.ptr for b in d_in], [c.size for c in clouds], [b.ptr for b in d_out], caps),
                                      write_header=False, want_sizes=True)
    blobs = []
    for c, o, w in zip(clouds, d_out, written):
        hinfo = synth.info_xyzi(c.size // 16)
        hinfo.compression_opt = NONE
        blobs.append(cb.EncodeHeader(hinfo) + o.body()[:w].tobytes())
    before = cb.kernel_launch_count()
    st = _check_batch(oracle, blobs, device)
    assert st == [0] * len(blobs)
    if device:
        # the launches of the check above: decode_blobs once, then every frame alone for the comparison
        dec = cb.PointcloudDecoder()
        ins = [_Buf(len(b), True, src=b) for b in blobs]
        outs = [_Buf(_need(b), True) for b in blobs]
        n = len(blobs)
        before = cb.kernel_launch_count()
        rc = cb.lib().cldn_b200_decode_blobs(dec._h, n, (C.c_void_p * n)(*[b.ptr for b in ins]), (C.c_size_t * n)(*[len(b) for b in blobs]),
                                             (C.c_void_p * n)(*[o.ptr for o in outs]), (C.c_size_t * n)(*[_need(b) for b in blobs]), 1,
                                             (C.c_int32 * n)(), None)
        assert rc == 0
        blobs_launches = cb.kernel_launch_count() - before
        # one decode_batch of a same-layout batch with as many frames (uniform size)
        m = 70_000
        u_blob = _encode(synth.info_xyzi(m), _xyzi(m, seed=5)[1])
        hdr = cb.DecodeHeader(u_blob)[1]
        u_in = [_Buf(len(u_blob) - hdr, True, src=u_blob[hdr:]) for _ in range(n)]
        u_out = [_Buf(m * 16, True) for _ in range(n)]
        before = cb.kernel_launch_count()
        dec.decode_batch_device(cb.DecodeHeader(u_blob)[0], dec.make_device_batch([b.ptr for b in u_in], [len(u_blob) - hdr] * n,
                                                                                  [b.ptr for b in u_out], [m * 16] * n), sync=True)
        batch_launches = cb.kernel_launch_count() - before
        assert blobs_launches <= batch_launches + 1, (blobs_launches, batch_launches)   # + the header gather


@pytest.mark.gpu
@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
def test_varying_sizes_after_the_viz_preprocessor(oracle, device):
    from cloudini_b200.ros import VizPreprocessor
    pp = VizPreprocessor()
    blobs = []
    for k in range(4 if EMULATED else 16):
        info, cloud = synth.cloud_viz(20_000 if EMULATED else 150_000, seed=40 + k)
        new_info, data, applied = pp.run(info, cloud)
        assert applied
        new_info.compression_opt = NONE
        blobs.append(cb.PointcloudEncoder(new_info).encode(data))
    assert len({_info_of(b).width for b in blobs}) > 1
    assert _check_batch(oracle, blobs, device) == [0] * len(blobs)


# ---- 2. mixed layouts, versions and compressions ---------------------------------------------------------------------
def _mixed_blobs(seed):
    n = 9_000 if EMULATED else 70_000
    out = []
    out.append(_encode(*synth.cloud_c1(n // 3, seed=seed)))
    for v in (3, 4, 5):
        for comp in (NONE, LZ4, ZSTD):
            info, cloud = synth.cloud_c2(n + 101 * v + comp, seed=seed + v)
            out.append(_encode(info, cloud, comp, version=v))
    out.append(_encode(*synth.cloud_c3(n + 7, seed=seed + 1), compression=ZSTD))
    out.append(_encode(*synth.cloud_c3(n // 2, seed=seed + 2)))
    out.append(_encode(*synth.cloud_c4_mixed_frame(1, az=256 if EMULATED else 2032), compression=LZ4))
    info, cloud = synth.cloud_lossless(n // 2, seed=seed + 3)
    out.append(_encode(info, cloud, ZSTD))
    info, cloud = synth.cloud_lossless(n // 3, seed=seed + 4, lossless=False, stamp_res=None)
    out.append(_encode(info, cloud))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
def test_mixed_layouts_versions_and_compressions_in_one_call(oracle, device, monkeypatch):
    monkeypatch.delenv("CLDN_B200_ZSTD_HOST", raising=False)
    blobs = _mixed_blobs(3)
    order = np.random.default_rng(1).permutation(len(blobs))
    blobs = [blobs[i] for i in order]
    assert {(_info_of(b).compression_opt, _info_of(b).version) for b in blobs} >= {(c, v) for c in (NONE, LZ4, ZSTD) for v in (3, 4, 5)}
    assert _check_batch(oracle, blobs, device) == [0] * len(blobs)
    if not device:   # the Python binding, zero-filled outputs
        for b, (s, info, out) in zip(blobs, cb.PointcloudDecoder().decode_blobs(blobs)):
            assert s == 0 and info.width == _info_of(b).width
            if info.compression_opt == NONE or oracle.kind != "port":
                want = np.zeros(_need(b), dtype=np.uint8)
                oracle.decode(b, want)
                assert np.array_equal(out, want)


# ---- 3. damaged frames among good ones -------------------------------------------------------------------------------
def _payload_at(blob):
    return cb.DecodeHeader(blob)[1]


def _damaged(blob, kind, rng):
    b = bytearray(blob)
    h = _payload_at(blob)
    if kind == "bitflip":
        i = h + 4 + int(rng.integers(0, max(1, len(b) - h - 4)))
        b[i] ^= 1 << int(rng.integers(8))
    elif kind == "truncate":
        b = b[:h + int(rng.integers(0, len(b) - h))]
    elif kind == "chunk_prefix":
        b[h:h + 4] = (0xFFFFFF00 | int(rng.integers(256))).to_bytes(4, "little")
    elif kind == "header_line":
        b[3] = ord("X")
    elif kind == "v2":
        b[10:12] = b"02"
    return bytes(b)


KINDS = ["bitflip", "truncate", "chunk_prefix", "header_line", "v2", "short_output"]


@pytest.mark.gpu
@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
@pytest.mark.parametrize("where", ["first", "middle", "last", "all"])
def test_damaged_frames_among_good_ones(oracle, device, where):
    rng = np.random.default_rng(["first", "middle", "last", "all"].index(where))
    n = 6_000 if EMULATED else 60_000
    good = [_encode(*synth.cloud_c2(n + k, seed=70 + k), compression=[NONE, ZSTD, LZ4][k % 3]) for k in range(6)]
    for kind in KINDS + ["zstd_frame"]:
        blobs = list(good)
        caps = [_need(b) for b in blobs]
        at = {"first": [0], "middle": [3], "last": [len(blobs) - 1], "all": list(range(len(blobs)))}[where]
        for i in at:
            if kind == "short_output":
                caps[i] -= 1
            elif kind == "zstd_frame":
                z = [j for j in range(len(blobs)) if _info_of(blobs[j]).compression_opt == ZSTD][0]
                src = bytearray(blobs[z])
                h = _payload_at(blobs[z])
                src[h + 4 + 6] ^= 0x40            # inside the first ZSTD frame's header / first block
                blobs[i] = bytes(src)
            else:
                blobs[i] = _damaged(blobs[i], kind, rng)
        if kind not in ("short_output", "zstd_frame"):
            caps = [max(_need(b), c) if i in at else c for i, (b, c) in enumerate(zip(blobs, caps))]
        st = _check_batch(oracle, blobs, device, caps)
        for i in range(len(blobs)):
            if i not in at:
                assert st[i] == 0, (kind, i)
        if kind in ("header_line", "short_output", "chunk_prefix"):
            assert all(st[i] != 0 for i in at), kind
        if kind == "v2":
            assert all(st[i] == -5 for i in at)


def _device_launches(fn):
    before = cb.kernel_launch_count()
    fn()
    return cb.kernel_launch_count() - before


def _blobs_device_call(dec, blobs, caps=None):
    caps = caps or [_need(b) for b in blobs]
    ins = [_Buf(len(b), True, src=b) for b in blobs]
    outs = [_Buf(c, True) for c in caps]
    n = len(blobs)
    status = (C.c_int32 * n)()
    cb.lib().cldn_b200_decode_blobs(dec._h, n, (C.c_void_p * n)(*[b.ptr for b in ins]), (C.c_size_t * n)(*[len(b) for b in blobs]),
                                    (C.c_void_p * n)(*[o.ptr for o in outs]), (C.c_size_t * n)(*caps), 1, status, None)
    return list(status)


@pytest.mark.gpu
@pytest.mark.parametrize("comp", [NONE, LZ4, ZSTD], ids=["none", "lz4", "zstd"])
def test_a_group_is_one_fused_batch_launch(comp):
    # equal frames: decode_blobs launches exactly what decode_batch of the same payloads launches, plus the header gather
    n_pts = 9_000 if EMULATED else 70_000
    blobs = [_encode(*synth.cloud_c2(n_pts, seed=60 + k), compression=comp) for k in range(6)]
    dec = cb.PointcloudDecoder()
    _blobs_device_call(dec, blobs)   # warm: buffers grown, plan cached
    blobs_launches = _device_launches(lambda: _blobs_device_call(dec, blobs))
    info, h = cb.DecodeHeader(blobs[0])
    ins = [_Buf(len(b) - h, True, src=b[h:]) for b in blobs]
    outs = [_Buf(_need(b), True) for b in blobs]
    batch = dec.make_device_batch([b.ptr for b in ins], [len(b) - h for b in blobs], [o.ptr for o in outs], [_need(b) for b in blobs])
    batch_launches = _device_launches(lambda: dec.decode_batch_device(info, batch, sync=True))
    assert blobs_launches == batch_launches + 1, (blobs_launches, batch_launches)


@pytest.mark.gpu
@pytest.mark.parametrize("comp", [NONE, ZSTD], ids=["none", "zstd"])
def test_a_damaged_frame_costs_only_its_own_second_decode(comp):
    # the per-frame error words name the damaged frame: only it is decoded again, not its whole group
    n_pts = 9_000 if EMULATED else 70_000
    blobs = [_encode(*synth.cloud_c2(n_pts + k, seed=80 + k), compression=comp) for k in range(8)]
    dec = cb.PointcloudDecoder()
    _blobs_device_call(dec, blobs)
    clean = _device_launches(lambda: _blobs_device_call(dec, blobs))
    bad = list(blobs)
    bad[5] = _damaged(blobs[5], "chunk_prefix", np.random.default_rng(3))
    st = []
    damaged = _device_launches(lambda: st.extend(_blobs_device_call(dec, bad)))
    assert st == [0] * 5 + [-4] + [0] * 2
    alone = _device_launches(lambda: _alone(bad[5], _need(bad[5]), True))
    assert damaged == clean + alone, (damaged, clean, alone)


# ---- 4. seeded fuzz --------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_random_batches_with_random_damage(oracle):
    trials = int(os.environ.get("CLDN_B200_BLOBS_TRIALS", "6" if EMULATED else "40"))
    rng = np.random.default_rng(2024)
    n = 4_000 if EMULATED else 40_000
    pool = []
    for k in range(8):
        comp = [NONE, LZ4, ZSTD][k % 3]
        if k % 4 == 3:
            pool.append(_encode(*synth.cloud_c3(n // 2 + k, seed=k), compression=comp))
        else:
            pool.append(_encode(*synth.cloud_c2(int(rng.integers(0, n)), seed=k), compression=comp, version=3 + k % 3))
    for t in range(trials):
        m = int(rng.integers(1, 9))
        blobs = [pool[int(rng.integers(len(pool)))] for _ in range(m)]
        caps = [_need(b) for b in blobs]
        for i in range(m):
            if rng.random() < 0.35:
                kind = KINDS[int(rng.integers(len(KINDS)))]
                if kind == "short_output":
                    caps[i] = max(0, caps[i] - 1)
                elif len(blobs[i]) > _payload_at(blobs[i]) + 8:
                    blobs[i] = _damaged(blobs[i], kind, rng)
                    caps[i] = max(caps[i], _need(blobs[i]))
        _check_batch(oracle, blobs, bool(t % 2), caps)


@pytest.mark.gpu
def test_python_api_reports_statuses_and_infos(oracle):
    good = _encode(*synth.cloud_c2(5_000, seed=3), compression=ZSTD)
    bad = _damaged(good, "header_line", np.random.default_rng(0))
    dec = cb.PointcloudDecoder()
    res = dec.decode_blobs([good, bad, b""])
    assert res[0][0] == 0 and res[0][1].width == 5_000 and res[0][2] is not None
    assert res[1][0] == -3 and res[1][1] is None and res[1][2] is None and "magic" in dec.frame_error(1)
    assert res[2][0] == -3 and dec.frame_error(0) == ""
    ins = [_Buf(len(good), True, src=good), _Buf(len(bad), True, src=bad)]
    outs = [_Buf(5_000 * 16, True), _Buf(16, True)]
    st, infos = dec.decode_blobs_device([b.ptr for b in ins], [len(good), len(bad)], [o.ptr for o in outs], [5_000 * 16, 16])
    assert st == [0, -3] and infos[0].point_step == 16 and infos[1] is None
    assert np.array_equal(outs[0].body(), _want(oracle, good, 5_000 * 16, True))
    assert dec.decode_blobs([]) == [] and dec.decode_blobs_device([], [], [], []) == ([], [])


# ---- 5. the same file under the CPU emulation ------------------------------------------------------------------------
@pytest.mark.skipif(EMULATED, reason="already running under the emulation")
@pytest.mark.parametrize("order,workers", [("fwd", "1"), ("fwd", "8"), ("rand", "1"), ("rand", "8")])
def test_this_file_under_emulation(lib_built, order, workers):
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from test_cusim_kernels import _run_gpu_suite
    import platform
    if platform.machine() != "x86_64":
        pytest.skip("cusim's context switch is x86-64 only")
    sys.path.insert(0, os.path.join(ROOT, "tests", "cusim"))
    import build_cusim
    env = {"CUSIM_ORDER": order, "CUSIM_WORKERS": workers}
    if order == "rand":
        env["CUSIM_JITTER"] = "1"
    out = _run_gpu_suite(build_cusim.build(), env, ["tests/test_gpu_decode_blobs.py"])
    assert " passed" in out and "failed" not in out


@pytest.mark.skipif(EMULATED, reason="already running under the emulation")
def test_mixed_damaged_batch_under_thread_sanitizer(lib_built, tmp_path):
    # tests/cusim/blobs_racecheck_main.cpp: one decode_blobs call over NONE / ZSTD / LZ4 groups with a forged chunk prefix and
    # a damaged header, every CUDA thread a ThreadSanitizer fiber (strict model: a shuffle is no fence)
    import platform
    if platform.machine() != "x86_64":
        pytest.skip("cusim's context switch is x86-64 only")
    here = os.path.join(ROOT, "tests", "cusim")
    sys.path.insert(0, here)
    import build_cusim
    from cloudini_b200.build import SOURCES
    try:
        build_cusim.build_racecheck()   # the instrumented kernels and C ABI (objects next to its own driver)
    except subprocess.CalledProcessError as e:
        pytest.skip(f"ThreadSanitizer toolchain unavailable: {e}")
    objs = [os.path.join(build_cusim.OUT_DIR, os.path.splitext(s)[0] + "_tsan.o") for s in SOURCES + ["cusim.cpp"]]
    drv, exe = str(tmp_path / "blobs_main.o"), str(tmp_path / "blobs_racecheck")
    subprocess.check_call(["g++", "-std=c++17", "-O0", "-g", "-fPIC", "-pthread", "-w", "-fsanitize=thread", "-I", here, "-I",
                           os.path.join(ROOT, "include"), "-x", "c++", "-c", os.path.join(here, "blobs_racecheck_main.cpp"), "-o", drv])
    subprocess.check_call(["g++", "-fsanitize=thread", "-pthread", "-o", exe, drv, *objs, "-ldl"])
    env = dict(os.environ, TSAN_OPTIONS="halt_on_error=0 report_signal_unsafe=0", CUSIM_WORKERS="4", CUSIM_TSAN_STRICT="1")
    env.pop("LD_PRELOAD", None)
    r = subprocess.run([exe], env=env, capture_output=True, text=True, timeout=1500)
    if "FATAL: ThreadSanitizer" in r.stderr:
        pytest.skip("ThreadSanitizer cannot run in this environment: " + r.stderr[-200:])
    assert r.returncode == 0 and "blobs_racecheck: done" in r.stdout, r.stdout[-2000:] + r.stderr[-3000:]
    assert "WARNING: ThreadSanitizer" not in r.stderr, r.stderr[-4000:]


@pytest.mark.skipif(EMULATED or not os.environ.get("CLDN_CUSIM_ASAN"),
                    reason="opt-in (CLDN_CUSIM_ASAN=1): this file under an AddressSanitizer build of the emulation")
def test_this_file_under_asan(lib_built):
    sys.path.insert(0, os.path.join(ROOT, "tests", "cusim"))
    import build_cusim
    lib = build_cusim.build(asan=True)
    libasan = subprocess.check_output(["gcc", "-print-file-name=libasan.so"], text=True).strip()
    libstdcxx = subprocess.check_output(["gcc", "-print-file-name=libstdc++.so.6"], text=True).strip()
    env = dict(os.environ, CLDN_B200_LIB=lib, CLDN_B200_ALLOW_EMULATION="tests-only", LD_PRELOAD=f"{libasan} {libstdcxx}",
               ASAN_OPTIONS="detect_leaks=0")
    r = subprocess.run([sys.executable, "-m", "pytest", "-x", "-q", "-m", "gpu", "-p", "no:cacheprovider", "tests/test_gpu_decode_blobs.py"],
                       cwd=ROOT, env=env, capture_output=True, text=True, timeout=3000)
    assert r.returncode == 0 and "AddressSanitizer" not in (r.stdout + r.stderr), r.stdout[-3000:] + r.stderr[-3000:]
