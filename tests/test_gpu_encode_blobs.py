"""cldn_b200_encode_blobs and cldn_b200_viz_lossy_preprocess_batch: batches of clouds of any size, one call each.

encode_blobs: blob f must be byte-identical to set_dims(w_f, h_f) + encode(write_header = 1) with the same handle, which
for NONE (and host-pointer LZ4 / ZSTD) is the reference's PointcloudEncoder(info with w_f, h_f).encode(cloud_f).
viz batch: every frame must give what the single call gives that cloud, which is the oracle's applyVizLossyPreprocessing.
Outputs sit between guard bytes and are pre-filled, so a write outside a frame's buffer, or any write by a refused call,
is seen.
"""
import ctypes as C
import os
import subprocess
import sys
import threading

import numpy as np
import pytest

import cloudini_b200 as cb
from cloudini_b200 import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMULATED = bool(os.environ.get("CLDN_B200_LIB"))   # tests/cusim: the same checks on smaller inputs
GUARD = 64
G_BYTE, PAD_BYTE = 0xA7, 0x5A
NONE, LZ4, ZSTD = cb.CompressionOption.NONE, cb.CompressionOption.LZ4, cb.CompressionOption.ZSTD
BIG = 70_000 if EMULATED else 300_000
SHUFFLED_LANES = EMULATED and os.environ.get("CUSIM_ORDER", "fwd") != "fwd"


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


def _src(cloud, device):
    return _Buf(max(cloud.size, 1), device, src=cloud.tobytes() + b"\0" * (cloud.size == 0))


def _with_dims(info, w, h):
    return cb.EncodingInfo(**{**info.__dict__, "fields": list(info.fields), "width": int(w), "height": int(h)})


def _worst(info, n, dims=None):
    w, h = dims if dims else (n, 1)
    return cb.MaxCompressedSize(_with_dims(info, w, h), n, True)


def _encode_blobs(enc, clouds, device, caps=None, dims=None, widths_only=False):
    """Runs encode_blobs on guarded buffers. Returns (rc, message, blobs, guards intact, outputs untouched)."""
    info = enc.getEncodingInfo()
    n = len(clouds)
    m = max(n, 1)
    pts = [c.size // info.point_step for c in clouds]
    caps = caps or [_worst(info, p, dims[f] if dims else None) for f, p in enumerate(pts)]
    ins = [_src(c, device) for c in clouds]
    outs = [_Buf(c, device) for c in caps]
    widths = (C.c_uint32 * m)(*[d[0] for d in dims]) if dims else None
    heights = (C.c_uint32 * m)(*[d[1] for d in dims]) if dims and not widths_only else None
    if widths_only:
        widths = (C.c_uint32 * m)(*pts)
    written = (C.c_size_t * m)()
    rc = cb.lib().cldn_b200_encode_blobs(enc._h, n, (C.c_void_p * m)(*[b.ptr for b in ins]), (C.c_size_t * m)(*[c.size for c in clouds]),
                                         widths, heights, (C.c_void_p * m)(*[o.ptr for o in outs]), (C.c_size_t * m)(*caps), written,
                                         1 if device else 0)
    msg = cb.lib().cldn_b200_last_error().decode() if rc else ""
    bodies = [o.body() for o in outs]
    blobs = [bodies[f][:written[f]].tobytes() for f in range(n)] if rc == 0 else None
    guards = all(o.guards_intact() for o in outs) and all(i.guards_intact() for i in ins)
    untouched = all((b == PAD_BYTE).all() for b in bodies)
    return rc, msg, blobs, guards, untouched


def _alone(enc, cloud, device, dims=None):
    """set_dims + encode(write_header = 1) with the same handle: the blob encode_blobs must reproduce."""
    info = enc.getEncodingInfo()
    n = cloud.size // info.point_step
    w, h = dims if dims else (n, 1)
    L = cb.lib()
    from cloudini_b200 import ros
    ros._L()
    assert L.cldn_b200_encoder_set_dims(enc._h, w, h) == 0
    cap = _worst(info, n, (w, h))
    src, out = _src(cloud, device), _Buf(cap, device)
    written = C.c_size_t(0)
    rc = L.cldn_b200_encode(enc._h, src.ptr, cloud.size, out.ptr, cap, 1, C.byref(written), 1 if device else 0)
    assert rc == 0, L.cldn_b200_last_error().decode()
    assert L.cldn_b200_encoder_set_dims(enc._h, info.width, info.height) == 0
    return out.body()[:written.value].tobytes()


def _device_u64(ptr, n):
    """n uint64 words at a device address."""
    if EMULATED:
        got = (C.c_uint64 * n)()
        C.memmove(got, ptr, 8 * n)
        return list(got)
    import torch

    class _View:
        __cuda_array_interface__ = {"shape": (n,), "typestr": "<i8", "data": (ptr, False), "version": 3}
    return [int(v) for v in torch.as_tensor(_View(), device="cuda").cpu().tolist()]


def _sizes(seed, k=6):
    rng = np.random.default_rng(seed)
    return [0, 1, 32767, 32768, 32769] + [int(x) for x in rng.integers(0, BIG, 2 if EMULATED else k)]


def _layout(name, n, seed, version=5):
    """(info, cloud) of n points for each layout the encoder treats differently."""
    if name == "xyzi":        # step 16, the fast XYZI kernel
        info, cloud = synth.cloud_c2(n, seed=seed)
    elif name == "xyz":       # step 12
        info, cloud = synth.cloud_c1(n, seed=seed)
    elif name == "c3":        # padded step 32, V5 Palette / DeltaRle sections
        info, cloud = synth.cloud_c3(n, seed=seed, version=version)
    elif name == "xyzirt":    # step 22, FloatN + V5 section
        info, cloud = synth.cloud_c4_mixed_frame(1, seed=seed, az=max(1, (n + 63) // 64))
    elif name == "gorilla":   # the DDS layout with a resolution-less FLOAT64 (Gorilla at v >= 4)
        info, cloud = synth.cloud_lossless(n, seed=seed, lossless=False, stamp_res=None)
    elif name == "lossless":
        info, cloud = synth.cloud_lossless(n, seed=seed)
    elif name == "enc_none":
        info, cloud = synth.cloud_c2(n, seed=seed)
        info.encoding_opt = cb.EncodingOptions.NONE
    else:
        raise ValueError(name)
    info.version = version
    info.compression_opt = NONE
    info.width, info.height = 0, 1
    return info, np.ascontiguousarray(cloud[:n * info.point_step])


LAYOUTS = ["xyzi", "xyz", "c3", "xyzirt", "gorilla", "lossless", "enc_none"]


def _clouds(name, sizes, seed, version=5):
    info = _layout(name, 1, seed, version)[0]
    return info, [_layout(name, n, seed + k, version)[1] for k, n in enumerate(sizes)]


# ---- 1. parity with the oracle, frame by frame -------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
@pytest.mark.parametrize("version", [3, 4, 5])
@pytest.mark.parametrize("layout", LAYOUTS)
def test_blobs_equal_the_oracle_frame_by_frame(oracle, layout, version, device):
    sizes = _sizes(LAYOUTS.index(layout) * 10 + version)
    info, clouds = _clouds(layout, sizes, 100 + version, version)
    enc = cb.PointcloudEncoder(info)
    rc, msg, blobs, guards, _ = _encode_blobs(enc, clouds, device)
    assert rc == 0, msg
    assert guards, "a byte outside a frame's buffer changed"
    for f, (cloud, blob) in enumerate(zip(clouds, blobs)):
        n = cloud.size // info.point_step
        assert blob == oracle.encode(_with_dims(info, n, 1), cloud), (layout, version, f, n)


@pytest.mark.gpu
@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
@pytest.mark.parametrize("layout", ["xyzi", "c3"])
def test_one_byte_short_names_the_frame_and_writes_nothing(layout, device):
    sizes = _sizes(5)
    info, clouds = _clouds(layout, sizes, 7)
    enc = cb.PointcloudEncoder(info)
    caps = [_worst(info, c.size // info.point_step) for c in clouds]
    for bad in (0, 3, len(clouds) - 1):
        short = list(caps)
        short[bad] -= 1
        rc, msg, _, guards, untouched = _encode_blobs(enc, clouds, device, short)
        assert rc == -2 and msg == f"frame {bad}: Output buffer too small for worst-case compressed size", msg
        assert guards and untouched
    rc, msg, blobs, guards, _ = _encode_blobs(enc, clouds, device, caps)   # exactly the worst case is enough
    assert rc == 0 and guards, msg


# ---- 2. stage 2 ----------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_device_lz4_equals_set_dims_and_encode():
    sizes = _sizes(21)
    for layout in ("xyzi", "c3"):
        info, clouds = _clouds(layout, sizes, 30)
        info.compression_opt = LZ4
        enc = cb.PointcloudEncoder(info)
        rc, msg, blobs, guards, _ = _encode_blobs(enc, clouds, True)
        assert rc == 0 and guards, msg
        for f, cloud in enumerate(clouds):
            alone = _alone(enc, cloud, True)
            if SHUFFLED_LANES:
                # the LZ4 kernel's shared hash table keeps whichever lane's store lands last; the emulation's shuffled
                # lane order changes that winner (encode_batch's blobs change the same way), so only the points must agree
                decoded = cb.PointcloudDecoder().decode_blobs([blobs[f], alone])
                assert decoded[0][0] == decoded[1][0] == 0 and np.array_equal(decoded[0][2], decoded[1][2]), (layout, f)
            else:
                assert blobs[f] == alone, (layout, f)


@pytest.mark.gpu
@pytest.mark.parametrize("comp", [LZ4, ZSTD], ids=["lz4", "zstd"])
def test_host_stage2_equals_the_reference(oracle, comp):
    if oracle.kind != "reference":
        pytest.skip("the compiled reference is not available")
    sizes = _sizes(31, 3)
    info, clouds = _clouds("xyzi", sizes, 40)
    info.compression_opt = comp
    enc = cb.PointcloudEncoder(info)
    rc, msg, blobs, guards, _ = _encode_blobs(enc, clouds, False)
    assert rc == 0 and guards, msg
    for f, cloud in enumerate(clouds):
        assert blobs[f] == oracle.encode(_with_dims(info, cloud.size // 16, 1), cloud), f
        assert blobs[f] == _alone(enc, cloud, False), f


@pytest.mark.gpu
def test_device_zstd_is_refused_like_encode_batch():
    info, clouds = _clouds("xyzi", [10, 20], 3)
    info.compression_opt = ZSTD
    enc = cb.PointcloudEncoder(info)
    rc, msg, _, guards, untouched = _encode_blobs(enc, clouds, True)
    assert rc == -5 and "host-pointer API" in msg and guards and untouched


# ---- 3. dims -------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
def test_explicit_dims_and_their_refusals(oracle, device):
    w = 256 if EMULATED else 1024
    info, clouds = _clouds("xyzi", [64 * w, 5000, 0], 50)
    dims = [(w, 64), (5000, 1), (0, 7)]
    enc = cb.PointcloudEncoder(info)
    rc, msg, blobs, guards, _ = _encode_blobs(enc, clouds, device, dims=dims)
    assert rc == 0 and guards, msg
    for f, cloud in enumerate(clouds):
        assert blobs[f] == oracle.encode(_with_dims(info, *dims[f]), cloud), f
        assert blobs[f] == _alone(enc, cloud, device, dims[f]), f
    assert cb.DecodeHeader(blobs[0])[0].height == 64
    bad = [(w, 64), (5001, 1), (0, 7)]
    rc, msg, _, guards, untouched = _encode_blobs(enc, clouds, device, caps=[_worst(info, c.size // 16, d) for c, d in zip(clouds, dims)], dims=bad)
    assert rc == -1 and msg.startswith("frame 1: ") and guards and untouched, msg
    rc, msg, _, guards, untouched = _encode_blobs(enc, clouds, device, widths_only=True)
    assert rc == -1 and guards and untouched, msg


# ---- 4. handle state and round trip --------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
def test_handle_header_and_later_batches_are_unchanged(device):
    info, clouds = _clouds("c3", [5000, 5000], 60)
    info.width = 5000
    enc = cb.PointcloudEncoder(info)
    header_before = enc.getHeader()
    outs = [np.zeros(_worst(info, 5000), dtype=np.uint8) for _ in clouds]
    before = enc.encode_batch_host(clouds, outs)
    before_bytes = [o[:w].tobytes() for o, w in zip(outs, before)]
    other = [_layout("c3", n, 61 + n)[1] for n in (17, 40000, 3)]
    assert _encode_blobs(enc, other, device)[0] == 0
    hp, hn = C.c_void_p(), C.c_size_t()
    assert cb.lib().cldn_b200_encoder_header(enc._h, C.byref(hp), C.byref(hn)) == 0
    assert C.string_at(hp.value, hn.value) == header_before
    outs = [np.zeros(_worst(info, 5000), dtype=np.uint8) for _ in clouds]
    after = enc.encode_batch_host(clouds, outs)
    assert [o[:w].tobytes() for o, w in zip(outs, after)] == before_bytes


@pytest.mark.gpu
@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
def test_round_trip_through_decode_blobs(oracle, device):
    sizes = _sizes(70)
    info, clouds = _clouds("xyzirt", sizes, 71)
    enc = cb.PointcloudEncoder(info)
    rc, msg, blobs, _, _ = _encode_blobs(enc, clouds, device)
    assert rc == 0, msg
    for (st, dinfo, out), blob in zip(cb.PointcloudDecoder().decode_blobs(blobs), blobs):
        assert st == 0
        want = np.zeros(dinfo.width * dinfo.point_step, dtype=np.uint8)
        oracle.decode(blob, want)
        assert np.array_equal(out, want)


@pytest.mark.gpu
def test_python_api():
    info, clouds = _clouds("xyzi", [100, 0, 64 * 8], 80)
    enc = cb.PointcloudEncoder(info)
    blobs = enc.encode_blobs(clouds, dims=[(100, 1), (0, 1), (8, 64)])
    assert [cb.DecodeHeader(b)[0].height for b in blobs] == [1, 1, 64]
    assert blobs[0] == _alone(enc, clouds[0], False)
    ins = [_src(c, True) for c in clouds]
    caps = [_worst(info, c.size // 16) for c in clouds]
    outs = [_Buf(c, True) for c in caps]
    sizes = enc.encode_blobs_device([b.ptr for b in ins], [c.size for c in clouds], [o.ptr for o in outs], caps)
    assert [o.body()[:s].tobytes() for o, s in zip(outs, sizes)] == enc.encode_blobs(clouds)
    assert enc.encode_blobs_device([b.ptr for b in ins], [c.size for c in clouds], [o.ptr for o in outs], caps, want_sizes=False) is None
    enc.sync()
    assert _device_u64(enc.sizes_device_ptr(), 3) == sizes   # whole blob sizes, headers included
    with pytest.raises(RuntimeError, match="frame 0"):
        enc.encode_blobs([np.zeros(17, dtype=np.uint8)])
    assert enc.encode_blobs([]) == []


# ---- 5. launch counts ----------------------------------------------------------------------------------------------
def _launches(fn):
    before = cb.kernel_launch_count()
    fn()
    return cb.kernel_launch_count() - before


@pytest.mark.gpu
@pytest.mark.parametrize("layout,comp", [("xyzi", NONE), ("c3", NONE), ("xyzi", LZ4)], ids=["xyzi", "c3", "xyzi-lz4"])
def test_encode_blobs_launches_encode_batch_plus_one(layout, comp):
    sizes = _sizes(90)
    info, clouds = _clouds(layout, sizes, 91)
    info.compression_opt = comp
    enc = cb.PointcloudEncoder(info)
    ins = [_src(c, True) for c in clouds]
    caps = [_worst(info, c.size // info.point_step) for c in clouds]
    outs = [_Buf(c, True) for c in caps]
    args = ([b.ptr for b in ins], [c.size for c in clouds], [o.ptr for o in outs], caps)
    enc.encode_blobs_device(*args)   # warm: buffers grown
    blobs = _launches(lambda: enc.encode_blobs_device(*args))
    batch = _launches(lambda: enc.encode_batch_device(enc.make_device_batch(*args), write_header=True, want_sizes=True))
    assert blobs == batch + 1, (blobs, batch)


@pytest.mark.gpu
@pytest.mark.parametrize("frames", [1, 7, 128])
def test_viz_batch_is_two_launches(frames):
    from cloudini_b200.ros import VizPreprocessor
    pp = VizPreprocessor()
    n = 300 if EMULATED else 3000
    info = synth.cloud_viz(1)[0]
    clouds = [synth.cloud_viz(n + k, seed=k)[1] for k in range(frames)]
    ins = [_src(c, True) for c in clouds]
    outs = [_Buf(c.size, True) for c in clouds]
    args = (info, [b.ptr for b in ins], [c.size for c in clouds], [o.ptr for o in outs], [c.size for c in clouds])
    assert _launches(lambda: pp.run_batch_device(*args)) == 2
    assert _launches(lambda: pp.run_batch(info, clouds)) == 2


# ---- 6. viz batch against the single call and the oracle ------------------------------------------------------------
def _viz_batch(pp, info, clouds, device, caps=None):
    """Runs the viz batch on guarded buffers. Returns (rc, message, [(info, survivors, kept, applied)], guards intact)."""
    n = len(clouds)
    m = max(n, 1)
    caps = caps or [c.size for c in clouds]
    ins = [_src(c, device) for c in clouds]
    outs = [_Buf(max(cap, 1), device) for cap in caps]
    c = cb._to_c(info)
    kept, applied, infos = (C.c_size_t * m)(), (C.c_int * m)(), (cb._CInfo * m)()
    from cloudini_b200 import ros
    rc = ros._L().cldn_b200_viz_lossy_preprocess_batch(pp._h, C.byref(c), n, (C.c_void_p * m)(*[b.ptr for b in ins]),
                                                       (C.c_size_t * m)(*[x.size for x in clouds]), (C.c_void_p * m)(*[o.ptr for o in outs]),
                                                       (C.c_size_t * m)(*caps), kept, applied, infos, 1 if device else 0)
    msg = cb.lib().cldn_b200_last_error().decode() if rc else ""
    res = []
    for f in range(n):
        body = outs[f].body()
        res.append((cb._from_c(infos[f]), body, int(kept[f]), bool(applied[f])))
    guards = all(o.guards_intact() for o in outs) and all(i.guards_intact() for i in ins)
    return rc, msg, res, guards


def _check_viz(oracle, pp, info, clouds, device):
    rc, msg, res, guards = _viz_batch(pp, info, clouds, device)
    assert rc == 0, msg
    assert guards, "a byte outside a frame's buffer changed"
    from cloudini_b200.ros import VizPreprocessor
    single = VizPreprocessor()
    step = info.point_step
    for f, (cloud, (after, body, kept, applied)) in enumerate(zip(clouds, res)):
        s_info, s_out, s_applied = single.run(info, cloud)
        assert applied == s_applied, f
        if not applied:
            assert kept == (cloud.size // step if step else 0)
            assert (body == PAD_BYTE).all(), f"frame {f}: a no-op frame's output was written"
            assert cb.EncodingInfoToYAML(after) == cb.EncodingInfoToYAML(info)
            continue
        assert kept == s_out.size // step
        assert np.array_equal(body[:kept * step], s_out), f
        assert (body[kept * step:] == PAD_BYTE).all(), f
        assert cb.EncodingInfoToYAML(after) == cb.EncodingInfoToYAML(s_info)
        o_info, o_out = oracle.viz_preprocess(info, cloud)
        assert np.array_equal(s_out, o_out) and o_info.width == kept, f
    return res


def _special(kind, n, step, seed):
    info, cloud = synth.cloud_viz(max(n, 1), seed=seed, step=step)
    pts = cloud.reshape(-1, step)
    if kind == "empty":
        return cloud[:0]
    if kind == "nan":
        pts[:, 0:4] = np.frombuffer(np.float32(np.nan).tobytes(), dtype=np.uint8)
    elif kind == "one_voxel":
        pts[:, 0:12] = np.frombuffer(np.array([1.0, 2.0, 3.0], dtype=np.float32).tobytes(), dtype=np.uint8)
    return np.ascontiguousarray(pts.reshape(-1)[:n * step])


@pytest.mark.gpu
@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
@pytest.mark.parametrize("step", [12, 16, 22, 32, 280])
def test_viz_batch_equals_the_single_call(oracle, step, device):
    from cloudini_b200.ros import VizPreprocessor
    pp = VizPreprocessor()
    n = 9_000 if EMULATED else 90_000
    info = synth.cloud_viz(1, step=step)[0]
    clouds = [synth.cloud_viz(n, seed=1, step=step)[1], _special("empty", 0, step, 2), _special("nan", 500, step, 3),
              synth.cloud_viz(1, seed=4, step=step)[1], _special("one_voxel", 2000, step, 5),
              synth.cloud_viz(n // 3 + 7, seed=6, step=step)[1], _special("empty", 0, step, 7)]
    _check_viz(oracle, pp, info, clouds, device)
    # the same handle, another batch (fewer, larger and smaller frames)
    _check_viz(oracle, pp, info, [synth.cloud_viz(2 * n + 1, seed=8, step=step)[1], synth.cloud_viz(3, seed=9, step=step)[1]], device)


def _noop_layouts():
    base = synth.cloud_viz(1)[0]
    out = []
    i = _with_dims(base, 0, 1); i.fields = i.fields[:2]; out.append(("two_fields", i))
    i = _with_dims(base, 0, 1); i.fields = [cb.PointField(f.name, f.offset, f.type, None if k == 1 else f.resolution) for k, f in enumerate(i.fields)]; out.append(("no_resolution", i))
    i = _with_dims(base, 0, 1); i.fields = [cb.PointField(f.name, f.offset, f.type, 0.002 if k == 2 else f.resolution) for k, f in enumerate(i.fields)]; out.append(("unequal_resolution", i))
    i = _with_dims(base, 0, 1); i.fields = [cb.PointField(f.name, f.offset, cb.FieldType.FLOAT64 if k == 0 else f.type, f.resolution) for k, f in enumerate(i.fields)]; out.append(("not_float32", i))
    i = _with_dims(base, 0, 1); i.fields = [cb.PointField(f.name, [0, 4, 12, 8][k], f.type, f.resolution) for k, f in enumerate(i.fields)]; out.append(("not_contiguous", i))
    for r in (0.0, -0.001, float("inf"), float("nan")):
        i = _with_dims(base, 0, 1); i.fields = [cb.PointField(f.name, f.offset, f.type, r if k < 3 else f.resolution) for k, f in enumerate(i.fields)]
        out.append((f"resolution_{r}", i))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
def test_viz_batch_no_op_layouts(oracle, device):
    from cloudini_b200.ros import VizPreprocessor
    pp = VizPreprocessor()
    clouds = [synth.cloud_viz(n, seed=n)[1] for n in (3000, 0, 17)]
    for name, info in _noop_layouts():
        before = cb.kernel_launch_count()
        res = _check_viz(oracle, pp, info, clouds, device)
        assert cb.kernel_launch_count() == before, name
        assert not any(r[3] for r in res), name


@pytest.mark.gpu
@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
def test_viz_batch_argument_errors_name_the_frame_and_launch_nothing(device):
    from cloudini_b200.ros import VizPreprocessor
    pp = VizPreprocessor()
    info = synth.cloud_viz(1)[0]
    clouds = [synth.cloud_viz(n, seed=n)[1] for n in (300, 200, 100)]
    before = cb.kernel_launch_count()
    rc, msg, res, guards = _viz_batch(pp, info, clouds, device, caps=[300 * 16, 200 * 16 - 1, 0])
    assert rc == -2 and msg == "frame 1: viz preprocessing: output buffer smaller than the input cloud", msg
    assert guards and all((r[1] == PAD_BYTE).all() for r in res)
    assert cb.kernel_launch_count() == before
    bad = _with_dims(info, 0, 1)
    bad.fields = [cb.PointField(f.name, f.offset + 8, f.type, f.resolution) for f in info.fields[:3]]
    rc, msg, _, _ = _viz_batch(pp, bad, [clouds[0][:0], clouds[1]], device)
    assert rc == -1 and msg == "frame 1: xyz fields lie outside the point", msg


@pytest.mark.gpu
def test_viz_batch_a_million_points_next_to_single_points(oracle):
    from cloudini_b200.ros import VizPreprocessor
    pp = VizPreprocessor()
    big = 150_000 if EMULATED else 1_200_000
    info = synth.cloud_viz(1)[0]
    clouds = [synth.cloud_viz(1, seed=1)[1], synth.cloud_viz(big, seed=2)[1], synth.cloud_viz(1, seed=3)[1], _special("nan", 1, 16, 4)]
    _check_viz(oracle, pp, info, clouds, True)


# ---- 7. the pipeline: viz batch -> encode_blobs, device-resident ----------------------------------------------------
@pytest.mark.gpu
def test_viz_batch_then_encode_blobs_equals_the_oracle(oracle):
    from cloudini_b200.ros import VizPreprocessor
    pp = VizPreprocessor()
    n = 12_000 if EMULATED else 150_000
    info = synth.cloud_viz(1)[0]
    info.width = 0   # what an empty cloud's message says; the other frames get their survivor count
    clouds = [synth.cloud_viz(n + 997 * k, seed=10 + k)[1] for k in range(5)] + [synth.cloud_viz(0)[1]]
    ins = [_src(c, True) for c in clouds]
    mid = [_Buf(max(c.size, 1), True) for c in clouds]
    res = pp.run_batch_device(info, [b.ptr for b in ins], [c.size for c in clouds], [b.ptr for b in mid], [c.size for c in clouds])
    enc_info = res[0][0]
    enc = cb.PointcloudEncoder(enc_info)
    kept = [k for _, k, _ in res]
    caps = [_worst(enc_info, k) for k in kept]
    outs = [_Buf(c, True) for c in caps]
    sizes = enc.encode_blobs_device([b.ptr for b in mid], [k * 16 for k in kept], [o.ptr for o in outs], caps)
    for f, cloud in enumerate(clouds):
        o_info, o_out = oracle.viz_preprocess(info, cloud)
        o_info.compression_opt = NONE
        want = oracle.encode(o_info, o_out)
        assert outs[f].body()[:sizes[f]].tobytes() == want, f


# ---- 8. threads ----------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_two_handles_on_two_threads(oracle):
    from cloudini_b200.ros import VizPreprocessor
    n = 8_000 if EMULATED else 80_000
    jobs = []
    for t, layout in enumerate(("xyzi", "c3")):
        info, clouds = _clouds(layout, [n, 1, n // 2 + t, 0, 32769], 200 + t)
        jobs.append((info, clouds, [synth.cloud_viz(n // (k + 1), seed=300 + 10 * t + k)[1] for k in range(4)], bool(t)))

    def work(job):
        info, clouds, viz, device = job
        enc, pp = cb.PointcloudEncoder(info), VizPreprocessor()
        out = []
        for _ in range(3):
            rc, msg, blobs, guards, _ = _encode_blobs(enc, clouds, device)
            assert rc == 0 and guards, msg
            rc, msg, res, guards = _viz_batch(pp, synth.cloud_viz(1)[0], viz, device)
            assert rc == 0 and guards, msg
            out.append((blobs, [r[1][:r[2] * 16].tobytes() for r in res]))
        return out

    alone = [work(j) for j in jobs]
    got = [None, None]
    errors = []

    def run(k):
        try:
            got[k] = work(jobs[k])
        except BaseException as e:  # noqa: BLE001 -- reported below
            errors.append(e)

    threads = [threading.Thread(target=run, args=(k,)) for k in range(2)]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    assert not errors, errors
    assert got == alone


# ---- 9. seeded fuzz ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_random_batches(oracle):
    from cloudini_b200.ros import VizPreprocessor
    trials = int(os.environ.get("CLDN_B200_ENCODE_BLOBS_TRIALS", "4" if EMULATED else "24"))
    rng = np.random.default_rng(4242)
    pp = VizPreprocessor()
    encs = {}
    for t in range(trials):
        layout = LAYOUTS[int(rng.integers(len(LAYOUTS)))]
        version = int(rng.integers(3, 6))
        m = int(rng.integers(1, 9))
        sizes = [int(rng.choice([0, 1, int(rng.integers(0, BIG // 4)), 32768])) for _ in range(m)]
        info, clouds = _clouds(layout, sizes, 1000 + t, version)
        key = (layout, version)
        enc = encs.get(key) or encs.setdefault(key, cb.PointcloudEncoder(info))
        device = bool(t % 2)
        rc, msg, blobs, guards, _ = _encode_blobs(enc, clouds, device)
        assert rc == 0 and guards, (t, msg)
        for f, cloud in enumerate(clouds):
            assert blobs[f] == oracle.encode(_with_dims(info, cloud.size // info.point_step, 1), cloud), (t, layout, version, f)
        step = int(rng.choice([12, 16, 22, 32]))
        viz = [synth.cloud_viz(int(rng.integers(0, BIG // 4)), seed=2000 + 10 * t + k, step=step)[1] for k in range(int(rng.integers(1, 7)))]
        _check_viz(oracle, pp, synth.cloud_viz(1, step=step)[0], viz, device)


# ---- 10. the same file under the CPU emulation ---------------------------------------------------------------------
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
    out = _run_gpu_suite(build_cusim.build(), env, ["tests/test_gpu_encode_blobs.py"])
    assert " passed" in out and "failed" not in out


@pytest.mark.skipif(EMULATED, reason="already running under the emulation")
def test_viz_batch_and_encode_blobs_under_thread_sanitizer(lib_built, tmp_path):
    # tests/cusim/encode_blobs_racecheck_main.cpp: one viz batch and one encode_blobs over mixed sizes, every CUDA thread
    # a ThreadSanitizer fiber (strict model: a shuffle is no fence)
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
    drv, exe = str(tmp_path / "encode_blobs_main.o"), str(tmp_path / "encode_blobs_racecheck")
    subprocess.check_call(["g++", "-std=c++17", "-O0", "-g", "-fPIC", "-pthread", "-w", "-fsanitize=thread", "-I", here, "-I",
                           os.path.join(ROOT, "include"), "-x", "c++", "-c", os.path.join(here, "encode_blobs_racecheck_main.cpp"), "-o", drv])
    subprocess.check_call(["g++", "-fsanitize=thread", "-pthread", "-o", exe, drv, *objs, "-ldl"])
    env = dict(os.environ, TSAN_OPTIONS="halt_on_error=0 report_signal_unsafe=0", CUSIM_WORKERS="4", CUSIM_TSAN_STRICT="1")
    env.pop("LD_PRELOAD", None)
    r = subprocess.run([exe], env=env, capture_output=True, text=True, timeout=1500)
    if "FATAL: ThreadSanitizer" in r.stderr:
        pytest.skip("ThreadSanitizer cannot run in this environment: " + r.stderr[-200:])
    assert r.returncode == 0 and "encode_blobs_racecheck: done" in r.stdout, r.stdout[-2000:] + r.stderr[-3000:]
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
    r = subprocess.run([sys.executable, "-m", "pytest", "-x", "-q", "-m", "gpu", "-p", "no:cacheprovider", "tests/test_gpu_encode_blobs.py"],
                       cwd=ROOT, env=env, capture_output=True, text=True, timeout=3000)
    assert r.returncode == 0 and "AddressSanitizer" not in (r.stdout + r.stderr), r.stdout[-3000:] + r.stderr[-3000:]
