"""CLDN_MEM_DEVICE_POINTS: clouds and decoded points in device memory, blobs and payloads in host memory.

The memory kind takes the routes of CLDN_MEM_HOST with the points read and written in place, so everything it gives is
compared with what CLDN_MEM_HOST gives the same input: blob bytes, decoded bytes (padding included), statuses and
messages. Device buffers sit between guard bytes and are pre-filled, so a write outside a buffer is seen. Under the CPU
emulation (tests/cusim) the device buffers come from the emulation's own cudaMalloc, so that CUSIM_HOSTCHECK=1 turns a
host access to a caller's device points into a failure (test_this_file_under_emulation).
"""
import ctypes as C
import os
import platform
import subprocess
import sys

import numpy as np
import pytest

import cloudini_b200 as cb
from cloudini_b200 import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMULATED = bool(os.environ.get("CLDN_B200_LIB"))
GUARD = 64
G_BYTE, FILL = 0xA7, 0xCD
HOST, DEVICE, DEVICE_POINTS = cb.MEM_HOST, cb.MEM_DEVICE, cb.MEM_DEVICE_POINTS
NONE, LZ4, ZSTD = cb.CompressionOption.NONE, cb.CompressionOption.LZ4, cb.CompressionOption.ZSTD
COMPS = [NONE, LZ4, ZSTD]
VERSIONS = [5] if EMULATED else [3, 4, 5]
MULTI = 40_000 if EMULATED else 200_000              # a frame of several 32768-point chunks
SIZES = [0, 1, 32769, MULTI] if EMULATED else [0, 1, 32767, 32768, 32769, MULTI]
LAYOUTS = ["xyz", "xyzi", "xyzirt", "c3", "gorilla", "xor", "copy"]
UNALIGNED = {"xyzirt": 3}                             # device clouds / outputs of step-22 points at an odd address


def _cusim():
    L = cb.lib()
    L._ZN5cusim12device_allocEm.restype = C.c_void_p
    L._ZN5cusim12device_allocEm.argtypes = [C.c_size_t]
    L._ZN5cusim11device_freeEPv.argtypes = [C.c_void_p]
    return L


class _Dev:
    """`cap` bytes of device memory at `off` bytes behind a guard, with a guard behind them (torch on the GPU, the
    emulation's cudaMalloc under cusim)."""

    def __init__(self, cap, fill=FILL, src=None, off=0):
        a = np.full(GUARD + off + cap + GUARD, G_BYTE, dtype=np.uint8)
        a[GUARD + off:GUARD + off + cap] = fill if src is None else np.frombuffer(src, dtype=np.uint8)
        self.cap, self.off, self.size = cap, off, a.size
        if EMULATED:
            self.base = _cusim()._ZN5cusim12device_allocEm(a.size)
            self._copy(self.base, a.ctypes.data)
        else:
            import torch
            self.t = torch.from_numpy(a).cuda()
            torch.cuda.synchronize()
            self.base = self.t.data_ptr()
        self.ptr = self.base + GUARD + off

    def _copy(self, dst, src):
        L = cb.lib()
        L._ZN5cusim19device_access_beginEv()
        C.memmove(dst, src, self.size)
        L._ZN5cusim17device_access_endEv()

    def all(self):
        if EMULATED:
            out = np.empty(self.size, dtype=np.uint8)
            self._copy(out.ctypes.data, self.base)
            return out
        import torch
        torch.cuda.synchronize()
        return self.t.cpu().numpy()

    def body(self):
        return self.all()[GUARD + self.off:GUARD + self.off + self.cap]

    def guards_intact(self):
        a = self.all()
        return bool((a[:GUARD + self.off] == G_BYTE).all() and (a[GUARD + self.off + self.cap:] == G_BYTE).all())

    def __del__(self):
        if EMULATED and getattr(self, "base", None):
            _cusim()._ZN5cusim11device_freeEPv(self.base)


class _Host:
    """The same for host memory (numpy)."""

    def __init__(self, cap, fill=FILL, src=None, off=0):
        self.a = np.full(GUARD + off + cap + GUARD, G_BYTE, dtype=np.uint8)
        self.a[GUARD + off:GUARD + off + cap] = fill if src is None else np.frombuffer(src, dtype=np.uint8)
        self.cap, self.off = cap, off
        self.ptr = self.a.ctypes.data + GUARD + off

    def all(self):
        return self.a

    body, guards_intact = _Dev.body, _Dev.guards_intact


def _points_buf(mem, cap, fill=FILL, src=None, off=0):
    """A buffer of points (a cloud to encode, a decode output) for memory kind `mem`."""
    return (_Dev if mem == DEVICE_POINTS else _Host)(cap, fill, src, off)


def _copy_fields(n, seed):
    F = cb.FieldType
    fields, off = [], 0
    for k in range(9):
        t = (F.UINT8, F.INT8, F.FLOAT32)[k % 3]
        fields.append(cb.PointField(f"c{k}", off, t, None))
        off += cb.SizeOf(t)
    info = cb.EncodingInfo(fields=fields, width=n, height=1, point_step=off, compression_opt=NONE, use_threads=False)
    return info, np.random.default_rng(seed).integers(0, 256, n * off, dtype=np.uint8)


def _layout(name, n, seed, version, comp):
    """(info, cloud) of n points of each layout family."""
    if name == "xyz":
        info, cloud = synth.cloud_c1(max(n, 1), seed=seed)
    elif name == "xyzi":
        info, cloud = synth.cloud_c2(max(n, 1), seed=seed)
    elif name == "xyzirt":     # step 22: FloatN + V5 section + scalar lossy float
        info, cloud = synth.cloud_c4_mixed_frame(seed, az=max(1, (n + 63) // 64))
    elif name == "c3":         # padded step 32, V5 Palette / DeltaRle sections
        info, cloud = synth.cloud_c3(max(n, 1), seed=seed, version=version)
    elif name == "gorilla":    # resolution-less FLOAT64: Gorilla at v >= 4
        info, cloud = synth.cloud_lossless(max(n, 1), seed=seed, lossless=False, stamp_res=None)
    elif name == "xor":        # LOSSLESS: XOR residuals
        info, cloud = synth.cloud_lossless(max(n, 1), seed=seed)
    elif name == "copy":       # every field copied
        info, cloud = _copy_fields(max(n, 1), seed)
    else:
        raise ValueError(name)
    info.version, info.compression_opt, info.use_threads = version, comp, False
    info.width, info.height = n, 1
    return info, np.ascontiguousarray(cloud[:n * info.point_step])


def _with_dims(info, w, h):
    return cb.EncodingInfo(**{**info.__dict__, "fields": list(info.fields), "width": int(w), "height": int(h)})


def _worst(info, nbytes, dims=None):
    n = nbytes // info.point_step
    w, h = dims if dims else (n, 1)
    return cb.MaxCompressedSize(_with_dims(info, w, h), n, True)


def _msg():
    return cb.lib().cldn_b200_last_error().decode()


def _arr(t, xs):
    return (t * max(len(xs), 1))(*xs)


def _encode(enc, api, clouds, mem, caps=None, dims=None, off=0):
    """One of the encode entry points on guarded buffers, clouds in `mem`'s point memory and blobs in host memory.
    Returns (rc, message, blobs, every guard intact)."""
    info = enc.getEncodingInfo()
    n = len(clouds)
    caps = caps or [_worst(info, c.size, dims[f] if dims else None) for f, c in enumerate(clouds)]
    ins = [_points_buf(mem, max(c.size, 1), src=c.tobytes() + b"\0" * (c.size == 0), off=off) for c in clouds]
    outs = [_Host(c) for c in caps]
    written = (C.c_size_t * max(n, 1))()
    L = cb.lib()
    in_p, in_b = _arr(C.c_void_p, [b.ptr for b in ins]), _arr(C.c_size_t, [c.size for c in clouds])
    out_p, cap_a = _arr(C.c_void_p, [o.ptr for o in outs]), _arr(C.c_size_t, caps)
    if api == "encode":
        rc = 0
        for f in range(n):
            w = C.c_size_t(0)
            rc = L.cldn_b200_encode(enc._h, in_p[f], clouds[f].size, out_p[f], caps[f], 1, C.byref(w), mem)
            if rc:
                break
            written[f] = w.value
    elif api == "batch":
        rc = L.cldn_b200_encode_batch(enc._h, n, in_p, in_b, out_p, cap_a, 1, written, mem)
    else:
        widths = _arr(C.c_uint32, [d[0] for d in dims]) if dims else None
        heights = _arr(C.c_uint32, [d[1] for d in dims]) if dims else None
        rc = L.cldn_b200_encode_blobs(enc._h, n, in_p, in_b, widths, heights, out_p, cap_a, written, mem)
    msg = _msg() if rc else ""
    blobs = [outs[f].body()[:written[f]].tobytes() for f in range(n)] if rc == 0 else None
    guards = all(o.guards_intact() for o in outs) and all(i.guards_intact() for i in ins)
    return rc, msg, blobs, guards


def _decode(dec, api, info, payloads, caps, mem, off=0):
    """decode (frame by frame) / decode_batch of header-less host payloads into outputs in `mem`'s point memory.
    Returns (rc, message, outputs, every guard intact)."""
    n = len(payloads)
    outs = [_points_buf(mem, c, off=off) for c in caps]
    srcs = [np.frombuffer(p + b"\0", dtype=np.uint8) for p in payloads]    # never a null pointer, even for b""
    L = cb.lib()
    c = cb._to_c(info)
    if api == "decode":
        rc = 0
        for f in range(n):
            rc = L.cldn_b200_decode(dec._h, C.byref(c), srcs[f].ctypes.data, len(payloads[f]), outs[f].ptr, caps[f], mem)
            if rc:
                break
    else:
        rc = L.cldn_b200_decode_batch(dec._h, C.byref(c), n, _arr(C.c_void_p, [s.ctypes.data for s in srcs]),
                                      _arr(C.c_size_t, [len(p) for p in payloads]), _arr(C.c_void_p, [o.ptr for o in outs]),
                                      _arr(C.c_size_t, caps), mem, 1)
    msg = _msg() if rc else ""
    return rc, msg, [o.body() for o in outs], all(o.guards_intact() for o in outs)


def _decode_blobs(dec, blobs, caps, mem):
    """decode_blobs of host blobs. Returns (rc, message, statuses, frame messages, decoded bytes, outputs, guards)."""
    n = len(blobs)
    outs = [_points_buf(mem, c) for c in caps]
    srcs = [np.frombuffer(b + b"\0", dtype=np.uint8) for b in blobs]
    status = (C.c_int32 * max(n, 1))()
    decoded = (C.c_size_t * max(n, 1))()
    rc = cb.lib().cldn_b200_decode_blobs(dec._h, n, _arr(C.c_void_p, [s.ctypes.data for s in srcs]), _arr(C.c_size_t, [len(b) for b in blobs]),
                                         _arr(C.c_void_p, [o.ptr for o in outs]), _arr(C.c_size_t, caps), mem, status, decoded)
    msg = _msg() if rc else ""
    return (rc, msg, list(status)[:n], [dec.frame_error(f) for f in range(n)], list(decoded)[:n], [o.body() for o in outs],
            all(o.guards_intact() for o in outs))


def _field_mask(info):
    """True at the bytes of a point that some declared field covers."""
    m = np.zeros(info.point_step, dtype=bool)
    for f in info.fields:
        m[f.offset:f.offset + cb.SizeOf(f.type)] = True
    return m


# ---- encode ------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("version", VERSIONS)
@pytest.mark.parametrize("comp", COMPS, ids=["none", "lz4", "zstd"])
@pytest.mark.parametrize("layout", LAYOUTS)
def test_encode_equals_host_and_oracle(oracle, layout, comp, version):
    info = _layout(layout, 0, 1, version, comp)[0]
    clouds = [_layout(layout, n, 10 + k, version, comp)[1] for k, n in enumerate(SIZES)]
    enc = cb.PointcloudEncoder(info)
    off = UNALIGNED.get(layout, 0)
    for api in ("encode", "batch", "blobs"):
        rc0, msg0, want, guards0 = _encode(enc, api, clouds, HOST)
        rc2, msg2, got, guards2 = _encode(enc, api, clouds, DEVICE_POINTS, off=off)
        assert rc0 == 0 and rc2 == 0, (api, msg0, msg2)
        assert guards0 and guards2, f"{api}: a byte outside a buffer changed"
        for f, (n, a, b) in enumerate(zip(SIZES, want, got)):
            assert b == a, (api, f, n)
            if comp == NONE or oracle.kind == "reference":                      # the C port has no stage 2
                # encode / encode_batch write the handle's header, encode_blobs one with the frame's own dims
                assert b == oracle.encode(_with_dims(info, n, 1) if api == "blobs" else info, clouds[f]), (api, f, n)


@pytest.mark.gpu
@pytest.mark.parametrize("comp", COMPS, ids=["none", "lz4", "zstd"])
@pytest.mark.parametrize("layout", ["xyzi", "c3"])
def test_encode_blobs_with_per_frame_dims(oracle, layout, comp):
    dims = [(100, 60), (0, 4), (32769, 1), (7, 9), (1, 1)]
    info = _layout(layout, 0, 2, 5, comp)[0]
    clouds = [_layout(layout, w * h, 20 + k, 5, comp)[1] for k, (w, h) in enumerate(dims)]
    enc = cb.PointcloudEncoder(info)
    rc0, msg0, want, _ = _encode(enc, "blobs", clouds, HOST, dims=dims)
    rc2, msg2, got, guards = _encode(enc, "blobs", clouds, DEVICE_POINTS, dims=dims)
    assert rc0 == 0 and rc2 == 0 and guards, (msg0, msg2)
    assert got == want
    assert enc.encode_blobs_from_device([0] * 0, [], None) == []
    if comp == NONE or oracle.kind == "reference":
        for (w, h), cloud, blob in zip(dims, clouds, got):
            assert blob == oracle.encode(_with_dims(info, w, h), cloud)


@pytest.mark.gpu
def test_python_wrappers(oracle):
    info, cloud = _layout("xyzi", 50_000, 3, 5, ZSTD)
    enc = cb.PointcloudEncoder(info)
    src = _Dev(cloud.size, src=cloud.tobytes())
    blob = enc.encode_device(src.ptr, cloud.size)
    assert blob == enc.encode(cloud)
    assert enc.encode_device(src.ptr, cloud.size, write_header=False) == enc.encode(cloud, write_header=False)
    for cut in (1, 5):                                                   # the same refusal as encode() of that cloud
        with pytest.raises(RuntimeError) as host:
            enc.encode(cloud[:-cut])
        with pytest.raises(RuntimeError) as dev:
            enc.encode_device(src.ptr, cloud.size - cut)
        assert str(dev.value) == str(host.value) == "Input cloud_data size is not a multiple of point_step"
    clouds = [cloud, _layout("xyzi", 1000, 4, 5, ZSTD)[1]]
    srcs = [src, _Dev(clouds[1].size, src=clouds[1].tobytes())]
    dims = [(50_000, 1), (10, 100)]
    assert enc.encode_blobs_from_device([s.ptr for s in srcs], [c.size for c in clouds], dims) == enc.encode_blobs(clouds, dims)
    assert enc.encode_blobs_from_device([s.ptr for s in srcs], [c.size for c in clouds]) == enc.encode_blobs(clouds)

    dec = cb.PointcloudDecoder()
    dinfo, hdr = cb.DecodeHeader(blob)
    out = _Dev(cloud.size)
    dec.decode_to_device(dinfo, blob[hdr:], out.ptr, out.cap)
    assert np.array_equal(out.body(), cb.PointcloudDecoder().decode(dinfo, blob[hdr:]))
    outs = [_Dev(c.size) for c in clouds]
    blobs = enc.encode_blobs(clouds) + [b"CLOUDINI_V05\nnot a header"]
    outs.append(_Dev(16))
    status, infos = dec.decode_blobs_to_device(blobs, [o.ptr for o in outs], [o.cap for o in outs])
    host = cb.PointcloudDecoder().decode_blobs(blobs)
    assert status == [h[0] for h in host] and status[:2] == [0, 0] and status[2] != 0
    assert infos[:2] == [h[1] for h in host[:2]] and infos[2] is None
    for o, h in zip(outs[:2], host[:2]):
        assert np.array_equal(o.body(), h[2])


@pytest.mark.gpu
@pytest.mark.parametrize("comp", COMPS, ids=["none", "lz4", "zstd"])
def test_encode_refusals_equal_host(comp):
    info, cloud = _layout("c3", 40_000, 5, 5, comp)
    enc = cb.PointcloudEncoder(info)
    clouds = [cloud, _layout("c3", 3, 6, 5, comp)[1]]
    caps = [_worst(info, c.size) for c in clouds]
    cases = [("short", clouds, [caps[0], caps[1] - 1]),
             ("ragged", [clouds[0], clouds[1][:-5]], [caps[0], caps[1]])]
    for what, cl, cp in cases:
        for api in ("encode", "batch", "blobs"):
            rc0, msg0, _, g0 = _encode(enc, api, cl, HOST, caps=cp)
            rc2, msg2, _, g2 = _encode(enc, api, cl, DEVICE_POINTS, caps=cp)
            assert rc0 != 0 and (rc2, msg2) == (rc0, msg0), (what, api)
            assert g0 and g2
    L = cb.lib()
    src = _Dev(cloud.size, src=cloud.tobytes())
    out = _Host(caps[0])
    w = C.c_size_t(0)
    assert L.cldn_b200_encode(enc._h, src.ptr, cloud.size, out.ptr, caps[0], 1, C.byref(w), 3) == -1 and _msg() == "bad mem kind"


# ---- decode ------------------------------------------------------------------------------------------------------------
def _blobs(layout, sizes, version, comp, seed):
    """Host blobs of `layout` (kind 0) and the clouds they encode."""
    info = _layout(layout, 0, seed, version, comp)[0]
    clouds = [_layout(layout, n, seed + k, version, comp)[1] for k, n in enumerate(sizes)]
    return cb.PointcloudEncoder(info).encode_blobs(clouds), clouds


@pytest.mark.gpu
@pytest.mark.parametrize("version", VERSIONS)
@pytest.mark.parametrize("comp", COMPS, ids=["none", "lz4", "zstd"])
@pytest.mark.parametrize("layout", LAYOUTS)
def test_decode_equals_host(layout, comp, version):
    off = UNALIGNED.get(layout, 0)
    blobs, _ = _blobs(layout, SIZES, version, comp, 30)
    dec = cb.PointcloudDecoder()
    for blob in blobs:                                              # decode, frame by frame
        info, hdr = cb.DecodeHeader(blob)
        need = info.width * info.height * info.point_step
        rc0, m0, want, g0 = _decode(dec, "decode", info, [blob[hdr:]], [need], HOST)
        rc2, m2, got, g2 = _decode(dec, "decode", info, [blob[hdr:]], [need], DEVICE_POINTS, off=off)
        assert rc0 == 0 and rc2 == 0 and g0 and g2, (m0, m2)
        assert np.array_equal(got[0], want[0]), info.width
        if need:
            rows = got[0].reshape(-1, info.point_step)
            assert (rows[:, ~_field_mask(info)] == FILL).all(), "a padding byte changed"
    n = SIZES[-2]                                                    # decode_batch: frames of one info
    blobs, _ = _blobs(layout, [n] * 3, version, comp, 40)
    info, hdr = cb.DecodeHeader(blobs[0])
    payloads = [b[cb.DecodeHeader(b)[1]:] for b in blobs]
    caps = [n * info.point_step + 5] * 3
    rc0, m0, want, _ = _decode(dec, "batch", info, payloads, caps, HOST)
    rc2, m2, got, guards = _decode(dec, "batch", info, payloads, caps, DEVICE_POINTS, off=off)
    assert rc0 == 0 and rc2 == 0 and guards, (m0, m2)
    for a, b in zip(want, got):
        assert np.array_equal(a, b)


@pytest.mark.gpu
def test_decode_blobs_mixed_batch():
    blobs = []
    for k, (layout, comp, version) in enumerate([("xyzi", NONE, 5), ("c3", ZSTD, 5), ("xyzirt", LZ4, 4), ("xor", ZSTD, 3),
                                                  ("xyzi", ZSTD, 5), ("gorilla", NONE, 4), ("c3", NONE, 3), ("copy", LZ4, 5)]):
        blobs += _blobs(layout, [SIZES[k % len(SIZES)], 1 + 997 * k], version, comp, 50 + k)[0]
    caps = [(lambda i: i.width * i.height * i.point_step)(cb.DecodeHeader(b)[0]) + 3 for b in blobs]
    dec = cb.PointcloudDecoder()
    want = _decode_blobs(dec, blobs, caps, HOST)
    got = _decode_blobs(dec, blobs, caps, DEVICE_POINTS)
    assert want[0] == 0 and got[:5] == want[:5]
    assert got[6], "a byte outside an output changed"
    for a, b in zip(want[5], got[5]):
        assert np.array_equal(a, b)


def _damaged(blob, at, value):
    b = bytearray(blob)
    b[at:at + len(value)] = value
    return bytes(b)


@pytest.mark.gpu
def test_errors_equal_host():
    # good and damaged frames in one batch: per frame, the same status and message as CLDN_MEM_HOST
    good, _ = _blobs("xyzi", [40_000, 5000], 5, NONE, 60)
    zs, _ = _blobs("c3", [40_000, 3000], 5, ZSTD, 61)
    lz, _ = _blobs("xyzirt", [9000], 5, LZ4, 62)
    hz = cb.DecodeHeader(zs[0])[1]
    hl = cb.DecodeHeader(lz[0])[1]
    hg, hg1 = cb.DecodeHeader(good[0])[1], cb.DecodeHeader(good[1])[1]
    blobs = [good[0],
             _damaged(good[0], hg, b"\xff\xff\xff\x7f"),                  # chunk size past the payload
             good[0][:len(good[0]) - 40],                                 # chunk cut short
             _damaged(zs[0], hz + 4, b"\0\0\0\0"),                        # ZSTD frame magic
             _damaged(lz[0], hl + 4, b"\xff" * 12),                       # LZ4 literal run past the block
             b"CLOUDINX" + good[1][8:],                                   # header
             good[1][:hg1] + good[1],                                      # payload that still carries its header
             zs[1], lz[0], good[1]]
    caps = []
    for b in blobs:
        try:
            i = cb.DecodeHeader(b)[0]
            caps.append(i.width * i.height * i.point_step)
        except RuntimeError:
            caps.append(64)
    caps[7] -= 1                                                          # too small an output
    dec = cb.PointcloudDecoder()
    want = _decode_blobs(dec, blobs, caps, HOST)
    got = _decode_blobs(dec, blobs, caps, DEVICE_POINTS)
    assert got[:5] == want[:5], (got[2], want[2], got[3], want[3])
    assert got[6], "a byte outside an output changed"
    st = want[2]
    assert st[0] == 0 and st[8] == 0 and st[9] == 0 and all(s != 0 for s in st[1:8]), (st, want[3])
    for f in (0, 8, 9):
        assert np.array_equal(want[5][f], got[5][f])
    # the same payloads through decode, alone
    for f, b in enumerate(blobs):
        try:
            info, hdr = cb.DecodeHeader(b)
        except RuntimeError:
            continue
        r0 = _decode(dec, "decode", info, [b[hdr:]], [caps[f]], HOST)
        r2 = _decode(dec, "decode", info, [b[hdr:]], [caps[f]], DEVICE_POINTS)
        assert r2[:2] == r0[:2] and r2[3], f
        if r0[0] == 0:
            assert np.array_equal(r0[2][0], r2[2][0])
    # a device output one byte too small for decode_batch
    info, hdr = cb.DecodeHeader(good[0])
    need = info.width * info.point_step
    r0 = _decode(dec, "batch", info, [good[0][hdr:]], [need - 1], HOST)
    r2 = _decode(dec, "batch", info, [good[0][hdr:]], [need - 1], DEVICE_POINTS)
    assert r0[0] == -2 and r2[:2] == r0[:2] and r2[3] and (r2[2][0] == FILL).all()
    assert cb.lib().cldn_b200_decode(dec._h, C.byref(cb._to_c(info)), None, 0, None, 0, 3) == -1 and _msg() == "bad mem kind"


# ---- streams -----------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.skipif(EMULATED, reason="torch streams: the GPU only")
def test_consumer_on_the_callers_stream_sees_the_points():
    import torch
    info, cloud = _layout("xyzi", 1_000_000, 70, 5, NONE)
    blob = cb.PointcloudEncoder(info).encode(cloud)
    dinfo, hdr = cb.DecodeHeader(blob)
    want = cb.PointcloudDecoder().decode(dinfo, blob[hdr:])
    s = torch.cuda.Stream()
    dec = cb.PointcloudDecoder(stream=s.cuda_stream)
    payload = np.frombuffer(blob[hdr:], dtype=np.uint8)
    out = torch.full((cloud.size,), FILL, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    rc = cb.lib().cldn_b200_decode_batch(dec._h, C.byref(cb._to_c(dinfo)), 1, _arr(C.c_void_p, [payload.ctypes.data]),
                                         _arr(C.c_size_t, [payload.size]), _arr(C.c_void_p, [out.data_ptr()]),
                                         _arr(C.c_size_t, [cloud.size]), DEVICE_POINTS, 0)
    assert rc == 0, _msg()
    with torch.cuda.stream(s):
        seen = out.clone()                                               # the consumer, enqueued behind the decode
    s.synchronize()
    assert np.array_equal(seen.cpu().numpy(), want)
    dec.sync()


@pytest.mark.gpu
@pytest.mark.skipif(EMULATED, reason="torch streams: the GPU only")
def test_encoder_reads_what_a_producer_kernel_wrote():
    import torch
    info, cloud = _layout("xyzi", 1_000_000, 71, 5, ZSTD)
    want = cb.PointcloudEncoder(info).encode(cloud)
    staged = torch.from_numpy(cloud.copy()).cuda()
    dst = torch.full_like(staged, FILL)
    torch.cuda.synchronize()
    producer, s = torch.cuda.Stream(), torch.cuda.Stream()
    enc = cb.PointcloudEncoder(info, stream=s.cuda_stream)
    with torch.cuda.stream(producer):
        torch.cuda._sleep(20_000_000)                                    # the write lands well after the encode is called
        dst.copy_(staged)
        ev = torch.cuda.Event()
        ev.record(producer)
    s.wait_event(ev)
    assert enc.encode_device(dst.data_ptr(), cloud.size) == want


@pytest.mark.gpu
@pytest.mark.skipif(EMULATED, reason="torch streams: the GPU only")
def test_host_decode_after_an_asynchronous_device_points_decode():
    # decode_batch(..., CLDN_MEM_DEVICE_POINTS, sync = 0) returns while its decode still waits on the handle's stream (held
    # back here by a sleep kernel) and reads the payload staged in the decoder's buffer. A CLDN_MEM_HOST decode on the same
    # handle right after it stages its own payload in that buffer: its upload must wait for the earlier decode.
    import torch
    n = 500_000
    info, cloud_a = _layout("xyzi", n, 80, 5, NONE)
    cloud_b = _layout("xyzi", n, 81, 5, NONE)[1]
    enc = cb.PointcloudEncoder(info)
    blob_a, blob_b = enc.encode(cloud_a), enc.encode(cloud_b)
    dinfo, hdr = cb.DecodeHeader(blob_a)
    assert cb.DecodeHeader(blob_b) == (dinfo, hdr)                      # one plan, no synchronisation for a new layout
    pay_a, pay_b = blob_a[hdr:], blob_b[hdr:]
    ref = cb.PointcloudDecoder()
    want_a, want_b = ref.decode(dinfo, pay_a), ref.decode(dinfo, pay_b)
    s = torch.cuda.Stream()
    dec = cb.PointcloudDecoder(stream=s.cuda_stream)
    dec.decode(dinfo, pay_a)                                             # plan and staging buffer sized for both frames
    dec.decode(dinfo, pay_b)
    out_a = torch.full((cloud_a.size,), FILL, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    src_a = np.frombuffer(pay_a, dtype=np.uint8)
    with torch.cuda.stream(s):
        torch.cuda._sleep(200_000_000)                                   # ~0.1 s before frame A's decode may start
    rc = cb.lib().cldn_b200_decode_batch(dec._h, C.byref(cb._to_c(dinfo)), 1, _arr(C.c_void_p, [src_a.ctypes.data]),
                                         _arr(C.c_size_t, [src_a.size]), _arr(C.c_void_p, [out_a.data_ptr()]),
                                         _arr(C.c_size_t, [cloud_a.size]), DEVICE_POINTS, 0)
    assert rc == 0, _msg()
    got_b = dec.decode(dinfo, pay_b)                                     # CLDN_MEM_HOST, at once
    dec.sync()
    assert np.array_equal(got_b, want_b)
    assert np.array_equal(out_a.cpu().numpy(), want_a), "frame A was decoded from another frame's payload"


# ---- emulation -----------------------------------------------------------------------------------------------------------
def test_this_file_under_emulation(lib_built):
    # CUSIM_HOSTCHECK=1: every cudaMalloc region, the caller's device points included, is inaccessible to host code outside a
    # kernel / cudaMemcpy; CUSIM_ASYNC=1: a blob, size or status copied down reads as garbage until the host synchronises
    if platform.machine() != "x86_64":
        pytest.skip("cusim's context switch is x86-64 only")
    if EMULATED:
        pytest.skip("already under the emulation")
    sys.path.insert(0, os.path.join(ROOT, "tests", "cusim"))
    import build_cusim
    env = dict(os.environ, CLDN_B200_LIB=build_cusim.build(), CLDN_B200_ALLOW_EMULATION="tests-only", CUSIM_HOSTCHECK="1", CUSIM_ASYNC="1")
    cmd = [sys.executable, "-m", "pytest", "-x", "-q", "-m", "gpu", "-p", "no:cacheprovider", os.path.abspath(__file__)]
    r = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=2400)
    assert r.returncode == 0 and " passed" in r.stdout and "failed" not in r.stdout, r.stdout[-4000:] + r.stderr[-2000:]
