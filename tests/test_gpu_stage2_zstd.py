"""ZSTD decompression on the device (cldn_zstd.cu): blobs compressed with ZSTD -- Cloudini's default -- decode through the
device-pointer API, and through the host-pointer API without libzstd on the decode path.

The blobs come from the compiled reference where it is available (ref.encode calls ZSTD_compress(..., 1) per chunk,
codec_common.cpp:241-250), else from the host-pointer encoder, which makes the same libzstd call. The expected points
are the oracle's decode of the same blob with stage 2 undone by libzstd.
"""
import os
import struct

import numpy as np
import pytest

import cloudini_b200 as cb
from cloudini_b200 import synth
from test_gpu_parity import _Dev

pytestmark = pytest.mark.gpu
ZSTD = cb.CompressionOption.ZSTD


def _cases():
    n = 70_000
    info, cloud = synth.cloud_c2(n, seed=31)
    yield "xyzi", info, [cloud, synth.cloud_c2(n, seed=32)[1], synth.cloud_c2(n, seed=33)[1]]
    flat = np.tile(np.array([1.5, -2.25, 0.125, 7.0], dtype=np.float32), n).view(np.uint8)
    rnd = np.random.default_rng(5).normal(0, 50.0, (n, 4)).astype(np.float32).view(np.uint8).reshape(-1)
    yield "flat+random", synth.info_xyzi(n), [np.array(flat), rnd]
    info, cloud = synth.cloud_c3(40_001, seed=8)
    yield "c3", info, [cloud]
    info, cloud = synth.cloud_c4_mixed_frame(3)
    yield "xyzirt", info, [cloud, synth.cloud_c4_mixed_frame(4)[1]]
    yield "tiny", synth.info_xyzi(3), [synth.cloud_c2(3, seed=1)[1]]
    rng = np.random.default_rng(77)
    base = np.cumsum(rng.normal(0, 0.02, (977, 4)), axis=0).astype(np.float32)
    m = 2 * 32768 + 5
    yield "periodic-ragged", synth.info_xyzi(m), [np.ascontiguousarray(np.tile(base, (m // 977 + 1, 1))[:m]).view(np.uint8).reshape(-1)]


@pytest.fixture(scope="module")
def blob_source(_ref_oracle):
    """encode(info, cloud) -> ZSTD blob: the compiled reference, else the host-pointer encoder (the same libzstd call)."""
    if _ref_oracle is not None:
        return _ref_oracle.encode
    return lambda info, cloud: cb.PointcloudEncoder(info).encode(cloud)


@pytest.fixture(scope="module")
def zstd_host_route():
    """Context: CLDN_B200_ZSTD_HOST=1 (libzstd on the host) while active."""
    class _Route:
        def __enter__(self):
            os.environ["CLDN_B200_ZSTD_HOST"] = "1"

        def __exit__(self, *a):
            os.environ.pop("CLDN_B200_ZSTD_HOST", None)
    return _Route()


def _device_decode(info, payloads, n_bytes, fill=0):
    dec = cb.PointcloudDecoder()
    d_in = [_Dev(src=np.frombuffer(p, dtype=np.uint8)) if len(p) else _Dev(size=16) for p in payloads]
    d_out = [_Dev(src=np.full(n_bytes, fill, dtype=np.uint8)) for _ in payloads]
    batch = dec.make_device_batch([t.ptr for t in d_in], [len(p) for p in payloads], [t.ptr for t in d_out], [n_bytes] * len(payloads))
    dec.decode_batch_device(info, batch, sync=True)
    return [o.numpy() for o in d_out]


def _host_decode(info, payload, n_bytes, fill=0):
    out = np.full(n_bytes, fill, dtype=np.uint8)
    cb.PointcloudDecoder().decode(info, payload, out)
    return out


def _want(oracle, blob, n_bytes, fill):
    out = np.full(n_bytes, fill, dtype=np.uint8)
    oracle.decode(blob, out)
    return out


@pytest.mark.parametrize("case", list(_cases()), ids=lambda c: c[0])
def test_zstd_blobs_decode_bit_exact_through_both_apis(oracle, blob_source, case):
    name, info, clouds = case
    info.compression_opt = ZSTD
    n_bytes = clouds[0].size
    blobs = [blob_source(info, c) for c in clouds]
    dinfo, hdr = cb.DecodeHeader(blobs[0])
    assert dinfo.compression_opt == ZSTD
    wants = [_want(oracle, b, n_bytes, 0x2E) for b in blobs]   # 0x2E: padding bytes must come back untouched
    got = _device_decode(dinfo, [b[hdr:] for b in blobs], n_bytes, 0x2E)
    for g, w in zip(got, wants):
        assert np.array_equal(g, w), name
    for b, w in zip(blobs, wants):
        assert np.array_equal(_host_decode(dinfo, b[hdr:], n_bytes, 0x2E), w), name


def test_many_frames_per_batch_and_damaged_batches(oracle):
    n = 40_000
    info, _ = synth.cloud_c2(n, seed=1)
    info.compression_opt = ZSTD
    clouds = [synth.cloud_c2(n, seed=100 + k)[1] for k in range(24)]
    enc = cb.PointcloudEncoder(info)
    blobs = [enc.encode(c) for c in clouds]
    dinfo, hdr = cb.DecodeHeader(blobs[0])
    got = _device_decode(dinfo, [b[hdr:] for b in blobs], n * 16)
    for g, b in zip(got, blobs):
        assert np.array_equal(g, _want(oracle, b, n * 16, 0))
    good = blobs[3][hdr:]
    c0 = struct.unpack_from("<I", good)[0]
    bad = struct.pack("<I", c0 - 5) + good[4:4 + c0 - 5] + good[4 + c0:]   # chunk 0's frame loses its last 5 bytes
    with pytest.raises(RuntimeError, match="ZSTD decompression failed"):
        _device_decode(dinfo, [b[hdr:] for b in blobs[:3]] + [bytes(bad)] + [b[hdr:] for b in blobs[4:8]], n * 16)
    again = _device_decode(dinfo, [b[hdr:] for b in blobs[8:12]], n * 16)   # the handle recovers: the next batch is intact
    for g, b in zip(again, blobs[8:12]):
        assert np.array_equal(g, _want(oracle, b, n * 16, 0))


def _damage(rng, payload: bytes) -> bytes:
    b = bytearray(payload)
    kind = rng.integers(4)
    if kind == 0:
        for _ in range(int(rng.integers(1, 4))):
            b[int(rng.integers(len(b)))] ^= 1 << int(rng.integers(8))
    elif kind == 1:
        del b[int(rng.integers(1, len(b))):]
    elif kind == 2:
        b[4 + int(rng.integers(0, 40))] = int(rng.integers(256))          # frame / block / literals headers of chunk 0
    else:
        c0 = struct.unpack_from("<I", b)[0]
        b[4 + c0 - 1 - int(rng.integers(0, 16))] ^= 1 << int(rng.integers(8))  # the end of chunk 0's sequences
    return bytes(b)


def _status(fn):
    try:
        return "ok", fn()
    except RuntimeError:
        return "error", None


def test_damaged_blobs_fail_exactly_like_libzstd(zstd_host_route):
    # the device route (default) and the libzstd route (CLDN_B200_ZSTD_HOST=1) of the host-pointer API: the same
    # outcome and, when both succeed, the same points -- on intact and on damaged payloads
    n = 40_000
    info, cloud = synth.cloud_c2(n, seed=3)
    info.compression_opt = ZSTD
    blob = cb.PointcloudEncoder(info).encode(cloud)
    dinfo, hdr = cb.DecodeHeader(blob)
    rng = np.random.default_rng(int(os.environ.get("CLDN_B200_FUZZ_SEED", "2026")))
    count = int(os.environ.get("CLDN_ZSTD_GPU_DAMAGED", "150"))
    outcomes = {"ok": 0, "error": 0}
    for trial in range(count):
        bad = _damage(rng, blob[hdr:]) if trial else blob[hdr:]
        dev = _status(lambda: _host_decode(dinfo, bad, n * 16, 0x11))
        with zstd_host_route:
            host = _status(lambda: _host_decode(dinfo, bad, n * 16, 0x11))
        assert dev[0] == host[0], trial
        if dev[0] == "ok":
            assert np.array_equal(dev[1], host[1]), trial
        outcomes[dev[0]] += 1
        # the device-pointer API agrees too
        dptr = _status(lambda: _device_decode(dinfo, [bad], n * 16, 0x11)[0])
        assert dptr[0] == dev[0], trial
        if dptr[0] == "ok":
            assert np.array_equal(dptr[1], dev[1]), trial
    assert outcomes["error"] > count // 4 and outcomes["ok"] >= 1


def test_default_host_route_runs_the_zstd_kernel(zstd_host_route):
    n = 70_000
    info, cloud = synth.cloud_c2(n, seed=9)
    info.compression_opt = ZSTD
    blob = cb.PointcloudEncoder(info).encode(cloud)
    dinfo, hdr = cb.DecodeHeader(blob)
    before = cb.kernel_launch_count()
    a = _host_decode(dinfo, blob[hdr:], n * 16)
    device_launches = cb.kernel_launch_count() - before
    with zstd_host_route:
        before = cb.kernel_launch_count()
        b = _host_decode(dinfo, blob[hdr:], n * 16)
        host_launches = cb.kernel_launch_count() - before
    assert np.array_equal(a, b)
    assert device_launches >= host_launches + 2   # the chunk decompressor and the re-framing kernel


def test_device_pointer_api_decodes_what_it_refused_before():
    # a blob written with the default compression: before the device decompressor, the device-pointer API refused it
    # ("stage 2 is undone before the stage-1 decode")
    n = 33_000
    info, cloud = synth.cloud_c2(n, seed=12)
    info.compression_opt = ZSTD   # EncodingInfo's default
    blob = cb.PointcloudEncoder(info).encode(cloud)
    dinfo, hdr = cb.DecodeHeader(blob)
    got = _device_decode(dinfo, [blob[hdr:]], n * 16)[0]
    assert np.array_equal(got, _host_decode(dinfo, blob[hdr:], n * 16))


def test_dds_converter_decompresses_the_references_zstd_message(ref):
    # the reference's own compressed message (ZSTD), as tests/test_gpu_ros.py builds it, through the converter's
    # decompress direction: byte-identical to the reference's PointCloud2
    import ctypes as C
    from cloudini_b200 import ros
    L = cb.lib()
    u32, vp = C.c_uint32, C.c_void_p
    L.cldn_b200_ConvertCompressedMsgToPointCloud2Msg.restype, L.cldn_b200_ConvertCompressedMsgToPointCloud2Msg.argtypes = u32, [vp, u32, vp, u32]
    from cloudini_b200 import FieldType as FT
    XYZI = [("x", 0, FT.FLOAT32), ("y", 4, FT.FLOAT32), ("z", 8, FT.FLOAT32), ("intensity", 12, FT.FLOAT32)]
    info, cloud = synth.cloud_c2(30_000, seed=8)
    msg = synth.pointcloud2_msg(XYZI, 16, cloud)
    try:
        comp = np.frombuffer(ref.ros_compress(bytes(msg), {}, 0.001, False, 1, 2, 5), dtype=np.uint8)
        want = ref.ros_decompress(bytes(comp), len(msg) + 64)
    except (KeyError, LookupError, NotImplementedError) as e:
        pytest.skip(f"the compiled reference is not available: {e}")
    full = np.zeros(len(msg) + 64, dtype=np.uint8)
    m = L.cldn_b200_ConvertCompressedMsgToPointCloud2Msg(comp.ctypes.data, comp.size, full.ctypes.data, full.size)
    assert m > 0 and bytes(full[:m]) == want
    del ros
