"""Stage 2 on the device for encoders that ask for it (cldn_b200_encoder_set_stage2_on_device): ZSTD frames of
Huffman-coded literal blocks (cldn_zstd_enc.cu) and LZ4 blocks (cldn_lz4.cu), for all three memory kinds.

The frames are not libzstd's bytes, so they are checked for what they promise: every chunk's frame, given to libzstd's
ZSTD_decompress, is that chunk's stage-1 bytes from the oracle's NONE encode; every blob decodes to the oracle's points
through every decode route; a blob's bytes do not depend on the memory kind, the call, the batch or the run; the frame
uses every block form the coder has; and its size stays within a few per cent of ZSTD_compress(level 1) on the same
chunks. Outputs sit between guard bytes.
"""
import ctypes as C
import os
import platform
import random
import struct
import subprocess
import sys
import threading

import numpy as np
import pytest

import cloudini_b200 as cb
from cloudini_b200 import FieldType as FT
from cloudini_b200 import synth
from test_gpu_device_points import _Dev, _Host, _arr, _field_mask, _layout, _msg, _with_dims
from zstd_corpus import compress, decompress, zstd_lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMULATED = bool(os.environ.get("CLDN_B200_LIB"))
HOST, DEVICE, DEVICE_POINTS = cb.MEM_HOST, cb.MEM_DEVICE, cb.MEM_DEVICE_POINTS
MEMS = [HOST, DEVICE, DEVICE_POINTS]
NONE, LZ4, ZSTD = cb.CompressionOption.NONE, cb.CompressionOption.LZ4, cb.CompressionOption.ZSTD
VERSIONS = [5] if EMULATED else [3, 4, 5]
MULTI = 70_000 if EMULATED else 200_000
SIZES = [0, 1, 32767, 32768, 32769, MULTI]
LAYOUTS = ["xyz", "xyzi", "xyzirt", "c3", "gorilla", "xor", "copy"]
SEEDS = [3, 7, 14] if EMULATED else [3, 7, 14, 21, 28, 35, 42]
BLOCK = 32 * 1024                       # stage-1 bytes per ZSTD block (cldn_zstd_enc.cu kZeBlock)
MIN_HUFF = 64                           # fewer bytes in a block: a raw block (kZeMinHuff)
ERR_INVALID_ARGUMENT, ERR_BUFFER_TOO_SMALL, ERR_UNSUPPORTED = -1, -2, -5


def _chunks(payload):
    """The chunk bodies of a header-less payload ([u32 size][bytes])*."""
    out, p = [], 0
    while p < len(payload):
        (n,) = struct.unpack_from("<I", payload, p)
        out.append(payload[p + 4:p + 4 + n])
        p += 4 + n
    assert p == len(payload)
    return out


def _encoder(info, comp, on=True):
    info = _with_dims(info, info.width, info.height)
    info.compression_opt = comp
    enc = cb.PointcloudEncoder(info)
    enc.set_stage2_on_device(on)
    return enc


def _exact_caps(info, api, clouds, dims=None):
    """MaxCompressedSize of every frame with the header it is written with: encode_blobs the frame's own dims,
    encode / encode_batch the handle's."""
    def hdr_dims(f, c):
        return dims[f] if dims else (c.size // info.point_step, 1) if api == "blobs" else (info.width, info.height)
    return [cb.MaxCompressedSize(_with_dims(info, *hdr_dims(f, c)), c.size // info.point_step, True) for f, c in enumerate(clouds)]


def _run(enc, api, clouds, mem, caps=None, dims=None):
    """One encode entry point with clouds in `mem`'s point memory, blobs in `mem`'s blob memory, all between guards.
    Returns (rc, message, blobs, every guard intact)."""
    info = enc.getEncodingInfo()
    n = len(clouds)
    caps = caps or _exact_caps(info, api, clouds, dims)
    pts = _Dev if mem in (DEVICE, DEVICE_POINTS) else _Host
    ins = [pts(max(c.size, 1), src=c.tobytes() + b"\0" * (c.size == 0)) for c in clouds]
    outs = [(_Dev if mem == DEVICE else _Host)(cap) for cap in caps]
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


def _payload(blob):
    return blob[cb.DecodeHeader(blob)[1]:]


def _decode_blobs(blobs, mem):
    """decode_blobs of host blobs into `mem`'s point memory: (rc, statuses, outputs)."""
    caps = [(lambda i: max(i.width * i.height * i.point_step, 1))(cb.DecodeHeader(b)[0]) for b in blobs]
    outs = [(_Dev if mem == DEVICE_POINTS else _Host)(c) for c in caps]
    srcs = [np.frombuffer(b + b"\0", dtype=np.uint8) for b in blobs]
    status = (C.c_int32 * len(blobs))()
    decoded = (C.c_size_t * len(blobs))()
    dec = cb.PointcloudDecoder()
    rc = cb.lib().cldn_b200_decode_blobs(dec._h, len(blobs), _arr(C.c_void_p, [s.ctypes.data for s in srcs]),
                                         _arr(C.c_size_t, [len(b) for b in blobs]), _arr(C.c_void_p, [o.ptr for o in outs]),
                                         _arr(C.c_size_t, caps), mem, status, decoded)
    assert all(o.guards_intact() for o in outs)
    return rc, list(status), [o.body()[:d] for o, d in zip(outs, decoded)]


def _check_frames(z, oracle, info, clouds, blobs):
    """Every chunk frame of every blob is, through libzstd / liblz4's format, the oracle's stage-1 chunk."""
    plain_info = _with_dims(info, info.width, info.height)
    plain_info.compression_opt = NONE
    for cloud, blob in zip(clouds, blobs):
        want = _chunks(oracle.encode(_with_dims(plain_info, cloud.size // info.point_step, 1), cloud, write_header=False))
        got = _chunks(_payload(blob))
        assert len(got) == len(want)
        for a, b in zip(want, got):
            if info.compression_opt == ZSTD:
                assert len(b) <= z.ZSTD_compressBound(len(a))
                ok, out = decompress(z, b, len(a))
                assert ok and out == a
            else:
                out = C.create_string_buffer(len(a) + 1)
                assert _lz4().LZ4_decompress_safe(b, out, len(b), len(a) + 1) == len(a)
                assert out.raw[:len(a)] == a


_LZ4 = None


def _lz4():
    global _LZ4
    if _LZ4 is None:
        try:
            _LZ4 = C.CDLL("liblz4.so.1")
        except OSError:
            pytest.skip("liblz4.so.1 is not installed")
        _LZ4.LZ4_decompress_safe.argtypes = [C.c_char_p, C.c_void_p, C.c_int, C.c_int]
    return _LZ4


def _check_decodes(oracle, info, clouds, blobs, monkeypatch):
    """Every blob decodes to the oracle's points: decode_blobs (host and device points), the host libzstd route, and the
    compiled reference where it exists."""
    plain = _with_dims(info, info.width, info.height)
    plain.compression_opt = NONE
    want = []
    for cloud in clouds:
        ref = oracle.encode(_with_dims(plain, cloud.size // info.point_step, 1), cloud)
        out = np.zeros(cloud.size, dtype=np.uint8)
        if cloud.size:
            oracle.decode(ref, out)
        want.append(out)
    mask = np.tile(_field_mask(info), max((c.size // info.point_step for c in clouds), default=0))  # padding is left as it was
    routes = [("host", HOST, None), ("device", DEVICE_POINTS, None)]
    if info.compression_opt == ZSTD:
        routes.append(("zstd_host", HOST, "1"))
    for name, mem, zhost in routes:
        if zhost:
            monkeypatch.setenv("CLDN_B200_ZSTD_HOST", zhost)
        rc, status, outs = _decode_blobs(blobs, mem)
        monkeypatch.delenv("CLDN_B200_ZSTD_HOST", raising=False)
        assert rc == 0 and status == [0] * len(blobs), (name, status)
        for w, g in zip(want, outs):
            assert np.array_equal(w[mask[:w.size]], g[mask[:g.size]]), name
    if oracle.kind == "reference":
        for w, blob in zip(want, blobs):
            out = np.zeros(w.size, dtype=np.uint8)
            if w.size:
                oracle.decode(blob, out)
            assert np.array_equal(out[mask[:w.size]], w[mask[:w.size]]), "reference"


def _cases():
    return [(name, None) for name in LAYOUTS] + [(f"random{s}", s) for s in SEEDS]


def _case(name, seed, version, sizes):
    if seed is None:
        info = _layout(name, 0, 1, version, ZSTD)[0]
        return info, [_layout(name, n, 10 + k, version, ZSTD)[1] for k, n in enumerate(sizes)]
    info, cloud = synth.random_layout_case(seed)
    info.use_threads = False
    n = cloud.size // info.point_step
    cuts = sorted({0, 1, n // 2, n})
    return _with_dims(info, n, 1), [np.ascontiguousarray(cloud[:k * info.point_step]) for k in cuts]


# ---- 1. frame validity ---------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("version", VERSIONS)
@pytest.mark.parametrize("name,seed", _cases(), ids=[c[0] for c in _cases()])
def test_frames_are_valid_and_decode_everywhere(oracle, name, seed, version, monkeypatch):
    z = zstd_lib()
    if seed is not None and version != VERSIONS[-1]:
        pytest.skip("random layouts carry their own wire version")
    info, clouds = _case(name, seed, version, SIZES)
    info.compression_opt = NONE
    try:
        oracle.encode(info, clouds[-1])
    except RuntimeError:
        pytest.skip("a layout the reference refuses")
    info.compression_opt = ZSTD
    enc = _encoder(info, ZSTD)
    first = None
    for mem in MEMS:
        for api in ("blobs", "encode", "batch"):          # encode_blobs first: headers with each frame's own width
            rc, msg, blobs, guards = _run(enc, api, clouds, mem)
            assert rc == 0 and guards, (mem, api, msg)
            payloads = [_payload(b) for b in blobs]
            if first is None:
                first = payloads
                _check_frames(z, oracle, enc.getEncodingInfo(), clouds, blobs)
                _check_decodes(oracle, enc.getEncodingInfo(), clouds, blobs, monkeypatch)
            assert payloads == first, (mem, api)
            if api != "blobs":
                assert all(b[:len(enc.getHeader())] == enc.getHeader() for b in blobs)
            else:
                for c, b in zip(clouds, blobs):
                    assert cb.DecodeHeader(b)[0].width == c.size // info.point_step


# ---- 2. the same bytes everywhere, capacities, LZ4 ------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("comp", [ZSTD, LZ4], ids=["zstd", "lz4"])
def test_same_bytes_in_any_batch_and_capacity_rule(oracle, comp, monkeypatch):
    z = zstd_lib()
    rng = random.Random(5)
    nf = 12 if EMULATED else 128
    sizes = [rng.choice([0, 1, 77, 32768, 40_000, rng.randrange(1, 100_000 if EMULATED else 300_000)]) for _ in range(nf)]
    info = _layout("c3", 0, 1, 5, comp)[0]
    clouds = [_layout("c3", n, 100 + k, 5, comp)[1] for k, n in enumerate(sizes)]
    enc = _encoder(info, comp)
    rc, _, batch, guards = _run(enc, "blobs", clouds, DEVICE)
    assert rc == 0 and guards
    _check_frames(z, oracle, enc.getEncodingInfo(), clouds, batch)
    _check_decodes(oracle, enc.getEncodingInfo(), clouds[:8], batch[:8], monkeypatch)
    for mem in MEMS:
        rc, _, again, guards = _run(enc, "blobs", clouds, mem)        # a second run, every memory kind
        assert rc == 0 and guards and again == batch, mem
    for f in (0, 1, nf // 2, nf - 1):                                 # a frame alone
        other = _encoder(info, comp)
        rc, _, alone, _ = _run(other, "blobs", [clouds[f]], DEVICE)
        assert rc == 0 and alone[0] == batch[f], f
    # capacity: exactly MaxCompressedSize, and one byte short (the default policy's status and message)
    pick = [clouds[k] for k in (0, 2, 4)]
    default = _encoder(info, comp, on=False)
    for api in ("encode", "batch", "blobs"):
        exact = _exact_caps(enc.getEncodingInfo(), api, pick)
        for mem in MEMS:
            rc, msg, blobs, guards = _run(enc, api, pick, mem, caps=exact)
            assert rc == 0 and guards, (api, mem, msg)
            short = [exact[0], exact[1] - 1, exact[2]]
            rc, msg, _, guards = _run(enc, api, pick, mem, caps=short)
            ref_mem = HOST if (comp == ZSTD and mem == DEVICE) else mem
            rc0, msg0, _, _ = _run(default, api, pick, ref_mem, caps=short)
            assert guards and rc == rc0 == ERR_BUFFER_TOO_SMALL and msg == msg0, (api, mem, msg, msg0)


# ---- 3. every block form -----------------------------------------------------------------------------------------------
COPY_STEP = 32   # four copied UINT64 fields: any byte string of whole points is a stage-1 chunk, of up to 1 MB


def _copy_info(n):
    return cb.EncodingInfo(fields=[cb.PointField(f"f{k}", 8 * k, FT.UINT64) for k in range(4)], width=n, height=1,
                           point_step=COPY_STEP, encoding_opt=cb.EncodingOptions.NONE, compression_opt=ZSTD, use_threads=False,
                           version=4)


def _blocks(frame):
    """(type, size, last, literals byte 0, tree header byte, weights) per block of one frame written by the coder."""
    fhd = frame[4]
    p = 5 + (1, 2, 4, 8)[fhd >> 6]
    out = []
    while True:
        (h,) = struct.unpack_from("<I", frame[p:p + 3] + b"\0")
        last, bt, size = h & 1, (h >> 1) & 3, h >> 3
        p += 3
        if bt == 2:
            lh = (3, 3, 4, 5)[(frame[p] >> 2) & 3]
            hb = frame[p + lh]
            weights = [w for b in frame[p + lh + 1:p + lh + 1 + (hb - 127 + 1) // 2] for w in (b >> 4, b & 15)][:hb - 127] if hb >= 128 else None
            out.append((bt, size, last, frame[p], hb, weights))
        else:
            out.append((bt, size, last, None, None, None))
        p += 1 if bt == 1 else size
        if last:
            break
    assert p == len(frame)
    return out


def _max_bits(weights):
    total = sum(1 << (w - 1) for w in weights if w)
    return total.bit_length()     # highbit(total) + 1


@pytest.mark.gpu
def test_every_block_form_is_reached():
    z = zstd_lib()
    rng = random.Random(9)
    fib = [1, 1]
    while len(fib) < 16:
        fib.append(fib[-1] + fib[-2])
    fibs = b"".join(bytes([s]) * f for s, f in enumerate(fib))     # 16 symbols < 128: the deepest code is 15 > 11 bits
    corpus = {
        "rle": bytes([7]) * 5000,
        "random": rng.randbytes(70_000),                                 # 256 equally likely values: raw
        "high_symbols": bytes(rng.choice([0, 1, 2, 3, 200]) for _ in range(9000)),
        "low_symbols": bytes(rng.choice(b"abcdefgh") for _ in range(9000)),
        "fibonacci": (fibs * (40_000 // len(fibs) + 1))[:40_000],
        "dominant": bytes(rng.choice([0] * 200 + [1, 2]) for _ in range(20_000)),
        "short_tail": bytes(rng.choice(b"xyz") for _ in range(BLOCK + COPY_STEP)),
        "many_blocks": bytes(rng.randrange(0, 50) for _ in range(5 * BLOCK + 1000)),
    }
    seen = set()
    enc_cache = {}
    for name, data in corpus.items():
        data = data[:len(data) // COPY_STEP * COPY_STEP]
        n = len(data)
        enc = enc_cache.setdefault(n, _encoder(_copy_info(n // COPY_STEP), ZSTD))
        rc, msg, blobs, guards = _run(enc, "batch", [np.frombuffer(data, dtype=np.uint8)], DEVICE_POINTS)
        assert rc == 0 and guards, msg
        (frame,) = _chunks(_payload(blobs[0]))
        ok, out = decompress(z, frame, n)
        assert ok and out == data, name
        blocks = _blocks(frame)
        for bt, size, last, lit0, hb, weights in blocks:
            if bt == 1:
                seen.add("rle_block")
            elif bt == 0:
                seen.add("raw_block")
                if last and size < MIN_HUFF and len(blocks) > 1:
                    seen.add("short_tail")
            else:
                assert lit0 & 3 == 2 and (lit0 >> 2) & 3 != 0, name      # Huffman literals, four streams
                seen.add("fse_weights" if hb < 128 else "direct_weights")
                if weights is not None and _max_bits(weights) == 11:
                    seen.add("11_bit_code")
                if name == "dominant":
                    seen.add("dominant")
        if len(blocks) >= 5:
            seen.add("many_blocks")
    want = {"rle_block", "raw_block", "fse_weights", "direct_weights", "11_bit_code", "dominant", "short_tail", "many_blocks"}
    assert want <= seen, want - seen


# ---- 4. ratio against ZSTD_compress(level 1) ---------------------------------------------------------------------------
RATIO = [("cloud_c2", lambda: synth.cloud_c2(300_000 if EMULATED else 1_000_000, seed=1000), 1.02),
         ("cloud_c4_frame", lambda: synth.cloud_c4_frame(0), 1.02),
         ("cloud_c3", lambda: synth.cloud_c3(300_000 if EMULATED else 1_000_000), 1.03),
         ("cloud_viz", lambda: synth.cloud_viz(200_000), 1.06)]


@pytest.mark.gpu
@pytest.mark.parametrize("name,make,limit", RATIO, ids=[r[0] for r in RATIO])
def test_ratio_against_libzstd_level_1(oracle, name, make, limit):
    z = zstd_lib()
    info, cloud = make()
    info.compression_opt = NONE
    plain = _chunks(oracle.encode(info, cloud, write_header=False))
    enc = _encoder(info, ZSTD)
    rc, msg, blobs, _ = _run(enc, "batch", [cloud], DEVICE_POINTS)
    assert rc == 0, msg
    frames = _chunks(_payload(blobs[0]))
    ours = sum(map(len, frames))
    lib1 = sum(len(compress(z, c, 1)) for c in plain)
    for c, f in zip(plain, frames):
        assert len(f) <= len(c) + 3 * max(1, -(-len(c) // BLOCK)) + 13
    assert ours <= limit * lib1, f"{name}: {ours / lib1:.4f} x libzstd level 1 ({ours} / {lib1} bytes)"


# ---- 5. concurrency ----------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_two_handles_on_two_streams_equal_the_calls_alone():
    infos = [_layout("xyzi", 0, 1, 5, ZSTD)[0], _layout("xyzirt", 0, 1, 5, LZ4)[0]]
    comps = [ZSTD, LZ4]
    work = [[_layout(l, n, 300 + k, 5, c)[1] for k, n in enumerate([33_000, 5, 70_000])] for l, c in (("xyzi", ZSTD), ("xyzirt", LZ4))]
    alone = []
    for info, comp, clouds in zip(infos, comps, work):
        rc, _, blobs, _ = _run(_encoder(info, comp), "batch", clouds, DEVICE)
        assert rc == 0
        alone.append(blobs)
    encs = [_encoder(info, comp) for info, comp in zip(infos, comps)]   # each handle has its own stream
    got = [[], []]

    def worker(h):
        for mem in (DEVICE, HOST, DEVICE_POINTS, DEVICE):
            got[h].append(_run(encs[h], "batch", work[h], mem))

    threads = [threading.Thread(target=worker, args=(h,)) for h in (0, 1)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    for h in (0, 1):
        for rc, msg, blobs, guards in got[h]:
            assert rc == 0 and guards and blobs == alone[h], (h, msg)


# ---- 6. Python, launches, policy ---------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_python_policy_round_trip_and_launch_count():
    info, cloud = _layout("xyzi", 50_000, 3, 5, ZSTD)
    enc = cb.PointcloudEncoder(info)
    default = enc.encode(cloud)
    assert default == cb.PointcloudEncoder(info).encode(cloud)
    enc.set_stage2_on_device(True)
    on = enc.encode(cloud)
    assert on != default and cb.DecodeHeader(on) == cb.DecodeHeader(default)
    dinfo, hdr = cb.DecodeHeader(on)
    assert np.array_equal(cb.PointcloudDecoder().decode(dinfo, on[hdr:]), cb.PointcloudDecoder().decode(dinfo, default[hdr:]))
    assert enc.encode_blobs([cloud]) == [on]
    enc.set_stage2_on_device(False)
    assert enc.encode(cloud) == default
    assert cb.lib().cldn_b200_encoder_set_stage2_on_device(enc._h, 2) == ERR_INVALID_ARGUMENT
    # the default still refuses device blobs with ZSTD
    rc, msg, _, _ = _run(enc, "batch", [cloud], DEVICE)
    assert rc == ERR_UNSUPPORTED and "host-pointer API" in msg
    # launches: stage 1 + the compressor + the pack, whatever the batch
    enc.set_stage2_on_device(True)
    plain = _encoder(info, NONE)
    for clouds in ([cloud], [cloud] * 7):
        for comp_enc in (enc, _encoder(info, LZ4)):
            c0 = cb.kernel_launch_count()
            assert _run(plain, "batch", clouds, DEVICE)[0] == 0
            c1 = cb.kernel_launch_count()
            assert _run(comp_enc, "batch", clouds, DEVICE)[0] == 0
            c2 = cb.kernel_launch_count()
            assert c2 - c1 == (c1 - c0) + 2, (len(clouds), c1 - c0, c2 - c1)


class _Handle:
    """A library-owned encoder handle in the shape _run takes."""

    def __init__(self, h, info):
        self._h, self._info = h, info

    def getEncodingInfo(self):
        return self._info


@pytest.mark.gpu
def test_pool_encoders_refuse_the_policy_and_keep_the_library_bytes():
    # the per-thread pool's handles (cldn_b200_pool_encoder) are the ones the DDS converter and the ros shims use, and
    # those promise the system libraries' bytes
    from cloudini_b200 import ros
    L = cb.lib()
    L.cldn_b200_pool_encoder.argtypes = [C.POINTER(cb._CInfo), C.POINTER(C.c_void_p)]
    fields = [("x", 0, FT.FLOAT32), ("y", 4, FT.FLOAT32), ("z", 8, FT.FLOAT32), ("intensity", 12, FT.FLOAT32)]
    msg = synth.pointcloud2_msg(fields, 16, synth.cloud_viz(40_000, seed=5)[1])
    for comp in (ZSTD, LZ4):
        before = ros.convert_message(msg, {}, 0.001, False, cb.EncodingOptions.LOSSY, comp, 5)
        info = _layout("xyzi", 40_000, 3, 5, comp)[0]
        h = C.c_void_p()
        assert L.cldn_b200_pool_encoder(C.byref(cb._to_c(info)), C.byref(h)) == 0
        assert L.cldn_b200_encoder_set_stage2_on_device(h, 1) == ERR_INVALID_ARGUMENT and "pool encoder" in _msg()
        assert L.cldn_b200_encoder_set_stage2_on_device(h, 0) == 0
        assert ros.convert_message(msg, {}, 0.001, False, cb.EncodingOptions.LOSSY, comp, 5) == before
        # the pool's handle still encodes the library's bytes
        cloud = _layout("xyzi", 40_000, 3, 5, comp)[1]
        rc, msg_, blobs, _ = _run(_Handle(h, info), "batch", [cloud], HOST)
        assert rc == 0 and blobs == [cb.PointcloudEncoder(info).encode(cloud)], msg_


# ---- 7. the same file under the CPU emulation, and the kernels under ThreadSanitizer ------------------------------------
@pytest.mark.skipif(EMULATED, reason="already running under the emulation")
def test_this_file_under_emulation(lib_built):
    if platform.machine() != "x86_64":
        pytest.skip("cusim's context switch is x86-64 only")
    sys.path.insert(0, os.path.join(ROOT, "tests", "cusim"))
    import build_cusim
    env = dict(os.environ, CLDN_B200_LIB=build_cusim.build(), CLDN_B200_ALLOW_EMULATION="tests-only", CUSIM_HOSTCHECK="1", CUSIM_ASYNC="1")
    cmd = [sys.executable, "-m", "pytest", "-x", "-q", "-m", "gpu", "-p", "no:cacheprovider", os.path.abspath(__file__)]
    r = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=3000)
    assert r.returncode == 0 and " passed" in r.stdout and "failed" not in r.stdout, r.stdout[-4000:] + r.stderr[-2000:]


@pytest.mark.skipif(EMULATED, reason="already running under the emulation")
def test_device_stage2_under_thread_sanitizer(lib_built, tmp_path):
    # tests/cusim/zstd_encode_racecheck_main.cpp: ZSTD and LZ4 on the device for every memory kind, every CUDA thread a
    # ThreadSanitizer fiber (strict model: a shuffle is no fence)
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
    drv, exe = str(tmp_path / "zstd_encode_main.o"), str(tmp_path / "zstd_encode_racecheck")
    subprocess.check_call(["g++", "-std=c++17", "-O0", "-g", "-fPIC", "-pthread", "-w", "-fsanitize=thread", "-I", here, "-I",
                           os.path.join(ROOT, "include"), "-x", "c++", "-c", os.path.join(here, "zstd_encode_racecheck_main.cpp"), "-o", drv])
    subprocess.check_call(["g++", "-fsanitize=thread", "-pthread", "-o", exe, drv, *objs, "-ldl"])
    env = dict(os.environ, TSAN_OPTIONS="halt_on_error=0 report_signal_unsafe=0", CUSIM_WORKERS="4", CUSIM_TSAN_STRICT="1")
    env.pop("LD_PRELOAD", None)
    r = subprocess.run([exe], env=env, capture_output=True, text=True, timeout=1500)
    if "FATAL: ThreadSanitizer" in r.stderr:
        pytest.skip("ThreadSanitizer cannot run in this environment: " + r.stderr[-200:])
    assert r.returncode == 0 and "zstd_encode_racecheck: done" in r.stdout, r.stdout[-2000:] + r.stderr[-3000:]
    assert "WARNING: ThreadSanitizer" not in r.stderr, r.stderr[-4000:]
