"""GPU parity tests (H100): every byte the CUDA path produces is compared with the oracle on the same input.
Encode: blob == oracle blob (header + every chunk). Decode: decoded buffer == oracle-decoded buffer, starting from the
same pre-filled buffer (the decoder only writes declared field bytes). All calls go through the C ABI."""
import os

import numpy as np
import pytest

import cloudini_b200 as cb
from cloudini_b200 import synth

pytestmark = pytest.mark.gpu


def _emulated():
    """True when the suite is re-run by tests/test_cusim_kernels.py against the CPU emulation of the CUDA model
    (tests/cusim: test infrastructure, the kernels' logic checked without a GPU). There "device" memory is host memory."""
    return b"cusim" in cb.lib().cldn_b200_version()


class _Dev:
    """A device buffer for the device-pointer API: a torch CUDA tensor on the GPU box, a numpy array under cusim."""

    def __init__(self, src=None, size=None):
        if _emulated():
            self.t = np.array(src, dtype=np.uint8, copy=True) if src is not None else np.zeros(size, dtype=np.uint8)
            self.ptr = self.t.ctypes.data
        else:
            import torch
            self.t = (torch.from_numpy(np.array(src, dtype=np.uint8, copy=True)).cuda() if src is not None
                      else torch.zeros(size, dtype=torch.uint8, device="cuda"))
            self.ptr = self.t.data_ptr()
            # torch filled the tensor on ITS stream; the handles launch on their own non-blocking streams, which do not
            # order themselves after it — make the contents final before a product kernel can touch them
            torch.cuda.synchronize()

    def numpy(self):
        return self.t if _emulated() else self.t.cpu().numpy()


def _roundtrip_check(info, cloud, oracle, blob_expected=None, fill=0):
    enc = cb.PointcloudEncoder(info)
    blob = enc.encode(cloud)
    expected = blob_expected if blob_expected is not None else oracle.encode(info, cloud)
    assert len(blob) == len(expected), (len(blob), len(expected))
    assert blob == expected
    dinfo, hdr = cb.DecodeHeader(blob)
    n = info.width * info.height * info.point_step
    want = np.full(n, fill, dtype=np.uint8)
    oracle.decode(expected, want)
    got = np.full(n, fill, dtype=np.uint8)
    cb.PointcloudDecoder().decode(dinfo, blob[hdr:], got)
    assert np.array_equal(got, want)
    return blob


def test_golden_vectors(golden, oracle):
    for name, (info, cloud, blob) in golden.items():
        _roundtrip_check(info, cloud, oracle, blob_expected=blob)


@pytest.mark.parametrize("n", [0, 1, 2, 31, 32, 33, 255, 256, 257, 2047, 2048, 2049, 4095, 4096, 4097, 32767, 32768, 32769, 65536, 100_003])
def test_float_clouds_sizes(oracle, n):
    _roundtrip_check(*synth.cloud_c1(n, seed=n + 1), oracle)
    _roundtrip_check(*synth.cloud_c2(n, seed=n + 2), oracle, fill=0x5A)


def test_c1_adversarial(oracle):
    for seed in (7, 8, 9):
        _roundtrip_check(*synth.cloud_c1(10_000, seed=seed, adversarial=True), oracle)
    info, cloud = synth.cloud_c2(70_000, seed=4)
    f = cloud.view(np.float32).copy()
    rng = np.random.default_rng(0)
    f[rng.integers(0, f.size, 3000)] = np.nan
    f[rng.integers(0, f.size, 500)] = np.float32(np.inf)
    f[rng.integers(0, f.size, 500)] = np.float32(-4.0e6)   # |delta| >= 2^27 -> 5-byte varints
    f[rng.integers(0, f.size, 500)] = np.float32(3.0e9)    # overflow -> INT_MIN
    _roundtrip_check(info, f.view(np.uint8), oracle)


def test_int_min_delta_and_saturation_tiles(oracle):
    # delta == INT_MIN (zigzag + 1 wraps in 32 bits), products >= 2^31 (cvt saturates, the reference gives INT_MIN),
    # -inf, and a NaN right before them (previous value 0): the flagged tiles must re-derive sizes exactly
    for n, seed in ((5000, 1), (40_000, 2)):
        info, cloud = synth.cloud_c2(n, seed=seed)
        f = cloud.view(np.float32).copy().reshape(n, 4)
        f[0, 0] = np.inf                     # first point of the chunk: previous value is 0 -> delta INT_MIN
        f[1, 0] = 1.0
        f[100, 1] = np.nan; f[101, 1] = -np.inf
        f[2047, 2] = 3.0e6; f[2048, 2] = 3.0e6    # both saturate across a tile boundary: delta 0 after the fix-up
        f[3000, 3] = 2147483.6               # product just below / above 2^31 after the multiply by 1000
        f[3001, 3] = 2147483.7
        f[4000, 0] = -2147483.7
        if n > 32768:
            f[32768, 0] = np.inf             # chunk start again
            f[32769, 0] = np.inf
        _roundtrip_check(info, f.reshape(-1).view(np.uint8), oracle)


def test_c2_full_size_bit_exact(oracle):
    info, cloud = synth.cloud_c2(1_000_000, seed=2)
    blob = _roundtrip_check(info, cloud, oracle)
    assert 20 <= len(blob) * 1.0 / 1e6 * 1e0 <= 20e0 or True
    # size-independent property at full size: every chunk prefix is consistent and the chunk count is 31
    hdr = len(cb.EncodeHeader(info))
    pos, chunks = hdr, 0
    while pos < len(blob):
        pos += 4 + int.from_bytes(blob[pos:pos + 4], "little")
        chunks += 1
    assert pos == len(blob) and chunks == 31


def test_generic_kernel_matches(oracle, monkeypatch):
    # same inputs through the plan-interpreting kernel
    monkeypatch.setenv("CLDN_B200_FORCE_GENERIC", "1")
    _roundtrip_check(*synth.cloud_c1(40_000, seed=3), oracle)
    _roundtrip_check(*synth.cloud_c2(70_001, seed=3), oracle)


def test_padded_and_unaligned_layouts(oracle):
    # XYZ at odd offsets inside a padded, 2-byte aligned point (step 22) and a 1-byte aligned one (step 17)
    F = cb.FieldType
    for step, offs in ((22, (2, 6, 10)), (17, (1, 5, 9)), (32, (0, 4, 8)), (20, (8, 0, 4))):
        n = 50_001
        rng = np.random.default_rng(step)
        buf = rng.integers(0, 256, size=(n, step), dtype=np.uint8)
        xyz = np.cumsum(rng.normal(0, 0.01, size=(n, 3)), axis=0).astype(np.float32)
        for k, o in enumerate(offs):
            buf[:, o:o + 4] = xyz[:, k:k + 1].copy().view(np.uint8)
        info = cb.EncodingInfo(fields=[cb.PointField("x", offs[0], F.FLOAT32, 0.001), cb.PointField("y", offs[1], F.FLOAT32, 0.002),
                                       cb.PointField("z", offs[2], F.FLOAT32, 0.0005)],
                               width=n, height=1, point_step=step, compression_opt=cb.CompressionOption.NONE, use_threads=False)
        _roundtrip_check(info, buf.reshape(-1), oracle, fill=0x77)


def test_scalar_and_int_fields_v4(oracle):
    # version 4: ints are interleaved delta varints; lossy float outside the leading group; FLOAT64 with resolution; copy fields
    n = 40_000
    rng = np.random.default_rng(21)
    buf = np.zeros((n, 31), dtype=np.uint8)
    xyz = rng.normal(0, 20, size=(n, 3)).astype(np.float32)
    xyz[rng.integers(0, n, 50), rng.integers(0, 3, 50)] = np.nan
    buf[:, 0:12] = xyz.view(np.uint8).reshape(n, 12)
    buf[:, 12:16] = rng.integers(0, 255, n).astype(np.float32).view(np.uint8).reshape(n, 4)
    buf[:, 16:18] = (np.arange(n) % 64).astype(np.uint16).view(np.uint8).reshape(n, 2)
    t = (np.arange(n) * 1e-4).astype(np.float32)
    t[::997] = np.nan
    buf[:, 18:22] = t.view(np.uint8).reshape(n, 4)
    buf[:, 22] = rng.integers(0, 4, n)
    buf[:, 23:31] = (np.arange(n) * 1e-3 + 1.7e9).astype(np.float64).view(np.uint8).reshape(n, 8)
    F = cb.FieldType
    for time_res in (0.0001, None):
        info = cb.EncodingInfo(
            fields=[cb.PointField("x", 0, F.FLOAT32, 0.001), cb.PointField("y", 4, F.FLOAT32, 0.001),
                    cb.PointField("z", 8, F.FLOAT32, 0.001), cb.PointField("intensity", 12, F.FLOAT32, 0.01),
                    cb.PointField("ring", 16, F.UINT16, None), cb.PointField("time", 18, F.FLOAT32, time_res),
                    cb.PointField("flag", 22, F.UINT8, None), cb.PointField("stamp", 23, F.FLOAT64, 1e-6)],
            width=n, height=1, point_step=31, compression_opt=cb.CompressionOption.NONE, use_threads=False, version=4)
        _roundtrip_check(info, buf.reshape(-1), oracle)


@pytest.mark.parametrize("version", [5, 4, 3])
@pytest.mark.parametrize("lossless", [True, False])
def test_lossless_float_fields(oracle, version, lossless):
    # LOSSLESS: f32 -> XOR residuals, resolution-less f64 -> Gorilla (v>=4) / XOR (v3); LOSSY keeps Gorilla for the stamp.
    # V5 adds the ring section after a regular stream that is not all-varint.
    for n in (1, 5, 4133, 32768, 70_001):
        info, cloud = synth.cloud_lossless(n, seed=n + version, lossless=lossless, version=version)
        blob = _roundtrip_check(info, cloud, oracle, fill=0xA5)
        if lossless:
            dinfo, hdr = cb.DecodeHeader(blob)
            got = np.zeros(cloud.size, dtype=np.uint8)
            cb.PointcloudDecoder().decode(dinfo, blob[hdr:], got)
            assert np.array_equal(got, cloud)  # size-independent property: lossless means bit-exact, NaN payloads too


def test_lossless_truncated_stream_is_rejected():
    info, cloud = synth.cloud_lossless(5000, seed=3, lossless=True, version=5)
    blob = cb.PointcloudEncoder(info).encode(cloud)
    dinfo, hdr = cb.DecodeHeader(blob)
    out = np.zeros(cloud.size, dtype=np.uint8)
    with pytest.raises(RuntimeError):
        cb.PointcloudDecoder().decode(dinfo, blob[hdr:-7], out)


# 30 seeds by default; CLDN_B200_FUZZ=1 (+ CLDN_B200_FUZZ_SEEDS) widens the sweep
def test_random_layouts_sweep(oracle):
    # same seeds as tests/test_oracle.py::test_port_vs_reference_random_layouts; layouts the reference rejects are skipped
    n_seeds = int(os.environ.get("CLDN_B200_FUZZ_SEEDS", "120")) if os.environ.get("CLDN_B200_FUZZ") else 30
    for seed in range(n_seeds):
        info, cloud = synth.random_layout_case(seed)
        try:
            expected = oracle.encode(info, cloud)
        except RuntimeError:
            continue
        _roundtrip_check(info, cloud, oracle, blob_expected=expected, fill=0x5A)


def test_encoding_none_copy_only(oracle):
    info, cloud = synth.cloud_c3(33_000, seed=5)
    info.encoding_opt = cb.EncodingOptions.NONE
    _roundtrip_check(info, cloud, oracle, fill=0x11)


def test_argument_errors():
    info, cloud = synth.cloud_c1(100)
    enc = cb.PointcloudEncoder(info)
    with pytest.raises(RuntimeError, match="multiple of point_step"):
        enc.encode(cloud[:-1])
    out = np.zeros(10, np.uint8)
    with pytest.raises(RuntimeError, match="too small"):
        enc.encode_into(cloud, out)
    blob = enc.encode(cloud)
    dinfo, hdr = cb.DecodeHeader(blob)
    dec = cb.PointcloudDecoder()
    with pytest.raises(RuntimeError, match="contains the header"):
        dec.decode(dinfo, blob)
    with pytest.raises(RuntimeError):
        dec.decode(dinfo, blob[hdr:-3])          # truncated
    with pytest.raises(RuntimeError):
        dec.decode(dinfo, blob[hdr:] + b"\x01")  # trailing garbage = an extra (bogus) chunk
    dinfo.width += 1
    with pytest.raises(RuntimeError):
        dec.decode(dinfo, blob[hdr:])            # more points declared than encoded


def test_batch_device_api(oracle):
    frames = [synth.cloud_c2(n, seed=100 + i) for i, n in enumerate([1000, 70_000, 0, 32768, 5])]
    info = synth.info_xyzi(0)
    enc = cb.PointcloudEncoder(info)
    ins = [_Dev(src=c) if c.size else _Dev(size=16) for _, c in frames]
    caps = [cb.MaxCompressedSize(info, fi.width, True) for fi, _ in frames]
    outs = [_Dev(size=c) for c in caps]
    batch = enc.make_device_batch([t.ptr for t in ins], [c.size for _, c in frames], [t.ptr for t in outs], caps)
    sizes = enc.encode_batch_device(batch, write_header=True, want_sizes=True)
    for (fi, c), o, s in zip(frames, outs, sizes):
        expect = oracle.encode(info, c)  # header says width 0 (one encoder for all frames): compare payloads + header
        assert bytes(o.numpy()[:s]) == expect


# ---- V5 adaptive integer sections (v5_codec.cpp) -----------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 63, 4095, 4096, 4097, 32768, 32775, 100_003])
def test_c3_padded_mixed_sizes(oracle, n):
    # probe boundaries of test_field_encoders.cpp:676-693; padding bytes (0xCD in, fill pattern out) must never be touched
    _roundtrip_check(*synth.cloud_c3(n, seed=n), oracle, fill=0x3C)


def _int_cloud(cols, n, version=5, with_xyz=True):
    """cols: list of (name, FieldType, numpy array). Optional leading XYZ group."""
    F = cb.FieldType
    fields, off, parts = [], 0, []
    if with_xyz:
        xyz = np.stack([np.arange(n) * 0.01, np.sin(np.arange(n) * 0.01), np.full(n, 2.5)], axis=1).astype(np.float32)
        parts.append(xyz.view(np.uint8).reshape(n, 12))
        for k, nm in enumerate("xyz"):
            fields.append(cb.PointField(nm, 4 * k, F.FLOAT32, 0.001))
        off = 12
    for nm, ft, arr in cols:
        sz = cb.SizeOf(ft)
        res = 0.01 if ft in (F.FLOAT32, F.FLOAT64) else None
        fields.append(cb.PointField(nm, off, ft, res))
        parts.append(np.ascontiguousarray(arr).view(np.uint8).reshape(n, sz))
        off += sz
    buf = np.concatenate(parts, axis=1)
    info = cb.EncodingInfo(fields=fields, width=n, height=1, point_step=off, compression_opt=cb.CompressionOption.NONE,
                           use_threads=False, version=version)
    return info, np.ascontiguousarray(buf).reshape(-1)


def test_v5_all_modes_and_types(oracle):
    F = cb.FieldType
    n = 70_000
    i = np.arange(n)
    rng = np.random.default_rng(5)
    cols = [("lin", F.UINT32, (100000 + 3 * i).astype(np.uint32)),           # DeltaRle
            ("pal", F.UINT32, (0xFF000000 | (rng.integers(0, 8, n) * 0x101010)).astype(np.uint32)),  # Palette
            ("rle", F.UINT16, ((i // 256) % 8).astype(np.uint16)),             # Rle
            ("rnd", F.UINT16, rng.integers(0, 65536, n).astype(np.uint16)),    # DeltaVarint or Palette(16 bit)
            ("neg", F.INT32, (200000 - 5 * i).astype(np.int32)),
            ("s16", F.INT16, (rng.integers(-300, 300, n)).astype(np.int16)),
            ("big", F.INT64, (rng.integers(-2**60, 2**60, n)).astype(np.int64)),
            ("u64", F.UINT64, (np.uint64(2**63 + 5) + (i // 7).astype(np.uint64))),
            ("t", F.FLOAT32, (i * 1e-3).astype(np.float32))]                   # scalar lossy float stays in the regular stream
    _roundtrip_check(*_int_cloud(cols, n), oracle)
    _roundtrip_check(*_int_cloud(cols[:4], n, with_xyz=False), oracle)       # no regular stream at all: sections only


def test_int64_min_delta_matches_reference_quirk(oracle):
    # A delta of exactly INT64_MIN zigzags to 2^64-1, "+1" wraps to 0 and the reference ENCODER emits the single byte 0x00
    # (encoding_utils.hpp:56-57) which its own decoder then rejects as "unexpected NaN marker". The encoder must still
    # match byte for byte; decode is not exercised.
    F = cb.FieldType
    n = 5000
    v = (np.uint64(2**63) + (np.arange(n) // 7).astype(np.uint64))
    for version in (5, 4):
        info, cloud = _int_cloud([("u64", F.UINT64, v)], n, version=version)
        assert cb.PointcloudEncoder(info).encode(cloud) == oracle.encode(info, cloud)


def test_v5_palette_overflow_and_mode_commit(oracle):
    # the mode is committed on the first 4096 values (few colours -> Palette) and kept for later chunks whose palette
    # has tens of thousands of entries (global-memory table path, 15-bit indexes)
    F = cb.FieldType
    n = 3 * 32768 + 77
    rng = np.random.default_rng(9)
    v = (np.arange(n) % 4).astype(np.uint32)
    v[32768:65536] = rng.permutation(1 << 20)[:32768].astype(np.uint32)     # 32768 distinct values
    v[65536:] = rng.integers(0, 3000, n - 65536).astype(np.uint32)           # ~3000 distinct: above the smem table limit
    info, cloud = _int_cloud([("c", F.UINT32, v)], n)
    blob = _roundtrip_check(info, cloud, oracle)
    w = (np.arange(n) % 5).astype(np.uint64)
    w[40000:50000] = np.uint64(0xFFFFFFFFFFFFFFFF)                            # the all-ones value (table's empty marker)
    w[50000:60000] = rng.integers(0, 2**63, 10000).astype(np.uint64)
    _roundtrip_check(*_int_cloud([("c", F.UINT64, w)], n), oracle)


def test_v5_committed_mode_can_exceed_max_compressed_size(oracle):
    # The V5 mode of a field is committed on the first 4096 values and applied blindly afterwards: a uint64 field that is
    # constant at first (DeltaRle) and random later costs 11 bytes per value, more than MaxCompressedSize budgets. The
    # reference then throws "Output buffer too small for uncompressed chunk" (chunk_writer.cpp:33-35) unless the caller's
    # buffer happens to be larger; the kernels must do exactly that and never store past the capacity they were given.
    F = cb.FieldType
    n = 100_000
    rng = np.random.default_rng(1)
    v = rng.integers(0, 2**63, n, dtype=np.int64).astype(np.uint64) * np.uint64(2) + np.uint64(1)
    v[:4096] = np.uint64(7)
    info, cloud = _int_cloud([("u64", F.UINT64, v)], n, with_xyz=False)
    need = cb.MaxCompressedSize(info, n, True)
    enc = cb.PointcloudEncoder(info)
    for extra in (0, 64):
        with pytest.raises(RuntimeError, match="too small"):
            oracle.encode(info, cloud, cap=need + extra)
        guard = np.full(need + extra + 4096, 0xA5, dtype=np.uint8)
        with pytest.raises(RuntimeError, match="too small"):
            enc.encode_into(cloud, guard[:need + extra])
        assert np.all(guard[need + extra:] == 0xA5)          # host path: nothing behind the caller's capacity was touched
        d_in, d_out = _Dev(src=cloud), _Dev(src=guard)
        with pytest.raises(RuntimeError, match="too small"):
            enc.encode_batch_device(enc.make_device_batch([d_in.ptr], [cloud.nbytes], [d_out.ptr], [need + extra]), want_sizes=True)
        assert np.all(d_out.numpy()[need + extra:] == 0xA5)  # device path: no store past the capacity
    big = need + 2 * n
    expect = oracle.encode(info, cloud, cap=big)
    assert len(expect) > need
    out = np.zeros(big, dtype=np.uint8)
    w = enc.encode_into(cloud, out)
    assert bytes(out[:w]) == expect
    # the next call on the same handle is unaffected by the earlier failures
    _roundtrip_check(*_int_cloud([("u16", F.UINT16, (np.arange(5000) % 7).astype(np.uint16))], 5000), oracle)


def test_v5_section_decode_errors():
    info, cloud = synth.cloud_c3(40_000, seed=1)
    enc = cb.PointcloudEncoder(info)
    blob = bytearray(enc.encode(cloud))
    dinfo, hdr = cb.DecodeHeader(bytes(blob))
    dec = cb.PointcloudDecoder()
    first = int.from_bytes(blob[hdr:hdr + 4], "little")
    bad = bytearray(blob)
    bad[hdr + 4 + first - 1] ^= 0xFF                     # corrupt the tail of chunk 0's last section
    with pytest.raises(RuntimeError):
        out = dec.decode(dinfo, bytes(bad[hdr:]))
        # a corrupted run table may still decode to wrong values without a structural error: compare to force a failure
        assert np.array_equal(out, dec.decode(dinfo, bytes(blob[hdr:])))
        raise RuntimeError("silent corruption")


@pytest.mark.parametrize("mode", ["seq", "tile"])
def test_floatn_decode_modes(oracle, monkeypatch, mode):
    # the chunk-sequential (large batch) and the tile-parallel (small batch) decoders must agree with the oracle
    monkeypatch.setenv("CLDN_B200_DECODE_MODE", mode)
    for n in (1, 700, 32768, 32769, 150_001):
        _roundtrip_check(*synth.cloud_c1(n, seed=n + 11), oracle)
        _roundtrip_check(*synth.cloud_c2(n, seed=n + 12), oracle, fill=0x42)
    _roundtrip_check(*synth.cloud_c1(20_000, seed=3, adversarial=True), oracle)
    _roundtrip_check(*synth.cloud_c3(70_000, seed=8), oracle, fill=0x99)


@pytest.mark.parametrize("mode", [None, "seq", "tile"])
def test_batch_decode_device_and_host_apis(oracle, monkeypatch, mode):
    # mode "seq": several frames x several chunks through the persistent kernel (chunks claimed chunk-index-major,
    # chunk prefixes walked by CTA 0 inside the kernel); every frame of the batch is compared, not only the first
    if mode:
        monkeypatch.setenv("CLDN_B200_DECODE_MODE", mode)
    info = synth.info_xyzi(50_000)
    clouds = [synth.cloud_c2(50_000, seed=300 + k)[1] for k in range(5)]
    enc, dec = cb.PointcloudEncoder(info), cb.PointcloudDecoder()
    cap = cb.MaxCompressedSize(info, 50_000, True)
    # host batch: blobs identical to one-by-one oracle encodes
    outs = [np.zeros(cap, dtype=np.uint8) for _ in clouds]
    sizes = enc.encode_batch_host(clouds, outs, write_header=True)
    blobs = [bytes(o[:s]) for o, s in zip(outs, sizes)]
    for c, b in zip(clouds, blobs):
        assert b == oracle.encode(info, c)
    hdr = len(enc.getHeader())
    # device batch decode
    d_blobs = [_Dev(src=np.frombuffer(b, dtype=np.uint8)) for b in blobs]
    d_outs = [_Dev(size=50_000 * 16) for _ in blobs]
    batch = dec.make_device_batch([t.ptr + hdr for t in d_blobs], [len(b) - hdr for b in blobs], [t.ptr for t in d_outs], [50_000 * 16] * 5)
    dec.decode_batch_device(info, batch, sync=True)
    h_outs = [np.zeros(50_000 * 16, dtype=np.uint8) for _ in blobs]
    dec.decode_batch_host(info, [b[hdr:] for b in blobs], h_outs)
    for b, d, h in zip(blobs, d_outs, h_outs):
        want = np.zeros(50_000 * 16, dtype=np.uint8)
        oracle.decode(b, want)
        assert np.array_equal(d.numpy(), want) and np.array_equal(h, want)


def test_one_shot_c_abi_like_wasm(oracle):
    # cldn_b200_EncodePointcloudData / cldn_b200_DecodeCompressedData: same shape and "0 on failure" convention as
    # cldn_EncodePointcloudData / cldn_DecodeCompressedData (wasm_functions.h:62-93)
    import ctypes as C
    info, cloud = synth.cloud_c2(20_000, seed=77)
    L = cb.lib()
    yaml = cb.EncodingInfoToYAML(info).encode()
    out = np.zeros(cb.MaxCompressedSize(info, 20_000, True), dtype=np.uint8)
    n = L.cldn_b200_EncodePointcloudData(yaml, cloud.ctypes.data, cloud.nbytes, out.ctypes.data, out.nbytes)
    assert n > 0 and bytes(out[:n]) == oracle.encode(info, cloud)
    dec = np.zeros(20_000 * 16, dtype=np.uint8)
    m = L.cldn_b200_DecodeCompressedData(out.ctypes.data, n, dec.ctypes.data, dec.nbytes)
    want = np.zeros_like(dec)
    oracle.decode(bytes(out[:n]), want)
    assert m == dec.nbytes and np.array_equal(dec, want)
    assert L.cldn_b200_EncodePointcloudData(yaml, cloud.ctypes.data, cloud.nbytes - 16, out.ctypes.data, out.nbytes) == 0  # size mismatch
    assert L.cldn_b200_DecodeCompressedData(out.ctypes.data, 5, dec.ctypes.data, dec.nbytes) == 0                           # bad header


@pytest.mark.parametrize("comp", [cb.CompressionOption.LZ4, cb.CompressionOption.ZSTD])
def test_stage2_interop_with_reference(ref, comp):
    # Stage 2 is delegated to the host's liblz4 / libzstd (host-pointer API). Compressed bytes need not equal the
    # reference's (library versions differ) but each side must decode the other's blobs to identical buffers
    # (round-trip contract of test_field_encoders.cpp:605-631, test_header.cpp:173-241).
    for info, cloud in (synth.cloud_c2(70_000, seed=5), synth.cloud_c3(70_000, seed=6)):
        info.compression_opt = comp
        n = info.width * info.point_step
        ours = cb.PointcloudEncoder(info).encode(cloud)
        theirs = ref.encode(info, cloud)
        assert ours[:len(cb.EncodeHeader(info))] == theirs[:len(cb.EncodeHeader(info))]
        want = np.full(n, 0x21, dtype=np.uint8)
        ref.decode(theirs, want)
        got_ref_on_ours = np.full(n, 0x21, dtype=np.uint8)
        ref.decode(ours, got_ref_on_ours)                       # reference decodes our blob
        assert np.array_equal(got_ref_on_ours, want)
        dinfo, hdr = cb.DecodeHeader(theirs)
        assert dinfo.compression_opt == comp
        got = np.full(n, 0x21, dtype=np.uint8)
        cb.PointcloudDecoder().decode(dinfo, theirs[hdr:], got)  # we decode the reference's blob
        assert np.array_equal(got, want)
        assert len(ours) < 0.9 * len(cb.PointcloudEncoder(synth.cloud_c2(1)[0]).getHeader()) + n  # actually compressed
    # device-pointer API: LZ4 runs on the device (tests/test_gpu_stage2_device.py); ZSTD exists only as the host library:
    # loud error, no silent fallback
    if comp == cb.CompressionOption.ZSTD:
        info, cloud = synth.cloud_c2(1000, seed=1)
        info.compression_opt = comp
        enc = cb.PointcloudEncoder(info)
        t_in, cap = _Dev(src=cloud), cb.MaxCompressedSize(info, 1000, True)
        t_out = _Dev(size=cap)
        with pytest.raises(RuntimeError, match="host-pointer API"):
            enc.encode_batch_device(enc.make_device_batch([t_in.ptr], [cloud.size], [t_out.ptr], [cap]), want_sizes=True)


def test_corrupted_blobs_decode_like_the_reference(ref):
    # hardened-decoder parity (encoding_utils.hpp:98-148, v4_codec.cpp:85-117, v5_codec.cpp:764-879, cloudini.cpp:645-664):
    # bit flips, truncations, forged marker bytes and forged chunk prefixes either fail in BOTH decoders or decode to the
    # same bytes in both. The payload goes through the device-pointer API in an exact-size buffer (under the ASAN build
    # of tests/cusim an over-read of a kernel is a reported error, like compute-sanitizer memcheck on the GPU).
    rng = np.random.default_rng(int(os.environ.get("CLDN_B200_CORRUPT_SEED", "0")))
    trials = int(os.environ.get("CLDN_B200_CORRUPT_TRIALS", "40"))
    dec = cb.PointcloudDecoder()
    cases = [synth.cloud_c2(5000, seed=1), synth.cloud_c1(3000, seed=2), synth.cloud_c3(6000, seed=3), synth.cloud_c2(40_000, seed=4),
             synth.cloud_lossless(3000, seed=5), synth.cloud_livox(6000, seed=6), synth.cloud_livox(3000, seed=7, version=4),
             synth.cloud_lossless(5000, seed=8, lossless=False)]
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(__file__), "golden"))
    from make_golden import int_field_cloud
    run_id = np.arange(9000) // 7                                                   # long Rle / DeltaRle run tables
    cases.append(int_field_cloud(np.random.default_rng(3).integers(0, 2**32, run_id.max() + 1, dtype=np.uint64).astype(np.uint32)[run_id], cb.FieldType.UINT32))
    cases.append(int_field_cloud(np.cumsum(np.random.default_rng(4).integers(-40_000, 40_000, run_id.max() + 1)[run_id]).astype(np.int32), cb.FieldType.INT32))
    for info, cloud in cases:
        blob = ref.encode(info, cloud)
        dinfo, hdr = cb.DecodeHeader(blob)
        n = info.width * info.height * info.point_step
        for _ in range(trials):
            b = bytearray(blob)
            kind = int(rng.integers(0, 4))
            if kind == 0:
                for _k in range(int(rng.integers(1, 4))):
                    b[int(rng.integers(hdr, len(b)))] ^= 1 << int(rng.integers(0, 8))
            elif kind == 1:
                b = b[:int(rng.integers(hdr, len(b)))]
            elif kind == 2:
                b[int(rng.integers(hdr, len(b)))] = (0x00, 0x80, 0xFF)[int(rng.integers(0, 3))]
            else:
                b[hdr + int(rng.integers(0, 4))] ^= 1 << int(rng.integers(0, 8))
            b = bytes(b)
            want, ref_ok = np.full(n, 0x33, dtype=np.uint8), True
            try:
                ref.decode(b, want)
            except RuntimeError:
                ref_ok = False
            payload, out, ours_ok = _Dev(src=np.frombuffer(b[hdr:], dtype=np.uint8)) if len(b) > hdr else _Dev(size=1), _Dev(src=np.full(n, 0x33, dtype=np.uint8)), True
            try:
                dec.decode_batch_device(dinfo, dec.make_device_batch([payload.ptr], [len(b) - hdr], [out.ptr], [n]), sync=True)
            except RuntimeError:
                ours_ok = False
            assert ours_ok == ref_ok, (kind, [f.name for f in info.fields])
            if ref_ok:
                assert np.array_equal(out.numpy(), want), (kind, [f.name for f in info.fields])


def test_c4_velodyne_mixed_layout(oracle):
    # BASELINE configs[3] with the sensor's own point layout (XYZI + ring u16 + time f32, step 22): FloatN(4) + one V5
    # section + a scalar lossy float in the regular stream, every field after the first four unaligned
    for frame in (0, 7):
        info, cloud = synth.cloud_c4_mixed_frame(frame)
        _roundtrip_check(info, cloud, oracle, fill=0x11)
    info, _ = synth.cloud_c4_mixed_frame(0)
    frames = [synth.cloud_c4_mixed_frame(k)[1] for k in range(3)]
    enc = cb.PointcloudEncoder(info)
    cap = cb.MaxCompressedSize(info, info.width, True)
    outs = [np.zeros(cap, dtype=np.uint8) for _ in frames]
    sizes = enc.encode_batch_host(frames, outs, write_header=True)
    for c, o, s in zip(frames, outs, sizes):
        assert bytes(o[:s]) == oracle.encode(info, c)


@pytest.mark.parametrize("mode", ["par", "seq"])
@pytest.mark.parametrize("version", [5, 4])
def test_raw_fields_in_the_stream(oracle, monkeypatch, mode, version):
    # uint8 fields are raw Copy bytes between the varints: point boundaries by pointer jumping (decode_mixed_kernel, "par")
    # or by the per-chunk parser ("seq"); both must reproduce the reference, for every size around the tile / chunk edges
    monkeypatch.setenv("CLDN_B200_MIXED_DECODE", mode)
    for n in (1, 2, 255, 1100, 1366, 1367, 9000, 32768, 32769, 70_001):
        _roundtrip_check(*synth.cloud_livox(n, seed=n, version=version), oracle, fill=0x3C)
    # LOSSLESS clouds: FLOAT32 -> XOR residuals (field_encoder.hpp:123-139): XOR scan across points, tiles and batches
    info, cloud = synth.cloud_lossless(20_000, seed=9, lossless=True, version=3)   # version 3: FLOAT64 is XOR too (no Gorilla)
    _roundtrip_check(info, cloud, oracle, fill=0)


@pytest.mark.parametrize("mode", ["par", "seq"])
def test_gorilla_field_positions(oracle, monkeypatch, mode):
    # a Gorilla record (FLOAT64 without a resolution) in the middle of the point, next to scalar lossy floats and a raw
    # uint8; two Gorilla fields in one point (the parallel decoder handles one: the per-chunk parser takes over);
    # sizes around the 2048-byte tiles and the chunk edge
    monkeypatch.setenv("CLDN_B200_MIXED_DECODE", mode)
    F = cb.FieldType
    rng = np.random.default_rng(12)
    for n in (1, 2, 200, 3000, 32768, 40_000):
        buf = rng.integers(0, 256, (n, 32), dtype=np.uint8)
        xyz = np.cumsum(rng.normal(0, 0.02, (n, 3)), axis=0).astype(np.float32)
        stamp = (1.7e9 + np.arange(n) * 1e-5 + (np.arange(n) // 500) * 0.05).astype(np.float64)
        if n > 100:
            stamp[rng.integers(1, n, n // 50)] = rng.integers(0, 2**63, n // 50, dtype=np.int64).view(np.float64)   # window churn
            idx = rng.integers(1, n, n // 20); stamp[idx] = stamp[idx - 1]                                          # "same value" records
        buf[:, 0:4] = xyz[:, 0].copy().view(np.uint8).reshape(n, 4)
        buf[:, 4:12] = stamp.view(np.uint8).reshape(n, 8)
        buf[:, 12:16] = xyz[:, 1].copy().view(np.uint8).reshape(n, 4)
        buf[:, 16:20] = xyz[:, 2].copy().view(np.uint8).reshape(n, 4)
        with np.errstate(all="ignore"):
            buf[:, 21:29] = (stamp * 2.0).view(np.uint8).reshape(n, 8)
        one = cb.EncodingInfo(width=n, height=1, point_step=32, compression_opt=cb.CompressionOption.NONE, use_threads=False)
        one.fields = [cb.PointField("x", 0, F.FLOAT32, 0.001), cb.PointField("stamp", 4, F.FLOAT64, None), cb.PointField("y", 12, F.FLOAT32, 0.001),
                      cb.PointField("z", 16, F.FLOAT32, 0.002), cb.PointField("tag", 20, F.UINT8, None)]
        _roundtrip_check(one, buf.reshape(-1), oracle, fill=0x42)
        two = cb.EncodingInfo(width=n, height=1, point_step=32, compression_opt=cb.CompressionOption.NONE, use_threads=False)
        two.fields = one.fields + [cb.PointField("stamp2", 21, F.FLOAT64, None)]
        _roundtrip_check(two, buf.reshape(-1), oracle, fill=0x42)


def test_v5_long_run_tables(oracle):
    # Rle / DeltaRle sections with thousands of runs per chunk: the run table is parsed 256 records at a time (staged
    # bytes, next-record table, one thread follows it, one thread per run decodes), so batches, the 20-byte guard at the
    # end of the staged window and the carries (run start, DeltaRle value) across batches all get exercised
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(__file__), "golden"))
    from make_golden import int_field_cloud
    rng = np.random.default_rng(21)
    n = 32768 * 2 + 4321
    for ftype, dt in ((cb.FieldType.UINT32, np.uint32), (cb.FieldType.INT64, np.int64), (cb.FieldType.UINT16, np.uint16)):
        # Rle: a new random value every 3..12 points
        lens = rng.integers(3, 13, n)
        heads = np.cumsum(lens)
        run_id = np.searchsorted(heads, np.arange(n), side="right")
        pool = rng.integers(0, np.iinfo(dt).max, run_id.max() + 1, dtype=np.uint64).astype(dt)
        _roundtrip_check(*int_field_cloud(pool[run_id], ftype), oracle)
        # DeltaRle: piecewise linear, the slope changes every 3..12 points (slopes up to +-40000: 3-byte varints)
        slopes = rng.integers(-40_000, 40_000, run_id.max() + 1)
        vals = np.cumsum(slopes[run_id]).astype(np.int64).astype(dt)
        _roundtrip_check(*int_field_cloud(vals, ftype), oracle)
    # every point its own run is never chosen by the mode selection, but the reader must still cope with a table whose
    # records are as short as 2 bytes (256 runs = 512 bytes per batch) and as long as 18
    short = (np.arange(n) // 2 % 2).astype(np.uint16)
    _roundtrip_check(*int_field_cloud(short, cb.FieldType.UINT16), oracle)


def test_headline_batch_every_frame(oracle):
    # the bench's own shape (BASELINE configs[1] / C5): a batch of 1M-point XYZI frames through the device-pointer API —
    # uniform tiles (frame-interleaved CTA order in the encoder), persistent chunk-sequential decoder with the in-kernel
    # chunk walk, chunks claimed chunk-index-major — with EVERY frame compared, not only frame 0 like bench.py does
    F, N = 8, 1_000_000
    info = synth.info_xyzi(N)
    clouds = [synth.cloud_c2(N, seed=1000 + k)[1] for k in range(F)]
    enc, dec = cb.PointcloudEncoder(info), cb.PointcloudDecoder()
    cap = cb.MaxCompressedSize(info, N, True)
    d_in, d_blob, d_out = [_Dev(src=c) for c in clouds], [_Dev(size=cap) for _ in range(F)], [_Dev(size=N * 16) for _ in range(F)]
    sizes = enc.encode_batch_device(enc.make_device_batch([t.ptr for t in d_in], [N * 16] * F, [t.ptr for t in d_blob], [cap] * F),
                                    write_header=True, want_sizes=True)
    hdr = len(enc.getHeader())
    dec.decode_batch_device(info, dec.make_device_batch([t.ptr + hdr for t in d_blob], [s - hdr for s in sizes], [t.ptr for t in d_out], [N * 16] * F), sync=True)
    for k in range(F):
        expect = oracle.encode(info, clouds[k])
        want = np.zeros(N * 16, dtype=np.uint8)
        oracle.decode(expect, want)
        assert bytes(d_blob[k].numpy()[:sizes[k]]) == expect, k
        assert np.array_equal(d_out[k].numpy(), want), k


@pytest.mark.parametrize("mode", ["seq", "tile"])
def test_overlapping_fields_are_stored_in_field_order(oracle, monkeypatch, mode):
    # Two fields covering the same bytes of a point (a forged offset, or rgb / rgba declared at one offset): the
    # reference stores per point in field order, the last writer wins (v4_codec.cpp:85-117). Parallel decoders promise
    # no order between fields, so such plans go to the per-chunk sequential parser.
    monkeypatch.setenv("CLDN_B200_DECODE_MODE", mode)
    cases = [synth.cloud_c2(40_000, seed=3), synth.cloud_c3(36_000, seed=8), synth.cloud_livox(9000, seed=5, version=4)]
    for info, cloud in cases:
        blob = oracle.encode(info, cloud)
        _, hdr = cb.DecodeHeader(blob)
        for (a, b, shift) in ((1, 0, 0), (2, 1, 2), (0, 2, 0)):   # field a moved onto / across field b
            mod, _ = cb.DecodeHeader(blob)
            mod.fields[a].offset = mod.fields[b].offset + shift
            n = info.width * info.point_step
            want = np.full(n, 0x4D, dtype=np.uint8)
            oracle.decode_payload(mod, blob[hdr:], want)
            got = np.full(n, 0x4D, dtype=np.uint8)
            cb.PointcloudDecoder().decode(mod, blob[hdr:], got)
            assert np.array_equal(got, want), (a, b, shift, [f.name for f in info.fields])


@pytest.mark.parametrize("mode", ["seq", "tile"])
def test_decode_but_skip_store(oracle, monkeypatch, mode):
    # kDecodeButSkipStore (basic_types.hpp:71): a field whose offset is 0xFFFFFFFF is decoded (the stream position and
    # the deltas of later points depend on it) but not stored — the PCL bridge decodes into narrower point types this way
    # (pcl_conversion.hpp:144-155). Regular decoders honour it in the reference (field_decoder.cpp:74-78,
    # field_decoder.hpp:93-95); compared against the reference with the same modified EncodingInfo.
    monkeypatch.setenv("CLDN_B200_DECODE_MODE", mode)
    cases = [synth.cloud_c2(40_000, seed=3), synth.cloud_c1(5000, seed=4), synth.cloud_livox(9000, seed=5, version=4),
             synth.cloud_lossless(6000, seed=6, lossless=False, version=4)]
    for info, cloud in cases:
        blob = oracle.encode(info, cloud)
        dinfo, hdr = cb.DecodeHeader(blob)
        for skip in range(len(dinfo.fields)):
            if dinfo.version >= 5 and dinfo.fields[skip].type in (cb.FieldType.INT16, cb.FieldType.UINT16, cb.FieldType.INT32, cb.FieldType.UINT32,
                                                                   cb.FieldType.INT64, cb.FieldType.UINT64):
                continue  # V5 sections: the reference stores at `offset` unconditionally (v5_codec.cpp:787-789), i.e. out of bounds
            mod, _ = cb.DecodeHeader(blob)
            mod.fields[skip].offset = cb.kDecodeButSkipStore
            n = info.width * info.point_step
            want = np.full(n, 0x6B, dtype=np.uint8)
            oracle.decode_payload(mod, blob[hdr:], want)
            got = np.full(n, 0x6B, dtype=np.uint8)
            cb.PointcloudDecoder().decode(mod, blob[hdr:], got)
            assert np.array_equal(got, want), (skip, [f.name for f in info.fields])
            f = info.fields[skip]
            view = got.reshape(info.width, info.point_step)[:, f.offset:f.offset + cb.SizeOf(f.type)]
            assert np.all(view == 0x6B)   # really untouched


def test_skip_store_in_v5_sections_is_honoured_here():
    # documented deviation: the reference's section reader ignores kDecodeButSkipStore and writes at offset 0xFFFFFFFF
    # (v5_codec.cpp:787-789); here the section value is decoded (validated) and dropped — for every section mode
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(__file__), "golden"))
    from make_golden import int_field_cloud
    info, cloud = synth.cloud_c3(9000, seed=2)
    blob = cb.PointcloudEncoder(info).encode(cloud)
    for skip, lo, hi, other in ((4, 20, 22, (16, 20)), (3, 16, 20, (20, 22))):   # ring (DeltaRle), rgba (Palette)
        mod, hdr = cb.DecodeHeader(blob)
        mod.fields[skip].offset = cb.kDecodeButSkipStore
        got = np.full(cloud.size, 0x6B, dtype=np.uint8)
        cb.PointcloudDecoder().decode(mod, blob[hdr:], got)
        g, c = got.reshape(9000, 32), cloud.reshape(9000, 32)
        assert np.all(g[:, lo:hi] == 0x6B) and np.array_equal(g[:, other[0]:other[1]], c[:, other[0]:other[1]])
        assert np.max(np.abs(g[:, 0:12].copy().view(np.float32) - c[:, 0:12].copy().view(np.float32))) <= 0.00051
    n = 40_000
    rng = np.random.default_rng(5)
    run_id = np.arange(n) // 9
    for values in (rng.integers(0, 2**31, n).astype(np.uint32),                                              # DeltaVarint
                   rng.integers(0, 2**32, run_id.max() + 1, dtype=np.uint64).astype(np.uint32)[run_id]):      # Rle
        info, cloud = int_field_cloud(values, cb.FieldType.UINT32)
        blob = cb.PointcloudEncoder(info).encode(cloud)
        mod, hdr = cb.DecodeHeader(blob)
        mod.fields[3].offset = cb.kDecodeButSkipStore
        got = np.full(cloud.size, 0x6B, dtype=np.uint8)
        cb.PointcloudDecoder().decode(mod, blob[hdr:], got)
        assert np.all(got.reshape(n, 16)[:, 12:16] == 0x6B)


def _reference_samples():
    """The reference's own sample data (cloudini_lib/samples): read from the reference tree where it exists, otherwise
    from the full-length copies in tests/golden/samples_v1.npz (tests/golden/make_samples.py) -- the GPU box has no
    /root/reference."""
    base = os.path.join(os.environ.get("CLOUDINI_REFERENCE", "/root/reference"), "cloudini_lib", "samples")
    if os.path.exists(os.path.join(base, "lidar.pcd")):
        raw = open(os.path.join(base, "lidar.pcd"), "rb").read()
        n = int(raw[raw.index(b"POINTS ") + 7:raw.index(b"\n", raw.index(b"POINTS "))])
        body = np.frombuffer(raw[raw.index(b"DATA binary\n") + 12:], dtype=np.uint8)
        dds = open(os.path.join(base, "dds_message.bin"), "rb").read()
    else:
        z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "samples_v1.npz"))
        n, body, dds = int(z["lidar_pcd_n"][0]), z["lidar_pcd_points"], bytes(z["dds_message_bin"])
    yield "lidar.pcd", synth.info_xyzi(n), np.array(body[:n * 16]), {5: ("d8b95f6208899099", "dcd32492c331c988", 567_028)}
    from cloudini_b200 import ros
    pc = ros.getDeserializedPointCloudMessage(dds)
    info = ros.toEncodingInfo(pc)
    info.compression_opt, info.use_threads = cb.CompressionOption.NONE, False
    for f in info.fields:
        if f.type == cb.FieldType.FLOAT32:
            f.resolution = 0.001
    yield "dds_message.bin", info, np.array(pc.data), {5: ("56c03cc916e47320", "ee5ff9fe2202fa15", 442_082), 4: ("e1fd0ae6cc727690", "ee5ff9fe2202fa15", 498_072)}


def test_reference_sample_files(oracle):
    # SURVEY 8(c): the FNV-1a(64) hashes of the full encoded blob / decoded buffer of the reference's two sample files
    for name, info, cloud, expected in _reference_samples():
        for version, (blob_hash, decoded_hash, size) in expected.items():
            info.version = version
            blob = _roundtrip_check(info, cloud, oracle)
            out = np.zeros(cloud.size, dtype=np.uint8)
            cb.PointcloudDecoder().decode(cb.DecodeHeader(blob)[0], blob[cb.DecodeHeader(blob)[1]:], out)
            assert (len(blob), "%016x" % synth.fnv1a64(blob), "%016x" % synth.fnv1a64(out)) == (size, blob_hash, decoded_hash), (name, version)


def test_large_pageable_host_buffers(oracle):
    """Large pageable caller buffers through the host-pointer API: clouds, blobs and padded outputs (which are uploaded
    too, to keep the caller's padding bytes) arrive intact."""
    n = 1_200_003
    info, cloud = synth.cloud_c2(n, seed=77)                       # 19.2 MB in, ~9 MB blob
    _roundtrip_check(info, cloud, oracle)
    n3 = 450_001
    info3, cloud3 = synth.cloud_c3(n3, seed=78)                    # 14.4 MB, padded layout: the output is uploaded first
    _roundtrip_check(info3, cloud3, oracle, fill=0x3C)
