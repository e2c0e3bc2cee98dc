"""The fast FloatN readers / writers must (a) really be the kernels that run on plain clouds and (b) hand everything
they cannot prove plain to the careful kernels, with bytes identical to the oracle either way. All through the C ABI."""
import numpy as np
import pytest

import cloudini_b200 as cb
from cloudini_b200 import synth
from test_gpu_parity import _Dev

pytestmark = pytest.mark.gpu


def _encode_all(info, clouds, oracle):
    blobs = [oracle.encode(info, c) for c in clouds]
    hdr = len(cb.PointcloudEncoder(info).getHeader())
    return blobs, hdr


def _decode_batch(info, blobs, hdr, n_bytes, fill=0):
    dec = cb.PointcloudDecoder()
    d_blobs = [_Dev(src=np.frombuffer(b, dtype=np.uint8)) for b in blobs]
    d_outs = [_Dev(src=np.full(n_bytes, fill, dtype=np.uint8)) for _ in blobs]
    batch = dec.make_device_batch([t.ptr + hdr for t in d_blobs], [len(b) - hdr for b in blobs], [t.ptr for t in d_outs], [n_bytes] * len(blobs))
    dec.decode_batch_device(info, batch, sync=True)
    return [d.numpy() for d in d_outs], dec.last_stats()


def _want(oracle, blob, n_bytes, fill=0):
    w = np.full(n_bytes, fill, dtype=np.uint8)
    oracle.decode(blob, w)
    return w


@pytest.mark.parametrize("n", [1, 7, 8, 9, 1023, 1024, 1025, 32767, 32768, 32769, 40_001, 100_000])
def test_fast_reader_takes_plain_clouds(oracle, monkeypatch, n):
    monkeypatch.setenv("CLDN_B200_DECODE_MODE", "seq")
    for make, step, fill in ((synth.cloud_c2, 16, 0), (synth.cloud_c1, 12, 0x5A)):
        frames = 3
        made = [make(n, seed=40 + k) for k in range(frames)]
        info = made[0][0]
        blobs, hdr = _encode_all(info, [m[1] for m in made], oracle)
        outs, (fast, redo) = _decode_batch(info, blobs, hdr, n * step, fill)
        chunks = frames * ((n + 32767) // 32768)
        assert (fast, redo) == (chunks, 0), (fast, redo, chunks)
        for b, o in zip(blobs, outs):
            assert np.array_equal(o, _want(oracle, b, n * step, fill))


def test_fast_reader_hands_over_what_it_cannot_prove_plain(oracle, monkeypatch):
    monkeypatch.setenv("CLDN_B200_DECODE_MODE", "seq")
    n = 70_000
    info, plain = synth.cloud_c2(n, seed=5)
    pts = plain.view(np.float32).reshape(n, 4).copy()
    nan_cloud = pts.copy(); nan_cloud[40_000, 1] = np.nan                 # one NaN marker in chunk 1
    wide_cloud = pts.copy(); wide_cloud[100, 0] = np.float32(3.0e6)        # a 5-byte varint (and the jump back) in chunk 0
    tail_cloud = pts.copy(); tail_cloud[n - 1, 3] = np.nan                 # NaN in the very last value of the stream
    clouds = [plain, nan_cloud.view(np.uint8).reshape(-1), wide_cloud.view(np.uint8).reshape(-1), tail_cloud.view(np.uint8).reshape(-1)]
    blobs, hdr = _encode_all(info, clouds, oracle)
    outs, (fast, redo) = _decode_batch(info, blobs, hdr, n * 16, 0x11)
    assert fast == 4 * 3 and redo == 3, (fast, redo)
    for b, o in zip(blobs, outs):
        assert np.array_equal(o, _want(oracle, b, n * 16, 0x11))


def test_fast_reader_on_damaged_streams_reports_like_the_careful_one(oracle, monkeypatch):
    # truncated bodies / forged sizes: the fast reader must not decide anything itself; the error and its message come
    # from the careful kernel, exactly as with CLDN_B200_DECODE_FAST=0
    n = 50_000
    info, cloud = synth.cloud_c2(n, seed=6)
    blob = oracle.encode(info, cloud)
    hdr = len(cb.PointcloudEncoder(info).getHeader())
    rng = np.random.default_rng(7)
    for trial in range(12):
        bad = bytearray(blob)
        kind = trial % 3
        if kind == 0:      # cut the payload
            bad = bad[:hdr + int(rng.integers(5, len(blob) - hdr))]
        elif kind == 1:    # flip bytes inside a chunk
            for _ in range(4):
                bad[hdr + 8 + int(rng.integers(0, len(blob) - hdr - 8))] = int(rng.integers(0, 256))
        else:              # zero byte (NaN marker) in the middle
            bad[hdr + 4 + int(rng.integers(0, 100_000))] = 0
        results = []
        for fastflag in ("1", "0"):
            monkeypatch.setenv("CLDN_B200_DECODE_MODE", "seq")
            monkeypatch.setenv("CLDN_B200_DECODE_FAST", fastflag)
            out = np.full(n * 16, 0x33, dtype=np.uint8)
            try:
                cb.PointcloudDecoder().decode(info, bytes(bad[hdr:]), out)
                results.append(("ok", out.tobytes()))
            except RuntimeError as e:
                results.append(("err", str(e)))
        assert results[0][0] == results[1][0], (trial, results[0][0], results[1][0])
        if results[0][0] == "ok":
            assert results[0][1] == results[1][1], trial
        elif kind != 1:    # (four flipped bytes can be four defects: which one is named is first-found, chunks decode concurrently)
            assert results[0][1] == results[1][1], (trial, results[0][1], results[1][1])


def test_fast_reader_layouts(oracle, monkeypatch):
    # padded / unaligned outputs and skipped fields go through the generic store path of the same kernel
    monkeypatch.setenv("CLDN_B200_DECODE_MODE", "seq")
    for n in (5_000, 66_000):
        info, cloud = synth.cloud_c3(n, seed=n, version=5)   # XYZ + V5 sections, step 32
        blob = oracle.encode(info, cloud)
        dinfo, hdr = cb.DecodeHeader(blob)
        got = np.full(n * 32, 0x77, dtype=np.uint8)
        cb.PointcloudDecoder().decode(dinfo, blob[hdr:], got)
        assert np.array_equal(got, _want(oracle, blob, n * 32, 0x77))


# ---- encoder -------------------------------------------------------------------------------------------------------
def _xyzi_adversarial(n, seed):
    info, cloud = synth.cloud_c2(n, seed=seed)
    rng = np.random.default_rng(seed)
    pts = cloud.view(np.float32).reshape(n, 4).copy()
    flat = pts.reshape(-1)
    k = max(n // 200, 1)
    idx = rng.choice(flat.size, size=min(5 * k, flat.size), replace=False)
    q = max(len(idx) // 5, 1)
    flat[idx[:q]] = np.nan
    flat[idx[q:2 * q]] = rng.choice(np.array([np.inf, -np.inf, 3e9, -3e9, 2.2e6, -2.2e6, 33554.4, -33554.5], dtype=np.float32), size=len(idx[q:2 * q]))
    flat[idx[2 * q:3 * q]] = (rng.integers(-5000, 5000, size=len(idx[2 * q:3 * q])).astype(np.float32) + 0.5) * np.float32(0.001)  # .5 ties
    flat[idx[3 * q:4 * q]] = rng.normal(0, 1e-4, size=len(idx[3 * q:4 * q])).astype(np.float32)
    flat[idx[4 * q:]] = np.float32(-0.0)
    return info, np.ascontiguousarray(pts).view(np.uint8).reshape(-1)


@pytest.mark.parametrize("n", [1, 8, 1023, 1024, 1025, 4096, 4097, 32768, 32769, 70_000])
def test_fast_writer_sizes_and_edges(oracle, n):
    # tiles of 1024 points, groups of 4 tiles per CTA, chunk boundaries every 32 tiles, the partial last tile
    info, cloud = synth.cloud_c2(n, seed=n)
    assert cb.PointcloudEncoder(info).encode(cloud) == oracle.encode(info, cloud)
    info, cloud = _xyzi_adversarial(n, seed=n + 1)   # NaN / inf / huge / tie values: those tiles take the exact path
    assert cb.PointcloudEncoder(info).encode(cloud) == oracle.encode(info, cloud)


def test_fast_writer_near_the_range_limit(oracle):
    # |v * mul| just below / at / above 2^25 (the fast path's bound) and deltas that need exactly 4 / 5 varint bytes
    n = 3000
    info, cloud = synth.cloud_c2(n, seed=9)
    pts = cloud.view(np.float32).reshape(n, 4).copy()
    lim = np.float32(33554.432)  # 2^25 mm
    for i, v in enumerate([lim, -lim, np.nextafter(lim, np.float32(0)), np.nextafter(lim, np.float32(1e9)), np.float32(33554.0), np.float32(-33554.3)]):
        pts[100 + 300 * i, i % 3] = v
    pts[2000, 0] = np.float32(134217.7); pts[2001, 0] = np.float32(-134217.7)   # delta 2^28: a 5-byte varint
    cloud = np.ascontiguousarray(pts).view(np.uint8).reshape(-1)
    assert cb.PointcloudEncoder(info).encode(cloud) == oracle.encode(info, cloud)


def test_fast_writer_batches(oracle):
    # uniform batch (frame-interleaved groups) through the device API, with one frame full of NaNs, and a 4-byte
    # misaligned input (the kernel then loads field by field)
    F, n = 5, 40_000
    info = synth.info_xyzi(n)
    clouds = [synth.cloud_c2(n, seed=70 + k)[1] for k in range(F)]
    clouds[2] = _xyzi_adversarial(n, seed=99)[1]
    enc = cb.PointcloudEncoder(info)
    cap = cb.MaxCompressedSize(info, n, True)
    d_in = [_Dev(src=c) for c in clouds]
    d_blob = [_Dev(size=cap) for _ in range(F)]
    sizes = enc.encode_batch_device(enc.make_device_batch([t.ptr for t in d_in], [n * 16] * F, [t.ptr for t in d_blob], [cap] * F),
                                    write_header=True, want_sizes=True)
    for k in range(F):
        assert bytes(d_blob[k].numpy()[:sizes[k]]) == oracle.encode(info, clouds[k]), k
    shifted = _Dev(size=n * 16 + 16)
    if hasattr(shifted.t, "cpu"):
        import torch
        shifted.t[4:4 + n * 16] = torch.from_numpy(clouds[0]).to(shifted.t.device)
        torch.cuda.synchronize()
    else:
        shifted.t[4:4 + n * 16] = clouds[0]
    out = _Dev(size=cap)
    sizes = enc.encode_batch_device(enc.make_device_batch([shifted.ptr + 4], [n * 16], [out.ptr], [cap]), write_header=True, want_sizes=True)
    assert bytes(out.numpy()[:sizes[0]]) == oracle.encode(info, clouds[0])


def test_fast_writer_large_and_ragged_batches(oracle):
    # more frames than the kernel caches records for (32), frames of different sizes (no uniform tile order), empty frames
    rng = np.random.default_rng(3)
    sizes_pts = [int(x) for x in rng.integers(1, 5000, 44)] + [0, 256, 257, 32768, 33000, 0]
    F = len(sizes_pts)
    info = synth.info_xyzi(1)
    clouds = [synth.cloud_c2(max(n, 1), seed=500 + k)[1][:n * 16] for k, n in enumerate(sizes_pts)]
    clouds[5] = _xyzi_adversarial(sizes_pts[5] or 1, seed=77)[1][:sizes_pts[5] * 16]
    enc = cb.PointcloudEncoder(info)
    caps = [cb.MaxCompressedSize(synth.info_xyzi(max(n, 1)), n, True) + 64 for n in sizes_pts]
    d_in = [_Dev(src=c) if c.size else _Dev(size=16) for c in clouds]
    d_blob = [_Dev(size=c) for c in caps]
    sizes = enc.encode_batch_device(enc.make_device_batch([t.ptr for t in d_in], [n * 16 for n in sizes_pts], [t.ptr for t in d_blob], caps),
                                    write_header=False, want_sizes=True)
    for k, n in enumerate(sizes_pts):
        one = synth.info_xyzi(n)
        want = oracle.encode(one, clouds[k], write_header=False) if n else b""
        assert bytes(d_blob[k].numpy()[:sizes[k]]) == want, (k, n)


# ---- sensor layouts with scalar lossy floats behind the FloatN group (Velodyne XYZIRT ...) -----------------------------
def _xyzirt(n, seed, time_scale=1.0):
    info, cloud = synth.cloud_c4_mixed_frame(seed)
    n0 = info.width
    reps = (n + n0 - 1) // n0
    buf = np.tile(cloud.reshape(n0, 22), (reps, 1))[:n].copy()
    t = (np.arange(n, dtype=np.float64) * 1e-4 * time_scale).astype(np.float32)
    buf[:, 18:22] = t.view(np.uint8).reshape(n, 4)
    info.width = n
    return info, np.ascontiguousarray(buf).reshape(-1)


def test_mixed_float_layouts_take_the_fast_paths(oracle, monkeypatch):
    monkeypatch.setenv("CLDN_B200_DECODE_MODE", "seq")
    F = cb.FieldType
    for n in (1, 511, 512, 513, 40_000, 70_001):
        cases = [_xyzirt(n, 3)]
        # three scalar lossy floats and no FloatN group at all (an int field first breaks the leading group), step 20
        rng = np.random.default_rng(n)
        raw = np.zeros((n, 20), dtype=np.uint8)
        raw[:, 0:4] = (np.arange(n) % 5).astype(np.uint32).view(np.uint8).reshape(n, 4)
        for k in range(3):
            raw[:, 4 + 4 * k:8 + 4 * k] = np.cumsum(rng.normal(0, 0.05, n)).astype(np.float32).view(np.uint8).reshape(n, 4)
        info = cb.EncodingInfo(fields=[cb.PointField("id", 0, F.UINT32, None), cb.PointField("a", 4, F.FLOAT32, 0.001), cb.PointField("b", 8, F.FLOAT32, 0.002),
                                       cb.PointField("c", 12, F.FLOAT32, 0.0005)],
                               width=n, height=1, point_step=20, compression_opt=cb.CompressionOption.NONE, use_threads=False, version=5)
        cases.append((info, raw.reshape(-1)))
        for info, cloud in cases:
            blob = oracle.encode(info, cloud)
            assert cb.PointcloudEncoder(info).encode(cloud) == blob
            hdr = len(cb.PointcloudEncoder(info).getHeader())
            outs, (fast, redo) = _decode_batch(info, [blob, blob], hdr, cloud.size, 0x19)
            chunks = 2 * ((n + 32767) // 32768)
            assert (fast, redo) == (chunks, 0), (n, fast, redo)
            for o in outs:
                assert np.array_equal(o, _want(oracle, blob, cloud.size, 0x19))


def test_mixed_float_layouts_hand_over_what_is_not_plain(oracle, monkeypatch):
    monkeypatch.setenv("CLDN_B200_DECODE_MODE", "seq")
    n = 70_000
    info, plain = _xyzirt(n, 5)
    pts = plain.reshape(n, 22).copy()
    nan_c = pts.copy(); nan_c[40_000, 18:22] = np.frombuffer(np.float32(np.nan).tobytes(), dtype=np.uint8)   # NaN in the scalar field
    wide_c = pts.copy(); wide_c[100, 0:4] = np.frombuffer(np.float32(3.0e6).tobytes(), dtype=np.uint8)        # 5-byte varint
    _, big_t = _xyzirt(n, 5, time_scale=5000.0)        # time * 1e5 leaves the int32 range half way through the cloud
    clouds = [plain, nan_c.reshape(-1), wide_c.reshape(-1), big_t]
    blobs, hdr = _encode_all(info, clouds, oracle)
    for c, b in zip(clouds, blobs):
        assert cb.PointcloudEncoder(info).encode(c) == b
    outs, (fast, redo) = _decode_batch(info, blobs, hdr, n * 22, 0x44)
    assert fast == 4 * 3 and redo >= 3, (fast, redo)
    for b, o in zip(blobs, outs):
        assert np.array_equal(o, _want(oracle, b, n * 22, 0x44))


@pytest.mark.parametrize("shift", [0, 2, 16])
def test_whole_row_copy_out_at_any_output_address(oracle, monkeypatch, shift):
    """Layouts whose fields cover every byte of a point leave the fast reader as whole rows (16-byte stores) when the output
    is 16-byte aligned, and field by field otherwise: same bytes, nothing outside [out, out + n * step) is touched."""
    monkeypatch.setenv("CLDN_B200_DECODE_MODE", "seq")
    for n in (129, 40_003):
        made = [_xyzirt(n, 5), synth.cloud_c1(n, seed=9)]
        for info, cloud in made:
            blob = oracle.encode(info, cloud)
            hdr = len(cb.PointcloudEncoder(info).getHeader())
            dec = cb.PointcloudDecoder()
            d_blob = _Dev(src=np.frombuffer(blob, dtype=np.uint8))
            guard = 64
            d_out = _Dev(src=np.full(cloud.size + 2 * guard + 32, 0xA7, dtype=np.uint8))
            base = d_out.ptr + guard
            base += (-base) % 16 + shift                      # 16-byte aligned + shift
            batch = dec.make_device_batch([d_blob.ptr + hdr], [len(blob) - hdr], [base], [cloud.size])
            dec.decode_batch_device(info, batch, sync=True)
            fast, redo = dec.last_stats()
            assert (fast, redo) == ((n + 32767) // 32768, 0)
            got = d_out.numpy()
            o0 = base - d_out.ptr
            assert np.array_equal(got[o0:o0 + cloud.size], _want(oracle, blob, cloud.size, 0xA7))
            assert np.all(got[:o0] == 0xA7) and np.all(got[o0 + cloud.size:] == 0xA7)


# ---- V5 sections ahead of the regular stream (side mode) -------------------------------------------------------------
def _decode_batch_side(info, blobs, hdr, n_bytes, fill, shift=0):
    dec = cb.PointcloudDecoder()
    d_blobs = [_Dev(src=np.frombuffer(b, dtype=np.uint8)) for b in blobs]
    d_outs = [_Dev(src=np.full(n_bytes + 64, fill, dtype=np.uint8)) for _ in blobs]
    bases = [t.ptr + (-t.ptr) % 16 + shift for t in d_outs]
    batch = dec.make_device_batch([t.ptr + hdr for t in d_blobs], [len(b) - hdr for b in blobs], bases, [n_bytes] * len(blobs))
    dec.decode_batch_device(info, batch, sync=True)
    outs = []
    for d, b in zip(d_outs, bases):
        a = d.numpy()
        o0 = b - d.ptr
        assert np.all(a[:o0] == fill) and np.all(a[o0 + n_bytes:] == fill)
        outs.append(a[o0:o0 + n_bytes])
    return outs, dec.last_stats(), dec.last_sections_ahead()


def _int_sections_layout(n, seed, with_u64=False, only_u64=False):
    """XYZ (FloatN) + int16 / uint32 / (uint64) / uint16 adaptive fields, padded step 40: every V5 mode shows up. The side
    mode carries at most 8 bytes of section values per point (1024-point tiles): with_u64 = 16 bytes, sections behind."""
    F = cb.FieldType
    rng = np.random.default_rng(seed)
    raw = np.full((n, 40), 0xEE, dtype=np.uint8)
    xyz = np.cumsum(rng.normal(0, 0.01, (n, 3)), axis=0).astype(np.float32)
    raw[:, 0:12] = xyz.view(np.uint8).reshape(n, 12)
    a = (rng.integers(-300, 300, n)).astype(np.int16)                                   # DeltaVarint
    b = rng.choice(np.array([7, 1 << 20, 0xFFFFFFF0, 12345], dtype=np.uint32), n)       # Palette
    c = (np.arange(n, dtype=np.uint64) // 900) * np.uint64(1 << 33)                     # Rle (64-bit)
    d = (np.arange(n) % 128).astype(np.uint16)                                          # DeltaRle
    raw[:, 12:14] = a.view(np.uint8).reshape(n, 2)
    raw[:, 16:20] = b.view(np.uint8).reshape(n, 4)
    raw[:, 24:32] = c.view(np.uint8).reshape(n, 8)
    raw[:, 32:34] = d.view(np.uint8).reshape(n, 2)
    fields = [cb.PointField("x", 0, F.FLOAT32, 0.001), cb.PointField("y", 4, F.FLOAT32, 0.001), cb.PointField("z", 8, F.FLOAT32, 0.001)]
    if only_u64:
        fields.append(cb.PointField("c", 24, F.UINT64, None))
    else:
        fields += [cb.PointField("a", 12, F.INT16, None), cb.PointField("b", 16, F.UINT32, None)]
        if with_u64:
            fields.append(cb.PointField("c", 24, F.UINT64, None))
        fields.append(cb.PointField("d", 32, F.UINT16, None))
    info = cb.EncodingInfo(fields=fields, width=n, height=1, point_step=40, compression_opt=cb.CompressionOption.NONE, use_threads=False, version=5)
    return info, raw.reshape(-1)


@pytest.mark.parametrize("shift", [0, 2])
@pytest.mark.parametrize("n", [1, 9, 1024, 4097, 32768, 32769, 70_001])
def test_sections_ahead_same_bytes_as_sections_behind(oracle, monkeypatch, n, shift):
    monkeypatch.setenv("CLDN_B200_DECODE_MODE", "seq")
    cases = [synth.cloud_c3(n, seed=n, version=5), _xyzirt(n, 3), _int_sections_layout(n, n), _int_sections_layout(n, n + 1, only_u64=True)]
    for info, cloud in cases:
        step = info.point_step
        clouds = [cloud, np.ascontiguousarray(cloud.reshape(n, step)[::-1]).reshape(-1)]
        blobs, hdr = _encode_all(info, clouds, oracle)
        seen = {}
        for flag in ("1", "0"):
            monkeypatch.setenv("CLDN_B200_DECODE_SIDE", flag)
            outs, (fast, redo), ahead = _decode_batch_side(info, blobs, hdr, n * step, 0x5C, shift)
            assert ahead == (flag == "1"), (n, flag)
            assert (fast, redo) == (2 * ((n + 32767) // 32768), 0), (n, flag, fast, redo)
            seen[flag] = outs
        for b, o1, o0 in zip(blobs, seen["1"], seen["0"]):
            want = _want(oracle, b, n * step, 0x5C)
            assert np.array_equal(o1, want), (n, shift)
            assert np.array_equal(o0, want), (n, shift)


def test_sections_ahead_with_chunks_for_the_careful_kernels(oracle, monkeypatch):
    """NaN markers / wide values in the regular stream: the chunk's sections were decoded ahead, its rows were not merged; the
    careful kernels decode stream and sections again. Batches mix plain and redone chunks."""
    monkeypatch.setenv("CLDN_B200_DECODE_MODE", "seq")
    monkeypatch.setenv("CLDN_B200_DECODE_SIDE", "1")   # (unpadded one-section layouts like XYZIRT only take it when asked)
    n = 70_000
    for make in (lambda: synth.cloud_c3(n, seed=11, version=5), lambda: _xyzirt(n, 5), lambda: _int_sections_layout(n, 12)):
        info, plain = make()
        step = info.point_step
        pts = plain.reshape(n, step).copy()
        nan_c = pts.copy(); nan_c[40_000, 4:8] = np.frombuffer(np.float32(np.nan).tobytes(), dtype=np.uint8)
        wide_c = pts.copy(); wide_c[100, 0:4] = np.frombuffer(np.float32(3.0e6).tobytes(), dtype=np.uint8)
        last_c = pts.copy(); last_c[n - 1, 8:12] = np.frombuffer(np.float32(np.nan).tobytes(), dtype=np.uint8)
        clouds = [plain, nan_c.reshape(-1), wide_c.reshape(-1), last_c.reshape(-1)]
        blobs, hdr = _encode_all(info, clouds, oracle)
        outs, (fast, redo), ahead = _decode_batch_side(info, blobs, hdr, n * step, 0x21)
        assert ahead and fast == 12 and redo == 3, (fast, redo, ahead)
        for b, o in zip(blobs, outs):
            assert np.array_equal(o, _want(oracle, b, n * step, 0x21))


def test_sections_ahead_on_damaged_blobs_reports_like_sections_behind(oracle, monkeypatch):
    """Damage anywhere in a V5 blob (stream, section modes, palettes, run tables, trailing bytes): same outcome, same message
    and -- when the blob still decodes -- same bytes with the sections ahead of or behind the regular stream."""
    n = 40_000
    rng = np.random.default_rng(99)
    for info, cloud in (synth.cloud_c3(n, seed=21, version=5), _int_sections_layout(n, 22)):
        step = info.point_step
        blob = oracle.encode(info, cloud)
        hdr = len(cb.PointcloudEncoder(info).getHeader())
        # where chunk 0's sections start: its stream ends there
        size0 = int(np.frombuffer(blob[hdr:hdr + 4], dtype=np.uint32)[0])
        for trial in range(24):
            bad = bytearray(blob)
            kind = trial % 6
            if kind == 0:      # cut the payload
                bad = bad[:hdr + int(rng.integers(5, len(blob) - hdr))]
            elif kind == 1:    # flip bytes anywhere
                for _ in range(3):
                    bad[hdr + 4 + int(rng.integers(0, len(blob) - hdr - 4))] = int(rng.integers(0, 256))
            elif kind == 2:    # flip bytes near the end of chunk 0 (its sections)
                for _ in range(3):
                    bad[hdr + 4 + size0 - 1 - int(rng.integers(0, min(size0 - 1, 3000)))] = int(rng.integers(0, 256))
            elif kind == 3:    # one terminator more / less in the stream: the sections start elsewhere
                at = hdr + 4 + int(rng.integers(10, size0 // 2))
                bad[at] ^= 0x80
            elif kind == 4:    # chunk 0 claims one byte less than it has (trailing byte for chunk 0, shifted chunk 1)
                bad[hdr:hdr + 4] = np.uint32(size0 - 1).tobytes()
            else:              # zero byte (NaN marker) in the stream
                bad[hdr + 4 + int(rng.integers(0, size0 // 2))] = 0
            results = []
            for flag in ("1", "0"):
                monkeypatch.setenv("CLDN_B200_DECODE_MODE", "seq")
                monkeypatch.setenv("CLDN_B200_DECODE_SIDE", flag)
                out = np.full(n * step, 0x33, dtype=np.uint8)
                try:
                    cb.PointcloudDecoder().decode(info, bytes(bad[hdr:]), out)
                    results.append(("ok", out.tobytes()))
                except RuntimeError as e:
                    results.append(("err", str(e)))
            if kind in (1, 2) and results[0][0] == results[1][0] == "err":
                continue  # several damaged places = several defects: both orders fail, which defect is named is first-found (chunks decode concurrently)
            assert results[0] == results[1], (trial, kind, results[0][0], results[1][0], results[0][1][:80] if results[0][0] == "err" else "", results[1][1][:80] if results[1][0] == "err" else "")


def test_sections_ahead_limits(oracle, monkeypatch):
    """More adaptive fields than the side arrays carry: sections behind the stream, same bytes. Defaults: padded layouts take
    the side mode, an unpadded layout with one section field (XYZIRT) does not."""
    monkeypatch.setenv("CLDN_B200_DECODE_MODE", "seq")
    monkeypatch.delenv("CLDN_B200_DECODE_SIDE", raising=False)
    for (info, cloud), expect in ((synth.cloud_c3(3000, seed=1, version=5), True), (_xyzirt(3000, 3), False)):
        blob = oracle.encode(info, cloud)
        hdr = len(cb.PointcloudEncoder(info).getHeader())
        outs, _, ahead = _decode_batch_side(info, [blob], hdr, cloud.size, 0x42)
        assert ahead == expect
        assert np.array_equal(outs[0], _want(oracle, blob, cloud.size, 0x42))
    F = cb.FieldType
    n = 5_000
    rng = np.random.default_rng(4)
    raw = np.zeros((n, 32), dtype=np.uint8)
    raw[:, 0:12] = np.cumsum(rng.normal(0, 0.01, (n, 3)), axis=0).astype(np.float32).view(np.uint8).reshape(n, 12)
    fields = [cb.PointField("x", 0, F.FLOAT32, 0.001), cb.PointField("y", 4, F.FLOAT32, 0.001), cb.PointField("z", 8, F.FLOAT32, 0.001)]
    for k in range(5):
        raw[:, 12 + 4 * k:16 + 4 * k] = rng.integers(0, 50, n).astype(np.uint32).view(np.uint8).reshape(n, 4)
        fields.append(cb.PointField(f"i{k}", 12 + 4 * k, F.UINT32, None))
    info = cb.EncodingInfo(fields=fields, width=n, height=1, point_step=32, compression_opt=cb.CompressionOption.NONE, use_threads=False, version=5)
    blob = oracle.encode(info, raw.reshape(-1))
    hdr = len(cb.PointcloudEncoder(info).getHeader())
    outs, (fast, redo), ahead = _decode_batch_side(info, [blob], hdr, n * 32, 0x42)
    assert not ahead and (fast, redo) == (1, 0)
    assert np.array_equal(outs[0], _want(oracle, blob, n * 32, 0x42))
    # 16 bytes of section values per point: more than a tile's shared-memory budget
    info, cloud = _int_sections_layout(n, 8, with_u64=True)
    blob = oracle.encode(info, cloud)
    hdr = len(cb.PointcloudEncoder(info).getHeader())
    outs, (fast, redo), ahead = _decode_batch_side(info, [blob], hdr, n * 40, 0x42)
    assert not ahead and (fast, redo) == (1, 0)
    assert np.array_equal(outs[0], _want(oracle, blob, n * 40, 0x42))
