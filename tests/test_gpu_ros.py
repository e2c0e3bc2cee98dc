"""SURVEY.md §8(f) N2 + N3 on the GPU (also re-run under tests/cusim by test_cusim_kernels.py): the viz preprocessing
kernels and the DDS envelope conversions, byte-for-byte against the reference (cloudini_lib/src/ros_msg_utils.cpp) or,
where the reference .so is unavailable, against the committed golden messages generated from it."""
import os
import subprocess

import numpy as np
import pytest

import cloudini_b200 as cb
from cloudini_b200 import ros, synth
from cloudini_b200 import FieldType as FT

pytestmark = pytest.mark.gpu
# order: the N2 envelope (host code around hardware-verified kernels) first, the N3 kernels (no hardware run yet) last

XYZI = [("x", 0, FT.FLOAT32), ("y", 4, FT.FLOAT32), ("z", 8, FT.FLOAT32), ("intensity", 12, FT.FLOAT32)]
VELO = [("x", 0, FT.FLOAT32), ("y", 4, FT.FLOAT32), ("z", 8, FT.FLOAT32), ("intensity", 12, FT.FLOAT32),
        ("ring", 16, FT.UINT16), ("time", 18, FT.FLOAT32), ("stamp", 24, FT.FLOAT64)]


def _same_info(a, b):
    return (a.width, a.height, a.point_step) == (b.width, b.height, b.point_step) and \
        [(f.name, f.offset, int(f.type), None if f.resolution is None else np.float32(f.resolution)) for f in a.fields] == \
        [(f.name, f.offset, int(f.type), None if f.resolution is None else np.float32(f.resolution)) for f in b.fields]


# ---- N2: DDS envelope ----------------------------------------------------------------------------------------------------
def _convert(msg, profile, default_resolution, viz, compression, version=5, encoding=cb.EncodingOptions.LOSSY):
    """The converter's per-message step (tools/src/mcap_converter.cpp:184-204) through the product API."""
    pc = ros.getDeserializedPointCloudMessage(msg)
    ros.applyResolutionProfile(profile, pc.fields, default_resolution)
    if viz:
        ros.applyVizLossyPreprocessing(pc)
    info = ros.toEncodingInfo(pc)
    info.encoding_opt, info.compression_opt, info.version, info.use_threads = encoding, compression, version, False
    return ros.convertPointCloud2ToCompressedCloud(pc, info)


def _cases():
    rng = np.random.default_rng(9)
    velo = rng.integers(0, 256, (20_000, 32), dtype=np.uint8)
    velo[:, :12] = np.stack(synth._lidar_xyz(20_000, rng), axis=1).view(np.uint8)
    velo[:, 12:16] = rng.integers(0, 255, 20_000).astype(np.float32).view(np.uint8).reshape(-1, 1, 4)[:, 0]
    velo[:, 16:18] = (np.arange(20_000) % 64).astype(np.uint16).view(np.uint8).reshape(-1, 2)
    velo[:, 18:22] = (np.arange(20_000) * 1e-5).astype(np.float32).view(np.uint8).reshape(-1, 4)
    velo[:, 24:32] = (1.7e9 + np.arange(20_000) * 1e-6).astype(np.float64).view(np.uint8).reshape(-1, 8)
    yield "xyzi", synth.pointcloud2_msg(XYZI, 16, synth.cloud_viz(40_000, seed=5)[1]), {}, 0.001
    yield "velodyne", synth.pointcloud2_msg(VELO, 32, velo, frame_id="velodyne"), {"intensity": 0.0, "time": 1e-4}, 0.002
    yield "organized", synth.pointcloud2_msg(XYZI[:3], 12, synth.cloud_c1(64 * 50, seed=1)[1], width=64, height=50, frame_id="", is_dense=False), {}, 0.001
    yield "empty", synth.pointcloud2_msg(XYZI, 16, np.zeros(0, dtype=np.uint8)), {}, 0.001


@pytest.mark.parametrize("viz", [False, True])
def test_compress_message_matches_reference(ref, viz):
    for name, msg, profile, res in _cases():
        for version in (5, 4):
            got = _convert(msg, profile, res, viz, cb.CompressionOption.NONE, version)
            want = ref.ros_compress(msg, profile, res, viz, 1, 0, version)
            assert got == want, (name, version, len(got), len(want))


def test_non_canonical_is_dense_byte_is_carried_like_the_reference(ref):
    # found by tests/fuzz/fuzz_dds_messages.py: a CDR bool that is neither 0 nor 1 leaves the reference unchanged
    msg = bytearray(synth.pointcloud2_msg(XYZI, 16, synth.cloud_viz(300, seed=2)[1]))
    assert msg[-1] == 1  # is_dense is the last byte of a PointCloud2 message
    msg[-1] = 0x7C
    msg = bytes(msg)
    comp = _convert(msg, {}, 0.001, False, cb.CompressionOption.NONE)
    assert comp == ref.ros_compress(msg, {}, 0.001, False, 1, 0, 5)
    back = ros.convertCompressedCloudToPointCloud2(ros.getDeserializedPointCloudMessage(comp))
    assert back == ref.ros_decompress(comp, len(msg) + 4096) and back[-1] == 0x7C


def test_decompress_message_matches_reference(ref):
    for name, msg, profile, res in _cases():
        comp = ref.ros_compress(msg, profile, res, False, 1, 0, 5)
        pc = ros.getDeserializedPointCloudMessage(comp)
        got = ros.convertCompressedCloudToPointCloud2(pc)
        want = ref.ros_decompress(comp, len(msg) + 4096)
        assert got == want, name
        # and a message compressed by the product decodes identically through the reference
        ours = _convert(msg, profile, res, True, cb.CompressionOption.NONE)
        assert ros.convertCompressedCloudToPointCloud2(ros.getDeserializedPointCloudMessage(ours)) == ref.ros_decompress(ours, len(msg) + 4096)


@pytest.mark.parametrize("comp", [cb.CompressionOption.ZSTD, cb.CompressionOption.LZ4])
def test_stage2_messages_interoperate(ref, comp):
    # default toEncodingInfo compression is ZSTD: compressed bytes differ between library versions, the round trip must not
    name, msg, profile, res = next(_cases())
    ours = _convert(msg, profile, res, False, comp)
    fused = ros.convert_message(msg, profile, res, True, cb.EncodingOptions.LOSSY, comp, 5)   # stage 2 after the fused stage 1
    assert ref.ros_decompress(fused, len(msg) + 4096) == ref.ros_decompress(ref.ros_compress(msg, profile, res, True, 1, int(comp), 5), len(msg) + 4096)
    theirs = ref.ros_compress(msg, profile, res, False, 1, int(comp), 5)
    want = ref.ros_decompress(theirs, len(msg) + 4096)
    assert ref.ros_decompress(ours, len(msg) + 4096) == want
    assert ros.convertCompressedCloudToPointCloud2(ros.getDeserializedPointCloudMessage(theirs)) == want


def test_golden_messages(golden_ros):
    # no reference needed: fixtures generated from it by tests/golden/make_golden_ros.py
    for name, g in golden_ros.items():
        got = _convert(g["msg"], g["profile"], g["default_resolution"], g["viz"], cb.CompressionOption.NONE)
        assert got == g["compressed"], name
        # the same step as ONE library call (payload device resident between preprocessing and encode, pooled handles):
        # twice, so that the second call runs on reused handles with another width than the first left behind
        for _ in range(2):
            fused = ros.convert_message(g["msg"], g["profile"], g["default_resolution"], g["viz"], cb.EncodingOptions.LOSSY,
                                        cb.CompressionOption.NONE, 5)
            assert fused == g["compressed"], name
        back = ros.convertCompressedCloudToPointCloud2(ros.getDeserializedPointCloudMessage(g["compressed"]))
        assert back == g["restored"], name


def test_dds_roundtrip_like_the_reference_test(golden_ros):
    # cloudini_lib/test/test_ros_msg.cpp:91-144 (DDS_Roundtrip) on the committed excerpt of samples/dds_message.bin:
    # parsed infos, then encode / decode with xyz + intensity at 1 mm: floats within the resolution, ring and the
    # (unaligned, offset 18) FLOAT64 timestamp exactly (Gorilla), default ZSTD stage 2
    if "dds_sample_4000" not in golden_ros:
        pytest.skip("golden excerpt of the reference's sample message not present")
    pc = ros.getDeserializedPointCloudMessage(golden_ros["dds_sample_4000"]["msg"])
    info = ros.toEncodingInfo(pc)
    assert [(f.name, f.offset, f.type) for f in info.fields] == [("x", 0, FT.FLOAT32), ("y", 4, FT.FLOAT32), ("z", 8, FT.FLOAT32),
                                                                ("intensity", 12, FT.FLOAT32), ("ring", 16, FT.UINT16), ("timestamp", 18, FT.FLOAT64)]
    assert (info.width, info.height, info.point_step) == (4000, 1, 26)
    assert info.encoding_opt == cb.EncodingOptions.LOSSY and info.compression_opt == cb.CompressionOption.ZSTD and info.version == 5
    for k in range(4):
        info.fields[k].resolution = 0.001
    original = np.array(pc.data)
    blob = cb.PointcloudEncoder(info).encode(original)
    dinfo, hdr = cb.DecodeHeader(blob)
    assert [(f.name, f.offset, f.type) for f in dinfo.fields] == [(f.name, f.offset, f.type) for f in info.fields]
    decoded = np.zeros(original.size, dtype=np.uint8)
    cb.PointcloudDecoder().decode(dinfo, blob[hdr:], decoded)
    a, b = original.reshape(4000, 26), decoded.reshape(4000, 26)
    fa, fb = a[:, :16].copy().view(np.float32), b[:, :16].copy().view(np.float32)
    ok = np.isfinite(fa)
    assert np.all(np.abs(fa[ok] - fb[ok]) <= 0.001) and np.array_equal(np.isnan(fa), np.isnan(fb))
    assert np.array_equal(a[:, 16:18], b[:, 16:18]) and np.array_equal(a[:, 18:26], b[:, 18:26])


def test_wasm_shaped_message_functions(ref):
    # the DDS-message half of the reference's C ABI (wasm_functions.cpp:58-226) through the GPU codec
    import ctypes as C
    L = cb.lib()
    vp, u32 = C.c_void_p, C.c_uint32
    L.cldn_b200_ComputeCompressedSize.restype, L.cldn_b200_ComputeCompressedSize.argtypes = u32, [vp, u32, C.c_float]
    L.cldn_b200_EncodePointcloudMessage.restype, L.cldn_b200_EncodePointcloudMessage.argtypes = u32, [vp, u32, C.c_float, vp, u32]
    L.cldn_b200_DecodeCompressedMessage.restype, L.cldn_b200_DecodeCompressedMessage.argtypes = u32, [vp, u32, vp, u32]
    L.cldn_b200_ConvertCompressedMsgToPointCloud2Msg.restype, L.cldn_b200_ConvertCompressedMsgToPointCloud2Msg.argtypes = u32, [vp, u32, vp, u32]
    info, cloud = synth.cloud_c2(30_000, seed=8)
    msg = np.frombuffer(synth.pointcloud2_msg(XYZI, 16, cloud), dtype=np.uint8)
    out = np.zeros(msg.size, dtype=np.uint8)
    n = L.cldn_b200_EncodePointcloudMessage(msg.ctypes.data, msg.size, 0.001, out.ctypes.data, out.size)
    assert n > 0 and n == L.cldn_b200_ComputeCompressedSize(msg.ctypes.data, msg.size, 0.001)
    blob = bytes(out[:n])
    dinfo, hdr = cb.DecodeHeader(blob)
    assert dinfo.compression_opt == cb.CompressionOption.ZSTD and all(f.resolution == pytest.approx(0.001) for f in dinfo.fields)
    want = np.zeros(cloud.size, dtype=np.uint8)
    ref.decode(blob, want)                                     # the reference reads what the message encoder wrote
    pc = ros.getDeserializedPointCloudMessage(bytes(msg))
    pc.data = np.frombuffer(blob, dtype=np.uint8)              # wrap the blob like the publisher does: a CompressedPointCloud2 message
    einfo = ros.toEncodingInfo(pc)
    for f in einfo.fields:
        f.resolution = 0.001
    comp = np.frombuffer(ref.ros_compress(bytes(msg), {}, 0.001, False, 1, 2, 5), dtype=np.uint8)   # the reference's own compressed message (ZSTD)
    raw = np.zeros(cloud.size, dtype=np.uint8)
    assert L.cldn_b200_DecodeCompressedMessage(comp.ctypes.data, comp.size, raw.ctypes.data, raw.size) == cloud.size
    assert np.array_equal(raw, want)
    full = np.zeros(msg.size + 64, dtype=np.uint8)
    m = L.cldn_b200_ConvertCompressedMsgToPointCloud2Msg(comp.ctypes.data, comp.size, full.ctypes.data, full.size)
    assert m > 0 and bytes(full[:m]) == ref.ros_decompress(bytes(comp), msg.size + 64)
    # failures return 0: size mismatch (width * height * point_step != data), output too small, garbage
    bad = np.frombuffer(synth.pointcloud2_msg(XYZI, 16, cloud, width=29_999), dtype=np.uint8)
    assert L.cldn_b200_EncodePointcloudMessage(bad.ctypes.data, bad.size, 0.001, out.ctypes.data, out.size) == 0
    assert L.cldn_b200_EncodePointcloudMessage(msg.ctypes.data, msg.size, 0.001, out.ctypes.data, 100) == 0
    assert L.cldn_b200_DecodeCompressedMessage(comp.ctypes.data, 40, raw.ctypes.data, raw.size) == 0


# ---- N3: applyVizLossyPreprocessing ------------------------------------------------------------------------------------
@pytest.mark.parametrize("n,step", [(1, 16), (2, 16), (255, 16), (256, 12), (2049, 16), (40_000, 16), (100_003, 32), (30_000, 22), (5_000, 280)])
def test_viz_preprocess_matches_reference(oracle, n, step):
    info, cloud = synth.cloud_viz(n, seed=n, step=step)
    pp = ros.VizPreprocessor()
    got_info, got, applied = pp.run(info, cloud)
    want_info, want = oracle.viz_preprocess(info, cloud)
    assert applied and got.size == want.size and np.array_equal(got, want)
    assert _same_info(got_info, want_info)
    if n >= 2049:
        assert want_info.width < n  # the input really has NaNs / duplicates
    # the handle is reusable (epoch-tagged status words, re-cleared table): same answer again, then a different cloud
    assert np.array_equal(pp.run(info, cloud)[1], want)
    info2, cloud2 = synth.cloud_viz(max(1, n // 3), seed=n + 1, step=step)
    assert np.array_equal(pp.run(info2, cloud2)[1], oracle.viz_preprocess(info2, cloud2)[1])


def test_viz_preprocess_golden(golden_viz):
    pp = ros.VizPreprocessor()
    for name, (info, cloud, after, kept) in golden_viz.items():
        got_info, got, applied = pp.run(info, cloud)
        assert applied and np.array_equal(got, kept) and _same_info(got_info, after), name


def test_viz_preprocess_edge_cases(oracle):
    pp = ros.VizPreprocessor()
    # all points in one voxel / all NaN / huge coordinates (21-bit truncation of the key, lround overflow) / res 0.5 ties
    info, cloud = synth.cloud_viz(5000, seed=3)
    f = cloud.view(np.float32).reshape(-1, 4).copy()
    f[:, :3] = np.float32(1.2344)
    for case in ("one_voxel", "all_nan", "huge", "ties"):
        g = f.copy()
        if case == "all_nan":
            g[:, 1] = np.nan
        elif case == "huge":
            rng = np.random.default_rng(1)
            g[:, :3] = rng.choice(np.array([1.0e4, -1.0e4, 1048.575, 1048.576, -1048.577, 3.0e9, -3.0e9, 1.0e30, 2097.152, 0.0005, -0.0005, 4194.304],
                                           dtype=np.float32), (5000, 3))
        elif case == "ties":
            g[:, :3] = (np.arange(15000, dtype=np.float32).reshape(5000, 3) % 7) * np.float32(0.25) - np.float32(0.75)
        inf = info
        if case == "ties":
            inf = synth.cloud_viz(1, seed=1)[0]
            inf.width = 5000
            for k in range(3):
                inf.fields[k].resolution = 0.5
        got_info, got, applied = pp.run(inf, g.reshape(-1).view(np.uint8))
        want_info, want = oracle.viz_preprocess(inf, g.reshape(-1).view(np.uint8))
        assert applied and np.array_equal(got, want), case
        assert _same_info(got_info, want_info), case
    # FLOAT64 fields without a resolution get 1e-6; with one they keep it
    rng = np.random.default_rng(2)
    raw = rng.integers(0, 256, 32 * 1000, dtype=np.uint8)
    raw.reshape(1000, 32)[:, :12] = np.stack(synth._lidar_xyz(1000, rng), axis=1).view(np.uint8)
    inf = cb.EncodingInfo(width=1000, height=1, point_step=32, compression_opt=cb.CompressionOption.NONE, use_threads=False)
    inf.fields = [cb.PointField("a", 0, FT.FLOAT32, 0.01), cb.PointField("b", 4, FT.FLOAT32, 0.01), cb.PointField("c", 8, FT.FLOAT32, 0.01),
                  cb.PointField("t", 16, FT.FLOAT64, None), cb.PointField("u", 24, FT.FLOAT64, 0.5)]
    got_info, got, applied = pp.run(inf, raw)
    want_info, want = oracle.viz_preprocess(inf, raw)
    assert applied and np.array_equal(got, want) and _same_info(got_info, want_info)
    assert got_info.fields[3].resolution == pytest.approx(1e-6) and got_info.fields[4].resolution == 0.5


def test_viz_preprocess_no_op_conditions(oracle):
    pp = ros.VizPreprocessor()
    info, cloud = synth.cloud_viz(1000, seed=1)
    variants = []
    a = synth.cloud_viz(1000, seed=1)[0]; a.fields[1].resolution = 0.002; variants.append(a)          # resolutions differ
    b = synth.cloud_viz(1000, seed=1)[0]; b.fields[2].offset = 12; variants.append(b)                  # not consecutive
    c = synth.cloud_viz(1000, seed=1)[0]; c.fields[0].type = FT.INT32; variants.append(c)              # not FLOAT32
    d = synth.cloud_viz(1000, seed=1)[0]; d.fields = d.fields[:2]; variants.append(d)                  # fewer than 3 fields
    e = synth.cloud_viz(1000, seed=1)[0]
    for k in range(3):
        e.fields[k].resolution = None
    variants.append(e)                                                                                  # no resolution
    for v in variants:
        got_info, got, applied = pp.run(v, cloud)
        assert not applied and got_info is v and np.array_equal(got, cloud)
        want_info, want = oracle.viz_preprocess(v, cloud)
        assert np.array_equal(want, cloud)
    assert pp.run(info, np.zeros(0, dtype=np.uint8))[2] is False                                        # empty cloud


def test_viz_preprocess_device_pointers(oracle):
    from test_gpu_parity import _Dev
    info, cloud = synth.cloud_viz(70_000, seed=11)
    d_in, d_out = _Dev(src=cloud), _Dev(size=cloud.size)
    new_info, kept, applied = ros.VizPreprocessor().run_device(info, d_in.ptr, cloud.size, d_out.ptr, cloud.size)
    want_info, want = oracle.viz_preprocess(info, cloud)
    assert applied and kept == want_info.width and np.array_equal(d_out.numpy()[:kept * 16], want)


def test_viz_then_encode_matches_reference_pipeline(oracle):
    # preprocessing feeds the encoder: the blob equals the reference's encode of the reference's preprocessed cloud
    info, cloud = synth.cloud_viz(60_000, seed=21)
    new_info, kept, _ = ros.VizPreprocessor().run(info, cloud)
    want_info, want = oracle.viz_preprocess(info, cloud)
    assert cb.PointcloudEncoder(new_info).encode(kept) == oracle.encode(want_info, want)


# ---- the cloudini_ros C++ shim (include/cloudini_b200/ros_msg_utils.hpp) through its converter-step executable ---------
def test_ros_shim_converter_step_matches_golden(lib_built, golden_ros, tmp_path):
    # the C++ shim reproduces the reference converter's output (golden messages generated from the reference)
    from test_cpp_shim import _compile_ros, _run_env
    ros_exe = _compile_ros(lib_built, tmp_path)
    for name in ("xyzi_viz", "xyz_organized", "dds_sample_4000"):
        if name not in golden_ros:  # the sample excerpt exists only when the goldens were generated next to the reference tree
            continue
        g = golden_ros[name]
        src, comp, rest = tmp_path / "in.msg", tmp_path / "out.comp", tmp_path / "out.rest"
        src.write_bytes(g["msg"])
        out = subprocess.run([ros_exe, str(src), str(comp), str(rest), repr(g["default_resolution"]), "1" if g["viz"] else "0"],
                             capture_output=True, text=True, timeout=120, env=_run_env(tmp_path))
        assert out.returncode == 0 and "ros_shim_convert: ok" in out.stdout, out.stdout + out.stderr
        assert comp.read_bytes() == g["compressed"], name
        assert rest.read_bytes() == g["restored"], name
