"""Secondary measurements that ride along with bench.py as `extras` (never the headline, never able to break it: bench.py
runs this file in a child process with a timeout and records whatever JSON line it prints, or the error).

  viz   applyVizLossyPreprocessing kernels (SURVEY 8(f) N3) on a device-resident 1M-point XYZI cloud: ms per call,
        survivors checked against a numpy restatement of "finite && first point of its voxel" (no oracle involved)
  c3    BASELINE configs[2]: 1M-point XYZ + rgba u32 + ring u16 (V5 adaptive sections), 32 frames, encode / decode ms
  c4    BASELINE configs[3] with the Velodyne XYZIRT layout (step 22), 64 frames of 130 048 points, encode / decode ms
  msg   the DDS converter step (parse -> profile -> viz -> compress message) on one 1M-point PointCloud2, host buffers
  zstd  the headline's 128 XYZI frames compressed once with ZSTD level 1 (what Cloudini ships, host-pointer encoder):
        device-resident ZSTD + stage-1 decode per batch, one-message host-pointer decode latency, libzstd decompression
        of the same chunks on one host core, bytes per point; parity with the oracle before any number
"""
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

import cloudini_b200 as cb  # noqa: E402
from cloudini_b200 import ros, synth  # noqa: E402


def hbm_peak():
    """HBM3 bandwidth of the H100 SXM data sheet (700 W board), in GB/s."""
    return 3350.0


def numpy_first_voxel_mask(cloud, step, res):
    """finite && first occurrence of (lround(x/res), lround(y/res), lround(z/res)) truncated to 21 bits per axis."""
    n = cloud.size // step
    xyz = cloud.reshape(n, step)[:, :12].copy().view(np.float32)
    finite = np.isfinite(xyz).all(axis=1)
    inv = np.float32(1.0) / np.float32(res)
    prod = (xyz * inv).astype(np.float32)
    q = np.where(finite[:, None], np.sign(prod) * np.floor(np.abs(prod).astype(np.float64) + 0.5), 0).astype(np.int64)
    u = (q + (1 << 20)) & ((1 << 21) - 1)
    key = u[:, 0] | (u[:, 1] << 21) | (u[:, 2] << 42)
    key[~finite] = -1 - np.arange(np.count_nonzero(~finite))
    _, first = np.unique(key, return_index=True)
    mask = np.zeros(n, dtype=bool)
    mask[first] = True
    return mask & finite


def bench_viz(out):
    n = 1_000_000
    info, cloud = synth.cloud_viz(n, seed=77)
    d_in = torch.from_numpy(cloud).cuda()
    d_out = torch.zeros(cloud.size, dtype=torch.uint8, device="cuda")
    pp = ros.VizPreprocessor()
    new_info, kept, applied = pp.run_device(info, d_in.data_ptr(), cloud.size, d_out.data_ptr(), cloud.size)
    mask = numpy_first_voxel_mask(cloud, 16, 0.001)
    want = cloud.reshape(n, 16)[mask].reshape(-1)
    ok = bool(applied and kept == int(mask.sum()) and np.array_equal(d_out[:kept * 16].cpu().numpy(), want))
    reps = 20
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        pp.run_device(info, d_in.data_ptr(), cloud.size, d_out.data_ptr(), cloud.size)  # synchronous (4-byte count read-back)
    ms = (time.perf_counter() - t0) / reps * 1e3
    out["viz_preprocess"] = {"points": n, "kept": int(kept), "ms_per_call": ms, "mpoints_s": n / ms / 1e3, "matches_numpy_restatement": ok,
                             "algorithmic_bytes": int(n * 16 + kept * 16), "gbs": (n * 16 + kept * 16) / ms / 1e6,
                             "frac_of_hbm": (n * 16 + kept * 16) / ms / 1e6 / hbm_peak()}
    # preprocessing straight into the encoder, everything device resident
    enc = cb.PointcloudEncoder(new_info)
    cap = cb.MaxCompressedSize(new_info, kept, True)
    d_blob = torch.zeros(cap, dtype=torch.uint8, device="cuda")
    batch = enc.make_device_batch([d_out.data_ptr()], [kept * 16], [d_blob.data_ptr()], [cap])
    enc.encode_batch_device(batch, write_header=True, want_sizes=True)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        pp.run_device(info, d_in.data_ptr(), cloud.size, d_out.data_ptr(), cloud.size)
        enc.encode_batch_device(batch, write_header=True, want_sizes=True)
    out["viz_then_encode"] = {"ms_per_frame": (time.perf_counter() - t0) / reps * 1e3}


def bench_c3(out):
    F, n = 32, 1_000_000   # 992 chunks: one per resident CTA of the chunk-sequential reader, like the headline batch
    info, _ = synth.cloud_c3(n)
    clouds = [synth.cloud_c3(n, seed=3 + k)[1] for k in range(F)]
    s = torch.cuda.Stream()
    torch.cuda.set_stream(s)
    enc, dec = cb.PointcloudEncoder(info, stream=s.cuda_stream), cb.PointcloudDecoder(stream=s.cuda_stream)
    step = info.point_step
    d_in = [torch.from_numpy(c).cuda() for c in clouds]
    cap = cb.MaxCompressedSize(info, n, True)
    d_blob = [torch.empty(cap, dtype=torch.uint8, device="cuda") for _ in range(F)]
    d_out = [torch.zeros(n * step, dtype=torch.uint8, device="cuda") for _ in range(F)]
    eb = enc.make_device_batch([t.data_ptr() for t in d_in], [n * step] * F, [t.data_ptr() for t in d_blob], [cap] * F)
    sizes = enc.encode_batch_device(eb, True, want_sizes=True)
    hdr = len(enc.getHeader())
    db = dec.make_device_batch([t.data_ptr() + hdr for t in d_blob], [x - hdr for x in sizes], [t.data_ptr() for t in d_out], [n * step] * F)
    dec.decode_batch_device(info, db, sync=True)
    # size-independent property instead of the oracle: the integer channels survive the round trip exactly, the floats
    # within half a resolution step
    got = d_out[0].cpu().numpy().reshape(n, step)
    src = clouds[0].reshape(n, step)
    ints_ok = bool(np.array_equal(got[:, 16:22], src[:, 16:22]))
    f_err = float(np.max(np.abs(got[:, :12].copy().view(np.float32) - src[:, :12].copy().view(np.float32))))
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    te = td = 0.0
    reps = 10
    for _ in range(3):
        enc.encode_batch_device(eb, True)
        dec.decode_batch_device(info, db, sync=False)
    for _ in range(reps):
        ev[0].record()
        enc.encode_batch_device(eb, True)
        ev[1].record()
        dec.decode_batch_device(info, db, sync=False)
        ev[2].record()
        torch.cuda.synchronize()
        te += ev[0].elapsed_time(ev[1])
        td += ev[1].elapsed_time(ev[2])
    te, td = te / reps, td / reps
    S = float(np.mean(sizes)) - hdr
    algo = F * (n * step + S)
    out["c3_v5_sections"] = {"frames": F, "points": n, "point_step": step, "stage1_B_per_pt": S / n, "encode_ms": te, "decode_ms": td,
                             "encode_mpts": F * n / te / 1e3, "decode_mpts": F * n / td / 1e3, "encode_gbs": algo / te / 1e6,
                             "decode_gbs": algo / td / 1e6, "encode_frac_of_hbm": algo / te / 1e6 / hbm_peak(),
                             "decode_frac_of_hbm": algo / td / 1e6 / hbm_peak(), "ints_roundtrip_exact": ints_ok, "max_float_error": f_err}


def bench_c4_mixed(out):
    """BASELINE configs[3] with the sensor's own layout (XYZI + ring u16 + time f32, step 22, generic kernels + V5 section)."""
    F = 256   # 1024 chunks: the chunk-sequential readers want at least one chunk per resident CTA (7 per SM, 924 on 132 SMs)
    info, _ = synth.cloud_c4_mixed_frame(0)
    clouds = [synth.cloud_c4_mixed_frame(k)[1] for k in range(F)]
    n, step = info.width, info.point_step
    s = torch.cuda.Stream()
    torch.cuda.set_stream(s)
    enc, dec = cb.PointcloudEncoder(info, stream=s.cuda_stream), cb.PointcloudDecoder(stream=s.cuda_stream)
    d_in = [torch.from_numpy(c).cuda() for c in clouds]
    cap = cb.MaxCompressedSize(info, n, True)
    d_blob = [torch.empty(cap, dtype=torch.uint8, device="cuda") for _ in range(F)]
    d_out = [torch.zeros(n * step, dtype=torch.uint8, device="cuda") for _ in range(F)]
    eb = enc.make_device_batch([t.data_ptr() for t in d_in], [n * step] * F, [t.data_ptr() for t in d_blob], [cap] * F)
    sizes = enc.encode_batch_device(eb, True, want_sizes=True)
    hdr = len(enc.getHeader())
    db = dec.make_device_batch([t.data_ptr() + hdr for t in d_blob], [x - hdr for x in sizes], [t.data_ptr() for t in d_out], [n * step] * F)
    dec.decode_batch_device(info, db, sync=True)
    got, src = d_out[0].cpu().numpy().reshape(n, step), clouds[0].reshape(n, step)
    ring_ok = bool(np.array_equal(got[:, 16:18], src[:, 16:18]))
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    te = td = 0.0
    reps = 10
    for _ in range(2):
        enc.encode_batch_device(eb, True)
        dec.decode_batch_device(info, db, sync=False)
    for _ in range(reps):
        ev[0].record()
        enc.encode_batch_device(eb, True)
        ev[1].record()
        dec.decode_batch_device(info, db, sync=False)
        ev[2].record()
        torch.cuda.synchronize()
        te += ev[0].elapsed_time(ev[1])
        td += ev[1].elapsed_time(ev[2])
    te, td = te / reps, td / reps
    S = float(np.mean(sizes)) - hdr
    out["c4_velodyne_xyzirt"] = {"frames": F, "points": n, "point_step": step, "stage1_B_per_pt": S / n, "encode_ms": te, "decode_ms": td,
                                 "encode_mpts": F * n / te / 1e3, "decode_mpts": F * n / td / 1e3, "ring_roundtrip_exact": ring_ok,
                                 "encode_gbs": F * (n * step + S) / te / 1e6, "decode_gbs": F * (n * step + S) / td / 1e6,
                                 "encode_frac_of_hbm": F * (n * step + S) / te / 1e6 / hbm_peak(),
                                 "decode_frac_of_hbm": F * (n * step + S) / td / 1e6 / hbm_peak()}


def bench_msg(out):
    from cloudini_b200 import FieldType as FT
    n = 1_000_000
    fields = [("x", 0, FT.FLOAT32), ("y", 4, FT.FLOAT32), ("z", 8, FT.FLOAT32), ("intensity", 12, FT.FLOAT32)]
    msg = synth.pointcloud2_msg(fields, 16, synth.cloud_viz(n, seed=78)[1])
    pp = ros.VizPreprocessor()

    def step(viz):
        pc = ros.getDeserializedPointCloudMessage(msg)
        ros.applyResolutionProfile({}, pc.fields, 0.001)
        if viz:
            ros.applyVizLossyPreprocessing(pc, pp)
        info = ros.toEncodingInfo(pc)
        info.compression_opt, info.use_threads = cb.CompressionOption.NONE, False
        return ros.convertPointCloud2ToCompressedCloud(pc, info)

    res = {}
    for viz in (False, True):
        comp = step(viz)
        back = ros.convertCompressedCloudToPointCloud2(ros.getDeserializedPointCloudMessage(comp))
        t0 = time.perf_counter()
        for _ in range(5):
            step(viz)
        res["viz" if viz else "plain"] = {"ms_per_message": (time.perf_counter() - t0) / 5 * 1e3, "compressed_bytes": len(comp),
                                          "restored_bytes": len(back)}
    for viz in (False, True):   # the same step as one library call: payload device resident between viz and encode, pooled handles
        want = step(viz)
        got = ros.convert_message(msg, {}, 0.001, viz, cb.EncodingOptions.LOSSY, cb.CompressionOption.NONE, 5)
        t0 = time.perf_counter()
        for _ in range(10):
            ros.convert_message(msg, {}, 0.001, viz, cb.EncodingOptions.LOSSY, cb.CompressionOption.NONE, 5)
        res["fused_viz" if viz else "fused_plain"] = {"ms_per_message": (time.perf_counter() - t0) / 10 * 1e3, "same_bytes_as_the_five_calls": got == want}
    out["dds_converter_step"] = dict(res, points=n, note="pageable host message in, host message out; plain / viz: the five mirror calls "
                                     "(pooled handles); fused_*: cldn_b200_ros_convert_msg")


def bench_zstd(out):
    import ctypes as C
    import struct
    from oracle.client import best_oracle
    F, n = 128, 1_000_000
    info, _ = synth.cloud_c2(n, seed=1000)
    info.compression_opt = cb.CompressionOption.ZSTD
    enc = cb.PointcloudEncoder(info)
    clouds = [synth.cloud_c2(n, seed=1000 + k)[1] for k in range(F)]   # the headline step's frames (bench.py)
    blobs = [enc.encode(c) for c in clouds]
    hdr = cb.DecodeHeader(blobs[0])[1]
    s = torch.cuda.Stream()
    torch.cuda.set_stream(s)
    dec = cb.PointcloudDecoder(stream=s.cuda_stream)
    d_in = [torch.from_numpy(np.frombuffer(b[hdr:], dtype=np.uint8).copy()).cuda() for b in blobs]
    d_out = [torch.zeros(n * 16, dtype=torch.uint8, device="cuda") for _ in range(F)]
    db = dec.make_device_batch([t.data_ptr() for t in d_in], [t.numel() for t in d_in], [t.data_ptr() for t in d_out], [n * 16] * F)
    dec.decode_batch_device(info, db, sync=True)
    # parity: the oracle's decode of the same blob (libzstd + stage 1), every 16th frame
    oracle = best_oracle()
    ok = True
    for k in range(F):
        if k % 16 == 0:
            want = np.zeros(n * 16, dtype=np.uint8)
            oracle.decode(blobs[k], want)
            ok = ok and bool(np.array_equal(d_out[k].cpu().numpy(), want))
    if not ok:
        out["zstd_decode"] = {"parity": "MISMATCH against the oracle"}
        return
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    for _ in range(2):
        dec.decode_batch_device(info, db, sync=False)
    reps, t = 5, 0.0
    for _ in range(reps):
        ev[0].record()
        dec.decode_batch_device(info, db, sync=False)
        ev[1].record()
        torch.cuda.synchronize()
        t += ev[0].elapsed_time(ev[1])
    dev_ms = t / reps
    host_dec = cb.PointcloudDecoder()
    outbuf = np.zeros(n * 16, dtype=np.uint8)
    host_dec.decode(info, blobs[0][hdr:], outbuf)
    t0 = time.perf_counter()
    for _ in range(5):
        host_dec.decode(info, blobs[0][hdr:], outbuf)
    host_ms = (time.perf_counter() - t0) / 5 * 1e3
    z = C.CDLL("libzstd.so.1")
    z.ZSTD_decompress.restype = C.c_size_t
    z.ZSTD_decompress.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]
    chunks, pos, p0 = [], 0, blobs[0][hdr:]
    while pos < len(p0):
        (c,) = struct.unpack_from("<I", p0, pos)
        chunks.append(p0[pos + 4:pos + 4 + c])
        pos += 4 + c
    dst = C.create_string_buffer(1 << 20)
    stage1 = 0
    t0 = time.perf_counter()
    for _ in range(5):
        stage1 = sum(z.ZSTD_decompress(dst, 1 << 20, c, len(c)) for c in chunks)
    lib_ms = (time.perf_counter() - t0) / 5 * 1e3
    zbytes = float(np.mean([len(b) - hdr for b in blobs]))
    out["zstd_decode"] = {"frames": F, "points": n, "parity": f"bit-exact vs {oracle.kind} oracle (every 16th frame)",
                          "zstd_B_per_pt": zbytes / n, "stage1_B_per_pt": stage1 / n,
                          "device_batch_ms": dev_ms, "device_ms_per_frame": dev_ms / F, "device_mpts": F * n / dev_ms / 1e3,
                          "host_api_one_message_ms": host_ms, "libzstd_one_core_ms_per_frame": lib_ms,
                          "libzstd_one_core_mbs": stage1 / lib_ms / 1e3}


if __name__ == "__main__":
    out = {}
    for name, fn in (("viz", bench_viz), ("c3", bench_c3), ("c4", bench_c4_mixed), ("msg", bench_msg), ("zstd", bench_zstd)):
        try:
            fn(out)
        except Exception as e:  # noqa: BLE001 — an extra must never take the others down
            out[name + "_error"] = f"{type(e).__name__}: {e}"[:300]
    print(json.dumps(out), flush=True)
