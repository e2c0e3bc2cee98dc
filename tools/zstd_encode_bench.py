"""ZSTD stage 2 on the device (cldn_b200_encoder_set_stage2_on_device) against the system libzstd route, and against
device LZ4 and no stage 2:

  single  one 1M-point XYZI frame (synth.cloud_c2), CLDN_MEM_DEVICE_POINTS: libzstd route vs device route;
  batch   128 XYZI frames of 130 048 points, CLDN_MEM_DEVICE: device ZSTD vs device LZ4 vs NONE;
  viz     128 viz clouds of 100k..300k points (synth.cloud_viz) through encode_blobs, CLDN_MEM_DEVICE_POINTS:
          libzstd route vs device route.

Outputs are checked first: every chunk frame of every blob must give its stage-1 bytes back through libzstd's
ZSTD_decompress. Times are medians of --steps runs in which the variants of a case alternate, wall clock around
synchronous calls. The coder's kernel time (zstd_compress_blocks_kernel) comes from a separate torch.profiler run (the
kernel is launched inside the library, between other kernels of the same call, so CUDA events recorded by the caller
cannot bracket it alone); its bytes/s counts stage-1 bytes in + compressed bytes out. The same profiler run splits one
device-route call into its kernels, copies and runtime calls ("breakdown": device time per kernel / copy, host time per
runtime call, ms per call), to show where the route's time goes besides the coder. Prints one JSON line with the
card's name, power limit and SM clock read in the same run.

    python tools/zstd_encode_bench.py [--steps 20] [--warmup 3]
"""
import argparse
import json
import os
import struct
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import cloudini_b200 as cb  # noqa: E402
from cloudini_b200 import synth  # noqa: E402
from blobs_bench import _gpu_state  # noqa: E402
from zstd_corpus import decompress, zstd_lib  # noqa: E402

NONE, LZ4, ZSTD = cb.CompressionOption.NONE, cb.CompressionOption.LZ4, cb.CompressionOption.ZSTD


def _chunks(payload):
    out, p = [], 0
    while p < len(payload):
        (n,) = struct.unpack_from("<I", payload, p)
        out.append(payload[p + 4:p + 4 + n])
        p += 4 + n
    return out


def _encoder(info, comp, on):
    info = cb.EncodingInfo(**{**info.__dict__, "fields": list(info.fields), "compression_opt": comp})
    enc = cb.PointcloudEncoder(info, device=0)
    enc.set_stage2_on_device(on)
    return enc


def _alternate(variants, steps, warmup):
    """Median ms of every variant, the variants run in turn within each step."""
    import torch
    for _ in range(warmup):
        for fn in variants.values():
            fn()
    ts = {k: [] for k in variants}
    for _ in range(steps):
        for k, fn in variants.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            ts[k].append((time.perf_counter() - t0) * 1e3)
    return {k: float(np.median(v)) for k, v in ts.items()}


def _coder_ms(fn, calls=5):
    """(mean ms per call of the ZSTD block kernel, breakdown of a call), from torch.profiler."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            fn()
        torch.cuda.synchronize()
    ev = prof.key_averages()
    us = sum(e.device_time_total for e in ev if "zstd_compress_blocks_kernel" in e.key)
    dev = sorted(((e.key[:60], e.device_time_total / 1e3 / calls) for e in ev if e.device_time_total > 0), key=lambda x: -x[1])[:8]
    host = sorted(((e.key[:60], e.cpu_time_total / 1e3 / calls) for e in ev if e.key.startswith("cuda")), key=lambda x: -x[1])[:8]
    return us / 1e3 / calls, {"device_ms": dict(dev), "runtime_host_ms": dict(host)}


def _check(z, stage1_payloads, blobs):
    """Every chunk frame of every blob decompresses (libzstd) to the stage-1 chunk. Returns (stage-1 bytes, frame bytes)."""
    s1 = out = 0
    for plain, blob in zip(stage1_payloads, blobs):
        want, got = _chunks(plain), _chunks(blob[cb.DecodeHeader(blob)[1]:])
        assert len(want) == len(got)
        for a, b in zip(want, got):
            ok, back = decompress(z, b, len(a))
            assert ok and back == a, "a device frame does not round-trip through libzstd"
            s1 += len(a)
            out += len(b)
    return s1, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    import torch
    assert b"cusim" not in cb.lib().cldn_b200_version(), "refusing the cusim test emulation"
    z = zstd_lib()
    res = {"gpu": _gpu_state(), "steps": a.steps}

    # ---- single: one 1M-point XYZI frame, device points, host blob -------------------------------------------------
    info, cloud = synth.cloud_c2(1_000_000, seed=1000)
    dev = torch.from_numpy(cloud.reshape(-1).view(np.uint8).copy()).cuda()
    torch.cuda.synchronize()
    lib_enc, dev_enc, plain = _encoder(info, ZSTD, False), _encoder(info, ZSTD, True), _encoder(info, NONE, False)
    stage1 = plain.encode(cloud)
    b_lib, b_dev = lib_enc.encode_device(dev.data_ptr(), dev.numel()), dev_enc.encode_device(dev.data_ptr(), dev.numel())
    s1, out = _check(z, [stage1[cb.DecodeHeader(stage1)[1]:]], [b_dev])
    n = cloud.size // info.point_step
    t = _alternate({"libzstd": lambda: lib_enc.encode_device(dev.data_ptr(), dev.numel()),
                    "device": lambda: dev_enc.encode_device(dev.data_ptr(), dev.numel())}, a.steps, a.warmup)
    coder, split = _coder_ms(lambda: dev_enc.encode_device(dev.data_ptr(), dev.numel()))
    res["single_1M_xyzi"] = {
        "ms": t, "gpoints_s": {k: n / v / 1e6 for k, v in t.items()},
        "bytes_per_point": {"libzstd": len(b_lib) / n, "device": len(b_dev) / n},
        "coder_ms": coder, "coder_gb_s": (s1 + out) / coder / 1e6, "breakdown": split}

    # ---- batch: 128 headline frames, device memory ------------------------------------------------------------------
    frames, pts = 128, 130_048
    clouds = [synth.cloud_c2(pts, seed=2000 + k)[1] for k in range(frames)]
    info = synth.cloud_c2(pts, seed=2000)[0]
    ins = [torch.from_numpy(c.reshape(-1).view(np.uint8).copy()).cuda() for c in clouds]
    encs = {"zstd_device": _encoder(info, ZSTD, True), "lz4_device": _encoder(info, LZ4, False), "none": _encoder(info, NONE, False)}
    cap = max(cb.MaxCompressedSize(e.getEncodingInfo(), pts, True) for e in encs.values())
    outs = torch.empty(frames * cap, dtype=torch.uint8, device="cuda")
    import ctypes as C
    a_in = (C.c_void_p * frames)(*[x.data_ptr() for x in ins])
    a_inb = (C.c_size_t * frames)(*[x.numel() for x in ins])
    a_out = (C.c_void_p * frames)(*[outs.data_ptr() + f * cap for f in range(frames)])
    a_cap = (C.c_size_t * frames)(*([cap] * frames))
    args = (frames, a_in, a_inb, a_out, a_cap)
    sizes = {k: e.encode_batch_device(args, want_sizes=True) for k, e in encs.items()}
    encs["zstd_device"].encode_batch_device(args, want_sizes=True)   # the blobs to check are the last ones written
    host = outs.cpu().numpy()
    zblobs = [host[f * cap:f * cap + sizes["zstd_device"][f]].tobytes() for f in range(frames)]
    plain = _encoder(info, NONE, False)
    s1, out = _check(z, [plain.encode(c, write_header=False) for c in clouds], zblobs)
    t = _alternate({k: (lambda e=e: e.encode_batch_device(args, want_sizes=True)) for k, e in encs.items()}, a.steps, a.warmup)
    coder, split = _coder_ms(lambda: encs["zstd_device"].encode_batch_device(args, want_sizes=True))
    res["batch_128_headline"] = {
        "ms": t, "gpoints_s": {k: frames * pts / v / 1e6 for k, v in t.items()},
        "bytes_per_point": {k: sum(v) / (frames * pts) for k, v in sizes.items()},
        "libzstd_bytes_per_point": sum(len(_encoder(info, ZSTD, False).encode(c)) for c in clouds[:8]) / (8 * pts),
        "coder_ms": coder, "coder_gb_s": (s1 + out) / coder / 1e6, "breakdown": split}
    del outs, ins

    # ---- viz: 128 viz clouds through encode_blobs, device points, host blobs -----------------------------------------
    rng = np.random.default_rng(9)
    viz = [synth.cloud_viz(int(rng.integers(100_000, 300_001)), seed=1000 + k) for k in range(128)]
    info = viz[0][0]
    vdev = [torch.from_numpy(c.reshape(-1).view(np.uint8).copy()).cuda() for _, c in viz]
    torch.cuda.synchronize()
    ptrs, nbytes = [x.data_ptr() for x in vdev], [x.numel() for x in vdev]
    lib_enc, dev_enc = _encoder(info, ZSTD, False), _encoder(info, ZSTD, True)
    b_lib, b_dev = lib_enc.encode_blobs_from_device(ptrs, nbytes), dev_enc.encode_blobs_from_device(ptrs, nbytes)
    stage1 = [_encoder(info, NONE, False).encode_blobs([c])[0] for _, c in viz]
    s1, out = _check(z, [b[cb.DecodeHeader(b)[1]:] for b in stage1], b_dev)
    npts = sum(nbytes) // info.point_step
    t = _alternate({"libzstd": lambda: lib_enc.encode_blobs_from_device(ptrs, nbytes),
                    "device": lambda: dev_enc.encode_blobs_from_device(ptrs, nbytes)}, a.steps, a.warmup)
    coder, split = _coder_ms(lambda: dev_enc.encode_blobs_from_device(ptrs, nbytes))
    res["viz_128_encode_blobs"] = {
        "ms": t, "gpoints_s": {k: npts / v / 1e6 for k, v in t.items()},
        "bytes_per_point": {"libzstd": sum(map(len, b_lib)) / npts, "device": sum(map(len, b_dev)) / npts},
        "coder_ms": coder, "coder_gb_s": (s1 + out) / coder / 1e6, "breakdown": split}
    res["gpu_after"] = _gpu_state()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
