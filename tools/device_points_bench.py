"""Points on the GPU, blobs in host memory: CLDN_MEM_DEVICE_POINTS against what a caller does without it.

decode: host blobs -> cldn_b200_decode_blobs(CLDN_MEM_HOST) into pinned buffers -> torch H2D of the points, against
        cldn_b200_decode_blobs(CLDN_MEM_DEVICE_POINTS) straight into the device buffers;
encode: device clouds -> torch D2H into pinned buffers -> cldn_b200_encode_blobs(CLDN_MEM_HOST), against
        cldn_b200_encode_blobs(CLDN_MEM_DEVICE_POINTS) reading the device clouds in place.

Two workloads: one 1M-point XYZI frame (synth.cloud_c2), and a batch of --frames varying-size clouds (synth.cloud_viz,
100k..300k points, step 16), each with compression NONE and ZSTD. Blobs and decoded points of the two routes are
compared byte for byte before any timing. Times are medians of --steps runs, wall clock around synchronous calls, the
two routes alternating, after --warmup runs of each. For NONE, `libzstd_alone_ms` is the host time of ZSTD_compress
(level 1) over the same stage-1 chunks, the part of a ZSTD encode that no memory kind changes. Prints one JSON line
with the card's name and power limit.

    python tools/device_points_bench.py [--points 1000000] [--frames 128] [--steps 20] [--warmup 3]
"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import cloudini_b200 as cb  # noqa: E402
from cloudini_b200 import synth  # noqa: E402
from blobs_bench import _gpu_state  # noqa: E402


def _ptrs(xs):
    return (C.c_void_p * len(xs))(*xs)


def _sizes(xs):
    return (C.c_size_t * len(xs))(*xs)


def _alternating_ms(fa, fb, steps, warmup):
    """Medians (ms) of fa and fb, run in turn, each timed between two device synchronisations."""
    import torch
    for _ in range(warmup):
        fa()
        fb()
    ta, tb = [], []
    for _ in range(steps):
        for fn, ts in ((fa, ta), (fb, tb)):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            ts.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(ta)), float(np.median(tb))


def _case(L, info0, clouds, comp, steps, warmup):
    import torch
    n = len(clouds)
    step = info0.point_step
    pts = [c.size // step for c in clouds]
    info = cb.EncodingInfo(**{**info0.__dict__, "fields": list(info0.fields), "compression_opt": comp, "width": pts[0], "height": 1})
    enc = cb.PointcloudEncoder(info)
    caps = [cb.MaxCompressedSize(cb.EncodingInfo(**{**info.__dict__, "width": p}), p, True) for p in pts]
    d_clouds = [torch.from_numpy(c).cuda() for c in clouds]
    h_clouds = [torch.empty(c.size, dtype=torch.uint8, pin_memory=True) for c in clouds]
    outs = {m: [np.empty(c, dtype=np.uint8) for c in caps] for m in (cb.MEM_HOST, cb.MEM_DEVICE_POINTS)}
    written = {m: (C.c_size_t * n)() for m in outs}
    nbytes = _sizes([c.size for c in clouds])
    cap_a = _sizes(caps)
    args = {cb.MEM_HOST: (_ptrs([t.data_ptr() for t in h_clouds]), _ptrs([o.ctypes.data for o in outs[cb.MEM_HOST]])),
            cb.MEM_DEVICE_POINTS: (_ptrs([t.data_ptr() for t in d_clouds]), _ptrs([o.ctypes.data for o in outs[cb.MEM_DEVICE_POINTS]]))}
    torch.cuda.synchronize()

    def encode(mem):
        ins, out_p = args[mem]
        assert L.cldn_b200_encode_blobs(enc._h, n, ins, nbytes, None, None, out_p, cap_a, written[mem], mem) == 0, cb._err()

    def enc_host():
        for h, d in zip(h_clouds, d_clouds):
            h.copy_(d, non_blocking=True)
        torch.cuda.synchronize()
        encode(cb.MEM_HOST)

    def enc_dev():
        encode(cb.MEM_DEVICE_POINTS)

    enc_host()
    enc_dev()
    blobs = [outs[cb.MEM_HOST][f][:written[cb.MEM_HOST][f]].tobytes() for f in range(n)]
    assert blobs == [outs[cb.MEM_DEVICE_POINTS][f][:written[cb.MEM_DEVICE_POINTS][f]].tobytes() for f in range(n)], \
        "blobs differ between the two encode routes"
    enc_ms = _alternating_ms(enc_host, enc_dev, steps, warmup)

    src = [np.frombuffer(b, dtype=np.uint8) for b in blobs]
    b_ptr, b_size = _ptrs([s.ctypes.data for s in src]), _sizes([s.size for s in src])
    need = [c.size for c in clouds]
    h_out = [torch.zeros(c, dtype=torch.uint8, pin_memory=True) for c in need]
    d_out = {m: [torch.zeros(c, dtype=torch.uint8, device="cuda") for c in need] for m in (cb.MEM_HOST, cb.MEM_DEVICE_POINTS)}
    out_args = {cb.MEM_HOST: _ptrs([t.data_ptr() for t in h_out]), cb.MEM_DEVICE_POINTS: _ptrs([t.data_ptr() for t in d_out[cb.MEM_DEVICE_POINTS]])}
    need_a = _sizes(need)
    status = (C.c_int32 * n)()
    dec = cb.PointcloudDecoder()
    torch.cuda.synchronize()

    def decode(mem):
        assert L.cldn_b200_decode_blobs(dec._h, n, b_ptr, b_size, out_args[mem], need_a, mem, status, None) == 0, cb._err()

    def dec_host():
        decode(cb.MEM_HOST)
        for d, h in zip(d_out[cb.MEM_HOST], h_out):
            d.copy_(h, non_blocking=True)
        torch.cuda.synchronize()

    def dec_dev():
        decode(cb.MEM_DEVICE_POINTS)

    dec_host()
    dec_dev()
    torch.cuda.synchronize()
    assert all(torch.equal(a, b) for a, b in zip(d_out[cb.MEM_HOST], d_out[cb.MEM_DEVICE_POINTS])), "decoded points differ between the routes"
    dec_ms = _alternating_ms(dec_host, dec_dev, steps, warmup)

    total = sum(pts)
    stage_bytes = sum(len(b) for b in blobs)
    extra = {}
    if comp == cb.CompressionOption.NONE:
        extra["libzstd_alone_ms"] = round(_libzstd_ms(blobs), 3)

    def entry(ms):
        return {"host_plus_torch_copy_ms": round(ms[0], 3), "device_points_ms": round(ms[1], 3), "speedup": round(ms[0] / ms[1], 3),
                "device_points_mpoints_per_s": round(total / ms[1] / 1e3, 1)}
    return {"frames": n, "points": total, "blob_bytes_per_point": round(stage_bytes / total, 3), "encode": entry(enc_ms), "decode": entry(dec_ms),
            **extra}


def _libzstd_ms(blobs):
    """Host time of ZSTD_compress at level 1 (what the ZSTD encode route calls per chunk) over the stage-1 chunks of
    these NONE blobs, alone: the part of a ZSTD encode that does not depend on where the points are."""
    z = C.CDLL("libzstd.so.1")
    z.ZSTD_compress.restype = C.c_size_t
    z.ZSTD_compress.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_int]
    chunks = []
    for b in blobs:
        p = np.frombuffer(b, dtype=np.uint8)[cb.DecodeHeader(b)[1]:]
        i = 0
        while i < p.size:
            k = int(p[i:i + 4].view(np.uint32)[0])
            chunks.append(p[i + 4:i + 4 + k])
            i += 4 + k
    dst = np.empty(2 * max((c.size for c in chunks), default=0) + 1024, dtype=np.uint8)
    t0 = time.perf_counter()
    for c in chunks:
        z.ZSTD_compress(dst.ctypes.data, dst.size, c.ctypes.data, c.size, 1)
    return (time.perf_counter() - t0) * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--points", type=int, default=1_000_000)
    ap.add_argument("--frames", type=int, default=128)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "needs a CUDA device"
    L = cb.lib()
    assert b"cusim" not in L.cldn_b200_version(), "refusing the cusim test emulation"
    res = {"gpu": _gpu_state(), "steps": a.steps}
    one_info, one = synth.cloud_c2(a.points, seed=2)
    rng = np.random.default_rng(9)
    batch = []
    for k in range(a.frames):
        viz_info, cloud = synth.cloud_viz(int(rng.integers(100_000, 300_001)), seed=1000 + k)
        batch.append(cloud)
    for name, info, clouds in (("one_xyzi_frame", one_info, [one]), ("viz_batch", viz_info, batch)):
        for comp in (cb.CompressionOption.NONE, cb.CompressionOption.ZSTD):
            res[f"{name}_{comp.name.lower()}"] = _case(L, info, clouds, comp, a.steps, a.warmup)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
