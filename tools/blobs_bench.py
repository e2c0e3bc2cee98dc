"""Device-resident decode of frames of different sizes: cldn_b200_decode_blobs against the per-frame cldn_b200_decode loop
(the only way to decode such frames without it) and against a uniform cldn_b200_decode_batch of the same total points.

The frames are 128 XYZI clouds of 100k..300k points after the viz preprocessor (which drops a different number of points
from every frame), encoded without stage 2. Prints one JSON line; times are medians of --steps runs, wall clock around
synchronous calls.

    python tools/blobs_bench.py [--frames 128] [--steps 20] [--warmup 3]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import cloudini_b200 as cb  # noqa: E402
from cloudini_b200 import synth  # noqa: E402
from cloudini_b200.ros import VizPreprocessor  # noqa: E402


def _median_ms(fn, steps, warmup):
    import torch
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(steps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(ts))


def _gpu_state():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        return q
    except Exception as e:  # reporting only
        return f"unavailable: {e}"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=128)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    import torch
    assert b"cusim" not in cb.lib().cldn_b200_version(), "refusing the cusim test emulation"
    rng = np.random.default_rng(9)
    pp = VizPreprocessor()
    blobs, infos = [], []
    for k in range(a.frames):
        info, cloud = synth.cloud_viz(int(rng.integers(100_000, 300_001)), seed=1000 + k)
        new_info, data, applied = pp.run(info, cloud)
        assert applied
        new_info.compression_opt = cb.CompressionOption.NONE
        blob = cb.PointcloudEncoder(new_info).encode(data)
        blobs.append(blob)
        infos.append(cb.DecodeHeader(blob))
    n = len(blobs)
    pts = [i.width * i.height for i, _ in infos]
    step = infos[0][0].point_step
    d_blobs = [torch.from_numpy(np.frombuffer(b, dtype=np.uint8).copy()).cuda() for b in blobs]
    d_outs = [torch.zeros(p * step, dtype=torch.uint8, device="cuda") for p in pts]
    torch.cuda.synchronize()
    dec = cb.PointcloudDecoder()
    L = cb.lib()
    a_in = (C.c_void_p * n)(*[t.data_ptr() for t in d_blobs])
    a_inb = (C.c_size_t * n)(*[len(b) for b in blobs])
    a_out = (C.c_void_p * n)(*[t.data_ptr() for t in d_outs])
    a_cap = (C.c_size_t * n)(*[p * step for p in pts])
    status = (C.c_int32 * n)()

    def blobs_call():
        assert L.cldn_b200_decode_blobs(dec._h, n, a_in, a_inb, a_out, a_cap, 1, status, None) == 0

    c_infos = [cb._to_c(i) for i, _ in infos]

    def loop_call():
        for f in range(n):
            h = infos[f][1]
            assert L.cldn_b200_decode(dec._h, C.byref(c_infos[f]), d_blobs[f].data_ptr() + h, len(blobs[f]) - h,
                                      d_outs[f].data_ptr(), pts[f] * step, 1) == 0

    blobs_call()
    want = [t.cpu().numpy().copy() for t in d_outs]
    for t in d_outs:
        t.zero_()
    loop_call()
    assert all(np.array_equal(w, t.cpu().numpy()) for w, t in zip(want, d_outs)), "decode_blobs differs from the per-frame decode"

    # uniform batch: the same total points in n equal frames of the same kind of cloud
    m = sum(pts) // n
    info_u, cloud_u = synth.cloud_viz(m * 2, seed=7)
    new_u, data_u, _ = pp.run(info_u, cloud_u)
    data_u = data_u[:m * step]
    new_u.width, new_u.height, new_u.compression_opt = m, 1, cb.CompressionOption.NONE
    u_blob = cb.PointcloudEncoder(new_u).encode(data_u)
    u_info, u_h = cb.DecodeHeader(u_blob)
    u_in = [torch.from_numpy(np.frombuffer(u_blob[u_h:], dtype=np.uint8).copy()).cuda() for _ in range(n)]
    u_out = [torch.zeros(m * step, dtype=torch.uint8, device="cuda") for _ in range(n)]
    torch.cuda.synchronize()
    batch = dec.make_device_batch([t.data_ptr() for t in u_in], [len(u_blob) - u_h] * n, [t.data_ptr() for t in u_out], [m * step] * n)

    def uniform_call():
        dec.decode_batch_device(u_info, batch, sync=True)

    total = sum(pts)
    res = {"frames": n, "points_total": total, "points_min": min(pts), "points_max": max(pts), "point_step": step,
           "gpu": _gpu_state()}
    for name, fn, p in (("decode_blobs", blobs_call, total), ("per_frame_decode", loop_call, total), ("uniform_decode_batch", uniform_call, m * n)):
        before = cb.kernel_launch_count()
        fn()
        launches = cb.kernel_launch_count() - before
        ms = _median_ms(fn, a.steps, a.warmup)
        res[name] = {"ms": round(ms, 3), "gpoints_per_s": round(p / ms / 1e6, 3), "launches": launches}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
