"""Device-resident clouds of different sizes encoded without the host: cldn_b200_encode_blobs_async (and a CUDA graph that
captured it) against cldn_b200_encode_blobs(CLDN_MEM_DEVICE, written) and a uniform cldn_b200_encode_batch of the same
total points.

The workload of tools/blobs_async_bench.py: 128 XYZI clouds of 100k..300k points after the viz preprocessor (which drops a
different number of points from every frame), encoded without stage 2, with the device LZ4 coder and with the device
ZSTD coder. Every blob is checked byte for byte against encode_blobs before anything is timed. Times are medians of
--steps rounds, wall clock around a synchronise; the calls take turns inside every round. Prints one JSON line.

    python tools/encode_blobs_async_bench.py [--frames 128] [--steps 20] [--warmup 3]
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


def _gpu_state():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # reporting only
        return f"unavailable: {e}"


def _workload(frames):
    rng = np.random.default_rng(9)
    pp = VizPreprocessor()
    out = []
    for k in range(frames):
        info, cloud = synth.cloud_viz(int(rng.integers(100_000, 300_001)), seed=1000 + k)
        new_info, data, applied = pp.run(info, cloud)
        assert applied
        out.append((new_info, np.ascontiguousarray(data)))
    return out


def _encoder(info, comp, stream=0):
    info.compression_opt = comp
    info.width, info.height = 0, 1
    enc = cb.PointcloudEncoder(info, stream=stream)
    if comp != cb.CompressionOption.NONE:
        enc.set_stage2_on_device(True)
    return enc


def _run(comp, work, steps, warmup):
    import torch
    n = len(work)
    info = work[0][0]
    step = info.point_step
    pts = [d.size // step for _, d in work]
    s = torch.cuda.Stream()
    enc = _encoder(info, comp, s.cuda_stream)
    ref = _encoder(info, comp)
    L = cb.lib()
    d_in = [torch.from_numpy(d).cuda() for _, d in work]
    caps = [cb.MaxCompressedSize(_with(info, comp, p), p, True) for p in pts]
    r_out = [torch.zeros(c, dtype=torch.uint8, device="cuda") for c in caps]
    a_out = [torch.zeros(c, dtype=torch.uint8, device="cuda") for c in caps]
    a_in = (C.c_void_p * n)(*[t.data_ptr() for t in d_in])
    a_inb = (C.c_size_t * n)(*[d.size for _, d in work])
    a_out_p = (C.c_void_p * n)(*[t.data_ptr() for t in r_out])
    a_cap = (C.c_size_t * n)(*caps)
    written_host = (C.c_size_t * n)()
    desc = cb.pack_cloud_descs([(t.data_ptr(), d.size, o.data_ptr(), c) for t, (_, d), o, c in zip(d_in, work, a_out, caps)])
    d_status = torch.zeros(n, dtype=torch.int32, device="cuda")
    d_written = torch.zeros(n, dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    enc.prepare_blobs(n, max(pts))

    def blobs_call():
        assert L.cldn_b200_encode_blobs(ref._h, n, a_in, a_inb, None, None, a_out_p, a_cap, written_host, 1) == 0

    def async_call():
        enc.encode_blobs_async(desc.data_ptr(), n, d_status.data_ptr(), d_written.data_ptr())
        s.synchronize()

    def same():
        w = d_written.cpu().tolist()
        return d_status.cpu().tolist() == [0] * n and all(
            w[f] == written_host[f] and torch.equal(a_out[f][:w[f]], r_out[f][:w[f]]) for f in range(n))

    # blobs first: the async call against encode_blobs, byte for byte
    blobs_call()
    async_call()
    assert same(), "encode_blobs_async differs from encode_blobs"
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        enc.encode_blobs_async(desc.data_ptr(), n, d_status.data_ptr(), d_written.data_ptr())
    for t in a_out:
        t.zero_()
    d_status.fill_(99)
    torch.cuda.synchronize()
    g.replay()
    torch.cuda.synchronize()
    assert same(), "the graph replay differs from encode_blobs"

    def graph_call():
        g.replay()
        torch.cuda.synchronize()

    # uniform batch: the same total points in n equal frames of the first cloud's kind
    m = sum(pts) // n
    u_info, u_cloud = synth.cloud_viz(m * 2, seed=7)
    u_info, u_data, _ = VizPreprocessor().run(u_info, u_cloud)
    u_data = np.ascontiguousarray(u_data[:m * step])
    uenc = _encoder(u_info, comp)
    u_cap = cb.MaxCompressedSize(_with(u_info, comp, m), m, True)
    u_in = torch.from_numpy(u_data).cuda()
    u_out = [torch.zeros(u_cap, dtype=torch.uint8, device="cuda") for _ in range(n)]
    torch.cuda.synchronize()
    batch = uenc.make_device_batch([u_in.data_ptr()] * n, [u_data.size] * n, [t.data_ptr() for t in u_out], [u_cap] * n)

    def uniform_call():
        uenc.encode_batch_device(batch, want_sizes=True)

    uniform_call()

    calls = {"encode_blobs": blobs_call, "encode_blobs_async": async_call, "graph_replay": graph_call, "uniform_encode_batch": uniform_call}
    launches = {}
    for name, fn in calls.items():
        before = cb.kernel_launch_count()
        fn()
        launches[name] = cb.kernel_launch_count() - before
    launches["graph_replay"] = launches["encode_blobs_async"]   # the captured kernels (a replay launches through the graph)
    for _ in range(warmup):
        for fn in calls.values():
            fn()
    times = {k: [] for k in calls}
    for r in range(steps):
        names = list(calls)
        for name in names[r % len(names):] + names[:r % len(names)]:   # rotate who goes first
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            calls[name]()
            torch.cuda.synchronize()
            times[name].append((time.perf_counter() - t0) * 1e3)
    total = sum(pts)
    out = {"points_total": total, "points_min": min(pts), "points_max": max(pts)}
    for name in calls:
        ms = float(np.median(times[name]))
        p = m * n if name == "uniform_encode_batch" else total
        out[name] = {"ms": round(ms, 3), "gpoints_per_s": round(p / ms / 1e6, 3), "launches": launches[name]}
    return out


def _with(info, comp, points):
    return cb.EncodingInfo(**{**info.__dict__, "fields": list(info.fields), "width": int(points), "height": 1, "compression_opt": comp})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=128)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    assert a.steps >= 20, "medians of at least 20 rounds"
    assert b"cusim" not in cb.lib().cldn_b200_version(), "refusing the cusim test emulation"
    work = _workload(a.frames)
    res = {"frames": a.frames, "gpu": _gpu_state()}
    for name, comp in (("none", cb.CompressionOption.NONE), ("lz4", cb.CompressionOption.LZ4), ("zstd", cb.CompressionOption.ZSTD)):
        res[name] = _run(comp, work, a.steps, a.warmup)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
