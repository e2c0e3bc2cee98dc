"""Device-resident blobs of different sizes without the host: cldn_b200_decode_blobs_async (and a CUDA graph that
captured it) against cldn_b200_decode_blobs and a uniform cldn_b200_decode_batch of the same total points.

The workload of tools/blobs_bench.py: 128 XYZI clouds of 100k..300k points after the viz preprocessor (which drops a
different number of points from every frame), encoded without stage 2 and with ZSTD. Every output is checked byte for
byte before anything is timed. Times are medians of --steps rounds, wall clock around a synchronise; the calls take
turns inside every round. Prints one JSON line.

    python tools/blobs_async_bench.py [--frames 128] [--steps 20] [--warmup 3]
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


def _workload(frames, comp):
    rng = np.random.default_rng(9)
    pp = VizPreprocessor()
    blobs = []
    for k in range(frames):
        info, cloud = synth.cloud_viz(int(rng.integers(100_000, 300_001)), seed=1000 + k)
        new_info, data, applied = pp.run(info, cloud)
        assert applied
        new_info.compression_opt = comp
        blobs.append(cb.PointcloudEncoder(new_info).encode(data))
    return blobs


def _run(comp, frames, steps, warmup):
    import torch
    blobs = _workload(frames, comp)
    n = len(blobs)
    infos = [cb.DecodeHeader(b)[0] for b in blobs]
    pts = [i.width * i.height for i in infos]
    step = infos[0].point_step
    s = torch.cuda.Stream()
    dec = cb.PointcloudDecoder(stream=s.cuda_stream)
    ref = cb.PointcloudDecoder()
    L = cb.lib()
    d_blobs = [torch.from_numpy(np.frombuffer(b, dtype=np.uint8).copy()).cuda() for b in blobs]
    d_outs = [torch.zeros(p * step, dtype=torch.uint8, device="cuda") for p in pts]
    a_outs = [torch.zeros(p * step, dtype=torch.uint8, device="cuda") for p in pts]
    a_in = (C.c_void_p * n)(*[t.data_ptr() for t in d_blobs])
    a_inb = (C.c_size_t * n)(*[len(b) for b in blobs])
    a_out = (C.c_void_p * n)(*[t.data_ptr() for t in d_outs])
    a_cap = (C.c_size_t * n)(*[p * step for p in pts])
    status = (C.c_int32 * n)()
    desc = cb.pack_blob_descs([(t.data_ptr(), len(b), o.data_ptr(), p * step) for t, b, o, p in zip(d_blobs, blobs, a_outs, pts)])
    d_status = torch.zeros(n, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    dec.prepare_blobs(infos[0], n, max(pts))

    def blobs_call():
        assert L.cldn_b200_decode_blobs(ref._h, n, a_in, a_inb, a_out, a_cap, 1, status, None) == 0

    def async_call():
        dec.decode_blobs_async(desc.data_ptr(), n, d_status.data_ptr())
        s.synchronize()

    # outputs first: the async call against decode_blobs, byte for byte
    blobs_call()
    async_call()
    assert d_status.cpu().tolist() == [0] * n
    assert all(torch.equal(x, y) for x, y in zip(d_outs, a_outs)), "decode_blobs_async differs from decode_blobs"
    with torch.cuda.stream(s):
        dec.decode_blobs_async(desc.data_ptr(), n, d_status.data_ptr())
    s.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        dec.decode_blobs_async(desc.data_ptr(), n, d_status.data_ptr())
    for t in a_outs:
        t.zero_()
    d_status.fill_(99)
    torch.cuda.synchronize()
    g.replay()
    torch.cuda.synchronize()
    assert d_status.cpu().tolist() == [0] * n
    assert all(torch.equal(x, y) for x, y in zip(d_outs, a_outs)), "the graph replay differs from decode_blobs"

    def graph_call():
        g.replay()
        torch.cuda.synchronize()

    # uniform batch: the same total points in n equal frames of the same kind of cloud (stage 1 only, as decode_batch takes
    # header-less payloads; a ZSTD uniform batch includes its stage 2)
    m = sum(pts) // n
    pp = VizPreprocessor()
    info_u, cloud_u = synth.cloud_viz(m * 2, seed=7)
    new_u, data_u, _ = pp.run(info_u, cloud_u)
    data_u = data_u[:m * step]
    new_u.width, new_u.height, new_u.compression_opt = m, 1, comp
    u_blob = cb.PointcloudEncoder(new_u).encode(data_u)
    u_info, u_h = cb.DecodeHeader(u_blob)
    u_in = [torch.from_numpy(np.frombuffer(u_blob[u_h:], dtype=np.uint8).copy()).cuda() for _ in range(n)]
    u_out = [torch.zeros(m * step, dtype=torch.uint8, device="cuda") for _ in range(n)]
    torch.cuda.synchronize()
    batch = ref.make_device_batch([t.data_ptr() for t in u_in], [len(u_blob) - u_h] * n, [t.data_ptr() for t in u_out], [m * step] * n)

    def uniform_call():
        ref.decode_batch_device(u_info, batch, sync=True)

    uniform_call()
    want_u = torch.from_numpy(cb.PointcloudDecoder().decode(u_info, u_blob[u_h:])).cuda()
    assert all(torch.equal(t, want_u) for t in u_out), "decode_batch differs from the host-pointer decode"

    calls = {"decode_blobs": blobs_call, "decode_blobs_async": async_call, "graph_replay": graph_call, "uniform_decode_batch": uniform_call}
    launches = {}
    for name, fn in calls.items():
        before = cb.kernel_launch_count()
        fn()
        launches[name] = cb.kernel_launch_count() - before
    launches["graph_replay"] = launches["decode_blobs_async"]   # the captured kernels (a replay launches through the graph)
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
        p = m * n if name == "uniform_decode_batch" else total
        out[name] = {"ms": round(ms, 3), "gpoints_per_s": round(p / ms / 1e6, 3), "launches": launches[name]}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=128)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    assert a.steps >= 20, "medians of at least 20 rounds"
    assert b"cusim" not in cb.lib().cldn_b200_version(), "refusing the cusim test emulation"
    res = {"frames": a.frames, "gpu": _gpu_state()}
    for name, comp in (("none", cb.CompressionOption.NONE), ("zstd", cb.CompressionOption.ZSTD)):
        res[name] = _run(comp, a.frames, a.steps, a.warmup)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
