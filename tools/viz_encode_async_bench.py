"""The converter step on device-resident clouds, three ways, taking turns inside every round:

  sync    cldn_b200_viz_lossy_preprocess_batch + cldn_b200_encode_blobs(CLDN_MEM_DEVICE, written): the survivor counts
          come back to the host, which builds the encoder's inputs from them;
  async   cldn_b200_viz_lossy_preprocess_batch_async + cldn_b200_encode_blobs_async + one synchronise: the preprocessing
          writes the encoder's descriptors on the device;
  graph   the replay of a CUDA graph that captured the async pair.

The workload of tools/encode_blobs_bench.py: 128 raw viz clouds of 100k..300k points in device memory, encoded without
stage 2 and with the device ZSTD coder. Every blob of async and graph is checked byte for byte against sync before
anything is timed. Times are medians of --steps rounds, wall clock around a synchronise. Prints one JSON line with the
card's name, power limit and SM clock. --profile DIR writes a separate torch.profiler run of sync and async, split by
kernel, to DIR.

    python tools/viz_encode_async_bench.py [--frames 128] [--steps 20] [--warmup 3] [--profile DIR]
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
from cloudini_b200 import ros, synth  # noqa: E402


def _gpu_state():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # reporting only
        return f"unavailable: {e}"


def _run(comp, clouds, info, steps, warmup, profile_dir):
    import torch
    n = len(clouds)
    step = info.point_step
    pts = [c.size // step for c in clouds]
    s = torch.cuda.Stream()
    d_in = [torch.from_numpy(c).cuda() for c in clouds]
    mid_a = [torch.zeros(c.size, dtype=torch.uint8, device="cuda") for c in clouds]
    mid_b = [torch.zeros(c.size, dtype=torch.uint8, device="cuda") for c in clouds]
    pp_a, pp_b = ros.VizPreprocessor(), ros.VizPreprocessor(stream=s.cuda_stream)
    after = pp_b.prepare_batch(info, n, max(pts))
    after.compression_opt = comp
    caps = [cb.MaxCompressedSize(cb.EncodingInfo(**{**after.__dict__, "width": p, "height": 1}), p, True) for p in pts]
    out_a = [torch.zeros(c, dtype=torch.uint8, device="cuda") for c in caps]
    out_b = [torch.zeros(c, dtype=torch.uint8, device="cuda") for c in caps]

    def encoder(stream=0):
        enc = cb.PointcloudEncoder(after, stream=stream)
        if comp != cb.CompressionOption.NONE:
            enc.set_stage2_on_device(True)
        return enc

    enc_a, enc_b = encoder(), encoder(s.cuda_stream)
    enc_b.prepare_blobs(n, max(pts))
    L = cb.lib()
    in_args = ([t.data_ptr() for t in d_in], [c.size for c in clouds], [t.data_ptr() for t in mid_a], [c.size for c in clouds])
    out_p = (C.c_void_p * n)(*[t.data_ptr() for t in out_a])
    mid_p = (C.c_void_p * n)(*in_args[2])
    cap_p = (C.c_size_t * n)(*caps)
    written_a = (C.c_size_t * n)()
    vdesc = ros.pack_viz_descs([(t.data_ptr(), c.size, m.data_ptr(), c.size) for t, c, m in zip(d_in, clouds, mid_b)])
    edesc = cb.pack_cloud_descs([(0, 0, o.data_ptr(), c) for o, c in zip(out_b, caps)])
    v_status, e_status = (torch.zeros(n, dtype=torch.int32, device="cuda") for _ in range(2))
    written_b = torch.zeros(n, dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()

    def sync_call():
        res = pp_a.run_batch_device(info, *in_args)
        kept_bytes = (C.c_size_t * n)(*[k * step for _, k, _ in res])
        assert L.cldn_b200_encode_blobs(enc_a._h, n, mid_p, kept_bytes, None, None, out_p, cap_p, written_a, 1) == 0

    def enqueue():
        pp_b.run_batch_async(vdesc.data_ptr(), n, v_status.data_ptr(), encode_descs_ptr=edesc.data_ptr())
        enc_b.encode_blobs_async(edesc.data_ptr(), n, e_status.data_ptr(), written_b.data_ptr())

    def async_call():
        enqueue()
        s.synchronize()

    def same():
        w = written_b.cpu().tolist()
        return (v_status.cpu().tolist() == [0] * n and e_status.cpu().tolist() == [0] * n
                and all(w[f] == written_a[f] and torch.equal(out_b[f][:w[f]], out_a[f][:w[f]]) for f in range(n)))

    sync_call()
    async_call()
    assert same(), "the async chain differs from the sync chain"
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        enqueue()
    for t in out_b:
        t.zero_()
    e_status.fill_(99)
    torch.cuda.synchronize()
    g.replay()
    torch.cuda.synchronize()
    assert same(), "the graph replay differs from the sync chain"

    def graph_call():
        g.replay()
        torch.cuda.synchronize()

    calls = {"sync": sync_call, "async": async_call, "graph": graph_call}
    launches = {}
    for name, fn in calls.items():
        before = cb.kernel_launch_count()
        fn()
        launches[name] = cb.kernel_launch_count() - before
    launches["graph"] = launches["async"]   # the captured kernels (a replay launches through the graph)
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
        out[name] = {"ms": round(ms, 3), "ms_min": round(min(times[name]), 3), "ms_max": round(max(times[name]), 3),
                     "gpoints_per_s": round(total / ms / 1e6, 3), "launches": launches[name]}
    if profile_dir:
        from torch.profiler import ProfilerActivity, profile
        os.makedirs(profile_dir, exist_ok=True)
        for name in ("sync", "async"):
            with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
                for _ in range(5):
                    calls[name]()
                torch.cuda.synchronize()
            tag = f"{name}_{comp.name.lower()}"
            prof.export_chrome_trace(os.path.join(profile_dir, f"{tag}.json"))
            with open(os.path.join(profile_dir, f"{tag}.txt"), "w") as fh:
                fh.write(prof.key_averages().table(sort_by="cuda_time_total", row_limit=40))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=128)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--profile", default="")
    a = ap.parse_args()
    assert a.steps >= 20, "medians of at least 20 rounds"
    assert b"cusim" not in cb.lib().cldn_b200_version(), "refusing the cusim test emulation"
    rng = np.random.default_rng(9)
    clouds = []
    for k in range(a.frames):
        info, cloud = synth.cloud_viz(int(rng.integers(100_000, 300_001)), seed=1000 + k)
        clouds.append(cloud)
    info.width = 0
    res = {"frames": a.frames, "gpu": _gpu_state()}
    for name, comp in (("none", cb.CompressionOption.NONE), ("zstd", cb.CompressionOption.ZSTD)):
        res[name] = _run(comp, clouds, info, a.steps, a.warmup, a.profile)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
