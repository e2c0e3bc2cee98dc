"""Device-resident viz preprocessing + encode of clouds of different sizes, the producer side of tools/blobs_bench.py:
cldn_b200_viz_lossy_preprocess_batch + cldn_b200_encode_blobs against the per-frame loop (viz call, set_dims, encode:
the only way to make such blobs without them), and a uniform cldn_b200_encode_batch of the same total points.

The frames are 128 XYZI clouds of 100k..300k points (synth.cloud_viz, which drops a different number of points from
every frame), encoded without stage 2. Before timing, the loop's and the batch's blobs are checked to be byte-identical.
Prints one JSON line; times are medians of --steps runs, wall clock around synchronous calls.

    python tools/encode_blobs_bench.py [--frames 128] [--steps 20] [--warmup 3]
"""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import cloudini_b200 as cb  # noqa: E402
from cloudini_b200 import synth  # noqa: E402
from cloudini_b200.ros import VizPreprocessor  # noqa: E402
from blobs_bench import _gpu_state, _median_ms  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=128)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    import torch
    assert b"cusim" not in cb.lib().cldn_b200_version(), "refusing the cusim test emulation"
    rng = np.random.default_rng(9)
    clouds = []
    for k in range(a.frames):
        info, cloud = synth.cloud_viz(int(rng.integers(100_000, 300_001)), seed=1000 + k)
        clouds.append(cloud)
    n = len(clouds)
    step = info.point_step
    pts = [c.size // step for c in clouds]
    d_in = [torch.from_numpy(c).cuda() for c in clouds]
    d_mid = [torch.zeros(c.size, dtype=torch.uint8, device="cuda") for c in clouds]
    pp = VizPreprocessor()
    res0 = pp.run_batch_device(info, [t.data_ptr() for t in d_in], [c.size for c in clouds], [t.data_ptr() for t in d_mid],
                               [c.size for c in clouds])
    enc_info = res0[0][0]
    caps = [cb.MaxCompressedSize(enc_info, p, False) + 4096 for p in pts]   # any survivor count, with its header
    d_out_a = [torch.zeros(c, dtype=torch.uint8, device="cuda") for c in caps]
    d_out_b = [torch.zeros(c, dtype=torch.uint8, device="cuda") for c in caps]
    torch.cuda.synchronize()
    enc_a, enc_b = cb.PointcloudEncoder(enc_info), cb.PointcloudEncoder(enc_info)
    L = cb.lib()
    from cloudini_b200 import ros
    ros._L()
    sizes_a = [0] * n
    sizes_b = []

    def loop_call():
        written = C.c_size_t(0)
        for f in range(n):
            _, kept, applied = pp.run_device(info, d_in[f].data_ptr(), clouds[f].size, d_mid[f].data_ptr(), clouds[f].size)
            assert applied
            assert L.cldn_b200_encoder_set_dims(enc_a._h, kept, 1) == 0
            assert L.cldn_b200_encode(enc_a._h, d_mid[f].data_ptr(), kept * step, d_out_a[f].data_ptr(), caps[f], 1,
                                      C.byref(written), 1) == 0
            sizes_a[f] = written.value

    in_args = ([t.data_ptr() for t in d_in], [c.size for c in clouds], [t.data_ptr() for t in d_mid], [c.size for c in clouds])
    out_ptrs = [t.data_ptr() for t in d_out_b]

    def batch_call():
        res = pp.run_batch_device(info, *in_args)
        sizes_b[:] = enc_b.encode_blobs_device(in_args[2], [k * step for _, k, _ in res], out_ptrs, caps)

    loop_call()
    batch_call()
    assert sizes_a == sizes_b, "blob sizes differ between the per-frame loop and the batch calls"
    assert all(torch.equal(x[:s], y[:s]) for x, y, s in zip(d_out_a, d_out_b, sizes_a)), "blobs differ between the loop and the batch"
    kept = [k for _, k, _ in pp.run_batch_device(info, *in_args)]

    # uniform encode_batch: n equal frames holding the same total survivors (the largest frame's first m), no viz step
    m = sum(kept) // n
    u_info = cb.EncodingInfo(**{**enc_info.__dict__, "width": m})
    u_src = d_mid[int(np.argmax(kept))][:m * step]
    u_cap = cb.MaxCompressedSize(u_info, m, True)
    u_out = [torch.zeros(u_cap, dtype=torch.uint8, device="cuda") for _ in range(n)]
    enc_c = cb.PointcloudEncoder(u_info)
    u_args = enc_c.make_device_batch([u_src.data_ptr()] * n, [m * step] * n, [t.data_ptr() for t in u_out], [u_cap] * n)

    def uniform_call():
        enc_c.encode_batch_device(u_args, write_header=True, want_sizes=True)

    total = sum(pts)
    res = {"frames": n, "points_in_total": total, "points_in_min": min(pts), "points_in_max": max(pts), "points_kept_total": sum(kept),
           "point_step": step, "gpu": _gpu_state()}
    for name, fn, p in (("per_frame_loop", loop_call, total), ("viz_batch_plus_encode_blobs", batch_call, total),
                        ("uniform_encode_batch", uniform_call, m * n)):
        before = cb.kernel_launch_count()
        fn()
        launches = cb.kernel_launch_count() - before
        ms = _median_ms(fn, a.steps, a.warmup)
        res[name] = {"ms": round(ms, 3), "gpoints_per_s": round(p / ms / 1e6, 3), "launches": launches}
    res["uniform_encode_batch"]["note"] = "encode only, survivors already in place, equal frames"
    print(json.dumps(res))


if __name__ == "__main__":
    main()
