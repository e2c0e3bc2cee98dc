"""Device-resident clouds of four layouts, interleaved, into complete blobs: cldn_b200_encode_mixed_blobs (one call)
against one encoder per layout with cldn_b200_encode_blobs (one call, one synchronisation and one size read-back per
layout) and against the per-frame loop (set_dims + encode, one synchronisation per frame).

The frames are 128 clouds of 100k..300k points from cloudini_b200.synth, cycling XYZI (step 16), XYZ (step 12), C3
(padded step 32, V5 sections) and XYZIRT (step 22), for NONE and LZ4, into device blobs (CLDN_MEM_DEVICE) and host blobs
(CLDN_MEM_DEVICE_POINTS). Before timing, the three ways' blobs are checked to be byte-identical. Times are medians of
--steps rounds, the three ways alternating inside each round, wall clock around synchronous calls. Prints one JSON line
per (compression, memory kind) and the GPU's name, power limit and SM clock read in the same run.

    python tools/encode_mixed_bench.py [--frames 128] [--steps 20] [--warmup 3]
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

LAYOUTS = ["xyzi", "xyz", "c3", "xyzirt"]


def _cloud(name, n, seed):
    if name == "xyzi":
        info, cloud = synth.cloud_c2(n, seed=seed)
    elif name == "xyz":
        info, cloud = synth.cloud_c1(n, seed=seed)
    elif name == "c3":
        info, cloud = synth.cloud_c3(n, seed=seed)
    else:
        info, cloud = synth.cloud_c4_mixed_frame(1, seed=seed, az=(n + 63) // 64)
    info.width, info.height = 0, 0
    return info, np.ascontiguousarray(cloud[:n * info.point_step])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=128)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    import torch
    assert b"cusim" not in cb.lib().cldn_b200_version(), "refusing the cusim test emulation"
    rng = np.random.default_rng(11)
    frames = [_cloud(LAYOUTS[k % 4], int(rng.integers(100_000, 300_001)), 500 + k) for k in range(a.frames)]
    n = len(frames)
    d_in = [torch.from_numpy(c).cuda() for _, c in frames]
    torch.cuda.synchronize()
    in_ptrs, in_bytes = [t.data_ptr() for t in d_in], [c.size for _, c in frames]
    gpu = _gpu_state()
    for comp in (cb.CompressionOption.NONE, cb.CompressionOption.LZ4):
        infos = []
        for info, _ in frames:
            info = cb.EncodingInfo(**{**info.__dict__, "fields": list(info.fields)})
            info.compression_opt = comp
            infos.append(info)
        caps = [cb.MaxCompressedSize(cb.EncodingInfo(**{**i.__dict__, "fields": list(i.fields), "width": b // i.point_step, "height": 1}),
                                     b // i.point_step, True) for i, b in zip(infos, in_bytes)]
        groups = [list(range(k, n, 4)) for k in range(4)]
        for mem in (cb.MEM_DEVICE, cb.MEM_DEVICE_POINTS):
            device_out = mem == cb.MEM_DEVICE
            outs = {}
            for way in ("mixed", "per_layout", "per_frame"):
                if device_out:
                    bufs = [torch.zeros(c, dtype=torch.uint8, device="cuda") for c in caps]
                    outs[way] = (bufs, [t.data_ptr() for t in bufs])
                else:
                    bufs = [np.zeros(c, dtype=np.uint8) for c in caps]
                    outs[way] = (bufs, [b.ctypes.data for b in bufs])
            torch.cuda.synchronize()
            me = cb.MixedEncoder()
            encs = [cb.PointcloudEncoder(infos[g[0]]) for g in groups]
            sizes = {w: [0] * n for w in outs}
            L = cb.lib()
            # the argument arrays are made once, as a caller that encodes the same topics batch after batch would keep them
            c_infos = (cb._CInfo * n)(*[cb._to_c(i) for i in infos])
            c_mixed = ((C.c_void_p * n)(*in_ptrs), (C.c_size_t * n)(*in_bytes), (C.c_void_p * n)(*outs["mixed"][1]), (C.c_size_t * n)(*caps))

            def mixed():
                st = (C.c_int32 * n)()
                w = (C.c_size_t * n)()
                rc = L.cldn_b200_encode_mixed_blobs(me._h, n, c_infos, *c_mixed, mem, st, w)
                assert rc == 0, L.cldn_b200_last_error()
                sizes["mixed"] = list(w)

            def per_layout():
                p = outs["per_layout"][1]
                for enc, g in zip(encs, groups):
                    m = len(g)
                    w = (C.c_size_t * m)()
                    rc = L.cldn_b200_encode_blobs(enc._h, m, (C.c_void_p * m)(*[in_ptrs[f] for f in g]), (C.c_size_t * m)(*[in_bytes[f] for f in g]),
                                                  None, None, (C.c_void_p * m)(*[p[f] for f in g]), (C.c_size_t * m)(*[caps[f] for f in g]), w, mem)
                    assert rc == 0, L.cldn_b200_last_error()
                    for i, f in enumerate(g):
                        sizes["per_layout"][f] = w[i]

            def per_frame():
                p = outs["per_frame"][1]
                for k, g in enumerate(groups):
                    for f in g:
                        assert L.cldn_b200_encoder_set_dims(encs[k]._h, in_bytes[f] // infos[f].point_step, 1) == 0
                        w = C.c_size_t(0)
                        rc = L.cldn_b200_encode(encs[k]._h, in_ptrs[f], in_bytes[f], p[f], caps[f], 1, C.byref(w), mem)
                        assert rc == 0, L.cldn_b200_last_error()
                        sizes["per_frame"][f] = w.value

            from cloudini_b200 import ros
            ros._L()   # declares cldn_b200_encoder_set_dims
            fns = {"mixed": mixed, "per_layout": per_layout, "per_frame": per_frame}
            launches = {}
            for w, fn in fns.items():
                fn()
                before = cb.kernel_launch_count()
                fn()
                launches[w] = cb.kernel_launch_count() - before
            torch.cuda.synchronize()

            def blob(way, f):
                b = outs[way][0][f]
                return (b[:sizes[way][f]].cpu().numpy() if device_out else b[:sizes[way][f]]).tobytes()
            for f in range(n):
                assert blob("mixed", f) == blob("per_layout", f) == blob("per_frame", f), (comp, mem, f)
            for _ in range(a.warmup):
                for fn in fns.values():
                    fn()
            ts = {w: [] for w in fns}
            order = list(fns)
            for s in range(a.steps):
                for w in order[s % 3:] + order[:s % 3]:
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    fns[w]()
                    torch.cuda.synchronize()
                    ts[w].append((time.perf_counter() - t0) * 1e3)
            print(json.dumps({"compression": comp.name, "mem": "device" if device_out else "device_points", "frames": n,
                              "points": int(sum(in_bytes[f] // infos[f].point_step for f in range(n))),
                              "ms": {w: round(float(np.median(v)), 3) for w, v in ts.items()}, "launches": launches,
                              "blobs_identical": True, "gpu": gpu}), flush=True)
            me.close()
            for e in encs:
                e.close()


if __name__ == "__main__":
    main()
