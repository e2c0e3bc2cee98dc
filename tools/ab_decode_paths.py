"""A/B of the decoders for plans that the terminator ranking cannot handle (raw / XOR / Gorilla fields in the stream):
parallel boundary search (decode_mixed_kernel / decode_gorilla_kernel) vs the per-chunk parser (decode_sequential_kernel),
single cloud (latency) and a batch (throughput). Development / reporting aid; prints one JSON line per case."""
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

import cloudini_b200 as cb  # noqa: E402
from cloudini_b200 import synth  # noqa: E402


def run(name, info, clouds, reps=10):
    n, step, F = info.width, info.point_step, len(clouds)
    enc = cb.PointcloudEncoder(info)
    cap = cb.MaxCompressedSize(info, n, True)
    d_in = [torch.from_numpy(c).cuda() for c in clouds]
    d_blob = [torch.empty(cap, dtype=torch.uint8, device="cuda") for _ in range(F)]
    d_out = [torch.zeros(n * step, dtype=torch.uint8, device="cuda") for _ in range(F)]
    eb = enc.make_device_batch([t.data_ptr() for t in d_in], [n * step] * F, [t.data_ptr() for t in d_blob], [cap] * F)
    sizes = enc.encode_batch_device(eb, True, want_sizes=True)
    hdr = len(enc.getHeader())
    res = {"case": name, "frames": F, "points": n, "point_step": step, "stage1_B_per_pt": (float(np.mean(sizes)) - hdr) / n}
    enc.encode_batch_device(eb, True)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        enc.encode_batch_device(eb, True)
    enc.sync()
    res["encode_ms"] = (time.perf_counter() - t0) / reps * 1e3
    outs = {}
    for mode in ("par", "seq"):
        os.environ["CLDN_B200_MIXED_DECODE"] = mode
        dec = cb.PointcloudDecoder()
        db = dec.make_device_batch([t.data_ptr() + hdr for t in d_blob], [x - hdr for x in sizes], [t.data_ptr() for t in d_out], [n * step] * F)
        dec.decode_batch_device(info, db, sync=True)
        outs[mode] = d_out[0].cpu().numpy().copy()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(reps):
            dec.decode_batch_device(info, db, sync=False)
        dec.sync()
        res[f"decode_{mode}_ms"] = (time.perf_counter() - t0) / reps * 1e3
    res["modes_agree"] = bool(np.array_equal(outs["par"], outs["seq"]))
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    for n, F in ((64_000, 1), (1_000_000, 1), (130_048, 64), (130_048, 512)):
        info, _ = synth.cloud_livox(n)
        run(f"livox (uint8 raw fields) {n} x{F}", info, [synth.cloud_livox(n, seed=k)[1] for k in range(min(F, 16))] * (F // min(F, 16)))
        info, _ = synth.cloud_lossless(n, lossless=False)
        run(f"dds layout (f64 Gorilla timestamp) {n} x{F}", info, [synth.cloud_lossless(n, seed=k, lossless=False)[1] for k in range(min(F, 16))] * (F // min(F, 16)))
