import sys, os, numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))); sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, 'tests', 'golden'))
import cloudini_b200 as cb
from cloudini_b200 import synth
from oracle.client import RefOracle
from make_golden import int_field_cloud
ref = RefOracle()
rng = np.random.default_rng(int(sys.argv[1]))
trials = int(sys.argv[2])
run_id = np.arange(3000) // 5
cases = {
  "c2_small": synth.cloud_c2(700, seed=1), "c2_3chunks": synth.cloud_c2(70_000, seed=2), "c1": synth.cloud_c1(900, seed=3),
  "c3": synth.cloud_c3(2500, seed=4), "c3_v4": synth.cloud_c3(2500, seed=4, version=4),
  "livox": synth.cloud_livox(1500, seed=5), "livox_v4": synth.cloud_livox(1500, seed=5, version=4),
  "lossless_v3": synth.cloud_lossless(800, seed=6, lossless=True, version=3), "lossless_v5": synth.cloud_lossless(800, seed=6, lossless=True, version=5),
  "c4mixed": synth.cloud_c4_mixed_frame(0, az=40),
  "rle": int_field_cloud(np.random.default_rng(3).integers(0, 2**32, run_id.max()+1, dtype=np.uint64).astype(np.uint32)[run_id], cb.FieldType.UINT32),
  "deltarle_i64": int_field_cloud(np.cumsum(np.random.default_rng(4).integers(-2**40, 2**40, run_id.max()+1)[run_id]).astype(np.int64), cb.FieldType.INT64),
  "delta_u16": int_field_cloud(np.random.default_rng(5).integers(0, 65536, 3000).astype(np.uint16), cb.FieldType.UINT16),
}
only = sys.argv[3].split(",") if len(sys.argv) > 3 else list(cases)
dec = cb.PointcloudDecoder()
total = {"ok_same":0, "both_fail":0, "mismatch":0}
for name in only:
    info, cloud = cases[name]
    blob = ref.encode(info, cloud)
    dinfo, hdr = cb.DecodeHeader(blob)
    n = cloud.size
    modes = [("CLDN_B200_DECODE_MODE", m) for m in ("seq", "tile")] if name.startswith(("c2", "c1")) else [("CLDN_B200_MIXED_DECODE", m) for m in ("par", "seq")]
    mm = 0
    for t in range(trials):
        b = bytearray(blob)
        k = int(rng.integers(0, 4))
        if k == 0:
            for _ in range(int(rng.integers(1, 3))): b[int(rng.integers(hdr, len(b)))] = int(rng.integers(0, 256))
        elif k == 1: b[int(rng.integers(hdr, len(b)))] ^= 1 << int(rng.integers(0, 8))
        elif k == 2: b = b[:int(rng.integers(hdr, len(b)))]
        else:
            i = int(rng.integers(hdr, len(b) - 1)); del b[i:i + int(rng.integers(1, 4))]     # drop bytes: everything behind shifts
        b = bytes(b)
        want = np.full(n, 0x33, np.uint8); rok = True
        try: ref.decode(b, want)
        except RuntimeError: rok = False
        bad = False
        for var, m in modes:
            os.environ[var] = m
            got = np.full(n, 0x33, np.uint8); ook = True
            try:
                if os.environ.get("FUZZ_DEVICE_API"):  # exact-size "device" buffers: with the ASAN emulation an over-read is a report
                    payload = np.frombuffer(b[hdr:], dtype=np.uint8).copy() if len(b) > hdr else np.zeros(1, np.uint8)
                    dec.decode_batch_device(dinfo, dec.make_device_batch([payload.ctypes.data], [len(b) - hdr], [got.ctypes.data], [n]), sync=True)
                else:
                    dec.decode(dinfo, b[hdr:], got)
            except RuntimeError: ook = False
            if ook != rok or (rok and not np.array_equal(got, want)):
                bad = True
                if mm < 3: print("MISMATCH", name, m, "ref_ok", rok, "ours_ok", ook, "kind", k)
        if bad: mm += 1; total["mismatch"] += 1
        elif rok: total["ok_same"] += 1
        else: total["both_fail"] += 1
    print(name, "mismatches", mm, flush=True)
print(total)
