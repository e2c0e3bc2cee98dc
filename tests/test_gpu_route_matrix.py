"""Every layout through every kernel route, at the batch sizes, pointer offsets and field counts that switch kernels.

The codec picks its encode and decode kernels from the layout, the batch's total chunk count (chunk-sequential readers
from SMs + SMs/8 chunks on, a persistent grid of at most 8 CTAs per SM that claims further chunks from a counter), the
uniformity of the frames' chunk counts, pointer alignment and memory kind. Each case here encodes a batch through one
encode API and decodes it through one decode API, under one route (the default selection or one of the switches that
force a kernel), with inputs and outputs placed at a byte offset from a 16-byte boundary:
  * every encode must be byte-identical to the oracle's blob;
  * every decode starts from a pre-filled output with guard bytes around every frame and must equal the oracle's decode.
The product of all dimensions is subsampled with a fixed seed; every (layout, route) pair appears. What the library
reports about the route it took (fast-reader chunks, hand-overs, sections ahead, launches) goes into a ledger, and the
test fails if the default selection never took one of the routes it should take somewhere in the matrix.
"""
import ctypes as C
import functools
import os
import sys

import numpy as np
import pytest

import cloudini_b200 as cb
from cloudini_b200 import synth

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_gpu_encode_blobs import G_BYTE, PAD_BYTE, _Buf  # noqa: E402
from test_gpu_fast_paths import _int_sections_layout  # noqa: E402
from test_gpu_parity import _Dev  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMULATED = bool(os.environ.get("CLDN_B200_LIB"))
F = cb.FieldType
NONE, LZ4, ZSTD = cb.CompressionOption.NONE, cb.CompressionOption.LZ4, cb.CompressionOption.ZSTD
MEM_HOST, MEM_DEVICE = 0, 1
CHUNK = 32768
OFFSETS = (0, 1, 4, 8)
# bytes of decoded points one case may hold: large enough for a 2-chunk frame of every layout on the GPU
BUDGET = (12 << 20) if EMULATED else (160 << 20)


@functools.lru_cache(maxsize=None)
def _sms():
    if EMULATED:
        return int(os.environ.get("CUSIM_SMS", "132"))
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _cross():
    return _sms() + _sms() // 8                 # decode_tiles_sequential: chunk-sequential readers from here on


def _grid_chunks():
    return (3 if EMULATED else 8) * _sms()      # the persistent grid's largest size: one more chunk is a second claim


# name -> the switches it sets; the variables a route does not set are removed
ROUTE_ENV = ("CLDN_B200_DECODE_MODE", "CLDN_B200_DECODE_FAST", "CLDN_B200_DECODE_SIDE", "CLDN_B200_FORCE_CHUNK_DECODE",
             "CLDN_B200_FORCE_GENERIC", "CLDN_B200_ENC_FAST", "CLDN_B200_ZSTD_HOST", "CLDN_B200_MIXED_DECODE")
ROUTES = {
    "default": {},
    "seq": {"CLDN_B200_DECODE_MODE": "seq"},
    "tile": {"CLDN_B200_DECODE_MODE": "tile"},
    "careful": {"CLDN_B200_DECODE_MODE": "seq", "CLDN_B200_DECODE_FAST": "0"},
    "side0": {"CLDN_B200_DECODE_MODE": "seq", "CLDN_B200_DECODE_SIDE": "0"},
    "side1": {"CLDN_B200_DECODE_MODE": "seq", "CLDN_B200_DECODE_SIDE": "1"},
    "chunk": {"CLDN_B200_FORCE_CHUNK_DECODE": "1"},
    "generic": {"CLDN_B200_FORCE_GENERIC": "1"},
    "enc_fast0": {"CLDN_B200_ENC_FAST": "0"},
}
DECODE_APIS = ("decode", "batch_host", "batch_device", "blobs_host", "blobs_device")
ENCODE_APIS = ("encode", "batch_device", "blobs_device")


# ---- layouts ---------------------------------------------------------------------------------------------------------
def _fill(fields, step, n, seed):
    """n points of `step` bytes: plausible values in every field (random walks, palettes, runs), 0xCD padding."""
    rng = np.random.default_rng(seed)
    buf = np.full((n, step), 0xCD, dtype=np.uint8)
    npt = {F.INT8: np.int8, F.UINT8: np.uint8, F.INT16: np.int16, F.UINT16: np.uint16, F.INT32: np.int32, F.UINT32: np.uint32,
           F.FLOAT32: np.float32, F.FLOAT64: np.float64, F.INT64: np.int64, F.UINT64: np.uint64}
    for k, f in enumerate(fields):
        t = npt[f.type]
        if f.type in (F.FLOAT32, F.FLOAT64):
            v = (np.cumsum(rng.normal(0, 0.05, n)) + (1.7e9 if f.type == F.FLOAT64 else 0.0)).astype(t)
            if n > 100:
                v[rng.integers(0, n, 3)] = np.nan
        else:
            kind = k % 3
            if kind == 0:
                v = (np.arange(n) * (k % 5 + 1) + k).astype(t)                       # DeltaRle
            elif kind == 1:
                v = rng.integers(0, 6, n).astype(t)                                   # Palette
            else:
                v = ((np.arange(n) // 97) % 7).astype(t)                              # Rle
        sz = cb.SizeOf(f.type)
        buf[:, f.offset:f.offset + sz] = np.ascontiguousarray(v).view(np.uint8).reshape(n, sz)
    return buf.reshape(-1)


def _info(fields, step, version=5, encoding=cb.EncodingOptions.LOSSY):
    return cb.EncodingInfo(fields=fields, width=0, height=1, point_step=step, encoding_opt=encoding, compression_opt=NONE,
                           use_threads=False, version=version)


def _xyz(o=0, res=0.001):
    return [cb.PointField("x", o, F.FLOAT32, res), cb.PointField("y", o + 4, F.FLOAT32, res), cb.PointField("z", o + 8, F.FLOAT32, res)]


def _named_layouts():
    n = 600 if EMULATED else 4096
    out = [("c1", *synth.cloud_c1(n, seed=1, adversarial=True)),      # NaN / inf / 5-byte varints: the careful redo
           ("c2", *synth.cloud_c2(n, seed=2)),
           ("c3", *synth.cloud_c3(n, seed=3)),
           ("xyzirt", *synth.cloud_c4_mixed_frame(0, az=max(1, n // 64))),
           ("dds_lossy", *synth.cloud_lossless(n, seed=5, lossless=False, stamp_res=None)),
           ("dds_lossless", *synth.cloud_lossless(n, seed=6, lossless=True))]
    fields = [cb.PointField("x", 0, F.FLOAT32, 0.001), cb.PointField("stamp", 4, F.FLOAT64, None), cb.PointField("y", 12, F.FLOAT32, 0.001),
              cb.PointField("z", 16, F.FLOAT32, 0.002), cb.PointField("tag", 20, F.UINT8, None), cb.PointField("stamp2", 21, F.FLOAT64, None)]
    out.append(("two_gorilla", _info(fields, 32), _fill(fields, 32, n, 7)))
    info, cloud = synth.cloud_c2(n, seed=8)
    info.fields.append(cb.PointField("i2", 10, F.FLOAT32, 0.01))           # overlaps z and intensity
    out.append(("overlap", info, cloud))
    info, cloud = synth.cloud_c3(n, seed=9)
    info.encoding_opt = cb.EncodingOptions.NONE
    out.append(("enc_none", info, cloud))
    info, cloud = _int_sections_layout(n, 10, with_u64=True)                 # 4 section fields: side mode's limit
    out.append(("int4", info, cloud))
    info, cloud = _int_sections_layout(n, 11, with_u64=True)
    rows = cloud.reshape(n, 40).copy()
    rows[:, 36:40] = (np.arange(n) // 33 % 9).astype(np.uint32).view(np.uint8).reshape(n, 4)
    info.fields.append(cb.PointField("e", 36, F.UINT32, None))              # 5: sections behind the stream
    out.append(("int5", info, rows.reshape(-1)))
    # Ouster-style: xyz, padding, intensity, t, reflectivity, ring, ambient, padding, range, padding (step 48)
    fields = _xyz() + [cb.PointField("intensity", 16, F.FLOAT32, 0.01), cb.PointField("t", 20, F.UINT32, None),
                       cb.PointField("reflectivity", 24, F.UINT16, None), cb.PointField("ring", 26, F.UINT16, None),
                       cb.PointField("ambient", 28, F.UINT16, None), cb.PointField("range", 32, F.UINT32, None)]
    out.append(("ouster", _info(fields, 48), _fill(fields, 48, n, 12)))
    # Hesai-style: xyz + intensity f32, timestamp f64 without resolution, ring u16 (step 26)
    fields = _xyz() + [cb.PointField("intensity", 12, F.FLOAT32, 0.01), cb.PointField("timestamp", 16, F.FLOAT64, None),
                       cb.PointField("ring", 24, F.UINT16, None)]
    out.append(("hesai", _info(fields, 26), _fill(fields, 26, n, 13)))
    # wide points: fields spread over the whole point, the last one ending at its last byte
    for step in (257, 1000, 4096):
        fields = _xyz(3) + [cb.PointField("intensity", step // 3, F.FLOAT32, 0.01), cb.PointField("ring", step // 2, F.UINT16, None),
                            cb.PointField("stamp", (2 * step) // 3, F.FLOAT64, 1e-6), cb.PointField("tail", step - 4, F.UINT32, None)]
        out.append((f"wide{step}", _info(fields, step), _fill(fields, step, n, step)))
    # 32 fields: the ABI's limit, and 32 op / section slots of the plan
    ints = [F.INT16, F.UINT16, F.INT32, F.UINT32, F.INT64, F.UINT64]
    fields, off = _xyz(), 12
    for k in range(29):
        t = ints[k % len(ints)]
        fields.append(cb.PointField(f"i{k}", off, t, None))
        off += cb.SizeOf(t)
    out.append(("ints29", _info(fields, off), _fill(fields, off, n, 14)))
    fields = [cb.PointField(f"f{k}", 4 * k, F.FLOAT32, 0.001 * (1 + k % 4)) for k in range(32)]
    out.append(("lossy32", _info(fields, 128), _fill(fields, 128, n, 15)))
    fields, off = [], 0
    for k in range(32):
        t = (F.UINT8, F.INT8, F.FLOAT32)[k % 3]
        fields.append(cb.PointField(f"c{k}", off, t, None))
        off += cb.SizeOf(t)
    out.append(("copy32", _info(fields, off), _fill(fields, off, n, 16)))
    return out


def _route_seeds():
    """synth.random_layout_case seeds: CLDN_B200_ROUTE_SEEDS is a count (default 60) or a comma-separated list."""
    v = os.environ.get("CLDN_B200_ROUTE_SEEDS", "60")
    return [int(s) for s in v.split(",")] if "," in v else list(range(int(v)))


def _layouts():
    out = []
    for seed in _route_seeds():
        info, cloud = synth.random_layout_case(seed)
        out.append((f"random{seed}", info, cloud))
    return out + _named_layouts()


def _plan(info):
    """What the planner makes of a layout (cldn_host.cpp build_plan): (floatn_only, fast reader applies, section count)."""
    lossy = info.encoding_opt == cb.EncodingOptions.LOSSY
    lead = 0
    if lossy:
        for f in info.fields:
            if f.type != F.FLOAT32 or f.resolution is None:
                break
            lead += 1
    lead = lead if lead in (3, 4) else 0
    adaptive = (F.INT16, F.UINT16, F.INT32, F.UINT32, F.INT64, F.UINT64)
    v5 = info.version >= 5 and lossy and any(f.type in adaptive for f in info.fields[lead:])
    if not v5 and info.encoding_opt == cb.EncodingOptions.NONE:
        return False, False, 0
    rest = [f for f in info.fields[lead:] if not (v5 and f.type in adaptive)]
    sections = len(info.fields) - lead - len(rest)
    floatn_only = lead > 0 and not rest
    scalar = all(f.type == F.FLOAT32 and f.resolution is not None and lossy for f in rest)
    regular = sorted((f.offset, f.offset + cb.SizeOf(f.type)) for f in info.fields[:lead] + rest)
    overlap = any(b[0] < a[1] for a, b in zip(regular, regular[1:]))     # such plans go to the per-chunk parser
    fast = scalar and not overlap and 3 <= lead + len(rest) <= 6
    return floatn_only, fast, sections


def _padded(info):
    cover = np.zeros(info.point_step, dtype=bool)
    for f in info.fields:
        cover[f.offset:f.offset + cb.SizeOf(f.type)] = True
    return not cover.all()


class _Layout:
    def __init__(self, name, info, cloud, oracle):
        self.name, self.step = name, info.point_step
        self.family = "random" if name.startswith("random") else name
        self.info = cb.EncodingInfo(**{**info.__dict__, "fields": list(info.fields), "width": 0, "height": 1, "compression_opt": NONE})
        self.base = np.ascontiguousarray(cloud).reshape(-1)
        self.n0 = self.base.size // self.step
        self.oracle = oracle
        self.floatn_only, self.fast, self.sections = _plan(self.info)
        self.padded = _padded(self.info)
        self._clouds, self._blobs, self._want, self._caps, self._payloads = {}, {}, {}, {}, {}

    def dims(self, k, comp=NONE):
        return cb.EncodingInfo(**{**self.info.__dict__, "fields": list(self.info.fields), "width": int(k), "compression_opt": comp})

    def cloud(self, k, v):
        """k points; variant v starts at another point of the base cloud (a few distinct frames per size)."""
        key = (k, v)
        if key not in self._clouds:
            shift = (v * 7919 % max(self.n0, 1)) * self.step
            self._clouds[key] = np.resize(np.roll(self.base, -shift), k * self.step)
        return self._clouds[key]

    def blob(self, k, v, comp=NONE):
        key = (k, v, comp)
        if key not in self._blobs:
            self._blobs[key] = self.oracle.encode(self.dims(k, comp), self.cloud(k, v))
        return self._blobs[key]

    def cap(self, k):
        if k not in self._caps:
            self._caps[k] = cb.MaxCompressedSize(self.dims(k), k, True)
        return self._caps[k]

    def payload(self, k, v):
        """The blob without its header: what encode_batch writes."""
        if (k, v) not in self._payloads:
            b = self.blob(k, v)
            self._payloads[(k, v)] = b[cb.DecodeHeader(b)[1]:]
        return self._payloads[(k, v)]

    def want(self, k, v):
        """The oracle's decode of the frame onto a PAD_BYTE-filled buffer."""
        key = (k, v)
        if key not in self._want:
            out = np.full(k * self.step, PAD_BYTE, dtype=np.uint8)
            self.oracle.decode(self.blob(k, v), out)
            self._want[key] = out
        return self._want[key]


# ---- batch shapes ----------------------------------------------------------------------------------------------------
def _shape(lay, shape, rng):
    """[(points, variant)] of one batch. 'one': one frame; '<target>_u': every frame one chunk, the same point count;
    '<target>_m': 1- and 2-chunk frames mixed (1, 32767, 32768 and 32769 points) and filled up with small frames."""
    if shape == "one":
        pool = [k for k in (1, 17, 32767, 32768, 32769, lay.n0) if k * lay.step <= BUDGET]
        return [(int(rng.choice(pool)), 0)]
    target = {"below": _cross() - 1, "at": _cross(), "big": _grid_chunks() + 1}[shape[:-2]]
    if shape.endswith("_u"):
        pool = [k for k in (1, 2, 17, 300, min(lay.n0, CHUNK), 32767, 32768) if target * k * lay.step <= BUDGET]
        k = int(rng.choice(pool))
        return [(k, f % 3) for f in range(target)]
    frames, chunks, used = [], 0, 0
    for k in (32769, 1, 32768, 32767):
        c = (k + CHUNK - 1) // CHUNK
        if chunks + c <= target and used + k * lay.step <= BUDGET:
            frames.append((k, len(frames) % 2))
            chunks, used = chunks + c, used + k * lay.step
    small = (1, 2, 17, 300, 5)
    while chunks < target:
        frames.append((small[chunks % len(small)], chunks % 2))
        chunks += 1
    order = rng.permutation(len(frames))
    return [frames[i] for i in order]


def _chunks(frames):
    return sum((k + CHUNK - 1) // CHUNK for k, _ in frames)


# ---- guarded arenas --------------------------------------------------------------------------------------------------
class _Arena:
    """Regions of the given sizes in one guarded buffer (_Buf: guards in front and behind), each starting `off` bytes past
    a 16-byte boundary with at least 16 guard bytes before it; `fills` are the regions' initial contents."""

    def __init__(self, fills, device, off):
        pos, at = 0, []
        for r in fills:
            pos = (pos + 16 + 15) // 16 * 16 + off
            at.append(pos)
            pos += r.size
        total = pos + 16
        img = np.full(total, G_BYTE, dtype=np.uint8)
        for p, r in zip(at, fills):
            img[p:p + r.size] = r
        self.at, self.sizes, self.img, self.device = at, [r.size for r in fills], img, device
        self.buf = _Buf(total, device, src=img.tobytes())
        self.ptrs = [self.buf.ptr + p for p in at]

    def read(self):
        return self.buf.body()

    def guards_intact(self):
        got = self.read()
        mask = np.ones(got.size, dtype=bool)
        for p, s in zip(self.at, self.sizes):
            mask[p:p + s] = False
        return self.buf.guards_intact() and bool((got[mask] == G_BYTE).all())

    def region(self, got, f):
        return got[self.at[f]:self.at[f] + self.sizes[f]]


def _inputs(datas, device, off):
    """Read-only inputs (clouds, blobs, payloads) at `off` bytes past a 16-byte boundary: device memory through _Dev."""
    pos, at = 0, []
    for d in datas:
        pos = (pos + 15) // 16 * 16 + off
        at.append(pos)
        pos += max(d.size, 1)
    img = np.zeros(pos + 16, dtype=np.uint8)
    for p, d in zip(at, datas):
        img[p:p + d.size] = d
    if device:
        keep = _Dev(src=img)
        base = keep.ptr
    else:
        keep = img
        base = img.ctypes.data
    return keep, [base + p for p in at]


def _arr(t, xs):
    return (t * max(len(xs), 1))(*xs)


# ---- one case --------------------------------------------------------------------------------------------------------
def _run_encode(lay, enc, api, frames, device, off_in, off_out):
    L = cb.lib()
    clouds = [lay.cloud(k, v) for k, v in frames]
    expect = [lay.blob(k, v) for k, v in frames]
    caps = [lay.cap(k) for k, _ in frames]
    keep, ins = _inputs(clouds, device, off_in)
    outs = _Arena([np.full(c, PAD_BYTE, dtype=np.uint8) for c in caps], device, off_out)
    mem = MEM_DEVICE if device else MEM_HOST
    n = len(frames)
    written = (C.c_size_t * max(n, 1))()
    if api == "encode":
        assert n == 1
        assert L.cldn_b200_encoder_set_dims(enc._h, frames[0][0], 1) == 0
        w = C.c_size_t(0)
        rc = L.cldn_b200_encode(enc._h, ins[0], clouds[0].size, outs.ptrs[0], caps[0], 1, C.byref(w), mem)
        written[0] = w.value
    elif api == "batch_device":
        rc = L.cldn_b200_encode_batch(enc._h, n, _arr(C.c_void_p, ins), _arr(C.c_size_t, [c.size for c in clouds]),
                                      _arr(C.c_void_p, outs.ptrs), _arr(C.c_size_t, caps), 0, written, mem)
        expect = [lay.payload(k, v) for k, v in frames]
    else:
        rc = L.cldn_b200_encode_blobs(enc._h, n, _arr(C.c_void_p, ins), _arr(C.c_size_t, [c.size for c in clouds]), None, None,
                                      _arr(C.c_void_p, outs.ptrs), _arr(C.c_size_t, caps), written, mem)
    if rc != 0:
        return f"encode {api}: rc {rc}: {L.cldn_b200_last_error().decode()}"
    got = outs.read()
    for f in range(n):
        if written[f] != len(expect[f]) or outs.region(got, f)[:written[f]].tobytes() != expect[f]:
            return f"encode {api}: frame {f} ({frames[f][0]} points) differs from the oracle's blob"
    if not outs.guards_intact():
        return f"encode {api}: a byte outside the frames' buffers changed"
    del keep
    return None


def _run_decode(lay, dec, api, frames, comps, device, off_in, off_out):
    L = cb.lib()
    blobs = [np.frombuffer(lay.blob(k, v, c), dtype=np.uint8) for (k, v), c in zip(frames, comps)]
    wants = [lay.want(k, v) for k, v in frames]
    outs = _Arena([np.full(w.size, PAD_BYTE, dtype=np.uint8) for w in wants], device, off_out)
    mem = MEM_DEVICE if device else MEM_HOST
    n = len(frames)
    if api in ("decode", "batch_host", "batch_device"):
        info, hdr = cb.DecodeHeader(lay.blob(*frames[0]))
        payloads = [b[hdr:] for b in blobs]
        keep, ins = _inputs(payloads, device, off_in)
        c = cb._to_c(info)
        if api == "decode":
            rc = L.cldn_b200_decode(dec._h, C.byref(c), ins[0], payloads[0].size, outs.ptrs[0], outs.sizes[0], mem)
        else:
            rc = L.cldn_b200_decode_batch(dec._h, C.byref(c), n, _arr(C.c_void_p, ins), _arr(C.c_size_t, [p.size for p in payloads]),
                                          _arr(C.c_void_p, outs.ptrs), _arr(C.c_size_t, outs.sizes), mem, 1)
        if rc != 0:
            return f"decode {api}: rc {rc}: {L.cldn_b200_last_error().decode()}"
    else:
        keep, ins = _inputs(blobs, device, off_in)
        status, _ = dec._blobs(n, _arr(C.c_void_p, ins), _arr(C.c_size_t, [b.size for b in blobs]), _arr(C.c_void_p, outs.ptrs),
                               _arr(C.c_size_t, outs.sizes), mem)
        bad = [f for f in range(n) if status[f] != 0]
        if bad:
            return f"decode {api}: frame {bad[0]} status {status[bad[0]]}: {dec.frame_error(bad[0])}"
    got = outs.read()
    for f in range(n):
        if not np.array_equal(outs.region(got, f), wants[f]):
            return f"decode {api}: frame {f} ({frames[f][0]} points, {comps[f].name}) differs from the oracle's decode"
    if not outs.guards_intact():
        return f"decode {api}: a byte outside the frames' outputs changed"
    del keep
    return None


def _plan_cases(layouts, oracle):
    """(layout, route, shape, decode api, encode api, device, offsets, compressions) per case, from a fixed seed."""
    rng = np.random.default_rng(20261017)
    cases = []
    for lay in layouts:
        for route in ROUTES:
            shapes = ["one", f"below_{'um'[int(rng.integers(2))]}", f"at_{'um'[int(rng.integers(2))]}", f"big_{'um'[int(rng.integers(2))]}"] \
                if route == "default" else [str(rng.choice(["one", "below_u", "below_m", "at_u", "at_m"]))]   # the switches force a
                # kernel at a small size; the default selection takes every shape, the persistent grid's second claims included
            for shape in shapes:
                frames = _shape(lay, shape, rng)
                dapis = [a for a in DECODE_APIS if (a != "decode" or shape == "one") and
                         (not a.startswith("batch") or len({k for k, _ in frames}) == 1)]
                eapis = [a for a in ENCODE_APIS if a != "encode" or shape == "one"]
                if route == "default" and _chunks(frames) >= _cross():
                    # the ledger's cases: device memory, decoded in one launch (the host APIs stage a batch in pieces)
                    dapis = [a for a in dapis if a.endswith("device")]
                dapi = str(rng.choice(dapis))
                device = dapi.endswith("device") or (dapi == "decode" and bool(rng.integers(2)))
                comps = [NONE] * len(frames)
                # (decode_blobs decodes each compression as a group of its own: the ledger's default cases above the
                # crossover keep one group, so that what the library reports is the route of the whole batch)
                mixable = not (route == "default" and _chunks(frames) >= _cross())
                if dapi.startswith("blobs") and oracle.kind != "port" and mixable and rng.random() < 0.3:
                    comps = [(NONE, LZ4, ZSTD)[f % 3] for f in range(len(frames))]
                eapi = str(rng.choice(eapis))
                edevice = eapi != "encode" or bool(rng.integers(2))
                if eapi == "batch_device" and rng.random() < 0.3:
                    edevice = False     # the same call with host memory
                offs = [int(rng.choice(OFFSETS)) for _ in range(4)]
                cases.append((lay, route, shape, frames, dapi, device, comps, eapi, edevice, offs))
    return cases


@pytest.fixture(scope="module")
def layouts(oracle):
    out, skipped = [], []
    for name, info, cloud in _layouts():
        lay = _Layout(name, info, cloud, oracle)
        try:
            lay.blob(1, 0)
        except RuntimeError:        # a layout the oracle refuses (as test_random_layouts_sweep skips them)
            skipped.append(name)
            continue
        out.append(lay)
    return out, skipped


@pytest.mark.gpu
def test_route_matrix(oracle, layouts, monkeypatch, capsys):
    from cloudini_b200 import ros
    ros._L()    # binds cldn_b200_encoder_set_dims
    lays, skipped = layouts
    cases = _plan_cases(lays, oracle)
    assert {(c[0].name, c[1]) for c in cases} == {(lay.name, r) for lay in lays for r in ROUTES}
    dec = cb.PointcloudDecoder()
    failures, ledger = [], []
    for lay, route, shape, frames, dapi, device, comps, eapi, edevice, offs in cases:
        for var in ROUTE_ENV:
            monkeypatch.delenv(var, raising=False)
        for var, val in ROUTES[route].items():
            monkeypatch.setenv(var, val)
        where = f"{lay.name} route={route} shape={shape} frames={len(frames)} chunks={_chunks(frames)}"
        # an encoder fixes its tile size when it is made, from the switches then in force: one per case, freed after it
        # (hundreds of handles grown for thousand-frame batches would not fit the device together)
        enc = cb.PointcloudEncoder(lay.dims(1))
        try:
            msg = _run_encode(lay, enc, eapi, frames, edevice, offs[0], offs[1])
            if msg:
                failures.append(f"{where} {'device' if edevice else 'host'} in+{offs[0]} out+{offs[1]}: {msg}")
            launches = cb.kernel_launch_count()
            msg = _run_decode(lay, dec, dapi, frames, comps, device, offs[2], offs[3])
            launches = cb.kernel_launch_count() - launches
            if msg:
                failures.append(f"{where} {'device' if device else 'host'} in+{offs[2]} out+{offs[3]}: {msg}")
            stats, ahead = dec.last_stats(), dec.last_sections_ahead()
        except RuntimeError as e:
            failures.append(f"{where} {dapi}/{eapi}: {e}")
            continue
        finally:
            enc.close()
        one_group = len(set(comps)) == 1
        ledger.append((lay, route, shape, _chunks(frames), dapi, one_group, stats, ahead, launches))
    for var in ROUTE_ENV:
        monkeypatch.delenv(var, raising=False)

    def seen(pred):
        return sum(1 for lay, route, shape, chunks, dapi, one, st, ahead, _ in ledger
                   if route == "default" and one and pred(lay, chunks, st, ahead))
    above = lambda chunks: chunks >= _cross()  # noqa: E731
    required = {
        "fast FloatN reader, random layout": seen(lambda l, ch, st, a: above(ch) and l.family == "random" and l.floatn_only and st[0] > 0),
        "fast general reader": seen(lambda l, ch, st, a: above(ch) and not l.floatn_only and l.fast and st[0] > 0),
        "side mode, padded multi-section layout": seen(lambda l, ch, st, a: above(ch) and a and l.padded and l.sections >= 2),
        "hand-over to the careful kernel": seen(lambda l, ch, st, a: above(ch) and st[1] > 0),
        "tile-parallel below the crossover": seen(lambda l, ch, st, a: 0 < ch < _cross() and l.floatn_only and st[0] == 0),
    }
    with capsys.disabled():
        print(f"\nroute matrix: {len(cases)} cases over {len(lays)} layouts, {len(skipped)} refused by the oracle {skipped}; "
              f"SMs {_sms()}, crossover {_cross()} chunks, persistent grid up to {_grid_chunks()} chunks")
        for route in ROUTES:
            rows = [r for r in ledger if r[1] == route]
            print(f"  {route:9s} cases {len(rows):4d}  fast chunks {sum(r[6][0] for r in rows):7d}  handed over {sum(r[6][1] for r in rows):5d}"
                  f"  sections ahead {sum(1 for r in rows if r[7]):3d}  decode launches {sum(r[8] for r in rows):6d}")
        for what, count in required.items():
            print(f"  default selection, {what}: {count} cases")
        for line in failures[:25]:
            print("  FAILED", line)
    assert not failures, f"{len(failures)} of {len(cases)} cases failed:\n" + "\n".join(failures[:25])
    missing = [what for what, count in required.items() if count == 0]
    assert not missing, f"the default selection never took: {missing}"


# ---- viz compaction shapes -------------------------------------------------------------------------------------------
VIZ_STEPS = (36, 48, 96, 128, 801, 1000, 4096)


def _viz_tile(step):
    """viz_compact_kernel's points per tile (cldn_preproc.cu: 256 threads x 8, 4, 2 or 1 points)."""
    ppt = 8
    while ppt > 1 and 256 * ppt * step > (64 << 10):
        ppt >>= 1
    return 256 * ppt


def _viz_case(step, xo, seed, n):
    info, cloud = synth.cloud_viz(n, seed=seed, step=step)
    rows = cloud.reshape(n, step).copy()
    rows[:, xo:xo + 12] = cloud.reshape(n, step)[:, 0:12]
    info.fields = _xyz(xo)
    return info, rows.reshape(-1)


@pytest.mark.gpu
@pytest.mark.parametrize("step", VIZ_STEPS)
def test_viz_compaction_shapes(oracle, step):
    from cloudini_b200 import ros
    pp = ros.VizPreprocessor()
    tile = _viz_tile(step)
    L = ros._L()
    for xo in (0, 8, step - 12):
        sizes = [tile + 1, 1, 2 * tile + 1, tile - 1, 0, tile]
        clouds = [_viz_case(step, xo, 100 * xo + k, n)[1] for k, n in enumerate(sizes)]
        info = _viz_case(step, xo, 0, 1)[0]
        wants = [oracle.viz_preprocess(info, c) for c in clouds]
        for device, off in ((False, 0), (True, 0), (True, 1), (True, 4)):
            keep, ins = _inputs(clouds, device, off)
            outs = _Arena([np.full(max(c.size, 1), PAD_BYTE, dtype=np.uint8) for c in clouds], device, (off * 3) % 8)
            m = len(clouds)
            kept, applied, infos = (C.c_size_t * m)(), (C.c_int * m)(), (cb._CInfo * m)()
            rc = L.cldn_b200_viz_lossy_preprocess_batch(pp._h, C.byref(cb._to_c(info)), m, _arr(C.c_void_p, ins),
                                                        _arr(C.c_size_t, [c.size for c in clouds]), _arr(C.c_void_p, outs.ptrs),
                                                        _arr(C.c_size_t, outs.sizes), kept, applied, infos, MEM_DEVICE if device else MEM_HOST)
            assert rc == 0, cb.lib().cldn_b200_last_error().decode()
            got = outs.read()
            for f, (c, (o_info, o_out)) in enumerate(zip(clouds, wants)):
                body = outs.region(got, f)
                where = (step, xo, device, off, f, sizes[f])
                if c.size == 0:
                    assert kept[f] == 0 and (body == PAD_BYTE).all(), where
                    continue
                assert applied[f] and kept[f] == o_out.size // step == o_info.width, where
                assert np.array_equal(body[:o_out.size], o_out), where
                assert (body[o_out.size:] == PAD_BYTE).all(), where
            assert outs.guards_intact(), (step, xo, device, off)
            # the single call on the cloud that crosses a tile boundary by one point
            one = _Arena([np.full(clouds[0].size, PAD_BYTE, dtype=np.uint8)], device, off)
            k1, a1 = C.c_size_t(0), C.c_int(0)
            rc = L.cldn_b200_viz_lossy_preprocess(pp._h, C.byref(cb._to_c(info)), C.c_void_p(ins[0]), clouds[0].size,
                                                      C.c_void_p(one.ptrs[0]), clouds[0].size, C.byref(k1), C.byref(a1),
                                                      MEM_DEVICE if device else MEM_HOST)
            assert rc == 0 and a1.value and k1.value == kept[0], (step, xo, device, off)
            g1 = one.read()
            assert np.array_equal(one.region(g1, 0)[:wants[0][1].size], wants[0][1]) and one.guards_intact(), (step, xo, device, off)
            del keep


# ---- the same file under the CPU emulation (not a GPU test: it runs in the CPU suite) -------------------------------
@pytest.mark.skipif(EMULATED, reason="already running under the emulation")
@pytest.mark.parametrize("order,workers", [("fwd", "1"), ("fwd", "8"), ("rand", "1"), ("rand", "8")])
def test_this_file_under_emulation(lib_built, order, workers):
    # 4 SMs: the crossover is 4 chunks and the persistent grid 12, so a small batch reaches every route
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from test_cusim_kernels import _run_gpu_suite
    import platform
    if platform.machine() != "x86_64":
        pytest.skip("cusim's context switch is x86-64 only")
    sys.path.insert(0, os.path.join(ROOT, "tests", "cusim"))
    import build_cusim
    # (seed 36 is a random layout whose regular stream is one FloatN group: the fast FloatN reader's random case)
    env = {"CUSIM_ORDER": order, "CUSIM_WORKERS": workers, "CUSIM_SMS": "4", "CLDN_B200_ROUTE_SEEDS": "0,1,2,3,4,5,6,7,36"}
    if order == "rand":
        env["CUSIM_JITTER"] = "1"
    out = _run_gpu_suite(build_cusim.build(), env, ["-s", "tests/test_gpu_route_matrix.py"])
    assert " passed" in out and "failed" not in out
