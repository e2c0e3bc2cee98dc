"""V5 adaptive integer sections against the oracle at every palette width, table path, mode tie and run boundary.

What the section kernels run depends on the values of a field: which of the four modes the probe commits (the first
min(4096, chunk 0) values, strict `<` in the order DeltaVarint, Palette, Rle, DeltaRle), which writer packs it (fields of
2 or 4 bytes: the staged writer; 8 bytes: the in-place writer), which palette table holds it (shared memory up to 2048
distinct values, the global-memory overflow pool above), and how the reader unpacks index units and run-table batches.
The cases here are built to reach each of those shapes on purpose:
  * every blob is byte-equal to the oracle's, and every decode (into a buffer pre-filled with a non-zero byte, so that
    padding is checked too) byte-equal to the oracle's decode; where the oracle refuses, the message must match;
  * a plain model of the probe (written from the wire format) must pick the mode byte the oracle wrote, and the size of
    a whole-chunk probe's section;
  * a parser walks the oracle's blobs into sections, and test_every_listed_shape_is_reached fails if a shape the cases
    were built for never appears.
"""
import functools
import os
import platform
import sys

import numpy as np
import pytest

import cloudini_b200 as cb

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_gpu_parity import _Dev  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMULATED = bool(os.environ.get("CLDN_B200_LIB"))   # tests/cusim: the same shapes on smaller frames
F = cb.FieldType
NONE = cb.CompressionOption.NONE
CHUNK, PROBE, RUN_PAR = 32768, 4096, 256            # points per chunk, probe window, run records per reader batch
SMEM_DISTINCT = 2048                                # the shared-memory palette table's limit
FILL = 0xA7
NP = {F.INT16: np.int16, F.UINT16: np.uint16, F.INT32: np.int32, F.UINT32: np.uint32, F.INT64: np.int64, F.UINT64: np.uint64}
STAGED, IN_PLACE = (F.INT16, F.UINT16, F.INT32, F.UINT32), (F.INT64, F.UINT64)
DELTA, PALETTE, RLE, DRLE = range(4)
MODE_NAMES = ("DeltaVarint", "Palette", "Rle", "DeltaRle")
# The decode switches: the side, fast and careful readers are chunk-sequential, so they are forced with MODE=seq (a
# frame of a few chunks takes the tile-parallel / per-chunk kernels by default)
ROUTES = {"default": {}, "seq": {"CLDN_B200_DECODE_MODE": "seq"},
          "careful": {"CLDN_B200_DECODE_MODE": "seq", "CLDN_B200_DECODE_FAST": "0"},
          "side0": {"CLDN_B200_DECODE_MODE": "seq", "CLDN_B200_DECODE_SIDE": "0"},
          "side1": {"CLDN_B200_DECODE_MODE": "seq", "CLDN_B200_DECODE_SIDE": "1"}}
ROUTE_ENV = ("CLDN_B200_DECODE_SIDE", "CLDN_B200_DECODE_MODE", "CLDN_B200_DECODE_FAST")


def _writer(t):
    return "staged" if t in STAGED else "in-place"


# ---- the model: selectBestAdaptiveIntMode on a probe window ----------------------------------------------------------
def _vlen(u):
    """LEB128 bytes of each uint64."""
    n = np.ones(u.shape, dtype=np.int64)
    for k in range(1, 10):
        n += u >= np.uint64(1 << (7 * k))
    return n


def _zigzag_plus1(d):
    """The varint payload of a signed delta: zigzag, plus one (0 is the NaN marker), wrapping like uint64."""
    with np.errstate(over="ignore"):
        return ((d << np.int64(1)) ^ (d >> np.int64(63))).view(np.uint64) + np.uint64(1)


def _deltas(v):
    """Each value minus its predecessor (0 in front of the first) as int64, wrapping: the field's ToInt64 values."""
    x = v.astype(np.int64).view(np.uint64) if v.dtype != np.uint64 else v
    return np.diff(x, prepend=np.uint64(0)).view(np.int64)


def _raw(v):
    return v.view(np.dtype(f"u{v.itemsize}")).astype(np.uint64)


def _bits(u):
    """bitsForPaletteIndex of each palette size."""
    b = np.zeros(np.shape(u), dtype=np.int64)
    for k in range(16):
        b += np.asarray(u) - 1 >= (1 << k)
    return b


def _prefix_sizes(v):
    """[4, len(v)]: the four section sizes (DeltaVarint, Palette, Rle, DeltaRle) of every prefix v[:n], n = 1..len(v)."""
    n, bpv = len(v), v.itemsize
    idx = np.arange(n)
    d = _deltas(v)
    dl = _vlen(_zigzag_plus1(d))
    raw = _raw(v)
    first = np.zeros(n, dtype=bool)
    first[np.unique(raw, return_index=True)[1]] = True
    u = np.cumsum(first)
    pal = 3 + u * bpv + (_bits(u) * (idx + 1) + 7) // 8

    def runs(head, value_bytes):
        start = np.maximum.accumulate(np.where(head, idx, 0))
        rid = np.cumsum(head) - 1
        heads = np.flatnonzero(head)
        full = value_bytes[heads] + _vlen(np.diff(np.append(heads, n)).astype(np.uint64))
        before = np.concatenate([[0], np.cumsum(full)])[rid]
        return 5 + before + value_bytes[start] + _vlen((idx - start + 1).astype(np.uint64))

    head = np.ones(n, dtype=bool)
    head[1:] = raw[1:] != raw[:-1]
    rle = runs(head, np.full(n, bpv))
    head = np.ones(n, dtype=bool)
    head[1:] = d[1:] != d[:-1]
    drle = runs(head, dl)
    return np.stack([1 + np.cumsum(dl), pal, rle, drle])


def _select(sizes):
    best, mode = sizes[DELTA], DELTA
    for m in (PALETTE, RLE, DRLE):
        if sizes[m] < best:
            best, mode = sizes[m], m
    return mode


def _model(v):
    """(mode, the four sizes) of a field's values as the probe sees them."""
    sizes = [int(s) for s in _prefix_sizes(v[:PROBE])[:, -1]]
    return _select(sizes), sizes


# ---- the parser: blob -> chunks -> sections ----------------------------------------------------------------------------
def _chunk_bodies(blob):
    _, p = cb.DecodeHeader(blob)
    out = []
    while p < len(blob):
        size = int.from_bytes(blob[p:p + 4], "little")
        out.append(blob[p + 4:p + 4 + size])
        p += 4 + size
    assert p == len(blob)
    return out


def _uvarint(b, p):
    v = s = 0
    while True:
        v |= (b[p] & 0x7F) << s
        p, s = p + 1, s + 7
        if b[p - 1] < 0x80:
            return v, p


def _parse_sections(body, bpvs, n):
    """The sections of a chunk body that holds nothing else: one dict per field."""
    p, out = 0, []
    a = np.frombuffer(body, dtype=np.uint8)
    for bpv in bpvs:
        sec = {"mode": body[p], "n": n, "bpv": bpv}
        if sec["mode"] == DELTA:
            end = p + 1 + int(np.flatnonzero(a[p + 1:] < 0x80)[n - 1]) + 1
        elif sec["mode"] == PALETTE:
            count = int.from_bytes(body[p + 1:p + 3], "little")
            sec["count"], sec["bits"] = count, int(_bits(count))
            sec["palette"] = [int.from_bytes(body[p + 3 + k * bpv:p + 3 + (k + 1) * bpv], "little") for k in range(count)]
            end = p + 3 + count * bpv + (sec["bits"] * n + 7) // 8
        else:
            runs = int.from_bytes(body[p + 1:p + 5], "little")
            q, lens, widths, nan_diff = p + 5, [], set(), False
            for _ in range(runs):
                if sec["mode"] == RLE:
                    q += bpv
                else:
                    nan_diff |= body[q] == 0x00                 # the reference's encoding of a diff of exactly INT64_MIN
                    _, q = _uvarint(body, q)
                length, q2 = _uvarint(body, q)
                lens.append(length)
                widths.add(q2 - q)
                q = q2
            sec.update(runs=runs, lens=lens, len_widths=widths, nan_diff=nan_diff)
            end = q
        sec["size"] = end - p
        out.append(sec)
        p = end
    assert p == len(body), "sections do not fill the chunk"
    return out


# ---- layouts and clouds ------------------------------------------------------------------------------------------------
class _Group:
    """Frames of one layout: `lead` lossy float32 lanes (a FloatN group), the section fields, `scalars` lossy float32
    fields behind them, each field `pad` bytes behind the previous one. frames[f] holds the values of each section field
    of frame f. `claims` are shapes the construction reached by itself (mode ties), which the model check confirms; `big`
    frames get a capacity above MaxCompressedSize; `side` layouts fit the side-mode reader (a regular stream of 3..6
    lossy floats, at most 4 section fields whose values fill one 8 KB tile), which the side1 route must then take."""

    def __init__(self, name, types, frames, lead=0, scalars=0, pad=0, claims=(), big=False, side=False):
        fields = [cb.PointField(c, 4 * k, F.FLOAT32, 0.001) for k, c in enumerate("xyzi"[:lead])]
        off = 4 * lead
        for k, t in enumerate(types):
            off += pad
            fields.append(cb.PointField(f"f{k}", off, t, None))
            off += cb.SizeOf(t)
        for k in range(scalars):
            off += pad
            fields.append(cb.PointField(f"s{k}", off, F.FLOAT32, 0.01))
            off += 4
        self.name, self.types, self.frames, self.lead, self.big, self.side = name, list(types), frames, lead, big, side
        self.step = off + pad
        self.fields = fields
        self.claims = set(claims)
        self.sections = [f for f in fields if f.type in NP]

    def info(self, n, sections_only=False):
        fields = self.sections if sections_only else self.fields
        return cb.EncodingInfo(fields=list(fields), width=n, height=1, point_step=self.step, encoding_opt=cb.EncodingOptions.LOSSY,
                               compression_opt=NONE, use_threads=False, version=5)

    def cloud(self, f):
        cols = self.frames[f]
        n = len(cols[0])
        rows = np.full((n, self.step), 0xCD, dtype=np.uint8)
        t = np.arange(n) * 0.013
        for k, fld in enumerate(f for f in self.fields if f.type == F.FLOAT32):
            v = (np.cos(t + k) * (20 + k)).astype(np.float32)
            if k < self.lead:
                v[7 + k::997] = np.nan
            rows[:, fld.offset:fld.offset + 4] = v.view(np.uint8).reshape(n, 4)
        for fld, c in zip(self.sections, cols):
            c = np.ascontiguousarray(c, dtype=NP[fld.type])
            rows[:, fld.offset:fld.offset + c.itemsize] = c.view(np.uint8).reshape(n, c.itemsize)
        return rows.reshape(-1)

    def cap(self, f):
        n = len(self.frames[f][0])
        need = cb.MaxCompressedSize(self.info(n), n, True)
        return need + 12 * n * len(self.sections) if self.big else need


def _distinct(rng, t, d, ones=False):
    """d distinct values of type t (the all-ones bit pattern among them when `ones`)."""
    it = np.iinfo(NP[t])
    if cb.SizeOf(t) == 2:
        raw = rng.permutation(1 << 16)[:d].astype(np.uint64)
    else:
        raw = np.unique(rng.integers(0, 2 ** (8 * cb.SizeOf(t)), 2 * d + 16, dtype=np.uint64))
        raw = rng.permutation(raw)[:d]
    if ones:
        raw[0] = np.uint64(2 ** (8 * cb.SizeOf(t)) - 1)
        assert len(np.unique(raw)) == d
    return raw.astype(np.dtype(f"u{it.bits // 8}")).view(NP[t])


def _with_distinct(rng, t, n, d, ones=False):
    """n values holding exactly d distinct ones, in random order."""
    vals = _distinct(rng, t, d, ones)
    pick = np.concatenate([np.arange(d), rng.integers(0, d, n - d)])
    return vals[rng.permutation(pick)]


def _exact(rng, t, n, d, ones=False):
    """n values, the first 4096 of them two values (one when d == 1), exactly d distinct in all."""
    vals = _distinct(rng, t, d, ones)
    k = min(d, 2)
    head = vals[np.arange(min(PROBE, n)) % k]
    tail_n = n - len(head)
    assert tail_n >= d - k, (n, d)
    tail = np.concatenate([np.arange(k, d), rng.integers(0, d, tail_n - (d - k))]) if tail_n else np.zeros(0, dtype=np.int64)
    return np.concatenate([head, vals[rng.permutation(tail).astype(np.int64)]])


# 1, 2, 3, 4, 5, 8, 9, 16, 17, ..., 2^k, 2^k + 1, ..., 32768: every index width from 0 to 15 at both of its ends
LADDER = [1, 2, 3, 4, 5] + [d for k in range(3, 15) for d in (1 << k, (1 << k) + 1)] + [CHUNK]


def _ladder_group():
    """Palette widths: one field of every type, chunk k of the frame holding LADDER[k] distinct values (the all-ones
    value among 5 and 4097 of them: the dedicated slot of both tables)."""
    rng = np.random.default_rng(1)
    ladder = LADDER if not EMULATED else [1, 2, 3] + [(1 << k) + 1 for k in range(2, 15)]
    types = [F.INT16, F.UINT16, F.INT32, F.UINT32, F.INT64, F.UINT64]
    cols = []
    for t in types:
        chunks = [_exact(rng, t, CHUNK, 2)]
        for d in ladder:
            chunks.append(_with_distinct(rng, t, CHUNK, d, ones=t in IN_PLACE and d in (5, 4097)))
        chunks.append(_with_distinct(rng, t, 1003, 5))      # a last partial chunk: 1003 = 8 * 125 + 3
        cols.append(np.concatenate(chunks))
    return [_Group("ladder", types, [cols])]


def _remainder_group():
    """Every width, for both writers, in frames of every length mod 8 (single-chunk frames: the last chunk is chunk 0).
    Field w of each writer holds 2^(w-1) + 1 distinct values in even frames and 2^w in odd ones (w = 0: one value); 2048
    and 2049 distinct values are the two tables' edge, and the frames' overflowing items add up to more than 64."""
    rng = np.random.default_rng(2)
    base = 20480 if not EMULATED else 12288
    top = 16 if not EMULATED else 14
    types = [STAGED[w % 4] for w in range(top)] + [IN_PLACE[w % 2] for w in range(top)]
    frames = []
    for r in range(9 if not EMULATED else 4):
        n = base + (r if not EMULATED else (0, 3, 5, 7)[r])
        cols = []
        for k, t in enumerate(types):
            w = k % top
            d = 1 if w == 0 else min((1 << (w - 1)) + 1 if r % 2 == 0 else 1 << w, n - PROBE + 2)
            cols.append(_exact(rng, t, n, d, ones=t in IN_PLACE and w in (3, 12)))
        frames.append(cols)
    return [_Group("remainders", types, frames)]


def _overflow_groups():
    """More than 64 items for the overflow pool of 64 CTAs: 22 fields x 3 chunks of one frame, and 66 single-chunk frames
    of one batch whose probe window itself has more than 2048 distinct values (the brute-force count)."""
    rng = np.random.default_rng(3)
    types = [(F.UINT16, F.INT64)[k % 2] for k in range(22)]
    one = [np.concatenate([_exact(rng, t, CHUNK, 2), _with_distinct(rng, t, CHUNK, 3000), _with_distinct(rng, t, CHUNK, 2500),
                           _with_distinct(rng, t, 5003, 3000)]) for t in types]
    pool = rng.permutation(1 << 16)[:3000].astype(np.uint16)
    frames = [[pool[rng.integers(0, 3000, PROBE)]] for _ in range(66)]
    return [_Group("overflow_frame", types, [one]), _Group("overflow_batch", [F.UINT16], frames)]


# ---- mode ties ---------------------------------------------------------------------------------------------------------
def _segments(rng, t, n, kinds=range(7)):
    """Values of mixed character (walks, constant runs, ramps, few-valued noise, wide noise, short constant runs of wide
    values, constant runs of a few wide values) for the tie search."""
    lo, hi = (0, 60000) if t == F.UINT16 else (-(1 << 40), 1 << 40)
    out, v = [], int(rng.integers(lo // 2 + hi // 4, hi // 2))
    kinds = list(kinds)
    while sum(len(s) for s in out) < n:
        kind, m = kinds[int(rng.integers(len(kinds)))], int(rng.integers(20, 600))
        if kind == 0:
            s = v + np.cumsum(rng.integers(-3, 4, m))
        elif kind == 1:
            s = np.repeat(v + rng.integers(-200, 200, m // 8 + 1), rng.integers(1, 40, m // 8 + 1))[:m]
        elif kind == 2:
            s = v + np.cumsum(np.repeat(rng.integers(-9, 10, m // 10 + 1), rng.integers(2, 30, m // 10 + 1))[:m])
        elif kind == 3:
            s = v + rng.integers(0, int(rng.integers(2, 300)), m) * int(rng.integers(1, 50))
        elif kind == 4:
            s = rng.integers(lo, hi, m)
        elif kind == 5:
            s = np.repeat(rng.integers(lo, hi, m), rng.integers(1, 7, m))[:m]
        else:
            s = np.repeat(rng.integers(lo, hi, 6)[rng.integers(0, 6, m)], rng.integers(1, 40, m))[:m]
        s = np.clip(s, lo, hi)
        v = int(s[-1])
        out.append(s)
    return np.concatenate(out)[:n].astype(NP[t])


PAIRS = [(a, b) for a in range(4) for b in range(a + 1, 4)]


def _tie_frames(t):
    """Probe windows (whole single-chunk frames) where two modes' sizes are equal or one byte apart, both below the
    other two, for all six pairs; found by scanning the prefixes of mixed-character arrays with the model."""
    want = {(a, b, dd) for a, b in PAIRS for dd in (-1, 0, 1)}
    found = {}
    for seed in range(1500):
        rng = np.random.default_rng(1000 + seed)
        v = _segments(rng, t, PROBE, rng.permutation(7)[:int(rng.integers(1, 4))])
        s = _prefix_sizes(v)
        for a, b in PAIRS:
            others = np.min(np.delete(s, [a, b], axis=0), axis=0)
            ok = np.maximum(s[a], s[b]) < others
            for dd in (-1, 0, 1):
                if (a, b, dd) in found:
                    continue
                hit = np.flatnonzero(ok & (s[a] - s[b] == dd) & (np.arange(PROBE) >= 7))
                if hit.size:
                    found[(a, b, dd)] = v[:int(hit[int(rng.integers(hit.size))]) + 1]
        if want <= found.keys():
            break
    missing = want - found.keys()
    assert not missing or t != F.UINT16, f"no probe window found for {missing}"   # (the reach test asks for all of them)
    return found


def _bruteforce_frames():
    """Single-chunk UINT16 frames whose probe holds more than 2048 distinct values (the brute-force count) and where
    Palette wins by one byte or loses by one byte."""
    found = {}
    for seed in range(400):
        rng = np.random.default_rng(5000 + seed)
        pool = np.sort(rng.permutation(1 << 16)[:int(rng.integers(2300, 4000))]).astype(np.uint16)
        near = rng.random() * 0.6          # a share of steps to a neighbouring pool value: 2-byte deltas
        pick = rng.integers(0, len(pool), PROBE)
        walk = np.clip(np.cumsum(rng.integers(-2, 3, PROBE)) + len(pool) // 2, 0, len(pool) - 1)
        v = pool[np.where(rng.random(PROBE) < near, walk, pick)]
        s = _prefix_sizes(v)
        first = np.zeros(PROBE, dtype=bool)
        first[np.unique(v, return_index=True)[1]] = True
        many = np.cumsum(first) > SMEM_DISTINCT
        others = np.min(np.delete(s, PALETTE, axis=0), axis=0)
        for dd in (-1, 1):
            hit = np.flatnonzero(many & (s[PALETTE] - others == dd))
            if dd not in found and hit.size:
                found[dd] = v[:int(hit[0]) + 1]
        if len(found) == 2:
            break
    assert len(found) == 2, f"no brute-force window found for {set((-1, 1)) - found.keys()}"
    return found


def _tie_groups():
    """Per type: the tie windows, the brute-force windows, frames of 4096 and 4097 points, all in one batch (frames of
    one layout that commit different modes)."""
    groups = []
    for t in (F.UINT16, F.INT64):
        ties = _tie_frames(t)
        claims = {("tie", MODE_NAMES[a], MODE_NAMES[b], dd) for a, b, dd in ties}
        frames = [[v] for v in ties.values()]
        rng = np.random.default_rng(7)
        for n in (PROBE, PROBE + 1):
            frames.append([_segments(rng, t, n)])
        if t == F.UINT16:
            bf = _bruteforce_frames()
            claims |= {("brute-force count", "Palette wins" if dd < 0 else "Palette loses") for dd in bf}
            frames += [[v] for v in bf.values()]
        groups.append(_Group(f"ties_{t.name}", [t], frames, lead=3, claims=claims, side=True))
    return groups


# ---- run tables and committed modes ------------------------------------------------------------------------------------
def _lens_chunks():
    """Run lengths per chunk: 1, 127, 128, 16383, 16384; one run of 32768; kRunPar - 1 .. 2 kRunPar + 1 runs."""
    out = [[16384, 16383, 1], [1, 127, 128] * 128, [CHUNK]]
    for r in (RUN_PAR - 1, RUN_PAR, RUN_PAR + 1, 2 * RUN_PAR - 1, 2 * RUN_PAR, 2 * RUN_PAR + 1):
        out.append([CHUNK // r + (1 if k < CHUNK % r else 0) for k in range(r)])
    if EMULATED:
        out = out[:4] + out[5:7]
    return out


def _rle_values(rng, t, lens):
    vals = _distinct(rng, t, len(lens) + 1)
    return np.repeat(vals[:len(lens)], lens)


def _drle_values(t, lens):
    """Runs of equal deltas with these lengths, the first delta equal to the first value (prev = 0 at a chunk start)."""
    slopes = np.where(np.arange(len(lens)) % 2 == 0, 1, 2)
    return np.cumsum(np.repeat(slopes, lens)).astype(NP[t])


def _run_groups():
    rng = np.random.default_rng(4)
    types = [F.UINT16, F.UINT16, F.INT32, F.INT32, F.INT64, F.UINT64]
    cols = []
    for k, t in enumerate(types):
        drle = k % 2 == 1
        probe_lens = [64] * (CHUNK // 64)
        chunks = [_drle_values(t, probe_lens) if drle else _rle_values(rng, t, probe_lens)]
        for lens in _lens_chunks() + [[100] * 77 + [77]]:
            chunks.append(_drle_values(t, lens) if drle else _rle_values(rng, t, lens))
        cols.append(np.concatenate(chunks))
    groups = [_Group("runs", types, [cols])]
    # DeltaRle at the 64-bit extremes: deltas of INT64_MAX, INT64_MIN + 1, 2^62, -1 (decodes), and a frame with a delta
    # of exactly INT64_MIN, which the reference's encoder writes as a single 0x00 and its decoder refuses
    ext = [np.int64(2**63 - 1), np.int64(-2**63 + 1), np.int64(2**62), np.int64(-1), np.int64(3)]
    deltas = np.repeat(np.array(ext * 40, dtype=np.int64), 50)
    with np.errstate(over="ignore"):
        v = np.cumsum(deltas.view(np.uint64))
    mn = np.repeat(np.array([0, 1 << 63, 1 << 63, 5, (1 << 63) + 5], dtype=np.uint64), [300, 1, 400, 300, 500])
    frames = [[v.view(np.int64), v], [mn.view(np.int64), mn]]
    groups.append(_Group("extremes", [F.INT64, F.UINT64], frames, lead=4, scalars=2, side=True))
    # a committed mode that is bad for later chunks: Rle / DeltaRle on the probe, then every point its own value
    bad = []
    for k, t in enumerate([F.UINT16, F.UINT16, F.INT32, F.INT64, F.UINT64, F.INT32]):
        first = _drle_values(t, [40] * (CHUNK // 40) + [CHUNK % 40]) if k % 2 else _rle_values(rng, t, [40] * (CHUNK // 40) + [CHUNK % 40])
        bad.append((t, np.concatenate([first, _distinct(rng, t, CHUNK), _distinct(rng, t, 7001)])))
    groups.append(_Group("bad_commit", [t for t, _ in bad], [[c for _, c in bad]], big=True))
    return groups


# ---- batches and layouts -----------------------------------------------------------------------------------------------
def _layout_groups():
    """Three section fields, alone or between a FloatN group of 4 lanes and a scalar lossy float (a regular stream of 5
    values: side mode's reader takes 14 bytes of sections per point), padded or not; each frame commits another mix of
    modes for the same fields."""
    rng = np.random.default_rng(6)
    types = [F.UINT16, F.INT32, F.UINT64]
    n_of = (40000, 4097, 70001, 300) if not EMULATED else (33000, 4097, 300)

    def col(kind, t, n):
        if kind == PALETTE:
            return _with_distinct(rng, t, n, 13)
        if kind == RLE:
            return _rle_values(rng, t, [37] * (n // 37) + ([n % 37] if n % 37 else []))
        if kind == DRLE:
            return _drle_values(t, [50] * (n // 50) + ([n % 50] if n % 50 else []))
        return _segments(rng, t, n) if t != F.INT32 else np.cumsum(rng.integers(-5000, 5000, n)).astype(np.int32)

    frames = []
    for f, n in enumerate(n_of):
        frames.append([col((f + k) % 4, t, n) for k, t in enumerate(types)])
    return [_Group(f"layout_{'lead' if lead else 'bare'}_{'pad' if pad else 'tight'}", types, frames, lead=4 if lead else 0,
                   scalars=1 if lead else 0, pad=pad, side=lead)
            for lead in (False, True) for pad in (0, 3)]


@functools.lru_cache(maxsize=None)
def _groups():
    out = []
    for make in (_ladder_group, _remainder_group, _overflow_groups, _tie_groups, _run_groups, _layout_groups):
        out += make()
    return {g.name: g for g in out}


# ---- the oracle's blobs, checked against the model and parsed ------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def _expected(oracle, name):
    """Per frame: (blob or None, the oracle's error message or None)."""
    g = _groups()[name]
    out = []
    for f in range(len(g.frames)):
        n = len(g.frames[f][0])
        try:
            out.append((oracle.encode(g.info(n), g.cloud(f), cap=g.cap(f)), None))
        except RuntimeError as e:
            out.append((None, str(e)))
    return out


@functools.lru_cache(maxsize=None)
def _shapes(oracle, name):
    """Checks every frame's sections against the model and returns the shapes they reach."""
    g = _groups()[name]
    seen = set(g.claims)
    bpvs = [cb.SizeOf(t) for t in g.types]
    overflow_total, frame_modes = 0, set()
    for f, (blob, err) in enumerate(_expected(oracle, name)):
        cols = g.frames[f]
        n = len(cols[0])
        assert blob is not None, f"{name} frame {f}: the oracle refused it: {err}"
        if len(g.sections) < len(g.fields):
            # the sections are the tail of every chunk: the same cloud encoded with its section fields alone gives them
            twin = _chunk_bodies(oracle.encode(g.info(n, sections_only=True), g.cloud(f), cap=g.cap(f)))
            full = _chunk_bodies(blob)
            assert len(twin) == len(full) and all(a.endswith(b) for a, b in zip(full, twin)), f"{name} frame {f}"
            bodies = twin
        else:
            bodies = _chunk_bodies(blob)
        models = [_model(c) for c in cols]
        overflow = 0
        for c, body in enumerate(bodies):
            m = min(CHUNK, n - c * CHUNK)
            for k, (sec, t, (mode, sizes)) in enumerate(zip(_parse_sections(body, bpvs, m), g.types, models)):
                where = f"{name} frame {f} chunk {c} field {k} ({t.name}, {n} points)"
                assert sec["mode"] == mode, f"{where}: the oracle committed {MODE_NAMES[sec['mode']]}, the model {MODE_NAMES[mode]} {sizes}"
                if n <= PROBE:
                    assert sec["size"] == sizes[mode], f"{where}: section of {sec['size']} bytes, the model says {sizes[mode]}"
                w = _writer(t)
                if mode == PALETTE:
                    bits = sec["bits"]
                    seen |= {("palette width", t.name, bits), ("palette width, length mod 8", w, bits, m % 8)}
                    if sec["count"] in (SMEM_DISTINCT, SMEM_DISTINCT + 1):
                        seen.add(("palette of", w, sec["count"]))
                    if bpvs[k] == 8 and (1 << 64) - 1 in sec["palette"]:
                        seen.add(("all-ones value", "shared table" if sec["count"] <= SMEM_DISTINCT else "global table"))
                    overflow += sec["count"] > SMEM_DISTINCT
                elif mode in (RLE, DRLE):
                    mn = MODE_NAMES[mode]
                    seen |= {("run length bytes", mn, b) for b in sec["len_widths"]}
                    seen |= {("run length", mn, x) for x in set(sec["lens"]) & {1, 127, 128, 16383, 16384, CHUNK}}
                    if sec["runs"] in (RUN_PAR - 1, RUN_PAR, RUN_PAR + 1, 2 * RUN_PAR - 1, 2 * RUN_PAR, 2 * RUN_PAR + 1):
                        seen.add(("runs in a chunk", mn, sec["runs"]))
                    if sec["nan_diff"]:
                        seen.add(("DeltaRle diff of INT64_MIN",))
                    if c > 0 and len(np.unique(cols[k][c * CHUNK:c * CHUNK + m])) == m:
                        seen.add(("committed mode, every later point its own value", mn))
        frame_modes.add(tuple(mode for mode, _ in models))
        overflow_total += overflow
        if overflow > 64:
            seen.add(("overflowing items", "one frame"))
        if n <= PROBE:
            seen.add(("probe", "whole chunk"))
        if n in (PROBE, PROBE + 1):
            seen.add(("probe", f"{n} points"))
    if overflow_total > 64 and len(g.frames) > 1:
        seen.add(("overflowing items", "one batch"))
    if len(frame_modes) > 1:
        seen.add(("one batch, different modes",))
    return frozenset(seen)


def _required():
    writers = ("staged", "in-place")
    req = {("palette width", t.name, b) for t in STAGED + IN_PLACE for b in range(16)}
    req |= {("palette width, length mod 8", w, b, r) for w in writers for b in range(16) for r in range(8)}
    req |= {("palette of", w, c) for w in writers for c in (SMEM_DISTINCT, SMEM_DISTINCT + 1)}
    req |= {("all-ones value", "shared table"), ("all-ones value", "global table")}
    req |= {("overflowing items", "one frame"), ("overflowing items", "one batch")}
    req |= {("tie", MODE_NAMES[a], MODE_NAMES[b], dd) for a, b in PAIRS for dd in (-1, 0, 1)}
    req |= {("brute-force count", "Palette wins"), ("brute-force count", "Palette loses")}
    req |= {("probe", "whole chunk"), ("probe", "4096 points"), ("probe", "4097 points")}
    req |= {("committed mode, every later point its own value", m) for m in ("Rle", "DeltaRle")}
    for m in ("Rle", "DeltaRle"):
        req |= {("run length bytes", m, b) for b in (1, 2, 3)}
        req |= {("run length", m, x) for x in (1, 127, 128, 16383, 16384, CHUNK)}
        req |= {("runs in a chunk", m, r) for r in (RUN_PAR - 1, RUN_PAR, RUN_PAR + 1, 2 * RUN_PAR - 1, 2 * RUN_PAR, 2 * RUN_PAR + 1)}
    req |= {("DeltaRle diff of INT64_MIN",), ("one batch, different modes",)}
    return req


def test_every_listed_shape_is_reached(oracle):
    # the model agrees with the oracle on every frame (asserted inside _shapes), and the cases reach what they were built for
    seen = set().union(*(_shapes(oracle, name) for name in _groups()))
    missing = _required() - seen
    assert not missing, f"{len(missing)} shapes never reached: {sorted(missing)[:40]}"


# ---- the kernels against the oracle ------------------------------------------------------------------------------------
GROUP_NAMES = ["ladder", "remainders", "overflow_frame", "overflow_batch", "ties_UINT16", "ties_INT64", "runs", "extremes",
               "bad_commit"] + [f"layout_{a}_{b}" for a in ("bare", "lead") for b in ("tight", "pad")]


@pytest.mark.gpu
@pytest.mark.parametrize("name", GROUP_NAMES)
def test_sections_equal_the_oracle(oracle, name, monkeypatch):
    g = _groups()[name]
    _shapes(oracle, name)
    expected = _expected(oracle, name)
    clouds = [g.cloud(f) for f in range(len(g.frames))]
    points = [len(c[0]) for c in g.frames]
    # encode: the whole group through encode_blobs (host memory: a launch per frame) and through one launch of
    # encode_blobs_device, or frame by frame into a capacity above MaxCompressedSize
    if not g.big:
        enc = cb.PointcloudEncoder(g.info(points[0]))
        got = enc.encode_blobs(clouds)
        for f, (blob, _) in enumerate(expected):
            assert got[f] == blob, f"{name} frame {f} ({points[f]} points): the blob differs from the oracle's"
        caps = [g.cap(f) for f in range(len(clouds))]
        ins = [_Dev(src=c) for c in clouds]
        outs = [_Dev(src=np.full(c, FILL, dtype=np.uint8)) for c in caps]
        sizes = enc.encode_blobs_device([d.ptr for d in ins], [c.nbytes for c in clouds], [o.ptr for o in outs], caps)
        for f, (blob, _) in enumerate(expected):
            assert bytes(outs[f].numpy()[:sizes[f]]) == blob, f"{name} frame {f} ({points[f]} points): encode_blobs_device differs"
    else:
        for f, (blob, _) in enumerate(expected):
            info, cap = g.info(points[f]), g.cap(f)
            enc = cb.PointcloudEncoder(info)
            out = np.full(cap + 256, FILL, dtype=np.uint8)
            w = enc.encode_into(clouds[f], out[:cap])
            assert bytes(out[:w]) == blob and (out[cap:] == FILL).all(), f"{name} frame {f}"
            need = cb.MaxCompressedSize(info, points[f], True)
            try:
                theirs = None
                oracle.encode(info, clouds[f], cap=need)
            except RuntimeError as e:
                theirs = str(e)
            try:
                ours = None
                w = enc.encode_into(clouds[f], out[:need])
            except RuntimeError as e:
                ours = str(e)
            if theirs is None:
                assert ours is None and bytes(out[:w]) == blob, f"{name} frame {f} at MaxCompressedSize: {ours}"
            else:
                assert ours == theirs, f"{name} frame {f} at MaxCompressedSize: {ours!r} vs {theirs!r}"
    # decode every frame under every route, into pre-filled buffers
    wants = []
    for f, (blob, _) in enumerate(expected):
        want = np.full(points[f] * g.step, FILL, dtype=np.uint8)
        try:
            oracle.decode(blob, want)
            wants.append((want, None))
        except RuntimeError as e:
            wants.append((None, str(e)))
    dec = cb.PointcloudDecoder()
    for route, env in ROUTES.items():
        for var in ROUTE_ENV:
            monkeypatch.delenv(var, raising=False)
        for var, val in env.items():
            monkeypatch.setenv(var, val)
        for f, ((blob, _), (want, theirs)) in enumerate(zip(expected, wants)):
            info, hdr = cb.DecodeHeader(blob)
            got = np.full(points[f] * g.step, FILL, dtype=np.uint8)
            try:
                ours = None
                dec.decode(info, blob[hdr:], got)
            except RuntimeError as e:
                ours = str(e)
            where = f"{name} frame {f} ({points[f]} points) route {route}"
            if theirs is None:
                assert ours is None, f"{where}: {ours}"
                assert np.array_equal(got, want), f"{where}: the decode differs from the oracle's"
            else:
                assert ours == theirs, f"{where}: {ours!r} vs {theirs!r}"
            if route == "side1" and g.side and ours is None:
                assert dec.last_sections_ahead(), f"{where}: the sections were not decoded ahead of the stream (side mode)"
            if route in ("side0", "careful"):
                assert not dec.last_sections_ahead(), f"{where}: side mode ran"
    for var in ROUTE_ENV:
        monkeypatch.delenv(var, raising=False)
    # and the group's blobs as one batch of complete blobs
    outs = [np.full(p * g.step, FILL, dtype=np.uint8) for p in points]
    res = dec.decode_blobs([b for b, _ in expected], outs)
    for f, ((status, _, _), (want, theirs)) in enumerate(zip(res, wants)):
        if theirs is None:
            assert status == 0 and np.array_equal(outs[f], want), f"{name} frame {f}: decode_blobs status {status}: {dec.frame_error(f) if status else ''}"
        else:
            assert status != 0 and dec.frame_error(f) == theirs, f"{name} frame {f}: decode_blobs status {status}: {dec.frame_error(f)!r} vs {theirs!r}"


# ---- the same file under the CPU emulation (not a GPU test: it runs in the CPU suite) -------------------------------
@pytest.mark.skipif(EMULATED, reason="already running under the emulation")
@pytest.mark.parametrize("order,workers", [("fwd", "1"), ("rand", "8")])
def test_this_file_under_emulation(lib_built, order, workers):
    if platform.machine() != "x86_64":
        pytest.skip("cusim's context switch is x86-64 only")
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    sys.path.insert(0, os.path.join(ROOT, "tests", "cusim"))
    from test_cusim_kernels import _run_gpu_suite
    import build_cusim
    env = {"CUSIM_ORDER": order, "CUSIM_WORKERS": workers}
    if order == "rand":
        env["CUSIM_JITTER"] = "1"
    out = _run_gpu_suite(build_cusim.build(), env, ["tests/test_gpu_v5_sections.py"])
    assert " passed" in out and "failed" not in out
