"""cldn_b200_decode_blobs_async: device-resident blobs of one prepared layout and any point counts, decoded without the
host, so that the call can be captured in a CUDA graph.

Every frame's status and output must equal cldn_b200_decode_blobs on the same blobs (and the oracle's decode), except
where the async call refuses what decode_blobs would decode: a header that is not the prepared layout's canonical
header, and more points than prepared. Outputs sit between guard bytes with a pre-filled padding (the _Buf of
test_gpu_decode_blobs.py), so a write outside a frame's buffer or into its padding is seen.
"""
import os
import subprocess
import sys

import numpy as np
import pytest

import cloudini_b200 as cb
from cloudini_b200 import synth

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)
import test_gpu_decode_blobs as base  # noqa: E402  (guarded buffers, the decode_blobs reference, damage kinds)

EMULATED = base.EMULATED
NONE, LZ4, ZSTD = cb.CompressionOption.NONE, cb.CompressionOption.LZ4, cb.CompressionOption.ZSTD
MAX_POINTS = 34_000 if EMULATED else 100_000
OK, BAD_HEADER, TOO_SMALL, CORRUPT, UNSUPPORTED = 0, -3, -2, -4, -5


class _Dev:
    """A device copy of a numpy array (torch on the GPU, the array itself under cusim)."""

    def __init__(self, a):
        self.a = np.ascontiguousarray(a)
        if EMULATED:
            self.t, self.ptr = self.a, self.a.ctypes.data
        else:
            import torch
            self.t = torch.from_numpy(self.a.view(np.uint8).reshape(-1).copy()).cuda()
            self.ptr = self.t.data_ptr()

    def get(self):
        if EMULATED:
            return self.a.copy()
        return self.t.cpu().numpy().view(self.a.dtype).reshape(self.a.shape)


def _padded(n, seed):
    """XYZ in a 20-byte point: 8 bytes of padding no field covers."""
    info, cloud = synth.cloud_c1(n, seed=seed)
    buf = np.full((n, 20), 0xCD, dtype=np.uint8)
    buf[:, :12] = cloud.reshape(n, 12)
    info.point_step = 20
    return info, buf.reshape(-1)


def _xyzirt(n, seed):
    info, cloud = synth.cloud_c4_mixed_frame(seed, az=(n + 63) // 64 or 1)
    return info, cloud[:n * info.point_step]


LAYOUTS = {
    "xyzi": lambda n, s: synth.cloud_c2(n, seed=s),
    "xyz": lambda n, s: synth.cloud_c1(n, seed=s),
    "c3_sections": lambda n, s: synth.cloud_c3(n, seed=s),
    "xyzirt": _xyzirt,
    "lossless_dds": lambda n, s: synth.cloud_lossless(n, seed=s),
    "padded": _padded,
}


def _blob(layout, n, comp, seed):
    info, cloud = LAYOUTS[layout](n, seed)
    return base._encode(info, cloud, comp)


def _layout_info(blob):
    return cb.DecodeHeader(blob)[0]


def _run_async(dec, blobs, caps):
    """Device blobs + descriptors + statuses, one decode_blobs_async call. Returns (statuses, decoded, outputs, guards)."""
    ins = [base._Buf(max(len(b), 1), True, src=bytes(b) + b"\0" * (len(b) == 0)) for b in blobs]
    outs = [base._Buf(c, True) for c in caps]
    n = len(blobs)
    desc = _Dev(cb.blob_descs([(i.ptr, len(b), o.ptr, c) for i, b, o, c in zip(ins, blobs, outs, caps)]))
    status = _Dev(np.full(n, 99, dtype=np.int32))
    decoded = _Dev(np.full(n, 7, dtype=np.uint64))
    dec.decode_blobs_async(desc.ptr, n, status.ptr, decoded.ptr)
    dec.sync()
    guards = all(o.guards_intact() for o in outs) and all(i.guards_intact() for i in ins)
    return [int(s) for s in status.get()], [int(d) for d in decoded.get()], [o.body().copy() for o in outs], guards


def _check(dec, blobs, caps, want_status=None, oracle=None):
    """Async call vs decode_blobs on the same blobs; want_status overrides decode_blobs' status of some frames."""
    st, decoded, outs, guards = _run_async(dec, blobs, caps)
    assert guards, "a byte outside a frame's buffer changed"
    ref_st, _, ref_outs, ref_guards = base._decode_blobs(blobs, caps, True)
    assert ref_guards
    for f in range(len(blobs)):
        want = (want_status or {}).get(f, ref_st[f])
        assert st[f] == want, (f, st[f], want, ref_st[f])
        if st[f] == OK:
            assert decoded[f] == base._need(blobs[f]), f
            assert np.array_equal(outs[f], ref_outs[f]), f"frame {f} differs from decode_blobs"
            if oracle is not None:
                assert np.array_equal(outs[f], base._want(oracle, blobs[f], caps[f], True)), f"frame {f} differs from the oracle"
        else:
            assert decoded[f] == 0, f
    return st


# The decode routes of test_gpu_route_matrix.py that a prepared shape can take, set before prepare_blobs (which sizes
# the route's scratch). Small prepared shapes take the tile-parallel / per-chunk routes by default; "seq" and the
# variants below force the chunk-sequential readers (fast reader, careful reader, side mode on and off), which claim
# chunk slots and wait for their descriptors -- the code that meets empty slots. Under the emulation (CUSIM_SMS=4)
# the default already is chunk-sequential.
ROUTE_ENV = ("CLDN_B200_DECODE_MODE", "CLDN_B200_DECODE_FAST", "CLDN_B200_DECODE_SIDE")
ROUTES = {
    "default": {},
    "seq": {"CLDN_B200_DECODE_MODE": "seq"},
    "tile": {"CLDN_B200_DECODE_MODE": "tile"},
    "careful": {"CLDN_B200_DECODE_MODE": "seq", "CLDN_B200_DECODE_FAST": "0"},
    "side0": {"CLDN_B200_DECODE_MODE": "seq", "CLDN_B200_DECODE_SIDE": "0"},
    "side1": {"CLDN_B200_DECODE_MODE": "seq", "CLDN_B200_DECODE_SIDE": "1"},
}
RUN_ROUTES = ["default", "tile", "careful", "side1"] if EMULATED else list(ROUTES)


def _route(monkeypatch, route):
    for k in ROUTE_ENV:
        monkeypatch.delenv(k, raising=False)
    for k, v in ROUTES[route].items():
        monkeypatch.setenv(k, v)


def _sizes(seed):
    rng = np.random.default_rng(seed)
    return [0, 1, 32768, 32769, MAX_POINTS] + [int(x) for x in rng.integers(2, MAX_POINTS, 1 if EMULATED else 5)]


# ---- parity with decode_blobs ---------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("comp", [NONE, LZ4, ZSTD], ids=["none", "lz4", "zstd"])
@pytest.mark.parametrize("layout", list(LAYOUTS))
@pytest.mark.parametrize("route", RUN_ROUTES)
def test_varying_point_counts_equal_decode_blobs(oracle, layout, comp, route, monkeypatch):
    _route(monkeypatch, route)
    sizes = _sizes(len(layout) * 3 + comp)
    blobs = [_blob(layout, n, comp, 10 + k) for k, n in enumerate(sizes)]
    dec = cb.PointcloudDecoder()
    dec.prepare_blobs(_layout_info(blobs[0]), len(blobs) + 3, MAX_POINTS)
    st = _check(dec, blobs, [base._need(b) for b in blobs], oracle=oracle)
    assert st == [OK] * len(blobs)
    # fewer frames than prepared, in another order, with room to spare after every frame
    order = list(reversed(range(len(blobs))))[:4]
    _check(dec, [blobs[i] for i in order], [base._need(blobs[i]) + 48 for i in order])


# ---- damage among good frames ---------------------------------------------------------------------------------------
def _other_layout(blob):
    info = _layout_info(blob)
    info.fields[0].resolution = info.fields[0].resolution * 2
    return cb.EncodeHeader(info) + blob[base._payload_at(blob):]


def _leading_zero(blob):
    h = base._payload_at(blob)
    text = blob[:h]
    i = text.index(b"\nwidth: ") + 8
    return text[:i] + b"0" + text[i:] + blob[h:]


KINDS = ["truncate", "chunk_prefix", "bitflip", "stage2_frame", "other_layout", "leading_zero", "too_many_points", "short_output"]


@pytest.mark.gpu
@pytest.mark.parametrize("comp", [NONE, LZ4, ZSTD], ids=["none", "lz4", "zstd"])
@pytest.mark.parametrize("where", ["first", "middle", "last", "all"])
@pytest.mark.parametrize("route", ["default", "seq", "careful"])
def test_damaged_frames_among_good_ones(comp, where, route, monkeypatch):
    _route(monkeypatch, route)
    rng = np.random.default_rng(["first", "middle", "last", "all"].index(where) + 10 * comp)
    n_pts = 6_000 if EMULATED else 50_000
    good = [_blob("xyzi", n_pts + 1000 * k, comp, 70 + k) for k in range(5)]
    dec = cb.PointcloudDecoder()
    dec.prepare_blobs(_layout_info(good[0]), len(good), MAX_POINTS)
    at = {"first": [0], "middle": [2], "last": [len(good) - 1], "all": list(range(len(good)))}[where]
    for kind in KINDS:
        blobs, caps, want = list(good), [base._need(b) for b in good], {}
        for i in at:
            if kind == "short_output":
                caps[i] -= 1
                want[i] = TOO_SMALL
            elif kind == "other_layout":
                blobs[i] = _other_layout(blobs[i])
                want[i] = BAD_HEADER
            elif kind == "leading_zero":
                blobs[i] = _leading_zero(blobs[i])
                want[i] = BAD_HEADER
            elif kind == "too_many_points":
                blobs[i] = _blob("xyzi", MAX_POINTS + 1, comp, 99)
                caps[i] = base._need(blobs[i])
                want[i] = UNSUPPORTED
            elif kind == "stage2_frame":
                src = bytearray(blobs[i])
                src[base._payload_at(blobs[i]) + 4 + 6] ^= 0x40   # inside the first chunk's LZ4 / ZSTD frame (NONE: its stream)
                blobs[i] = bytes(src)
            else:
                blobs[i] = base._damaged(blobs[i], kind, rng)
        st = _check(dec, blobs, caps, want)
        assert all(st[i] == OK for i in range(len(blobs)) if i not in at), kind
        if kind in ("truncate", "chunk_prefix"):
            assert all(st[i] == CORRUPT for i in at), (kind, st)


# ---- the shape the chunk-sequential readers take by their own choice ---------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("comp", [NONE, ZSTD], ids=["none", "zstd"])
@pytest.mark.parametrize("layout", ["xyzi", "c3_sections", "xyzirt"])
def test_a_prepared_shape_past_the_sequential_threshold(oracle, layout, comp, monkeypatch):
    # 40 frames of up to 4 chunks: 160 chunk slots, past the 148 at which a 132-SM H100 picks the chunk-sequential readers
    # (fast FloatN reader for XYZI, side mode for C3, fast general reader for XYZIRT) without any override; most slots
    # are empty, the frames before, between and after them hold 0 .. MAX_POINTS points, two are damaged
    _route(monkeypatch, "default")
    frames = 12 if EMULATED else 40
    rng = np.random.default_rng(comp + len(layout))
    sizes = [0, 1, 32769, MAX_POINTS] + [int(x) for x in rng.integers(1, MAX_POINTS, frames - 4)]
    blobs = [_blob(layout, n, comp, 400 + k) for k, n in enumerate(sizes)]
    dec = cb.PointcloudDecoder()
    dec.prepare_blobs(_layout_info(blobs[0]), frames, MAX_POINTS)
    st = _check(dec, blobs, [base._need(b) for b in blobs], oracle=oracle)
    assert st == [OK] * frames
    blobs[5] = base._damaged(blobs[5], "chunk_prefix", rng)
    blobs[-1] = base._damaged(blobs[-1], "truncate", rng)
    st = _check(dec, blobs, [base._need(b) for b in blobs])
    assert st[5] == CORRUPT and all(st[f] == OK for f in range(frames) if f not in (5, frames - 1))
    # fewer frames than prepared: the tables and slots of the rest are empty
    st = _check(dec, blobs[:7], [base._need(b) for b in blobs[:7]])
    assert st[5] == CORRUPT


# ---- asynchrony, graphs, launches, concurrency -----------------------------------------------------------------------
def _viz_blobs(comp, count, seed):
    out = []
    for k in range(count):
        n = int(np.random.default_rng(seed + k).integers(1, MAX_POINTS))
        out.append(_blob("xyzi", n, comp, seed + k))
    return out


@pytest.mark.gpu
@pytest.mark.skipif(EMULATED, reason="needs a CUDA stream")
def test_the_call_returns_before_the_stream_runs():
    import torch
    s = torch.cuda.Stream()
    dec = cb.PointcloudDecoder(stream=s.cuda_stream)
    blobs = _viz_blobs(ZSTD, 6, 5)
    dec.prepare_blobs(_layout_info(blobs[0]), 6, MAX_POINTS)
    caps = [base._need(b) for b in blobs]
    ins = [base._Buf(len(b), True, src=b) for b in blobs]
    outs = [base._Buf(c, True) for c in caps]
    desc = cb.pack_blob_descs([(i.ptr, len(b), o.ptr, c) for i, b, o, c in zip(ins, blobs, outs, caps)])
    status = torch.full((6,), 99, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        torch.cuda._sleep(200_000_000)   # ~0.1 s of the stream ahead of the call
    dec.decode_blobs_async(desc.data_ptr(), 6, status.data_ptr())
    assert not s.query(), "the call waited for the stream"
    s.synchronize()
    assert status.cpu().tolist() == [0] * 6
    ref_st, _, ref_outs, _ = base._decode_blobs(blobs, caps, True)
    assert ref_st == [0] * 6
    for o, r in zip(outs, ref_outs):
        assert np.array_equal(o.body(), r)


@pytest.mark.gpu
@pytest.mark.skipif(EMULATED, reason="needs CUDA graphs")
@pytest.mark.parametrize("comp", [NONE, LZ4, ZSTD], ids=["none", "lz4", "zstd"])
def test_captured_graph_replays_new_blobs_in_the_same_buffers(comp):
    import torch
    s = torch.cuda.Stream()
    dec = cb.PointcloudDecoder(stream=s.cuda_stream)
    n_max = 8
    first = _viz_blobs(comp, n_max, 300)
    dec.prepare_blobs(_layout_info(first[0]), n_max, MAX_POINTS)
    blob_cap = max(len(_blob("xyzi", MAX_POINTS, comp, 1)), max(len(b) for b in first)) + 4096
    out_cap = MAX_POINTS * 16
    arena = torch.zeros(n_max * blob_cap, dtype=torch.uint8, device="cuda")
    outs = torch.zeros(n_max * out_cap, dtype=torch.uint8, device="cuda")
    desc = torch.zeros(n_max * 32, dtype=torch.uint8, device="cuda")
    status = torch.zeros(n_max, dtype=torch.int32, device="cuda")
    decoded = torch.zeros(n_max, dtype=torch.int64, device="cuda")

    def load(blobs, caps):
        for f, b in enumerate(blobs):
            arena[f * blob_cap:f * blob_cap + len(b)].copy_(torch.frombuffer(bytearray(b), dtype=torch.uint8))
        outs.fill_(base.PAD_BYTE)
        cb.pack_blob_descs([(arena.data_ptr() + f * blob_cap, len(b), outs.data_ptr() + f * out_cap, caps[f])
                            for f, b in enumerate(blobs)], out=desc)
        torch.cuda.synchronize()

    load(first, [base._need(b) for b in first])
    with torch.cuda.stream(s):   # warm-up outside the capture
        dec.decode_blobs_async(desc.data_ptr(), n_max, status.data_ptr(), decoded.data_ptr())
    s.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        dec.decode_blobs_async(desc.data_ptr(), n_max, status.data_ptr(), decoded.data_ptr())
    for rnd in range(2):
        blobs = _viz_blobs(comp, n_max, 500 + 50 * rnd)
        caps = [base._need(b) for b in blobs]
        rng = np.random.default_rng(rnd)
        bad = int(rng.integers(n_max))
        blobs[bad] = base._damaged(blobs[bad], ["truncate", "chunk_prefix"][rnd], rng)
        caps[bad] = max(caps[bad], base._need(blobs[bad]))
        if rnd == 1:
            caps[(bad + 1) % n_max] -= 1
        load(blobs, caps)
        g.replay()
        torch.cuda.synchronize()
        ref_st, _, ref_outs, _ = base._decode_blobs(blobs, caps, True)
        got = status.cpu().tolist()
        assert got == ref_st, (rnd, got, ref_st)
        assert ref_st[bad] != 0
        host = outs.cpu().numpy()
        for f in range(n_max):
            if got[f] == 0:
                assert decoded[f].item() == base._need(blobs[f])
                assert np.array_equal(host[f * out_cap:f * out_cap + caps[f]], ref_outs[f]), (rnd, f)
    # a call the prepared shape cannot hold, and a decoder never prepared, fail with a status inside a capture
    for d, n in ((dec, n_max + 1), (cb.PointcloudDecoder(stream=s.cuda_stream), 1)):
        g2 = torch.cuda.CUDAGraph()
        with pytest.raises(RuntimeError):
            with torch.cuda.graph(g2, stream=s):
                d.decode_blobs_async(desc.data_ptr(), n, status.data_ptr())
    torch.cuda.synchronize()


@pytest.mark.gpu
@pytest.mark.parametrize("comp", [NONE, LZ4, ZSTD], ids=["none", "lz4", "zstd"])
def test_launches_per_call_do_not_depend_on_the_frames(comp):
    dec = cb.PointcloudDecoder()
    pool = _viz_blobs(comp, 6, 900) + [_blob("xyzi", 0, comp, 1), _blob("xyzi", MAX_POINTS, comp, 2)]
    dec.prepare_blobs(_layout_info(pool[0]), len(pool), MAX_POINTS)
    counts = set()
    for sel in ([0], [6], [7], list(range(len(pool))), [1, 6, 3]):
        blobs = [pool[i] for i in sel]
        before = cb.kernel_launch_count()
        st, _, _, _ = _run_async(dec, blobs, [base._need(b) for b in blobs])
        counts.add(cb.kernel_launch_count() - before)
        assert st == [0] * len(blobs)
    assert len(counts) == 1, counts


@pytest.mark.gpu
@pytest.mark.skipif(EMULATED, reason="needs CUDA streams")
def test_two_handles_on_two_streams_equal_each_call_alone():
    import torch
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    decs = [cb.PointcloudDecoder(stream=s.cuda_stream) for s in streams]
    sets = [_viz_blobs(ZSTD, 5, 40), _viz_blobs(ZSTD, 5, 80)]
    for d, b in zip(decs, sets):
        d.prepare_blobs(_layout_info(b[0]), 5, MAX_POINTS)
    alone = [_run_async(d, b, [base._need(x) for x in b]) for d, b in zip(decs, sets)]
    runs = []
    for d, b in zip(decs, sets):
        caps = [base._need(x) for x in b]
        ins = [base._Buf(len(x), True, src=x) for x in b]
        outs = [base._Buf(c, True) for c in caps]
        desc = cb.pack_blob_descs([(i.ptr, len(x), o.ptr, c) for i, x, o, c in zip(ins, b, outs, caps)])
        status = torch.full((5,), 99, dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()
        runs.append((ins, outs, desc, status))
    for d, (ins, outs, desc, status) in zip(decs, runs):   # both enqueued before either is waited for
        d.decode_blobs_async(desc.data_ptr(), 5, status.data_ptr())
    torch.cuda.synchronize()
    for (st, _, a_outs, _), (_, outs, _, status) in zip(alone, runs):
        assert status.cpu().tolist() == st == [0] * 5
        for a, o in zip(a_outs, outs):
            assert np.array_equal(a, o.body())


@pytest.mark.gpu
def test_prepare_refusals_and_other_calls_keep_working(oracle):
    dec = cb.PointcloudDecoder()
    blobs = _viz_blobs(NONE, 3, 20)
    info = _layout_info(blobs[0])
    with pytest.raises(RuntimeError):
        dec.decode_blobs_async(0, 1, 0)           # nothing prepared
    v2 = _layout_info(blobs[0])
    v2.version = 2
    with pytest.raises(RuntimeError):
        dec.prepare_blobs(v2, 3, MAX_POINTS)
    with pytest.raises(RuntimeError):
        dec.prepare_blobs(info, 0, MAX_POINTS)
    dec.prepare_blobs(info, 3, MAX_POINTS)
    # decode_blobs on the same handle between async calls leaves the prepared state alone
    assert base._decode_blobs(blobs, [base._need(b) for b in blobs], True)[0] == [0] * 3
    assert _check(dec, blobs, [base._need(b) for b in blobs], oracle=oracle) == [0] * 3
    # a valid blob of another layout is refused: decode_blobs decodes it
    other = _blob("xyz", 1000, NONE, 3)
    assert _check(dec, [other, blobs[0]], [base._need(other), base._need(blobs[0])], {0: BAD_HEADER}) == [BAD_HEADER, 0]


# ---- the same file under the CPU emulation ---------------------------------------------------------------------------
@pytest.mark.skipif(EMULATED, reason="already running under the emulation")
@pytest.mark.parametrize("order,workers", [("fwd", "8"), ("rand", "8")])
def test_this_file_under_emulation(lib_built, order, workers):
    from test_cusim_kernels import _run_gpu_suite
    import platform
    if platform.machine() != "x86_64":
        pytest.skip("cusim's context switch is x86-64 only")
    sys.path.insert(0, os.path.join(ROOT, "tests", "cusim"))
    import build_cusim
    # 4 SMs: the default route of every prepared shape here is chunk-sequential (persistent CTAs claiming chunk slots)
    env = {"CUSIM_ORDER": order, "CUSIM_WORKERS": workers, "CUSIM_SMS": "4"}
    if order == "rand":
        env["CUSIM_JITTER"] = "1"
    out = _run_gpu_suite(build_cusim.build(), env, ["tests/test_gpu_decode_blobs_async.py"])
    assert " passed" in out and "failed" not in out


@pytest.mark.skipif(EMULATED, reason="already running under the emulation")
def test_async_batch_under_thread_sanitizer(lib_built, tmp_path):
    # tests/cusim/blobs_async_racecheck_main.cpp: decode_blobs_async calls of NONE / LZ4 / ZSTD blobs with damaged frames
    # and empty chunk slots, every CUDA thread a ThreadSanitizer fiber (strict model: a shuffle is no fence)
    import platform
    if platform.machine() != "x86_64":
        pytest.skip("cusim's context switch is x86-64 only")
    here = os.path.join(ROOT, "tests", "cusim")
    sys.path.insert(0, here)
    import build_cusim
    from cloudini_b200.build import SOURCES
    try:
        build_cusim.build_racecheck()
    except subprocess.CalledProcessError as e:
        pytest.skip(f"ThreadSanitizer toolchain unavailable: {e}")
    objs = [os.path.join(build_cusim.OUT_DIR, os.path.splitext(s)[0] + "_tsan.o") for s in SOURCES + ["cusim.cpp"]]
    drv, exe = str(tmp_path / "blobs_async_main.o"), str(tmp_path / "blobs_async_racecheck")
    subprocess.check_call(["g++", "-std=c++17", "-O0", "-g", "-fPIC", "-pthread", "-w", "-fsanitize=thread", "-I", here, "-I",
                           os.path.join(ROOT, "include"), "-x", "c++", "-c", os.path.join(here, "blobs_async_racecheck_main.cpp"), "-o", drv])
    subprocess.check_call(["g++", "-fsanitize=thread", "-pthread", "-o", exe, drv, *objs, "-ldl"])
    env = dict(os.environ, TSAN_OPTIONS="halt_on_error=0 report_signal_unsafe=0", CUSIM_WORKERS="4", CUSIM_TSAN_STRICT="1",
               CUSIM_SMS="2")   # 2 SMs: the chunk-sequential readers, whose CTAs claim slots past each other
    env.pop("LD_PRELOAD", None)
    r = subprocess.run([exe], env=env, capture_output=True, text=True, timeout=1500)
    if "FATAL: ThreadSanitizer" in r.stderr:
        pytest.skip("ThreadSanitizer cannot run in this environment: " + r.stderr[-200:])
    assert r.returncode == 0 and "blobs_async_racecheck: done" in r.stdout, r.stdout[-2000:] + r.stderr[-3000:]
    assert "WARNING: ThreadSanitizer" not in r.stderr, r.stderr[-4000:]
