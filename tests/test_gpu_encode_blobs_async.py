"""cldn_b200_encode_blobs_async: device-resident clouds of the encoder's layout and any point counts, encoded into complete
device blobs without the host, so that the call can be captured in a CUDA graph.

Every frame's status, blob size and bytes must equal cldn_b200_encode_blobs of that frame alone on the same handle (and
for NONE the oracle's encode), except for the one refusal of the async call: more points than prepared. Outputs sit
between guard bytes with a pre-filled padding (the _Buf of test_gpu_encode_blobs.py), so that a write outside a frame's
buffer, or any write by a frame refused before the encode, is seen.
"""
import os
import subprocess
import sys

import numpy as np
import pytest

import cloudini_b200 as cb

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)
import test_gpu_encode_blobs as base  # noqa: E402  (guarded buffers, layouts, the encode_blobs reference)

EMULATED = base.EMULATED
NONE, LZ4, ZSTD = cb.CompressionOption.NONE, cb.CompressionOption.LZ4, cb.CompressionOption.ZSTD
COMPS = {"none": NONE, "lz4": LZ4, "zstd": ZSTD}
MAX_POINTS = 34_000 if EMULATED else 100_000
OK, INVALID, TOO_SMALL, UNSUPPORTED = 0, -1, -2, -5


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


class Frame:
    """One frame of a call: a cloud (None: a NULL cloud pointer of `nbytes`), its output capacity and dims."""

    def __init__(self, cloud, cap, dims=None, nbytes=None, offset=0):
        self.cloud, self.cap, self.dims, self.offset = cloud, cap, dims, offset
        self.nbytes = cloud.size if nbytes is None else nbytes


def _encoder(info, comp):
    info.compression_opt = comp
    enc = cb.PointcloudEncoder(info)
    if comp == ZSTD:
        enc.set_stage2_on_device(True)
    return enc


def _frame(info, cloud, dims=None, short=0):
    n = cloud.size // info.point_step
    return Frame(cloud, base._worst(info, n, dims) - short, dims)


def _src(fr):
    """The cloud in device memory, `offset` bytes past a 16-byte aligned base."""
    if fr.cloud is None:
        return None, 0
    buf = base._Buf(max(fr.cloud.size + fr.offset, 1), True, src=b"\0" * fr.offset + fr.cloud.tobytes() + b"\0" * (fr.cloud.size + fr.offset == 0))
    return buf, buf.ptr + fr.offset


def _run_async(enc, frames, spare=0):
    """One encode_blobs_async call. `spare` more descriptors (and outputs) follow the call's frames and must stay untouched.
    Returns (statuses, written, output bodies, guards intact, spare outputs untouched)."""
    srcs = [_src(fr) for fr in frames]
    outs = [base._Buf(fr.cap, True) for fr in frames]
    extra = [base._Buf(64, True) for _ in range(spare)]
    descs = [(ptr or 0, fr.nbytes, o.ptr, fr.cap, *(fr.dims or (0, 0))) for (_, ptr), fr, o in zip(srcs, frames, outs)]
    descs += [(srcs[0][1] or 0, frames[0].nbytes, o.ptr, 64, 0, 0) for o in extra]
    desc = _Dev(cb.cloud_descs(descs))
    n = len(frames)
    status = _Dev(np.full(n + spare, 99, dtype=np.int32))
    written = _Dev(np.full(n + spare, 7, dtype=np.uint64))
    enc.encode_blobs_async(desc.ptr, n, status.ptr, written.ptr)
    enc.sync()
    guards = all(o.guards_intact() for o in outs + extra) and all(b.guards_intact() for b, _ in srcs if b is not None)
    st, wr = status.get(), written.get()
    spare_ok = all((o.body() == base.PAD_BYTE).all() for o in extra) and all(st[n:] == 99) and all(wr[n:] == 7)
    return [int(s) for s in st[:n]], [int(w) for w in wr[:n]], [o.body().copy() for o in outs], guards, spare_ok


def _same_blob(a, b):
    """Blob equality; under the emulation's shuffled lane order LZ4 blobs need only decode to the same points: the LZ4
    kernel's shared hash table keeps whichever lane's store lands last, and the shuffled order changes that winner (the
    blobs of encode_blobs change the same way)."""
    if a == b:
        return True
    if not (base.SHUFFLED_LANES and a and b and cb.DecodeHeader(a)[0].compression_opt == LZ4):
        return False
    (sa, _, pa), (sb, _, pb) = cb.PointcloudDecoder().decode_blobs([a, b])
    return sa == sb == 0 and np.array_equal(pa, pb)


def _reference(enc, fr):
    """(status, blob) of cldn_b200_encode_blobs on that frame alone, with this handle."""
    if fr.cloud is None:
        return INVALID, None
    rc, _, blobs, guards, _ = base._encode_blobs(enc, [fr.cloud], True, caps=[fr.cap], dims=[fr.dims] if fr.dims else None)
    assert guards
    return rc, (blobs[0] if rc == 0 else None)


def _check(enc, frames, want=None, oracle=None, spare=0):
    """Async call vs encode_blobs frame by frame; want overrides the reference status of some frames (the async refusal).
    A frame refused before the encode must leave its output as it was."""
    info = enc.getEncodingInfo()
    st, wr, bodies, guards, spare_ok = _run_async(enc, frames, spare)
    assert guards, "a byte outside a frame's buffer changed"
    assert spare_ok, "a frame past the call's frames was touched"
    blobs = []
    for f, fr in enumerate(frames):
        ref_st, ref_blob = _reference(enc, fr)
        expect = (want or {}).get(f, ref_st)
        assert st[f] == expect, (f, st[f], expect, ref_st)
        if st[f] == OK:
            got = bodies[f][:wr[f]].tobytes()
            assert _same_blob(got, ref_blob), f"frame {f} differs from encode_blobs"
            if oracle is not None and info.compression_opt == NONE:
                n = fr.cloud.size // info.point_step
                assert got == oracle.encode(base._with_dims(info, *(fr.dims or (n, 1))), fr.cloud), f"frame {f} differs from the oracle"
            blobs.append(got)
        else:
            assert wr[f] == 0, f
            if st[f] in (INVALID, UNSUPPORTED) or (st[f] == TOO_SMALL and ref_st == TOO_SMALL and fr.cap < base._worst(info, fr.nbytes // info.point_step, fr.dims)):
                assert (bodies[f] == base.PAD_BYTE).all(), f"refused frame {f} wrote into its output"
            blobs.append(None)
    return st, blobs


def _sizes(seed):
    rng = np.random.default_rng(seed)
    return [0, 1, 32767, 32768, 32769, MAX_POINTS] + [int(x) for x in rng.integers(2, MAX_POINTS, 1 if EMULATED else 3)]


ROUTES = {"default": {}, "generic": {"CLDN_B200_FORCE_GENERIC": "1"}, "no_fast": {"CLDN_B200_ENC_FAST": "0"}}


def _route(monkeypatch, route):
    for k in ("CLDN_B200_FORCE_GENERIC", "CLDN_B200_ENC_FAST"):
        monkeypatch.delenv(k, raising=False)
    for k, v in ROUTES[route].items():
        monkeypatch.setenv(k, v)


def _round_trip(oracle, blobs, clouds):
    """The blobs decode through decode_blobs_async as the oracle decodes the NONE blobs of the same clouds (stage 2 is
    lossless)."""
    info = cb.DecodeHeader(blobs[0])[0]
    dec = cb.PointcloudDecoder()
    dec.prepare_blobs(info, len(blobs), MAX_POINTS)
    caps = []
    for b in blobs:
        i = cb.DecodeHeader(b)[0]
        caps.append(max(i.width * i.height * i.point_step, 1))
    ins = [base._Buf(len(b), True, src=b) for b in blobs]
    outs = [base._Buf(c, True, fill=0) for c in caps]
    desc = _Dev(cb.blob_descs([(i.ptr, len(b), o.ptr, c) for i, b, o, c in zip(ins, blobs, outs, caps)]))
    status = _Dev(np.full(len(blobs), 99, dtype=np.int32))
    dec.decode_blobs_async(desc.ptr, len(blobs), status.ptr)
    dec.sync()
    assert [int(s) for s in status.get()] == [OK] * len(blobs)
    for b, cloud, o, c in zip(blobs, clouds, outs, caps):
        plain = cb.DecodeHeader(b)[0]
        plain.compression_opt = NONE
        want = np.zeros(c, dtype=np.uint8)
        oracle.decode(oracle.encode(plain, cloud), want)
        assert np.array_equal(o.body(), want)


# ---- parity with encode_blobs ---------------------------------------------------------------------------------------
PARITY_LAYOUTS = [("xyzi", 5), ("xyz", 5), ("c3", 4), ("c3", 5), ("xyzirt", 5), ("gorilla", 5), ("lossless", 5), ("enc_none", 5)]


@pytest.mark.gpu
@pytest.mark.parametrize("comp", list(COMPS))
@pytest.mark.parametrize("layout,version", PARITY_LAYOUTS, ids=[f"{l}_v{v}" for l, v in PARITY_LAYOUTS])
@pytest.mark.parametrize("route", list(ROUTES))
def test_varying_point_counts_equal_encode_blobs(oracle, layout, version, comp, route, monkeypatch):
    if EMULATED and route != "default" and layout not in ("xyzi", "c3"):
        pytest.skip("the emulation runs the other routes on the layouts that switch kernels")
    _route(monkeypatch, route)
    sizes = _sizes(len(layout) * 7 + version + 3 * COMPS[comp])
    info, clouds = base._clouds(layout, sizes, 40 + version, version)
    enc = _encoder(info, COMPS[comp])
    enc.prepare_blobs(len(clouds) + 2, MAX_POINTS)
    info = enc.getEncodingInfo()
    frames = [_frame(info, c) for c in clouds]
    st, blobs = _check(enc, frames, oracle=oracle, spare=2)
    assert st == [OK] * len(frames)
    if route == "default":
        _round_trip(oracle, blobs, clouds)
    # fewer frames, in another order, with room to spare behind every blob
    order = list(reversed(range(len(clouds))))[:3]
    _check(enc, [Frame(clouds[i], frames[i].cap + 48) for i in order])


# ---- refusals among good frames -------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("comp", list(COMPS))
@pytest.mark.parametrize("layout", ["xyzi", "c3"])
def test_refused_frames_among_good_ones(layout, comp):
    info, clouds = base._clouds(layout, [5000, 32768, 32769, 2000], 9)
    enc = _encoder(info, COMPS[comp])
    enc.prepare_blobs(8, MAX_POINTS)
    info = enc.getEncodingInfo()
    good = [_frame(info, c) for c in clouds]
    step = info.point_step
    too_many = base._layout(layout, MAX_POINTS + 1, 3)[1]
    cases = {
        "not_whole_points": (Frame(np.concatenate([clouds[1], np.zeros(1, np.uint8)]), good[1].cap + 8), INVALID),
        "null_cloud": (Frame(None, good[1].cap, nbytes=clouds[1].size), INVALID),
        "dims_mismatch": (Frame(clouds[2], good[2].cap + 8, dims=(7, 5)), INVALID),
        "too_many_points": (_frame(info, too_many), UNSUPPORTED),
    }
    for at in (0, 2, 3):   # a chunk-sized frame's neighbours on both sides
        for kind, (bad, want) in cases.items():
            frames = list(good)
            frames[at] = bad
            st, _ = _check(enc, frames, want={at: want})
            assert st[at] == want and all(st[f] == OK for f in range(len(frames)) if f != at), (kind, st)
        # capacity: exactly the need is enough, one byte less is refused, on both sides of a chunk boundary
        for c in (clouds[1], clouds[2]):
            frames = list(good)
            frames[at] = _frame(info, c)
            assert _check(enc, frames)[0] == [OK] * len(frames)
            frames[at] = _frame(info, c, short=1)
            st, _ = _check(enc, frames)
            assert st[at] == TOO_SMALL and all(st[f] == OK for f in range(len(frames)) if f != at)


@pytest.mark.gpu
@pytest.mark.parametrize("comp", list(COMPS))
def test_explicit_dims_write_their_headers(comp):
    info, clouds = base._clouds("xyzirt", [6000, 4096, 0, 30000], 21)
    enc = _encoder(info, COMPS[comp])
    enc.prepare_blobs(4, MAX_POINTS)
    info = enc.getEncodingInfo()
    dims = [(100, 60), (64, 64), (0, 7), (30000, 1)]
    frames = [_frame(info, c, d) for c, d in zip(clouds, dims)]
    st, blobs = _check(enc, frames)
    assert st == [OK] * 4
    for c, d, b in zip(clouds, dims, blobs):
        assert _same_blob(b, base._alone(enc, c, True, d))


@pytest.mark.gpu
def test_v5_committed_mode_overflow_fails_its_frame_alone(oracle):
    # test_gpu_parity.py's case: a uint64 field constant for 4096 values (DeltaRle committed) and random after it costs
    # more than MaxCompressedSize; encode_blobs then fails with BUFFER_TOO_SMALL, unless the capacity is larger
    from test_gpu_parity import _int_cloud
    F = cb.FieldType
    n = 100_000
    rng = np.random.default_rng(1)
    v = rng.integers(0, 2**63, n, dtype=np.int64).astype(np.uint64) * np.uint64(2) + np.uint64(1)
    v[:4096] = np.uint64(7)
    info, cloud = _int_cloud([("u64", F.UINT64, v)], n, with_xyz=False)
    info.width, info.height = 0, 1
    _, calm = _int_cloud([("u64", F.UINT64, np.full(n, 3, dtype=np.uint64))], n, with_xyz=False)
    enc = cb.PointcloudEncoder(info)
    enc.prepare_blobs(3, n)
    over = _frame(info, cloud)
    st, _ = _check(enc, [_frame(info, calm), over, _frame(info, calm)], oracle=oracle)
    assert st == [OK, TOO_SMALL, OK]
    st, blobs = _check(enc, [Frame(cloud, over.cap + 2 * n)])
    assert blobs[0] == oracle.encode(base._with_dims(info, n, 1), cloud, cap=over.cap + 2 * n)
    assert st == [OK] and len(blobs[0]) > over.cap


@pytest.mark.gpu
@pytest.mark.parametrize("comp", list(COMPS))
@pytest.mark.parametrize("layout", ["xyzi", "xyz", "xyzirt"])
def test_misaligned_clouds_give_the_same_blobs(layout, comp):
    info, clouds = base._clouds(layout, [3000, 32769, 1025], 31)
    enc = _encoder(info, COMPS[comp])
    enc.prepare_blobs(3, MAX_POINTS)
    info = enc.getEncodingInfo()
    aligned = _check(enc, [_frame(info, c) for c in clouds])[1]
    for off in (4, 8):
        frames = [_frame(info, c) for c in clouds]
        for fr in frames[1:]:
            fr.offset = off
        assert all(_same_blob(x, y) for x, y in zip(_check(enc, frames)[1], aligned))


# ---- asynchrony, graphs, launches, concurrency ------------------------------------------------------------------------
def _xyzi(n, seed):
    return base._layout("xyzi", n, seed)


@pytest.mark.gpu
@pytest.mark.skipif(EMULATED, reason="needs a CUDA stream")
def test_the_call_returns_before_the_stream_runs():
    import torch
    s = torch.cuda.Stream()
    info = _xyzi(1, 0)[0]
    info.compression_opt = LZ4
    enc = cb.PointcloudEncoder(info, stream=s.cuda_stream)
    enc.prepare_blobs(6, MAX_POINTS)
    clouds = [_xyzi(5000 * (k + 1), k)[1] for k in range(6)]
    frames = [_frame(info, c) for c in clouds]
    srcs = [_src(fr) for fr in frames]
    outs = [base._Buf(fr.cap, True) for fr in frames]
    desc = cb.pack_cloud_descs([(p, fr.nbytes, o.ptr, fr.cap) for (_, p), fr, o in zip(srcs, frames, outs)])
    status = torch.full((6,), 99, dtype=torch.int32, device="cuda")
    written = torch.zeros(6, dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        torch.cuda._sleep(200_000_000)   # ~0.1 s of the stream ahead of the call
    enc.encode_blobs_async(desc.data_ptr(), 6, status.data_ptr(), written.data_ptr())
    assert not s.query(), "the call waited for the stream"
    s.synchronize()
    assert status.cpu().tolist() == [0] * 6
    for fr, o, w in zip(frames, outs, written.cpu().tolist()):
        assert o.body()[:w].tobytes() == _reference(enc, fr)[1]


@pytest.mark.gpu
@pytest.mark.skipif(EMULATED, reason="needs CUDA graphs")
@pytest.mark.parametrize("comp", list(COMPS))
@pytest.mark.parametrize("layout", ["xyzi", "c3"])
def test_captured_graph_replays_new_clouds_in_the_same_buffers(layout, comp):
    import torch
    s = torch.cuda.Stream()
    info = base._layout(layout, 1, 0)[0]
    info.compression_opt = COMPS[comp]
    enc = cb.PointcloudEncoder(info, stream=s.cuda_stream)
    if COMPS[comp] == ZSTD:
        enc.set_stage2_on_device(True)
    n_max = 8
    enc.prepare_blobs(n_max, MAX_POINTS)
    step = info.point_step
    cloud_cap = MAX_POINTS * step + 64
    blob_cap = base._worst(info, MAX_POINTS) + 4096
    clouds_t = torch.zeros(n_max * cloud_cap, dtype=torch.uint8, device="cuda")
    outs = torch.zeros(n_max * blob_cap, dtype=torch.uint8, device="cuda")
    desc = torch.zeros(n_max * 40, dtype=torch.uint8, device="cuda")
    status = torch.zeros(n_max, dtype=torch.int32, device="cuda")
    written = torch.zeros(n_max, dtype=torch.int64, device="cuda")

    def load(clouds, caps, nbytes):
        for f, c in enumerate(clouds):
            clouds_t[f * cloud_cap:f * cloud_cap + c.size].copy_(torch.from_numpy(c))
        outs.fill_(base.PAD_BYTE)
        cb.pack_cloud_descs([(clouds_t.data_ptr() + f * cloud_cap, nbytes[f], outs.data_ptr() + f * blob_cap, caps[f])
                             for f in range(len(clouds))], out=desc)
        torch.cuda.synchronize()

    first = [base._layout(layout, 1000 * (f + 1), f)[1] for f in range(n_max)]
    load(first, [base._worst(info, c.size // step) for c in first], [c.size for c in first])
    with torch.cuda.stream(s):   # warm-up outside the capture
        enc.encode_blobs_async(desc.data_ptr(), n_max, status.data_ptr(), written.data_ptr())
    s.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        enc.encode_blobs_async(desc.data_ptr(), n_max, status.data_ptr(), written.data_ptr())
    for rnd in range(3):
        rng = np.random.default_rng(rnd)
        sizes = [int(x) for x in rng.integers(0, MAX_POINTS, n_max)]
        sizes[rnd] = MAX_POINTS
        clouds = [base._layout(layout, n, 100 * rnd + f)[1] for f, n in enumerate(sizes)]
        caps = [base._worst(info, n) for n in sizes]
        nbytes = [c.size for c in clouds]
        bad = (rnd + 3) % n_max
        if rnd == 0:
            caps[bad] -= 1
        elif rnd == 1:
            nbytes[bad] += 1
        else:
            caps[bad] = max(caps[bad], base._worst(info, MAX_POINTS + 1))
            nbytes[bad] = (MAX_POINTS + 1) * step
        load(clouds, caps, nbytes)
        g.replay()
        torch.cuda.synchronize()
        got, sizes_w = status.cpu().tolist(), written.cpu().tolist()
        host = outs.cpu().numpy()
        assert got[bad] == [TOO_SMALL, INVALID, UNSUPPORTED][rnd], (rnd, got)
        assert (host[bad * blob_cap:(bad + 1) * blob_cap] == base.PAD_BYTE).all()
        for f in range(n_max):
            if f == bad:
                continue
            ref = _reference(enc, Frame(clouds[f], caps[f]))
            assert got[f] == ref[0] == OK, (rnd, f, got[f])
            assert host[f * blob_cap:f * blob_cap + sizes_w[f]].tobytes() == ref[1], (rnd, f)
    # a call the prepared shape cannot hold, and an encoder never prepared, fail inside a capture
    for e, n in ((enc, n_max + 1), (cb.PointcloudEncoder(info, stream=s.cuda_stream), 1)):
        g2 = torch.cuda.CUDAGraph()
        with pytest.raises(RuntimeError):
            with torch.cuda.graph(g2, stream=s):
                e.encode_blobs_async(desc.data_ptr(), n, status.data_ptr())
    torch.cuda.synchronize()


@pytest.mark.gpu
@pytest.mark.parametrize("comp", list(COMPS))
@pytest.mark.parametrize("layout", ["xyzi", "c3", "gorilla"])
def test_launches_per_call_do_not_depend_on_the_frames(layout, comp):
    info, pool = base._clouds(layout, [0, 1, 5000, 32769, MAX_POINTS], 8)
    enc = _encoder(info, COMPS[comp])
    enc.prepare_blobs(len(pool), MAX_POINTS)
    info = enc.getEncodingInfo()
    counts = set()
    for sel in ([0], [4], [1, 3], list(range(len(pool)))):
        before = cb.kernel_launch_count()
        st, _, _, _, _ = _run_async(enc, [_frame(info, pool[i]) for i in sel])
        counts.add(cb.kernel_launch_count() - before)
        assert st == [OK] * len(sel)
    assert len(counts) == 1, counts


@pytest.mark.gpu
@pytest.mark.skipif(EMULATED, reason="needs CUDA streams")
def test_two_handles_on_two_streams_equal_each_call_alone():
    import torch
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    info = _xyzi(1, 0)[0]
    info.compression_opt = ZSTD
    encs = [cb.PointcloudEncoder(info, stream=s.cuda_stream) for s in streams]
    sets = [[_xyzi(int(n), k)[1] for k, n in enumerate(np.random.default_rng(seed).integers(1, MAX_POINTS, 5))] for seed in (40, 80)]
    for e in encs:
        e.set_stage2_on_device(True)
        e.prepare_blobs(5, MAX_POINTS)
    runs = []
    for clouds in sets:
        frames = [_frame(info, c) for c in clouds]
        srcs = [_src(fr) for fr in frames]
        outs = [base._Buf(fr.cap, True) for fr in frames]
        desc = cb.pack_cloud_descs([(p, fr.nbytes, o.ptr, fr.cap) for (_, p), fr, o in zip(srcs, frames, outs)])
        status = torch.full((5,), 99, dtype=torch.int32, device="cuda")
        written = torch.zeros(5, dtype=torch.int64, device="cuda")
        torch.cuda.synchronize()
        runs.append((frames, srcs, outs, desc, status, written))
    for e, (_, _, _, desc, status, written) in zip(encs, runs):   # both enqueued before either is waited for
        e.encode_blobs_async(desc.data_ptr(), 5, status.data_ptr(), written.data_ptr())
    torch.cuda.synchronize()
    for e, (frames, _, outs, _, status, written) in zip(encs, runs):
        assert status.cpu().tolist() == [0] * 5
        alone = _run_async(e, frames)
        for f, (o, w) in enumerate(zip(outs, written.cpu().tolist())):
            assert o.body()[:w].tobytes() == alone[2][f][:alone[1][f]].tobytes() == _reference(e, frames[f])[1]


@pytest.mark.gpu
def test_prepare_refusals_and_other_calls_keep_working(oracle):
    info, clouds = base._clouds("xyzi", [3000, 30000, 0], 60)
    enc = cb.PointcloudEncoder(info)
    with pytest.raises(RuntimeError):
        enc.encode_blobs_async(0, 1, 0)           # nothing prepared
    with pytest.raises(RuntimeError):
        enc.prepare_blobs(0, MAX_POINTS)
    with pytest.raises(RuntimeError):
        enc.prepare_blobs(3, 2**32)
    zinfo = base._layout("xyzi", 1, 0)[0]
    zinfo.compression_opt = ZSTD
    with pytest.raises(RuntimeError):
        cb.PointcloudEncoder(zinfo).prepare_blobs(3, MAX_POINTS)   # ZSTD needs the device coder
    enc.prepare_blobs(3, MAX_POINTS)
    frames = [_frame(info, c) for c in clouds]
    first = _check(enc, frames, oracle=oracle)[1]
    # encode, encode_batch, encode_blobs and set_dims between async calls change neither result
    host = enc.encode(clouds[0])
    assert base._encode_blobs(enc, clouds, True)[0] == 0
    src, out = base._src(clouds[0], True), base._Buf(frames[0].cap, True)
    batch = enc.encode_blobs_device([src.ptr], [clouds[0].size], [out.ptr], [frames[0].cap])
    assert cb.lib().cldn_b200_encoder_set_dims(enc._h, 10, 300) == 0
    assert _check(enc, frames, oracle=oracle)[1] == first
    assert cb.lib().cldn_b200_encoder_set_dims(enc._h, 0, 1) == 0
    assert enc.encode(clouds[0]) == host and batch[0] == len(first[0])
    # set_stage2_on_device applies from the next prepare: a ZSTD shape prepared with the device coder stays prepared
    zenc = cb.PointcloudEncoder(zinfo)
    zenc.set_stage2_on_device(True)
    zenc.prepare_blobs(3, MAX_POINTS)
    zframes = [_frame(zinfo, c) for c in clouds]
    zst = _check(zenc, zframes)[1]   # (ZSTD blobs do not depend on the lane order)
    zenc.set_stage2_on_device(False)
    st, _, bodies, _, _ = _run_async(zenc, zframes)
    assert st == [OK] * 3 and all(b[:len(z)].tobytes() == z for b, z in zip(bodies, zst))
    with pytest.raises(RuntimeError):
        zenc.prepare_blobs(3, MAX_POINTS)


# ---- the same file under the CPU emulation ---------------------------------------------------------------------------
@pytest.mark.skipif(EMULATED, reason="already running under the emulation")
@pytest.mark.parametrize("order", ["fwd", "rand"])
def test_this_file_under_emulation(lib_built, order):
    from test_cusim_kernels import _run_gpu_suite
    import platform
    if platform.machine() != "x86_64":
        pytest.skip("cusim's context switch is x86-64 only")
    sys.path.insert(0, os.path.join(ROOT, "tests", "cusim"))
    import build_cusim
    # 4 SMs: a persistent XYZI grid of few CTAs, which take tile slots (real and empty) by ticket
    env = {"CUSIM_ORDER": order, "CUSIM_WORKERS": "8", "CUSIM_SMS": "4"}
    if order == "rand":
        env["CUSIM_JITTER"] = "1"
    out = _run_gpu_suite(build_cusim.build(), env, ["tests/test_gpu_encode_blobs_async.py"])
    assert " passed" in out and "failed" not in out


@pytest.mark.skipif(EMULATED, reason="already running under the emulation")
def test_async_encode_under_thread_sanitizer(lib_built, tmp_path):
    # tests/cusim/encode_blobs_async_racecheck_main.cpp: encode_blobs_async calls of NONE / LZ4 / ZSTD with refused frames
    # and empty tile and chunk slots, every CUDA thread a ThreadSanitizer fiber (strict model: a shuffle is no fence)
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
    drv, exe = str(tmp_path / "encode_async_main.o"), str(tmp_path / "encode_async_racecheck")
    subprocess.check_call(["g++", "-std=c++17", "-O0", "-g", "-fPIC", "-pthread", "-w", "-fsanitize=thread", "-I", here, "-I",
                           os.path.join(ROOT, "include"), "-x", "c++", "-c", os.path.join(here, "encode_blobs_async_racecheck_main.cpp"), "-o", drv])
    subprocess.check_call(["g++", "-fsanitize=thread", "-pthread", "-o", exe, drv, *objs, "-ldl"])
    env = dict(os.environ, TSAN_OPTIONS="halt_on_error=0 report_signal_unsafe=0", CUSIM_WORKERS="4", CUSIM_TSAN_STRICT="1",
               CUSIM_SMS="2")   # 2 SMs: a persistent XYZI grid of few CTAs drawing tickets for real and empty tile slots
    env.pop("LD_PRELOAD", None)
    r = subprocess.run([exe], env=env, capture_output=True, text=True, timeout=1500)
    if "FATAL: ThreadSanitizer" in r.stderr:
        pytest.skip("ThreadSanitizer cannot run in this environment: " + r.stderr[-200:])
    assert r.returncode == 0 and "encode_blobs_async_racecheck: done" in r.stdout, r.stdout[-2000:] + r.stderr[-3000:]
    assert "WARNING: ThreadSanitizer" not in r.stderr, r.stderr[-4000:]
