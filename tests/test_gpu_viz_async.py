"""cldn_b200_viz_lossy_preprocess_batch_async: the viz preprocessing of device-resident clouds of one prepared layout,
without the host, so that it and cldn_b200_encode_blobs_async can be captured in one CUDA graph.

Every frame's status, kept count, applied flag and output bytes must equal cldn_b200_viz_lossy_preprocess(...,
CLDN_MEM_DEVICE) of that cloud alone (and the oracle's applyVizLossyPreprocessing), except for the one refusal of the async
call: more points than prepared. Inputs and outputs sit between guard bytes with a pre-filled padding (the _Buf of
test_gpu_encode_blobs.py); descriptors, outputs and result entries past the call's frames hold sentinels that must
survive.
"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import cloudini_b200 as cb
from cloudini_b200 import ros, synth

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)
import test_gpu_encode_blobs as base  # noqa: E402  (guarded buffers, _special, _noop_layouts)
import test_gpu_encode_blobs_async as eba  # noqa: E402  (device arrays, blob equality)
from test_gpu_route_matrix import _viz_case, _viz_tile  # noqa: E402

EMULATED = base.EMULATED
NONE, LZ4, ZSTD = cb.CompressionOption.NONE, cb.CompressionOption.LZ4, cb.CompressionOption.ZSTD
COMPS = {"none": NONE, "lz4": LZ4, "zstd": ZSTD}
OK, INVALID, TOO_SMALL, UNSUPPORTED = 0, -1, -2, -5
MAX_POINTS = 6_000 if EMULATED else 40_000
PAD = base.PAD_BYTE
SENTINEL_DESC = (0x1111, 0x2222, 0x3333, 0x4444, 5, 6)   # a cloud_desc entry: out and capacity must survive
ST0, KEPT0, APPLIED0 = 99, 7, 55


class Frame:
    """One frame of a call: a cloud (None: a NULL cloud pointer of `nbytes`), its output capacity (None: a NULL output)
    and the offset of both device pointers past a 16-byte aligned base."""

    def __init__(self, cloud, cap=-1, nbytes=None, offset=0):
        self.cloud, self.offset = cloud, offset
        self.nbytes = cloud.size if nbytes is None else nbytes
        self.cap = self.nbytes if cap == -1 else cap


def _src(fr):
    if fr.cloud is None:
        return None, 0
    size = fr.cloud.size + fr.offset
    buf = base._Buf(max(size, 1), True, src=b"\0" * fr.offset + fr.cloud.tobytes() + b"\0" * (size == 0))
    return buf, buf.ptr + fr.offset


def _out(fr):
    if fr.cap is None:
        return None, 0
    buf = base._Buf(fr.cap + fr.offset, True)
    return buf, buf.ptr + fr.offset


def _single(pp, info, fr):
    """(status, kept, applied, output body) of cldn_b200_viz_lossy_preprocess(..., CLDN_MEM_DEVICE) on the frame alone."""
    (src, ptr), (out, optr) = _src(fr), _out(fr)
    kept, applied = C.c_size_t(0), C.c_int(0)
    rc = ros._L().cldn_b200_viz_lossy_preprocess(pp._h, C.byref(cb._to_c(info)), ptr or None, fr.nbytes, optr or None,
                                                 fr.cap or 0, C.byref(kept), C.byref(applied), cb.MEM_DEVICE)
    body = out.body()[fr.offset:].copy() if out is not None else None
    return rc, kept.value, applied.value, body


class Run:
    """One async call on guarded buffers, with `spare` descriptors, outputs and result entries past its frames."""

    def __init__(self, pp, info, frames, spare=2, encode=True):
        self.srcs = [_src(fr) for fr in frames]
        self.outs = [_out(fr) for fr in frames]
        step = info.point_step
        decoy = synth.cloud_viz(3, seed=99, step=step)[1] if step else np.zeros(0, np.uint8)
        self.decoy_src = base._Buf(max(decoy.size, 1), True, src=decoy.tobytes() + b"\0" * (decoy.size == 0))
        self.extra = [base._Buf(max(decoy.size, 1), True) for _ in range(spare)]
        descs = [(p, fr.nbytes, op, fr.cap or 0) for (_, p), (_, op), fr in zip(self.srcs, self.outs, frames)]
        descs += [(self.decoy_src.ptr, decoy.size, o.ptr, o.cap) for o in self.extra]
        n, m = len(frames), len(frames) + spare
        self.desc = eba._Dev(ros.viz_descs(descs))
        self.status = eba._Dev(np.full(m, ST0, dtype=np.int32))
        self.kept = eba._Dev(np.full(m, KEPT0, dtype=np.uint64))
        self.applied = eba._Dev(np.full(m, APPLIED0, dtype=np.int32))
        self.enc = eba._Dev(cb.cloud_descs([SENTINEL_DESC] * m)) if encode else None
        pp.run_batch_async(self.desc.ptr, n, self.status.ptr, self.kept.ptr, self.applied.ptr, self.enc.ptr if encode else 0)
        pp.sync()
        st, kept, applied = self.status.get(), self.kept.get(), self.applied.get()
        self.st, self.k, self.a = [int(x) for x in st[:n]], [int(x) for x in kept[:n]], [int(x) for x in applied[:n]]
        self.encode = self.enc.get() if encode else None
        self.bodies = [o.body()[fr.offset:].copy() if o is not None else None for (o, _), fr in zip(self.outs, frames)]
        self.guards = (all(o.guards_intact() for o, _ in self.outs if o is not None)
                       and all(b.guards_intact() and np.array_equal(b.body()[fr.offset:fr.offset + fr.cloud.size], fr.cloud)
                               for (b, _), fr in zip(self.srcs, frames) if b is not None))
        self.spare_ok = (all((o.body() == PAD).all() and o.guards_intact() for o in self.extra)
                         and (st[n:] == ST0).all() and (kept[n:] == KEPT0).all() and (applied[n:] == APPLIED0).all()
                         and (not encode or (self.encode[n:] == cb.cloud_descs([SENTINEL_DESC])[0]).all()))


def _check(pp, info, frames, want=None, oracle=None, spare=2):
    """The async call against the single call frame by frame; `want` overrides the single call's status of some frames
    (the async refusal). Returns the Run."""
    r = Run(pp, info, frames, spare)
    assert r.guards, "a byte outside a frame's buffer, or an input, changed"
    assert r.spare_ok, "something of a frame past the call's frames was touched"
    single = ros.VizPreprocessor()
    step = info.point_step
    for f, fr in enumerate(frames):
        rc, k1, a1, body1 = _single(single, info, fr)
        expect = (want or {}).get(f, rc)
        assert r.st[f] == expect, (f, r.st[f], expect, rc)
        e = r.encode[f]
        assert e[2] == SENTINEL_DESC[2] and e[3] == SENTINEL_DESC[3] and e[4] == 0, f
        if r.st[f] != OK:
            assert r.k[f] == (fr.nbytes // step if step else 0) and r.a[f] == 0, (f, r.k[f], r.a[f])
            assert r.bodies[f] is None or (r.bodies[f] == PAD).all(), f"refused frame {f} wrote into its output"
            assert e[0] == 0 and e[1] == 1, f
            continue
        assert (r.k[f], r.a[f]) == (k1, a1), (f, r.k[f], r.a[f], k1, a1)
        if not a1:
            assert r.bodies[f] is None or (r.bodies[f] == PAD).all(), f"frame {f} was not applied but its output changed"
            assert e[0] == (r.srcs[f][1] or 0) and e[1] == fr.nbytes, f
            continue
        assert np.array_equal(r.bodies[f], body1), f"frame {f} differs from the single call"
        assert (r.bodies[f][k1 * step:] == PAD).all(), f
        assert e[0] == r.outs[f][1] and e[1] == k1 * step, f
        if oracle is not None:
            o_info, o_out = oracle.viz_preprocess(info, fr.cloud)
            assert o_info.width == k1 and np.array_equal(r.bodies[f][:k1 * step], o_out), f"frame {f} differs from the oracle"
    return r


def _at(cloud, step, xo):
    """The cloud with its xyz bytes moved to offset xo (as _viz_case places them)."""
    rows = cloud.reshape(-1, step).copy()
    rows[:, xo:xo + 12] = cloud.reshape(-1, step)[:, 0:12]
    return rows.reshape(-1)


# ---- 1. every frame equals the single call and the oracle -------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("step", [12, 16, 22, 32, 280])
def test_every_frame_equals_the_single_call(oracle, step):
    tile = _viz_tile(step)
    sizes = [0, 1, tile - 1, tile, tile + 1, 2 * tile + 1, MAX_POINTS]
    pp = ros.VizPreprocessor()
    for xo in sorted({xo for xo in (0, 8, step - 12) if xo + 12 <= step}):
        info = _viz_case(step, xo, 0, 1)[0]
        info.width, info.height = 0, 1
        after = pp.prepare_batch(info, 12, MAX_POINTS)
        assert after.width == after.height == 0
        clouds = [_viz_case(step, xo, 10 * xo + k, n)[1] if n else np.zeros(0, np.uint8) for k, n in enumerate(sizes)]
        clouds += [_at(base._special("nan", 500, step, 3), step, xo), _at(base._special("one_voxel", 2000, step, 5), step, xo),
                   base._special("empty", 0, step, 7)]
        frames = [Frame(c, offset=(0, 1, 4)[k % 3]) for k, c in enumerate(clouds)]
        _check(pp, info, frames, oracle=oracle)
        # fewer frames than the last call, in another order, with room to spare
        _check(pp, info, [Frame(clouds[k], cap=clouds[k].size + 40, offset=4) for k in (6, 1, 5)], oracle=oracle)


# ---- 2. refused frames fail alone ---------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_refused_frames_fail_alone(oracle):
    info = synth.cloud_viz(1)[0]
    info.width = 0
    pp = ros.VizPreprocessor()
    pp.prepare_batch(info, 6, MAX_POINTS)
    good = [synth.cloud_viz(n, seed=k)[1] for k, n in enumerate([3000, 2049, 1, 4096])]
    big = synth.cloud_viz(MAX_POINTS + 1, seed=8)[1]
    cases = {
        "null_cloud": (Frame(None, cap=good[1].size, nbytes=good[1].size), INVALID),
        "one_byte_short": (Frame(good[1], cap=good[1].size - 1), TOO_SMALL),
        "null_out": (Frame(good[1], cap=None), TOO_SMALL),
        "too_many_points": (Frame(big), UNSUPPORTED),
    }
    for at in (0, 2, 3):
        for kind, (bad, want) in cases.items():
            frames = [Frame(c) for c in good]
            frames[at] = bad
            r = _check(pp, info, frames, want={at: want}, oracle=oracle)
            assert r.st[at] == want and all(r.st[f] == OK for f in range(len(frames)) if f != at), (kind, r.st)
    # xyz outside the point: every non-empty frame of the layout is refused, an empty one stays OK
    bad = base._with_dims(info, 0, 1)
    bad.fields = [cb.PointField(f.name, f.offset + 8, f.type, f.resolution) for f in info.fields[:3]]
    pp.prepare_batch(bad, 4, MAX_POINTS)
    r = _check(pp, bad, [Frame(good[0]), Frame(good[0][:0]), Frame(good[2])])
    assert r.st == [INVALID, OK, INVALID] and r.a == [0, 0, 0]


# ---- 3. no-op layouts -----------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_no_op_layouts_pass_every_frame_through():
    pp = ros.VizPreprocessor()
    clouds = [synth.cloud_viz(n, seed=n)[1] for n in (3000, 0, 17)]
    for name, info in base._noop_layouts():
        after = pp.prepare_batch(info, 5, MAX_POINTS)
        assert cb.EncodingInfoToYAML(after) == cb.EncodingInfoToYAML(info), name
        before = cb.kernel_launch_count()
        r = _check(pp, info, [Frame(c, offset=k) for k, c in enumerate(clouds)] + [Frame(None, nbytes=64)], want={3: INVALID})
        assert cb.kernel_launch_count() - before == 2, name
        assert r.st == [OK, OK, OK, INVALID] and r.a == [0] * 4 and r.k == [3000, 0, 17, 4], name


# ---- 4. the chain into encode_blobs_async ---------------------------------------------------------------------------------
def _float64_layout(n, seed):
    """The viz XYZI layout followed by a FLOAT64 stamp without a resolution (which the preprocessing gives 1e-6)."""
    info, cloud = synth.cloud_viz(n, seed=seed, step=24)
    rows = cloud.reshape(n, 24)
    rows[:, 16:24] = (1.7e9 + np.arange(n, dtype=np.float64) * 1e-5).view(np.uint8).reshape(n, 8)
    info.fields.append(cb.PointField("t", 16, cb.FieldType.FLOAT64, None))
    info.width = 0
    return info, rows.reshape(-1)


def _chain_clouds(layout, sizes, seed):
    if layout == "xyzi":
        info = synth.cloud_viz(1)[0]
        info.width = 0
        return info, [synth.cloud_viz(n, seed=seed + k)[1] for k, n in enumerate(sizes)]
    return _float64_layout(1, seed)[0], [_float64_layout(n, seed + k)[1] for k, n in enumerate(sizes)]


def _sync_chain(info, comp, clouds):
    """The current chain: viz_lossy_preprocess_batch, then encode_blobs (widths = heights = NULL) with an encoder created
    from an applied frame's info. Returns one blob per frame."""
    pp = ros.VizPreprocessor()
    ins = [base._src(c, True) for c in clouds]
    mid = [base._Buf(max(c.size, 1), True) for c in clouds]
    res = pp.run_batch_device(info, [b.ptr for b in ins], [c.size for c in clouds], [b.ptr for b in mid], [c.size for c in clouds])
    enc_info = next(r[0] for r in res if r[2])
    enc_info.compression_opt = comp
    enc = eba._encoder(enc_info, comp)
    kept = [k for _, k, _ in res]
    caps = [base._worst(enc_info, k) for k in kept]
    outs = [base._Buf(c, True) for c in caps]
    sizes = enc.encode_blobs_device([b.ptr for b in mid], [k * info.point_step for k in kept], [o.ptr for o in outs], caps)
    return [o.body()[:s].tobytes() for o, s in zip(outs, sizes)]


@pytest.mark.gpu
@pytest.mark.parametrize("comp", list(COMPS))
@pytest.mark.parametrize("layout", ["xyzi", "float64"])
def test_chain_into_encode_blobs_async(oracle, layout, comp):
    sizes = [5000, 0, 1, MAX_POINTS, 2049, 3000]
    info, clouds = _chain_clouds(layout, sizes, 20)
    step = info.point_step
    pp = ros.VizPreprocessor()
    after = pp.prepare_batch(info, len(clouds) + 1, MAX_POINTS)
    if layout == "float64":
        assert after.fields[4].resolution == pytest.approx(1e-6)
    after.compression_opt = COMPS[comp]
    enc = eba._encoder(after, COMPS[comp])
    enc.prepare_blobs(len(clouds) + 1, MAX_POINTS)
    bad = 4   # one frame refused by the preprocessing: its output one byte short
    frames = [Frame(c, cap=c.size - (f == bad)) for f, c in enumerate(clouds)]
    srcs, mids = [_src(fr) for fr in frames], [_out(fr) for fr in frames]
    caps = [base._worst(after, c.size // step) for c in clouds]
    blobs = [base._Buf(c, True) for c in caps]
    vdesc = eba._Dev(ros.viz_descs([(p, fr.nbytes, op, fr.cap) for (_, p), (_, op), fr in zip(srcs, mids, frames)]))
    edesc = eba._Dev(cb.cloud_descs([(0, 0, b.ptr, c) for b, c in zip(blobs, caps)]))
    n = len(frames)
    vst, est = eba._Dev(np.full(n, ST0, np.int32)), eba._Dev(np.full(n, ST0, np.int32))
    written = eba._Dev(np.zeros(n, np.uint64))
    pp.run_batch_async(vdesc.ptr, n, vst.ptr, encode_descs_ptr=edesc.ptr)
    enc.encode_blobs_async(edesc.ptr, n, est.ptr, written.ptr)
    enc.sync()
    vs, es, wr = vst.get().tolist(), est.get().tolist(), written.get().tolist()
    assert vs == [TOO_SMALL if f == bad else OK for f in range(n)], vs
    assert es == [INVALID if f == bad else OK for f in range(n)], es
    assert (blobs[bad].body() == PAD).all() and all(b.guards_intact() for b in blobs)
    want = _sync_chain(info, COMPS[comp], [c for f, c in enumerate(clouds) if f != bad])
    got = [b.body()[:w].tobytes() for f, (b, w) in enumerate(zip(blobs, wr)) if f != bad]
    good = [c for f, c in enumerate(clouds) if f != bad]
    for f, (g, w, c) in enumerate(zip(got, want, good)):
        assert eba._same_blob(g, w), f"frame {f} differs from the sync chain"
        # the reference leaves an empty cloud's info as it is, so a FLOAT64 field without a resolution keeps none there,
        # while the chain's one encoder (and the sync chain's) states 1e-6 for every frame
        if COMPS[comp] == NONE and (c.size or layout == "xyzi"):
            o_info, o_out = oracle.viz_preprocess(info, c)
            o_info.compression_opt = NONE
            assert g == oracle.encode(o_info, o_out), f"frame {f} differs from the oracle"


# ---- 5. one graph captures both calls ---------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.skipif(EMULATED, reason="needs CUDA graphs")
@pytest.mark.parametrize("comp", list(COMPS))
def test_one_graph_captures_preprocessing_and_encode(comp):
    import torch
    s = torch.cuda.Stream()
    info = synth.cloud_viz(1)[0]
    info.width = 0
    step, n_max = info.point_step, 8
    pp = ros.VizPreprocessor(stream=s.cuda_stream)
    after = pp.prepare_batch(info, n_max, MAX_POINTS)
    after.compression_opt = COMPS[comp]
    enc = cb.PointcloudEncoder(after, stream=s.cuda_stream)
    if COMPS[comp] == ZSTD:
        enc.set_stage2_on_device(True)
    enc.prepare_blobs(n_max, MAX_POINTS)
    cloud_cap = (MAX_POINTS + 1) * step + 64
    blob_cap = base._worst(after, MAX_POINTS + 1) + 4096
    clouds_t = torch.zeros(n_max * cloud_cap, dtype=torch.uint8, device="cuda")
    mid = torch.zeros(n_max * cloud_cap, dtype=torch.uint8, device="cuda")
    blobs = torch.zeros(n_max * blob_cap, dtype=torch.uint8, device="cuda")
    vdesc = torch.zeros(n_max * 32, dtype=torch.uint8, device="cuda")
    edesc = cb.pack_cloud_descs([(0, 0, blobs.data_ptr() + f * blob_cap, blob_cap) for f in range(n_max)])
    vst, est = (torch.zeros(n_max, dtype=torch.int32, device="cuda") for _ in range(2))
    kept, written = (torch.zeros(n_max, dtype=torch.int64, device="cuda") for _ in range(2))
    applied = torch.zeros(n_max, dtype=torch.int32, device="cuda")

    def call():
        pp.run_batch_async(vdesc.data_ptr(), n_max, vst.data_ptr(), kept.data_ptr(), applied.data_ptr(), edesc.data_ptr())
        enc.encode_blobs_async(edesc.data_ptr(), n_max, est.data_ptr(), written.data_ptr())

    def load(clouds, descs):
        for f, c in enumerate(clouds):
            clouds_t[f * cloud_cap:f * cloud_cap + c.size].copy_(torch.from_numpy(c))
        mid.fill_(PAD)
        blobs.fill_(PAD)
        ros.pack_viz_descs(descs, out=vdesc)
        cb.pack_cloud_descs([(0, 0, blobs.data_ptr() + f * blob_cap, blob_cap) for f in range(n_max)], out=edesc)
        torch.cuda.synchronize()

    def cloud_at(f):
        return clouds_t.data_ptr() + f * cloud_cap

    def mid_at(f):
        return mid.data_ptr() + f * cloud_cap

    first = [synth.cloud_viz(1000 * (f + 1), seed=f)[1] for f in range(n_max)]
    load(first, [(cloud_at(f), c.size, mid_at(f), cloud_cap) for f, c in enumerate(first)])
    with torch.cuda.stream(s):   # warm-up outside the capture
        call()
    s.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        call()
    for rnd in range(4):
        rng = np.random.default_rng(rnd)
        sizes = [int(x) for x in rng.integers(0, MAX_POINTS, n_max)]
        sizes[rnd] = MAX_POINTS
        bad = (rnd + 3) % n_max
        if rnd == 3:
            sizes[bad] = MAX_POINTS + 1
        clouds = [synth.cloud_viz(n, seed=100 * rnd + f)[1] for f, n in enumerate(sizes)]
        descs = [(cloud_at(f), c.size, mid_at(f), cloud_cap) for f, c in enumerate(clouds)]
        want_viz = [TOO_SMALL, INVALID, TOO_SMALL, UNSUPPORTED][rnd]
        if rnd == 0:
            descs[bad] = (cloud_at(bad), clouds[bad].size, mid_at(bad), clouds[bad].size - 1)
        elif rnd == 1:
            descs[bad] = (0, clouds[bad].size, mid_at(bad), cloud_cap)
        elif rnd == 2:
            descs[bad] = (cloud_at(bad), clouds[bad].size, 0, cloud_cap)
        load(clouds, descs)
        g.replay()
        torch.cuda.synchronize()
        vs, es = vst.cpu().tolist(), est.cpu().tolist()
        assert vs[bad] == want_viz and es[bad] == INVALID, (rnd, vs, es)
        host = blobs.cpu().numpy()
        assert (host[bad * blob_cap:(bad + 1) * blob_cap] == PAD).all()
        good = [f for f in range(n_max) if f != bad]
        want = _sync_chain(info, COMPS[comp], [clouds[f] for f in good])
        wr = written.cpu().tolist()
        for f, w in zip(good, want):
            assert vs[f] == es[f] == OK, (rnd, f, vs[f], es[f])
            assert host[f * blob_cap:f * blob_cap + wr[f]].tobytes() == w, (rnd, f)
    # a call the prepared shape cannot hold, and a preprocessor never prepared, fail inside a capture
    for p, n in ((pp, n_max + 1), (ros.VizPreprocessor(stream=s.cuda_stream), 1)):
        g2 = torch.cuda.CUDAGraph()
        with pytest.raises(RuntimeError):
            with torch.cuda.graph(g2, stream=s):
                p.run_batch_async(vdesc.data_ptr(), n, vst.data_ptr())
    torch.cuda.synchronize()


# ---- 6. launches ----------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_launches_per_call_do_not_depend_on_the_frames():
    info = synth.cloud_viz(1)[0]
    pool = [synth.cloud_viz(n, seed=n)[1] for n in (0, 1, 5000, 2049, MAX_POINTS)]
    pp = ros.VizPreprocessor()
    pp.prepare_batch(info, len(pool), MAX_POINTS)
    counts = set()
    for sel in ([0], [4], [1, 3], list(range(len(pool)))):
        before = cb.kernel_launch_count()
        r = Run(pp, info, [Frame(pool[i]) for i in sel])
        counts.add(cb.kernel_launch_count() - before)
        assert r.st == [OK] * len(sel)
    assert counts == {5}, counts


# ---- 7. prepare refusals; the other calls keep working --------------------------------------------------------------------
def _bodies(r):
    return [b.tobytes() for b in r.bodies], r.st, r.k, r.a


@pytest.mark.gpu
def test_prepare_refusals_and_other_calls_keep_working(oracle):
    info = synth.cloud_viz(1)[0]
    pp = ros.VizPreprocessor()
    with pytest.raises(RuntimeError):
        pp.run_batch_async(0, 1, 0)                 # nothing prepared
    with pytest.raises(RuntimeError):
        pp.prepare_batch(info, 0, MAX_POINTS)
    with pytest.raises(RuntimeError):
        pp.prepare_batch(info, 3, 2**30 + 1)
    with pytest.raises(RuntimeError):
        pp.prepare_batch(info, 2**31, 10)
    pp.prepare_batch(info, 3, MAX_POINTS)
    with pytest.raises(RuntimeError):
        pp.run_batch_async(0, 1, 0)                 # NULL descriptors
    empty = eba._Dev(np.full(4, ST0, np.int32))
    pp.run_batch_async(empty.ptr, 0, empty.ptr)     # no frames: no work
    pp.sync()
    assert (empty.get() == ST0).all()
    clouds = [synth.cloud_viz(n, seed=n + 1)[1] for n in (3000, 4097, 0)]
    first = _bodies(_check(pp, info, [Frame(c) for c in clouds], oracle=oracle))
    # the single and batch calls between async calls give what a fresh handle gives, and change nothing of the async state
    fresh = ros.VizPreprocessor()
    other = [synth.cloud_viz(n, seed=n + 5)[1] for n in (700, 9000)]
    for c in other:
        assert [x.tobytes() for x in pp.run(info, c)[1:2]] == [x.tobytes() for x in fresh.run(info, c)[1:2]]
    got = pp.run_batch(info, other)
    assert [g[1].tobytes() for g in got] == [g[1].tobytes() for g in fresh.run_batch(info, other)]
    assert _bodies(_check(pp, info, [Frame(c) for c in clouds])) == first
    # a new prepare with another layout
    info32 = synth.cloud_viz(1, step=32)[0]
    pp.prepare_batch(info32, 2, MAX_POINTS)
    _check(pp, info32, [Frame(synth.cloud_viz(n, seed=n, step=32)[1]) for n in (2500, 1)], oracle=oracle)


# ---- 8. two preprocessors on two streams ----------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.skipif(EMULATED, reason="needs CUDA streams")
def test_two_preprocessors_on_two_streams():
    import torch
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    info = synth.cloud_viz(1)[0]
    pps = [ros.VizPreprocessor(stream=s.cuda_stream) for s in streams]
    for p in pps:
        p.prepare_batch(info, 5, MAX_POINTS)
    sets = [[synth.cloud_viz(int(n), seed=k + seed)[1] for k, n in enumerate(np.random.default_rng(seed).integers(1, MAX_POINTS, 5))]
            for seed in (40, 80)]
    runs = []
    for clouds in sets:
        frames = [Frame(c) for c in clouds]
        srcs, outs = [_src(fr) for fr in frames], [_out(fr) for fr in frames]
        desc = ros.pack_viz_descs([(p, fr.nbytes, op, fr.cap) for (_, p), (_, op), fr in zip(srcs, outs, frames)])
        status = torch.full((5,), ST0, dtype=torch.int32, device="cuda")
        kept = torch.zeros(5, dtype=torch.int64, device="cuda")
        torch.cuda.synchronize()
        runs.append((frames, srcs, outs, desc, status, kept))
    for p, (_, _, _, desc, status, kept) in zip(pps, runs):   # both enqueued before either is waited for
        p.run_batch_async(desc.data_ptr(), 5, status.data_ptr(), kept.data_ptr())
    torch.cuda.synchronize()
    single = ros.VizPreprocessor()
    for (frames, _, outs, _, status, kept) in runs:
        assert status.cpu().tolist() == [OK] * 5
        for fr, (o, _), k in zip(frames, outs, kept.cpu().tolist()):
            rc, k1, _, body = _single(single, info, fr)
            assert rc == OK and k == k1 and np.array_equal(o.body(), body)


# ---- 9. the same file under the CPU emulation ---------------------------------------------------------------------------
def _x86():
    import platform
    if platform.machine() != "x86_64":
        pytest.skip("cusim's context switch is x86-64 only")


@pytest.mark.skipif(EMULATED, reason="already running under the emulation")
@pytest.mark.parametrize("order", ["fwd", "rand"])
def test_this_file_under_emulation(lib_built, order):
    from test_cusim_kernels import _run_gpu_suite
    _x86()
    sys.path.insert(0, os.path.join(ROOT, "tests", "cusim"))
    import build_cusim
    env = {"CUSIM_ORDER": order, "CUSIM_WORKERS": "8"}
    if order == "rand":
        env["CUSIM_JITTER"] = "1"
    out = _run_gpu_suite(build_cusim.build(), env, ["tests/test_gpu_viz_async.py"])
    assert " passed" in out and "failed" not in out


@pytest.mark.skipif(EMULATED, reason="already running under the emulation")
def test_this_file_with_host_checks(lib_built):
    # CUSIM_HOSTCHECK=1: every cudaMalloc region is inaccessible to host code outside a kernel or a copy, so a host read of
    # a descriptor or a count fails; CUSIM_ASYNC=1: a device-to-host copy reads as garbage until the host synchronises
    from test_cusim_kernels import _run_gpu_suite
    _x86()
    sys.path.insert(0, os.path.join(ROOT, "tests", "cusim"))
    import build_cusim
    out = _run_gpu_suite(build_cusim.build(), {"CUSIM_HOSTCHECK": "1", "CUSIM_ASYNC": "1"}, ["tests/test_gpu_viz_async.py"])
    assert " passed" in out and "failed" not in out


@pytest.mark.skipif(EMULATED, reason="already running under the emulation")
def test_async_viz_under_thread_sanitizer(lib_built, tmp_path):
    # tests/cusim/viz_async_racecheck_main.cpp: async calls with refused frames, empty frame slots and partial last tiles,
    # every CUDA thread a ThreadSanitizer fiber (strict model: a shuffle is no fence)
    _x86()
    here = os.path.join(ROOT, "tests", "cusim")
    sys.path.insert(0, here)
    import build_cusim
    from cloudini_b200.build import SOURCES
    try:
        build_cusim.build_racecheck()
    except subprocess.CalledProcessError as e:
        pytest.skip(f"ThreadSanitizer toolchain unavailable: {e}")
    objs = [os.path.join(build_cusim.OUT_DIR, os.path.splitext(s)[0] + "_tsan.o") for s in SOURCES + ["cusim.cpp"]]
    drv, exe = str(tmp_path / "viz_async_main.o"), str(tmp_path / "viz_async_racecheck")
    subprocess.check_call(["g++", "-std=c++17", "-O0", "-g", "-fPIC", "-pthread", "-w", "-fsanitize=thread", "-I", here, "-I",
                           os.path.join(ROOT, "include"), "-x", "c++", "-c", os.path.join(here, "viz_async_racecheck_main.cpp"), "-o", drv])
    subprocess.check_call(["g++", "-fsanitize=thread", "-pthread", "-o", exe, drv, *objs, "-ldl"])
    env = dict(os.environ, TSAN_OPTIONS="halt_on_error=0 report_signal_unsafe=0", CUSIM_WORKERS="4", CUSIM_TSAN_STRICT="1")
    env.pop("LD_PRELOAD", None)
    r = subprocess.run([exe], env=env, capture_output=True, text=True, timeout=1500)
    if "FATAL: ThreadSanitizer" in r.stderr:
        pytest.skip("ThreadSanitizer cannot run in this environment: " + r.stderr[-200:])
    assert r.returncode == 0 and "viz_async_racecheck: done" in r.stdout, r.stdout[-2000:] + r.stderr[-3000:]
    assert "WARNING: ThreadSanitizer" not in r.stderr, r.stderr[-4000:]
