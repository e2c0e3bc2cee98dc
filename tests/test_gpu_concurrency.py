"""Distinct handles used at the same time: several host threads, each with its own encoder / decoder / preprocessor, and
handles bound to the caller's streams. A single handle is not thread-safe; distinct handles are (one handle per thread
or stream, include/cloudini_b200.h), and that is how the DDS converter's per-thread handle pools, a node decoding several
topics and bench.py's end-to-end pipelines use the library.

Every expected result is computed on the main thread before any worker starts: by the oracle where it has the answer,
else by the same call made alone. Device buffers are allocated and read back on the main thread; the workers only call
the library. Every output is compared bit for bit, device buffers sit between guard bytes and decode outputs are
pre-filled, so a write outside a frame's own bytes is seen.
"""
import ctypes as C
import os
import threading
import traceback

import numpy as np
import pytest

import cloudini_b200 as cb
from cloudini_b200 import ros, synth
from test_gpu_decode_blobs import EMULATED, PAD_BYTE, _Buf, _check_batch, _damaged, _need

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NONE, LZ4 = cb.CompressionOption.NONE, cb.CompressionOption.LZ4
ROUNDS = 3


def _run_threads(workers):
    """Starts every worker at once (barrier) and re-raises the first failure with its thread's traceback."""
    errors = [None] * len(workers)
    gate = threading.Barrier(len(workers))

    def run(k):
        try:
            gate.wait()
            workers[k]()
        except BaseException:   # noqa: B902 -- reported on the main thread
            errors[k] = traceback.format_exc()

    threads = [threading.Thread(target=run, args=(k,)) for k in range(len(workers))]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    failed = [e for e in errors if e]
    assert not failed, "\n".join(failed)


def _want_points(oracle, info, cloud):
    """The oracle's decode of the oracle's encode of `cloud` (NONE stage 2), into a pre-filled buffer."""
    i = cb.EncodingInfo(**{**info.__dict__, "compression_opt": NONE})
    out = np.full(cloud.size, PAD_BYTE, dtype=np.uint8)
    oracle.decode(oracle.encode(i, cloud), out)
    return out


# ---- a. one layout per thread, host and device APIs ---------------------------------------------------------------------
def _layouts():
    n = 12_000 if EMULATED else 60_000
    xyzi_n = 20_000 if EMULATED else 300_000   # 4 x 300k points: 1172 tiles, more than the persistent encoder's grid
    yield "c2_xyzi", synth.cloud_c2(xyzi_n, seed=1), NONE, 4
    yield "c1", synth.cloud_c1(n, seed=2, adversarial=True), NONE, 2
    yield "c3_v5", synth.cloud_c3(n + 3, seed=3), NONE, 2
    info, cloud = synth.cloud_c4_mixed_frame(2, az=256 if EMULATED else 2032)
    yield "xyzirt", (info, cloud), NONE, 2
    yield "livox", synth.cloud_livox(n, seed=5), NONE, 2
    yield "gorilla", synth.cloud_lossless(n // 2, seed=6), NONE, 2
    yield "lz4_xyzi", synth.cloud_c2(xyzi_n // 2, seed=7), LZ4, 2


class _Case:
    """One thread's layout and rounds: the host API, an asynchronous device batch and a synchronous device batch."""

    def __init__(self, oracle, name, info, clouds, comp):
        self.name, self.comp, self.frames = name, comp, len(clouds)
        self.info = cb.EncodingInfo(**{**info.__dict__, "compression_opt": comp, "use_threads": False})
        self.clouds = clouds
        self.nbytes = clouds[0].size
        self.want_pts = [_want_points(oracle, info, c) for c in clouds]
        if comp == NONE:
            self.want_blob = [oracle.encode(self.info, c) for c in clouds]
        else:   # LZ4 blocks are not canonical: the same device call made alone, whose points must be the oracle's
            self.want_blob = _device_encode_alone(self.info, clouds)
            for b, w in zip(self.want_blob, self.want_pts):
                assert np.array_equal(_device_decode_alone(b, self.nbytes), w)
        self.hinfo, self.hdr = cb.DecodeHeader(self.want_blob[0])
        self.cap = cb.MaxCompressedSize(self.info, info.width, True)
        self.kinds = [1 + r % 2 for r in range(ROUNDS)] if comp != NONE else [r % 3 for r in range(ROUNDS)]
        # device buffers for every device round, made here on the main thread
        self.d_in = [[_Buf(self.nbytes, True, src=c.tobytes()) for c in clouds] if k else None for k in self.kinds]
        self.d_out = [[_Buf(self.cap, True) for _ in clouds] if k else None for k in self.kinds]
        self.d_blob = [[_Buf(len(b), True, src=b) for b in self.want_blob] if k else None for k in self.kinds]
        self.d_pts = [[_Buf(self.nbytes, True) for _ in clouds] if k else None for k in self.kinds]
        self.host_results, self.sizes = {}, {}

    def work(self):
        enc = cb.PointcloudEncoder(self.info)
        dec = cb.PointcloudDecoder()
        for r, kind in enumerate(self.kinds):
            if kind == 0:
                blobs = [enc.encode(c) for c in self.clouds]
                outs = []
                for b in blobs:
                    out = np.full(self.nbytes, PAD_BYTE, dtype=np.uint8)
                    dec.decode(self.hinfo, b[self.hdr:], out)
                    outs.append(out)
                self.host_results[r] = (blobs, outs)
                continue
            ins, outs = self.d_in[r], self.d_out[r]
            batch = enc.make_device_batch([b.ptr for b in ins], [self.nbytes] * self.frames, [o.ptr for o in outs], [self.cap] * self.frames)
            if kind == 1:
                enc.encode_batch_device(batch)    # asynchronous
                enc.sync()
            else:
                self.sizes[r] = enc.encode_batch_device(batch, want_sizes=True)
            lens = [len(b) - self.hdr for b in self.want_blob]
            dbatch = dec.make_device_batch([b.ptr + self.hdr for b in self.d_blob[r]], lens, [o.ptr for o in self.d_pts[r]], [self.nbytes] * self.frames)
            dec.decode_batch_device(self.hinfo, dbatch, sync=(kind == 2))
            if kind == 1:
                dec.sync()
        enc.close()
        dec.close()

    def check(self):
        for r, kind in enumerate(self.kinds):
            for f in range(self.frames):
                where = (self.name, r, f)
                if kind == 0:
                    blobs, outs = self.host_results[r]
                    assert blobs[f] == self.want_blob[f], where
                    assert np.array_equal(outs[f], self.want_pts[f]), where
                    continue
                o, p = self.d_out[r][f], self.d_pts[r][f]
                assert o.body()[:len(self.want_blob[f])].tobytes() == self.want_blob[f], where
                assert np.array_equal(p.body(), self.want_pts[f]), where
                assert o.guards_intact() and p.guards_intact(), where
            if r in self.sizes:
                assert self.sizes[r] == [len(b) for b in self.want_blob], (self.name, r)


def _device_encode_alone(info, clouds):
    enc = cb.PointcloudEncoder(info)
    caps = [cb.MaxCompressedSize(info, c.size // info.point_step, True) for c in clouds]
    ins = [_Buf(c.size, True, src=c.tobytes()) for c in clouds]
    outs = [_Buf(cap, True) for cap in caps]
    sizes = enc.encode_batch_device(enc.make_device_batch([b.ptr for b in ins], [c.size for c in clouds], [o.ptr for o in outs], caps),
                                    want_sizes=True)
    return [o.body()[:s].tobytes() for o, s in zip(outs, sizes)]


def _device_decode_alone(blob, nbytes):
    info, h = cb.DecodeHeader(blob)
    dec = cb.PointcloudDecoder()
    src, dst = _Buf(len(blob) - h, True, src=blob[h:]), _Buf(nbytes, True)
    dec.decode_batch_device(info, dec.make_device_batch([src.ptr], [len(blob) - h], [dst.ptr], [nbytes]), sync=True)
    return dst.body().copy()


def _layout_cases(oracle):
    cases = []
    for name, (info, cloud), comp, frames in _layouts():
        # the frames of a batch differ: frame f is the first cloud with its points rotated by 97 f
        n = info.width
        clouds = [np.roll(cloud.reshape(n, info.point_step), 97 * f, axis=0).reshape(-1).copy() for f in range(frames)]
        cases.append(_Case(oracle, name, info, clouds, comp))
    return cases


def test_one_layout_per_thread_host_and_device_apis(oracle):
    cases = _layout_cases(oracle)
    assert len(cases) == 7
    _run_threads([c.work for c in cases])
    for c in cases:
        c.check()


# ---- b. two persistent XYZI encoders on two streams, enqueued back to back ------------------------------------------------
def test_two_device_encoders_on_two_streams_back_to_back(oracle):
    # Both grids are in flight together: each encoder's CTAs may find part of the GPU taken by the other's. Its tiles are
    # handed out in order from a ticket counter, so every tile a look-back waits for belongs to a CTA that is running.
    n, frames = (20_000, 4) if EMULATED else (300_000, 4)
    info = synth.info_xyzi(n)
    clouds = [[synth.cloud_c2(n, seed=100 + 10 * e + k)[1] for k in range(frames)] for e in range(2)]
    want = [[oracle.encode(info, c) for c in cl] for cl in clouds]
    cap = cb.MaxCompressedSize(info, n, True)
    encs = [cb.PointcloudEncoder(info) for _ in range(2)]
    reps = 2
    ins = [[[_Buf(c.size, True, src=c.tobytes()) for c in clouds[e]] for _ in range(reps)] for e in range(2)]
    outs = [[[_Buf(cap, True) for _ in range(frames)] for _ in range(reps)] for e in range(2)]
    batches = [[encs[e].make_device_batch([b.ptr for b in ins[e][r]], [n * 16] * frames, [o.ptr for o in outs[e][r]], [cap] * frames)
                for r in range(reps)] for e in range(2)]
    for r in range(reps):
        for e in range(2):
            encs[e].encode_batch_device(batches[e][r])   # asynchronous: nothing waits until all four batches are enqueued
    for e in encs:
        e.sync()
    for e in range(2):
        for r in range(reps):
            for f in range(frames):
                o = outs[e][r][f]
                assert o.body()[:len(want[e][f])].tobytes() == want[e][f], (e, r, f)
                assert o.guards_intact()


# ---- c. viz preprocessing and the DDS converter on threads ---------------------------------------------------------------
def test_viz_preprocessing_and_message_conversion_on_threads(oracle, golden_ros):
    # viz_compact_kernel needs 32,800 B of dynamic shared memory at step 16, 65,568 B at step 32 and 71,712 B at step 280:
    # threads that set the kernel's limit to what their own launch needs would lower it under each other's launches
    n = 6_000 if EMULATED else 100_000
    inputs = [synth.cloud_viz(n if step != 280 else n // 10, seed=step, step=step) for step in (16, 32, 280, 12)]
    want = [oracle.viz_preprocess(info, cloud) for info, cloud in inputs]
    got = [[] for _ in inputs]

    def viz(k):
        def run():
            pp = ros.VizPreprocessor()
            for _ in range(ROUNDS):
                got[k].append(pp.run(*inputs[k]))
        return run

    messages = list(golden_ros.items())
    converted = []

    def convert():
        for _ in range(ROUNDS):
            for name, g in messages:
                converted.append((name, ros.convert_message(g["msg"], g["profile"], g["default_resolution"], g["viz"],
                                                            cb.EncodingOptions.LOSSY, NONE, 5)))

    _run_threads([viz(k) for k in range(len(inputs))] + [convert])
    for k, (w_info, w) in enumerate(want):
        assert len(got[k]) == ROUNDS
        for g_info, g, applied in got[k]:
            assert applied and np.array_equal(g, w), inputs[k][0].point_step
            assert (g_info.width, g_info.point_step) == (w_info.width, w_info.point_step)
    assert len(converted) == ROUNDS * len(messages)
    for name, blob in converted:
        assert blob == golden_ros[name]["compressed"], name


# ---- d, e. decode_blobs on two threads; the launch counter over concurrent work ------------------------------------------
def _blobs_job(seed, damage):
    from test_gpu_decode_blobs import _mixed_blobs
    rng = np.random.default_rng(seed)
    blobs = _mixed_blobs(seed)
    blobs = [blobs[i] for i in rng.permutation(len(blobs))]
    caps = [_need(b) for b in blobs]
    for i, kind in damage:
        if kind == "short_output":
            caps[i] -= 1
        else:
            blobs[i] = _damaged(blobs[i], kind, rng)
            caps[i] = max(caps[i], _need(blobs[i]))
    return blobs, caps


class _BlobsRun:
    """One decode_blobs call on guarded device buffers made in advance."""

    def __init__(self, dec, blobs, caps):
        self.dec, self.blobs, self.caps = dec, blobs, caps
        self.ins = [_Buf(max(len(b), 1), True, src=bytes(b) + b"\0" * (len(b) == 0)) for b in blobs]
        self.outs = [_Buf(c, True) for c in caps]

    def run(self):
        n = len(self.blobs)
        status = (C.c_int32 * n)()
        rc = cb.lib().cldn_b200_decode_blobs(self.dec._h, n, (C.c_void_p * n)(*[b.ptr for b in self.ins]),
                                             (C.c_size_t * n)(*[len(b) for b in self.blobs]), (C.c_void_p * n)(*[o.ptr for o in self.outs]),
                                             (C.c_size_t * n)(*self.caps), 1, status, None)
        self.rc, self.status = rc, list(status)
        self.msgs = [self.dec.frame_error(f) for f in range(n)]

    def result(self):
        assert all(o.guards_intact() for o in self.outs) and all(i.guards_intact() for i in self.ins)
        return self.rc, self.status, self.msgs, [o.body().copy() for o in self.outs]


def test_decode_blobs_on_two_threads_and_the_launch_counter(oracle):
    jobs = [_blobs_job(3, [(2, "bitflip"), (7, "chunk_prefix"), (11, "short_output")]), _blobs_job(5, [(0, "header_line"), (5, "truncate")])]
    decs = [cb.PointcloudDecoder() for _ in jobs]
    # alone, on the main thread: the expected statuses, messages and bytes, and the launches each job makes
    alone, launches = [], []
    for dec, (blobs, caps) in zip(decs, jobs):
        st = _check_batch(oracle, blobs, True, caps)   # good frames against the oracle, every frame against its single decode
        assert any(s != 0 for s in st) and any(s == 0 for s in st)
        r = _BlobsRun(dec, blobs, caps)
        before = cb.kernel_launch_count()
        r.run()
        launches.append(cb.kernel_launch_count() - before)
        alone.append(r.result())
        assert alone[-1][1] == st
    runs = [[_BlobsRun(dec, *job) for _ in range(ROUNDS)] for dec, job in zip(decs, jobs)]
    before = cb.kernel_launch_count()
    _run_threads([lambda rs=rs: [r.run() for r in rs] for rs in runs])
    # every kernel launch of the concurrent run is counted once: the counter is atomic
    assert cb.kernel_launch_count() - before == ROUNDS * sum(launches)
    for k, rs in enumerate(runs):
        for r in rs:
            rc, st, msgs, outs = r.result()
            assert (rc, st, msgs) == alone[k][:3], k
            assert all(np.array_equal(a, b) for a, b in zip(outs, alone[k][3])), k


# ---- f. caller streams ---------------------------------------------------------------------------------------------------
@pytest.mark.skipif(EMULATED, reason="torch streams need the GPU")
def test_caller_streams_ordered_by_torch_events(oracle):
    import torch
    n, frames = 60_000, 12     # more asynchronous calls than the 8 pinned upload slots of a handle
    info = synth.info_xyzi(n)
    clouds = [synth.cloud_c2(n, seed=300 + k)[1] for k in range(frames)]
    want_blob = [oracle.encode(info, c) for c in clouds]
    want_pts = [_want_points(oracle, info, c) for c in clouds]
    hinfo, hdr = cb.DecodeHeader(want_blob[0])
    cap = cb.MaxCompressedSize(info, n, True)
    staged = [torch.from_numpy(c.copy()).cuda() for c in clouds]
    torch.cuda.synchronize()
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    enc = cb.PointcloudEncoder(info, stream=s1.cuda_stream)
    dec = cb.PointcloudDecoder(stream=s2.cuda_stream)
    with torch.cuda.stream(s1):
        ins = [t.clone() for t in staged]                      # written by torch kernels on s1, not synchronised
        outs = [torch.full((cap,), PAD_BYTE, dtype=torch.uint8, device="cuda") for _ in range(frames)]
        for k in range(frames):
            enc.encode_batch_device(enc.make_device_batch([ins[k].data_ptr()], [n * 16], [outs[k].data_ptr()], [cap]))
        done = torch.cuda.Event()
        done.record(s1)
    s2.wait_event(done)
    with torch.cuda.stream(s2):
        pts = [torch.full((n * 16,), PAD_BYTE, dtype=torch.uint8, device="cuda") for _ in range(frames)]
        for k in range(frames):
            dec.decode_batch_device(hinfo, dec.make_device_batch([outs[k].data_ptr() + hdr], [len(want_blob[k]) - hdr], [pts[k].data_ptr()], [n * 16]))
        got_blob = [outs[k][:len(want_blob[k])].cpu().numpy() for k in range(frames)]   # read with torch on s2
        got_pts = [p.cpu().numpy() for p in pts]
    enc.sync()
    dec.sync()
    for k in range(frames):
        assert got_blob[k].tobytes() == want_blob[k], k
        assert np.array_equal(got_pts[k], want_pts[k]), k


@pytest.mark.skipif(EMULATED, reason="torch streams need the GPU")
def test_preprocessor_encoder_and_decoder_sharing_one_caller_stream(oracle):
    # the DDS converter's handle pool: one stream per thread, shared by its preprocessor, encoder and decoder
    import torch
    info, cloud = synth.cloud_viz(80_000, seed=21, step=32)
    w_info, w_kept = oracle.viz_preprocess(info, cloud)
    w_info.compression_opt = NONE
    want_blob = oracle.encode(w_info, w_kept)
    want_pts = np.full(w_kept.size, PAD_BYTE, dtype=np.uint8)
    oracle.decode(want_blob, want_pts)
    hinfo, hdr = cb.DecodeHeader(want_blob)
    s = torch.cuda.Stream()
    src = torch.from_numpy(cloud.copy()).cuda()
    torch.cuda.synchronize()
    pp = ros.VizPreprocessor(stream=s.cuda_stream)
    enc = cb.PointcloudEncoder(w_info, stream=s.cuda_stream)
    dec = cb.PointcloudDecoder(stream=s.cuda_stream)
    cap = cb.MaxCompressedSize(w_info, w_info.width, True)
    with torch.cuda.stream(s):
        d_in = src.clone()
        kept = torch.full((cloud.size,), PAD_BYTE, dtype=torch.uint8, device="cuda")
        blob = torch.full((cap,), PAD_BYTE, dtype=torch.uint8, device="cuda")
        pts = torch.full((w_kept.size,), PAD_BYTE, dtype=torch.uint8, device="cuda")
        new_info, n_kept, applied = pp.run_device(info, d_in.data_ptr(), cloud.size, kept.data_ptr(), cloud.size)
        assert applied and n_kept == w_info.width
        enc.encode_batch_device(enc.make_device_batch([kept.data_ptr()], [w_kept.size], [blob.data_ptr()], [cap]))
        dec.decode_batch_device(hinfo, dec.make_device_batch([blob.data_ptr() + hdr], [len(want_blob) - hdr], [pts.data_ptr()], [w_kept.size]))
        got_kept = kept[:w_kept.size].cpu().numpy()
        got_blob = blob[:len(want_blob)].cpu().numpy().tobytes()
        got_pts = pts.cpu().numpy()
    assert np.array_equal(got_kept, w_kept)
    assert got_blob == want_blob
    assert np.array_equal(got_pts, want_pts)


# ---- g. two GPUs -----------------------------------------------------------------------------------------------------------
def _gpu_count():
    if EMULATED:
        return 1
    import torch
    return torch.cuda.device_count()


@pytest.mark.skipif(_gpu_count() < 2, reason="needs two GPUs")
def test_handles_on_two_devices_from_threads(oracle):
    # The dynamic shared memory limit is per device: device 0 raises viz_compact_kernel's limit to 71,712 B first, then
    # a thread whose current device is 0 uses device-1 handles, which must raise it on device 1 as well.
    info, cloud = synth.cloud_viz(20_000, seed=280, step=280)
    w_info, w = oracle.viz_preprocess(info, cloud)
    x_info, x_cloud = synth.cloud_c2(300_000, seed=9)
    x_want = oracle.encode(x_info, x_cloud)
    assert np.array_equal(ros.VizPreprocessor(device=0).run(info, cloud)[1], w)
    got = {0: [], 1: []}

    def on(device):
        def run():
            pp, enc = ros.VizPreprocessor(device=device), cb.PointcloudEncoder(x_info, device=device)
            for _ in range(ROUNDS):
                got[device].append((pp.run(info, cloud)[1], enc.encode(x_cloud)))
        return run

    _run_threads([on(0), on(1)])
    for device in (0, 1):
        assert len(got[device]) == ROUNDS
        for kept, blob in got[device]:
            assert np.array_equal(kept, w), device
            assert blob == x_want, device
