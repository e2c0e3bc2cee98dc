"""The device ZSTD decompressor (cloudini_b200/csrc/cldn_zstd.cu) against libzstd, without a GPU (tests/cusim).

tests/cusim/zstd_main.cpp runs the unmodified kernel source under the CUDA emulation on one chunk body per launch. The
contract it checks is the one the host-pointer API relies on: for every body, the kernel produces exactly the bytes of
ZSTD_decompress(dst, cap, body, size), and fails exactly when ZSTD_decompress fails, also on damaged input.

The corpus is compressed here with the system libzstd (ctypes) from stage-1 chunks of the C oracle: levels 1 / 3 / 19 / -5,
a content checksum, no content size, streaming with a flush every few KB (many blocks per frame: treeless literals and
repeat tables), a constant chunk, 0 / 1 / 3-point chunks, two frames with a skippable frame between them. A block-header
inspector counts which format features the corpus exercises; the test fails if one of them is missing.
"""
import ctypes as C
import os
import platform
import random
import struct
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HERE = os.path.join(ROOT, "tests", "cusim")
sys.path.insert(0, HERE)
sys.path.insert(0, ROOT)

pytestmark = pytest.mark.skipif(platform.machine() != "x86_64", reason="cusim's context switch is x86-64 only")


# ---- libzstd through ctypes ------------------------------------------------------------------------------------------
class _In(C.Structure):
    _fields_ = [("src", C.c_void_p), ("size", C.c_size_t), ("pos", C.c_size_t)]


class _Out(C.Structure):
    _fields_ = [("dst", C.c_void_p), ("size", C.c_size_t), ("pos", C.c_size_t)]


def zstd_lib():
    try:
        z = C.CDLL("libzstd.so.1")
    except OSError:
        pytest.skip("libzstd.so.1 is not installed")
    z.ZSTD_compress.restype = C.c_size_t
    z.ZSTD_compress.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_int]
    z.ZSTD_decompress.restype = C.c_size_t
    z.ZSTD_decompress.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]
    z.ZSTD_isError.restype = C.c_uint
    z.ZSTD_isError.argtypes = [C.c_size_t]
    z.ZSTD_compressBound.restype = C.c_size_t
    z.ZSTD_compressBound.argtypes = [C.c_size_t]
    z.ZSTD_createCCtx.restype = C.c_void_p
    z.ZSTD_freeCCtx.argtypes = [C.c_void_p]
    z.ZSTD_CCtx_setParameter.restype = C.c_size_t
    z.ZSTD_CCtx_setParameter.argtypes = [C.c_void_p, C.c_int, C.c_int]
    z.ZSTD_compress2.restype = C.c_size_t
    z.ZSTD_compress2.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]
    z.ZSTD_compressStream2.restype = C.c_size_t
    z.ZSTD_compressStream2.argtypes = [C.c_void_p, C.POINTER(_Out), C.POINTER(_In), C.c_int]
    return z


C_LEVEL, C_CONTENT_SIZE, C_CHECKSUM = 100, 200, 201
E_CONTINUE, E_FLUSH, E_END = 0, 1, 2


def compress(z, data: bytes, level=1, checksum=None, content_size=None) -> bytes:
    cap = z.ZSTD_compressBound(len(data))
    dst = C.create_string_buffer(cap)
    if checksum is None and content_size is None:
        r = z.ZSTD_compress(dst, cap, data, len(data), level)
    else:
        cc = z.ZSTD_createCCtx()
        z.ZSTD_CCtx_setParameter(cc, C_LEVEL, level)
        if checksum is not None:
            z.ZSTD_CCtx_setParameter(cc, C_CHECKSUM, int(checksum))
        if content_size is not None:
            z.ZSTD_CCtx_setParameter(cc, C_CONTENT_SIZE, int(content_size))
        r = z.ZSTD_compress2(cc, dst, cap, data, len(data))
        z.ZSTD_freeCCtx(cc)
    assert not z.ZSTD_isError(r)
    return dst.raw[:r]


def compress_flushing(z, data: bytes, level: int, every: int) -> bytes:
    """Streaming compression with ZSTD_e_flush every `every` bytes: many blocks in one (windowed) frame."""
    cc = z.ZSTD_createCCtx()
    z.ZSTD_CCtx_setParameter(cc, C_LEVEL, level)
    cap = z.ZSTD_compressBound(len(data)) + 64 * (len(data) // every + 2)
    dst = C.create_string_buffer(cap)
    src = C.create_string_buffer(data, len(data))
    out = _Out(C.cast(dst, C.c_void_p), cap, 0)
    for start in range(0, len(data) + 1, every):
        end = min(start + every, len(data))
        inp = _In(C.cast(src, C.c_void_p).value + start, end - start, 0)
        op = E_END if end == len(data) else E_FLUSH
        while True:
            r = z.ZSTD_compressStream2(cc, C.byref(out), C.byref(inp), op)
            assert not z.ZSTD_isError(r)
            if r == 0 and inp.pos == inp.size:
                break
        if op == E_END:
            break
    z.ZSTD_freeCCtx(cc)
    return dst.raw[:out.pos]


def decompress(z, body: bytes, cap: int):
    """(ok, bytes) of ZSTD_decompress(dst, cap, body, len(body))."""
    dst = C.create_string_buffer(max(cap, 1))
    r = z.ZSTD_decompress(dst, cap, body, len(body))
    if z.ZSTD_isError(r):
        return False, b""
    return True, dst.raw[:r]


# ---- corpus --------------------------------------------------------------------------------------------------------
def split_chunks(payload: bytes):
    out, pos = [], 0
    while pos < len(payload):
        (n,) = struct.unpack_from("<I", payload, pos)
        out.append(payload[pos + 4:pos + 4 + n])
        pos += 4 + n
    return out


def stage1_chunks():
    """Stage-1 chunk bodies (C oracle, no stage 2) of the C2, C3 and C4 layouts, plus 1- and 3-point chunks."""
    import cloudini_b200 as cb
    from cloudini_b200 import synth
    from oracle.client import PortOracle
    port = PortOracle()
    chunks = {}
    for name, (info, cloud) in (("c2", synth.cloud_c2(40_000, seed=2)), ("c3", synth.cloud_c3(33_000, seed=3)),
                                ("c4", synth.cloud_c4_mixed_frame(0)), ("c2_1pt", synth.cloud_c2(1, seed=5)),
                                ("c2_3pt", synth.cloud_c2(3, seed=6))):
        info.compression_opt = cb.CompressionOption.NONE
        body = split_chunks(port.encode(info, cloud, write_header=False))
        for k, c in enumerate(body[:2]):
            chunks[f"{name}_{k}"] = c
    return chunks


def hand_frames():
    """Frames libzstd's compressor does not write on its own: a 0-point chunk (empty body), a raw literals section with
    a 2-byte count of 0 sequences, a 1-byte and a 4-byte content size, a dictionary-ID field of 0, and raw / RLE blocks
    above the 128 KB block maximum (accepted by ZSTD_decompress)."""
    def frame(fhd, extra, blocks):
        return struct.pack("<I", 0xFD2FB528) + bytes([fhd]) + extra + b"".join(blocks)

    def bh(last, btype, size):
        v = (size << 3) | (btype << 1) | last
        return struct.pack("<I", v)[:3]
    raw = bytes(range(200))
    out = {
        "empty_body": b"",
        "fcs1_raw": frame(0x20, bytes([200]), [bh(1, 0, 200) + raw]),                       # single segment, 1-byte FCS
        "fcs4_did0": frame(0x81 | 0x20, bytes([0]) + struct.pack("<I", 200), [bh(1, 0, 200) + raw]),  # 1-byte DID 0, 4-byte FCS
        "windowed_raw": frame(0x00, bytes([0x08]), [bh(0, 0, 100) + raw[:100], bh(1, 0, 100) + raw[100:]]),
        # compressed block: raw literals (5 bytes) + a 2-byte sequence count of 0 (then the modes byte, predefined tables)
        "nseq_long0": frame(0x20, bytes([5]), [bh(1, 2, 1 + 5 + 3) + bytes([5 << 3]) + b"abcde" + bytes([0x80, 0x00, 0x00])]),
        # RLE literals: libzstd writes them only for a block whose > 63 literals are one byte value
        "rle_literals": frame(0x20, bytes([20]), [bh(1, 2, 3) + bytes([(20 << 3) | 1, 0x41, 0])]),
        "raw_200k": frame(0x00, bytes([0x30]), [bh(1, 0, 200_000) + bytes(random.Random(1).randbytes(200_000))]),
        "rle_300k": frame(0x00, bytes([0x30]), [bh(1, 1, 300_000) + b"\x07"]),
    }
    return out


def build_corpus(z):
    """name -> frame bytes (all valid: libzstd decompresses every one)."""
    chunks = stage1_chunks()
    corpus = {}
    for name, data in chunks.items():
        for lvl in (1, 3, 19, -5):
            corpus[f"{name}_L{lvl}"] = compress(z, data, lvl)
    big = chunks["c4_0"]
    corpus["c4_checksum"] = compress(z, big, 1, checksum=1)
    corpus["c2_checksum_L19"] = compress(z, chunks["c2_0"], 19, checksum=1)
    corpus["c4_no_content_size"] = compress(z, big, 1, content_size=0)
    corpus["c3_no_content_size"] = compress(z, chunks["c3_0"], 3, content_size=0)
    for lvl in (1, 3, 19):
        corpus[f"c4_flush4k_L{lvl}"] = compress_flushing(z, big, lvl, 4096)
        corpus[f"c2_flush3k_L{lvl}"] = compress_flushing(z, chunks["c2_0"], lvl, 3000)
    corpus["constant"] = compress(z, bytes([0x5A]) * 40_000, 1)
    corpus["small_text"] = compress(z, b"cloudini " * 3, 1)
    a, b = compress(z, chunks["c3_1"], 1), compress(z, chunks["c2_1pt_0"], 3)
    corpus["two_frames_skippable"] = a + struct.pack("<II", 0x184D2A5B, 5) + b"skip!" + b
    # inputs shaped to bring out the rarer table modes: one record changing in one byte (RLE offset / literal-length
    # codes) and word-like text flushed every KB (treeless literals: a block reusing the previous Huffman table)
    rng = random.Random(3)
    seg = bytes(rng.randrange(256) for _ in range(64))
    corpus["runs_flush1k_L1"] = compress_flushing(z, b"".join(seg + b"A" * (1 + rng.randrange(2)) for _ in range(1500)), 1, 1024)
    rec, recs = bytearray(rng.randbytes(32)), []
    for _ in range(2000):
        rec[5] = rng.randrange(256)
        recs.append(bytes(rec))
    corpus["records_flush4k_L3"] = compress_flushing(z, b"".join(recs), 3, 4096)
    words = [bytes(rng.choice(b"etaoinshrdlu") for _ in range(rng.randrange(2, 9))) for _ in range(400)]
    corpus["words_flush1k_L3"] = compress_flushing(z, b" ".join(rng.choice(words) for _ in range(12000)), 3, 1024)
    corpus.update(hand_frames())
    return corpus


# ---- block-header inspector --------------------------------------------------------------------------------------------
def inspect(body: bytes, feats: dict):
    """Counts the format features of `body` (a valid ZSTD chunk body) into feats."""
    def add(k):
        feats[k] = feats.get(k, 0) + 1
    pos = 0
    while len(body) - pos >= 5:
        (magic,) = struct.unpack_from("<I", body, pos)
        if magic & 0xFFFFFFF0 == 0x184D2A50:
            add("skippable_frame")
            (sz,) = struct.unpack_from("<I", body, pos + 4)
            pos += 8 + sz
            continue
        add("frame")
        fhd = body[pos + 4]
        single, fcs_code, did_code = (fhd >> 5) & 1, fhd >> 6, fhd & 3
        add("single_segment" if single else "windowed_frame")
        if fhd & 4:
            add("checksum")
        fcs_size = (single if fcs_code == 0 else 1 << fcs_code)
        add(f"fcs_bytes_{fcs_size}")
        p = pos + 5 + (0 if single else 1) + (0, 1, 2, 4)[did_code] + fcs_size
        while True:
            (h,) = struct.unpack_from("<I", body[p:p + 3] + b"\0")
            last, btype, bsize = h & 1, (h >> 1) & 3, h >> 3
            p += 3
            add(("raw_block", "rle_block", "compressed_block")[btype])
            if btype == 2:
                blk = body[p:p + bsize]
                lt, lhl = blk[0] & 3, (blk[0] >> 2) & 3
                add(("raw_literals", "rle_literals", "huffman_literals", "treeless_literals")[lt])
                if lt <= 1:
                    lh = (1, 2, 1, 3)[lhl]
                    lsz = (blk[0] >> 3) if lh == 1 else (struct.unpack_from("<H", blk)[0] >> 4 if lh == 2 else (blk[0] | blk[1] << 8 | blk[2] << 16) >> 4)
                    used = lh + (lsz if lt == 0 else 1)
                else:
                    add("huffman_1_stream" if lhl == 0 else "huffman_4_streams")
                    (lhc,) = struct.unpack_from("<I", blk)
                    if lhl <= 1:
                        lh, csz = 3, (lhc >> 14) & 0x3FF
                    elif lhl == 2:
                        lh, csz = 4, lhc >> 18
                    else:
                        lh, csz = 5, (lhc >> 22) + (blk[4] << 10)
                    if lt == 2:
                        add("huffman_weights_direct" if blk[lh] >= 128 else "huffman_weights_fse")
                    used = lh + csz
                ns = blk[used]
                q = used + 1
                if ns == 0:
                    add("no_sequences")
                else:
                    if ns == 255:
                        q += 2
                    elif ns >= 128:
                        q += 1
                    modes = blk[q]
                    for name, m in (("ll", modes >> 6), ("of", (modes >> 4) & 3), ("ml", (modes >> 2) & 3)):
                        add(f"{name}_" + ("predefined", "rle", "fse", "repeat")[m])
            p += 1 if btype == 1 else bsize
            if last:
                break
        if fhd & 4:
            p += 4
        pos = p


REQUIRED = ["frame", "skippable_frame", "single_segment", "windowed_frame", "checksum", "fcs_bytes_0", "fcs_bytes_1", "fcs_bytes_2",
            "fcs_bytes_4", "raw_block", "rle_block", "compressed_block", "raw_literals", "rle_literals", "huffman_literals",
            "treeless_literals", "huffman_1_stream", "huffman_4_streams", "huffman_weights_fse", "no_sequences",
            "ll_predefined", "ll_rle", "ll_fse", "ll_repeat", "of_predefined", "of_rle", "of_fse", "of_repeat",
            "ml_predefined", "ml_rle", "ml_fse", "ml_repeat"]


# ---- the emulated kernel ---------------------------------------------------------------------------------------------
def build_driver(variant="plain"):
    """tests/cusim/_build/zstd_<variant>: zstd_main.cpp + the emulated cldn_zstd.cu / cldn_lz4.cu (+ cusim.cpp)."""
    import build_cusim
    out_dir = os.path.join(build_cusim.OUT_DIR, "zstd_" + variant)
    gen = os.path.join(out_dir, "csrc")
    os.makedirs(gen, exist_ok=True)
    for f in os.listdir(build_cusim.CSRC):
        with open(os.path.join(build_cusim.CSRC, f)) as fh:
            text = fh.read()
        with open(os.path.join(gen, f), "w") as fh:
            fh.write(build_cusim.transform(text, f))
    common = ["-std=c++17", "-g", "-fPIC", "-ffp-contract=off", "-fno-strict-aliasing", "-pthread", "-I", HERE, "-I", gen, "-w"]
    exe = os.path.join(out_dir, "zstd_main")
    srcs = [os.path.join(gen, "cldn_zstd.cu"), os.path.join(gen, "cldn_lz4.cu"), os.path.join(HERE, "zstd_main.cpp"), os.path.join(HERE, "cusim.cpp")]
    objs, procs = [], []
    for src in srcs:
        flags = list(common)
        own = src.endswith("cusim.cpp")
        if variant == "plain":
            flags.append("-O1")
        elif variant == "asan":
            ub = "alignment,shift-exponent,float-cast-overflow,integer-divide-by-zero"
            flags += ["-O1", "-fsanitize=address", "-fsanitize=" + ub, "-fno-sanitize-recover=" + ub, "-fno-omit-frame-pointer"]
        else:  # tsan: kernels and driver instrumented, the scheduler announces its fibers (see build_cusim.build_racecheck)
            flags += ["-O0"] + (["-DCUSIM_TSAN=1"] if own else ["-fsanitize=thread"])
        obj = os.path.join(out_dir, os.path.basename(src) + ".o")
        procs.append((src, obj, subprocess.Popen(["g++", *flags, "-x", "c++", "-c", src, "-o", obj], stdout=subprocess.PIPE,
                                                 stderr=subprocess.STDOUT, text=True)))
    for src, obj, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            raise RuntimeError(f"g++ failed on {src}:\n{out[-4000:]}")
        objs.append(obj)
    link = {"plain": [], "asan": ["-fsanitize=address", "-fsanitize=alignment,shift-exponent,float-cast-overflow,integer-divide-by-zero"],
            "tsan": ["-fsanitize=thread"]}[variant]
    subprocess.check_call(["g++", "-pthread", *link, "-o", exe, *objs, "-ldl"])
    return exe


def run_kernel(exe, cases, tmp_path, env=None):
    """cases: [(cap, body)] -> [(ok, bytes)] from the emulated kernel."""
    src, dst = str(tmp_path / "cases.bin"), str(tmp_path / "results.bin")
    with open(src, "wb") as f:
        f.write(struct.pack("<I", len(cases)))
        for cap, body in cases:
            f.write(struct.pack("<II", cap, len(body)) + body)
    r = subprocess.run([exe, src, dst], env=dict(os.environ, **(env or {})), capture_output=True, text=True, timeout=3000)
    assert r.returncode == 0 and "zstd_main: done" in r.stdout, r.stdout[-2000:] + r.stderr[-4000:]
    out, raw, pos = [], open(dst, "rb").read(), 0
    for _ in cases:
        ok, n = struct.unpack_from("<II", raw, pos)
        pos += 8
        out.append((bool(ok), raw[pos:pos + n]))
        pos += n
    return out, r


def cap_for(z, body):
    ok, data = decompress(z, body, 1 << 22)
    return max(len(data), 1) + 64 if ok else 1 << 20


def damage(rng, body: bytes) -> bytes:
    """One seeded corruption: bit flips, truncation, forged block size, forged table header bytes, appended bytes."""
    b = bytearray(body)
    kind = rng.randrange(6)
    if not b:
        return bytes([rng.randrange(256) for _ in range(rng.randrange(1, 12))])
    if kind == 0:
        for _ in range(rng.randrange(1, 4)):
            i = rng.randrange(len(b))
            b[i] ^= 1 << rng.randrange(8)
    elif kind == 1:
        del b[rng.randrange(len(b)):]
    elif kind == 2 and len(b) > 12:   # block header: first block after a frame header of 5..14 bytes
        i = rng.randrange(5, min(len(b) - 3, 18))
        v = int.from_bytes(b[i:i + 3], "little") ^ (1 << rng.randrange(3, 24))
        b[i:i + 3] = v.to_bytes(3, "little")
    elif kind == 3 and len(b) > 20:   # bytes where literal / sequence / table headers sit
        for _ in range(rng.randrange(1, 3)):
            i = rng.randrange(5, min(len(b), 64))
            b[i] = rng.randrange(256)
    elif kind == 4 and len(b) > 8:    # the end of the sequence bitstream (offsets, lengths, final states)
        i = len(b) - 1 - rng.randrange(min(len(b) - 1, 24))
        b[i] ^= 1 << rng.randrange(8)
    else:
        b += bytes([rng.randrange(256) for _ in range(rng.randrange(1, 6))])
    return bytes(b)


@pytest.fixture(scope="module")
def z():
    return zstd_lib()


@pytest.fixture(scope="module")
def corpus(z):
    return build_corpus(z)


@pytest.fixture(scope="module")
def driver():
    return build_driver("plain")


def test_corpus_covers_the_format(corpus):
    feats = {}
    for body in corpus.values():
        inspect(body, feats)
    missing = [k for k in REQUIRED if not feats.get(k)]
    assert not missing, f"the corpus lacks {missing}: {feats}"


def test_every_frame_decodes_to_libzstd_bytes(z, corpus, driver, tmp_path):
    names = sorted(corpus)
    cases = [(cap_for(z, corpus[k]), corpus[k]) for k in names]
    got, _ = run_kernel(driver, cases, tmp_path)
    for name, (cap, body), (ok, data) in zip(names, cases, got):
        want = decompress(z, body, cap)
        assert want[0], name
        assert (ok, data) == want, name


def test_output_bound_is_the_capacity(z, corpus, driver, tmp_path):
    # exactly the decompressed size fits; one byte less fails, as ZSTD_decompress with that capacity does
    names = [k for k in sorted(corpus) if decompress(z, corpus[k], 1 << 22)[1]][:12]
    cases = []
    for k in names:
        n = len(decompress(z, corpus[k], 1 << 22)[1])
        cases += [(n, corpus[k]), (n - 1, corpus[k])]
    got, _ = run_kernel(driver, cases, tmp_path)
    for (cap, body), res in zip(cases, got):
        assert res == decompress(z, body, cap), cap


def _known_gap(body, res, want):
    """The one documented difference (see the damaged-frames test): accepted here, refused by libzstd, 4 Huffman streams."""
    feats = {}
    try:
        inspect(body, feats)
    except (IndexError, struct.error):
        pass
    return res[0] and not want[0] and bool(feats.get("huffman_4_streams"))


def _damaged_cases(z, corpus, count, seed):
    rng = random.Random(seed)
    names = sorted(k for k in corpus if len(corpus[k]) < 200_000)
    cases = []
    for _ in range(count):
        body = damage(rng, corpus[names[rng.randrange(len(names))]])
        cases.append((cap_for(z, body) if rng.random() < 0.8 else rng.randrange(1, 1 << 18), body))
    return cases


def test_damaged_frames_fail_exactly_when_libzstd_fails(z, corpus, driver, tmp_path):
    n = int(os.environ.get("CLDN_ZSTD_DAMAGED", "3000"))
    cases = _damaged_cases(z, corpus, n, seed=20260)
    got, _ = run_kernel(driver, cases, tmp_path)
    bad, lenient = [], []
    for i, ((cap, b), res) in enumerate(zip(cases, got)):
        want = decompress(z, b, cap)
        if res == want:
            continue
        # Known gap: libzstd's 4-stream fast Huffman loop checks, where its bulk loop happens to stop, that no stream has
        # read more than 8 bytes before its own start; the kernel models the loop's leniency but not that stop point, so
        # such a stream may be accepted here and refused by libzstd. Never the other way round, never other bytes.
        if _known_gap(b, res, want):
            lenient.append(i)
        else:
            bad.append((i, len(b), cap))
    accepted = sum(1 for ok, _ in got if ok)
    assert not bad, f"{len(bad)} of {n} differ from libzstd (first: {bad[:5]}); {accepted} accepted"
    assert len(lenient) <= n // 1000, lenient
    assert 0 < accepted < n   # both outcomes occur


def test_racecheck_under_thread_sanitizer(z, corpus, tmp_path):
    # every lane is a ThreadSanitizer fiber, CUSIM_TSAN_STRICT: a shuffle is no fence; an unsynchronised pair of accesses
    # to the shared tables, the literal scratch or the output slot is a report
    try:
        exe = build_driver("tsan")
    except (RuntimeError, subprocess.CalledProcessError) as e:
        pytest.skip(f"ThreadSanitizer toolchain unavailable: {e}")
    keep = ["c4_0_L1", "c4_flush4k_L19", "c2_0_L19", "c3_0_L3", "c4_checksum", "two_frames_skippable", "constant", "nseq_long0"]
    cases = [(cap_for(z, corpus[k]), corpus[k]) for k in keep] + _damaged_cases(z, corpus, 40, seed=7)
    env = {"TSAN_OPTIONS": "halt_on_error=0 report_signal_unsafe=0", "CUSIM_TSAN_STRICT": "1", "CUSIM_WORKERS": "2"}
    got, r = run_kernel(exe, cases, tmp_path, env)
    if "FATAL: ThreadSanitizer" in r.stderr:
        pytest.skip("ThreadSanitizer cannot run in this environment")
    assert r.stderr.count("WARNING: ThreadSanitizer") == 0, r.stderr[-4000:]
    for (cap, body), res in zip(cases, got):
        want = decompress(z, body, cap)
        assert res == want or _known_gap(body, res, want)


@pytest.mark.skipif(not os.environ.get("CLDN_CUSIM_ASAN"), reason="opt-in (CLDN_CUSIM_ASAN=1): the decompressor under AddressSanitizer")
def test_no_out_of_bounds_access_under_asan(z, corpus, tmp_path):
    exe = build_driver("asan")
    cases = [(cap_for(z, corpus[k]), corpus[k]) for k in sorted(corpus)] + _damaged_cases(z, corpus, 600, seed=11)
    got, r = run_kernel(exe, cases, tmp_path, {"ASAN_OPTIONS": "detect_leaks=0"})
    assert "AddressSanitizer" not in r.stderr, r.stderr[-4000:]
    for (cap, body), res in zip(cases, got):
        want = decompress(z, body, cap)
        assert res == want or _known_gap(body, res, want)
