"""The device ZSTD decompressor (cloudini_b200/csrc/cldn_zstd.cu) against libzstd, without a GPU (tests/cusim).

tests/cusim/zstd_main.cpp runs the unmodified kernel source under the CUDA emulation on one chunk body per launch. The
contract it checks is the one the host-pointer API relies on: for every body, the kernel produces exactly the bytes of
ZSTD_decompress(dst, cap, body, size), and fails exactly when ZSTD_decompress fails, also on damaged input.

The corpus is compressed here with the system libzstd (ctypes) from stage-1 chunks of the C oracle: levels 1 / 3 / 19 / -5,
a content checksum, no content size, streaming with a flush every few KB (many blocks per frame: treeless literals and
repeat tables), a constant chunk, 0 / 1 / 3-point chunks, two frames with a skippable frame between them. A block-header
inspector counts which format features the corpus exercises; the test fails if one of them is missing. The libzstd
bindings, the hand-written frames, the inspector and the corruption live in tests/zstd_corpus.py, which
tests/test_gpu_zstd_format.py shares to run the same format features through the product's API on the GPU.
"""
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

from zstd_corpus import REQUIRED, _known_gap, compress, compress_flushing, damage, decompress, hand_frames, inspect, zstd_lib  # noqa: E402

pytestmark = pytest.mark.skipif(platform.machine() != "x86_64", reason="cusim's context switch is x86-64 only")


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
