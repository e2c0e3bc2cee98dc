"""ZSTD corpus helpers shared by the device decompressor's tests (tests/test_cusim_zstd.py under the CPU emulation,
tests/test_gpu_zstd_format.py on the GPU): libzstd through ctypes, frames libzstd's compressor does not write on its own,
a block-header inspector that names the format features a body uses, and a seeded corruption.
"""
import ctypes as C
import random
import struct

import pytest


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


# ZSTD_cParameter values (zstd.h, stable API)
C_LEVEL, C_WINDOW_LOG, C_STRATEGY, C_CONTENT_SIZE, C_CHECKSUM, C_LDM = 100, 101, 107, 200, 201, 160
E_CONTINUE, E_FLUSH, E_END = 0, 1, 2


def compress(z, data: bytes, level=1, checksum=None, content_size=None, **params) -> bytes:
    """One frame of `data`. params: window_log, strategy (1 fast .. 9 btultra2), ldm (long-distance matching)."""
    cap = z.ZSTD_compressBound(len(data))
    dst = C.create_string_buffer(cap)
    if checksum is None and content_size is None and not params:
        r = z.ZSTD_compress(dst, cap, data, len(data), level)
    else:
        cc = z.ZSTD_createCCtx()
        z.ZSTD_CCtx_setParameter(cc, C_LEVEL, level)
        if checksum is not None:
            z.ZSTD_CCtx_setParameter(cc, C_CHECKSUM, int(checksum))
        if content_size is not None:
            z.ZSTD_CCtx_setParameter(cc, C_CONTENT_SIZE, int(content_size))
        for key, p in (("window_log", C_WINDOW_LOG), ("strategy", C_STRATEGY), ("ldm", C_LDM)):
            if key in params:
                assert not z.ZSTD_isError(z.ZSTD_CCtx_setParameter(cc, p, int(params[key]))), key
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


# ---- frames written by hand ------------------------------------------------------------------------------------------
def _frame(fhd, extra, blocks):
    return struct.pack("<I", 0xFD2FB528) + bytes([fhd]) + extra + b"".join(blocks)


def _bh(last, btype, size):
    v = (size << 3) | (btype << 1) | last
    return struct.pack("<I", v)[:3]


def _lit_header(ltype, n):
    """Raw (0) / RLE (1) literals section header for n literals: 1 byte below 32, else 2 bytes (n < 4096)."""
    if n < 32:
        return bytes([(n << 3) | ltype])
    assert n < 4096
    return struct.pack("<H", (n << 4) | (1 << 2) | ltype)


BLOCK_MAX = 131072   # Block_Maximum_Size


def hand_frames(step=None):
    """Frames libzstd's compressor does not write on its own: a 0-point chunk (empty body), a raw literals section with
    a 2-byte count of 0 sequences, a 1-byte and a 4-byte content size, a dictionary-ID field of 0, and raw / RLE blocks
    above the 128 KB block maximum (accepted by ZSTD_decompress).

    With `step`, every frame decompresses to a whole number of step-byte points, so that it is a valid chunk body of a
    layout whose stage 1 is a plain copy; the empty body, and blocks that would exceed one 32768-point chunk, are left out."""
    def size(n):   # n bytes, or the nearest whole number of points at or above it (at least one)
        return n if step is None else max(1, -(-n // step)) * step

    def fits(n):
        return step is None or n <= 32768 * step
    def whole(n):   # n bytes, or the whole points below it
        return n if step is None else n // step * step
    rng = random.Random(1)
    n200, n5, n20 = max(size(1), whole(200)), size(5), size(20)
    raw = bytes(range(200)) if step is None else bytes(rng.randrange(256) for _ in range(n200))
    lits = b"abcde" if step is None else bytes(rng.randrange(256) for _ in range(n5))
    lh5, lh20 = _lit_header(0, n5), _lit_header(1, n20)
    out = {
        # single segment, 1-byte FCS
        "fcs1_raw": _frame(0x20, bytes([n200]), [_bh(1, 0, n200) + raw]),
        # 1-byte DID 0, 4-byte FCS
        "fcs4_did0": _frame(0x81 | 0x20, bytes([0]) + struct.pack("<I", n200), [_bh(1, 0, n200) + raw]),
        "windowed_raw": _frame(0x00, bytes([0x08]), [_bh(0, 0, n200 // 2) + raw[:n200 // 2], _bh(1, 0, n200 - n200 // 2) + raw[n200 // 2:]]),
        # compressed block: raw literals + a 2-byte sequence count of 0 (then the modes byte, predefined tables)
        "nseq_long0": _frame(0x20, bytes([n5]), [_bh(1, 2, len(lh5) + n5 + 3) + lh5 + lits + bytes([0x80, 0x00, 0x00])]),
        # RLE literals: libzstd writes them only for a block whose > 63 literals are one byte value
        "rle_literals": _frame(0x20, bytes([n20]), [_bh(1, 2, len(lh20) + 2) + lh20 + bytes([0x41, 0])]),
    }
    if step is None:
        out["empty_body"] = b""
    big_raw, big_rle = whole(200_000), whole(300_000)
    if fits(big_raw) and big_raw > BLOCK_MAX:
        out["raw_200k"] = _frame(0x00, bytes([0x30]), [_bh(1, 0, big_raw) + bytes(random.Random(1).randbytes(big_raw))])
    if fits(big_rle) and big_rle > BLOCK_MAX:
        out["rle_300k"] = _frame(0x00, bytes([0x30]), [_bh(1, 1, big_rle) + b"\x07"])
    if step is not None and 32768 * step > BLOCK_MAX:   # a full chunk of one byte value: one RLE block
        out["rle_full_chunk"] = _frame(0x00, bytes([0x48]), [_bh(1, 1, 32768 * step) + b"\x3c"])
    return out


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


# ---- damage --------------------------------------------------------------------------------------------------------
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


def _known_gap(body, res, want):
    """The one documented difference (cldn_zstd.cu, top): accepted by the kernel, refused by libzstd, 4 Huffman streams."""
    feats = {}
    try:
        inspect(body, feats)
    except (IndexError, struct.error):
        pass
    return res[0] and not want[0] and bool(feats.get("huffman_4_streams"))
