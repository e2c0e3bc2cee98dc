"""The encode routes against each other: every memory kind and stage-2 placement must return the same status for the
same cloud and capacity, and where they succeed, blobs whose chunks are the same stage-1 bytes, so the same points.

The clouds are V5 frames whose committed mode costs more than MaxCompressedSize budgets (see
test_gpu_parity.py::test_v5_committed_mode_can_exceed_max_compressed_size): one whose stage-1 bytes overflow the
compressed routes' stage-1 arena, and one whose overflow fits in the arena's slack.
"""
import ctypes as C

import numpy as np
import pytest

import cloudini_b200 as cb
from test_gpu_parity import _int_cloud
from test_gpu_zstd_encode import DEVICE, MEMS, _chunks, _lz4, _payload, _run
from zstd_corpus import decompress, zstd_lib

pytestmark = pytest.mark.gpu

NONE, LZ4, ZSTD = cb.CompressionOption.NONE, cb.CompressionOption.LZ4, cb.CompressionOption.ZSTD


def _committed_mode_cloud(n, comp):
    """A uint64 field that is constant for its first 4096 values (DeltaRle is committed) and random after them."""
    rng = np.random.default_rng(1)
    v = rng.integers(0, 2**63, n, dtype=np.int64).astype(np.uint64) * np.uint64(2) + np.uint64(1)
    v[:4096] = np.uint64(7)
    info, cloud = _int_cloud([("u64", cb.FieldType.UINT64, v)], n, with_xyz=False)
    info.compression_opt = comp
    return info, cloud


def _stage1(blob, comp, sizes):
    """The chunks of a blob decompressed by libzstd / liblz4, given the size of each stage-1 chunk."""
    out = []
    for body, size in zip(_chunks(_payload(blob)), sizes):
        if comp == ZSTD:
            ok, plain = decompress(zstd_lib(), body, size)
            out.append(plain if ok else None)
        else:
            buf = C.create_string_buffer(size + 1)
            out.append(buf.raw[:size] if _lz4().LZ4_decompress_safe(body, buf, len(body), size + 1) == size else None)
    return out


# 100_000 points: 2134 stage-1 bytes over MaxCompressedSize, more than the arena's 64 bytes per chunk and 64 more.
# 93_700 points: 108 bytes over, within the arena's 256 bytes of slack.
@pytest.mark.parametrize("n,comp", [
    (100_000, LZ4), (100_000, ZSTD), (93_700, ZSTD),
    pytest.param(93_700, LZ4, marks=pytest.mark.xfail(strict=True, reason=(
        "the device LZ4 coder gives each chunk a slot of LZ4_COMPRESSBOUND of the per-chunk MaxCompressedSize; a chunk "
        "past it makes lz4_compress_chunks_kernel raise DEV_ERR_LZ4 (CLDN_ERR_CORRUPT_DATA, 'LZ4 decompression "
        "failed'), while liblz4 runs out of the caller's capacity (CLDN_ERR_BUFFER_TOO_SMALL)"))),
])
def test_committed_mode_overflow_is_the_same_on_every_route(oracle, n, comp):
    info, cloud = _committed_mode_cloud(n, comp)
    plain = _committed_mode_cloud(n, NONE)[0]
    want = _chunks(oracle.encode(plain, cloud, write_header=False, cap=2 * cb.MaxCompressedSize(info, n, True)))
    outcomes = {}
    for on_device in (False, True):
        enc = cb.PointcloudEncoder(info)
        enc.set_stage2_on_device(on_device)
        for mem in MEMS:
            if mem == DEVICE and comp == ZSTD and not on_device:
                continue  # ZSTD into device blobs needs the device coder
            rc, msg, blobs, guards = _run(enc, "batch", [cloud], mem)
            assert guards, (mem, on_device)
            outcomes[(mem, on_device)] = (rc, msg, _stage1(blobs[0], comp, [len(c) for c in want]) if rc == 0 else None)
    assert len({rc for rc, _, _ in outcomes.values()}) == 1, {k: v[:2] for k, v in outcomes.items()}
    for route, (rc, _, stage1) in outcomes.items():
        assert rc != 0 or stage1 == want, route
