"""cloudini_b200 — host-side Python mirror of the reference's codec interface on top of the C ABI.

The product is ``lib/libcloudini_b200.so`` (hand-written sm_90a kernels behind ``include/cloudini_b200.h``). This
module only binds it with ctypes and mirrors the names of the reference's public API
(``cloudini_lib/include/cloudini_lib/cloudini.hpp``): ``EncodingInfo``, ``PointField``, ``EncodeHeader``,
``DecodeHeader``, ``MaxCompressedSize``, ``PointcloudEncoder.encode`` and ``PointcloudDecoder.decode`` — same argument
meaning, same error behaviour (``RuntimeError`` where the reference throws ``std::runtime_error``).

There is no CPU implementation here: without the compiled library (or without a GPU for the compute calls) every
entry point raises.
"""
from __future__ import annotations

import ctypes as C
import enum
import os
from dataclasses import dataclass, field, replace
from typing import List, Optional, Sequence

__all__ = [
    "FieldType", "EncodingOptions", "CompressionOption", "PointField", "EncodingInfo", "EncodingInfoToYAML",
    "EncodingInfoFromYAML", "EncodeHeader", "DecodeHeader", "MaxCompressedSize", "PointcloudEncoder",
    "PointcloudDecoder", "SizeOf", "lib", "library_path", "kernel_launch_count", "kDecodeButSkipStore",
]

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.environ.get("CLDN_B200_LIB") or os.path.join(_HERE, "lib", "libcloudini_b200.so")
CLDN_MAX_FIELDS = 32
CLDN_MAX_NAME = 64
kDecodeButSkipStore = 0xFFFFFFFF  # basic_types.hpp:71
MEM_HOST, MEM_DEVICE = 0, 1
MEM_DEVICE_POINTS = 2  # points (clouds, decoded outputs) in device memory, blobs and payloads in host memory


class FieldType(enum.IntEnum):  # basic_types.hpp:29-48
    UNKNOWN = 0
    INT8 = 1
    UINT8 = 2
    INT16 = 3
    UINT16 = 4
    INT32 = 5
    UINT32 = 6
    FLOAT32 = 7
    FLOAT64 = 8
    INT64 = 9
    UINT64 = 10


class EncodingOptions(enum.IntEnum):  # cloudini.hpp:31-43
    NONE = 0
    LOSSY = 1
    LOSSLESS = 2


class CompressionOption(enum.IntEnum):  # cloudini.hpp:45-53
    NONE = 0
    LZ4 = 1
    ZSTD = 2


def SizeOf(t: FieldType) -> int:  # basic_types.hpp:73-96
    return {1: 1, 2: 1, 3: 2, 4: 2, 5: 4, 6: 4, 7: 4, 8: 8, 9: 8, 10: 8}.get(int(t), 0)


@dataclass
class PointField:  # basic_types.hpp:50-66
    name: str = ""
    offset: int = 0
    type: FieldType = FieldType.UNKNOWN
    resolution: Optional[float] = None


@dataclass
class EncodingInfo:  # cloudini.hpp:65-111
    fields: List[PointField] = field(default_factory=list)
    width: int = 0
    height: int = 1
    point_step: int = 0
    encoding_opt: EncodingOptions = EncodingOptions.LOSSY
    encoding_config: str = ""
    compression_opt: CompressionOption = CompressionOption.ZSTD
    use_threads: bool = True
    version: int = 5


class _CField(C.Structure):
    _fields_ = [("name", C.c_char * CLDN_MAX_NAME), ("offset", C.c_uint32), ("type", C.c_uint8),
                ("has_resolution", C.c_uint8), ("reserved_", C.c_uint8 * 2), ("resolution", C.c_float)]


class _CInfo(C.Structure):
    _fields_ = [("width", C.c_uint32), ("height", C.c_uint32), ("point_step", C.c_uint32),
                ("encoding_opt", C.c_uint8), ("compression_opt", C.c_uint8), ("version", C.c_uint8),
                ("use_threads", C.c_uint8), ("n_fields", C.c_uint32), ("fields", _CField * CLDN_MAX_FIELDS),
                ("encoding_config", C.c_char * 128)]


_lib = None


def library_path() -> str:
    return _LIB_PATH


def lib():
    """Loads the compiled C-ABI library. Fails loudly when it has not been built (no fallback path exists)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(_LIB_PATH):
        raise RuntimeError(
            f"{_LIB_PATH} is missing: build it with `python -m cloudini_b200.build` (nvcc, sm_90a). "
            "cloudini_b200 has no CPU or PyTorch fallback.")
    L = C.CDLL(_LIB_PATH)
    vp, sz, u8p = C.c_void_p, C.c_size_t, C.POINTER(C.c_uint8)
    L.cldn_b200_version.restype = C.c_char_p
    if b"cusim" in L.cldn_b200_version() and os.environ.get("CLDN_B200_ALLOW_EMULATION") != "tests-only":
        # tests/cusim (the CUDA model emulated on the CPU) exists to test kernel logic without a GPU; it is not a way to
        # run this package without one
        raise RuntimeError(f"{_LIB_PATH} is the cusim test emulation, not the product library: refusing to load it "
                           "(tests/test_cusim_kernels.py sets CLDN_B200_ALLOW_EMULATION=tests-only for its sub-runs)")
    L.cldn_b200_last_error.restype = C.c_char_p
    L.cldn_b200_kernel_launch_count.restype = C.c_uint64
    L.cldn_b200_bind_host_thread_to_device.argtypes = [C.c_int]
    L.cldn_b200_info_init.argtypes = [C.POINTER(_CInfo)]
    L.cldn_b200_info_to_yaml.argtypes = [C.POINTER(_CInfo), C.c_char_p, sz, C.POINTER(sz)]
    L.cldn_b200_info_from_yaml.argtypes = [C.c_char_p, sz, C.POINTER(_CInfo)]
    L.cldn_b200_encode_header.argtypes = [C.POINTER(_CInfo), vp, sz, C.POINTER(sz)]
    L.cldn_b200_encode_header_binary.argtypes = [C.POINTER(_CInfo), vp, sz, C.POINTER(sz)]
    L.cldn_b200_decode_header.argtypes = [vp, sz, C.POINTER(_CInfo), C.POINTER(sz)]
    L.cldn_b200_max_compressed_size.argtypes = [C.POINTER(_CInfo), sz, C.c_int]
    L.cldn_b200_max_compressed_size.restype = sz
    L.cldn_b200_encoder_create.argtypes = [C.POINTER(_CInfo), C.c_int, vp, C.POINTER(vp)]
    L.cldn_b200_encoder_destroy.argtypes = [vp]
    L.cldn_b200_encoder_destroy.restype = None
    L.cldn_b200_encoder_header.argtypes = [vp, C.POINTER(vp), C.POINTER(sz)]
    L.cldn_b200_encode.argtypes = [vp, vp, sz, vp, sz, C.c_int, C.POINTER(sz), C.c_int]
    L.cldn_b200_encode_batch.argtypes = [vp, sz, C.POINTER(vp), C.POINTER(sz), C.POINTER(vp), C.POINTER(sz), C.c_int,
                                         C.POINTER(sz), C.c_int]
    L.cldn_b200_encode_blobs.argtypes = [vp, sz, C.POINTER(vp), C.POINTER(sz), C.POINTER(C.c_uint32), C.POINTER(C.c_uint32),
                                         C.POINTER(vp), C.POINTER(sz), C.POINTER(sz), C.c_int]
    L.cldn_b200_encoder_sizes_device.argtypes = [vp]
    L.cldn_b200_encoder_sizes_device.restype = vp
    L.cldn_b200_encoder_sync.argtypes = [vp]
    L.cldn_b200_decoder_create.argtypes = [C.c_int, vp, C.POINTER(vp)]
    L.cldn_b200_decoder_destroy.argtypes = [vp]
    L.cldn_b200_decoder_destroy.restype = None
    L.cldn_b200_decode.argtypes = [vp, C.POINTER(_CInfo), vp, sz, vp, sz, C.c_int]
    L.cldn_b200_decode_batch.argtypes = [vp, C.POINTER(_CInfo), sz, C.POINTER(vp), C.POINTER(sz), C.POINTER(vp),
                                         C.POINTER(sz), C.c_int, C.c_int]
    L.cldn_b200_decode_blobs.argtypes = [vp, sz, C.POINTER(vp), C.POINTER(sz), C.POINTER(vp), C.POINTER(sz), C.c_int,
                                         C.POINTER(C.c_int32), C.POINTER(sz)]
    L.cldn_b200_decoder_frame_error.argtypes = [vp, sz]
    L.cldn_b200_decoder_frame_error.restype = C.c_char_p
    L.cldn_b200_decoder_frame_info.argtypes = [vp, sz, C.POINTER(_CInfo)]
    L.cldn_b200_decoder_sync.argtypes = [vp]
    L.cldn_b200_decoder_last_stats.argtypes = [vp, C.POINTER(C.c_uint32)]
    L.cldn_b200_decoder_last_sections_ahead.argtypes = [vp]
    L.cldn_b200_EncodePointcloudData.argtypes = [C.c_char_p, vp, C.c_uint32, vp, C.c_uint32]
    L.cldn_b200_EncodePointcloudData.restype = C.c_uint32
    L.cldn_b200_DecodeCompressedData.argtypes = [vp, C.c_uint32, vp, C.c_uint32]
    L.cldn_b200_DecodeCompressedData.restype = C.c_uint32
    _lib = L
    return L


def _err() -> str:
    return lib().cldn_b200_last_error().decode("utf-8", "replace")


def _check(rc: int):
    if rc != 0:
        raise RuntimeError(_err() or f"cloudini_b200 error {rc}")


def kernel_launch_count() -> int:
    return int(lib().cldn_b200_kernel_launch_count())


def bind_host_thread_to_device(device: int = -1) -> int:
    """Pins the calling thread (and threads it starts later) to the CPUs next to `device` (NVML's CPU affinity), so that
    pinned buffers allocated afterwards are NUMA-local to the GPU. Returns the number of CPUs in the set (0: unchanged)."""
    return int(lib().cldn_b200_bind_host_thread_to_device(device))


def _to_c(info: EncodingInfo) -> _CInfo:
    if len(info.fields) > CLDN_MAX_FIELDS:
        raise RuntimeError("too many fields")
    c = _CInfo()
    c.width, c.height, c.point_step = info.width, info.height, info.point_step
    c.encoding_opt, c.compression_opt = int(info.encoding_opt), int(info.compression_opt)
    c.version, c.use_threads = int(info.version), 1 if info.use_threads else 0
    c.n_fields = len(info.fields)
    c.encoding_config = info.encoding_config.encode("utf-8", "surrogateescape")
    for i, f in enumerate(info.fields):
        c.fields[i].name = f.name.encode("utf-8", "surrogateescape")
        c.fields[i].offset = f.offset
        c.fields[i].type = int(f.type)
        c.fields[i].has_resolution = 0 if f.resolution is None else 1
        c.fields[i].resolution = 0.0 if f.resolution is None else float(f.resolution)
    return c


def _from_c(c: _CInfo) -> EncodingInfo:
    info = EncodingInfo(width=c.width, height=c.height, point_step=c.point_step,
                        encoding_opt=EncodingOptions(c.encoding_opt) if c.encoding_opt <= 2 else int(c.encoding_opt),
                        compression_opt=CompressionOption(c.compression_opt) if c.compression_opt <= 2 else int(c.compression_opt),
                        use_threads=bool(c.use_threads), version=c.version,
                        encoding_config=c.encoding_config.decode("utf-8", "surrogateescape"))
    for i in range(c.n_fields):
        f = c.fields[i]
        # a forged legacy header can carry any type byte (the reference casts it unchecked, cloudini.cpp:405): keep the number
        info.fields.append(PointField(f.name.decode("utf-8", "surrogateescape"), f.offset, FieldType(f.type) if f.type <= 10 else int(f.type),
                                      float(f.resolution) if f.has_resolution else None))
    return info


def EncodingInfoToYAML(info: EncodingInfo) -> str:  # cloudini.cpp:165-190
    c = _to_c(info)
    need = C.c_size_t(0)
    lib().cldn_b200_info_to_yaml(C.byref(c), None, 0, C.byref(need))
    buf = C.create_string_buffer(need.value)
    _check(lib().cldn_b200_info_to_yaml(C.byref(c), buf, need.value, None))
    return buf.value.decode("utf-8", "surrogateescape")


def EncodingInfoFromYAML(yaml: str) -> EncodingInfo:  # cloudini.cpp:192-230
    c = _CInfo()
    raw = yaml.encode("utf-8", "surrogateescape")
    _check(lib().cldn_b200_info_from_yaml(raw, len(raw), C.byref(c)))
    return _from_c(c)


def EncodeHeader(info: EncodingInfo, binary: bool = False) -> bytes:
    """cloudini.cpp:294-344: the YAML header every encoder writes, or (binary=True) HeaderEncoding::BINARY."""
    c = _to_c(info)
    fn = lib().cldn_b200_encode_header_binary if binary else lib().cldn_b200_encode_header
    need = C.c_size_t(0)
    fn(C.byref(c), None, 0, C.byref(need))
    buf = (C.c_uint8 * need.value)()
    _check(fn(C.byref(c), buf, need.value, None))
    return bytes(buf)


def DecodeHeader(blob) -> tuple:
    """cloudini.cpp:353-428. Returns (EncodingInfo, header_bytes); the reference advances the caller's view instead."""
    raw = bytes(blob) if not isinstance(blob, (bytes, bytearray)) else blob
    buf = (C.c_uint8 * len(raw)).from_buffer_copy(raw) if len(raw) else (C.c_uint8 * 1)()
    c = _CInfo()
    used = C.c_size_t(0)
    _check(lib().cldn_b200_decode_header(buf, len(raw), C.byref(c), C.byref(used)))
    return _from_c(c), used.value


def MaxCompressedSize(info: EncodingInfo, points_count: int, include_header: bool = True) -> int:  # cloudini.cpp:249-292
    c = _to_c(info)
    n = lib().cldn_b200_max_compressed_size(C.byref(c), points_count, 1 if include_header else 0)
    if n == 0 and (info.point_step == 0 or points_count > 0 or include_header):
        raise RuntimeError(_err())
    return n


def _host_ptr(obj):
    """Returns (address, nbytes, keepalive) of a bytes-like / numpy / CPU torch object."""
    import numpy as np
    if hasattr(obj, "data_ptr"):  # torch CPU tensor
        t = obj.contiguous()
        return t.data_ptr(), t.numel() * t.element_size(), t
    a = np.frombuffer(obj, dtype=np.uint8) if isinstance(obj, (bytes, bytearray, memoryview)) else np.ascontiguousarray(obj)
    return a.ctypes.data, a.nbytes, a


class PointcloudEncoder:
    """Cloudini::PointcloudEncoder (cloudini.hpp:154-211) backed by the sm_90a kernels."""

    def __init__(self, info: EncodingInfo, device: int = -1, stream: int = 0):
        self._info = info
        self._c = _to_c(info)
        self._h = C.c_void_p()
        _check(lib().cldn_b200_encoder_create(C.byref(self._c), device, C.c_void_p(stream or None), C.byref(self._h)))
        hp, hn = C.c_void_p(), C.c_size_t()
        _check(lib().cldn_b200_encoder_header(self._h, C.byref(hp), C.byref(hn)))
        self._header = C.string_at(hp.value, hn.value)

    def getEncodingInfo(self) -> EncodingInfo:
        return self._info

    def getHeader(self) -> bytes:
        return self._header

    def close(self):
        if getattr(self, "_h", None) and self._h.value:
            lib().cldn_b200_encoder_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # size_t encode(ConstBufferView cloud_data, std::vector<uint8_t>& output)  (cloudini.cpp:501-520)
    def encode(self, cloud_data, write_header: bool = True) -> bytes:
        import numpy as np
        addr, nbytes, keep = _host_ptr(cloud_data)
        if self._info.point_step == 0:
            raise RuntimeError("point_step cannot be 0")
        if nbytes % self._info.point_step:
            raise RuntimeError("Input cloud_data size is not a multiple of point_step")
        cap = MaxCompressedSize(self._info, nbytes // self._info.point_step, True)
        out = np.empty(max(cap, 1), dtype=np.uint8)
        written = C.c_size_t(0)
        _check(lib().cldn_b200_encode(self._h, addr, nbytes, out.ctypes.data, cap, 1 if write_header else 0,
                                      C.byref(written), MEM_HOST))
        del keep
        return out[:written.value].tobytes()

    # size_t encode(ConstBufferView, BufferView& output, bool write_header)  (cloudini.cpp:522-623), host buffers
    def encode_into(self, cloud_data, output, write_header: bool = True) -> int:
        addr, nbytes, keep = _host_ptr(cloud_data)
        oaddr, ocap, okeep = _host_ptr(output)
        written = C.c_size_t(0)
        _check(lib().cldn_b200_encode(self._h, addr, nbytes, oaddr, ocap, 1 if write_header else 0, C.byref(written), MEM_HOST))
        return written.value

    def encode_batch_host(self, clouds: Sequence, outputs: Sequence, write_header: bool = True) -> List[int]:
        n = len(clouds)
        ins = [_host_ptr(c) for c in clouds]
        outs = [_host_ptr(o) for o in outputs]
        a_in = (C.c_void_p * n)(*[p[0] for p in ins])
        a_inb = (C.c_size_t * n)(*[p[1] for p in ins])
        a_out = (C.c_void_p * n)(*[p[0] for p in outs])
        a_cap = (C.c_size_t * n)(*[p[1] for p in outs])
        written = (C.c_size_t * n)()
        _check(lib().cldn_b200_encode_batch(self._h, n, a_in, a_inb, a_out, a_cap, 1 if write_header else 0, written, MEM_HOST))
        return list(written)

    def make_device_batch(self, in_ptrs: Sequence[int], in_bytes: Sequence[int], out_ptrs: Sequence[int],
                          out_caps: Sequence[int]):
        """Pre-marshals the pointer arrays of a device-resident batch (see encode_batch_device)."""
        n = len(in_ptrs)
        return (n, (C.c_void_p * n)(*in_ptrs), (C.c_size_t * n)(*in_bytes), (C.c_void_p * n)(*out_ptrs),
                (C.c_size_t * n)(*out_caps))

    def encode_batch_device(self, batch, write_header: bool = True, want_sizes: bool = False):
        """Device pointers in, device pointers out; asynchronous on the encoder's stream unless want_sizes."""
        n, a_in, a_inb, a_out, a_cap = batch
        written = (C.c_size_t * n)() if want_sizes else None
        _check(lib().cldn_b200_encode_batch(self._h, n, a_in, a_inb, a_out, a_cap, 1 if write_header else 0, written, MEM_DEVICE))
        return list(written) if want_sizes else None

    @staticmethod
    def _dims(n: int, dims):
        """(widths, heights) ctypes arrays for encode_blobs: None for width = points, height = 1."""
        if dims is None:
            return None, None
        if len(dims) != n:
            raise RuntimeError("dims must have one (width, height) per frame")
        m = max(n, 1)
        return (C.c_uint32 * m)(*[int(w) for w, _ in dims]), (C.c_uint32 * m)(*[int(h) for _, h in dims])

    def encode_blobs(self, clouds: Sequence, dims: Optional[Sequence] = None) -> List[bytes]:
        """Complete blobs of host clouds of this encoder's layout, each with a header stating its own dims: ``dims`` is
        one (width, height) per cloud, or None for (points, 1). Blob f equals what set_dims(w_f, h_f) + encode(cloud_f)
        give; this encoder's header is not changed."""
        import numpy as np
        n = len(clouds)
        m = max(n, 1)
        widths, heights = self._dims(n, dims)
        ins = [_host_ptr(c) for c in clouds]
        caps = [self._blob_cap(nbytes, dims[k] if dims is not None else None) for k, (_, nbytes, _) in enumerate(ins)]
        outs = [np.empty(max(c, 1), dtype=np.uint8) for c in caps]
        written = (C.c_size_t * m)()
        _check(lib().cldn_b200_encode_blobs(self._h, n, (C.c_void_p * m)(*[p[0] for p in ins]), (C.c_size_t * m)(*[p[1] for p in ins]),
                                            widths, heights, (C.c_void_p * m)(*[o.ctypes.data for o in outs]), (C.c_size_t * m)(*caps),
                                            written, MEM_HOST))
        del ins
        return [outs[f][:written[f]].tobytes() for f in range(n)]

    def encode_blobs_device(self, in_ptrs: Sequence[int], in_bytes: Sequence[int], out_ptrs: Sequence[int], out_caps: Sequence[int],
                            dims: Optional[Sequence] = None, want_sizes: bool = True):
        """encode_blobs for device-resident clouds and outputs (device addresses). Returns the blob sizes, or None when
        want_sizes is False: the call is then asynchronous and the sizes stay at sizes_device_ptr()."""
        n = len(in_ptrs)
        m = max(n, 1)
        widths, heights = self._dims(n, dims)
        written = (C.c_size_t * m)() if want_sizes else None
        _check(lib().cldn_b200_encode_blobs(self._h, n, (C.c_void_p * m)(*in_ptrs), (C.c_size_t * m)(*in_bytes), widths, heights,
                                            (C.c_void_p * m)(*out_ptrs), (C.c_size_t * m)(*out_caps), written, MEM_DEVICE))
        return [int(written[f]) for f in range(n)] if want_sizes else None

    def _blob_cap(self, nbytes: int, dims=None) -> int:
        """Capacity of the blob of a cloud of `nbytes` for encode_blobs / encode_blobs_from_device: MaxCompressedSize with
        the header of its dims ((width, height), None for (points, 1)), or 1 byte for a cloud that is not a whole number
        of points, which the library then reports as that frame's error."""
        step = self._info.point_step
        if not step or nbytes % step:
            return 1
        w, h = dims if dims is not None else (nbytes // step, 1)
        return MaxCompressedSize(replace(self._info, width=int(w), height=int(h)), nbytes // step, True)

    def encode_device(self, ptr: int, nbytes: int, write_header: bool = True) -> bytes:
        """encode() of a device-resident cloud (a device address of `nbytes`): the blob comes back in host memory, as
        encode() writes it. The cloud is read on this encoder's stream."""
        import numpy as np
        if self._info.point_step == 0:
            raise RuntimeError("point_step cannot be 0")
        if nbytes % self._info.point_step:
            raise RuntimeError("Input cloud_data size is not a multiple of point_step")
        cap = MaxCompressedSize(self._info, nbytes // self._info.point_step, True)
        out = np.empty(max(cap, 1), dtype=np.uint8)
        written = C.c_size_t(0)
        _check(lib().cldn_b200_encode(self._h, ptr, nbytes, out.ctypes.data, cap, 1 if write_header else 0, C.byref(written),
                                      MEM_DEVICE_POINTS))
        return out[:written.value].tobytes()

    def encode_blobs_from_device(self, in_ptrs: Sequence[int], in_bytes: Sequence[int], dims: Optional[Sequence] = None) -> List[bytes]:
        """encode_blobs() of device-resident clouds (device addresses): complete blobs in host memory, byte-identical to
        what encode_blobs() gives the same clouds in host memory."""
        import numpy as np
        n = len(in_ptrs)
        m = max(n, 1)
        widths, heights = self._dims(n, dims)
        caps = [self._blob_cap(int(b), dims[f] if dims is not None else None) for f, b in enumerate(in_bytes)]
        outs = [np.empty(max(c, 1), dtype=np.uint8) for c in caps]
        written = (C.c_size_t * m)()
        _check(lib().cldn_b200_encode_blobs(self._h, n, (C.c_void_p * m)(*in_ptrs), (C.c_size_t * m)(*in_bytes), widths, heights,
                                            (C.c_void_p * m)(*[o.ctypes.data for o in outs]), (C.c_size_t * m)(*caps), written,
                                            MEM_DEVICE_POINTS))
        return [outs[f][:written[f]].tobytes() for f in range(n)]

    def sizes_device_ptr(self) -> int:
        return int(lib().cldn_b200_encoder_sizes_device(self._h) or 0)

    def sync(self):
        _check(lib().cldn_b200_encoder_sync(self._h))


class PointcloudDecoder:
    """Cloudini::PointcloudDecoder (cloudini.hpp:216-244) backed by the sm_90a kernels."""

    def __init__(self, device: int = -1, stream: int = 0):
        self._h = C.c_void_p()
        _check(lib().cldn_b200_decoder_create(device, C.c_void_p(stream or None), C.byref(self._h)))

    def close(self):
        if getattr(self, "_h", None) and self._h.value:
            lib().cldn_b200_decoder_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # void decode(info, compressed_data (no header), std::vector<uint8_t>& output)  (cloudini.hpp:229-233)
    def decode(self, info: EncodingInfo, compressed_data, output=None):
        """Returns the decoded bytes; `output` (numpy uint8, pre-filled) is decoded in place when given — only
        declared field bytes are overwritten, like the reference."""
        import numpy as np
        need = info.width * info.height * info.point_step
        if output is None:
            output = np.zeros(need, dtype=np.uint8)  # std::vector::resize zero-fills
        addr, nbytes, keep = _host_ptr(compressed_data)
        oaddr, ocap, okeep = _host_ptr(output)
        c = _to_c(info)
        _check(lib().cldn_b200_decode(self._h, C.byref(c), addr, nbytes, oaddr, ocap, MEM_HOST))
        return output

    def make_device_batch(self, in_ptrs, in_bytes, out_ptrs, out_caps):
        n = len(in_ptrs)
        return (n, (C.c_void_p * n)(*in_ptrs), (C.c_size_t * n)(*in_bytes), (C.c_void_p * n)(*out_ptrs),
                (C.c_size_t * n)(*out_caps))

    def decode_batch_device(self, info: EncodingInfo, batch, sync: bool = False):
        n, a_in, a_inb, a_out, a_cap = batch
        c = _to_c(info)
        _check(lib().cldn_b200_decode_batch(self._h, C.byref(c), n, a_in, a_inb, a_out, a_cap, MEM_DEVICE, 1 if sync else 0))

    def decode_batch_host(self, info: EncodingInfo, payloads: Sequence, outputs: Sequence):
        n = len(payloads)
        ins = [_host_ptr(p) for p in payloads]
        outs = [_host_ptr(o) for o in outputs]
        c = _to_c(info)
        _check(lib().cldn_b200_decode_batch(self._h, C.byref(c), n, (C.c_void_p * n)(*[p[0] for p in ins]),
                                            (C.c_size_t * n)(*[p[1] for p in ins]), (C.c_void_p * n)(*[p[0] for p in outs]),
                                            (C.c_size_t * n)(*[p[1] for p in outs]), MEM_HOST, 1))

    def _blobs(self, n, a_in, a_inb, a_out, a_cap, mem):
        status = (C.c_int32 * max(n, 1))()
        lib().cldn_b200_decode_blobs(self._h, n, a_in, a_inb, a_out, a_cap, mem, status, None)
        infos = []
        for f in range(n):
            c = _CInfo()
            _check(lib().cldn_b200_decoder_frame_info(self._h, f, C.byref(c)))
            infos.append(_from_c(c) if c.version else None)  # zeroed where the header did not parse
        return [int(status[f]) for f in range(n)], infos

    def decode_blobs(self, blobs: Sequence, outputs: Optional[Sequence] = None):
        """Complete blobs (header included, as encode() returns them) in any mix of layouts, point counts, wire versions
        3..5 and compressions, host memory. Frames of one layout and compression are decoded together. Returns one
        (status, EncodingInfo | None, output | None) per blob: status 0 or the negative cldn_status_t that DecodeHeader +
        decode give that blob alone (its message: frame_error(f)); output is None for a failed frame. `outputs` (numpy
        uint8, pre-filled) are decoded in place when given; only declared field bytes are overwritten."""
        import numpy as np
        n = len(blobs)
        if outputs is None:
            outputs = []
            for b in blobs:
                try:
                    info, _ = DecodeHeader(b)
                    outputs.append(np.zeros(info.width * info.height * info.point_step, dtype=np.uint8))
                except (RuntimeError, MemoryError, ValueError):   # the decoder reports the frame's status
                    outputs.append(np.zeros(0, dtype=np.uint8))
        ins = [_host_ptr(b) for b in blobs]
        outs = [_host_ptr(o) for o in outputs]
        status, infos = self._blobs(n, (C.c_void_p * max(n, 1))(*[p[0] for p in ins]), (C.c_size_t * max(n, 1))(*[p[1] for p in ins]),
                                    (C.c_void_p * max(n, 1))(*[p[0] for p in outs]), (C.c_size_t * max(n, 1))(*[p[1] for p in outs]),
                                    MEM_HOST)
        return [(status[f], infos[f], outputs[f] if status[f] == 0 else None) for f in range(n)]

    def decode_blobs_device(self, ptrs: Sequence[int], sizes: Sequence[int], out_ptrs: Sequence[int], out_caps: Sequence[int]):
        """decode_blobs for device-resident blobs and outputs (device addresses). Returns (statuses, EncodingInfos), an
        info being None where the header did not parse."""
        n = len(ptrs)
        m = max(n, 1)
        return self._blobs(n, (C.c_void_p * m)(*ptrs), (C.c_size_t * m)(*sizes), (C.c_void_p * m)(*out_ptrs),
                           (C.c_size_t * m)(*out_caps), MEM_DEVICE)

    def decode_to_device(self, info: EncodingInfo, payload, out_ptr: int, out_cap: int):
        """decode() of a host payload (no header) into a device buffer of `out_cap` bytes at device address `out_ptr`,
        in place: only declared field bytes are written. Ordered on this decoder's stream; synchronous."""
        addr, nbytes, keep = _host_ptr(payload)
        c = _to_c(info)
        _check(lib().cldn_b200_decode(self._h, C.byref(c), addr, nbytes, out_ptr, out_cap, MEM_DEVICE_POINTS))
        del keep

    def decode_blobs_to_device(self, blobs: Sequence, out_ptrs: Sequence[int], out_caps: Sequence[int]):
        """decode_blobs() of host blobs into device buffers (device addresses). Returns (statuses, EncodingInfos) as
        decode_blobs_device() does; statuses and frame_error(f) are those decode_blobs() gives the same blobs."""
        n = len(blobs)
        m = max(n, 1)
        ins = [_host_ptr(b) for b in blobs]
        r = self._blobs(n, (C.c_void_p * m)(*[p[0] for p in ins]), (C.c_size_t * m)(*[p[1] for p in ins]),
                        (C.c_void_p * m)(*out_ptrs), (C.c_size_t * m)(*out_caps), MEM_DEVICE_POINTS)
        del ins
        return r

    def frame_error(self, f: int) -> str:
        """Message of frame f of the last decode_blobs / decode_blobs_device ("" when it decoded)."""
        return lib().cldn_b200_decoder_frame_error(self._h, f).decode("utf-8", "replace")

    def sync(self):
        _check(lib().cldn_b200_decoder_sync(self._h))

    def last_stats(self):
        """(chunks taken by the chunk-sequential fast reader, chunks it handed to the careful reader) of the last batch."""
        st = (C.c_uint32 * 2)()
        _check(lib().cldn_b200_decoder_last_stats(self._h, st))
        return int(st[0]), int(st[1])

    def last_sections_ahead(self) -> bool:
        """True if the last batch decoded its V5 sections ahead of the regular stream (merged row writes)."""
        r = lib().cldn_b200_decoder_last_sections_ahead(self._h)
        _check(r if r < 0 else 0)
        return r == 1
