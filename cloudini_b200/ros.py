"""Host-side Python mirror of ``cloudini_ros`` (cloudini_lib/include/cloudini_lib/ros_msg_utils.hpp) on top of the C ABI
``include/cloudini_b200_ros.h`` — SURVEY.md §8(f) rows N2 (DDS envelope) and N3 (viz preprocessing).

Same names and argument meaning as the reference: ``getDeserializedPointCloudMessage``, ``applyResolutionProfile``,
``toEncodingInfo``, ``convertPointCloud2ToCompressedCloud``, ``convertCompressedCloudToPointCloud2``,
``applyVizLossyPreprocessing``. The CDR header is parsed / written by host code in the library; every byte of point data
goes through the GPU codec / the preprocessing kernels (no CPU implementation exists here).
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, field
from typing import Dict, List, Optional

import numpy as np

from . import (CLDN_MAX_FIELDS, MEM_DEVICE, MEM_HOST, CompressionOption, EncodingInfo, EncodingOptions, FieldType,
               PointcloudDecoder, PointcloudEncoder, PointField, _CField, _CInfo, _check, _from_c, _to_c, blob_descs, lib,
               pack_blob_descs)

__all__ = ["RosPointCloud2", "getDeserializedPointCloudMessage", "applyResolutionProfile", "toEncodingInfo",
           "convertPointCloud2ToCompressedCloud", "convertCompressedCloudToPointCloud2", "applyVizLossyPreprocessing",
           "VizPreprocessor", "viz_descs", "pack_viz_descs"]


class _CRosMsg(C.Structure):
    _fields_ = [("cdr_header", C.c_uint8 * 4), ("stamp_sec", C.c_int32), ("stamp_nsec", C.c_uint32),
                ("frame_id", C.c_void_p), ("frame_id_len", C.c_uint32), ("height", C.c_uint32),
                ("width", C.c_uint32), ("n_fields", C.c_uint32), ("fields", _CField * CLDN_MAX_FIELDS),
                ("is_bigendian", C.c_uint8), ("is_dense", C.c_uint8), ("point_step", C.c_uint32),
                ("row_step", C.c_uint32), ("data", C.c_void_p), ("data_bytes", C.c_size_t)]


_bound = False


def _L():
    global _bound
    L = lib()
    if not _bound:
        vp, sz = C.c_void_p, C.c_size_t
        L.cldn_b200_preproc_create.argtypes = [C.c_int, vp, C.POINTER(vp)]
        L.cldn_b200_preproc_destroy.argtypes = [vp]
        L.cldn_b200_preproc_destroy.restype = None
        L.cldn_b200_viz_lossy_preprocess.argtypes = [vp, C.POINTER(_CInfo), vp, sz, vp, sz, C.POINTER(sz), C.POINTER(C.c_int), C.c_int]
        L.cldn_b200_viz_lossy_preprocess_batch.argtypes = [vp, C.POINTER(_CInfo), sz, C.POINTER(vp), C.POINTER(sz), C.POINTER(vp),
                                                           C.POINTER(sz), C.POINTER(sz), C.POINTER(C.c_int), C.POINTER(_CInfo), C.c_int]
        L.cldn_b200_preproc_prepare_batch.argtypes = [vp, C.POINTER(_CInfo), sz, C.c_uint64, C.POINTER(_CInfo)]
        L.cldn_b200_viz_lossy_preprocess_batch_async.argtypes = [vp, sz, vp, vp, vp, vp, vp]
        L.cldn_b200_preproc_sync.argtypes = [vp]
        L.cldn_b200_ros_parse.argtypes = [vp, sz, C.POINTER(_CRosMsg)]
        L.cldn_b200_ros_to_encoding_info.argtypes = [C.POINTER(_CRosMsg), C.POINTER(_CInfo)]
        L.cldn_b200_ros_apply_resolution_profile.argtypes = [C.POINTER(_CField), C.POINTER(C.c_uint32), C.POINTER(C.c_char_p),
                                                             C.POINTER(C.c_float), sz, C.POINTER(C.c_float)]
        L.cldn_b200_ros_compress_msg.argtypes = [vp, C.POINTER(_CRosMsg), vp, sz, C.POINTER(sz)]
        L.cldn_b200_ros_decompress_msg.argtypes = [vp, C.POINTER(_CRosMsg), vp, sz, C.POINTER(sz)]
        L.cldn_b200_encoder_info.argtypes = [vp, C.POINTER(_CInfo)]
        L.cldn_b200_encoder_set_dims.argtypes = [vp, C.c_uint32, C.c_uint32]
        L.cldn_b200_ros_convert_msg.argtypes = [vp, sz, C.POINTER(C.c_char_p), C.POINTER(C.c_float), sz, C.POINTER(C.c_float), C.c_int, C.c_int,
                                                C.c_int, C.c_int, vp, sz, C.POINTER(sz)]
        _bound = True
    return L


@dataclass
class RosPointCloud2:
    """cloudini_ros::RosPointCloud2 (ros_msg_utils.hpp:32-148). ``data`` is the point payload (or the compressed blob of
    a CompressedPointCloud2) as a uint8 array; after parsing it is a view into ``msg``."""
    msg: bytes = b""
    cdr_header: bytes = bytes([0, 1, 0, 0])
    stamp_sec: int = 0
    stamp_nsec: int = 0
    frame_id: str = ""
    height: int = 1
    width: int = 0
    fields: List[PointField] = field(default_factory=list)
    point_step: int = 0
    row_step: int = 0
    is_bigendian: bool = False
    is_dense: bool = True
    data: np.ndarray = field(default_factory=lambda: np.zeros(0, dtype=np.uint8))
    data_offset: int = 0  # where `data` started inside `msg` when it was parsed

    def _c_view(self):
        """(C struct, keepalive objects) describing this object for the header writer."""
        c = _CRosMsg()
        c.cdr_header[:] = list(self.cdr_header)
        c.stamp_sec, c.stamp_nsec = self.stamp_sec, self.stamp_nsec
        frame = self.frame_id.encode("utf-8", "surrogateescape")
        fbuf = C.create_string_buffer(frame, len(frame) + 1)
        c.frame_id, c.frame_id_len = C.cast(fbuf, C.c_void_p).value, len(frame)
        c.height, c.width, c.point_step, c.row_step = self.height, self.width, self.point_step, self.row_step
        c.is_bigendian, c.is_dense = (1 if self.is_bigendian else 0), int(self.is_dense) & 0xFF
        if len(self.fields) > CLDN_MAX_FIELDS:
            raise RuntimeError("too many fields")
        c.n_fields = len(self.fields)
        for i, f in enumerate(self.fields):
            c.fields[i].name = f.name.encode("utf-8", "surrogateescape")
            c.fields[i].offset, c.fields[i].type = f.offset, int(f.type)
            c.fields[i].has_resolution = 0 if f.resolution is None else 1
            c.fields[i].resolution = 0.0 if f.resolution is None else float(f.resolution)
        data = np.ascontiguousarray(self.data, dtype=np.uint8)
        c.data, c.data_bytes = (data.ctypes.data if data.size else None), data.size
        return c, (fbuf, data)


def getDeserializedPointCloudMessage(dds_msg) -> RosPointCloud2:  # ros_msg_utils.cpp:54-95
    raw = bytes(dds_msg)
    c = _CRosMsg()
    buf = np.frombuffer(raw, dtype=np.uint8)
    _check(_L().cldn_b200_ros_parse(buf.ctypes.data if len(raw) else None, len(raw), C.byref(c)))
    base = buf.ctypes.data
    f0 = (c.frame_id or base) - base
    d0 = (c.data or base) - base
    pc = RosPointCloud2(msg=raw, cdr_header=bytes(c.cdr_header), stamp_sec=c.stamp_sec, stamp_nsec=c.stamp_nsec,
                        frame_id=raw[f0:f0 + c.frame_id_len].decode("utf-8", "surrogateescape"),
                        height=c.height, width=c.width, point_step=c.point_step, row_step=c.row_step,
                        is_bigendian=bool(c.is_bigendian),
                        # a non-canonical CDR bool (byte > 1) leaves the reference the way it came in (it memcpy's the
                        # byte into a C++ bool and back, ros_msg_utils.cpp:89,164): keep the byte, truthiness unchanged
                        is_dense=(bool(c.is_dense) if c.is_dense <= 1 else int(c.is_dense)),
                        data=buf[d0:d0 + c.data_bytes], data_offset=d0)
    for i in range(c.n_fields):
        f = c.fields[i]
        pc.fields.append(PointField(f.name.decode("utf-8", "surrogateescape"), f.offset, FieldType(f.type) if f.type <= 10 else f.type, None))
    return pc


def applyResolutionProfile(profile: Dict[str, float], fields: List[PointField], default_resolution: Optional[float] = None):
    """ros_msg_utils.cpp:217-238 — edits ``fields`` in place (profile resolution 0 removes the field)."""
    n = C.c_uint32(len(fields))
    arr = (_CField * CLDN_MAX_FIELDS)()
    for i, f in enumerate(fields):
        arr[i].name = f.name.encode("utf-8", "surrogateescape")
        arr[i].offset, arr[i].type = f.offset, int(f.type)
        arr[i].has_resolution = 0 if f.resolution is None else 1
        arr[i].resolution = 0.0 if f.resolution is None else float(f.resolution)
    names = (C.c_char_p * max(1, len(profile)))(*[k.encode("utf-8", "surrogateescape") for k in profile])
    res = (C.c_float * max(1, len(profile)))(*[float(v) for v in profile.values()])
    dflt = C.byref(C.c_float(default_resolution)) if default_resolution is not None else None
    _check(_L().cldn_b200_ros_apply_resolution_profile(arr, C.byref(n), names, res, len(profile), dflt))
    fields[:] = [PointField(arr[i].name.decode("utf-8", "surrogateescape"), arr[i].offset, FieldType(arr[i].type) if arr[i].type <= 10 else arr[i].type,
                            float(arr[i].resolution) if arr[i].has_resolution else None) for i in range(n.value)]


def toEncodingInfo(pc: RosPointCloud2) -> EncodingInfo:  # ros_msg_utils.cpp:122-131
    c = _CInfo()
    m, _keep = pc._c_view()
    _check(_L().cldn_b200_ros_to_encoding_info(C.byref(m), C.byref(c)))
    return _from_c(c)


_ENCODERS: Dict[tuple, PointcloudEncoder] = {}   # per layout: the reference builds an encoder per message (:198); here that
_DECODERS: Dict[int, PointcloudDecoder] = {}      # would mean streams, device buffers and pinned memory per message


def _layout_key(info: EncodingInfo, device: int) -> tuple:
    return (device, info.point_step, int(info.encoding_opt), int(info.compression_opt), info.version,
            tuple((f.name, f.offset, int(f.type), f.resolution) for f in info.fields))


def _pooled_encoder(info: EncodingInfo, device: int) -> PointcloudEncoder:
    key = _layout_key(info, device)
    enc = _ENCODERS.get(key)
    if enc is None:
        if len(_ENCODERS) >= 8:
            _ENCODERS.pop(next(iter(_ENCODERS)))
        enc = _ENCODERS[key] = PointcloudEncoder(info, device=device)
    _check(_L().cldn_b200_encoder_set_dims(enc._h, info.width, info.height))
    return enc


def convertPointCloud2ToCompressedCloud(pc: RosPointCloud2, encoding_info: EncodingInfo, device: int = -1) -> bytes:
    """ros_msg_utils.cpp:167-213. Returns the serialised CompressedPointCloud2 message."""
    enc = _pooled_encoder(encoding_info, device)
    m, _keep = pc._c_view()
    need = C.c_size_t(0)
    _check(_L().cldn_b200_ros_compress_msg(enc._h, C.byref(m), None, 0, C.byref(need)))
    out = np.zeros(need.value, dtype=np.uint8)
    w = C.c_size_t(0)
    _check(_L().cldn_b200_ros_compress_msg(enc._h, C.byref(m), out.ctypes.data, out.size, C.byref(w)))
    return bytes(out[:w.value])


def convertCompressedCloudToPointCloud2(pc: RosPointCloud2, device: int = -1) -> bytes:
    """ros_msg_utils.cpp:134-165. Returns the serialised PointCloud2 message."""
    dec = _DECODERS.get(device)
    if dec is None:
        dec = _DECODERS[device] = PointcloudDecoder(device=device)
    m, _keep = pc._c_view()
    need = C.c_size_t(0)
    _check(_L().cldn_b200_ros_decompress_msg(dec._h, C.byref(m), None, 0, C.byref(need)))
    out = np.zeros(need.value, dtype=np.uint8)
    w = C.c_size_t(0)
    _check(_L().cldn_b200_ros_decompress_msg(dec._h, C.byref(m), out.ctypes.data, out.size, C.byref(w)))
    return bytes(out[:w.value])


def convert_message(msg: bytes, profile: Optional[Dict[str, float]] = None, default_resolution: Optional[float] = None, viz: bool = False,
                    encoding_opt=None, compression_opt=None, version: int = 5) -> bytes:
    """The converter's per-message step (tools/src/mcap_converter.cpp:184-204) as ONE library call: parse, resolution
    profile, optional viz preprocessing, encode, write the CompressedPointCloud2 message. The payload is uploaded once and
    stays on the GPU in between; handles come from the library's per-thread pool."""
    from . import CompressionOption, EncodingOptions
    profile = profile or {}
    raw = bytes(msg)
    buf = np.frombuffer(raw, dtype=np.uint8)
    names = (C.c_char_p * max(1, len(profile)))(*[k.encode("utf-8", "surrogateescape") for k in profile])
    res = (C.c_float * max(1, len(profile)))(*[float(v) for v in profile.values()])
    dflt = C.byref(C.c_float(default_resolution)) if default_resolution is not None else None
    eo = int(EncodingOptions.LOSSY if encoding_opt is None else encoding_opt)
    co = int(CompressionOption.ZSTD if compression_opt is None else compression_opt)
    L = _L()
    need = C.c_size_t(0)
    args = (buf.ctypes.data if len(raw) else None, len(raw), names, res, len(profile), dflt, 1 if viz else 0, eo, co, int(version))
    _check(L.cldn_b200_ros_convert_msg(*args, None, 0, C.byref(need)))
    out = np.empty(need.value, dtype=np.uint8)
    w = C.c_size_t(0)
    _check(L.cldn_b200_ros_convert_msg(*args, out.ctypes.data, out.size, C.byref(w)))
    return bytes(out[:w.value])


class VizPreprocessor:
    """Handle of the preprocessing kernels (voxel hash table, tile status words, staging buffers)."""

    def __init__(self, device: int = -1, stream: int = 0):
        self._h = C.c_void_p()
        _check(_L().cldn_b200_preproc_create(device, C.c_void_p(stream or None), C.byref(self._h)))

    def __del__(self):
        try:
            if self._h:
                _L().cldn_b200_preproc_destroy(self._h)
                self._h = None
        except Exception:
            pass

    def run(self, info: EncodingInfo, cloud, out=None):
        """Returns (new_info, survivors as a uint8 array, applied). ``info`` is not modified."""
        arr = np.frombuffer(cloud, dtype=np.uint8) if isinstance(cloud, (bytes, bytearray, memoryview)) \
            else np.ascontiguousarray(cloud).view(np.uint8).reshape(-1)
        c = _to_c(info)
        if out is None:
            out = np.zeros(max(arr.size, 1), dtype=np.uint8)
        kept, applied = C.c_size_t(0), C.c_int(0)
        _check(_L().cldn_b200_viz_lossy_preprocess(self._h, C.byref(c), arr.ctypes.data if arr.size else None, arr.size,
                                                   out.ctypes.data, out.size, C.byref(kept), C.byref(applied), MEM_HOST))
        if not applied.value:  # the reference's early returns: nothing changes
            return info, arr, False
        new_info = _from_c(c)
        new_info.use_threads = info.use_threads
        return new_info, out[:kept.value * info.point_step], True

    def run_device(self, info: EncodingInfo, in_ptr: int, nbytes: int, out_ptr: int, out_capacity: int):
        """Device-pointer variant: returns (new_info, kept_points, applied); survivors are at out_ptr."""
        c = _to_c(info)
        kept, applied = C.c_size_t(0), C.c_int(0)
        _check(_L().cldn_b200_viz_lossy_preprocess(self._h, C.byref(c), C.c_void_p(in_ptr), nbytes, C.c_void_p(out_ptr), out_capacity,
                                                   C.byref(kept), C.byref(applied), MEM_DEVICE))
        return (_from_c(c) if applied.value else info), kept.value, bool(applied.value)

    def _batch(self, info: EncodingInfo, n: int, in_ptrs, in_bytes, out_ptrs, out_caps, mem: int):
        m = max(n, 1)
        c = _to_c(info)
        kept, applied, infos = (C.c_size_t * m)(), (C.c_int * m)(), (_CInfo * m)()
        _check(_L().cldn_b200_viz_lossy_preprocess_batch(self._h, C.byref(c), n, (C.c_void_p * m)(*in_ptrs), (C.c_size_t * m)(*in_bytes),
                                                         (C.c_void_p * m)(*out_ptrs), (C.c_size_t * m)(*out_caps), kept, applied,
                                                         infos, mem))
        out = []
        for f in range(n):
            new_info = info
            if applied[f]:
                new_info = _from_c(infos[f])
                new_info.use_threads = info.use_threads
            out.append((new_info, int(kept[f]), bool(applied[f])))
        return out

    def run_batch(self, info: EncodingInfo, clouds):
        """``run`` for a list of host clouds of one layout, in one launch pair: returns one (new_info, survivors as a uint8
        array, applied) per cloud, with run's no-op convention (the input array and ``info`` when not applied)."""
        arrs = [np.frombuffer(c, dtype=np.uint8) if isinstance(c, (bytes, bytearray, memoryview))
                else np.ascontiguousarray(c).view(np.uint8).reshape(-1) for c in clouds]
        outs = [np.zeros(max(a.size, 1), dtype=np.uint8) for a in arrs]
        res = self._batch(info, len(arrs), [a.ctypes.data if a.size else None for a in arrs], [a.size for a in arrs],
                          [o.ctypes.data for o in outs], [o.size for o in outs], MEM_HOST)
        return [(new_info, outs[f][:kept * info.point_step] if applied else arrs[f], applied)
                for f, (new_info, kept, applied) in enumerate(res)]

    def run_batch_device(self, info: EncodingInfo, in_ptrs, in_bytes, out_ptrs, out_caps):
        """Device-pointer variant of run_batch: returns one (new_info, kept_points, applied) per cloud; survivors are at
        out_ptrs[f]."""
        return self._batch(info, len(in_ptrs), in_ptrs, in_bytes, out_ptrs, out_caps, MEM_DEVICE)

    def prepare_batch(self, info: EncodingInfo, max_frames: int, max_points: int) -> EncodingInfo:
        """Prepares run_batch_async() for calls of at most `max_frames` device clouds of layout `info` with at most
        `max_points` points each. Returns the layout of an applied frame with width = height = 0 (``info`` itself for a
        layout the preprocessing leaves alone): the EncodingInfo of the encoder that follows. See
        cldn_b200_preproc_prepare_batch."""
        c, after = _to_c(info), _CInfo()
        _check(_L().cldn_b200_preproc_prepare_batch(self._h, C.byref(c), max_frames, max_points, C.byref(after)))
        new_info = _from_c(after)
        new_info.use_threads = info.use_threads
        return new_info

    def run_batch_async(self, frames_ptr: int, n: int, status_ptr: int, kept_ptr: int = 0, applied_ptr: int = 0,
                        encode_descs_ptr: int = 0):
        """Enqueues the preprocessing of n device clouds on the handle's stream and returns (graph capturable).
        frames_ptr: device address of n descriptors (pack_viz_descs); status_ptr: device int32[n]; kept_ptr: device
        uint64[n] or 0; applied_ptr: device int32[n] or 0; encode_descs_ptr: device address of n cloud descriptors
        (cloudini_b200.pack_cloud_descs) whose cloud and size the call points at each frame's result, or 0. See
        cldn_b200_viz_lossy_preprocess_batch_async."""
        _check(_L().cldn_b200_viz_lossy_preprocess_batch_async(self._h, n, frames_ptr or None, status_ptr or None, kept_ptr or None,
                                                               applied_ptr or None, encode_descs_ptr or None))

    def sync(self):
        """Waits for the handle's stream."""
        _check(_L().cldn_b200_preproc_sync(self._h))


def viz_descs(descs):
    """numpy uint64 array [n, 4] of cldn_viz_desc_t: one (cloud_ptr, cloud_bytes, out_ptr, capacity) per frame, device
    addresses and sizes as run_batch_async() reads them (the layout of cldn_blob_desc_t)."""
    return blob_descs(descs)


def pack_viz_descs(descs, out=None):
    """The descriptors of viz_descs() in device memory, as pack_blob_descs() places them (32 bytes per frame). Returns
    the tensor; its data_ptr() is run_batch_async()'s frames_ptr."""
    return pack_blob_descs(descs, out)


def applyVizLossyPreprocessing(pc: RosPointCloud2, preprocessor: Optional[VizPreprocessor] = None) -> None:
    """ros_msg_utils.cpp:249-341 — edits ``pc`` in place (data, width, height, row_step, FLOAT64 resolutions)."""
    pp = preprocessor or VizPreprocessor()
    info = EncodingInfo(fields=list(pc.fields), width=pc.width, height=pc.height, point_step=pc.point_step)
    new_info, data, applied = pp.run(info, np.ascontiguousarray(pc.data, dtype=np.uint8))
    if not applied:
        return
    pc.data = data
    pc.width, pc.height = new_info.width, 1
    pc.row_step = pc.point_step * pc.width
    pc.fields = new_info.fields
