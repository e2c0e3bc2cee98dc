// SURVEY.md §8(f) N2 — the DDS / ROS 2 envelope around the codec (cloudini_lib/src/ros_msg_utils.cpp:54-238).
// Host code: the CDR header of a PointCloud2 message is a few hundred bytes of text-like fields; the point payload is
// never touched here — it goes to the GPU codec through the C ABI (cldn_b200_encode / cldn_b200_decode).
// CDR rules restated from the reference's vendored nanocdr (include/cloudini_lib/contrib/nanocdr.hpp:252-293 decoder
// header checks, :346-368 / :391-414 primitives aligned to their size relative to the byte after the 4-byte
// encapsulation header, :313-333 / :417-424 strings = u32 length including the NUL + bytes).
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <string>
#include <vector>

#include "../../include/cloudini_b200_ros.h"
#include "cldn_plan.h"

using cldn::set_error;

namespace {

struct CdrReader {
  const uint8_t* base;
  size_t size, pos = 4;
  bool big = false;
  bool ok = true;
  const char* why = "";
  size_t remaining() const { return size - pos; }
  void align(size_t n) {  // nanocdr.hpp:135-138 (origin = buffer + 4)
    const size_t a = (n - ((pos - 4) % n)) & (n - 1);
    pos += (a <= remaining()) ? a : remaining();  // trim_front clamps; the size check that follows reports the error
  }
  uint32_t u32() {
    align(4);
    if (remaining() < 4) { fail("Decode: not enough data to decode"); return 0; }
    uint32_t v;
    memcpy(&v, base + pos, 4);
    pos += 4;
    return big ? __builtin_bswap32(v) : v;
  }
  uint8_t u8() {
    if (remaining() < 1) { fail("Decode: not enough data to decode"); return 0; }
    return base[pos++];
  }
  // returns offset / length (NUL stripped) of a string
  void str(size_t* off, uint32_t* len) {
    const uint32_t n = u32();
    if (!ok) return;
    if (remaining() < n) { fail("Decode: not enough data to decode (string)"); return; }
    *off = pos;
    *len = (n > 0 && base[pos + n - 1] == 0) ? n - 1 : n;
    pos += n;
  }
  void fail(const char* w) { if (ok) { ok = false; why = w; } }
};

struct CdrWriter {
  std::vector<uint8_t> buf;
  bool big = false;
  void align(size_t n) {  // nanocdr.hpp:196-199: (size - 4) % n
    const size_t a = (n - ((buf.size() - 4) % n)) & (n - 1);
    buf.resize(buf.size() + a);
  }
  void u32(uint32_t v) {
    align(4);
    if (big) v = __builtin_bswap32(v);
    const size_t at = buf.size();
    buf.resize(at + 4);
    memcpy(buf.data() + at, &v, 4);
  }
  void u8(uint8_t v) { buf.push_back(v); }
  void str(const char* s, size_t len) {
    u32(static_cast<uint32_t>(len + 1));
    buf.insert(buf.end(), reinterpret_cast<const uint8_t*>(s), reinterpret_cast<const uint8_t*>(s) + len);
    buf.push_back(0);
  }
};

// writePointCloudHeader (ros_msg_utils.cpp:97-120) after the 4-byte encapsulation header
void write_pc_header(CdrWriter& w, const cldn_ros_msg_t& m) {
  w.buf.assign({0, m.cdr_header[1], 0, 0});  // nanocdr.hpp:381-387
  w.big = (m.cdr_header[1] & 1u) == 0;
  w.u32(static_cast<uint32_t>(m.stamp_sec));
  w.u32(m.stamp_nsec);
  w.str(m.frame_id ? m.frame_id : "", m.frame_id ? m.frame_id_len : 0);
  w.u32(m.height);
  w.u32(m.width);
  w.u32(m.n_fields);
  for (uint32_t i = 0; i < m.n_fields; ++i) {
    w.str(m.fields[i].name, strlen(m.fields[i].name));
    w.u32(m.fields[i].offset);
    w.u8(m.fields[i].type);
    w.u32(1);  // count, not used
  }
  w.u8(0);  // is_bigendian, not used
  w.u32(m.point_step);
  w.u32(m.point_step * m.width);
}

}  // namespace

extern "C" {

int cldn_b200_ros_parse(const void* dds_msg, size_t msg_bytes, cldn_ros_msg_t* out) {
  if (!dds_msg || !out) { set_error("null argument"); return CLDN_ERR_INVALID_ARGUMENT; }
  memset(out, 0, sizeof(*out));
  const uint8_t* p = static_cast<const uint8_t*>(dds_msg);
  if (msg_bytes < 4) { set_error("Decode: not enough data to decode"); return CLDN_ERR_CORRUPT_DATA; }
  if (p[0] != 0) { set_error("Invalid CDR header: expected first byte to be 0"); return CLDN_ERR_CORRUPT_DATA; }
  if ((p[1] & 0xFEu) != 0) { set_error("Unexpected encoding received."); return CLDN_ERR_CORRUPT_DATA; }  // only PLAIN_CDR (DDS_CDR default)
  if (p[2] != 0 || p[3] != 0) { set_error("Extended header not supported"); return CLDN_ERR_CORRUPT_DATA; }
  memcpy(out->cdr_header, p, 4);
  CdrReader r{p, msg_bytes};
  r.big = (p[1] & 1u) == 0;
  out->stamp_sec = static_cast<int32_t>(r.u32());
  out->stamp_nsec = r.u32();
  size_t frame_off = 4;
  r.str(&frame_off, &out->frame_id_len);
  out->frame_id = reinterpret_cast<const char*>(p) + frame_off;
  out->height = r.u32();
  out->width = r.u32();
  const uint32_t n_fields = r.u32();
  if (r.ok && n_fields > CLDN_MAX_FIELDS) {
    set_error("PointCloud2 with %u fields: this build handles at most %d", n_fields, CLDN_MAX_FIELDS);
    return CLDN_ERR_UNSUPPORTED;
  }
  for (uint32_t i = 0; r.ok && i < n_fields; ++i) {
    size_t off = 0;
    uint32_t len = 0;
    r.str(&off, &len);
    if (!r.ok) break;
    if (len >= CLDN_MAX_NAME) { set_error("field name longer than %d characters", CLDN_MAX_NAME - 1); return CLDN_ERR_UNSUPPORTED; }
    // the reference keeps such a name as a std::string with the NUL inside and writes it back at full length; a C
    // string cannot, and silently shortening it would change the bytes of the converted message
    if (memchr(p + off, 0, len)) { set_error("field name with an embedded NUL character"); return CLDN_ERR_UNSUPPORTED; }
    cldn_field_t& f = out->fields[i];
    memcpy(f.name, p + off, len);
    f.name[len] = 0;
    f.offset = r.u32();
    f.type = r.u8();
    (void)r.u32();  // count
  }
  out->n_fields = r.ok ? n_fields : 0;
  out->is_bigendian = r.u8();
  out->point_step = r.u32();
  out->row_step = r.u32();
  const uint32_t data_len = r.u32();
  if (r.ok && r.remaining() < data_len) r.fail("Decode: not enough data to decode (string)");
  if (r.ok) {
    out->data = p + r.pos;
    out->data_bytes = data_len;
    r.pos += data_len;
  }
  out->is_dense = r.u8();
  if (!r.ok) { set_error("%s", r.why); return CLDN_ERR_CORRUPT_DATA; }
  return CLDN_OK;
}

int cldn_b200_ros_to_encoding_info(const cldn_ros_msg_t* msg, cldn_info_t* info) {
  if (!msg || !info) { set_error("null argument"); return CLDN_ERR_INVALID_ARGUMENT; }
  cldn_b200_info_init(info);  // LOSSY + ZSTD are the EncodingInfo defaults toEncodingInfo sets again (:127-128)
  info->height = msg->height;
  info->width = msg->width;
  info->point_step = msg->point_step;
  info->encoding_opt = CLDN_ENC_LOSSY;
  info->compression_opt = CLDN_COMP_ZSTD;
  info->n_fields = msg->n_fields;
  memcpy(info->fields, msg->fields, sizeof(cldn_field_t) * msg->n_fields);
  return CLDN_OK;
}

int cldn_b200_ros_apply_resolution_profile(cldn_field_t* fields, uint32_t* n_fields, const char* const* names,
                                           const float* resolutions, size_t n_profile, const float* default_resolution) {
  if (!fields || !n_fields || (n_profile && (!names || !resolutions))) { set_error("null argument"); return CLDN_ERR_INVALID_ARGUMENT; }
  if (*n_fields > CLDN_MAX_FIELDS) { set_error("too many fields"); return CLDN_ERR_INVALID_ARGUMENT; }
  // std::map semantics: the profile is keyed by name; with duplicate names in the arrays the LAST entry is the one a
  // caller building the map with operator[] would end up with
  auto find = [&](const char* name) -> const float* {
    for (size_t k = n_profile; k-- > 0;) if (strcmp(names[k], name) == 0) return &resolutions[k];
    return nullptr;
  };
  uint32_t w = 0;
  for (uint32_t i = 0; i < *n_fields; ++i) {  // erase-remove of fields whose profile resolution is 0 (:221-229)
    const float* r = find(fields[i].name);
    if (r && *r == 0.0f) continue;
    if (w != i) fields[w] = fields[i];
    ++w;
  }
  for (uint32_t i = w; i < *n_fields; ++i) memset(&fields[i], 0, sizeof(cldn_field_t));
  *n_fields = w;
  for (uint32_t i = 0; i < w; ++i) {  // :231-237
    cldn_field_t& f = fields[i];
    if (const float* r = find(f.name)) {
      f.has_resolution = 1;
      f.resolution = *r;
    } else if (default_resolution && f.type == CLDN_FLOAT32) {
      f.has_resolution = 1;
      f.resolution = *default_resolution;
    }
  }
  return CLDN_OK;
}

int cldn_b200_ros_compress_msg(cldn_encoder_t* enc, const cldn_ros_msg_t* msg, void* out, size_t out_capacity, size_t* written) {
  if (!enc || !msg || (!msg->data && msg->data_bytes)) { set_error("null argument"); return CLDN_ERR_INVALID_ARGUMENT; }
  const uint8_t* data = msg->data;
  const size_t data_bytes = msg->data_bytes;
  cldn_info_t info;
  if (int rc = cldn_b200_encoder_info(enc, &info)) return rc;
  CdrWriter w;
  write_pc_header(w, *msg);
  w.u32(0);  // compressed_data length, patched below (:177-181)
  const size_t size_at = w.buf.size() - 4, prev = w.buf.size();
  size_t blob_cap = 0;
  if (data_bytes != 0) {
    if (info.point_step == 0) { set_error("convertPointCloud2ToCompressedCloud: point_step cannot be 0"); return CLDN_ERR_INVALID_ARGUMENT; }
    blob_cap = cldn_b200_max_compressed_size(&info, data_bytes / info.point_step, 1);  // :193-196
    if (blob_cap == 0) return CLDN_ERR_INVALID_ARGUMENT;
  }
  const size_t worst = prev + blob_cap + 1 + 3 + 4 + 9;
  if (!out) {
    if (written) *written = worst;
    return CLDN_OK;
  }
  if (out_capacity < worst) { set_error("output buffer smaller than the worst-case message (%zu bytes)", worst); return CLDN_ERR_BUFFER_TOO_SMALL; }
  uint8_t* o = static_cast<uint8_t*>(out);
  memcpy(o, w.buf.data(), prev);
  size_t blob = 0;
  if (data_bytes != 0) {
    if (int rc = cldn_b200_encode(enc, data, data_bytes, o + prev, blob_cap, 1, &blob, CLDN_MEM_HOST)) return rc;
    const uint32_t sz = static_cast<uint32_t>(blob);
    memcpy(o + size_at, &sz, 4);  // the reference memcpy's the native value, whatever the message's endianness (:203)
  }
  // trailing fields (:209-212): is_dense (1 byte, no alignment), then format = "cloudini" (u32 length 9 aligned to 4
  // relative to the byte after the encapsulation header, characters, NUL)
  size_t pos = prev + blob;
  o[pos++] = msg->is_dense;
  while ((pos - 4) % 4) o[pos++] = 0;
  uint32_t len = 9;
  if (w.big) len = __builtin_bswap32(len);
  memcpy(o + pos, &len, 4);
  memcpy(o + pos + 4, "cloudini", 9);
  if (written) *written = pos + 13;
  return CLDN_OK;
}

int cldn_b200_ros_decompress_msg(cldn_decoder_t* dec, const cldn_ros_msg_t* msg, void* out, size_t out_capacity, size_t* written) {
  if (!dec || !msg || (!msg->data && msg->data_bytes)) { set_error("null argument"); return CLDN_ERR_INVALID_ARGUMENT; }
  // uint32 arithmetic like the reference (width * height * point_step, :136)
  const size_t cloud_bytes = static_cast<uint32_t>(msg->width * msg->height * msg->point_step);
  CdrWriter w;
  write_pc_header(w, *msg);
  w.u32(static_cast<uint32_t>(cloud_bytes));
  const size_t prev = w.buf.size();
  const size_t total = prev + cloud_bytes + 1;
  if (!out) {
    if (written) *written = total;
    return CLDN_OK;
  }
  if (out_capacity < total) { set_error("output buffer smaller than the message (%zu bytes)", total); return CLDN_ERR_BUFFER_TOO_SMALL; }
  uint8_t* o = static_cast<uint8_t*>(out);
  memcpy(o, w.buf.data(), prev);
  if (cloud_bytes != 0) {
    const uint8_t* blob = msg->data;
    cldn_info_t info;
    size_t hdr = 0;
    if (int rc = cldn_b200_decode_header(blob, msg->data_bytes, &info, &hdr)) return rc;
    memset(o + prev, 0, cloud_bytes);  // std::vector::resize zero-fills; the decoder only writes declared field bytes (:153)
    if (int rc = cldn_b200_decode(dec, &info, blob + hdr, msg->data_bytes - hdr, o + prev, cloud_bytes, CLDN_MEM_HOST)) return rc;
  }
  o[prev + cloud_bytes] = msg->is_dense;
  if (written) *written = total;
  return CLDN_OK;
}

}  // extern "C"

// ---- per-thread handle pool: the converter step and the one-shots below reuse handles instead of creating streams, device
// buffers and pinned memory for every message (handles are single-threaded, so the pool is too; it is never torn down:
// at process exit the driver may already be gone) ---------------------------------------------------------------------------
namespace {
struct LayoutKey {
  cldn_info_t info;  // width / height zeroed
  bool same(const cldn_info_t& o) const {
    if (info.point_step != o.point_step || info.encoding_opt != o.encoding_opt || info.compression_opt != o.compression_opt ||
        info.version != o.version || info.n_fields != o.n_fields) return false;
    for (uint32_t i = 0; i < o.n_fields; ++i) {
      const cldn_field_t &a = info.fields[i], &b = o.fields[i];
      if (strncmp(a.name, b.name, CLDN_MAX_NAME) != 0 || a.offset != b.offset || a.type != b.type || a.has_resolution != b.has_resolution ||
          (a.has_resolution && memcmp(&a.resolution, &b.resolution, 4) != 0)) return false;
    }
    return true;
  }
};
struct HandlePool {
  cudaStream_t stream = nullptr;
  std::vector<std::pair<LayoutKey, cldn_encoder_t*>> encoders;  // most recently used first
  cldn_decoder_t* decoder = nullptr;
  cldn_preproc_t* preproc = nullptr;
  uint8_t *d_in = nullptr, *d_mid = nullptr, *d_blob = nullptr;
  size_t cap_in = 0, cap_mid = 0, cap_blob = 0;
  bool ready() {
    if (stream) return true;
    return cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking) == cudaSuccess;
  }
  static bool grow(uint8_t** p, size_t* cap, size_t need) {
    if (need <= *cap) return true;
    if (*p) cudaFree(*p);
    *p = nullptr; *cap = 0;
    const size_t want = need + need / 4 + 4096;
    if (cudaMalloc(reinterpret_cast<void**>(p), want) != cudaSuccess) return false;
    *cap = want;
    return true;
  }
  cldn_encoder_t* encoder_for(const cldn_info_t& info) {
    for (size_t i = 0; i < encoders.size(); ++i) {
      if (encoders[i].first.same(info)) {
        auto hit = encoders[i];
        encoders.erase(encoders.begin() + i);
        encoders.insert(encoders.begin(), hit);
        if (cldn_b200_encoder_set_dims(hit.second, info.width, info.height) != CLDN_OK) return nullptr;
        return hit.second;
      }
    }
    if (!ready()) { set_error("cudaStreamCreate failed"); return nullptr; }
    cldn_encoder_t* enc = nullptr;
    if (cldn_b200_encoder_create(&info, -1, stream, &enc) != CLDN_OK) return nullptr;
    cldn::encoder_mark_pooled(enc);  // the converter and the shims promise the system libraries' bytes
    LayoutKey k;
    k.info = info;
    encoders.insert(encoders.begin(), {k, enc});
    if (encoders.size() > 8) {  // bounded: a process talks to a handful of sensor layouts
      cldn_b200_encoder_destroy(encoders.back().second);
      encoders.pop_back();
    }
    return enc;
  }
  cldn_decoder_t* the_decoder() {
    if (!decoder && ready() && cldn_b200_decoder_create(-1, stream, &decoder) != CLDN_OK) decoder = nullptr;
    return decoder;
  }
  cldn_preproc_t* the_preproc() {
    if (!preproc && ready() && cldn_b200_preproc_create(-1, stream, &preproc) != CLDN_OK) preproc = nullptr;
    return preproc;
  }
};
HandlePool& pool() {
  static thread_local HandlePool* p = new HandlePool();  // deliberately leaked (see above)
  return *p;
}
}  // namespace

extern "C" int cldn_b200_pool_encoder(const cldn_info_t* info, cldn_encoder_t** out) {
  if (!info || !out) { set_error("null argument"); return CLDN_ERR_INVALID_ARGUMENT; }
  *out = pool().encoder_for(*info);
  return *out ? CLDN_OK : CLDN_ERR_INVALID_ARGUMENT;
}
extern "C" int cldn_b200_pool_decoder(cldn_decoder_t** out) {
  if (!out) { set_error("null argument"); return CLDN_ERR_INVALID_ARGUMENT; }
  *out = pool().the_decoder();
  return *out ? CLDN_OK : CLDN_ERR_CUDA;
}
extern "C" int cldn_b200_pool_preproc(cldn_preproc_t** out) {
  if (!out) { set_error("null argument"); return CLDN_ERR_INVALID_ARGUMENT; }
  *out = pool().the_preproc();
  return *out ? CLDN_OK : CLDN_ERR_CUDA;
}

extern "C" int cldn_b200_ros_convert_msg(const void* dds_msg, size_t msg_bytes, const char* const* names, const float* resolutions,
                                         size_t n_profile, const float* default_resolution, int viz, int encoding_opt,
                                         int compression_opt, int version, void* out, size_t out_capacity, size_t* written) {
  cldn_ros_msg_t m;
  if (int rc = cldn_b200_ros_parse(dds_msg, msg_bytes, &m)) return rc;
  if (int rc = cldn_b200_ros_apply_resolution_profile(m.fields, &m.n_fields, names, resolutions, n_profile, default_resolution)) return rc;
  cldn_info_t info;
  if (int rc = cldn_b200_ros_to_encoding_info(&m, &info)) return rc;
  info.encoding_opt = static_cast<uint8_t>(encoding_opt);
  info.compression_opt = static_cast<uint8_t>(compression_opt);
  info.version = static_cast<uint8_t>(version);
  info.use_threads = 0;
  HandlePool& P = pool();
  if (!P.ready()) { set_error("cudaStreamCreate failed"); return CLDN_ERR_CUDA; }
  const size_t step = m.point_step;
  const size_t points_in = step ? m.data_bytes / step : 0;
  // worst-case size of the output message (before preprocessing: it only ever shrinks the cloud)
  {
    cldn_encoder_t* probe = P.encoder_for(info);
    if (!probe) return CLDN_ERR_INVALID_ARGUMENT;
    size_t worst = 0;
    if (int rc = cldn_b200_ros_compress_msg(probe, &m, nullptr, 0, &worst)) return rc;
    if (!out) { if (written) *written = worst; return CLDN_OK; }
    if (out_capacity < worst) { set_error("output buffer smaller than the worst-case message (%zu bytes)", worst); return CLDN_ERR_BUFFER_TOO_SMALL; }
  }
  if (compression_opt != CLDN_COMP_NONE || m.data_bytes == 0 || step == 0 || m.data_bytes % step != 0) {
    // stage 2 runs in the host libraries (and degenerate messages take the plain path): preprocessing through the host API
    std::vector<uint8_t> kept_data;
    if (viz && m.data_bytes) {
      cldn_preproc_t* pp = P.the_preproc();
      if (!pp) return CLDN_ERR_CUDA;
      kept_data.resize(m.data_bytes);
      size_t kept = 0;
      int applied = 0;
      if (int rc = cldn_b200_viz_lossy_preprocess(pp, &info, m.data, m.data_bytes, kept_data.data(), kept_data.size(), &kept, &applied, CLDN_MEM_HOST)) return rc;
      if (applied) {
        m.data = kept_data.data(); m.data_bytes = kept * step; m.width = info.width; m.height = 1; m.row_step = m.point_step * m.width;
        for (uint32_t i = 0; i < info.n_fields; ++i) m.fields[i] = info.fields[i];
      }
    }
    cldn_encoder_t* enc = P.encoder_for(info);
    if (!enc) return CLDN_ERR_INVALID_ARGUMENT;
    return cldn_b200_ros_compress_msg(enc, &m, out, out_capacity, written);
  }
  // ---- device-resident: one upload, kernels, one download ----
  if (!HandlePool::grow(&P.d_in, &P.cap_in, m.data_bytes)) { set_error("cudaMalloc failed"); return CLDN_ERR_CUDA; }
  if (cudaMemcpyAsync(P.d_in, m.data, m.data_bytes, cudaMemcpyHostToDevice, P.stream) != cudaSuccess) { set_error("upload failed"); return CLDN_ERR_CUDA; }
  const uint8_t* d_cloud = P.d_in;
  size_t n_points = points_in;
  if (viz) {
    cldn_preproc_t* pp = P.the_preproc();
    if (!pp) return CLDN_ERR_CUDA;
    if (!HandlePool::grow(&P.d_mid, &P.cap_mid, m.data_bytes)) { set_error("cudaMalloc failed"); return CLDN_ERR_CUDA; }
    size_t kept = 0;
    int applied = 0;
    if (int rc = cldn_b200_viz_lossy_preprocess(pp, &info, P.d_in, m.data_bytes, P.d_mid, P.cap_mid, &kept, &applied, CLDN_MEM_DEVICE)) return rc;
    if (applied) {
      d_cloud = P.d_mid; n_points = kept;
      m.width = info.width; m.height = 1; m.row_step = m.point_step * m.width;
      for (uint32_t i = 0; i < info.n_fields; ++i) m.fields[i] = info.fields[i];
    }
  }
  cldn_encoder_t* enc = P.encoder_for(info);
  if (!enc) return CLDN_ERR_INVALID_ARGUMENT;
  const size_t blob_cap = cldn_b200_max_compressed_size(&info, n_points, 1);
  if (blob_cap == 0) return CLDN_ERR_INVALID_ARGUMENT;
  if (!HandlePool::grow(&P.d_blob, &P.cap_blob, blob_cap)) { set_error("cudaMalloc failed"); return CLDN_ERR_CUDA; }
  size_t blob = 0;
  if (int rc = cldn_b200_encode(enc, d_cloud, n_points * step, P.d_blob, blob_cap, 1, &blob, CLDN_MEM_DEVICE)) return rc;
  // message: header, u32 blob size, blob, is_dense, "cloudini" (convertPointCloud2ToCompressedCloud, :167-213)
  CdrWriter w;
  write_pc_header(w, m);
  w.u32(0);
  const size_t size_at = w.buf.size() - 4, prev = w.buf.size();
  uint8_t* o = static_cast<uint8_t*>(out);
  memcpy(o, w.buf.data(), prev);
  if (cudaMemcpyAsync(o + prev, P.d_blob, blob, cudaMemcpyDeviceToHost, P.stream) != cudaSuccess || cudaStreamSynchronize(P.stream) != cudaSuccess) {
    set_error("download failed");
    return CLDN_ERR_CUDA;
  }
  const uint32_t sz = static_cast<uint32_t>(blob);
  memcpy(o + size_at, &sz, 4);
  size_t pos = prev + blob;
  o[pos++] = m.is_dense;
  while ((pos - 4) % 4) o[pos++] = 0;
  uint32_t len = 9;
  if (w.big) len = __builtin_bswap32(len);
  memcpy(o + pos, &len, 4);
  memcpy(o + pos + 4, "cloudini", 9);
  if (written) *written = pos + 13;
  return CLDN_OK;
}

extern "C" {

// ---- the DDS-message half of the reference's own C ABI (src/wasm_functions.cpp:24-226) ------------------------------------
uint32_t cldn_b200_GetHeaderAsYAML(const void* encoded_data, uint32_t encoded_data_size, char* output_yaml, uint32_t capacity) {
  if (!encoded_data || !output_yaml) { set_error("null argument"); return 0; }
  cldn_info_t info;
  size_t hdr = 0, need = 0;
  if (cldn_b200_decode_header(static_cast<const uint8_t*>(encoded_data), encoded_data_size, &info, &hdr) != CLDN_OK) return 0;
  cldn_b200_info_to_yaml(&info, nullptr, 0, &need);  // strlen + 1
  std::vector<char> text(need);
  if (cldn_b200_info_to_yaml(&info, text.data(), text.size(), nullptr) != CLDN_OK) return 0;
  const uint32_t n = static_cast<uint32_t>(need ? need - 1 : 0);
  if (n > capacity) { set_error("output buffer too small for the YAML text (%u bytes)", n); return 0; }
  memcpy(output_yaml, text.data(), n);  // like the reference: no terminator is written (:36-38)
  return n;
}

uint32_t cldn_b200_GetHeaderAsYAMLFromDDS(const void* raw_dds_msg, uint32_t dds_msg_size, char* output_yaml, uint32_t capacity) {
  cldn_ros_msg_t m;
  if (cldn_b200_ros_parse(raw_dds_msg, dds_msg_size, &m) != CLDN_OK) return 0;
  return cldn_b200_GetHeaderAsYAML(m.data, static_cast<uint32_t>(m.data_bytes), output_yaml, capacity);
}

uint32_t cldn_b200_GetDecompressedSize(const void* encoded_dds_msg, uint32_t encoded_dds_size) {
  cldn_ros_msg_t m;
  if (cldn_b200_ros_parse(encoded_dds_msg, encoded_dds_size, &m) != CLDN_OK) return 0;
  return m.height * m.width * m.point_step;
}

// parse + toEncodingInfo + "every FLOAT32 field gets `resolution`" (wasm_functions.cpp:63-73, 184-194)
static bool message_encoding_info(const void* msg, uint32_t size, float resolution, cldn_ros_msg_t* m, cldn_info_t* info) {
  if (cldn_b200_ros_parse(msg, size, m) != CLDN_OK || cldn_b200_ros_to_encoding_info(m, info) != CLDN_OK) return false;
  for (uint32_t i = 0; i < info->n_fields; ++i) {
    if (info->fields[i].type == CLDN_FLOAT32) {
      info->fields[i].has_resolution = 1;
      info->fields[i].resolution = resolution;
    }
  }
  return true;
}

static uint32_t encode_message_payload(const cldn_ros_msg_t& m, const cldn_info_t& info, std::vector<uint8_t>* blob) {
  cldn_encoder_t* enc = pool().encoder_for(info);  // reused across messages of the same layout
  if (!enc) return 0;
  const size_t cap = info.point_step ? cldn_b200_max_compressed_size(&info, m.data_bytes / info.point_step, 1) : 0;
  blob->resize(cap);
  size_t written = 0;
  const int rc = cap ? cldn_b200_encode(enc, m.data, m.data_bytes, blob->data(), blob->size(), 1, &written, CLDN_MEM_HOST) : CLDN_ERR_INVALID_ARGUMENT;
  return rc == CLDN_OK ? static_cast<uint32_t>(written) : 0;
}

uint32_t cldn_b200_ComputeCompressedSize(const void* dds_msg, uint32_t dds_msg_size, float resolution) {
  cldn_ros_msg_t m;
  cldn_info_t info;
  if (!message_encoding_info(dds_msg, dds_msg_size, resolution, &m, &info)) return 0;
  const size_t expected = static_cast<size_t>(m.width) * m.height * m.point_step;
  if (m.data_bytes != expected && (m.width == 0 || m.height == 0)) return 0;  // :81-86
  std::vector<uint8_t> blob;
  return encode_message_payload(m, info, &blob);
}

uint32_t cldn_b200_EncodePointcloudMessage(const void* pointcloud_msg, uint32_t msg_size, float resolution, void* output_data,
                                           uint32_t capacity) {
  if (!output_data) { set_error("null argument"); return 0; }
  cldn_ros_msg_t m;
  cldn_info_t info;
  if (!message_encoding_info(pointcloud_msg, msg_size, resolution, &m, &info)) return 0;
  const size_t expected = static_cast<size_t>(m.width) * m.height * m.point_step;
  if (m.data_bytes != expected) { set_error("Data size mismatch"); return 0; }  // :197-201
  std::vector<uint8_t> blob;
  const uint32_t n = encode_message_payload(m, info, &blob);
  if (n == 0) return 0;
  if (n > capacity) { set_error("Output buffer too small for encoded message"); return 0; }  // :217-220
  memcpy(output_data, blob.data(), n);
  return n;
}

uint32_t cldn_b200_ConvertCompressedMsgToPointCloud2Msg(const void* compressed_msg, uint32_t msg_size, void* output_msg, uint32_t capacity) {
  if (!output_msg) { set_error("null argument"); return 0; }
  cldn_ros_msg_t m;
  if (cldn_b200_ros_parse(compressed_msg, msg_size, &m) != CLDN_OK) return 0;
  cldn_decoder_t* dec = pool().the_decoder();
  if (!dec) return 0;
  size_t written = 0;
  const int rc = cldn_b200_ros_decompress_msg(dec, &m, output_msg, capacity, &written);
  return rc == CLDN_OK ? static_cast<uint32_t>(written) : 0;
}

uint32_t cldn_b200_DecodeCompressedMessage(const void* compressed_msg, uint32_t msg_size, void* output_data, uint32_t capacity) {
  cldn_ros_msg_t m;
  if (cldn_b200_ros_parse(compressed_msg, msg_size, &m) != CLDN_OK) return 0;
  return cldn_b200_DecodeCompressedData(m.data, static_cast<uint32_t>(m.data_bytes), output_data, capacity);
}

}  // extern "C"
