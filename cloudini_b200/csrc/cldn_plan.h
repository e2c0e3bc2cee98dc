// Internal (not part of the C ABI): flat POD description of how one EncodingInfo maps to the byte stream.
//
// This is the GPU counterpart of the reference's vector<unique_ptr<FieldEncoder>> / V5EncoderPlan:
// the planner (cldn_host.cpp) mirrors LeadingLossyFloatFieldCount / CreateCompatibleEncoder / CreateCompatibleDecoder
// (cloudini_lib/src/codec_common.cpp:69-198), BuildV4Encoders/Decoders (v4_codec.cpp:26-64), UsesV5Codec and
// buildV5Plan / getV5AdaptiveFields (v5_codec.cpp:719-763,883-892) and hands the kernels a fixed-size table
// instead of virtual objects.
#pragma once
#include <stddef.h>
#include <stdint.h>

#include "../../include/cloudini_b200.h"

namespace cldn {

constexpr uint32_t kChunkPoints = CLDN_POINTS_PER_CHUNK;  // codec_common.hpp:28
constexpr uint32_t kProbePoints = 4096;                   // v5_codec.cpp:76 kAdaptiveModeProbePoints
constexpr int kMaxOps = CLDN_MAX_FIELDS;

// One entry of the interleaved "regular" stream (one reference FieldEncoder/FieldDecoder object).
enum OpKind : uint8_t {
  OP_FLOATN = 0,     // FieldEncoderFloatN_Lossy  field_encoder.cpp:24-91   (3 or 4 f32 lanes, int32 ties-to-even)
  OP_F32_LOSSY = 1,  // FieldEncoderFloat_Lossy<float>   field_encoder.hpp:99-118,343-357 (int64, half away from zero)
  OP_F64_LOSSY = 2,  // FieldEncoderFloat_Lossy<double>
  OP_INT = 3,        // FieldEncoderInt<T>  field_encoder.hpp:72-94 (V4 interleaved delta varint)
  OP_COPY = 4,       // FieldEncoderCopy    field_encoder.hpp:51-67 (raw bytes)
  OP_XOR32 = 5,      // FieldEncoderFloat_XOR<float>     field_encoder.hpp:123-139,360-370 (raw XOR with the previous bits)
  OP_XOR64 = 6,      // FieldEncoderFloat_XOR<double>
  OP_GORILLA64 = 7,  // FieldEncoderFloat_Gorilla<double> field_encoder.hpp:157-312 (bit-packed, byte-aligned per value)
};

struct RegOp {
  uint8_t kind;      // OpKind
  uint8_t lanes;     // OP_FLOATN: 3|4, else 1
  uint8_t type;      // cldn_field_type_t of the field (OP_INT / OP_COPY)
  uint8_t size;      // bytes of the raw field (SizeOf(type))
  uint32_t offset[4];  // byte offset(s) inside the point; CLDN_SKIP_STORE_OFFSET honoured on decode
  float enc_mul_f[4];  // FloatN: 1.0F/res (field_encoder.cpp:34); F32_LOSSY: float(1.0/double(res)) (field_encoder.hpp:101-102)
  float dec_mul_f[4];  // decoder multiplier = resolution (field_decoder.cpp:33, field_decoder.hpp:113)
  double enc_mul_d;    // F64_LOSSY: 1.0/double(res)
  double dec_mul_d;    // F64_LOSSY: double(res)
};

// One V5 adaptive integer field (v5_codec.cpp:40-66 V5AdaptiveIntField).
struct SectionField {
  uint32_t offset;
  uint8_t type;  // cldn_field_type_t (INT16..UINT64)
  uint8_t bpv;   // bytes per value
  uint16_t field_index;
};

struct Plan {
  uint32_t point_step;
  uint32_t n_ops;
  RegOp ops[kMaxOps];
  uint32_t n_sections;  // > 0  <=>  UsesV5Codec(info)
  SectionField sections[kMaxOps];
  uint32_t max_point_bytes;   // worst-case bytes per point of the regular stream (this build's own bound, <= reference's)
  uint32_t min_point_bytes;   // BuildV4Decoders' min_encoded_point_bytes (v4_codec.cpp:43-63)
  uint32_t values_per_point;  // number of varint-coded values per point in the regular stream (if all_varint)
  uint8_t uses_v5;
  uint8_t floatn_only;  // regular stream is exactly one OP_FLOATN  -> specialised kernels
  uint8_t all_varint;   // every regular op is varint/NaN-marker coded -> terminator-scan decode applies
  uint8_t all_fixed;    // every regular op is fixed size (COPY)
  uint8_t supported;    // 0 if the plan contains ops this build cannot run at all
  uint8_t n_gorilla;    // number of OP_GORILLA64 ops (they need the sequential per-chunk pre-pass / decoder)
  uint8_t regular_overlap;  // decoder: two stored fields of the regular stream cover the same byte of a point. The reference
                            // stores per point in field order (last writer wins, v4_codec.cpp:85-117); only the per-chunk
                            // sequential decoder reproduces that order, so such plans are routed to it
  uint8_t pad_[1];
};

// Builds the ENCODER plan. Returns CLDN_OK or a negative status (message via set_error()).
int build_encode_plan(const cldn_info_t& info, Plan* plan);
// Builds the DECODER plan (CreateCompatibleDecoder has extra legacy branches, codec_common.cpp:157-198).
int build_decode_plan(const cldn_info_t& info, Plan* plan);

bool uses_v5_codec(const cldn_info_t& info);
size_t leading_lossy_float_count(const cldn_info_t& info);
size_t max_serialized_field_size(const cldn_field_t& f, uint8_t encoding_opt, bool* ok);

void set_error(const char* fmt, ...);
// Marks an encoder as one of the per-thread pool's (cldn_ros.cpp): the converter and the shims hand it to callers that
// were promised the system libraries' bytes, so it refuses cldn_b200_encoder_set_stage2_on_device(enc, 1).
void encoder_mark_pooled(cldn_encoder_t* enc);
int size_of_type(uint8_t type);

}  // namespace cldn
