/*
 * cloudini_b200 — C ABI of the H100-native (sm_90a) Cloudini stage-1 point-cloud codec.
 *
 * This is the drop-in boundary: plain pointers and sizes, no C++ / torch types. Every entry point names the
 * reference interface it replaces (paths relative to the reference tree, cloudini_lib/...). The reference-side
 * bindings a maintainer would add on top of this header are shown in INTEGRATION.md; a header-only C++ shim that
 * re-creates Cloudini::PointcloudEncoder / PointcloudDecoder on top of it lives in include/cloudini_b200/cloudini.hpp.
 *
 * Conventions
 *  - All functions return CLDN_OK (0) or a negative cldn_status_t; cldn_b200_last_error() returns the message of the
 *    last failure on the calling thread. The reference throws std::runtime_error at the same places (cited below) and
 *    its own C ABI (include/cloudini_lib/wasm_functions.h:30-93) maps every failure to "return 0".
 *  - There is NO CPU fallback. Entry points that launch kernels fail with CLDN_ERR_CUDA when no sm_90 device exists.
 *    Pure host helpers (header, YAML, sizing, planning) work without a GPU.
 *  - Buffers are owned by the caller. `mem` says where they live: CLDN_MEM_HOST (pageable or pinned host memory;
 *    the library stages through pinned buffers and its own stream — this is the drop-in path used by
 *    cloudini_ros/src/cloudini_publisher_plugin.cpp:73-74), CLDN_MEM_DEVICE (device pointers; launch-only,
 *    asynchronous on the handle's stream) or CLDN_MEM_DEVICE_POINTS (points in device memory, blobs and payloads in
 *    host memory: see cldn_mem_t).
 *  - Handles are not thread-safe (same as the reference's PointcloudEncoder, cloudini.hpp:185-208): one handle per
 *    thread / stream.
 */
#ifndef CLOUDINI_B200_H_
#define CLOUDINI_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define CLDN_MAX_FIELDS 32
#define CLDN_MAX_NAME 64
#define CLDN_POINTS_PER_CHUNK 32768u /* codec_common.hpp:28 kPointsPerChunk */
#define CLDN_ENCODING_VERSION 5      /* cloudini.hpp:63 kEncodingVersion */
#define CLDN_SKIP_STORE_OFFSET 0xFFFFFFFFu /* basic_types.hpp:71 kDecodeButSkipStore */

typedef enum cldn_status_t {
  CLDN_OK = 0,
  CLDN_ERR_INVALID_ARGUMENT = -1, /* reference: std::runtime_error from argument validation (cloudini.cpp:502-507) */
  CLDN_ERR_BUFFER_TOO_SMALL = -2, /* cloudini.cpp:531-534, v4_codec.cpp:93-95 */
  CLDN_ERR_BAD_HEADER = -3,       /* cloudini.cpp:353-372 */
  CLDN_ERR_CORRUPT_DATA = -4,     /* encoding_utils.hpp:98-148, v5_codec.cpp:764-879, cloudini.cpp:645-664 */
  CLDN_ERR_UNSUPPORTED = -5,      /* a plan this build does not accelerate (see DESIGN.md "out of scope") */
  CLDN_ERR_CUDA = -6,             /* CUDA runtime failure / no sm_90 device: there is no CPU fallback */
  CLDN_ERR_INTERNAL = -7
} cldn_status_t;

/* basic_types.hpp:29-48 FieldType (values 1..8 match sensor_msgs/PointField) */
typedef enum cldn_field_type_t {
  CLDN_UNKNOWN = 0, CLDN_INT8 = 1, CLDN_UINT8 = 2, CLDN_INT16 = 3, CLDN_UINT16 = 4, CLDN_INT32 = 5,
  CLDN_UINT32 = 6, CLDN_FLOAT32 = 7, CLDN_FLOAT64 = 8, CLDN_INT64 = 9, CLDN_UINT64 = 10
} cldn_field_type_t;

/* cloudini.hpp:31-53 EncodingOptions / CompressionOption */
typedef enum cldn_encoding_opt_t { CLDN_ENC_NONE = 0, CLDN_ENC_LOSSY = 1, CLDN_ENC_LOSSLESS = 2 } cldn_encoding_opt_t;
typedef enum cldn_compression_opt_t { CLDN_COMP_NONE = 0, CLDN_COMP_LZ4 = 1, CLDN_COMP_ZSTD = 2 } cldn_compression_opt_t;

/* Where the buffers of a call live.
 * CLDN_MEM_HOST: clouds, blobs, payloads and decoded points are host memory.
 * CLDN_MEM_DEVICE: all of them are device memory.
 * CLDN_MEM_DEVICE_POINTS: point clouds (encode inputs) and decoded points (decode outputs) are DEVICE pointers; blobs
 *   and payloads (encode outputs, decode inputs) are HOST pointers. For a GPU producer or consumer of messages that
 *   travel through host memory: only the compressed bytes cross PCIe. Accepted by cldn_b200_encode, _encode_batch,
 *   _encode_blobs, cldn_b200_decode, _decode_batch and _decode_blobs. It takes the routes of CLDN_MEM_HOST with the
 *   points read and written in place, so:
 *   - every blob equals what CLDN_MEM_HOST writes for the same cloud: stage 2 runs through the system liblz4 / libzstd
 *     (LZ4 and ZSTD blobs are the reference's bytes; ZSTD is supported);
 *   - every decoded buffer equals what CLDN_MEM_HOST gives: only declared field bytes of the caller's device buffer are
 *     written (padding untouched). Stage 2 is undone as for CLDN_MEM_HOST: ZSTD on the device (the system libzstd with
 *     CLDN_B200_ZSTD_HOST=1), LZ4 by the system liblz4 on the host, then uploaded;
 *   - statuses and messages (per frame, cldn_b200_decoder_frame_error) are those of CLDN_MEM_HOST: damaged blobs,
 *     too-small capacities, a payload that still carries its header, a cloud that is not a whole number of points.
 *     Nothing is written outside [0, capacity) of any buffer, host or device;
 *   - device memory is ordered on the handle's stream only, as for CLDN_MEM_DEVICE. Encode returns when the blobs and
 *     `written` are in host memory; decode_blobs returns with the statuses; decode / decode_batch return once the host
 *     payloads are no longer read, and `sync` == 0 leaves the device error word to cldn_b200_decoder_sync, as for
 *     CLDN_MEM_DEVICE. */
typedef enum cldn_mem_t { CLDN_MEM_HOST = 0, CLDN_MEM_DEVICE = 1, CLDN_MEM_DEVICE_POINTS = 2 } cldn_mem_t;

/* POD mirror of Cloudini::PointField (basic_types.hpp:50-66) */
typedef struct cldn_field_t {
  char name[CLDN_MAX_NAME]; /* NUL-terminated */
  uint32_t offset;          /* byte offset inside a point; CLDN_SKIP_STORE_OFFSET on decode = decode but do not store */
  uint8_t type;             /* cldn_field_type_t */
  uint8_t has_resolution;   /* std::optional<float>::has_value() */
  uint8_t reserved_[2];
  float resolution;         /* max quantisation error = resolution / 2 */
} cldn_field_t;

/* POD mirror of Cloudini::EncodingInfo (cloudini.hpp:65-111) */
typedef struct cldn_info_t {
  uint32_t width;
  uint32_t height;
  uint32_t point_step;
  uint8_t encoding_opt;    /* cldn_encoding_opt_t, default LOSSY */
  uint8_t compression_opt; /* cldn_compression_opt_t. NONE everywhere. LZ4: both APIs (device kernels; the host-pointer
                              API hands each chunk to the system liblz4). ZSTD: decode with both APIs on the device;
                              encode with host blobs only (CLDN_MEM_HOST, CLDN_MEM_DEVICE_POINTS), each chunk handed to
                              the system libzstd (dlopen) */
  uint8_t version;         /* wire version 2..5, default 5 */
  uint8_t use_threads;     /* accepted for API parity; ignored (there is no stage-2 worker thread here) */
  uint32_t n_fields;
  cldn_field_t fields[CLDN_MAX_FIELDS];
  char encoding_config[128];
} cldn_info_t;

typedef struct cldn_encoder cldn_encoder_t; /* replaces Cloudini::PointcloudEncoder (cloudini.hpp:154-211) */
typedef struct cldn_decoder cldn_decoder_t; /* replaces Cloudini::PointcloudDecoder (cloudini.hpp:216-244) */

/* ---- library ------------------------------------------------------------------------------------------------- */
const char* cldn_b200_version(void);
/* Message of the last failure on this thread ("" if none). Replaces e.what() of the reference's exceptions. */
const char* cldn_b200_last_error(void);
/* Number of kernels this library has launched in this process (bench.py reports it as gpu_launches). */
uint64_t cldn_b200_kernel_launch_count(void);
/* Host-side placement for the host-pointer API (no reference counterpart: the reference never leaves the CPU).
 * Binds the CALLING thread (and the threads it creates afterwards) to the CPUs of the NUMA node that `device` (-1: the
 * current one) hangs off, as NVML reports them, so that buffers the thread allocates and pins from now on are local to
 * the GPU's PCIe root: on a two-socket host a remote node halves the achievable host<->device bandwidth when several
 * GPUs stream at once. Returns the number of CPUs in the set, 0 if NVML / the affinity call is unavailable (nothing
 * changed), or a negative status. */
int cldn_b200_bind_host_thread_to_device(int device);

/* ---- configuration <-> text (host only) ---------------------------------------------------------------------- */
void cldn_b200_info_init(cldn_info_t* info); /* EncodingInfo defaults, cloudini.hpp:65-90 */
/* EncodingInfoToYAML (cloudini.cpp:165-190). Writes a NUL-terminated string; *needed (optional) gets strlen+1. */
int cldn_b200_info_to_yaml(const cldn_info_t* info, char* out, size_t capacity, size_t* needed);
/* EncodingInfoFromYAML (cloudini.cpp:192-230). `version` is taken from the text. */
int cldn_b200_info_from_yaml(const char* yaml, size_t yaml_len, cldn_info_t* info);

/* ---- header + sizing (host only) ----------------------------------------------------------------------------- */
/* EncodeHeader, YAML flavour (cloudini.cpp:294-318): "CLOUDINI_V" + 2 digits + '\n' + yaml + '\0'. */
int cldn_b200_encode_header(const cldn_info_t* info, uint8_t* out, size_t capacity, size_t* written);
/* EncodeHeader, HeaderEncoding::BINARY (cloudini.cpp:319-344): the legacy fixed-layout header (magic + version digits,
 * width, height, point_step, options, fields). PointcloudEncoder never writes it (cloudini.cpp:430-440 uses YAML);
 * it exists for callers of the free function. Call with out == NULL to query the size through *written. */
int cldn_b200_encode_header_binary(const cldn_info_t* info, uint8_t* out, size_t capacity, size_t* written);
/* DecodeHeader (cloudini.cpp:353-428): YAML and legacy binary headers. `blob` must be host memory.
 * *header_bytes = number of bytes consumed (the reference advances the caller's view by the same amount). */
int cldn_b200_decode_header(const uint8_t* blob, size_t blob_bytes, cldn_info_t* info, size_t* header_bytes);
/* MaxCompressedSize (cloudini.cpp:249-292). Returns 0 and sets the error on failure (point_step == 0 ...). */
size_t cldn_b200_max_compressed_size(const cldn_info_t* info, size_t points_count, int include_header);

/* ---- encoder -------------------------------------------------------------------------------------------------- */
/* PointcloudEncoder::PointcloudEncoder(info) (cloudini.cpp:430-440). `device` = CUDA ordinal, -1 = current.
 * `stream` = cudaStream_t to bind (NULL = a private non-blocking stream owned by the handle).
 * Device-pointer calls (CLDN_MEM_DEVICE) are ordered on that stream only: buffers another stream is still writing —
 * the legacy default stream included, a non-blocking stream does not wait for it — must be complete (or the
 * producer's stream passed here) before the call. */
int cldn_b200_encoder_create(const cldn_info_t* info, int device, void* stream, cldn_encoder_t** out);
void cldn_b200_encoder_destroy(cldn_encoder_t* enc);
/* getHeader() (cloudini.hpp:176-178) */
int cldn_b200_encoder_header(const cldn_encoder_t* enc, const uint8_t** header, size_t* header_bytes);
/* getEncodingInfo() (cloudini.hpp:171-173): the EncodingInfo the encoder was created from. */
int cldn_b200_encoder_info(const cldn_encoder_t* enc, cldn_info_t* info);

/* PointcloudEncoder::encode(ConstBufferView, BufferView&, bool write_header) (cloudini.cpp:522-623).
 * Point count = cloud_bytes / point_step (width*height of the info is NOT consulted, as in the reference).
 * `out_capacity` must be >= MaxCompressedSize(info, n, false) + (write_header ? header : 0) (cloudini.cpp:531-534).
 * CLDN_MEM_HOST: synchronous; *written is valid on return.
 * CLDN_MEM_DEVICE: kernels are enqueued on the handle's stream; the call then waits for the 8-byte size read-back
 *   unless `written` is NULL, in which case it returns right after enqueueing (size stays in cldn_b200_encoder_sizes_device). */
int cldn_b200_encode(cldn_encoder_t* enc, const void* cloud, size_t cloud_bytes, void* out, size_t out_capacity,
                     int write_header, size_t* written, int mem);

/* Batch of independent frames with the same layout (one PointcloudEncoder::encode per frame in the reference,
 * e.g. cloudini_publisher_plugin.cpp:55-77 once per message). One fused launch covers all frames.
 * clouds[i]/outs[i] are per-frame pointers (host array of pointers, pointing to `mem` memory).
 * written_host may be NULL for CLDN_MEM_DEVICE (fully asynchronous; sizes stay on the device). */
int cldn_b200_encode_batch(cldn_encoder_t* enc, size_t n_frames, const void* const* clouds, const size_t* cloud_bytes,
                           void* const* outs, const size_t* out_capacities, int write_header, size_t* written_host,
                           int mem);
/* Batch of frames of this encoder's layout, each written as a complete blob whose header states the frame's own
 * width / height (no reference counterpart: the reference builds a PointcloudEncoder per message). Blob f is
 * byte-identical to cldn_b200_encoder_set_dims(enc, widths[f], heights[f]) + cldn_b200_encode(..., write_header = 1)
 * with this handle. widths and heights are both NULL (width = point count, height = 1) or both given, with
 * widths[f] * heights[f] equal to frame f's point count. Every frame is checked before anything launches, in the order
 * of cldn_b200_encode with that frame's header length; the first bad frame's status is returned with
 * "frame <f>: <message>" and no output byte is written. Memory kinds, compression options and their refusals are those of
 * cldn_b200_encode_batch; with CLDN_MEM_DEVICE and written_host == NULL the call is asynchronous, and
 * cldn_b200_encoder_sizes_device then holds the blob sizes, headers included. The handle's header and dims are unchanged.
 * Device pointers: the encode_batch launches plus one launch that puts the headers in front of the payloads. */
int cldn_b200_encode_blobs(cldn_encoder_t* enc, size_t n_frames, const void* const* clouds, const size_t* cloud_bytes,
                           const uint32_t* widths, const uint32_t* heights, void* const* outs, const size_t* out_capacities,
                           size_t* written_host, int mem);
/* Device array (uint64 per frame of the last batch) with the encoded sizes; valid after the stream is synchronised. */
const uint64_t* cldn_b200_encoder_sizes_device(const cldn_encoder_t* enc);
/* Re-uses an encoder for messages of the same layout but another width / height (no reference counterpart: the
 * reference constructs a PointcloudEncoder per message, ros_msg_utils.cpp:198, which here would mean streams, device
 * buffers and pinned memory per message). Only the header text changes. Synchronises the handle's stream. */
int cldn_b200_encoder_set_dims(cldn_encoder_t* enc, uint32_t width, uint32_t height);
/* Waits for everything enqueued on the handle's stream; reports device-side errors of the last call. */
int cldn_b200_encoder_sync(cldn_encoder_t* enc);

/* ---- decoder -------------------------------------------------------------------------------------------------- */
int cldn_b200_decoder_create(int device, void* stream, cldn_decoder_t** out);
void cldn_b200_decoder_destroy(cldn_decoder_t* dec);

/* PointcloudDecoder::decode(info, compressed_data WITHOUT header, output) (cloudini.cpp:635-668).
 * Output must hold width*height*point_step bytes; only declared field bytes are written (padding is untouched,
 * field_decoder.cpp:74-78). Errors of the reference's hardened decoder surface as CLDN_ERR_CORRUPT_DATA. */
int cldn_b200_decode(cldn_decoder_t* dec, const cldn_info_t* info, const void* payload, size_t payload_bytes,
                     void* out, size_t out_capacity, int mem);

/* Batch of header-less payloads sharing one `info`. Asynchronous for CLDN_MEM_DEVICE when `sync` == 0. */
int cldn_b200_decode_batch(cldn_decoder_t* dec, const cldn_info_t* info, size_t n_frames,
                           const void* const* payloads, const size_t* payload_bytes, void* const* outs,
                           const size_t* out_capacities, int mem, int sync);
/* Complete blobs (header + payload, as PointcloudEncoder::encode writes them), in any mix of layouts, point counts,
 * wire versions 3..5 and compression options (no reference counterpart: the reference decodes one message per call).
 * Frames that share a layout and compression option are decoded in ONE fused launch, whatever their point counts
 * (LZ4 / ZSTD frames: those that also share the points of a chunk, min(points, 32768)). Synchronous for both memory
 * kinds. With CLDN_MEM_DEVICE the headers are read with one gather launch of every blob's first 4 KB.
 * status[f] (host array, always filled): CLDN_OK or the status that cldn_b200_decode_header + cldn_b200_decode return
 * for that blob alone. decoded_bytes[f] (optional): width*height*point_step of the frame, 0 when it failed.
 * A good frame's output holds exactly what cldn_b200_decode writes (padding bytes untouched); a failed frame's output
 * bytes are unspecified, and no frame's bytes outside outs[f][0, out_capacities[f]) are written.
 * Each frame of a fused launch has its own device error word; a frame that failed is decoded once more alone for its
 * exact status and message, the good frames of its group are not decoded again.
 * Returns CLDN_OK when every frame decoded. Otherwise it returns the status of the lowest-index failed frame, and
 * cldn_b200_last_error() reads "frame <f>: <message>". */
int cldn_b200_decode_blobs(cldn_decoder_t* dec, size_t n_frames, const void* const* blobs, const size_t* blob_bytes,
                           void* const* outs, const size_t* out_capacities, int mem, int32_t* status,
                           size_t* decoded_bytes);
/* Message of frame f of this handle's last cldn_b200_decode_blobs ("" when it decoded). */
const char* cldn_b200_decoder_frame_error(const cldn_decoder_t* dec, size_t f);
/* EncodingInfo read from the header of frame f of this handle's last cldn_b200_decode_blobs (zeroed when the header
 * did not parse). */
int cldn_b200_decoder_frame_info(const cldn_decoder_t* dec, size_t f, cldn_info_t* info);
int cldn_b200_decoder_sync(cldn_decoder_t* dec);
/* Diagnostics of the LAST FloatN batch decode of this handle (no reference counterpart; synchronises the stream):
 * stats[0] = chunks claimed by the chunk-sequential reader, stats[1] = chunks it handed to the careful reader
 * (NaN markers, varints of 5+ bytes, damaged streams). Both 0 when the batch took another kernel. */
int cldn_b200_decoder_last_stats(cldn_decoder_t* dec, uint32_t stats[2]);
/* 1 if the LAST batch decode of this handle decoded its V5 sections ahead of the regular stream and merged them into the
 * rows the chunk-sequential reader writes (large batches of FloatN / lossy-float layouts with 1..4 adaptive integer
 * fields; CLDN_B200_DECODE_SIDE=0 turns it off), else 0. No reference counterpart; negative status on a null handle. */
int cldn_b200_decoder_last_sections_ahead(cldn_decoder_t* dec);

/* ---- one-shot convenience, same shape as the reference's own C ABI ------------------------------------------- */
/* cldn_EncodePointcloudData (wasm_functions.h:88-93 / wasm_functions.cpp:217-248): YAML config + raw points -> blob
 * with header. Host memory. Returns the encoded size, 0 on any failure (the reference convention). */
uint32_t cldn_b200_EncodePointcloudData(const char* header_as_yaml, const void* pc_data, uint32_t pc_data_size,
                                        void* output_data, uint32_t output_capacity);
/* cldn_DecodeCompressedData (wasm_functions.h:62-72 / wasm_functions.cpp:143-167): blob with header -> raw points.
 * Host memory. Returns the decoded size (width*height*point_step), 0 on failure. */
uint32_t cldn_b200_DecodeCompressedData(const void* encoded_data, uint32_t encoded_data_size, void* output_data,
                                        uint32_t output_capacity);

#ifdef __cplusplus
}
#endif
#endif /* CLOUDINI_B200_H_ */
