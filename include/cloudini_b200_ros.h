/*
 * cloudini_b200 — C ABI of the callers either side of the codec (SURVEY.md §8(f) rows N2 and N3):
 *   N3  applyVizLossyPreprocessing  (cloudini_lib/src/ros_msg_utils.cpp:249-341): NaN/inf drop + order-preserving voxel
 *       de-duplication as sm_90a kernels directly in front of the encode launch;
 *   N2  the DDS / ROS 2 envelope    (cloudini_lib/src/ros_msg_utils.cpp:54-238): CDR (de)serialisation of
 *       sensor_msgs/msg/PointCloud2 and point_cloud_interfaces/msg/CompressedPointCloud2 around the codec.
 * Same conventions as cloudini_b200.h (status codes, cldn_b200_last_error(), caller-owned buffers, no CPU fallback for
 * anything that touches point data: the envelope functions parse / write the small CDR header on the host and hand the
 * point payload to the GPU codec).
 */
#ifndef CLOUDINI_B200_ROS_H_
#define CLOUDINI_B200_ROS_H_

#include "cloudini_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* ---- N3: visualisation-oriented lossy preprocessing ------------------------------------------------------------- */
typedef struct cldn_preproc cldn_preproc_t; /* owns the voxel hash table, tile status words and staging buffers */

int cldn_b200_preproc_create(int device, void* stream, cldn_preproc_t** out);
void cldn_b200_preproc_destroy(cldn_preproc_t* pp);

/* applyVizLossyPreprocessing(RosPointCloud2&) (ros_msg_utils.cpp:249-341, contract ros_msg_utils.hpp:198-221).
 *  - the geometry triple is detected structurally: fields[0..2] FLOAT32 with the same resolution at offsets b, b+4, b+8
 *    (names are never read); without it, with a non-positive / non-finite resolution or with an empty cloud the call is
 *    a no-op exactly like the reference: *applied = 0, `info` and `out` untouched, *kept_points = input point count;
 *  - points whose x, y or z is NaN / +-inf are dropped; of the points that quantise (lround(v * (1/res)), 21 bits per
 *    axis, packVoxelKey21 ros_msg_utils.cpp:42-49) to the same voxel only the FIRST survives; survivors keep their order
 *    and all `point_step` bytes;
 *  - on success `info` is updated like pc_info: width = kept, height = 1, every FLOAT64 field without a resolution gets
 *    1e-6 (so the planner routes it through the lossy coder).
 * `cloud` / `out` live in `mem` memory; `out_capacity` >= cloud_bytes is always enough. CLDN_MEM_DEVICE: the kernels run
 * on the handle's stream and the call waits for the 4-byte survivor count. */
int cldn_b200_viz_lossy_preprocess(cldn_preproc_t* pp, cldn_info_t* info, const void* cloud, size_t cloud_bytes,
                                   void* out, size_t out_capacity, size_t* kept_points, int* applied, int mem);

/* The same preprocessing for n_frames clouds of one layout `info` (no reference counterpart: the reference handles one
 * message per call). Frame f's output bytes, kept_points[f], applied[f] and infos_out[f] (optional, n_frames entries) are
 * what cldn_b200_viz_lossy_preprocess gives that cloud alone, `info` in and out being infos_out[f]: a layout without the
 * triple or with a bad resolution makes every frame a no-op, an empty cloud only its own frame (applied[f] = 0, output
 * untouched, infos_out[f] = *info). Every frame is checked before anything launches; the first bad frame's status is
 * returned with "frame <f>: <message>". One insert and one compact launch cover all frames, followed by one read-back
 * of the survivor counts and one synchronisation, for both memory kinds. Workspace: about 28 bytes per point of the
 * batch, kept by the handle. */
int cldn_b200_viz_lossy_preprocess_batch(cldn_preproc_t* pp, const cldn_info_t* info, size_t n_frames,
                                         const void* const* clouds, const size_t* cloud_bytes, void* const* outs,
                                         const size_t* out_capacities, size_t* kept_points, int* applied,
                                         cldn_info_t* infos_out, int mem);

/* Device-resident clouds of ONE layout and any point counts, preprocessed without the host, so that the converter step
 * (preprocessing, then cldn_b200_encode_blobs_async) runs on device pointers and can be captured in one CUDA graph.
 *
 * cldn_b200_preproc_prepare_batch: once per layout and shape, outside any capture. Width and height of `info` are
 * ignored. It decides from the layout alone whether the reference's early returns apply (no xyz triple, or a resolution
 * that is not positive and finite: a no-op layout). It allocates every device buffer a call of up to `max_frames`
 * clouds of up to `max_points_per_frame` points needs, apart from the buffers of the handle's single and batch calls:
 * a table region of 2 * max_points slots (rounded up to 1024) of 12 bytes, 4 bytes of slot per point and the tile
 * status words, per frame: about 28 bytes per point of max_frames * max_points_per_frame (none for a no-op layout).
 * `info_after` (optional) receives the layout an applied frame's infos_out[f] has, with width = height = 0 (every
 * FLOAT64 field without a resolution gets 1e-6), or *info for a no-op layout: cldn_b200_encoder_create(info_after, ...)
 * gives the encoder the chain needs. Refuses max_frames == 0 or >= 2^31 (CLDN_ERR_INVALID_ARGUMENT),
 * max_points_per_frame > 2^30, the single call's limit, and shapes of 2^31 insert blocks or compaction tiles or more
 * (CLDN_ERR_UNSUPPORTED). Waits for the handle's stream. A new prepare replaces the previous state; graphs captured
 * before it are then invalid. cldn_b200_viz_lossy_preprocess and _batch keep working and do not disturb it.
 *
 * cldn_b200_viz_lossy_preprocess_batch_async: enqueues on the handle's stream and returns. No host synchronisation,
 * allocation, pageable copy or host->device copy; the launches and their grids depend only on the prepared layout and
 * shape, not on n_frames or on the point counts. Returns CLDN_ERR_INVALID_ARGUMENT, before anything is enqueued, without
 * a prepared layout, with n_frames > max_frames, or with d_frames or d_status NULL; n_frames == 0 is CLDN_OK with no
 * work. `d_frames`: DEVICE array of n_frames cldn_viz_desc_t. For every frame f < n_frames, d_status[f] (int32),
 * d_kept[f] (uint64, optional) and d_applied[f] (int32, optional) are what cldn_b200_viz_lossy_preprocess(...,
 * CLDN_MEM_DEVICE) returns and writes for that cloud alone, with its checks in its order:
 *   CLDN_ERR_INVALID_ARGUMENT  a NULL cloud with cloud_bytes > 0; xyz fields outside the point (non-empty clouds);
 *   CLDN_ERR_UNSUPPORTED       more than 2^30 points;
 *   CLDN_ERR_BUFFER_TOO_SMALL  a NULL `out`, or capacity < points * point_step;
 * and, checked last, the one refusal of this call alone:
 *   CLDN_ERR_UNSUPPORTED       a non-empty cloud of an applying layout with more points than max_points_per_frame.
 * A failed frame gets kept = cloud_bytes / point_step and applied = 0, as the single call leaves them. Survivors go to
 * out[0, kept * point_step); no other byte of `out` is written, and a no-op or failed frame's output is untouched.
 * Nothing of the frames >= n_frames is read or written.
 * `d_encode` (optional): DEVICE array of n_frames cldn_cloud_desc_t whose out / capacity the caller set, for the blobs.
 * The call writes only cloud, cloud_bytes, width and height of each:
 *   applied:         cloud = out,   cloud_bytes = kept * point_step, width = height = 0;
 *   OK, not applied: cloud = cloud, cloud_bytes = cloud_bytes,       width = height = 0;
 *   failed:          cloud = NULL,  cloud_bytes = 1,                 width = height = 0, which
 *                    cldn_b200_encode_blobs_async refuses with CLDN_ERR_INVALID_ARGUMENT before writing anything.
 * cldn_b200_encode_blobs_async(enc, n_frames, d_encode, ...) enqueued behind it on the same stream, with `enc` created
 * from info_after, then gives every good frame the blob cldn_b200_viz_lossy_preprocess_batch + cldn_b200_encode_blobs
 * (widths = heights = NULL) give it.
 *
 * cldn_b200_preproc_sync: waits for the handle's stream and reports its CUDA error. */
typedef struct cldn_viz_desc_t { /* all device pointers */
  const void* cloud;
  uint64_t cloud_bytes;
  void* out;                      /* survivors; must not overlap `cloud` */
  uint64_t capacity;
} cldn_viz_desc_t;
int cldn_b200_preproc_prepare_batch(cldn_preproc_t* pp, const cldn_info_t* info, size_t max_frames,
                                    uint64_t max_points_per_frame, cldn_info_t* info_after);
int cldn_b200_viz_lossy_preprocess_batch_async(cldn_preproc_t* pp, size_t n_frames, const void* d_frames,
                                               int32_t* d_status, uint64_t* d_kept, int32_t* d_applied,
                                               cldn_cloud_desc_t* d_encode);
int cldn_b200_preproc_sync(cldn_preproc_t* pp);

/* ---- N2: DDS envelope ------------------------------------------------------------------------------------------- */
/* Parsed view of a CDR-serialised sensor_msgs/msg/PointCloud2 or point_cloud_interfaces/msg/CompressedPointCloud2
 * (cloudini_ros::RosPointCloud2, ros_msg_utils.hpp:32-148). `frame_id` and `data` are views (into the message that was
 * parsed, or into whatever buffers the caller sets them to before re-serialising). */
typedef struct cldn_ros_msg_t {
  uint8_t cdr_header[4];     /* nanocdr::CdrHeader as found on the wire: {0, encapsulation, 0, 0} */
  int32_t stamp_sec;
  uint32_t stamp_nsec;
  const char* frame_id;      /* header.frame_id, NOT NUL-terminated */
  uint32_t frame_id_len;     /* without the trailing NUL */
  uint32_t height, width;
  uint32_t n_fields;
  cldn_field_t fields[CLDN_MAX_FIELDS]; /* has_resolution = 0 after parsing (the message carries none) */
  uint8_t is_bigendian, is_dense;
  uint32_t point_step, row_step;
  const uint8_t* data;       /* PointCloud2::data / CompressedPointCloud2::compressed_data */
  size_t data_bytes;
} cldn_ros_msg_t;

/* getDeserializedPointCloudMessage (ros_msg_utils.cpp:54-95). Host memory. Little-endian PLAIN_CDR like the reference's
 * callers produce; CLDN_ERR_CORRUPT_DATA where nanocdr throws ("not enough data", bad header). */
int cldn_b200_ros_parse(const void* dds_msg, size_t msg_bytes, cldn_ros_msg_t* out);

/* toEncodingInfo (ros_msg_utils.cpp:122-131): LOSSY + ZSTD defaults, fields copied. */
int cldn_b200_ros_to_encoding_info(const cldn_ros_msg_t* msg, cldn_info_t* info);

/* applyResolutionProfile (ros_msg_utils.cpp:217-238) on a field list (msg->fields / &msg->n_fields — the reference's
 * converter applies it to the message's own fields, tools/src/mcap_converter.cpp:189, so removed fields also leave the
 * re-written message header): a profile entry of 0 removes the field, other entries set the field's resolution,
 * FLOAT32 fields without an entry get *default_resolution when it is non-NULL. */
int cldn_b200_ros_apply_resolution_profile(cldn_field_t* fields, uint32_t* n_fields, const char* const* names,
                                           const float* resolutions, size_t n_profile, const float* default_resolution);

/* convertPointCloud2ToCompressedCloud (ros_msg_utils.cpp:167-213): PointCloud2 message -> CompressedPointCloud2
 * message (same CDR header, width/height/fields/point_step, compressed_data = Cloudini blob with header, is_dense,
 * format "cloudini"). The point payload is encoded on the GPU through `enc` (created from `encoding_info`; its
 * compression_opt may be LZ4/ZSTD: host-pointer API). The payload is msg->data / msg->data_bytes — after
 * cldn_b200_viz_lossy_preprocess point them (and msg->width / height) at the preprocessed cloud, like pc_info.data.
 * Query the worst-case size with out == NULL (*written receives it). */
int cldn_b200_ros_compress_msg(cldn_encoder_t* enc, const cldn_ros_msg_t* msg, void* out, size_t out_capacity,
                               size_t* written);

/* convertCompressedCloudToPointCloud2 (ros_msg_utils.cpp:134-165): CompressedPointCloud2 message -> PointCloud2 message,
 * the blob decoded on the GPU through `dec` straight into the output message. out == NULL queries the exact size. */
int cldn_b200_ros_decompress_msg(cldn_decoder_t* dec, const cldn_ros_msg_t* msg, void* out, size_t out_capacity,
                                 size_t* written);

/* The converter's per-message step (tools/src/mcap_converter.cpp:184-204: getDeserializedPointCloudMessage ->
 * applyResolutionProfile -> [applyVizLossyPreprocessing] -> toEncodingInfo + options -> convertPointCloud2ToCompressedCloud)
 * as ONE call, host message in, host message out. Same bytes as the five calls; what differs is where the payload lives:
 * it is uploaded once, stays in HBM between the preprocessing and the encode kernels (only the 4-byte survivor count and
 * the 8-byte blob size come back), and encoder / preprocessor / staging buffers come from a per-thread pool keyed by the
 * layout instead of being created per message. compression_opt != NONE: stage 1 as above, then the host libraries.
 * out == NULL queries a worst-case size. */
int cldn_b200_ros_convert_msg(const void* dds_msg, size_t msg_bytes, const char* const* names, const float* resolutions,
                              size_t n_profile, const float* default_resolution, int viz, int encoding_opt,
                              int compression_opt, int version, void* out, size_t out_capacity, size_t* written);

/* Handles of the calling thread's pool (created on first use, owned by the library, never to be destroyed by the caller;
 * valid for this thread only). The reference constructs encoder / decoder objects per message, which costs it nothing;
 * a GPU handle owns streams, device buffers and pinned memory, so the per-message callers (the shims of
 * convertPointCloud2ToCompressedCloud & co.) take theirs from here. The encoder is re-dimensioned to info->width / height.
 * It keeps the system libraries' stage-2 bytes: cldn_b200_encoder_set_stage2_on_device(enc, 1) refuses it
 * (CLDN_ERR_INVALID_ARGUMENT). cldn_b200_ros_compress_msg uses the handle it is given, with that handle's policy. */
int cldn_b200_pool_encoder(const cldn_info_t* info, cldn_encoder_t** out);
int cldn_b200_pool_decoder(cldn_decoder_t** out);
int cldn_b200_pool_preproc(cldn_preproc_t** out);

/* ---- the rest of the reference's own C ABI (include/cloudini_lib/wasm_functions.h:30-93, src/wasm_functions.cpp), the
 * functions that take DDS messages. Same shape and "return 0 on any failure" convention; every output pointer is
 * followed by its capacity (the WASM module trusts the caller's allocation instead). Host memory. ------------------- */
/* cldn_GetHeaderAsYAML (wasm_functions.cpp:24-44): YAML text of the blob's header (not NUL-terminated); returns its size. */
uint32_t cldn_b200_GetHeaderAsYAML(const void* encoded_data, uint32_t encoded_data_size, char* output_yaml, uint32_t capacity);
/* cldn_GetHeaderAsYAMLFromDDS (:46-56): same, the blob is the compressed_data of a CompressedPointCloud2 message. */
uint32_t cldn_b200_GetHeaderAsYAMLFromDDS(const void* raw_dds_msg, uint32_t dds_msg_size, char* output_yaml, uint32_t capacity);
/* cldn_ComputeCompressedSize (:58-93): full GPU encode of a PointCloud2 message (every FLOAT32 field at `resolution`,
 * toEncodingInfo defaults: LOSSY + ZSTD), only the size is returned. */
uint32_t cldn_b200_ComputeCompressedSize(const void* dds_msg, uint32_t dds_msg_size, float resolution);
/* cldn_GetDecompressedSize (:95-106): height * width * point_step of the message; nothing is decoded. */
uint32_t cldn_b200_GetDecompressedSize(const void* encoded_dds_msg, uint32_t encoded_dds_size);
/* cldn_ConvertCompressedMsgToPointCloud2Msg (:108-125): CompressedPointCloud2 message -> PointCloud2 message. */
uint32_t cldn_b200_ConvertCompressedMsgToPointCloud2Msg(const void* compressed_msg, uint32_t msg_size, void* output_msg,
                                                        uint32_t capacity);
/* cldn_DecodeCompressedMessage (:127-148): CompressedPointCloud2 message -> raw point data. */
uint32_t cldn_b200_DecodeCompressedMessage(const void* compressed_msg, uint32_t msg_size, void* output_data, uint32_t capacity);
/* cldn_EncodePointcloudMessage (:178-226): PointCloud2 message -> Cloudini blob with header (every FLOAT32 field at
 * `resolution`); 0 when data size != width * height * point_step or the blob does not fit `capacity`. */
uint32_t cldn_b200_EncodePointcloudMessage(const void* pointcloud_msg, uint32_t msg_size, float resolution, void* output_data,
                                           uint32_t capacity);

#ifdef __cplusplus
}
#endif
#endif /* CLOUDINI_B200_ROS_H_ */
