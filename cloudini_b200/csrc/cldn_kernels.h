// Internal launch interface between the C-ABI layer (cldn_api.cu) and the kernels.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "cldn_plan.h"

namespace cldn {

// One frame (one PointcloudEncoder::encode call in the reference) of a fused batch launch.
struct EncFrame {
  const uint8_t* in;     // n_points * point_step bytes
  uint8_t* out;          // start of the blob (header goes here when write_header)
  uint64_t out_cap;      // bytes available at `out`: every store is checked against it (a committed V5 mode can exceed
                         // the reference's worst-case formula; the reference then throws, chunk_writer.cpp:33-35)
  uint32_t n_points;
  uint32_t tile_begin;   // global index of this frame's first tile (exclusive scan of n_tiles over the batch)
  uint32_t n_tiles;
  uint32_t n_chunks;
  // V5: exclusive scan over chunks of the total adaptive-section bytes ((n_chunks + 1) entries), else nullptr.
  const uint32_t* sec_excl;
  // Gorilla ops: records precomputed by the sequential pre-pass, 12 bytes per (op, point): bytes 0..9 record, byte 11 length
  const uint8_t* side;
};

struct EncLaunch {
  const EncFrame* frames;  // device
  uint32_t n_frames;
  uint32_t n_tiles_total;
  const Plan* plan;        // device copy
  const uint8_t* header;   // device copy of the blob header
  uint32_t header_bytes;   // 0 when write_header == false
  uint64_t* status;        // n_tiles_total tile status words
  uint32_t epoch;
  uint64_t* sizes;         // per frame: total bytes written (header included)
  uint32_t* err;
  uint32_t tile_points;    // 256 * I (choose_tile_points)
  uint32_t flags;          // kEncInputsAligned16 / kEncAlignPerFrame
  uint32_t uniform_tiles;  // > 0: every frame has exactly this many tiles (frame = tile / uniform_tiles, no search)
  uint32_t* tile_ticket;   // one word, zeroed per launch: the persistent XYZI kernel's CTAs take their tiles from it in order
  uint32_t* frame_err;     // nullptr, or one word per frame that takes that frame's errors (frame_err_word)
  uint32_t empty_slots;    // 1: every frame owns uniform_tiles tile slots, and the slots t >= n_tiles are empty
};
constexpr uint32_t kEncInputsAligned16 = 1u;  // every frame's input base is 16-byte aligned (checked on the host)
constexpr uint32_t kEncAlignPerFrame = 2u;    // the host has not seen the inputs: each frame's base is checked on the device
// Whether frame input `in` takes the 16-byte loads.
__device__ __forceinline__ bool enc_input_aligned16(uint32_t flags, const uint8_t* in) {
  return (flags & kEncInputsAligned16) || ((flags & kEncAlignPerFrame) && (reinterpret_cast<uintptr_t>(in) & 15u) == 0u);
}
uint32_t choose_tile_points(const Plan& plan);

// Interleaved regular stream + chunk framing. Returns the number of kernels launched.
int launch_encode_regular(const Plan& host_plan, const EncLaunch& L, cudaStream_t stream);
int launch_gorilla_prepass(const Plan& host_plan, const EncLaunch& L, cudaStream_t stream);

constexpr int kMaxSideFields = 4;   // V5 section fields the side mode carries (more: the sections are decoded behind the stream)
struct DecFrame {
  const uint8_t* payload;  // header-less payload
  uint64_t payload_bytes;
  uint8_t* out;
  uint32_t n_points;       // width * height
  uint32_t n_chunks;
  uint32_t chunk_begin;    // global index of this frame's first chunk
  uint32_t pad_;
};

struct DecLaunch {
  const DecFrame* frames;  // device
  uint32_t n_frames;
  uint32_t n_chunks_total;
  const Plan* plan;          // device copy
  uint64_t* chunk_offsets;   // per global chunk: byte offset of the chunk BODY inside its payload
  uint32_t* chunk_sizes;     // per global chunk: body size
  uint32_t* err;
  // tile-parallel path (FloatN-only regular streams)
  uint32_t* chunk_tiles;       // per global chunk: number of 8 KB byte tiles
  uint32_t* chunk_tile_begin;  // exclusive scan of chunk_tiles, (n_chunks_total + 1) entries
  uint32_t* stream_end;        // per global chunk: bytes of the regular stream (start of the V5 sections)
  uint32_t* chunk_frame;       // per global chunk: frame index
  uint32_t* tile_chunk;        // per tile: global chunk index
  uint64_t* tstatus;           // per tile: look-back 1 (value counts)
  uint32_t* tsums;             // per tile: 2 x 8 words, look-back 2 (aggregate record, inclusive record)
  uint32_t* chunk_counter;     // 4 words, zeroed per launch: [0] chunk claims, [1] redo claims, [2] walk ticket, [3] redo count
  uint32_t* redo_list;         // chunks the fast chunk-sequential kernel handed to the careful one (n_chunks_total entries)
  uint32_t redo_mode;          // careful kernel: 1 = decode exactly the chunks of redo_list (descriptors are already published)
  uint64_t* chunk_desc;        // chunk-sequential kernel: 2 self-validating words per chunk, [tag:24][offset:40] and
                               // [tag:24][size:32], published by CTA 0 while it walks the chunk prefixes
  uint32_t desc_tag;           // tag of this launch (never 0)
  uint32_t uniform_chunks;     // > 0: every frame has this many chunks (chunks are then claimed chunk-index-major)
  uint32_t sections_only;      // decode_chunks_kernel: the regular stream was decoded elsewhere, start at stream_end[]
  uint32_t tile_capacity;      // records allocated (== tile_grid)
  uint32_t tile_grid;          // host upper bound on the number of tiles
  uint32_t chunk_bytes_max;    // > 0: tile_grid was sized from a prepared shape whose chunk bodies hold at most this many
                               // bytes; count_tiles_kernel fails a larger chunk's frame instead of tiling it
  uint32_t epoch;
  // Side mode (V5 sections decoded AHEAD of the regular stream, large batches): stream_end_kernel finds where every chunk's
  // regular stream ends, the section reader writes its values into compact arrays -- section s of global chunk gc at
  // side + side_off[s] + gc * kChunkPoints * bpv -- and the fast reader merges them into the rows it writes, so that
  // every output sector is written once instead of once per pass.
  uint8_t* side;               // nullptr: off
  uint64_t side_off[kMaxSideFields];
  uint32_t side_mode;          // decode_chunks_kernel, sections_only: 1 = store into the side arrays; any anomaly marks the
                               // chunk (stream_end = 0xFFFFFFFF) for the careful kernels instead of raising the error word
  uint32_t* frame_err;         // nullptr, or one word per frame (zeroed per launch) that takes that frame's errors
  uint32_t empty_slots;        // 1: some chunk slots are empty (chunk_slot_empty); the chunk-sequential readers check
                               // a claimed slot before they wait for its descriptor
};

// Error word of frame f: its own word when the launch has per-frame words, else the launch word (so launches without
// them report exactly as before). A frame's errors go to its own word only: a raised launch word in a launch with
// per-frame words means an error that no frame claimed.
template <class Launch>
__device__ __forceinline__ uint32_t* frame_err_word(const Launch& L, uint32_t f) { return L.frame_err ? L.frame_err + f : L.err; }
template <class Launch>
__device__ __forceinline__ void report_frame_error(const Launch& L, uint32_t f, uint32_t code) { atomicCAS(frame_err_word(L, f), 0u, code); }

// Whether global chunk gc, which lies in frame F's range, is not one of F's chunks. cldn_b200_decode_blobs_async gives every
// frame the same number of chunk slots (those of the prepared maximum of points), so the slots past a frame's own chunks --
// all of them for a frame refused before the decode -- are empty, and a kernel leaves an empty slot at once. Every other
// launch packs the frames' chunks back to back and has no empty slot. (DecFrame and Lz4Frame)
template <class Frame>
__device__ __forceinline__ bool chunk_slot_empty(const Frame& F, uint32_t gc) { return gc - F.chunk_begin >= F.n_chunks; }

// Frame of global chunk gc: gc / uniform_chunks, else the last frame that begins at or before gc.
__device__ __forceinline__ uint32_t dec_frame_of(const DecLaunch& L, uint32_t gc) {
  if (L.uniform_chunks) return gc / L.uniform_chunks;
  uint32_t lo = 0, hi = L.n_frames - 1;
  while (lo < hi) {
    const uint32_t mid = (lo + hi + 1) >> 1;
    if (L.frames[mid].chunk_begin <= gc) lo = mid; else hi = mid - 1;
  }
  return lo;
}

int launch_decode(const Plan& host_plan, const DecLaunch& L, cudaStream_t stream);
int launch_decode_tiles(const Plan& host_plan, const DecLaunch& L, cudaStream_t stream);
int launch_decode_fast(const Plan& host_plan, const DecLaunch& L, int sm_count, cudaStream_t stream);
bool decode_fast_general_plan(const Plan& host_plan);  // a FloatN group and / or scalar lossy floats, 3..6 values per point
bool decode_fast_whole_rows(const Plan& host_plan);    // ... whose regular + section fields cover every byte of a point
bool decode_fast_enabled();  // CLDN_B200_DECODE_FAST=0 keeps the careful chunk-sequential kernel alone
bool decode_tiles_sequential(uint32_t n_chunks_total);  // which of the two FloatN kernels launch_decode_tiles will pick
uint32_t decode_tile_bytes();
// Side mode applies to this plan (1..kMaxSideFields section fields, CLDN_B200_DECODE_SIDE != 0) / to this launch
bool decode_side_plan(const Plan& host_plan);
bool decode_side_active(const Plan& host_plan, const DecLaunch& L);
size_t decode_side_bytes(const Plan& host_plan, uint64_t n_chunks_total, uint64_t side_off[kMaxSideFields]);
int launch_stream_end(const Plan& host_plan, const DecLaunch& L, cudaStream_t stream);

// V5 adaptive integer sections (encode side).
struct SecLaunch {
  const EncFrame* frames;
  uint32_t n_frames;
  uint32_t n_chunks_total;       // over the batch
  const uint32_t* chunk_frame;   // per global chunk: frame index
  const uint32_t* chunk_first;   // per frame: global index of its first chunk
  const Plan* plan;
  uint8_t* modes;                // [n_frames][n_sections] committed AdaptiveIntMode
  uint8_t* scratch;              // [n_chunks_total][n_sections][sec_stride] section bytes
  uint32_t sec_stride;
  uint32_t* sec_sizes;           // [n_chunks_total][n_sections]
  uint32_t* sec_excl;            // per frame region: (n_chunks + 1) entries, laid out at chunk_first[f] + f
  uint64_t* hash_scratch;        // palette hash tables
  uint32_t* err;
  uint32_t header_bytes;
  uint32_t* frame_err;           // nullptr, or one word per frame (frame_err_word)
  uint32_t empty_slots;          // 1: chunk slots past a frame's n_chunks are empty, and the kernels leave them at once
};
int launch_encode_sections(const Plan& host_plan, const SecLaunch& L, cudaStream_t stream);
size_t palette_overflow_scratch_bytes();
int launch_place_sections(const Plan& host_plan, const SecLaunch& L, const uint64_t* status, uint32_t epoch,
                          uint32_t tile_points, cudaStream_t stream);

// ---- stage 2 on the device (LZ4 blocks per chunk; cldn_lz4.cu) ----------------------------------------------------------
struct Lz4Frame {
  // compress: stage-1 payload of the frame ([u32 size][bytes])*, its byte count (device word written by the stage-1
  // kernels), and where the finished blob goes
  const uint8_t* plain;
  const uint64_t* plain_bytes;
  uint8_t* blob_out;
  uint64_t blob_cap;
  // decompress: the blob's payload ([u32 csize][LZ4 block])* and where the re-framed stage-1 payload goes
  const uint8_t* packed_in;
  uint64_t packed_in_bytes;
  uint8_t* plain_out;
  uint64_t plain_cap;
  uint32_t n_chunks;
  uint32_t chunk_begin;  // global index of the frame's first chunk
};
struct Lz4Launch {
  const Lz4Frame* frames;      // device
  uint32_t n_frames;
  uint32_t n_chunks_total;
  const uint32_t* chunk_frame; // per global chunk: frame index
  uint8_t* scratch;            // n_chunks_total slots of slot_stride bytes
  uint32_t slot_stride;
  uint32_t* chunk_sizes;       // per global chunk: bytes in its slot
  uint64_t* sizes;             // per frame: bytes written by the pack kernel (0: did not fit)
  uint32_t* err;
  uint32_t* frame_err;         // decompression: nullptr, or one word per frame (see frame_err_word)
  // ZSTD compression: a chunk's compressed bytes are the concatenation of several pieces (one per block). Chunk gc owns
  // pieces block_begin[gc] .. block_begin[gc + 1] - 1, and the slots of `scratch` and `chunk_sizes` are per piece.
  // nullptr: one piece per chunk (LZ4).
  const uint32_t* block_begin = nullptr;  // n_chunks_total + 1 entries
  uint32_t n_blocks_total = 0;
  // compression: 1 when chunk slots past a frame's n_chunks are empty (cldn_b200_encode_blobs_async); decompression
  // always checks them (chunk_slot_empty)
  uint32_t empty_slots = 0;
};
// Compression: one LZ4 block per chunk, then the blobs are packed (launch_stage2_pack)
int launch_lz4_compress(const Lz4Launch& L, const uint8_t* header, uint32_t header_bytes, cudaStream_t stream);
// Blob f = header + ([u32 size][the chunk's pieces])* into F.blob_out; a blob that does not fit F.blob_cap raises
// DEV_ERR_ENCODE_OUTPUT_SMALL and writes sizes[f] = 0, else sizes[f] = its bytes.
int launch_stage2_pack(const Lz4Launch& L, const uint8_t* header, uint32_t header_bytes, cudaStream_t stream);
int launch_lz4_decompress(const Lz4Launch& L, cudaStream_t stream);
// Re-frames the slots of L (chunk_sizes[] bytes each) into one stage-1 payload per frame at plain_out; a payload that
// does not fit plain_cap raises `fail_code`.
int launch_stage2_unpack(const Lz4Launch& L, uint32_t fail_code, cudaStream_t stream);

// ---- ZSTD frames per chunk on the device (cldn_zstd.cu) ------------------------------------------------------------------
// The chunk table, slots and frames are those of the LZ4 path (L.frames[f].packed_in: ([u32 csize][ZSTD frames])*).
// Every chunk decompresses exactly as ZSTD_decompress(slot, body_cap, body, csize) does, failing exactly when it fails;
// a failure raises DEV_ERR_ZSTD. A frame whose payload holds more chunks than n_chunks raises DEV_ERR_CHUNK_COUNT.
struct ZstdLaunch {
  Lz4Launch L;
  uint32_t body_cap;       // bytes a chunk may decompress to (<= L.slot_stride)
  uint32_t n_ctas;         // grid of the decompressor: warps walk the chunks with a grid stride
  uint8_t* lit_scratch;    // n_ctas * zstd_warps_per_cta() regions of zstd_lit_scratch_bytes(body_cap) bytes
};
uint32_t zstd_warps_per_cta();
// ---- ZSTD compression on the device (cldn_zstd_enc.cu) -----------------------------------------------------------------
// Every chunk of L becomes one ZSTD frame of Huffman-coded literal blocks of zstd_enc_block_bytes() stage-1 bytes (the
// pieces of L.block_begin, zstd_enc_slot_bytes() each), then the blobs are packed (launch_stage2_pack).
uint32_t zstd_enc_block_bytes();
uint32_t zstd_enc_slot_bytes();
int launch_zstd_compress(const Lz4Launch& L, const uint8_t* header, uint32_t header_bytes, cudaStream_t stream);
size_t zstd_lit_scratch_bytes(uint32_t body_cap);
int launch_zstd_decompress(const ZstdLaunch& Z, cudaStream_t stream);

// ---- headers of device-resident blobs (cldn_lz4.cu) --------------------------------------------------------------------
// One launch: tab = [n source addresses][n byte counts][n offsets into dst]; blob f's bytes go to dst + offset[f].
int launch_gather_prefixes(const uint64_t* tab, uint32_t n, uint8_t* dst, cudaStream_t stream);
// Headers of blobs encoded without one (cldn_b200_encode_blobs), one launch: tab = [n blob addresses][n + 1 offsets into
// the packed header bytes][packed header bytes]; header f is copied to blob f and its length added to sizes[f]. With
// `slots` (2n words, cldn_b200_encode_mixed_blobs): sizes[slots[n + f]] = from[slots[f]] + that length instead.
int launch_place_headers(const uint64_t* tab, uint32_t n, uint64_t* sizes, cudaStream_t stream, const uint64_t* from = nullptr,
                         const uint32_t* slots = nullptr);

// ---- complete device blobs of one prepared layout, without the host (cldn_b200_decode_blobs_async; cldn_blobs_async.cu) ---
struct BlobDesc {  // cldn_blob_desc_t
  const uint8_t* blob;
  uint64_t blob_bytes;
  uint8_t* out;
  uint64_t capacity;
};
struct AsyncLaunch {
  const BlobDesc* desc;       // device, n_frames
  uint32_t n_frames;
  uint32_t n_tables;          // frames of the prepared shape (>= n_frames): the tables of frames n_frames.. are written empty
  const uint8_t* tmpl;        // the layout's header with width and height cut out: part 0 | part 1 | part 2 ('\0' included)
  uint32_t tmpl_len[3];
  uint64_t max_points;
  uint32_t point_step;
  uint32_t slots;             // chunk slots per frame (frame f: f * slots ..)
  uint32_t compression;       // CLDN_COMP_*
  DecFrame* frames;           // stage 1
  Lz4Frame* lz_frames;        // stage 2 (LZ4 / ZSTD)
  uint8_t* s1;                // stage-1 payloads after stage 2: frame f at s1 + f * s1_stride
  uint64_t s1_stride;
  const uint64_t* s1_sizes;   // stage 2: bytes of every frame's stage-1 payload (Lz4Launch::sizes)
  const uint32_t* chunk_sizes;  // stage 2: bytes every chunk decompressed to (Lz4Launch::chunk_sizes)
  uint64_t chunk_a, chunk_b;  // stage-1 worst case of a chunk of p > 0 points: chunk_a + chunk_b * p bytes
  uint32_t* frame_err;        // one word per frame, zeroed before the launches
  uint32_t* err;              // the launches' word (errors no frame claimed)
  int32_t* status;            // device, n_frames
  uint64_t* decoded;          // device, n_frames, optional
};
// Header check and frame tables; status[f] = CLDN_OK or the header / size refusal.
int launch_blobs_async_headers(const AsyncLaunch& A, cudaStream_t stream);
// After stage 2: a frame's stage-1 payload size goes into its DecFrame, a frame stage 2 failed leaves stage 1 out.
int launch_blobs_async_link(const AsyncLaunch& A, cudaStream_t stream);
// status[f] / decoded[f] from the frame's error word.
int launch_blobs_async_status(const AsyncLaunch& A, cudaStream_t stream);

// ---- device clouds of the encoder's layout, without the host (cldn_b200_encode_blobs_async; cldn_blobs_async.cu) -------
struct CloudDesc {  // cldn_cloud_desc_t
  const uint8_t* cloud;
  uint64_t cloud_bytes;
  uint8_t* out;
  uint64_t capacity;
  uint32_t width, height;
};
struct EncAsyncLaunch {
  const CloudDesc* desc;      // device, n_frames
  uint32_t n_frames;
  uint32_t n_tables;          // frames of the prepared shape (>= n_frames): the tables of frames n_frames.. are written empty
  const uint8_t* tmpl;        // the layout's header with width and height cut out: part 0 | part 1 | part 2 ('\0' included)
  uint32_t tmpl_len[3];
  uint32_t point_step;
  uint64_t max_points;
  // MaxCompressedSize (without header) of n points: n / kChunkPoints full chunks of full_chunk bytes, and a last chunk of
  // r = n % kChunkPoints points of 4 + bound(r * per_point + chunk_extra) bytes; bound is the stage-2 worst case of
  // `compression`. full_chunk_s1 / the NONE bound: the same for the stage-1 arena of the compressed layouts.
  uint64_t per_point;
  uint32_t chunk_extra;
  uint32_t compression;       // CLDN_COMP_* of the blobs
  uint64_t full_chunk, full_chunk_s1;
  uint32_t tile_points;
  uint32_t tiles_per_frame;   // tile slots of a frame (frame f: f * tiles_per_frame ..)
  uint32_t slots;             // chunk slots of a frame (frame f: f * slots ..)
  EncFrame* frames;           // stage 1
  Lz4Frame* lz_frames;        // stage 2 (LZ4 / ZSTD), else nullptr
  uint8_t* s1;                // stage 2: stage-1 arena of frame f at s1 + f * s1_stride
  uint64_t s1_stride;
  uint32_t* sec_excl;         // V5: frame f's (slots + 1) entries at sec_excl + f * (slots + 1), else nullptr
  uint8_t* side;              // Gorilla records: frame f's at side + f * side_stride, else nullptr
  uint64_t side_stride;
  uint64_t* sizes;            // per frame: payload bytes (EncLaunch::sizes, Lz4Launch::sizes)
  uint32_t* hdr_len;          // per frame: header bytes of a good frame, 0 else
  uint32_t* frame_err;        // one word per frame, zeroed before the launches
  uint32_t* err;              // the launches' word (errors no frame claimed)
  int32_t* status;            // device, n_frames
  uint64_t* written;          // device, n_frames, optional
};
// Frame checks, headers and frame tables; status[f] = CLDN_OK or the refusal.
int launch_encode_async_frames(const EncAsyncLaunch& A, cudaStream_t stream);
// status[f] / written[f] from the frame's error word.
int launch_encode_async_status(const EncAsyncLaunch& A, cudaStream_t stream);

uint64_t kernel_launch_count();
void count_launch(int n = 1);  // process-wide, atomic: handles on other threads count into the same total

// Raises `kernel`'s dynamic shared memory limit on the current device to at least `bytes` and never lowers it. The limit
// is one value per (device, kernel) for the whole process, so a launch site that set exactly what its own launch needs
// could lower it between another thread's set and that thread's launch, and the other launch would then fail. The limit
// is a cap, not a reservation: occupancy and the launch itself take the launch's own size.
cudaError_t raise_smem_limit_ptr(const void* kernel, size_t bytes);
template <typename K>
inline cudaError_t raise_smem_limit(K* kernel, size_t bytes) { return raise_smem_limit_ptr((const void*)kernel, bytes); }

}  // namespace cldn
