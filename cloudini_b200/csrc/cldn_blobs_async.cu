// cldn_b200_decode_blobs_async: complete device-resident blobs of ONE prepared layout, decoded without the host.
//
// Every blob of such a call starts with the layout's canonical header (cldn_b200_encode_header), which differs from blob
// to blob only in its width and height numbers. So a warp per frame compares the blob's first bytes with the template
// cut around those two numbers, parses them, and writes the frame's tables; the decode kernels then read every count
// from those tables. Every frame owns the same number of chunk slots (those of the prepared maximum of points): slots past
// a frame's own chunks are empty and the kernels leave them (chunk_slot_empty), so nothing the host launches depends on
// the frames: the tables and grids are those of the prepared max_frames, whatever the call's frame count. Statuses are
// folded on the device as well.
//
// cldn_b200_encode_blobs_async is the same arrangement for the encoder: a warp per frame checks the frame as
// cldn_b200_encode_blobs does, writes its header (the template with the frame's width and height) and its tables into
// tile and chunk slots of the prepared maximum; the stage-1 and stage-2 kernels leave the empty slots.
#include "cldn_device.cuh"
#include "cldn_kernels.h"

namespace cldn {

constexpr int kAsyncWarps = 4;  // frames per CTA of the header kernel

// Blob bytes [at, at + len) equal tmpl[0, len). Called by the whole warp with the same arguments.
__device__ __forceinline__ bool warp_bytes_equal(const uint8_t* blob, uint64_t blob_bytes, uint64_t at, const uint8_t* tmpl,
                                                 uint32_t len, uint32_t lane) {
  if (at > blob_bytes || blob_bytes - at < len) return false;
  bool ok = true;
  for (uint32_t i = lane; i < len; i += 32) ok = ok && blob[at + i] == tmpl[i];
  return !__any_sync(0xffffffffu, !ok);
}

// A number as EncodingInfoToYAML writes it ("%u"): 1..10 digits, no leading zero unless it is "0", at most 2^32 - 1.
// Returns the digits it used, 0 for anything else.
__device__ __forceinline__ uint32_t parse_canonical_u32(const uint8_t* p, uint64_t avail, uint32_t* value) {
  uint64_t v = 0;
  uint32_t k = 0;
  while (k < avail && k < 11 && p[k] >= '0' && p[k] <= '9') {
    v = v * 10 + (p[k] - '0');
    ++k;
  }
  if (k == 0 || k > 10 || v > 0xFFFFFFFFull || (k > 1 && p[0] == '0')) return 0;
  *value = static_cast<uint32_t>(v);
  return k;
}

// One warp per frame.
__global__ void __launch_bounds__(kAsyncWarps * 32) blobs_async_headers_kernel(const AsyncLaunch A) {
  const uint32_t lane = threadIdx.x & 31u;
  const uint32_t f = blockIdx.x * kAsyncWarps + (threadIdx.x >> 5);
  if (f >= A.n_tables) return;
  const bool real = f < A.n_frames;  // the tables past the call's frames are written empty
  BlobDesc D = {nullptr, 0, nullptr, 0};
  if (real) D = A.desc[f];
  uint32_t w = 0, h = 0, k = 0;
  uint64_t at = A.tmpl_len[0];
  bool ok = D.blob != nullptr && warp_bytes_equal(D.blob, D.blob_bytes, 0, A.tmpl, A.tmpl_len[0], lane);
  if (ok) {
    k = parse_canonical_u32(D.blob + at, D.blob_bytes - at, &w);
    ok = k > 0;
    at += k;
  }
  ok = ok && warp_bytes_equal(D.blob, D.blob_bytes, at, A.tmpl + A.tmpl_len[0], A.tmpl_len[1], lane);
  if (ok) {
    at += A.tmpl_len[1];
    k = parse_canonical_u32(D.blob + at, D.blob_bytes - at, &h);
    ok = k > 0;
    at += k;
  }
  ok = ok && warp_bytes_equal(D.blob, D.blob_bytes, at, A.tmpl + A.tmpl_len[0] + A.tmpl_len[1], A.tmpl_len[2], lane);
  at += A.tmpl_len[2];
  if (lane != 0) return;
  const uint64_t points = static_cast<uint64_t>(w) * h;
  int32_t st = CLDN_OK;
  if (!ok) st = CLDN_ERR_BAD_HEADER;
  else if (points > A.max_points) st = CLDN_ERR_UNSUPPORTED;
  else if (points * A.point_step > D.capacity) st = CLDN_ERR_BUFFER_TOO_SMALL;
  else if (A.compression == CLDN_COMP_ZSTD && points == 0 && D.blob_bytes != at) st = CLDN_ERR_CORRUPT_DATA;  // no chunk to hold them
  const bool good = st == CLDN_OK;
  DecFrame F;
  F.out = D.out;
  F.n_points = good ? static_cast<uint32_t>(points) : 0u;
  F.n_chunks = good ? static_cast<uint32_t>((points + kChunkPoints - 1) / kChunkPoints) : 0u;
  F.chunk_begin = f * A.slots;
  F.pad_ = 0;
  const uint8_t* payload = good ? D.blob + at : nullptr;
  const uint64_t payload_bytes = good ? D.blob_bytes - at : 0;
  if (A.compression == CLDN_COMP_NONE) {
    F.payload = payload;
    F.payload_bytes = payload_bytes;
  } else {
    F.payload = A.s1 + f * A.s1_stride;
    F.payload_bytes = 0;  // blobs_async_link_kernel
    Lz4Frame Z;
    Z.plain = nullptr;
    Z.plain_bytes = nullptr;
    Z.blob_out = nullptr;
    Z.blob_cap = 0;
    Z.packed_in = payload;
    Z.packed_in_bytes = payload_bytes;
    Z.plain_out = A.s1 + f * A.s1_stride;
    Z.plain_cap = A.s1_stride;
    Z.n_chunks = F.n_chunks;
    Z.chunk_begin = F.chunk_begin;
    A.lz_frames[f] = Z;
  }
  A.frames[f] = F;
  if (real) A.status[f] = st;
}

// One thread per frame, after stage 2.
__global__ void blobs_async_link_kernel(const AsyncLaunch A) {
  const uint32_t f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= A.n_frames || A.status[f] != CLDN_OK) return;
  DecFrame& F = A.frames[f];
  bool failed = A.frame_err[f] != 0u;
  const uint32_t p = F.n_points;
  if (!failed && p > 0 && p < kChunkPoints) {
    // cldn_b200_decode_blobs bounds the decompressed chunk of a frame of fewer points than a chunk by that frame's own
    // stage-1 worst case (the slot here is the prepared maximum's): a chunk past it fails as it does there
    const uint64_t body_cap = A.chunk_a + A.chunk_b * p + 64;
    const bool zstd = A.compression == CLDN_COMP_ZSTD;
    if (A.chunk_sizes[F.chunk_begin] > (zstd ? body_cap : (body_cap + 15) & ~15ull)) {
      report_frame_error(A, f, zstd ? DEV_ERR_ZSTD : DEV_ERR_LZ4);
      failed = true;
    }
  }
  if (failed) {  // stage 1 leaves the frame out
    F.n_points = 0;
    F.n_chunks = 0;
    F.payload_bytes = 0;
  } else {
    F.payload_bytes = A.s1_sizes[f];
  }
}

// One CTA.
__global__ void __launch_bounds__(256) blobs_async_status_kernel(const AsyncLaunch A) {
  __shared__ uint32_t s_err;
  if (threadIdx.x == 0) s_err = *A.err;
  __syncthreads();
  for (uint32_t f = threadIdx.x; f < A.n_frames; f += blockDim.x) {
    int32_t st = A.status[f];
    if (st == CLDN_OK && (A.frame_err[f] != 0u || s_err != 0u)) st = CLDN_ERR_CORRUPT_DATA;
    A.status[f] = st;
    if (A.decoded) A.decoded[f] = st == CLDN_OK ? static_cast<uint64_t>(A.frames[f].n_points) * A.point_step : 0ull;
  }
  __syncthreads();
  if (threadIdx.x == 0) *A.err = 0u;
}

int launch_blobs_async_headers(const AsyncLaunch& A, cudaStream_t stream) {
  blobs_async_headers_kernel<<<(A.n_tables + kAsyncWarps - 1) / kAsyncWarps, kAsyncWarps * 32, 0, stream>>>(A);
  count_launch(1);
  return 1;
}

int launch_blobs_async_link(const AsyncLaunch& A, cudaStream_t stream) {
  blobs_async_link_kernel<<<(A.n_frames + 127) / 128, 128, 0, stream>>>(A);
  count_launch(1);
  return 1;
}

int launch_blobs_async_status(const AsyncLaunch& A, cudaStream_t stream) {
  blobs_async_status_kernel<<<1, 256, 0, stream>>>(A);
  count_launch(1);
  return 1;
}

// ---- cldn_b200_encode_blobs_async -----------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t decimal_digits(uint32_t v) {
  uint32_t k = 1;
  while (v >= 10u) { v /= 10u; ++k; }
  return k;
}
// v as "%u" into p (decimal_digits(v) bytes).
__device__ __forceinline__ void put_decimal(uint8_t* p, uint32_t v, uint32_t digits) {
  for (uint32_t k = digits; k-- > 0;) { p[k] = static_cast<uint8_t>('0' + v % 10u); v /= 10u; }
}
__device__ __forceinline__ uint64_t lz4_bound_dev(uint64_t n) { return n + n / 255u + 16u; }
__device__ __forceinline__ uint64_t zstd_bound_dev(uint64_t n) {
  return n + (n >> 8) + (n < (128u << 10) ? (((128u << 10) - n) >> 11) : 0u);
}
// MaxCompressedSize(info, n, false) of cldn_host.cpp: full chunks of `full` bytes, then the last, partial chunk.
__device__ __forceinline__ uint64_t max_compressed_dev(const EncAsyncLaunch& A, uint64_t n, uint32_t compression, uint64_t full) {
  const uint64_t r = n % kChunkPoints;
  uint64_t total = (n / kChunkPoints) * full;
  if (r) {
    const uint64_t in = r * A.per_point + A.chunk_extra;
    total += 4u + (compression == CLDN_COMP_LZ4 ? lz4_bound_dev(in) : compression == CLDN_COMP_ZSTD ? zstd_bound_dev(in) : in);
  }
  return total;
}

// One warp per frame: the checks of check_encode_frame in its order, then the dims, then the prepared maximum.
__global__ void __launch_bounds__(kAsyncWarps * 32) encode_async_frames_kernel(const EncAsyncLaunch A) {
  const uint32_t lane = threadIdx.x & 31u;
  const uint32_t f = blockIdx.x * kAsyncWarps + (threadIdx.x >> 5);
  if (f >= A.n_tables) return;
  const bool real = f < A.n_frames;  // the tables past the call's frames are written empty
  CloudDesc D = {nullptr, 0, nullptr, 0, 0, 0};
  if (real) D = A.desc[f];
  const uint64_t n = D.cloud_bytes / A.point_step;
  const bool own_dims = D.width != 0u || D.height != 0u;
  const uint32_t w = own_dims ? D.width : static_cast<uint32_t>(n), h = own_dims ? D.height : 1u;
  const uint32_t dw = decimal_digits(w), dh = decimal_digits(h);
  const uint32_t hdr = A.tmpl_len[0] + A.tmpl_len[1] + A.tmpl_len[2] + dw + dh;
  int32_t st = CLDN_OK;
  if (!real) st = CLDN_ERR_INVALID_ARGUMENT;
  else if (D.cloud_bytes % A.point_step) st = CLDN_ERR_INVALID_ARGUMENT;
  else if (D.capacity < max_compressed_dev(A, n, A.compression, A.full_chunk) + hdr) st = CLDN_ERR_BUFFER_TOO_SMALL;
  else if (n > 0xFFFFFFFFull) st = CLDN_ERR_UNSUPPORTED;
  else if ((n > 0 && !D.cloud) || !D.out) st = CLDN_ERR_INVALID_ARGUMENT;
  else if (static_cast<uint64_t>(w) * h != n) st = CLDN_ERR_INVALID_ARGUMENT;
  else if (n > A.max_points) st = CLDN_ERR_UNSUPPORTED;
  const bool good = st == CLDN_OK;
  if (good) {  // the header: template part 0, width, part 1, height, part 2
    uint8_t* o = D.out;
    for (uint32_t i = lane; i < A.tmpl_len[0]; i += 32) o[i] = A.tmpl[i];
    o += A.tmpl_len[0];
    if (lane == 0) put_decimal(o, w, dw);
    o += dw;
    for (uint32_t i = lane; i < A.tmpl_len[1]; i += 32) o[i] = A.tmpl[A.tmpl_len[0] + i];
    o += A.tmpl_len[1];
    if (lane == 0) put_decimal(o, h, dh);
    o += dh;
    for (uint32_t i = lane; i < A.tmpl_len[2]; i += 32) o[i] = A.tmpl[A.tmpl_len[0] + A.tmpl_len[1] + i];
  }
  if (lane != 0) return;
  const uint32_t pts = good ? static_cast<uint32_t>(n) : 0u;
  const uint32_t n_chunks = (pts + kChunkPoints - 1) / kChunkPoints;
  uint8_t* payload = good ? D.out + hdr : nullptr;
  const uint64_t payload_cap = good ? D.capacity - hdr : 0;
  EncFrame F;
  F.in = good ? D.cloud : nullptr;
  F.n_points = pts;
  F.tile_begin = f * A.tiles_per_frame;
  F.n_tiles = (pts + A.tile_points - 1) / A.tile_points;
  F.n_chunks = n_chunks;
  F.sec_excl = A.sec_excl ? A.sec_excl + static_cast<uint64_t>(f) * (A.slots + 1) : nullptr;
  F.side = A.side ? A.side + f * A.side_stride : nullptr;
  if (A.lz_frames) {
    // stage 1 into the frame's arena, bounded as encode_blobs bounds it for this frame: the stage-1 worst case plus 64
    // bytes per chunk and 64 more (stage1_arena_bytes)
    uint8_t* arena = A.s1 + f * A.s1_stride;
    F.out = arena;
    const uint64_t arena_cap = max_compressed_dev(A, pts, CLDN_COMP_NONE, A.full_chunk_s1) + 64ull * (n_chunks + 1);
    F.out_cap = good ? (arena_cap < A.s1_stride ? arena_cap : A.s1_stride) : 0;
    Lz4Frame Z;
    Z.plain = arena;
    Z.plain_bytes = A.sizes + f;
    Z.blob_out = payload;
    Z.blob_cap = payload_cap;
    Z.packed_in = nullptr;
    Z.packed_in_bytes = 0;
    Z.plain_out = nullptr;
    Z.plain_cap = 0;
    Z.n_chunks = n_chunks;
    Z.chunk_begin = f * A.slots;
    A.lz_frames[f] = Z;
  } else {
    F.out = payload;
    F.out_cap = payload_cap;
  }
  A.frames[f] = F;
  A.hdr_len[f] = good ? hdr : 0u;
  if (real) A.status[f] = st;
}

// One CTA.
__global__ void __launch_bounds__(256) encode_async_status_kernel(const EncAsyncLaunch A) {
  __shared__ uint32_t s_err;
  if (threadIdx.x == 0) s_err = *A.err;
  __syncthreads();
  for (uint32_t f = threadIdx.x; f < A.n_frames; f += blockDim.x) {
    int32_t st = A.status[f];
    const uint32_t code = A.frame_err[f] != 0u ? A.frame_err[f] : s_err;
    // as check_device_error reads the error word after cldn_b200_encode_blobs
    if (st == CLDN_OK && code != 0u) st = code == DEV_ERR_ENCODE_OUTPUT_SMALL ? CLDN_ERR_BUFFER_TOO_SMALL : CLDN_ERR_CORRUPT_DATA;
    A.status[f] = st;
    if (A.written) A.written[f] = st == CLDN_OK ? A.hdr_len[f] + A.sizes[f] : 0ull;
  }
  __syncthreads();
  if (threadIdx.x == 0) *A.err = 0u;
}

int launch_encode_async_frames(const EncAsyncLaunch& A, cudaStream_t stream) {
  encode_async_frames_kernel<<<(A.n_tables + kAsyncWarps - 1) / kAsyncWarps, kAsyncWarps * 32, 0, stream>>>(A);
  count_launch(1);
  return 1;
}

int launch_encode_async_status(const EncAsyncLaunch& A, cudaStream_t stream) {
  encode_async_status_kernel<<<1, 256, 0, stream>>>(A);
  count_launch(1);
  return 1;
}

}  // namespace cldn
