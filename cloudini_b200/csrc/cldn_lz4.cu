// Stage 2 on the device, LZ4 only (SURVEY §8(f) N1 / BASELINE configs[3]): every chunk's stage-1 bytes are compressed
// into an LZ4 *block* (the format LZ4_compress_default / LZ4_decompress_safe speak, which is what the reference calls per
// chunk: cloudini_lib/src/codec_common.cpp:220-299, chunk_writer.cpp:42-47) without leaving HBM.
//
// north_star delegates stage 2 to nvCOMP; this image has no nvCOMP (probed on the GPU box: gpurun_out/r2_start/probe.txt),
// so the block coder is written here. It is not byte-identical to liblz4's output -- no two LZ4 compressors are -- but
// every block it writes is a valid LZ4 block: the stock reference decodes the blobs (tests/test_gpu_stage2_device.py),
// and the decompressor below accepts whatever liblz4 wrote.
//
//  compress    one warp per chunk. 128 consecutive positions per step (4 per lane, all of a step's loads in flight together):
//              every lane hashes the 4 bytes at its positions, reads the candidates the table holds and verifies them by
//              content over EIGHT bytes; the first verified position (ballots) becomes the match, which the warp extends 32
//              bytes per ballot; literals leave as aligned 16-byte stores. Greedy, 2048-entry table in shared memory: 16-bit
//              position (candidates are rebuilt modulo 64 KB) + 16-bit tag of the hashed value, so that only candidates that
//              very likely hold the same four bytes are fetched; always checked by content (stale or uninitialised entries
//              are harmless). Why 8 bytes: on varint streams 4-byte repeats are everywhere and each saves about
//              one byte, while a sequence costs the warp a chain of dependent global round trips -- the round-1 coder
//              (4-byte matches, 32 positions per step) spent far more time for a few per cent of size.
//  decompress  one warp per chunk: the (cheap, serial) sequence headers are parsed by all lanes in lock step, literal and
//              match bytes move cooperatively (overlapping matches with offset < 32 by the closed form k mod offset).
//  pack        one CTA per frame: exclusive scan of the chunk sizes, then [u32 size][bytes] back to back behind the header.
#include <stdio.h>

#include "cldn_device.cuh"
#include "cldn_kernels.h"
#include "cldn_stage2.cuh"

namespace cldn {

constexpr int kLzThreads = 128;          // 4 warps = 4 chunks per CTA
constexpr int kLzWarps = kLzThreads / 32;
constexpr uint32_t kLzHashBits = 11;    // 2048 entries of (16-bit tag << 16 | 16-bit position) per warp = 8 KB
constexpr int kLzR = 4;                  // positions per lane and step of the compressor
constexpr int kLzMinMatch = 6;           // 4 (the format's minimum) .. 8: shortest match the compressor takes.
// Sizes on config 4 (1000 x 130 048-point XYZI frames, 6.802 stage-1 bytes per point; liblz4: 6.61): minimum match
//   5: 6.747 B per point    6: 6.797    8: 6.825 (the block framing outweighs the matches). Shorter minimum matches were
// slower to encode and decode; 6 never expands and was close to 8 in time.

__device__ __forceinline__ uint32_t lz_mix(uint32_t v) { return v * 2654435761u; }
__device__ __forceinline__ uint32_t lz_slot(uint32_t m) { return m >> (32u - kLzHashBits); }           // top bits: the table slot
__device__ __forceinline__ uint32_t lz_tag(uint32_t m) { return (m << kLzHashBits) & 0xFFFF0000u; }   // the 16 bits below them, moved to the entry's top half

// Length field of a sequence: nibble value 15 is followed by bytes of 255 and a last byte < 255 (uniform over the warp).
__device__ __forceinline__ uint32_t lz_ext_bytes(uint32_t len) { return len >= 15u ? (len - 15u) / 255u + 1u : 0u; }
__device__ __forceinline__ void lz_write_ext(uint8_t* dst, uint32_t len, uint32_t lane) {  // len >= 15
  const uint32_t rest = len - 15u, full = rest / 255u;
  for (uint32_t k = lane; k < full; k += 32u) dst[k] = 255u;
  if (lane == 0) dst[full] = static_cast<uint8_t>(rest - full * 255u);
}

// One full warp. Returns the compressed size, 0 if `cap` is too small.
__device__ uint32_t lz4_compress_warp(const uint8_t* __restrict__ src, uint32_t n, uint8_t* __restrict__ dst, uint32_t cap,
                                      uint32_t* table) {
  const uint32_t lane = threadIdx.x & 31u;
  uint32_t ip = 0, anchor = 0, op = 0;
  // LZ4 block rules: the last match starts at least 12 bytes before the end, the last 5 bytes are literals
  const uint32_t mflimit = n > 12u ? n - 12u : 0u;
  const uint32_t matchlimit = n > 5u ? n - 5u : 0u;
  // the aligned word pairs lz_load32 reads must stay inside [src & ~3, src + n + 3]: positions < mflimit read <= n - 9
  while (ip < mflimit) {
    // ---- kLzR * 32 positions: position ip + 32 r + lane is lane's r-th; every load of the step is issued before the first use ----
    // the input is read once, front to back, one dependent step after the other: ask for it ahead of the steps (one lane per
    // 128-byte line: 2 KB ahead into L2, 512 bytes ahead into L1)
    {
      const uint32_t a2 = ip + 2048u + 128u * lane, a1 = ip + 512u + 128u * lane;
      if (lane < kLzR && a2 < n) lz_prefetch(src + a2, false);
      if (lane < kLzR && a1 < n) lz_prefetch(src + a1, true);
    }
    uint2 v[kLzR];
    uint32_t stored[kLzR];
    bool ok[kLzR];
#pragma unroll
    for (int r = 0; r < kLzR; ++r) {
      const uint32_t p = ip + 32u * r + lane;
      ok[r] = p < mflimit;
      v[r] = ok[r] ? lz_load64(src + p) : make_uint2(0u, 0u);
    }
    uint32_t mix[kLzR];
#pragma unroll
    for (int r = 0; r < kLzR; ++r) {
      mix[r] = lz_mix(v[r].x);
      stored[r] = table[lz_slot(mix[r])];
    }
    __syncwarp();
#pragma unroll
    for (int r = 0; r < kLzR; ++r) {
      if (ok[r]) table[lz_slot(mix[r])] = lz_tag(mix[r]) | ((ip + 32u * r + lane) & 0xFFFFu);
    }
    __syncwarp();
    uint32_t cand[kLzR];
    uint2 cv[kLzR];
    bool maybe[kLzR];
#pragma unroll
    for (int r = 0; r < kLzR; ++r) {
      const uint32_t p = ip + 32u * r + lane;
      const uint32_t d = (p - stored[r]) & 0xFFFFu;
      cand[r] = p - d;
      // the entry's tag: 16 more bits of the hash. Without it nearly every position verified a stale candidate -- 128 scattered
      // sectors from L2 per 128 bytes of input, which is what the round-1 coder's time went into
      maybe[r] = ok[r] && d != 0u && d <= p && (stored[r] & 0xFFFF0000u) == lz_tag(mix[r]);
      cv[r] = maybe[r] ? lz_load64(src + cand[r]) : make_uint2(0u, 0u);
    }
    uint32_t mp = 0xFFFFFFFFu, ref = 0, len = 0;
#pragma unroll
    for (int r = 0; r < kLzR; ++r) {
      // equal leading bytes among the eight in registers (8 = all of them: the match may go on)
      const uint32_t dx = cv[r].x ^ v[r].x, dy = cv[r].y ^ v[r].y;
      const uint32_t common = dx ? static_cast<uint32_t>(__ffs(static_cast<int>(dx)) - 1) >> 3 : 4u + (dy ? static_cast<uint32_t>(__ffs(static_cast<int>(dy)) - 1) >> 3 : 4u);
      const bool valid = maybe[r] && common >= static_cast<uint32_t>(kLzMinMatch);
      const uint32_t mask = __ballot_sync(0xffffffffu, valid);
      if (mp == 0xFFFFFFFFu && mask != 0u) {
        const int first = __ffs(static_cast<int>(mask)) - 1;
        mp = ip + 32u * r + static_cast<uint32_t>(first);
        ref = __shfl_sync(0xffffffffu, cand[r], first);
        len = __shfl_sync(0xffffffffu, common, first);
      }
    }
    if (mp == 0xFFFFFFFFu) { ip += 32u * kLzR; continue; }
    // (mp < mflimit = n - 12: the eight compared bytes end in front of the last five, which must stay literals)
    while (len >= 8u) {  // the match may go on: 32 more bytes per round
      const uint32_t q = mp + len + lane;
      const bool eq = q < matchlimit && src[q] == src[ref + len + lane];
      const uint32_t ne = __ballot_sync(0xffffffffu, !eq);
      if (ne) { len += static_cast<uint32_t>(__ffs(static_cast<int>(ne)) - 1); break; }
      len += 32u;
    }
    const uint32_t lit = mp - anchor, ml = len - 4u;
    const uint32_t need = 1u + lz_ext_bytes(lit) + lit + 2u + lz_ext_bytes(ml);
    if (op + need + 16u > cap) return 0u;  // (+ room for the final literals' header)
    if (lane == 0) dst[op] = static_cast<uint8_t>((lit >= 15u ? 15u : lit) << 4 | (ml >= 15u ? 15u : ml));
    op += 1u;
    if (lit >= 15u) { lz_write_ext(dst + op, lit, lane); op += lz_ext_bytes(lit); }
    lz_copy(dst + op, src + anchor, lit, lane, 32u);
    op += lit;
    if (lane == 0) { dst[op] = static_cast<uint8_t>(mp - ref); dst[op + 1] = static_cast<uint8_t>((mp - ref) >> 8); }
    op += 2u;
    if (ml >= 15u) { lz_write_ext(dst + op, ml, lane); op += lz_ext_bytes(ml); }
    ip = mp + len;
    anchor = ip;
  }
  const uint32_t lit = n - anchor;
  if (op + 1u + lz_ext_bytes(lit) + lit > cap) return 0u;
  if (lane == 0) dst[op] = static_cast<uint8_t>((lit >= 15u ? 15u : lit) << 4);
  op += 1u;
  if (lit >= 15u) { lz_write_ext(dst + op, lit, lane); op += lz_ext_bytes(lit); }
  lz_copy(dst + op, src + anchor, lit, lane, 32u);
  op += lit;
  __syncwarp();
  return op;
}

// One full warp. Returns the decompressed size, 0xFFFFFFFF for a malformed block / a block that does not fit `cap`.
__device__ uint32_t lz4_decompress_warp(const uint8_t* __restrict__ src, uint32_t n, uint8_t* dst, uint32_t cap) {
  const uint32_t lane = threadIdx.x & 31u;
  uint32_t ip = 0, op = 0;
  if (n == 0) return 0xFFFFFFFFu;
  while (true) {
    if (ip >= n) return 0xFFFFFFFFu;
    const uint32_t token = src[ip++];
    uint32_t lit = token >> 4;
    if (lit == 15u) {
      uint32_t b;
      do {
        if (ip >= n) return 0xFFFFFFFFu;
        b = src[ip++];
        lit += b;
      } while (b == 255u);
    }
    if (lit > n - ip || lit > cap - op) return 0xFFFFFFFFu;
    lz_copy(dst + op, src + ip, lit, lane, 32u);
    ip += lit;
    op += lit;
    if (ip >= n) break;  // a block ends with literals
    if (n - ip < 2u) return 0xFFFFFFFFu;
    const uint32_t offset = static_cast<uint32_t>(src[ip]) | (static_cast<uint32_t>(src[ip + 1]) << 8);
    ip += 2u;
    if (offset == 0u || offset > op) return 0xFFFFFFFFu;
    uint32_t ml = token & 15u;
    if (ml == 15u) {
      uint32_t b;
      do {
        if (ip >= n) return 0xFFFFFFFFu;
        b = src[ip++];
        ml += b;
      } while (b == 255u);
    }
    ml += 4u;
    if (ml > cap - op) return 0xFFFFFFFFu;
    __syncwarp();  // the literals just written may be the match's source
    if (offset >= 32u) {
      for (uint32_t base = 0; base < ml; base += 32u) {
        const uint32_t k = base + lane;
        if (k < ml) dst[op + k] = dst[op + k - offset];
        __syncwarp();  // a later round may read what this one wrote
      }
    } else {
      const uint8_t* pat = dst + op - offset;  // the match repeats these `offset` bytes
      for (uint32_t k = lane; k < ml; k += 32u) dst[op + k] = pat[k % offset];
      __syncwarp();
    }
    op += ml;
  }
  __syncwarp();
  return op;
}

// grid: ceil(n_chunks_total / 4) CTAs of 4 warps; warp -> (frame, chunk) through chunk_frame[]
__global__ void __launch_bounds__(kLzThreads) lz4_compress_chunks_kernel(const Lz4Launch L) {
  __shared__ uint32_t s_table[kLzWarps][1u << kLzHashBits];
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31u;
  const uint32_t gc = blockIdx.x * kLzWarps + warp;
  if (gc >= L.n_chunks_total) return;
  const uint32_t f = L.chunk_frame[gc];
  const Lz4Frame F = L.frames[f];
  if (L.empty_slots && chunk_slot_empty(F, gc)) return;
  const uint32_t c = gc - F.chunk_begin;
  uint64_t body = 0;
  const uint32_t n = lz_find_chunk(F.plain, *F.plain_bytes, c, &body);
  uint32_t csize = 0;
  if (n != 0xFFFFFFFFu) csize = lz4_compress_warp(F.plain + body, n, L.scratch + static_cast<size_t>(gc) * L.slot_stride, L.slot_stride, s_table[warp]);
  if (lane == 0) {
    L.chunk_sizes[gc] = csize;
    if (csize == 0u) report_frame_error(L, f, DEV_ERR_LZ4);  // cannot happen with slots of LZ4_COMPRESSBOUND size
  }
}

__global__ void __launch_bounds__(kLzThreads) lz4_decompress_chunks_kernel(const Lz4Launch L) {
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31u;
  const uint32_t gc = blockIdx.x * kLzWarps + warp;
  if (gc >= L.n_chunks_total) return;
  const uint32_t f = L.chunk_frame[gc];
  const Lz4Frame F = L.frames[f];
  if (chunk_slot_empty(F, gc)) return;
  const uint32_t c = gc - F.chunk_begin;
  uint64_t body = 0;
  const uint32_t n = lz_find_chunk(F.packed_in, F.packed_in_bytes, c, &body);
  uint32_t dsize = 0xFFFFFFFFu;
  if (n != 0xFFFFFFFFu) dsize = lz4_decompress_warp(F.packed_in + body, n, L.scratch + static_cast<size_t>(gc) * L.slot_stride, L.slot_stride);
  if (lane == 0) {
    L.chunk_sizes[gc] = dsize == 0xFFFFFFFFu ? 0u : dsize;
    if (n == 0xFFFFFFFFu) report_frame_error(L, f, DEV_ERR_CHUNK_SIZE);  // "Invalid chunk size found while decoding"
    else if (dsize == 0xFFFFFFFFu) report_frame_error(L, f, DEV_ERR_LZ4);  // "LZ4 decompression failed"
  }
}

// One CTA per frame: ([u32 size][bytes])* of the frame's chunks, back to back at `dst` (behind `header_bytes` bytes of
// header, which are copied too); the frame's total goes to sizes[f]. Stores are checked against dst_cap. A chunk's bytes
// are its slot, or with L.block_begin the concatenation of its pieces (ZSTD compression).
// (shared by the ZSTD decompressor, launch_stage2_unpack: `unpack_err` is the code of a re-framed payload that does not fit)
__global__ void __launch_bounds__(256) lz4_pack_frames_kernel(const Lz4Launch L, const uint8_t* header, uint32_t header_bytes, int to_blob,
                                                              uint32_t unpack_err) {
  const uint32_t f = blockIdx.x;
  const Lz4Frame F = L.frames[f];
  uint8_t* dst = to_blob ? F.blob_out : F.plain_out;
  const uint64_t cap = to_blob ? F.blob_cap : F.plain_cap;
  __shared__ unsigned long long s_pos;
  uint64_t pos = header_bytes;
  if (header_bytes <= cap) {
    for (uint32_t k = threadIdx.x; k < header_bytes; k += blockDim.x) dst[k] = header[k];
  }
  bool fits = header_bytes <= cap;
  for (uint32_t c = 0; c < F.n_chunks; ++c) {
    const uint32_t gc = F.chunk_begin + c;
    const uint32_t p0 = L.block_begin ? L.block_begin[gc] : gc, p1 = L.block_begin ? L.block_begin[gc + 1] : gc + 1;
    uint64_t sz = 0;
    for (uint32_t p = p0; p < p1; ++p) sz += L.chunk_sizes[p];
    if (pos + 4ull + sz > cap) { fits = false; break; }
    if (threadIdx.x == 0) store_u32(dst + pos, static_cast<uint32_t>(sz));
    pos += 4ull;
    for (uint32_t p = p0; p < p1; ++p) {
      const uint32_t psz = L.chunk_sizes[p];
      lz_copy(dst + pos, L.scratch + static_cast<size_t>(p) * L.slot_stride, psz, threadIdx.x, blockDim.x);
      pos += psz;
    }
  }
  if (threadIdx.x == 0) {
    s_pos = pos;
    L.sizes[f] = fits ? pos : 0ull;
    if (!fits) report_frame_error(L, f, to_blob ? DEV_ERR_ENCODE_OUTPUT_SMALL : unpack_err);
  }
  (void)s_pos;
}

int launch_stage2_pack(const Lz4Launch& L, const uint8_t* header, uint32_t header_bytes, cudaStream_t stream) {
  if (L.n_frames == 0) return 0;
  lz4_pack_frames_kernel<<<L.n_frames, 256, 0, stream>>>(L, header, header_bytes, 1, DEV_ERR_LZ4);
  count_launch(1);
  return 1;
}

int launch_lz4_compress(const Lz4Launch& L, const uint8_t* header, uint32_t header_bytes, cudaStream_t stream) {
  if (L.n_frames == 0) return 0;
  int n = 0;
  if (L.n_chunks_total) {
    lz4_compress_chunks_kernel<<<(L.n_chunks_total + kLzWarps - 1) / kLzWarps, kLzThreads, 0, stream>>>(L);
    count_launch(1);
    ++n;
  }
  return n + launch_stage2_pack(L, header, header_bytes, stream);
}

int launch_lz4_decompress(const Lz4Launch& L, cudaStream_t stream) {
  if (L.n_frames == 0) return 0;
  int n = 0;
  if (L.n_chunks_total) {
    lz4_decompress_chunks_kernel<<<(L.n_chunks_total + kLzWarps - 1) / kLzWarps, kLzThreads, 0, stream>>>(L);
    ++n;
  }
  lz4_pack_frames_kernel<<<L.n_frames, 256, 0, stream>>>(L, nullptr, 0, 0, DEV_ERR_LZ4);
  count_launch(n + 1);
  return n + 1;
}

int launch_stage2_unpack(const Lz4Launch& L, uint32_t fail_code, cudaStream_t stream) {
  if (L.n_frames == 0) return 0;
  lz4_pack_frames_kernel<<<L.n_frames, 256, 0, stream>>>(L, nullptr, 0, 0, fail_code);
  count_launch(1);
  return 1;
}

// One CTA per blob; tab holds n source addresses, n byte counts and n destination offsets.
__global__ void __launch_bounds__(256) gather_prefixes_kernel(const uint64_t* tab, uint32_t n, uint8_t* dst) {
  const uint32_t f = blockIdx.x;
  const uint8_t* src = reinterpret_cast<const uint8_t*>(tab[f]);
  lz_copy(dst + tab[2ull * n + f], src, static_cast<uint32_t>(tab[n + f]), threadIdx.x, blockDim.x);
}

int launch_gather_prefixes(const uint64_t* tab, uint32_t n, uint8_t* dst, cudaStream_t stream) {
  if (n == 0) return 0;
  gather_prefixes_kernel<<<n, 256, 0, stream>>>(tab, n, dst);
  count_launch(1);
  return 1;
}

// One CTA per blob; tab holds n destination addresses and n + 1 offsets into the packed header bytes that follow it.
// Blob f's header goes in front of its payload, and the payload size in sizes[f] becomes the blob size. With `slots`
// (2n words), the payload size is from[slots[f]] and the blob size goes to sizes[slots[n + f]].
__global__ void __launch_bounds__(256) place_headers_kernel(const uint64_t* tab, uint32_t n, uint64_t* sizes, const uint64_t* from,
                                                            const uint32_t* slots) {
  const uint32_t f = blockIdx.x;
  const uint8_t* packed = reinterpret_cast<const uint8_t*>(tab + 2ull * n + 1);
  const uint64_t begin = tab[n + f], bytes = tab[n + f + 1] - begin;
  lz_copy(reinterpret_cast<uint8_t*>(tab[f]), packed + begin, static_cast<uint32_t>(bytes), threadIdx.x, blockDim.x);
  if (threadIdx.x != 0) return;
  if (slots) sizes[slots[n + f]] = from[slots[f]] + bytes;
  else sizes[f] += bytes;
}

int launch_place_headers(const uint64_t* tab, uint32_t n, uint64_t* sizes, cudaStream_t stream, const uint64_t* from,
                         const uint32_t* slots) {
  if (n == 0) return 0;
  place_headers_kernel<<<n, 256, 0, stream>>>(tab, n, sizes, from, slots);
  count_launch(1);
  return 1;
}

}  // namespace cldn
