// Stage-1 ENCODE kernels: interleaved regular stream + chunk framing, one fused launch for a batch of frames.
//
// Replaces the per-point x per-encoder loop of EncodeV4Stage1Chunk (cloudini_lib/src/v4_codec.cpp:66-83) /
// EncodeV5Stage1's regular part (v5_codec.cpp:920-932) and WriteStage1Chunk's u32 framing (chunk_writer.cpp:27-48).
//
// Grid = one CTA per tile of T = 256*I points (T divides the 32768-point chunk, so tiles never straddle chunks).
//  pass A   every thread quantises its points, takes the delta to the previous point and sizes the varints;
//  scan     warp scans of per-point byte counts give tile-local offsets and the tile's size, which is published at once
//           as the aggregate of a decoupled look-back over the frame's tiles (input is read exactly once from HBM);
//  pass B   the LEB128 bytes are formed and stored byte-wise into a shared-memory staging buffer at their offsets,
//           while warp 0 polls the look-back window between its iterations;
//  copy-out the staged bytes are streamed to their final (arbitrarily aligned) position with 16-byte stores;
//  framing  the last tile of every chunk back-patches the chunk's u32 size prefix, the last tile of a frame writes
//           the frame's total size.
#include <stdio.h>

#include <atomic>
#include <map>
#include <mutex>
#include <utility>

#include "cldn_device.cuh"
#include "cldn_kernels.h"

namespace cldn {

// ------------------------------------------------------------------------------------------------------------------
// Per-point evaluation of an arbitrary regular-stream plan (generic path; also the 5-byte slow path of the FloatN
// kernel). `prev` is the previous point of the same chunk or nullptr at a chunk start: every reference encoder only
// keeps the previous point's quantised value (0 after reset() or after a NaN), so it is recomputed instead of carried.
template <class Sink>
__device__ __forceinline__ void encode_point_ops(const Plan& plan, const uint8_t* __restrict__ pt,
                                                 const uint8_t* __restrict__ prev, Sink& sink,
                                                 const uint8_t* __restrict__ side = nullptr, uint32_t side_stride = 0) {
  uint32_t gorilla_idx = 0;
  for (uint32_t k = 0; k < plan.n_ops; ++k) {
    const RegOp& op = plan.ops[k];
    switch (op.kind) {
      case OP_XOR32: case OP_XOR64: {  // field_encoder.hpp:360-370: residual = bits ^ previous point's bits (0 at a chunk start)
        const uint64_t cur = load_raw_bits(pt + op.offset[0], op.size);
        const uint64_t pb = prev ? load_raw_bits(prev + op.offset[0], op.size) : 0ull;
        sink.put_le(cur ^ pb, op.size);
      } break;
      case OP_GORILLA64: {  // record built by gorilla_prepass_kernel (the window state is sequential along the chunk)
        const uint8_t* rec = side + static_cast<size_t>(gorilla_idx) * side_stride;
        sink.put_raw(rec, rec[11]);
        ++gorilla_idx;
      } break;
      case OP_FLOATN: {  // field_encoder.cpp:42-91
        for (int l = 0; l < op.lanes; ++l) {
          const float v = __uint_as_float(load_u32(pt + op.offset[l]));
          if (isnan(v)) { sink.put_byte(0); continue; }
          const int32_t q = quant_i32_x86(v, op.enc_mul_f[l]);
          int32_t pq = 0;
          if (prev) {
            const float pv = __uint_as_float(load_u32(prev + op.offset[l]));
            if (!isnan(pv)) pq = quant_i32_x86(pv, op.enc_mul_f[l]);
          }
          const int32_t d = static_cast<int32_t>(static_cast<uint32_t>(q) - static_cast<uint32_t>(pq));  // _mm_sub_epi32
          sink.put_varint(zigzag_plus1(static_cast<int64_t>(d)));
        }
      } break;
      case OP_F32_LOSSY: {  // field_encoder.hpp:343-357
        const float v = __uint_as_float(load_u32(pt + op.offset[0]));
        if (isnan(v)) { sink.put_byte(0); break; }
        const int64_t q = quant_i64_f32(v, op.enc_mul_f[0]);
        int64_t pq = 0;
        if (prev) {
          const float pv = __uint_as_float(load_u32(prev + op.offset[0]));
          if (!isnan(pv)) pq = quant_i64_f32(pv, op.enc_mul_f[0]);
        }
        sink.put_varint(zigzag_plus1(static_cast<int64_t>(static_cast<uint64_t>(q) - static_cast<uint64_t>(pq))));
      } break;
      case OP_F64_LOSSY: {
        const double v = __longlong_as_double(static_cast<long long>(load_u64(pt + op.offset[0])));
        if (isnan(v)) { sink.put_byte(0); break; }
        const int64_t q = quant_i64_f64(v, op.enc_mul_d);
        int64_t pq = 0;
        if (prev) {
          const double pv = __longlong_as_double(static_cast<long long>(load_u64(prev + op.offset[0])));
          if (!isnan(pv)) pq = quant_i64_f64(pv, op.enc_mul_d);
        }
        sink.put_varint(zigzag_plus1(static_cast<int64_t>(static_cast<uint64_t>(q) - static_cast<uint64_t>(pq))));
      } break;
      case OP_INT: {  // field_encoder.hpp:78-85
        const int64_t v = load_int_as_i64(pt + op.offset[0], op.type);
        const int64_t pv = prev ? load_int_as_i64(prev + op.offset[0], op.type) : 0;
        sink.put_varint(zigzag_plus1(static_cast<int64_t>(static_cast<uint64_t>(v) - static_cast<uint64_t>(pv))));
      } break;
      default:  // OP_COPY, field_encoder.hpp:56-60
        sink.put_raw(pt + op.offset[0], op.size);
        break;
    }
  }
}

// Frame lookup: last frame whose tile_begin <= tile (empty frames share tile_begin with their successor).
__device__ __forceinline__ uint32_t find_frame(const EncFrame* __restrict__ frames, uint32_t n_frames, uint32_t tile) {
  uint32_t lo = 0, hi = n_frames - 1;
  while (lo < hi) {
    const uint32_t mid = (lo + hi + 1) >> 1;
    if (frames[mid].tile_begin <= tile) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// Header copy + bookkeeping for frames without any tile (0 points); run by CTA 0.
__device__ __forceinline__ void handle_empty_frames(const EncLaunch& L) {
  for (uint32_t f = threadIdx.x; f < L.n_frames; f += blockDim.x) {
    if (L.frames[f].n_tiles == 0) {
      for (uint32_t i = 0; i < L.header_bytes; ++i) L.frames[f].out[i] = L.header[i];
      L.sizes[f] = L.header_bytes;
    }
  }
}

// Common tail of both encode kernels: copy-out, chunk prefix back-patch, frame size.
//  total   = bytes staged by this tile, excl = data bytes of all earlier tiles of the frame (look-back result)
template <uint32_t T>  // points per tile: a power of two that divides the chunk, so the divisions below are shifts
__device__ __forceinline__ void finish_tile(const EncLaunch& L, const EncFrame& F, uint32_t frame_idx, uint32_t t,
                                            const uint8_t* stage, uint32_t total, uint64_t excl) {
  constexpr uint32_t tiles_per_chunk = kChunkPoints / T;
  const uint32_t chunk = t / tiles_per_chunk;
  const uint64_t sec_before = F.sec_excl ? F.sec_excl[chunk] : 0;
  uint8_t* payload = F.out + L.header_bytes;
  // data position: one u32 prefix per chunk up to and including mine, all earlier data, all earlier chunks' sections
  const uint64_t at = 4ull * (chunk + 1) + excl + sec_before;
  const bool fits = L.header_bytes + at + total <= F.out_cap;  // "Output buffer too small for uncompressed chunk"
  if (fits) copy_stage_to_global(stage, total, payload + at);
  else if (threadIdx.x == 0) report_frame_error(L, frame_idx, DEV_ERR_ENCODE_OUTPUT_SMALL);
  if (t == 0 && L.header_bytes <= F.out_cap) {
    for (uint32_t i = threadIdx.x; i < L.header_bytes; i += blockDim.x) F.out[i] = L.header[i];
  }
  const bool last_of_frame = (t + 1 == F.n_tiles);
  const bool last_of_chunk = last_of_frame || ((t + 1) % tiles_per_chunk == 0);
  if (last_of_chunk && threadIdx.x == 0) {
    const uint32_t first = chunk * tiles_per_chunk;
    const uint64_t data_before_chunk = (first == 0) ? 0 : wait_inclusive(L.status, F.tile_begin + first - 1, L.epoch);
    const uint64_t sec_mine = F.sec_excl ? (F.sec_excl[chunk + 1] - F.sec_excl[chunk]) : 0;
    const uint64_t body = (excl + total) - data_before_chunk + sec_mine;
    if (L.header_bytes + 4ull * (chunk + 1) + data_before_chunk + sec_before <= F.out_cap) {
      store_u32(payload + 4ull * chunk + data_before_chunk + sec_before, static_cast<uint32_t>(body));  // chunk_writer.cpp:33-40
    }
    if (last_of_frame) {
      L.sizes[frame_idx] = L.header_bytes + 4ull * F.n_chunks + excl + total + (F.sec_excl ? F.sec_excl[F.n_chunks] : 0);
    }
  }
}

// ------------------------------------------------------------------------------------------------------------------
// Generic kernel: any supported plan. Thread-blocked point assignment (thread owns I consecutive points).
template <int I>
__global__ void __launch_bounds__(kThreads) encode_generic_kernel(const EncLaunch L) {
  extern __shared__ __align__(16) uint8_t dyn_smem[];
  __shared__ uint32_t s_scan[kThreads / 32 + 1];
  __shared__ unsigned long long s_excl;
  Plan& plan = *reinterpret_cast<Plan*>(dyn_smem);
  uint8_t* stage = dyn_smem + ((sizeof(Plan) + 15) & ~size_t(15));

  {  // plan -> shared memory (uniform reads afterwards)
    const uint32_t* src = reinterpret_cast<const uint32_t*>(L.plan);
    uint32_t* dst = reinterpret_cast<uint32_t*>(&plan);
    for (uint32_t i = threadIdx.x; i < sizeof(Plan) / 4; i += blockDim.x) dst[i] = src[i];
  }
  if (blockIdx.x == 0) handle_empty_frames(L);
  // Batches of equally sized frames: consecutive CTAs take the same tile of consecutive frames, so the predecessors a
  // tile has to look back at (same frame) were dispatched n_frames CTAs earlier and have usually published already.
  // (Still in-order: a tile's predecessors always have a smaller blockIdx.)
  const uint32_t fi = L.uniform_tiles ? blockIdx.x % L.n_frames : find_frame(L.frames, L.n_frames, blockIdx.x);
  const EncFrame F = L.frames[fi];
  const uint32_t t = L.uniform_tiles ? blockIdx.x / L.n_frames : blockIdx.x - F.tile_begin;
  if (L.empty_slots && t >= F.n_tiles) return;  // an empty tile slot (EncLaunch::empty_slots)
  const uint32_t tile = F.tile_begin + t;  // index of the tile's status word
  const uint32_t T = kThreads * I;
  const uint32_t p0 = t * T + threadIdx.x * I;
  const uint32_t step = L.plan->point_step;
  __syncthreads();

  uint32_t len[I];
  uint32_t mine = 0;
#pragma unroll
  for (int i = 0; i < I; ++i) {
    const uint32_t p = p0 + i;
    len[i] = 0;
    if (p < F.n_points) {
      const uint8_t* pt = F.in + static_cast<size_t>(p) * step;
      const uint8_t* prev = (p % kChunkPoints) ? pt - step : nullptr;
      CountSink cs;
      encode_point_ops(plan, pt, prev, cs, F.side ? F.side + static_cast<size_t>(p) * 12 : nullptr, F.n_points * 12u);
      len[i] = cs.n;
    }
    mine += len[i];
  }
  uint32_t total;
  uint32_t off = block_exclusive_scan(mine, s_scan, &total);
  if (threadIdx.x == 0) {
    st_relaxed_u64(L.status + tile, pack_status(t == 0 ? kFlagIncl : kFlagAgg, L.epoch, total));
  }
#pragma unroll
  for (int i = 0; i < I; ++i) {
    const uint32_t p = p0 + i;
    if (p < F.n_points) {
      const uint8_t* pt = F.in + static_cast<size_t>(p) * step;
      const uint8_t* prev = (p % kChunkPoints) ? pt - step : nullptr;
      ByteSink bs{stage + off};
      encode_point_ops(plan, pt, prev, bs, F.side ? F.side + static_cast<size_t>(p) * 12 : nullptr, F.n_points * 12u);
      off += len[i];
    }
  }
  if (threadIdx.x < 32) {
    const uint64_t e = tile_lookback(L.status, F.tile_begin, tile, L.epoch, total);
    if (threadIdx.x == 0) s_excl = e;
  }
  __syncthreads();
  finish_tile<kThreads * I>(L, F, fi, t, stage, total, s_excl);
}

// ------------------------------------------------------------------------------------------------------------------
// Specialised kernel: the regular stream is exactly one FloatN op (C1/C2 XYZ / XYZI; also the float part of C3).
//   VEC4 = packed XYZI float32x4 at a 16-byte aligned base: one coalesced LDG.128 per point.
// Warp-blocked point assignment: warp w owns points [w*32*I, (w+1)*32*I), lane l takes point 32*i + l of iteration i,
// so loads are perfectly coalesced, the previous point comes from a lane shuffle and each iteration's output is one
// contiguous byte run.
struct FloatNParams {
  uint32_t offset[4];
  float mul[4];
  uint32_t point_step;
};

// u in [1, 2^28): LEB128 bytes of u packed little-endian into one word (continuation bits included).
__device__ __forceinline__ uint32_t varint_word_28(uint32_t u) {
  // 7-bit groups -> bytes: adding the masked upper part to itself shifts it left by one, three times.
  uint32_t x = u + (u & 0xFFFFFF80u);
  x = x + (x & 0xFFFF8000u);
  x = x + (x & 0xFF800000u);
  // continuation flag on every byte below the most significant non-zero byte
  const uint32_t g = x >> 8;
  const uint32_t h = g | (g >> 8) | (g >> 16);
  return x | ((h + 0x007F7F7Fu) & 0x00808080u);
}

template <int N, int I, bool VEC4, int MINB>
__global__ void __launch_bounds__(kThreads, MINB) encode_floatn_kernel(const EncLaunch L, const FloatNParams P) {
  extern __shared__ __align__(16) uint8_t dyn_smem[];
  __shared__ uint32_t s_wtot[kThreads / 32];
  __shared__ unsigned long long s_excl;
  uint8_t* stage = dyn_smem;
  uint32_t* stage32 = reinterpret_cast<uint32_t*>(dyn_smem);

  if (blockIdx.x == 0) handle_empty_frames(L);
  // Batches of equally sized frames: consecutive CTAs take the same tile of consecutive frames, so the predecessors a
  // tile has to look back at (same frame) were dispatched n_frames CTAs earlier and have usually published already.
  // (Still in-order: a tile's predecessors always have a smaller blockIdx.)
  const uint32_t fi = L.uniform_tiles ? blockIdx.x % L.n_frames : find_frame(L.frames, L.n_frames, blockIdx.x);
  const EncFrame F = L.frames[fi];
  const uint32_t t = L.uniform_tiles ? blockIdx.x / L.n_frames : blockIdx.x - F.tile_begin;
  if (L.empty_slots && t >= F.n_tiles) return;  // an empty tile slot (EncLaunch::empty_slots)
  const uint32_t tile = F.tile_begin + t;  // index of the tile's status word
  constexpr uint32_t T = kThreads * I;
  // VEC4 launches whose frames' alignment only the device knows take the 16-byte loads frame by frame
  const bool vec4 = VEC4 && enc_input_aligned16(L.flags, F.in);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint32_t tile_p0 = t * T;
  const uint32_t warp_p0 = tile_p0 + warp * 32 * I;
  const uint32_t step = P.point_step;

  // ---- loads (all issued before use: I independent 16-byte requests per thread) ----
  float v[I][N];
#pragma unroll
  for (int i = 0; i < I; ++i) {
    const uint32_t p = warp_p0 + 32 * i + lane;
    if (p < F.n_points) {
      if (vec4) {
        const float4 q = __ldcs(reinterpret_cast<const float4*>(F.in) + p);
        v[i][0] = q.x; v[i][1] = q.y; v[i][2] = q.z;
        if (N == 4) v[i][N - 1] = q.w;
      } else {
        const uint8_t* pt = F.in + static_cast<size_t>(p) * step;
#pragma unroll
        for (int k = 0; k < N; ++k) v[i][k] = __uint_as_float(load_u32(pt + P.offset[k]));
      }
    } else {
#pragma unroll
      for (int k = 0; k < N; ++k) v[i][k] = 0.f;
    }
  }
  // previous point of the warp's first point (0 at a chunk start; T divides the chunk so only tile_p0 can be one)
  int32_t carry[N];
#pragma unroll
  for (int k = 0; k < N; ++k) carry[k] = 0;
  if (warp_p0 % kChunkPoints != 0 && warp_p0 < F.n_points) {
    const uint8_t* pt = F.in + static_cast<size_t>(warp_p0 - 1) * step;
#pragma unroll
    for (int k = 0; k < N; ++k) {
      const float pv = __uint_as_float(load_u32(pt + P.offset[k]));
      carry[k] = isnan(pv) ? 0 : quant_i32_x86(pv, P.mul[k]);
    }
  }

  // ---- phase 1: quantise, delta, varint bytes (as words), per-point sizes ----
  uint32_t r[I][N];   // zigzag + 1 of each value (0 for the NaN marker)
  // one word of bookkeeping per point: [2:0] len(v0)  [6:3] len(v0..v1)  [10:7] len(v0..v2)  [15:11] total length
  // [31:16] byte offset of the point inside the warp's run (filled in after the scan)
  uint32_t meta[I];
  // Anything the 4-byte fast path cannot represent sends the whole tile to the exact byte-wise path, which recomputes
  // the sizes too: a zigzag value >= 2^28 - 1 (5-byte varint; `wide` collects the bits of zz and zz + 1) and a product
  // >= 2^31 (cvt saturates to INT_MAX where the reference's cvtps2dq gives INT_MIN; `smax` tracks the largest product).
  uint32_t wide = 0;
  float smax = 0.0f;
#pragma unroll
  for (int i = 0; i < I; ++i) {
    uint32_t acc = 0, packed = 0;
#pragma unroll
    for (int k = 0; k < N; ++k) {
      const bool nan = isnan(v[i][k]);
      // NaN input gives q = 0 here (cvt.rni of NaN), which is exactly what the next point must see as "previous"
      // (field_encoder.cpp:79-82)
      const float sc = __fmul_rn(v[i][k], P.mul[k]);
      const int32_t q = __float2int_rn(sc);
      smax = fmaxf(smax, sc);
      // previous point: lane-1 of this iteration; lane 0 takes lane 31 of the previous iteration (one rotate per value)
      const int32_t rot = __shfl_sync(0xffffffffu, q, (lane + 31) & 31);
      const int32_t prev = (lane == 0) ? carry[k] : rot;
      carry[k] = rot;  // only lane 0 uses it (it holds lane 31's value of this iteration)
      const uint32_t d = static_cast<uint32_t>(q) - static_cast<uint32_t>(prev);
      const uint32_t zz = (d << 1) ^ static_cast<uint32_t>(static_cast<int32_t>(d) >> 31);
      // zz + 1 may wrap for zz = 2^32 - 1 (then `wide` has bit 31 from zz); NaN lanes become the single 0x00 byte
      const uint32_t u = nan ? 0u : zz + 1u;
      wide |= nan ? 0u : (zz | u);
      uint32_t b;  // index of the highest set bit (bfind, not 31 - clz: one instruction)
      asm("bfind.u32 %0, %1;" : "=r"(b) : "r"(u | 1u));
      const uint32_t lenm1 = (b * 37u) >> 8;            // floor(b / 7) for b <= 34
      r[i][k] = u;  // the LEB128 bytes are formed in the packing loop, after the tile's size has been published
      acc += lenm1 + 1u;
      if (k < N - 1) packed |= acc << (k == 0 ? 0 : k == 1 ? 3 : 7);
    }
    meta[i] = (N == 4) ? (packed | (acc << 11)) : (packed | (acc << 7) | (acc << 11));
  }
  // the fast path also assumes a full tile; the (single) partial tile of a frame takes the byte-wise path too
  const uint32_t big = ((wide >> 28) != 0u || smax >= 2147483648.0f || tile_p0 + T > F.n_points) ? 1u : 0u;
  const int any_big = __syncthreads_or(static_cast<int>(big));
  if (any_big) {
    // exact sizes, evaluated like the reference does (field_encoder.cpp:42-91); the byte-wise emission below follows them
#pragma unroll 1
    for (int i = 0; i < I; ++i) {
      const uint32_t p = warp_p0 + 32 * i + lane;
      uint32_t len = 0;
      if (p < F.n_points) {
        const uint8_t* pt = F.in + static_cast<size_t>(p) * step;
        const uint8_t* prevp = (p % kChunkPoints) ? pt - step : nullptr;
#pragma unroll
        for (int k = 0; k < N; ++k) {
          const float x = __uint_as_float(load_u32(pt + P.offset[k]));
          if (isnan(x)) { len += 1; continue; }
          const int32_t q = quant_i32_x86(x, P.mul[k]);
          int32_t pq = 0;
          if (prevp) {
            const float px = __uint_as_float(load_u32(prevp + P.offset[k]));
            if (!isnan(px)) pq = quant_i32_x86(px, P.mul[k]);
          }
          const int32_t d = static_cast<int32_t>(static_cast<uint32_t>(q) - static_cast<uint32_t>(pq));
          len += varint_len(zigzag_plus1(static_cast<int64_t>(d)));
        }
      }
      meta[i] = len << 11;
    }
  }
  // ---- warp-level exclusive offsets: 10-bit fields, three iterations per shuffle scan (32 * 20 = 640 < 1024) ----
  uint32_t run = 0;   // bytes of earlier iterations of this warp
#pragma unroll
  for (int g = 0; g < I; g += 3) {
    uint32_t pk = meta[g] >> 11;
    if (g + 1 < I) pk |= (meta[g + 1] >> 11) << 10;
    if (g + 2 < I) pk |= (meta[g + 2] >> 11) << 20;
    uint32_t inc = pk;
#pragma unroll
    for (int dlt = 1; dlt < 32; dlt <<= 1) {
      const uint32_t x = __shfl_up_sync(0xffffffffu, inc, dlt);
      if (lane >= dlt) inc += x;
    }
    const uint32_t tot = __shfl_sync(0xffffffffu, inc, 31);
    const uint32_t exc = inc - pk;
    meta[g] |= (run + (exc & 1023u)) << 16;
    run += tot & 1023u;
    if (g + 1 < I) { meta[g + 1] |= (run + ((exc >> 10) & 1023u)) << 16; run += (tot >> 10) & 1023u; }
    if (g + 2 < I) { meta[g + 2] |= (run + ((exc >> 20) & 1023u)) << 16; run += (tot >> 20) & 1023u; }
  }
  if (lane == 0) s_wtot[warp] = run;
  __syncthreads();
  uint32_t wbase = 0, total = 0;
#pragma unroll
  for (int w = 0; w < kThreads / 32; ++w) {
    const uint32_t x = s_wtot[w];
    if (w < warp) wbase += x;
    total += x;
  }
  // ---- tile base: warp 0 publishes the aggregate now and polls the look-back window between its packing
  //      iterations, so that waiting for the slowest predecessor overlaps with useful work ----
  LookbackPoll lb;
  if (warp == 0) {
    lb.begin(L.status, F.tile_begin, tile, L.epoch, total);
    lb.issue(L.status, F.tile_begin, L.epoch);
  }

  // ---- phase 2: pack bytes into the staging buffer at tile-local offsets ----
  if (!any_big) {
    // every value leaves with byte stores straight at its position: a byte exists iff the one below it carries the
    // continuation flag, so no record assembly, no shifts across word boundaries and no neighbour merging is needed
#pragma unroll
    for (int i = 0; i < I; ++i) {
      if (warp == 0) {  // the status words asked for one iteration ago have arrived by now
        lb.eval(L.epoch);
        lb.issue(L.status, F.tile_begin, L.epoch);
      }
      uint8_t* dst = stage + wbase + (meta[i] >> 16);
#pragma unroll
      for (int k = 0; k < N; ++k) {
        const uint32_t pre = k == 0 ? 0u : k == 1 ? (meta[i] & 7u) : k == 2 ? ((meta[i] >> 3) & 15u) : ((meta[i] >> 7) & 15u);
        const uint32_t nxt = k == 0 ? (meta[i] & 7u) : k == 1 ? ((meta[i] >> 3) & 15u) : k == 2 ? ((meta[i] >> 7) & 15u) : ((meta[i] >> 11) & 31u);
        uint8_t* q = dst + pre;
        // 7-bit groups -> bytes: adding the masked upper part to itself shifts it left by one, three times
        const uint32_t u = r[i][k];
        uint32_t x = u + (u & 0xFFFFFF80u);
        x = x + (x & 0xFFFF8000u);
        x = x + (x & 0xFF800000u);
        uint32_t fl;  // continuation flags below the top byte (length 1..4 here)
        asm("shr.b32 %0, %1, %2;" : "=r"(fl) : "r"(0x00808080u), "r"(32u - 8u * (nxt - pre)));
        x |= fl;
        q[0] = static_cast<uint8_t>(x);
        if (x & 0x80u) q[1] = static_cast<uint8_t>(x >> 8);
        if (x & 0x8000u) q[2] = static_cast<uint8_t>(x >> 16);
        if (x & 0x800000u) q[3] = static_cast<uint8_t>(x >> 24);
      }
    }
  } else {
    // slow path (some |delta| >= 2^27): re-evaluate byte-wise, exactly like the generic kernel
#pragma unroll 1
    for (int i = 0; i < I; ++i) {
      const uint32_t p = warp_p0 + 32 * i + lane;
      if (p < F.n_points) {
        const uint8_t* pt = F.in + static_cast<size_t>(p) * step;
        const uint8_t* prevp = (p % kChunkPoints) ? pt - step : nullptr;
        ByteSink bs{stage + wbase + (meta[i] >> 16)};
#pragma unroll
        for (int k = 0; k < N; ++k) {
          const float x = __uint_as_float(load_u32(pt + P.offset[k]));
          if (isnan(x)) { bs.put_byte(0); continue; }
          const int32_t q = quant_i32_x86(x, P.mul[k]);
          int32_t pq = 0;
          if (prevp) {
            const float px = __uint_as_float(load_u32(prevp + P.offset[k]));
            if (!isnan(px)) pq = quant_i32_x86(px, P.mul[k]);
          }
          const int32_t d = static_cast<int32_t>(static_cast<uint32_t>(q) - static_cast<uint32_t>(pq));
          bs.put_varint(zigzag_plus1(static_cast<int64_t>(d)));
        }
      }
    }
  }
  if (warp == 0) {
    const uint64_t ex = lb.finish(L.status, F.tile_begin, tile, L.epoch, total);
    if (lane == 0) s_excl = ex;
  }
  __syncthreads();
  finish_tile<kThreads * I>(L, F, fi, t, stage, total, s_excl);
}

// ------------------------------------------------------------------------------------------------------------------
static std::atomic<uint64_t> g_launches{0};
uint64_t kernel_launch_count() { return g_launches.load(std::memory_order_relaxed); }
void count_launch(int n) { g_launches.fetch_add(static_cast<uint64_t>(n), std::memory_order_relaxed); }

cudaError_t raise_smem_limit_ptr(const void* kernel, size_t bytes) {
  static std::mutex mutex;
  static std::map<std::pair<int, const void*>, size_t> marks;  // highest limit set so far, per device context
  int dev = 0;
  if (const cudaError_t e = cudaGetDevice(&dev)) return e;
  std::lock_guard<std::mutex> lock(mutex);  // check and set together: two raising threads must not leave the smaller value
  size_t& mark = marks[{dev, kernel}];
  if (bytes <= mark) return cudaSuccess;
  const cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(bytes));
  if (e == cudaSuccess) mark = bytes;
  return e;
}

template <typename K>
static cudaError_t set_smem(K* kernel, size_t bytes) { return raise_smem_limit(kernel, bytes); }

template <int N, int I, int MINB>
static int launch_floatn(const Plan& plan, const EncLaunch& L, bool vec4, cudaStream_t stream) {
  FloatNParams P;
  for (int k = 0; k < 4; ++k) {
    P.offset[k] = plan.ops[0].offset[k];
    P.mul[k] = plan.ops[0].enc_mul_f[k];
  }
  P.point_step = plan.point_step;
  const size_t smem = static_cast<size_t>(kThreads) * I * 5 * N + 64;
  if (vec4) {
    auto k = encode_floatn_kernel<N, I, true, MINB>;
    if (set_smem(k, smem) != cudaSuccess) return -1;
    k<<<L.n_tiles_total, kThreads, smem, stream>>>(L, P);
  } else {
    auto k = encode_floatn_kernel<N, I, false, MINB>;
    if (set_smem(k, smem) != cudaSuccess) return -1;
    k<<<L.n_tiles_total, kThreads, smem, stream>>>(L, P);
  }
  count_launch();
  return 1;
}

// Gorilla pre-pass: one WARP per (chunk, Gorilla op) leaves a 12-byte record per point (bytes 0..9 the encoded value,
// byte 11 its length); the generic kernel then copies the record like any other field. Side layout: [op][point][12].
// The only sequential part of the coder is the (leading, trailing) window of the last "new window" record
// (field_encoder.hpp:262-296): a value keeps the window when its XOR fits into it, otherwise it starts a new one. The warp
// takes 32 consecutive values at a time; every lane knows its own XOR / leading / trailing zeros, and the window each lane
// sees is resolved with one ballot per window change inside the group (the first lane that does not fit becomes the
// new window for the lanes behind it) instead of 32 dependent steps.
constexpr int kGorillaThreads = 256;
__global__ void __launch_bounds__(kGorillaThreads) gorilla_prepass_kernel(const EncLaunch L) {
  const EncFrame F = L.frames[blockIdx.x];
  const Plan& plan = *L.plan;
  const uint32_t items = F.n_chunks * plan.n_gorilla;
  const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5, n_warps = blockDim.x >> 5;
  for (uint32_t it = warp; it < items; it += n_warps) {  // warp-uniform
    const uint32_t chunk = it / plan.n_gorilla, g = it % plan.n_gorilla;
    uint32_t seen = 0, offset = 0;
    for (uint32_t k = 0; k < plan.n_ops; ++k) {
      if (plan.ops[k].kind == OP_GORILLA64) {
        if (seen == g) offset = plan.ops[k].offset[0];
        ++seen;
      }
    }
    const uint32_t p0 = chunk * kChunkPoints;
    const uint32_t n = min(kChunkPoints, F.n_points - p0);
    uint8_t* side = const_cast<uint8_t*>(F.side) + (static_cast<size_t>(g) * F.n_points + p0) * 12;
    uint32_t win_lead = 255u, win_trail = 0u;  // GorillaState::reset(): no window yet
    uint64_t last = 0;                         // bits of the value before this group
    for (uint32_t base = 0; base < n; base += 32u) {  // warp-uniform
      const uint32_t i = base + lane;
      const bool valid = i < n;
      const uint64_t cur = valid ? load_u64(F.in + static_cast<size_t>(p0 + i) * plan.point_step + offset) : 0ull;
      uint64_t prev = __shfl_up_sync(0xffffffffu, cur, 1);
      if (lane == 0) prev = last;
      last = __shfl_sync(0xffffffffu, cur, 31);
      const bool first = (i == 0);
      const uint64_t x = cur ^ prev;
      const uint32_t lz = static_cast<uint32_t>(__clzll(static_cast<long long>(x)));
      const uint32_t tz = x ? static_cast<uint32_t>(__ffsll(static_cast<long long>(x)) - 1) : 0u;
      const bool uses_window = valid && !first && x != 0ull;
      // resolve the window every lane sees: lanes up to and including the first one that does not fit see the current
      // window; that lane's (min(lz, 31), tz) is the window of the lanes behind it, and so on
      uint32_t my_lead = win_lead, my_trail = win_trail;
      uint32_t cursor = 0;  // lanes below it are settled
      while (true) {        // warp-uniform trip count
        const bool fits = win_lead != 255u && lz >= win_lead && tz >= win_trail;
        const uint32_t misfit = __ballot_sync(0xffffffffu, uses_window && !fits && lane >= cursor);
        if (lane >= cursor) { my_lead = win_lead; my_trail = win_trail; }
        if (misfit == 0u) break;
        const int j = __ffs(misfit) - 1;
        win_lead = __shfl_sync(0xffffffffu, lz > 31u ? 31u : lz, j);
        win_trail = __shfl_sync(0xffffffffu, tz, j);
        cursor = static_cast<uint32_t>(j) + 1u;
      }
      if (valid) {
        GorillaState st;
        st.prev_bits = prev; st.leading = my_lead; st.trailing = my_trail; st.first = first;
        uint8_t rec[12];
        const uint32_t len = gorilla_encode(st, cur, rec);
        uint8_t* dst = side + static_cast<size_t>(i) * 12;
        for (uint32_t b = 0; b < len; ++b) dst[b] = rec[b];
        dst[11] = static_cast<uint8_t>(len);
      }
    }
  }
}

int launch_gorilla_prepass(const Plan& plan, const EncLaunch& L, cudaStream_t stream) {
  if (plan.n_gorilla == 0 || L.n_frames == 0) return 0;
  gorilla_prepass_kernel<<<L.n_frames, kGorillaThreads, 0, stream>>>(L);
  count_launch();
  return 1;
}

// Header + size for a batch that only holds empty frames (no tile exists to do it).
__global__ void empty_frames_kernel(const EncLaunch L) { handle_empty_frames(L); }

}  // namespace cldn
#include "cldn_encode_fast.cuh"
#include "cldn_encode_points.cuh"
namespace cldn {

// Points per tile for a plan: the largest I in {8,4,2,1} whose staging buffer fits comfortably.
uint32_t choose_tile_points(const Plan& plan) {
  if (encode_fast_applies(plan)) return encode_fast_tile_points();
  {
    PointsParams pp;
    if (encode_points_applies(plan, &pp)) return encode_points_tile(plan);
  }
  if (plan.floatn_only) return kThreads * 8;
  const size_t budget = 96 * 1024;
  for (int I = 8; I >= 1; I >>= 1) {
    if (static_cast<size_t>(kThreads) * I * plan.max_point_bytes + sizeof(Plan) + 64 <= budget) return kThreads * I;
  }
  return kThreads;
}

int launch_encode_regular(const Plan& plan, const EncLaunch& L, cudaStream_t stream) {
  if (L.n_tiles_total == 0) {
    empty_frames_kernel<<<1, kThreads, 0, stream>>>(L);
    count_launch();
    return 1;
  }
  const char* force = getenv("CLDN_B200_FORCE_GENERIC");
  bool muls_ok = true;  // the fast kernel relies on 0 < mul < inf (a NaN product then implies a NaN input)
  if (plan.floatn_only) {
    for (int k = 0; k < plan.ops[0].lanes; ++k) {
      const float m = plan.ops[0].enc_mul_f[k];
      if (!(m > 0.0f) || m > 3.0e38f) muls_ok = false;
    }
  }
  if (!(force && force[0] == '1') && encode_fast_applies(plan) && L.tile_points == encode_fast_tile_points()) {
    return launch_encode_fast(plan, L, stream);
  }
  {
    PointsParams pp;
    if (!(force && force[0] == '1') && !encode_fast_applies(plan) && encode_points_applies(plan, &pp) && L.tile_points == encode_points_tile(plan)) {
      return launch_encode_points(plan, L, pp, stream);
    }
  }
  if (plan.floatn_only && muls_ok && !(force && force[0] == '1')) {
    const RegOp& op = plan.ops[0];
    const bool packed4 = op.lanes == 4 && plan.point_step == 16 && op.offset[0] == 0 && op.offset[1] == 4 &&
                         op.offset[2] == 8 && op.offset[3] == 12;
    // LDG.128 needs 16-byte aligned frame bases (kEncAlignPerFrame: the kernel checks each frame's)
    const bool vec4 = packed4 && (L.flags & (kEncInputsAligned16 | kEncAlignPerFrame));
    if (L.tile_points != kThreads * 8) return -1;
    if (op.lanes == 4) return launch_floatn<4, 8, 3>(plan, L, vec4, stream);
    return launch_floatn<3, 8, 3>(plan, L, false, stream);
  }
  const EncLaunch& LL = L;
  const uint32_t I = LL.tile_points / kThreads;
  const size_t smem = ((sizeof(Plan) + 15) & ~size_t(15)) + static_cast<size_t>(LL.tile_points) * plan.max_point_bytes + 64;
#define CLDN_LAUNCH_GENERIC(II)                                                         \
  {                                                                                     \
    auto k = encode_generic_kernel<II>;                                                 \
    if (set_smem(k, smem) != cudaSuccess) return -1;                                    \
    k<<<LL.n_tiles_total, kThreads, smem, stream>>>(LL);                                \
  }
  switch (I) {
    case 8: CLDN_LAUNCH_GENERIC(8) break;
    case 4: CLDN_LAUNCH_GENERIC(4) break;
    case 2: CLDN_LAUNCH_GENERIC(2) break;
    default: CLDN_LAUNCH_GENERIC(1) break;
  }
#undef CLDN_LAUNCH_GENERIC
  count_launch();
  return 1;
}

}  // namespace cldn
