// Stage-1 DECODE kernels.
//
// Replaces PointcloudDecoder::decode's chunk walk (cloudini_lib/src/cloudini.cpp:645-664), DecodeV4Stage1Chunk
// (v4_codec.cpp:85-117), DecodeV5Stage1Chunk (v5_codec.cpp:984-1012) and decodeV5AdaptiveIntSection (:764-879).
//
// Work decomposition: one CTA per 32768-point chunk (chunks are independently decodable: every decoder resets at a
// chunk start). Inside a chunk the byte stream is processed in tiles of kDecTileBytes bytes:
//   pass A  (byte-parallel)  a byte with a clear MSB terminates a value (the 0x00 NaN marker too), so the number of
//           terminators before a byte is the index of the value it belongs to; each thread scans 16-byte vectors,
//           a CTA scan ranks the terminators, and the thread owning a terminator reassembles the varint behind it;
//   pass B  (point-parallel) values are regrouped per point / per field ("slot"), a segmented CTA scan (reset at NaN)
//           turns deltas into absolute quantised values, which are scaled and scattered into the strided output.
// Plans whose regular stream holds raw (Copy) fields cannot be ranked by terminators: all-Copy plans have a fixed
// point size and are trivially parallel; mixed plans fall back to a sequential per-chunk parser (one thread per chunk).
#include <stdio.h>

#include "cldn_device.cuh"
#include "cldn_kernels.h"

namespace cldn {

constexpr int kDecVecPerThread = 2;
constexpr int kDecTileBytes = kThreads * 16 * kDecVecPerThread;  // 8192
constexpr int kLookBehind = 16;

// One varint-coded value per point ("slot") of the regular stream, or the single slot of a DeltaVarint section.
enum SlotKind : uint8_t { SLOT_FLOATN = 0, SLOT_F32 = 1, SLOT_F64 = 2, SLOT_INT = 3 };
struct DecSlot {
  uint32_t offset;
  uint8_t kind;
  uint8_t size;  // bytes stored for SLOT_INT
  uint8_t pad_[2];
  float mul_f;
  double mul_d;
};

// ------------------------------------------------------------------------------------------------------------------
// Chunk table: cloudini.cpp:645-664. One thread per frame walks the u32 prefixes (a dependent chain by construction).
__global__ void walk_chunks_kernel(const DecLaunch L) {
  const uint32_t f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= L.n_frames) return;
  const DecFrame F = L.frames[f];
  uint64_t pos = 0;
  for (uint32_t c = 0; c < F.n_chunks; ++c) {
    uint64_t body = 0;
    uint32_t size = 0;
    if (pos >= F.payload_bytes) {
      report_frame_error(L, f, DEV_ERR_CHUNK_COUNT);  // "Encoded data ended before all declared points were decoded"
    } else if (F.payload_bytes - pos < 4) {
      report_frame_error(L, f, DEV_ERR_TRUNCATED);    // decode<uint32_t>: not enough input data
      pos = F.payload_bytes;
    } else {
      size = load_u32(F.payload + pos);
      pos += 4;
      if (size > F.payload_bytes - pos) {
        report_frame_error(L, f, DEV_ERR_CHUNK_SIZE);  // "Invalid chunk size found while decoding"
        size = 0;
        pos = F.payload_bytes;
      }
      body = pos;
      pos += size;
    }
    L.chunk_offsets[F.chunk_begin + c] = body;
    L.chunk_sizes[F.chunk_begin + c] = size;
  }
  if (pos < F.payload_bytes) report_frame_error(L, f, DEV_ERR_CHUNK_COUNT);  // "more chunks than declared points"
}

// ------------------------------------------------------------------------------------------------------------------
// Shared-memory working set of the chunk decoder.
struct DecShared {
  uint32_t scan[kThreads / 32 + 1];
  uint32_t values_done;      // values of the current stream decoded so far
  uint32_t stream_end;       // byte offset (inside the chunk body) one past the stream's last value
  uint32_t stop;             // stream finished (or failed)
  uint32_t pad_;
  long long carry[kMaxOps];  // per slot: absolute quantised value of the last decoded point
  long long seg_sum[kThreads / 32][4];
  uint32_t seg_rst[kThreads / 32];
};

// Segmented-sum element for NS slots processed together: sum[j] is the sum of deltas since the last reset (NaN) of
// slot j, bit j of rst tells whether a reset happened inside the range.
// Wrapping add (FieldDecoderFloatN_Lossy adds in int32 with wrap-around, field_decoder.cpp:68).
__device__ __forceinline__ int32_t wadd(int32_t a, int32_t b) { return static_cast<int32_t>(static_cast<uint32_t>(a) + static_cast<uint32_t>(b)); }
__device__ __forceinline__ long long wadd(long long a, long long b) {
  return static_cast<long long>(static_cast<unsigned long long>(a) + static_cast<unsigned long long>(b));
}

template <typename AccT, int NS>
struct Seg {
  AccT sum[NS];
  uint32_t rst;
};
template <typename AccT, int NS>
__device__ __forceinline__ Seg<AccT, NS> seg_combine(const Seg<AccT, NS>& a, const Seg<AccT, NS>& b) {  // a then b
  Seg<AccT, NS> r;
#pragma unroll
  for (int j = 0; j < NS; ++j) r.sum[j] = ((b.rst >> j) & 1u) ? b.sum[j] : wadd(a.sum[j], b.sum[j]);
  r.rst = a.rst | b.rst;
  return r;
}
template <typename AccT, int NS>
__device__ __forceinline__ Seg<AccT, NS> seg_shfl_up(const Seg<AccT, NS>& a, int d) {
  Seg<AccT, NS> r;
#pragma unroll
  for (int j = 0; j < NS; ++j) r.sum[j] = __shfl_up_sync(0xffffffffu, a.sum[j], d);
  r.rst = __shfl_up_sync(0xffffffffu, a.rst, d);
  return r;
}

// CTA-wide EXCLUSIVE segmented scan. smem: per-warp aggregates. Also returns the CTA total in *total.
template <typename AccT, int NS>
__device__ __forceinline__ Seg<AccT, NS> block_seg_exclusive(const Seg<AccT, NS>& mine, long long (*w_sum)[4],
                                                             uint32_t* w_rst, Seg<AccT, NS>* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  Seg<AccT, NS> inc = mine;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const Seg<AccT, NS> up = seg_shfl_up<AccT, NS>(inc, d);
    if (lane >= d) inc = seg_combine<AccT, NS>(up, inc);
  }
  if (lane == 31) {
#pragma unroll
    for (int j = 0; j < NS; ++j) w_sum[warp][j] = static_cast<long long>(inc.sum[j]);
    w_rst[warp] = inc.rst;
  }
  __syncthreads();
  Seg<AccT, NS> prefix;  // combination of all earlier warps
#pragma unroll
  for (int j = 0; j < NS; ++j) prefix.sum[j] = 0;
  prefix.rst = 0;
  Seg<AccT, NS> tot = prefix;
#pragma unroll
  for (int w = 0; w < kThreads / 32; ++w) {
    Seg<AccT, NS> x;
#pragma unroll
    for (int j = 0; j < NS; ++j) x.sum[j] = static_cast<AccT>(w_sum[w][j]);
    x.rst = w_rst[w];
    if (w < warp) prefix = seg_combine<AccT, NS>(prefix, x);
    tot = seg_combine<AccT, NS>(tot, x);
  }
  *total = tot;
  // exclusive = prefix (+) inclusive-of-previous-lane
  Seg<AccT, NS> prev_lane = seg_shfl_up<AccT, NS>(inc, 1);
  Seg<AccT, NS> res = prefix;
  if (lane > 0) res = seg_combine<AccT, NS>(prefix, prev_lane);
  __syncthreads();  // w_sum / w_rst may be reused by the caller
  return res;
}

// Stores one decoded value of a slot.
template <typename AccT>
__device__ __forceinline__ void store_slot_value(uint8_t* point, const DecSlot& s, AccT value, bool nan) {
  if (s.offset == CLDN_SKIP_STORE_OFFSET) return;  // kDecodeButSkipStore (basic_types.hpp:71)
  uint8_t* dst = point + s.offset;
  switch (s.kind) {
    case SLOT_FLOATN:  // field_decoder.cpp:62-70
    case SLOT_F32: {   // field_decoder.hpp:331-353
      float f;
      if (nan) f = __uint_as_float(0x7FC00000u);  // std::numeric_limits<float>::quiet_NaN()
      else if (s.kind == SLOT_FLOATN) f = __fmul_rn(__int2float_rn(static_cast<int32_t>(value)), s.mul_f);
      else f = __fmul_rn(__ll2float_rn(static_cast<long long>(value)), s.mul_f);
      store_u32(dst, __float_as_uint(f));
    } break;
    case SLOT_F64: {
      double d;
      if (nan) d = __longlong_as_double(0x7FF8000000000000ll);
      else d = __dmul_rn(__ll2double_rn(static_cast<long long>(value)), s.mul_d);
      store_u64(dst, static_cast<uint64_t>(__double_as_longlong(d)));
    } break;
    default:  // SLOT_INT: memcpy(&value, sizeof(IntType)) (field_decoder.hpp:93-95)
      store_low_bytes(dst, static_cast<uint64_t>(static_cast<long long>(value)), s.size);
      break;
  }
}

// ------------------------------------------------------------------------------------------------------------------
// Decodes a stream of `n_points * K` varint-coded values (K slots per point, interleaved) that starts at `src`
// (at most `avail` readable bytes) and scatters them to out + point * step + slot.offset.
// KT > 0: compile-time K with 32-bit accumulators (FloatN: wrapping int32 adds, field_decoder.cpp:68);
// KT == 0: run-time K, 64-bit accumulators, one slot at a time.
// Returns (to all threads) the number of bytes consumed, or 0xFFFFFFFF after reporting an error.
template <int KT>
__device__ uint32_t decode_varint_stream(const uint8_t* __restrict__ src, uint32_t avail, uint32_t n_points, int K_rt,
                                         const DecSlot* __restrict__ slots, uint8_t* __restrict__ out, uint32_t step,
                                         DecShared& sh, uint8_t* tile_bytes, uint8_t* vals_raw, uint32_t* nanbits,
                                         uint32_t* err) {
  using AccT = typename std::conditional<(KT > 0), int32_t, long long>::type;
  const int K = KT > 0 ? KT : K_rt;
  AccT* vals = reinterpret_cast<AccT*>(vals_raw);
  const uint32_t V = n_points * static_cast<uint32_t>(K);
  if (threadIdx.x == 0) {
    sh.values_done = 0;
    sh.stream_end = 0;
    sh.stop = (V == 0) ? 1u : 0u;
  }
  for (int j = threadIdx.x; j < K; j += blockDim.x) sh.carry[j] = 0;
  __syncthreads();
  if (V == 0) return 0;

  // tiles are aligned to 16 bytes in global memory so that every thread issues aligned 16-byte loads
  const uintptr_t src_addr = reinterpret_cast<uintptr_t>(src);
  const uint32_t mis = static_cast<uint32_t>(src_addr & 15u);
  const uint8_t* aligned = src - mis;  // tile k covers stream bytes [k*TB - mis, (k+1)*TB - mis)

  for (uint32_t tile = 0;; ++tile) {
    const int64_t tile_b0 = static_cast<int64_t>(tile) * kDecTileBytes - mis;  // stream offset of the tile's first byte
    if (tile_b0 >= static_cast<int64_t>(avail)) {
      // ran out of bytes before all values were seen: "Truncated encoded data" (v4_codec.cpp:102-104)
      if (threadIdx.x == 0) report_error(err, DEV_ERR_TRUNCATED);
      return 0xFFFFFFFFu;
    }
    // ---- load: tile_bytes[kLookBehind + i] = stream byte (tile_b0 + i); bytes outside [0, avail) read as 0x80 ----
#pragma unroll
    for (int vv = 0; vv < kDecVecPerThread; ++vv) {
      const uint32_t i = (vv * kThreads + threadIdx.x) * 16u;
      const int64_t b = tile_b0 + i;
      uint4 q = make_uint4(0x80808080u, 0x80808080u, 0x80808080u, 0x80808080u);
      if (b >= 0 && b + 16 <= static_cast<int64_t>(avail)) {
        q = *reinterpret_cast<const uint4*>(aligned + static_cast<size_t>(tile) * kDecTileBytes + i);
      } else if (b + 16 > 0 && b < static_cast<int64_t>(avail)) {  // stream edge: only touch bytes inside the stream
        uint32_t w[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
        for (int k = 0; k < 16; ++k) {
          const int64_t bb = b + k;
          if (bb >= 0 && bb < static_cast<int64_t>(avail)) {
            w[k >> 2] = (w[k >> 2] & ~(0xFFu << (8 * (k & 3)))) | (static_cast<uint32_t>(src[bb]) << (8 * (k & 3)));
          }
        }
        q = make_uint4(w[0], w[1], w[2], w[3]);
      }
      *reinterpret_cast<uint4*>(tile_bytes + kLookBehind + i) = q;
    }
    if (threadIdx.x < 4) {  // look-behind: the 16 stream bytes before the tile (0x80 before the stream start)
      uint32_t w = 0x80808080u;
      const int64_t b = tile_b0 - 16 + 4 * static_cast<int64_t>(threadIdx.x);
      if (tile > 0) {
        w = *reinterpret_cast<const uint32_t*>(aligned + static_cast<size_t>(tile) * kDecTileBytes - 16 + 4 * threadIdx.x);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          if (b + k < 0) w = (w & ~(0xFFu << (8 * k))) | (0x80u << (8 * k));
        }
      }
      // a terminator must separate the look-behind from the stream start: byte (-1) is treated as a terminator
      reinterpret_cast<uint32_t*>(tile_bytes)[threadIdx.x] = w;
    }
    __syncthreads();

    // ---- pass A: rank terminators ----
    uint32_t tmask[kDecVecPerThread];
    uint32_t cnt = 0;
#pragma unroll
    for (int vv = 0; vv < kDecVecPerThread; ++vv) {
      const uint32_t i = (vv * kThreads + threadIdx.x) * 16u;
      const uint4 q = *reinterpret_cast<const uint4*>(tile_bytes + kLookBehind + i);
      const uint32_t w[4] = {~q.x & 0x80808080u, ~q.y & 0x80808080u, ~q.z & 0x80808080u, ~q.w & 0x80808080u};
      uint32_t m = 0;
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        // gather bits 7,15,23,31 into 4 consecutive bits
        const uint32_t x = w[k];
        m |= (((x >> 7) & 1u) | ((x >> 14) & 2u) | ((x >> 21) & 4u) | ((x >> 28) & 8u)) << (4 * k);
      }
      tmask[vv] = m;
      cnt += __popc(m);
    }
    // thread order must follow byte order: vector vv of thread t sits at (vv*kThreads + t)*16, so scan per vv
    uint32_t vbase[kDecVecPerThread];
    uint32_t tile_values = 0;
#pragma unroll
    for (int vv = 0; vv < kDecVecPerThread; ++vv) {
      uint32_t tot;
      const uint32_t ex = block_exclusive_scan(__popc(tmask[vv]), sh.scan, &tot);
      vbase[vv] = tile_values + ex;
      tile_values += tot;
      __syncthreads();
    }
    const uint32_t done = sh.values_done;
    const uint32_t want = V - done;                       // values still missing
    const uint32_t take = tile_values < want ? tile_values : want;

    // ---- pass A2: reassemble the varint behind every terminator and park it at its tile-local value index ----
    for (uint32_t i = threadIdx.x; i < (take + 31u) / 32u; i += blockDim.x) nanbits[i] = 0;
    __syncthreads();
#pragma unroll
    for (int vv = 0; vv < kDecVecPerThread; ++vv) {
      uint32_t m = tmask[vv];
      uint32_t vi = vbase[vv];
      const uint32_t i0 = (vv * kThreads + threadIdx.x) * 16u;
      while (m && vi < take) {
        const int j = __ffs(m) - 1;
        m &= m - 1;
        const uint8_t* endp = tile_bytes + kLookBehind + i0 + j;  // terminator byte
        // walk back over continuation bytes (at most 9; byte -1 of the stream reads as a terminator-less 0x80 guard
        // only inside the look-behind, where the stream start is protected by the explicit bound below)
        const int64_t spos = tile_b0 + i0 + j;  // stream offset of the terminator
        int nb = 1;
        while (nb < 11 && spos - nb >= 0 && (endp[-nb] & 0x80u)) ++nb;
        bool bad = false;
        unsigned long long u = 0;
        if (nb > 10) { bad = true; report_error(err, DEV_ERR_VARINT_OVERFLOW); }
        else {
#pragma unroll 1
          for (int k = 0; k < nb; ++k) {
            const unsigned long long payload = endp[-(nb - 1) + k] & 0x7Fu;
            if (k == 9 && payload > 1) { bad = true; report_error(err, DEV_ERR_VARINT_OVERFLOW); }  // encoding_utils.hpp:127-129
            u |= payload << (7 * k);
          }
        }
        bool nan = false;
        AccT delta = 0;
        if (!bad) {
          if (u == 0) {
            // single 0x00 = NaN marker for float slots; anything else is "unexpected NaN marker"
            const DecSlot& s = slots[(done + vi) % static_cast<uint32_t>(K)];
            if (nb == 1 && s.kind != SLOT_INT) nan = true;
            else report_error(err, DEV_ERR_NAN_MARKER);
          } else {
            delta = static_cast<AccT>(unzigzag(u - 1ull));
          }
        }
        vals[vi] = delta;
        if (nan) atomicOr(&nanbits[vi >> 5], 1u << (vi & 31));
        if (done + vi + 1 == V) sh.stream_end = static_cast<uint32_t>(spos + 1);
        ++vi;
      }
    }
    __syncthreads();

    // ---- pass B: per point / per slot prefix sums and scatter ----
    if (take > 0) {
      const uint32_t first_pt = done / K;
      const uint32_t last_pt = (done + take - 1) / K;
      const uint32_t npts = last_pt - first_pt + 1;
      const uint32_t per_thread = (npts + kThreads - 1) / kThreads;
      const uint32_t my0 = first_pt + threadIdx.x * per_thread;
      uint32_t my1 = my0 + per_thread;
      if (my1 > last_pt + 1) my1 = last_pt + 1;
      if (KT > 0) {
        constexpr int NS = KT > 0 ? KT : 1;
        Seg<AccT, NS> mine;
#pragma unroll
        for (int j = 0; j < NS; ++j) mine.sum[j] = 0;
        mine.rst = 0;
        for (uint32_t p = my0; p < my1; ++p) {
#pragma unroll
          for (int j = 0; j < NS; ++j) {
            const int64_t lv = static_cast<int64_t>(p) * NS + j - done;
            if (lv >= 0 && lv < static_cast<int64_t>(take)) {
              if ((nanbits[lv >> 5] >> (lv & 31)) & 1u) { mine.sum[j] = 0; mine.rst |= 1u << j; }
              else mine.sum[j] = wadd(mine.sum[j], vals[lv]);
            }
          }
        }
        Seg<AccT, NS> total;
        Seg<AccT, NS> ex = block_seg_exclusive<AccT, NS>(mine, sh.seg_sum, sh.seg_rst, &total);
        AccT cur[NS];
#pragma unroll
        for (int j = 0; j < NS; ++j) {
          cur[j] = ((ex.rst >> j) & 1u) ? ex.sum[j] : wadd(static_cast<AccT>(sh.carry[j]), ex.sum[j]);
        }
        for (uint32_t p = my0; p < my1; ++p) {
          uint8_t* point = out + static_cast<size_t>(p) * step;
#pragma unroll
          for (int j = 0; j < NS; ++j) {
            const int64_t lv = static_cast<int64_t>(p) * NS + j - done;
            if (lv >= 0 && lv < static_cast<int64_t>(take)) {
              const bool nan = (nanbits[lv >> 5] >> (lv & 31)) & 1u;
              if (nan) cur[j] = 0; else cur[j] = wadd(cur[j], vals[lv]);
              store_slot_value<AccT>(point, slots[j], cur[j], nan);
            }
          }
        }
        __syncthreads();
        if (threadIdx.x == 0) {
#pragma unroll
          for (int j = 0; j < NS; ++j) {
            sh.carry[j] = ((total.rst >> j) & 1u) ? static_cast<long long>(total.sum[j])
                                                  : static_cast<long long>(wadd(static_cast<AccT>(sh.carry[j]), total.sum[j]));
          }
        }
      } else {
        // run-time K: one slot at a time with 64-bit accumulators
        for (int j = 0; j < K; ++j) {
          Seg<long long, 1> mine;
          mine.sum[0] = 0;
          mine.rst = 0;
          for (uint32_t p = my0; p < my1; ++p) {
            const int64_t lv = static_cast<int64_t>(p) * K + j - done;
            if (lv >= 0 && lv < static_cast<int64_t>(take)) {
              if ((nanbits[lv >> 5] >> (lv & 31)) & 1u) { mine.sum[0] = 0; mine.rst = 1u; }
              else mine.sum[0] = wadd(mine.sum[0], static_cast<long long>(vals[lv]));
            }
          }
          Seg<long long, 1> total;
          Seg<long long, 1> ex = block_seg_exclusive<long long, 1>(mine, sh.seg_sum, sh.seg_rst, &total);
          long long cur = ex.rst ? ex.sum[0] : wadd(sh.carry[j], ex.sum[0]);
          for (uint32_t p = my0; p < my1; ++p) {
            const int64_t lv = static_cast<int64_t>(p) * K + j - done;
            if (lv >= 0 && lv < static_cast<int64_t>(take)) {
              const bool nan = (nanbits[lv >> 5] >> (lv & 31)) & 1u;
              if (nan) cur = 0; else cur = wadd(cur, static_cast<long long>(vals[lv]));
              store_slot_value<long long>(out + static_cast<size_t>(p) * step, slots[j], cur, nan);
            }
          }
          __syncthreads();
          if (threadIdx.x == 0) sh.carry[j] = total.rst ? total.sum[0] : wadd(sh.carry[j], total.sum[0]);
        }
      }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      sh.values_done = done + take;
      if (done + take == V) sh.stop = 1;
    }
    __syncthreads();
    if (sh.stop) break;
  }
  return sh.stream_end;
}

// ------------------------------------------------------------------------------------------------------------------
// V5 adaptive integer sections (decodeV5AdaptiveIntSection, v5_codec.cpp:764-879). Executed by the whole CTA.
__device__ __forceinline__ uint32_t bits_for_palette(uint32_t count) {  // bitsForPaletteIndex, v5_codec.cpp:196-207
  if (count <= 1) return 0;
  return 32u - __clz(count - 1u);
}

// plain LEB128 (readUVarint, v5_codec.cpp:176-194). Returns bytes consumed, 0 on error.
__device__ __forceinline__ uint32_t read_uvarint(const uint8_t* p, uint32_t avail, unsigned long long* out, uint32_t* err) {
  unsigned long long v = 0;
  uint32_t shift = 0, n = 0;
  while (true) {
    if (n >= avail) { report_error(err, DEV_ERR_TRUNCATED); return 0; }
    const uint8_t b = p[n++];
    v |= static_cast<unsigned long long>(b & 0x7Fu) << shift;
    if (!(b & 0x80u)) break;
    shift += 7;
    if (shift >= 64) { report_error(err, DEV_ERR_VARINT_OVERFLOW); return 0; }
  }
  *out = v;
  return n;
}
// zigzag varint (decodeVarint, encoding_utils.hpp:98-148). Returns bytes consumed, 0 on error.
__device__ __forceinline__ uint32_t read_varint(const uint8_t* p, uint32_t avail, long long* out, uint32_t* err) {
  unsigned long long v = 0;
  uint32_t n = 0;
  while (true) {
    if (n >= avail) { report_error(err, n == 0 ? DEV_ERR_TRUNCATED : DEV_ERR_TRUNCATED); return 0; }
    const uint8_t b = p[n];
    const unsigned long long payload = b & 0x7Fu;
    if (n >= 10 || (n == 9 && payload > 1)) { report_error(err, DEV_ERR_VARINT_OVERFLOW); return 0; }
    v |= payload << (7 * n);
    ++n;
    if (!(b & 0x80u)) break;
  }
  if (v == 0) { report_error(err, DEV_ERR_NAN_MARKER); return 0; }
  *out = unzigzag(v - 1ull);
  return n;
}

constexpr int kRunBatch = 512;
struct RunBatch {
  unsigned long long value[kRunBatch];  // Rle: raw value; DeltaRle: value BEFORE the run's first point
  long long diff[kRunBatch];            // DeltaRle only
  uint32_t start[kRunBatch + 1];        // chunk-local index of the run's first point
  uint32_t n;
  uint32_t pos;       // parse position (bytes into the section) after this batch
  uint32_t runs_left;
  unsigned long long prev;  // DeltaRle: running value in front of the next batch
};

// ---- parallel parse of a run table (Rle: raw value + uvarint length, DeltaRle: varint delta + uvarint length) -----------
// The table is a chain of variable-length records, so the reference walks it with one dependent parse per run. Here the
// next kRunPar * 20 bytes are staged in shared memory, every byte position computes where the following record would
// start IF a record started there (one or two terminator bits, plus the raw bytes of an Rle value), ONE thread follows
// that table from the batch's first byte (one shared-memory load per run) and then every thread decodes one run with
// the careful readers; run starts and DeltaRle values come from two CTA scans.
constexpr uint32_t kRunPar = kThreads;        // runs per iteration (one per thread)
constexpr uint32_t kRunRecMax = 20;           // a record is at most 10 + 10 bytes (8 + 10 for Rle)
constexpr uint32_t kRunStage = 5632;          // >= kRunPar * kRunRecMax, multiple of 32
constexpr uint32_t kRunNone = 0xFFFFu;

__device__ __forceinline__ uint32_t run_skip_varint(const uint32_t* tb, uint32_t p, uint32_t S) {
  if (p >= S) return kRunNone;
  const uint32_t w = p >> 5, sh = p & 31u;
  const uint32_t lo = __funnelshift_r(tb[w], tb[w + 1], sh);  // 32 terminator bits from p on: a varint has at most 10 bytes
  if (lo == 0u) return kRunNone;
  return p + static_cast<uint32_t>(__ffs(static_cast<int>(lo)));
}
__device__ __forceinline__ unsigned long long block_exclusive_sum_u64(unsigned long long v, long long (*scratch)[4], unsigned long long* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  unsigned long long inc = v;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const unsigned long long t = __shfl_up_sync(0xffffffffu, inc, d);
    if (lane >= d) inc += t;
  }
  if (lane == 31) scratch[warp][0] = static_cast<long long>(inc);
  __syncthreads();
  unsigned long long before = 0, all = 0;
#pragma unroll
  for (int w = 0; w < kThreads / 32; ++w) {
    const unsigned long long x = static_cast<unsigned long long>(scratch[w][0]);
    if (w < warp) before += x;
    all += x;
  }
  *total = all;
  __syncthreads();
  return before + inc - v;
}

// Decodes one section starting at src (avail bytes). Returns bytes consumed or 0xFFFFFFFF on error.
template <int KT>
__device__ uint32_t decode_section(const uint8_t* __restrict__ src, uint32_t avail, uint32_t n_points,
                                   const SectionField& sf, uint8_t* __restrict__ out, uint32_t step, DecShared& sh,
                                   uint8_t* tile_bytes, uint8_t* vals_raw, uint32_t* nanbits, RunBatch& rb,
                                   DecSlot* sec_slot, uint32_t* err) {
  if (avail < 1) {
    if (threadIdx.x == 0) report_error(err, DEV_ERR_BAD_MODE);  // "missing mode byte"
    return 0xFFFFFFFFu;
  }
  const uint8_t mode = src[0];
  if (mode > 3) {
    if (threadIdx.x == 0) report_error(err, DEV_ERR_BAD_MODE);
    return 0xFFFFFFFFu;
  }
  const uint32_t bpv = sf.bpv;
  if (mode == 0) {  // DeltaVarint: n_points zigzag varints, prev = 0
    if (threadIdx.x == 0) {
      sec_slot->offset = sf.offset;
      sec_slot->kind = SLOT_INT;
      sec_slot->size = sf.bpv;
    }
    __syncthreads();
    const uint32_t used = decode_varint_stream<0>(src + 1, avail - 1, n_points, 1, sec_slot, out, step, sh, tile_bytes,
                                                  vals_raw, nanbits, err);
    return used == 0xFFFFFFFFu ? used : used + 1;
  }
  if (mode == 1) {  // Palette
    if (avail < 3) {
      if (threadIdx.x == 0) report_error(err, DEV_ERR_TRUNCATED);
      return 0xFFFFFFFFu;
    }
    const uint32_t count = load_u16(src + 1);
    if (count == 0) {
      if (threadIdx.x == 0) report_error(err, DEV_ERR_PALETTE);  // "empty palette"
      return 0xFFFFFFFFu;
    }
    const uint64_t pal_bytes = static_cast<uint64_t>(count) * bpv;
    const uint32_t bits = bits_for_palette(count);
    const uint64_t idx_bytes = (static_cast<uint64_t>(bits) * n_points + 7u) / 8u;
    if (3ull + pal_bytes + idx_bytes > avail) {
      if (threadIdx.x == 0) report_error(err, DEV_ERR_PALETTE);  // truncated palette / indexes
      return 0xFFFFFFFFu;
    }
    const uint8_t* pal = src + 3;
    const uint8_t* idx = pal + pal_bytes;
    // 8 indexes are exactly `bits` bytes: a thread unpacks the unit [8 u, 8 u + 8) from bytes [u * bits, (u + 1) * bits) --
    // its loads are independent of each other (the per-value version chained three byte loads per point)
    const uint32_t units = (n_points + 7u) / 8u;
    const bool store = sf.offset != CLDN_SKIP_STORE_OFFSET;
    for (uint32_t u = threadIdx.x; u < units; u += blockDim.x) {
      unsigned long long lo = 0, hi = 0;
      if (bits) {
        const uint32_t b0 = u * bits;
        const uint32_t nb = static_cast<uint32_t>(idx_bytes - b0 < bits ? idx_bytes - b0 : bits);
        const uint8_t* pb = idx + b0;
#pragma unroll 4
        for (uint32_t b = 0; b < nb; ++b) {
          const unsigned long long byte = pb[b];
          if (b < 8u) lo |= byte << (8u * b); else hi |= byte << (8u * (b - 8u));
        }
      }
      const uint32_t mask = (1u << bits) - 1u;   // bits <= 16
#pragma unroll
      for (uint32_t j = 0; j < 8u; ++j) {
        const uint32_t i = 8u * u + j;
        if (i >= n_points) break;
        const uint32_t sh_ = j * bits;
        uint32_t k;
        if (sh_ >= 64u) k = static_cast<uint32_t>(hi >> (sh_ - 64u));
        else k = static_cast<uint32_t>(lo >> sh_) | (sh_ + bits > 64u ? static_cast<uint32_t>(hi << (64u - sh_)) : 0u);
        k &= mask;
        if (k >= count) { report_error(err, DEV_ERR_PALETTE); continue; }  // "palette index out of range"
        // kDecodeButSkipStore: the reference's section reader stores at `offset` unconditionally (v5_codec.cpp:787-789),
        // i.e. 4 GB behind the buffer; here the value is validated and dropped like the regular decoders do
        if (store) store_low_bytes(out + static_cast<size_t>(i) * step + sf.offset, load_raw_bits(pal + static_cast<size_t>(k) * bpv, bpv), bpv);
      }
    }
    return static_cast<uint32_t>(3ull + pal_bytes + idx_bytes);
  }
  // Rle (2) / DeltaRle (3): a run table is parsed in batches of kRunPar records, then expanded by all threads.
  if (avail < 5) {
    if (threadIdx.x == 0) report_error(err, DEV_ERR_TRUNCATED);
    return 0xFFFFFFFFu;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    rb.runs_left = load_u32(src + 1);
    rb.pos = 5;
    rb.start[0] = 0;
    rb.value[0] = 0;
  }
  __syncthreads();
  uint32_t out_index = 0;          // points produced so far (uniform)
  if (threadIdx.x == 0) rb.prev = 0;
  uint8_t* sb = vals_raw;                                                        // staged bytes of the run table
  uint32_t* tb = reinterpret_cast<uint32_t*>(sb + kRunStage + 32);              // terminator bits
  uint16_t* nx = reinterpret_cast<uint16_t*>(tb + kRunStage / 32 + 4);          // next record start per byte position
  uint16_t* rs = nx + kRunStage;                                                 // record starts of this batch [kRunPar + 2]
  uint32_t* hmask = reinterpret_cast<uint32_t*>(nx);                             // once the records are parsed: run-start marks of the
  uint32_t* hpre = hmask + kChunkPoints / 32;                                    //   batch's points + their word-prefix counts
  static_assert(2 * (kChunkPoints / 32) * 4 <= kRunStage * 2, "marks and prefix counts alias the next-record table");
  while (true) {
    const uint32_t pos = rb.pos;
    const uint32_t want = rb.runs_left < kRunPar ? rb.runs_left : kRunPar;
    const uint32_t rest = avail - pos;
    const uint32_t S = rest < kRunStage ? rest : kRunStage;
    const bool more_behind = rest > kRunStage;
    for (uint32_t i = threadIdx.x; i < kRunStage + 32; i += blockDim.x) sb[i] = i < S ? src[pos + i] : 0x80u;
    __syncthreads();
    for (uint32_t w = threadIdx.x; w < kRunStage / 32 + 4; w += blockDim.x) {
      uint32_t m = 0;
      if (w * 32u < S) {
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          const uint32_t t = ~*reinterpret_cast<const uint32_t*>(sb + w * 32u + 4 * k) & 0x80808080u;
          m |= (((t >> 7) & 1u) | ((t >> 14) & 2u) | ((t >> 21) & 4u) | ((t >> 28) & 8u)) << (4 * k);
        }
      }
      tb[w] = m;  // bytes behind S read as 0x80: no terminator there
    }
    __syncthreads();
    if (mode == 3) {
      // a DeltaRle record is two varints: record r ends at terminator 2 r + 1 of the staged bytes. Word-prefix counts
      // of the terminator bits (one CTA scan) rank every terminator; the odd-ranked ones name the next record's start.
      uint32_t* tpre = reinterpret_cast<uint32_t*>(nx);                 // [kRunStage / 32 + 4] terminators in front of word w
      const uint32_t nw = kRunStage / 32 + 4;
      uint32_t terms_total;
      {
        const uint32_t w = threadIdx.x;
        const uint32_t c = w < nw ? __popc(tb[w]) : 0u;
        static_assert(kRunStage / 32 + 4 <= kThreads, "one terminator word per thread");
        const uint32_t before = block_exclusive_scan_n<kThreads>(c, sh.scan, &terms_total);
        if (w < nw) tpre[w] = before;
      }
      __syncthreads();
      const uint32_t complete = terms_total >> 1;                        // records that end inside the staged bytes
      // records taken this batch; a table that ends (or is damaged) inside the staged bytes hands its first incomplete
      // record to the careful readers below, which say what is wrong with it
      uint32_t n = complete < want ? complete : want;
      if (n < want && (!more_behind || n == 0u)) n += 1u;
      for (uint32_t b = threadIdx.x; b < S; b += blockDim.x) {
        const uint32_t w = b >> 5, k = b & 31u;
        const uint32_t word = tb[w];
        if ((word >> k) & 1u) {
          const uint32_t rank = tpre[w] + __popc(word & ((1u << k) - 1u));
          if ((rank & 1u) && (rank >> 1) + 1u <= n) rs[(rank >> 1) + 1u] = static_cast<uint16_t>(b + 1u);
        }
      }
      if (threadIdx.x == 0) {
        rs[0] = 0;
        if (n > complete) rs[n] = static_cast<uint16_t>(kRunNone);
        rb.n = n;
      }
      __syncthreads();
    } else {
      for (uint32_t b = threadIdx.x; b < S; b += blockDim.x) {
        uint32_t p = b + bpv;
        if (p > S) p = kRunNone;
        if (p != kRunNone) p = run_skip_varint(tb, p, S);
        nx[b] = static_cast<uint16_t>(p);
      }
      __syncthreads();
      if (threadIdx.x == 0) {
        uint32_t n = 0, p = 0;
        while (n < want) {
          if (n > 0 && more_behind && p + kRunRecMax > S) break;  // the record may continue behind the staged bytes: next batch
          rs[n++] = static_cast<uint16_t>(p);
          p = p < S ? nx[p] : kRunNone;  // a record that would start behind the last byte is a truncated table
          if (p == kRunNone) break;      // truncated / malformed record: the careful readers below say what is wrong with it
        }
        rs[n] = static_cast<uint16_t>(p);
        rb.n = n;
      }
      __syncthreads();
    }
    {
      const uint32_t n = rb.n;
      const uint32_t r = threadIdx.x;
      bool bad = false;
      unsigned long long run_len = 0, raw = 0;
      long long diff = 0;
      uint32_t q = 0;
      if (r < n) {
        q = rs[r];
        if (mode == 2) {
          if (rest - q < bpv) { report_error(err, DEV_ERR_RLE); bad = true; }  // "truncated RLE value"
          else { raw = load_raw_bits(sb + q, bpv); q += bpv; }
        } else {
          const uint32_t lim = (rest - q) < (S - q) ? (rest - q) : (S - q);
          const uint32_t c = read_varint(sb + q, lim, &diff, err);
          if (!c) bad = true;
          q += c;
        }
        if (!bad) {
          const uint32_t lim = (rest - q) < (S - q) ? (rest - q) : (S - q);
          const uint32_t c2 = read_uvarint(sb + q, lim, &run_len, err);
          if (!c2) bad = true;
          q += c2;
        }
      }
      if (__syncthreads_or(bad ? 1 : 0)) return 0xFFFFFFFFu;
      // run starts: exclusive sum of the lengths (64-bit: a forged length must not wrap)
      unsigned long long len_total, prod_total;
      const unsigned long long before = block_exclusive_sum_u64(r < n ? run_len : 0ull, sh.seg_sum, &len_total);
      const unsigned long long oi = static_cast<unsigned long long>(out_index) + before;
      if (r < n && (oi > n_points || run_len > static_cast<unsigned long long>(n_points) - oi)) {  // "run exceeds point count"
        report_error(err, DEV_ERR_RLE);
        bad = true;
      }
      // DeltaRle: the value in front of run r is prev + sum over earlier runs of diff * length (wrapping like the reference)
      const unsigned long long prod = (r < n && mode == 3) ? static_cast<unsigned long long>(diff) * run_len : 0ull;
      const unsigned long long pbefore = block_exclusive_sum_u64(prod, sh.seg_sum, &prod_total);
      if (__syncthreads_or(bad ? 1 : 0)) return 0xFFFFFFFFu;
      // Which run does point i belong to? One bit per point of the batch marks the run starts; a point's run is the
      // number of marks up to it (word-prefix counts + one popc) -- two shared-memory loads instead of a binary search
      // over the starts (8 dependent loads; 45 % of the kernel's instructions on a 64-ring `ring` field). Empty runs
      // set no mark and get no slot.
      const bool ne = r < n && run_len > 0ull;
      uint32_t ne_total;
      const uint32_t slot = block_exclusive_scan_n<kThreads>(ne ? 1u : 0u, sh.scan, &ne_total);
      const uint32_t batch_pts = static_cast<uint32_t>(len_total);       // validated above: <= n_points - out_index
      const uint32_t mw = (batch_pts + 31u) / 32u;
      for (uint32_t w = threadIdx.x; w < mw; w += blockDim.x) hmask[w] = 0u;
      __syncthreads();
      if (ne) {
        const uint32_t rel = static_cast<uint32_t>(oi) - out_index;
        atomicOr(&hmask[rel >> 5], 1u << (rel & 31u));
        rb.start[slot] = static_cast<uint32_t>(oi);
        rb.value[slot] = mode == 2 ? raw : rb.prev + pbefore;
        rb.diff[slot] = diff;
      }
      if (r + 1 == n) rb.pos = pos + q;
      __syncthreads();  // marks complete; everybody has read rb.prev / rb.runs_left / rb.n
      {
        constexpr uint32_t kPer = kChunkPoints / 32 / kThreads;           // mask words per thread
        const uint32_t w0 = kPer * threadIdx.x;
        uint32_t c = 0;
#pragma unroll
        for (uint32_t k = 0; k < kPer; ++k) c += (w0 + k < mw) ? __popc(hmask[w0 + k]) : 0u;
        uint32_t marks;
        uint32_t before = block_exclusive_scan_n<kThreads>(c, sh.scan, &marks);
#pragma unroll
        for (uint32_t k = 0; k < kPer; ++k) {
          if (w0 + k < mw) { hpre[w0 + k] = before; before += __popc(hmask[w0 + k]); }
        }
      }
      if (threadIdx.x == 0) {
        rb.start[ne_total] = out_index + batch_pts;
        rb.n = ne_total;
        rb.prev += prod_total;
        rb.runs_left -= n;
      }
    }
    __syncthreads();
    const uint32_t n = rb.n;
    const uint32_t lo_pt = out_index, hi_pt = rb.start[n];
    for (uint32_t i = lo_pt + threadIdx.x; i < hi_pt; i += blockDim.x) {
      const uint32_t rel = i - lo_pt, w = rel >> 5;
      const uint32_t run = hpre[w] + __popc(hmask[w] & (0xFFFFFFFFu >> (31u - (rel & 31u)))) - 1u;
      unsigned long long v = rb.value[run];
      if (mode == 3) v += static_cast<unsigned long long>(rb.diff[run]) * static_cast<unsigned long long>(i - rb.start[run] + 1);
      if (sf.offset != CLDN_SKIP_STORE_OFFSET) store_low_bytes(out + static_cast<size_t>(i) * step + sf.offset, v, bpv);
    }
    out_index = hi_pt;
    const uint32_t left = rb.runs_left;
    __syncthreads();
    if (left == 0) break;
  }
  if (out_index != n_points) {
    if (threadIdx.x == 0) report_error(err, DEV_ERR_RLE);  // "run count does not fill chunk"
    return 0xFFFFFFFFu;
  }
  return rb.pos;
}

// ------------------------------------------------------------------------------------------------------------------
// One CTA per chunk: regular stream (varint-coded plans) followed by the V5 sections.
template <int KT>
__global__ void __launch_bounds__(kThreads) decode_chunks_kernel(const DecLaunch L) {
  extern __shared__ __align__(16) uint8_t dyn_smem[];
  __shared__ DecShared sh;
  __shared__ DecSlot s_slots[kMaxOps + 1];
  __shared__ uint32_t s_frame;
  __shared__ uint32_t s_side_err;   // side mode: the error word of this chunk's sections
  // dynamic smem: tile bytes | values | nan bits | run batch
  uint8_t* tile_bytes = dyn_smem;
  uint8_t* vals_raw = tile_bytes + kLookBehind + kDecTileBytes + 16;
  constexpr size_t kValBytes = static_cast<size_t>(kDecTileBytes) * (KT > 0 ? 4 : 8);
  uint32_t* nanbits = reinterpret_cast<uint32_t*>(vals_raw + kValBytes);
  RunBatch& rb = *reinterpret_cast<RunBatch*>(reinterpret_cast<uint8_t*>(nanbits) + kDecTileBytes / 8);

  uint32_t gc = blockIdx.x;
  if (L.redo_mode) {  // only the chunks the fast reader handed over (NaN markers, 5+ byte varints, wide scalars, damage)
    if (gc >= L.chunk_counter[3]) return;
    gc = L.redo_list[gc];
  }
  if (threadIdx.x == 0) {
    uint32_t lo = 0, hi = L.n_frames - 1;
    while (lo < hi) {
      const uint32_t mid = (lo + hi + 1) >> 1;
      if (L.frames[mid].chunk_begin <= gc) lo = mid; else hi = mid - 1;
    }
    s_frame = lo;
    s_side_err = 0u;
  }
  const Plan& plan = *L.plan;
  // expand the regular ops into slots
  if (threadIdx.x == 0) {
    int ns = 0;
    for (uint32_t k = 0; k < plan.n_ops; ++k) {
      const RegOp& op = plan.ops[k];
      for (int l = 0; l < op.lanes; ++l) {
        DecSlot& s = s_slots[ns++];
        s.offset = op.offset[l];
        s.size = op.size;
        s.mul_f = op.dec_mul_f[l];
        s.mul_d = op.dec_mul_d;
        s.kind = op.kind == OP_FLOATN ? SLOT_FLOATN : op.kind == OP_F32_LOSSY ? SLOT_F32 : op.kind == OP_F64_LOSSY ? SLOT_F64 : SLOT_INT;
      }
    }
  }
  __syncthreads();
  const DecFrame F = L.frames[s_frame];
  const uint32_t c = gc - F.chunk_begin;
  const uint32_t n_points = min(kChunkPoints, F.n_points - c * kChunkPoints);
  const uint8_t* body = F.payload + L.chunk_offsets[gc];
  const uint32_t body_bytes = L.chunk_sizes[gc];
  uint8_t* out = F.out + static_cast<size_t>(c) * kChunkPoints * plan.point_step;

  // Side mode: the sections are decoded AHEAD of the regular stream (stream_end_kernel said where they start) into compact
  // per-chunk arrays that the fast reader merges into the rows it writes. Nothing is reported from here then: whatever
  // is wrong with a section marks the chunk, and the careful kernels decode it again in the reference's order (regular
  // stream first), so the first error a caller sees is the one the reference would raise.
  const bool side = L.sections_only != 0u && L.side_mode != 0u;
  uint32_t* const err = side ? &s_side_err : frame_err_word(L, s_frame);
  uint32_t pos = 0;
  if (L.sections_only) {
    // the regular stream was decoded by another kernel; sections start where it ended
    pos = L.stream_end[gc];
    if (pos > body_bytes) return;  // regular stream failed (error already reported / chunk already marked)
  } else if (plan.values_per_point > 0) {
    const uint32_t used = decode_varint_stream<KT>(body, body_bytes, n_points, static_cast<int>(plan.values_per_point), s_slots,
                                                   out, plan.point_step, sh, tile_bytes, vals_raw, nanbits, err);
    if (used == 0xFFFFFFFFu) return;
    pos = used;
  }
  for (uint32_t s = 0; s < plan.n_sections; ++s) {
    SectionField sf = plan.sections[s];
    uint8_t* dst = out;
    uint32_t dstep = plan.point_step;
    if (side) {
      dst = L.side + L.side_off[s] + static_cast<size_t>(gc) * kChunkPoints * sf.bpv;
      dstep = sf.bpv;
      if (sf.offset != CLDN_SKIP_STORE_OFFSET) sf.offset = 0;
    }
    const uint32_t used = decode_section<KT>(body + pos, body_bytes - pos, n_points, sf, dst, dstep,
                                             sh, tile_bytes, vals_raw, nanbits, rb, &s_slots[kMaxOps], err);
    if (used == 0xFFFFFFFFu) {
      if (side && threadIdx.x == 0) L.stream_end[gc] = 0xFFFFFFFFu;
      return;
    }
    pos += used;
    __syncthreads();
  }
  // DecodeV5Stage1Chunk rejects trailing bytes (v5_codec.cpp:1008-1010); DecodeV4Stage1Chunk does not check.
  if (plan.uses_v5 && pos != body_bytes && threadIdx.x == 0) report_error(err, DEV_ERR_TRAILING);
  if (side) {
    __syncthreads();
    if (threadIdx.x == 0 && s_side_err != 0u) L.stream_end[gc] = 0xFFFFFFFFu;
  }
}

// ------------------------------------------------------------------------------------------------------------------
// All-Copy plans (encoding NONE, or LOSSY clouds made of INT8 / resolution-less FLOAT32 fields only): fixed point
// size, every point independent. One thread per point.
__global__ void __launch_bounds__(kThreads) decode_fixed_kernel(const DecLaunch L) {
  const Plan& plan = *L.plan;
  const uint32_t gc = blockIdx.y;
  uint32_t lo = 0, hi = L.n_frames - 1;
  while (lo < hi) {
    const uint32_t mid = (lo + hi + 1) >> 1;
    if (L.frames[mid].chunk_begin <= gc) lo = mid; else hi = mid - 1;
  }
  const DecFrame F = L.frames[lo];
  const uint32_t c = gc - F.chunk_begin;
  const uint32_t n_points = min(kChunkPoints, F.n_points - c * kChunkPoints);
  const uint8_t* body = F.payload + L.chunk_offsets[gc];
  const uint32_t body_bytes = L.chunk_sizes[gc];
  const uint32_t psize = plan.min_point_bytes;
  if (static_cast<uint64_t>(n_points) * psize > body_bytes) {
    if (threadIdx.x == 0 && blockIdx.x == 0) report_frame_error(L, lo, DEV_ERR_TRUNCATED);
    return;
  }
  uint8_t* out = F.out + static_cast<size_t>(c) * kChunkPoints * plan.point_step;
  for (uint32_t p = blockIdx.x * blockDim.x + threadIdx.x; p < n_points; p += gridDim.x * blockDim.x) {
    const uint8_t* src = body + static_cast<size_t>(p) * psize;
    uint8_t* dst = out + static_cast<size_t>(p) * plan.point_step;
    for (uint32_t k = 0; k < plan.n_ops; ++k) {
      const RegOp& op = plan.ops[k];
      if (op.offset[0] != CLDN_SKIP_STORE_OFFSET) store_low_bytes(dst + op.offset[0], load_raw_bits(src, op.size), op.size);
      src += op.size;
    }
  }
}

// ------------------------------------------------------------------------------------------------------------------
// Sequential fallback for regular streams that mix raw (Copy) and varint fields: one thread per chunk walks the
// stream exactly like DecodeV4Stage1Chunk. Sections (if any) are then decoded by the same thread.
__global__ void decode_sequential_kernel(const DecLaunch L) {
  const uint32_t gc = blockIdx.x * blockDim.x + threadIdx.x;
  if (gc >= L.n_chunks_total) return;
  const Plan& plan = *L.plan;
  uint32_t lo = 0, hi = L.n_frames - 1;
  while (lo < hi) {
    const uint32_t mid = (lo + hi + 1) >> 1;
    if (L.frames[mid].chunk_begin <= gc) lo = mid; else hi = mid - 1;
  }
  const DecFrame F = L.frames[lo];
  const uint32_t c = gc - F.chunk_begin;
  const uint32_t n_points = min(kChunkPoints, F.n_points - c * kChunkPoints);
  const uint8_t* p = F.payload + L.chunk_offsets[gc];
  uint32_t avail = L.chunk_sizes[gc];
  uint8_t* out = F.out + static_cast<size_t>(c) * kChunkPoints * plan.point_step;
  long long prev[kMaxOps];      // per op: previous quantised value / previous raw bits (FloatN uses prev4)
  int32_t prev4[4] = {0, 0, 0, 0};
  uint8_t g_lead[kMaxOps], g_trail[kMaxOps], g_first[kMaxOps];
  for (int i = 0; i < kMaxOps; ++i) { prev[i] = 0; g_lead[i] = 255; g_trail[i] = 0; g_first[i] = 1; }
  const uint8_t* const body = p;
  if (L.stream_end) L.stream_end[gc] = 0xFFFFFFFFu;  // stays so if the stream turns out to be malformed
  for (uint32_t pt = 0; pt < n_points; ++pt) {
    if (!plan.uses_v5 && avail < plan.min_point_bytes) { report_frame_error(L, lo, DEV_ERR_TRUNCATED); return; }  // v4_codec.cpp:102-104
    uint8_t* point = out + static_cast<size_t>(pt) * plan.point_step;
    for (uint32_t k = 0; k < plan.n_ops; ++k) {
      const RegOp& op = plan.ops[k];
      if (op.kind == OP_COPY) {
        if (avail < op.size) { report_frame_error(L, lo, DEV_ERR_TRUNCATED); return; }
        if (op.offset[0] != CLDN_SKIP_STORE_OFFSET) store_low_bytes(point + op.offset[0], load_raw_bits(p, op.size), op.size);
        p += op.size; avail -= op.size;
        continue;
      }
      if (op.kind == OP_XOR32 || op.kind == OP_XOR64) {  // field_decoder.hpp:356-370
        if (avail < op.size) { report_frame_error(L, lo, DEV_ERR_TRUNCATED); return; }
        const unsigned long long res = load_raw_bits(p, op.size);
        p += op.size; avail -= op.size;
        prev[k] = static_cast<long long>(static_cast<unsigned long long>(prev[k]) ^ res);
        if (op.offset[0] != CLDN_SKIP_STORE_OFFSET) store_low_bytes(point + op.offset[0], static_cast<uint64_t>(prev[k]), op.size);
        continue;
      }
      if (op.kind == OP_GORILLA64) {  // field_decoder.hpp:257-300
        GorillaState st;
        st.prev_bits = static_cast<uint64_t>(prev[k]); st.leading = g_lead[k]; st.trailing = g_trail[k]; st.first = g_first[k] != 0;
        uint64_t v;
        const uint32_t c = gorilla_decode(st, p, avail, &v);
        if (!c) { report_frame_error(L, lo, DEV_ERR_TRUNCATED); return; }
        p += c; avail -= c;
        prev[k] = static_cast<long long>(st.prev_bits); g_lead[k] = static_cast<uint8_t>(st.leading); g_trail[k] = static_cast<uint8_t>(st.trailing); g_first[k] = 0;
        if (op.offset[0] != CLDN_SKIP_STORE_OFFSET) store_u64(point + op.offset[0], v);
        continue;
      }
      for (int l = 0; l < op.lanes; ++l) {
        if (avail == 0) { report_frame_error(L, lo, DEV_ERR_TRUNCATED); return; }
        DecSlot s;
        s.offset = op.offset[l]; s.size = op.size; s.mul_f = op.dec_mul_f[l]; s.mul_d = op.dec_mul_d;
        s.kind = op.kind == OP_FLOATN ? SLOT_FLOATN : op.kind == OP_F32_LOSSY ? SLOT_F32 : op.kind == OP_F64_LOSSY ? SLOT_F64 : SLOT_INT;
        if (p[0] == 0 && s.kind != SLOT_INT) {
          if (op.kind == OP_FLOATN) prev4[l] = 0; else prev[k] = 0;
          store_slot_value<long long>(point, s, 0, true);
          ++p; --avail;
          continue;
        }
        long long diff;
        const uint32_t n = read_varint(p, avail, &diff, frame_err_word(L, lo));
        if (!n) return;
        p += n; avail -= n;
        long long value;
        if (op.kind == OP_FLOATN) { prev4[l] = wadd(static_cast<int32_t>(diff), prev4[l]); value = prev4[l]; }
        else { prev[k] = wadd(prev[k], diff); value = prev[k]; }
        store_slot_value<long long>(point, s, value, false);
      }
    }
  }
  if (L.stream_end) L.stream_end[gc] = static_cast<uint32_t>(p - body);  // V5: the sections start here
}

// ------------------------------------------------------------------------------------------------------------------
// Mixed plans: varint-coded fields AND raw (Copy) / XOR fields in the regular stream (sensor layouts with uint8 fields,
// LOSSLESS float clouds). Raw bytes carry no terminator structure, so the terminator ranking of decode_varint_stream does
// not find value boundaries; the one-thread-per-chunk parser above does, at the speed of a single GPU thread.
// This kernel finds the POINT boundaries in parallel instead (one CTA per chunk, tiles of kMixTile candidate positions):
//   1. bytes of the tile (+ kMixLook look-ahead) are staged in shared memory, one terminator bit per byte;
//   2. every byte position b computes next(b): where the following point would start IF a point started at b (skip
//      n varints = n terminator bits, skip the fixed bytes, segment by segment) — independent of everything before b;
//   3. the true boundaries are the orbit of the tile's entry position under next(): pointer doubling builds the 2^k-hop
//      table and the list of the first 2^(k+1) boundaries in round k (log2 rounds, all threads);
//   4. one thread per point then decodes its tokens with the careful readers (errors exactly where the reference's
//      decoders throw), and per-field CTA scans (segmented sums with NaN reset, XOR scans) turn deltas into values.
// Gorilla fields stay with the per-chunk parser: a record's length depends on the running window, so next(b) is not a
// function of b alone.
constexpr uint32_t kMixTile = 8192;   // candidate point starts per tile (tile-local positions [0, kMixTile))
constexpr uint32_t kMixLook = 512;    // a point that starts inside the tile may extend this far behind it
constexpr uint32_t kMixBatch = kThreads;
constexpr uint32_t kMixNone = 0xFFFFu;
constexpr uint32_t kMixBitWords = (kMixTile + kMixLook) / 32 + 4;

enum MixKind : uint8_t { MIX_VAR = 0, MIX_COPY = 1, MIX_XOR = 2 };
struct MixToken {
  uint8_t kind;    // MixKind
  uint8_t size;    // raw bytes (COPY / XOR), stored bytes (INT)
  uint16_t index;  // index among the VAR tokens or among the fixed tokens of a point
  DecSlot slot;    // VAR: how to turn the accumulated value into the field
  uint32_t offset; // COPY / XOR: byte offset inside the point
};
struct MixShared {
  MixToken tok[kMaxOps + 4];
  uint8_t seg_nvar[kMaxOps + 4], seg_nfix[kMaxOps + 4];  // next(): n varints, then n fixed bytes, segment by segment
  uint32_t n_tok, n_seg, n_var, n_fix;
  uint32_t n_found;   // boundaries found in this tile
  uint32_t fail;
  long long carry[kMaxOps + 4];            // per VAR token: last absolute value
  unsigned long long xcarry[kMaxOps + 4];  // per fixed token (XOR): last raw bits
  unsigned long long xscan[kThreads / 32];
};

// 64 terminator bits starting at bit position p
__device__ __forceinline__ uint64_t mix_window(const uint32_t* tbits, uint32_t p) {
  const uint32_t w = p >> 5, sh = p & 31u;
  const uint32_t a = tbits[w], b = tbits[w + 1], c = tbits[w + 2];
  return static_cast<uint64_t>(__funnelshift_r(a, b, sh)) | (static_cast<uint64_t>(__funnelshift_r(b, c, sh)) << 32);
}
// Start of the point that follows a point starting at local position p (kMixNone if it cannot be told from this tile).
__device__ __forceinline__ uint32_t mix_next(const MixShared& ms, const uint32_t* tbits, uint32_t p, uint32_t limit) {
  for (uint32_t s = 0; s < ms.n_seg; ++s) {
    uint32_t k = ms.seg_nvar[s];
    while (k) {
      if (p >= limit) return kMixNone;
      uint64_t w = mix_window(tbits, p);
      const uint32_t c = static_cast<uint32_t>(__popcll(w));
      if (c >= k) {
        for (uint32_t i = 1; i < k; ++i) w &= w - 1ull;
        p += static_cast<uint32_t>(__ffsll(static_cast<long long>(w)));
        k = 0;
      } else {
        k -= c;
        p += 64u;
      }
    }
    p += ms.seg_nfix[s];
    if (p > limit) return kMixNone;
  }
  return p;
}
__device__ __forceinline__ unsigned long long mix_block_xor_exclusive(unsigned long long v, unsigned long long* scratch,
                                                                     unsigned long long* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  unsigned long long inc = v;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const unsigned long long t = __shfl_up_sync(0xffffffffu, inc, d);
    if (lane >= d) inc ^= t;
  }
  if (lane == 31) scratch[warp] = inc;
  __syncthreads();
  unsigned long long before = 0, all = 0;
#pragma unroll
  for (int w = 0; w < kThreads / 32; ++w) {
    const unsigned long long x = scratch[w];
    if (w < warp) before ^= x;
    all ^= x;
  }
  *total = all;
  __syncthreads();  // scratch is reused by the next scan
  return before ^ inc ^ v;
}

__global__ void __launch_bounds__(kThreads) decode_mixed_kernel(const DecLaunch L) {
  extern __shared__ __align__(16) uint8_t dyn_smem[];
  __shared__ DecShared sh;
  __shared__ MixShared ms;
  __shared__ uint32_t s_frame;
  // dynamic smem: bytes | terminator bits | 2 jump tables | boundary list | per-batch values
  uint8_t* bytes = dyn_smem;
  uint32_t* tbits = reinterpret_cast<uint32_t*>(bytes + kMixTile + kMixLook + 32);
  uint16_t* jump0 = reinterpret_cast<uint16_t*>(tbits + kMixBitWords);
  uint16_t* jump1 = jump0 + kMixTile;
  uint16_t* starts = jump1 + kMixTile;  // [kMixTile + 2]
  long long* vals = reinterpret_cast<long long*>(reinterpret_cast<uint8_t*>(starts) + ((kMixTile + 2) * 2 + 15) / 16 * 16);

  const uint32_t gc = blockIdx.x;
  const Plan& plan = *L.plan;
  if (threadIdx.x == 0) {
    uint32_t lo = 0, hi = L.n_frames - 1;
    while (lo < hi) {
      const uint32_t mid = (lo + hi + 1) >> 1;
      if (L.frames[mid].chunk_begin <= gc) lo = mid; else hi = mid - 1;
    }
    s_frame = lo;
    // token program of one point, in stream order
    uint32_t nt = 0, nv = 0, nf = 0, nseg = 0;
    uint32_t run_var = 0, run_fix = 0;
    for (uint32_t k = 0; k < plan.n_ops; ++k) {
      const RegOp& op = plan.ops[k];
      const bool fixed = op.kind == OP_COPY || op.kind == OP_XOR32 || op.kind == OP_XOR64;
      for (int l = 0; l < (fixed ? 1 : op.lanes); ++l) {
        MixToken& t = ms.tok[nt++];
        if (fixed) {
          t.kind = op.kind == OP_COPY ? MIX_COPY : MIX_XOR;
          t.size = op.size;
          t.index = static_cast<uint16_t>(nf++);
          t.offset = op.offset[0];
          run_fix += op.size;
        } else {
          if (run_fix) { ms.seg_nvar[nseg] = static_cast<uint8_t>(run_var); ms.seg_nfix[nseg] = static_cast<uint8_t>(run_fix); ++nseg; run_var = run_fix = 0; }
          t.kind = MIX_VAR;
          t.size = op.size;
          t.index = static_cast<uint16_t>(nv++);
          t.offset = op.offset[l];
          t.slot.offset = op.offset[l];
          t.slot.size = op.size;
          t.slot.mul_f = op.dec_mul_f[l];
          t.slot.mul_d = op.dec_mul_d;
          t.slot.kind = op.kind == OP_FLOATN ? SLOT_FLOATN : op.kind == OP_F32_LOSSY ? SLOT_F32 : op.kind == OP_F64_LOSSY ? SLOT_F64 : SLOT_INT;
          ++run_var;
        }
      }
    }
    if (run_var || run_fix) { ms.seg_nvar[nseg] = static_cast<uint8_t>(run_var); ms.seg_nfix[nseg] = static_cast<uint8_t>(run_fix); ++nseg; }
    ms.n_tok = nt; ms.n_var = nv; ms.n_fix = nf; ms.n_seg = nseg;
    ms.fail = 0;
    for (uint32_t i = 0; i < kMaxOps + 4; ++i) { ms.carry[i] = 0; ms.xcarry[i] = 0; }
  }
  __syncthreads();
  const DecFrame F = L.frames[s_frame];
  const uint32_t c = gc - F.chunk_begin;
  const uint32_t n_points = min(kChunkPoints, F.n_points - c * kChunkPoints);
  const uint8_t* body = F.payload + L.chunk_offsets[gc];
  const uint32_t size = L.chunk_sizes[gc];
  uint8_t* out = F.out + static_cast<size_t>(c) * kChunkPoints * plan.point_step;
  const uint32_t n_var = ms.n_var, n_fix = ms.n_fix, n_tok = ms.n_tok;
  uint8_t* nanflag = reinterpret_cast<uint8_t*>(vals + static_cast<size_t>(kMixBatch) * n_var);
  unsigned long long* raws = reinterpret_cast<unsigned long long*>(nanflag + ((static_cast<size_t>(kMixBatch) * n_var + 15) / 16) * 16);
  if (L.stream_end && threadIdx.x == 0) L.stream_end[gc] = 0xFFFFFFFFu;  // stays so if the stream turns out to be malformed

  uint32_t done = 0;   // points decoded so far
  uint32_t t0 = 0;     // chunk-body offset of the next point
  while (done < n_points) {
    if (t0 >= size) {  // points are still missing but the bytes are used up: "Truncated encoded data" (v4_codec.cpp:102-104)
      if (threadIdx.x == 0) report_frame_error(L, s_frame, DEV_ERR_TRUNCATED);
      return;
    }
    // ---- 1. stage [a0, a0 + kMixTile + kMixLook) with a0 = t0 rounded down to a 16-byte aligned ADDRESS ----
    const uint32_t mis = static_cast<uint32_t>((reinterpret_cast<uintptr_t>(body) + t0) & 15u);
    const int64_t a0 = static_cast<int64_t>(t0) - mis;  // may be negative at the chunk start: those bytes are never read
    const int64_t avail_local = static_cast<int64_t>(size) - a0;
    const uint32_t limit = static_cast<uint32_t>(avail_local < static_cast<int64_t>(kMixTile + kMixLook) ? avail_local : kMixTile + kMixLook);
    for (uint32_t v = threadIdx.x; v < (kMixTile + kMixLook) / 16; v += blockDim.x) {
      const int64_t b = a0 + static_cast<int64_t>(v) * 16;
      uint4 q = make_uint4(0x80808080u, 0x80808080u, 0x80808080u, 0x80808080u);
      if (b >= 0 && b + 16 <= static_cast<int64_t>(size)) {
        q = *reinterpret_cast<const uint4*>(body + b);
      } else if (b + 16 > 0 && b < static_cast<int64_t>(size)) {
        uint32_t w[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
        for (int k = 0; k < 16; ++k) {
          const int64_t bb = b + k;
          if (bb >= 0 && bb < static_cast<int64_t>(size)) w[k >> 2] = (w[k >> 2] & ~(0xFFu << (8 * (k & 3)))) | (static_cast<uint32_t>(body[bb]) << (8 * (k & 3)));
        }
        q = make_uint4(w[0], w[1], w[2], w[3]);
      }
      *reinterpret_cast<uint4*>(bytes + v * 16) = q;
    }
    __syncthreads();
    for (uint32_t w = threadIdx.x; w < kMixBitWords; w += blockDim.x) {
      uint32_t m = 0;
      if (w * 32u < limit) {
        const uint4 lo = *reinterpret_cast<const uint4*>(bytes + w * 32u);
        const uint4 hi = *reinterpret_cast<const uint4*>(bytes + w * 32u + 16u);
        const uint32_t x[8] = {lo.x, lo.y, lo.z, lo.w, hi.x, hi.y, hi.z, hi.w};
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          const uint32_t t = ~x[k] & 0x80808080u;  // MSB clear = the byte ends a varint
          m |= (((t >> 7) & 1u) | ((t >> 14) & 2u) | ((t >> 21) & 4u) | ((t >> 28) & 8u)) << (4 * k);
        }
        if (w * 32u + 32u > limit) m &= (1u << (limit - w * 32u)) - 1u;  // nothing behind the last byte
        if (w * 32u < mis) m &= ~((1u << (mis - w * 32u > 31u ? 31u : mis - w * 32u)) - 1u);  // bytes in front of the entry are not ours
      }
      tbits[w] = m;
    }
    __syncthreads();
    // ---- 2. next(b) for every candidate start ----
    for (uint32_t b = threadIdx.x; b < kMixTile; b += blockDim.x) {
      uint32_t nx = kMixNone;
      if (b >= mis && b < limit) nx = mix_next(ms, tbits, b, limit);
      jump0[b] = static_cast<uint16_t>(nx);
      starts[b] = static_cast<uint16_t>(kMixNone);
    }
    if (threadIdx.x == 0) {  // (thread 0 also owns b = 0 in the loop above: program order)
      starts[0] = static_cast<uint16_t>(mis);  // boundary 0 = the tile's entry
      starts[kMixTile] = starts[kMixTile + 1] = static_cast<uint16_t>(kMixNone);
      ms.n_found = 1;
    }
    __syncthreads();
    // ---- 3. pointer doubling: round k appends boundaries 2^k .. 2^(k+1)-1 and squares the jump table ----
    uint16_t* jt = jump0;
    uint16_t* jn = jump1;
    uint32_t exit_pos = kMixNone;
    for (uint32_t step = 1; step < kMixTile; step <<= 1) {  // a tile holds at most kMixTile boundaries (one per byte)
      int grew = 0;
      for (uint32_t i = threadIdx.x; i < step; i += blockDim.x) {
        const uint32_t b = starts[i];
        if (b != kMixNone) {
          const uint32_t t = jt[b];
          if (t < kMixTile) { starts[i + step] = static_cast<uint16_t>(t); grew = 1; }
        }
      }
      if (!__syncthreads_or(grew)) { exit_pos = jt[mis]; break; }  // no boundary beyond 2^k: jt[entry] already left the tile
      for (uint32_t b = threadIdx.x; b < kMixTile; b += blockDim.x) {
        const uint32_t t = jt[b];
        jn[b] = (t < kMixTile) ? jt[t] : static_cast<uint16_t>(t);
      }
      __syncthreads();
      uint16_t* sw = jt; jt = jn; jn = sw;
      exit_pos = jt[mis];
    }
    {  // number of boundaries = first unset entry of the list
      uint32_t mine = 0;
      for (uint32_t i = threadIdx.x; i < kMixTile; i += blockDim.x) if (starts[i] != kMixNone) mine = i + 1;
      atomicMax(&ms.n_found, mine);
    }
    __syncthreads();
    const uint32_t found = ms.n_found;
    const uint32_t take = found < n_points - done ? found : n_points - done;
    if (threadIdx.x == 0) starts[found] = static_cast<uint16_t>(exit_pos);  // end of the last point of the tile
    __syncthreads();
    // ---- 4. + 5. batches of one point per thread ----
    for (uint32_t b0 = 0; b0 < take; b0 += kMixBatch) {
      const uint32_t i = b0 + threadIdx.x;
      const bool active = i < take;
      bool bad = false;
      if (active) {
        uint32_t p = starts[i];
        for (uint32_t t = 0; t < n_tok; ++t) {
          const MixToken& tk = ms.tok[t];
          if (tk.kind == MIX_VAR) {
            long long diff = 0;
            uint8_t nan = 0;
            if (p >= limit) { report_frame_error(L, s_frame, DEV_ERR_TRUNCATED); bad = true; break; }
            if (bytes[p] == 0 && tk.slot.kind != SLOT_INT) { nan = 1; ++p; }  // NaN marker (field_decoder.cpp:57-61)
            else {
              const uint32_t n = read_varint(bytes + p, limit - p, &diff, frame_err_word(L, s_frame));
              if (!n) { bad = true; break; }
              p += n;
            }
            vals[static_cast<size_t>(threadIdx.x) * n_var + tk.index] = diff;
            nanflag[static_cast<size_t>(threadIdx.x) * n_var + tk.index] = nan;
          } else {
            if (p + tk.size > limit) { report_frame_error(L, s_frame, DEV_ERR_TRUNCATED); bad = true; break; }
            raws[static_cast<size_t>(threadIdx.x) * n_fix + tk.index] = load_raw_bits(bytes + p, tk.size);
            p += tk.size;
          }
        }
      }
      if (__syncthreads_or(bad ? 1 : 0)) return;  // the error word is set; the host reports it
      uint8_t* point = out + static_cast<size_t>(done + i) * plan.point_step;
      for (uint32_t t = 0; t < n_tok; ++t) {
        const MixToken& tk = ms.tok[t];
        if (tk.kind == MIX_VAR) {
          const long long d = active ? vals[static_cast<size_t>(threadIdx.x) * n_var + tk.index] : 0;
          const bool nan = active && nanflag[static_cast<size_t>(threadIdx.x) * n_var + tk.index] != 0;
          Seg<long long, 1> mine;
          mine.sum[0] = nan ? 0 : d;
          mine.rst = nan ? 1u : 0u;
          Seg<long long, 1> total;
          const Seg<long long, 1> ex = block_seg_exclusive<long long, 1>(mine, sh.seg_sum, sh.seg_rst, &total);
          const long long before = ex.rst ? ex.sum[0] : wadd(ms.carry[tk.index], ex.sum[0]);
          if (active) store_slot_value<long long>(point, tk.slot, nan ? 0 : wadd(before, d), nan);
          __syncthreads();
          if (threadIdx.x == 0) ms.carry[tk.index] = total.rst ? total.sum[0] : wadd(ms.carry[tk.index], total.sum[0]);
        } else if (tk.kind == MIX_XOR) {  // field_decoder.hpp:356-370: value = residual ^ previous value
          const unsigned long long r = active ? raws[static_cast<size_t>(threadIdx.x) * n_fix + tk.index] : 0ull;
          unsigned long long total;
          const unsigned long long ex = mix_block_xor_exclusive(r, ms.xscan, &total);
          const unsigned long long v = ms.xcarry[tk.index] ^ ex ^ r;
          if (active && tk.offset != CLDN_SKIP_STORE_OFFSET) store_low_bytes(point + tk.offset, v, tk.size);
          __syncthreads();
          if (threadIdx.x == 0) ms.xcarry[tk.index] ^= total;
        } else if (active && tk.offset != CLDN_SKIP_STORE_OFFSET) {
          store_low_bytes(point + tk.offset, raws[static_cast<size_t>(threadIdx.x) * n_fix + tk.index], tk.size);
        }
      }
      __syncthreads();
    }
    done += take;
    const uint32_t end_local = starts[take];  // start of the first point that was NOT taken (or the tile's exit)
    __syncthreads();                          // everybody has read the list before the next tile rewrites it
    if (done < n_points) {
      if (end_local == kMixNone || end_local <= mis) {  // the path left the tile through a point this tile cannot delimit
        if (threadIdx.x == 0) report_frame_error(L, s_frame, DEV_ERR_TRUNCATED);
        return;
      }
      t0 = static_cast<uint32_t>(a0 + end_local);
    } else {
      if (end_local == kMixNone) { if (threadIdx.x == 0) report_frame_error(L, s_frame, DEV_ERR_TRUNCATED); return; }
      if (L.stream_end && threadIdx.x == 0) L.stream_end[gc] = static_cast<uint32_t>(a0 + end_local);  // V5: the sections start here
    }
  }
  if (n_points == 0 && L.stream_end && threadIdx.x == 0) L.stream_end[gc] = 0;
}

static size_t mixed_smem_bytes(const Plan& plan) {
  size_t n_var = 0, n_fix = 0;
  for (uint32_t k = 0; k < plan.n_ops; ++k) {
    const RegOp& op = plan.ops[k];
    if (op.kind == OP_COPY || op.kind == OP_XOR32 || op.kind == OP_XOR64) ++n_fix; else n_var += op.lanes;
  }
  size_t bytes = kMixTile + kMixLook + 32 + kMixBitWords * 4 + 2 * kMixTile * 2;
  bytes += ((kMixTile + 2) * 2 + 15) / 16 * 16;
  bytes += kMixBatch * n_var * 8;
  bytes += (kMixBatch * n_var + 15) / 16 * 16;
  bytes += kMixBatch * n_fix * 8 + 64;
  return bytes;
}
// The parallel boundary search applies when a point's length is a function of its own bytes (no Gorilla window) and a
// point fits the look-ahead of a tile.
static bool mixed_plan_ok(const Plan& plan) {
  if (plan.n_gorilla != 0 || plan.max_point_bytes > kMixLook || plan.n_ops == 0) return false;
  const char* e = getenv("CLDN_B200_MIXED_DECODE");  // "par" / "seq": explicit choice
  return !(e && e[0] == 's');
}

// ------------------------------------------------------------------------------------------------------------------
// Plans with ONE Gorilla field (FLOAT64 without a resolution — the timestamps of most sensor drivers) next to varint /
// raw / XOR fields. A Gorilla record is byte aligned but its length is not a function of its own bytes: a "reuse window"
// record is 2 + meaningful(window) bits long. Only the BYTE length of such a record matters for the boundaries, i.e. one
// of 10 classes (0 = no window yet, 1..9 = bytes of a reuse record), and a "new window" record announces the class that
// follows it. So next() becomes a function of (position, class): every thread fills next(b, c) for its positions and all
// classes (the work in front of the record is shared), ONE thread then follows the tile's entry through the table (one
// shared-memory load per point instead of a full parse) and all threads decode: varints / raw fields as in
// decode_mixed_kernel, the Gorilla values by a "last new-window record" scan (which window does a reuse record see) and
// an XOR scan (value = xor of all residuals so far).
constexpr uint32_t kGorTile = 2048;
constexpr uint32_t kGorClasses = 10;
constexpr uint32_t kGorBitWords = (kGorTile + kMixLook) / 32 + 4;
constexpr uint32_t kGorNone = 0xFFFFFFFFu;
constexpr uint8_t MIX_GORILLA = 3;

// Header of the Gorilla record at p (field_decoder.hpp:257-300), read with the same truncation tests as gorilla_decode.
// kind: 0 same value (1 byte), 1 reuse window, 2 new window; returns false when the header itself is truncated.
struct GorHeader { uint32_t kind, lead, meaningful; };
__device__ __forceinline__ bool gor_header(const uint8_t* p, uint32_t avail, GorHeader* h) {
  BitWindow w(p, avail);
  uint64_t flag, control, lead, m1;
  h->kind = 0; h->lead = 0; h->meaningful = 0;
  if (!w.read(1, &flag)) return false;
  if (flag == 0) return true;
  if (!w.read(1, &control)) return false;
  if (control == 0) { h->kind = 1; return true; }
  if (!w.read(5, &lead) || !w.read(6, &m1)) return false;
  h->kind = 2; h->lead = static_cast<uint32_t>(lead); h->meaningful = static_cast<uint32_t>(m1) + 1u;
  return true;
}
// position after one varint that starts at p (kMixNone if its terminator is not within 64 bytes / the data)
__device__ __forceinline__ uint32_t gor_skip_varint(const uint32_t* tbits, uint32_t p, uint32_t limit) {
  if (p >= limit) return kMixNone;
  const uint64_t w = mix_window(tbits, p);
  if (w == 0ull) return kMixNone;
  return p + static_cast<uint32_t>(__ffsll(static_cast<long long>(w)));
}
// Walks tokens [t_begin, t_end) that hold no Gorilla record.
__device__ __forceinline__ uint32_t gor_skip_tokens(const MixShared& ms, const uint32_t* tbits, uint32_t p, uint32_t limit,
                                                    uint32_t t_begin, uint32_t t_end) {
  for (uint32_t t = t_begin; t < t_end && p != kMixNone; ++t) {
    if (ms.tok[t].kind == MIX_VAR) p = gor_skip_varint(tbits, p, limit);
    else { p += ms.tok[t].size; if (p > limit) p = kMixNone; }
  }
  return p;
}
// exclusive "latest valid entry" scan: v = (1 << 16) | payload for threads that define a window, 0 otherwise
__device__ __forceinline__ uint32_t gor_block_last_exclusive(uint32_t v, uint32_t* scratch, uint32_t* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint32_t inc = v;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const uint32_t t = __shfl_up_sync(0xffffffffu, inc, d);
    if (lane >= d && inc == 0u) inc = t;
  }
  if (lane == 31) scratch[warp] = inc;
  uint32_t prev = __shfl_up_sync(0xffffffffu, inc, 1);
  if (lane == 0) prev = 0;
  __syncthreads();
  uint32_t before = 0, all = 0;
#pragma unroll
  for (int w = 0; w < kThreads / 32; ++w) {
    const uint32_t x = scratch[w];
    if (w < warp && x) before = x;
    if (x) all = x;
  }
  *total = all;
  __syncthreads();
  return prev ? prev : before;
}

__global__ void __launch_bounds__(kThreads) decode_gorilla_kernel(const DecLaunch L) {
  extern __shared__ __align__(16) uint8_t dyn_smem[];
  __shared__ DecShared sh;
  __shared__ MixShared ms;
  __shared__ uint32_t s_frame, s_gtok, s_found, s_exit, s_exit_class, s_window, s_class;
  __shared__ uint32_t s_lastscan[kThreads / 32];
  uint8_t* bytes = dyn_smem;
  uint32_t* tbits = reinterpret_cast<uint32_t*>(bytes + kGorTile + kMixLook + 32);
  uint32_t* table = tbits + kGorBitWords;                       // [kGorClasses][kGorTile]: next position | next class << 16
  uint8_t* q = reinterpret_cast<uint8_t*>(table + kGorClasses * kGorTile);
  uint16_t* starts = reinterpret_cast<uint16_t*>(q);  // [kGorTile + 2]
  q += ((kGorTile + 2) * 2 + 15) / 16 * 16;
  uint8_t* cls = q;                                    // [kGorTile + 2] class in front of every point
  q += (kGorTile + 2 + 15) / 16 * 16;
  long long* vals = reinterpret_cast<long long*>(q);

  const uint32_t gc = blockIdx.x;
  const Plan& plan = *L.plan;
  if (threadIdx.x == 0) {
    uint32_t lo = 0, hi = L.n_frames - 1;
    while (lo < hi) {
      const uint32_t mid = (lo + hi + 1) >> 1;
      if (L.frames[mid].chunk_begin <= gc) lo = mid; else hi = mid - 1;
    }
    s_frame = lo;
    uint32_t nt = 0, nv = 0, nf = 0;
    for (uint32_t k = 0; k < plan.n_ops; ++k) {
      const RegOp& op = plan.ops[k];
      const bool fixed = op.kind == OP_COPY || op.kind == OP_XOR32 || op.kind == OP_XOR64;
      const int lanes = (fixed || op.kind == OP_GORILLA64) ? 1 : op.lanes;
      for (int l = 0; l < lanes; ++l) {
        MixToken& t = ms.tok[nt];
        t.size = op.size;
        t.offset = op.offset[l];
        if (op.kind == OP_GORILLA64) { t.kind = MIX_GORILLA; t.index = 0; s_gtok = nt; }
        else if (fixed) { t.kind = op.kind == OP_COPY ? MIX_COPY : MIX_XOR; t.index = static_cast<uint16_t>(nf++); }
        else {
          t.kind = MIX_VAR;
          t.index = static_cast<uint16_t>(nv++);
          t.slot.offset = op.offset[l]; t.slot.size = op.size; t.slot.mul_f = op.dec_mul_f[l]; t.slot.mul_d = op.dec_mul_d;
          t.slot.kind = op.kind == OP_FLOATN ? SLOT_FLOATN : op.kind == OP_F32_LOSSY ? SLOT_F32 : op.kind == OP_F64_LOSSY ? SLOT_F64 : SLOT_INT;
        }
        ++nt;
      }
    }
    ms.n_tok = nt; ms.n_var = nv; ms.n_fix = nf; ms.n_seg = 0;
    for (uint32_t i = 0; i < kMaxOps + 4; ++i) { ms.carry[i] = 0; ms.xcarry[i] = 0; }
    s_window = 0;  // no window yet ((1 << 16) | lead << 8 | trail once there is one)
    s_class = 0;
  }
  __syncthreads();
  const DecFrame F = L.frames[s_frame];
  const uint32_t c = gc - F.chunk_begin;
  const uint32_t n_points = min(kChunkPoints, F.n_points - c * kChunkPoints);
  const uint8_t* body = F.payload + L.chunk_offsets[gc];
  const uint32_t size = L.chunk_sizes[gc];
  uint8_t* out = F.out + static_cast<size_t>(c) * kChunkPoints * plan.point_step;
  const uint32_t n_var = ms.n_var, n_fix = ms.n_fix, n_tok = ms.n_tok, gtok = s_gtok;
  uint8_t* nanflag = reinterpret_cast<uint8_t*>(vals + static_cast<size_t>(kMixBatch) * n_var);
  unsigned long long* raws = reinterpret_cast<unsigned long long*>(nanflag + ((static_cast<size_t>(kMixBatch) * n_var + 15) / 16) * 16);
  if (L.stream_end && threadIdx.x == 0) L.stream_end[gc] = 0xFFFFFFFFu;

  uint32_t done = 0, t0 = 0;
  while (done < n_points) {
    if (t0 >= size) { if (threadIdx.x == 0) report_frame_error(L, s_frame, DEV_ERR_TRUNCATED); return; }
    // ---- 1. stage the tile and its terminator bits (as in decode_mixed_kernel) ----
    const uint32_t mis = static_cast<uint32_t>((reinterpret_cast<uintptr_t>(body) + t0) & 15u);
    const int64_t a0 = static_cast<int64_t>(t0) - mis;
    const int64_t avail_local = static_cast<int64_t>(size) - a0;
    const uint32_t limit = static_cast<uint32_t>(avail_local < static_cast<int64_t>(kGorTile + kMixLook) ? avail_local : kGorTile + kMixLook);
    for (uint32_t v = threadIdx.x; v < (kGorTile + kMixLook) / 16; v += blockDim.x) {
      const int64_t b = a0 + static_cast<int64_t>(v) * 16;
      uint4 q = make_uint4(0x80808080u, 0x80808080u, 0x80808080u, 0x80808080u);
      if (b >= 0 && b + 16 <= static_cast<int64_t>(size)) {
        q = *reinterpret_cast<const uint4*>(body + b);
      } else if (b + 16 > 0 && b < static_cast<int64_t>(size)) {
        uint32_t w[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
        for (int k = 0; k < 16; ++k) {
          const int64_t bb = b + k;
          if (bb >= 0 && bb < static_cast<int64_t>(size)) w[k >> 2] = (w[k >> 2] & ~(0xFFu << (8 * (k & 3)))) | (static_cast<uint32_t>(body[bb]) << (8 * (k & 3)));
        }
        q = make_uint4(w[0], w[1], w[2], w[3]);
      }
      *reinterpret_cast<uint4*>(bytes + v * 16) = q;
    }
    __syncthreads();
    for (uint32_t w = threadIdx.x; w < kGorBitWords; w += blockDim.x) {
      uint32_t m = 0;
      if (w * 32u < limit) {
        const uint4 lo = *reinterpret_cast<const uint4*>(bytes + w * 32u);
        const uint4 hi = *reinterpret_cast<const uint4*>(bytes + w * 32u + 16u);
        const uint32_t x[8] = {lo.x, lo.y, lo.z, lo.w, hi.x, hi.y, hi.z, hi.w};
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          const uint32_t t = ~x[k] & 0x80808080u;
          m |= (((t >> 7) & 1u) | ((t >> 14) & 2u) | ((t >> 21) & 4u) | ((t >> 28) & 8u)) << (4 * k);
        }
        if (w * 32u + 32u > limit) m &= (1u << (limit - w * 32u)) - 1u;
      }
      tbits[w] = m;
    }
    __syncthreads();
    // ---- 2. next(b, class) ----
    for (uint32_t b = threadIdx.x; b < kGorTile; b += blockDim.x) {
      uint32_t pg = kMixNone;
      if (b >= mis && b < limit) pg = gor_skip_tokens(ms, tbits, b, limit, 0, gtok);
      GorHeader h;
      const bool header_ok = pg != kMixNone && pg < limit && gor_header(bytes + pg, limit - pg, &h);
      for (uint32_t cl = 0; cl < kGorClasses; ++cl) {
        uint32_t e = kGorNone;
        if (header_ok) {
          uint32_t len = 1, ncl = cl;
          bool ok = true;
          if (h.kind == 1) len = cl ? cl : 9u;  // reuse: the class IS the length (no window yet: 2 + 65 bits, see gorilla_decode)
          else if (h.kind == 2) { len = (13u + h.meaningful + 7u) >> 3; ncl = (2u + h.meaningful + 7u) >> 3; }
          if (ok && pg + len <= limit) {
            const uint32_t pe = gor_skip_tokens(ms, tbits, pg + len, limit, gtok + 1, n_tok);
            if (pe != kMixNone) e = pe | (ncl << 16);
          }
        }
        table[cl * kGorTile + b] = e;
      }
    }
    __syncthreads();
    // ---- 3. one thread follows the entry through the table ----
    if (threadIdx.x == 0) {
      uint32_t i = 0, p = mis, cl = s_class;
      while (p < kGorTile && i < kGorTile) {
        starts[i] = static_cast<uint16_t>(p);
        cls[i] = static_cast<uint8_t>(cl);
        uint32_t e;
        if (done == 0 && i == 0) {  // first point of the chunk: the record is the 64 raw bits, no window afterwards
          const uint32_t pg = gor_skip_tokens(ms, tbits, p, limit, 0, gtok);
          e = kGorNone;
          if (pg != kMixNone && pg + 8u <= limit) {
            const uint32_t pe = gor_skip_tokens(ms, tbits, pg + 8u, limit, gtok + 1, n_tok);
            if (pe != kMixNone) e = pe;  // class 0
          }
        } else {
          e = table[cl * kGorTile + p];
        }
        ++i;
        if (e == kGorNone) { p = kMixNone; break; }
        p = e & 0xFFFFu;
        cl = e >> 16;
      }
      s_found = i;
      s_exit = p;
      s_exit_class = cl;
      starts[i] = static_cast<uint16_t>(p);
    }
    __syncthreads();
    const uint32_t found = s_found;
    const uint32_t take = found < n_points - done ? found : n_points - done;
    // ---- 4. + 5. batches of one point per thread ----
    for (uint32_t b0 = 0; b0 < take; b0 += kMixBatch) {
      const uint32_t i = b0 + threadIdx.x;
      const bool active = i < take;
      bool bad = false;
      uint32_t g_pos = 0, g_new = 0;  // g_new: (1 << 16) | lead << 8 | trail when this point's record opens a window
      const bool g_first = active && done == 0 && i == 0;
      if (active) {
        uint32_t p = starts[i];
        for (uint32_t t = 0; t < n_tok; ++t) {
          const MixToken& tk = ms.tok[t];
          if (tk.kind == MIX_VAR) {
            long long diff = 0;
            uint8_t nan = 0;
            if (p >= limit) { report_frame_error(L, s_frame, DEV_ERR_TRUNCATED); bad = true; break; }
            if (bytes[p] == 0 && tk.slot.kind != SLOT_INT) { nan = 1; ++p; }
            else {
              const uint32_t n = read_varint(bytes + p, limit - p, &diff, frame_err_word(L, s_frame));
              if (!n) { bad = true; break; }
              p += n;
            }
            vals[static_cast<size_t>(threadIdx.x) * n_var + tk.index] = diff;
            nanflag[static_cast<size_t>(threadIdx.x) * n_var + tk.index] = nan;
          } else if (tk.kind == MIX_GORILLA) {
            g_pos = p;
            uint32_t len = 8;
            if (!g_first) {
              GorHeader h;
              if (p >= limit || !gor_header(bytes + p, limit - p, &h)) { report_frame_error(L, s_frame, DEV_ERR_TRUNCATED); bad = true; break; }
              if (h.kind == 0) len = 1;
              else if (h.kind == 1) len = cls[i] ? cls[i] : 9u;  // reuse (before any window: a 65-bit field, like the reference)
              else {
                len = (13u + h.meaningful + 7u) >> 3;
                g_new = (1u << 16) | (h.lead << 8) | ((64u - h.lead - h.meaningful) & 0xFFu);
              }
            }
            if (p + len > limit) { report_frame_error(L, s_frame, DEV_ERR_TRUNCATED); bad = true; break; }
            p += len;
          } else {
            if (p + tk.size > limit) { report_frame_error(L, s_frame, DEV_ERR_TRUNCATED); bad = true; break; }
            raws[static_cast<size_t>(threadIdx.x) * n_fix + tk.index] = load_raw_bits(bytes + p, tk.size);
            p += tk.size;
          }
        }
      }
      if (__syncthreads_or(bad ? 1 : 0)) return;
      // the window every record sees: the latest "new window" record in front of it (this batch, else the carry)
      uint32_t win_total;
      const uint32_t win_ex = gor_block_last_exclusive(g_new, s_lastscan, &win_total);
      const uint32_t win = win_ex ? win_ex : s_window;
      unsigned long long xres = 0;
      if (active) {
        GorillaState st;
        st.prev_bits = 0;
        st.first = g_first;
        st.leading = win ? ((win >> 8) & 0xFFu) : 255u;
        st.trailing = win ? (win & 0xFFu) : 0u;
        uint64_t v = 0;
        if (!gorilla_decode(st, bytes + g_pos, limit - g_pos, &v)) { report_frame_error(L, s_frame, DEV_ERR_TRUNCATED); bad = true; }
        xres = v;  // previous bits 0: the value IS the residual (the first record: the raw bits)
      }
      if (__syncthreads_or(bad ? 1 : 0)) return;
      uint8_t* point = out + static_cast<size_t>(done + i) * plan.point_step;
      for (uint32_t t = 0; t < n_tok; ++t) {
        const MixToken& tk = ms.tok[t];
        if (tk.kind == MIX_VAR) {
          const long long d = active ? vals[static_cast<size_t>(threadIdx.x) * n_var + tk.index] : 0;
          const bool nan = active && nanflag[static_cast<size_t>(threadIdx.x) * n_var + tk.index] != 0;
          Seg<long long, 1> mine;
          mine.sum[0] = nan ? 0 : d;
          mine.rst = nan ? 1u : 0u;
          Seg<long long, 1> total;
          const Seg<long long, 1> ex = block_seg_exclusive<long long, 1>(mine, sh.seg_sum, sh.seg_rst, &total);
          const long long before = ex.rst ? ex.sum[0] : wadd(ms.carry[tk.index], ex.sum[0]);
          if (active) store_slot_value<long long>(point, tk.slot, nan ? 0 : wadd(before, d), nan);
          __syncthreads();
          if (threadIdx.x == 0) ms.carry[tk.index] = total.rst ? total.sum[0] : wadd(ms.carry[tk.index], total.sum[0]);
        } else if (tk.kind == MIX_XOR || tk.kind == MIX_GORILLA) {
          const bool g = tk.kind == MIX_GORILLA;
          const uint32_t ci = g ? static_cast<uint32_t>(kMaxOps + 3) : tk.index;  // the Gorilla field's carry lives in the last slot
          const unsigned long long r = !active ? 0ull : g ? xres : raws[static_cast<size_t>(threadIdx.x) * n_fix + tk.index];
          unsigned long long total;
          const unsigned long long ex = mix_block_xor_exclusive(r, ms.xscan, &total);
          const unsigned long long v = ms.xcarry[ci] ^ ex ^ r;
          if (active && tk.offset != CLDN_SKIP_STORE_OFFSET) {
            if (g) store_u64(point + tk.offset, v); else store_low_bytes(point + tk.offset, v, tk.size);
          }
          __syncthreads();
          if (threadIdx.x == 0) ms.xcarry[ci] ^= total;
        } else if (active && tk.offset != CLDN_SKIP_STORE_OFFSET) {
          store_low_bytes(point + tk.offset, raws[static_cast<size_t>(threadIdx.x) * n_fix + tk.index], tk.size);
        }
      }
      if (threadIdx.x == 0 && win_total) s_window = win_total;
      __syncthreads();
    }
    done += take;
    const uint32_t end_local = starts[take];
    const uint32_t exit_class = s_exit_class;
    __syncthreads();
    if (done < n_points) {
      if (end_local == kMixNone || end_local <= mis) { if (threadIdx.x == 0) report_frame_error(L, s_frame, DEV_ERR_TRUNCATED); return; }
      t0 = static_cast<uint32_t>(a0 + end_local);
      if (threadIdx.x == 0) s_class = exit_class;
      __syncthreads();
    } else {
      if (end_local == kMixNone) { if (threadIdx.x == 0) report_frame_error(L, s_frame, DEV_ERR_TRUNCATED); return; }
      if (L.stream_end && threadIdx.x == 0) L.stream_end[gc] = static_cast<uint32_t>(a0 + end_local);
    }
  }
  if (n_points == 0 && L.stream_end && threadIdx.x == 0) L.stream_end[gc] = 0;
}

static size_t gorilla_smem_bytes(const Plan& plan) {
  size_t n_var = 0, n_fix = 0;
  for (uint32_t k = 0; k < plan.n_ops; ++k) {
    const RegOp& op = plan.ops[k];
    if (op.kind == OP_GORILLA64) continue;
    if (op.kind == OP_COPY || op.kind == OP_XOR32 || op.kind == OP_XOR64) ++n_fix; else n_var += op.lanes;
  }
  size_t bytes = kGorTile + kMixLook + 32 + kGorBitWords * 4 + kGorClasses * kGorTile * 4;
  bytes += ((kGorTile + 2) * 2 + 15) / 16 * 16 + (kGorTile + 2 + 15) / 16 * 16;
  bytes += kMixBatch * n_var * 8;
  bytes += (kMixBatch * n_var + 15) / 16 * 16;
  bytes += kMixBatch * n_fix * 8 + 64;
  return bytes;
}
static bool gorilla_plan_ok(const Plan& plan) {
  if (plan.n_gorilla != 1 || plan.max_point_bytes > kMixLook) return false;
  const char* e = getenv("CLDN_B200_MIXED_DECODE");
  return !(e && e[0] == 's');
}

// ------------------------------------------------------------------------------------------------------------------
static size_t dec_smem_bytes(bool k32) {
  return kLookBehind + kDecTileBytes + 16 + static_cast<size_t>(kDecTileBytes) * (k32 ? 4 : 8) + kDecTileBytes / 8 +
         sizeof(RunBatch) + 16;
}

// The V5 sections of every chunk (or, redo = true, of the chunks on the redo list), starting at stream_end[]; side = true
// stores into the side arrays (see DecLaunch::side) instead of the rows.
static int launch_sections_only(const DecLaunch& L, cudaStream_t stream, bool side, bool redo) {
  DecLaunch S = L;
  S.sections_only = 1;
  S.side_mode = side ? 1u : 0u;
  S.redo_mode = redo ? 1u : 0u;
  const size_t smem = dec_smem_bytes(false);
  auto k = decode_chunks_kernel<0>;
  if (raise_smem_limit(k, smem) != cudaSuccess) return -1;
  k<<<L.n_chunks_total, kThreads, smem, stream>>>(S);  // redo: CTAs beyond the redo list return at once
  return 1;
}

bool decode_side_plan(const Plan& plan) {
  const char* e = getenv("CLDN_B200_DECODE_SIDE");
  if (e && e[0] == '0') return false;
  if (plan.n_sections == 0 || plan.n_sections > static_cast<uint32_t>(kMaxSideFields) || plan.regular_overlap) return false;
  // Measured (Velodyne XYZIRT, 256 frames): a layout without padding and with ONE section field gains nothing -- the section
  // reader's direct stores cost less than pre-pass + side arrays + merge. Padded layouts (every store of
  // every pass a sector read-modify-write) and several section fields are where writing each row once pays
  if (e == nullptr && plan.n_sections == 1 && decode_fast_whole_rows(plan)) return false;
  uint32_t sum = 0;
  for (uint32_t s = 0; s < plan.n_sections; ++s) {
    const uint32_t b = plan.sections[s].bpv;
    if (!(b == 1 || b == 2 || b == 4 || b == 8)) return false;
    sum += b;
  }
  // the fast reader keeps one tile of section values in 8 KB of shared memory (tiles: 1024 points for <= 4 values per point, else 512)
  const uint32_t tile_points = plan.values_per_point <= 4 ? 1024u : 512u;
  return sum * tile_points <= 8192u;
}
size_t decode_side_bytes(const Plan& plan, uint64_t n_chunks_total, uint64_t side_off[kMaxSideFields]) {
  uint64_t at = 0;
  for (uint32_t s = 0; s < static_cast<uint32_t>(kMaxSideFields); ++s) {
    side_off[s] = at;
    if (s < plan.n_sections) at += ((n_chunks_total * kChunkPoints * plan.sections[s].bpv) + 255u) & ~255ull;
  }
  return static_cast<size_t>(at);
}
bool decode_side_active(const Plan& plan, const DecLaunch& L) {
  return L.side != nullptr && L.n_chunks_total > 0 && L.redo_list != nullptr && L.chunk_desc != nullptr && L.stream_end != nullptr &&
         L.chunk_counter != nullptr && decode_side_plan(plan) && decode_fast_general_plan(plan) &&
         decode_tiles_sequential(L.n_chunks_total) && decode_fast_enabled();
}

int launch_decode(const Plan& plan, const DecLaunch& L, cudaStream_t stream) {
  int launches = 0;
  if (L.n_chunks_total == 0 && L.n_frames == 0) return 0;
  // the chunk-sequential FloatN kernel walks the chunk prefixes itself (CTA 0) while the other CTAs already decode
  // float-varint streams beyond the FloatN-only ones (a FloatN group + scalar lossy floats: Velodyne XYZIRT ...): the fast
  // chunk-sequential reader for large batches, the generic per-chunk kernel for whatever it hands over
  const bool fast_general = L.n_chunks_total > 0 && !plan.floatn_only && L.redo_list != nullptr && L.chunk_desc != nullptr &&
                            decode_fast_general_plan(plan) && decode_tiles_sequential(L.n_chunks_total) && decode_fast_enabled();
  const bool fused_walk = fast_general || (L.n_chunks_total > 0 && L.tile_grid > 0 && L.chunk_desc != nullptr &&
                                           decode_tiles_sequential(L.n_chunks_total) && !plan.regular_overlap);
  if (!fused_walk) {
    walk_chunks_kernel<<<(L.n_frames + 127) / 128, 128, 0, stream>>>(L);
    ++launches;
  }
  if (L.n_chunks_total > 0 && plan.regular_overlap) {
    // overlapping stored fields: the reference's store order (per point, field order, last writer wins) is only kept by
    // the one-thread-per-chunk parser; sections follow in field order like everywhere else
    decode_sequential_kernel<<<(L.n_chunks_total + 31) / 32, 32, 0, stream>>>(L);
    ++launches;
    if (plan.n_sections > 0) {
      DecLaunch S = L;
      S.sections_only = 1;
      const size_t smem = dec_smem_bytes(false);
      auto k = decode_chunks_kernel<0>;
      if (raise_smem_limit(k, smem) != cudaSuccess) return -1;
      k<<<L.n_chunks_total, kThreads, smem, stream>>>(S);
      ++launches;
    }
  } else if (fast_general) {
    int sms = 0, dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    cudaMemsetAsync(L.chunk_counter, 0, 4 * sizeof(uint32_t), stream);
    const bool side = decode_side_active(plan, L);
    if (side) {
      // sections first, into the side arrays; the fast reader writes every row once, section fields included
      if (launch_stream_end(plan, L, stream) < 0 || launch_sections_only(L, stream, true, false) < 0) return -1;
      launches += 2;
    }
    if (launch_decode_fast(plan, L, sms > 0 ? sms : 132, stream) < 0) return -1;
    ++launches;
    {
      DecLaunch R = L;
      R.redo_mode = 1;
      const size_t smem = dec_smem_bytes(false);
      auto k = decode_chunks_kernel<0>;
      if (raise_smem_limit(k, smem) != cudaSuccess) return -1;
      k<<<L.n_chunks_total, kThreads, smem, stream>>>(R);  // CTAs beyond the redo list return at once; regular stream + sections
      ++launches;
    }
    if (plan.n_sections > 0 && !side) {
      if (launch_sections_only(L, stream, false, false) < 0) return -1;
      ++launches;
    }
  } else if (L.n_chunks_total > 0 && L.tile_grid > 0) {
    // FloatN-only regular stream: tile-parallel kernel; V5 sections (if any) by the per-chunk kernel afterwards -- or, large
    // batches in side mode, ahead of it (launch_decode_tiles then runs the merging fast reader and the sections of the
    // chunks it handed to the careful kernel follow)
    const bool side = decode_side_active(plan, L);
    if (side) {
      cudaMemsetAsync(L.chunk_counter, 0, 4 * sizeof(uint32_t), stream);
      if (launch_stream_end(plan, L, stream) < 0 || launch_sections_only(L, stream, true, false) < 0) return -1;
      launches += 2;
    }
    const int n = launch_decode_tiles(plan, L, stream);
    if (n < 0) return -1;
    launches += n;
    if (plan.n_sections > 0) {
      if (launch_sections_only(L, stream, false, side) < 0) return -1;
      ++launches;
    }
  } else if (L.n_chunks_total > 0) {
    const bool varint_ok = plan.all_varint || plan.n_ops == 0;
    if (varint_ok) {
      const int K = static_cast<int>(plan.values_per_point);
      const bool f3 = plan.floatn_only && K == 3, f4 = plan.floatn_only && K == 4;
      const size_t smem = dec_smem_bytes(f3 || f4);
      if (f4) {
        auto k = decode_chunks_kernel<4>;
        if (raise_smem_limit(k, smem) != cudaSuccess) return -1;
        k<<<L.n_chunks_total, kThreads, smem, stream>>>(L);
      } else if (f3) {
        auto k = decode_chunks_kernel<3>;
        if (raise_smem_limit(k, smem) != cudaSuccess) return -1;
        k<<<L.n_chunks_total, kThreads, smem, stream>>>(L);
      } else {
        auto k = decode_chunks_kernel<0>;
        if (raise_smem_limit(k, smem) != cudaSuccess) return -1;
        k<<<L.n_chunks_total, kThreads, smem, stream>>>(L);
      }
      ++launches;
    } else if (plan.all_fixed && plan.n_sections == 0) {
      dim3 grid(kChunkPoints / kThreads / 4, L.n_chunks_total);
      decode_fixed_kernel<<<grid, kThreads, 0, stream>>>(L);
      ++launches;
    } else {
      // raw / XOR fields mixed into the stream: point boundaries by parallel pointer jumping (decode_mixed_kernel);
      // Gorilla fields: one thread per chunk parses the stream like the reference does.
      // V5 sections (if any) are then decoded by the per-chunk section reader from where the stream ended
      if (mixed_plan_ok(plan)) {
        const size_t msmem = mixed_smem_bytes(plan);
        if (raise_smem_limit(decode_mixed_kernel, msmem) != cudaSuccess) return -1;
        decode_mixed_kernel<<<L.n_chunks_total, kThreads, msmem, stream>>>(L);
      } else if (gorilla_plan_ok(plan)) {
        const size_t gsmem = gorilla_smem_bytes(plan);
        if (raise_smem_limit(decode_gorilla_kernel, gsmem) != cudaSuccess) return -1;
        decode_gorilla_kernel<<<L.n_chunks_total, kThreads, gsmem, stream>>>(L);
      } else {
        decode_sequential_kernel<<<(L.n_chunks_total + 31) / 32, 32, 0, stream>>>(L);
      }
      ++launches;
      if (plan.n_sections > 0) {
        DecLaunch S = L;
        S.sections_only = 1;
        const size_t smem = dec_smem_bytes(false);
        auto k = decode_chunks_kernel<0>;
        if (raise_smem_limit(k, smem) != cudaSuccess) return -1;
        k<<<L.n_chunks_total, kThreads, smem, stream>>>(S);
        ++launches;
      }
    }
  }
  count_launch(launches);
  return launches;
}

}  // namespace cldn
