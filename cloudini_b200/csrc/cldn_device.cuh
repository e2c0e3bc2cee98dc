// Device-side building blocks shared by the encode / decode / V5-section kernels (sm_90a).
// Arithmetic contract: SURVEY.md Appendix B; each helper cites the reference expression it must match bit-for-bit.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "cldn_plan.h"

namespace cldn {

constexpr int kThreads = 256;  // CTA size of all streaming kernels

// Device error word (one per handle). First error wins; host maps it to CLDN_ERR_CORRUPT_DATA + message.
enum DevError : uint32_t {
  DEV_OK = 0,
  DEV_ERR_TRUNCATED = 1,       // "Truncated encoded data" (v4_codec.cpp:103) / decodeVarint truncated (encoding_utils.hpp:123)
  DEV_ERR_VARINT_OVERFLOW = 2, // encoding_utils.hpp:128,135
  DEV_ERR_NAN_MARKER = 3,      // "unexpected NaN marker" encoding_utils.hpp:141-143
  DEV_ERR_TRAILING = 4,        // "V5 chunk has trailing bytes after decode" v5_codec.cpp:1008-1010
  DEV_ERR_BAD_MODE = 5,        // v5_codec.cpp:772-775
  DEV_ERR_PALETTE = 6,         // v5_codec.cpp:797-823
  DEV_ERR_RLE = 7,             // v5_codec.cpp:836-877
  DEV_ERR_CHUNK_SIZE = 8,      // "Invalid chunk size found while decoding" cloudini.cpp:653-655
  DEV_ERR_CHUNK_COUNT = 9,     // cloudini.cpp:648-650,662-664
  DEV_ERR_OUTPUT_SMALL = 10,
  DEV_ERR_LZ4 = 12,                  // "LZ4 decompression failed" codec_common.cpp:279-281
  DEV_ERR_ENCODE_OUTPUT_SMALL = 11,  // "Output buffer too small for uncompressed chunk" chunk_writer.cpp:33-35
  DEV_ERR_ZSTD = 13,                 // "ZSTD decompression failed" codec_common.cpp:290-293
};

__device__ __forceinline__ void report_error(uint32_t* err, uint32_t code) { atomicCAS(err, 0u, code); }

// ---- relaxed / acquire-release global accessors for the tile status words ---------------------------------------
__device__ __forceinline__ uint64_t ld_relaxed_u64(const uint64_t* p) {
  uint64_t v;
  asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_relaxed_u64(uint64_t* p, uint64_t v) {
  asm volatile("st.relaxed.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_u32(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_u32(uint32_t* p, uint32_t v) {
  asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

// ---- unaligned little-endian field access (PointCloud2 layouts such as step 22/26 are not 4-byte aligned) -------
__device__ __forceinline__ uint32_t load_u32(const uint8_t* p) {
  const uintptr_t a = reinterpret_cast<uintptr_t>(p);
  if ((a & 3u) == 0) return *reinterpret_cast<const uint32_t*>(p);
  if ((a & 1u) == 0) {
    const uint16_t* h = reinterpret_cast<const uint16_t*>(p);
    return static_cast<uint32_t>(h[0]) | (static_cast<uint32_t>(h[1]) << 16);
  }
  return static_cast<uint32_t>(p[0]) | (static_cast<uint32_t>(p[1]) << 8) | (static_cast<uint32_t>(p[2]) << 16) |
         (static_cast<uint32_t>(p[3]) << 24);
}
__device__ __forceinline__ uint64_t load_u64(const uint8_t* p) {
  const uintptr_t a = reinterpret_cast<uintptr_t>(p);
  if ((a & 7u) == 0) return *reinterpret_cast<const uint64_t*>(p);
  return static_cast<uint64_t>(load_u32(p)) | (static_cast<uint64_t>(load_u32(p + 4)) << 32);
}
__device__ __forceinline__ uint32_t load_u16(const uint8_t* p) {
  const uintptr_t a = reinterpret_cast<uintptr_t>(p);
  if ((a & 1u) == 0) return *reinterpret_cast<const uint16_t*>(p);
  return static_cast<uint32_t>(p[0]) | (static_cast<uint32_t>(p[1]) << 8);
}
__device__ __forceinline__ void store_u32(uint8_t* p, uint32_t v) {
  const uintptr_t a = reinterpret_cast<uintptr_t>(p);
  if ((a & 3u) == 0) { *reinterpret_cast<uint32_t*>(p) = v; return; }
  if ((a & 1u) == 0) {
    uint16_t* h = reinterpret_cast<uint16_t*>(p);
    h[0] = static_cast<uint16_t>(v); h[1] = static_cast<uint16_t>(v >> 16);
    return;
  }
  p[0] = static_cast<uint8_t>(v); p[1] = static_cast<uint8_t>(v >> 8);
  p[2] = static_cast<uint8_t>(v >> 16); p[3] = static_cast<uint8_t>(v >> 24);
}
__device__ __forceinline__ void store_u16(uint8_t* p, uint32_t v) {
  const uintptr_t a = reinterpret_cast<uintptr_t>(p);
  if ((a & 1u) == 0) { *reinterpret_cast<uint16_t*>(p) = static_cast<uint16_t>(v); return; }
  p[0] = static_cast<uint8_t>(v); p[1] = static_cast<uint8_t>(v >> 8);
}
__device__ __forceinline__ void store_u64(uint8_t* p, uint64_t v) {
  const uintptr_t a = reinterpret_cast<uintptr_t>(p);
  if ((a & 7u) == 0) { *reinterpret_cast<uint64_t*>(p) = v; return; }
  store_u32(p, static_cast<uint32_t>(v));
  store_u32(p + 4, static_cast<uint32_t>(v >> 32));
}
// Stores the low `bytes` (1,2,4,8) bytes of v: writeRawBitsToPoint (v5_codec.cpp:121-123), FieldDecoderInt (field_decoder.hpp:93-95).
__device__ __forceinline__ void store_low_bytes(uint8_t* p, uint64_t v, int bytes) {
  if (bytes == 4) store_u32(p, static_cast<uint32_t>(v));
  else if (bytes == 2) store_u16(p, static_cast<uint32_t>(v));
  else if (bytes == 8) store_u64(p, v);
  else p[0] = static_cast<uint8_t>(v);
}
// ToInt64<T> (encoding_utils.hpp:69-73) / readIntAsI64 (v5_codec.cpp:97-115): sign- or zero-extend by field type.
__device__ __forceinline__ int64_t load_int_as_i64(const uint8_t* p, uint8_t type) {
  switch (type) {
    case CLDN_INT16: return static_cast<int16_t>(load_u16(p));
    case CLDN_UINT16: return static_cast<int64_t>(load_u16(p));
    case CLDN_INT32: return static_cast<int32_t>(load_u32(p));
    case CLDN_UINT32: return static_cast<int64_t>(load_u32(p));
    case CLDN_INT8: return static_cast<int8_t>(p[0]);
    case CLDN_UINT8: return static_cast<int64_t>(p[0]);
    default: return static_cast<int64_t>(load_u64(p));  // INT64 / UINT64 (reinterpreted)
  }
}
// readRawBits (v5_codec.cpp:117-121)
__device__ __forceinline__ uint64_t load_raw_bits(const uint8_t* p, int bytes) {
  if (bytes == 4) return load_u32(p);
  if (bytes == 2) return load_u16(p);
  if (bytes == 8) return load_u64(p);
  return p[0];
}

// ---- quantisation ----------------------------------------------------------------------------------------------
// cast_vector4f_to_vector4i (intrinsics.hpp:288-293): _mm_round_ps(NEAREST) + _mm_cvtps_epi32 -> ties-to-even int32,
// "integer indefinite" 0x80000000 for NaN / +-inf / |s| >= 2^31. cvt.rni.s32.f32 saturates and maps NaN to 0, so
// everything that is not provably < 2^31 is forced to INT_MIN (negative overflow already saturates to INT_MIN).
__device__ __forceinline__ int32_t quant_i32_x86(float v, float mul) {
  const float s = __fmul_rn(v, mul);  // _mm_mul_ps: IEEE RN, never contracted into an FMA
  const int32_t q = __float2int_rn(s);
  return (s < 2147483648.0f) ? q : static_cast<int32_t>(0x80000000u);
}
// static_cast<int64_t>(std::round(v * mul)) (field_encoder.hpp:351): half away from zero, then cvttss2si whose
// out-of-range / NaN result is the 64-bit "integer indefinite" 0x8000000000000000.
__device__ __forceinline__ int64_t quant_i64_f32(float v, float mul) {
  const float r = roundf(__fmul_rn(v, mul));
  if (!(r < 9223372036854775808.0f) || r < -9223372036854775808.0f) return static_cast<int64_t>(0x8000000000000000ull);
  return __float2ll_rz(r);
}
__device__ __forceinline__ int64_t quant_i64_f64(double v, double mul) {
  const double r = round(__dmul_rn(v, mul));
  if (!(r < 9223372036854775808.0) || r < -9223372036854775808.0) return static_cast<int64_t>(0x8000000000000000ull);
  return __double2ll_rz(r);
}

// ---- zigzag + varint (encodeVarint64, encoding_utils.hpp:55-67) --------------------------------------------------
__device__ __forceinline__ uint64_t zigzag_plus1(int64_t v) {
  return ((static_cast<uint64_t>(v) << 1) ^ static_cast<uint64_t>(v >> 63)) + 1ull;  // wraps to 0 for INT64_MIN, like the reference
}
__device__ __forceinline__ int varint_len(uint64_t u) {
  const int bits = 64 - __clzll(static_cast<long long>(u | 1ull));
  return (bits + 6) / 7;
}
// plain LEB128 length (appendUVarint, v5_codec.cpp:160-174)
__device__ __forceinline__ int uvarint_len(uint64_t u) { return varint_len(u); }

// Inverse zigzag (encoding_utils.hpp:144-146) applied to (uval - 1).
__device__ __forceinline__ int64_t unzigzag(uint64_t uval_minus1) {
  return static_cast<int64_t>((uval_minus1 >> 1) ^ (0ull - (uval_minus1 & 1ull)));
}

// ---- sinks: the same per-point op code runs once to count bytes and once to emit them ---------------------------
struct CountSink {
  uint32_t n = 0;
  __device__ __forceinline__ void put_varint(uint64_t u) { n += varint_len(u); }
  __device__ __forceinline__ void put_byte(uint8_t) { n += 1; }
  __device__ __forceinline__ void put_raw(const uint8_t*, int size) { n += size; }
  __device__ __forceinline__ void put_le(uint64_t, int size) { n += size; }
};
struct ByteSink {
  uint8_t* p;
  __device__ __forceinline__ void put_varint(uint64_t u) {
    while (u > 0x7Full) {
      *p++ = static_cast<uint8_t>((u & 0x7Full) | 0x80ull);
      u >>= 7;
    }
    *p++ = static_cast<uint8_t>(u);
  }
  __device__ __forceinline__ void put_byte(uint8_t b) { *p++ = b; }
  __device__ __forceinline__ void put_raw(const uint8_t* src, int size) {
    for (int i = 0; i < size; ++i) *p++ = src[i];
  }
  __device__ __forceinline__ void put_le(uint64_t v, int size) {  // low `size` bytes, little endian
    for (int i = 0; i < size; ++i) *p++ = static_cast<uint8_t>(v >> (8 * i));
  }
};

// ---- Gorilla / Chimp-style bit packing of one FLOAT64 (field_encoder.hpp:157-312) -----------------------------------
// Bits are appended LSB-first and every value is flushed to a byte boundary. State = previous bits + the window
// (leading, trailing) of the last "new window" record; leading == 255 is the reference's "no window yet" sentinel.
struct GorillaState {
  uint64_t prev_bits;
  uint32_t leading, trailing;
  bool first;
  __device__ __forceinline__ void reset() { prev_bits = 0; leading = 255u; trailing = 0; first = true; }
};
struct BitAcc {  // up to 128 bits
  uint64_t lo = 0, hi = 0;
  uint32_t n = 0;
  __device__ __forceinline__ void put(uint64_t bits, uint32_t nbits) {
    if (nbits < 64u) bits &= (1ull << nbits) - 1ull;
    if (n < 64u) {
      lo |= bits << n;
      if (n + nbits > 64u) hi |= bits >> (64u - n);  // n >= 1 here
    } else {
      hi |= bits << (n - 64u);
    }
    n += nbits;
  }
};
// Encodes `cur`; writes the record to out[0..len) and returns len (1..10).
__device__ __forceinline__ uint32_t gorilla_encode(GorillaState& st, uint64_t cur, uint8_t* out) {
  BitAcc a;
  if (st.first) {
    st.first = false;
    st.prev_bits = cur;
    a.put(cur, 64);
  } else {
    const uint64_t x = cur ^ st.prev_bits;
    st.prev_bits = cur;
    if (x == 0) {
      a.put(0, 1);
    } else {
      a.put(1, 1);
      const uint32_t leading = static_cast<uint32_t>(__clzll(static_cast<long long>(x)));
      const uint32_t trailing = static_cast<uint32_t>(__ffsll(static_cast<long long>(x)) - 1);
      if (st.leading != 255u && leading >= st.leading && trailing >= st.trailing) {
        a.put(0, 1);
        a.put(x >> st.trailing, 64u - st.leading - st.trailing);
      } else {
        a.put(1, 1);
        const uint32_t stored = leading > 31u ? 31u : leading;
        const uint32_t meaningful = 64u - stored - trailing;
        a.put(stored, 5);
        a.put(meaningful - 1u, 6);
        a.put(x >> trailing, meaningful);
        st.leading = stored;
        st.trailing = trailing;
      }
    }
  }
  const uint32_t bytes = (a.n + 7u) >> 3;
  for (uint32_t i = 0; i < bytes; ++i) out[i] = static_cast<uint8_t>(i < 8u ? (a.lo >> (8u * i)) : (a.hi >> (8u * (i - 8u))));
  return bytes;
}
// The next <= 10 bytes of the stream (one Gorilla record is at most 2 + 5 + 6 + 64 = 77 bits) as a 128-bit window;
// bit fields are then cut out of registers instead of being gathered bit by bit from memory.
struct BitWindow {
  uint64_t lo = 0, hi = 0;
  uint32_t avail;  // bytes that really exist behind p
  uint32_t bp = 0; // bit position of the next field
  __device__ __forceinline__ BitWindow(const uint8_t* p, uint32_t avail_) : avail(avail_) {
    if (avail_ >= 10u) {
      lo = load_u64(p);
      hi = load_u16(p + 8);
    } else {
#pragma unroll
      for (uint32_t b = 0; b < 8u; ++b) if (b < avail_) lo |= static_cast<uint64_t>(p[b]) << (8u * b);
      if (avail_ > 8u) hi = p[8];
    }
  }
  // Reads nbits (<= 64). Returns false when the field does not lie inside the available bytes (same test, in the same
  // order, as the reference's bit reader: truncated input is reported at the first field that crosses the end).
  __device__ __forceinline__ bool read(uint32_t nbits, uint64_t* out) {
    if ((bp + nbits + 7u) / 8u > avail) return false;
    uint64_t v = bp == 0 ? lo : (bp < 64u ? ((lo >> bp) | (hi << (64u - bp))) : (hi >> (bp - 64u)));
    if (nbits < 64u) v &= (1ull << nbits) - 1ull;
    bp += nbits;
    *out = v;
    return true;
  }
};
// Decodes one value (field_decoder.hpp:257-300). Returns the bytes consumed, 0 when the input is truncated / malformed.
__device__ __forceinline__ uint32_t gorilla_decode(GorillaState& st, const uint8_t* p, uint32_t avail, uint64_t* value) {
  BitWindow w(p, avail);
  uint64_t v;
  if (st.first) {
    st.first = false;
    if (!w.read(64, &v)) return 0;
    st.prev_bits = v;
  } else {
    uint64_t flag;
    if (!w.read(1, &flag)) return 0;
    if (flag == 0) {
      v = st.prev_bits;
    } else {
      uint64_t control, bits, x;
      if (!w.read(1, &control)) return 0;
      if (control == 0) {
        // uint8_t(64 - prev_leading - prev_trailing) (field_decoder.hpp:274). After a new-window record this is that
        // record's bit count again (1..64) whatever the stored leading / trailing were; before any window the sentinel
        // 255 makes it 65: the reference then reads a 65-bit field and keeps its low 64 bits (getBits, :213-241).
        const uint32_t meaningful = (64u - st.leading - st.trailing) & 0xFFu;
        if (meaningful > 65u) return 0;  // unreachable with the states this decoder can be in
        if (!w.read(meaningful > 64u ? 64u : meaningful, &bits)) return 0;
        if (meaningful > 64u) { uint64_t dropped; if (!w.read(1, &dropped)) return 0; }
        // `bits << prev_trailing_` with a uint8_t count: a forged new-window record (leading + bits > 64) leaves a count
        // of 192..255 behind; the reference's shift is the x86 one (count mod 64), which is what its blobs decode to
        x = bits << (st.trailing & 63u);
      } else {
        uint64_t lead, m1;
        if (!w.read(5, &lead) || !w.read(6, &m1)) return 0;
        const uint32_t meaningful = static_cast<uint32_t>(m1) + 1u;
        if (!w.read(meaningful, &bits)) return 0;
        const uint32_t trailing = (64u - static_cast<uint32_t>(lead) - meaningful) & 0xFFu;
        x = bits << (trailing & 63u);  // see above: x86 shift semantics for forged records (trailing >= 64)
        st.leading = static_cast<uint32_t>(lead);
        st.trailing = trailing;
      }
      v = x ^ st.prev_bits;
      st.prev_bits = v;
    }
  }
  *value = v;
  return (w.bp + 7u) >> 3;
}

// ---- block-wide exclusive scan of one uint32 per thread (kThreads threads) --------------------------------------
// Returns the exclusive prefix; *total receives the block sum. `scratch` = 8+1 uint32 in shared memory.
__device__ __forceinline__ uint32_t block_exclusive_scan(uint32_t v, uint32_t* scratch, uint32_t* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint32_t inc = v;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const uint32_t t = __shfl_up_sync(0xffffffffu, inc, d);
    if (lane >= d) inc += t;
  }
  if (lane == 31) scratch[warp] = inc;
  __syncthreads();
  if (warp == 0) {
    uint32_t w = (lane < kThreads / 32) ? scratch[lane] : 0;
    uint32_t winc = w;
#pragma unroll
    for (int d = 1; d < kThreads / 32; d <<= 1) {
      const uint32_t t = __shfl_up_sync(0xffffffffu, winc, d);
      if (lane >= d) winc += t;
    }
    if (lane < kThreads / 32) scratch[lane] = winc - w;
    if (lane == kThreads / 32 - 1) scratch[kThreads / 32] = winc;
  }
  __syncthreads();
  const uint32_t res = scratch[warp] + inc - v;
  *total = scratch[kThreads / 32];
  return res;
}

// The same for a CTA of NT threads (NT a multiple of 32, <= 1024). `scratch` = NT/32 + 1 words.
template <int NT>
__device__ __forceinline__ uint32_t block_exclusive_scan_n(uint32_t v, uint32_t* scratch, uint32_t* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint32_t inc = v;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const uint32_t t = __shfl_up_sync(0xffffffffu, inc, d);
    if (lane >= d) inc += t;
  }
  if (lane == 31) scratch[warp] = inc;
  __syncthreads();
  uint32_t before = 0, all = 0;
#pragma unroll
  for (int w = 0; w < NT / 32; ++w) {
    const uint32_t c = scratch[w];
    if (w < warp) before += c;
    all += c;
  }
  __syncthreads();  // scratch may be reused at once
  *total = all;
  return before + inc - v;
}

// cp.async (LDGSTS): 16 bytes global -> shared without a register round trip; groups complete in commit order
__device__ __forceinline__ void async_copy16(void* smem_dst, const void* gmem_src) {
#ifdef CLDN_CUSIM
  *reinterpret_cast<uint4*>(smem_dst) = *reinterpret_cast<const uint4*>(gmem_src);
#else
  const uint32_t d = static_cast<uint32_t>(__cvta_generic_to_shared(smem_dst));
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(d), "l"(gmem_src) : "memory");
#endif
}
__device__ __forceinline__ void async_commit() {
#ifndef CLDN_CUSIM
  asm volatile("cp.async.commit_group;" ::: "memory");
#endif
}
__device__ __forceinline__ void async_wait_all_but_last() {
#ifndef CLDN_CUSIM
  asm volatile("cp.async.wait_group 1;" ::: "memory");
#endif
}
__device__ __forceinline__ void async_wait_all() {
#ifndef CLDN_CUSIM
  asm volatile("cp.async.wait_group 0;" ::: "memory");
#endif
}
// ---- tile status word for the decoupled look-back ---------------------------------------------------------------
// [63:62] flag (0 = invalid, 1 = tile aggregate, 2 = inclusive prefix)   [61:40] launch epoch   [39:0] byte count
constexpr uint64_t kFlagAgg = 1ull, kFlagIncl = 2ull;
__device__ __forceinline__ uint64_t pack_status(uint64_t flag, uint32_t epoch, uint64_t value) {
  return (flag << 62) | (static_cast<uint64_t>(epoch & 0x3FFFFFu) << 40) | (value & 0xFFFFFFFFFFull);
}
__device__ __forceinline__ uint32_t status_flag(uint64_t s, uint32_t epoch) {
  return (static_cast<uint32_t>(s >> 40) & 0x3FFFFFu) == (epoch & 0x3FFFFFu) ? static_cast<uint32_t>(s >> 62) : 0u;
}
__device__ __forceinline__ uint64_t status_value(uint64_t s) { return s & 0xFFFFFFFFFFull; }

// Warp-wide decoupled look-back (executed by one full warp). `first` = global index of the first tile of the scan
// domain (frame), `me` = this tile. Publishes the aggregate, resolves the exclusive prefix, publishes the inclusive
// prefix. Tiles are dispatched in increasing blockIdx order, so every predecessor is resident or finished.
__device__ __forceinline__ uint64_t tile_lookback(uint64_t* status, uint32_t first, uint32_t me, uint32_t epoch,
                                                  uint64_t aggregate) {
  const int lane = threadIdx.x & 31;
  if (me == first) {
    if (lane == 0) st_relaxed_u64(status + me, pack_status(kFlagIncl, epoch, aggregate));
    return 0;
  }
  if (lane == 0) st_relaxed_u64(status + me, pack_status(kFlagAgg, epoch, aggregate));
  uint64_t exclusive = 0;
  int64_t idx = static_cast<int64_t>(me) - 1;
  while (true) {
    const int64_t mine = idx - lane;
    uint64_t s = pack_status(kFlagIncl, epoch, 0);  // virtual tiles before `first` contribute an inclusive 0
    if (mine >= static_cast<int64_t>(first)) {
      do { s = ld_relaxed_u64(status + mine); } while (status_flag(s, epoch) == 0);
    }
    const uint32_t incl_mask = __ballot_sync(0xffffffffu, status_flag(s, epoch) == kFlagIncl);
    const int stop = incl_mask ? (__ffs(incl_mask) - 1) : 31;  // nearest predecessor holding an inclusive prefix
    uint64_t v = (lane <= stop) ? status_value(s) : 0;
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(0xffffffffu, v, d);
    exclusive += v;
    if (incl_mask) break;
    idx -= 32;
  }
  if (lane == 0) st_relaxed_u64(status + me, pack_status(kFlagIncl, epoch, exclusive + aggregate));
  return exclusive;
}

// The same look-back as a resumable state machine (one full warp): begin() publishes the aggregate, issue() requests
// the status words of the current 32-tile window, eval() consumes them if every tile of the window has published at
// least its aggregate (otherwise the window is simply asked for again later), finish() blocks until the exclusive
// prefix is known and publishes the inclusive one. The caller interleaves issue()/eval() with useful work so that the
// wait for the slowest predecessor does not stall the CTA.
struct LookbackPoll {
  int64_t idx;         // nearest tile not yet accounted for
  uint64_t exclusive;  // sum of the tiles in (idx, me)
  uint64_t s;          // this lane's status word in flight
  bool done;
  bool published = false;   // poll_once() already wrote the inclusive prefix

  // `publish` = false: another warp of the CTA publishes this tile's words; this warp only resolves the prefix for itself
  __device__ __forceinline__ void begin(uint64_t* status, uint32_t first, uint32_t me, uint32_t epoch, uint64_t aggregate, bool publish = true) {
    const int lane = threadIdx.x & 31;
    exclusive = 0;
    idx = static_cast<int64_t>(me) - 1;
    done = (me == first);
    published = false;
    s = 0;
    if (publish && lane == 0) st_relaxed_u64(status + me, pack_status(done ? kFlagIncl : kFlagAgg, epoch, aggregate));
  }
  __device__ __forceinline__ void issue(const uint64_t* status, uint32_t first, uint32_t epoch) {
    if (done) return;
    const int64_t mine = idx - (threadIdx.x & 31);
    s = pack_status(kFlagIncl, epoch, 0);  // virtual tiles before `first` contribute an inclusive 0
    if (mine >= static_cast<int64_t>(first)) s = ld_relaxed_u64(status + mine);
  }
  __device__ __forceinline__ void eval(uint32_t epoch) {
    if (done) return;
    const int lane = threadIdx.x & 31;
    const uint32_t flag = status_flag(s, epoch);
    if (!__all_sync(0xffffffffu, flag != 0u)) return;  // somebody in the window has not published yet: ask again later
    const uint32_t incl_mask = __ballot_sync(0xffffffffu, flag == kFlagIncl);
    const int stop = incl_mask ? (__ffs(incl_mask) - 1) : 31;
    uint64_t v = (lane <= stop) ? status_value(s) : 0;
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(0xffffffffu, v, d);
    exclusive += v;
    if (incl_mask) done = true; else idx -= 32;
  }
  // One non-blocking step for a warp that has other work between polls: evaluates the words asked for by the last issue(),
  // publishes this tile's inclusive prefix the moment it is known (successors stop walking here), else asks again.
  __device__ __forceinline__ void poll_once(uint64_t* status, uint32_t first, uint32_t me, uint32_t epoch, uint64_t aggregate) {
    if (done) return;
    eval(epoch);
    if (done) {
      if (me != first && (threadIdx.x & 31) == 0) st_relaxed_u64(status + me, pack_status(kFlagIncl, epoch, exclusive + aggregate));
      published = true;
    } else {
      issue(status, first, epoch);
    }
  }
  __device__ __forceinline__ uint64_t finish(uint64_t* status, uint32_t first, uint32_t me, uint32_t epoch, uint64_t aggregate, bool publish = true) {
    const bool was_first = (me == first);
    while (!done) {
      issue(status, first, epoch);
      eval(epoch);
    }
    if (publish && !published && !was_first && (threadIdx.x & 31) == 0) st_relaxed_u64(status + me, pack_status(kFlagIncl, epoch, exclusive + aggregate));
    return exclusive;
  }
};

// Spins until tile `t` has published its inclusive prefix and returns it (one thread).
__device__ __forceinline__ uint64_t wait_inclusive(const uint64_t* status, uint32_t t, uint32_t epoch) {
  uint64_t s;
  do { s = ld_relaxed_u64(status + t); } while (status_flag(s, epoch) != kFlagIncl);
  return status_value(s);
}

// ---- staged tile -> global copy -----------------------------------------------------------------------------------
// Copies `n` bytes from shared memory (`stage`, 16-byte aligned, readable up to n+16) to an arbitrarily aligned global
// address with 16-byte coalesced stores for the aligned body and byte stores for the <=15-byte head and tail.
__device__ __forceinline__ void copy_stage_to_global(const uint8_t* stage, uint32_t n, uint8_t* g) {
  const uint32_t a = static_cast<uint32_t>(reinterpret_cast<uintptr_t>(g) & 15u);
  uint32_t head = (16u - a) & 15u;
  if (head > n) head = n;
  const uint32_t nvec = (n - head) >> 4;
  const uint32_t tail_begin = head + (nvec << 4);
  if (threadIdx.x < head) g[threadIdx.x] = stage[threadIdx.x];
  if (threadIdx.x >= 32 && threadIdx.x - 32 < n - tail_begin) {
    g[tail_begin + threadIdx.x - 32] = stage[tail_begin + threadIdx.x - 32];
  }
  const uint32_t sh = (head & 3u) * 8u;
  const uint32_t* w = reinterpret_cast<const uint32_t*>(stage + (head & ~3u));
  uint4* gv = reinterpret_cast<uint4*>(g + head);
  if (sh == 0) {
    for (uint32_t j = threadIdx.x; j < nvec; j += blockDim.x) {
      const uint32_t* q = w + 4 * j;
      gv[j] = make_uint4(q[0], q[1], q[2], q[3]);
    }
  } else {
    for (uint32_t j = threadIdx.x; j < nvec; j += blockDim.x) {
      const uint32_t* q = w + 4 * j;
      const uint32_t w0 = q[0], w1 = q[1], w2 = q[2], w3 = q[3], w4 = q[4];
      gv[j] = make_uint4(__funnelshift_r(w0, w1, sh), __funnelshift_r(w1, w2, sh), __funnelshift_r(w2, w3, sh),
                         __funnelshift_r(w3, w4, sh));
    }
  }
}

}  // namespace cldn
