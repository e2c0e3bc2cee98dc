// Stage 2 on the device, ZSTD decompression (RFC 8878). Cloudini compresses every chunk with ZSTD_compress(..., 1) by
// default (codec_common.cpp:241-250); this file turns such chunk bodies back into stage-1 bytes without leaving HBM.
//
// Contract: for one chunk body, the result equals ZSTD_decompress(slot, body_cap, body, csize) of libzstd 1.5 -- the same
// bytes whenever it succeeds, and a failure exactly when it fails, damaged input included. Where libzstd is more lenient
// than the RFC, the decoder follows libzstd, because the host-pointer API used to call it and must not change behaviour:
//   * Huffman tables of up to 12 bits are accepted (the RFC says 11);
//   * raw / RLE blocks are not held to the 128 KB block maximum, compressed blocks only by their compressed size;
//     window logs up to 31 are accepted (ZSTD_decompress has no window limit of its own);
//   * the sequence bitstream is read like libzstd's 64-bit bit container (it also updates the FSE states after the last
//     sequence, and only an under-consumed stream is an error), so bits read past the end give what libzstd reads;
//   * 4-stream Huffman literals that libzstd's x86-64 fast loop takes need no end mark and need not be consumed exactly.
//     Not modelled: where that loop stops and refuses a stream that read more than 8 bytes before its own start, so a
//     rare damaged block (about 1 in 3000 damaged frames in tests/test_cusim_zstd.py) is accepted here, refused there.
// Formats: one or more frames and skippable frames per chunk, every header layout, content checksums (XXH64), raw / RLE /
// compressed blocks, raw / RLE / Huffman / treeless literals with 1 or 4 streams, predefined / RLE / FSE / repeat
// sequence tables, repeat offsets. Not supported: dictionaries (a Dictionary_ID other than 0 is an error, as without a
// dictionary in libzstd) and the legacy pre-1.0 formats.
//
//  layout     one warp per chunk (grid-stride over the chunk table of the LZ4 path); the Huffman table (4096 entries) and
//             the LL / OF / ML FSE tables live in shared memory per warp, the block's literals in a global scratch region
//             per warp (<= 128 KB).
//  parsing    frame, block, literals and sequence headers are parsed by all lanes in lock step (uniform registers);
//             what needs a table or an array -- Huffman weights, FSE headers, table construction -- is done by lane 0,
//             which publishes its result through shared memory.
//  literals   Huffman streams: lanes 0..3 decode the four streams of a block at the same time (lane 0 the single stream).
//  sequences  decoded by every lane in lock step (the same bits, the same table entries), executed by the warp: literal
//             bytes with 16-byte stores, matches in rounds of `offset` bytes (a pattern for offsets below 32).
#include <stdint.h>

#include "cldn_device.cuh"
#include "cldn_kernels.h"
#include "cldn_stage2.cuh"

namespace cldn {

constexpr int kZsThreads = 64;  // 2 warps = 2 chunks per CTA (about 15 KB of tables each)
constexpr int kZsWarps = kZsThreads / 32;
constexpr uint32_t kZsBad = 0xFFFFFFFFu;
constexpr uint32_t kZsBlockMax = 131072u;  // Block_Maximum_Size
constexpr uint32_t kZsHufLogMax = 12u;
constexpr uint32_t kZsWindowLogMax = 31u;  // frame header check of ZSTD_getFrameHeader (64-bit builds)

__constant__ int16_t kZsLLNorm[36] = {4, 3, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 1, 1, 1, 2, 2, 2, 2, 2, 2, 2, 2, 2, 3, 2, 1, 1, 1, 1, 1, -1, -1, -1, -1};
__constant__ int16_t kZsMLNorm[53] = {1, 4, 3, 2, 2, 2, 2, 2, 2, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1,
                                      1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, -1, -1, -1, -1, -1, -1, -1};
__constant__ int16_t kZsOFNorm[29] = {1, 1, 1, 1, 1, 1, 2, 2, 2, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, -1, -1, -1, -1, -1};
__constant__ uint32_t kZsLLBase[36] = {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16, 18, 20, 22, 24, 28, 32, 40, 48, 64,
                                       128, 256, 512, 1024, 2048, 4096, 8192, 16384, 32768, 65536};
__constant__ uint8_t kZsLLBits[36] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 3, 3, 4, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16};
__constant__ uint32_t kZsMLBase[53] = {3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16, 17, 18, 19, 20, 21, 22, 23, 24, 25, 26, 27, 28, 29, 30, 31, 32, 33, 34,
                                       35, 37, 39, 41, 43, 47, 51, 59, 67, 83, 99, 131, 259, 515, 1027, 2051, 4099, 8195, 16387, 32771, 65539};
__constant__ uint8_t kZsMLBits[53] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0,
                                      1, 1, 1, 1, 2, 2, 3, 3, 4, 4, 5, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16};

// FSE decoding table entry: symbol | nbBits << 8 | next-state base << 16
struct ZsSmem {
  uint16_t huf[1u << kZsHufLogMax];  // symbol << 8 | code length
  uint32_t seq[3][512];              // LL, OF, ML
  uint32_t wfse[64];                 // Huffman weights (table log <= 6)
  uint8_t wgt[256];
  uint32_t res[8];                   // lane 0 (or lanes 0..3) -> warp
};

__device__ __forceinline__ uint32_t zs_highbit(uint32_t v) { return 31u - static_cast<uint32_t>(__clz(static_cast<int>(v))); }
__device__ __forceinline__ uint32_t zs_rd16(const uint8_t* p) { return static_cast<uint32_t>(p[0]) | (static_cast<uint32_t>(p[1]) << 8); }
__device__ __forceinline__ uint32_t zs_rd24(const uint8_t* p) { return zs_rd16(p) | (static_cast<uint32_t>(p[2]) << 16); }
__device__ __forceinline__ uint32_t zs_rd32(const uint8_t* p) { return zs_rd24(p) | (static_cast<uint32_t>(p[3]) << 24); }
__device__ __forceinline__ uint64_t zs_rd64(const uint8_t* p) { return load_u64(p); }  // reads [p, p + 8) only
// 8 bytes at off of a range of n bytes: through the aligned words covering them (two or three loads) while those stay
// inside the range, else byte-exact
__device__ __forceinline__ uint64_t zs_rd64_in(const uint8_t* base, uint32_t off, uint32_t n) {
  if (off + 11u <= n) {
    const uint2 v = lz_load64(base + off);
    return static_cast<uint64_t>(v.x) | (static_cast<uint64_t>(v.y) << 32);
  }
  return load_u64(base + off);
}

// ---- backward bitstream, read as libzstd's 64-bit BIT_DStream_t reads it ----------------------------------------------
struct ZsBits {
  uint64_t c;           // container: the 8 bytes at start + off (fewer for a short stream)
  uint32_t used;        // bits of the container consumed, from the top
  uint32_t off;
  uint32_t n;           // bytes from start to the end of the stream
  const uint8_t* start;
};
enum : int { ZS_UNFINISHED = 0, ZS_END_OF_BUFFER = 1, ZS_COMPLETED = 2, ZS_OVERFLOW = 3 };

__device__ __forceinline__ bool zs_bits_init(ZsBits& b, const uint8_t* src, uint32_t n) {
  if (n < 1u) return false;
  const uint32_t last = src[n - 1];
  if (last == 0u) return false;  // no end mark
  b.start = src;
  b.n = n;
  if (n >= 8u) {
    b.off = n - 8u;
    b.c = zs_rd64(src + b.off);
    b.used = 8u - zs_highbit(last);
  } else {
    b.off = 0;
    uint64_t c = 0;
    for (uint32_t k = 0; k < n; ++k) c |= static_cast<uint64_t>(src[k]) << (8u * k);
    b.c = c;
    b.used = 8u - zs_highbit(last) + (8u - n) * 8u;
  }
  return true;
}
// BIT_lookBits: a window that starts past the container wraps around it (what libzstd reads on a corrupted stream)
__device__ __forceinline__ uint32_t zs_look(const ZsBits& b, uint32_t nb) {
  return static_cast<uint32_t>((b.c >> ((64u - b.used - nb) & 63u)) & ((1ull << nb) - 1ull));
}
__device__ __forceinline__ uint32_t zs_look_fast(const ZsBits& b, uint32_t nb) {  // nb >= 1; zeros past the container
  return static_cast<uint32_t>((b.c << (b.used & 63u)) >> ((64u - nb) & 63u));
}
__device__ __forceinline__ uint32_t zs_read(ZsBits& b, uint32_t nb) { const uint32_t v = zs_look(b, nb); b.used += nb; return v; }
__device__ __forceinline__ uint32_t zs_read_fast(ZsBits& b, uint32_t nb) { const uint32_t v = zs_look_fast(b, nb); b.used += nb; return v; }
__device__ __forceinline__ int zs_reload(ZsBits& b) {
  if (b.used > 64u) return ZS_OVERFLOW;
  if (b.off >= 8u) {
    b.off -= b.used >> 3;
    b.used &= 7u;
    b.c = zs_rd64_in(b.start, b.off, b.n);
    return ZS_UNFINISHED;
  }
  if (b.off == 0u) return b.used < 64u ? ZS_END_OF_BUFFER : ZS_COMPLETED;
  uint32_t nbytes = b.used >> 3;
  int r = ZS_UNFINISHED;
  if (nbytes > b.off) { nbytes = b.off; r = ZS_END_OF_BUFFER; }
  b.off -= nbytes;
  b.used -= nbytes * 8u;
  b.c = zs_rd64_in(b.start, b.off, b.n);
  return r;
}

// ---- FSE table headers (lane 0) -------------------------------------------------------------------------------------
// Normalized counts of an FSE table description: returns the bytes it occupies, kZsBad if it is malformed. *maxsv is the
// largest symbol allowed on entry and the last one described on return. Reads past `hb` see zeros (the header is copied
// into 8 zeroed bytes when shorter than that); a description longer than hb is an error.
__device__ uint32_t zs_ncount_body(const uint8_t* src, int iend, int16_t* norm, uint32_t* maxsv, uint32_t* tlog) {
  const uint32_t max1 = *maxsv + 1u;
  for (uint32_t s = 0; s < max1; ++s) norm[s] = 0;
  int ip = 0;
  uint32_t bits = zs_rd32(src);
  int nb = static_cast<int>(bits & 0xFu) + 5;
  if (nb > 15) return kZsBad;
  bits >>= 4;
  int bit_count = 4;
  *tlog = static_cast<uint32_t>(nb);
  int remaining = (1 << nb) + 1;
  int threshold = 1 << nb;
  nb++;
  uint32_t charnum = 0;
  bool prev0 = false;
  auto advance = [&]() {
    if (ip <= iend - 7 || ip + (bit_count >> 3) <= iend - 4) {
      ip += bit_count >> 3;
      bit_count &= 7;
    } else {
      bit_count -= 8 * (iend - 4 - ip);
      bit_count &= 31;
      ip = iend - 4;
    }
    bits = zs_rd32(src + ip) >> bit_count;
  };
  for (;;) {
    if (prev0) {
      int repeats = (__ffs(static_cast<int>(~bits | 0x80000000u)) - 1) >> 1;
      while (repeats >= 12) {
        charnum += 36u;
        if (ip <= iend - 7) {
          ip += 3;
        } else {
          bit_count -= 8 * (iend - 7 - ip);
          bit_count &= 31;
          ip = iend - 4;
        }
        bits = zs_rd32(src + ip) >> bit_count;
        repeats = (__ffs(static_cast<int>(~bits | 0x80000000u)) - 1) >> 1;
      }
      charnum += 3u * static_cast<uint32_t>(repeats);
      bits >>= 2 * repeats;
      bit_count += 2 * repeats;
      charnum += bits & 3u;
      bit_count += 2;
      if (charnum >= max1) break;
      advance();
    }
    {
      const int max = (2 * threshold - 1) - remaining;
      int count;
      if (static_cast<int>(bits & static_cast<uint32_t>(threshold - 1)) < max) {
        count = static_cast<int>(bits & static_cast<uint32_t>(threshold - 1));
        bit_count += nb - 1;
      } else {
        count = static_cast<int>(bits & static_cast<uint32_t>(2 * threshold - 1));
        if (count >= threshold) count -= max;
        bit_count += nb;
      }
      count--;
      if (count >= 0) remaining -= count;
      else remaining += count;
      norm[charnum++] = static_cast<int16_t>(count);
      prev0 = count == 0;
      if (remaining < threshold) {
        if (remaining <= 1) break;
        nb = static_cast<int>(zs_highbit(static_cast<uint32_t>(remaining))) + 1;
        threshold = 1 << (nb - 1);
      }
      if (charnum >= max1) break;
      advance();
    }
  }
  if (remaining != 1) return kZsBad;
  if (charnum > max1) return kZsBad;
  if (bit_count > 32) return kZsBad;
  *maxsv = charnum - 1u;
  ip += (bit_count + 7) >> 3;
  return static_cast<uint32_t>(ip);
}
__device__ uint32_t zs_ncount(const uint8_t* src, uint32_t hb, int16_t* norm, uint32_t* maxsv, uint32_t* tlog) {
  if (hb < 8u) {
    uint8_t buf[8];
    for (uint32_t k = 0; k < 8u; ++k) buf[k] = k < hb ? src[k] : 0u;
    const uint32_t r = zs_ncount_body(buf, 8, norm, maxsv, tlog);
    return (r == kZsBad || r > hb) ? kZsBad : r;
  }
  return zs_ncount_body(src, static_cast<int>(hb), norm, maxsv, tlog);
}

// Decoding table of normalized counts (RFC 8878 4.1.1). Returns false when a symbol holds half the table or more (no
// 0-bit-free "fast" decode: FSE_decompress then reads with BIT_readBits, which matters only for corrupted streams).
__device__ bool zs_build_fse(uint32_t* t, const int16_t* norm, uint32_t maxsv, uint32_t tlog) {
  uint16_t next[256];
  const uint32_t size = 1u << tlog;
  uint32_t high = size - 1u;
  const int large = 1 << (tlog - 1u);
  bool fast = true;
  for (uint32_t s = 0; s <= maxsv; ++s) {
    if (norm[s] == -1) {
      t[high--] = s;
      next[s] = 1;
    } else {
      if (norm[s] >= large) fast = false;
      next[s] = static_cast<uint16_t>(norm[s]);
    }
  }
  const uint32_t step = (size >> 1) + (size >> 3) + 3u, mask = size - 1u;
  uint32_t pos = 0;
  for (uint32_t s = 0; s <= maxsv; ++s) {
    for (int i = 0; i < norm[s]; ++i) {
      t[pos] = s;
      do { pos = (pos + step) & mask; } while (pos > high);
    }
  }
  for (uint32_t u = 0; u < size; ++u) {
    const uint32_t s = t[u] & 0xFFu;
    const uint32_t ns = next[s]++;
    const uint32_t nbits = tlog - zs_highbit(ns);
    const uint32_t base = (ns << nbits) - size;
    t[u] = s | (nbits << 8) | (base << 16);
  }
  return fast;
}

__device__ __forceinline__ uint32_t zs_fse_sym(const uint32_t* t, uint32_t& st, ZsBits& b, bool fast) {
  const uint32_t e = t[st];
  const uint32_t nb = (e >> 8) & 0xFFu;
  st = (e >> 16) + (fast ? zs_read_fast(b, nb) : zs_read(b, nb));
  return e & 0xFFu;
}

// Huffman weights compressed with FSE (two interleaved states, FSE_decompress): the number of weights, kZsBad.
__device__ uint32_t zs_fse_weights(ZsSmem* s, const uint8_t* src, uint32_t n) {
  int16_t norm[256];
  uint32_t maxsv = 255, tlog = 0;
  const uint32_t hs = zs_ncount(src, n, norm, &maxsv, &tlog);
  if (hs == kZsBad || tlog > 6u) return kZsBad;
  const bool fast = zs_build_fse(s->wfse, norm, maxsv, tlog);
  ZsBits b;
  if (!zs_bits_init(b, src + hs, n - hs)) return kZsBad;
  uint32_t st1 = zs_read(b, tlog);
  zs_reload(b);
  uint32_t st2 = zs_read(b, tlog);
  zs_reload(b);
  uint8_t* w = s->wgt;
  uint32_t op = 0;
  for (;;) {
    const bool more = zs_reload(b) == ZS_UNFINISHED;
    if (!(more && op < 252u)) break;
    w[op] = zs_fse_sym(s->wfse, st1, b, fast);
    w[op + 1] = zs_fse_sym(s->wfse, st2, b, fast);
    w[op + 2] = zs_fse_sym(s->wfse, st1, b, fast);
    w[op + 3] = zs_fse_sym(s->wfse, st2, b, fast);
    op += 4u;
  }
  for (;;) {
    if (op > 253u) return kZsBad;
    w[op++] = zs_fse_sym(s->wfse, st1, b, fast);
    if (zs_reload(b) == ZS_OVERFLOW) { w[op++] = zs_fse_sym(s->wfse, st2, b, fast); break; }
    if (op > 253u) return kZsBad;
    w[op++] = zs_fse_sym(s->wfse, st2, b, fast);
    if (zs_reload(b) == ZS_OVERFLOW) { w[op++] = zs_fse_sym(s->wfse, st1, b, fast); break; }
  }
  return op;
}

// Huffman tree description -> s->huf. Returns the description's size, kZsBad; *tlog = the table log.
__device__ uint32_t zs_huf_read(ZsSmem* s, const uint8_t* src, uint32_t n, uint32_t* tlog_out) {
  if (n == 0u) return kZsBad;
  uint32_t isize = src[0], osize;
  uint8_t* w = s->wgt;
  if (isize >= 128u) {  // direct: 4-bit weights
    osize = isize - 127u;
    isize = (osize + 1u) / 2u;
    if (isize + 1u > n) return kZsBad;
    for (uint32_t k = 0; k < osize; k += 2u) {
      w[k] = src[1 + k / 2] >> 4;
      w[k + 1] = src[1 + k / 2] & 15u;
    }
  } else {
    if (isize + 1u > n) return kZsBad;
    osize = zs_fse_weights(s, src + 1, isize);
    if (osize == kZsBad) return kZsBad;
  }
  uint32_t rank[kZsHufLogMax + 1];
  for (uint32_t k = 0; k <= kZsHufLogMax; ++k) rank[k] = 0;
  uint32_t total = 0;
  for (uint32_t k = 0; k < osize; ++k) {
    if (w[k] > kZsHufLogMax) return kZsBad;
    rank[w[k]]++;
    total += (1u << w[k]) >> 1;
  }
  if (total == 0u) return kZsBad;
  const uint32_t tlog = zs_highbit(total) + 1u;
  if (tlog > kZsHufLogMax) return kZsBad;
  const uint32_t rest = (1u << tlog) - total;
  if ((1u << zs_highbit(rest)) != rest) return kZsBad;  // the implied last weight must complete a power of two
  const uint32_t lastw = zs_highbit(rest) + 1u;
  w[osize] = static_cast<uint8_t>(lastw);
  rank[lastw]++;
  if (rank[1] < 2u || (rank[1] & 1u)) return kZsBad;
  const uint32_t nsym = osize + 1u;
  // codes: weight 1 (longest) first, symbols ascending within a weight; weight w covers 2^(w-1) entries
  uint32_t pos = 0;
  for (uint32_t wt = 1; wt <= tlog; ++wt) {
    if (rank[wt] == 0u) continue;
    const uint32_t len = 1u << (wt - 1u), nbits = tlog + 1u - wt;
    for (uint32_t sym = 0; sym < nsym; ++sym) {
      if (w[sym] != wt) continue;
      const uint16_t e = static_cast<uint16_t>((sym << 8) | nbits);
      for (uint32_t k = 0; k < len; ++k) s->huf[pos + k] = e;
      pos += len;
    }
  }
  *tlog_out = tlog;
  return isize + 1u;
}

// One Huffman stream (one lane): cnt symbols into out; false unless the stream is consumed exactly.
// lenient: libzstd's 4-stream fast decoder (x86-64, streams of >= 16 / 8 / 8 / 8 bytes, table log <= 11) neither needs
// the end mark nor checks that a stream is consumed exactly, and a stream may read on into the bytes of the streams
// before it (down to `first`, the start of stream 1); the decoder follows it there.
__device__ bool zs_huf_stream(const uint16_t* huf, uint32_t tlog, const uint8_t* src, uint32_t n, uint8_t* out, uint32_t cnt,
                              bool lenient, const uint8_t* first) {
  ZsBits b;
  if (lenient) {
    const uint32_t back = static_cast<uint32_t>(src - first);
    const uint32_t last = src[n - 1];
    b.start = first;
    b.n = back + n;
    b.off = back + n - 8u;
    b.c = zs_rd64(first + b.off);
    b.used = last ? 8u - zs_highbit(last) : 0u;
  } else if (!zs_bits_init(b, src, n)) {
    return false;
  }
  for (uint32_t k = 0; k < cnt; ++k) {
    const uint32_t e = huf[zs_look_fast(b, tlog)];
    out[k] = static_cast<uint8_t>(e >> 8);
    b.used += e & 0xFFu;
    zs_reload(b);
  }
  if (lenient) return true;
  zs_reload(b);
  return b.off == 0u && b.used == 64u;
}

// Literals of a Huffman-coded section: 1 stream (lane 0) or 4 (lanes 0..3). Uniform result.
__device__ bool zs_huf_literals(ZsSmem* s, uint32_t tlog, const uint8_t* src, uint32_t n, uint8_t* lit, uint32_t lsize, bool single) {
  const uint32_t lane = threadIdx.x & 31u;
  uint32_t ok = 1;
  if (single) {
    if (lane == 0) s->res[4] = zs_huf_stream(s->huf, tlog, src, n, lit, lsize, false, src) ? 1u : 0u;
    __syncwarp();
    ok = s->res[4];
    __syncwarp();
    return ok != 0u;
  }
  if (n < 10u) return false;
  const uint32_t l1 = zs_rd16(src), l2 = zs_rd16(src + 2), l3 = zs_rd16(src + 4);
  if (l1 + l2 + l3 + 6u > n) return false;
  const uint32_t l4 = n - (l1 + l2 + l3 + 6u);
  const uint32_t seg = (lsize + 3u) / 4u;
  if (3u * seg > lsize) return false;
  const bool lenient = tlog <= 11u && l1 >= 16u && l2 >= 8u && l3 >= 8u && l4 >= 8u && 3u * seg < lsize;
  if (lane < 4u) {
    const uint32_t in_off = lane == 0 ? 6u : lane == 1 ? 6u + l1 : lane == 2 ? 6u + l1 + l2 : 6u + l1 + l2 + l3;
    const uint32_t in_n = lane == 0 ? l1 : lane == 1 ? l2 : lane == 2 ? l3 : l4;
    const uint32_t cnt = lane < 3u ? seg : lsize - 3u * seg;
    s->res[4 + lane] = zs_huf_stream(s->huf, tlog, src + in_off, in_n, lit + lane * seg, cnt, lenient, src + 6) ? 1u : 0u;
  }
  __syncwarp();
  ok = s->res[4] & s->res[5] & s->res[6] & s->res[7];
  __syncwarp();
  return ok != 0u;
}

// Builds one sequence table (LL = 0, OF = 1, ML = 2) in `mode`; returns the header bytes used, kZsBad. Uniform.
__device__ uint32_t zs_seq_table(ZsSmem* s, int which, uint32_t mode, const uint8_t* src, uint32_t n, bool have_tables, uint32_t* tlog) {
  const uint32_t lane = threadIdx.x & 31u;
  const uint32_t maxsv = which == 0 ? 35u : which == 1 ? 31u : 52u;
  const uint32_t maxlog = which == 1 ? 8u : 9u;
  if (mode == 3u) return have_tables ? 0u : kZsBad;  // repeat: the previous block's table
  if (mode == 1u) {                                    // RLE: one symbol, no state bits
    if (n == 0u || src[0] > maxsv) return kZsBad;
    if (lane == 0) s->seq[which][0] = src[0];
    __syncwarp();
    *tlog = 0;
    return 1u;
  }
  uint32_t used = 0, log = 0;
  if (lane == 0) {
    int16_t norm[64];
    uint32_t sv = maxsv;
    if (mode == 0u) {  // predefined distribution
      const int16_t* d = which == 0 ? kZsLLNorm : which == 1 ? kZsOFNorm : kZsMLNorm;
      sv = which == 0 ? 35u : which == 1 ? 28u : 52u;
      for (uint32_t k = 0; k <= sv; ++k) norm[k] = d[k];
      log = which == 1 ? 5u : 6u;
      used = 0;
    } else {
      used = zs_ncount(src, n, norm, &sv, &log);
      if (used != kZsBad && log > maxlog) used = kZsBad;
    }
    if (used != kZsBad) zs_build_fse(s->seq[which], norm, sv, log);
    s->res[0] = used;
    s->res[1] = log;
  }
  __syncwarp();
  used = s->res[0];
  log = s->res[1];
  __syncwarp();
  *tlog = log;
  return used;
}

// ---- XXH64 (content checksum) ----------------------------------------------------------------------------------------
constexpr uint64_t kP1 = 11400714785074694791ull, kP2 = 14029467366897019727ull, kP3 = 1609587929392839161ull,
                   kP4 = 9650029242287828579ull, kP5 = 2870177450012600261ull;
__device__ __forceinline__ uint64_t zs_rotl(uint64_t x, int r) { return (x << r) | (x >> (64 - r)); }
__device__ __forceinline__ uint64_t zs_xround(uint64_t acc, uint64_t in) { return zs_rotl(acc + in * kP2, 31) * kP1; }
__device__ __forceinline__ uint64_t zs_xmerge(uint64_t acc, uint64_t v) { return (acc ^ zs_xround(0, v)) * kP1 + kP4; }
__device__ uint64_t zs_xxh64(const uint8_t* p, uint64_t len) {
  uint64_t h, i = 0;
  if (len >= 32u) {
    uint64_t v1 = kP1 + kP2, v2 = kP2, v3 = 0, v4 = 0ull - kP1;
    for (; i + 32u <= len; i += 32u) {
      v1 = zs_xround(v1, zs_rd64(p + i));
      v2 = zs_xround(v2, zs_rd64(p + i + 8));
      v3 = zs_xround(v3, zs_rd64(p + i + 16));
      v4 = zs_xround(v4, zs_rd64(p + i + 24));
    }
    h = zs_rotl(v1, 1) + zs_rotl(v2, 7) + zs_rotl(v3, 12) + zs_rotl(v4, 18);
    h = zs_xmerge(h, v1); h = zs_xmerge(h, v2); h = zs_xmerge(h, v3); h = zs_xmerge(h, v4);
  } else {
    h = kP5;
  }
  h += len;
  for (; i + 8u <= len; i += 8u) h = zs_rotl(h ^ zs_xround(0, zs_rd64(p + i)), 27) * kP1 + kP4;
  if (i + 4u <= len) { h = zs_rotl(h ^ (static_cast<uint64_t>(zs_rd32(p + i)) * kP1), 23) * kP2 + kP3; i += 4u; }
  for (; i < len; ++i) h = zs_rotl(h ^ (p[i] * kP5), 11) * kP1;
  h ^= h >> 33; h *= kP2; h ^= h >> 29; h *= kP3; h ^= h >> 32;
  return h;
}

// ---- one chunk ------------------------------------------------------------------------------------------------------
struct ZsFrameState {
  uint32_t rep[3];
  bool lit_tables, seq_tables;  // a Huffman / FSE table exists for treeless literals / repeat modes
  uint32_t huf_log, ll_log, of_log, ml_log;
};

// Match of `ml` bytes at dst[op] from `offset` bytes back (the warp; everything before dst + op is published).
__device__ __forceinline__ void zs_match(uint8_t* dst, uint32_t op, uint32_t ml, uint32_t offset, uint32_t lane) {
  if (offset >= 32u) {
    for (uint32_t done = 0; done < ml; done += offset) {  // rounds of `offset` bytes: a round reads only older rounds
      const uint32_t n = min(offset, ml - done);
      uint8_t* d = dst + op + done;
      const uint8_t* from = d - offset;
      for (uint32_t k = lane; k < n; k += 32u) d[k] = from[k];
      __syncwarp();
    }
  } else {
    const uint8_t* pat = dst + op - offset;
    for (uint32_t k = lane; k < ml; k += 32u) dst[op + k] = pat[k % offset];
    __syncwarp();
  }
}

// A compressed block at src[0, n) into dst[op, cap). Returns the bytes written, kZsBad. Uniform.
__device__ uint32_t zs_block(ZsSmem* s, ZsFrameState& fs, const uint8_t* src, uint32_t n, uint8_t* dst, uint32_t op, uint32_t cap,
                             uint32_t frame_start, uint8_t* litbuf) {
  const uint32_t lane = threadIdx.x & 31u;
  if (n >= kZsBlockMax) return kZsBad;
  if (n < 2u) return kZsBad;
  const uint32_t room = cap - op, lit_room = min(room, kZsBlockMax);
  // ---- literals section ----
  const uint32_t b0 = src[0], ltype = b0 & 3u, lhl = (b0 >> 2) & 3u;
  const uint8_t* lits;
  uint32_t lsize, used;
  if (ltype <= 1u) {  // raw / RLE
    const uint32_t lh = lhl == 1u ? 2u : lhl == 3u ? 3u : 1u;
    if (lh + ltype > n) return kZsBad;  // the header (and the RLE byte) must be there
    lsize = lh == 1u ? b0 >> 3 : lh == 2u ? zs_rd16(src) >> 4 : zs_rd24(src) >> 4;
    if (ltype == 0u) {
      if (lsize > lit_room || lh + lsize > n) return kZsBad;
      lits = src + lh;
      used = lh + lsize;
    } else {
      if (lsize > lit_room) return kZsBad;
      const uint8_t v = src[lh];
      for (uint32_t k = lane; k < lsize; k += 32u) litbuf[k] = v;
      __syncwarp();
      lits = litbuf;
      used = lh + 1u;
    }
  } else {  // Huffman: compressed (2) or treeless (3)
    if (ltype == 3u && !fs.lit_tables) return kZsBad;
    if (n < 5u) return kZsBad;
    const uint32_t lhc = zs_rd32(src);
    uint32_t lh, csize;
    const bool single = lhl == 0u;
    if (lhl <= 1u) { lh = 3u; lsize = (lhc >> 4) & 0x3FFu; csize = (lhc >> 14) & 0x3FFu; }
    else if (lhl == 2u) { lh = 4u; lsize = (lhc >> 4) & 0x3FFFu; csize = lhc >> 18; }
    else { lh = 5u; lsize = (lhc >> 4) & 0x3FFFFu; csize = (lhc >> 22) + (static_cast<uint32_t>(src[4]) << 10); }
    if (lsize > kZsBlockMax) return kZsBad;
    if (!single && lsize < 6u) return kZsBad;
    if (csize + lh > n) return kZsBad;
    if (lsize > lit_room) return kZsBad;
    const uint8_t* hs = src + lh;
    uint32_t hn = csize;
    if (ltype == 2u) {
      if (hn == 0u) return kZsBad;
      uint32_t r = 0, log = 0;
      if (lane == 0) { r = zs_huf_read(s, hs, hn, &log); s->res[0] = r; s->res[1] = log; }
      __syncwarp();
      r = s->res[0];
      log = s->res[1];
      __syncwarp();
      if (r == kZsBad || r >= hn) return kZsBad;
      fs.huf_log = log;
      hs += r;
      hn -= r;
    }
    if (!zs_huf_literals(s, fs.huf_log, hs, hn, litbuf, lsize, single)) return kZsBad;
    fs.lit_tables = true;
    lits = litbuf;
    used = lh + csize;
  }
  // ---- sequences section ----
  const uint8_t* ip = src + used;
  uint32_t left = n - used;
  if (left < 1u) return kZsBad;
  uint32_t nseq = ip[0];
  ip++; left--;
  uint32_t lp = 0;  // literals consumed
  uint32_t o = op;
  if (nseq == 0u) {
    if (left != 0u) return kZsBad;
  } else {
    if (nseq == 255u) {
      if (left < 2u) return kZsBad;
      nseq = zs_rd16(ip) + 0x7F00u;
      ip += 2; left -= 2;
    } else if (nseq > 127u) {
      if (left < 1u) return kZsBad;
      nseq = ((nseq - 128u) << 8) + ip[0];
      ip++; left--;
    }
    // (a 2-byte count may still say 0: the tables are read, the bitstream is not)
    if (left < 1u) return kZsBad;
    const uint32_t modes = ip[0];
    ip++; left--;  // (libzstd 1.5 ignores the reserved low bits)
    uint32_t r = zs_seq_table(s, 0, modes >> 6, ip, left, fs.seq_tables, &fs.ll_log);
    if (r == kZsBad) return kZsBad;
    ip += r; left -= r;
    r = zs_seq_table(s, 1, (modes >> 4) & 3u, ip, left, fs.seq_tables, &fs.of_log);
    if (r == kZsBad) return kZsBad;
    ip += r; left -= r;
    r = zs_seq_table(s, 2, (modes >> 2) & 3u, ip, left, fs.seq_tables, &fs.ml_log);
    if (r == kZsBad) return kZsBad;
    ip += r; left -= r;
  }
  if (nseq != 0u) {
    fs.seq_tables = true;
    ZsBits b;
    if (!zs_bits_init(b, ip, left)) return kZsBad;
    uint32_t sll = zs_read(b, fs.ll_log);
    zs_reload(b);
    uint32_t sof = zs_read(b, fs.of_log);
    zs_reload(b);
    uint32_t sml = zs_read(b, fs.ml_log);
    zs_reload(b);
    uint32_t rep0 = fs.rep[0], rep1 = fs.rep[1], rep2 = fs.rep[2];
    for (;;) {
      const uint32_t ell = s->seq[0][sll], eof = s->seq[1][sof], eml = s->seq[2][sml];
      const uint32_t llc = ell & 0xFFu, mlc = eml & 0xFFu, ofc = eof & 0xFFu;
      const uint32_t llb = kZsLLBits[llc], mlb = kZsMLBits[mlc];
      const uint32_t total_bits = llb + mlb + ofc;
      uint32_t offset;
      if (ofc > 1u) {
        offset = ((1u << ofc) - 3u) + zs_read_fast(b, ofc);
        rep2 = rep1; rep1 = rep0; rep0 = offset;
      } else {
        const uint32_t ll0 = kZsLLBase[llc] == 0u ? 1u : 0u;
        if (ofc == 0u) {
          offset = ll0 ? rep1 : rep0;
          if (ll0) { rep1 = rep0; rep0 = offset; }
        } else {
          const uint32_t idx = 1u + ll0 + zs_read_fast(b, 1);
          uint32_t t = idx == 3u ? rep0 - 1u : idx == 1u ? rep1 : rep2;
          t += t == 0u ? 1u : 0u;
          if (idx != 1u) rep2 = rep1;
          rep1 = rep0;
          rep0 = offset = t;
        }
      }
      uint32_t ml = kZsMLBase[mlc];
      if (mlb) ml += zs_read_fast(b, mlb);
      if (total_bits >= 31u) zs_reload(b);
      uint32_t ll = kZsLLBase[llc];
      if (llb) ll += zs_read_fast(b, llb);
      // libzstd 1.5 updates the states after the last sequence too (the end check below accepts the overflow)
      sll = (ell >> 16) + zs_read(b, (ell >> 8) & 0xFFu);
      sml = (eml >> 16) + zs_read(b, (eml >> 8) & 0xFFu);
      sof = (eof >> 16) + zs_read(b, (eof >> 8) & 0xFFu);
      // execute
      if (ll > lsize - lp) return kZsBad;
      if (static_cast<uint64_t>(ll) + ml > cap - o) return kZsBad;
      if (offset > o + ll - frame_start) return kZsBad;
      lz_copy(dst + o, lits + lp, ll, lane, 32u);
      lp += ll;
      o += ll;
      __syncwarp();  // the literals just written may be the match's source
      zs_match(dst, o, ml, offset, lane);
      o += ml;
      if (--nseq == 0u) break;
      zs_reload(b);
    }
    if (zs_reload(b) < ZS_COMPLETED) return kZsBad;
    fs.rep[0] = rep0; fs.rep[1] = rep1; fs.rep[2] = rep2;
  }
  const uint32_t last = lsize - lp;
  if (last > cap - o) return kZsBad;
  lz_copy(dst + o, lits + lp, last, lane, 32u);
  o += last;
  __syncwarp();
  return o - op;
}

// One full warp: ZSTD_decompress(dst, cap, src, n). Returns the decompressed size, kZsBad.
__device__ uint32_t zstd_decompress_warp(ZsSmem* s, const uint8_t* __restrict__ src, uint32_t n, uint8_t* dst, uint32_t cap, uint8_t* litbuf) {
  const uint32_t lane = threadIdx.x & 31u;
  uint32_t pos = 0, op = 0;
  while (n - pos >= 5u) {
    const uint8_t* f = src + pos;
    const uint32_t magic = zs_rd32(f);
    if ((magic & 0xFFFFFFF0u) == 0x184D2A50u) {  // skippable frame
      if (n - pos < 8u) return kZsBad;
      const uint32_t sz = zs_rd32(f + 4);
      if (sz + 8u < sz) return kZsBad;
      if (sz + 8u > n - pos) return kZsBad;
      pos += sz + 8u;
      continue;
    }
    const uint32_t rem = n - pos;
    if (rem < 9u) return kZsBad;
    const uint32_t fhd = f[4];
    const uint32_t did_code = fhd & 3u, single = (fhd >> 5) & 1u, fcs_code = fhd >> 6, checksum = (fhd >> 2) & 1u;
    const uint32_t did_size = did_code == 3u ? 4u : did_code;
    const uint32_t fcs_size = fcs_code == 0u ? single : (1u << fcs_code);
    const uint32_t hsize = 5u + (single ? 0u : 1u) + did_size + fcs_size;
    if (rem < hsize + 3u) return kZsBad;
    if (magic != 0xFD2FB528u) return kZsBad;
    if (fhd & 8u) return kZsBad;  // reserved bit
    uint32_t hp = 5;
    if (!single) {
      const uint32_t wlog = (f[hp] >> 3) + 10u;
      if (wlog > kZsWindowLogMax) return kZsBad;
      hp++;
    }
    uint32_t did = 0;
    if (did_size == 1u) did = f[hp];
    else if (did_size == 2u) did = zs_rd16(f + hp);
    else if (did_size == 4u) did = zs_rd32(f + hp);
    if (did != 0u) return kZsBad;  // no dictionary
    hp += did_size;
    uint64_t fcs = ~0ull;
    if (fcs_size == 1u) fcs = f[hp];
    else if (fcs_size == 2u) fcs = zs_rd16(f + hp) + 256u;
    else if (fcs_size == 4u) fcs = zs_rd32(f + hp);
    else if (fcs_size == 8u) fcs = static_cast<uint64_t>(zs_rd32(f + hp)) | (static_cast<uint64_t>(zs_rd32(f + hp + 4)) << 32);
    uint32_t p = pos + hsize;
    const uint32_t frame_start = op;
    ZsFrameState fs;
    fs.rep[0] = 1; fs.rep[1] = 4; fs.rep[2] = 8;
    fs.lit_tables = fs.seq_tables = false;
    fs.huf_log = fs.ll_log = fs.of_log = fs.ml_log = 0;
    for (;;) {
      if (n - p < 3u) return kZsBad;
      const uint32_t bh = zs_rd24(src + p);
      const uint32_t last = bh & 1u, btype = (bh >> 1) & 3u, bsize = bh >> 3;
      p += 3u;
      if (btype == 3u) return kZsBad;
      const uint32_t csize = btype == 1u ? 1u : bsize;
      if (csize > n - p) return kZsBad;
      uint32_t out;
      if (btype == 0u) {  // raw
        if (bsize > cap - op) return kZsBad;
        lz_copy(dst + op, src + p, bsize, lane, 32u);
        out = bsize;
      } else if (btype == 1u) {  // RLE
        if (bsize > cap - op) return kZsBad;
        const uint8_t v = src[p];
        for (uint32_t k = lane; k < bsize; k += 32u) dst[op + k] = v;
        out = bsize;
      } else {
        out = zs_block(s, fs, src + p, csize, dst, op, cap, frame_start, litbuf);
        if (out == kZsBad) return kZsBad;
      }
      __syncwarp();
      op += out;
      p += csize;
      if (last) break;
    }
    if (fcs != ~0ull && static_cast<uint64_t>(op - frame_start) != fcs) return kZsBad;
    if (checksum) {
      if (n - p < 4u) return kZsBad;
      const uint32_t want = zs_rd32(src + p);
      if (static_cast<uint32_t>(zs_xxh64(dst + frame_start, op - frame_start)) != want) return kZsBad;
      p += 4u;
    }
    pos = p;
  }
  if (pos != n) return kZsBad;  // trailing bytes that cannot start a frame
  return op;
}

// Literal scratch per warp: a block's literals never exceed the block maximum or the room left in the slot.
__host__ __device__ __forceinline__ size_t zs_lit_stride(uint32_t body_cap) {
  return (static_cast<size_t>(body_cap < kZsBlockMax ? body_cap : kZsBlockMax) + 31u) & ~size_t(15);
}

// grid: Z.n_ctas CTAs of kZsWarps warps; warp w decompresses chunks w, w + all warps, ... (literals: its scratch region)
__global__ void __launch_bounds__(kZsThreads) zstd_decompress_chunks_kernel(const ZstdLaunch Z) {
  __shared__ ZsSmem s_zs[kZsWarps];
  const Lz4Launch& L = Z.L;
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31u;
  const uint32_t w = blockIdx.x * kZsWarps + warp;
  uint8_t* litbuf = Z.lit_scratch + static_cast<size_t>(w) * zs_lit_stride(Z.body_cap);
  for (uint32_t gc = w; gc < L.n_chunks_total; gc += gridDim.x * kZsWarps) {
    const uint32_t f = L.chunk_frame[gc];
    const Lz4Frame F = L.frames[f];
    const uint32_t c = gc - F.chunk_begin;
    uint64_t body = 0;
    const uint32_t n = lz_find_chunk(F.packed_in, F.packed_in_bytes, c, &body);
    uint32_t dsize = kZsBad;
    if (n != 0xFFFFFFFFu) dsize = zstd_decompress_warp(&s_zs[warp], F.packed_in + body, n, L.scratch + static_cast<size_t>(gc) * L.slot_stride, Z.body_cap, litbuf);
    if (lane == 0) {
      L.chunk_sizes[gc] = dsize == kZsBad ? 0u : dsize;
      if (n == 0xFFFFFFFFu) report_error(L.err, DEV_ERR_CHUNK_SIZE);  // "Invalid chunk size found while decoding"
      else if (dsize == kZsBad) report_error(L.err, DEV_ERR_ZSTD);    // "ZSTD decompression failed"
      else if (c + 1u == F.n_chunks && body + n != F.packed_in_bytes) report_error(L.err, DEV_ERR_CHUNK_COUNT);  // more chunks than points
    }
    __syncwarp();
  }
}

uint32_t zstd_warps_per_cta() { return kZsWarps; }
size_t zstd_lit_scratch_bytes(uint32_t body_cap) { return zs_lit_stride(body_cap); }

int launch_zstd_decompress(const ZstdLaunch& Z, cudaStream_t stream) {
  if (Z.L.n_frames == 0) return 0;
  int n = 0;
  if (Z.L.n_chunks_total) {
    zstd_decompress_chunks_kernel<<<Z.n_ctas, kZsThreads, 0, stream>>>(Z);
    count_launch(1);
    ++n;
  }
  return n + launch_stage2_unpack(Z.L, DEV_ERR_ZSTD, stream);
}

}  // namespace cldn
