// DECODE of FloatN-only regular streams, large batches: the chunk-sequential FAST kernel.
//
// Same arithmetic as FieldDecoderFloatN_Lossy::decode (cloudini_lib/src/field_decoder.cpp:43-86) for the common case --
// every value 1..4 bytes long, no NaN marker -- and nothing else: a chunk that holds anything the fast reader cannot
// prove to be that case (a 0x00 NaN marker, a varint of 5+ bytes, a malformed marker, a truncated stream) is put on the
// launch's redo list and decoded from scratch by the careful chunk-sequential kernel (cldn_decode_tiles.cu), which also
// owns every error report. So this kernel never has to be exact about the rare cases, only about detecting them.
//
// Shape (what makes it ~2.4x cheaper in instructions than the kernel it fronts):
//  * a tile is a fixed number of POINTS (128 threads x 8 points), not a fixed number of bytes: every thread decodes
//    exactly 8 points = 8K values, fields are static, the decoded prefix values live in a static register array and no
//    per-thread rotation / run length / division exists anywhere;
//  * the bytes of a tile are staged once (coalesced 16-byte loads) in a window sized from the previous tile's length;
//    terminator bits (MSB clear) are ranked with one CTA scan; every thread finds the byte behind terminator 8K*t - 1
//    by a two-level search of the scan (warp totals, lane totals) and a select inside the owner's mask words;
//  * one straight-line reader per value: 4-byte window at the running bit position, m ^ (m - 1) isolates the value,
//    two add/mask steps un-spread the 7-bit groups, un-zigzag and the per-field running sum are one multiply-add;
//  * per-field sums: warp shuffle scan + 4 warp totals (one barrier); floats are staged per warp in a 16-byte-slot
//    array (XOR-swizzled, conflict-free both ways) and leave with 16-byte coalesced stores;
//  * 128-thread CTAs, 7 per SM: a 32-frame batch (992 chunks) is resident at once -- no quarter-full last wave.
// Included by cldn_decode_tiles.cu (shares its chunk walk and select table; the build has no relocatable device code).
#pragma once

namespace cldn {

constexpr int kFT = 128;                     // threads per CTA
constexpr int kFW = kFT / 32;                // warps
// points per thread and tile: FP = 8 for <= 4 values per point (1024-point tiles), 4 for 5 or 6 (512-point tiles): the
// decoded prefix values of a thread stay in registers, a point's floats in one 16-byte (two for 5 / 6 values) staging slot
// Values 0 .. n_floatn-1 of a point are the FloatN group (int32 arithmetic, wrapping like the reference's Vector4i); the
// rest are scalar lossy FLOAT32 fields, which the reference accumulates in int64 (field_decoder.hpp:331-353): the fast
// reader keeps 64-bit bases for them and hands the chunk to the careful kernel if a value leaves the int32 range.
constexpr int kFastDecMinBlocks = 7;   // resident CTAs per SM the register allocation aims at (8 spills; 6 loses more than it gains)
struct FastDecParams {
  float mul[6];
  uint32_t off[6];
  uint32_t n_floatn;
  uint32_t rows;   // 1: the regular fields and the V5 section fields together cover every byte of a point, whole rows may be written
  // side mode (SIDE instantiations): the V5 section fields whose values wait in DecLaunch::side
  uint32_t n_side;
  uint32_t side_offset[kMaxSideFields];   // byte offset inside a point (CLDN_SKIP_STORE_OFFSET: decoded, not stored)
  uint32_t side_bpv[kMaxSideFields];
};
constexpr int kFUnit = 16;                   // bytes per unit: a thread's slice of the window is `nu` units (nu odd: the
constexpr int kFMaxUnits = 11;                //   16-byte reads of a warp are then conflict-free at any count)
constexpr int kFLead = 16;                   // bytes in front of the window (never read as data; keeps indices > 0)
constexpr int kFWinBytes = kFMaxUnits * kFT * kFUnit;   // 22528
constexpr int kFWinAlloc = kFLead + kFWinBytes + 160;   // a thread's reader may run 32 values x 4 bytes (garbage behind its last real
                                                        // point) + two prefetched words past the window
constexpr int kFMaskWords = (kFMaxUnits * kFUnit + 31) / 32; // 6 words of terminator bits per thread
static_assert(kFT * 8 * 16 <= kFWinAlloc, "the float staging aliases the window");
// SIDE: the tile's section values (cp.async at the tile start) live behind a window of at most 9 units per thread -- enough
// for every tile the fast reader accepts (<= 4 bytes per value, <= 16 bytes per point and thread slot) -- so that window +
// values + the static shared memory still fit 7 CTAs per SM (a 32-frame batch is one chunk per resident CTA: with 6 per SM
// a seventh of the chunks waits for a second round and the launch takes twice as long -- measured)
constexpr int kFSideMaxUnits = 9;
constexpr int kFSideOff = (kFLead + kFSideMaxUnits * kFT * kFUnit + 160 + 15) & ~15;   // 18608
constexpr int kFSideBytes = 8192;                        // sum over the section fields of tile points * bpv fits here (decode_side_plan)
static_assert(kFT * 8 * 16 <= kFSideOff, "the float staging aliases the window, not the section values");

struct FastShared {
  uint32_t wcnt[kFW];                 // terminators per warp
  uint32_t lane_incl[kFT];            // warp-local inclusive terminator counts
  uint32_t masks[kFMaskWords][kFT];   // terminator bits of every thread's slice (word-major: conflict-free)
  int32_t wsum[kFW][6];               // per-warp field sums (int32, wrapping: FloatN fields)
  long long wsum64[kFW][6];           // scalar lossy fields: the reference keeps them in int64
  uint32_t next_cursor;               // window byte index (incl. kFLead) one past the tile's last value
  uint32_t chunk;                     // claimed chunk
  unsigned long long desc[2];
  // the claimed chunk, re-read from here in every tile instead of living in registers across the tile loop
  const uint8_t* body;                // first byte of the chunk body
  const uint8_t* pay_lo;              // the frame's payload [pay_lo, pay_hi): nothing outside may be read
  const uint8_t* pay_hi;
  uint8_t* out;                       // output of the chunk's first point
  uint32_t size;                      // body bytes
  uint32_t n_points;
};

// (a & m) | (b & ~m) in one LOP3; min of three in one VIMNMX3
__device__ __forceinline__ uint32_t bitselect(uint32_t m, uint32_t a, uint32_t b) {
  uint32_t d;
  asm("lop3.b32 %0, %1, %2, %3, 0xCA;" : "=r"(d) : "r"(m), "r"(a), "r"(b));
  return d;
}
// 16 bytes at g, byte by byte, reading only inside [lo, hi); bytes outside read as 0x80 (never terminate anything).
__device__ __noinline__ uint4 load_vector_bounded(const uint8_t* g, const uint8_t* lo, const uint8_t* hi) {
  uint32_t w0 = 0, w1 = 0, w2 = 0, w3 = 0;
#pragma unroll 1
  for (int b = 0; b < 16; ++b) {
    const uint8_t* gb = g + b;
    const uint32_t v = ((gb >= lo && gb < hi) ? static_cast<uint32_t>(*gb) : 0x80u) << (8 * (b & 3));
    if (b < 4) w0 |= v; else if (b < 8) w1 |= v; else if (b < 12) w2 |= v; else w3 |= v;
  }
  return make_uint4(w0, w1, w2, w3);
}
__device__ __forceinline__ void prefetch_l2(const void* p) {
  asm volatile("prefetch.global.L2 [%0];" ::"l"(p));
}
__device__ __forceinline__ uint32_t min3_u32(uint32_t a, uint32_t b, uint32_t c) {
#ifdef CLDN_CUSIM
  return min(a, min(b, c));
#else
  return __vimin3_u32(a, b, c);
#endif
}

__device__ __forceinline__ uint32_t nth_set_bit32(uint32_t m, uint32_t n, const uint32_t* __restrict__ table) {
  uint32_t base = 0;
#pragma unroll
  for (int by = 0; by < 3; ++by) {
    const uint32_t c = __popc(m & 0xFFu);
    if (n >= c) { n -= c; m >>= 8; base += 8u; }
  }
  return base + ((__ldg(&table[m & 0xFFu]) >> (4u * n)) & 7u);
}

// One value of a side array (naturally aligned: the arrays start at 256-byte boundaries, values are bpv = 1 / 2 / 4 / 8 bytes)
__device__ __forceinline__ uint64_t load_side_value(const uint8_t* p, uint32_t bpv) {
  if (bpv == 2) return *reinterpret_cast<const uint16_t*>(p);
  if (bpv == 4) return *reinterpret_cast<const uint32_t*>(p);
  if (bpv == 8) return *reinterpret_cast<const uint64_t*>(p);
  return p[0];
}

// SIDE: the chunk's V5 sections were decoded ahead of this kernel into DecLaunch::side (stream_end_kernel found where
// they start); their values are merged into the rows as they are written, so every output sector is written by ONE pass.
template <int K, int FP, bool MIXED, bool ROWS, int NF, bool SIDE>   // NF: lanes of the leading FloatN group (K when !MIXED)
__global__ void __launch_bounds__(kFT, kFastDecMinBlocks) decode_floatn_fast_kernel(const DecLaunch L, const FastDecParams Q) {
  constexpr int kFP = FP;
  constexpr int kFTilePts = kFT * FP;
  constexpr int kSlots = K <= 4 ? 1 : 2;                     // 16-byte staging slots per point
  constexpr int kMaxU = SIDE ? (kFSideMaxUnits < kFMaxUnits ? kFSideMaxUnits : kFMaxUnits) : kFMaxUnits;   // window units per thread
  extern __shared__ __align__(16) uint8_t dyn_smem[];
  __shared__ FastShared sh;
  uint8_t* win = dyn_smem;                                    // kFLead + window bytes
  uint4* ostage = reinterpret_cast<uint4*>(dyn_smem);         // aliases the window once every thread has parsed its run
  constexpr int VPT = kFP * K;                                // values per thread
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint32_t step = L.plan->point_step;
  float mul[K];
  uint32_t off[K];
#pragma unroll
  for (int f = 0; f < K; ++f) { mul[f] = Q.mul[f]; off[f] = Q.off[f]; }
  constexpr uint32_t n_floatn = MIXED ? static_cast<uint32_t>(NF) : static_cast<uint32_t>(K);   // compile time: the int64 side of a
                                                                                               // mixed plan exists only for its scalar fields

  // Whichever CTA draws ticket 0 -- by construction one that is running -- follows the u32 chunk prefixes of every
  // frame (cloudini.cpp:645-664) and publishes them; everybody else starts decoding and only waits for its own chunk.
  if (threadIdx.x == 0) sh.chunk = atomicAdd(L.chunk_counter + 2, 1u);
  __syncthreads();
  if (sh.chunk == 0u) {
    for (uint32_t f = threadIdx.x; f < L.n_frames; f += kFT) walk_frame_publish(L, f);
  }
  __syncthreads();

  while (true) {
    if (threadIdx.x == 0) {
      const uint32_t i = atomicAdd(L.chunk_counter, 1u);
      uint32_t gc_ = i;
      if (i < L.n_chunks_total) {
        if (L.uniform_chunks) gc_ = (i % L.n_frames) * L.uniform_chunks + i / L.n_frames;
        unsigned long long w0, w1;
        do {
          w0 = ld_relaxed_u64(L.chunk_desc + 2ull * gc_);
          w1 = ld_relaxed_u64(L.chunk_desc + 2ull * gc_ + 1);
        } while (static_cast<uint32_t>(w0 >> 40) != L.desc_tag || static_cast<uint32_t>(w1 >> 40) != L.desc_tag);
        sh.desc[0] = w0 & 0xFFFFFFFFFFull;
        sh.desc[1] = w1 & 0xFFFFFFFFull;
      }
      sh.chunk = gc_;
    }
    __syncthreads();
    const uint32_t gc = sh.chunk;
    if (gc >= L.n_chunks_total) return;
    uint32_t fidx;
    if (L.uniform_chunks) {
      fidx = gc / L.uniform_chunks;
    } else {
      uint32_t lo = 0, hi = L.n_frames - 1;
      while (lo < hi) {
        const uint32_t mid = (lo + hi + 1) >> 1;
        if (L.frames[mid].chunk_begin <= gc) lo = mid; else hi = mid - 1;
      }
      fidx = lo;
    }
    const uint32_t n_points = [&] {
      const DecFrame F = L.frames[fidx];
      const uint32_t chunk = gc - F.chunk_begin;
      const uint32_t n = min(kChunkPoints, F.n_points - chunk * kChunkPoints);
      if (threadIdx.x == 0) {
        sh.body = F.payload + sh.desc[0];
        sh.size = static_cast<uint32_t>(sh.desc[1]);
        sh.pay_lo = F.payload;
        sh.pay_hi = F.payload + F.payload_bytes;
        sh.out = F.out + static_cast<size_t>(chunk) * kChunkPoints * step;
        sh.n_points = n;
      }
      return n;
    }();
    __syncthreads();
    uint8_t* const out = sh.out;
    const uint32_t size = sh.size;
    bool aligned4 = ((reinterpret_cast<uintptr_t>(out) | step) & 3u) == 0u;
#pragma unroll
    for (int f = 0; f < K; ++f) aligned4 = aligned4 && (off[f] & 3u) == 0u && off[f] != CLDN_SKIP_STORE_OFFSET;
    bool dense4 = K == 4 && aligned4 && step == 16u && (reinterpret_cast<uintptr_t>(out) & 15u) == 0u;
#pragma unroll
    for (int f = 0; f < K; ++f) dense4 = dense4 && off[f] == 4u * f;
    // Whole-row copy-out: when every byte of a point belongs to a decoded field (regular or V5 section -- the section
    // reader runs behind this kernel and overwrites its bytes), the warp builds its 32 * FP points as contiguous rows in
    // shared memory and writes them with 16-byte stores. Per-field 4-byte stores of 32 lanes touch one 32-byte sector
    // per lane and field (XYZIRT, step 22: 16 sectors per store instruction measured, 5x the row bytes through L2).
    // A warp's staging holds 4 KB: layouts whose 32 * FP rows need more go out in 2, 4 or 8 passes of contiguous rows (the
    // owner lanes of a pass fill it, everybody copies it out). A layout with padding bytes keeps per-field stores: the
    // padding must keep what the caller's buffer holds. Fetching the old rows to write whole ones was measured, slower on
    // C3 (a second 32 B per point from DRAM, and every pass of a warp waits for them).
    uint32_t rows_shift = 0;
    while (((step * (32u * kFP)) >> rows_shift) > 4096u && rows_shift < 3u) ++rows_shift;
    const bool rows = ROWS && !dense4 && Q.rows != 0u && ((step * (32u * kFP)) >> rows_shift) <= 4096u && (reinterpret_cast<uintptr_t>(out) & 15u) == 0u;
    uint32_t row_align = step;
#pragma unroll
    for (int f = 0; f < K; ++f) row_align |= off[f];
    __syncthreads();  // everybody has read sh.chunk / sh.desc before thread 0 may claim the next chunk

    int32_t carry[K];
    long long carry64[MIXED ? K : 1];
#pragma unroll
    for (int f = 0; f < K; ++f) { carry[f] = 0; if (MIXED) carry64[f] = 0; }
    uint32_t cursor = 0;                      // stream byte offset of the next tile's first value
    uint32_t est = 0;                         // bytes of the previous tile (0: none yet)
    bool redo = (size == 0u);                 // an empty body cannot hold n_points > 0 points: the careful kernel reports it
    if (SIDE) redo = redo || L.stream_end[gc] == 0xFFFFFFFFu;   // no stream end / a damaged section: nothing to merge, the careful kernels decide
    for (uint32_t pt0 = 0; pt0 < n_points && !redo; pt0 += kFTilePts) {
      const uint32_t tile_pts = min(static_cast<uint32_t>(kFTilePts), n_points - pt0);
      const uint32_t n_vals = tile_pts * K;
      const uint32_t remaining = size - cursor;                                // stream bytes from the cursor on
      if (remaining < n_vals) { redo = true; break; }                          // not even one byte per value left
      const uint8_t* const body = sh.body;
      const uint8_t* first = body + cursor;
      const uint32_t c0 = static_cast<uint32_t>(reinterpret_cast<uintptr_t>(first) & 15u);
      const uint8_t* abase = first - c0;                                       // window byte i <-> abase[i]
      if (est == 0) est = static_cast<uint32_t>((static_cast<uint64_t>(size) * tile_pts) / n_points);
      uint32_t want = c0 + est + (est >> 3) + 96u;
      uint32_t nu = (want + (kFT * kFUnit - 1)) / (kFT * kFUnit);
      nu = nu < 3u ? 3u : (nu | 1u);
      if (nu > kMaxU) nu = kMaxU;
      if (SIDE) {
        // the tile's section values (whole tile: a chunk's slot holds kChunkPoints values whatever its point count) are
        // requested now and land while the window is staged and parsed
        uint32_t soff = 0;
        for (uint32_t s = 0; s < Q.n_side; ++s) {
          const uint32_t bpv = Q.side_bpv[s];
          const uint8_t* src = L.side + L.side_off[s] + (static_cast<size_t>(gc) * kChunkPoints + pt0) * bpv;
          const uint32_t bytes = kFTilePts * bpv;
          for (uint32_t u = 16u * threadIdx.x; u < bytes; u += 16u * kFT) {
            async_copy16(reinterpret_cast<uint4*>(dyn_smem + kFSideOff + soff + u), reinterpret_cast<const uint4*>(src + u));
          }
          soff += bytes;
        }
        async_commit();
      }
      uint32_t m[kFMaskWords];
      uint32_t total, incl, cnt;
      while (true) {
        // ---- stage the window: coalesced 16-byte loads, vector v <-> bytes [16 v, 16 v + 16) ----
        // vectors [v_lo, v_hi) lie completely inside the payload (only the very first / last ones of a frame can stick out)
        const uint32_t n_vec = nu * kFT;
        const uint8_t* const pay_lo = sh.pay_lo;
        const uint8_t* const pay_end = sh.pay_hi;
        const uint32_t v_lo = abase < pay_lo ? 1u : 0u;
        const uint64_t room = static_cast<uint64_t>(pay_end - abase) >> 4;
        const uint32_t v_hi = room < n_vec ? static_cast<uint32_t>(room) : n_vec;
        const uint4* gv = reinterpret_cast<const uint4*>(abase) + threadIdx.x;
        uint4* sv = reinterpret_cast<uint4*>(win + kFLead) + threadIdx.x;
        if (v_lo == 0u && v_hi == n_vec) {
          // the whole window lies inside the payload (every tile but the first / last few of a frame): cp.async, global ->
          // shared without the register round trip, every request of the thread in flight at once (measured faster than
          // plain loads + stores)
#pragma unroll
          for (int r = 0; r < kMaxU; ++r) {
            if (r < static_cast<int>(nu)) async_copy16(sv + r * kFT, gv + r * kFT);
          }
          async_commit();
          async_wait_all();
        } else {
#pragma unroll 1
          for (uint32_t r = 0; r < nu; ++r) {
            const uint32_t v = r * kFT + threadIdx.x;
            sv[r * kFT] = (v >= v_lo && v < v_hi) ? __ldcs(gv + r * kFT) : load_vector_bounded(abase + 16u * v, pay_lo, pay_end);
          }
        }
        if (SIDE) async_wait_all();   // (the section values too; a no-op in the widening rounds)
        __syncthreads();
        // ---- terminator bits of my slice: nu units of 16 bytes, bit i of the mask <-> slice byte i ----
        const uint32_t slice0 = threadIdx.x * nu * kFUnit;                     // window byte of my first unit
#pragma unroll
        for (int r = 0; r < kFMaskWords; ++r) m[r] = 0;
#pragma unroll
        for (int u = 0; u < kMaxU; ++u) {
          if (u < static_cast<int>(nu)) {
            const uint4 q = *reinterpret_cast<const uint4*>(win + kFLead + slice0 + kFUnit * u);
            // (x * 0x00204081) >> 28 collects bits 7, 15, 23, 31 into a nibble
            const uint32_t b16 = (((~q.x & 0x80808080u) * 0x00204081u) >> 28) | ((((~q.y & 0x80808080u) * 0x00204081u) >> 28) << 4) |
                                 ((((~q.z & 0x80808080u) * 0x00204081u) >> 28) << 8) | ((((~q.w & 0x80808080u) * 0x00204081u) >> 28) << 12);
            m[u / 2] |= b16 << (16 * (u % 2));
          }
        }
        // bytes in front of the cursor (thread 0, c0 < 16) and past the end of the chunk are not values
        if (threadIdx.x == 0) m[0] &= ~((1u << c0) - 1u);
        const uint32_t wend = c0 + remaining;                                  // window byte one past the chunk
        if (wend < nu * (kFT * kFUnit)) {
#pragma unroll
          for (int r = 0; r < kFMaskWords; ++r) {
            const uint32_t b0 = slice0 + 32u * r;
            if (b0 >= wend) m[r] = 0;
            else if (wend - b0 < 32u) m[r] &= (1u << (wend - b0)) - 1u;
          }
        }
        cnt = 0;
#pragma unroll
        for (int r = 0; r < kFMaskWords; ++r) cnt += __popc(m[r]);
        incl = cnt;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
          const uint32_t t = __shfl_up_sync(0xffffffffu, incl, d);
          if (lane >= d) incl += t;
        }
        if (lane == 31) sh.wcnt[warp] = incl;
        sh.lane_incl[threadIdx.x] = incl;
#pragma unroll
        for (int r = 0; r < kFMaskWords; ++r) sh.masks[r][threadIdx.x] = m[r];
        __syncthreads();
        total = 0;
#pragma unroll
        for (int w = 0; w < kFW; ++w) total += sh.wcnt[w];
        if (total >= n_vals) break;
        // too few values in the window: widen it if the chunk has more bytes, otherwise give the chunk to the careful kernel
        if (nu >= kMaxU || wend <= nu * (kFT * kFUnit)) { redo = true; break; }
        nu = min(static_cast<uint32_t>(kMaxU), nu + 2u);
        __syncthreads();  // everybody has read wcnt before the next round overwrites it
      }
      if (redo) break;

      // ---- first byte of my run: one past terminator (VPT * t - 1); thread 0 starts at the cursor ----
      const uint32_t v0 = threadIdx.x * VPT;
      uint32_t start = kFLead + c0;
      if (threadIdx.x > 0 && v0 < n_vals) {
        uint32_t e = v0 - 1u;                                                  // rank of the terminator in the tile
        uint32_t w = 0;
#pragma unroll
        for (int k = 0; k < kFW - 1; ++k) {
          const uint32_t c = sh.wcnt[k];
          if (w == static_cast<uint32_t>(k) && e >= c) { e -= c; w = k + 1; }
        }
        // smallest lane of warp w whose inclusive count exceeds e
        const uint32_t* li = sh.lane_incl + 32u * w;
        uint32_t lo = 0;
#pragma unroll
        for (int s = 16; s > 0; s >>= 1) {
          if (li[lo + s - 1] <= e) lo += s;
        }
        const uint32_t owner = 32u * w + lo;
        uint32_t n = e - (lo ? li[lo - 1] : 0u);                               // index among the owner's terminators
        uint32_t word = sh.masks[0][owner], wbase = 0;
#pragma unroll
        for (int r = 1; r < kFMaskWords; ++r) {
          const uint32_t c = __popc(word);
          if (wbase == 32u * (r - 1) && n >= c) { n -= c; word = sh.masks[r][owner]; wbase = 32u * r; }
        }
        start = kFLead + owner * nu * kFUnit + wbase + nth_set_bit32(word, n, kNthBit) + 1u;
      }

      // ---- parse my 8 points; P[j][f] = sum of my deltas of field f up to and including point j ----
      const uint32_t my_pts = v0 < n_vals ? min(static_cast<uint32_t>(kFP), (n_vals - v0) / K) : 0u;
      if (my_pts == 0u) start = kFLead;   // nothing of mine: parse whatever is there (ignored) from a safe place
      int32_t P[kFP][K];
      uint32_t trk = 0xFFFFFFFFu, trs = 0xFFFFFFFFu;
      uint32_t pb = start * 8u, pbs = 0;
      {
        int32_t acc[K];
#pragma unroll
        for (int f = 0; f < K; ++f) acc[f] = 0;
        const uint32_t* win32 = reinterpret_cast<const uint32_t*>(win);
        // rolling 64-bit window: the shared-memory loads follow the WORD index, which only ever steps by one, so the next
        // word is in a register before it is needed and no load sits on the value-to-value dependency chain
        uint32_t wi = pb >> 5;
        uint32_t lo = win32[wi], hi = win32[wi + 1], nx = win32[wi + 2u];   // (kFWinAlloc leaves room behind the window)
#pragma unroll
        for (int j = 0; j < kFP; ++j) {
#pragma unroll
          for (int f = 0; f < K; ++f) {
            const uint32_t w = __funnelshift_r(lo, hi, pb);                    // the 4 bytes at the bit position pb
            const uint32_t t = ~w & 0x80808080u;                               // terminators among them
            const uint32_t msk = t ^ (t - 1u);                                 // everything up to the first one (all if none)
            uint32_t x = w & 0x7F7F7F7Fu & msk;                                // the value's payload bits
            trk = min3_u32(trk, t, x);                                         // 0 <=> no terminator in 4 bytes, or a zero value
            pb += __popc(msk);
            if ((pb >> 5) != wi) {                                             // a value is at most 32 bits: one word step at most
              ++wi;
              lo = hi;
              hi = nx;
              nx = win32[wi + 2u];
            }
            // (nine instructions per value as compiled: compare, address, three moves, increment, predicated load, two copies.
            // Two shorter forms were measured at the end of round 2 -- selects, which the compiler turns into compare + select +
            // a predicated load of `hi` (5 instructions), and a mask from wi - wn with two LOP3 and an unconditional load (6):
            // both slower per 128 frames. Fewer instructions, slower: the kernel is not bound by issue slots
            // alone at this point of the loop)
            x = x - ((x >> 1) & 0x3F803F80u);                                  // 7-bit groups -> 14-bit groups
            const uint32_t z = bitselect(0x3FFFu, x, x >> 2);                  // -> uval = zigzag + 1 (28 bits)
            // un-zigzag of z - 1: odd z -> +(z >> 1), even z -> -(z >> 1); bit 0 of z is bit 0 of the window
            const int32_t sgn = static_cast<int32_t>(w & 1u) * 2 - 1;
            acc[f] = static_cast<int32_t>(static_cast<uint32_t>(acc[f]) + (z >> 1) * static_cast<uint32_t>(sgn));
            P[j][f] = acc[f];
          }
          if (static_cast<uint32_t>(j + 1) == my_pts) { trs = trk; pbs = pb; }  // my last real point
        }
      }
      // a 0x00 marker / zero value or a value without a terminator inside 4 bytes among my real values
      const bool bad = my_pts > 0u && trs == 0u;
      int32_t tot[K];
#pragma unroll
      for (int f = 0; f < K; ++f) tot[f] = my_pts > 0u ? P[kFP - 1][f] : 0;
      if (my_pts > 0u && my_pts < static_cast<uint32_t>(kFP)) {
#pragma unroll
        for (int j = 0; j < kFP - 1; ++j) {
          if (static_cast<uint32_t>(j + 1) == my_pts) {
#pragma unroll
            for (int f = 0; f < K; ++f) tot[f] = P[j][f];
          }
        }
      }
      // the thread that owns the tile's last point knows where the next tile starts
      if (my_pts > 0u && v0 + my_pts * K == n_vals) sh.next_cursor = pbs >> 3;
      int32_t inc[K];
#pragma unroll
      for (int f = 0; f < K; ++f) inc[f] = tot[f];
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
#pragma unroll
        for (int f = 0; f < K; ++f) {
          const int32_t up = __shfl_up_sync(0xffffffffu, inc[f], d);
          if (lane >= d) inc[f] = static_cast<int32_t>(static_cast<uint32_t>(inc[f]) + static_cast<uint32_t>(up));
        }
      }
      long long inc64[MIXED ? K : 1];
      if (MIXED) {  // scalar fields: the same scan in 64 bits (a warp's sum of 4-byte deltas does not fit 32)
#pragma unroll
        for (int f = 0; f < K; ++f) inc64[f] = tot[f];
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
#pragma unroll
          for (int f = 0; f < K; ++f) {
            if (static_cast<uint32_t>(f) >= n_floatn) {
              const long long up = __shfl_up_sync(0xffffffffu, inc64[f], d);
              if (lane >= d) inc64[f] += up;
            }
          }
        }
      }
      if (lane == 31) {
#pragma unroll
        for (int f = 0; f < K; ++f) {
          sh.wsum[warp][f] = inc[f];
          if (MIXED) sh.wsum64[warp][f] = inc64[f];
        }
      }
      const int any_bad = __syncthreads_or(bad ? 1 : 0);  // also: every thread is done with the window bytes
      if (any_bad) { redo = true; break; }
      int32_t base[K];
      long long base64[MIXED ? K : 1];
#pragma unroll
      for (int f = 0; f < K; ++f) {
        uint32_t b = static_cast<uint32_t>(carry[f]), c = static_cast<uint32_t>(carry[f]);
#pragma unroll
        for (int w = 0; w < kFW; ++w) {
          const uint32_t s = static_cast<uint32_t>(sh.wsum[w][f]);
          if (w < warp) b += s;
          c += s;
        }
        carry[f] = static_cast<int32_t>(c);
        base[f] = static_cast<int32_t>(b + static_cast<uint32_t>(inc[f]) - static_cast<uint32_t>(tot[f]));
        if (MIXED && static_cast<uint32_t>(f) >= n_floatn) {
          long long b64 = carry64[f], c64 = carry64[f];
#pragma unroll
          for (int w = 0; w < kFW; ++w) {
            const long long s64 = sh.wsum64[w][f];
            if (w < warp) b64 += s64;
            c64 += s64;
          }
          carry64[f] = c64;
          base64[f] = b64 + inc64[f] - tot[f];
        }
      }
      const uint32_t ncur = sh.next_cursor;
      const uint32_t used = ncur - (kFLead + c0);
      // the next tile's bytes are asked into L2 now (its loads are issued behind this tile's conversion and copy-out)
      if (pt0 + kFTilePts < n_points) {
        const uint32_t ahead = cursor + used + threadIdx.x * 128u;
        if (ahead < size && threadIdx.x * 128u < used + (used >> 2) + 256u) prefetch_l2(body + ahead);
      }
      // ---- floats into my warp's staging slots (16 bytes per point, two for 5 / 6 values; a lane's 8 slots are XOR-swizzled
      //      with its index so that both the lane-blocked writes and the point-strided reads are conflict-free) ----
      uint4* wst = ostage + warp * (32 * 8);
      uint4* const my_slots = wst + 8 * lane;
      const uint32_t lx = lane & 7;
      bool wide = false;   // a scalar lossy value left the int32 range: the careful kernel (int64 like the reference) decides
      // MODE: 0 = 16-byte slots, 4 / 2 / 1 = whole rows assembled with 4- / 2- / 1-byte stores. One instantiation of the
      // loop per mode behind a CTA-uniform branch: as one loop the three row variants were if-converted and every tile
      // issued all of them (25 predicated-off instructions per point on XYZIRT).
      uint8_t* row0 = reinterpret_cast<uint8_t*>(wst) + static_cast<uint32_t>(kFP * lane) * step;   // my first row in the staging (row modes)
      auto emit = [&](auto mode_tag) {
        constexpr int MODE = decltype(mode_tag)::value;
#pragma unroll
        for (int j = 0; j < kFP; ++j) {
          uint32_t fl[kSlots * 4];
#pragma unroll
          for (int f = 0; f < kSlots * 4; ++f) fl[f] = 0;
#pragma unroll
          for (int f = 0; f < K; ++f) {
            int32_t v = static_cast<int32_t>(static_cast<uint32_t>(base[f]) + static_cast<uint32_t>(P[j][f]));
            if (MIXED && static_cast<uint32_t>(f) >= n_floatn) {
              const long long v64 = base64[f] + P[j][f];
              v = static_cast<int32_t>(v64);
              wide = wide || (v64 != static_cast<long long>(v));
            }
            fl[f] = __float_as_uint(__fmul_rn(__int2float_rn(v), mul[f]));
          }
          if (MODE != 0) {
            uint8_t* row = row0 + static_cast<uint32_t>(j) * step;
#pragma unroll
            for (int f = 0; f < K; ++f) {
              uint8_t* d = row + off[f];
              if (MODE == 4) {
                *reinterpret_cast<uint32_t*>(d) = fl[f];
              } else if (MODE == 2) {
                *reinterpret_cast<uint16_t*>(d) = static_cast<uint16_t>(fl[f]);
                *reinterpret_cast<uint16_t*>(d + 2) = static_cast<uint16_t>(fl[f] >> 16);
              } else {
                d[0] = static_cast<uint8_t>(fl[f]); d[1] = static_cast<uint8_t>(fl[f] >> 8);
                d[2] = static_cast<uint8_t>(fl[f] >> 16); d[3] = static_cast<uint8_t>(fl[f] >> 24);
              }
            }
          } else if (kSlots == 1) {
            my_slots[j ^ lx] = make_uint4(fl[0], fl[1], fl[2], fl[3]);
          } else {
            my_slots[(2 * j) ^ lx] = make_uint4(fl[0], fl[1], fl[2], fl[3]);
            my_slots[(2 * j + 1) ^ lx] = make_uint4(fl[4], fl[5], fl[6], fl[7]);
          }
        }
      };
      // ---- copy-out: lane l of iteration i takes point 32 i + l of the warp's 32 * FP ----
      const uint32_t wp0 = pt0 + warp * (32 * kFP);
      const uint32_t wn = wp0 < n_points ? min(static_cast<uint32_t>(32 * kFP), n_points - wp0) : 0u;
      uint8_t* dst0 = sh.out + static_cast<size_t>(wp0 + lane) * step;
      if (!ROWS || !rows) {
        emit(std::integral_constant<int, 0>{});
        __syncwarp();
      }
      if (ROWS && rows) {
        // ---- whole rows, 1 << rows_shift passes of contiguous rows through the warp's 4 KB ----
        const uint32_t lpp = 32u >> rows_shift;            // owner lanes per pass
        const uint32_t rpp = lpp * kFP;                    // rows per pass
        uint8_t* const wsb = reinterpret_cast<uint8_t*>(wst);
        row0 = wsb + static_cast<uint32_t>(kFP * (lane & (lpp - 1u))) * step;
        for (uint32_t h = 0; h < (1u << rows_shift); ++h) {
          const uint32_t p_lo = h * rpp;
          const uint32_t cnt_rows = wn > p_lo ? min(rpp, wn - p_lo) : 0u;
          const uint32_t total = cnt_rows * step;          // bytes of this pass; its first byte is 16-byte aligned
          uint8_t* dst = sh.out + static_cast<size_t>(wp0 + p_lo) * step;
          const uint32_t tail0 = total & ~15u;
          if ((static_cast<uint32_t>(lane) >> (5u - rows_shift)) == h) {
            if ((row_align & 3u) == 0u) emit(std::integral_constant<int, 4>{});
            else if ((row_align & 1u) == 0u) emit(std::integral_constant<int, 2>{});
            else emit(std::integral_constant<int, 1>{});
            if (SIDE) {
              // the section values of my kFP consecutive points go into my rows (bytes: a row may sit at any alignment)
              uint32_t soff = 0;
              for (uint32_t s = 0; s < Q.n_side; ++s) {
                const uint32_t bpv = Q.side_bpv[s], so = Q.side_offset[s];
                const uint8_t* sv = dyn_smem + kFSideOff + soff + threadIdx.x * kFP * bpv;
                soff += kFTilePts * bpv;
                if (so == CLDN_SKIP_STORE_OFFSET) continue;
                uint8_t* d = row0 + so;
                for (uint32_t j = 0; j < static_cast<uint32_t>(kFP); ++j) {
                  for (uint32_t b = 0; b < bpv; ++b) d[j * step + b] = sv[j * bpv + b];
                }
              }
            }
          }
          __syncwarp();
          for (uint32_t o = 16u * lane; o + 16u <= total; o += 512u) {
            __stcs(reinterpret_cast<uint4*>(dst + o), *reinterpret_cast<const uint4*>(wsb + o));
          }
          if (tail0 + lane < total) dst[tail0 + lane] = wsb[tail0 + lane];
          __syncwarp();   // the next pass refills the staging
        }
      } else if (kSlots == 1) {
        // slot of point 32 i + l: owner lane 4 i + (l >> 3), its point l & 7 -> 8 (4 i + (l >> 3)) + ((l & 7) ^ ((4 i + (l >> 3)) & 7))
        const uint32_t lh = lane >> 3, ll = lane & 7;
        const uint4* rd_even = wst + 8 * lh + (ll ^ lh);          // i even: (4 i + lh) & 7 == lh
        const uint4* rd_odd = wst + 8 * lh + (ll ^ (lh + 4));     // i odd:  (4 i + lh) & 7 == lh + 4
        if (dense4 && wn == static_cast<uint32_t>(32 * kFP)) {
#pragma unroll
          for (int i = 0; i < kFP; ++i) {
            const uint4 v = ((i & 1) ? rd_odd : rd_even)[32 * i];
            __stcs(reinterpret_cast<uint4*>(dst0 + 512 * i), v);
          }
        } else {
#pragma unroll
          for (int i = 0; i < kFP; ++i) {
            const uint32_t q = 32u * i + lane;
            if (q < wn) {
              const uint4 v = ((i & 1) ? rd_odd : rd_even)[32 * i];
              uint8_t* dst = dst0 + static_cast<size_t>(32 * i) * step;
              const uint32_t vv[4] = {v.x, v.y, v.z, v.w};
              if (dense4) {
                __stcs(reinterpret_cast<uint4*>(dst), v);
              } else if (aligned4) {
                // (neighbouring fields inside one aligned 8 bytes as ONE 8-byte store: measured on C3 -- no gain)
#pragma unroll
                for (int f = 0; f < K; ++f) __stcs(reinterpret_cast<unsigned int*>(dst + off[f]), vv[f]);
              } else {
#pragma unroll
                for (int f = 0; f < K; ++f) {
                  if (off[f] != CLDN_SKIP_STORE_OFFSET) store_u32(dst + off[f], vv[f]);
                }
              }
            }
          }
        }
      } else {
        // two slots per point, 4 points per lane: point 32 i + l belongs to lane 8 i + (l >> 2), its point l & 3
        const uint32_t lo4 = lane >> 2, lj = lane & 3;
        const uint4* rd0 = wst + 8 * lo4 + ((2 * lj) ^ lo4);
        const uint4* rd1 = wst + 8 * lo4 + ((2 * lj + 1) ^ lo4);
#pragma unroll
        for (int i = 0; i < kFP; ++i) {
          const uint32_t q = 32u * i + lane;
          if (q < wn) {
            const uint4 a = rd0[64 * i], b = rd1[64 * i];
            uint8_t* dst = dst0 + static_cast<size_t>(32 * i) * step;
            const uint32_t vv[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
            if (aligned4) {
#pragma unroll
              for (int f = 0; f < K; ++f) __stcs(reinterpret_cast<unsigned int*>(dst + off[f]), vv[f]);
            } else {
#pragma unroll
              for (int f = 0; f < K; ++f) {
                if (off[f] != CLDN_SKIP_STORE_OFFSET) store_u32(dst + off[f], vv[f]);
              }
            }
          }
        }
      }
      if (SIDE && !rows) {
        // per-point copy-out of the section fields: lane l of iteration i takes point 32 i + l like the floats above, so a
        // point's section bytes follow its floats into the same sectors while they are still in L2
        uint32_t soff = 0;
        for (uint32_t s = 0; s < Q.n_side; ++s) {
          const uint32_t bpv = Q.side_bpv[s], so = Q.side_offset[s];
          const uint8_t* sv = dyn_smem + kFSideOff + soff + (static_cast<uint32_t>(warp) * (32 * kFP) + lane) * bpv;
          soff += kFTilePts * bpv;
          if (so == CLDN_SKIP_STORE_OFFSET) continue;
          uint8_t* d = dst0 + so;
          const bool al = ((static_cast<uint32_t>(reinterpret_cast<uintptr_t>(d)) | step) & (bpv - 1u)) == 0u;
          if (bpv == 4u && al) {
#pragma unroll
            for (int i = 0; i < kFP; ++i) {
              if (32u * i + lane < wn) __stcs(reinterpret_cast<unsigned int*>(d + static_cast<size_t>(32 * i) * step), *reinterpret_cast<const uint32_t*>(sv + 128 * i));
            }
          } else if (bpv == 2u && al) {
#pragma unroll
            for (int i = 0; i < kFP; ++i) {
              if (32u * i + lane < wn) *reinterpret_cast<uint16_t*>(d + static_cast<size_t>(32 * i) * step) = *reinterpret_cast<const uint16_t*>(sv + 64 * i);
            }
          } else {
#pragma unroll 1
            for (int i = 0; i < kFP; ++i) {
              if (32u * i + lane < wn) {
                uint8_t* dp = d + static_cast<size_t>(32 * i) * step;
                for (uint32_t b = 0; b < bpv; ++b) dp[b] = sv[32u * i * bpv + b];
              }
            }
          }
        }
      }
      est = used;
      cursor += used;
      // the staging slots alias the window the next tile is about to load
      if (MIXED) {
        if (__syncthreads_or(wide ? 1 : 0)) { redo = true; break; }
      } else {
        __syncthreads();
      }
    }
    if (redo) {
      if (threadIdx.x == 0) {
        L.redo_list[atomicAdd(L.chunk_counter + 3, 1u)] = gc;
        L.stream_end[gc] = 0xFFFFFFFFu;  // the careful kernel owns this chunk now (its sections too)
      }
    } else if (SIDE && cursor != L.stream_end[gc]) {
      // (cannot happen for a stream the tile loop accepted: it ends behind its n_points * K-th terminator, which is what
      // the pre-pass looked for. Kept as a cross-check: the merged section values belong to that position.)
      if (threadIdx.x == 0) {
        L.redo_list[atomicAdd(L.chunk_counter + 3, 1u)] = gc;
        L.stream_end[gc] = 0xFFFFFFFFu;
      }
    } else if (threadIdx.x == 0) {
      L.stream_end[gc] = cursor;  // V5: the sections start here
    }
    if (SIDE) __syncthreads();  // everybody has compared the pre-pass's stream end before thread 0 may have replaced it
  }
}

size_t decode_fast_smem_bytes(bool side) {
  if (side) return static_cast<size_t>(kFSideOff + kFSideBytes);
  return static_cast<size_t>(kFWinAlloc);
}

template <int K, int FP, bool MIXED, bool ROWS, int NF, bool SIDE>
static int launch_fast_one(const FastDecParams& Q, const DecLaunch& L, int sm_count, cudaStream_t stream) {
  const size_t smem = decode_fast_smem_bytes(SIDE);
  auto k = decode_floatn_fast_kernel<K, FP, MIXED, ROWS, NF, SIDE>;
  if (raise_smem_limit(k, smem) != cudaSuccess) return -1;
  int per_sm = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k, kFT, smem) != cudaSuccess || per_sm < 1) per_sm = 1;
  const uint32_t grid = min(L.n_chunks_total, static_cast<uint32_t>(per_sm * sm_count));
  k<<<grid, kFT, smem, stream>>>(L, Q);
  return 1;
}
template <int K, int FP, bool MIXED, bool ROWS, int NF>
static int launch_fast(const FastDecParams& Q, const DecLaunch& L, int sm_count, cudaStream_t stream) {
  return Q.n_side ? launch_fast_one<K, FP, MIXED, ROWS, NF, true>(Q, L, sm_count, stream)
                  : launch_fast_one<K, FP, MIXED, ROWS, NF, false>(Q, L, sm_count, stream);
}

// Plans the fast reader takes: every value of the regular stream is a 32-bit float varint -- one leading FloatN group and /
// or scalar lossy FLOAT32 fields --, 3 .. 6 values per point.
bool decode_fast_plan(const Plan& plan, FastDecParams* Q) {
  if (!plan.all_varint || plan.n_ops == 0 || plan.n_gorilla || plan.regular_overlap) return false;
  uint32_t nv = 0;
  Q->n_floatn = 0;
  for (uint32_t i = 0; i < plan.n_ops; ++i) {
    const RegOp& op = plan.ops[i];
    if (op.kind == OP_FLOATN && i == 0) {
      for (int l = 0; l < op.lanes; ++l) { Q->mul[nv] = op.dec_mul_f[l]; Q->off[nv] = op.offset[l]; ++nv; }
      Q->n_floatn = op.lanes;
    } else if (op.kind == OP_F32_LOSSY) {
      if (nv >= 6) return false;
      Q->mul[nv] = op.dec_mul_f[0]; Q->off[nv] = op.offset[0]; ++nv;
    } else {
      return false;
    }
  }
  if (nv < 3 || nv > 6) return false;
  for (uint32_t k = nv; k < 6; ++k) { Q->mul[k] = 0.f; Q->off[k] = 0; }
  Q->n_side = 0;   // launch_decode_fast fills the side fields in when the launch runs in side mode
  for (int k = 0; k < kMaxSideFields; ++k) { Q->side_offset[k] = CLDN_SKIP_STORE_OFFSET; Q->side_bpv[k] = 1; }
  // rows: every byte of [0, point_step) is written by a regular field (4 bytes each here) or by a V5 section field
  Q->rows = 0;
  if (plan.point_step <= 64) {
    uint64_t covered = 0;
    bool ok = true;
    for (uint32_t k = 0; k < nv; ++k) {
      if (Q->off[k] == CLDN_SKIP_STORE_OFFSET || Q->off[k] + 4u > plan.point_step) { ok = false; break; }
      covered |= 0xFull << Q->off[k];
    }
    for (uint32_t s2 = 0; ok && s2 < plan.n_sections; ++s2) {
      const SectionField& sf = plan.sections[s2];
      if (sf.offset == CLDN_SKIP_STORE_OFFSET || sf.offset + sf.bpv > plan.point_step) { ok = false; break; }
      covered |= ((1ull << sf.bpv) - 1ull) << sf.offset;
    }
    const uint64_t all = plan.point_step == 64 ? ~0ull : ((1ull << plan.point_step) - 1ull);
    // (padding bytes: per-field stores. Rows assembled in shared memory and stored word by word with the padding masked
    // were measured on C3, 32 x 1M points, step 32: slower. The rows of a thread's 8 consecutive points lie 8 * 32 bytes
    // apart in the staging, so every shared-memory store of the row assembly is a 32-way bank conflict.)
    if (ok) Q->rows = covered == all ? 1 : 0;
  }
  return true;
}

bool decode_fast_general_plan(const Plan& plan) {
  FastDecParams Q;
  return decode_fast_plan(plan, &Q);
}
bool decode_fast_whole_rows(const Plan& plan) {
  FastDecParams Q;
  return decode_fast_plan(plan, &Q) && Q.rows == 1;
}

// ---- side mode pre-pass: where does the regular stream of every chunk end? ----------------------------------------------
// The V5 sections of a chunk start behind its regular stream, whose length is only known once it has been decoded -- or
// counted: every value is one varint (or a 0x00 NaN marker), i.e. exactly one byte with a clear top bit, so the stream ends
// right behind the chunk's (n_points * K)-th such byte. One CTA per chunk counts them 512 bytes per warp and step, finds
// the 512-byte block holding that terminator from the block counts and the byte inside it with one warp. It also does
// the launch's chunk walk (ticket 0, like the fast reader, which then finds the descriptors published). A chunk without
// that many terminators inside the longest possible stream gets 0xFFFFFFFF: the careful kernels report what is wrong.
constexpr int kSeT = 256;
constexpr uint32_t kSeBlock = 512;                                 // bytes per warp step
constexpr uint32_t kSeMaxBlocks = (kChunkPoints * 6u * 10u) / kSeBlock + 2u;  // 6 values of at most 10 bytes per point

__device__ __forceinline__ uint32_t terminator_bits16(const uint4& q) {
  return (((~q.x & 0x80808080u) * 0x00204081u) >> 28) | ((((~q.y & 0x80808080u) * 0x00204081u) >> 28) << 4) |
         ((((~q.z & 0x80808080u) * 0x00204081u) >> 28) << 8) | ((((~q.w & 0x80808080u) * 0x00204081u) >> 28) << 12);
}

__global__ void __launch_bounds__(kSeT) stream_end_kernel(const DecLaunch L, const uint32_t K) {
  __shared__ uint16_t s_cnt[kSeMaxBlocks];
  __shared__ uint32_t s_scan[kSeT / 32 + 1];
  __shared__ unsigned long long s_desc[2];
  __shared__ uint32_t s_ticket, s_found, s_rank;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) { s_ticket = atomicAdd(L.chunk_counter + 2, 1u); s_found = 0xFFFFFFFFu; s_rank = 0; }
  __syncthreads();
  if (s_ticket == 0u) {
    for (uint32_t f = threadIdx.x; f < L.n_frames; f += kSeT) walk_frame_publish(L, f);
  }
  const uint32_t gc = blockIdx.x;
  if (gc >= L.n_chunks_total) return;
  if (threadIdx.x == 0) {
    unsigned long long w0, w1;
    do {
      w0 = ld_relaxed_u64(L.chunk_desc + 2ull * gc);
      w1 = ld_relaxed_u64(L.chunk_desc + 2ull * gc + 1);
    } while (static_cast<uint32_t>(w0 >> 40) != L.desc_tag || static_cast<uint32_t>(w1 >> 40) != L.desc_tag);
    s_desc[0] = w0 & 0xFFFFFFFFFFull;
    s_desc[1] = w1 & 0xFFFFFFFFull;
  }
  __syncthreads();
  uint32_t fidx;
  if (L.uniform_chunks) {
    fidx = gc / L.uniform_chunks;
  } else {
    uint32_t lo = 0, hi = L.n_frames - 1;
    while (lo < hi) {
      const uint32_t mid = (lo + hi + 1) >> 1;
      if (L.frames[mid].chunk_begin <= gc) lo = mid; else hi = mid - 1;
    }
    fidx = lo;
  }
  const DecFrame F = L.frames[fidx];
  const uint32_t n_points = min(kChunkPoints, F.n_points - (gc - F.chunk_begin) * kChunkPoints);
  const uint32_t size = static_cast<uint32_t>(s_desc[1]);
  const uint32_t N = n_points * K;                                   // <= 32768 * 6
  if (N == 0u || size < N) {                                         // (an empty chunk has no stream: its sections start at 0)
    if (threadIdx.x == 0) L.stream_end[gc] = N == 0u ? 0u : 0xFFFFFFFFu;
    return;
  }
  const uint8_t* body = F.payload + s_desc[0];
  const uint8_t* pay_lo = F.payload;
  const uint8_t* pay_hi = F.payload + F.payload_bytes;
  const uint32_t limit = size < N * 10u ? size : N * 10u;            // (N * 10 <= 1 966 080)
  const uint32_t c0 = static_cast<uint32_t>(reinterpret_cast<uintptr_t>(body) & 15u);
  const uint8_t* abase = body - c0;                                  // window byte i <-> abase[i]; the stream is [c0, c0 + limit)
  const uint32_t wend = c0 + limit;
  const uint32_t nblk = (wend + kSeBlock - 1u) / kSeBlock;           // <= kSeMaxBlocks
  // terminator bits of the 16 bytes at window offset o, bytes outside the stream masked off
  auto unit_bits = [&](uint32_t o) -> uint32_t {
    if (o >= wend) return 0u;
    const uint8_t* g = abase + o;
    const uint4 q = (g >= pay_lo && g + 16 <= pay_hi) ? __ldg(reinterpret_cast<const uint4*>(g)) : load_vector_bounded(g, pay_lo, pay_hi);
    uint32_t m = terminator_bits16(q);
    if (o < c0) m &= ~((1u << (c0 - o)) - 1u);                        // (only the first unit: c0 < 16)
    if (wend - o < 16u) m &= (1u << (wend - o)) - 1u;
    return m;
  };
  // blocks [b_lo, b_hi) lie completely inside the stream and the payload: four of a warp's loads in flight, no masking
  const uint32_t b_lo = 1u;
  uint32_t b_hi = nblk > 0u ? nblk - 1u : 0u;
  if (abase + static_cast<size_t>(b_hi) * kSeBlock > pay_hi) b_hi = 0u;   // (cannot happen: the stream lies inside the payload)
  constexpr uint32_t kWarps = kSeT / 32;
  uint32_t b = b_lo + warp;
  for (; b + 3u * kWarps < b_hi; b += 4u * kWarps) {
    uint4 q[4];
#pragma unroll
    for (int r = 0; r < 4; ++r) q[r] = __ldg(reinterpret_cast<const uint4*>(abase + static_cast<size_t>(b + r * kWarps) * kSeBlock) + lane);
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      uint32_t c = __popc(terminator_bits16(q[r]));
#pragma unroll
      for (int d = 16; d > 0; d >>= 1) c += __shfl_xor_sync(0xffffffffu, c, d);
      if (lane == 0) s_cnt[b + r * kWarps] = static_cast<uint16_t>(c);
    }
  }
  for (; b < b_hi; b += kWarps) {
    uint32_t c = __popc(terminator_bits16(__ldg(reinterpret_cast<const uint4*>(abase + static_cast<size_t>(b) * kSeBlock) + lane)));
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) c += __shfl_xor_sync(0xffffffffu, c, d);
    if (lane == 0) s_cnt[b] = static_cast<uint16_t>(c);
  }
  // the first and the last block: bytes outside the stream / the payload masked off
  if (warp < 2) {
    const uint32_t be = warp == 0 ? 0u : nblk - 1u;
    if (warp == 0 || nblk > 1u) {
      uint32_t c = __popc(unit_bits(be * kSeBlock + 16u * lane));
#pragma unroll
      for (int d = 16; d > 0; d >>= 1) c += __shfl_xor_sync(0xffffffffu, c, d);
      if (lane == 0) s_cnt[be] = static_cast<uint16_t>(c);
    }
  }
  __syncthreads();
  // the block holding terminator N (1-based): thread t scans blocks [t * per, (t + 1) * per)
  const uint32_t per = (nblk + kSeT - 1u) / kSeT;
  uint32_t mine = 0;
  for (uint32_t i = 0; i < per; ++i) {
    const uint32_t b = threadIdx.x * per + i;
    if (b < nblk) mine += s_cnt[b];
  }
  uint32_t total;
  uint32_t before = block_exclusive_scan_n<kSeT>(mine, s_scan, &total);
  if (before < N && before + mine >= N) {
    for (uint32_t i = 0; i < per; ++i) {
      const uint32_t b = threadIdx.x * per + i;
      const uint32_t c = b < nblk ? s_cnt[b] : 0u;
      if (before + c >= N) { s_found = b; s_rank = N - before; break; }
      before += c;
    }
  }
  __syncthreads();
  const uint32_t fb = s_found;
  if (fb == 0xFFFFFFFFu) {
    if (threadIdx.x == 0) L.stream_end[gc] = 0xFFFFFFFFu;
    return;
  }
  if (warp == 0) {
    const uint32_t o = fb * kSeBlock + 16u * lane;
    uint32_t m = unit_bits(o);
    const uint32_t c = __popc(m);
    uint32_t inc = c;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const uint32_t t = __shfl_up_sync(0xffffffffu, inc, d);
      if (lane >= d) inc += t;
    }
    const uint32_t r = s_rank;                                        // 1-based inside the block
    if (inc - c < r && r <= inc) {
      for (uint32_t i = inc - c + 1u; i < r; ++i) m &= m - 1u;        // drop the terminators in front of it
      L.stream_end[gc] = o + static_cast<uint32_t>(__ffs(static_cast<int>(m))) - c0;   // one past it, relative to the body
    }
  }
}

int launch_stream_end(const Plan& plan, const DecLaunch& L, cudaStream_t stream) {
  if (plan.values_per_point == 0 || plan.values_per_point > 6) return -1;
  stream_end_kernel<<<L.n_chunks_total, kSeT, 0, stream>>>(L, plan.values_per_point);
  return 1;
}

int launch_decode_fast(const Plan& plan, const DecLaunch& L, int sm_count, cudaStream_t stream) {
  FastDecParams Q;
  if (!decode_fast_plan(plan, &Q)) return -1;
  if (decode_side_active(plan, L)) {
    Q.n_side = plan.n_sections;
    for (uint32_t s2 = 0; s2 < plan.n_sections; ++s2) {
      Q.side_offset[s2] = plan.sections[s2].offset;
      Q.side_bpv[s2] = plan.sections[s2].bpv;
    }
  }
  const uint32_t nv = plan.values_per_point;
  // whole-row copy-out is a separate instantiation: its extra live state costs the dense XYZI reader (which never needs it:
  // one 16-byte store per point already) 4 % when it is merely a run-time branch
  bool dense_xyzi = nv == 4 && plan.point_step == 16;
  for (uint32_t k = 0; k < 4; ++k) dense_xyzi = dense_xyzi && Q.off[k] == 4 * k;
  const bool rows = Q.rows != 0 && !dense_xyzi;
  if (Q.n_floatn == nv) {
    if (nv == 4) return rows ? launch_fast<4, 8, false, true, 4>(Q, L, sm_count, stream) : launch_fast<4, 8, false, false, 4>(Q, L, sm_count, stream);
    return rows ? launch_fast<3, 8, false, true, 3>(Q, L, sm_count, stream) : launch_fast<3, 8, false, false, 3>(Q, L, sm_count, stream);
  }
  // mixed plans: (values per point, FloatN lanes) -- the group has 0, 3 or 4 lanes and at least one scalar field follows it
#define CLDN_FAST_MIXED(KK, FPP, NFF) \
  if (nv == KK && Q.n_floatn == NFF) return rows ? launch_fast<KK, FPP, true, true, NFF>(Q, L, sm_count, stream) : launch_fast<KK, FPP, true, false, NFF>(Q, L, sm_count, stream);
  CLDN_FAST_MIXED(3, 8, 0) CLDN_FAST_MIXED(4, 8, 0) CLDN_FAST_MIXED(4, 8, 3)
  CLDN_FAST_MIXED(5, 4, 0) CLDN_FAST_MIXED(5, 4, 3) CLDN_FAST_MIXED(5, 4, 4)
  CLDN_FAST_MIXED(6, 4, 0) CLDN_FAST_MIXED(6, 4, 3) CLDN_FAST_MIXED(6, 4, 4)
#undef CLDN_FAST_MIXED
  return -1;
}

}  // namespace cldn
