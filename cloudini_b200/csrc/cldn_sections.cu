// V5 adaptive integer sections, ENCODE side.
//
// Replaces the adaptive-int half of EncodeV5Stage1 (cloudini_lib/src/v5_codec.cpp:900-963): mode analysis on the
// first 4096 values of a call (:258-421), the four section writers (:423-491) and the placement of the sections
// behind each chunk's interleaved stream.
//
// Kernels (all stream-ordered, no host round trip):
//   probe_modes_kernel     one CTA per (frame, int field): the four candidate sizes on the probe window -> mode byte
//   encode_sections_kernel one CTA per (chunk, int field): section bytes into a scratch slot + their size
//   palette_overflow_kernel  rare: chunks with more distinct values than the shared-memory table holds
//   scan_sections_kernel   per frame: exclusive scan over chunks of the section bytes (feeds the regular kernel's
//                          output positions)
//   place_sections_kernel  after the regular stream kernel: copies every section behind its chunk's stream
#include <stdio.h>
#include <stdlib.h>

#include "cldn_device.cuh"
#include "cldn_kernels.h"

namespace cldn {

constexpr uint32_t kSmemPaletteSlots = 4096;   // open addressing, at most half full -> 2048 distinct values per chunk
constexpr uint32_t kGlobalPaletteSlots = 65536;  // 32768 values per chunk at most -> never more than half full
constexpr uint64_t kEmptyKey = 0xFFFFFFFFFFFFFFFFull;
constexpr uint32_t kOverflowTables = 64;
constexpr uint32_t kPlacePiece = 16384;   // bytes per staged piece of place_sections_kernel
constexpr int kSecThreads = 1024;  // one CTA per SM (shared-memory bound): use all its warp slots to hide the strided loads

// CTA-wide exclusive scan for kSecThreads threads; scratch = 33 uint32. Same contract as block_exclusive_scan.
__device__ __forceinline__ uint32_t sec_exclusive_scan(uint32_t v, uint32_t* scratch, uint32_t* total) {
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
    const uint32_t w = scratch[lane];
    uint32_t winc = w;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const uint32_t t = __shfl_up_sync(0xffffffffu, winc, d);
      if (lane >= d) winc += t;
    }
    scratch[lane] = winc - w;
    if (lane == 31) scratch[32] = winc;
  }
  __syncthreads();
  const uint32_t res = scratch[warp] + inc - v;
  *total = scratch[32];
  return res;
}

struct SecItem {
  const uint8_t* base;  // first point of the chunk + field offset
  uint32_t n;           // values in the chunk
  uint32_t step;
  uint8_t type;
  uint8_t bpv;
};

__device__ __forceinline__ int64_t item_value(const SecItem& it, uint32_t i) {
  return load_int_as_i64(it.base + static_cast<size_t>(i) * it.step, it.type);
}
__device__ __forceinline__ uint64_t item_raw(const SecItem& it, uint32_t i) {
  return load_raw_bits(it.base + static_cast<size_t>(i) * it.step, it.bpv);
}
// delta of value i to its predecessor inside the chunk (prev = 0 at the chunk start), wrapping like the reference's int64 math
__device__ __forceinline__ int64_t item_delta(const SecItem& it, uint32_t i) {
  const uint64_t v = static_cast<uint64_t>(item_value(it, i));
  const uint64_t p = i ? static_cast<uint64_t>(item_value(it, i - 1)) : 0ull;
  return static_cast<int64_t>(v - p);
}
__device__ __forceinline__ uint32_t bits_for_index(uint32_t unique) {  // bitsForPaletteIndex, v5_codec.cpp:196-207
  return unique <= 1 ? 0u : 32u - __clz(unique - 1u);
}
__device__ __forceinline__ uint64_t mix64(uint64_t x) {  // table placement only; any hash gives the same bytes
  x ^= x >> 33;
  x *= 0xff51afd7ed558ccdull;
  x ^= x >> 33;
  return x;
}

__device__ __forceinline__ uint32_t block_sum(uint32_t v, uint32_t* scratch) {
  uint32_t total;
  sec_exclusive_scan(v, scratch, &total);
  __syncthreads();
  return total;
}

// ---- run analysis shared by the probe and the writers ------------------------------------------------------------
// head(i): value i starts a new run. Rle compares raw values (v5_codec.cpp:301-318), DeltaRle compares deltas (:269-288).
template <bool DELTA>
__device__ __forceinline__ bool run_head(const SecItem& it, uint32_t i) {
  if (i == 0) return true;
  if (DELTA) return item_delta(it, i) != item_delta(it, i - 1);
  return item_raw(it, i) != item_raw(it, i - 1);
}

// Builds the list of run-head positions of the first `n` values into heads[] (uint16, position < 32768); returns the
// number of runs to every thread. Tile loop of kThreads*8 values, thread-blocked so that ranks follow value order.
template <bool DELTA>
__device__ uint32_t build_heads(const SecItem& it, uint32_t n, uint16_t* heads, uint32_t* scan) {
  uint32_t base = 0;
  for (uint32_t t0 = 0; t0 < n; t0 += kSecThreads * 8) {
    uint32_t flags = 0;
    const uint32_t i0 = t0 + threadIdx.x * 8;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      if (i0 + k < n && run_head<DELTA>(it, i0 + k)) flags |= 1u << k;
    }
    uint32_t total;
    uint32_t rank = base + sec_exclusive_scan(__popc(flags), scan, &total);
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      if (flags & (1u << k)) heads[rank++] = static_cast<uint16_t>(i0 + k);
    }
    base += total;
    __syncthreads();
  }
  return base;
}

template <bool DELTA>
__device__ __forceinline__ uint32_t run_bytes(const SecItem& it, uint32_t head, uint32_t len) {
  const uint32_t lb = uvarint_len(len);
  if (DELTA) return varint_len(zigzag_plus1(item_delta(it, head))) + lb;
  return it.bpv + lb;
}

// ---- section writers -----------------------------------------------------------------------------------------------
// DeltaVarint (mode 0), appendDeltaVarintSection v5_codec.cpp:423-432. Returns the section size.
__device__ uint32_t write_delta_section(const SecItem& it, uint8_t* out, uint32_t* scan) {
  if (threadIdx.x == 0) out[0] = 0;
  uint32_t base = 1;
  for (uint32_t t0 = 0; t0 < it.n; t0 += kSecThreads * 8) {
    const uint32_t i0 = t0 + threadIdx.x * 8;
    uint64_t u[8];
    uint32_t mine = 0;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      u[k] = 0;
      if (i0 + k < it.n) {
        u[k] = zigzag_plus1(item_delta(it, i0 + k));
        mine += varint_len(u[k]);
      }
    }
    uint32_t total;
    uint32_t off = base + sec_exclusive_scan(mine, scan, &total);
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      if (i0 + k < it.n) {
        ByteSink bs{out + off};
        bs.put_varint(u[k]);
        off = static_cast<uint32_t>(bs.p - out);
      }
    }
    base += total;
    __syncthreads();
  }
  return base;
}

// Rle (mode 2, v5_codec.cpp:471-491) / DeltaRle (mode 3, :447-460). Returns the section size.
template <bool DELTA>
__device__ uint32_t write_run_section(const SecItem& it, uint8_t* out, uint16_t* heads, uint32_t* scan) {
  const uint32_t runs = build_heads<DELTA>(it, it.n, heads, scan);
  if (threadIdx.x == 0) {
    out[0] = DELTA ? 3 : 2;
    store_u32(out + 1, runs);
  }
  uint32_t base = 5;
  for (uint32_t r0 = 0; r0 < runs; r0 += kSecThreads * 8) {
    const uint32_t q0 = r0 + threadIdx.x * 8;
    uint32_t mine = 0;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const uint32_t r = q0 + k;
      if (r < runs) {
        const uint32_t h = heads[r];
        const uint32_t len = ((r + 1 < runs) ? heads[r + 1] : it.n) - h;
        mine += run_bytes<DELTA>(it, h, len);
      }
    }
    uint32_t total;
    uint32_t off = base + sec_exclusive_scan(mine, scan, &total);
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const uint32_t r = q0 + k;
      if (r < runs) {
        const uint32_t h = heads[r];
        const uint32_t len = ((r + 1 < runs) ? heads[r + 1] : it.n) - h;
        ByteSink bs{out + off};
        if (DELTA) {
          bs.put_varint(zigzag_plus1(item_delta(it, h)));
        } else {
          const uint64_t raw = item_raw(it, h);
          for (int b = 0; b < it.bpv; ++b) bs.put_byte(static_cast<uint8_t>(raw >> (8 * b)));
        }
        uint64_t l = len;  // appendUVarint
        while (l > 0x7F) { bs.put_byte(static_cast<uint8_t>((l & 0x7F) | 0x80)); l >>= 7; }
        bs.put_byte(static_cast<uint8_t>(l));
        off = static_cast<uint32_t>(bs.p - out);
      }
    }
    base += total;
    __syncthreads();
  }
  return base;
}

// ---- palette ---------------------------------------------------------------------------------------------------------
// Open-addressing table (shared or global memory): keys[slot] = raw value, firsts[slot] = smallest index holding it,
// ranks[slot] = position in first-appearance order. The all-ones raw value cannot be a key (it is the empty marker);
// it only exists for 64-bit fields and gets the dedicated slot `slots` (one past the table).
struct PaletteTable {
  unsigned long long* keys;
  uint32_t* firsts;
  uint16_t* ranks;
  uint32_t slots;  // power of two; entry [slots] is the dedicated slot of the all-ones value
};

__device__ __forceinline__ uint32_t palette_find(const PaletteTable& T, uint64_t raw) {
  if (raw == kEmptyKey) return T.slots;
  uint32_t h = static_cast<uint32_t>(mix64(raw)) & (T.slots - 1);
  while (T.keys[h] != raw) h = (h + 1) & (T.slots - 1);
  return h;
}

// Inserts all values; returns false (to all threads) if more than slots/2 distinct values show up.
__device__ bool palette_insert_all(const PaletteTable& T, const SecItem& it, uint32_t n, uint32_t* s_count) {
  for (uint32_t i = threadIdx.x; i <= T.slots; i += blockDim.x) {
    T.keys[i] = kEmptyKey;
    T.firsts[i] = 0xFFFFFFFFu;
  }
  if (threadIdx.x == 0) *s_count = 0;
  __syncthreads();
  for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) {
    if (*reinterpret_cast<volatile uint32_t*>(s_count) > T.slots / 2) break;
    const uint64_t raw = item_raw(it, i);
    uint32_t h;
    if (raw == kEmptyKey) {
      h = T.slots;
    } else {
      h = static_cast<uint32_t>(mix64(raw)) & (T.slots - 1);
      while (true) {
        const unsigned long long k = T.keys[h];
        if (k == raw) break;
        if (k == kEmptyKey) {
          const unsigned long long old = atomicCAS(&T.keys[h], kEmptyKey, static_cast<unsigned long long>(raw));
          if (old == kEmptyKey) { atomicAdd(s_count, 1u); break; }
          if (old == raw) break;
        }
        h = (h + 1) & (T.slots - 1);
      }
    }
    // indexes arrive in roughly rising order, so after its first few appearances a value's entry is already below i:
    // the plain read keeps 32768 atomics off a handful of addresses (8 colours -> 4096 serialised updates each)
    if (reinterpret_cast<volatile uint32_t*>(T.firsts)[h] > i) atomicMin(&T.firsts[h], i);
  }
  __syncthreads();
  const bool ok = *s_count <= T.slots / 2;
  __syncthreads();
  return ok;
}

// Number of distinct values among the first n (probe) — or 0xFFFFFFFF when the table overflowed.
__device__ uint32_t palette_count_distinct(const PaletteTable& T, const SecItem& it, uint32_t n, uint32_t* s_count,
                                           uint32_t* scan) {
  if (!palette_insert_all(T, it, n, s_count)) return 0xFFFFFFFFu;
  const uint32_t special = (T.firsts[T.slots] != 0xFFFFFFFFu) ? 1u : 0u;
  return *s_count + special;
}

// Palette section (mode 1), appendPaletteSection v5_codec.cpp:462-469 + appendBitpackedIndexes :209-227.
// idx16 = shared uint16[32768]. Returns the section size or 0xFFFFFFFF if the table overflowed.
__device__ uint32_t write_palette_section(const PaletteTable& T, const SecItem& it, uint8_t* out, uint16_t* idx16,
                                          uint32_t* s_count, uint32_t* scan) {
  if (!palette_insert_all(T, it, it.n, s_count)) return 0xFFFFFFFFu;
  // ranks in first-appearance order: value i is a "first" iff the table says its smallest index is i
  uint32_t base = 0;
  for (uint32_t t0 = 0; t0 < it.n; t0 += kSecThreads * 8) {
    const uint32_t i0 = t0 + threadIdx.x * 8;
    uint32_t flags = 0;
    uint32_t slot[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      slot[k] = 0;
      if (i0 + k < it.n) {
        slot[k] = palette_find(T, item_raw(it, i0 + k));
        if (T.firsts[slot[k]] == i0 + k) flags |= 1u << k;
      }
    }
    uint32_t total;
    uint32_t rank = base + sec_exclusive_scan(__popc(flags), scan, &total);
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      if (flags & (1u << k)) {
        T.ranks[slot[k]] = static_cast<uint16_t>(rank);
        const uint64_t raw = item_raw(it, i0 + k);
        uint8_t* dst = out + 3 + static_cast<size_t>(rank) * it.bpv;
        for (int b = 0; b < it.bpv; ++b) dst[b] = static_cast<uint8_t>(raw >> (8 * b));
        ++rank;
      }
    }
    base += total;
    __syncthreads();
  }
  const uint32_t unique = base;
  if (threadIdx.x == 0) {
    out[0] = 1;
    store_u16(out + 1, unique & 0xFFFFu);  // static_cast<uint16_t>(palette.size())
  }
  for (uint32_t i = threadIdx.x; i < it.n; i += blockDim.x) idx16[i] = T.ranks[palette_find(T, item_raw(it, i))];
  __syncthreads();
  const uint32_t bits = bits_for_index(unique);
  const uint32_t idx_bytes = static_cast<uint32_t>((static_cast<uint64_t>(bits) * it.n + 7u) / 8u);
  uint8_t* ib = out + 3 + static_cast<size_t>(unique) * it.bpv;
  if (bits) {
    // every thread assembles whole output bytes: byte b holds stream bits [8b, 8b+8), index i sits at bit i*bits (LSB first)
    for (uint32_t b = threadIdx.x; b < idx_bytes; b += blockDim.x) {
      const uint32_t lo = 8u * b;
      uint32_t i = lo / bits;
      uint32_t acc = 0;
      while (i < it.n && i * bits < lo + 8u) {
        const int32_t sh = static_cast<int32_t>(i * bits) - static_cast<int32_t>(lo);
        const uint32_t v = idx16[i];
        acc |= sh >= 0 ? (v << sh) : (v >> (-sh));
        ++i;
      }
      ib[b] = static_cast<uint8_t>(acc);
    }
  }
  __syncthreads();
  return 3u + unique * it.bpv + idx_bytes;
}

// ---- shared memory layout of the section kernels -------------------------------------------------------------------
struct SecShared {
  uint32_t scan[kSecThreads / 32 + 1];
  uint32_t count;
  uint32_t pad_[2];
  unsigned long long keys[kSmemPaletteSlots + 1];
  uint32_t firsts[kSmemPaletteSlots + 1];
  uint16_t ranks[kSmemPaletteSlots + 2];
  uint16_t idx16[kChunkPoints + 2];  // palette indexes / run heads
};

__device__ __forceinline__ SecItem make_item(const EncFrame& F, const Plan& plan, uint32_t chunk, uint32_t sec) {
  SecItem it;
  const SectionField& sf = plan.sections[sec];
  it.base = F.in + static_cast<size_t>(chunk) * kChunkPoints * plan.point_step + sf.offset;
  it.n = min(kChunkPoints, F.n_points - chunk * kChunkPoints);
  it.step = plan.point_step;
  it.type = sf.type;
  it.bpv = sf.bpv;
  return it;
}

// ---- probe: selectBestAdaptiveIntMode on the first min(4096, chunk 0) values (v5_codec.cpp:387-421, 934-949) ------
__global__ void __launch_bounds__(kSecThreads, 1) probe_modes_kernel(const SecLaunch L) {
  extern __shared__ __align__(16) uint8_t dyn_smem[];
  SecShared& sh = *reinterpret_cast<SecShared*>(dyn_smem);
  const Plan& plan = *L.plan;
  const uint32_t ns = plan.n_sections;
  const uint32_t f = blockIdx.x / ns, s = blockIdx.x % ns;
  if (blockIdx.x == 0 && threadIdx.x == 0) L.sec_sizes[L.n_chunks_total * ns] = 0;   // the writers' overflow flag
  const EncFrame F = L.frames[f];
  if (F.n_points == 0) return;
  SecItem it = make_item(F, plan, 0, s);
  const uint32_t n = it.n > kProbePoints ? kProbePoints : it.n;  // whole chunk when it has <= 4096 points
  it.n = n;

  // DeltaVarint: 1 + sum of varint sizes
  uint32_t mine = 0;
  for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) mine += varint_len(zigzag_plus1(item_delta(it, i)));
  const uint32_t delta_bytes = 1u + block_sum(mine, sh.scan);

  // Rle / DeltaRle: 1 + 4 + sum over runs
  uint32_t rle_bytes, drle_bytes;
  {
    const uint32_t runs = build_heads<false>(it, n, sh.idx16, sh.scan);
    mine = 0;
    for (uint32_t r = threadIdx.x; r < runs; r += blockDim.x) {
      const uint32_t h = sh.idx16[r];
      mine += run_bytes<false>(it, h, ((r + 1 < runs) ? sh.idx16[r + 1] : n) - h);
    }
    rle_bytes = 5u + block_sum(mine, sh.scan);
  }
  {
    const uint32_t runs = build_heads<true>(it, n, sh.idx16, sh.scan);
    mine = 0;
    for (uint32_t r = threadIdx.x; r < runs; r += blockDim.x) {
      const uint32_t h = sh.idx16[r];
      mine += run_bytes<true>(it, h, ((r + 1 < runs) ? sh.idx16[r + 1] : n) - h);
    }
    drle_bytes = 5u + block_sum(mine, sh.scan);
  }
  // Palette: 1 + 2 + U*bpv + ceil(bits*n/8). 4096 probe values never overflow the table when it has >= 8192 slots;
  // with 4096 slots more than 2048 distinct values overflow -> palette then costs at least 2048*bpv + 12*4096/8 bytes,
  // which is still compared exactly via the global fallback below.
  PaletteTable T{sh.keys, sh.firsts, sh.ranks, kSmemPaletteSlots};
  uint32_t unique = palette_count_distinct(T, it, n, &sh.count, sh.scan);
  if (unique == 0xFFFFFFFFu) {
    // > 2048 distinct values among <= 4096 (rare): exact distinct count by brute force over the probe window (rare path, n <= 4096): value i is new iff no j < i equals it
    mine = 0;
    for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) {
      const uint64_t raw = item_raw(it, i);
      bool seen = false;
      for (uint32_t j = 0; j < i && !seen; ++j) seen = item_raw(it, j) == raw;
      mine += seen ? 0u : 1u;
    }
    unique = block_sum(mine, sh.scan);
  }
  const uint32_t bits = bits_for_index(unique);
  const uint32_t pal_bytes = 3u + unique * it.bpv + static_cast<uint32_t>((static_cast<uint64_t>(bits) * n + 7u) / 8u);

  if (threadIdx.x == 0) {
    uint32_t best = delta_bytes;
    uint8_t mode = 0;
    if (pal_bytes < best) { best = pal_bytes; mode = 1; }
    if (rle_bytes < best) { best = rle_bytes; mode = 2; }
    if (drle_bytes < best) { mode = 3; }
    L.modes[f * ns + s] = mode;
  }
}

// ---- sections ---------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kSecThreads, 1) encode_sections_kernel(const SecLaunch L) {
  extern __shared__ __align__(16) uint8_t dyn_smem[];
  SecShared& sh = *reinterpret_cast<SecShared*>(dyn_smem);
  const Plan& plan = *L.plan;
  const uint32_t ns = plan.n_sections;
  const uint32_t gc = blockIdx.x / ns, s = blockIdx.x % ns;
  if (plan.sections[s].bpv <= 4) return;  // encode_sections_staged_kernel
  const uint32_t f = L.chunk_frame[gc];
  const EncFrame F = L.frames[f];
  const uint32_t chunk = gc - L.chunk_first[f];
  if (L.empty_slots && chunk >= F.n_chunks) return;
  const SecItem it = make_item(F, plan, chunk, s);
  uint8_t* out = L.scratch + static_cast<size_t>(blockIdx.x) * L.sec_stride;
  const uint8_t mode = L.modes[f * ns + s];
  uint32_t size;
  switch (mode) {
    case 0: size = write_delta_section(it, out, sh.scan); break;
    case 2: size = write_run_section<false>(it, out, sh.idx16, sh.scan); break;
    case 3: size = write_run_section<true>(it, out, sh.idx16, sh.scan); break;
    default: {
      PaletteTable T{sh.keys, sh.firsts, sh.ranks, kSmemPaletteSlots};
      size = write_palette_section(T, it, out, sh.idx16, &sh.count, sh.scan);
    } break;
  }
  if (threadIdx.x == 0) {
    L.sec_sizes[blockIdx.x] = size;  // 0xFFFFFFFF = palette overflow, finished by the next kernel
    if (size == 0xFFFFFFFFu) atomicOr(L.sec_sizes + L.n_chunks_total * ns, 1u);   // "some item overflowed" (word behind the sizes)
  }
}

// ---- staged writers: fields of at most 4 bytes ------------------------------------------------------------------------
// The writers above fetch a value from the strided cloud every time they look at it: 3-4 sector loads per value, most of
// them from L2 (a chunk's field spans 32768 sectors = 1 MB, four times the L1), and the kernel waits on them (ncu:
// long-scoreboard 24 per issue, issue slots 19 % busy). Here the chunk's values are loaded ONCE, 32 independent loads in
// flight per thread, into 128 KB of shared memory; every pass of the four modes then runs from there.
//   layout   value i lives in word i ^ ((i >> 5) & 31): conflict-free both for the point-strided passes (lane = i & 31) and
//            for the thread-blocked passes (thread t owns values 32 t .. 32 t + 31, the order the output needs)
//   runs     one flag bit per value (mask word t = values of thread t, built with one ballot per warp and 32 values) and a
//            32-word summary of the non-empty mask words: the run that starts at a head ends at the next set bit, found
//            with two count-trailing-zeros -- no compacted head list
//   palette  same table as above; ranks in first-appearance order from the "first occurrence" flag bits; then every value
//            is replaced in place by its rank and 8 values are packed into exactly `bits` bytes by one thread
struct StagedShared {
  uint32_t scan[kSecThreads / 32 + 1];
  uint32_t count;
  uint32_t summary[32];
  uint32_t mask[kChunkPoints / 32];
  unsigned long long keys[kSmemPaletteSlots + 1];
  uint32_t firsts[kSmemPaletteSlots + 1];
  uint16_t ranks[kSmemPaletteSlots + 2];
  uint32_t vals[kChunkPoints];
};

__device__ __forceinline__ uint32_t sidx(uint32_t i) { return i ^ ((i >> 5) & 31u); }
// Signed fields are stored sign-extended to 32 bits (equal raw values stay equal, the low bpv bytes are the raw value), so
// ToInt64<T> is one widening conversion chosen by a CTA-uniform flag instead of a switch over the field type per value.
struct StagedItem {
  const uint32_t* vals;
  uint32_t n;
  bool is_signed;
  uint8_t bpv;
  __device__ __forceinline__ uint32_t raw(uint32_t i) const { return vals[sidx(i)]; }
  __device__ __forceinline__ int64_t value(uint32_t i) const {
    const uint32_t v = vals[sidx(i)];
    return is_signed ? static_cast<int64_t>(static_cast<int32_t>(v)) : static_cast<int64_t>(v);
  }
  __device__ __forceinline__ int64_t delta(uint32_t i) const { return value(i) - (i ? value(i - 1) : 0ll); }
};

// next set bit of the flag mask behind position i (exclusive), n if there is none
__device__ __forceinline__ uint32_t next_flag(const StagedShared& sh, uint32_t i, uint32_t n) {
  const uint32_t w = i >> 5, k = i & 31u;
  const uint32_t m = k == 31u ? 0u : (sh.mask[w] >> (k + 1u));
  if (m) return i + static_cast<uint32_t>(__ffs(static_cast<int>(m)));
  uint32_t s = w >> 5;
  const uint32_t kw = w & 31u;
  uint32_t sm = kw == 31u ? 0u : ((sh.summary[s] >> (kw + 1u)) << (kw + 1u));
  while (sm == 0u) {
    if (++s >= 32u) return n;
    sm = sh.summary[s];
  }
  const uint32_t w2 = 32u * s + static_cast<uint32_t>(__ffs(static_cast<int>(sm)) - 1);
  return 32u * w2 + static_cast<uint32_t>(__ffs(static_cast<int>(sh.mask[w2])) - 1);
}

// flag bits from a predicate over the values, evaluated point-strided (one ballot per warp and 32 values) + the summary
template <typename Pred>
__device__ __forceinline__ void build_flags(StagedShared& sh, uint32_t n, Pred pred) {
  const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
#pragma unroll 4
  for (uint32_t it = 0; it < kChunkPoints / kSecThreads; ++it) {
    const uint32_t i = it * kSecThreads + threadIdx.x;
    const bool f = i < n && pred(i);
    const uint32_t b = __ballot_sync(0xffffffffu, f);
    if (lane == 0) sh.mask[it * (kSecThreads / 32) + warp] = b;
  }
  __syncthreads();
  {
    const uint32_t b = __ballot_sync(0xffffffffu, sh.mask[32u * warp + lane] != 0u);
    if (lane == 0) sh.summary[warp] = b;
  }
  __syncthreads();
}

__device__ uint32_t staged_delta_section(StagedShared& sh, const StagedItem& it, uint8_t* out) {
  if (threadIdx.x == 0) out[0] = 0;
  const uint32_t i0 = 32u * threadIdx.x;
  const uint32_t cnt = i0 < it.n ? min(32u, it.n - i0) : 0u;
  uint32_t mine = 0;
  {
    int64_t prev = i0 && cnt ? it.value(i0 - 1) : 0ll;
    for (uint32_t k = 0; k < cnt; ++k) {
      const int64_t v = it.value(i0 + k);
      mine += varint_len(zigzag_plus1(v - prev));
      prev = v;
    }
  }
  uint32_t total;
  const uint32_t off = 1u + sec_exclusive_scan(mine, sh.scan, &total);
  {
    ByteSink bs{out + off};
    int64_t prev = i0 && cnt ? it.value(i0 - 1) : 0ll;
    for (uint32_t k = 0; k < cnt; ++k) {
      const int64_t v = it.value(i0 + k);
      bs.put_varint(zigzag_plus1(v - prev));
      prev = v;
    }
  }
  __syncthreads();
  return 1u + total;
}

template <bool DELTA>
__device__ uint32_t staged_run_section(StagedShared& sh, const StagedItem& it, uint8_t* out) {
  if (DELTA) build_flags(sh, it.n, [&](uint32_t i) { return i == 0u || it.delta(i) != it.delta(i - 1); });
  else build_flags(sh, it.n, [&](uint32_t i) { return i == 0u || it.raw(i) != it.raw(i - 1); });
  const uint32_t i0 = 32u * threadIdx.x;
  const uint32_t m = sh.mask[threadIdx.x];
  uint32_t mine = 0;
  for (uint32_t r = m; r; r &= r - 1u) {
    const uint32_t h = i0 + static_cast<uint32_t>(__ffs(static_cast<int>(r)) - 1);
    const uint32_t len = next_flag(sh, h, it.n) - h;
    mine += (DELTA ? static_cast<uint32_t>(varint_len(zigzag_plus1(it.delta(h)))) : static_cast<uint32_t>(it.bpv)) + uvarint_len(len);
  }
  uint32_t total, runs;
  const uint32_t off = 5u + sec_exclusive_scan(mine, sh.scan, &total);
  __syncthreads();
  sec_exclusive_scan(__popc(m), sh.scan, &runs);
  if (threadIdx.x == 0) {
    out[0] = DELTA ? 3 : 2;
    store_u32(out + 1, runs);
  }
  ByteSink bs{out + off};
  for (uint32_t r = m; r; r &= r - 1u) {
    const uint32_t h = i0 + static_cast<uint32_t>(__ffs(static_cast<int>(r)) - 1);
    uint32_t l = next_flag(sh, h, it.n) - h;
    if (DELTA) {
      bs.put_varint(zigzag_plus1(it.delta(h)));
    } else {
      const uint32_t raw = it.raw(h);
      for (int b = 0; b < it.bpv; ++b) bs.put_byte(static_cast<uint8_t>(raw >> (8 * b)));
    }
    while (l > 0x7Fu) { bs.put_byte(static_cast<uint8_t>((l & 0x7Fu) | 0x80u)); l >>= 7; }  // appendUVarint
    bs.put_byte(static_cast<uint8_t>(l));
  }
  __syncthreads();
  return 5u + total;
}

__device__ uint32_t staged_palette_section(StagedShared& sh, const StagedItem& it, uint8_t* out) {
  PaletteTable T{sh.keys, sh.firsts, sh.ranks, kSmemPaletteSlots};
  for (uint32_t i = threadIdx.x; i <= T.slots; i += blockDim.x) {
    T.keys[i] = kEmptyKey;
    T.firsts[i] = 0xFFFFFFFFu;
  }
  if (threadIdx.x == 0) sh.count = 0;
  __syncthreads();
  for (uint32_t i = threadIdx.x; i < it.n; i += blockDim.x) {
    if (*reinterpret_cast<volatile uint32_t*>(&sh.count) > T.slots / 2) break;
    const uint64_t raw = it.raw(i);  // <= 32 bits: never the empty marker
    uint32_t h = static_cast<uint32_t>(mix64(raw)) & (T.slots - 1);
    while (true) {
      const unsigned long long k = T.keys[h];
      if (k == raw) break;
      if (k == kEmptyKey) {
        const unsigned long long old = atomicCAS(&T.keys[h], kEmptyKey, static_cast<unsigned long long>(raw));
        if (old == kEmptyKey) { atomicAdd(&sh.count, 1u); break; }
        if (old == raw) break;
      }
      h = (h + 1) & (T.slots - 1);
    }
    if (reinterpret_cast<volatile uint32_t*>(T.firsts)[h] > i) atomicMin(&T.firsts[h], i);
  }
  __syncthreads();
  if (sh.count > T.slots / 2) return 0xFFFFFFFFu;  // more distinct values than the table holds: palette_overflow_kernel
  build_flags(sh, it.n, [&](uint32_t i) { return T.firsts[palette_find(T, it.raw(i))] == i; });
  const uint32_t i0 = 32u * threadIdx.x;
  const uint32_t m = sh.mask[threadIdx.x];
  uint32_t unique;
  uint32_t rank = sec_exclusive_scan(__popc(m), sh.scan, &unique);
  for (uint32_t r = m; r; r &= r - 1u) {
    const uint32_t i = i0 + static_cast<uint32_t>(__ffs(static_cast<int>(r)) - 1);
    const uint32_t raw = it.raw(i);
    T.ranks[palette_find(T, raw)] = static_cast<uint16_t>(rank);
    uint8_t* dst = out + 3 + static_cast<size_t>(rank) * it.bpv;
    for (int b = 0; b < it.bpv; ++b) dst[b] = static_cast<uint8_t>(raw >> (8 * b));
    ++rank;
  }
  if (threadIdx.x == 0) {
    out[0] = 1;
    store_u16(out + 1, unique & 0xFFFFu);  // static_cast<uint16_t>(palette.size())
  }
  __syncthreads();
  uint32_t* vals = const_cast<uint32_t*>(it.vals);
  for (uint32_t i = threadIdx.x; i < it.n; i += blockDim.x) vals[sidx(i)] = T.ranks[palette_find(T, vals[sidx(i)])];
  __syncthreads();
  const uint32_t bits = bits_for_index(unique);
  const uint32_t idx_bytes = static_cast<uint32_t>((static_cast<uint64_t>(bits) * it.n + 7u) / 8u);
  uint8_t* ib = out + 3 + static_cast<size_t>(unique) * it.bpv;
  if (bits) {
    // 8 indexes are exactly `bits` bytes: unit u = values 8 u .. 8 u + 7 -> bytes [u * bits, (u + 1) * bits), LSB first
    const uint32_t units = (it.n + 7u) / 8u;
    for (uint32_t u = threadIdx.x; u < units; u += blockDim.x) {
      unsigned long long lo = 0, hi = 0;
#pragma unroll
      for (uint32_t k = 0; k < 8; ++k) {
        const uint32_t i = 8u * u + k;
        const unsigned long long v = i < it.n ? vals[sidx(i)] : 0u;
        const uint32_t sh_ = k * bits;
        if (sh_ < 64u) {
          lo |= v << sh_;
          if (sh_ + bits > 64u) hi |= v >> (64u - sh_);
        } else {
          hi |= v << (sh_ - 64u);
        }
      }
      const uint32_t b0 = u * bits;
      const uint32_t nb = min(bits, idx_bytes - b0);
      for (uint32_t b = 0; b < nb; ++b) ib[b0 + b] = static_cast<uint8_t>(b < 8u ? (lo >> (8u * b)) : (hi >> (8u * (b - 8u))));
    }
  }
  __syncthreads();
  return 3u + unique * it.bpv + idx_bytes;
}

__global__ void __launch_bounds__(kSecThreads, 1) encode_sections_staged_kernel(const SecLaunch L) {
  extern __shared__ __align__(16) uint8_t dyn_smem[];
  StagedShared& sh = *reinterpret_cast<StagedShared*>(dyn_smem);
  const Plan& plan = *L.plan;
  const uint32_t ns = plan.n_sections;
  const uint32_t gc = blockIdx.x / ns, s = blockIdx.x % ns;
  if (plan.sections[s].bpv > 4) return;  // 64-bit fields: encode_sections_kernel
  const uint32_t f = L.chunk_frame[gc];
  const EncFrame F = L.frames[f];
  const uint32_t chunk = gc - L.chunk_first[f];
  if (L.empty_slots && chunk >= F.n_chunks) return;
  const SecItem src = make_item(F, plan, chunk, s);
  const bool is_signed = src.type == CLDN_INT8 || src.type == CLDN_INT16 || src.type == CLDN_INT32;
  const uint32_t ext_shift = 32u - 8u * src.bpv;
  // the one pass over the cloud: 32 independent strided loads per thread
#pragma unroll 8
  for (uint32_t k = 0; k < kChunkPoints / kSecThreads; ++k) {
    const uint32_t i = k * kSecThreads + threadIdx.x;
    if (i < src.n) {
      const uint32_t raw = static_cast<uint32_t>(item_raw(src, i));
      sh.vals[sidx(i)] = is_signed ? static_cast<uint32_t>(static_cast<int32_t>(raw << ext_shift) >> ext_shift) : raw;
    }
  }
  __syncthreads();
  const StagedItem it{sh.vals, src.n, is_signed, src.bpv};
  uint8_t* out = L.scratch + static_cast<size_t>(blockIdx.x) * L.sec_stride;
  const uint8_t mode = L.modes[f * ns + s];
  uint32_t size;
  switch (mode) {
    case 0: size = staged_delta_section(sh, it, out); break;
    case 2: size = staged_run_section<false>(sh, it, out); break;
    case 3: size = staged_run_section<true>(sh, it, out); break;
    default: size = staged_palette_section(sh, it, out); break;
  }
  if (threadIdx.x == 0) {
    L.sec_sizes[blockIdx.x] = size;  // 0xFFFFFFFF = palette overflow, finished by the next kernel
    if (size == 0xFFFFFFFFu) atomicOr(L.sec_sizes + L.n_chunks_total * ns, 1u);   // "some item overflowed" (word behind the sizes)
  }
}

// Chunks whose palette does not fit the shared-memory table: same algorithm on a 65536-slot table in global memory.
// A fixed pool of kOverflowTables CTAs, each owning one table, sweeps the (normally empty) list of flagged items.
__global__ void __launch_bounds__(kSecThreads, 1) palette_overflow_kernel(const SecLaunch L) {
  extern __shared__ __align__(16) uint8_t dyn_smem[];
  SecShared& sh = *reinterpret_cast<SecShared*>(dyn_smem);
  const Plan& plan = *L.plan;
  const uint32_t ns = plan.n_sections;
  const uint32_t items = L.n_chunks_total * ns;
  if (L.sec_sizes[items] == 0u) return;   // no writer overflowed its shared-memory table (the normal case)
  // table layout per CTA: keys[65537] u64 | firsts[65537] u32 | ranks[65538] u16
  const size_t words_per_table = (kGlobalPaletteSlots + 1) + (kGlobalPaletteSlots + 2) / 2 + (kGlobalPaletteSlots + 8) / 4;
  unsigned long long* basep = reinterpret_cast<unsigned long long*>(L.hash_scratch) + words_per_table * blockIdx.x;
  PaletteTable T;
  T.keys = basep;
  T.firsts = reinterpret_cast<uint32_t*>(basep + kGlobalPaletteSlots + 1);
  T.ranks = reinterpret_cast<uint16_t*>(T.firsts + kGlobalPaletteSlots + 2);
  T.slots = kGlobalPaletteSlots;
  for (uint32_t item = blockIdx.x; item < items; item += gridDim.x) {
    if (L.sec_sizes[item] != 0xFFFFFFFFu) continue;
    const uint32_t gc = item / ns, s = item % ns;
    const uint32_t f = L.chunk_frame[gc];
    const EncFrame F = L.frames[f];
    if (L.empty_slots && gc - L.chunk_first[f] >= F.n_chunks) continue;  // (an empty slot's size word is never written)
    const SecItem it = make_item(F, plan, gc - L.chunk_first[f], s);
    uint8_t* out = L.scratch + static_cast<size_t>(item) * L.sec_stride;
    const uint32_t size = write_palette_section(T, it, out, sh.idx16, &sh.count, sh.scan);
    if (threadIdx.x == 0) L.sec_sizes[item] = size;
    __syncthreads();
  }
}

// Per frame: sec_excl[c] = section bytes of all chunks before c (n_chunks + 1 entries). One warp per frame: lanes take
// chunks 32 at a time, a shuffle scan gives the running sums (a thread per frame walked 31 dependent loads).
__global__ void scan_sections_kernel(const SecLaunch L) {
  const uint32_t f = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const uint32_t lane = threadIdx.x & 31u;
  if (f >= L.n_frames) return;
  const uint32_t ns = L.plan->n_sections;
  const uint32_t c0 = L.chunk_first[f];
  const uint32_t nc = L.frames[f].n_chunks;
  uint32_t* excl = L.sec_excl + c0 + f;
  uint32_t acc = 0;
  for (uint32_t b = 0; b < nc; b += 32u) {
    const uint32_t c = b + lane;
    uint32_t mine = 0;
    if (c < nc) {
      for (uint32_t s = 0; s < ns; ++s) mine += L.sec_sizes[(c0 + c) * ns + s];
    }
    uint32_t inc = mine;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const uint32_t t = __shfl_up_sync(0xffffffffu, inc, d);
      if (lane >= static_cast<uint32_t>(d)) inc += t;
    }
    if (c < nc) excl[c] = acc + inc - mine;
    acc += __shfl_sync(0xffffffffu, inc, 31);
  }
  if (lane == 0) excl[nc] = acc;
}

// After the regular kernel: chunk c's sections go right behind its interleaved stream.
__global__ void __launch_bounds__(kThreads) place_sections_kernel(const SecLaunch L, const uint64_t* status, uint32_t epoch,
                                                                   uint32_t tile_points) {
  const Plan& plan = *L.plan;
  const uint32_t ns = plan.n_sections;
  const uint32_t gc = blockIdx.x / ns, s = blockIdx.x % ns;
  const uint32_t f = L.chunk_frame[gc];
  const EncFrame F = L.frames[f];
  const uint32_t chunk = gc - L.chunk_first[f];
  if (L.empty_slots && chunk >= F.n_chunks) return;
  const uint32_t tiles_per_chunk = kChunkPoints / tile_points;
  uint32_t last_tile = (chunk + 1) * tiles_per_chunk - 1;
  if (last_tile >= F.n_tiles) last_tile = F.n_tiles - 1;
  const uint64_t data_incl = status_value(status[F.tile_begin + last_tile]);  // inclusive data bytes up to this chunk's end
  uint64_t pos = L.header_bytes + 4ull * (chunk + 1) + data_incl + F.sec_excl[chunk];
  for (uint32_t k = 0; k < s; ++k) pos += L.sec_sizes[gc * ns + k];
  const uint32_t size = L.sec_sizes[blockIdx.x];
  const uint8_t* src = L.scratch + static_cast<size_t>(blockIdx.x) * L.sec_stride;
  uint8_t* dst = F.out + pos;
  if (pos + size > F.out_cap) {  // the reference: "Output buffer too small for uncompressed chunk" (chunk_writer.cpp:33-35)
    if (threadIdx.x == 0) report_frame_error(L, f, DEV_ERR_ENCODE_OUTPUT_SMALL);
    return;
  }
  // through shared memory in 16 KB pieces: 16-byte loads from the (aligned) scratch slot, 16-byte stores at whatever alignment
  // the section lands on (copy_stage_to_global shifts the words) -- the byte loop this replaces moved 14 MB one byte at a time
  __shared__ uint4 stage4[(kPlacePiece + 32) / 16];   // (a uint4 array: 16-byte aligned without an attribute)
  uint8_t* stage = reinterpret_cast<uint8_t*>(stage4);
  for (uint32_t p0 = 0; p0 < size; p0 += kPlacePiece) {
    const uint32_t len = min(kPlacePiece, size - p0);
    const uint4* sv = reinterpret_cast<const uint4*>(src + p0);
    for (uint32_t v = threadIdx.x; v < (len + 15u) / 16u; v += blockDim.x) reinterpret_cast<uint4*>(stage)[v] = sv[v];
    __syncthreads();
    copy_stage_to_global(stage, len, dst + p0);
    __syncthreads();
  }
}

// ------------------------------------------------------------------------------------------------------------------
size_t palette_overflow_scratch_bytes() {
  const size_t words_per_table = (kGlobalPaletteSlots + 1) + (kGlobalPaletteSlots + 2) / 2 + (kGlobalPaletteSlots + 8) / 4;
  return words_per_table * 8 * kOverflowTables;
}

int launch_encode_sections(const Plan& plan, const SecLaunch& L, cudaStream_t stream) {
  if (L.n_chunks_total == 0) return 0;
  const size_t smem = sizeof(SecShared) + 16;
  if (raise_smem_limit(probe_modes_kernel, smem) != cudaSuccess) return -1;
  if (raise_smem_limit(encode_sections_kernel, smem) != cudaSuccess) return -1;
  if (raise_smem_limit(palette_overflow_kernel, smem) != cudaSuccess) return -1;
  // fields of <= 4 bytes: the staged writers (values loaded once into shared memory); 64-bit fields: the writers that
  // read the cloud in place
  bool any_small = false, any_wide = false;
  for (uint32_t s = 0; s < plan.n_sections; ++s) (plan.sections[s].bpv <= 4 ? any_small : any_wide) = true;
  int launched = 3;
  probe_modes_kernel<<<L.n_frames * plan.n_sections, kSecThreads, smem, stream>>>(L);
  if (any_small) {
    const size_t smem2 = sizeof(StagedShared) + 16;
    if (raise_smem_limit(encode_sections_staged_kernel, smem2) != cudaSuccess) return -1;
    encode_sections_staged_kernel<<<L.n_chunks_total * plan.n_sections, kSecThreads, smem2, stream>>>(L);
    ++launched;
  }
  if (any_wide) {
    encode_sections_kernel<<<L.n_chunks_total * plan.n_sections, kSecThreads, smem, stream>>>(L);
    ++launched;
  }
  palette_overflow_kernel<<<kOverflowTables, kSecThreads, smem, stream>>>(L);
  scan_sections_kernel<<<(L.n_frames * 32 + 127) / 128, 128, 0, stream>>>(L);
  count_launch(launched);
  return launched;
}

int launch_place_sections(const Plan& plan, const SecLaunch& L, const uint64_t* status, uint32_t epoch, uint32_t tile_points,
                          cudaStream_t stream) {
  if (L.n_chunks_total == 0) return 0;
  place_sections_kernel<<<L.n_chunks_total * plan.n_sections, kThreads, 0, stream>>>(L, status, epoch, tile_points);
  count_launch(1);
  return 1;
}

}  // namespace cldn
