// DECODE of FloatN-only regular streams (XYZ / XYZI: BASELINE configs C1, C2, C5 and the float part of C3).
//
// Same arithmetic as FieldDecoderFloatN_Lossy::decode (cloudini_lib/src/field_decoder.cpp:43-86), different shape:
// the chunk's byte stream is cut into fixed 8 KB tiles (256 threads x 2 16-byte vectors). Inside a tile a byte with a
// clear MSB ends a value: a CTA scan ranks the terminators, every thread takes a run of ceil(values / 256) consecutive
// values (the start of the run is the byte behind the (run * VT - 1)-th terminator, found with a small table), decodes
// them with a streaming 4-byte window, and the per-field running values come from a CTA segmented scan (reset at NaN).
// Two kernels share these building blocks:
//   decode_chunks_seq_kernel  large batches: persistent CTAs claim whole chunks from a counter and carry the value
//                             count and the per-field values from tile to tile in registers; CTA 0 also walks the u32
//                             chunk prefixes and publishes them while the others are already decoding;
//   decode_tiles_kernel       small batches: one CTA per tile of every chunk, two decoupled look-backs over the tiles
//                             of a chunk: (1) number of values before the tile, (2) per-field sum since the last reset.
#include <stdio.h>

#include <type_traits>

#include "cldn_device.cuh"
#include "cldn_kernels.h"

namespace cldn {

constexpr int kVec = 2;        // adjacent 16-byte vectors per thread
constexpr int kDT = 256;       // threads per decode CTA (tile = kDT * 16 * kVec stream bytes)
constexpr int kSeqMinBlocks = 3;   // resident CTAs per SM of the tile and chunk-sequential readers
constexpr int kTB = kDT * 16 * kVec;  // stream bytes per tile (8192)
constexpr int kTLook = 16;     // look-behind bytes staged in front of the tile
constexpr uint32_t kRecWords = 8;  // look-back record: sum[4], rst, flag, pad, pad
constexpr int kOStageOffset = (kTLook + kTB + 16 + 2 * kDT + 64 + 15) / 16 * 16;  // float staging of dense layouts
constexpr int kOStageBytes = (3 + kTB + 4) * 4;  // at most one value per stream byte (+ alignment slack)

// ---- per-chunk tile counts and their exclusive scan (grid of the tile kernel is an upper bound computed on the host)
__global__ void count_tiles_kernel(const DecLaunch L) {
  const uint32_t gc = blockIdx.x * blockDim.x + threadIdx.x;
  if (gc >= L.n_chunks_total) return;
  // frame of this chunk
  uint32_t lo = 0, hi = L.n_frames - 1;
  while (lo < hi) {
    const uint32_t mid = (lo + hi + 1) >> 1;
    if (L.frames[mid].chunk_begin <= gc) lo = mid; else hi = mid - 1;
  }
  L.chunk_frame[gc] = lo;
  if (chunk_slot_empty(L.frames[lo], gc)) {  // no tile
    L.chunk_tiles[gc] = 0;
    L.stream_end[gc] = 0xFFFFFFFFu;
    return;
  }
  const uint8_t* body = L.frames[lo].payload + L.chunk_offsets[gc];
  const uint32_t mis = static_cast<uint32_t>(reinterpret_cast<uintptr_t>(body) & 15u);
  const uint32_t size = L.chunk_sizes[gc];
  L.stream_end[gc] = 0xFFFFFFFFu;  // set by the tile that decodes the chunk's last regular value
  if (L.chunk_bytes_max && size > L.chunk_bytes_max) {  // past the bound the grid was sized from: no tile, the frame fails
    L.chunk_tiles[gc] = 0;
    report_frame_error(L, lo, DEV_ERR_CHUNK_SIZE);
    return;
  }
  L.chunk_tiles[gc] = size ? (size + mis + kTB - 1) / kTB : 0;
  const uint32_t chunk = gc - L.frames[lo].chunk_begin;
  const uint32_t n_points = min(kChunkPoints, L.frames[lo].n_points - chunk * kChunkPoints);
  if (size == 0 && n_points * L.plan->values_per_point > 0) report_frame_error(L, lo, DEV_ERR_TRUNCATED);
}

// single CTA: exclusive scan of chunk_tiles -> chunk_tile_begin[0..n], total in chunk_tile_begin[n]
__global__ void scan_tiles_kernel(const DecLaunch L) {
  __shared__ uint32_t s_scan[kThreads / 32 + 1];
  uint32_t base = 0;
  for (uint32_t c0 = 0; c0 < L.n_chunks_total; c0 += kThreads) {
    const uint32_t c = c0 + threadIdx.x;
    const uint32_t v = c < L.n_chunks_total ? L.chunk_tiles[c] : 0;
    uint32_t total;
    const uint32_t ex = block_exclusive_scan(v, s_scan, &total);
    if (c < L.n_chunks_total) {
      L.chunk_tile_begin[c] = base + ex;
      for (uint32_t k = 0; k < v; ++k) L.tile_chunk[base + ex + k] = c;  // tile -> chunk table (<= ~60 tiles per chunk)
    }
    base += total;
    __syncthreads();
  }
  if (threadIdx.x == 0) L.chunk_tile_begin[L.n_chunks_total] = base;
}

// ---- segmented sums over K int32 slots ------------------------------------------------------------------------------
template <int K>
struct SegK {
  int32_t sum[K];
  uint32_t rst;
};
__device__ __forceinline__ int32_t wadd32(int32_t a, int32_t b) { return static_cast<int32_t>(static_cast<uint32_t>(a) + static_cast<uint32_t>(b)); }
template <int K>
__device__ __forceinline__ SegK<K> seg_then(const SegK<K>& a, const SegK<K>& b) {  // a earlier in the stream than b
  SegK<K> r;
#pragma unroll
  for (int j = 0; j < K; ++j) r.sum[j] = ((b.rst >> j) & 1u) ? b.sum[j] : wadd32(a.sum[j], b.sum[j]);
  r.rst = a.rst | b.rst;
  return r;
}
template <int K>
__device__ __forceinline__ SegK<K> seg_shfl_up(const SegK<K>& a, int d) {
  SegK<K> r;
#pragma unroll
  for (int j = 0; j < K; ++j) r.sum[j] = __shfl_up_sync(0xffffffffu, a.sum[j], d);
  r.rst = __shfl_up_sync(0xffffffffu, a.rst, d);
  return r;
}
template <int K>
__device__ __forceinline__ SegK<K> seg_shfl(const SegK<K>& a, int src) {
  SegK<K> r;
#pragma unroll
  for (int j = 0; j < K; ++j) r.sum[j] = __shfl_sync(0xffffffffu, a.sum[j], src);
  r.rst = __shfl_sync(0xffffffffu, a.rst, src);
  return r;
}
template <int K>
__device__ __forceinline__ SegK<K> seg_identity() {
  SegK<K> r;
#pragma unroll
  for (int j = 0; j < K; ++j) r.sum[j] = 0;
  r.rst = 0;
  return r;
}

struct TileShared {
  uint32_t scan[kDT / 32 + 1];
  uint32_t done;  // values of this chunk before the tile
  int32_t w_sum[kDT / 32][4];
  uint32_t w_rst[kDT / 32];
  int32_t carry[4];
};

// ---- look-back 2 records: K self-validating 64-bit words per tile ---------------------------------------------------
// word j = [63:42] epoch  [41:38] reset mask (word 0 only)  [33:32] state (1 aggregate, 2 inclusive)  [31:0] sum[j]
// Every word carries its own tag, so no fence / flag ordering is needed: a reader retries until all K words show the
// current epoch and the same state.
__device__ __forceinline__ uint64_t rec_word(uint32_t epoch, uint32_t rst, uint32_t state, int32_t sum) {
  return (static_cast<uint64_t>(epoch & 0x3FFFFFu) << 42) | (static_cast<uint64_t>(rst & 0xFu) << 38) |
         (static_cast<uint64_t>(state & 3u) << 32) | static_cast<uint32_t>(sum);
}
template <int K>
__device__ __forceinline__ void publish_words(uint64_t* rec, const SegK<K>& v, uint32_t epoch, uint32_t state) {
#pragma unroll
  for (int j = 0; j < K; ++j) st_relaxed_u64(rec + j, rec_word(epoch, j == 0 ? v.rst : 0u, state, v.sum[j]));
}
// Returns the state (0 = not ready / torn) and fills v.
template <int K>
__device__ __forceinline__ uint32_t read_words(const uint64_t* rec, uint32_t epoch, SegK<K>& v) {
  uint64_t w[K];
#pragma unroll
  for (int j = 0; j < K; ++j) w[j] = ld_relaxed_u64(rec + j);
  const uint32_t state = static_cast<uint32_t>(w[0] >> 32) & 3u;
  bool ok = state != 0;
#pragma unroll
  for (int j = 0; j < K; ++j) {
    ok = ok && (static_cast<uint32_t>(w[j] >> 42) == (epoch & 0x3FFFFFu)) && ((static_cast<uint32_t>(w[j] >> 32) & 3u) == state);
    v.sum[j] = static_cast<int32_t>(static_cast<uint32_t>(w[j]));
  }
  v.rst = static_cast<uint32_t>(w[0] >> 38) & 0xFu;
  return ok ? state : 0u;
}

// Warp-wide look-back over the records of the tiles [first, me) of a chunk; returns the combination of all
// predecessors (stream order) to every lane.
template <int K>
__device__ __forceinline__ SegK<K> sums_lookback(const uint64_t* recs, uint32_t first, uint32_t me, uint32_t epoch) {
  const int lane = threadIdx.x & 31;
  SegK<K> acc = seg_identity<K>();  // combination of the predecessors inspected so far (they all FOLLOW the next batch)
  int64_t idx = static_cast<int64_t>(me) - 1;
  while (idx >= static_cast<int64_t>(first)) {
    const int64_t mine = idx - lane;
    SegK<K> r = seg_identity<K>();
    bool is_incl = true;  // virtual tiles before the chunk start: inclusive identity
    if (mine >= static_cast<int64_t>(first)) {
      uint32_t st;
      do { st = read_words<K>(recs + mine * 4, epoch, r); } while (st == 0);
      is_incl = (st == 2u);
    }
    const uint32_t incl_mask = __ballot_sync(0xffffffffu, is_incl);
    const int stop = incl_mask ? (__ffs(incl_mask) - 1) : 31;
    if (lane > stop) r = seg_identity<K>();
    // ordered reduction: lane index grows backwards in the stream, so lane l's partial (lanes 0..l) = r_l then partial(l-1)
    SegK<K> inc = r;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const SegK<K> up = seg_shfl_up<K>(inc, d);
      if (lane >= d) inc = seg_then<K>(inc, up);
    }
    const SegK<K> batch = seg_shfl<K>(inc, 31);  // lanes > stop hold identities, so lane 31 has the batch up to `stop`
    acc = seg_then<K>(batch, acc);
    if (incl_mask) break;
    idx -= 32;
  }
  return acc;
}

// Per-thread value run in LOCAL slot numbering: value k of the run is local slot k % K; its global field is
// (phase + k) % K with phase = (values before the run) % K, so accumulators and per-field constants are rotated once
// per thread instead of specialising the unrolled loops per phase.
template <int K, int VTMAX>
__device__ __forceinline__ SegK<K> run_reduce_local(const int32_t (&d)[VTMAX], unsigned long long nanm, uint32_t n) {
  SegK<K> m = seg_identity<K>();
  if (nanm == 0ull) {  // no NaN marker in my run (the common case): plain wrapping sums
#pragma unroll
    for (int k = 0; k < VTMAX; ++k) {
      if (k >= static_cast<int>(n)) break;
      m.sum[k % K] = wadd32(m.sum[k % K], d[k]);
    }
    return m;
  }
#pragma unroll
  for (int k = 0; k < VTMAX; ++k) {
    if (k >= static_cast<int>(n)) break;
    const int j = k % K;
    if ((nanm >> k) & 1ull) { m.sum[j] = 0; m.rst |= 1u << j; }
    else m.sum[j] = wadd32(m.sum[j], d[k]);
  }
  return m;
}
// out[l] = in[(l + phase) % K]: a two-stage barrel rotation (K == 4) / two selects per element (K == 3)
template <int K, typename T>
__device__ __forceinline__ void rotate_k(const T (&in)[K], uint32_t phase, T (&out)[K]) {
  if (K == 4) {
    const bool p1 = phase & 1u, p2 = phase & 2u;
    T t[K];
#pragma unroll
    for (int l = 0; l < K; ++l) t[l] = p1 ? in[(l + 1) % K] : in[l];
#pragma unroll
    for (int l = 0; l < K; ++l) out[l] = p2 ? t[(l + 2) % K] : t[l];
  } else {
    const bool p1 = phase == 1u, p2 = phase == 2u;
#pragma unroll
    for (int l = 0; l < K; ++l) out[l] = p1 ? in[(l + 1) % K] : (p2 ? in[(l + 2) % K] : in[l]);
  }
}
// local slot l -> global field (l + phase) % K
template <int K>
__device__ __forceinline__ SegK<K> seg_to_global(const SegK<K>& a, uint32_t phase) {
  SegK<K> r;
  rotate_k<K, int32_t>(a.sum, (K - phase) % K, r.sum);  // r.sum[g] = a.sum[(g - phase) mod K]
  r.rst = ((a.rst << phase) | (a.rst >> (K - phase))) & ((1u << K) - 1u);
  return r;
}
// MODE 0: any layout (byte-wise stores, skipped fields honoured); 1: 4-byte aligned fields, direct 4-byte stores;
// 2: dense float32xK points (step == 4K, offsets 0,4,..): the floats are staged in shared memory (`ostage`, indexed by
//    the value's position in the tile) and leave with coalesced 16-byte stores (copy_out_dense) -- a direct store
//    would touch one 32-byte sector per value.
template <int K, int VTMAX, int MODE>
__device__ __forceinline__ void run_emit_local(const int32_t (&d)[VTMAX], unsigned long long nanm, uint32_t n, const int32_t (&cur_global)[K],
                                               uint32_t phase, uint8_t* out, uint32_t pbase, uint32_t step, const float (&mul)[4],
                                               const uint32_t (&off)[4], uint32_t* ostage = nullptr) {
  constexpr bool ALIGNED4 = MODE >= 1;
  // rotate the running values and the per-field constants into local numbering
  int32_t cur[K];
  float lmul[K], gmul[K];
  uint32_t loff[K], goff[K];
#pragma unroll
  for (int g = 0; g < K; ++g) { gmul[g] = mul[g]; goff[g] = off[g]; }
  rotate_k<K, int32_t>(cur_global, phase, cur);
  rotate_k<K, float>(gmul, phase, lmul);
  rotate_k<K, uint32_t>(goff, phase, loff);
  if (MODE == 2 && nanm == 0ull) {  // dense layout, no NaN in my run
#pragma unroll
    for (int k = 0; k < VTMAX; ++k) {
      if (k >= static_cast<int>(n)) break;
      const int l = k % K;
      cur[l] = wadd32(cur[l], d[k]);
      ostage[k] = __float_as_uint(__fmul_rn(__int2float_rn(cur[l]), lmul[l]));
    }
    return;
  }
#pragma unroll
  for (int k = 0; k < VTMAX; ++k) {
    if (k >= static_cast<int>(n)) break;
    const int l = k % K;
    const bool nan = (nanm >> k) & 1ull;
    if (nan) cur[l] = 0; else cur[l] = wadd32(cur[l], d[k]);
    if (MODE == 2) {
      const float f = nan ? __uint_as_float(0x7FC00000u) : __fmul_rn(__int2float_rn(cur[l]), lmul[l]);
      ostage[k] = __float_as_uint(f);
    } else if (ALIGNED4 || loff[l] != CLDN_SKIP_STORE_OFFSET) {  // ALIGNED4 implies that no field is skipped
      const float f = nan ? __uint_as_float(0x7FC00000u) : __fmul_rn(__int2float_rn(cur[l]), lmul[l]);
      // point of value k: pbase + (phase + k) / K = pbase + k / K + (k % K + phase >= K)
      const uint32_t p = pbase + k / K + ((l + phase >= static_cast<uint32_t>(K)) ? 1u : 0u);
      uint8_t* dst = out + static_cast<size_t>(p) * step + loff[l];
      if (ALIGNED4) __stcs(reinterpret_cast<unsigned int*>(dst), __float_as_uint(f));  // st.global (the pointer comes from a table)
      else store_u32(dst, __float_as_uint(f));
    }
  }
}

// Dense layouts: the tile's `take` floats (staged at ostage[(done & 3) + i]) are the floats [done, done + take) of the
// chunk's output; staging index and global index agree modulo 4, so whole 16-byte vectors move with LDS.128 / STG.128.
__device__ __forceinline__ void copy_out_dense(const uint32_t* ostage, uint8_t* out, uint32_t done, uint32_t take) {
  const uint32_t a = done & 3u, end = a + take;
  uint32_t* g = reinterpret_cast<uint32_t*>(out) + (done - a);
  for (uint32_t s4 = threadIdx.x * 4u; s4 < end; s4 += kDT * 4u) {
    if (s4 >= a && s4 + 4u <= end) {
      __stcs(reinterpret_cast<uint4*>(g + s4), *reinterpret_cast<const uint4*>(ostage + s4));
    } else {
#pragma unroll
      for (uint32_t j = 0; j < 4u; ++j) {
        if (s4 + j >= a && s4 + j < end) __stcs(g + s4 + j, ostage[s4 + j]);
      }
    }
  }
}


// ---- tile building blocks shared by the tile-parallel and the chunk-sequential kernel -------------------------------
// Loads tile `t` of a chunk body into tile_bytes (with a 16-byte look-behind) and returns this thread's terminator mask.
// tile_bytes[kTLook + i] = stream byte tile_b0 + i; every thread owns kVec adjacent 16-byte vectors.
// Bytes before the stream start read as 0x00 ("boundary": a value can never extend across them, and they are not
// counted as values); bytes past the end read as 0x80 (never terminate anything).
// True when this thread's vector vv of tile t lies completely inside the stream (plain aligned 16-byte load).
__device__ __forceinline__ bool tile_vector_interior(uint32_t size, int64_t tile_b0, int vv) {
  const int64_t b = tile_b0 + (threadIdx.x * kVec + vv) * 16u;
  return b >= 0 && b + 16 <= static_cast<int64_t>(size);
}
__device__ __forceinline__ uint4 tile_vector_fetch(const uint8_t* aligned, uint32_t t, int vv) {
  return __ldcs(reinterpret_cast<const uint4*>(aligned + static_cast<size_t>(t) * kTB + (threadIdx.x * kVec + vv) * 16u));
}

__device__ __forceinline__ uint32_t tile_load_masks(uint8_t* tile_bytes, const uint8_t* aligned, const uint8_t* body, uint32_t size,
                                                    uint32_t t, int64_t tile_b0, bool have_pre = false, uint4 pre = uint4()) {
  uint32_t tmask = 0;  // bit j: byte j of my kVec*16 bytes ends a value (and lies inside the stream)
#pragma unroll
  for (int vv = 0; vv < kVec; ++vv) {
    const uint32_t i = (threadIdx.x * kVec + vv) * 16u;
    const int64_t b = tile_b0 + i;
    uint32_t w0, w1, w2, w3;
    if (b >= 0 && b + 16 <= static_cast<int64_t>(size)) {
      const uint4 q = (have_pre && vv == 0) ? pre : __ldcs(reinterpret_cast<const uint4*>(aligned + static_cast<size_t>(t) * kTB + i));
      w0 = q.x; w1 = q.y; w2 = q.z; w3 = q.w;
    } else {
      w0 = w1 = w2 = w3 = 0;
#pragma unroll
      for (int k = 0; k < 16; ++k) {
        const int64_t bb = b + k;
        uint32_t byte = 0x80u;
        if (bb < 0) byte = 0u;
        else if (bb < static_cast<int64_t>(size)) byte = body[bb];
        const uint32_t v = byte << (8 * (k & 3));
        if ((k >> 2) == 0) w0 |= v; else if ((k >> 2) == 1) w1 |= v; else if ((k >> 2) == 2) w2 |= v; else w3 |= v;
      }
    }
    *reinterpret_cast<uint4*>(tile_bytes + kTLook + i) = make_uint4(w0, w1, w2, w3);
    // terminator flags: bit 7 of every byte inverted; (x * 0x00204081) >> 28 collects bits 7,15,23,31 into a nibble
    const uint32_t x0 = ~w0 & 0x80808080u, x1 = ~w1 & 0x80808080u, x2 = ~w2 & 0x80808080u, x3 = ~w3 & 0x80808080u;
    uint32_t m16 = ((x0 * 0x00204081u) >> 28) | (((x1 * 0x00204081u) >> 28) << 4) | (((x2 * 0x00204081u) >> 28) << 8) |
                   (((x3 * 0x00204081u) >> 28) << 12);
    if (b < 0) {  // bytes before the stream start are not values
      const int64_t nb = -b;
      m16 &= nb >= 16 ? 0u : (0xFFFFu << nb);
    }
    tmask |= m16 << (16 * vv);
  }
  if (threadIdx.x < 4) {  // look-behind
    uint32_t v = 0;  // before the stream start: boundaries
    if (t > 0) {
      v = *reinterpret_cast<const uint32_t*>(aligned + static_cast<size_t>(t) * kTB - 16 + 4 * threadIdx.x);
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        if (tile_b0 - 16 + 4 * static_cast<int64_t>(threadIdx.x) + k < 0) v &= ~(0xFFu << (8 * k));
      }
    }
    reinterpret_cast<uint32_t*>(tile_bytes)[threadIdx.x] = v;
  }
  return tmask;
}

// CTA scan of the terminator counts; then every run t of VT consecutive values gets the tile byte index (biased by
// kTLook) of its first byte in start16[t]: value q starts right behind terminator q-1, which is found in the owner's
// 16-bit mask. No per-value position list is built. Returns the number of values in the tile; ends with a barrier.
// kNthBit[b] holds, 4 bits each, the positions of the set bits of the byte b in increasing order.
__device__ const uint32_t kNthBit[256] = {
    0x00000000u, 0x00000000u, 0x00000001u, 0x00000010u, 0x00000002u, 0x00000020u, 0x00000021u, 0x00000210u,
    0x00000003u, 0x00000030u, 0x00000031u, 0x00000310u, 0x00000032u, 0x00000320u, 0x00000321u, 0x00003210u,
    0x00000004u, 0x00000040u, 0x00000041u, 0x00000410u, 0x00000042u, 0x00000420u, 0x00000421u, 0x00004210u,
    0x00000043u, 0x00000430u, 0x00000431u, 0x00004310u, 0x00000432u, 0x00004320u, 0x00004321u, 0x00043210u,
    0x00000005u, 0x00000050u, 0x00000051u, 0x00000510u, 0x00000052u, 0x00000520u, 0x00000521u, 0x00005210u,
    0x00000053u, 0x00000530u, 0x00000531u, 0x00005310u, 0x00000532u, 0x00005320u, 0x00005321u, 0x00053210u,
    0x00000054u, 0x00000540u, 0x00000541u, 0x00005410u, 0x00000542u, 0x00005420u, 0x00005421u, 0x00054210u,
    0x00000543u, 0x00005430u, 0x00005431u, 0x00054310u, 0x00005432u, 0x00054320u, 0x00054321u, 0x00543210u,
    0x00000006u, 0x00000060u, 0x00000061u, 0x00000610u, 0x00000062u, 0x00000620u, 0x00000621u, 0x00006210u,
    0x00000063u, 0x00000630u, 0x00000631u, 0x00006310u, 0x00000632u, 0x00006320u, 0x00006321u, 0x00063210u,
    0x00000064u, 0x00000640u, 0x00000641u, 0x00006410u, 0x00000642u, 0x00006420u, 0x00006421u, 0x00064210u,
    0x00000643u, 0x00006430u, 0x00006431u, 0x00064310u, 0x00006432u, 0x00064320u, 0x00064321u, 0x00643210u,
    0x00000065u, 0x00000650u, 0x00000651u, 0x00006510u, 0x00000652u, 0x00006520u, 0x00006521u, 0x00065210u,
    0x00000653u, 0x00006530u, 0x00006531u, 0x00065310u, 0x00006532u, 0x00065320u, 0x00065321u, 0x00653210u,
    0x00000654u, 0x00006540u, 0x00006541u, 0x00065410u, 0x00006542u, 0x00065420u, 0x00065421u, 0x00654210u,
    0x00006543u, 0x00065430u, 0x00065431u, 0x00654310u, 0x00065432u, 0x00654320u, 0x00654321u, 0x06543210u,
    0x00000007u, 0x00000070u, 0x00000071u, 0x00000710u, 0x00000072u, 0x00000720u, 0x00000721u, 0x00007210u,
    0x00000073u, 0x00000730u, 0x00000731u, 0x00007310u, 0x00000732u, 0x00007320u, 0x00007321u, 0x00073210u,
    0x00000074u, 0x00000740u, 0x00000741u, 0x00007410u, 0x00000742u, 0x00007420u, 0x00007421u, 0x00074210u,
    0x00000743u, 0x00007430u, 0x00007431u, 0x00074310u, 0x00007432u, 0x00074320u, 0x00074321u, 0x00743210u,
    0x00000075u, 0x00000750u, 0x00000751u, 0x00007510u, 0x00000752u, 0x00007520u, 0x00007521u, 0x00075210u,
    0x00000753u, 0x00007530u, 0x00007531u, 0x00075310u, 0x00007532u, 0x00075320u, 0x00075321u, 0x00753210u,
    0x00000754u, 0x00007540u, 0x00007541u, 0x00075410u, 0x00007542u, 0x00075420u, 0x00075421u, 0x00754210u,
    0x00007543u, 0x00075430u, 0x00075431u, 0x00754310u, 0x00075432u, 0x00754320u, 0x00754321u, 0x07543210u,
    0x00000076u, 0x00000760u, 0x00000761u, 0x00007610u, 0x00000762u, 0x00007620u, 0x00007621u, 0x00076210u,
    0x00000763u, 0x00007630u, 0x00007631u, 0x00076310u, 0x00007632u, 0x00076320u, 0x00076321u, 0x00763210u,
    0x00000764u, 0x00007640u, 0x00007641u, 0x00076410u, 0x00007642u, 0x00076420u, 0x00076421u, 0x00764210u,
    0x00007643u, 0x00076430u, 0x00076431u, 0x00764310u, 0x00076432u, 0x00764320u, 0x00764321u, 0x07643210u,
    0x00000765u, 0x00007650u, 0x00007651u, 0x00076510u, 0x00007652u, 0x00076520u, 0x00076521u, 0x00765210u,
    0x00007653u, 0x00076530u, 0x00076531u, 0x00765310u, 0x00076532u, 0x00765320u, 0x00765321u, 0x07653210u,
    0x00007654u, 0x00076540u, 0x00076541u, 0x00765410u, 0x00076542u, 0x00765420u, 0x00765421u, 0x07654210u,
    0x00076543u, 0x00765430u, 0x00765431u, 0x07654310u, 0x00765432u, 0x07654320u, 0x07654321u, 0x76543210u};
// Position of the n-th (0-based) set bit of a mask of up to 32 bits (n < popc(m)).
__device__ __forceinline__ uint32_t nth_set_bit(uint32_t m, uint32_t n) {
  uint32_t base = 0;
#pragma unroll
  for (int by = 0; by < 2 * kVec - 1; ++by) {
    const uint32_t c = __popc(m & 0xFFu);
    if (n >= c) { n -= c; m >>= 8; base += 8u; }
  }
  return base + ((__ldg(&kNthBit[m & 0xFFu]) >> (4u * n)) & 7u);
}

// CTA exclusive scan of one count per thread with a single barrier: every warp re-scans the warp totals itself.
__device__ __forceinline__ uint32_t tile_count_scan(uint32_t v, uint32_t* scratch, uint32_t* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  constexpr int NW = kDT / 32;
  uint32_t inc = v;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const uint32_t t = __shfl_up_sync(0xffffffffu, inc, d);
    if (lane >= d) inc += t;
  }
  if (lane == 31) scratch[warp] = inc;
  __syncthreads();
  uint32_t w = lane < NW ? scratch[lane] : 0u;
#pragma unroll
  for (int d = 1; d < NW; d <<= 1) {
    const uint32_t t = __shfl_up_sync(0xffffffffu, w, d);
    if (lane >= d) w += t;
  }
  *total = __shfl_sync(0xffffffffu, w, NW - 1);
  const uint32_t before = __shfl_sync(0xffffffffu, w, warp > 0 ? warp - 1 : 0);
  return (warp > 0 ? before : 0u) + inc - v;
}

template <int K>
__device__ __forceinline__ uint32_t tile_rank_starts(uint32_t tmask, const uint8_t* tile_bytes, uint16_t* start16, uint32_t* scan,
                                                     uint32_t* vt_out) {
  uint32_t tile_cnt;
  const uint32_t c = __popc(tmask);
  const uint32_t rank = tile_count_scan(c, scan, &tile_cnt);
  const uint32_t VT = max(1u, (tile_cnt + kDT - 1) / kDT);  // values per thread (runs need not start at a field 0)
  *vt_out = VT;
  const uint32_t base = kTLook + threadIdx.x * kVec * 16u;
  if (c) {
    if (rank == 0) {
      // first byte of value 0: walk back from its terminator over continuation bytes (at most 10; stops at a boundary)
      const int e = static_cast<int>(base) + __ffs(tmask) - 1;
      int st = e;
      while (st > 0 && e - st < 11 && (tile_bytes[st - 1] & 0x80u)) --st;
      start16[0] = static_cast<uint16_t>(st);
    }
    // run starts among my terminators: value q starts right behind terminator q - 1 = my (q - 1 - rank)-th one
    for (uint32_t q = (rank / VT + 1u) * VT; q <= rank + c && q < tile_cnt; q += VT) {
      start16[q / VT] = static_cast<uint16_t>(base + nth_set_bit(tmask, q - 1u - rank) + 1u);
    }
  }
  __syncthreads();
  return tile_cnt;
}

// Values of 5..10 bytes starting at tile byte `ptr`: returns (bad << 40) | (len << 32) | uint32(delta).
__device__ __noinline__ unsigned long long decode_wide_at(const uint8_t* tile_bytes, uint32_t ptr) {
  unsigned long long u = 0;
  uint32_t len = 0, bad = 0;
  while (true) {
    if (len >= 10u) { bad = DEV_ERR_VARINT_OVERFLOW; break; }
    const uint32_t byte = tile_bytes[ptr + len];
    const unsigned long long payload = byte & 0x7Fu;
    if (len == 9u && payload > 1) bad = DEV_ERR_VARINT_OVERFLOW;  // encoding_utils.hpp:127-129
    u |= payload << (7 * len);
    ++len;
    if (!(byte & 0x80u)) break;
  }
  if (!bad && u == 0) bad = DEV_ERR_NAN_MARKER;
  const uint32_t delta = bad ? 0u : static_cast<uint32_t>(static_cast<int32_t>(unzigzag(u - 1ull)));
  return (static_cast<unsigned long long>(bad) << 40) | (static_cast<unsigned long long>(len) << 32) | delta;
}

// Streams this thread's run of n_run consecutive values (starting at tile byte `ptr`) into registers: every value is
// cut out of a 4-byte window read at the current byte position; the window's terminator flags give its length.
template <int VTMAX>
__device__ __forceinline__ void tile_decode_run(const uint8_t* tile_bytes, uint32_t ptr, uint32_t n_run, int32_t (&d)[VTMAX],
                                                unsigned long long& nanm, uint32_t& badcode, uint32_t& badk) {
  nanm = 0;
  badcode = 0;
  badk = 0xFFFFFFFFu;
#pragma unroll
  for (int k = 0; k < VTMAX; ++k) {
    if (k >= static_cast<int>(n_run)) break;
    const uint32_t* wp = reinterpret_cast<const uint32_t*>(tile_bytes + (ptr & ~3u));
    const uint32_t lo = __funnelshift_r(wp[0], wp[1], 8u * (ptr & 3u));  // the 4 bytes at ptr
    const uint32_t m = ~lo & 0x80808080u;                                 // terminators among them
    int32_t delta = 0;
    uint32_t len;
    if (m) {
      const uint32_t lowbit = m & (0u - m);                               // flag bit of the value's last byte
      uint32_t hb;
      asm("bfind.u32 %0, %1;" : "=r"(hb) : "r"(lowbit));                  // 7, 15, 23 or 31
      len = (hb >> 3) + 1u;
      uint32_t x = lo & (lowbit * 2u - 1u) & 0x7F7F7F7Fu;                 // the value's bytes without their flags
      x = x - ((x & 0x7F007F00u) >> 1);                                   // 7-bit groups -> 14-bit groups
      x = (x & 0x3FFFu) | ((x >> 2) & 0x0FFFC000u);                       // -> 28-bit uval = zigzag + 1
      if (x == 0u) {  // uval 0: the NaN marker if it is the single byte 0x00, otherwise "unexpected NaN marker"
        if (len == 1u) nanm |= 1ull << k;
        else if (badk == 0xFFFFFFFFu) { badcode = DEV_ERR_NAN_MARKER; badk = k; }
      } else {
        // un-zigzag of x - 1: odd x -> x >> 1, even x -> -(x >> 1) = (x * +-1) >> 1 (the multiplies run on the FMA pipe)
        const int32_t sgn = static_cast<int32_t>((x & 1u) * 2u) - 1;
        delta = (static_cast<int32_t>(x) * sgn) >> 1;
      }
    } else {
      const unsigned long long r = decode_wide_at(tile_bytes, ptr);
      const uint32_t bad = static_cast<uint32_t>(r >> 40);
      len = static_cast<uint32_t>(r >> 32) & 0xFFu;
      delta = static_cast<int32_t>(static_cast<uint32_t>(r));
      if (bad && badk == 0xFFFFFFFFu) { badcode = bad; badk = k; }
    }
    d[k] = delta;
    ptr += len;
  }
}

// Branch-free variant for the common case (every value at most 4 bytes, no malformed NaN marker): returns false if
// the run has to be decoded again by tile_decode_run (d / nanm are then meaningless). With FUSED the per-field sums of
// the run (local slot numbering, no NaN reset) are accumulated on the way.
template <int K, int VTMAX, bool FUSED>
__device__ __forceinline__ bool tile_decode_run_fast(const uint8_t* tile_bytes, uint32_t ptr, uint32_t n_run, int32_t (&d)[VTMAX],
                                                     unsigned long long& nanm, int32_t (&sum)[K]) {
  uint32_t nan_lo = 0, nan_hi = 0, mmin = 0xFFFFFFFFu, badacc = 0;
#pragma unroll
  for (int j = 0; j < K; ++j) sum[j] = 0;
#pragma unroll
  for (int k = 0; k < VTMAX; ++k) {
    if (k >= static_cast<int>(n_run)) break;
    const uint32_t* wp = reinterpret_cast<const uint32_t*>(tile_bytes + (ptr & ~3u));
    const uint32_t lo = __funnelshift_r(wp[0], wp[1], 8u * (ptr & 3u));  // the 4 bytes at ptr
    const uint32_t m = ~lo & 0x80808080u;                                 // terminators among them
    mmin = min(mmin, m);                                                  // 0: a value longer than 4 bytes -> slow path
    const uint32_t lowbit = m & (0u - m);                                 // flag bit of the value's last byte
    uint32_t hb;
    asm("bfind.u32 %0, %1;" : "=r"(hb) : "r"(lowbit));                    // 7, 15, 23 or 31 (all ones if m == 0)
    const uint32_t lenm1 = (hb >> 3) & 3u;
    uint32_t x = lo & (lowbit * 2u - 1u) & 0x7F7F7F7Fu;                   // the value's bytes without their flags
    x = x - ((x & 0x7F007F00u) >> 1);                                     // 7-bit groups -> 14-bit groups
    x = (x & 0x3FFFu) | ((x >> 2) & 0x0FFFC000u);                         // -> 28-bit uval = zigzag + 1
    if (x == 0u) {  // NaN marker (must be the single byte 0x00; anything longer is malformed -> slow path reports it)
      if (k < 32) nan_lo |= 1u << (k & 31); else nan_hi |= 1u << (k & 31);
      badacc |= lenm1;
    }
    // un-zigzag of x - 1: odd x -> x >> 1, even x -> -(x >> 1) = (x * +-1) >> 1; x == 0 gives 0
    const int32_t sgn = static_cast<int32_t>((x & 1u) * 2u) - 1;
    const int32_t delta = (static_cast<int32_t>(x) * sgn) >> 1;
    d[k] = delta;
    if (FUSED) sum[k % K] = wadd32(sum[k % K], delta);
    ptr += lenm1 + 1u;
  }
  nanm = (static_cast<unsigned long long>(nan_hi) << 32) | nan_lo;
  return mmin != 0u && badacc == 0u;
}

// Tile byte index (biased) one past value `idx` of the run that starts at `ptr` (single thread; used for stream_end).
__device__ __forceinline__ uint32_t run_end_after(const uint8_t* tile_bytes, uint32_t ptr, uint32_t idx) {
  for (uint32_t k = 0; k <= idx; ++k) {
    uint32_t n = 0;
    while (n < 10u && (tile_bytes[ptr + n] & 0x80u)) ++n;
    ptr += n + 1u;
  }
  return ptr;
}

// CTA-wide exclusive segmented scan of one SegK per thread (two barriers); *total = combination of all threads.
template <int K>
__device__ __forceinline__ SegK<K> cta_seg_exclusive(const SegK<K>& mine, TileShared& sh, SegK<K>* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  SegK<K> inc = mine;
  if (!__any_sync(0xffffffffu, mine.rst != 0u)) {
    // no NaN reset in this warp (the common case): plain wrapping prefix sums
#pragma unroll
    for (int dd = 1; dd < 32; dd <<= 1) {
#pragma unroll
      for (int j = 0; j < K; ++j) {
        const int32_t up = __shfl_up_sync(0xffffffffu, inc.sum[j], dd);
        if (lane >= dd) inc.sum[j] = wadd32(inc.sum[j], up);
      }
    }
  } else {
#pragma unroll
    for (int dd = 1; dd < 32; dd <<= 1) {
      const SegK<K> up = seg_shfl_up<K>(inc, dd);
      if (lane >= dd) inc = seg_then<K>(up, inc);
    }
  }
  if (lane == 31) {
#pragma unroll
    for (int j = 0; j < K; ++j) sh.w_sum[warp][j] = inc.sum[j];
    sh.w_rst[warp] = inc.rst;
  }
  __syncthreads();
  // every warp scans the kDT/32 warp totals with its first lanes (3 shuffle steps) instead of looping over them
  constexpr int NW = kDT / 32;
  SegK<K> wt = seg_identity<K>();
  if (lane < NW) {
#pragma unroll
    for (int j = 0; j < K; ++j) wt.sum[j] = sh.w_sum[lane][j];
    wt.rst = sh.w_rst[lane];
  }
  if (!__any_sync(0xffffffffu, wt.rst != 0u)) {
#pragma unroll
    for (int dd = 1; dd < NW; dd <<= 1) {
#pragma unroll
      for (int j = 0; j < K; ++j) {
        const int32_t up = __shfl_up_sync(0xffffffffu, wt.sum[j], dd);
        if (lane >= dd) wt.sum[j] = wadd32(wt.sum[j], up);
      }
    }
  } else {
#pragma unroll
    for (int dd = 1; dd < NW; dd <<= 1) {
      const SegK<K> up = seg_shfl_up<K>(wt, dd);
      if (lane >= dd) wt = seg_then<K>(up, wt);
    }
  }
  const SegK<K> tot = seg_shfl<K>(wt, NW - 1);
  SegK<K> prefix = seg_shfl<K>(wt, warp > 0 ? warp - 1 : 0);
  if (warp == 0) prefix = seg_identity<K>();
  *total = tot;
  SegK<K> ex = prefix;
  const SegK<K> prev_lane = seg_shfl_up<K>(inc, 1);
  if (lane > 0) ex = seg_then<K>(prefix, prev_lane);
  return ex;
}

// ---- tile-parallel kernel: one CTA per 8 KB tile, two decoupled look-backs (small batches / single frames) ----------
template <int K>
__global__ void __launch_bounds__(kDT, kSeqMinBlocks) decode_tiles_kernel(const DecLaunch L, float m0, float m1, float m2, float m3,
                                                                   uint32_t o0, uint32_t o1, uint32_t o2, uint32_t o3) {
  extern __shared__ __align__(16) uint8_t dyn_smem[];
  __shared__ TileShared sh;
  uint8_t* tile_bytes = dyn_smem;                                               // kTLook + kTB + 16
  uint16_t* start16 = reinterpret_cast<uint16_t*>(dyn_smem + kTLook + kTB + 16);  // kDT entries: first byte of every run
  uint32_t* ostage = reinterpret_cast<uint32_t*>(dyn_smem + kOStageOffset);
  constexpr int VTMAX = ((kTB / kDT) + K - 1) / K * K;                     // values per thread if every value is one byte

  const uint32_t gt = blockIdx.x;
  if (gt >= L.chunk_tile_begin[L.n_chunks_total]) return;
  const uint32_t gc = L.tile_chunk[gt];
  const DecFrame F = L.frames[L.chunk_frame[gc]];
  const uint32_t chunk = gc - F.chunk_begin;
  const uint32_t n_points = min(kChunkPoints, F.n_points - chunk * kChunkPoints);
  const uint32_t V = n_points * K;
  const uint32_t first_tile = L.chunk_tile_begin[gc];
  const uint32_t t = gt - first_tile;
  const uint8_t* body = F.payload + L.chunk_offsets[gc];
  const uint32_t size = L.chunk_sizes[gc];
  const uint32_t mis = static_cast<uint32_t>(reinterpret_cast<uintptr_t>(body) & 15u);
  const uint8_t* aligned = body - mis;
  const int64_t tile_b0 = static_cast<int64_t>(t) * kTB - mis;  // stream offset of tile byte 0
  const uint32_t step = L.plan->point_step;
  uint8_t* out = F.out + static_cast<size_t>(chunk) * kChunkPoints * step;
  const bool aligned4 = (((reinterpret_cast<uintptr_t>(out) | step | o0 | o1 | o2 | (K == 4 ? o3 : 0u)) & 3u) == 0u) &&
      o0 != CLDN_SKIP_STORE_OFFSET && o1 != CLDN_SKIP_STORE_OFFSET && o2 != CLDN_SKIP_STORE_OFFSET && (K < 4 || o3 != CLDN_SKIP_STORE_OFFSET);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint64_t* recs = reinterpret_cast<uint64_t*>(L.tsums);

  const uint32_t tmask = tile_load_masks(tile_bytes, aligned, body, size, t, tile_b0);
  uint32_t VT;
  const uint32_t tile_cnt = tile_rank_starts<K>(tmask, tile_bytes, start16, sh.scan, &VT);
  // ---- look-back 1 (warp 0): values before this tile; overlapped with the value decoding of the other warps ----
  if (warp == 0) {
    const uint64_t ex = tile_lookback(L.tstatus, first_tile, gt, L.epoch, tile_cnt);
    if (lane == 0) sh.done = static_cast<uint32_t>(ex > 0xFFFFFFFFull ? 0xFFFFFFFFull : ex);
  }
  // ---- every thread decodes a run of VT consecutive values (VT a multiple of K) into registers ----
  const uint32_t v0 = threadIdx.x * VT;
  const uint32_t n_run = v0 < tile_cnt ? min(VT, tile_cnt - v0) : 0u;
  int32_t d[VTMAX];
  unsigned long long nanm;
  uint32_t badcode, badk;
  tile_decode_run<VTMAX>(tile_bytes, n_run ? start16[threadIdx.x] : 0u, n_run, d, nanm, badcode, badk);
  __syncthreads();
  const uint32_t done = sh.done;
  // Tiles past the end of the regular stream (V5 sections / trailing bytes) are never waited on by anyone.
  if (done >= V) return;
  const uint32_t take = min(tile_cnt, V - done);
  // "ran out of bytes": the chunk's last tile still misses values (v4_codec.cpp:102-104)
  if (t + 1 == L.chunk_tiles[gc] && done + tile_cnt < V && threadIdx.x == 0) report_frame_error(L, L.chunk_frame[gc], DEV_ERR_TRUNCATED);
  if (take > 0 && done + take == V && threadIdx.x == (take - 1) / VT) {  // first byte after the regular stream
    L.stream_end[gc] = static_cast<uint32_t>(tile_b0 + run_end_after(tile_bytes, start16[threadIdx.x], (take - 1) - v0) - kTLook);
  }
  const uint32_t n_mine = v0 < take ? min(VT, take - v0) : 0u;  // my values that belong to the regular stream
  if (badk < n_mine) report_frame_error(L, L.chunk_frame[gc], badcode);            // bytes past the stream may be anything: only real values count

  // ---- per-field segmented sums of my run; the field of value k is (done + v0 + k) % K = (done % K + k) % K ----
  const uint32_t phase = (done + v0) % K;
  const SegK<K> mine = seg_to_global<K>(run_reduce_local<K, VTMAX>(d, nanm, n_mine), phase);
  SegK<K> total;
  const SegK<K> ex = cta_seg_exclusive<K>(mine, sh, &total);
  // ---- look-back 2: per-field value at the tile start ----
  if (warp == 0) {
    SegK<K> carry_in = seg_identity<K>();
    if (t == 0) {
      if (lane == 0) publish_words<K>(recs + static_cast<size_t>(gt) * 4, total, L.epoch, 2u);
    } else {
      if (lane == 0) publish_words<K>(recs + static_cast<size_t>(gt) * 4, total, L.epoch, 1u);
      carry_in = sums_lookback<K>(recs, first_tile, gt, L.epoch);
      if (lane == 0) publish_words<K>(recs + static_cast<size_t>(gt) * 4, seg_then<K>(carry_in, total), L.epoch, 2u);
    }
    if (lane == 0) {
#pragma unroll
      for (int j = 0; j < K; ++j) sh.carry[j] = carry_in.sum[j];  // sum since the last reset == absolute value (0 at chunk start)
    }
  }
  __syncthreads();
  const float mul[4] = {m0, m1, m2, m3};
  const uint32_t off[4] = {o0, o1, o2, o3};
  int32_t cur[K];
#pragma unroll
  for (int j = 0; j < K; ++j) cur[j] = ((ex.rst >> j) & 1u) ? ex.sum[j] : wadd32(sh.carry[j], ex.sum[j]);
  const uint32_t pbase = (done + v0) / K;  // point of my first value
  const bool dense = aligned4 && step == 4u * K && o0 == 0u && o1 == 4u && o2 == 8u && (K < 4 || o3 == 12u) &&
      (reinterpret_cast<uintptr_t>(out) & 15u) == 0u;
  if (dense) {
    run_emit_local<K, VTMAX, 2>(d, nanm, n_mine, cur, phase, out, pbase, step, mul, off, ostage + (done & 3u) + v0);
    __syncthreads();
    copy_out_dense(ostage, out, done, take);
  } else if (aligned4) run_emit_local<K, VTMAX, 1>(d, nanm, n_mine, cur, phase, out, pbase, step, mul, off);
  else run_emit_local<K, VTMAX, 0>(d, nanm, n_mine, cur, phase, out, pbase, step, mul, off);
}

// One thread follows the chunk prefixes of frame f (same checks and error codes as walk_chunks_kernel) and publishes
// each chunk twice: plain tables for the kernels that run afterwards (V5 sections), and two self-validating words
// ([tag:24][value:40]) that the decoding CTAs of this launch poll -- every word carries its own tag, so no fence orders
// them. A chunk that cannot be located is published with size 0 (the decoder then reports the truncation).
__device__ __forceinline__ void walk_frame_publish(const DecLaunch& L, uint32_t f) {
  const DecFrame F = L.frames[f];
  const unsigned long long tag = static_cast<unsigned long long>(L.desc_tag) << 40;
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
    const uint32_t gc = F.chunk_begin + c;
    L.chunk_offsets[gc] = body;
    L.chunk_sizes[gc] = size;
    st_relaxed_u64(L.chunk_desc + 2ull * gc, tag | (body & 0xFFFFFFFFFFull));
    st_relaxed_u64(L.chunk_desc + 2ull * gc + 1, tag | size);
  }
  if (pos < F.payload_bytes) report_frame_error(L, f, DEV_ERR_CHUNK_COUNT);  // "more chunks than declared points"
}

// ---- chunk-sequential kernel: a persistent CTA walks the tiles of one chunk after the other (large batches) ---------
// No inter-CTA communication at all: the value count and the per-field running values are carried in shared memory
// from tile to tile; chunks are claimed from an atomic counter so that the SMs stay balanced.
template <int K>
__global__ void __launch_bounds__(kDT, kSeqMinBlocks) decode_chunks_seq_kernel(const DecLaunch L, float m0, float m1, float m2, float m3,
                                                                        uint32_t o0, uint32_t o1, uint32_t o2, uint32_t o3) {
  extern __shared__ __align__(16) uint8_t dyn_smem[];
  __shared__ TileShared sh;
  __shared__ uint32_t s_chunk;
  uint8_t* tile_bytes = dyn_smem;
  uint16_t* start16 = reinterpret_cast<uint16_t*>(dyn_smem + kTLook + kTB + 16);
  uint32_t* ostage = reinterpret_cast<uint32_t*>(dyn_smem + kOStageOffset);
  constexpr int VTMAX = ((kTB / kDT) + K - 1) / K * K;
  __shared__ unsigned long long s_desc[2];
  const float mul[4] = {m0, m1, m2, m3};
  const uint32_t off[4] = {o0, o1, o2, o3};
  const uint32_t step = L.plan->point_step;

  // Whichever CTA draws ticket 0 -- by construction one that is running, whatever the block scheduler does -- follows
  // the u32 chunk prefixes of every frame (cloudini.cpp:645-664, the same checks as walk_chunks_kernel) and publishes
  // every chunk as soon as it is known; the other CTAs start decoding at once and only wait for the descriptor of the
  // chunk they claimed. (redo mode: the fast kernel of the same launch has published every descriptor already)
  if (!L.redo_mode) {
    if (threadIdx.x == 0) s_chunk = atomicAdd(L.chunk_counter + 2, 1u);
    __syncthreads();
    if (s_chunk == 0u) {
      for (uint32_t f = threadIdx.x; f < L.n_frames; f += kDT) walk_frame_publish(L, f);
    }
    __syncthreads();
  }

  while (true) {
    if (threadIdx.x == 0) {
      uint32_t i, gc_;
      if (L.redo_mode) {  // only the chunks the fast kernel could not prove to be "plain"
        i = atomicAdd(L.chunk_counter + 1, 1u);
        gc_ = i < L.chunk_counter[3] ? L.redo_list[i] : 0xFFFFFFFFu;
        i = gc_;
      } else {
        i = atomicAdd(L.chunk_counter, 1u);
        gc_ = i;
      }
      if (i < L.n_chunks_total) {
        // equal frames: claim chunk-index-major (all chunk 0s first), so early claims never wait long for the walk
        if (L.uniform_chunks && !L.redo_mode) gc_ = (i % L.n_frames) * L.uniform_chunks + i / L.n_frames;
        if (!L.empty_slots || !chunk_slot_empty(L.frames[dec_frame_of(L, gc_)], gc_)) {  // nobody publishes an empty slot
          unsigned long long w0, w1;
          do {
            w0 = ld_relaxed_u64(L.chunk_desc + 2ull * gc_);
            w1 = ld_relaxed_u64(L.chunk_desc + 2ull * gc_ + 1);
          } while (static_cast<uint32_t>(w0 >> 40) != L.desc_tag || static_cast<uint32_t>(w1 >> 40) != L.desc_tag);
          s_desc[0] = w0 & 0xFFFFFFFFFFull;
          s_desc[1] = w1 & 0xFFFFFFFFull;
          L.stream_end[gc_] = 0xFFFFFFFFu;  // set by the tile that decodes the chunk's last regular value
        }
      }
      s_chunk = gc_;
    }
    __syncthreads();
    const uint32_t gc = s_chunk;
    if (gc >= L.n_chunks_total) return;
    const uint32_t fidx = dec_frame_of(L, gc);
    const DecFrame F = L.frames[fidx];
    if (chunk_slot_empty(F, gc)) {
      __syncthreads();  // everybody has read s_chunk before thread 0 may claim the next chunk
      continue;
    }
    const uint32_t chunk = gc - F.chunk_begin;
    const uint32_t n_points = min(kChunkPoints, F.n_points - chunk * kChunkPoints);
    const uint32_t V = n_points * K;
    const uint8_t* body = F.payload + s_desc[0];
    const uint32_t size = static_cast<uint32_t>(s_desc[1]);
    const uint32_t mis = static_cast<uint32_t>(reinterpret_cast<uintptr_t>(body) & 15u);
    const uint8_t* aligned = body - mis;
    const uint32_t n_tiles = size ? (size + mis + kTB - 1) / kTB : 0u;
    __syncthreads();  // everybody has read s_chunk / s_desc before thread 0 may claim the next chunk
    uint8_t* out = F.out + static_cast<size_t>(chunk) * kChunkPoints * step;
    const bool aligned4 = (((reinterpret_cast<uintptr_t>(out) | step | o0 | o1 | o2 | (K == 4 ? o3 : 0u)) & 3u) == 0u) &&
      o0 != CLDN_SKIP_STORE_OFFSET && o1 != CLDN_SKIP_STORE_OFFSET && o2 != CLDN_SKIP_STORE_OFFSET && (K < 4 || o3 != CLDN_SKIP_STORE_OFFSET);
    const bool dense = aligned4 && step == 4u * K && o0 == 0u && o1 == 4u && o2 == 8u && (K < 4 || o3 == 12u) &&
        (reinterpret_cast<uintptr_t>(out) & 15u) == 0u;
    uint32_t done = 0;
    int32_t carry[K];
#pragma unroll
    for (int j = 0; j < K; ++j) carry[j] = 0;
    // software prefetch: the next tile's (first) vector is requested before the current tile is processed
    bool have_pre = false;
    uint4 pre = make_uint4(0, 0, 0, 0);
    for (uint32_t t = 0; t < n_tiles && done < V; ++t) {
      const int64_t tile_b0 = static_cast<int64_t>(t) * kTB - mis;
      const uint32_t tmask = tile_load_masks(tile_bytes, aligned, body, size, t, tile_b0, have_pre, pre);
      have_pre = (t + 1 < n_tiles) && tile_vector_interior(size, tile_b0 + kTB, 0);
      if (have_pre) pre = tile_vector_fetch(aligned, t + 1, 0);
      uint32_t VT;
      const uint32_t tile_cnt = tile_rank_starts<K>(tmask, tile_bytes, start16, sh.scan, &VT);
      const uint32_t v0 = threadIdx.x * VT;
      const uint32_t take = min(tile_cnt, V - done);
      const uint32_t n_mine = v0 < take ? min(VT, take - v0) : 0u;  // my values that belong to the regular stream
      const uint32_t run_ptr = n_mine ? start16[threadIdx.x] : 0u;
      int32_t d[VTMAX];
      unsigned long long nanm;
      SegK<K> local;  // per-field sums of my run in local slot numbering
      local.rst = 0;
      const bool fast_ok = tile_decode_run_fast<K, VTMAX, true>(tile_bytes, run_ptr, n_mine, d, nanm, local.sum);
      if (!fast_ok) {  // a value longer than 4 bytes or a malformed marker: the careful reader decides
        uint32_t badcode, badk;
        tile_decode_run<VTMAX>(tile_bytes, run_ptr, n_mine, d, nanm, badcode, badk);
        if (badk < n_mine) report_frame_error(L, fidx, badcode);
      }
      if (!fast_ok || nanm != 0ull) local = run_reduce_local<K, VTMAX>(d, nanm, n_mine);  // sums with NaN resets
      if (take > 0 && done + take == V && threadIdx.x == (take - 1) / VT) {
        L.stream_end[gc] = static_cast<uint32_t>(tile_b0 + run_end_after(tile_bytes, start16[threadIdx.x], (take - 1) - v0) - kTLook);
      }
      const uint32_t phase = (done + v0) % K;
      const SegK<K> mine = seg_to_global<K>(local, phase);
      SegK<K> total;
      const SegK<K> ex = cta_seg_exclusive<K>(mine, sh, &total);
      int32_t cur[K];
#pragma unroll
      for (int j = 0; j < K; ++j) cur[j] = ((ex.rst >> j) & 1u) ? ex.sum[j] : wadd32(carry[j], ex.sum[j]);
      if (dense) run_emit_local<K, VTMAX, 2>(d, nanm, n_mine, cur, phase, out, (done + v0) / K, step, mul, off, ostage + (done & 3u) + v0);
      else if (aligned4) run_emit_local<K, VTMAX, 1>(d, nanm, n_mine, cur, phase, out, (done + v0) / K, step, mul, off);
      else run_emit_local<K, VTMAX, 0>(d, nanm, n_mine, cur, phase, out, (done + v0) / K, step, mul, off);
#pragma unroll
      for (int j = 0; j < K; ++j) carry[j] = ((total.rst >> j) & 1u) ? total.sum[j] : wadd32(carry[j], total.sum[j]);
      __syncthreads();  // tile_bytes / start16 / sh are reused by the next tile; ostage is complete
      // the staged floats leave while the next tile is loaded and ranked (ostage is not written again before the
      // barriers of the next tile's scans)
      if (dense) copy_out_dense(ostage, out, done, take);
      done += take;
    }
    if (done < V && threadIdx.x == 0) report_frame_error(L, fidx, DEV_ERR_TRUNCATED);  // v4_codec.cpp:102-104
  }
}

}  // namespace cldn
#include "cldn_decode_fast.cuh"
namespace cldn {

// ------------------------------------------------------------------------------------------------------------------
size_t decode_tiles_smem_bytes() { return static_cast<size_t>(kOStageOffset) + kOStageBytes; }
uint32_t decode_tile_bytes() { return kTB; }

template <int K>
static int launch_floatn_decode(const RegOp& op, const DecLaunch& L, bool sequential, int sm_count, cudaStream_t stream) {
  const size_t smem = decode_tiles_smem_bytes();
  const float m3 = K == 4 ? op.dec_mul_f[3] : 0.f;
  const uint32_t o3 = K == 4 ? op.offset[3] : 0u;
  if (sequential) {
    auto k = decode_chunks_seq_kernel<K>;
    if (raise_smem_limit(k, smem) != cudaSuccess) return -1;
    int per_sm = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k, kDT, smem) != cudaSuccess || per_sm < 1) per_sm = 1;
    const uint32_t grid = min(L.n_chunks_total, static_cast<uint32_t>(per_sm * sm_count));
    if (!L.redo_mode) cudaMemsetAsync(L.chunk_counter, 0, 4 * sizeof(uint32_t), stream);
    k<<<grid, kDT, smem, stream>>>(L, op.dec_mul_f[0], op.dec_mul_f[1], op.dec_mul_f[2], m3, op.offset[0], op.offset[1], op.offset[2], o3);
  } else {
    auto k = decode_tiles_kernel<K>;
    if (raise_smem_limit(k, smem) != cudaSuccess) return -1;
    k<<<L.tile_grid, kDT, smem, stream>>>(L, op.dec_mul_f[0], op.dec_mul_f[1], op.dec_mul_f[2], m3, op.offset[0], op.offset[1], op.offset[2], o3);
  }
  return 1;
}

static int device_sm_count() {
  static const int sm_count = [] {  // (a function-local static: handles on several threads may ask first at once)
    int dev = 0, n = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    return n > 0 ? n : 132;  // H100 SXM
  }();
  return sm_count;
}

// Large batches: one persistent CTA per chunk (no look-back latency); small ones: one CTA per tile (parallel inside a chunk).
bool decode_tiles_sequential(uint32_t n_chunks_total) {
  const int sm_count = device_sm_count();
  const char* mode = getenv("CLDN_B200_DECODE_MODE");  // "seq" | "tile" (development override)
  bool sequential = n_chunks_total >= static_cast<uint32_t>(sm_count + sm_count / 8);  // measured crossover: ~1.1 chunks per SM
  if (mode && mode[0] == 's') sequential = true;
  if (mode && mode[0] == 't') sequential = false;
  return sequential;
}

// CLDN_B200_DECODE_FAST=0 keeps the careful chunk-sequential kernel alone (A/B measurements, bisecting).
bool decode_fast_enabled() {
  const char* e = getenv("CLDN_B200_DECODE_FAST");
  return !(e && e[0] == '0');
}

int launch_decode_tiles(const Plan& plan, const DecLaunch& L, cudaStream_t stream) {
  const RegOp& op = plan.ops[0];
  const int sm_count = device_sm_count();
  const bool sequential = decode_tiles_sequential(L.n_chunks_total);
  if (sequential && !L.chunk_desc) return -1;
  int launches = 0;
  if (!(sequential && L.chunk_desc)) {  // the sequential kernel derives these per chunk itself
    count_tiles_kernel<<<(L.n_chunks_total + 127) / 128, 128, 0, stream>>>(L);
    ++launches;
  }
  if (!sequential) {
    scan_tiles_kernel<<<1, kThreads, 0, stream>>>(L);
    ++launches;
  }
  if (sequential && decode_fast_enabled() && L.redo_list) {
    // fast kernel first; whatever it could not prove plain (NaN markers, 5+ byte varints, damage) goes to the careful
    // kernel, which is launched on a small grid and returns at once when the redo list is empty
    if (!decode_side_active(plan, L)) cudaMemsetAsync(L.chunk_counter, 0, 4 * sizeof(uint32_t), stream);  // (side mode: zeroed before its pre-pass)
    if (launch_decode_fast(plan, L, sm_count, stream) < 0) return -1;
    DecLaunch R = L;
    R.redo_mode = 1;
    const int n = op.lanes == 4 ? launch_floatn_decode<4>(op, R, true, sm_count, stream)
                                : launch_floatn_decode<3>(op, R, true, sm_count, stream);
    return n < 0 ? -1 : launches + 1 + n;
  }
  const int n = op.lanes == 4 ? launch_floatn_decode<4>(op, L, sequential, sm_count, stream)
                              : launch_floatn_decode<3>(op, L, sequential, sm_count, stream);
  return n < 0 ? -1 : launches + n;
}

}  // namespace cldn
