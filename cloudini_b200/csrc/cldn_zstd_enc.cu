// Stage 2 on the device, ZSTD compression (RFC 8878), for encoders that asked for it
// (cldn_b200_encoder_set_stage2_on_device). Every chunk's stage-1 bytes become one ZSTD frame that libzstd, the
// reference and cldn_zstd.cu decode to the same bytes; the frames are not ZSTD_compress's bytes.
//
// Only the entropy stage of ZSTD is used: a block is its literals, Huffman-coded, and zero sequences. There is no match
// search, so blocks are independent and the work is data-parallel over them. On lidar stage-1 bytes (varints, deltas)
// matches are rare, and an order-0 Huffman code per block comes within a few per cent of ZSTD_compress(level 1)
// (DESIGN.md §7 has the measured ratios).
//
//  grid     one CTA per block of kZeBlock stage-1 bytes, over the blocks of every chunk of every frame of the batch. Chunk
//           gc owns pieces block_begin[gc] .. block_begin[gc + 1] - 1 (room for its worst-case size, filled on the host:
//           the real sizes are only known on the device); a CTA whose block lies past its chunk's end writes an empty
//           piece and exits (about 2-3x the real blocks on XYZI data). Each CTA finds its chunk by walking the frame's
//           [u32 size] chain from the start (lz_find_chunk, as the LZ4 compressor does): quadratic in the chunks of a
//           frame, a few dozen hops for today's frames (31 for 1M points).
//  block    1. byte histogram (per-warp sub-histograms in shared memory);
//           2. code lengths <= 11 bits: Huffman tree of the (count, symbol)-sorted symbols, then the lengths are limited and
//              made a complete code by moving leaves between lengths (thread 0; ties go by symbol value, so the result
//              never depends on the order of atomics);
//           3. tree description: 4-bit weights when the last symbol is < 128, else FSE-compressed weights (accuracy log 6,
//              two interleaved states);
//           4. four Huffman streams: every thread encodes a contiguous run of one stream at a bit offset from a scan of
//              the runs' code lengths, into shared memory; a backward reader meets the symbols in forward order;
//           5. the piece: [frame header, block 0 only][block header][literals header][tree][jump table][streams][0].
//           An RLE block when every byte is equal; a raw block when fewer than kZeMinHuff bytes remain, when the weights do
//           not fit their form, or when the compressed block is not smaller.
//  frame    magic, single-segment frame header with Frame_Content_Size (the layout ZSTD_compress writes for a chunk), the
//           blocks, Last_Block on the last one, no checksum. Its size is at most ZSTD_COMPRESSBOUND(chunk):
//             frame <= 4 (magic) + 1 (FHD) + 4 (FCS, chunks < 4 GB) + sum over blocks of (3 + block bytes)
//                    = n + 9 + 3 * ceil(n / kZeBlock)   for a chunk of n bytes (an empty chunk: one empty raw block),
//             ZSTD_COMPRESSBOUND(n) = n + n / 256 + (n < 128 KB ? (128 KB - n) / 2048 : 0).
//           With kZeBlock = 32 KB: below 3146 bytes the frame is one block (12 bytes over n) and (128 KB - n) / 2048 >= 62;
//           from there on 3 * ceil(n / 32 KB) + 9 <= 3 n / 32768 + 12 <= n / 256. So MaxCompressedSize (the sum of the
//           chunk bounds) stays the capacity rule.
//  pack     lz4_pack_frames_kernel (cldn_lz4.cu) concatenates a chunk's pieces behind its [u32 size].
#include <stdint.h>

#include "cldn_device.cuh"
#include "cldn_kernels.h"
#include "cldn_stage2.cuh"

namespace cldn {

// Stage-1 bytes per block (<= Block_Maximum_Size). In one paired run of both builds on the H100
// (tools/zstd_encode_bench.py), 32 KB against 128 KB gave smaller output (6.33 against 6.41 B per point on 1M-point XYZI
// frames: the tables follow the data more closely) and a faster coder (0.24 against 0.32 ms for one such frame, 3.4
// against 4.0 ms for 128 viz clouds). Occupancy is the likely reason: a 128 KB block needs 128 KB of dynamic shared
// memory, so one CTA per SM; at 32 KB the registers bound it (40 x 512 = 20480 of 65536: three CTAs per SM), and one
// CTA's serial steps (thread 0's table) overlap the others' parallel ones.
constexpr uint32_t kZeBlock = 32u * 1024u;
constexpr int kZeThreads = 512;
constexpr int kZeWarps = kZeThreads / 32;
constexpr int kZeRunsPerStream = kZeThreads / 4;
constexpr uint32_t kZeMaxBits = 11u;        // longest Huffman code (RFC 8878 §4.2.1)
constexpr uint32_t kZeMinHuff = 64u;        // four streams need >= 6 literals; below 64 the tables and the jump table do not pay
constexpr uint32_t kZeFrameHeaderMax = 9u;  // magic + FHD + 4-byte Frame_Content_Size
constexpr uint32_t kZeHead = 160u;          // shared bytes in front of the streams: frame header 9 + block header 3 +
                                            // literals header 5 + tree description 1 + 127 + jump table 6 = 151
constexpr uint32_t kZeSlot = (kZeFrameHeaderMax + 3u + kZeBlock + 15u) & ~15u;  // bytes of one piece
constexpr uint32_t kZeSmem = kZeHead + kZeBlock + 16u;                            // dynamic shared memory
static_assert(kZeBlock >= 3146u && kZeBlock <= 131072u && kZeBlock % 16u == 0u, "Block_Maximum_Size, and the bound above");
static_assert((kZeBlock / 4u) * kZeMaxBits / 8u + 1u < 65536u, "a stream's size must fit the 16-bit jump table");
static_assert(kZeWarps * 256u * 4u <= kZeBlock, "the sub-histograms live in the stream buffer");

uint32_t zstd_enc_block_bytes() { return kZeBlock; }
uint32_t zstd_enc_slot_bytes() { return kZeSlot; }

struct ZeShared {
  uint32_t cnt[256];
  uint32_t code[256];      // code << 8 | length, 0 for an unused symbol
  uint16_t sorted[256];    // used symbols by (count, symbol), ascending
  uint32_t iw[256];        // Huffman tree: weights of the internal nodes, in creation order
  uint16_t lpar[256];      // parent of sorted leaf i
  uint16_t ipar[256];      // parent of internal node j
  uint8_t idep[256];       // depth of internal node j
  uint8_t weight[256];
  uint8_t tree[128];       // tree description: header byte + weights
  uint32_t warp_bits[kZeWarps];
  uint32_t tree_bytes;     // 0: no usable table (raw block)
  uint32_t maxlen;
};

__device__ __forceinline__ uint32_t ze_highbit(uint32_t v) { return 31u - static_cast<uint32_t>(__clz(static_cast<int>(v))); }

// Forward bit writer (LSB first) into a small byte array; `ok` falls when it would pass `cap` bytes.
struct ZeBits {
  uint8_t* out;
  uint32_t cap, pos;
  uint64_t acc;
  uint32_t fill;
  bool ok;
  __device__ void put(uint32_t v, uint32_t nb) {
    acc |= static_cast<uint64_t>(v) << fill;
    fill += nb;
    while (fill >= 8u) {
      if (pos < cap) out[pos] = static_cast<uint8_t>(acc);
      else ok = false;
      ++pos;
      acc >>= 8;
      fill -= 8u;
    }
  }
  __device__ uint32_t close() {  // pads to a byte; returns the byte count
    if (fill) put(0u, 8u - fill);
    return pos;
  }
};

// FSE-compressed Huffman weights (RFC 8878 §4.2.1.2, §4.1.1): w[0..nw) with nw >= 2, values <= kZeMaxBits. Writes the
// table description and the two-state bitstream to out[0..127); returns their bytes, 0 when they do not fit or when
// the weights take a single value (a one-symbol FSE table has no bits to end on). Thread 0 alone.
__device__ uint32_t ze_fse_weights(const uint8_t* w, uint32_t nw, uint8_t* out) {
  constexpr uint32_t AL = 6u, T = 1u << AL;
  uint32_t hist[kZeMaxBits + 1];
  for (uint32_t v = 0; v <= kZeMaxBits; ++v) hist[v] = 0;
  for (uint32_t i = 0; i < nw; ++i) ++hist[w[i]];
  uint32_t maxv = 0, distinct = 0, big = 0;
  for (uint32_t v = 0; v <= kZeMaxBits; ++v) {
    if (!hist[v]) continue;
    maxv = v;
    ++distinct;
    if (hist[v] > hist[big]) big = v;
  }
  if (distinct < 2u) return 0u;
  // normalized counts summing to T: floor(T * share), at least 1, the rest to the most frequent value
  int nc[kZeMaxBits + 1];
  int sum = 0;
  for (uint32_t v = 0; v <= kZeMaxBits; ++v) {
    nc[v] = hist[v] ? max(1, static_cast<int>(hist[v] * T / nw)) : 0;
    sum += nc[v];
  }
  nc[big] += static_cast<int>(T) - sum;
  if (nc[big] < 1) return 0u;
  ZeBits bw{out, 127u, 0u, 0ull, 0u, true};
  // table description: accuracy log - 5, then count + 1 per value in the variable-width form, a run of zero counts
  // as 2-bit repeat flags behind the first of them
  bw.put(AL - 5u, 4u);
  int remaining = static_cast<int>(T) + 1, threshold = static_cast<int>(T);
  uint32_t nbits = AL + 1u;
  for (uint32_t v = 0; v <= maxv && remaining > 1;) {
    const int value = nc[v] + 1, lim = 2 * threshold - 1 - remaining;
    if (value < lim) bw.put(static_cast<uint32_t>(value), nbits - 1u);
    else if (value < threshold) bw.put(static_cast<uint32_t>(value), nbits);
    else bw.put(static_cast<uint32_t>(value + lim), nbits);
    remaining -= nc[v];
    while (remaining < threshold) { --nbits; threshold >>= 1; }
    if (nc[v] == 0) {
      uint32_t z = 0;
      while (v + 1u + z <= maxv && nc[v + 1u + z] == 0) ++z;
      v += 1u + z;
      for (; z >= 3u; z -= 3u) bw.put(3u, 2u);
      bw.put(z, 2u);
    } else {
      ++v;
    }
  }
  const uint32_t head = bw.close();
  // decoding table: the spread of RFC 8878 §4.1.1, then each value's states in increasing order
  uint8_t spread[T], states[T];
  uint32_t cum[kZeMaxBits + 2];
  {
    uint32_t p = 0;
    for (uint32_t v = 0; v <= maxv; ++v) {
      for (int i = 0; i < nc[v]; ++i) { spread[p] = static_cast<uint8_t>(v); p = (p + (T >> 1) + (T >> 3) + 3u) & (T - 1u); }
    }
    cum[0] = 0;
    for (uint32_t v = 0; v <= maxv; ++v) cum[v + 1] = cum[v] + static_cast<uint32_t>(nc[v]);
    uint32_t fill[kZeMaxBits + 1];
    for (uint32_t v = 0; v <= maxv; ++v) fill[v] = 0;
    for (uint32_t x = 0; x < T; ++x) states[cum[spread[x]] + fill[spread[x]]++] = static_cast<uint8_t>(x);
  }
  // bitstream, written back to front: the decoder reads state 1 (w[0]), state 2 (w[1]), then the update bits of w[0],
  // w[1], ..., w[nw - 3]. The update after w[nw - 2] finds the stream empty -- its state has at least one bit to read (the
  // first state of its value: c < T) -- and the decoder ends with w[nw - 1] from the other state.
  ZeBits bs{out + head, 127u - head, 0u, 0ull, 0u, head < 127u};
  uint32_t st[2];
  st[(nw - 1u) & 1u] = states[cum[w[nw - 1u]]];
  st[(nw - 2u) & 1u] = states[cum[w[nw - 2u]]];
  for (int k = static_cast<int>(nw) - 3; k >= 0; --k) {
    const uint32_t v = w[k], c = static_cast<uint32_t>(nc[v]);
    const uint32_t y = st[k & 1] + T;  // the state that decodes w[k + 2], plus T
    uint32_t nb = AL - ze_highbit(c);
    if ((y >> nb) < c) --nb;
    bs.put(y & ((1u << nb) - 1u), nb);
    st[k & 1] = states[cum[v] + (y >> nb) - c];
  }
  bs.put(st[1], AL);
  bs.put(st[0], AL);
  bs.put(1u, 1u);  // end mark
  const uint32_t body = bs.close();
  if (!bw.ok || !bs.ok || head + body > 127u) return 0u;
  return head + body;
}

// Thread 0: code lengths (<= kZeMaxBits, a complete code) of the m >= 2 used symbols, their weights and the tree
// description. Leaves S.tree_bytes = 0 when no description fits.
__device__ void ze_build_table(ZeShared& S, uint32_t m) {
  // Huffman tree over the ascending leaves: two queues (leaves, internal nodes in creation order)
  uint32_t li = 0, qi = 0;
  for (uint32_t j = 0; j + 1u < m; ++j) {
    uint32_t sum = 0;
    for (int t = 0; t < 2; ++t) {
      if (li < m && (qi >= j || S.cnt[S.sorted[li]] <= S.iw[qi])) { sum += S.cnt[S.sorted[li]]; S.lpar[li++] = static_cast<uint16_t>(j); }
      else { sum += S.iw[qi]; S.ipar[qi++] = static_cast<uint16_t>(j); }
    }
    S.iw[j] = sum;
  }
  S.idep[m - 2u] = 0;
  for (int j = static_cast<int>(m) - 3; j >= 0; --j) S.idep[j] = static_cast<uint8_t>(min(S.idep[S.ipar[j]] + 1, 250));
  // leaves per length, deeper ones clamped to the limit; then the Kraft sum (units of 2^-L) is brought to exactly 1
  constexpr uint32_t L = kZeMaxBits;
  uint32_t bl[L + 2];
  for (uint32_t l = 0; l <= L + 1u; ++l) bl[l] = 0;
  for (uint32_t i = 0; i < m; ++i) ++bl[min(static_cast<uint32_t>(S.idep[S.lpar[i]]) + 1u, L)];
  uint32_t kraft = 0;
  for (uint32_t l = 1; l <= L; ++l) kraft += bl[l] << (L - l);
  while (kraft > (1u << L)) {  // too many short codes: lengthen the longest code below the limit
    uint32_t l = L - 1u;
    while (bl[l] == 0u) --l;
    --bl[l];
    ++bl[l + 1u];
    kraft -= 1u << (L - l - 1u);
  }
  while (kraft < (1u << L)) {  // room left: shorten the shortest code that fits in it
    const uint32_t room = (1u << L) - kraft;
    uint32_t l = 2;
    while (bl[l] == 0u || (1u << (L - l)) > room) ++l;
    --bl[l];
    ++bl[l - 1u];
    kraft += 1u << (L - l);
  }
  // the most frequent symbols take the shortest codes
  uint32_t l = 1;
  for (int i = static_cast<int>(m) - 1; i >= 0; --i) {
    while (bl[l] == 0u) ++l;
    --bl[l];
    S.idep[i] = static_cast<uint8_t>(l);  // (idep is free again: now the length of sorted leaf i)
  }
  const uint32_t maxlen = l;
  uint32_t last = 0;
  for (uint32_t s = 0; s < 256u; ++s) S.weight[s] = 0;
  for (uint32_t i = 0; i < m; ++i) {
    const uint32_t s = S.sorted[i];
    S.weight[s] = static_cast<uint8_t>(maxlen + 1u - S.idep[i]);
    last = max(last, s);
  }
  S.maxlen = maxlen;
  // weights of symbols 0 .. last - 1 (the last symbol's weight is implied)
  if (last < 128u) {
    S.tree[0] = static_cast<uint8_t>(127u + last);
    for (uint32_t k = 0; k < (last + 1u) / 2u; ++k) {
      S.tree[1u + k] = static_cast<uint8_t>(S.weight[2u * k] << 4 | (2u * k + 1u < last ? S.weight[2u * k + 1u] : 0u));
    }
    S.tree_bytes = 1u + (last + 1u) / 2u;
  } else {
    const uint32_t b = ze_fse_weights(S.weight, last, S.tree + 1);
    S.tree[0] = static_cast<uint8_t>(b);
    S.tree_bytes = b ? 1u + b : 0u;
  }
}

// Little-endian 3-byte block header
__device__ __forceinline__ void ze_block_header(uint8_t* p, bool last, uint32_t type, uint32_t size) {
  const uint32_t v = (last ? 1u : 0u) | type << 1 | size << 3;
  p[0] = static_cast<uint8_t>(v);
  p[1] = static_cast<uint8_t>(v >> 8);
  p[2] = static_cast<uint8_t>(v >> 16);
}

// Frame header of a chunk of `s` bytes: single segment, Frame_Content_Size in 1 / 2 (s - 256) / 4 bytes. Returns its size.
__device__ __forceinline__ uint32_t ze_frame_header(uint8_t* p, uint32_t s) {
  const uint32_t fcs = s < 256u ? 0u : s < 65536u + 256u ? 1u : 2u;
  p[0] = 0x28; p[1] = 0xB5; p[2] = 0x2F; p[3] = 0xFD;
  p[4] = static_cast<uint8_t>(fcs << 6 | 0x20u);
  const uint32_t v = fcs == 1u ? s - 256u : s;
  const uint32_t nb = fcs == 0u ? 1u : fcs == 1u ? 2u : 4u;
  for (uint32_t k = 0; k < nb; ++k) p[5u + k] = static_cast<uint8_t>(v >> (8u * k));
  return 5u + nb;
}

__global__ void __launch_bounds__(kZeThreads) zstd_compress_blocks_kernel(const Lz4Launch L) {
  extern __shared__ __align__(16) uint8_t ze_out[];
  __shared__ ZeShared S;
  __shared__ uint32_t s_start;  // where the piece's bytes start in ze_out (compressed) / the raw bytes start in dst
  const uint32_t b = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31u;
  // the chunk of this piece: the last gc with block_begin[gc] <= b
  uint32_t lo = 0, hi = L.n_chunks_total;
  while (hi - lo > 1u) {
    const uint32_t mid = (lo + hi) >> 1;
    if (L.block_begin[mid] <= b) lo = mid;
    else hi = mid;
  }
  const uint32_t gc = lo, k = b - L.block_begin[gc], allotted = L.block_begin[gc + 1u] - L.block_begin[gc];
  const uint32_t f = L.chunk_frame[gc];
  const Lz4Frame F = L.frames[f];
  if (L.empty_slots && chunk_slot_empty(F, gc)) return;
  uint64_t body = 0;
  const uint32_t s = lz_find_chunk(F.plain, *F.plain_bytes, gc - F.chunk_begin, &body);
  const uint32_t nblk = s == 0xFFFFFFFFu ? 0u : max(1u, (s + kZeBlock - 1u) / kZeBlock);
  uint8_t* dst = L.scratch + static_cast<size_t>(b) * L.slot_stride;
  if (s == 0xFFFFFFFFu || nblk > allotted || k >= nblk) {
    if (tid == 0) {
      L.chunk_sizes[b] = 0u;
      // (a stage-1 chunk that is not where the chunk table says, or larger than its worst case: cannot happen)
      if (k == 0u && (s == 0xFFFFFFFFu || nblk > allotted)) report_frame_error(L, f, DEV_ERR_ENCODE_OUTPUT_SMALL);
    }
    return;
  }
  const uint32_t n = min(kZeBlock, s - k * kZeBlock);
  const uint8_t* src = F.plain + body + static_cast<size_t>(k) * kZeBlock;
  const bool last = k + 1u == nblk;

  // ---- 1. histogram: warp sub-histograms in the stream buffer, aligned 16-byte loads over the block -----------------
  uint32_t* wh = reinterpret_cast<uint32_t*>(ze_out + kZeHead);
  for (uint32_t i = tid; i < kZeWarps * 256u; i += kZeThreads) wh[i] = 0u;
  __syncthreads();
  {
    const uintptr_t a0 = reinterpret_cast<uintptr_t>(src) & ~uintptr_t(15), a1 = (reinterpret_cast<uintptr_t>(src) + n + 15u) & ~uintptr_t(15);
    const uint32_t nv = static_cast<uint32_t>((a1 - a0) >> 4), lead = static_cast<uint32_t>(reinterpret_cast<uintptr_t>(src) - a0);
    uint32_t* h = wh + warp * 256u;
    for (uint32_t v = tid; v < nv; v += kZeThreads) {
      const uint4 q = reinterpret_cast<const uint4*>(a0)[v];
      const uint32_t w4[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
      for (uint32_t j = 0; j < 16u; ++j) {
        const uint32_t at = 16u * v + j;  // offset from a0
        if (at >= lead && at < lead + n) atomicAdd(&h[(w4[j >> 2] >> (8u * (j & 3u))) & 0xFFu], 1u);
      }
    }
  }
  __syncthreads();
  if (tid < 256u) {
    uint32_t c = 0;
    for (uint32_t w = 0; w < kZeWarps; ++w) c += wh[w * 256u + tid];
    S.cnt[tid] = c;
  }
  __syncthreads();

  // ---- 2. block form --------------------------------------------------------------------------------------------
  const bool rle = n > 0u && S.cnt[src[0]] == n;
  bool huff = !rle && n >= kZeMinHuff;
  if (huff) {
    if (tid < 256u) {
      const uint32_t c = S.cnt[tid];
      if (c) {
        uint32_t rank = 0;
        for (uint32_t t = 0; t < 256u; ++t) {
          const uint32_t ct = S.cnt[t];
          rank += ct != 0u && (ct < c || (ct == c && t < tid));
        }
        S.sorted[rank] = static_cast<uint16_t>(tid);
      }
    }
    __syncthreads();
    if (tid == 0) {
      uint32_t m = 0;
      for (uint32_t t = 0; t < 256u; ++t) m += S.cnt[t] != 0u;
      ze_build_table(S, m);  // m >= 2: the block is not RLE
    }
    __syncthreads();
    huff = S.tree_bytes != 0u;
  }
  uint32_t streams_bytes = 0, sb[4] = {0, 0, 0, 0}, lh = 0, run_a = 0, run_e = 0, run_off = 0;
  if (huff) {
    // canonical codes: symbols by (weight, symbol) take consecutive ranges of the 2^maxlen-entry decoding table
    if (tid < 256u) {
      const uint32_t w = S.weight[tid];
      uint32_t code = 0;
      if (w) {
        uint32_t start = 0;
        for (uint32_t t = 0; t < 256u; ++t) {
          const uint32_t wt = S.weight[t];
          if (wt != 0u && (wt < w || (wt == w && t < tid))) start += 1u << (wt - 1u);
        }
        code = (start >> (w - 1u)) << 8 | (S.maxlen + 1u - w);
      }
      S.code[tid] = code;
    }
    __syncthreads();
    // ---- 3. runs: stream j = tid / kZeRunsPerStream; (n + 3) / 4 literals in streams 1..3, the rest in stream 4 ---------
    const uint32_t seg = (n + 3u) / 4u, j = tid / kZeRunsPerStream, i = tid % kZeRunsPerStream;
    const uint32_t s_begin = j * seg, s_len = j < 3u ? seg : n - 3u * seg;
    const uint32_t per = (seg + kZeRunsPerStream - 1u) / kZeRunsPerStream;
    run_a = min(s_begin + i * per, s_begin + s_len);
    run_e = min(run_a + per, s_begin + s_len);
    uint32_t bits = 0;
    for (uint32_t p = run_a; p < run_e; ++p) bits += S.code[src[p]] & 0xFFu;
    // bits of the later runs of the same stream: the stream is written back to front
    uint32_t suf = bits;
#pragma unroll
    for (uint32_t d = 1; d < 32u; d <<= 1) {
      const uint32_t y = __shfl_down_sync(0xffffffffu, suf, d);
      if (lane + d < 32u) suf += y;
    }
    if (lane == 0) S.warp_bits[warp] = suf;
    __syncthreads();
    constexpr uint32_t wps = kZeRunsPerStream / 32;  // warps per stream
    run_off = suf - bits;
    for (uint32_t w = warp + 1u; w < (j + 1u) * wps; ++w) run_off += S.warp_bits[w];
    uint32_t total_bits[4];
    for (uint32_t q = 0; q < 4u; ++q) {
      total_bits[q] = 0;
      for (uint32_t w = q * wps; w < (q + 1u) * wps; ++w) total_bits[q] += S.warp_bits[w];
      sb[q] = total_bits[q] / 8u + 1u;  // + the end mark
      streams_bytes += sb[q];
    }
    lh = n < 1024u ? 3u : n < 16384u ? 4u : 5u;
    const uint32_t lit_c = S.tree_bytes + 6u + streams_bytes;
    huff = lh + lit_c + 1u < n;
    if (huff) {
      // ---- 4. streams into shared memory at kZeHead ------------------------------------------------------------------
      __syncthreads();  // every thread has read the sub-histograms' space for the last time (warp_bits: above)
      uint32_t* ow = reinterpret_cast<uint32_t*>(ze_out + kZeHead);
      for (uint32_t x = tid; x < (streams_bytes + 7u) / 4u; x += kZeThreads) ow[x] = 0u;
      __syncthreads();
      uint32_t base = 0;
      for (uint32_t q = 0; q < j; ++q) base += sb[q];
      uint32_t pos = base * 8u + run_off;
      uint32_t word = pos >> 5, fill = pos & 31u;
      uint64_t acc = 0;
      for (uint32_t p = run_e; p > run_a; --p) {
        const uint32_t c = S.code[src[p - 1u]];
        acc |= static_cast<uint64_t>(c >> 8) << fill;
        fill += c & 0xFFu;
        if (fill >= 32u) {
          atomicOr(&ow[word], static_cast<uint32_t>(acc));
          acc >>= 32;
          fill -= 32u;
          ++word;
        }
      }
      if (fill) atomicOr(&ow[word], static_cast<uint32_t>(acc));
      if (i == 0u) {  // end mark behind the stream's first symbol
        const uint32_t e = base * 8u + total_bits[j];
        atomicOr(&ow[e >> 5], 1u << (e & 31u));
      }
      __syncthreads();
    }
  }

  // ---- 5. the piece --------------------------------------------------------------------------------------------------
  if (huff) {
    const uint32_t lit_c = S.tree_bytes + 6u + streams_bytes, content = lh + lit_c + 1u;
    const uint32_t head_bytes = 3u + lh + S.tree_bytes + 6u;
    if (tid == 0) {
      uint8_t fhb[kZeFrameHeaderMax];
      const uint32_t f = k == 0u ? ze_frame_header(fhb, s) : 0u;
      uint8_t* p = ze_out + kZeHead - head_bytes - f;
      for (uint32_t x = 0; x < f; ++x) p[x] = fhb[x];
      p += f;
      ze_block_header(p, last, 2u, content);
      p += 3;
      // Literals_Block_Type 2, Size_Format 1 / 2 / 3 (four streams, 10 / 14 / 18-bit sizes), Regenerated_Size, Compressed_Size
      const uint32_t sbits = lh == 3u ? 10u : lh == 4u ? 14u : 18u;
      const uint64_t hdr = 2ull | static_cast<uint64_t>(lh - 2u) << 2 | static_cast<uint64_t>(n) << 4 | static_cast<uint64_t>(lit_c) << (4u + sbits);
      for (uint32_t x = 0; x < lh; ++x) p[x] = static_cast<uint8_t>(hdr >> (8u * x));
      p += lh;
      for (uint32_t x = 0; x < S.tree_bytes; ++x) p[x] = S.tree[x];
      p += S.tree_bytes;
      for (uint32_t q = 0; q < 3u; ++q) { p[2u * q] = static_cast<uint8_t>(sb[q]); p[2u * q + 1u] = static_cast<uint8_t>(sb[q] >> 8); }
      ze_out[kZeHead + streams_bytes] = 0u;  // Number_of_Sequences
      s_start = kZeHead - head_bytes - f;
      L.chunk_sizes[b] = f + 3u + content;
    }
    __syncthreads();
    lz_copy(dst, ze_out + s_start, kZeHead + streams_bytes + 1u - s_start, tid, kZeThreads);
    return;
  }
  if (tid == 0) {
    const uint32_t f = k == 0u ? ze_frame_header(dst, s) : 0u;
    ze_block_header(dst + f, last, rle ? 1u : 0u, n);
    if (rle) dst[f + 3u] = src[0];
    L.chunk_sizes[b] = f + 3u + (rle ? 1u : n);
    s_start = f + 3u;
  }
  __syncthreads();
  if (!rle) lz_copy(dst + s_start, src, n, tid, kZeThreads);
}

int launch_zstd_compress(const Lz4Launch& L, const uint8_t* header, uint32_t header_bytes, cudaStream_t stream) {
  if (L.n_frames == 0) return 0;
  int n = 0;
  if (L.n_blocks_total) {
    if (raise_smem_limit(zstd_compress_blocks_kernel, kZeSmem) != cudaSuccess) return -1;
    zstd_compress_blocks_kernel<<<L.n_blocks_total, kZeThreads, kZeSmem, stream>>>(L);
    count_launch(1);
    ++n;
  }
  const int p = launch_stage2_pack(L, header, header_bytes, stream);
  return p < 0 ? p : n + p;
}

}  // namespace cldn
