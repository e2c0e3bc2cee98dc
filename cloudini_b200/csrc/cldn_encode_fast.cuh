// ENCODE of packed XYZI float32x4 clouds (point_step 16, 16-byte aligned frames): the FAST FloatN kernel.
// Included by cldn_encode.cu (shares finish_tile / find_frame; the build has no relocatable device code).
//
// Same bytes as FieldEncoderFloatN_Lossy::encode (cloudini_lib/src/field_encoder.cpp:42-91) + WriteStage1Chunk's framing
// (chunk_writer.cpp:27-48). Shape:
//  * thread-blocked points: a thread owns 8 consecutive points of a 1024-point tile, so the previous point is a
//    register (no shuffle / select per value) and the thread's bytes are ONE contiguous run of the output;
//  * the tile is loaded with coalesced 16-byte loads and transposed through shared memory inside each warp
//    (16-byte slots, XOR-swizzled: conflict-free both ways);
//  * pass 1 (per value: FMUL, F2I, |s| tracking with max.NaN, delta, zigzag + 1, 7-bit groups -> bytes with two
//    add/mask steps, continuation flags from the top bit) keeps the finished LEB128 words in registers and sums their
//    lengths; one warp scan + 4 warp totals give every thread its byte offset;
//  * pass 2 streams the words through a 64-bit register window and flushes aligned 32-bit words straight to their final
//    place in the staging buffer: a thread starts its window with the last bytes of its predecessor (every thread
//    publishes the last 4 bytes of its run before the scan), so words shared by two threads are written once, whole;
//  * a CTA walks a group of 4 consecutive tiles of one frame: one decoupled look-back per group, the other tiles know
//    their prefix locally and publish it as inclusive at once.
// Anything the 4-byte fast path cannot represent -- NaN / inf input, |v * mul| >= 2^25 (so that every delta fits 4
// varint bytes and no product reaches the x86 "integer indefinite" range), a partial tile -- sends the TILE to the exact
// byte-wise path below, which evaluates everything like the reference does.
#pragma once

namespace cldn {

constexpr int kET = 128;                  // threads per CTA
constexpr int kFastEncMinBlocks = 6;      // resident CTAs per SM the register allocation aims at
constexpr int kEW = kET / 32;
constexpr int kEP = 8;                    // points per thread and tile
constexpr int kETilePts = kET * kEP;      // 1024
constexpr int kEBufBytes = kETilePts * 16;          // one input buffer = one tile of transposed points (later: its staged bytes)
constexpr int kECarefulBytes = kETilePts * 20 + 64; // worst case of the exact path: 5 bytes per value
constexpr int kESmemBytes = (2 * kEBufBytes > kECarefulBytes ? 2 * kEBufBytes : kECarefulBytes) + 64;

struct EncFastShared {
  uint32_t wtot[kEW];        // bytes per warp
  uint32_t wtail[kEW];       // last 4 bytes of every warp's run (top byte = most recent)
  unsigned long long excl;   // look-back result of the group's first tile
  uint32_t scan[kET / 32 + 1];
  uint32_t first;            // the CTA's first tile and ...
  uint32_t ticket;           // ... the tile it takes next (thread 0 draws both from L.tile_ticket)
};

__device__ __forceinline__ float max_nan(float a, float b) {  // NaN if either is NaN (fmaxf would drop it)
  float d;
  asm("max.NaN.f32 %0, %1, %2;" : "=f"(d) : "f"(a), "f"(b));
  return d;
}
__device__ __forceinline__ uint32_t top_bit(uint32_t x) {  // index of the most significant set bit; 0xFFFFFFFF for 0
  uint32_t b;
  asm("bfind.u32 %0, %1;" : "=r"(b) : "r"(x));
  return b;
}
__device__ __forceinline__ uint32_t low_mask(uint32_t n) {  // (1 << n) - 1, all ones for n >= 32: one BMSK
  uint32_t d;
  asm("bmsk.clamp.b32 %0, %1, %2;" : "=r"(d) : "r"(0), "r"(n));
  return d;
}
__device__ __forceinline__ uint32_t bitselect_e(uint32_t m, uint32_t a, uint32_t b) {  // (a & m) | (b & ~m), one LOP3
  uint32_t d;
  asm("lop3.b32 %0, %1, %2, %3, 0xCA;" : "=r"(d) : "r"(m), "r"(a), "r"(b));
  return d;
}

// Exact byte-wise evaluation of one tile (thread t owns points 8 t .. 8 t + 7), like the reference (field_encoder.cpp:42-91).
// Returns the tile's byte count; the bytes are in `stage`. All threads of the CTA call it.
template <int N>
__device__ __noinline__ uint32_t encode_tile_careful(const EncFrame& F, const FloatNParams& P, uint32_t tile_p0, uint8_t* stage,
                                                     uint32_t* scan_scratch) {
  const uint32_t step = P.point_step;
  uint32_t len[kEP];
  uint32_t mine = 0;
#pragma unroll 1
  for (int i = 0; i < kEP; ++i) {
    const uint32_t p = tile_p0 + threadIdx.x * kEP + i;
    uint32_t l = 0;
    if (p < F.n_points) {
      const uint8_t* pt = F.in + static_cast<size_t>(p) * step;
      const uint8_t* prevp = (p % kChunkPoints) ? pt - step : nullptr;
#pragma unroll
      for (int k = 0; k < N; ++k) {
        const float x = __uint_as_float(load_u32(pt + P.offset[k]));
        if (isnan(x)) { l += 1; continue; }
        const int32_t q = quant_i32_x86(x, P.mul[k]);
        int32_t pq = 0;
        if (prevp) {
          const float px = __uint_as_float(load_u32(prevp + P.offset[k]));
          if (!isnan(px)) pq = quant_i32_x86(px, P.mul[k]);
        }
        const int32_t d = static_cast<int32_t>(static_cast<uint32_t>(q) - static_cast<uint32_t>(pq));
        l += varint_len(zigzag_plus1(static_cast<int64_t>(d)));
      }
    }
    len[i] = l;
    mine += l;
  }
  __syncthreads();  // the staging buffer may still hold the transposed input other warps are reading
  uint32_t total;
  uint32_t off = block_exclusive_scan_n<kET>(mine, scan_scratch, &total);
#pragma unroll 1
  for (int i = 0; i < kEP; ++i) {
    const uint32_t p = tile_p0 + threadIdx.x * kEP + i;
    if (p < F.n_points) {
      const uint8_t* pt = F.in + static_cast<size_t>(p) * step;
      const uint8_t* prevp = (p % kChunkPoints) ? pt - step : nullptr;
      ByteSink bs{stage + off};
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
      off += len[i];
    }
  }
  return total;
}

// Alternatives measured slower during development: one tile per CTA (the load latency is exposed at every CTA start);
// four consecutive tiles per CTA (the next group's look-back waits for this CTA's LAST tile: the frame serialises);
// independent 256-point warp tiles without any CTA barrier (four times as many status words: the look-back gets deeper);
// warp-private buffers with one barrier per tile, with and without deferring the copy-out by one tile (every warp
// following the look-back costs more than the two barriers it saves).
// Persistent CTAs: every CTA takes its tiles in the launch's global tile order (frame-interleaved for uniform batches, so
// the tiles a look-back depends on are being processed by other CTAs at the same time) from a ticket counter. While
// tile i is quantised and packed, the CTA's next tile is already on its way into the other input buffer (cp.async, 16
// bytes per lane, straight into the transposed slots): the load latency that a one-tile-per-CTA kernel exposes at every
// CTA start (measured: a third of all stall samples) is hidden behind the previous tile's arithmetic.
// Also measured (commit 5f46c71 has the code: CLDN_FAST_ENC_PIPE=1/2, removed again): pass 1 of tile i + 1 between pass 2 of tile i and its
// look-back result, with and without the barrier behind the copy-out: slower either way -- the
// later inclusive prefix makes every successor's look-back longer than the wait it hides.
// Why tickets: a CTA spins on aggregates of tiles with a smaller global index. A tile is only ever held by a CTA that has
// started, and a CTA handles its tiles in increasing order, so the smallest unfinished tile is always the current tile
// of a running CTA and can finish. A fixed assignment (CTA b takes b, b + G, ...) would need all G CTAs resident at
// once, which no longer holds when kernels of other streams or handles occupy part of the GPU.
__device__ __forceinline__ void tile_coords(const EncLaunch& L, uint32_t i, uint32_t* fi, uint32_t* t) {
  if (L.uniform_tiles) {
    *fi = i % L.n_frames;
    *t = i / L.n_frames;
  } else {
    *fi = find_frame(L.frames, L.n_frames, i);
    *t = i - L.frames[*fi].tile_begin;
  }
}

__global__ void __launch_bounds__(kET, kFastEncMinBlocks) encode_xyzi_fast_kernel(const EncLaunch L, const FloatNParams P) {
  extern __shared__ __align__(16) uint8_t dyn_smem[];
  __shared__ EncFastShared sh;
  __shared__ EncFrame s_F[2];
  __shared__ FloatNParams s_P;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const bool aligned16 = (L.flags & kEncInputsAligned16) != 0u;

  if (blockIdx.x == 0) handle_empty_frames(L);
  if (threadIdx.x == 0) {
    sh.first = atomicAdd(L.tile_ticket, 1u);
    if (sh.first < L.n_tiles_total) {
      uint32_t f0, t0;
      tile_coords(L, sh.first, &f0, &t0);
      s_F[0] = L.frames[f0];
    }
    s_P = P;
  }
  __syncthreads();
  const uint32_t i = sh.first;
  if (i >= L.n_tiles_total) return;
  uint32_t fi, t;
  tile_coords(L, i, &fi, &t);

  // asks for the 1024 points of tile t of frame F into `buf` (transposed slots); false if the tile is not eligible
  auto prefetch = [&](const EncFrame& F, uint32_t tt, uint8_t* buf) -> bool {
    const uint32_t p0 = tt * kETilePts;
    if (!aligned16 || p0 + kETilePts > F.n_points) return false;
    const uint4* src = reinterpret_cast<const uint4*>(F.in) + p0 + warp * (32 * kEP) + lane;
    uint4* wsl = reinterpret_cast<uint4*>(buf) + warp * (32 * kEP);
#pragma unroll
    for (int k = 0; k < kEP; ++k) {
      const uint32_t q = 32u * k + lane, ol = q >> 3;
      async_copy16(wsl + 8 * ol + ((q & 7u) ^ (ol & 7u)), src + 32 * k);
    }
    return true;
  };
  bool have_cur = prefetch(s_F[0], t, dyn_smem);
  async_commit();
  if (threadIdx.x == 0) sh.ticket = atomicAdd(L.tile_ticket, 1u);
  __syncthreads();

  for (uint32_t cur = 0;; cur ^= 1u) {
    const EncFrame& F = s_F[cur];
    uint8_t* buf = dyn_smem + cur * kEBufBytes;            // this tile's transposed input, then its staged output
    uint8_t* stage = buf;
    // ---- the next tile of this CTA goes into the other buffer now ----
    const uint32_t nxt = sh.ticket;   // (rewritten only behind the barriers below)
    bool have_next = false;
    uint32_t nfi = 0, nt = 0;
    if (nxt < L.n_tiles_total) {
      tile_coords(L, nxt, &nfi, &nt);
      if (threadIdx.x == 0) s_F[cur ^ 1u] = L.frames[nfi];
      // (every thread needs the frame's input pointer and size for its own copies: read them from the table directly)
      const EncFrame* NF = L.frames + nfi;
      const uint32_t p0 = nt * kETilePts;
      if (aligned16 && p0 + kETilePts <= NF->n_points) {
        const uint4* src = reinterpret_cast<const uint4*>(NF->in) + p0 + warp * (32 * kEP) + lane;
        uint4* wsl = reinterpret_cast<uint4*>(dyn_smem + (cur ^ 1u) * kEBufBytes) + warp * (32 * kEP);
#pragma unroll
        for (int k = 0; k < kEP; ++k) {
          const uint32_t q = 32u * k + lane, ol = q >> 3;
          async_copy16(wsl + 8 * ol + ((q & 7u) ^ (ol & 7u)), src + 32 * k);
        }
        have_next = true;
      }
    }
    async_commit();

    const uint32_t tile = F.tile_begin + t;
    const uint32_t tile_p0 = t * kETilePts;
    const bool full = tile_p0 + kETilePts <= F.n_points;
    uint32_t total = 0;
    bool fast = full;
    uint32_t X[kEP][4];
    uint32_t mine = 0, tail4 = 0;
    if (full) {
      const uint32_t wp0 = tile_p0 + warp * (32 * kEP);
      uint4* wsl = reinterpret_cast<uint4*>(buf) + warp * (32 * kEP);
      if (have_cur) {
        async_wait_all_but_last();   // this tile's copies have landed (the next tile's may still be in flight)
      } else {
        // ---- load + transpose inside the warp: lane l of iteration k loads point 32 k + l of the warp's 256 ----
#pragma unroll
        for (int k = 0; k < kEP; ++k) {
          const uint32_t q = 32u * k + lane;
          uint4 v;
          if (aligned16) {
            v = __ldcs(reinterpret_cast<const uint4*>(F.in) + wp0 + q);
          } else {
            const uint8_t* pt = F.in + static_cast<size_t>(wp0 + q) * 16u;
            v = make_uint4(load_u32(pt), load_u32(pt + 4), load_u32(pt + 8), load_u32(pt + 12));
          }
          const uint32_t ol = q >> 3;  // owner lane; slot of point j of lane l: 8 l + (j ^ (l & 7))
          wsl[8 * ol + ((q & 7u) ^ (ol & 7u))] = v;
        }
      }
      // previous point of my first point: 0 at a chunk start, else quantised like any point
      const uint32_t p_first = wp0 + lane * kEP;
      uint4 pvu = make_uint4(0, 0, 0, 0);
      if (lane == 0 && (p_first % kChunkPoints) != 0) {
        const uint8_t* pt = F.in + static_cast<size_t>(p_first - 1) * 16u;
        pvu = make_uint4(load_u32(pt), load_u32(pt + 4), load_u32(pt + 8), load_u32(pt + 12));
      }
      __syncwarp();
      if (lane != 0) {
        const uint32_t pl = lane - 1;
        pvu = wsl[8 * pl + (7u ^ (pl & 7u))];
      }
      float trk = 0.0f;
      int32_t prev[4];
      {
        const float pf[4] = {__uint_as_float(pvu.x), __uint_as_float(pvu.y), __uint_as_float(pvu.z), __uint_as_float(pvu.w)};
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const float s = __fmul_rn(pf[k], P.mul[k]);
          trk = max_nan(trk, fabsf(s));
          prev[k] = __float2int_rn(s);
        }
      }
      // ---- pass 1: LEB128 words of my 32 values + their total length ----
      uint32_t nbl[3] = {0, 0, 0};  // bit lengths of my last three values (for the tail word)
#pragma unroll
      for (int j = 0; j < kEP; ++j) {
        const uint4 u = wsl[8 * lane + (j ^ (lane & 7))];
        const float pf[4] = {__uint_as_float(u.x), __uint_as_float(u.y), __uint_as_float(u.z), __uint_as_float(u.w)};
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const float s = __fmul_rn(pf[k], P.mul[k]);   // _mm_mul_ps: IEEE RN, never contracted
          trk = max_nan(trk, fabsf(s));
          const int32_t q = __float2int_rn(s);          // cvtps2dq under the default MXCSR: ties to even
          const uint32_t d = static_cast<uint32_t>(q) - static_cast<uint32_t>(prev[k]);
          prev[k] = q;
          const uint32_t zz1 = ((d << 1) ^ static_cast<uint32_t>(static_cast<int32_t>(d) >> 31)) + 1u;  // < 2^28 on the fast path
          // 7-bit groups -> bytes: 14-bit halves into 16-bit lanes, then the upper 7 bits of each lane one bit up
          uint32_t x = (zz1 & 0xFFFFC000u) * 3u + zz1;           // lo14 + hi14 * 2^16 (one LOP3 + one IMAD)
          x = x + (x & 0x3F803F80u);
          const uint32_t b = top_bit(x);                           // inside the value's last byte (garbage tiles: x may be 0)
          x |= low_mask(b) & 0x00808080u;                          // continuation flags on every byte below it
          X[j][k] = x;
          mine += b >> 3;
          if (j == kEP - 1 && k >= 1) nbl[k - 1] = (b & 0x18u) + 8u;
        }
      }
      mine += kEP * 4;
      // last 4 bytes of my run (top byte = most recent): the successor starts its window with them
      tail4 = __funnelshift_rc(tail4, X[kEP - 1][1], nbl[0]);
      tail4 = __funnelshift_rc(tail4, X[kEP - 1][2], nbl[1]);
      tail4 = __funnelshift_rc(tail4, X[kEP - 1][3], nbl[2]);
      fast = trk < 33554432.0f;  // 2^25; false for NaN
    }
    // ---- offsets: warp scan + warp totals ----
    uint32_t inc = mine;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const uint32_t up = __shfl_up_sync(0xffffffffu, inc, d);
      if (lane >= d) inc += up;
    }
    uint32_t ptail = __shfl_up_sync(0xffffffffu, tail4, 1);
    if (lane == 31) { sh.wtot[warp] = inc; sh.wtail[warp] = tail4; }
    const int any_slow = __syncthreads_or(fast ? 0 : 1);  // also: every warp is done with its transposed input
    LookbackPoll lb;
    if (!any_slow) {
      uint32_t wbase = 0;
#pragma unroll
      for (int w = 0; w < kEW; ++w) {
        const uint32_t c = sh.wtot[w];
        if (w < warp) wbase += c;
        total += c;
      }
      // the tile's size is final: publish it before the bytes are packed, so that successors never wait for pass 2
      if (warp == 0) {
        lb.begin(L.status, F.tile_begin, tile, L.epoch, total);
        lb.issue(L.status, F.tile_begin, L.epoch);
      }
      if (lane == 0) ptail = warp > 0 ? sh.wtail[warp - 1] : 0u;
      const uint32_t off = wbase + inc - mine;
      // ---- pass 2: 64-bit window, aligned word flushes ----
      // `bit` = bit position of the next byte in the tile's stream; the window's low word is the aligned word holding it
      uint32_t bit = 8u * off;
      uint32_t lo = __funnelshift_rc(ptail, 0u, 32u - (bit & 31u));   // the last off % 4 bytes of the predecessor (0 if none)
      uint32_t wa = (bit >> 3) & ~3u;                                 // byte address of that word in the staging buffer
#pragma unroll
      for (int j = 0; j < kEP; ++j) {
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const uint32_t x = X[j][k];
          const uint32_t b = top_bit(x);
          lo |= __funnelshift_l(0u, x, bit);                 // x << (bit % 32)
          const uint32_t hi = __funnelshift_l(x, 0u, bit);   // x >> (32 - bit % 32), 0 for bit % 32 == 0
          bit += (b & 0x18u) + 8u;
          const uint32_t wn = (bit >> 3) & ~3u;
          if (wn != wa) { *reinterpret_cast<uint32_t*>(stage + wa) = lo; lo = hi; }
          wa = wn;
        }
      }
      if (threadIdx.x == kET - 1 && (bit & 31u) != 0u) *reinterpret_cast<uint32_t*>(stage + wa) = lo;  // nobody follows the tile's last thread
    } else {
      // exact path: up to 20 bytes per point, staged from the start of the dynamic shared memory across BOTH input buffers --
      // the next tile's copies are drained first and the tile is loaded again, synchronously, when its turn comes
      async_wait_all();
      __syncthreads();
      have_next = false;
      stage = dyn_smem;
      total = encode_tile_careful<4>(F, s_P, tile_p0, stage, sh.scan);
      if (warp == 0) lb.begin(L.status, F.tile_begin, tile, L.epoch, total);
    }
    // ---- the tile's place in the frame ----
    if (warp == 0) {
      const uint64_t e = lb.finish(L.status, F.tile_begin, tile, L.epoch, total);
      if (lane == 0) sh.excl = e;
    }
    __syncthreads();  // staged bytes + sh.excl complete (and s_F[cur ^ 1] written)
    finish_tile<kETilePts>(L, F, fi, t, stage, total, sh.excl);
    // the ticket for the tile after next is drawn just before that tile's copies are issued
    if (threadIdx.x == 0 && nxt < L.n_tiles_total) sh.ticket = atomicAdd(L.tile_ticket, 1u);
    __syncthreads();  // this buffer receives the tile after next (and sh.ticket is published)
    if (nxt >= L.n_tiles_total) break;
    have_cur = have_next;
    fi = nfi;
    t = nt;
  }
  async_wait_all();
}

static bool encode_fast_enabled() {
  const char* e = getenv("CLDN_B200_ENC_FAST");
  return !(e && e[0] == '0');
}
// Plans / batches the fast kernel takes: exactly one FloatN op over packed float32x4 at offsets 0,4,8,12 of a 16-byte point.
bool encode_fast_applies(const Plan& plan) {
  if (!plan.floatn_only || !encode_fast_enabled()) return false;
  const RegOp& op = plan.ops[0];
  if (!(op.lanes == 4 && plan.point_step == 16 && op.offset[0] == 0 && op.offset[1] == 4 && op.offset[2] == 8 && op.offset[3] == 12)) return false;
  for (int k = 0; k < 4; ++k) {
    const float m = op.enc_mul_f[k];
    if (!(m > 0.0f) || m > 3.0e38f) return false;  // the |s| < 2^25 test must imply a finite, non-NaN input
  }
  return true;
}
uint32_t encode_fast_tile_points() { return kETilePts; }

static int launch_encode_fast(const Plan& plan, const EncLaunch& L, cudaStream_t stream) {
  FloatNParams P;
  for (int k = 0; k < 4; ++k) {
    P.offset[k] = plan.ops[0].offset[k];
    P.mul[k] = plan.ops[0].enc_mul_f[k];
  }
  P.point_step = plan.point_step;
  const size_t smem = kESmemBytes;
  auto k = encode_xyzi_fast_kernel;
  if (set_smem(k, smem) != cudaSuccess) return -1;
  // persistent grid of one GPU's worth of CTAs; they take their tiles from the ticket counter, so none has to be resident
  static const int resident = [&] {
    int dev = 0, sms = 0, per_sm = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k, kET, smem) != cudaSuccess || per_sm < 1) per_sm = 1;
    return std::max(1, sms) * per_sm;
  }();
  const uint32_t grid = std::min<uint32_t>(L.n_tiles_total, static_cast<uint32_t>(resident));
  if (cudaMemsetAsync(L.tile_ticket, 0, sizeof(uint32_t), stream) != cudaSuccess) return -1;
  k<<<grid, kET, smem, stream>>>(L, P);
  count_launch();
  return 1;
}

}  // namespace cldn
