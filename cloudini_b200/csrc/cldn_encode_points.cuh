// ENCODE of real sensor layouts whose regular stream is all 32-bit float varints: one FloatN group (x y z [intensity])
// followed by scalar lossy FLOAT32 fields (a Velodyne `time`, ...), any point_step, any field offsets, any alignment --
// XYZ (step 12), padded XYZ + V5 integer sections (step 32), XYZIRT (step 22). Included by cldn_encode.cu.
//
// Same bytes as the reference's per-point loop over FieldEncoderFloatN_Lossy::encode (field_encoder.cpp:42-91) and
// FieldEncoderFloat_Lossy<float>::encode (field_encoder.hpp:343-357), framing as in chunk_writer.cpp:27-48. The packed
// XYZI layout has its own kernel (cldn_encode_fast.cuh); this one trades its transposed 16-byte slots for a raw copy of
// the tile's bytes in shared memory, from which every lane reads its own points field by field.
//  * tile = 128 lanes x EP points (EP = 8 for <= 4 values per point, 4 above: the LEB128 words of a lane stay in registers);
//  * pass 1: value -> quantise (FloatN: cvt.rni of v * (1/res), ties to even; scalar: roundf of v * float(1/res), half away
//    from zero) -> delta to the previous point (a register) -> zigzag + 1 -> LEB128 word; lengths summed;
//  * one CTA scan, the tile's size published for the decoupled look-back, pass 2 with the 64-bit window / aligned word
//    flushes of the XYZI kernel, finish_tile (copy-out, chunk prefix, V5 section offsets).
// A tile with a NaN / inf, a product >= 2^25 in magnitude or fewer points than a full tile goes through the plan
// interpreter (encode_point_ops), byte by byte, exactly like the generic kernel.
#pragma once

namespace cldn {

constexpr int kPT = 128;  // threads per CTA

struct PointsParams {
  uint32_t offset[6];
  float mul[6];
  uint32_t n_floatn;   // the first n_floatn values are the FloatN group (ties to even), the rest scalar lossy (half away)
  uint32_t point_step;
};

// Field reads from the staged tile. On the device the address is a 32-bit shared-window address and the loads are
// ld.shared: through a generic `const uint8_t*` every read cost 64-bit pointer arithmetic and a generic load (17
// instructions per value measured; the kernel is instruction-bound).
#ifdef CLDN_CUSIM
typedef const uint8_t* SmemAddr;
__device__ __forceinline__ SmemAddr smem_addr(const uint8_t* p) { return p; }
template <bool ALIGNED4>
__device__ __forceinline__ uint32_t smem_load_u32(SmemAddr base, uint32_t byte_off) {
  if (ALIGNED4) return *reinterpret_cast<const uint32_t*>(base + byte_off);
  const uintptr_t a = reinterpret_cast<uintptr_t>(base + byte_off);
  const uint32_t* w = reinterpret_cast<const uint32_t*>(a & ~uintptr_t(3));
  return __funnelshift_r(w[0], w[1], 8u * static_cast<uint32_t>(a & 3u));
}
#else
typedef uint32_t SmemAddr;
__device__ __forceinline__ SmemAddr smem_addr(const uint8_t* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }
__device__ __forceinline__ uint32_t lds_u32(uint32_t a) {
  uint32_t v;
  asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(a));
  return v;
}
template <bool ALIGNED4>
__device__ __forceinline__ uint32_t smem_load_u32(SmemAddr base, uint32_t byte_off) {
  const uint32_t a = base + byte_off;
  if (ALIGNED4) return lds_u32(a);
  const uint32_t w = a & ~3u;
  return __funnelshift_r(lds_u32(w), lds_u32(w + 4u), 8u * a);   // the funnel shift takes the low 5 bits: 8 * (a & 3)
}
#endif

template <int NV, int EP, bool ALIGNED4, int NF>   // NF: lanes of the leading FloatN group (ties to even); the others round half away
__global__ void __launch_bounds__(kPT) encode_points_fast_kernel(const EncLaunch L, const PointsParams P) {
  constexpr uint32_t T = kPT * EP;
  extern __shared__ __align__(16) uint8_t dyn_smem[];
  __shared__ uint32_t s_wtot[kPT / 32], s_wtail[kPT / 32], s_scan[kPT / 32 + 1];
  __shared__ unsigned long long s_excl;
  const Plan& plan = *L.plan;                                            // exact path only (rare): read in place
  uint8_t* raw = dyn_smem;                                               // tile bytes, the previous point in front of them
  uint8_t* stage = raw;                                                  // staged output aliases them after pass 1
  const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  const uint32_t step = P.point_step;

  if (blockIdx.x == 0) handle_empty_frames(L);
  const uint32_t fi = L.uniform_tiles ? blockIdx.x % L.n_frames : find_frame(L.frames, L.n_frames, blockIdx.x);
  const EncFrame F = L.frames[fi];
  const uint32_t t = L.uniform_tiles ? blockIdx.x / L.n_frames : blockIdx.x - F.tile_begin;
  if (L.empty_slots && t >= F.n_tiles) return;  // an empty tile slot (EncLaunch::empty_slots)
  const uint32_t tile = F.tile_begin + t;
  const uint32_t tile_p0 = t * T;
  const bool full = tile_p0 + T <= F.n_points;
  const bool chunk_start = (tile_p0 % kChunkPoints) == 0;

  // ---- the tile's bytes (and the point in front of it) into shared memory: [raw + 16 - step .. raw + 16 + T * step) ----
  // The shared copy starts at the same address modulo 16 as the global bytes, so that all but the first and last few bytes
  // move as 16-byte vectors with every load of a thread in flight at once (word-wise copies: 22 dependent-looking loop
  // iterations per thread and 23 % of the kernel's stall samples on XYZIRT).
  uint8_t* pts = raw + ((step + 15u) & ~15u) + 16u;    // point 0 of the tile (moved below); the previous point sits in front of it
  if (full) {
    const uint8_t* g0 = F.in + static_cast<size_t>(tile_p0) * step;
    const uint32_t lead = chunk_start ? 0u : step;
    const uint8_t* g = g0 - lead;
    const uint32_t bytes = T * step + lead;
    pts += (static_cast<uint32_t>(reinterpret_cast<uintptr_t>(g)) - static_cast<uint32_t>(reinterpret_cast<uintptr_t>(pts - lead))) & 15u;
    uint8_t* s = pts - lead;
    const uint32_t head = min((16u - static_cast<uint32_t>(reinterpret_cast<uintptr_t>(g) & 15u)) & 15u, bytes);
    if (threadIdx.x < head) s[threadIdx.x] = g[threadIdx.x];
    const uint32_t nvec = (bytes - head) >> 4;
    const uint4* gv = reinterpret_cast<const uint4*>(g + head);
    uint4* sv = reinterpret_cast<uint4*>(s + head);
    for (uint32_t i = threadIdx.x; i < nvec; i += kPT) async_copy16(sv + i, gv + i);   // cp.async: no register round trip
    async_commit();
    const uint32_t done = head + 16u * nvec;
    if (threadIdx.x < bytes - done) s[done + threadIdx.x] = g[done + threadIdx.x];
    async_wait_all();
  }
  __syncthreads();

  uint32_t X[EP][NV];
  uint32_t mine = 0, tail4 = 0;
  bool fast = full;
  if (full) {
    const uint32_t p_local = threadIdx.x * EP;
    float trk = 0.0f;
    int32_t prev[NV];
    if (threadIdx.x == 0 && chunk_start) {
#pragma unroll
      for (int k = 0; k < NV; ++k) prev[k] = 0;
    } else {
      const SmemAddr pp = smem_addr(pts) + (static_cast<int32_t>(p_local) - 1) * static_cast<int32_t>(step);
#pragma unroll
      for (int k = 0; k < NV; ++k) {
        const float v = __uint_as_float(smem_load_u32<ALIGNED4>(pp, P.offset[k]));
        const float s = __fmul_rn(v, P.mul[k]);
        trk = max_nan(trk, fabsf(s));
        prev[k] = k < NF ? __float2int_rn(s) : __float2int_rn(roundf(s));
      }
    }
    uint32_t nbl[3] = {0, 0, 0};
#pragma unroll
    for (int j = 0; j < EP; ++j) {
      const SmemAddr pt = smem_addr(pts) + (p_local + j) * step;
#pragma unroll
      for (int k = 0; k < NV; ++k) {
        const float v = __uint_as_float(smem_load_u32<ALIGNED4>(pt, P.offset[k]));
        const float s = __fmul_rn(v, P.mul[k]);                 // IEEE RN product, never contracted
        trk = max_nan(trk, fabsf(s));
        // FloatN: cvtps2dq, ties to even. Scalar: static_cast<int64_t>(std::round(s)), half away from zero; identical to
        // the 64-bit value while |s| < 2^25 (checked below)
        const int32_t q = k < NF ? __float2int_rn(s) : __float2int_rn(roundf(s));
        const uint32_t d = static_cast<uint32_t>(q) - static_cast<uint32_t>(prev[k]);
        prev[k] = q;
        const uint32_t zz1 = ((d << 1) ^ static_cast<uint32_t>(static_cast<int32_t>(d) >> 31)) + 1u;
        uint32_t x = (zz1 & 0xFFFFC000u) * 3u + zz1;
        x = x + (x & 0x3F803F80u);
        const uint32_t b = top_bit(x);
        x |= low_mask(b) & 0x00808080u;
        X[j][k] = x;
        mine += b >> 3;
        // bit lengths of my last three values (for the tail word)
        if (j * NV + k >= EP * NV - 3) nbl[j * NV + k - (EP * NV - 3)] = (b & 0x18u) + 8u;
      }
    }
    mine += EP * NV;
    {
      constexpr int last = EP * NV - 1;
      tail4 = __funnelshift_rc(tail4, X[(last - 2) / NV][(last - 2) % NV], nbl[0]);
      tail4 = __funnelshift_rc(tail4, X[(last - 1) / NV][(last - 1) % NV], nbl[1]);
      tail4 = __funnelshift_rc(tail4, X[last / NV][last % NV], nbl[2]);
    }
    fast = trk < 33554432.0f;  // 2^25; false for NaN
  }
  // ---- offsets: warp scan + warp totals ----
  uint32_t inc = mine;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const uint32_t up = __shfl_up_sync(0xffffffffu, inc, d);
    if (lane >= static_cast<uint32_t>(d)) inc += up;
  }
  uint32_t ptail = __shfl_up_sync(0xffffffffu, tail4, 1);
  if (lane == 31) { s_wtot[warp] = inc; s_wtail[warp] = tail4; }
  const int any_slow = __syncthreads_or(fast ? 0 : 1);  // also: everybody is done with the raw tile bytes
  uint32_t total = 0;
  LookbackPoll lb;
  if (!any_slow) {
    uint32_t wbase = 0;
#pragma unroll
    for (int w = 0; w < kPT / 32; ++w) {
      const uint32_t c = s_wtot[w];
      if (static_cast<uint32_t>(w) < warp) wbase += c;
      total += c;
    }
    if (warp == 0) {
      lb.begin(L.status, F.tile_begin, tile, L.epoch, total);
      lb.issue(L.status, F.tile_begin, L.epoch);
    }
    if (lane == 0) ptail = warp > 0 ? s_wtail[warp - 1] : 0u;
    const uint32_t off = wbase + inc - mine;
    uint32_t bit = 8u * off;
    uint32_t lo = __funnelshift_rc(ptail, 0u, 32u - (bit & 31u));
    uint32_t wa = (bit >> 3) & ~3u;
#pragma unroll
    for (int j = 0; j < EP; ++j) {
#pragma unroll
      for (int k = 0; k < NV; ++k) {
        const uint32_t x = X[j][k];
        const uint32_t b = top_bit(x);
        lo |= __funnelshift_l(0u, x, bit);
        const uint32_t hi = __funnelshift_l(x, 0u, bit);
        bit += (b & 0x18u) + 8u;
        const uint32_t wn = (bit >> 3) & ~3u;
        if (wn != wa) { *reinterpret_cast<uint32_t*>(stage + wa) = lo; lo = hi; }
        wa = wn;
      }
    }
    if (threadIdx.x == kPT - 1 && (bit & 31u) != 0u) *reinterpret_cast<uint32_t*>(stage + wa) = lo;
  } else {
    // exact path: the plan interpreter, point by point, from global memory (like encode_generic_kernel)
    uint32_t len[EP];
    uint32_t cnt = 0;
#pragma unroll 1
    for (int j = 0; j < EP; ++j) {
      const uint32_t p = tile_p0 + threadIdx.x * EP + j;
      len[j] = 0;
      if (p < F.n_points) {
        const uint8_t* pt = F.in + static_cast<size_t>(p) * step;
        const uint8_t* prevp = (p % kChunkPoints) ? pt - step : nullptr;
        CountSink cs;
        encode_point_ops(plan, pt, prevp, cs);
        len[j] = cs.n;
      }
      cnt += len[j];
    }
    uint32_t off = block_exclusive_scan_n<kPT>(cnt, s_scan, &total);
#pragma unroll 1
    for (int j = 0; j < EP; ++j) {
      const uint32_t p = tile_p0 + threadIdx.x * EP + j;
      if (p < F.n_points) {
        const uint8_t* pt = F.in + static_cast<size_t>(p) * step;
        const uint8_t* prevp = (p % kChunkPoints) ? pt - step : nullptr;
        ByteSink bs{stage + off};
        encode_point_ops(plan, pt, prevp, bs);
        off += len[j];
      }
    }
    if (warp == 0) lb.begin(L.status, F.tile_begin, tile, L.epoch, total);
  }
  if (warp == 0) {
    const uint64_t e = lb.finish(L.status, F.tile_begin, tile, L.epoch, total);
    if (lane == 0) s_excl = e;
  }
  __syncthreads();
  finish_tile<T>(L, F, fi, t, stage, total, s_excl);
}

// Plans this kernel takes: the regular stream is [one FloatN group] + scalar lossy FLOAT32 fields, 3..6 values per point,
// every multiplier positive and finite (so that |v * mul| < 2^25 implies a finite input).
static bool encode_points_applies(const Plan& plan, PointsParams* P) {
  const char* e = getenv("CLDN_B200_ENC_FAST");
  if (e && e[0] == '0') return false;
  if (plan.n_gorilla || plan.n_ops == 0 || plan.n_ops > 4) return false;
  // a FloatN group alone stays with encode_floatn_kernel, which reads its 12 / 16 bytes per point straight from global
  // memory: staging whole points first costs more than it saves there (C3, step 32: measured slower)
  if (plan.n_ops < 2) return false;
  uint32_t nv = 0;
  P->n_floatn = 0;
  for (uint32_t i = 0; i < plan.n_ops; ++i) {
    const RegOp& op = plan.ops[i];
    if (op.kind == OP_FLOATN && i == 0) {
      for (int l = 0; l < op.lanes; ++l) { P->offset[nv] = op.offset[l]; P->mul[nv] = op.enc_mul_f[l]; ++nv; }
      P->n_floatn = op.lanes;
    } else if (op.kind == OP_F32_LOSSY) {
      if (nv >= 6) return false;
      P->offset[nv] = op.offset[0]; P->mul[nv] = op.enc_mul_f[0]; ++nv;
    } else {
      return false;
    }
  }
  if (nv < 3 || nv > 6) return false;
  for (uint32_t k = 0; k < nv; ++k) {
    if (!(P->mul[k] > 0.0f) || P->mul[k] > 3.0e38f) return false;
  }
  for (uint32_t k = nv; k < 6; ++k) { P->offset[k] = 0; P->mul[k] = 1.0f; }
  P->point_step = plan.point_step;
  if (plan.point_step > 64) return false;                      // raw tile in shared memory: 128 x 8 x step bytes
  return true;
}
static uint32_t encode_points_values(const Plan& plan) {
  uint32_t nv = 0;
  for (uint32_t i = 0; i < plan.n_ops; ++i) nv += plan.ops[i].kind == OP_FLOATN ? plan.ops[i].lanes : 1u;
  return nv;
}
constexpr int kPointsWideEP = 4;   // points per thread for 5 / 6 values per point (8: 40-48 values in registers)
static uint32_t encode_points_tile(const Plan& plan) { return encode_points_values(plan) <= 4 ? kPT * 8 : kPT * kPointsWideEP; }

template <int NV, int EP, int NF>
static int launch_points_nf(const Plan& plan, const EncLaunch& L, const PointsParams& P, cudaStream_t stream) {
  constexpr uint32_t T = kPT * EP;
  const size_t raw = ((plan.point_step + 15u) & ~15u) + 32 + static_cast<size_t>(T) * plan.point_step + 32;
  const size_t stg = static_cast<size_t>(T) * plan.max_point_bytes + 64;
  const size_t smem = std::max(raw, stg);
  bool aligned4 = (plan.point_step & 3u) == 0u;
  for (int k = 0; k < NV; ++k) aligned4 = aligned4 && (P.offset[k] & 3u) == 0u;
  // (the shared copy keeps the global misalignment of the tile's first byte modulo 16; with a 4-byte aligned layout and
  //  16-byte aligned frames every field read is one aligned word; kEncAlignPerFrame launches take the unaligned reads,
  //  which are right at any alignment)
  aligned4 = aligned4 && (L.flags & kEncInputsAligned16);
  if (aligned4) {
    auto k = encode_points_fast_kernel<NV, EP, true, NF>;
    if (set_smem(k, smem) != cudaSuccess) return -1;
    k<<<L.n_tiles_total, kPT, smem, stream>>>(L, P);
  } else {
    auto k = encode_points_fast_kernel<NV, EP, false, NF>;
    if (set_smem(k, smem) != cudaSuccess) return -1;
    k<<<L.n_tiles_total, kPT, smem, stream>>>(L, P);
  }
  count_launch();
  return 1;
}

// the FloatN group has 0 (no leading group), 3 or 4 lanes and is followed by at least one scalar field
template <int NV, int EP>
static int launch_points_nv(const Plan& plan, const EncLaunch& L, const PointsParams& P, cudaStream_t stream) {
  if (P.n_floatn == 0) return launch_points_nf<NV, EP, 0>(plan, L, P, stream);
  if (P.n_floatn == 3) {
    if (NV >= 4) return launch_points_nf<NV, EP, NV >= 4 ? 3 : 0>(plan, L, P, stream);
  } else if (P.n_floatn == 4) {
    if (NV >= 5) return launch_points_nf<NV, EP, NV >= 5 ? 4 : 0>(plan, L, P, stream);
  }
  return -1;
}

static int launch_encode_points(const Plan& plan, const EncLaunch& L, const PointsParams& P, cudaStream_t stream) {
  switch (encode_points_values(plan)) {
    case 3: return launch_points_nv<3, 8>(plan, L, P, stream);
    case 4: return launch_points_nv<4, 8>(plan, L, P, stream);
    case 5: return launch_points_nv<5, kPointsWideEP>(plan, L, P, stream);
    default: return launch_points_nv<6, kPointsWideEP>(plan, L, P, stream);
  }
}

}  // namespace cldn
