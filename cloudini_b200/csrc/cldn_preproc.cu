// SURVEY.md §8(f) N3 — applyVizLossyPreprocessing (cloudini_lib/src/ros_msg_utils.cpp:249-341) on the device, directly
// in front of the encode launch: drop points with a non-finite coordinate, keep the FIRST point of every voxel
// (lround(v / res) per axis, 21 bits each), preserve the order and every byte of the survivors.
//
// Two kernels over a batch of strided PointCloud2 buffers of one layout (HBM-bound byte work, no tensor cores). A frame
// table gives every cloud its own blocks, tiles, table region and status words; a block finds its cloud once by binary
// search over the first blocks, so a single cloud is a batch of one through the same two launches.
//   viz_insert_kernel   one thread per point: quantise, pack the 63-bit voxel key (packVoxelKey21, :42-49), insert it in
//                       the cloud's open-addressing region (64-bit CAS on the key, atomicMin on the cloud-local index of
//                       the first point that produced it) and remember the slot. The reference's set is order-dependent
//                       only through "first occurrence wins", which min(index) reproduces exactly for any insertion order.
//   viz_compact_kernel  tile of 256 x PPT points of one cloud per CTA: survivor = finite && first[slot] == own index; CTA
//                       scan of the flags, decoupled look-back over the cloud's tiles (same status words as the encoder),
//                       survivors are gathered into shared memory at rank * point_step and leave with 16-byte coalesced
//                       stores; the cloud's last tile writes its survivor count.
// Algorithmic bytes per point: point_step read + 4 (slot) written/read + kept/n * point_step written. Workspace: 12 B per
// table slot, ceil(2n / 1024) * 1024 slots per cloud, plus the 4-byte slot: about 28 B per point of the batch. Blocks run
// in frame-major order, so the regions being probed at any moment are those of the few clouds in flight, which fit in L2
// for clouds up to ~2M points (50 MB of L2 on the H100) even when the whole batch's tables do not.
#include <cuda_runtime.h>
#include <math.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <new>
#include <vector>

#include "../../include/cloudini_b200_ros.h"
#include "cldn_device.cuh"
#include "cldn_kernels.h"

namespace cldn {

constexpr unsigned long long kEmptyVoxel = ~0ull;  // keys use 63 bits
constexpr uint32_t kNoSlot = 0xFFFFFFFFu;

__device__ __forceinline__ uint64_t pack_voxel_key21(int32_t qx, int32_t qy, int32_t qz) {  // ros_msg_utils.cpp:42-49
  const uint64_t kAxisMask = (1ull << 21) - 1ull;
  const int64_t kBias = 1ll << 20;
  const uint64_t ux = static_cast<uint64_t>(static_cast<int64_t>(qx) + kBias) & kAxisMask;
  const uint64_t uy = static_cast<uint64_t>(static_cast<int64_t>(qy) + kBias) & kAxisMask;
  const uint64_t uz = static_cast<uint64_t>(static_cast<int64_t>(qz) + kBias) & kAxisMask;
  return ux | (uy << 21) | (uz << 42);
}
__device__ __forceinline__ uint32_t mix_voxel_key(uint64_t k) {  // any avalanche works: the result does not depend on it
  k ^= k >> 33; k *= 0xff51afd7ed558ccdull; k ^= k >> 33; k *= 0xc4ceb9fe1a85ec53ull; k ^= k >> 33;
  return static_cast<uint32_t>(k);
}
__device__ __forceinline__ bool finite_f32(uint32_t bits) { return (bits & 0x7F800000u) != 0x7F800000u; }  // std::isfinite

// One cloud of a launch. Blocks and compaction tiles never straddle clouds; every cloud has its own table region and
// its own run of status words, and point indices are cloud-local, so each cloud is processed exactly as if alone.
struct VizFrame {
  const uint8_t* in;
  uint8_t* out;
  uint32_t n_points;
  uint32_t block_begin;          // first insert block (exclusive scan of ceil(n / kThreads))
  uint32_t tile_begin;           // first compaction tile (exclusive scan of ceil(n / tile points))
  uint32_t table_size;           // slots of the cloud's region, a multiple of 1024 and >= 2n
  uint64_t table_base;           // first slot of the region in keys / firsts
  uint64_t slot_base;            // first entry of the cloud in slots (points of the clouds before it)
};

struct VizLaunch {
  const VizFrame* frames;        // device; nullptr: a batch of one, whose frame is `one`
  VizFrame one;                  // (saves the table upload in front of every single-cloud call)
  uint32_t n_frames;
  uint32_t point_step, xyz_offset;
  float inv_res;                 // 1.0f / resolution (ros_msg_utils.cpp:272)
  unsigned long long* keys;      // voxel keys, kEmptyVoxel when free
  uint32_t* firsts;              // smallest cloud-local point index that produced the key
  uint32_t* slots;               // per point: table slot (region-local) of every finite point, kNoSlot for dropped ones
  uint64_t* status;              // tile status words of the compaction look-back
  uint32_t epoch;
  uint32_t ppt;                  // points per thread of the compaction tiles
  uint32_t staged;               // 1: survivors are gathered in shared memory (tile bytes fit), 0: direct copies
  uint32_t* kept;                // per cloud: number of survivors
};

// Last cloud whose first block (tile) is <= b: empty clouds share their first block with the next one.
template <uint32_t VizFrame::*Begin>
__device__ __forceinline__ uint32_t find_viz_frame(const VizFrame* __restrict__ frames, uint32_t n_frames, uint32_t b) {
  uint32_t lo = 0, hi = n_frames - 1;
  while (lo < hi) {
    const uint32_t mid = (lo + hi + 1) >> 1;
    if (frames[mid].*Begin <= b) lo = mid; else hi = mid - 1;
  }
  return lo;
}

__global__ void __launch_bounds__(kThreads) viz_insert_kernel(VizLaunch L) {
  const VizFrame F = L.frames ? L.frames[find_viz_frame<&VizFrame::block_begin>(L.frames, L.n_frames, blockIdx.x)] : L.one;
  const uint32_t i = (blockIdx.x - F.block_begin) * kThreads + threadIdx.x;
  const uint32_t n = F.n_points;
  if (i >= n) return;
  uint32_t* slots = L.slots + F.slot_base;
  const uint8_t* p = F.in + static_cast<size_t>(i) * L.point_step + L.xyz_offset;
  const uint32_t bx = load_u32(p), by = load_u32(p + 4), bz = load_u32(p + 8);
  if (!finite_f32(bx) || !finite_f32(by) || !finite_f32(bz)) { slots[i] = kNoSlot; return; }  // :311-313
  // static_cast<int32_t>(std::lround(f * inv_res)) (:314-317): half away from zero in 64 bits, low 32 bits kept
  const int32_t qx = static_cast<int32_t>(quant_i64_f32(__uint_as_float(bx), L.inv_res));
  const int32_t qy = static_cast<int32_t>(quant_i64_f32(__uint_as_float(by), L.inv_res));
  const int32_t qz = static_cast<int32_t>(quant_i64_f32(__uint_as_float(bz), L.inv_res));
  const unsigned long long key = pack_voxel_key21(qx, qy, qz);
  unsigned long long* keys = L.keys + F.table_base;
  const uint32_t size = F.table_size;
  uint32_t h = static_cast<uint32_t>((static_cast<uint64_t>(mix_voxel_key(key)) * size) >> 32);  // multiply-shift range
  while (true) {
    const unsigned long long old = atomicCAS(&keys[h], kEmptyVoxel, key);
    if (old == kEmptyVoxel || old == key) break;
    h = (h + 1u == size) ? 0u : h + 1u;
  }
  atomicMin(&L.firsts[F.table_base + h], i);
  slots[i] = h;
}

__global__ void __launch_bounds__(kThreads) viz_compact_kernel(VizLaunch L) {
  extern __shared__ __align__(16) uint8_t dyn_smem[];
  __shared__ uint32_t s_scan[kThreads / 32 + 1];
  __shared__ unsigned long long s_excl;
  const uint32_t fi = L.frames ? find_viz_frame<&VizFrame::tile_begin>(L.frames, L.n_frames, blockIdx.x) : 0u;
  const VizFrame F = L.frames ? L.frames[fi] : L.one;
  const uint32_t tile_points = kThreads * L.ppt;
  const uint32_t n = F.n_points;
  const uint32_t tile = blockIdx.x - F.tile_begin;
  const uint32_t* slots = L.slots + F.slot_base;
  const uint32_t* firsts = L.firsts + F.table_base;
  const uint8_t* in = F.in;
  uint8_t* out = F.out;
  const uint32_t p0 = tile * tile_points + threadIdx.x * L.ppt;  // blocked: thread t owns ppt consecutive points
  uint32_t keep_mask = 0, mine = 0;
  for (uint32_t j = 0; j < L.ppt; ++j) {
    const uint32_t i = p0 + j;
    if (i < n) {
      const uint32_t s = slots[i];
      if (s != kNoSlot && firsts[s] == i) { keep_mask |= 1u << j; ++mine; }  // first occurrence of its voxel (:318-320)
    }
  }
  uint32_t total = 0;
  const uint32_t rank0 = block_exclusive_scan(mine, s_scan, &total);
  if (threadIdx.x < 32) {
    const uint64_t excl = tile_lookback(L.status, F.tile_begin, blockIdx.x, L.epoch, total);
    if (threadIdx.x == 0) {
      s_excl = excl;
      if ((tile + 1) * static_cast<uint64_t>(tile_points) >= n) L.kept[fi] = static_cast<uint32_t>(excl + total);  // last tile
    }
  }
  const uint32_t step = L.point_step;
  const bool words = ((reinterpret_cast<uintptr_t>(in) | reinterpret_cast<uintptr_t>(out) | step) & 3u) == 0;
  if (L.staged) {
    uint32_t r = rank0;
    for (uint32_t j = 0; j < L.ppt; ++j) {
      if (!((keep_mask >> j) & 1u)) continue;
      const uint8_t* src = in + static_cast<size_t>(p0 + j) * step;
      uint8_t* dst = dyn_smem + static_cast<size_t>(r) * step;
      if (words) {
        for (uint32_t b = 0; b < step; b += 4) *reinterpret_cast<uint32_t*>(dst + b) = *reinterpret_cast<const uint32_t*>(src + b);
      } else {
        for (uint32_t b = 0; b < step; ++b) dst[b] = src[b];
      }
      ++r;
    }
    __syncthreads();  // staging complete, s_excl visible
    copy_stage_to_global(dyn_smem, total * step, out + static_cast<size_t>(s_excl) * step);
  } else {
    __syncthreads();
    uint64_t r = s_excl + rank0;
    for (uint32_t j = 0; j < L.ppt; ++j) {
      if (!((keep_mask >> j) & 1u)) continue;
      const uint8_t* src = in + static_cast<size_t>(p0 + j) * step;
      uint8_t* dst = out + r * step;
      if (words) {
        for (uint32_t b = 0; b < step; b += 4) *reinterpret_cast<uint32_t*>(dst + b) = *reinterpret_cast<const uint32_t*>(src + b);
      } else {
        for (uint32_t b = 0; b < step; ++b) dst[b] = src[b];
      }
      ++r;
    }
  }
}

}  // namespace cldn

using namespace cldn;

namespace {
template <typename T>
struct Buf {
  T* p = nullptr;
  size_t cap = 0;
  bool reserve(size_t n, bool zero = false) {
    if (n <= cap) return true;
    if (p) cudaFree(p);
    p = nullptr; cap = 0;
    const size_t want = std::max<size_t>(n + n / 4, 64);
    if (cudaMalloc(reinterpret_cast<void**>(&p), want * sizeof(T)) != cudaSuccess) return false;
    cap = want;
    // the handle's stream is non-blocking (it does not order itself after the legacy stream the memset runs on)
    if (zero && (cudaMemset(p, 0, want * sizeof(T)) != cudaSuccess || cudaDeviceSynchronize() != cudaSuccess)) return false;
    return true;
  }
  void release() { if (p) cudaFree(p); p = nullptr; cap = 0; }
};
template <typename T>
struct PinnedBuf {
  T* p = nullptr;
  size_t cap = 0;
  bool reserve(size_t n) {
    if (n <= cap) return true;
    if (p) cudaFreeHost(p);
    p = nullptr; cap = 0;
    const size_t want = std::max<size_t>(n, 16);
    if (cudaMallocHost(reinterpret_cast<void**>(&p), want * sizeof(T)) != cudaSuccess) return false;
    cap = want;
    return true;
  }
  void release() { if (p) cudaFreeHost(p); p = nullptr; cap = 0; }
};

// Table slots of a cloud of n points: a multiple of 1024 that is at least 2n (load factor <= 1/2). The output does not
// depend on the size or the hash, only on the table holding every distinct voxel.
uint32_t viz_table_size(uint32_t n) { return ((2u * n + 1023u) / 1024u) * 1024u; }
}  // namespace

struct cldn_preproc {
  int device = 0;
  cudaStream_t stream = nullptr;
  bool own_stream = false;
  uint32_t epoch = 0;
  Buf<uint8_t> table;  // keys (8 B per slot) of every cloud's region, then firsts (4 B per slot)
  Buf<uint32_t> slots, kept;
  Buf<uint64_t> status;
  Buf<VizFrame> frames;
  Buf<uint8_t> d_in, d_out;
  PinnedBuf<VizFrame> h_frames;
  PinnedBuf<uint32_t> h_kept;
};

#define PP_CUDA(expr)                                                                                          \
  do {                                                                                                         \
    cudaError_t e__ = (expr);                                                                                  \
    if (e__ != cudaSuccess) {                                                                                  \
      set_error("CUDA error %s at %s:%d: %s", cudaGetErrorName(e__), __FILE__, __LINE__, cudaGetErrorString(e__)); \
      return CLDN_ERR_CUDA;                                                                                    \
    }                                                                                                          \
  } while (0)

// applyVizLossyPreprocessing on n_frames clouds of one layout: every cloud is checked first (in the single call's order),
// then one insert and one compact launch cover every cloud, then one read-back of the survivor counts. `name_frames`
// prefixes a frame's message with "frame <f>: " (the batch API); the single call reports it as it is.
static int viz_frames(cldn_preproc_t* pp, const cldn_info_t* info, size_t n_frames, const void* const* clouds,
                      const size_t* cloud_bytes, void* const* outs, const size_t* out_capacities, size_t* kept_points,
                      int* applied, cldn_info_t* infos_out, int mem, bool name_frames) {
  for (size_t f = 0; f < n_frames; ++f) {
    applied[f] = 0;
    kept_points[f] = info->point_step ? cloud_bytes[f] / info->point_step : 0;  // :274
    if (infos_out) infos_out[f] = *info;
  }
  // ---- the reference's early returns: nothing is modified (ros_msg_utils.cpp:250-278) ----
  bool noop = info->n_fields < 3 || info->point_step == 0;
  float xyz_res = 0.0f;
  uint32_t xyz_offset = 0;
  if (!noop) {
    const cldn_field_t &f0 = info->fields[0], &f1 = info->fields[1], &f2 = info->fields[2];
    const bool has_triple = f0.type == CLDN_FLOAT32 && f1.type == CLDN_FLOAT32 && f2.type == CLDN_FLOAT32 && f0.has_resolution &&
                            f1.has_resolution && f2.has_resolution && f0.resolution == f1.resolution &&
                            f0.resolution == f2.resolution && f1.offset == f0.offset + 4u && f2.offset == f0.offset + 8u;
    xyz_res = f0.resolution;
    xyz_offset = f0.offset;
    noop = !has_triple || !(xyz_res > 0.0f) || !isfinite(xyz_res);
  }
  auto fail = [&](size_t f, int rc, const char* msg) {
    if (name_frames) set_error("frame %zu: %s", f, msg);
    else set_error("%s", msg);
    return rc;
  };
  const uint32_t step = info->point_step;
  uint64_t total_points = 0, blocks = 0, tiles = 0, table = 0;
  uint32_t ppt = 8;
  while (ppt > 1 && static_cast<size_t>(kThreads) * ppt * step > (64u << 10)) ppt >>= 1;
  const bool staged = static_cast<size_t>(kThreads) * ppt * step <= (200u << 10);
  const uint32_t tile_points = kThreads * ppt;
  for (size_t f = 0; f < n_frames; ++f) {
    if (!clouds[f] && cloud_bytes[f]) return fail(f, CLDN_ERR_INVALID_ARGUMENT, "null argument");
    if (noop) continue;
    const size_t n_in = kept_points[f];
    if (n_in == 0) continue;
    // ---- from here on the cloud is rewritten ----
    if (n_in > (1u << 30)) return fail(f, CLDN_ERR_UNSUPPORTED, "viz preprocessing: more than 2^30 points in one cloud");
    if (static_cast<uint64_t>(xyz_offset) + 12u > step) return fail(f, CLDN_ERR_INVALID_ARGUMENT, "xyz fields lie outside the point");
    if (!outs[f] || out_capacities[f] < n_in * step) {
      return fail(f, CLDN_ERR_BUFFER_TOO_SMALL, "viz preprocessing: output buffer smaller than the input cloud");
    }
    total_points += n_in;
    blocks += (n_in + kThreads - 1) / kThreads;
    tiles += (n_in + tile_points - 1) / tile_points;
    table += viz_table_size(static_cast<uint32_t>(n_in));
  }
  if (total_points == 0) return CLDN_OK;
  if (blocks > 0x7FFFFFFFull || tiles > 0x7FFFFFFFull) return fail(0, CLDN_ERR_UNSUPPORTED, "viz preprocessing: batch too large");
  PP_CUDA(cudaSetDevice(pp->device));
  if (!pp->table.reserve(table * 12) || !pp->slots.reserve(total_points) || !pp->status.reserve(tiles, true) ||
      !pp->kept.reserve(n_frames) || !pp->frames.reserve(n_frames) || !pp->h_frames.reserve(n_frames) ||
      !pp->h_kept.reserve(n_frames)) {
    set_error("device allocation failed");
    return CLDN_ERR_CUDA;
  }
  std::vector<size_t> in_at(n_frames, 0), out_at(n_frames, 0);
  if (mem == CLDN_MEM_HOST) {  // staging: every cloud at a 256-byte-aligned offset
    size_t in_total = 0, out_total = 0;
    for (size_t f = 0; f < n_frames; ++f) {
      const size_t bytes = noop ? 0 : kept_points[f] * step;
      in_at[f] = in_total;
      out_at[f] = out_total;
      in_total += (bytes + 255) & ~size_t(255);
      out_total += (bytes + 255) & ~size_t(255);
    }
    if (!pp->d_in.reserve(in_total + 256) || !pp->d_out.reserve(out_total + 256)) { set_error("device allocation failed"); return CLDN_ERR_CUDA; }
  }
  VizFrame* hf = pp->h_frames.p;
  uint64_t b = 0, t = 0, tb = 0, sb = 0;
  for (size_t f = 0; f < n_frames; ++f) {
    const uint32_t n = static_cast<uint32_t>(kept_points[f]);
    VizFrame& F = hf[f];
    F.in = static_cast<const uint8_t*>(clouds[f]);
    F.out = static_cast<uint8_t*>(outs[f]);
    if (mem == CLDN_MEM_HOST) {
      F.in = pp->d_in.p + in_at[f];
      F.out = pp->d_out.p + out_at[f];
      if (n) PP_CUDA(cudaMemcpyAsync(pp->d_in.p + in_at[f], clouds[f], static_cast<size_t>(n) * step, cudaMemcpyHostToDevice, pp->stream));
    }
    F.n_points = n;
    F.block_begin = static_cast<uint32_t>(b);
    F.tile_begin = static_cast<uint32_t>(t);
    F.table_size = n ? viz_table_size(n) : 0;
    F.table_base = tb;
    F.slot_base = sb;
    b += (n + kThreads - 1) / kThreads;
    t += (n + tile_points - 1) / tile_points;
    tb += F.table_size;
    sb += n;
  }
  if (n_frames > 1) PP_CUDA(cudaMemcpyAsync(pp->frames.p, hf, n_frames * sizeof(VizFrame), cudaMemcpyHostToDevice, pp->stream));
  pp->epoch = (pp->epoch + 1) & 0x3FFFFFu;  // the status words keep 22 bits of it
  if (pp->epoch == 0) {  // wrapped: words zeroed at allocation would read as this launch's
    PP_CUDA(cudaMemsetAsync(pp->status.p, 0, pp->status.cap * sizeof(uint64_t), pp->stream));
    pp->epoch = 1;
  }
  VizLaunch L;
  L.frames = n_frames > 1 ? pp->frames.p : nullptr;
  L.one = hf[0];
  L.n_frames = static_cast<uint32_t>(n_frames);
  L.point_step = step; L.xyz_offset = xyz_offset;
  L.inv_res = 1.0f / xyz_res;
  L.keys = reinterpret_cast<unsigned long long*>(pp->table.p);
  L.firsts = reinterpret_cast<uint32_t*>(pp->table.p + table * 8);
  L.slots = pp->slots.p;
  L.status = pp->status.p; L.epoch = pp->epoch; L.ppt = ppt; L.staged = staged ? 1u : 0u; L.kept = pp->kept.p;
  PP_CUDA(cudaMemsetAsync(pp->table.p, 0xFF, table * 12, pp->stream));  // keys empty, firsts "no point yet"
  viz_insert_kernel<<<static_cast<uint32_t>(blocks), kThreads, 0, pp->stream>>>(L);
  const size_t smem = staged ? static_cast<size_t>(tile_points) * step + 32 : 0;
  PP_CUDA(raise_smem_limit(viz_compact_kernel, smem));
  viz_compact_kernel<<<static_cast<uint32_t>(tiles), kThreads, smem, pp->stream>>>(L);
  count_launch(2);
  PP_CUDA(cudaGetLastError());
  PP_CUDA(cudaMemcpyAsync(pp->h_kept.p, pp->kept.p, n_frames * sizeof(uint32_t), cudaMemcpyDeviceToHost, pp->stream));
  PP_CUDA(cudaStreamSynchronize(pp->stream));
  bool copied = false;
  for (size_t f = 0; f < n_frames; ++f) {
    if (hf[f].n_points == 0) continue;  // an empty cloud is a no-op (:276-278)
    const size_t kept = pp->h_kept.p[f];
    if (mem == CLDN_MEM_HOST && kept) {
      PP_CUDA(cudaMemcpyAsync(outs[f], pp->d_out.p + out_at[f], kept * step, cudaMemcpyDeviceToHost, pp->stream));
      copied = true;
    }
    kept_points[f] = kept;
    applied[f] = 1;
    if (infos_out) {  // pc_info bookkeeping (:327-340)
      cldn_info_t& o = infos_out[f];
      o.width = static_cast<uint32_t>(kept);
      o.height = 1;
      for (uint32_t i = 0; i < o.n_fields; ++i) {
        if (o.fields[i].type == CLDN_FLOAT64 && !o.fields[i].has_resolution) {
          o.fields[i].has_resolution = 1;
          o.fields[i].resolution = 1e-6f;
        }
      }
    }
  }
  if (copied) PP_CUDA(cudaStreamSynchronize(pp->stream));
  return CLDN_OK;
}

extern "C" {

int cldn_b200_preproc_create(int device, void* stream, cldn_preproc_t** out) {
  if (!out) { set_error("null argument"); return CLDN_ERR_INVALID_ARGUMENT; }
  *out = nullptr;
  int count = 0;
  if (cudaGetDeviceCount(&count) != cudaSuccess || count == 0) {
    set_error("no CUDA device: cloudini_b200 has no CPU fallback");
    return CLDN_ERR_CUDA;
  }
  if (device >= 0) PP_CUDA(cudaSetDevice(device));
  cldn_preproc* pp = new cldn_preproc();
  cudaGetDevice(&pp->device);
  if (stream) {
    pp->stream = static_cast<cudaStream_t>(stream);
  } else if (cudaStreamCreateWithFlags(&pp->stream, cudaStreamNonBlocking) == cudaSuccess) {
    pp->own_stream = true;
  } else {
    set_error("cudaStreamCreate failed");
    delete pp;
    return CLDN_ERR_CUDA;
  }
  if (!pp->h_kept.reserve(1) || !pp->kept.reserve(1, true)) {
    set_error("allocation failed");
    cldn_b200_preproc_destroy(pp);
    return CLDN_ERR_CUDA;
  }
  *out = pp;
  return CLDN_OK;
}

void cldn_b200_preproc_destroy(cldn_preproc_t* pp) {
  if (!pp) return;
  cudaSetDevice(pp->device);
  if (pp->stream) cudaStreamSynchronize(pp->stream);
  pp->table.release(); pp->slots.release(); pp->kept.release(); pp->status.release(); pp->frames.release();
  pp->d_in.release(); pp->d_out.release();
  pp->h_frames.release(); pp->h_kept.release();
  if (pp->own_stream && pp->stream) cudaStreamDestroy(pp->stream);
  delete pp;
}

int cldn_b200_viz_lossy_preprocess(cldn_preproc_t* pp, cldn_info_t* info, const void* cloud, size_t cloud_bytes, void* out,
                                   size_t out_capacity, size_t* kept_points, int* applied, int mem) {
  if (!pp || !info || (!cloud && cloud_bytes)) { set_error("null argument"); return CLDN_ERR_INVALID_ARGUMENT; }
  if (mem != CLDN_MEM_HOST && mem != CLDN_MEM_DEVICE) { set_error("bad memory kind"); return CLDN_ERR_INVALID_ARGUMENT; }
  size_t kept = 0;
  int done = 0;
  cldn_info_t after;
  int rc;
  try {
    rc = viz_frames(pp, info, 1, &cloud, &cloud_bytes, &out, &out_capacity, &kept, &done, &after, mem, false);
  } catch (const std::bad_alloc&) {
    set_error("out of memory");
    rc = CLDN_ERR_INTERNAL;
  }
  if (kept_points) *kept_points = kept;
  if (applied) *applied = done;
  if (rc == CLDN_OK && done) *info = after;
  return rc;
}

int cldn_b200_viz_lossy_preprocess_batch(cldn_preproc_t* pp, const cldn_info_t* info, size_t n_frames,
                                         const void* const* clouds, const size_t* cloud_bytes, void* const* outs,
                                         const size_t* out_capacities, size_t* kept_points, int* applied,
                                         cldn_info_t* infos_out, int mem) {
  if (!pp || !info || (n_frames && (!clouds || !cloud_bytes || !outs || !out_capacities || !kept_points || !applied))) {
    set_error("null argument");
    return CLDN_ERR_INVALID_ARGUMENT;
  }
  if (mem != CLDN_MEM_HOST && mem != CLDN_MEM_DEVICE) { set_error("bad memory kind"); return CLDN_ERR_INVALID_ARGUMENT; }
  try {
    return viz_frames(pp, info, n_frames, clouds, cloud_bytes, outs, out_capacities, kept_points, applied, infos_out, mem, true);
  } catch (const std::bad_alloc&) {
    set_error("out of memory");
    return CLDN_ERR_INTERNAL;
  }
}

}  // extern "C"
