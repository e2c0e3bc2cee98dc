// SURVEY.md §8(f) N3 — applyVizLossyPreprocessing (cloudini_lib/src/ros_msg_utils.cpp:249-341) on the device, directly
// in front of the encode launch: drop points with a non-finite coordinate, keep the FIRST point of every voxel
// (lround(v / res) per axis, 21 bits each), preserve the order and every byte of the survivors.
//
// Two kernels over the strided PointCloud2 buffer (HBM-bound byte work, no tensor cores):
//   viz_insert_kernel   one thread per point: quantise, pack the 63-bit voxel key (packVoxelKey21, :42-49), insert it in
//                       an open-addressing table (64-bit CAS on the key, atomicMin on the index of the first point that
//                       produced it) and remember the slot. The reference's set is order-dependent only through "first
//                       occurrence wins", which min(index) reproduces exactly for any insertion order.
//   viz_compact_kernel  tile of 256 x PPT points per CTA: survivor = finite && first[slot] == own index; CTA scan of
//                       the flags, decoupled look-back over the tiles (same status words as the encoder), survivors are
//                       gathered into shared memory at rank * point_step and leave with 16-byte coalesced stores.
// Algorithmic bytes per point: point_step read + 4 (slot) written/read + kept/n * point_step written; the table
// (12 B per slot, 2 slots per point) lives in L2 for frames up to ~4M points.
#include <cuda_runtime.h>
#include <math.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>

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

struct VizLaunch {
  const uint8_t* in;
  uint8_t* out;
  uint32_t n_points, point_step, xyz_offset;
  float inv_res;                 // 1.0f / resolution (ros_msg_utils.cpp:272)
  unsigned long long* keys;      // [capacity] voxel keys, kEmptyVoxel when free
  uint32_t* firsts;              // [capacity] smallest point index that produced the key
  uint32_t mask;                 // capacity - 1 (power of two)
  uint32_t* slots;               // [n_points] table slot of every finite point, kNoSlot for dropped ones
  uint64_t* status;              // tile status words of the compaction look-back
  uint32_t epoch;
  uint32_t ppt;                  // points per thread of the compaction tiles
  uint32_t staged;               // 1: survivors are gathered in shared memory (tile bytes fit), 0: direct copies
  uint32_t* kept;                // total number of survivors
};

__global__ void __launch_bounds__(kThreads) viz_insert_kernel(VizLaunch L) {
  const uint32_t i = blockIdx.x * kThreads + threadIdx.x;
  if (i >= L.n_points) return;
  const uint8_t* p = L.in + static_cast<size_t>(i) * L.point_step + L.xyz_offset;
  const uint32_t bx = load_u32(p), by = load_u32(p + 4), bz = load_u32(p + 8);
  if (!finite_f32(bx) || !finite_f32(by) || !finite_f32(bz)) { L.slots[i] = kNoSlot; return; }  // :311-313
  // static_cast<int32_t>(std::lround(f * inv_res)) (:314-317): half away from zero in 64 bits, low 32 bits kept
  const int32_t qx = static_cast<int32_t>(quant_i64_f32(__uint_as_float(bx), L.inv_res));
  const int32_t qy = static_cast<int32_t>(quant_i64_f32(__uint_as_float(by), L.inv_res));
  const int32_t qz = static_cast<int32_t>(quant_i64_f32(__uint_as_float(bz), L.inv_res));
  const unsigned long long key = pack_voxel_key21(qx, qy, qz);
  uint32_t h = mix_voxel_key(key) & L.mask;
  while (true) {
    const unsigned long long old = atomicCAS(&L.keys[h], kEmptyVoxel, key);
    if (old == kEmptyVoxel || old == key) break;
    h = (h + 1u) & L.mask;
  }
  atomicMin(&L.firsts[h], i);
  L.slots[i] = h;
}

__global__ void __launch_bounds__(kThreads) viz_compact_kernel(VizLaunch L) {
  extern __shared__ __align__(16) uint8_t dyn_smem[];
  __shared__ uint32_t s_scan[kThreads / 32 + 1];
  __shared__ unsigned long long s_excl;
  const uint32_t tile_points = kThreads * L.ppt;
  const uint32_t tile = blockIdx.x;
  const uint32_t p0 = tile * tile_points + threadIdx.x * L.ppt;  // blocked: thread t owns ppt consecutive points
  uint32_t keep_mask = 0, mine = 0;
  for (uint32_t j = 0; j < L.ppt; ++j) {
    const uint32_t i = p0 + j;
    if (i < L.n_points) {
      const uint32_t s = L.slots[i];
      if (s != kNoSlot && L.firsts[s] == i) { keep_mask |= 1u << j; ++mine; }  // first occurrence of its voxel (:318-320)
    }
  }
  uint32_t total = 0;
  const uint32_t rank0 = block_exclusive_scan(mine, s_scan, &total);
  if (threadIdx.x < 32) {
    const uint64_t excl = tile_lookback(L.status, 0u, tile, L.epoch, total);
    if (threadIdx.x == 0) {
      s_excl = excl;
      if (tile == gridDim.x - 1) *L.kept = static_cast<uint32_t>(excl + total);
    }
  }
  const uint32_t step = L.point_step;
  const bool words = ((reinterpret_cast<uintptr_t>(L.in) | reinterpret_cast<uintptr_t>(L.out) | step) & 3u) == 0;
  if (L.staged) {
    uint32_t r = rank0;
    for (uint32_t j = 0; j < L.ppt; ++j) {
      if (!((keep_mask >> j) & 1u)) continue;
      const uint8_t* src = L.in + static_cast<size_t>(p0 + j) * step;
      uint8_t* dst = dyn_smem + static_cast<size_t>(r) * step;
      if (words) {
        for (uint32_t b = 0; b < step; b += 4) *reinterpret_cast<uint32_t*>(dst + b) = *reinterpret_cast<const uint32_t*>(src + b);
      } else {
        for (uint32_t b = 0; b < step; ++b) dst[b] = src[b];
      }
      ++r;
    }
    __syncthreads();  // staging complete, s_excl visible
    copy_stage_to_global(dyn_smem, total * step, L.out + static_cast<size_t>(s_excl) * step);
  } else {
    __syncthreads();
    uint64_t r = s_excl + rank0;
    for (uint32_t j = 0; j < L.ppt; ++j) {
      if (!((keep_mask >> j) & 1u)) continue;
      const uint8_t* src = L.in + static_cast<size_t>(p0 + j) * step;
      uint8_t* dst = L.out + r * step;
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
}  // namespace

struct cldn_preproc {
  int device = 0;
  cudaStream_t stream = nullptr;
  bool own_stream = false;
  uint32_t epoch = 0;
  Buf<unsigned long long> keys;
  Buf<uint32_t> firsts, slots, kept;
  Buf<uint64_t> status;
  Buf<uint8_t> d_in, d_out;
  uint32_t* h_kept = nullptr;  // pinned
};

#define PP_CUDA(expr)                                                                                          \
  do {                                                                                                         \
    cudaError_t e__ = (expr);                                                                                  \
    if (e__ != cudaSuccess) {                                                                                  \
      set_error("CUDA error %s at %s:%d: %s", cudaGetErrorName(e__), __FILE__, __LINE__, cudaGetErrorString(e__)); \
      return CLDN_ERR_CUDA;                                                                                    \
    }                                                                                                          \
  } while (0)

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
  if (cudaMallocHost(reinterpret_cast<void**>(&pp->h_kept), sizeof(uint32_t)) != cudaSuccess || !pp->kept.reserve(1, true)) {
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
  pp->keys.release(); pp->firsts.release(); pp->slots.release(); pp->kept.release(); pp->status.release();
  pp->d_in.release(); pp->d_out.release();
  if (pp->h_kept) cudaFreeHost(pp->h_kept);
  if (pp->own_stream && pp->stream) cudaStreamDestroy(pp->stream);
  delete pp;
}

int cldn_b200_viz_lossy_preprocess(cldn_preproc_t* pp, cldn_info_t* info, const void* cloud, size_t cloud_bytes, void* out,
                                   size_t out_capacity, size_t* kept_points, int* applied, int mem) {
  if (!pp || !info || (!cloud && cloud_bytes)) { set_error("null argument"); return CLDN_ERR_INVALID_ARGUMENT; }
  if (mem != CLDN_MEM_HOST && mem != CLDN_MEM_DEVICE) { set_error("bad memory kind"); return CLDN_ERR_INVALID_ARGUMENT; }
  if (applied) *applied = 0;
  const size_t n_in = info->point_step ? cloud_bytes / info->point_step : 0;  // :274
  if (kept_points) *kept_points = n_in;
  // ---- the reference's early returns: nothing is modified (ros_msg_utils.cpp:250-278) ----
  if (info->n_fields < 3 || info->point_step == 0) return CLDN_OK;
  const cldn_field_t &f0 = info->fields[0], &f1 = info->fields[1], &f2 = info->fields[2];
  const bool has_triple = f0.type == CLDN_FLOAT32 && f1.type == CLDN_FLOAT32 && f2.type == CLDN_FLOAT32 && f0.has_resolution &&
                          f1.has_resolution && f2.has_resolution && f0.resolution == f1.resolution &&
                          f0.resolution == f2.resolution && f1.offset == f0.offset + 4u && f2.offset == f0.offset + 8u;
  if (!has_triple) return CLDN_OK;
  const float xyz_res = f0.resolution;
  if (!(xyz_res > 0.0f) || !isfinite(xyz_res)) return CLDN_OK;
  if (n_in == 0) return CLDN_OK;
  // ---- from here on the cloud is rewritten ----
  if (n_in > (1u << 30)) { set_error("viz preprocessing: more than 2^30 points in one cloud"); return CLDN_ERR_UNSUPPORTED; }
  if (static_cast<uint64_t>(f0.offset) + 12u > info->point_step) { set_error("xyz fields lie outside the point"); return CLDN_ERR_INVALID_ARGUMENT; }
  const size_t in_bytes = n_in * info->point_step;
  if (!out || out_capacity < in_bytes) { set_error("viz preprocessing: output buffer smaller than the input cloud"); return CLDN_ERR_BUFFER_TOO_SMALL; }
  PP_CUDA(cudaSetDevice(pp->device));
  const uint32_t n = static_cast<uint32_t>(n_in), step = info->point_step;
  uint32_t capacity = 1024;
  while (capacity < 2u * n) capacity <<= 1;
  uint32_t ppt = 8;
  while (ppt > 1 && static_cast<size_t>(kThreads) * ppt * step > (64u << 10)) ppt >>= 1;
  const bool staged = static_cast<size_t>(kThreads) * ppt * step <= (200u << 10);
  const uint32_t tile_points = kThreads * ppt, n_tiles = (n + tile_points - 1) / tile_points;
  if (!pp->keys.reserve(capacity) || !pp->firsts.reserve(capacity) || !pp->slots.reserve(n) || !pp->status.reserve(n_tiles, true)) {
    set_error("device allocation failed");
    return CLDN_ERR_CUDA;
  }
  const uint8_t* d_in = static_cast<const uint8_t*>(cloud);
  uint8_t* d_out = static_cast<uint8_t*>(out);
  if (mem == CLDN_MEM_HOST) {
    if (!pp->d_in.reserve(in_bytes) || !pp->d_out.reserve(in_bytes + 16)) { set_error("device allocation failed"); return CLDN_ERR_CUDA; }
    PP_CUDA(cudaMemcpyAsync(pp->d_in.p, cloud, in_bytes, cudaMemcpyHostToDevice, pp->stream));
    d_in = pp->d_in.p;
    d_out = pp->d_out.p;
  }
  VizLaunch L;
  L.in = d_in; L.out = d_out; L.n_points = n; L.point_step = step; L.xyz_offset = f0.offset;
  L.inv_res = 1.0f / xyz_res;
  L.keys = pp->keys.p; L.firsts = pp->firsts.p; L.mask = capacity - 1u; L.slots = pp->slots.p;
  L.status = pp->status.p; L.epoch = ++pp->epoch; L.ppt = ppt; L.staged = staged ? 1u : 0u; L.kept = pp->kept.p;
  PP_CUDA(cudaMemsetAsync(pp->keys.p, 0xFF, static_cast<size_t>(capacity) * sizeof(unsigned long long), pp->stream));
  PP_CUDA(cudaMemsetAsync(pp->firsts.p, 0xFF, static_cast<size_t>(capacity) * sizeof(uint32_t), pp->stream));
  viz_insert_kernel<<<(n + kThreads - 1) / kThreads, kThreads, 0, pp->stream>>>(L);
  const size_t smem = staged ? static_cast<size_t>(tile_points) * step + 32 : 0;
  PP_CUDA(raise_smem_limit(viz_compact_kernel, smem));
  viz_compact_kernel<<<n_tiles, kThreads, smem, pp->stream>>>(L);
  count_launch(2);
  PP_CUDA(cudaGetLastError());
  PP_CUDA(cudaMemcpyAsync(pp->h_kept, pp->kept.p, sizeof(uint32_t), cudaMemcpyDeviceToHost, pp->stream));
  PP_CUDA(cudaStreamSynchronize(pp->stream));
  const size_t kept = *pp->h_kept;
  if (mem == CLDN_MEM_HOST && kept) {
    PP_CUDA(cudaMemcpyAsync(out, pp->d_out.p, kept * step, cudaMemcpyDeviceToHost, pp->stream));
    PP_CUDA(cudaStreamSynchronize(pp->stream));
  }
  // pc_info bookkeeping (:327-340)
  info->width = static_cast<uint32_t>(kept);
  info->height = 1;
  for (uint32_t i = 0; i < info->n_fields; ++i) {
    if (info->fields[i].type == CLDN_FLOAT64 && !info->fields[i].has_resolution) {
      info->fields[i].has_resolution = 1;
      info->fields[i].resolution = 1e-6f;
    }
  }
  if (kept_points) *kept_points = kept;
  if (applied) *applied = 1;
  return CLDN_OK;
}

}  // extern "C"
