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
#include <memory>
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

// Table slots of a cloud of n points: a multiple of 1024 that is at least 2n (load factor <= 1/2). The output does not
// depend on the size or the hash, only on the table holding every distinct voxel.
__host__ __device__ __forceinline__ uint32_t viz_table_size(uint32_t n) { return ((2u * n + 1023u) / 1024u) * 1024u; }

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
  // a tile slot past the cloud's last tile (the prepared grid of the async call) joins no look-back and writes no count
  if (static_cast<uint64_t>(tile) * tile_points >= n) return;
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

// ---- device clouds of one prepared layout, without the host (cldn_b200_viz_lossy_preprocess_batch_async) ------------
// Every frame slot f of the prepared shape owns blocks [f * blocks_per_frame, ..), tiles [f * tiles_per_frame, ..), the
// table region [f * table_per_frame, ..) and the slots [f * max_points, ..), so the insert and compact grids are those of
// max_frames clouds of max_points points whatever the call holds. The frame kernel writes the frame table on the device;
// a frame that is not rewritten (refused, empty, no-op, or past n_frames) gets n_points = 0, and all its blocks and
// tiles leave at once.
struct VizDesc {  // cldn_viz_desc_t
  const uint8_t* cloud;
  uint64_t cloud_bytes;
  uint8_t* out;
  uint64_t capacity;
};

struct VizAsyncLaunch {
  const VizDesc* desc;           // device, n_frames
  uint32_t n_frames;
  uint32_t n_slots;              // prepared frames (>= n_frames): the frame table has this many entries
  uint32_t point_step, xyz_offset;
  uint32_t noop;                 // the layout is one of the reference's early returns
  uint32_t max_points;
  uint32_t blocks_per_frame, tiles_per_frame, table_per_frame, clear_blocks_per_frame;
  VizFrame* frames;
  int32_t* frame_status;         // per frame slot: the status the frame kernel decided
  const uint32_t* kept;          // per frame slot: survivors, written by the compaction's last tile
  unsigned long long* keys;
  uint32_t* firsts;
  // the call's outputs (device, n_frames entries)
  int32_t* status;
  uint64_t* kept_out;
  int32_t* applied;
  CloudDesc* encode;
};

constexpr uint32_t kVizClearSlots = 4096;  // table slots cleared per CTA

// One thread per frame slot: the per-frame checks of viz_frames in its order, then the prepared maximum.
__global__ void __launch_bounds__(kThreads) viz_async_frames_kernel(const VizAsyncLaunch A) {
  const uint32_t f = blockIdx.x * kThreads + threadIdx.x;
  if (f >= A.n_slots) return;
  VizDesc D = {nullptr, 0, nullptr, 0};
  if (f < A.n_frames) D = A.desc[f];
  const uint64_t n = A.point_step ? D.cloud_bytes / A.point_step : 0;
  int32_t st = !D.cloud && D.cloud_bytes ? CLDN_ERR_INVALID_ARGUMENT : CLDN_OK;
  const bool rewritten = st == CLDN_OK && !A.noop && n > 0;  // a no-op layout or an empty cloud is left as it is
  if (rewritten) {
    if (n > (1ull << 30)) st = CLDN_ERR_UNSUPPORTED;
    else if (static_cast<uint64_t>(A.xyz_offset) + 12u > A.point_step) st = CLDN_ERR_INVALID_ARGUMENT;
    else if (!D.out || D.capacity < n * A.point_step) st = CLDN_ERR_BUFFER_TOO_SMALL;
    else if (n > A.max_points) st = CLDN_ERR_UNSUPPORTED;  // the one refusal of the async call alone
  }
  const uint32_t pts = rewritten && st == CLDN_OK ? static_cast<uint32_t>(n) : 0u;
  VizFrame F;
  F.in = D.cloud;
  F.out = D.out;
  F.n_points = pts;
  F.block_begin = f * A.blocks_per_frame;
  F.tile_begin = f * A.tiles_per_frame;
  F.table_size = pts ? viz_table_size(pts) : 0u;
  F.table_base = static_cast<uint64_t>(f) * A.table_per_frame;
  F.slot_base = static_cast<uint64_t>(f) * A.max_points;
  A.frames[f] = F;
  A.frame_status[f] = st;
}

// keys = kEmptyVoxel and firsts = ~0 over [0, table_size) of every rewritten frame: the bytes cleared follow the
// frames' points, not the prepared maximum. table_size and the region bases are multiples of 1024 slots.
__global__ void __launch_bounds__(kThreads) viz_clear_kernel(const VizAsyncLaunch A) {
  const uint32_t f = blockIdx.x / A.clear_blocks_per_frame;
  const uint32_t begin = (blockIdx.x - f * A.clear_blocks_per_frame) * kVizClearSlots;
  const VizFrame F = A.frames[f];
  if (begin >= F.table_size) return;
  const uint32_t slots = min(kVizClearSlots, F.table_size - begin);
  const uint4 ones = make_uint4(~0u, ~0u, ~0u, ~0u);
  uint4* keys = reinterpret_cast<uint4*>(A.keys + F.table_base + begin);
  for (uint32_t i = threadIdx.x; i < slots / 2; i += kThreads) keys[i] = ones;
  uint4* firsts = reinterpret_cast<uint4*>(A.firsts + F.table_base + begin);
  for (uint32_t i = threadIdx.x; i < slots / 4; i += kThreads) firsts[i] = ones;
}

// One thread per frame of the call: status, kept, applied and the encoder's descriptor, from the frame table and the
// survivor counts.
__global__ void __launch_bounds__(kThreads) viz_async_finish_kernel(const VizAsyncLaunch A) {
  const uint32_t f = blockIdx.x * kThreads + threadIdx.x;
  if (f >= A.n_frames) return;
  const VizDesc D = A.desc[f];
  const int32_t st = A.frame_status[f];
  const bool applied = A.frames[f].n_points != 0u;
  const uint64_t kept = applied ? A.kept[f] : A.point_step ? D.cloud_bytes / A.point_step : 0;
  A.status[f] = st;
  if (A.kept_out) A.kept_out[f] = kept;
  if (A.applied) A.applied[f] = applied ? 1 : 0;
  if (A.encode) {  // cloud, cloud_bytes, width and height only: out and capacity are the caller's
    CloudDesc* E = A.encode + f;
    E->cloud = st != CLDN_OK ? nullptr : applied ? D.out : D.cloud;
    E->cloud_bytes = st != CLDN_OK ? 1u : applied ? kept * A.point_step : D.cloud_bytes;
    E->width = 0;
    E->height = 0;
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

// The reference's early returns that depend on the layout alone (ros_msg_utils.cpp:250-278): true when the layout has no
// xyz triple or a resolution that is not positive and finite, in which case every cloud of it is left as it is.
bool viz_noop_layout(const cldn_info_t& info, uint32_t* xyz_offset, float* xyz_res) {
  *xyz_offset = 0;
  *xyz_res = 0.0f;
  if (info.n_fields < 3 || info.point_step == 0) return true;
  const cldn_field_t &f0 = info.fields[0], &f1 = info.fields[1], &f2 = info.fields[2];
  const bool has_triple = f0.type == CLDN_FLOAT32 && f1.type == CLDN_FLOAT32 && f2.type == CLDN_FLOAT32 && f0.has_resolution &&
                          f1.has_resolution && f2.has_resolution && f0.resolution == f1.resolution &&
                          f0.resolution == f2.resolution && f1.offset == f0.offset + 4u && f2.offset == f0.offset + 8u;
  *xyz_res = f0.resolution;
  *xyz_offset = f0.offset;
  return !has_triple || !(*xyz_res > 0.0f) || !isfinite(*xyz_res);
}

// Compaction tiles of kThreads x ppt points; staged: the survivors of a tile are gathered in shared memory.
void viz_tiling(uint32_t step, uint32_t* ppt, bool* staged) {
  uint32_t p = 8;
  while (p > 1 && static_cast<size_t>(kThreads) * p * step > (64u << 10)) p >>= 1;
  *ppt = p;
  *staged = static_cast<size_t>(kThreads) * p * step <= (200u << 10);
}

// pc_info bookkeeping of an applied cloud (:327-340), apart from width and height
void viz_info_after(cldn_info_t* o) {
  for (uint32_t i = 0; i < o->n_fields; ++i) {
    if (o->fields[i].type == CLDN_FLOAT64 && !o->fields[i].has_resolution) {
      o->fields[i].has_resolution = 1;
      o->fields[i].resolution = 1e-6f;
    }
  }
}

// Device memory of exactly n elements, freed with its owner.
template <typename T>
struct DevArray {
  T* p = nullptr;
  DevArray() = default;
  DevArray(const DevArray&) = delete;
  DevArray& operator=(const DevArray&) = delete;
  ~DevArray() { if (p) cudaFree(p); }
  bool alloc(size_t n) { return cudaMalloc(reinterpret_cast<void**>(&p), std::max<size_t>(n, 1) * sizeof(T)) == cudaSuccess; }
};
}  // namespace

// The prepared state of cldn_b200_viz_lossy_preprocess_batch_async: separate from the buffers of the single and batch
// calls, so that those keep working between async calls and a captured graph stays valid until the next prepare.
struct VizAsync {
  size_t max_frames = 0;
  uint32_t ppt = 1;
  bool staged = false;
  size_t smem = 0;
  uint32_t insert_blocks = 0, compact_tiles = 0, clear_blocks = 0;
  DevArray<uint8_t> table;  // keys (8 B per slot) of every frame's region, then firsts (4 B per slot)
  DevArray<uint32_t> slots, kept;
  DevArray<uint64_t> status;
  DevArray<VizFrame> frames;
  DevArray<int32_t> frame_status;
  VizAsyncLaunch A{};  // all but the call's arrays
  VizLaunch L{};
};

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
  std::unique_ptr<VizAsync> async;  // cldn_b200_preproc_prepare_batch
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
  float xyz_res = 0.0f;
  uint32_t xyz_offset = 0;
  const bool noop = viz_noop_layout(*info, &xyz_offset, &xyz_res);
  auto fail = [&](size_t f, int rc, const char* msg) {
    if (name_frames) set_error("frame %zu: %s", f, msg);
    else set_error("%s", msg);
    return rc;
  };
  const uint32_t step = info->point_step;
  uint64_t total_points = 0, blocks = 0, tiles = 0, table = 0;
  uint32_t ppt;
  bool staged;
  viz_tiling(step, &ppt, &staged);
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
      viz_info_after(&o);
    }
  }
  if (copied) PP_CUDA(cudaStreamSynchronize(pp->stream));
  return CLDN_OK;
}

static int prepare_batch_impl(cldn_preproc_t* pp, const cldn_info_t* info, size_t max_frames, uint64_t max_points,
                              cldn_info_t* info_after) {
  if (!pp || !info) { set_error("null argument"); return CLDN_ERR_INVALID_ARGUMENT; }
  if (max_frames == 0 || max_frames > 0x7FFFFFFFull) { set_error("max_frames must be 1 .. 2^31 - 1"); return CLDN_ERR_INVALID_ARGUMENT; }
  if (max_points > (1u << 30)) { set_error("viz preprocessing: more than 2^30 points in one cloud"); return CLDN_ERR_UNSUPPORTED; }
  float xyz_res = 0.0f;
  uint32_t xyz_offset = 0;
  const bool noop = viz_noop_layout(*info, &xyz_offset, &xyz_res);
  const uint32_t step = info->point_step;
  uint32_t ppt;
  bool staged;
  viz_tiling(step, &ppt, &staged);
  const uint64_t points = std::max<uint64_t>(max_points, 1), tile_points = static_cast<uint64_t>(kThreads) * ppt;
  const uint64_t blocks_per_frame = (points + kThreads - 1) / kThreads, tiles_per_frame = (points + tile_points - 1) / tile_points;
  const uint32_t table_per_frame = viz_table_size(static_cast<uint32_t>(points));
  const uint32_t clear_per_frame = (table_per_frame + kVizClearSlots - 1) / kVizClearSlots;
  if (!noop && (max_frames * blocks_per_frame > 0x7FFFFFFFull || max_frames * tiles_per_frame > 0x7FFFFFFFull)) {
    set_error("max_frames * blocks or tiles per frame must be below 2^31");
    return CLDN_ERR_UNSUPPORTED;
  }
  PP_CUDA(cudaSetDevice(pp->device));
  PP_CUDA(cudaStreamSynchronize(pp->stream));  // kernels of an earlier prepared state may still read it
  pp->async.reset();
  std::unique_ptr<VizAsync> a(new VizAsync());
  a->max_frames = max_frames;
  const size_t table_slots = noop ? 0 : max_frames * table_per_frame;
  if (!a->frames.alloc(max_frames) || !a->frame_status.alloc(max_frames) || !a->kept.alloc(max_frames) ||
      !a->table.alloc(table_slots * 12) || !a->slots.alloc(noop ? 0 : max_frames * points) ||
      !a->status.alloc(noop ? 0 : max_frames * tiles_per_frame)) {
    set_error("device allocation failed");
    return CLDN_ERR_CUDA;
  }
  VizAsyncLaunch& A = a->A;
  A.n_slots = static_cast<uint32_t>(max_frames);
  A.point_step = step;
  A.xyz_offset = xyz_offset;
  A.noop = noop ? 1u : 0u;
  A.max_points = static_cast<uint32_t>(max_points);
  A.blocks_per_frame = static_cast<uint32_t>(blocks_per_frame);
  A.tiles_per_frame = static_cast<uint32_t>(tiles_per_frame);
  A.table_per_frame = table_per_frame;
  A.clear_blocks_per_frame = clear_per_frame;
  A.frames = a->frames.p;
  A.frame_status = a->frame_status.p;
  A.kept = a->kept.p;
  A.keys = reinterpret_cast<unsigned long long*>(a->table.p);
  A.firsts = reinterpret_cast<uint32_t*>(a->table.p + table_slots * 8);
  if (!noop) {
    a->ppt = ppt;
    a->staged = staged;
    a->smem = staged ? static_cast<size_t>(tile_points) * step + 32 : 0;
    a->insert_blocks = static_cast<uint32_t>(max_frames * blocks_per_frame);
    a->compact_tiles = static_cast<uint32_t>(max_frames * tiles_per_frame);
    a->clear_blocks = static_cast<uint32_t>(max_frames * clear_per_frame);
    PP_CUDA(raise_smem_limit(viz_compact_kernel, a->smem));
    VizLaunch& L = a->L;
    L.frames = a->frames.p;
    L.n_frames = static_cast<uint32_t>(max_frames);
    L.point_step = step;
    L.xyz_offset = xyz_offset;
    L.inv_res = 1.0f / xyz_res;
    L.keys = A.keys;
    L.firsts = A.firsts;
    L.slots = a->slots.p;
    L.status = a->status.p;
    L.epoch = 1;  // the words are cleared in every call
    L.ppt = ppt;
    L.staged = staged ? 1u : 0u;
    L.kept = a->kept.p;
  }
  if (info_after) {
    *info_after = *info;
    if (!noop) {
      info_after->width = info_after->height = 0;
      viz_info_after(info_after);
    }
  }
  pp->async = std::move(a);
  return CLDN_OK;
}

// Enqueues only. The launches and their grids are those of the prepared layout and shape, whatever the frames: a clear
// of the tile status words, the frame kernel, the table clear, insert and compact, the finish kernel (frame and finish
// kernels alone for a no-op layout).
static int preprocess_batch_async_impl(cldn_preproc_t* pp, size_t n, const void* d_frames, int32_t* d_status, uint64_t* d_kept,
                                       int32_t* d_applied, cldn_cloud_desc_t* d_encode) {
  if (!pp) { set_error("null argument"); return CLDN_ERR_INVALID_ARGUMENT; }
  VizAsync* a = pp->async.get();
  if (!a) { set_error("no prepared layout: call cldn_b200_preproc_prepare_batch first"); return CLDN_ERR_INVALID_ARGUMENT; }
  if (n > a->max_frames) { set_error("%zu frames: the shape was prepared for at most %zu", n, a->max_frames); return CLDN_ERR_INVALID_ARGUMENT; }
  if (!d_frames || !d_status) { set_error("null argument"); return CLDN_ERR_INVALID_ARGUMENT; }
  if (n == 0) return CLDN_OK;
  PP_CUDA(cudaSetDevice(pp->device));
  VizAsyncLaunch A = a->A;
  A.desc = static_cast<const VizDesc*>(d_frames);
  A.n_frames = static_cast<uint32_t>(n);
  A.status = d_status;
  A.kept_out = d_kept;
  A.applied = d_applied;
  A.encode = reinterpret_cast<CloudDesc*>(d_encode);
  const uint32_t frame_blocks = static_cast<uint32_t>((a->max_frames + kThreads - 1) / kThreads);
  if (!A.noop) PP_CUDA(cudaMemsetAsync(a->status.p, 0, static_cast<size_t>(a->compact_tiles) * sizeof(uint64_t), pp->stream));
  viz_async_frames_kernel<<<frame_blocks, kThreads, 0, pp->stream>>>(A);
  if (!A.noop) {
    viz_clear_kernel<<<a->clear_blocks, kThreads, 0, pp->stream>>>(A);
    viz_insert_kernel<<<a->insert_blocks, kThreads, 0, pp->stream>>>(a->L);
    viz_compact_kernel<<<a->compact_tiles, kThreads, a->smem, pp->stream>>>(a->L);
  }
  viz_async_finish_kernel<<<frame_blocks, kThreads, 0, pp->stream>>>(A);
  count_launch(A.noop ? 2 : 5);
  PP_CUDA(cudaGetLastError());
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
  pp->async.reset();
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

int cldn_b200_preproc_prepare_batch(cldn_preproc_t* pp, const cldn_info_t* info, size_t max_frames, uint64_t max_points_per_frame,
                                    cldn_info_t* info_after) {
  try {
    return prepare_batch_impl(pp, info, max_frames, max_points_per_frame, info_after);
  } catch (const std::bad_alloc&) {
    set_error("out of memory");
    return CLDN_ERR_INTERNAL;
  }
}

int cldn_b200_viz_lossy_preprocess_batch_async(cldn_preproc_t* pp, size_t n_frames, const void* d_frames, int32_t* d_status,
                                               uint64_t* d_kept, int32_t* d_applied, cldn_cloud_desc_t* d_encode) {
  return preprocess_batch_async_impl(pp, n_frames, d_frames, d_status, d_kept, d_applied, d_encode);
}

int cldn_b200_preproc_sync(cldn_preproc_t* pp) {
  if (!pp) { set_error("null argument"); return CLDN_ERR_INVALID_ARGUMENT; }
  PP_CUDA(cudaSetDevice(pp->device));
  PP_CUDA(cudaStreamSynchronize(pp->stream));
  return CLDN_OK;
}

}  // extern "C"
