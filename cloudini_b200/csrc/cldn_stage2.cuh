// Byte-moving helpers shared by the stage-2 kernels (LZ4 in cldn_lz4.cu, ZSTD in cldn_zstd.cu): unaligned loads and a
// cooperative copy that stores aligned 16-byte vectors. Reads never leave the aligned words covering the source range.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "cldn_device.cuh"

namespace cldn {

__device__ __forceinline__ uint32_t lz_load32(const uint8_t* p) {  // any alignment
  const uintptr_t a = reinterpret_cast<uintptr_t>(p);
  const uint32_t* w = reinterpret_cast<const uint32_t*>(a & ~uintptr_t(3));
  const uint32_t sh = static_cast<uint32_t>(a & 3u) * 8u;
  if (sh == 0) return w[0];
  return __funnelshift_r(w[0], w[1], sh);
}
__device__ __forceinline__ uint2 lz_load64(const uint8_t* p) {  // any alignment; reads the aligned words covering [p, p + 8)
  const uintptr_t a = reinterpret_cast<uintptr_t>(p);
  const uint32_t* w = reinterpret_cast<const uint32_t*>(a & ~uintptr_t(3));
  const uint32_t sh = static_cast<uint32_t>(a & 3u) * 8u;
  const uint32_t w0 = w[0], w1 = w[1];
  if (sh == 0) return make_uint2(w0, w1);
  const uint32_t w2 = w[2];
  return make_uint2(__funnelshift_r(w0, w1, sh), __funnelshift_r(w1, w2, sh));
}
// n bytes from src to dst by `nt` threads (this one is `tid`): 16-byte stores for the aligned body of dst, the (unaligned)
// source through aligned words + funnel shifts. Reads the aligned words covering [src, src + n) only.
__device__ __forceinline__ void lz_copy(uint8_t* __restrict__ dst, const uint8_t* __restrict__ src, uint32_t n, uint32_t tid, uint32_t nt) {
  uint32_t head = (16u - static_cast<uint32_t>(reinterpret_cast<uintptr_t>(dst) & 15u)) & 15u;
  if (head > n) head = n;
  for (uint32_t k = tid; k < head; k += nt) dst[k] = src[k];
  const uint8_t* s0 = src + head;
  const uint32_t a = static_cast<uint32_t>(reinterpret_cast<uintptr_t>(s0) & 3u);
  uint32_t nv = (n - head) >> 4;
  // an unaligned source: a vector reads one word more than its 16 bytes; the last one may only do so inside the range
  if (a != 0u && nv != 0u && ((n - head) & 15u) < 4u - a) --nv;
  const uint32_t* w = reinterpret_cast<const uint32_t*>(s0 - a);
  uint4* dv = reinterpret_cast<uint4*>(dst + head);
  if (a == 0u) {
    for (uint32_t v = tid; v < nv; v += nt) {
      const uint32_t* q = w + 4u * v;
      dv[v] = make_uint4(q[0], q[1], q[2], q[3]);
    }
  } else {
    const uint32_t sh = a * 8u;
    for (uint32_t v = tid; v < nv; v += nt) {
      const uint32_t* q = w + 4u * v;
      const uint32_t w0 = q[0], w1 = q[1], w2 = q[2], w3 = q[3], w4 = q[4];
      dv[v] = make_uint4(__funnelshift_r(w0, w1, sh), __funnelshift_r(w1, w2, sh), __funnelshift_r(w2, w3, sh), __funnelshift_r(w3, w4, sh));
    }
  }
  for (uint32_t k = head + (nv << 4) + tid; k < n; k += nt) dst[k] = src[k];
}
__device__ __forceinline__ void lz_prefetch(const void* p, bool l1) {
  if (l1) asm volatile("prefetch.global.L1 [%0];" ::"l"(p));
  else asm volatile("prefetch.global.L2 [%0];" ::"l"(p));
}

// Position of chunk `c` inside a framed payload ([u32 size][bytes])*: *body = offset of its bytes, returns its size;
// 0xFFFFFFFF if the chain leaves the payload. (<= a few dozen hops: every frame has ceil(points / 32768) chunks.)
__device__ __forceinline__ uint32_t lz_find_chunk(const uint8_t* payload, uint64_t bytes, uint32_t c, uint64_t* body) {
  uint64_t pos = 0;
  for (uint32_t k = 0;; ++k) {
    if (bytes - pos < 4u || pos > bytes) return 0xFFFFFFFFu;
    const uint32_t sz = load_u32(payload + pos);
    if (sz > bytes - pos - 4u) return 0xFFFFFFFFu;
    if (k == c) { *body = pos + 4u; return sz; }
    pos += 4ull + sz;
  }
}

}  // namespace cldn
