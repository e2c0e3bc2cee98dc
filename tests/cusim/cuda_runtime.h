// cusim — TEST INFRASTRUCTURE ONLY. A functional CPU emulation of the CUDA execution model, just large enough to run
// the *unmodified* kernel sources of cloudini_b200/csrc under the `-m "not gpu"` test suite (this container has no
// GPU; the real parity gate is `pytest -m gpu` on an H100). It is NOT a CPU fallback of the product:
//   * it is never built by cloudini_b200.build / __graft_entry__.build(), never shipped in cloudini_b200/lib and never
//     loaded by bench.py or smoke() (both refuse a library whose cldn_b200_version() reports "cusim");
//   * tests/cusim/build_cusim.py compiles the kernel sources with g++ against THIS header (it shadows
//     <cuda_runtime.h>) into tests/cusim/_build/libcloudini_b200_cusim.so, which only tests/test_cusim_kernels.py loads.
// Model: one OS thread runs one CTA at a time; the CTA's threads are cooperative fibers that switch at
// __syncthreads() and at every warp-collective (shuffle / ballot / vote), so barrier and warp semantics are exact and
// divergence bugs (a lane missing a collective) show up as a reported deadlock. CTAs are dispatched in increasing
// blockIdx order on several OS threads, so inter-CTA protocols (decoupled look-back, published descriptors) run with
// real concurrency. It checks the *logic* of a kernel (indexing, scans, packing, protocols); it says nothing about
// performance and little about memory-model races.
#pragma once
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <functional>

#define CLDN_CUSIM 1

// ---- qualifiers ----------------------------------------------------------------------------------------------------
#define __global__
#define __device__
#define __host__
#define __forceinline__ inline __attribute__((always_inline))
#define __launch_bounds__(...)
#define __align__(n) alignas(n)
#define __shared__ static thread_local
#define __constant__ static
#ifndef __restrict__
#define __restrict__ __restrict
#endif

// ---- vector types --------------------------------------------------------------------------------------------------
struct uint3 { unsigned x, y, z; };
struct dim3 {
  unsigned x, y, z;
  dim3(unsigned x_ = 1, unsigned y_ = 1, unsigned z_ = 1) : x(x_), y(y_), z(z_) {}
};
struct alignas(8) uint2 { unsigned x, y; };
struct alignas(16) uint4 { unsigned x, y, z, w; };
struct alignas(8) int2 { int x, y; };
struct alignas(16) int4 { int x, y, z, w; };
struct alignas(8) float2 { float x, y; };
struct alignas(16) float4 { float x, y, z, w; };
struct alignas(16) ulonglong2 { unsigned long long x, y; };
static inline uint2 make_uint2(unsigned x, unsigned y) { return uint2{x, y}; }
static inline uint4 make_uint4(unsigned x, unsigned y, unsigned z, unsigned w) { return uint4{x, y, z, w}; }
static inline int2 make_int2(int x, int y) { return int2{x, y}; }
static inline int4 make_int4(int x, int y, int z, int w) { return int4{x, y, z, w}; }
static inline float2 make_float2(float x, float y) { return float2{x, y}; }
static inline float4 make_float4(float x, float y, float z, float w) { return float4{x, y, z, w}; }
static inline ulonglong2 make_ulonglong2(unsigned long long x, unsigned long long y) { return ulonglong2{x, y}; }

// ---- scheduler interface (cusim.cpp) ---------------------------------------------------------------------------------
namespace cusim {
struct ThreadCoords { uint3 tid, bid, bdim, gdim; };  // plain data: written only by the (uninstrumented) scheduler
extern thread_local ThreadCoords tc;
void launch(dim3 grid, dim3 block, size_t smem_bytes, const std::function<void()>& body, const void* kernel = nullptr);
// the hardware's dynamic shared memory rules: 48 KB per CTA unless cudaFuncSetAttribute raised the kernel's limit
// (at most 227 KB); a launch beyond it fails with cudaErrorInvalidValue and runs nothing
int set_max_dyn_smem(const void* kernel, int bytes);
int take_last_error();
// "Device" memory is host memory here, so host code that dereferences a device pointer (a segmentation fault on the real
// machine) would go unnoticed. With CUSIM_HOSTCHECK=1 every cudaMalloc region is its own mapping that is only
// accessible while a kernel runs or a cudaMemcpy / cudaMemset is in progress (DeviceAccess); any other touch is reported
// and aborts. Not in the sanitizer builds (they need the instrumented heap).
// CUSIM_ASYNC=1: a cudaMemcpyAsync(DeviceToHost) delivers its bytes (captured at enqueue time, i.e. in stream order) only
// when the host synchronises with the stream — cudaStreamSynchronize, an event recorded behind it, cudaDeviceSynchronize —
// and the destination holds 0xEE until then, so host code that reads a result before synchronising gets garbage as it
// (sometimes) would on the GPU box.
bool defer_d2h(void* dst, const void* src, size_t n, void* stream);
void flush_d2h(void* stream, bool all);
void event_record(void* event, void* stream);
void event_sync(void* event);
void event_forget(void* event);
void* device_alloc(size_t bytes);
void device_free(void* p);
void device_access_begin();
void device_access_end();
struct DeviceAccess {
  DeviceAccess() { device_access_begin(); }
  ~DeviceAccess() { device_access_end(); }
};
void* dyn_smem();
// static __shared__ variables announce themselves (build_cusim.py adds the call behind every declaration) so that the
// scheduler can fill them with 0xA5 before a CTA starts: shared memory is NOT zero on the GPU, and a kernel whose
// result depends on an unwritten static shared variable must not pass here
void register_shared(void* p, size_t bytes);
void syncthreads();
int syncthreads_or(int pred);
void poll_yield();  // called by the spin-wait loads so that a producer in the same CTA can run
// Warp collective: deposits `v`, waits until every live lane of `mask` has arrived, returns the 32 deposited values.
// kind 0: value collective (shuffle / ballot / vote), kind 1: __syncwarp (the only warp-level primitive that CUDA defines as
// a memory fence among the participating lanes; the racecheck build can be told to honour exactly that: CUSIM_TSAN_STRICT=1)
const uint64_t* warp_exchange(unsigned mask, uint64_t v, unsigned* arrived_mask, int kind = 0);
unsigned lane_id();
uint64_t globaltimer_ns();
}  // namespace cusim

#define threadIdx (::cusim::tc.tid)
#define blockIdx (::cusim::tc.bid)
#define blockDim (::cusim::tc.bdim)
#define gridDim (::cusim::tc.gdim)
constexpr int warpSize = 32;

static inline void __syncthreads() { cusim::syncthreads(); }
static inline int __syncthreads_or(int p) { return cusim::syncthreads_or(p); }
static inline void __syncwarp(unsigned mask = 0xffffffffu) { unsigned a; cusim::warp_exchange(mask, 0, &a, 1); }
static inline void __threadfence() { __atomic_thread_fence(__ATOMIC_SEQ_CST); }
static inline void __threadfence_block() { __atomic_thread_fence(__ATOMIC_SEQ_CST); }

// ---- warp collectives ------------------------------------------------------------------------------------------------
namespace cusim {
template <class T> inline uint64_t to_bits(T v) { static_assert(sizeof(T) <= 8, "shuffle operand too wide"); uint64_t b = 0; memcpy(&b, &v, sizeof(T)); return b; }
template <class T> inline T from_bits(uint64_t b) { T v; memcpy(&v, &b, sizeof(T)); return v; }
}  // namespace cusim
template <class T> static inline T __shfl_sync(unsigned mask, T v, int src, int width = 32) {
  unsigned arrived; const uint64_t* s = cusim::warp_exchange(mask, cusim::to_bits(v), &arrived);
  const unsigned lane = cusim::lane_id();
  const unsigned from = (lane & ~static_cast<unsigned>(width - 1)) | (static_cast<unsigned>(src) & static_cast<unsigned>(width - 1));
  return ((arrived >> from) & 1u) ? cusim::from_bits<T>(s[from]) : v;
}
template <class T> static inline T __shfl_up_sync(unsigned mask, T v, unsigned d, int width = 32) {
  unsigned arrived; const uint64_t* s = cusim::warp_exchange(mask, cusim::to_bits(v), &arrived);
  const unsigned lane = cusim::lane_id(), base = lane & ~static_cast<unsigned>(width - 1);
  return (lane - base >= d && ((arrived >> (lane - d)) & 1u)) ? cusim::from_bits<T>(s[lane - d]) : v;
}
template <class T> static inline T __shfl_down_sync(unsigned mask, T v, unsigned d, int width = 32) {
  unsigned arrived; const uint64_t* s = cusim::warp_exchange(mask, cusim::to_bits(v), &arrived);
  const unsigned lane = cusim::lane_id(), base = lane & ~static_cast<unsigned>(width - 1);
  return (lane - base + d < static_cast<unsigned>(width) && ((arrived >> (lane + d)) & 1u)) ? cusim::from_bits<T>(s[lane + d]) : v;
}
template <class T> static inline T __shfl_xor_sync(unsigned mask, T v, int x, int width = 32) {
  unsigned arrived; const uint64_t* s = cusim::warp_exchange(mask, cusim::to_bits(v), &arrived);
  const unsigned from = cusim::lane_id() ^ static_cast<unsigned>(x);
  (void)width;
  return (from < 32u && ((arrived >> from) & 1u)) ? cusim::from_bits<T>(s[from]) : v;
}
static inline unsigned __ballot_sync(unsigned mask, int pred) {
  unsigned arrived; const uint64_t* s = cusim::warp_exchange(mask, pred ? 1u : 0u, &arrived);
  unsigned r = 0;
  for (unsigned l = 0; l < 32; ++l) if (((arrived >> l) & 1u) && s[l]) r |= 1u << l;
  return r;
}
static inline int __any_sync(unsigned mask, int pred) { return __ballot_sync(mask, pred) != 0u; }
static inline int __all_sync(unsigned mask, int pred) {
  unsigned arrived; const uint64_t* s = cusim::warp_exchange(mask, pred ? 1u : 0u, &arrived);
  for (unsigned l = 0; l < 32; ++l) if (((arrived >> l) & 1u) && !s[l]) return 0;
  return 1;
}

namespace cusim { template <class T> struct same { typedef T type; }; }
// ---- atomics (global memory is shared between the OS threads that run different CTAs) ---------------------------------
template <class T> static inline T atomicAdd(T* p, typename cusim::same<T>::type v) { return __atomic_fetch_add(p, v, __ATOMIC_SEQ_CST); }
template <class T> static inline T atomicSub(T* p, typename cusim::same<T>::type v) { return __atomic_fetch_sub(p, v, __ATOMIC_SEQ_CST); }
template <class T> static inline T atomicOr(T* p, typename cusim::same<T>::type v) { return __atomic_fetch_or(p, v, __ATOMIC_SEQ_CST); }
template <class T> static inline T atomicAnd(T* p, typename cusim::same<T>::type v) { return __atomic_fetch_and(p, v, __ATOMIC_SEQ_CST); }
template <class T> static inline T atomicExch(T* p, typename cusim::same<T>::type v) { return __atomic_exchange_n(p, v, __ATOMIC_SEQ_CST); }
template <class T> static inline T atomicCAS(T* p, typename cusim::same<T>::type cmp, typename cusim::same<T>::type v) { __atomic_compare_exchange_n(p, &cmp, v, false, __ATOMIC_SEQ_CST, __ATOMIC_SEQ_CST); return cmp; }
template <class T> static inline T atomicMin(T* p, typename cusim::same<T>::type v) {
  T old = __atomic_load_n(p, __ATOMIC_SEQ_CST);
  while (v < old && !__atomic_compare_exchange_n(p, &old, v, false, __ATOMIC_SEQ_CST, __ATOMIC_SEQ_CST)) {}
  return old;
}
template <class T> static inline T atomicMax(T* p, typename cusim::same<T>::type v) {
  T old = __atomic_load_n(p, __ATOMIC_SEQ_CST);
  while (v > old && !__atomic_compare_exchange_n(p, &old, v, false, __ATOMIC_SEQ_CST, __ATOMIC_SEQ_CST)) {}
  return old;
}

// ---- arithmetic intrinsics (bit-exact restatements of the PTX semantics the kernels rely on) --------------------------
static inline float __fmul_rn(float a, float b) { volatile float r = a * b; return r; }  // built with -ffp-contract=off
static inline double __dmul_rn(double a, double b) { volatile double r = a * b; return r; }
static inline float __fadd_rn(float a, float b) { volatile float r = a + b; return r; }
static inline int __float2int_rn(float s) {  // cvt.rni.s32.f32: NaN -> 0, saturating, ties to even
  if (s != s) return 0;
  if (s >= 2147483648.0f) return 2147483647;
  if (s <= -2147483648.0f) return static_cast<int>(0x80000000u);
  return static_cast<int>(lrintf(s));
}
static inline long long __float2ll_rz(float s) {  // cvt.rzi.s64.f32: NaN -> 0x8000000000000000, saturating
  if (s != s) return static_cast<long long>(0x8000000000000000ull);
  if (s >= 9223372036854775808.0f) return 0x7FFFFFFFFFFFFFFFll;
  if (s <= -9223372036854775808.0f) return static_cast<long long>(0x8000000000000000ull);
  return static_cast<long long>(s);
}
static inline long long __double2ll_rz(double s) {
  if (s != s) return static_cast<long long>(0x8000000000000000ull);
  if (s >= 9223372036854775808.0) return 0x7FFFFFFFFFFFFFFFll;
  if (s <= -9223372036854775808.0) return static_cast<long long>(0x8000000000000000ull);
  return static_cast<long long>(s);
}
static inline float __int2float_rn(int v) { return static_cast<float>(v); }
static inline float __uint2float_rn(unsigned v) { return static_cast<float>(v); }
static inline float __ll2float_rn(long long v) { return static_cast<float>(v); }
static inline double __ll2double_rn(long long v) { return static_cast<double>(v); }
static inline unsigned __float_as_uint(float f) { unsigned u; memcpy(&u, &f, 4); return u; }
static inline int __float_as_int(float f) { int u; memcpy(&u, &f, 4); return u; }
static inline float __uint_as_float(unsigned u) { float f; memcpy(&f, &u, 4); return f; }
static inline float __int_as_float(int u) { float f; memcpy(&f, &u, 4); return f; }
static inline long long __double_as_longlong(double d) { long long u; memcpy(&u, &d, 8); return u; }
static inline double __longlong_as_double(long long u) { double d; memcpy(&d, &u, 8); return d; }
static inline int __clz(int v) { return v == 0 ? 32 : __builtin_clz(static_cast<unsigned>(v)); }
static inline int __clzll(long long v) { return v == 0 ? 64 : __builtin_clzll(static_cast<unsigned long long>(v)); }
static inline int __ffs(int v) { return __builtin_ffs(v); }
static inline int __ffsll(long long v) { return __builtin_ffsll(v); }
static inline int __popc(unsigned v) { return __builtin_popcount(v); }
static inline int __popcll(unsigned long long v) { return __builtin_popcountll(v); }
static inline unsigned __brev(unsigned v) { unsigned r = 0; for (int i = 0; i < 32; ++i) r |= ((v >> i) & 1u) << (31 - i); return r; }
static inline unsigned __funnelshift_r(unsigned lo, unsigned hi, unsigned sh) { return static_cast<unsigned>(((static_cast<uint64_t>(hi) << 32) | lo) >> (sh & 31u)); }
static inline unsigned __funnelshift_l(unsigned lo, unsigned hi, unsigned sh) { return static_cast<unsigned>((((static_cast<uint64_t>(hi) << 32) | lo) << (sh & 31u)) >> 32); }
static inline unsigned __funnelshift_rc(unsigned lo, unsigned hi, unsigned sh) { if (sh > 32u) sh = 32u; return static_cast<unsigned>(((static_cast<uint64_t>(hi) << 32) | lo) >> sh); }
static inline unsigned __funnelshift_lc(unsigned lo, unsigned hi, unsigned sh) { if (sh > 32u) sh = 32u; return static_cast<unsigned>(((((static_cast<uint64_t>(hi) << 32) | lo) << sh) >> 32) & 0xffffffffu); }
static inline unsigned __byte_perm(unsigned a, unsigned b, unsigned sel) {
  const uint64_t v = (static_cast<uint64_t>(b) << 32) | a;
  unsigned r = 0;
  // prmt's sign-replication mode (bit 3 of a selector nibble) is not restated: refuse rather than guess
  if (sel & 0x8888u) { fprintf(stderr, "cusim: __byte_perm selector 0x%x uses the sign-replication bit\n", sel); abort(); }
  for (int i = 0; i < 4; ++i) r |= static_cast<unsigned>((v >> (8 * ((sel >> (4 * i)) & 7u))) & 0xFFu) << (8 * i);
  return r;
}
namespace cusim {
static inline unsigned bmsk_clamp(unsigned a, unsigned b) {
  if (a > 32u) a = 32u;
  if (b > 32u) b = 32u;
  const uint64_t m = (b >= 32u ? 0xffffffffull : ((1ull << b) - 1ull)) << a;
  return static_cast<unsigned>(m & 0xffffffffull);
}
static inline unsigned lop3(unsigned a, unsigned b, unsigned c, unsigned lut) {
  unsigned r = 0;
  for (int i = 0; i < 32; ++i) r |= ((lut >> ((((a >> i) & 1u) << 2) | (((b >> i) & 1u) << 1) | ((c >> i) & 1u))) & 1u) << i;
  return r;
}
}  // namespace cusim
static inline unsigned __umulhi(unsigned a, unsigned b) { return static_cast<unsigned>((static_cast<uint64_t>(a) * b) >> 32); }
static inline unsigned long long __umul64hi(unsigned long long a, unsigned long long b) { return static_cast<unsigned long long>((static_cast<unsigned __int128>(a) * b) >> 64); }
template <class T> static inline T __ldg(const T* p) { return *p; }
template <class T> static inline T __ldcs(const T* p) { return *p; }
template <class T> static inline T __ldcg(const T* p) { return *p; }
template <class T> static inline void __stcs(T* p, T v) { *p = v; }
template <class T> static inline void __stcg(T* p, T v) { *p = v; }

// CUDA's min/max overload set (mixed signed / unsigned arguments promote like the CUDA math headers do)
static inline int min(int a, int b) { return a < b ? a : b; }
static inline int max(int a, int b) { return a > b ? a : b; }
static inline unsigned min(unsigned a, unsigned b) { return a < b ? a : b; }
static inline unsigned max(unsigned a, unsigned b) { return a > b ? a : b; }
static inline unsigned min(int a, unsigned b) { return min(static_cast<unsigned>(a), b); }
static inline unsigned min(unsigned a, int b) { return min(a, static_cast<unsigned>(b)); }
static inline unsigned max(int a, unsigned b) { return max(static_cast<unsigned>(a), b); }
static inline unsigned max(unsigned a, int b) { return max(a, static_cast<unsigned>(b)); }
static inline long long min(long long a, long long b) { return a < b ? a : b; }
static inline long long max(long long a, long long b) { return a > b ? a : b; }
static inline unsigned long long min(unsigned long long a, unsigned long long b) { return a < b ? a : b; }
static inline unsigned long long max(unsigned long long a, unsigned long long b) { return a > b ? a : b; }
static inline unsigned long min(unsigned long a, unsigned long b) { return a < b ? a : b; }
static inline unsigned long max(unsigned long a, unsigned long b) { return a > b ? a : b; }
static inline long min(long a, long b) { return a < b ? a : b; }
static inline long max(long a, long b) { return a > b ? a : b; }
static inline float min(float a, float b) { return fminf(a, b); }
static inline float max(float a, float b) { return fmaxf(a, b); }

// ---- runtime API (everything is synchronous; "device" memory is host memory) ------------------------------------------
typedef int cudaError_t;
typedef struct CUstream_st* cudaStream_t;
typedef struct CUevent_st* cudaEvent_t;
enum { cudaSuccess = 0, cudaErrorInvalidValue = 1, cudaErrorMemoryAllocation = 2 };
enum cudaMemcpyKind { cudaMemcpyHostToHost = 0, cudaMemcpyHostToDevice = 1, cudaMemcpyDeviceToHost = 2, cudaMemcpyDeviceToDevice = 3, cudaMemcpyDefault = 4 };
enum cudaFuncAttribute { cudaFuncAttributeMaxDynamicSharedMemorySize = 8 };
enum cudaDeviceAttr { cudaDevAttrMultiProcessorCount = 16 };
enum { cudaStreamNonBlocking = 1, cudaEventDisableTiming = 2, cudaEventDefault = 0 };

namespace cusim { int sm_count(); }
static inline const char* cudaGetErrorString(cudaError_t e) { return e == 0 ? "no error" : "cusim error"; }
static inline const char* cudaGetErrorName(cudaError_t e) { return e == 0 ? "cudaSuccess" : "cusimError"; }
static inline cudaError_t cudaGetLastError() { return static_cast<cudaError_t>(::cusim::take_last_error()); }
static inline cudaError_t cudaPeekAtLastError() { return cudaSuccess; }
static inline cudaError_t cudaGetDeviceCount(int* n) { *n = 1; return cudaSuccess; }
static inline cudaError_t cudaGetDevice(int* d) { *d = 0; return cudaSuccess; }
static inline cudaError_t cudaSetDevice(int d) { return d == 0 ? cudaSuccess : cudaErrorInvalidValue; }
static inline cudaError_t cudaDeviceGetPCIBusId(char*, int, int) { return cudaErrorInvalidValue; }  // no PCI device behind the emulation
static inline cudaError_t cudaDeviceSynchronize() { ::cusim::flush_d2h(nullptr, true); return cudaSuccess; }
static inline cudaError_t cudaDeviceGetAttribute(int* v, cudaDeviceAttr a, int) { *v = (a == cudaDevAttrMultiProcessorCount) ? cusim::sm_count() : 0; return cudaSuccess; }
// fresh device memory holds whatever the previous owner left there: fill it with a pattern, so that code that relies on
// cudaMalloc returning zeros (it often does on a fresh process, not after memory has been recycled) fails here
static inline cudaError_t cudaMalloc(void** p, size_t n) {
  *p = ::cusim::device_alloc(n ? n : 256);
  return *p ? cudaSuccess : cudaErrorMemoryAllocation;
}
template <class T> static inline cudaError_t cudaMalloc(T** p, size_t n) { return cudaMalloc(reinterpret_cast<void**>(p), n); }
static inline cudaError_t cudaFree(void* p) { ::cusim::device_free(p); return cudaSuccess; }
static inline cudaError_t cudaMallocHost(void** p, size_t n) {
  if (posix_memalign(p, 256, n ? n : 256) != 0) return cudaErrorMemoryAllocation;
  memset(*p, 0xCD, n ? n : 256);
  return cudaSuccess;
}
template <class T> static inline cudaError_t cudaMallocHost(T** p, size_t n) { return cudaMallocHost(reinterpret_cast<void**>(p), n); }
static inline cudaError_t cudaFreeHost(void* p) { ::cusim::flush_d2h(nullptr, true); free(p); return cudaSuccess; }
static inline cudaError_t cudaMemcpy(void* d, const void* s, size_t n, cudaMemcpyKind) { ::cusim::DeviceAccess da; if (n) memmove(d, s, n); return cudaSuccess; }
static inline cudaError_t cudaMemcpyAsync(void* d, const void* s, size_t n, cudaMemcpyKind kind, cudaStream_t stream = nullptr) {
  ::cusim::DeviceAccess da;
  if (kind == cudaMemcpyDeviceToHost && ::cusim::defer_d2h(d, s, n, stream)) return cudaSuccess;
  if (n) memmove(d, s, n);
  return cudaSuccess;
}
static inline cudaError_t cudaMemset(void* d, int v, size_t n) { ::cusim::DeviceAccess da; if (n) memset(d, v, n); return cudaSuccess; }
static inline cudaError_t cudaMemsetAsync(void* d, int v, size_t n, cudaStream_t = nullptr) { ::cusim::DeviceAccess da; if (n) memset(d, v, n); return cudaSuccess; }
static inline cudaError_t cudaStreamCreate(cudaStream_t* s) { *s = reinterpret_cast<cudaStream_t>(malloc(8)); return cudaSuccess; }
static inline cudaError_t cudaStreamCreateWithFlags(cudaStream_t* s, unsigned) { return cudaStreamCreate(s); }
static inline cudaError_t cudaStreamDestroy(cudaStream_t s) { ::cusim::flush_d2h(s, false); free(s); return cudaSuccess; }
static inline cudaError_t cudaStreamSynchronize(cudaStream_t s) { ::cusim::flush_d2h(s, false); return cudaSuccess; }
static inline cudaError_t cudaStreamWaitEvent(cudaStream_t, cudaEvent_t, unsigned = 0) { return cudaSuccess; }
static inline cudaError_t cudaEventCreate(cudaEvent_t* e) { *e = reinterpret_cast<cudaEvent_t>(malloc(8)); return cudaSuccess; }
static inline cudaError_t cudaEventCreateWithFlags(cudaEvent_t* e, unsigned) { return cudaEventCreate(e); }
static inline cudaError_t cudaEventDestroy(cudaEvent_t e) { ::cusim::event_forget(e); free(e); return cudaSuccess; }
static inline cudaError_t cudaEventRecord(cudaEvent_t e, cudaStream_t s = nullptr) { ::cusim::event_record(e, s); return cudaSuccess; }
static inline cudaError_t cudaEventSynchronize(cudaEvent_t e) { ::cusim::event_sync(e); return cudaSuccess; }
static inline cudaError_t cudaEventQuery(cudaEvent_t e) { ::cusim::event_sync(e); return cudaSuccess; }
template <class F> static inline cudaError_t cudaFuncSetAttribute(F f, cudaFuncAttribute, int v) { return static_cast<cudaError_t>(::cusim::set_max_dyn_smem(reinterpret_cast<const void*>(f), v)); }
template <class F> static inline cudaError_t cudaOccupancyMaxActiveBlocksPerMultiprocessor(int* n, F, int, size_t) { *n = 3; return cudaSuccess; }
