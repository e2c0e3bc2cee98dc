// cusim scheduler — TEST INFRASTRUCTURE ONLY (see cuda_runtime.h in this directory for what this is and is not).
// One OS worker runs one CTA at a time; its threads are fibers (hand-rolled x86-64 context switch) scheduled
// round-robin, blocked fibers are skipped until their barrier / warp generation changes. A full pass without a
// runnable fiber is a deadlock (a lane skipped a collective, a barrier inside divergent code, ...) and aborts with a
// per-fiber report.
#include "cuda_runtime.h"

#include <signal.h>
#include <sys/mman.h>
#include <unistd.h>

#include <atomic>
#include <deque>
#include <map>
#include <chrono>
#include <mutex>
#include <thread>
#include <vector>

#if defined(__SANITIZE_ADDRESS__)
// AddressSanitizer build (tests/cusim/build_cusim.py --asan): the fiber switches are announced to the runtime so that
// its shadow stack bookkeeping follows them; "device" memory is then the instrumented heap, i.e. an out-of-bounds access
// of a kernel is reported like compute-sanitizer's memcheck would on the GPU.
#include <sanitizer/common_interface_defs.h>
#define CUSIM_ASAN 1
#else
#define CUSIM_ASAN 0
#endif

#if defined(CUSIM_TSAN)
// ThreadSanitizer build (tests/cusim/build_cusim.py --tsan -> racecheck executable): every CUDA thread is a TSAN fiber and
// the switches carry NO implicit synchronisation, so two threads of a CTA touching the same shared / global memory without
// a __syncthreads(), a warp collective or an atomic between them are reported — compute-sanitizer's racecheck without a
// GPU. This file itself is compiled uninstrumented (the scheduler's own bookkeeping is not kernel state); barriers and
// warp collectives publish their happens-before edges through __tsan_release / __tsan_acquire.
extern "C" {
void* __tsan_get_current_fiber(void);
void* __tsan_create_fiber(unsigned flags);
void __tsan_destroy_fiber(void* fiber);
void __tsan_switch_to_fiber(void* fiber, unsigned flags);
void __tsan_acquire(void* addr);
void __tsan_release(void* addr);
}
#define TSAN_SWITCH(f) __tsan_switch_to_fiber((f), 1u /* no_sync */)
#define TSAN_RELEASE(a) __tsan_release(a)
#define TSAN_ACQUIRE(a) __tsan_acquire(a)
#else
#define TSAN_SWITCH(f) ((void)0)
#define TSAN_RELEASE(a) ((void)0)
#define TSAN_ACQUIRE(a) ((void)0)
#endif

#if !defined(__x86_64__)
#error "cusim's context switch is written for x86-64"
#endif

extern "C" void cusim_switch(void** save_sp, void* new_sp);
asm(R"(
.text
.globl cusim_switch
.type cusim_switch,@function
cusim_switch:
  pushq %rbp
  pushq %rbx
  pushq %r12
  pushq %r13
  pushq %r14
  pushq %r15
  movq %rsp, (%rdi)
  movq %rsi, %rsp
  popq %r15
  popq %r14
  popq %r13
  popq %r12
  popq %rbx
  popq %rbp
  ret
.size cusim_switch,.-cusim_switch
)");

namespace cusim {

thread_local ThreadCoords tc;

namespace {

constexpr size_t kStackBytes = 256 * 1024;
constexpr unsigned kMaxThreads = 1024;

enum Wait : uint8_t { RUNNABLE = 0, WAIT_BARRIER, WAIT_WARP, WAIT_POLL, DONE };

struct Fiber {
  void* tsan = nullptr;        // TSAN fiber context (racecheck build)
  void* fake_stack = nullptr;  // ASAN fake-stack handle while the fiber is switched out
  void* sp = nullptr;
  char* stack = nullptr;
  Wait wait = RUNNABLE;
  uint32_t wait_gen = 0;
  uint32_t wait_warp = 0;
  uint3 tid{0, 0, 0};
};

struct Warp {
  uint64_t slot[2][32];
  unsigned arrived[2];
  unsigned arrived_final[2];
  uint32_t gen;
  unsigned live;  // lanes that exist and have not exited
};

struct Cta {
  Fiber fibers[kMaxThreads];
  Warp warps[kMaxThreads / 32];
  void* sched_sp = nullptr;
  unsigned n_threads = 0, cur = 0;
  unsigned live = 0, bar_arrived = 0;
  uint32_t bar_gen = 0;
  int bar_or_acc = 0, bar_or_res[2] = {0, 0};
  void* dyn = nullptr;
  size_t dyn_cap = 0;
  const std::function<void()>* body = nullptr;
  char* stacks = nullptr;
  void* sched_tsan = nullptr;             // TSAN context of the scheduler (the OS thread itself)
  char bar_sync = 0;                      // address the CTA barrier's happens-before edges hang on
  char start_sync = 0, end_sync = 0;      // launch -> thread start / thread exit -> CTA retired (two addresses: a thread that
                                          // exits must not become ordered before a thread that starts later)
  void* sched_fake_stack = nullptr;       // ASAN bookkeeping of the scheduler's (OS thread's) stack
  const void* sched_stack_bottom = nullptr;
  size_t sched_stack_size = 0;
};

thread_local Cta* g_cta = nullptr;
thread_local std::vector<std::pair<void*, size_t>> g_shared_regs;  // static __shared__ variables seen on this OS thread
}  // namespace

// The emulation's own locks. In the racecheck build they must not order the host threads that launch kernels: a lock
// that every launch takes would put a happens-before edge between any two host threads' library calls and hide their
// races. There they are spinlocks on atomics of this (uninstrumented) file, which ThreadSanitizer does not see.
#if defined(CUSIM_TSAN)
struct HostLock {
  std::atomic<bool> held{false};
  void lock() { while (held.exchange(true, std::memory_order_acquire)) std::this_thread::yield(); }
  void unlock() { held.store(false, std::memory_order_release); }
};
#else
typedef std::mutex HostLock;
#endif

namespace {

HostLock g_pool_mutex;
// CTA contexts (fiber stacks) are recycled between the launches of one host thread. The host thread takes them from its
// pool before it creates the launch's worker threads and returns them after it has joined them, so every reuse is
// ordered by that join and the next create. A worker must not return its context itself: on a busy machine a sibling
// worker of the same launch could start after that and take it, unordered. Sharing contexts between host threads would
// order those threads.
std::map<std::thread::id, std::vector<Cta*>> g_pool;

Cta* acquire_cta(std::thread::id host) {
  {
    std::lock_guard<HostLock> lock(g_pool_mutex);
    std::vector<Cta*>& pool = g_pool[host];
    if (!pool.empty()) { Cta* c = pool.back(); pool.pop_back(); return c; }
  }
  Cta* c = new Cta();
  c->stacks = static_cast<char*>(mmap(nullptr, kStackBytes * kMaxThreads, PROT_READ | PROT_WRITE,
                                      MAP_PRIVATE | MAP_ANONYMOUS | MAP_NORESERVE, -1, 0));
  if (c->stacks == MAP_FAILED) { fprintf(stderr, "cusim: mmap of fiber stacks failed\n"); abort(); }
  for (unsigned i = 0; i < kMaxThreads; ++i) c->fibers[i].stack = c->stacks + kStackBytes * i;
  return c;
}
void release_cta(Cta* c, std::thread::id host) {
  std::lock_guard<HostLock> lock(g_pool_mutex);
  g_pool[host].push_back(c);
}

void yield_to_scheduler() {
  Cta* c = g_cta;
  Fiber& f = c->fibers[c->cur];
#if CUSIM_ASAN
  __sanitizer_start_switch_fiber(&f.fake_stack, c->sched_stack_bottom, c->sched_stack_size);
#endif
  TSAN_SWITCH(c->sched_tsan);
  cusim_switch(&f.sp, c->sched_sp);
#if CUSIM_ASAN
  __sanitizer_finish_switch_fiber(f.fake_stack, &c->sched_stack_bottom, &c->sched_stack_size);
#endif
}

void release_barrier_if_complete(Cta* c) {
  if (c->live > 0 && c->bar_arrived >= c->live) {
    c->bar_arrived = 0;
    c->bar_or_res[c->bar_gen & 1u] = c->bar_or_acc;
    c->bar_or_acc = 0;
    c->bar_gen++;
  }
}

void release_warp_if_complete(Warp& w, unsigned mask_expected) {
  const unsigned b = w.gen & 1u;
  const unsigned need = mask_expected & w.live;
  if (need != 0 && (w.arrived[b] & need) == need) {
    w.arrived_final[b] = w.arrived[b];
    w.arrived[b] = 0;
    w.gen++;
  }
}

void fiber_main() {
  Cta* c = g_cta;
#if CUSIM_ASAN
  __sanitizer_finish_switch_fiber(nullptr, &c->sched_stack_bottom, &c->sched_stack_size);
#endif
  TSAN_ACQUIRE(&c->start_sync);  // everything the host did before the launch is visible to the kernel
  (*c->body)();
  TSAN_RELEASE(&c->end_sync);  // ... and the kernel's accesses are ordered before whatever follows the launch
  // thread exit: it no longer takes part in barriers or warp collectives
  Fiber& f = c->fibers[c->cur];
  f.wait = DONE;
  c->live--;
  release_barrier_if_complete(c);
  const unsigned linear = c->cur;
  Warp& w = c->warps[linear >> 5];
  w.live &= ~(1u << (linear & 31u));
  // a collective that was only waiting for this lane completes (CUDA ignores exited lanes)
  const unsigned b = w.gen & 1u;
  if (w.arrived[b] != 0 && w.live != 0 && (w.arrived[b] & w.live) == w.live) release_warp_if_complete(w, w.arrived[b]);
#if CUSIM_ASAN
  __sanitizer_start_switch_fiber(nullptr, c->sched_stack_bottom, c->sched_stack_size);  // this fiber is finished
#endif
  TSAN_SWITCH(c->sched_tsan);
  cusim_switch(&f.sp, c->sched_sp);
  fprintf(stderr, "cusim: finished fiber resumed\n");
  abort();
}

extern "C" void cusim_fiber_entry() { fiber_main(); }

void prepare_fiber(Fiber& f) {
  // initial frame consumed by cusim_switch: r15 r14 r13 r12 rbx rbp, then the "return address" = entry point
  uintptr_t top = reinterpret_cast<uintptr_t>(f.stack) + kStackBytes;
  top &= ~static_cast<uintptr_t>(15);
  uint64_t* p = reinterpret_cast<uint64_t*>(top);
  *--p = 0;                                                   // fake return address of the entry function
  *--p = reinterpret_cast<uint64_t>(&cusim_fiber_entry);      // popped by `ret`
  for (int i = 0; i < 6; ++i) *--p = 0;
  f.sp = p;
  f.wait = RUNNABLE;
}

void deadlock_report(Cta* c) {
  fprintf(stderr, "cusim: DEADLOCK in CTA (%u,%u,%u): no runnable thread. live=%u barrier arrived=%u\n", tc.bid.x, tc.bid.y,
          tc.bid.z, c->live, c->bar_arrived);
  unsigned shown = 0;
  for (unsigned i = 0; i < c->n_threads && shown < 40; ++i) {
    const Fiber& f = c->fibers[i];
    if (f.wait == DONE) continue;
    fprintf(stderr, "  thread %u: %s\n", i, f.wait == WAIT_BARRIER ? "at __syncthreads" : f.wait == WAIT_WARP ? "at a warp collective" : "?");
    ++shown;
  }
  abort();
}

void run_cta(Cta* c, dim3 grid, dim3 block, uint3 bid) {
  const unsigned n = block.x * block.y * block.z;
  c->n_threads = n;
  c->live = n;
  c->bar_arrived = 0;
  c->bar_or_acc = 0;
  for (unsigned w = 0; w < (n + 31) / 32; ++w) {
    Warp& W = c->warps[w];
    W.arrived[0] = W.arrived[1] = 0;
    W.gen = 0;
    const unsigned lanes = n - w * 32 >= 32 ? 32 : n - w * 32;
    W.live = lanes == 32 ? 0xffffffffu : ((1u << lanes) - 1u);
  }
  for (unsigned i = 0; i < n; ++i) {
    Fiber& f = c->fibers[i];
    f.tid = uint3{i % block.x, (i / block.x) % block.y, i / (block.x * block.y)};
    prepare_fiber(f);
#if defined(CUSIM_TSAN)
    f.tsan = __tsan_create_fiber(0);
#endif
  }
#if defined(CUSIM_TSAN)
  c->sched_tsan = __tsan_get_current_fiber();
  TSAN_RELEASE(&c->start_sync);
#endif
  tc.bid = bid;
  tc.bdim = uint3{block.x, block.y, block.z};
  tc.gdim = uint3{grid.x, grid.y, grid.z};
  // CUSIM_ORDER: fwd (default) | rev | rand — the order in which runnable threads are resumed within a pass. Results
  // must not depend on it; "rand" reshuffles every pass with a per-CTA seed.
  static const int order = [] { const char* e = getenv("CUSIM_ORDER"); return !e ? 0 : e[0] == 'r' && e[1] == 'e' ? 1 : e[0] == 'r' ? 2 : 0; }();
  uint64_t rng = 0x9E3779B97F4A7C15ull * (bid.x + 1u) + bid.y;
  unsigned done = 0;
  while (done < n) {
    bool progressed = false;
    unsigned rot = 0, stride = 1;
    if (order == 2) {
      rng = rng * 6364136223846793005ull + 1442695040888963407ull;
      rot = static_cast<unsigned>(rng >> 33) % n;
      stride = (n % 7u) ? 7u : ((n % 5u) ? 5u : ((n % 3u) ? 3u : 1u));  // co-prime with n for the usual block sizes
    }
    for (unsigned k = 0; k < n; ++k) {
      const unsigned i = order == 0 ? k : order == 1 ? n - 1 - k : static_cast<unsigned>((rot + static_cast<uint64_t>(k) * stride) % n);
      Fiber& f = c->fibers[i];
      if (f.wait == DONE) continue;
      if (f.wait == WAIT_BARRIER && c->bar_gen == f.wait_gen) continue;
      if (f.wait == WAIT_WARP && c->warps[f.wait_warp].gen == f.wait_gen) continue;
      f.wait = RUNNABLE;
      c->cur = i;
      tc.tid = f.tid;
#if CUSIM_ASAN
      __sanitizer_start_switch_fiber(&c->sched_fake_stack, f.stack, kStackBytes);
#endif
      TSAN_SWITCH(f.tsan);
      cusim_switch(&c->sched_sp, f.sp);
#if CUSIM_ASAN
      __sanitizer_finish_switch_fiber(c->sched_fake_stack, nullptr, nullptr);
#endif
      progressed = true;
      if (f.wait == DONE) ++done;
    }
    if (!progressed) deadlock_report(c);
  }
#if defined(CUSIM_TSAN)
  TSAN_ACQUIRE(&c->end_sync);
  for (unsigned i = 0; i < n; ++i) __tsan_destroy_fiber(c->fibers[i].tsan);
#endif
}

}  // namespace

int sm_count() {
  const char* e = getenv("CUSIM_SMS");
  const int v = e ? atoi(e) : 0;
  return v > 0 ? v : 132;
}

uint64_t globaltimer_ns() {
  return static_cast<uint64_t>(std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::steady_clock::now().time_since_epoch()).count());
}

unsigned lane_id() { return g_cta->cur & 31u; }

void* dyn_smem() { return g_cta->dyn; }

void register_shared(void* p, size_t bytes) {
  for (const auto& r : g_shared_regs) if (r.first == p) return;
  g_shared_regs.emplace_back(p, bytes);
}

void syncthreads() {
  Cta* c = g_cta;
  Fiber& f = c->fibers[c->cur];
  const uint32_t gen = c->bar_gen;
  TSAN_RELEASE(&c->bar_sync);
  c->bar_arrived++;
  release_barrier_if_complete(c);
  if (c->bar_gen == gen) {  // not the last arriver
    f.wait = WAIT_BARRIER;
    f.wait_gen = gen;
    yield_to_scheduler();
  }
  TSAN_ACQUIRE(&c->bar_sync);
}

int syncthreads_or(int pred) {
  Cta* c = g_cta;
  Fiber& f = c->fibers[c->cur];
  const uint32_t gen = c->bar_gen;
  TSAN_RELEASE(&c->bar_sync);
  c->bar_or_acc |= (pred != 0);
  c->bar_arrived++;
  release_barrier_if_complete(c);
  if (c->bar_gen == gen) {
    f.wait = WAIT_BARRIER;
    f.wait_gen = gen;
    yield_to_scheduler();
  }
  TSAN_ACQUIRE(&c->bar_sync);
  return c->bar_or_res[gen & 1u];
}

void poll_yield() {
  static const bool jitter = getenv("CUSIM_JITTER") != nullptr;
  if (jitter && (globaltimer_ns() & 63u) == 0u) std::this_thread::yield();
  Cta* c = g_cta;
  if (!c || c->n_threads <= 1) { std::this_thread::yield(); return; }
  c->fibers[c->cur].wait = WAIT_POLL;
  yield_to_scheduler();
}

const uint64_t* warp_exchange(unsigned mask, uint64_t v, unsigned* arrived_mask, int kind) {
#if defined(CUSIM_TSAN)
  static const bool strict = getenv("CUSIM_TSAN_STRICT") != nullptr;
  const bool fence = kind == 1 || !strict;
#else
  (void)kind;
#endif
  Cta* c = g_cta;
  const unsigned linear = c->cur, lane = linear & 31u;
  Warp& w = c->warps[linear >> 5];
  if (!((mask >> lane) & 1u)) {
    fprintf(stderr, "cusim: thread %u called a warp collective with mask %08x that excludes its own lane\n", linear, mask);
    abort();
  }
  const uint32_t gen = w.gen;
  const unsigned b = gen & 1u;
#if defined(CUSIM_TSAN)
  if (fence) TSAN_RELEASE(&w.gen);  // the collective orders the memory accesses of the lanes that take part in it
#endif
  w.slot[b][lane] = v;
  w.arrived[b] |= 1u << lane;
  release_warp_if_complete(w, mask);
  if (w.gen == gen) {
    Fiber& f = c->fibers[linear];
    f.wait = WAIT_WARP;
    f.wait_gen = gen;
    f.wait_warp = linear >> 5;
    yield_to_scheduler();
  }
#if defined(CUSIM_TSAN)
  if (fence) TSAN_ACQUIRE(&w.gen);
#endif
  *arrived_mask = w.arrived_final[b];
  return w.slot[b];
}

// ---- CUSIM_HOSTCHECK: device allocations the host may not touch ---------------------------------------------------------
static std::mutex g_dev_mutex;
static std::map<uintptr_t, size_t> g_dev_regions;  // base -> mapped bytes
static int g_dev_access = 0;
static bool hostcheck() {
#if CUSIM_ASAN || defined(CUSIM_TSAN)
  return false;
#else
  static const bool on = [] { const char* e = getenv("CUSIM_HOSTCHECK"); return e && e[0] == '1'; }();
  return on;
#endif
}
static void hostcheck_segv(int, siginfo_t* si, void*) {
  const uintptr_t a = reinterpret_cast<uintptr_t>(si->si_addr);
  bool ours = false;
  for (const auto& r : g_dev_regions) ours |= (a >= r.first && a < r.first + r.second);  // no lock: we are about to die
  if (ours) {
    static const char msg[] = "cusim hostcheck: host code touched device memory outside a kernel / cudaMemcpy (a segmentation fault on the GPU box)\n";
    (void)!write(2, msg, sizeof(msg) - 1);
  }
  signal(SIGSEGV, SIG_DFL);
  raise(SIGSEGV);
}
void* device_alloc(size_t bytes) {
  if (!hostcheck()) {
    void* p = nullptr;
    if (posix_memalign(&p, 256, bytes) != 0) return nullptr;
    memset(p, 0xCD, bytes);
    return p;
  }
  static const bool installed = [] {
    struct sigaction sa;
    memset(&sa, 0, sizeof(sa));
    sa.sa_sigaction = hostcheck_segv;
    sa.sa_flags = SA_SIGINFO;
    sigaction(SIGSEGV, &sa, nullptr);
    return true;
  }();
  (void)installed;
  const size_t mapped = (bytes + 4095) & ~static_cast<size_t>(4095);
  void* p = mmap(nullptr, mapped, PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS, -1, 0);
  if (p == MAP_FAILED) return nullptr;
  memset(p, 0xCD, mapped);
  std::lock_guard<std::mutex> lock(g_dev_mutex);
  g_dev_regions[reinterpret_cast<uintptr_t>(p)] = mapped;
  if (g_dev_access == 0) mprotect(p, mapped, PROT_NONE);
  return p;
}
void device_free(void* p) {
  if (!p) return;
  if (!hostcheck()) { free(p); return; }
  std::lock_guard<std::mutex> lock(g_dev_mutex);
  auto it = g_dev_regions.find(reinterpret_cast<uintptr_t>(p));
  if (it == g_dev_regions.end()) { fprintf(stderr, "cusim hostcheck: cudaFree of a pointer cudaMalloc did not return\n"); abort(); }
  munmap(p, it->second);
  g_dev_regions.erase(it);
}
void device_access_begin() {
  if (!hostcheck()) return;
  std::lock_guard<std::mutex> lock(g_dev_mutex);
  if (g_dev_access++ == 0) for (const auto& r : g_dev_regions) mprotect(reinterpret_cast<void*>(r.first), r.second, PROT_READ | PROT_WRITE);
}
void device_access_end() {
  if (!hostcheck()) return;
  std::lock_guard<std::mutex> lock(g_dev_mutex);
  if (--g_dev_access == 0) for (const auto& r : g_dev_regions) mprotect(reinterpret_cast<void*>(r.first), r.second, PROT_NONE);
}

// ---- CUSIM_ASYNC: device-to-host copies complete at the next synchronisation with their stream -----------------------------
struct PendingCopy { void* dst; std::vector<uint8_t> data; uint64_t seq; };
static std::mutex g_async_mutex;
static std::map<void*, std::deque<PendingCopy>> g_pending;         // per stream, in enqueue order
static std::map<void*, uint64_t> g_stream_seq;                      // copies enqueued so far on a stream
static std::map<void*, std::pair<void*, uint64_t>> g_events;        // event -> (stream, copies enqueued before the record)
static bool async_mode() {
  static const bool on = [] { const char* e = getenv("CUSIM_ASYNC"); return e && e[0] == '1'; }();
  return on;
}
static void deliver_locked(void* stream, uint64_t up_to) {
  auto it = g_pending.find(stream);
  if (it == g_pending.end()) return;
  while (!it->second.empty() && it->second.front().seq <= up_to) {
    PendingCopy& c = it->second.front();
    memcpy(c.dst, c.data.data(), c.data.size());
    it->second.pop_front();
  }
}
bool defer_d2h(void* dst, const void* src, size_t n, void* stream) {
  if (!async_mode() || n == 0) return false;
  std::lock_guard<std::mutex> lock(g_async_mutex);
  PendingCopy c{dst, std::vector<uint8_t>(static_cast<const uint8_t*>(src), static_cast<const uint8_t*>(src) + n), ++g_stream_seq[stream]};
  memset(dst, 0xEE, n);
  g_pending[stream].push_back(std::move(c));
  return true;
}
void flush_d2h(void* stream, bool all) {
  if (!async_mode()) return;
  std::lock_guard<std::mutex> lock(g_async_mutex);
  if (all) { for (auto& q : g_pending) deliver_locked(q.first, ~0ull); return; }
  deliver_locked(stream, ~0ull);
}
void event_record(void* event, void* stream) {
  if (!async_mode()) return;
  std::lock_guard<std::mutex> lock(g_async_mutex);
  g_events[event] = {stream, g_stream_seq[stream]};
}
void event_sync(void* event) {
  if (!async_mode()) return;
  std::lock_guard<std::mutex> lock(g_async_mutex);
  auto it = g_events.find(event);
  if (it != g_events.end()) deliver_locked(it->second.first, it->second.second);
}
void event_forget(void* event) {
  if (!async_mode()) return;
  std::lock_guard<std::mutex> lock(g_async_mutex);
  g_events.erase(event);
}

static HostLock g_attr_mutex;
static std::map<const void*, size_t> g_max_dyn_smem;
static thread_local int g_last_error = 0;  // like CUDA's: one error word per host thread
static HostLock g_launch_mutex;          // the emulated device runs one kernel at a time

// CUSIM_SMEM_MONOTONIC=1: a call that LOWERS a kernel's dynamic shared memory limit fails. The limit is one value per
// kernel for the whole process, so library code that lowers it can make a launch of another thread, which set a larger
// limit a moment earlier, fail; code that only ever raises it cannot. This mode finds the lowering calls without threads.
int set_max_dyn_smem(const void* kernel, int bytes) {
  if (bytes < 0 || bytes > 227 * 1024) return 1;  // cudaErrorInvalidValue
  static const bool monotonic = [] { const char* e = getenv("CUSIM_SMEM_MONOTONIC"); return e && e[0] == '1'; }();
  std::lock_guard<HostLock> lock(g_attr_mutex);
  auto it = g_max_dyn_smem.find(kernel);
  if (monotonic && it != g_max_dyn_smem.end() && static_cast<size_t>(bytes) < it->second) {
    fprintf(stderr, "cusim: cudaFuncSetAttribute lowers a kernel's dynamic shared memory limit from %zu to %d bytes (CUSIM_SMEM_MONOTONIC)\n", it->second, bytes);
    return 1;
  }
  g_max_dyn_smem[kernel] = static_cast<size_t>(bytes);
  return 0;
}
int take_last_error() { const int e = g_last_error; g_last_error = 0; return e; }

void launch(dim3 grid, dim3 block, size_t smem_bytes, const std::function<void()>& body, const void* kernel) {
  const uint64_t n_ctas = static_cast<uint64_t>(grid.x) * grid.y * grid.z;
  const unsigned n_threads = block.x * block.y * block.z;
  std::lock_guard<HostLock> one_kernel_at_a_time(g_launch_mutex);
  const std::thread::id host = std::this_thread::get_id();
  DeviceAccess device_access;
  if (kernel) {
    size_t allowed = 48 * 1024;
    {
      std::lock_guard<HostLock> lock(g_attr_mutex);
      auto it = g_max_dyn_smem.find(kernel);
      if (it != g_max_dyn_smem.end() && it->second > allowed) allowed = it->second;
    }
    if (smem_bytes > allowed) {
      fprintf(stderr, "cusim: launch with %zu bytes of dynamic shared memory, the kernel's limit is %zu (cudaFuncSetAttribute missing?)\n", smem_bytes, allowed);
      g_last_error = 1;
      return;
    }
  }
  if (n_ctas == 0 || n_threads == 0 || grid.y > 65535u || grid.z > 65535u || grid.x > 0x7FFFFFFFu || n_threads > 1024u) {
    // cudaErrorInvalidConfiguration on the GPU (an empty grid included): nothing runs and the error is left for
    // cudaGetLastError — a caller that launches unconditionally must see it here too
    fprintf(stderr, "cusim: invalid launch configuration: grid (%u,%u,%u) block (%u,%u,%u)\n", grid.x, grid.y, grid.z, block.x, block.y, block.z);
    g_last_error = 9;
    return;
  }
  if (n_threads > kMaxThreads) { fprintf(stderr, "cusim: block of %u threads\n", n_threads); abort(); }
  unsigned workers = std::thread::hardware_concurrency();
  if (const char* e = getenv("CUSIM_WORKERS")) workers = static_cast<unsigned>(atoi(e));
  if (workers < 1) workers = 1;
  if (workers > 16) workers = 16;
  if (workers > n_ctas) workers = static_cast<unsigned>(n_ctas);
  std::atomic<uint64_t> next{0};
  auto worker = [&](Cta* c) {
    g_cta = c;
    c->body = &body;
#if CUSIM_ASAN
    // exactly the bytes the launch asked for (rounded to the 16-byte granularity the kernels' staged copies may read),
    // so that a kernel running past its dynamic shared memory hits a redzone
    free(c->dyn);
    c->dyn_cap = ((smem_bytes + 15) & ~static_cast<size_t>(15)) + 64;
    if (posix_memalign(&c->dyn, 1024, c->dyn_cap - 64 ? c->dyn_cap - 64 : 16) != 0) abort();
#else
    if (smem_bytes + 64 > c->dyn_cap) {
      free(c->dyn);
      c->dyn_cap = smem_bytes + 64 < (256u << 10) ? (256u << 10) : smem_bytes + 64;
      if (posix_memalign(&c->dyn, 1024, c->dyn_cap) != 0) abort();
    }
#endif
    for (;;) {
      const uint64_t i = next.fetch_add(1);  // in-order dispatch, like the hardware's block scheduler
      if (i >= n_ctas) break;
      // poison shared memory so that reads of never-written bytes are reproducible and loud: the dynamic part always,
      // the static variables from the second CTA of this OS thread on (they register when their declaration first runs)
      for (const auto& r : g_shared_regs) memset(r.first, 0xA5, r.second);
      memset(c->dyn, 0xA5, CUSIM_ASAN ? c->dyn_cap - 64 : smem_bytes + 64);
      // CUSIM_JITTER=1: CTAs start after a random delay (and pollers give up their time slice now and then), so that the
      // inter-CTA protocols see many more interleavings than the OS scheduler produces on its own
      static const bool jitter = getenv("CUSIM_JITTER") != nullptr;
      if (jitter) {
        const uint64_t h = (i + 1) * 0x9E3779B97F4A7C15ull ^ static_cast<uint64_t>(globaltimer_ns());
        std::this_thread::sleep_for(std::chrono::microseconds((h >> 40) % 300));
      }
      const uint3 bid{static_cast<unsigned>(i % grid.x), static_cast<unsigned>((i / grid.x) % grid.y),
                      static_cast<unsigned>(i / (static_cast<uint64_t>(grid.x) * grid.y))};
      run_cta(c, grid, block, bid);
    }
    g_cta = nullptr;
  };
  // always on fresh OS threads: the caller's thread keeps its own (possibly small) stack out of the picture
  std::vector<Cta*> ctas(workers);
  for (Cta*& c : ctas) c = acquire_cta(host);
  std::vector<std::thread> pool;
  pool.reserve(workers);
  for (unsigned w = 0; w < workers; ++w) pool.emplace_back(worker, ctas[w]);
  for (auto& t : pool) t.join();
  for (Cta* c : ctas) release_cta(c, host);
}

}  // namespace cusim
