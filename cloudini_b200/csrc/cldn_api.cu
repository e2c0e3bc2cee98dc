// C-ABI layer: handles, device memory, stream plumbing and kernel launches. See include/cloudini_b200.h.
// There is deliberately no CPU implementation of the codec here: if CUDA is unavailable every compute entry point
// fails with CLDN_ERR_CUDA.
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <sched.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <memory>
#include <mutex>
#include <new>
#include <stdexcept>
#include <utility>
#include <string>
#include <vector>

#include "cldn_device.cuh"
#include "cldn_kernels.h"
#include "cldn_plan.h"

namespace cldn {
std::string info_to_yaml(const cldn_info_t& info);
int info_from_yaml(const char* yaml, size_t len, cldn_info_t* info);
size_t max_compressed_size(const cldn_info_t& info, size_t points, bool include_header, bool* ok);
std::vector<uint8_t> make_header(const cldn_info_t& info);
}  // namespace cldn

using namespace cldn;

#define CUDA_TRY(expr)                                                                          \
  do {                                                                                          \
    cudaError_t e__ = (expr);                                                                   \
    if (e__ != cudaSuccess) {                                                                   \
      set_error("CUDA error %s at %s:%d: %s", cudaGetErrorName(e__), __FILE__, __LINE__, cudaGetErrorString(e__)); \
      return CLDN_ERR_CUDA;                                                                     \
    }                                                                                           \
  } while (0)

namespace {

// Grow-only device / pinned-host buffers, freed with their handle.
template <typename T>
struct DevBuf {
  T* p = nullptr;
  size_t cap = 0;
  DevBuf() = default;
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
  ~DevBuf() { if (p) cudaFree(p); }
  int reserve(size_t n, bool zero = false) {
    if (n <= cap) return CLDN_OK;
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
    size_t want = std::max<size_t>(n, 16);
    CUDA_TRY(cudaMalloc(reinterpret_cast<void**>(&p), want * sizeof(T)));
    cap = want;
    if (zero) {
      // cudaMemset runs on the legacy stream and is asynchronous to the host; the handles' streams are non-blocking and
      // would not order their kernels behind it, so the zeroes are made final here (growth is rare)
      CUDA_TRY(cudaMemset(p, 0, want * sizeof(T)));
      CUDA_TRY(cudaDeviceSynchronize());
    }
    return CLDN_OK;
  }
};
template <typename T>
struct PinBuf {
  T* p = nullptr;
  size_t cap = 0;
  PinBuf() = default;
  PinBuf(const PinBuf&) = delete;
  PinBuf& operator=(const PinBuf&) = delete;
  ~PinBuf() { if (p) cudaFreeHost(p); }
  int reserve(size_t n) {
    if (n <= cap) return CLDN_OK;
    if (p) cudaFreeHost(p);
    p = nullptr;
    cap = 0;
    size_t want = std::max<size_t>(n, 16);
    CUDA_TRY(cudaMallocHost(reinterpret_cast<void**>(&p), want * sizeof(T)));
    cap = want;
    return CLDN_OK;
  }
};

// Ring of pinned upload slots: a slot is only rewritten by the host after the async copy that read it has completed
// (back-to-back asynchronous batch calls would otherwise race on a single pinned table).
template <typename T, int SLOTS = 8>
struct PinRing {
  PinBuf<T> slot[SLOTS];
  cudaEvent_t ev[SLOTS] = {};
  bool used[SLOTS] = {};
  int next = 0;
  PinRing() = default;
  PinRing(const PinRing&) = delete;
  PinRing& operator=(const PinRing&) = delete;
  ~PinRing() { for (cudaEvent_t e : ev) if (e) cudaEventDestroy(e); }
  // returns a host pointer with room for n elements
  int acquire(size_t n, T** out, int* idx) {
    const int i = next;
    next = (next + 1) % SLOTS;
    if (used[i]) CUDA_TRY(cudaEventSynchronize(ev[i]));
    if (!ev[i]) CUDA_TRY(cudaEventCreateWithFlags(&ev[i], cudaEventDisableTiming));
    if (int rc = slot[i].reserve(n)) return rc;
    *out = slot[i].p;
    *idx = i;
    return CLDN_OK;
  }
  int commit(int idx, cudaStream_t stream) {
    CUDA_TRY(cudaEventRecord(ev[idx], stream));
    used[idx] = true;
    return CLDN_OK;
  }
};

// Extra streams + an event pool for the host-pointer path: frame f+1 is uploaded while frame f is encoded and
// frame f-1 is downloaded (PCIe is full duplex), instead of one serial copy-compute-copy sequence.
struct CopyPipeline {
  cudaStream_t h2d = nullptr, d2h = nullptr;
  std::vector<cudaEvent_t> ev;
  CopyPipeline() = default;
  CopyPipeline(const CopyPipeline&) = delete;
  CopyPipeline& operator=(const CopyPipeline&) = delete;
  ~CopyPipeline() {
    for (cudaEvent_t e : ev) cudaEventDestroy(e);
    if (h2d) cudaStreamDestroy(h2d);
    if (d2h) cudaStreamDestroy(d2h);
  }
  int ensure(size_t n_events) {
    if (!h2d) CUDA_TRY(cudaStreamCreateWithFlags(&h2d, cudaStreamNonBlocking));
    if (!d2h) CUDA_TRY(cudaStreamCreateWithFlags(&d2h, cudaStreamNonBlocking));
    while (ev.size() < n_events) {
      cudaEvent_t e;
      CUDA_TRY(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
      ev.push_back(e);
    }
    return CLDN_OK;
  }
};

// ---- stage 2 (general-purpose compression of every chunk) ---------------------------------------------------------
// Not the product (north_star: delegated / bypassed) and not part of the GPU path: when a caller asks for LZ4 / ZSTD
// through the HOST-pointer API, the stage-1 bytes produced by the kernels are handed chunk by chunk to the system's
// liblz4 / libzstd (dlopen, like the reference links them: codec_common.cpp:220-299). Compressed bytes are not
// expected to equal the reference's (different library versions); they decompress to the same stage-1 bytes.
struct Stage2 {
  void* lz4 = nullptr;
  void* zstd = nullptr;
  int (*lz4_compress)(const char*, char*, int, int) = nullptr;
  int (*lz4_decompress)(const char*, char*, int, int) = nullptr;
  size_t (*zstd_compress)(void*, size_t, const void*, size_t, int) = nullptr;
  size_t (*zstd_decompress)(void*, size_t, const void*, size_t) = nullptr;
  unsigned (*zstd_is_error)(size_t) = nullptr;
  std::mutex mutex;  // handles on several threads may load a library first at the same time
  bool load(int option) {
    std::lock_guard<std::mutex> lock(mutex);
    if (option == CLDN_COMP_LZ4) {
      if (!lz4) {
        lz4 = dlopen("liblz4.so.1", RTLD_NOW);
        if (!lz4) lz4 = dlopen("liblz4.so", RTLD_NOW);
        if (lz4) {
          lz4_compress = reinterpret_cast<int (*)(const char*, char*, int, int)>(dlsym(lz4, "LZ4_compress_default"));
          lz4_decompress = reinterpret_cast<int (*)(const char*, char*, int, int)>(dlsym(lz4, "LZ4_decompress_safe"));
        }
      }
      if (!lz4_compress || !lz4_decompress) { set_error("stage 2: liblz4 is not available on this host"); return false; }
      return true;
    }
    if (!zstd) {
      zstd = dlopen("libzstd.so.1", RTLD_NOW);
      if (!zstd) zstd = dlopen("libzstd.so", RTLD_NOW);
      if (zstd) {
        zstd_compress = reinterpret_cast<size_t (*)(void*, size_t, const void*, size_t, int)>(dlsym(zstd, "ZSTD_compress"));
        zstd_decompress = reinterpret_cast<size_t (*)(void*, size_t, const void*, size_t)>(dlsym(zstd, "ZSTD_decompress"));
        zstd_is_error = reinterpret_cast<unsigned (*)(size_t)>(dlsym(zstd, "ZSTD_isError"));
      }
    }
    if (!zstd_compress || !zstd_decompress || !zstd_is_error) { set_error("stage 2: libzstd is not available on this host"); return false; }
    return true;
  }
};
static Stage2 g_stage2;

// Re-frames a stage-1 payload ([u32 size][body])* into ([u32 csize][compressed body])* — WriteStage1Chunk, chunk_writer.cpp:42-47.
static int stage2_compress_payload(int option, const uint8_t* src, size_t src_bytes, uint8_t* dst, size_t dst_cap, size_t* written) {
  size_t ip = 0, op = 0;
  while (ip < src_bytes) {
    uint32_t sz;
    memcpy(&sz, src + ip, 4);
    ip += 4;
    if (dst_cap - op < 4) { set_error("Output buffer too small for compressed chunk"); return CLDN_ERR_BUFFER_TOO_SMALL; }
    uint32_t csz = 0;
    if (option == CLDN_COMP_LZ4) {  // codec_common.cpp:232-237
      const int c = g_stage2.lz4_compress(reinterpret_cast<const char*>(src + ip), reinterpret_cast<char*>(dst + op + 4), static_cast<int>(sz),
                                          static_cast<int>(std::min<size_t>(dst_cap - op - 4, 0x7FFFFFFF)));
      if (c <= 0) { set_error("LZ4 compression failed"); return CLDN_ERR_BUFFER_TOO_SMALL; }
      csz = static_cast<uint32_t>(c);
    } else {                        // ZSTD level 1, codec_common.cpp:242
      const size_t c = g_stage2.zstd_compress(dst + op + 4, dst_cap - op - 4, src + ip, sz, 1);
      if (g_stage2.zstd_is_error(c)) { set_error("ZSTD compression failed"); return CLDN_ERR_BUFFER_TOO_SMALL; }
      csz = static_cast<uint32_t>(c);
    }
    memcpy(dst + op, &csz, 4);
    op += 4 + csz;
    ip += sz;
  }
  *written = op;
  return CLDN_OK;
}

// Inverse: ([u32 csize][compressed])* -> ([u32 size][stage-1 body])*; `max_body` bounds a decompressed chunk.
static int stage2_decompress_payload(int option, const uint8_t* src, size_t src_bytes, std::vector<uint8_t>& dst, size_t max_body) {
  size_t ip = 0;
  dst.clear();
  while (ip < src_bytes) {
    if (src_bytes - ip < 4) { set_error("decode: not enough input data"); return CLDN_ERR_CORRUPT_DATA; }
    uint32_t csz;
    memcpy(&csz, src + ip, 4);
    ip += 4;
    if (csz > src_bytes - ip) { set_error("Invalid chunk size found while decoding"); return CLDN_ERR_CORRUPT_DATA; }
    const size_t at = dst.size();
    dst.resize(at + 4 + max_body);
    uint32_t sz = 0;
    if (option == CLDN_COMP_LZ4) {
      const int r = g_stage2.lz4_decompress(reinterpret_cast<const char*>(src + ip), reinterpret_cast<char*>(dst.data() + at + 4), static_cast<int>(csz),
                                            static_cast<int>(std::min<size_t>(max_body, 0x7FFFFFFF)));
      if (r < 0) { set_error("LZ4 decompression failed"); return CLDN_ERR_CORRUPT_DATA; }
      sz = static_cast<uint32_t>(r);
    } else {
      const size_t r = g_stage2.zstd_decompress(dst.data() + at + 4, max_body, src + ip, csz);
      if (g_stage2.zstd_is_error(r)) { set_error("ZSTD decompression failed"); return CLDN_ERR_CORRUPT_DATA; }
      sz = static_cast<uint32_t>(r);
    }
    memcpy(dst.data() + at, &sz, 4);
    dst.resize(at + 4 + sz);
    ip += csz;
  }
  return CLDN_OK;
}

int select_device(int device) {
  int count = 0;
  cudaError_t e = cudaGetDeviceCount(&count);
  if (e != cudaSuccess || count == 0) {
    set_error("no CUDA device available (%s): cloudini_b200 has no CPU fallback", e == cudaSuccess ? "device count 0" : cudaGetErrorString(e));
    return CLDN_ERR_CUDA;
  }
  if (device >= 0) CUDA_TRY(cudaSetDevice(device));
  return CLDN_OK;
}

const char* dev_error_text(uint32_t code) {
  switch (code) {
    case DEV_ERR_TRUNCATED: return "Truncated encoded data: not enough bytes for a complete point";
    case DEV_ERR_VARINT_OVERFLOW: return "decodeVarint: value overflow";
    case DEV_ERR_NAN_MARKER: return "decodeVarint: unexpected NaN marker";
    case DEV_ERR_TRAILING: return "V5 chunk has trailing bytes after decode";
    case DEV_ERR_BAD_MODE: return "V5 adaptive int: missing or unknown mode byte";
    case DEV_ERR_PALETTE: return "V5 adaptive int: bad palette section";
    case DEV_ERR_RLE: return "V5 adaptive int: bad run-length section";
    case DEV_ERR_CHUNK_SIZE: return "Invalid chunk size found while decoding";
    case DEV_ERR_CHUNK_COUNT: return "Encoded data does not match the declared number of points (chunk count)";
    case DEV_ERR_OUTPUT_SMALL: return "Output buffer is too small to hold the decoded data";
    case DEV_ERR_ENCODE_OUTPUT_SMALL: return "Output buffer too small for uncompressed chunk";  // chunk_writer.cpp:33-35
    case DEV_ERR_LZ4: return "LZ4 decompression failed";  // codec_common.cpp:279-281
    case DEV_ERR_ZSTD: return "ZSTD decompression failed";  // codec_common.cpp:290-293
    default: return "unknown device error";
  }
}

}  // namespace

// =====================================================================================================================
// What the kernels read about one layout: an encoder has one, a mixed encoder (cldn_b200_encode_mixed_blobs) one per
// layout it has met.
struct EncLayout {
  cldn_info_t info;       // as given, except compression_opt = NONE (what the GPU path produces)
  cldn_info_t blob_info;  // the blob's layout: as given, compression_opt as declared
  int stage2 = 0;         // the caller's compression_opt
  Plan plan;
  std::vector<uint8_t> header;
  uint32_t tile_points = 0;
  DevBuf<Plan> d_plan;
  DevBuf<uint8_t> d_header;
};

// The stream and the scratch of a handle, shared by every layout it encodes.
struct EncScratch {
  bool stage2_on_device = false;  // cldn_b200_encoder_set_stage2_on_device
  std::vector<uint8_t> s2_tmp;
  int device = 0;
  cudaStream_t stream = nullptr;
  bool own_stream = false;
  uint32_t epoch = 0;
  size_t sizes_at = 0;  // first d_sizes slot of the frames being encoded (cldn_b200_encode_mixed_blobs: of the group)

  DevBuf<uint64_t> d_status;
  DevBuf<uint32_t> d_ticket;  // tile ticket of the persistent XYZI kernel
  DevBuf<EncFrame> d_frames;
  PinRing<EncFrame> h_frames;
  DevBuf<uint64_t> d_sizes;
  PinBuf<uint64_t> h_sizes;
  DevBuf<uint32_t> d_err;
  PinBuf<uint32_t> h_err;
  // host-memory path staging
  DevBuf<uint8_t> d_in, d_out;
  CopyPipeline pipe;
  // V5 section scratch
  DevBuf<uint8_t> d_modes;
  DevBuf<uint8_t> d_sec_scratch;
  DevBuf<uint32_t> d_sec_sizes;
  DevBuf<uint32_t> d_sec_excl;
  DevBuf<uint32_t> d_chunk_frame;
  PinRing<uint32_t> h_chunk_frame;
  DevBuf<uint64_t> d_hash;
  DevBuf<uint8_t> d_gorilla;  // Gorilla pre-pass records: [frame][op][point][12]
  // stage 2 on the device (LZ4, ZSTD): stage-1 arena, per-chunk (LZ4) / per-block (ZSTD) slots, chunk tables
  DevBuf<uint8_t> d_s1, d_lz_scratch;
  DevBuf<uint32_t> d_lz_chunk_frame, d_lz_chunk_sizes;
  DevBuf<Lz4Frame> d_lz_frames;
  PinRing<Lz4Frame> h_lz_frames;
  PinRing<uint32_t> h_lz_chunk_frame;
  // cldn_b200_encode_blobs: blob addresses, header offsets and the packed headers of a batch (launch_place_headers)
  DevBuf<uint8_t> d_blob_headers;
  PinRing<uint8_t> h_blob_headers;
};

struct AsyncEncode;  // cldn_b200_encoder_prepare_blobs
struct AsyncEncodeDeleter { void operator()(AsyncEncode* a) const; };

struct cldn_encoder : EncLayout, EncScratch {
  bool pooled = false;  // a handle of the per-thread pool (encoder_mark_pooled): keeps the libraries' bytes
  std::unique_ptr<AsyncEncode, AsyncEncodeDeleter> async;  // the prepared shape of cldn_b200_encode_blobs_async
};

// cldn_b200_encoder_create's refusals, in its order, and the host part of the layout of `info`.
static int plan_layout(const cldn_info_t& info, EncLayout& l) {
  Plan plan;
  if (int rc = build_encode_plan(info, &plan)) return rc;
  if (!plan.supported) {
    set_error("EncodingInfo contains a field encoder this build cannot run");
    return CLDN_ERR_UNSUPPORTED;
  }
  if (info.compression_opt > CLDN_COMP_ZSTD) { set_error("Unsupported compression option"); return CLDN_ERR_INVALID_ARGUMENT; }
  // ZSTD exists only as the host library; LZ4 also runs on the device, so a missing liblz4 only matters to the host-pointer API
  if (info.compression_opt == CLDN_COMP_ZSTD && !g_stage2.load(info.compression_opt)) return CLDN_ERR_UNSUPPORTED;
  l.info = info;
  l.blob_info = info;
  l.stage2 = info.compression_opt;        // the header declares it; the kernels always produce stage 1
  l.info.compression_opt = CLDN_COMP_NONE;
  l.plan = plan;
  l.header = make_header(info);
  l.tile_points = choose_tile_points(plan);
  return CLDN_OK;
}

// The device copies of the plan and the header (synchronous).
static int upload_layout(EncLayout& l) {
  if (int rc = l.d_plan.reserve(1)) return rc;
  if (int rc = l.d_header.reserve(l.header.size())) return rc;
  cudaError_t ce = cudaMemcpy(l.d_plan.p, &l.plan, sizeof(Plan), cudaMemcpyHostToDevice);
  if (ce == cudaSuccess) ce = cudaMemcpy(l.d_header.p, l.header.data(), l.header.size(), cudaMemcpyHostToDevice);
  if (ce != cudaSuccess) { set_error("cudaMemcpy failed: %s", cudaGetErrorString(ce)); return CLDN_ERR_CUDA; }
  return CLDN_OK;
}

// LZ4_COMPRESSBOUND (lz4.h): worst case of a block for n input bytes
static size_t lz4_bound(size_t n) { return n + n / 255 + 16; }

// The header of a layout with width = height = 0, cut around the two numbers: tmpl = part 0 | part 1 | part 2 with
// len[k] bytes each, so that the header of dims (w, h) is part 0, "%u" of w, part 1, "%u" of h, part 2. The headers the
// prepared async calls write (encode) and accept (decode) are built from it on the device.
static int header_template(const std::vector<uint8_t>& hdr, std::vector<uint8_t>* tmpl, uint32_t len[3]) {
  const std::string text(reinterpret_cast<const char*>(hdr.data()), hdr.size());
  const size_t w_at = text.find("\nwidth: 0\nheight: 0\n");
  if (w_at == std::string::npos) { set_error("the layout's header has no width / height lines"); return CLDN_ERR_INTERNAL; }
  len[0] = static_cast<uint32_t>(w_at + 8);
  len[1] = 9;
  len[2] = static_cast<uint32_t>(hdr.size() - (w_at + 19));
  tmpl->assign(hdr.begin(), hdr.begin() + len[0]);
  tmpl->insert(tmpl->end(), hdr.begin() + len[0] + 1, hdr.begin() + len[0] + 1 + len[1]);
  tmpl->insert(tmpl->end(), hdr.begin() + w_at + 19, hdr.end());
  return CLDN_OK;
}

namespace cldn {
void encoder_mark_pooled(cldn_encoder_t* enc) { enc->pooled = true; }
}  // namespace cldn

static int check_device_error(cudaStream_t stream, uint32_t* d_err, uint32_t* h_err) {
  CUDA_TRY(cudaMemcpyAsync(h_err, d_err, sizeof(uint32_t), cudaMemcpyDeviceToHost, stream));
  CUDA_TRY(cudaStreamSynchronize(stream));
  if (*h_err != DEV_OK) {
    const uint32_t code = *h_err;
    cudaMemsetAsync(d_err, 0, sizeof(uint32_t), stream);
    set_error("%s", dev_error_text(code));
    return code == DEV_ERR_ENCODE_OUTPUT_SMALL ? CLDN_ERR_BUFFER_TOO_SMALL : CLDN_ERR_CORRUPT_DATA;
  }
  return CLDN_OK;
}

extern "C" {

uint64_t cldn_b200_kernel_launch_count(void) { return kernel_launch_count(); }

int cldn_b200_bind_host_thread_to_device(int device) {
  if (int rc = select_device(device)) return rc;
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return 0;
  char bus_id[64] = {0};
  if (cudaDeviceGetPCIBusId(bus_id, sizeof(bus_id), dev) != cudaSuccess) return 0;
  // NVML through dlopen: the library has no link-time dependency on it
  static void* nvml = dlopen("libnvidia-ml.so.1", RTLD_NOW);
  if (!nvml) return 0;
  using InitFn = int (*)();
  using HandleFn = int (*)(const char*, void**);
  using AffFn = int (*)(void*, unsigned int, unsigned long*);
  InitFn init = reinterpret_cast<InitFn>(dlsym(nvml, "nvmlInit_v2"));
  HandleFn by_bus = reinterpret_cast<HandleFn>(dlsym(nvml, "nvmlDeviceGetHandleByPciBusId_v2"));
  AffFn affinity = reinterpret_cast<AffFn>(dlsym(nvml, "nvmlDeviceGetCpuAffinity"));
  if (!init || !by_bus || !affinity || init() != 0) return 0;
  void* handle = nullptr;
  if (by_bus(bus_id, &handle) != 0) return 0;
  constexpr unsigned kWords = 16;  // 1024 CPUs
  unsigned long words[kWords] = {0};
  if (affinity(handle, kWords, words) != 0) return 0;
  cpu_set_t set;
  CPU_ZERO(&set);
  int count = 0;
  for (unsigned w = 0; w < kWords; ++w) {
    for (unsigned b = 0; b < 8 * sizeof(unsigned long); ++b) {
      if ((words[w] >> b) & 1ul) { CPU_SET(w * 8 * sizeof(unsigned long) + b, &set); ++count; }
    }
  }
  if (count == 0 || sched_setaffinity(0, sizeof(set), &set) != 0) return 0;
  return count;
}

int cldn_b200_encoder_create(const cldn_info_t* info, int device, void* stream, cldn_encoder_t** out) {
  if (!info || !out) { set_error("null argument"); return CLDN_ERR_INVALID_ARGUMENT; }
  *out = nullptr;
  cldn_encoder* e = new cldn_encoder();
  if (int rc = plan_layout(*info, *e)) { delete e; return rc; }
  if (int rc = select_device(device)) { delete e; return rc; }
  cudaGetDevice(&e->device);
  if (stream) {
    e->stream = static_cast<cudaStream_t>(stream);
  } else {
    if (cudaStreamCreateWithFlags(&e->stream, cudaStreamNonBlocking) != cudaSuccess) {
      set_error("cudaStreamCreate failed");
      delete e;
      return CLDN_ERR_CUDA;
    }
    e->own_stream = true;
  }
  int rc = upload_layout(*e);
  if (!rc) rc = e->d_err.reserve(1, true);
  if (!rc) rc = e->h_err.reserve(1);
  if (rc) { cldn_b200_encoder_destroy(e); return rc; }
  *out = e;
  return CLDN_OK;
}

void cldn_b200_encoder_destroy(cldn_encoder_t* e) {
  if (!e) return;
  cudaSetDevice(e->device);
  if (e->stream) cudaStreamSynchronize(e->stream);
  const cudaStream_t own = e->own_stream ? e->stream : nullptr;
  delete e;  // the buffers free themselves
  if (own) cudaStreamDestroy(own);
}

int cldn_b200_encoder_header(const cldn_encoder_t* enc, const uint8_t** header, size_t* header_bytes) {
  if (!enc) { set_error("null encoder"); return CLDN_ERR_INVALID_ARGUMENT; }
  if (header) *header = enc->header.data();
  if (header_bytes) *header_bytes = enc->header.size();
  return CLDN_OK;
}

int cldn_b200_encoder_info(const cldn_encoder_t* enc, cldn_info_t* info) {
  if (!enc || !info) { set_error("null argument"); return CLDN_ERR_INVALID_ARGUMENT; }
  *info = enc->blob_info;
  return CLDN_OK;
}

const uint64_t* cldn_b200_encoder_sizes_device(const cldn_encoder_t* enc) { return enc ? enc->d_sizes.p : nullptr; }

int cldn_b200_encoder_set_dims(cldn_encoder_t* e, uint32_t width, uint32_t height) {
  if (!e) { set_error("null encoder"); return CLDN_ERR_INVALID_ARGUMENT; }
  if (e->info.width == width && e->info.height == height) return CLDN_OK;
  CUDA_TRY(cudaSetDevice(e->device));
  e->info.width = e->blob_info.width = width;
  e->info.height = e->blob_info.height = height;
  const std::vector<uint8_t> h = make_header(e->blob_info);
  // the device copy of the previous header may still be read by kernels in flight on the handle's stream
  CUDA_TRY(cudaStreamSynchronize(e->stream));
  if (int rc = e->d_header.reserve(h.size())) return rc;
  CUDA_TRY(cudaMemcpy(e->d_header.p, h.data(), h.size(), cudaMemcpyHostToDevice));
  e->header = h;
  return CLDN_OK;
}

int cldn_b200_encoder_set_stage2_on_device(cldn_encoder_t* e, int on) {
  if (!e) { set_error("null encoder"); return CLDN_ERR_INVALID_ARGUMENT; }
  if (on != 0 && on != 1) { set_error("on must be 0 or 1"); return CLDN_ERR_INVALID_ARGUMENT; }
  if (on == 1 && e->pooled) {
    set_error("a pool encoder (cldn_b200_pool_encoder) keeps the system libraries' stage-2 bytes: create an encoder of your own");
    return CLDN_ERR_INVALID_ARGUMENT;
  }
  e->stage2_on_device = on == 1;
  return CLDN_OK;
}

int cldn_b200_encoder_sync(cldn_encoder_t* e) {
  if (!e) { set_error("null encoder"); return CLDN_ERR_INVALID_ARGUMENT; }
  CUDA_TRY(cudaSetDevice(e->device));
  return check_device_error(e->stream, e->d_err.p, e->h_err.p);
}

}  // extern "C"

// No C++ exception may cross the C ABI (std::terminate under ctypes / C callers): allocation failures become a status.
template <class Fn>
static int guarded(Fn&& fn) {
  try {
    return fn();
  } catch (const std::bad_alloc&) {
    set_error("out of memory");
    return CLDN_ERR_INTERNAL;
  } catch (const std::exception& ex) {
    set_error("internal error: %s", ex.what());
    return CLDN_ERR_INTERNAL;
  }
}

// The encoder's rules for one frame, which every entry point checks on all frames before it uploads or launches
// anything: the reference's checks in its order (cloudini.cpp:523-534), then this library's own. `hdr` is the header
// bytes written in front of the payload at `out`.
static int check_encode_frame(const EncLayout& l, size_t hdr, const void* cloud, size_t cloud_bytes, const void* out,
                              size_t out_capacity) {
  const cldn_info_t& blob = l.blob_info;
  if (blob.point_step == 0) { set_error("point_step cannot be 0"); return CLDN_ERR_INVALID_ARGUMENT; }
  if (cloud_bytes % blob.point_step != 0) { set_error("Input cloud_data size is not a multiple of point_step"); return CLDN_ERR_INVALID_ARGUMENT; }
  const size_t n = cloud_bytes / blob.point_step;
  bool ok;
  const size_t need = max_compressed_size(blob, n, false, &ok) + hdr;
  if (!ok) return CLDN_ERR_INVALID_ARGUMENT;
  if (out_capacity < need) { set_error("Output buffer too small for worst-case compressed size"); return CLDN_ERR_BUFFER_TOO_SMALL; }
  if (n > 0xFFFFFFFFull) { set_error("too many points in one frame"); return CLDN_ERR_UNSUPPORTED; }
  if ((n > 0 && !cloud) || (need > 0 && !out)) { set_error("null frame pointer"); return CLDN_ERR_INVALID_ARGUMENT; }
  return CLDN_OK;
}

// How a batch is encoded. Device routes write CLDN_MEM_DEVICE blobs; host routes write host blobs from host clouds
// (CLDN_MEM_HOST) or device clouds (CLDN_MEM_DEVICE_POINTS).
enum EncodeRoute {
  kEncDevice,        // stage 1
  kEncDeviceStage2,  // stage 1, then LZ4 / ZSTD on the device
  kEncHostPlain,     // stage 1, pipelined upload / encode / download
  kEncHostStage2,    // stage 1 and LZ4 / ZSTD on the device, then download
  kEncHostLibrary,   // stage 1, download, then liblz4 / libzstd on the host
};

// The route for this encoder and memory kind, or the refusal. LZ4 runs on the device for device blobs; ZSTD, and LZ4
// into host blobs, run on the device only when the caller asked for it (cldn_b200_encoder_set_stage2_on_device).
static int choose_encode_route(const EncLayout& l, const EncScratch& s, int mem, EncodeRoute* route) {
  if (mem != CLDN_MEM_HOST && mem != CLDN_MEM_DEVICE && mem != CLDN_MEM_DEVICE_POINTS) { set_error("bad mem kind"); return CLDN_ERR_INVALID_ARGUMENT; }
  const bool device_blobs = mem == CLDN_MEM_DEVICE;
  if (l.stage2 == CLDN_COMP_NONE) {
    *route = device_blobs ? kEncDevice : kEncHostPlain;
  } else if (s.stage2_on_device || (device_blobs && l.stage2 == CLDN_COMP_LZ4)) {
    *route = device_blobs ? kEncDeviceStage2 : kEncHostStage2;
  } else if (device_blobs) {
    set_error("compression_opt %d needs the host-pointer API: ZSTD is delegated to the host library (LZ4 runs on the device)", l.stage2);
    return CLDN_ERR_UNSUPPORTED;
  } else {
    if (!g_stage2.load(l.stage2)) return CLDN_ERR_UNSUPPORTED;
    *route = kEncHostLibrary;
  }
  return CLDN_OK;
}

// The internal stage-1 arena of the compressed routes for a frame of n points: the stage-1 worst case plus 64 bytes per
// chunk and 64 more.
static size_t stage1_arena_bytes(const EncLayout& l, size_t n) {
  bool ok;
  return max_compressed_size(l.info, n, false, &ok) + 64 * ((n + kChunkPoints - 1) / kChunkPoints + 1);
}

// Device staging of a plain host blob. A committed V5 mode can exceed the reference's own worst-case formula (DeltaRle on
// a 64-bit field: 11 bytes per value against the 10 it budgets); the reference then succeeds iff the caller's buffer is
// large enough. Stage with room for the real worst case, never more than the caller gave: the kernels check every store
// against this bound.
static size_t plain_blob_staging(const EncLayout& l, size_t hdr, size_t cloud_bytes, size_t out_capacity) {
  const size_t n = cloud_bytes / l.info.point_step;
  bool ok;
  size_t worst = max_compressed_size(l.info, n, false, &ok) + hdr;
  for (uint32_t s = 0; s < l.plan.n_sections; ++s) {
    if (l.plan.sections[s].bpv == 8) worst += n + 16 * (n / kChunkPoints + 1);
  }
  return std::min(out_capacity, worst);
}

// Device staging of a host blob whose stage 2 runs on the device: a blob never exceeds its stage-1 arena plus the codec's
// framing. Never more than the caller gave.
static size_t stage2_blob_staging(const EncLayout& l, size_t hdr, size_t cloud_bytes, size_t out_capacity) {
  const size_t n = cloud_bytes / l.info.point_step, s1 = stage1_arena_bytes(l, n);
  return std::min(out_capacity, hdr + s1 + s1 / 128 + 32 * ((n + kChunkPoints - 1) / kChunkPoints) + 256);
}

// Device-pointer batches: the blob sizes into written_host, if asked for (one read-back, synchronises).
static int read_written(EncScratch& s, size_t n_frames, size_t* written_host) {
  if (!written_host) return CLDN_OK;
  if (int rc = s.h_sizes.reserve(n_frames)) return rc;
  CUDA_TRY(cudaMemcpyAsync(s.h_sizes.p, s.d_sizes.p, n_frames * sizeof(uint64_t), cudaMemcpyDeviceToHost, s.stream));
  if (int rc = check_device_error(s.stream, s.d_err.p, s.h_err.p)) return rc;
  for (size_t f = 0; f < n_frames; ++f) written_host[f] = static_cast<size_t>(s.h_sizes.p[f]);
  return CLDN_OK;
}

// Staging: n byte ranges at 256-byte-aligned offsets of `buf`, which grows to hold them with 256 bytes to
// spare; at[f] is where range f starts.
static int stage_layout(DevBuf<uint8_t>& buf, size_t n, const size_t* bytes, std::vector<void*>& at) {
  std::vector<size_t> off(n);
  size_t total = 0;
  for (size_t f = 0; f < n; ++f) {
    off[f] = total;
    total += (bytes[f] + 255) & ~size_t(255);
  }
  if (int rc = buf.reserve(total + 256)) return rc;
  at.resize(n);
  for (size_t f = 0; f < n; ++f) at[f] = buf.p + off[f];
  return CLDN_OK;
}

// Stage 1 from launch structs: the V5 sections (S, when the plan has them), the Gorilla pre-pass, the regular stream
// and the placement of the sections. cldn_b200_encode_batch and the prepared async call enqueue this same sequence.
static int launch_encode_stage1(const Plan& plan, const EncLaunch& L, const SecLaunch* S, cudaStream_t stream) {
  if (S && launch_encode_sections(plan, *S, stream) < 0) { set_error("section kernel launch failed"); return CLDN_ERR_CUDA; }
  if (launch_gorilla_prepass(plan, L, stream) < 0) { set_error("gorilla pre-pass launch failed"); return CLDN_ERR_CUDA; }
  if (launch_encode_regular(plan, L, stream) < 0) { set_error("encode kernel launch failed"); return CLDN_ERR_CUDA; }
  if (S && launch_place_sections(plan, *S, L.status, L.epoch, L.tile_points, stream) < 0) {
    set_error("section placement launch failed");
    return CLDN_ERR_CUDA;
  }
  CUDA_TRY(cudaGetLastError());
  return CLDN_OK;
}

// Stage 2 from its launch struct: the LZ4 or ZSTD chunk coder, then the pack into the blobs.
static int launch_encode_stage2(bool zstd, const Lz4Launch& Z, const uint8_t* header, uint32_t header_bytes, cudaStream_t stream) {
  if (zstd) {
    if (launch_zstd_compress(Z, header, header_bytes, stream) < 0) { set_error("ZSTD kernel launch failed"); return CLDN_ERR_CUDA; }
  } else if (launch_lz4_compress(Z, header, header_bytes, stream) < 0) {
    set_error("LZ4 kernel launch failed");
    return CLDN_ERR_CUDA;
  }
  CUDA_TRY(cudaGetLastError());
  return CLDN_OK;
}

// Bytes of one (chunk, section) slot of the V5 section scratch: the worst case of any mode is DeltaRle with one run per
// value, 5 + n * (max varint of the field + 1) bytes, plus the 16 bytes the vector copy of place_sections_kernel may read
// past the end.
static uint32_t section_stride(const Plan& plan) {
  uint32_t per_value = 0;
  for (uint32_t k = 0; k < plan.n_sections; ++k) {
    const uint32_t bpv = plan.sections[k].bpv;
    per_value = std::max<uint32_t>(per_value, (bpv == 2 ? 3u : bpv == 4 ? 5u : 10u) + 1u);
  }
  return 32 + kChunkPoints * per_value;
}

// Stage 1 of frames that passed check_encode_frame, or of staging their caller sized: fills their EncFrames and enqueues
// the kernels. Inputs and outputs are device pointers; the kernels check every store against out_capacities.
static int encode_batch_device(const EncLayout& l, EncScratch& s, size_t n_frames, const void* const* clouds, const size_t* cloud_bytes,
                               void* const* outs, const size_t* out_capacities, int write_header) {
  const cldn_info_t& info = l.info;
  EncFrame* hf = nullptr;
  int hf_slot = 0;
  if (int rc = s.h_frames.acquire(n_frames, &hf, &hf_slot)) return rc;
  if (int rc = s.d_frames.reserve(n_frames)) return rc;
  if (int rc = s.d_sizes.reserve(s.sizes_at + n_frames)) return rc;
  const uint32_t T = l.tile_points;
  const size_t hdr = write_header ? l.header.size() : 0;
  uint64_t tiles = 0, chunks = 0;
  bool aligned16 = true;
  for (size_t f = 0; f < n_frames; ++f) {
    const size_t n = cloud_bytes[f] / info.point_step;
    EncFrame& F = hf[f];
    F.in = static_cast<const uint8_t*>(clouds[f]);
    F.out = static_cast<uint8_t*>(outs[f]);
    F.out_cap = out_capacities[f];
    F.n_points = static_cast<uint32_t>(n);
    F.tile_begin = static_cast<uint32_t>(tiles);
    F.n_tiles = static_cast<uint32_t>((n + T - 1) / T);
    F.n_chunks = static_cast<uint32_t>((n + kChunkPoints - 1) / kChunkPoints);
    F.sec_excl = nullptr;
    tiles += F.n_tiles;
    chunks += F.n_chunks;
    if (reinterpret_cast<uintptr_t>(clouds[f]) & 15u) aligned16 = false;
  }
  if (tiles > 0x7FFFFFFFull) { set_error("batch too large"); return CLDN_ERR_UNSUPPORTED; }
  for (size_t f = 0; f < n_frames; ++f) hf[f].side = nullptr;
  if (l.plan.n_gorilla > 0) {
    // FieldEncoderFloat_Gorilla keeps a leading/trailing-zero window across the points of a chunk: a pre-pass walks
    // every chunk in order and leaves one 12-byte record per (op, point) for the (parallel) regular kernel to copy
    size_t total_points = 0;
    for (size_t f = 0; f < n_frames; ++f) total_points += hf[f].n_points;
    if (int rc = s.d_gorilla.reserve(total_points * 12 * l.plan.n_gorilla + 16)) return rc;
    size_t at = 0;
    for (size_t f = 0; f < n_frames; ++f) {
      hf[f].side = s.d_gorilla.p + at;
      at += static_cast<size_t>(hf[f].n_points) * 12 * l.plan.n_gorilla;
    }
  }
  if (int rc = s.d_status.reserve(static_cast<size_t>(tiles) + 1, true)) return rc;
  if (int rc = s.d_ticket.reserve(1)) return rc;
  s.epoch = (s.epoch + 1) & 0x3FFFFFu;
  if (s.epoch == 0) {  // epoch wrapped: stale words could alias
    CUDA_TRY(cudaMemsetAsync(s.d_status.p, 0, s.d_status.cap * sizeof(uint64_t), s.stream));
    s.epoch = 1;
  }
  EncLaunch L{};
  L.frames = s.d_frames.p;
  L.n_frames = static_cast<uint32_t>(n_frames);
  L.n_tiles_total = static_cast<uint32_t>(tiles);
  L.plan = l.d_plan.p;
  L.header = l.d_header.p;
  L.header_bytes = static_cast<uint32_t>(hdr);
  L.status = s.d_status.p;
  L.epoch = s.epoch;
  L.sizes = s.d_sizes.p + s.sizes_at;
  L.err = s.d_err.p;
  L.tile_points = T;
  L.flags = aligned16 ? kEncInputsAligned16 : 0u;
  L.uniform_tiles = 0;
  L.tile_ticket = s.d_ticket.p;
  if (n_frames > 0 && hf[0].n_tiles > 0) {
    bool uniform = true;
    for (size_t f = 1; f < n_frames; ++f) uniform = uniform && hf[f].n_tiles == hf[0].n_tiles;
    if (uniform) L.uniform_tiles = hf[0].n_tiles;
  }

  SecLaunch S{};
  if (l.plan.n_sections > 0) {
    // V5: adaptive integer sections are produced first (they determine where every later chunk starts).
    const uint32_t ns = l.plan.n_sections;
    const uint32_t stride = section_stride(l.plan);
    if (int rc = s.d_modes.reserve(n_frames * ns)) return rc;
    if (int rc = s.d_sec_scratch.reserve(static_cast<size_t>(chunks) * ns * stride)) return rc;
    if (int rc = s.d_sec_sizes.reserve(static_cast<size_t>(chunks) * ns + 1)) return rc;
    if (int rc = s.d_sec_excl.reserve(static_cast<size_t>(chunks) + n_frames + 1)) return rc;
    uint32_t* hcf = nullptr;
    int hcf_slot = 0;
    if (int rc = s.h_chunk_frame.acquire(static_cast<size_t>(chunks) + n_frames + 1, &hcf, &hcf_slot)) return rc;
    if (int rc = s.d_chunk_frame.reserve(static_cast<size_t>(chunks) + n_frames + 1)) return rc;
    if (int rc = s.d_hash.reserve(palette_overflow_scratch_bytes() / 8 + 16)) return rc;
    uint32_t cb = 0;
    for (size_t f = 0; f < n_frames; ++f) {
      EncFrame& F = hf[f];
      F.sec_excl = s.d_sec_excl.p + cb + f;  // (n_chunks + 1) entries per frame
      for (uint32_t c = 0; c < F.n_chunks; ++c) hcf[cb + c] = static_cast<uint32_t>(f);
      hcf[chunks + f] = cb;  // chunk_first[f]
      cb += F.n_chunks;
    }
    CUDA_TRY(cudaMemcpyAsync(s.d_chunk_frame.p, hcf, (chunks + n_frames) * sizeof(uint32_t), cudaMemcpyHostToDevice, s.stream));
    if (int rc = s.h_chunk_frame.commit(hcf_slot, s.stream)) return rc;
    S.frames = s.d_frames.p;
    S.n_frames = static_cast<uint32_t>(n_frames);
    S.n_chunks_total = static_cast<uint32_t>(chunks);
    S.chunk_frame = s.d_chunk_frame.p;
    S.chunk_first = s.d_chunk_frame.p + chunks;
    S.plan = l.d_plan.p;
    S.modes = s.d_modes.p;
    S.scratch = s.d_sec_scratch.p;
    S.sec_stride = stride;
    S.sec_sizes = s.d_sec_sizes.p;
    S.sec_excl = s.d_sec_excl.p;
    S.hash_scratch = s.d_hash.p;
    S.err = s.d_err.p;
    S.header_bytes = static_cast<uint32_t>(hdr);
  }
  CUDA_TRY(cudaMemcpyAsync(s.d_frames.p, hf, n_frames * sizeof(EncFrame), cudaMemcpyHostToDevice, s.stream));
  if (int rc = s.h_frames.commit(hf_slot, s.stream)) return rc;
  return launch_encode_stage1(l.plan, L, l.plan.n_sections > 0 ? &S : nullptr, s.stream);
}

// Stage 1 into an internal arena, then stage 2 on the device: one LZ4 block per chunk (cldn_lz4.cu) or one ZSTD frame
// per chunk (cldn_zstd_enc.cu), the blobs packed behind their headers into outs (device memory). The codec chooses the
// slots and the compress launch; the arena, the chunk tables and the pack are shared. Launches: stage 1 + 2.
static int encode_batch_device_stage2(const EncLayout& l, EncScratch& s, size_t n_frames, const void* const* clouds, const size_t* cloud_bytes,
                                      void* const* outs, const size_t* out_capacities, int write_header) {
  const cldn_info_t& info = l.info;  // compression NONE: what the stage-1 kernels produce
  const bool zstd = l.stage2 == CLDN_COMP_ZSTD;
  const size_t hdr = write_header ? l.header.size() : 0;
  const size_t zblock = zstd_enc_block_bytes();
  std::vector<size_t> s1_cap(n_frames), blocks_per_chunk(n_frames);
  size_t chunks = 0, max_chunk = 0, pieces = 0;
  for (size_t f = 0; f < n_frames; ++f) {
    const size_t n = cloud_bytes[f] / info.point_step, nc = (n + kChunkPoints - 1) / kChunkPoints;
    s1_cap[f] = stage1_arena_bytes(l, n);
    chunks += nc;
    bool ok;
    const size_t chunk_bound = max_compressed_size(info, std::min<size_t>(n, kChunkPoints), false, &ok) + 64;
    max_chunk = std::max(max_chunk, chunk_bound);
    blocks_per_chunk[f] = zstd ? std::max<size_t>(1, (chunk_bound + zblock - 1) / zblock) : 1;  // room for the worst case
    pieces += nc * blocks_per_chunk[f];
  }
  if (chunks > 0x7FFFFFFFull || pieces > 0x7FFFFFFFull) { set_error("batch too large"); return CLDN_ERR_UNSUPPORTED; }
  std::vector<void*> s1_ptr;
  if (int rc = stage_layout(s.d_s1, n_frames, s1_cap.data(), s1_ptr)) return rc;
  if (int rc = encode_batch_device(l, s, n_frames, clouds, cloud_bytes, s1_ptr.data(), s1_cap.data(), 0)) return rc;
  // chunk tables + slots: one per chunk (LZ4), one per block of a chunk's worst case (ZSTD)
  const size_t slot = zstd ? zstd_enc_slot_bytes() : (lz4_bound(max_chunk) + 15) & ~size_t(15);
  if (slot > 0xFFFFFFF0ull) { set_error("chunk too large for LZ4"); return CLDN_ERR_UNSUPPORTED; }
  if (int rc = s.d_lz_scratch.reserve(std::max<size_t>(pieces, 1) * slot)) return rc;
  if (int rc = s.d_lz_chunk_sizes.reserve(pieces + 1)) return rc;
  if (int rc = s.d_lz_chunk_frame.reserve(2 * chunks + 2)) return rc;  // chunk -> frame, then block_begin (ZSTD)
  if (int rc = s.d_lz_frames.reserve(n_frames)) return rc;
  Lz4Frame* hf = nullptr; int hf_slot = 0;
  uint32_t* hcf = nullptr; int hcf_slot = 0;
  if (int rc = s.h_lz_frames.acquire(n_frames, &hf, &hf_slot)) return rc;
  if (int rc = s.h_lz_chunk_frame.acquire(2 * chunks + 2, &hcf, &hcf_slot)) return rc;
  uint32_t cb = 0, pb = 0;
  for (size_t f = 0; f < n_frames; ++f) {
    const size_t n = cloud_bytes[f] / info.point_step;
    Lz4Frame& F = hf[f];
    memset(&F, 0, sizeof(F));
    F.plain = static_cast<uint8_t*>(s1_ptr[f]);
    F.plain_bytes = s.d_sizes.p + s.sizes_at + f;
    F.blob_out = static_cast<uint8_t*>(outs[f]);
    F.blob_cap = out_capacities[f];
    F.n_chunks = static_cast<uint32_t>((n + kChunkPoints - 1) / kChunkPoints);
    F.chunk_begin = cb;
    for (uint32_t c = 0; c < F.n_chunks; ++c) {
      hcf[cb + c] = static_cast<uint32_t>(f);
      hcf[chunks + cb + c] = pb;
      pb += static_cast<uint32_t>(blocks_per_chunk[f]);
    }
    cb += F.n_chunks;
  }
  hcf[2 * chunks] = pb;
  CUDA_TRY(cudaMemcpyAsync(s.d_lz_frames.p, hf, n_frames * sizeof(Lz4Frame), cudaMemcpyHostToDevice, s.stream));
  if (int rc = s.h_lz_frames.commit(hf_slot, s.stream)) return rc;
  CUDA_TRY(cudaMemcpyAsync(s.d_lz_chunk_frame.p, hcf, (2 * chunks + 1) * sizeof(uint32_t), cudaMemcpyHostToDevice, s.stream));
  if (int rc = s.h_lz_chunk_frame.commit(hcf_slot, s.stream)) return rc;
  Lz4Launch Z{};
  Z.frames = s.d_lz_frames.p;
  Z.n_frames = static_cast<uint32_t>(n_frames);
  Z.n_chunks_total = static_cast<uint32_t>(chunks);
  Z.chunk_frame = s.d_lz_chunk_frame.p;
  Z.scratch = s.d_lz_scratch.p;
  Z.slot_stride = static_cast<uint32_t>(slot);
  Z.chunk_sizes = s.d_lz_chunk_sizes.p;
  Z.sizes = s.d_sizes.p + s.sizes_at;   // the pack kernel overwrites the stage-1 sizes with the blob sizes (it runs after every reader)
  Z.err = s.d_err.p;
  if (zstd) {
    Z.block_begin = s.d_lz_chunk_frame.p + chunks;
    Z.n_blocks_total = static_cast<uint32_t>(pieces);
  }
  return launch_encode_stage2(zstd, Z, l.d_header.p, static_cast<uint32_t>(hdr), s.stream);
}

// Host blobs (CLDN_MEM_HOST, CLDN_MEM_DEVICE_POINTS) through device staging bounded by caps[f]: the clouds go up on the
// h2d stream (CLDN_MEM_HOST), the blobs are encoded on the handle's stream, and once a blob's 8-byte size is back,
// exactly that many bytes come down on the d2h stream. Stage 1 alone is pipelined frame by frame: frame f is encoded
// while later frames go up and earlier ones come down. Device stage 2 encodes the batch at once and is checked before
// anything comes down.
static int encode_host_blobs(const EncLayout& l, EncScratch& s, bool device_stage2, size_t n_frames, const void* const* clouds,
                             const size_t* cloud_bytes, void* const* outs, const size_t* caps, int write_header,
                             size_t* written_host, bool device_points) {
  std::vector<void*> slots, dout;
  std::vector<const void*> din(clouds, clouds + n_frames);
  if (!device_points) {
    if (int rc = stage_layout(s.d_in, n_frames, cloud_bytes, slots)) return rc;
  }
  if (int rc = stage_layout(s.d_out, n_frames, caps, dout)) return rc;
  if (int rc = s.pipe.ensure(2 * n_frames)) return rc;
  if (int rc = s.h_sizes.reserve(n_frames)) return rc;
  for (size_t f = 0; f < n_frames; ++f) {
    if (!device_points) {
      if (cloud_bytes[f]) CUDA_TRY(cudaMemcpyAsync(slots[f], clouds[f], cloud_bytes[f], cudaMemcpyHostToDevice, s.pipe.h2d));
      CUDA_TRY(cudaEventRecord(s.pipe.ev[2 * f], s.pipe.h2d));
      CUDA_TRY(cudaStreamWaitEvent(s.stream, s.pipe.ev[2 * f], 0));
      din[f] = slots[f];
    }
    if (device_stage2) continue;
    if (int rc = encode_batch_device(l, s, 1, &din[f], &cloud_bytes[f], &dout[f], &caps[f], write_header)) return rc;
    CUDA_TRY(cudaMemcpyAsync(s.h_sizes.p + f, s.d_sizes.p, sizeof(uint64_t), cudaMemcpyDeviceToHost, s.stream));
    CUDA_TRY(cudaEventRecord(s.pipe.ev[2 * f + 1], s.stream));
  }
  if (device_stage2) {
    if (int rc = encode_batch_device_stage2(l, s, n_frames, din.data(), cloud_bytes, dout.data(), caps, write_header)) return rc;
    CUDA_TRY(cudaMemcpyAsync(s.h_sizes.p, s.d_sizes.p, n_frames * sizeof(uint64_t), cudaMemcpyDeviceToHost, s.stream));
    if (int rc = check_device_error(s.stream, s.d_err.p, s.h_err.p)) return rc;
  }
  for (size_t f = 0; f < n_frames; ++f) {
    if (!device_stage2) CUDA_TRY(cudaEventSynchronize(s.pipe.ev[2 * f + 1]));
    const size_t sz = static_cast<size_t>(s.h_sizes.p[f]);
    if (sz > caps[f]) {  // the kernels refused the stores that did not fit and raised the error word
      if (int rc = check_device_error(s.stream, s.d_err.p, s.h_err.p)) return rc;
      set_error("Output buffer too small for uncompressed chunk");
      return CLDN_ERR_BUFFER_TOO_SMALL;
    }
    if (sz) CUDA_TRY(cudaMemcpyAsync(outs[f], dout[f], sz, cudaMemcpyDeviceToHost, s.pipe.d2h));
    if (written_host) written_host[f] = sz;
  }
  CUDA_TRY(cudaStreamSynchronize(s.pipe.d2h));
  return check_device_error(s.stream, s.d_err.p, s.h_err.p);
}

// Frames that passed check_encode_frame, through `route`. Device routes leave the blobs to the handle's stream and read
// the sizes back only into a given written_host; host routes return with their blobs complete.
static int encode_frames(const EncLayout& l, EncScratch& s, EncodeRoute route, int mem, size_t n_frames, const void* const* clouds,
                         const size_t* cloud_bytes, void* const* outs, const size_t* out_capacities, int write_header,
                         size_t* written_host) {
  const bool device_points = mem == CLDN_MEM_DEVICE_POINTS;
  const size_t hdr = write_header ? l.header.size() : 0;
  switch (route) {
    case kEncDevice:
      if (int rc = encode_batch_device(l, s, n_frames, clouds, cloud_bytes, outs, out_capacities, write_header)) return rc;
      return read_written(s, n_frames, written_host);
    case kEncDeviceStage2:
      if (int rc = encode_batch_device_stage2(l, s, n_frames, clouds, cloud_bytes, outs, out_capacities, write_header)) return rc;
      return read_written(s, n_frames, written_host);
    case kEncHostPlain:
    case kEncHostStage2: {
      const bool stage2 = route == kEncHostStage2;
      std::vector<size_t> caps(n_frames);
      for (size_t f = 0; f < n_frames; ++f) {
        caps[f] = (stage2 ? stage2_blob_staging : plain_blob_staging)(l, hdr, cloud_bytes[f], out_capacities[f]);
      }
      return encode_host_blobs(l, s, stage2, n_frames, clouds, cloud_bytes, outs, caps.data(), write_header, written_host, device_points);
    }
    case kEncHostLibrary:
      // stage 1 into host scratch, then every chunk through the system's liblz4 / libzstd behind the header; frame by
      // frame, so that the device staging holds one frame (the host compressor bounds this route, not the GPU)
      for (size_t f = 0; f < n_frames; ++f) {
        const size_t cap1 = stage1_arena_bytes(l, cloud_bytes[f] / l.info.point_step);
        s.s2_tmp.resize(cap1);
        void* s1_out = s.s2_tmp.data();
        size_t s1 = 0;
        if (int rc = encode_host_blobs(l, s, false, 1, &clouds[f], &cloud_bytes[f], &s1_out, &cap1, 0, &s1, device_points)) return rc;
        uint8_t* out = static_cast<uint8_t*>(outs[f]);
        if (hdr) memcpy(out, l.header.data(), hdr);
        size_t w = 0;
        if (int rc = stage2_compress_payload(l.stage2, s.s2_tmp.data(), s1, out + hdr, out_capacities[f] - hdr, &w)) return rc;
        if (written_host) written_host[f] = hdr + w;
      }
      return CLDN_OK;
  }
  set_error("unknown encode route");
  return CLDN_ERR_INTERNAL;
}

static int encode_batch_impl(cldn_encoder_t* e, size_t n_frames, const void* const* clouds, const size_t* cloud_bytes,
                             void* const* outs, const size_t* out_capacities, int write_header, size_t* written_host,
                             int mem) {
  if (!e || (n_frames && (!clouds || !cloud_bytes || !outs || !out_capacities))) {
    set_error("null argument");
    return CLDN_ERR_INVALID_ARGUMENT;
  }
  if (n_frames == 0) return CLDN_OK;
  EncodeRoute route;
  if (int rc = choose_encode_route(*e, *e, mem, &route)) return rc;
  const size_t hdr = write_header ? e->header.size() : 0;
  for (size_t f = 0; f < n_frames; ++f) {
    if (int rc = check_encode_frame(*e, hdr, clouds[f], cloud_bytes[f], outs[f], out_capacities[f])) return rc;
  }
  CUDA_TRY(cudaSetDevice(e->device));
  return encode_frames(*e, *e, route, mem, n_frames, clouds, cloud_bytes, outs, out_capacities, write_header, written_host);
}

// Complete blobs of frames with their own dims: each frame's header is made on the host, the payloads are encoded behind
// it (write_header = 0), and the headers are put in front of them afterwards (device blobs: one launch that also turns
// the payload sizes into blob sizes; host blobs: memcpy). The handle's header is not touched.
static int encode_blobs_impl(cldn_encoder_t* e, size_t n_frames, const void* const* clouds, const size_t* cloud_bytes,
                             const uint32_t* widths, const uint32_t* heights, void* const* outs, const size_t* out_capacities,
                             size_t* written_host, int mem) {
  if (!e || (n_frames && (!clouds || !cloud_bytes || !outs || !out_capacities))) {
    set_error("null argument");
    return CLDN_ERR_INVALID_ARGUMENT;
  }
  if (!widths != !heights) { set_error("widths and heights must both be given or both be NULL"); return CLDN_ERR_INVALID_ARGUMENT; }
  if (n_frames == 0) return CLDN_OK;
  EncodeRoute route;
  if (int rc = choose_encode_route(*e, *e, mem, &route)) return rc;
  std::vector<uint8_t> headers;          // frame f's header: headers[at[f], at[f + 1])
  std::vector<uint64_t> at(n_frames + 1, 0);
  std::vector<void*> payload(n_frames);
  std::vector<size_t> payload_cap(n_frames);
  auto frame_error = [](size_t f, int rc) {
    const std::string msg = cldn_b200_last_error();
    set_error("frame %zu: %s", f, msg.c_str());
    return rc;
  };
  for (size_t f = 0; f < n_frames; ++f) {
    cldn_info_t fi = e->blob_info;
    const size_t n = fi.point_step ? cloud_bytes[f] / fi.point_step : 0;
    fi.width = widths ? widths[f] : static_cast<uint32_t>(n);
    fi.height = heights ? heights[f] : 1u;
    const std::vector<uint8_t> h = make_header(fi);
    if (int rc = check_encode_frame(*e, h.size(), clouds[f], cloud_bytes[f], outs[f], out_capacities[f])) return frame_error(f, rc);
    if (static_cast<uint64_t>(fi.width) * fi.height != n) {
      set_error("width * height (%u x %u) differs from the %zu points of the cloud", fi.width, fi.height, n);
      return frame_error(f, CLDN_ERR_INVALID_ARGUMENT);
    }
    headers.insert(headers.end(), h.begin(), h.end());
    at[f + 1] = headers.size();
    payload[f] = static_cast<uint8_t*>(outs[f]) + h.size();
    payload_cap[f] = out_capacities[f] - h.size();
  }
  CUDA_TRY(cudaSetDevice(e->device));
  if (mem != CLDN_MEM_DEVICE) {
    std::vector<size_t> w(n_frames, 0);
    if (int rc = encode_frames(*e, *e, route, mem, n_frames, clouds, cloud_bytes, payload.data(), payload_cap.data(), 0, w.data())) return rc;
    for (size_t f = 0; f < n_frames; ++f) {
      memcpy(outs[f], headers.data() + at[f], at[f + 1] - at[f]);
      if (written_host) written_host[f] = (at[f + 1] - at[f]) + w[f];
    }
    return CLDN_OK;
  }
  if (int rc = encode_frames(*e, *e, route, mem, n_frames, clouds, cloud_bytes, payload.data(), payload_cap.data(), 0, nullptr)) return rc;
  const size_t tab_bytes = (2 * n_frames + 1) * sizeof(uint64_t) + headers.size();
  uint8_t* ht = nullptr;
  int slot = 0;
  if (int rc = e->h_blob_headers.acquire(tab_bytes, &ht, &slot)) return rc;
  if (int rc = e->d_blob_headers.reserve(tab_bytes)) return rc;
  uint64_t* tab = reinterpret_cast<uint64_t*>(ht);
  for (size_t f = 0; f < n_frames; ++f) tab[f] = reinterpret_cast<uintptr_t>(outs[f]);
  memcpy(tab + n_frames, at.data(), (n_frames + 1) * sizeof(uint64_t));
  memcpy(tab + 2 * n_frames + 1, headers.data(), headers.size());
  CUDA_TRY(cudaMemcpyAsync(e->d_blob_headers.p, ht, tab_bytes, cudaMemcpyHostToDevice, e->stream));
  if (int rc = e->h_blob_headers.commit(slot, e->stream)) return rc;
  if (launch_place_headers(reinterpret_cast<const uint64_t*>(e->d_blob_headers.p), static_cast<uint32_t>(n_frames), e->d_sizes.p,
                           e->stream) < 0) {
    set_error("header launch failed");
    return CLDN_ERR_CUDA;
  }
  CUDA_TRY(cudaGetLastError());
  return read_written(*e, n_frames, written_host);
}

// ---- device clouds of the encoder's layout, without the host (cldn_b200_encode_blobs_async) --------------------------
// Everything the calls of one prepared shape read: uploaded and allocated once by cldn_b200_encoder_prepare_blobs, apart
// from the handle's other scratch, so that a call allocates, copies from the host and synchronises nothing, and a CUDA
// graph that captured one stays valid until the next prepare. Every frame owns the tile and chunk slots of max_points;
// the frame kernel fills a frame's own and the encode kernels leave the rest (EncLaunch / SecLaunch / Lz4Launch
// ::empty_slots). Tile status words and error words are cleared inside every call, so a replayed graph starts clean.
struct AsyncEncode {
  size_t max_frames = 0;
  bool stage2 = false, zstd = false;
  DevBuf<uint8_t> d_tmpl;
  DevBuf<EncFrame> d_frames;
  DevBuf<Lz4Frame> d_lz_frames;
  DevBuf<uint64_t> d_sizes, d_status, d_hash;
  DevBuf<uint32_t> d_ticket, d_hdr_len, d_frame_err, d_err;
  DevBuf<uint8_t> d_gorilla, d_modes, d_sec_scratch, d_s1, d_lz_scratch;
  DevBuf<uint32_t> d_sec_sizes, d_sec_excl, d_chunk_frame, d_lz_chunk_frame, d_lz_chunk_sizes;
  EncAsyncLaunch A{};  // all but the call's arrays
  EncLaunch L{};
  SecLaunch S{};
  Lz4Launch Z{};
};
void AsyncEncodeDeleter::operator()(AsyncEncode* a) const { delete a; }

static int encoder_prepare_blobs_impl(cldn_encoder* e, size_t max_frames, uint64_t max_points) {
  if (!e) { set_error("null encoder"); return CLDN_ERR_INVALID_ARGUMENT; }
  if (max_frames == 0 || max_frames > 0x7FFFFFFFull) { set_error("max_frames must be 1 .. 2^31 - 1"); return CLDN_ERR_INVALID_ARGUMENT; }
  if (max_points > 0xFFFFFFFFull) { set_error("max_points_per_frame must be below 2^32"); return CLDN_ERR_UNSUPPORTED; }
  EncodeRoute route;
  if (int rc = choose_encode_route(*e, *e, CLDN_MEM_DEVICE, &route)) return rc;
  const Plan& plan = e->plan;
  const uint32_t T = e->tile_points;
  const uint64_t slots = (max_points + kChunkPoints - 1) / kChunkPoints, tiles_per_frame = (max_points + T - 1) / T;
  const uint64_t chunks = max_frames * slots, tiles = max_frames * tiles_per_frame;
  if (chunks > 0x7FFFFFFFull || tiles > 0x7FFFFFFFull) { set_error("max_frames * tiles or chunks per frame must be below 2^31"); return CLDN_ERR_UNSUPPORTED; }
  // MaxCompressedSize terms: a chunk of p points takes 4 + bound(p * per_point + chunk_extra) bytes
  bool ok1, ok2, ok3, ok4;
  const size_t m1 = max_compressed_size(e->info, 1, false, &ok1), m2 = max_compressed_size(e->info, 2, false, &ok2);
  const size_t full = max_compressed_size(e->blob_info, kChunkPoints, false, &ok3), full_s1 = max_compressed_size(e->info, kChunkPoints, false, &ok4);
  if (!ok1 || !ok2 || !ok3 || !ok4) return CLDN_ERR_INVALID_ARGUMENT;
  CUDA_TRY(cudaSetDevice(e->device));
  CUDA_TRY(cudaStreamSynchronize(e->stream));  // kernels of an earlier prepared state may still read it
  e->async.reset();
  std::unique_ptr<AsyncEncode, AsyncEncodeDeleter> a(new AsyncEncode());
  a->max_frames = max_frames;
  a->stage2 = route == kEncDeviceStage2;
  a->zstd = a->stage2 && e->stage2 == CLDN_COMP_ZSTD;
  cldn_info_t zero = e->blob_info;
  zero.width = zero.height = 0;
  std::vector<uint8_t> tmpl;
  EncAsyncLaunch& A = a->A;
  if (int rc = header_template(make_header(zero), &tmpl, A.tmpl_len)) return rc;
  std::vector<uint32_t> tables;  // host copies of the shape's tables, alive until the uploads below have completed
  std::vector<uint32_t> lz_tables;

  if (int rc = a->d_tmpl.reserve(tmpl.size())) return rc;
  CUDA_TRY(cudaMemcpyAsync(a->d_tmpl.p, tmpl.data(), tmpl.size(), cudaMemcpyHostToDevice, e->stream));
  if (int rc = a->d_frames.reserve(max_frames)) return rc;
  if (int rc = a->d_sizes.reserve(max_frames)) return rc;
  if (int rc = a->d_hdr_len.reserve(max_frames)) return rc;
  if (int rc = a->d_frame_err.reserve(max_frames)) return rc;
  if (int rc = a->d_err.reserve(1, true)) return rc;
  if (int rc = a->d_status.reserve(tiles + 1)) return rc;
  if (int rc = a->d_ticket.reserve(1)) return rc;
  A.tmpl = a->d_tmpl.p;
  A.point_step = e->info.point_step;
  A.max_points = max_points;
  A.per_point = m2 - m1;
  A.chunk_extra = static_cast<uint32_t>(m1 - 4 - (m2 - m1));
  A.compression = e->stage2;
  A.full_chunk = full;
  A.full_chunk_s1 = full_s1;
  A.tile_points = T;
  A.tiles_per_frame = static_cast<uint32_t>(tiles_per_frame);
  A.slots = static_cast<uint32_t>(slots);
  A.frames = a->d_frames.p;
  A.sizes = a->d_sizes.p;
  A.hdr_len = a->d_hdr_len.p;
  A.frame_err = a->d_frame_err.p;
  A.err = a->d_err.p;
  A.n_tables = static_cast<uint32_t>(max_frames);

  EncLaunch& L = a->L;
  L.frames = a->d_frames.p;
  L.n_frames = static_cast<uint32_t>(max_frames);
  L.n_tiles_total = static_cast<uint32_t>(tiles);
  L.plan = e->d_plan.p;
  L.header = nullptr;  // the frame kernel writes the headers
  L.header_bytes = 0;
  L.status = a->d_status.p;
  L.epoch = 1;         // the words are cleared in every call
  L.sizes = a->d_sizes.p;
  L.err = a->d_err.p;
  L.tile_points = T;
  L.flags = kEncAlignPerFrame;
  L.uniform_tiles = static_cast<uint32_t>(tiles_per_frame);
  L.tile_ticket = a->d_ticket.p;
  L.frame_err = a->d_frame_err.p;
  L.empty_slots = 1;
  if (plan.n_gorilla > 0) {
    A.side_stride = max_points * 12 * plan.n_gorilla;
    if (int rc = a->d_gorilla.reserve(max_frames * A.side_stride + 16)) return rc;
    A.side = a->d_gorilla.p;
  }
  if (plan.n_sections > 0) {
    // chunk slot gc belongs to frame gc / slots; chunk_first[f] = f * slots; frame f's sec_excl at f * (slots + 1)
    const uint32_t ns = plan.n_sections, stride = section_stride(plan);
    if (int rc = a->d_modes.reserve(max_frames * ns)) return rc;
    if (int rc = a->d_sec_scratch.reserve(chunks * ns * stride)) return rc;
    if (int rc = a->d_sec_sizes.reserve(chunks * ns + 1)) return rc;
    if (int rc = a->d_sec_excl.reserve(chunks + max_frames + 1)) return rc;
    if (int rc = a->d_chunk_frame.reserve(chunks + max_frames + 1)) return rc;
    if (int rc = a->d_hash.reserve(palette_overflow_scratch_bytes() / 8 + 16)) return rc;
    tables.resize(chunks + max_frames);
    for (uint64_t gc = 0; gc < chunks; ++gc) tables[gc] = static_cast<uint32_t>(gc / slots);
    for (size_t f = 0; f < max_frames; ++f) tables[chunks + f] = static_cast<uint32_t>(f * slots);
    CUDA_TRY(cudaMemcpyAsync(a->d_chunk_frame.p, tables.data(), tables.size() * sizeof(uint32_t), cudaMemcpyHostToDevice, e->stream));
    A.sec_excl = a->d_sec_excl.p;
    SecLaunch& S = a->S;
    S.frames = a->d_frames.p;
    S.n_frames = static_cast<uint32_t>(max_frames);
    S.n_chunks_total = static_cast<uint32_t>(chunks);
    S.chunk_frame = a->d_chunk_frame.p;
    S.chunk_first = a->d_chunk_frame.p + chunks;
    S.plan = e->d_plan.p;
    S.modes = a->d_modes.p;
    S.scratch = a->d_sec_scratch.p;
    S.sec_stride = stride;
    S.sec_sizes = a->d_sec_sizes.p;
    S.sec_excl = a->d_sec_excl.p;
    S.hash_scratch = a->d_hash.p;
    S.err = a->d_err.p;
    S.header_bytes = 0;
    S.frame_err = a->d_frame_err.p;
    S.empty_slots = 1;
  }
  if (a->stage2) {
    // stage-1 arenas of max_points (a frame's own stores are bounded by its stage1_arena_bytes), and the slots of
    // encode_batch_device_stage2 for chunks of min(max_points, kChunkPoints) points
    const uint64_t s1_stride = (stage1_arena_bytes(*e, max_points) + 255) & ~uint64_t(255);
    bool ok;
    const size_t chunk_bound = max_compressed_size(e->info, std::min<uint64_t>(max_points, kChunkPoints), false, &ok) + 64;
    const size_t zblock = zstd_enc_block_bytes();
    const uint64_t per_chunk = a->zstd ? std::max<size_t>(1, (chunk_bound + zblock - 1) / zblock) : 1, pieces = chunks * per_chunk;
    const size_t slot = a->zstd ? zstd_enc_slot_bytes() : (lz4_bound(chunk_bound) + 15) & ~size_t(15);
    if (pieces > 0x7FFFFFFFull) { set_error("max_frames * ZSTD blocks per frame must be below 2^31"); return CLDN_ERR_UNSUPPORTED; }
    if (slot > 0xFFFFFFF0ull) { set_error("chunk too large for LZ4"); return CLDN_ERR_UNSUPPORTED; }
    if (int rc = a->d_s1.reserve(std::max<uint64_t>(max_frames * s1_stride, 256))) return rc;
    if (int rc = a->d_lz_frames.reserve(max_frames)) return rc;
    if (int rc = a->d_lz_scratch.reserve(std::max<uint64_t>(pieces, 1) * slot)) return rc;
    if (int rc = a->d_lz_chunk_sizes.reserve(pieces + 1)) return rc;
    if (int rc = a->d_lz_chunk_frame.reserve(2 * chunks + 2)) return rc;  // chunk -> frame, then block_begin (ZSTD)
    lz_tables.resize(2 * chunks + 1);
    for (uint64_t gc = 0; gc < chunks; ++gc) {
      lz_tables[gc] = static_cast<uint32_t>(gc / slots);
      lz_tables[chunks + gc] = static_cast<uint32_t>(gc * per_chunk);
    }
    lz_tables[2 * chunks] = static_cast<uint32_t>(pieces);
    CUDA_TRY(cudaMemcpyAsync(a->d_lz_chunk_frame.p, lz_tables.data(), lz_tables.size() * sizeof(uint32_t), cudaMemcpyHostToDevice, e->stream));
    A.lz_frames = a->d_lz_frames.p;
    A.s1 = a->d_s1.p;
    A.s1_stride = s1_stride;
    Lz4Launch& Z = a->Z;
    Z.frames = a->d_lz_frames.p;
    Z.n_frames = static_cast<uint32_t>(max_frames);
    Z.n_chunks_total = static_cast<uint32_t>(chunks);
    Z.chunk_frame = a->d_lz_chunk_frame.p;
    Z.scratch = a->d_lz_scratch.p;
    Z.slot_stride = static_cast<uint32_t>(slot);
    Z.chunk_sizes = a->d_lz_chunk_sizes.p;
    Z.sizes = a->d_sizes.p;   // the pack kernel overwrites the stage-1 sizes with the payload sizes
    Z.err = a->d_err.p;
    Z.frame_err = a->d_frame_err.p;
    Z.empty_slots = 1;
    if (a->zstd) {
      Z.block_begin = a->d_lz_chunk_frame.p + chunks;
      Z.n_blocks_total = static_cast<uint32_t>(pieces);
    }
  }
  CUDA_TRY(cudaStreamSynchronize(e->stream));  // the uploads read host objects of this function
  e->async = std::move(a);
  return CLDN_OK;
}

// Enqueues only. The launches and their grids are those of the prepared shape, whatever the frames: two clears, the
// frame kernel, the stage-1 sequence of encode_batch, stage 2 when compressed, the status kernel.
static int encode_blobs_async_impl(cldn_encoder* e, size_t n, const void* d_frames, int32_t* d_status, uint64_t* d_written) {
  if (!e) { set_error("null encoder"); return CLDN_ERR_INVALID_ARGUMENT; }
  AsyncEncode* a = e->async.get();
  if (!a) { set_error("no prepared shape: call cldn_b200_encoder_prepare_blobs first"); return CLDN_ERR_INVALID_ARGUMENT; }
  if (n > a->max_frames) { set_error("%zu frames: the shape was prepared for at most %zu", n, a->max_frames); return CLDN_ERR_INVALID_ARGUMENT; }
  if (!d_frames || !d_status) { set_error("null argument"); return CLDN_ERR_INVALID_ARGUMENT; }
  if (n == 0) return CLDN_OK;
  CUDA_TRY(cudaSetDevice(e->device));
  EncAsyncLaunch A = a->A;
  A.desc = static_cast<const CloudDesc*>(d_frames);
  A.n_frames = static_cast<uint32_t>(n);
  A.status = d_status;
  A.written = d_written;
  CUDA_TRY(cudaMemsetAsync(a->d_frame_err.p, 0, a->max_frames * sizeof(uint32_t), e->stream));
  CUDA_TRY(cudaMemsetAsync(a->d_status.p, 0, a->L.n_tiles_total * sizeof(uint64_t), e->stream));
  launch_encode_async_frames(A, e->stream);
  if (int rc = launch_encode_stage1(e->plan, a->L, e->plan.n_sections > 0 ? &a->S : nullptr, e->stream)) return rc;
  if (a->stage2) {
    if (int rc = launch_encode_stage2(a->zstd, a->Z, nullptr, 0, e->stream)) return rc;
  }
  launch_encode_async_status(A, e->stream);
  CUDA_TRY(cudaGetLastError());
  return CLDN_OK;
}

extern "C" {

int cldn_b200_encode_batch(cldn_encoder_t* e, size_t n_frames, const void* const* clouds, const size_t* cloud_bytes,
                           void* const* outs, const size_t* out_capacities, int write_header, size_t* written_host,
                           int mem) {
  return guarded([&] { return encode_batch_impl(e, n_frames, clouds, cloud_bytes, outs, out_capacities, write_header, written_host, mem); });
}

int cldn_b200_encode(cldn_encoder_t* enc, const void* cloud, size_t cloud_bytes, void* out, size_t out_capacity,
                     int write_header, size_t* written, int mem) {
  const void* clouds[1] = {cloud};
  void* outs[1] = {out};
  return cldn_b200_encode_batch(enc, 1, clouds, &cloud_bytes, outs, &out_capacity, write_header, written, mem);
}

int cldn_b200_encode_blobs(cldn_encoder_t* e, size_t n_frames, const void* const* clouds, const size_t* cloud_bytes,
                           const uint32_t* widths, const uint32_t* heights, void* const* outs, const size_t* out_capacities,
                           size_t* written_host, int mem) {
  return guarded([&] { return encode_blobs_impl(e, n_frames, clouds, cloud_bytes, widths, heights, outs, out_capacities, written_host, mem); });
}

int cldn_b200_encoder_prepare_blobs(cldn_encoder_t* enc, size_t max_frames, uint64_t max_points_per_frame) {
  return guarded([&] { return encoder_prepare_blobs_impl(enc, max_frames, max_points_per_frame); });
}

int cldn_b200_encode_blobs_async(cldn_encoder_t* enc, size_t n_frames, const void* d_frames, int32_t* d_status, uint64_t* d_written) {
  return guarded([&] { return encode_blobs_async_impl(enc, n_frames, d_frames, d_status, d_written); });
}

}  // extern "C"

// =====================================================================================================================
// The device scratch of the stage-1 decode kernels (DecLaunch). A decoder has one for its calls, and one more for the
// shape that cldn_b200_decoder_prepare_blobs sized, so that neither invalidates the other.
struct DecStage1 {
  DevBuf<uint64_t> d_chunk_offsets;
  DevBuf<uint32_t> d_chunk_sizes;
  DevBuf<uint32_t> d_chunk_tiles, d_chunk_tile_begin, d_stream_end, d_tsums, d_chunk_frame, d_tile_chunk;
  DevBuf<uint64_t> d_tstatus;
  DevBuf<uint32_t> d_counter, d_redo;
  DevBuf<uint8_t> d_side;         // side mode: section values decoded ahead of the regular stream (DecLaunch::side)
  DevBuf<uint64_t> d_chunk_desc;  // chunk-sequential kernel: self-validating chunk descriptors (see walk_frame_publish)
  uint32_t desc_tag = 0;
  uint32_t epoch = 0;
  // the last launch of this scratch (cldn_b200_decoder_last_stats / _last_sections_ahead read the handle's own)
  bool fast_launched = false;  // it went through decode_floatn_fast_kernel
  uint32_t fast_chunks = 0;
  bool sections_ahead = false;  // it ran in side mode
};

// What the host knows about the frames of one stage-1 launch.
struct Stage1Shape {
  uint32_t n_frames = 0;
  uint64_t chunks = 0;          // chunk slots
  uint64_t tiles = 0;           // bound of the FloatN tiles of the launch (tile-parallel kernel)
  uint32_t uniform_chunks = 0;  // > 0: every frame has this many chunk slots
  // The launch may be replayed from a CUDA graph, with the same tag and epoch every time: the chunk descriptors and the
  // tile records are cleared in the launch instead of being told apart by a new tag / epoch per call.
  bool replayable = false;
  bool empty_slots = false;     // frames own fixed chunk slots, some of them empty (DecLaunch::empty_slots)
  uint64_t chunk_bytes_max = 0;  // > 0: `tiles` assumes chunk bodies of at most this many bytes (DecLaunch::chunk_bytes_max)
};

struct cldn_decoder;
static int launch_stage1(cldn_decoder* d, DecStage1& s, const Plan& plan, const Plan* d_plan, const DecFrame* d_frames,
                         const Stage1Shape& shape, uint32_t* err, uint32_t* frame_err, bool reserve_only);

struct AsyncBlobs;  // cldn_b200_decoder_prepare_blobs
struct AsyncBlobsDeleter { void operator()(AsyncBlobs* a) const; };

struct cldn_decoder {
  std::vector<uint8_t> s2_tmp;  // stage-2 decompression scratch (host-pointer API only)
  int device = 0;
  cudaStream_t stream = nullptr;
  bool own_stream = false;
  cldn_info_t info;  // info of the cached plan
  bool have_plan = false;
  Plan plan;
  bool has_padding = false;
  DevBuf<Plan> d_plan;
  DevBuf<DecFrame> d_frames;
  PinRing<DecFrame> h_frames;
  DevBuf<uint32_t> d_err;
  PinBuf<uint32_t> h_err;
  DevBuf<uint8_t> d_in, d_out;
  DecStage1 s1;
  // stage 2 on the device (LZ4)
  DevBuf<uint8_t> d_s1, d_lz_scratch;
  DevBuf<uint32_t> d_lz_chunk_frame, d_lz_chunk_sizes;
  DevBuf<Lz4Frame> d_lz_frames;
  DevBuf<uint64_t> d_lz_sizes;
  PinBuf<uint64_t> h_lz_sizes;
  PinRing<Lz4Frame> h_lz_frames;
  PinRing<uint32_t> h_lz_chunk_frame;
  DevBuf<uint8_t> d_zs_lit;        // ZSTD: literal scratch per decompressing warp
  CopyPipeline pipe;
  // cldn_b200_decode_blobs: the first bytes of device-resident blobs, and what the last call found for every frame
  DevBuf<uint64_t> d_blob_tab;
  PinBuf<uint64_t> h_blob_tab;
  DevBuf<uint8_t> d_prefix;
  PinBuf<uint8_t> h_prefix;
  // one error word per frame of the group being decoded (DecLaunch / Lz4Launch::frame_err); nullptr outside of it
  DevBuf<uint32_t> d_frame_err;
  PinBuf<uint32_t> h_frame_err;
  uint32_t* frame_err = nullptr;
  std::vector<std::string> frame_errors;
  std::vector<cldn_info_t> frame_infos;
  std::unique_ptr<AsyncBlobs, AsyncBlobsDeleter> async;  // cldn_b200_decoder_prepare_blobs
};

static bool same_fields(const cldn_info_t& a, const cldn_info_t& b) {
  if (a.point_step != b.point_step || a.encoding_opt != b.encoding_opt || a.compression_opt != b.compression_opt ||
      a.version != b.version || a.n_fields != b.n_fields) return false;
  for (uint32_t i = 0; i < a.n_fields; ++i) {
    const cldn_field_t &x = a.fields[i], &y = b.fields[i];
    if (x.offset != y.offset || x.type != y.type || x.has_resolution != y.has_resolution ||
        (x.has_resolution && memcmp(&x.resolution, &y.resolution, 4) != 0)) return false;
  }
  return true;
}

static bool same_info(const cldn_info_t& a, const cldn_info_t& b) {
  return a.width == b.width && a.height == b.height && same_fields(a, b);
}

// The stage-1 decoder plan of `info` (compression NONE), or the refusal.
static int make_decode_plan(const cldn_info_t& info, Plan* plan) {
  if (int rc = build_decode_plan(info, plan)) return rc;
  if (!plan->supported) {
    set_error("EncodingInfo contains a field decoder this build cannot run");
    return CLDN_ERR_UNSUPPORTED;
  }
  if (info.compression_opt != CLDN_COMP_NONE) {
    set_error("compression_opt %d: stage 2 is undone before the stage-1 decode (LZ4 and ZSTD on the device)", static_cast<int>(info.compression_opt));
    return CLDN_ERR_UNSUPPORTED;
  }
  if (info.version < 3) { set_error("wire version %d (single unframed chunk) is not supported", info.version); return CLDN_ERR_UNSUPPORTED; }
  return CLDN_OK;
}

// PointcloudDecoder::updateDecoders (cloudini.cpp:627-633)
static int decoder_update_plan(cldn_decoder* d, const cldn_info_t& info) {
  if (d->have_plan && same_info(d->info, info)) return CLDN_OK;
  Plan plan;
  if (int rc = make_decode_plan(info, &plan)) return rc;
  if (int rc = d->d_plan.reserve(1)) return rc;
  CUDA_TRY(cudaMemcpyAsync(d->d_plan.p, &plan, sizeof(Plan), cudaMemcpyHostToDevice, d->stream));
  CUDA_TRY(cudaStreamSynchronize(d->stream));  // `plan` is a stack object
  d->plan = plan;
  d->info = info;
  d->have_plan = true;
  // do the declared fields cover every byte of a point? (otherwise host outputs must round-trip their padding)
  // union of the field intervals, clipped to the point: at most CLDN_MAX_FIELDS of them, no point_step-sized table
  // (the header is untrusted: a forged point_step must not size an allocation)
  std::pair<uint64_t, uint64_t> iv[CLDN_MAX_FIELDS];
  uint32_t n_iv = 0;
  for (uint32_t i = 0; i < info.n_fields && n_iv < CLDN_MAX_FIELDS; ++i) {
    const uint64_t lo = info.fields[i].offset, hi = std::min<uint64_t>(lo + static_cast<uint64_t>(size_of_type(info.fields[i].type)), info.point_step);
    if (lo < hi) iv[n_iv++] = {lo, hi};
  }
  std::sort(iv, iv + n_iv);
  uint64_t covered_to = 0;
  bool gap = false;
  for (uint32_t i = 0; i < n_iv; ++i) {
    if (iv[i].first > covered_to) gap = true;
    covered_to = std::max(covered_to, iv[i].second);
  }
  d->has_padding = gap || covered_to < info.point_step;
  return CLDN_OK;
}

// `frame_points` (optional): points of every frame; nullptr gives every frame info.width * info.height points.
static int decode_batch_device(cldn_decoder* d, const cldn_info_t& info, size_t n_frames, const void* const* payloads,
                               const size_t* payload_bytes, void* const* outs, const size_t* out_capacities,
                               const uint64_t* frame_points) {
  d->s1.sections_ahead = false;
  if (int rc = decoder_update_plan(d, info)) return rc;
  const uint64_t wh = static_cast<uint64_t>(info.width) * info.height;
  for (size_t f = 0; f < (frame_points ? n_frames : 1); ++f) {
    if ((frame_points ? frame_points[f] : wh) > 0xFFFFFFFFull) { set_error("too many points"); return CLDN_ERR_UNSUPPORTED; }
  }
  DecFrame* hf = nullptr;
  int hf_slot = 0;
  if (int rc = d->h_frames.acquire(n_frames, &hf, &hf_slot)) return rc;
  if (int rc = d->d_frames.reserve(n_frames)) return rc;
  uint64_t chunks = 0;
  for (size_t f = 0; f < n_frames; ++f) {
    const uint64_t n_points = frame_points ? frame_points[f] : wh;
    const uint64_t out_need = n_points * info.point_step;
    if (out_capacities[f] < out_need) {
      set_error("Output buffer is too small to hold the decoded data");  // v4_codec.cpp:93-95 / v5_codec.cpp:991-993
      return CLDN_ERR_BUFFER_TOO_SMALL;
    }
    DecFrame& F = hf[f];
    F.payload = static_cast<const uint8_t*>(payloads[f]);
    F.payload_bytes = payload_bytes[f];
    F.out = static_cast<uint8_t*>(outs[f]);
    F.n_points = static_cast<uint32_t>(n_points);
    F.n_chunks = static_cast<uint32_t>((n_points + kChunkPoints - 1) / kChunkPoints);
    F.chunk_begin = static_cast<uint32_t>(chunks);
    F.pad_ = 0;
    chunks += F.n_chunks;
  }
  if (chunks > 0x7FFFFFFFull) { set_error("batch too large"); return CLDN_ERR_UNSUPPORTED; }
  CUDA_TRY(cudaMemcpyAsync(d->d_frames.p, hf, n_frames * sizeof(DecFrame), cudaMemcpyHostToDevice, d->stream));
  if (int rc = d->h_frames.commit(hf_slot, d->stream)) return rc;
  Stage1Shape shape;
  shape.n_frames = static_cast<uint32_t>(n_frames);
  shape.chunks = chunks;
  // tile-parallel path: every chunk adds at most 2 tiles of rounding / misalignment
  for (size_t f = 0; f < n_frames; ++f) shape.tiles += payload_bytes[f] / decode_tile_bytes() + 2ull * hf[f].n_chunks + 1;
  bool uniform = n_frames > 0 && hf[0].n_chunks > 0;
  for (size_t f = 1; f < n_frames; ++f) uniform = uniform && hf[f].n_chunks == hf[0].n_chunks;
  shape.uniform_chunks = uniform ? hf[0].n_chunks : 0u;
  return launch_stage1(d, d->s1, d->plan, d->d_plan.p, d->d_frames.p, shape, d->d_err.p, d->frame_err, false);
}

// The stage-1 kernels of one launch, routed by the plan and the host's view of the frames (`shape`); the frame table is on
// the device. reserve_only: size the scratch of this shape and launch nothing.
static int launch_stage1(cldn_decoder* d, DecStage1& s, const Plan& plan, const Plan* d_plan, const DecFrame* d_frames,
                         const Stage1Shape& shape, uint32_t* err, uint32_t* frame_err, bool reserve_only) {
  const uint64_t chunks = shape.chunks;
  if (int rc = s.d_chunk_offsets.reserve(static_cast<size_t>(chunks) + 1)) return rc;
  if (int rc = s.d_chunk_sizes.reserve(static_cast<size_t>(chunks) + 1)) return rc;
  DecLaunch L{};
  L.frames = d_frames;
  L.n_frames = shape.n_frames;
  L.n_chunks_total = static_cast<uint32_t>(chunks);
  L.plan = d_plan;
  L.chunk_offsets = s.d_chunk_offsets.p;
  L.chunk_sizes = s.d_chunk_sizes.p;
  L.err = err;
  L.frame_err = frame_err;
  L.empty_slots = shape.empty_slots ? 1u : 0u;
  if (plan.n_sections > 0 && chunks > 0 && (plan.regular_overlap || !(plan.all_varint || plan.n_ops == 0))) {
    // V5 with raw / XOR / Gorilla fields in the regular stream: the per-chunk parser records where the sections start
    if (int rc = s.d_stream_end.reserve(static_cast<size_t>(chunks) + 1)) return rc;
    L.stream_end = s.d_stream_end.p;
  }
  const char* force_env = getenv("CLDN_B200_FORCE_CHUNK_DECODE");
  const bool force_chunk = force_env && force_env[0] == '1';
  const bool fast_general = !plan.floatn_only && chunks > 0 && decode_fast_general_plan(plan) &&
                            decode_tiles_sequential(static_cast<uint32_t>(chunks)) && decode_fast_enabled() && !force_chunk;
  const bool tile_parallel = plan.floatn_only && chunks > 0 && !force_chunk;
  if (fast_general) {
    // float-varint streams with scalar lossy fields (Velodyne XYZIRT ...): fast chunk-sequential reader + redo list
    if (int rc = s.d_stream_end.reserve(static_cast<size_t>(chunks) + 1)) return rc;
    L.stream_end = s.d_stream_end.p;
  }
  if (tile_parallel) {
    const uint64_t tiles = shape.tiles;
    if (tiles > 0x7FFFFFFFull) { set_error("batch too large"); return CLDN_ERR_UNSUPPORTED; }
    if (int rc = s.d_chunk_tiles.reserve(static_cast<size_t>(chunks) + 1)) return rc;
    if (int rc = s.d_chunk_tile_begin.reserve(static_cast<size_t>(chunks) + 2)) return rc;
    if (int rc = s.d_stream_end.reserve(static_cast<size_t>(chunks) + 1)) return rc;
    if (int rc = s.d_chunk_frame.reserve(static_cast<size_t>(chunks) + 1)) return rc;
    if (int rc = s.d_tile_chunk.reserve(static_cast<size_t>(tiles) + 1)) return rc;
    const size_t old_cap = s.d_tstatus.cap;
    if (int rc = s.d_tstatus.reserve(static_cast<size_t>(tiles) + 1, true)) return rc;
    if (s.d_tstatus.cap != old_cap || s.d_tsums.cap < s.d_tstatus.cap * 16) {
      if (int rc = s.d_tsums.reserve(s.d_tstatus.cap * 16, true)) return rc;
    }
    // a replayable launch clears the records it will read: none on the chunk-sequential route, which has no tile records
    const bool clear = shape.replayable && !decode_tiles_sequential(static_cast<uint32_t>(chunks));
    if (!reserve_only) {
      s.epoch = shape.replayable ? 1u : (s.epoch + 1) & 0x3FFFFFu;
      if (s.epoch == 0 || clear) {
        CUDA_TRY(cudaMemsetAsync(s.d_tstatus.p, 0, (shape.replayable ? tiles + 1 : s.d_tstatus.cap) * sizeof(uint64_t), d->stream));
        CUDA_TRY(cudaMemsetAsync(s.d_tsums.p, 0, (shape.replayable ? 16 * (tiles + 1) : s.d_tsums.cap) * sizeof(uint32_t), d->stream));
        if (s.epoch == 0) s.epoch = 1;
      }
    }
    L.chunk_tiles = s.d_chunk_tiles.p;
    L.chunk_tile_begin = s.d_chunk_tile_begin.p;
    L.stream_end = s.d_stream_end.p;
    L.chunk_frame = s.d_chunk_frame.p;
    L.tile_chunk = s.d_tile_chunk.p;
    L.tstatus = s.d_tstatus.p;
    L.tsums = s.d_tsums.p;
    L.tile_capacity = static_cast<uint32_t>(s.d_tstatus.cap);
    L.tile_grid = static_cast<uint32_t>(tiles);
    L.chunk_bytes_max = static_cast<uint32_t>(shape.chunk_bytes_max);
    L.epoch = s.epoch;
  }
  if (fast_general || tile_parallel) {
    // chunk claim counters, the careful kernel's redo list and the self-validating chunk descriptors
    if (int rc = s.d_counter.reserve(4, true)) return rc;
    if (int rc = s.d_redo.reserve(static_cast<size_t>(chunks) + 1)) return rc;
    const size_t had = s.d_chunk_desc.cap;
    if (int rc = s.d_chunk_desc.reserve(2 * static_cast<size_t>(chunks) + 2)) return rc;
    if (!reserve_only) {
      s.desc_tag = shape.replayable ? 1u : (s.desc_tag + 1) & 0xFFFFFFu;
      if (s.d_chunk_desc.cap != had || s.desc_tag == 0 || shape.replayable) {  // fresh memory, tag wrap or replay: no stale word may carry a live tag
        CUDA_TRY(cudaMemsetAsync(s.d_chunk_desc.p, 0, (shape.replayable ? 2 * chunks + 2 : s.d_chunk_desc.cap) * sizeof(uint64_t), d->stream));
        if (s.desc_tag == 0) s.desc_tag = 1;
      }
    }
    L.chunk_counter = s.d_counter.p;
    L.redo_list = s.d_redo.p;
    L.chunk_desc = s.d_chunk_desc.p;
    L.desc_tag = s.desc_tag;
    L.uniform_chunks = shape.uniform_chunks;
  }
  const bool fast_launched = L.redo_list != nullptr && decode_tiles_sequential(L.n_chunks_total) && decode_fast_enabled() && !plan.regular_overlap;
  if (fast_launched && L.chunk_desc && L.stream_end && L.chunk_counter && decode_side_plan(plan) && decode_fast_general_plan(plan) && !force_chunk) {
    // V5 sections ahead of the regular stream: compact per-chunk arrays the fast reader merges into the rows (DecLaunch::side)
    const size_t side_bytes = decode_side_bytes(plan, chunks, L.side_off);
    if (int rc = s.d_side.reserve(side_bytes + 256)) return rc;
    L.side = s.d_side.p;
  }
  if (reserve_only) return CLDN_OK;
  s.fast_launched = fast_launched;
  s.sections_ahead = decode_side_active(plan, L);
  s.fast_chunks = fast_launched ? L.n_chunks_total : 0u;
  if (launch_decode(plan, L, d->stream) < 0) { set_error("decode kernel launch failed"); return CLDN_ERR_CUDA; }
  CUDA_TRY(cudaGetLastError());
  return CLDN_OK;
}

extern "C" {

int cldn_b200_decoder_create(int device, void* stream, cldn_decoder_t** out) {
  if (!out) { set_error("null argument"); return CLDN_ERR_INVALID_ARGUMENT; }
  *out = nullptr;
  if (int rc = select_device(device)) return rc;
  cldn_decoder* d = new cldn_decoder();
  cudaGetDevice(&d->device);
  if (stream) {
    d->stream = static_cast<cudaStream_t>(stream);
  } else {
    if (cudaStreamCreateWithFlags(&d->stream, cudaStreamNonBlocking) != cudaSuccess) {
      set_error("cudaStreamCreate failed");
      delete d;
      return CLDN_ERR_CUDA;
    }
    d->own_stream = true;
  }
  int rc = d->d_err.reserve(1, true);
  if (!rc) rc = d->h_err.reserve(1);
  if (rc) { cldn_b200_decoder_destroy(d); return rc; }
  *out = d;
  return CLDN_OK;
}

void cldn_b200_decoder_destroy(cldn_decoder_t* d) {
  if (!d) return;
  cudaSetDevice(d->device);
  if (d->stream) cudaStreamSynchronize(d->stream);
  const cudaStream_t own = d->own_stream ? d->stream : nullptr;
  delete d;  // the buffers free themselves
  if (own) cudaStreamDestroy(own);
}

int cldn_b200_decoder_sync(cldn_decoder_t* d) {
  if (!d) { set_error("null decoder"); return CLDN_ERR_INVALID_ARGUMENT; }
  CUDA_TRY(cudaSetDevice(d->device));
  return check_device_error(d->stream, d->d_err.p, d->h_err.p);
}

int cldn_b200_decoder_last_stats(cldn_decoder_t* d, uint32_t stats[2]) {
  if (!d || !stats) { set_error("null argument"); return CLDN_ERR_INVALID_ARGUMENT; }
  stats[0] = stats[1] = 0;
  CUDA_TRY(cudaSetDevice(d->device));
  if (!d->s1.d_counter.p || !d->s1.fast_launched) return CLDN_OK;
  uint32_t c[4] = {0, 0, 0, 0};
  CUDA_TRY(cudaStreamSynchronize(d->stream));
  CUDA_TRY(cudaMemcpy(c, d->s1.d_counter.p, sizeof(c), cudaMemcpyDeviceToHost));
  stats[0] = d->s1.fast_chunks;
  stats[1] = c[3];
  return CLDN_OK;
}

int cldn_b200_decoder_last_sections_ahead(cldn_decoder_t* d) {
  if (!d) { set_error("null argument"); return CLDN_ERR_INVALID_ARGUMENT; }
  return d->s1.sections_ahead ? 1 : 0;
}

}  // extern "C"

// Points of every frame of a batch and where each frame's re-framed stage-1 payload goes in the decoder's arena:
// `frame_points` as decode_batch_device takes it, every frame's chunks get a slot of `slot` bytes plus their u32 prefixes.
struct FrameChunks {
  std::vector<uint64_t> points;
  std::vector<size_t> s1_off, s1_cap;
  uint64_t max_points = 0;
  size_t arena = 0, chunks = 0;
  int init(const cldn_info_t& info, size_t n_frames, const uint64_t* frame_points) {
    points.resize(n_frames);
    for (size_t f = 0; f < n_frames; ++f) {
      points[f] = frame_points ? frame_points[f] : static_cast<uint64_t>(info.width) * info.height;
      if (points[f] > 0xFFFFFFFFull) { set_error("too many points"); return CLDN_ERR_UNSUPPORTED; }
      max_points = std::max(max_points, points[f]);
    }
    return CLDN_OK;
  }
  size_t frame_chunks(size_t f) const { return static_cast<size_t>((points[f] + kChunkPoints - 1) / kChunkPoints); }
  void place(size_t slot) {
    s1_off.resize(points.size());
    s1_cap.resize(points.size());
    for (size_t f = 0; f < points.size(); ++f) {
      s1_cap[f] = (frame_chunks(f) * (slot + 4) + 255) & ~size_t(255);
      s1_off[f] = arena;
      arena += s1_cap[f];
      chunks += frame_chunks(f);
    }
  }
};

// Bound of one decompressed chunk, as the host-pointer API has always passed it to ZSTD_decompress / LZ4_decompress_safe:
// the stage-1 worst case of a chunk, or the whole frame's bytes if larger (DecompressChunk's bound is w*h*step,
// cloudini.cpp:672-675), plus 64.
static size_t stage2_max_body(const cldn_info_t& info, size_t pts, bool* ok) {
  cldn_info_t plain = info;
  plain.compression_opt = CLDN_COMP_NONE;
  const size_t m = max_compressed_size(plain, std::min<size_t>(pts, kChunkPoints), false, ok);
  return std::max<size_t>(m, pts * info.point_step) + 64;
}

// CLDN_B200_ZSTD_HOST=1: the host-pointer API decompresses ZSTD with the system libzstd, chunk after chunk, as before the
// device decompressor existed (a comparison / bisecting aid).
static bool zstd_host_route() {
  const char* v = getenv("CLDN_B200_ZSTD_HOST");
  return v && v[0] == '1';
}

// The stage-2 kernels of one launch: every chunk of L is decompressed into its slot, LZ4 or ZSTD (`zstd`, into at most
// body_cap bytes), and the slots are re-framed into one stage-1 payload per frame (sizes in L.sizes). reserve_only: size
// the ZSTD literal scratch `lit` and launch nothing.
static int launch_stage2(cudaStream_t stream, bool zstd, const Lz4Launch& L, size_t body_cap, DevBuf<uint8_t>& lit, bool reserve_only) {
  if (zstd) {
    // one warp per chunk up to 2048 warps (literal scratch: <= 128 KB each), then a grid stride
    const uint32_t wpc = zstd_warps_per_cta();
    const size_t ctas = std::max<size_t>(1, std::min<size_t>((L.n_chunks_total + wpc - 1) / wpc, 2048 / wpc));
    if (int rc = lit.reserve(ctas * wpc * zstd_lit_scratch_bytes(static_cast<uint32_t>(body_cap)))) return rc;
    if (reserve_only) return CLDN_OK;
    ZstdLaunch Z{};
    Z.L = L;
    Z.body_cap = static_cast<uint32_t>(body_cap);
    Z.n_ctas = static_cast<uint32_t>(ctas);
    Z.lit_scratch = lit.p;
    if (launch_zstd_decompress(Z, stream) < 0) { set_error("ZSTD kernel launch failed"); return CLDN_ERR_CUDA; }
  } else if (!reserve_only && launch_lz4_decompress(L, stream) < 0) {
    set_error("LZ4 kernel launch failed");
    return CLDN_ERR_CUDA;
  }
  return CLDN_OK;
}

// Stage 2 on the device, LZ4 or ZSTD (info.compression_opt): every chunk is decompressed into a slot (cldn_lz4.cu,
// cldn_zstd.cu) and the slots are re-framed into one stage-1 payload per frame in the decoder's arena. On return p1 / b1
// are those payloads, behind one read-back of their sizes (8 bytes per frame) and one synchronisation. A slot holds the
// stage-1 worst case of a 32768-point chunk: a larger chunk body cannot be a stage-1 chunk and is refused as damaged.
// `frame_points` as decode_batch_device takes it: the frames of one launch share one chunk bound (that of the largest).
// `out_capacities`, if given, are checked before any scratch is sized from the (untrusted) header.
static int stage2_device(cldn_decoder* d, const cldn_info_t& info, size_t n_frames, const void* const* payloads,
                         const size_t* payload_bytes, const size_t* out_capacities, const uint64_t* frame_points,
                         std::vector<const void*>& p1, std::vector<size_t>& b1) {
  const bool zstd = info.compression_opt == CLDN_COMP_ZSTD;
  cldn_info_t plain = info;
  plain.compression_opt = CLDN_COMP_NONE;
  // ZSTD checks the capacity before the point counts, LZ4 after them; the two forms differ for point_step 0
  const uint64_t wh = static_cast<uint64_t>(info.width) * info.height;
  for (size_t f = 0; zstd && out_capacities && f < n_frames; ++f) {
    if (out_capacities[f] / std::max<uint32_t>(info.point_step, 1u) < (frame_points ? frame_points[f] : wh)) { set_error("Output buffer is too small to hold the decoded data"); return CLDN_ERR_BUFFER_TOO_SMALL; }
  }
  FrameChunks fc;
  if (int rc = fc.init(info, n_frames, frame_points)) return rc;
  for (size_t f = 0; !zstd && out_capacities && f < n_frames; ++f) {
    if (out_capacities[f] < fc.points[f] * info.point_step) { set_error("Output buffer is too small to hold the decoded data"); return CLDN_ERR_BUFFER_TOO_SMALL; }
  }
  bool ok;
  const size_t chunk_worst = max_compressed_size(plain, std::min<size_t>(fc.max_points, kChunkPoints), false, &ok) + 64;
  if (!ok) return CLDN_ERR_INVALID_ARGUMENT;
  // ZSTD: a chunk may decompress to max_body bytes (the host-pointer bound), but not beyond its slot
  const size_t body_cap = zstd ? std::min(stage2_max_body(info, fc.max_points, &ok), chunk_worst) : chunk_worst;
  const size_t slot = (body_cap + 15) & ~size_t(15);
  fc.place(slot);
  const size_t chunks = fc.chunks;
  if (chunks > 0x7FFFFFFFull || slot > 0xFFFFFFF0ull) { set_error("batch too large"); return CLDN_ERR_UNSUPPORTED; }
  for (size_t f = 0; zstd && f < n_frames; ++f) {  // a frame without points has no chunk to decompress
    if (fc.frame_chunks(f) == 0 && payload_bytes[f] != 0) { set_error("%s", dev_error_text(DEV_ERR_CHUNK_COUNT)); return CLDN_ERR_CORRUPT_DATA; }
  }
  if (int rc = d->d_s1.reserve(std::max<size_t>(fc.arena, 256))) return rc;
  if (int rc = d->d_lz_scratch.reserve(std::max<size_t>(chunks, 1) * slot)) return rc;
  if (int rc = d->d_lz_chunk_sizes.reserve(chunks + 1)) return rc;
  if (int rc = d->d_lz_chunk_frame.reserve(chunks + 1)) return rc;
  if (int rc = d->d_lz_frames.reserve(n_frames)) return rc;
  if (int rc = d->d_lz_sizes.reserve(n_frames)) return rc;
  if (int rc = d->h_lz_sizes.reserve(n_frames)) return rc;
  Lz4Frame* hf = nullptr; int hf_slot = 0;
  uint32_t* hcf = nullptr; int hcf_slot = 0;
  if (int rc = d->h_lz_frames.acquire(n_frames, &hf, &hf_slot)) return rc;
  if (int rc = d->h_lz_chunk_frame.acquire(chunks + 1, &hcf, &hcf_slot)) return rc;
  uint32_t cb = 0;
  for (size_t f = 0; f < n_frames; ++f) {
    Lz4Frame& F = hf[f];
    memset(&F, 0, sizeof(F));
    F.packed_in = static_cast<const uint8_t*>(payloads[f]);
    F.packed_in_bytes = payload_bytes[f];
    F.plain_out = d->d_s1.p + fc.s1_off[f];
    F.plain_cap = fc.s1_cap[f];
    F.n_chunks = static_cast<uint32_t>(fc.frame_chunks(f));
    F.chunk_begin = cb;
    for (uint32_t c = 0; c < F.n_chunks; ++c) hcf[cb + c] = static_cast<uint32_t>(f);
    cb += F.n_chunks;
  }
  CUDA_TRY(cudaMemcpyAsync(d->d_lz_frames.p, hf, n_frames * sizeof(Lz4Frame), cudaMemcpyHostToDevice, d->stream));
  if (int rc = d->h_lz_frames.commit(hf_slot, d->stream)) return rc;
  if (chunks) CUDA_TRY(cudaMemcpyAsync(d->d_lz_chunk_frame.p, hcf, chunks * sizeof(uint32_t), cudaMemcpyHostToDevice, d->stream));
  if (int rc = d->h_lz_chunk_frame.commit(hcf_slot, d->stream)) return rc;
  Lz4Launch L{};
  L.frames = d->d_lz_frames.p;
  L.n_frames = static_cast<uint32_t>(n_frames);
  L.n_chunks_total = static_cast<uint32_t>(chunks);
  L.chunk_frame = d->d_lz_chunk_frame.p;
  L.scratch = d->d_lz_scratch.p;
  L.slot_stride = static_cast<uint32_t>(slot);
  L.chunk_sizes = d->d_lz_chunk_sizes.p;
  L.sizes = d->d_lz_sizes.p;
  L.err = d->d_err.p;
  L.frame_err = d->frame_err;
  if (int rc = launch_stage2(d->stream, zstd, L, body_cap, d->d_zs_lit, false)) return rc;
  CUDA_TRY(cudaMemcpyAsync(d->h_lz_sizes.p, d->d_lz_sizes.p, n_frames * sizeof(uint64_t), cudaMemcpyDeviceToHost, d->stream));
  if (int rc = check_device_error(d->stream, d->d_err.p, d->h_err.p)) return rc;  // synchronises; damaged frames stop here
  p1.resize(n_frames);
  b1.resize(n_frames);
  for (size_t f = 0; f < n_frames; ++f) { p1[f] = d->d_s1.p + fc.s1_off[f]; b1[f] = static_cast<size_t>(d->h_lz_sizes.p[f]); }
  return CLDN_OK;
}

// The decoder writes only the declared field bytes: where the layout has padding, a staged output starts as the caller's
// bytes, so that the padding comes back unchanged.
static int stage_padding(const cldn_decoder* d, void* staged, const void* out, size_t bytes, cudaStream_t stream) {
  if (d->has_padding && bytes) CUDA_TRY(cudaMemcpyAsync(staged, out, bytes, cudaMemcpyHostToDevice, stream));
  return CLDN_OK;
}

// Host pointers, compression ZSTD: the payloads go up compressed, the device decompresses and decodes them, the points
// come back (with the caller's padding bytes, like the uncompressed host path). `device_out` (CLDN_MEM_DEVICE_POINTS):
// the points are decoded in place into the caller's device buffers and the error word is left to the caller.
static int decode_batch_host_zstd(cldn_decoder* d, const cldn_info_t& info, size_t n_frames, const void* const* payloads,
                                  const size_t* payload_bytes, void* const* outs, const uint64_t* frame_points, bool device_out) {
  std::vector<void*> din;
  if (int rc = stage_layout(d->d_in, n_frames, payload_bytes, din)) return rc;
  for (size_t f = 0; f < n_frames; ++f) {
    if (payload_bytes[f]) CUDA_TRY(cudaMemcpyAsync(din[f], payloads[f], payload_bytes[f], cudaMemcpyHostToDevice, d->stream));
  }
  std::vector<const void*> p1;
  std::vector<size_t> b1;
  if (int rc = stage2_device(d, info, n_frames, din.data(), payload_bytes, nullptr, frame_points, p1, b1)) return rc;
  cldn_info_t plain = info;
  plain.compression_opt = CLDN_COMP_NONE;
  if (int rc = decoder_update_plan(d, plain)) return rc;
  const size_t wh = static_cast<size_t>(info.width) * info.height;
  std::vector<size_t> caps(n_frames);
  for (size_t f = 0; f < n_frames; ++f) caps[f] = static_cast<size_t>(frame_points ? frame_points[f] : wh) * info.point_step;
  if (device_out) return decode_batch_device(d, plain, n_frames, p1.data(), b1.data(), outs, caps.data(), frame_points);
  std::vector<void*> dout;
  if (int rc = stage_layout(d->d_out, n_frames, caps.data(), dout)) return rc;
  for (size_t f = 0; f < n_frames; ++f) {
    if (int rc = stage_padding(d, dout[f], outs[f], caps[f], d->stream)) return rc;
  }
  if (int rc = decode_batch_device(d, plain, n_frames, p1.data(), b1.data(), dout.data(), caps.data(), frame_points)) return rc;
  for (size_t f = 0; f < n_frames; ++f) {
    if (caps[f]) CUDA_TRY(cudaMemcpyAsync(outs[f], dout[f], caps[f], cudaMemcpyDeviceToHost, d->stream));
  }
  return check_device_error(d->stream, d->d_err.p, d->h_err.p);
}

// Host pointers, no stage 2. `frame_points` as decode_batch_device takes it. `device_out` (CLDN_MEM_DEVICE_POINTS): the
// points are decoded in place into the caller's device buffers, and the call returns once the payloads have been read,
// leaving the error word to the caller.
static int decode_batch_host_plain(cldn_decoder* d, const cldn_info_t& info, size_t n_frames, const void* const* payloads,
                                   const size_t* payload_bytes, void* const* outs, const size_t* out_capacities,
                                   const uint64_t* frame_points, bool device_out) {
  if (int rc = decoder_update_plan(d, info)) return rc;
  const size_t wh = static_cast<size_t>(info.width) * info.height;
  std::vector<size_t> out_need(n_frames);
  for (size_t f = 0; f < n_frames; ++f) {
    out_need[f] = static_cast<size_t>(frame_points ? frame_points[f] : wh) * info.point_step;
    if (out_capacities[f] < out_need[f]) { set_error("Output buffer is too small to hold the decoded data"); return CLDN_ERR_BUFFER_TOO_SMALL; }
  }
  std::vector<void*> din, dout;
  if (int rc = stage_layout(d->d_in, n_frames, payload_bytes, din)) return rc;
  if (device_out) dout.assign(outs, outs + n_frames);
  else if (int rc = stage_layout(d->d_out, n_frames, out_need.data(), dout)) return rc;
  if (int rc = d->pipe.ensure(2 * n_frames + 1)) return rc;
  // an earlier CLDN_MEM_DEVICE_POINTS call may have returned with its decode still reading the staged payloads on the
  // handle's stream: whatever this call's memory kind, its uploads into d_in wait for that decode
  CUDA_TRY(cudaEventRecord(d->pipe.ev[2 * n_frames], d->stream));
  CUDA_TRY(cudaStreamWaitEvent(d->pipe.h2d, d->pipe.ev[2 * n_frames], 0));
  // frame f: upload on the h2d stream -> decode on the handle's stream -> download on the d2h stream
  for (size_t f = 0; f < n_frames; ++f) {
    if (payload_bytes[f]) CUDA_TRY(cudaMemcpyAsync(din[f], payloads[f], payload_bytes[f], cudaMemcpyHostToDevice, d->pipe.h2d));
    if (!device_out) {
      if (int rc = stage_padding(d, dout[f], outs[f], out_need[f], d->pipe.h2d)) return rc;
    }
    CUDA_TRY(cudaEventRecord(d->pipe.ev[2 * f], d->pipe.h2d));
    CUDA_TRY(cudaStreamWaitEvent(d->stream, d->pipe.ev[2 * f], 0));
    const uint64_t* pts = frame_points ? frame_points + f : nullptr;
    uint32_t* const group_err = d->frame_err;
    if (group_err) d->frame_err = group_err + f;  // one launch per frame: frame 0 of that launch is frame f of the group
    const int rc = decode_batch_device(d, info, 1, &din[f], &payload_bytes[f], &dout[f], &out_need[f], pts);
    d->frame_err = group_err;
    if (rc) return rc;
    if (device_out) continue;
    CUDA_TRY(cudaEventRecord(d->pipe.ev[2 * f + 1], d->stream));
    CUDA_TRY(cudaStreamWaitEvent(d->pipe.d2h, d->pipe.ev[2 * f + 1], 0));
    if (out_need[f]) CUDA_TRY(cudaMemcpyAsync(outs[f], dout[f], out_need[f], cudaMemcpyDeviceToHost, d->pipe.d2h));
  }
  if (device_out) {
    CUDA_TRY(cudaStreamSynchronize(d->pipe.h2d));  // the payloads have been read
    return CLDN_OK;
  }
  CUDA_TRY(cudaStreamSynchronize(d->pipe.d2h));
  // a failed decode must not hand back garbage silently: the error word is checked after everything has drained
  return check_device_error(d->stream, d->d_err.p, d->h_err.p);
}

// Whether decode_frames decodes frames of `info` in `mem` whole, with an error word per frame (DecLaunch /
// Lz4Launch::frame_err). The others go frame by frame: LZ4 with host payloads and CLDN_B200_ZSTD_HOST through the host
// libraries (decode_batch_impl), and compressions that no route decodes. CLDN_MEM_DEVICE_POINTS takes the host routes.
static bool route_has_frame_errors(int mem, const cldn_info_t& info) {
  switch (info.compression_opt) {
    case CLDN_COMP_NONE: return true;
    case CLDN_COMP_LZ4: return mem == CLDN_MEM_DEVICE;
    case CLDN_COMP_ZSTD: return mem == CLDN_MEM_DEVICE || !zstd_host_route();
    default: return false;
  }
}

// Frames that share `info`, each with frame_points[f] points (nullptr: info.width * info.height), through the one route
// of their memory kind and compression: device NONE, LZ4 or ZSTD (stage 2 then one fused stage-1 launch), host plain, or
// host ZSTD decompressed on the device. Host payloads (CLDN_MEM_HOST, CLDN_MEM_DEVICE_POINTS) take the host routes.
// Routes that write device points leave the error word to the caller; routes that write host points check it.
static int decode_frames(cldn_decoder* d, int mem, const cldn_info_t& info, size_t n_frames, const void* const* payloads,
                         const size_t* payload_bytes, void* const* outs, const size_t* out_capacities,
                         const uint64_t* frame_points) {
  if (mem != CLDN_MEM_DEVICE) {
    const bool device_out = mem == CLDN_MEM_DEVICE_POINTS;
    if (info.compression_opt == CLDN_COMP_ZSTD) return decode_batch_host_zstd(d, info, n_frames, payloads, payload_bytes, outs, frame_points, device_out);
    return decode_batch_host_plain(d, info, n_frames, payloads, payload_bytes, outs, out_capacities, frame_points, device_out);
  }
  if (info.compression_opt != CLDN_COMP_LZ4 && info.compression_opt != CLDN_COMP_ZSTD) {
    return decode_batch_device(d, info, n_frames, payloads, payload_bytes, outs, out_capacities, frame_points);
  }
  std::vector<const void*> p1;
  std::vector<size_t> b1;
  if (int rc = stage2_device(d, info, n_frames, payloads, payload_bytes, out_capacities, frame_points, p1, b1)) return rc;
  cldn_info_t plain = info;
  plain.compression_opt = CLDN_COMP_NONE;
  return decode_batch_device(d, plain, n_frames, p1.data(), b1.data(), outs, out_capacities, frame_points);
}

static int decode_batch_impl(cldn_decoder_t* d, const cldn_info_t* info, size_t n_frames, const void* const* payloads,
                             const size_t* payload_bytes, void* const* outs, const size_t* out_capacities, int mem, int sync) {
  if (!d || !info || (n_frames && (!payloads || !payload_bytes || !outs || !out_capacities))) {
    set_error("null argument");
    return CLDN_ERR_INVALID_ARGUMENT;
  }
  if (n_frames == 0) return CLDN_OK;
  CUDA_TRY(cudaSetDevice(d->device));
  if (mem == CLDN_MEM_DEVICE) {
    if (int rc = decode_frames(d, mem, *info, n_frames, payloads, payload_bytes, outs, out_capacities, nullptr)) return rc;
    if (sync) return check_device_error(d->stream, d->d_err.p, d->h_err.p);
    return CLDN_OK;
  }
  if (mem != CLDN_MEM_HOST && mem != CLDN_MEM_DEVICE_POINTS) { set_error("bad mem kind"); return CLDN_ERR_INVALID_ARGUMENT; }
  // the reference rejects a payload that still carries the header (cloudini.cpp:640-643)
  for (size_t f = 0; f < n_frames; ++f) {
    if (payload_bytes[f] >= 10 && memcmp(payloads[f], "CLOUDINI_V", 10) == 0) {
      set_error("compressed_data contains the header. You should use DecodeHeader first");
      return CLDN_ERR_INVALID_ARGUMENT;
    }
  }
  if (info->compression_opt != CLDN_COMP_NONE) {
    // stage 2 first (ZSTD: on the device; LZ4: host library), then the ordinary stage-1 decode of the re-framed payload
    if (info->compression_opt > CLDN_COMP_ZSTD) { set_error("Unsupported compression option"); return CLDN_ERR_INVALID_ARGUMENT; }
    const bool device_zstd = info->compression_opt == CLDN_COMP_ZSTD && !zstd_host_route();
    if (!device_zstd && !g_stage2.load(info->compression_opt)) return CLDN_ERR_UNSUPPORTED;
    cldn_info_t plain = *info;
    plain.compression_opt = CLDN_COMP_NONE;
    bool ok;
    const size_t pts = static_cast<size_t>(info->width) * info->height;
    for (size_t f = 0; f < n_frames; ++f) {  // before any scratch is sized from the (untrusted) header
      if (out_capacities[f] / std::max<uint32_t>(info->point_step, 1u) < pts) {
        set_error("Output buffer is too small to hold the decoded data");
        return CLDN_ERR_BUFFER_TOO_SMALL;
      }
    }
    const size_t max_body = stage2_max_body(*info, pts, &ok);
    if (!ok) return CLDN_ERR_INVALID_ARGUMENT;
    if (!device_zstd) {  // the host library, frame by frame
      for (size_t f = 0; f < n_frames; ++f) {
        if (int rc = stage2_decompress_payload(info->compression_opt, static_cast<const uint8_t*>(payloads[f]), payload_bytes[f], d->s2_tmp, max_body)) return rc;
        const void* p1 = d->s2_tmp.data();
        const size_t b1 = d->s2_tmp.size();
        if (int rc = decode_batch_impl(d, &plain, 1, &p1, &b1, &outs[f], &out_capacities[f], mem, 1)) return rc;
      }
      return CLDN_OK;
    }
  }
  if (int rc = decode_frames(d, mem, *info, n_frames, payloads, payload_bytes, outs, out_capacities, nullptr)) return rc;
  if (mem == CLDN_MEM_DEVICE_POINTS && sync) return check_device_error(d->stream, d->d_err.p, d->h_err.p);
  return CLDN_OK;
}

// ---- complete blobs, any mix of layouts and sizes (cldn_b200_decode_blobs) -----------------------------------------
constexpr size_t kBlobPrefix = 4096;  // bytes of every device-resident blob fetched for its header

// Whether a header whose first `len` bytes are at p may parse once more of the blob is read: a YAML header with no NUL
// yet, a binary header whose fields run past `len`. *want: bytes that would settle it, where the binary layout says so.
static bool header_runs_past(const uint8_t* p, size_t len, size_t* want) {
  *want = 0;
  if (len < 12 || memcmp(p, "CLOUDINI_V", 10) != 0) return false;
  auto digit = [](uint8_t c) -> int { return (c >= '0' && c <= '9') ? c - '0' : 0; };
  const int version = digit(p[10]) * 10 + digit(p[11]);
  if (version < 2 || version > CLDN_ENCODING_VERSION) return false;  // refused whatever follows
  if (len < 14) return true;
  if (p[12] == '\n' && p[13] != '{') return memchr(p + 13, 0, len - 13) == nullptr;
  size_t pos = 12 + 14;  // binary layout of cldn_b200_decode_header: width, height, point_step, options, field count
  if (len < pos) { *want = pos; return true; }
  uint16_t nf;
  memcpy(&nf, p + pos - 2, 2);
  if (nf > CLDN_MAX_FIELDS) return false;
  for (uint16_t i = 0; i < nf; ++i) {
    if (len < pos + 2) { *want = pos + 2; return true; }
    uint16_t nl;
    memcpy(&nl, p + pos, 2);
    pos += 2 + nl + 9;
    if (len < pos) { *want = pos; return true; }
  }
  return false;
}

// Headers of every blob, parsed by cldn_b200_decode_header: in place for host memory. Device blobs: one launch gathers
// the first min(blob_bytes, kBlobPrefix) bytes of every blob, packed back to back, behind one read-back and one
// synchronisation; a header that runs past its prefix is read again, twice as long each time (or as long as its binary
// layout says), until it parses or the blob ends, so every frame gets the status its complete header gives.
static int read_blob_headers(cldn_decoder* d, size_t n, const void* const* blobs, const size_t* blob_bytes, int mem,
                             std::vector<size_t>& hdr, int32_t* status) {
  hdr.assign(n, 0);
  auto parse = [&](size_t f, const uint8_t* p, size_t len) {
    status[f] = cldn_b200_decode_header(p, len, &d->frame_infos[f], &hdr[f]);
    d->frame_errors[f] = status[f] == CLDN_OK ? "" : cldn_b200_last_error();
    if (status[f] != CLDN_OK) d->frame_infos[f] = cldn_info_t{};
  };
  if (mem != CLDN_MEM_DEVICE) {  // host blobs
    for (size_t f = 0; f < n; ++f) parse(f, static_cast<const uint8_t*>(blobs[f]), blob_bytes[f]);
    return CLDN_OK;
  }
  if (n > 0x7FFFFFFFull) { set_error("batch too large"); return CLDN_ERR_UNSUPPORTED; }
  if (int rc = d->h_blob_tab.reserve(3 * n)) return rc;
  if (int rc = d->d_blob_tab.reserve(3 * n)) return rc;
  uint64_t* tab = d->h_blob_tab.p;
  size_t total = 0;
  for (size_t f = 0; f < n; ++f) {
    tab[f] = reinterpret_cast<uint64_t>(blobs[f]);
    tab[n + f] = blobs[f] ? std::min(blob_bytes[f], kBlobPrefix) : 0;
    tab[2 * n + f] = total;
    total += (tab[n + f] + 15) & ~size_t(15);
  }
  if (int rc = d->h_prefix.reserve(total + 16)) return rc;
  if (int rc = d->d_prefix.reserve(total + 16)) return rc;
  CUDA_TRY(cudaMemcpyAsync(d->d_blob_tab.p, tab, 3 * n * sizeof(uint64_t), cudaMemcpyHostToDevice, d->stream));
  if (launch_gather_prefixes(d->d_blob_tab.p, static_cast<uint32_t>(n), d->d_prefix.p, d->stream) < 0) { set_error("header gather launch failed"); return CLDN_ERR_CUDA; }
  CUDA_TRY(cudaGetLastError());
  if (total) CUDA_TRY(cudaMemcpyAsync(d->h_prefix.p, d->d_prefix.p, total, cudaMemcpyDeviceToHost, d->stream));
  CUDA_TRY(cudaStreamSynchronize(d->stream));
  std::vector<uint8_t> more;
  for (size_t f = 0; f < n; ++f) {
    if (!blobs[f]) { parse(f, nullptr, blob_bytes[f]); continue; }
    const uint8_t* p = d->h_prefix.p + tab[2 * n + f];
    size_t got = static_cast<size_t>(tab[n + f]), want = 0;
    while (got < blob_bytes[f] && header_runs_past(p, got, &want)) {
      got = std::min(blob_bytes[f], std::max(2 * got, want));
      more.resize(got);
      CUDA_TRY(cudaMemcpyAsync(more.data(), blobs[f], got, cudaMemcpyDeviceToHost, d->stream));
      CUDA_TRY(cudaStreamSynchronize(d->stream));
      p = more.data();
    }
    parse(f, p, got);
  }
  return CLDN_OK;
}

// The same layout, width and height aside: everything a plan and a header (but for its dims) depend on.
static bool same_layout(const cldn_info_t& a, const cldn_info_t& b) {
  if (!same_fields(a, b) || strncmp(a.encoding_config, b.encoding_config, sizeof(a.encoding_config)) != 0) return false;
  for (uint32_t i = 0; i < a.n_fields; ++i) {
    if (strncmp(a.fields[i].name, b.fields[i].name, CLDN_MAX_NAME) != 0) return false;
  }
  return true;
}

// Frames decoded by one fused launch: the same layout (width and height aside) and compression. LZ4 and ZSTD frames also
// share the bound of a decompressed chunk, which depends on the points of a chunk, so that every frame is bounded
// exactly as cldn_b200_decode bounds it.
static bool same_group(const cldn_info_t& a, uint64_t a_points, const cldn_info_t& b, uint64_t b_points) {
  if (!same_layout(a, b)) return false;
  return a.compression_opt == CLDN_COMP_NONE || std::min<uint64_t>(a_points, kChunkPoints) == std::min<uint64_t>(b_points, kChunkPoints);
}

// One group, synchronously, with an error word per frame (DecLaunch / Lz4Launch::frame_err). Device memory: one fused
// stage-1 launch (behind one stage-2 launch for LZ4 / ZSTD). Host memory: the staging of cldn_b200_decode_batch.
// frame_word[i] != 0: member i failed. A non-OK return (a CUDA error, a refused group, or an error no frame claimed)
// says nothing about any single member.
static int decode_blob_group(cldn_decoder* d, int mem, const cldn_info_t& info, size_t n, const void* const* payloads,
                             const size_t* payload_bytes, void* const* outs, const size_t* caps, const uint64_t* points,
                             std::vector<uint32_t>& frame_word) {
  if (int rc = d->d_frame_err.reserve(n)) return rc;
  if (int rc = d->h_frame_err.reserve(n)) return rc;
  CUDA_TRY(cudaMemsetAsync(d->d_frame_err.p, 0, n * sizeof(uint32_t), d->stream));
  d->frame_err = d->d_frame_err.p;
  int rc = decode_frames(d, mem, info, n, payloads, payload_bytes, outs, caps, points);
  // the launch word: errors no frame claimed (the routes that write host points have checked it)
  if (rc == CLDN_OK && mem != CLDN_MEM_HOST) rc = check_device_error(d->stream, d->d_err.p, d->h_err.p);
  d->frame_err = nullptr;
  if (rc) return rc;
  CUDA_TRY(cudaMemcpyAsync(d->h_frame_err.p, d->d_frame_err.p, n * sizeof(uint32_t), cudaMemcpyDeviceToHost, d->stream));
  CUDA_TRY(cudaStreamSynchronize(d->stream));
  frame_word.assign(d->h_frame_err.p, d->h_frame_err.p + n);
  return CLDN_OK;
}

// Every frame ends with the status cldn_b200_decode_header + cldn_b200_decode give it alone. Frames go through their
// group's fused launch, whose per-frame error words say which frames failed; only those are decoded again alone, which
// gives them exactly the single-blob status and message (the kernels report the first defect they meet, the reference
// the first in stream order). A group that fails as a whole (an error no frame claimed, a refused plan) has all its
// frames decoded alone. Frames that the single-frame path handles frame by frame anyway (LZ4 with host pointers,
// CLDN_B200_ZSTD_HOST) or refuses before any launch also take it directly.
static int decode_blobs_impl(cldn_decoder* d, size_t n, const void* const* blobs, const size_t* blob_bytes, void* const* outs,
                             const size_t* caps, int mem, int32_t* status, size_t* decoded_bytes) {
  if (!d || (n && !status)) { set_error("null argument"); return CLDN_ERR_INVALID_ARGUMENT; }
  d->frame_errors.assign(n, "frame not decoded");
  d->frame_infos.assign(n, cldn_info_t{});
  for (size_t f = 0; f < n; ++f) {
    status[f] = CLDN_ERR_INTERNAL;
    if (decoded_bytes) decoded_bytes[f] = 0;
  }
  auto result = [&]() -> int {
    for (size_t f = 0; f < n; ++f) {
      if (status[f] != CLDN_OK) { set_error("frame %zu: %s", f, d->frame_errors[f].c_str()); return status[f]; }
    }
    return CLDN_OK;
  };
  auto fail_all = [&](int rc) {
    const std::string msg = cldn_b200_last_error();
    for (size_t f = 0; f < n; ++f) { status[f] = rc; d->frame_errors[f] = msg; }
    return result();
  };
  if (n == 0) return CLDN_OK;
  if (!blobs || !blob_bytes || !outs || !caps) { set_error("null argument"); return fail_all(CLDN_ERR_INVALID_ARGUMENT); }
  if (mem != CLDN_MEM_HOST && mem != CLDN_MEM_DEVICE && mem != CLDN_MEM_DEVICE_POINTS) { set_error("bad mem kind"); return fail_all(CLDN_ERR_INVALID_ARGUMENT); }
  if (cudaSetDevice(d->device) != cudaSuccess) { set_error("cudaSetDevice failed"); return fail_all(CLDN_ERR_CUDA); }
  std::vector<size_t> hdr;
  if (int rc = read_blob_headers(d, n, blobs, blob_bytes, mem, hdr, status)) return fail_all(rc);

  std::vector<const void*> payload(n);
  std::vector<size_t> payload_bytes(n);
  std::vector<uint64_t> points(n);
  std::vector<uint8_t> todo(n), alone(n);
  for (size_t f = 0; f < n; ++f) {
    if (status[f] != CLDN_OK) continue;
    const cldn_info_t& I = d->frame_infos[f];
    todo[f] = 1;
    payload[f] = static_cast<const uint8_t*>(blobs[f]) + hdr[f];
    payload_bytes[f] = blob_bytes[f] - hdr[f];
    points[f] = static_cast<uint64_t>(I.width) * I.height;
    alone[f] = !route_has_frame_errors(mem, I) || I.version < 3 || points[f] > 0xFFFFFFFFull || points[f] * I.point_step > caps[f] ||
               (mem != CLDN_MEM_DEVICE && payload_bytes[f] >= 10 && memcmp(payload[f], "CLOUDINI_V", 10) == 0);
  }
  std::vector<size_t> members;
  std::vector<const void*> g_payload;
  std::vector<size_t> g_bytes, g_caps;
  std::vector<void*> g_outs;
  std::vector<uint64_t> g_points;
  std::vector<uint32_t> g_word;
  for (size_t f = 0; f < n; ++f) {
    if (!todo[f] || alone[f]) continue;
    members.clear();
    for (size_t g = f; g < n; ++g) {
      if (todo[g] && !alone[g] && same_group(d->frame_infos[f], points[f], d->frame_infos[g], points[g])) {
        members.push_back(g);
        todo[g] = 0;
      }
    }
    g_payload.clear(); g_bytes.clear(); g_caps.clear(); g_outs.clear(); g_points.clear();
    for (size_t g : members) {
      g_payload.push_back(payload[g]);
      g_bytes.push_back(payload_bytes[g]);
      g_outs.push_back(outs[g]);
      g_caps.push_back(caps[g]);
      g_points.push_back(points[g]);
    }
    // every member has its own point count: the group's info carries none, so that the decoder's cached plan (keyed by
    // the whole info) survives from call to call whatever the frames' sizes
    cldn_info_t layout = d->frame_infos[f];
    layout.width = layout.height = 0;
    const int rc = decode_blob_group(d, mem, layout, members.size(), g_payload.data(), g_bytes.data(), g_outs.data(),
                                     g_caps.data(), g_points.data(), g_word);
    for (size_t i = 0; i < members.size(); ++i) {
      const size_t g = members[i];
      if (rc != CLDN_OK || g_word[i] != 0) {
        todo[g] = 1;
        alone[g] = 1;
        continue;
      }
      status[g] = CLDN_OK;
      d->frame_errors[g].clear();
      if (decoded_bytes) decoded_bytes[g] = static_cast<size_t>(points[g] * d->frame_infos[g].point_step);
    }
  }
  for (size_t f = 0; f < n; ++f) {
    if (!todo[f]) continue;
    status[f] = decode_batch_impl(d, &d->frame_infos[f], 1, &payload[f], &payload_bytes[f], &outs[f], &caps[f], mem, 1);
    d->frame_errors[f] = status[f] == CLDN_OK ? "" : cldn_b200_last_error();
    if (status[f] == CLDN_OK && decoded_bytes) decoded_bytes[f] = static_cast<size_t>(points[f] * d->frame_infos[f].point_step);
  }
  return result();
}

// ---- complete device blobs of one prepared layout, without the host (cldn_b200_decode_blobs_async) ------------------
// Everything the calls of one prepared layout and shape read: uploaded and allocated once by
// cldn_b200_decoder_prepare_blobs, apart from the buffers of the handle's other calls, so that a call allocates, copies
// from the host and synchronises nothing, and a CUDA graph that captured one stays valid until the next prepare.
struct AsyncBlobs {
  cldn_info_t info;       // the layout as its header states it, width = height = 0
  Plan plan;              // stage 1 (compression NONE)
  size_t max_frames = 0;
  uint32_t slots = 0;     // chunk slots per frame: those of max_points
  uint64_t tiles_per_frame = 0;
  uint64_t chunk_bytes_max = 0;  // the chunk bodies the tile grid is sized for
  size_t body_cap = 0;    // stage 2: bytes a chunk may decompress to
  DevBuf<Plan> d_plan;
  DevBuf<uint8_t> d_tmpl;
  DevBuf<DecFrame> d_frames;
  DevBuf<Lz4Frame> d_lz_frames;
  DevBuf<uint32_t> d_lz_chunk_frame, d_lz_chunk_sizes;
  DevBuf<uint64_t> d_lz_sizes;
  DevBuf<uint8_t> d_s1, d_lz_scratch, d_zs_lit;
  DevBuf<uint32_t> d_frame_err, d_err;
  DecStage1 s1;
  AsyncLaunch A{};  // all but the call's arrays
  Lz4Launch Z{};    // all but the call's counts

  // every call launches the grids of max_frames frames: the frames past its own are empty
  Stage1Shape shape() const {
    Stage1Shape s;
    s.n_frames = static_cast<uint32_t>(max_frames);
    s.chunks = static_cast<uint64_t>(max_frames) * slots;
    s.tiles = static_cast<uint64_t>(max_frames) * tiles_per_frame;
    s.chunk_bytes_max = chunk_bytes_max;
    s.uniform_chunks = slots;
    s.replayable = true;
    s.empty_slots = true;
    return s;
  }
};
void AsyncBlobsDeleter::operator()(AsyncBlobs* a) const { delete a; }

static int prepare_blobs_impl(cldn_decoder* d, const cldn_info_t* layout, size_t max_frames, uint64_t max_points) {
  if (!d || !layout) { set_error("null argument"); return CLDN_ERR_INVALID_ARGUMENT; }
  if (max_frames == 0 || max_frames > 0x7FFFFFFFull) { set_error("max_frames must be 1 .. 2^31 - 1"); return CLDN_ERR_INVALID_ARGUMENT; }
  if (max_points > 0xFFFFFFFFull) { set_error("max_points_per_frame must be below 2^32"); return CLDN_ERR_UNSUPPORTED; }
  if (layout->version < 3 || layout->version > CLDN_ENCODING_VERSION) {
    set_error("wire version %d: cldn_b200_decode_blobs_async decodes versions 3 .. %d", layout->version, CLDN_ENCODING_VERSION);
    return CLDN_ERR_UNSUPPORTED;
  }
  if (layout->compression_opt > CLDN_COMP_ZSTD) { set_error("Unsupported compression option"); return CLDN_ERR_INVALID_ARGUMENT; }
  CUDA_TRY(cudaSetDevice(d->device));
  CUDA_TRY(cudaStreamSynchronize(d->stream));  // kernels of an earlier prepared state may still read it
  d->async.reset();
  std::unique_ptr<AsyncBlobs, AsyncBlobsDeleter> a(new AsyncBlobs());
  // the header every blob of the layout starts with, and the layout decode_blobs reads from it
  cldn_info_t zero = *layout;
  zero.width = zero.height = 0;
  const std::vector<uint8_t> hdr = make_header(zero);
  size_t used = 0;
  if (int rc = cldn_b200_decode_header(hdr.data(), hdr.size(), &a->info, &used)) return rc;
  std::vector<uint8_t> tmpl;
  uint32_t tmpl_len[3];
  if (int rc = header_template(hdr, &tmpl, tmpl_len)) return rc;
  cldn_info_t plain = a->info;
  plain.compression_opt = CLDN_COMP_NONE;
  if (int rc = make_decode_plan(plain, &a->plan)) return rc;
  const bool compressed = a->info.compression_opt != CLDN_COMP_NONE;
  a->max_frames = max_frames;
  a->slots = static_cast<uint32_t>((max_points + kChunkPoints - 1) / kChunkPoints);
  const uint64_t chunks = static_cast<uint64_t>(max_frames) * a->slots;
  if (chunks > 0x7FFFFFFFull) { set_error("max_frames * chunks per frame must be below 2^31"); return CLDN_ERR_UNSUPPORTED; }
  // stage-1 worst case of a chunk of p > 0 points: chunk_a + chunk_b * p (MaxCompressedSize of one chunk)
  bool ok1, ok2;
  const size_t m1 = max_compressed_size(plain, 1, false, &ok1), m2 = max_compressed_size(plain, 2, false, &ok2);
  if (!ok1 || !ok2) return CLDN_ERR_INVALID_ARGUMENT;
  const uint64_t chunk_b = m2 - m1, chunk_a = m1 - chunk_b;
  const uint64_t pc = std::min<uint64_t>(max_points, kChunkPoints);
  a->body_cap = pc ? chunk_a + chunk_b * pc + 64 : 64;  // stage2_device's bound for chunks of pc points
  const size_t slot = (a->body_cap + 15) & ~size_t(15);
  const uint64_t s1_stride = (a->slots * (slot + 4) + 255) & ~uint64_t(255);
  // bound of a chunk's stage-1 bytes for the tile grid: the worst case, with room for the V5 modes that exceed it (one
  // byte per value of a section and 16 more); a larger chunk, which no encoder writes, fails its frame alone
  const uint64_t chunk_bound = (pc ? chunk_a + chunk_b * pc : 0) + (pc + 16) * (a->plan.n_sections + 1) + 128;
  if (chunk_bound > 0xFFFFFFFFull) { set_error("prepared shape too large"); return CLDN_ERR_UNSUPPORTED; }
  a->chunk_bytes_max = chunk_bound;
  // a chunk of b bytes spans at most b / tile + 2 tiles (rounding and misalignment)
  a->tiles_per_frame = a->slots * (chunk_bound / decode_tile_bytes() + 2) + 1;
  if (static_cast<uint64_t>(max_frames) * a->tiles_per_frame > 0x7FFFFFFFull) { set_error("prepared shape too large"); return CLDN_ERR_UNSUPPORTED; }

  if (int rc = a->d_plan.reserve(1)) return rc;
  if (int rc = a->d_tmpl.reserve(tmpl.size())) return rc;
  CUDA_TRY(cudaMemcpyAsync(a->d_plan.p, &a->plan, sizeof(Plan), cudaMemcpyHostToDevice, d->stream));
  CUDA_TRY(cudaMemcpyAsync(a->d_tmpl.p, tmpl.data(), tmpl.size(), cudaMemcpyHostToDevice, d->stream));
  if (int rc = a->d_frames.reserve(max_frames)) return rc;
  if (int rc = a->d_frame_err.reserve(max_frames)) return rc;
  if (int rc = a->d_err.reserve(1, true)) return rc;
  AsyncLaunch& A = a->A;
  A.tmpl = a->d_tmpl.p;
  for (int k = 0; k < 3; ++k) A.tmpl_len[k] = tmpl_len[k];
  A.max_points = max_points;
  A.point_step = a->info.point_step;
  A.slots = a->slots;
  A.compression = a->info.compression_opt;
  A.frames = a->d_frames.p;
  A.chunk_a = chunk_a;
  A.chunk_b = chunk_b;
  A.frame_err = a->d_frame_err.p;
  A.err = a->d_err.p;
  if (compressed) {
    // stage 2: the chunk -> frame table is the prepared shape's (slot gc belongs to frame gc / slots)
    if (int rc = a->d_lz_frames.reserve(max_frames)) return rc;
    if (int rc = a->d_lz_sizes.reserve(max_frames)) return rc;
    if (int rc = a->d_lz_chunk_sizes.reserve(chunks + 1)) return rc;
    if (int rc = a->d_lz_chunk_frame.reserve(chunks + 1)) return rc;
    if (int rc = a->d_lz_scratch.reserve(std::max<uint64_t>(chunks, 1) * slot)) return rc;
    if (int rc = a->d_s1.reserve(std::max<uint64_t>(max_frames * s1_stride, 256))) return rc;
    std::vector<uint32_t> chunk_frame(chunks + 1, 0);
    for (uint64_t gc = 0; gc < chunks; ++gc) chunk_frame[gc] = static_cast<uint32_t>(gc / a->slots);
    CUDA_TRY(cudaMemcpyAsync(a->d_lz_chunk_frame.p, chunk_frame.data(), chunk_frame.size() * sizeof(uint32_t), cudaMemcpyHostToDevice, d->stream));
    Lz4Launch& Z = a->Z;
    Z.frames = a->d_lz_frames.p;
    Z.chunk_frame = a->d_lz_chunk_frame.p;
    Z.scratch = a->d_lz_scratch.p;
    Z.slot_stride = static_cast<uint32_t>(slot);
    Z.chunk_sizes = a->d_lz_chunk_sizes.p;
    Z.sizes = a->d_lz_sizes.p;
    Z.err = a->d_err.p;
    Z.frame_err = a->d_frame_err.p;
    Z.n_frames = static_cast<uint32_t>(max_frames);
    Z.n_chunks_total = static_cast<uint32_t>(chunks);
    if (int rc = launch_stage2(d->stream, A.compression == CLDN_COMP_ZSTD, Z, a->body_cap, a->d_zs_lit, true)) return rc;
    A.lz_frames = a->d_lz_frames.p;
    A.s1 = a->d_s1.p;
    A.s1_stride = s1_stride;
    A.s1_sizes = a->d_lz_sizes.p;
    A.chunk_sizes = a->d_lz_chunk_sizes.p;
  }
  A.n_tables = static_cast<uint32_t>(max_frames);
  if (int rc = launch_stage1(d, a->s1, a->plan, a->d_plan.p, a->d_frames.p, a->shape(), a->d_err.p, a->d_frame_err.p, true)) return rc;
  CUDA_TRY(cudaStreamSynchronize(d->stream));  // the uploads read host objects of this function
  d->async = std::move(a);
  return CLDN_OK;
}

// Enqueues only. The launches and their grids are those of the prepared shape, whatever the frames (header kernel,
// stage 2 + link kernel when compressed, the stage-1 launches of the prepared route, status kernel).
static int decode_blobs_async_impl(cldn_decoder* d, size_t n, const void* d_frames, int32_t* d_status, uint64_t* d_decoded) {
  if (!d) { set_error("null decoder"); return CLDN_ERR_INVALID_ARGUMENT; }
  AsyncBlobs* a = d->async.get();
  if (!a) { set_error("no prepared layout: call cldn_b200_decoder_prepare_blobs first"); return CLDN_ERR_INVALID_ARGUMENT; }
  if (n > a->max_frames) { set_error("%zu frames: the layout was prepared for at most %zu", n, a->max_frames); return CLDN_ERR_INVALID_ARGUMENT; }
  if (n == 0) return CLDN_OK;
  if (!d_frames || !d_status) { set_error("null argument"); return CLDN_ERR_INVALID_ARGUMENT; }
  CUDA_TRY(cudaSetDevice(d->device));
  AsyncLaunch A = a->A;
  A.desc = static_cast<const BlobDesc*>(d_frames);
  A.n_frames = static_cast<uint32_t>(n);
  A.status = d_status;
  A.decoded = d_decoded;
  CUDA_TRY(cudaMemsetAsync(a->d_frame_err.p, 0, a->max_frames * sizeof(uint32_t), d->stream));
  launch_blobs_async_headers(A, d->stream);
  if (A.compression != CLDN_COMP_NONE) {
    if (int rc = launch_stage2(d->stream, A.compression == CLDN_COMP_ZSTD, a->Z, a->body_cap, a->d_zs_lit, false)) return rc;
    launch_blobs_async_link(A, d->stream);
  }
  if (int rc = launch_stage1(d, a->s1, a->plan, a->d_plan.p, a->d_frames.p, a->shape(), a->d_err.p, a->d_frame_err.p, false)) return rc;
  launch_blobs_async_status(A, d->stream);
  CUDA_TRY(cudaGetLastError());
  return CLDN_OK;
}

extern "C" {

int cldn_b200_decode_batch(cldn_decoder_t* d, const cldn_info_t* info, size_t n_frames, const void* const* payloads,
                           const size_t* payload_bytes, void* const* outs, const size_t* out_capacities, int mem, int sync) {
  return guarded([&] { return decode_batch_impl(d, info, n_frames, payloads, payload_bytes, outs, out_capacities, mem, sync); });
}

int cldn_b200_decode_blobs(cldn_decoder_t* dec, size_t n_frames, const void* const* blobs, const size_t* blob_bytes,
                           void* const* outs, const size_t* out_capacities, int mem, int32_t* status, size_t* decoded_bytes) {
  return guarded([&] { return decode_blobs_impl(dec, n_frames, blobs, blob_bytes, outs, out_capacities, mem, status, decoded_bytes); });
}

int cldn_b200_decoder_prepare_blobs(cldn_decoder_t* dec, const cldn_info_t* layout, size_t max_frames, uint64_t max_points_per_frame) {
  return guarded([&] { return prepare_blobs_impl(dec, layout, max_frames, max_points_per_frame); });
}

int cldn_b200_decode_blobs_async(cldn_decoder_t* dec, size_t n_frames, const void* d_frames, int32_t* d_status, uint64_t* d_decoded_bytes) {
  return guarded([&] { return decode_blobs_async_impl(dec, n_frames, d_frames, d_status, d_decoded_bytes); });
}

const char* cldn_b200_decoder_frame_error(const cldn_decoder_t* dec, size_t f) {
  return dec && f < dec->frame_errors.size() ? dec->frame_errors[f].c_str() : "";
}

int cldn_b200_decoder_frame_info(const cldn_decoder_t* dec, size_t f, cldn_info_t* info) {
  if (!dec || !info) { set_error("null argument"); return CLDN_ERR_INVALID_ARGUMENT; }
  if (f >= dec->frame_infos.size()) { set_error("frame %zu: the last cldn_b200_decode_blobs had %zu frames", f, dec->frame_infos.size()); return CLDN_ERR_INVALID_ARGUMENT; }
  *info = dec->frame_infos[f];
  return CLDN_OK;
}

int cldn_b200_decode(cldn_decoder_t* dec, const cldn_info_t* info, const void* payload, size_t payload_bytes, void* out,
                     size_t out_capacity, int mem) {
  const void* payloads[1] = {payload};
  void* outs[1] = {out};
  return cldn_b200_decode_batch(dec, info, 1, payloads, &payload_bytes, outs, &out_capacity, mem, 1);
}

// ---- one-shot helpers shaped like the reference's WASM C ABI ------------------------------------------------------
uint32_t cldn_b200_EncodePointcloudData(const char* header_as_yaml, const void* pc_data, uint32_t pc_data_size,
                                        void* output_data, uint32_t output_capacity) {
  if (!header_as_yaml || !output_data) { set_error("null argument"); return 0; }
  cldn_info_t info;
  if (info_from_yaml(header_as_yaml, strlen(header_as_yaml), &info) != CLDN_OK) return 0;
  const uint64_t expected = static_cast<uint64_t>(info.width) * info.height * info.point_step;
  if (pc_data_size != expected) {  // wasm_functions.cpp:222-228
    set_error("Data size mismatch: expected %llu but got %u", static_cast<unsigned long long>(expected), pc_data_size);
    return 0;
  }
  cldn_encoder_t* enc = nullptr;
  if (cldn_b200_encoder_create(&info, -1, nullptr, &enc) != CLDN_OK) return 0;
  bool ok;
  const size_t cap = max_compressed_size(info, pc_data_size / info.point_step, true, &ok);
  std::vector<uint8_t> tmp(ok ? cap : 0);
  size_t written = 0;
  int rc = ok ? cldn_b200_encode(enc, pc_data, pc_data_size, tmp.data(), tmp.size(), 1, &written, CLDN_MEM_HOST) : CLDN_ERR_INVALID_ARGUMENT;
  cldn_b200_encoder_destroy(enc);
  if (rc != CLDN_OK) return 0;
  if (written > output_capacity) { set_error("Output buffer too small for encoded data. Need %zu bytes, got %u", written, output_capacity); return 0; }
  memcpy(output_data, tmp.data(), written);
  return static_cast<uint32_t>(written);
}

uint32_t cldn_b200_DecodeCompressedData(const void* encoded_data, uint32_t encoded_data_size, void* output_data,
                                        uint32_t output_capacity) {
  if (!encoded_data || !output_data) { set_error("null argument"); return 0; }
  cldn_info_t info;
  size_t hdr = 0;
  if (cldn_b200_decode_header(static_cast<const uint8_t*>(encoded_data), encoded_data_size, &info, &hdr) != CLDN_OK) return 0;
  const uint64_t decoded = static_cast<uint64_t>(info.width) * info.height * info.point_step;
  if (decoded > output_capacity) { set_error("output buffer too small"); return 0; }
  cldn_decoder_t* dec = nullptr;
  if (cldn_b200_decoder_create(-1, nullptr, &dec) != CLDN_OK) return 0;
  const int rc = cldn_b200_decode(dec, &info, static_cast<const uint8_t*>(encoded_data) + hdr, encoded_data_size - hdr,
                                  output_data, output_capacity, CLDN_MEM_HOST);
  cldn_b200_decoder_destroy(dec);
  return rc == CLDN_OK ? static_cast<uint32_t>(decoded) : 0;
}

}  // extern "C"

// =====================================================================================================================
// cldn_b200_encode_mixed_blobs: frames of any layouts through one handle, whose stream and scratch every layout shares.
// The layouts of the last kMixedLayouts calls' frames are kept (plan, header, device plan), at least those of the call
// in progress.
constexpr size_t kMixedLayouts = 16;

struct cldn_mixed_encoder : EncScratch {
  struct Cached {
    std::unique_ptr<EncLayout> layout;
    uint64_t used = 0;  // the last call with a frame of this layout
  };
  std::vector<Cached> layouts;
  uint64_t calls = 0;
  DevBuf<uint64_t> d_blob_sizes;  // blob sizes of the last CLDN_MEM_DEVICE call, one per frame (0: not encoded)
  std::vector<std::string> frame_errors;
};

// The layout of `info`, planned (cldn_b200_encoder_create's refusals) and uploaded the first time it is met.
static int mixed_layout(cldn_mixed_encoder* m, const cldn_info_t& info, EncLayout** out) {
  for (auto& c : m->layouts) {
    if (same_layout(c.layout->blob_info, info)) {
      c.used = m->calls;
      *out = c.layout.get();
      return CLDN_OK;
    }
  }
  std::unique_ptr<EncLayout> l(new EncLayout());
  if (int rc = plan_layout(info, *l)) return rc;
  l->info.width = l->info.height = l->blob_info.width = l->blob_info.height = 0;  // every frame's header states its own
  l->header = make_header(l->blob_info);
  if (int rc = upload_layout(*l)) return rc;
  *out = l.get();
  m->layouts.push_back({std::move(l), m->calls});
  return CLDN_OK;
}

// Drops the least recently used layouts beyond kMixedLayouts; an earlier asynchronous call may still read their plans.
static int trim_layouts(cldn_mixed_encoder* m) {
  if (m->layouts.size() <= kMixedLayouts) return CLDN_OK;
  CUDA_TRY(cudaStreamSynchronize(m->stream));
  std::sort(m->layouts.begin(), m->layouts.end(), [](const auto& a, const auto& b) { return a.used > b.used; });
  m->layouts.resize(kMixedLayouts);
  return CLDN_OK;
}

// Every frame gets the status cldn_b200_encoder_create(&infos[f]) + cldn_b200_encode_blobs give it alone: each is checked
// on the host with its own layout, and the good frames go through the fused batch path of their layout and route, one
// group after the other. Device blobs: the groups are enqueued back to back, one launch places every header and writes
// every blob size, and the sizes are read back once (not at all without `written`). Host blobs: each group returns
// complete, headers copied on the host. A group that fails on the device (which the worst-case capacities rule out) is
// encoded again frame by frame, so that only the guilty frame gets the status.
static int encode_mixed_impl(cldn_mixed_encoder* m, size_t n, const cldn_info_t* infos, const void* const* clouds,
                             const size_t* cloud_bytes, void* const* outs, const size_t* caps, int mem, int32_t* status,
                             size_t* written) {
  if (!m || (n && !status)) { set_error("null argument"); return CLDN_ERR_INVALID_ARGUMENT; }
  m->frame_errors.assign(n, "frame not encoded");
  for (size_t f = 0; f < n; ++f) {
    status[f] = CLDN_ERR_INTERNAL;
    if (written) written[f] = 0;
  }
  auto result = [&]() -> int {
    for (size_t f = 0; f < n; ++f) {
      if (status[f] != CLDN_OK) { set_error("frame %zu: %s", f, m->frame_errors[f].c_str()); return status[f]; }
    }
    return CLDN_OK;
  };
  auto fail = [&](size_t f, int rc) {
    status[f] = rc;
    m->frame_errors[f] = cldn_b200_last_error();
  };
  auto fail_all = [&](int rc) {
    for (size_t f = 0; f < n; ++f) fail(f, rc);
    return result();
  };
  if (n == 0) return CLDN_OK;
  if (!infos || !clouds || !cloud_bytes || !outs || !caps) { set_error("null argument"); return fail_all(CLDN_ERR_INVALID_ARGUMENT); }
  if (cudaSetDevice(m->device) != cudaSuccess) { set_error("cudaSetDevice failed"); return fail_all(CLDN_ERR_CUDA); }
  ++m->calls;
  if (int rc = trim_layouts(m)) return fail_all(rc);

  std::vector<EncLayout*> layout(n, nullptr);
  std::vector<EncodeRoute> route(n);
  std::vector<uint8_t> headers;  // frame f's header: headers[at[f], at[f + 1])
  std::vector<uint64_t> at(n + 1, 0);
  std::vector<void*> payload(n);
  std::vector<size_t> payload_cap(n);
  std::vector<std::vector<size_t>> groups;  // good frames of one layout and route, in call order
  for (size_t f = 0; f < n; ++f) {
    at[f + 1] = at[f];
    int rc = mixed_layout(m, infos[f], &layout[f]);
    if (!rc) rc = choose_encode_route(*layout[f], *m, mem, &route[f]);
    if (rc) { fail(f, rc); continue; }
    cldn_info_t fi = layout[f]->blob_info;
    const size_t pts = fi.point_step ? cloud_bytes[f] / fi.point_step : 0;
    fi.width = infos[f].width;
    fi.height = infos[f].height;
    if (fi.width == 0 && fi.height == 0) { fi.width = static_cast<uint32_t>(pts); fi.height = 1; }
    const std::vector<uint8_t> h = make_header(fi);
    rc = check_encode_frame(*layout[f], h.size(), clouds[f], cloud_bytes[f], outs[f], caps[f]);
    if (!rc && static_cast<uint64_t>(fi.width) * fi.height != pts) {
      set_error("width * height (%u x %u) differs from the %zu points of the cloud", fi.width, fi.height, pts);
      rc = CLDN_ERR_INVALID_ARGUMENT;
    }
    if (rc) { fail(f, rc); continue; }
    headers.insert(headers.end(), h.begin(), h.end());
    at[f + 1] = headers.size();
    payload[f] = static_cast<uint8_t*>(outs[f]) + h.size();
    payload_cap[f] = caps[f] - h.size();
    auto g = std::find_if(groups.begin(), groups.end(), [&](const std::vector<size_t>& G) {
      return layout[G[0]] == layout[f] && route[G[0]] == route[f];
    });
    if (g == groups.end()) groups.push_back({f});
    else g->push_back(f);
  }
  // the arrays of one group's frames
  std::vector<const void*> g_clouds;
  std::vector<size_t> g_bytes, g_caps, g_written;
  std::vector<void*> g_payload;
  auto gather = [&](const std::vector<size_t>& G) {
    g_clouds.clear(); g_bytes.clear(); g_caps.clear(); g_payload.clear();
    for (size_t f : G) {
      g_clouds.push_back(clouds[f]);
      g_bytes.push_back(cloud_bytes[f]);
      g_payload.push_back(payload[f]);
      g_caps.push_back(payload_cap[f]);
    }
    g_written.assign(G.size(), 0);
  };

  if (mem != CLDN_MEM_DEVICE) {
    auto run = [&](const std::vector<size_t>& G) -> int {
      gather(G);
      const size_t f0 = G[0];
      if (int rc = encode_frames(*layout[f0], *m, route[f0], mem, G.size(), g_clouds.data(), g_bytes.data(), g_payload.data(),
                                 g_caps.data(), 0, g_written.data())) return rc;
      for (size_t i = 0; i < G.size(); ++i) {
        const size_t f = G[i];
        memcpy(outs[f], headers.data() + at[f], at[f + 1] - at[f]);
        if (written) written[f] = (at[f + 1] - at[f]) + g_written[i];
        status[f] = CLDN_OK;
        m->frame_errors[f].clear();
      }
      return CLDN_OK;
    };
    for (const auto& G : groups) {
      if (run(G) == CLDN_OK) continue;
      for (size_t f : G) {
        if (int rc = run(std::vector<size_t>(1, f))) fail(f, rc);
      }
    }
    return result();
  }

  // device blobs: d_sizes holds the payload sizes group after group, d_blob_sizes the blob sizes frame by frame
  size_t good = 0;
  for (const auto& G : groups) good += G.size();
  if (int rc = m->d_sizes.reserve(good)) return fail_all(rc);
  if (int rc = m->d_blob_sizes.reserve(n)) return fail_all(rc);
  if (int rc = m->h_sizes.reserve(n)) return fail_all(rc);
  if (cudaMemsetAsync(m->d_blob_sizes.p, 0, n * sizeof(uint64_t), m->stream) != cudaSuccess) {
    set_error("cudaMemsetAsync failed");
    return fail_all(CLDN_ERR_CUDA);
  }
  auto enqueue = [&](const std::vector<std::vector<size_t>>& gs) -> int {
    std::vector<size_t> placed;
    std::vector<uint32_t> slots;
    for (const auto& G : gs) {
      gather(G);
      const size_t f0 = G[0];
      m->sizes_at = slots.size();
      const int rc = encode_frames(*layout[f0], *m, route[f0], mem, G.size(), g_clouds.data(), g_bytes.data(), g_payload.data(),
                                   g_caps.data(), 0, nullptr);
      m->sizes_at = 0;
      if (rc) return rc;
      for (size_t f : G) {
        placed.push_back(f);
        slots.push_back(static_cast<uint32_t>(slots.size()));
      }
    }
    const size_t np = placed.size();
    for (size_t f : placed) slots.push_back(static_cast<uint32_t>(f));
    // [np blob addresses][np + 1 header offsets][packed headers][pad][2 np slots]
    size_t hbytes = 0;
    for (size_t f : placed) hbytes += at[f + 1] - at[f];
    const size_t slots_at = ((2 * np + 1) * sizeof(uint64_t) + hbytes + 7) & ~size_t(7);
    const size_t tab_bytes = slots_at + slots.size() * sizeof(uint32_t);
    uint8_t* ht = nullptr;
    int slot = 0;
    if (int rc = m->h_blob_headers.acquire(tab_bytes, &ht, &slot)) return rc;
    if (int rc = m->d_blob_headers.reserve(tab_bytes)) return rc;
    uint64_t* tab = reinterpret_cast<uint64_t*>(ht);
    uint8_t* packed = ht + (2 * np + 1) * sizeof(uint64_t);
    tab[np] = 0;
    for (size_t i = 0; i < np; ++i) {
      const size_t f = placed[i], hb = at[f + 1] - at[f];
      tab[i] = reinterpret_cast<uintptr_t>(outs[f]);
      memcpy(packed + tab[np + i], headers.data() + at[f], hb);
      tab[np + i + 1] = tab[np + i] + hb;
    }
    memcpy(ht + slots_at, slots.data(), slots.size() * sizeof(uint32_t));
    CUDA_TRY(cudaMemcpyAsync(m->d_blob_headers.p, ht, tab_bytes, cudaMemcpyHostToDevice, m->stream));
    if (int rc = m->h_blob_headers.commit(slot, m->stream)) return rc;
    if (launch_place_headers(reinterpret_cast<const uint64_t*>(m->d_blob_headers.p), static_cast<uint32_t>(np), m->d_blob_sizes.p,
                             m->stream, m->d_sizes.p, reinterpret_cast<const uint32_t*>(m->d_blob_headers.p + slots_at)) < 0) {
      set_error("header launch failed");
      return CLDN_ERR_CUDA;
    }
    CUDA_TRY(cudaGetLastError());
    return CLDN_OK;
  };
  auto read_back = [&]() -> int {
    CUDA_TRY(cudaMemcpyAsync(m->h_sizes.p, m->d_blob_sizes.p, n * sizeof(uint64_t), cudaMemcpyDeviceToHost, m->stream));
    return check_device_error(m->stream, m->d_err.p, m->h_err.p);
  };
  auto done = [&](size_t f) {
    status[f] = CLDN_OK;
    m->frame_errors[f].clear();
    if (written) written[f] = static_cast<size_t>(m->h_sizes.p[f]);
  };
  int rc = enqueue(groups);
  if (rc == CLDN_OK && written) rc = read_back();
  if (rc == CLDN_OK) {
    for (const auto& G : groups) {
      for (size_t f : G) done(f);
    }
    return result();
  }
  for (const auto& G : groups) {
    for (size_t f : G) {
      int rf = enqueue(std::vector<std::vector<size_t>>(1, std::vector<size_t>(1, f)));
      if (!rf) rf = read_back();
      if (rf) fail(f, rf);
      else done(f);
    }
  }
  return result();
}

extern "C" {

int cldn_b200_mixed_encoder_create(int device, void* stream, cldn_mixed_encoder_t** out) {
  if (!out) { set_error("null argument"); return CLDN_ERR_INVALID_ARGUMENT; }
  *out = nullptr;
  if (int rc = select_device(device)) return rc;
  cldn_mixed_encoder* m = new cldn_mixed_encoder();
  cudaGetDevice(&m->device);
  if (stream) {
    m->stream = static_cast<cudaStream_t>(stream);
  } else {
    if (cudaStreamCreateWithFlags(&m->stream, cudaStreamNonBlocking) != cudaSuccess) {
      set_error("cudaStreamCreate failed");
      delete m;
      return CLDN_ERR_CUDA;
    }
    m->own_stream = true;
  }
  int rc = m->d_err.reserve(1, true);
  if (!rc) rc = m->h_err.reserve(1);
  if (rc) { cldn_b200_mixed_encoder_destroy(m); return rc; }
  *out = m;
  return CLDN_OK;
}

void cldn_b200_mixed_encoder_destroy(cldn_mixed_encoder_t* m) {
  if (!m) return;
  cudaSetDevice(m->device);
  if (m->stream) cudaStreamSynchronize(m->stream);
  const cudaStream_t own = m->own_stream ? m->stream : nullptr;
  delete m;  // the buffers and the layouts free themselves
  if (own) cudaStreamDestroy(own);
}

int cldn_b200_mixed_encoder_set_stage2_on_device(cldn_mixed_encoder_t* m, int on) {
  if (!m) { set_error("null encoder"); return CLDN_ERR_INVALID_ARGUMENT; }
  if (on != 0 && on != 1) { set_error("on must be 0 or 1"); return CLDN_ERR_INVALID_ARGUMENT; }
  m->stage2_on_device = on == 1;
  return CLDN_OK;
}

int cldn_b200_encode_mixed_blobs(cldn_mixed_encoder_t* m, size_t n_frames, const cldn_info_t* infos, const void* const* clouds,
                                 const size_t* cloud_bytes, void* const* outs, const size_t* out_capacities, int mem,
                                 int32_t* status, size_t* written) {
  return guarded([&] { return encode_mixed_impl(m, n_frames, infos, clouds, cloud_bytes, outs, out_capacities, mem, status, written); });
}

const char* cldn_b200_mixed_encoder_frame_error(const cldn_mixed_encoder_t* m, size_t f) {
  return m && f < m->frame_errors.size() ? m->frame_errors[f].c_str() : "";
}

const uint64_t* cldn_b200_mixed_encoder_sizes_device(const cldn_mixed_encoder_t* m) { return m ? m->d_blob_sizes.p : nullptr; }

size_t cldn_b200_mixed_encoder_cached_layouts(const cldn_mixed_encoder_t* m) { return m ? m->layouts.size() : 0; }

int cldn_b200_mixed_encoder_sync(cldn_mixed_encoder_t* m) {
  if (!m) { set_error("null encoder"); return CLDN_ERR_INVALID_ARGUMENT; }
  CUDA_TRY(cudaSetDevice(m->device));
  return check_device_error(m->stream, m->d_err.p, m->h_err.p);
}

}  // extern "C"
