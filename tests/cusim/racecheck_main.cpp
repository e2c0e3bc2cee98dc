// TEST INFRASTRUCTURE ONLY — driver of the ThreadSanitizer ("racecheck") build of tests/cusim.
// Runs the hot path's kernels (FloatN encode / both FloatN decoders, generic kernels, V5 sections, Gorilla pre-pass,
// viz preprocessing) on synthetic clouds through the C ABI. Every CUDA thread is a TSAN fiber, so an unsynchronised
// access pair inside a CTA, or between CTAs, is reported by the runtime; the round trips are sanity-checked only (the
// byte-exact comparisons live in the pytest suites).
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include <cuda_runtime.h>  // the cusim shim (this file is only ever compiled against it)

#include "cloudini_b200_ros.h"

// ---- positive / negative control of the detector itself ------------------------------------------------------------------
// racy: thread t writes s_buf[t], its neighbour reads it with nothing in between; fixed: the same with a __syncthreads().
static unsigned g_sink[256];
static unsigned g_buf[256];  // stands for global memory; s_buf below for shared memory
static void control_kernel(bool with_barrier) {
  __shared__ unsigned s_buf[256];
  s_buf[threadIdx.x] = threadIdx.x * 3u;
  g_buf[threadIdx.x] = threadIdx.x * 5u;
  if (with_barrier) __syncthreads();
  g_sink[threadIdx.x] = s_buf[(threadIdx.x + 1) & 255u] + g_buf[(threadIdx.x + 1) & 255u];
}

static uint32_t rng_state = 12345;
static uint32_t rnd() { rng_state = rng_state * 1664525u + 1013904223u; return rng_state >> 8; }

static void add_field(cldn_info_t& info, const char* name, uint32_t offset, uint8_t type, float res) {
  cldn_field_t& f = info.fields[info.n_fields++];
  memset(&f, 0, sizeof(f));
  strncpy(f.name, name, CLDN_MAX_NAME - 1);
  f.offset = offset; f.type = type; f.has_resolution = res > 0 ? 1 : 0; f.resolution = res;
}

static int roundtrip(const char* label, cldn_info_t info, const std::vector<uint8_t>& cloud, const char* decode_mode) {
  if (decode_mode) setenv("CLDN_B200_DECODE_MODE", decode_mode, 1); else unsetenv("CLDN_B200_DECODE_MODE");
  cldn_encoder_t* enc = nullptr;
  cldn_decoder_t* dec = nullptr;
  if (cldn_b200_encoder_create(&info, -1, nullptr, &enc) || cldn_b200_decoder_create(-1, nullptr, &dec)) { printf("%s: create failed: %s\n", label, cldn_b200_last_error()); return 1; }
  const size_t n = cloud.size() / info.point_step;
  std::vector<uint8_t> blob(cldn_b200_max_compressed_size(&info, n, 1)), back(cloud.size(), 0);
  size_t written = 0, hdr = 0;
  int rc = cldn_b200_encode(enc, cloud.data(), cloud.size(), blob.data(), blob.size(), 1, &written, CLDN_MEM_HOST);
  cldn_info_t dinfo;
  if (!rc) rc = cldn_b200_decode_header(blob.data(), written, &dinfo, &hdr);
  if (!rc) rc = cldn_b200_decode(dec, &dinfo, blob.data() + hdr, written - hdr, back.data(), back.size(), CLDN_MEM_HOST);
  cldn_b200_encoder_destroy(enc);
  cldn_b200_decoder_destroy(dec);
  if (rc) { printf("%s: failed: %s\n", label, cldn_b200_last_error()); return 1; }
  // xyz within 1 mm
  double worst = 0;
  for (size_t i = 0; i < n; ++i) {
    float a[3], b[3];
    memcpy(a, cloud.data() + i * info.point_step, 12);
    memcpy(b, back.data() + i * info.point_step, 12);
    for (int k = 0; k < 3; ++k) {  // |v| * 1000 >= 2^31 saturates by design (cvtps2dq "integer indefinite"): not a round-trip value
      if (std::isfinite(a[k]) && std::fabs(a[k]) < 2.0e6f) worst = std::fmax(worst, std::fabs(double(a[k]) - double(b[k])));
    }
  }
  printf("%s: %zu points -> %zu bytes, max xyz error %.6f %s\n", label, n, written, worst, worst <= 0.00101 ? "ok" : "BAD");
  return worst <= 0.00101 ? 0 : 1;
}

// warp-level variant: the neighbour is read after a shuffle. With shuffles modelled as fences (default) this is ordered;
// under CUSIM_TSAN_STRICT=1 (only __syncwarp / __syncthreads order memory, as the CUDA model defines it) it is a race.
static void control_shfl_kernel() {
  __shared__ unsigned s_buf[32];
  s_buf[threadIdx.x] = threadIdx.x * 7u;
  const unsigned other = __shfl_sync(0xffffffffu, threadIdx.x, (threadIdx.x + 1) & 31);
  g_sink[threadIdx.x] = s_buf[other];
}

int main(int argc, char** argv) {
  if (argc > 1 && !strcmp(argv[1], "--control-shfl")) { cusim::launch(dim3(1), dim3(32), 0, [] { control_shfl_kernel(); }); puts("control: shuffle kernel ran"); return 0; }
  if (argc > 1 && !strcmp(argv[1], "--control-racy")) { cusim::launch(dim3(1), dim3(256), 0, [] { control_kernel(false); }); puts("control: racy kernel ran"); return 0; }
  if (argc > 1 && !strcmp(argv[1], "--control-fixed")) { cusim::launch(dim3(1), dim3(256), 0, [] { control_kernel(true); }); puts("control: fixed kernel ran"); return 0; }
  int bad = 0;
  const size_t n = 70000;  // three chunks: look-backs, chunk walk, partial last tile
  // ---- C2: XYZI step 16 (FloatN fast kernels; sequential and tile-parallel decoders) ----
  {
    cldn_info_t info; cldn_b200_info_init(&info);
    info.width = n; info.height = 1; info.point_step = 16; info.compression_opt = CLDN_COMP_NONE;
    add_field(info, "x", 0, CLDN_FLOAT32, 0.001f); add_field(info, "y", 4, CLDN_FLOAT32, 0.001f);
    add_field(info, "z", 8, CLDN_FLOAT32, 0.001f); add_field(info, "intensity", 12, CLDN_FLOAT32, 0.001f);
    std::vector<uint8_t> cloud(n * 16);
    for (size_t i = 0; i < n; ++i) {
      float p[4] = {20.f * std::sin(0.001f * i), 20.f * std::cos(0.001f * i), 0.01f * float(i % 64), float(rnd() % 256)};
      if (rnd() % 97 == 0) p[rnd() % 3] = NAN;
      if (rnd() % 4001 == 0) p[0] = -4.0e6f;  // 5-byte varint -> byte-wise tile path
      memcpy(&cloud[i * 16], p, 16);
    }
    bad += roundtrip("c2/seq", info, cloud, "seq");
    bad += roundtrip("c2/tile", info, cloud, "tile");
    {  // a batch of equally sized frames: frame-interleaved CTA order in the encoder, chunk-index-major claims in the decoder
      unsetenv("CLDN_B200_DECODE_MODE");
      const size_t F = 3, fn = 40000;
      cldn_info_t binfo = info; binfo.width = fn;
      cldn_encoder_t* enc = nullptr; cldn_decoder_t* dec = nullptr;
      cldn_b200_encoder_create(&binfo, -1, nullptr, &enc); cldn_b200_decoder_create(-1, nullptr, &dec);
      const size_t cap = cldn_b200_max_compressed_size(&binfo, fn, 1);
      std::vector<std::vector<uint8_t>> blobs(F, std::vector<uint8_t>(cap)), outs(F, std::vector<uint8_t>(fn * 16));
      const void* ins[F]; void* bl[F]; size_t in_b[F], caps[F], wr[F];
      for (size_t f = 0; f < F; ++f) { ins[f] = cloud.data() + f * 1000 * 16; bl[f] = blobs[f].data(); in_b[f] = fn * 16; caps[f] = cap; }
      int rc = cldn_b200_encode_batch(enc, F, ins, in_b, bl, caps, 1, wr, CLDN_MEM_HOST);
      const uint8_t* hdr_p; size_t hdr = 0; cldn_b200_encoder_header(enc, &hdr_p, &hdr);
      const void* pl[F]; void* ou[F]; size_t pl_b[F], ou_b[F];
      for (size_t f = 0; f < F; ++f) { pl[f] = blobs[f].data() + hdr; pl_b[f] = wr[f] - hdr; ou[f] = outs[f].data(); ou_b[f] = fn * 16; }
      if (!rc) rc = cldn_b200_decode_batch(dec, &binfo, F, pl, pl_b, ou, ou_b, CLDN_MEM_HOST, 1);
      printf("c2/batch of %zu frames: %s\n", F, rc ? cldn_b200_last_error() : "ok");
      bad += rc != 0;
      cldn_b200_encoder_destroy(enc); cldn_b200_decoder_destroy(dec);
    }
    // ---- N3 on the same cloud ----
    cldn_preproc_t* pp = nullptr;
    std::vector<uint8_t> kept(cloud.size());
    size_t n_kept = 0; int applied = 0;
    cldn_info_t vinfo = info;
    if (cldn_b200_preproc_create(-1, nullptr, &pp) ||
        cldn_b200_viz_lossy_preprocess(pp, &vinfo, cloud.data(), cloud.size(), kept.data(), kept.size(), &n_kept, &applied, CLDN_MEM_HOST)) {
      printf("viz: failed: %s\n", cldn_b200_last_error()); ++bad;
    } else {
      printf("viz: %zu -> %zu points (applied %d)\n", n, n_kept, applied);
    }
    cldn_b200_preproc_destroy(pp);
  }
  // ---- C3-like: XYZ + rgba u32 + ring u16, step 32 (V5 sections: palette + delta-rle) ----
  {
    cldn_info_t info; cldn_b200_info_init(&info);
    info.width = n; info.height = 1; info.point_step = 32; info.compression_opt = CLDN_COMP_NONE;
    add_field(info, "x", 0, CLDN_FLOAT32, 0.001f); add_field(info, "y", 4, CLDN_FLOAT32, 0.001f); add_field(info, "z", 8, CLDN_FLOAT32, 0.001f);
    add_field(info, "rgba", 16, CLDN_UINT32, 0); add_field(info, "ring", 20, CLDN_UINT16, 0);
    std::vector<uint8_t> cloud(n * 32, 0xCD);
    for (size_t i = 0; i < n; ++i) {
      float p[3] = {0.001f * i, 1.f + 0.002f * float(i % 97), -3.f};
      uint32_t rgba = 0xFF000000u | ((rnd() % 8) * 0x101010u);
      uint16_t ring = uint16_t(i % 64);
      memcpy(&cloud[i * 32], p, 12); memcpy(&cloud[i * 32 + 16], &rgba, 4); memcpy(&cloud[i * 32 + 20], &ring, 2);
    }
    bad += roundtrip("c3/v5", info, cloud, nullptr);
  }
  // ---- DDS-sample layout: XYZI + ring u16 + FLOAT64 timestamp, step 26 (generic kernels, Gorilla pre-pass, one-Gorilla decoder) ----
  {
    cldn_info_t info; cldn_b200_info_init(&info);
    info.width = n; info.height = 1; info.point_step = 26; info.compression_opt = CLDN_COMP_NONE;
    add_field(info, "x", 0, CLDN_FLOAT32, 0.001f); add_field(info, "y", 4, CLDN_FLOAT32, 0.001f);
    add_field(info, "z", 8, CLDN_FLOAT32, 0.001f); add_field(info, "intensity", 12, CLDN_FLOAT32, 0.001f);
    add_field(info, "ring", 16, CLDN_UINT16, 0); add_field(info, "timestamp", 18, CLDN_FLOAT64, 0);
    std::vector<uint8_t> cloud(n * 26);
    for (size_t i = 0; i < n; ++i) {
      float p[4] = {5.f * std::sin(0.002f * i), 5.f * std::cos(0.002f * i), 0.02f * float(i % 32), float(rnd() % 100)};
      uint16_t ring = uint16_t(i % 32);
      double ts = 1.7e9 + 1e-5 * double(i) + (rnd() % 50 == 0 ? 0.1 : 0.0);
      memcpy(&cloud[i * 26], p, 16); memcpy(&cloud[i * 26 + 16], &ring, 2); memcpy(&cloud[i * 26 + 18], &ts, 8);
    }
    bad += roundtrip("dds-layout/gorilla", info, cloud, nullptr);
  }
  // ---- Livox-like: XYZI + two uint8 (raw Copy bytes in the stream) + u32, step 22: pointer-jumping decoder ----
  {
    cldn_info_t info; cldn_b200_info_init(&info);
    info.width = n; info.height = 1; info.point_step = 22; info.compression_opt = CLDN_COMP_NONE;
    add_field(info, "x", 0, CLDN_FLOAT32, 0.001f); add_field(info, "y", 4, CLDN_FLOAT32, 0.001f);
    add_field(info, "z", 8, CLDN_FLOAT32, 0.001f); add_field(info, "intensity", 12, CLDN_FLOAT32, 0.01f);
    add_field(info, "tag", 16, CLDN_UINT8, 0); add_field(info, "line", 17, CLDN_UINT8, 0); add_field(info, "offset_time", 18, CLDN_UINT32, 0);
    std::vector<uint8_t> cloud(n * 22);
    for (size_t i = 0; i < n; ++i) {
      float p[4] = {5.f * std::sin(0.002f * i), 5.f * std::cos(0.002f * i), 0.02f * float(i % 32), float(rnd() % 100)};
      uint8_t tag = uint8_t(rnd()), line = uint8_t(rnd());
      uint32_t ot = uint32_t(i * 100);
      memcpy(&cloud[i * 22], p, 16); cloud[i * 22 + 16] = tag; cloud[i * 22 + 17] = line; memcpy(&cloud[i * 22 + 18], &ot, 4);
    }
    bad += roundtrip("livox-layout/raw bytes in the stream", info, cloud, nullptr);
  }
  printf("racecheck_main: %s\n", bad ? "FAILED" : "done");
  return bad ? 1 : 0;
}
