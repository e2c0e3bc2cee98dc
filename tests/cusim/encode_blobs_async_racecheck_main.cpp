// TEST INFRASTRUCTURE ONLY — ThreadSanitizer driver for cldn_b200_encode_blobs_async (tests/test_gpu_encode_blobs_async.py).
// One prepared shape per compression (NONE, LZ4 and ZSTD on the device) of XYZI clouds, so that the persistent XYZI
// kernel draws tickets for real and empty tile slots: a call with fewer frames than prepared, frames of 0 .. 33000
// points, a frame that is not a whole number of points and one with more points than prepared. Every CUDA thread is a
// TSAN fiber; statuses and sizes are checked against cldn_b200_encode_blobs of each frame (the byte-exact comparisons
// live in the pytest file).
#include <cstdio>
#include <cstring>
#include <vector>

#include <cuda_runtime.h>  // the cusim shim (this file is only ever compiled against it)

#include "cloudini_b200.h"

static uint32_t rng_state = 4243;
static uint32_t rnd() { rng_state = rng_state * 1664525u + 1013904223u; return rng_state >> 8; }

static cldn_info_t xyzi(uint8_t compression) {
  cldn_info_t info;
  cldn_b200_info_init(&info);
  info.width = 0; info.height = 1; info.point_step = 16; info.compression_opt = compression;
  const char* names[4] = {"x", "y", "z", "intensity"};
  for (int k = 0; k < 4; ++k) {
    cldn_field_t& f = info.fields[info.n_fields++];
    memset(&f, 0, sizeof(f));
    strncpy(f.name, names[k], CLDN_MAX_NAME - 1);
    f.offset = 4 * k; f.type = 7; f.has_resolution = 1; f.resolution = 0.001f;
  }
  return info;
}

int main() {
  int bad = 0;
  const uint32_t max_points = 34000;
  for (uint8_t comp = 0; comp <= 2; ++comp) {
    const uint32_t sizes[] = {33000, 0, 2048, 5000, max_points + 1};
    const size_t n = sizeof(sizes) / sizeof(sizes[0]);
    cldn_info_t info = xyzi(comp);
    cldn_encoder_t* enc = nullptr;
    if (cldn_b200_encoder_create(&info, -1, nullptr, &enc) || (comp == 2 && cldn_b200_encoder_set_stage2_on_device(enc, 1))) {
      printf("create failed: %s\n", cldn_b200_last_error());
      return 1;
    }
    std::vector<std::vector<float>> clouds(n);
    std::vector<std::vector<uint8_t>> outs(n);
    std::vector<cldn_cloud_desc_t> desc(n);
    for (size_t f = 0; f < n; ++f) {
      clouds[f].resize(4 * static_cast<size_t>(sizes[f]) + 4);
      float w = 0;
      for (auto& v : clouds[f]) { w += (static_cast<int>(rnd() % 2001) - 1000) * 1e-5f; v = w; }
      cldn_info_t fi = info;
      fi.width = sizes[f];
      outs[f].assign(cldn_b200_max_compressed_size(&fi, sizes[f], 1), 0);
      desc[f] = {clouds[f].data(), 16ull * sizes[f] + (f == 3 ? 1 : 0), outs[f].data(), outs[f].size(), 0, 0};
    }
    std::vector<int32_t> status(n, 99);
    std::vector<uint64_t> written(n, 7);
    if (cldn_b200_encoder_prepare_blobs(enc, n + 2, max_points) ||
        cldn_b200_encode_blobs_async(enc, n, desc.data(), status.data(), written.data()) || cldn_b200_encoder_sync(enc)) {
      printf("call failed: %s\n", cldn_b200_last_error());
      return 1;
    }
    for (size_t f = 0; f < n; ++f) {
      const int32_t want = f == 3 ? CLDN_ERR_INVALID_ARGUMENT : f == 4 ? CLDN_ERR_UNSUPPORTED : CLDN_OK;
      size_t ref = 0;
      if (want == CLDN_OK) {
        std::vector<uint8_t> alone(outs[f].size());
        void* out = alone.data();
        const void* cloud = clouds[f].data();
        const size_t bytes = desc[f].cloud_bytes, cap = alone.size();
        if (cldn_b200_encode_blobs(enc, 1, &cloud, &bytes, nullptr, nullptr, &out, &cap, &ref, CLDN_MEM_DEVICE)) ref = 0;
      }
      printf("compression %d frame %zu: status %d written %llu (encode_blobs %zu)\n", comp, f, status[f],
             static_cast<unsigned long long>(written[f]), ref);
      bad += status[f] != want || written[f] != ref;
    }
    cldn_b200_encoder_destroy(enc);
  }
  if (bad) return 1;
  puts("encode_blobs_async_racecheck: done");
  return 0;
}
