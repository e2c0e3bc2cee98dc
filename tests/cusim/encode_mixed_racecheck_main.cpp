// TEST INFRASTRUCTURE ONLY — ThreadSanitizer driver for cldn_b200_encode_mixed_blobs (tests/test_gpu_encode_mixed.py).
// One device-blob batch and one host-blob batch through one handle, three layouts interleaved (XYZI step 16, XYZ step
// 12, XYZI with LZ4) over mixed sizes (empty, one point, several chunks). Every CUDA thread is a TSAN fiber; the blobs
// are checked against single-layout handles (the comparisons with the reference live in the pytest file).
#include <cstdio>
#include <cstring>
#include <vector>

#include <cuda_runtime.h>  // the cusim shim (this file is only ever compiled against it)

#include "cloudini_b200.h"

static uint32_t rng_state = 777;
static uint32_t rnd() { rng_state = rng_state * 1664525u + 1013904223u; return rng_state >> 8; }

static cldn_info_t layout(int k) {
  cldn_info_t info;
  cldn_b200_info_init(&info);
  const int fields = k == 1 ? 3 : 4;
  info.point_step = 4 * fields;
  info.compression_opt = k == 2 ? CLDN_COMP_LZ4 : CLDN_COMP_NONE;
  info.width = info.height = 0;
  const char* names[4] = {"x", "y", "z", "intensity"};
  for (int i = 0; i < fields; ++i) {
    cldn_field_t& f = info.fields[info.n_fields++];
    memset(&f, 0, sizeof(f));
    strncpy(f.name, names[i], CLDN_MAX_NAME - 1);
    f.offset = 4 * i; f.type = CLDN_FLOAT32; f.has_resolution = 1; f.resolution = 0.01f;
  }
  return info;
}

int main() {
  const uint32_t sizes[] = {40000, 0, 1, 9000, 33000, 5};
  const size_t n = sizeof(sizes) / sizeof(sizes[0]);
  std::vector<cldn_info_t> infos(n);
  std::vector<std::vector<float>> clouds(n);
  std::vector<const void*> in(n);
  std::vector<size_t> in_b(n), caps(n), written(n), alone_w(n);
  std::vector<std::vector<uint8_t>> blobs(n), alone(n);
  std::vector<void*> out(n), alone_out(n);
  std::vector<int32_t> status(n);
  for (size_t f = 0; f < n; ++f) {
    infos[f] = layout(static_cast<int>(f % 3));
    const size_t vals = infos[f].point_step / 4 * static_cast<size_t>(sizes[f]);
    clouds[f].resize(vals + 1);
    float w = 0;
    for (size_t i = 0; i < vals; ++i) { w += (static_cast<int>(rnd() % 2001) - 1000) * 1e-4f; clouds[f][i] = w; }
    in[f] = clouds[f].data();
    in_b[f] = 4 * vals;
    caps[f] = cldn_b200_max_compressed_size(&infos[f], sizes[f], 0) + 4096;
    blobs[f].assign(caps[f], 0);
    alone[f].assign(caps[f], 0);
    out[f] = blobs[f].data();
    alone_out[f] = alone[f].data();
  }
  cldn_mixed_encoder_t* m = nullptr;
  if (cldn_b200_mixed_encoder_create(-1, nullptr, &m)) { printf("create failed: %s\n", cldn_b200_last_error()); return 1; }
  int bad = 0;
  for (int mem : {CLDN_MEM_DEVICE, CLDN_MEM_HOST}) {
    if (cldn_b200_encode_mixed_blobs(m, n, infos.data(), in.data(), in_b.data(), out.data(), caps.data(), mem, status.data(),
                                     written.data())) {
      printf("encode_mixed_blobs failed: %s\n", cldn_b200_last_error());
      return 1;
    }
    for (size_t f = 0; f < n; ++f) {
      cldn_encoder_t* enc = nullptr;
      if (cldn_b200_encoder_create(&infos[f], -1, nullptr, &enc) ||
          cldn_b200_encode_blobs(enc, 1, &in[f], &in_b[f], nullptr, nullptr, &alone_out[f], &caps[f], &alone_w[f], mem)) {
        printf("single-layout encode failed: %s\n", cldn_b200_last_error());
        return 1;
      }
      cldn_b200_encoder_destroy(enc);
      const bool same = written[f] == alone_w[f] && memcmp(blobs[f].data(), alone[f].data(), written[f]) == 0;
      printf("mem %d blob %zu: %zu bytes, status %d, equal to the single-layout blob %d\n", mem, f, written[f], status[f], same);
      // the device LZ4 coder's bytes follow the lane order, which the emulation may shuffle: its sizes are not compared
      bad += status[f] != 0 || (!same && !(mem == CLDN_MEM_DEVICE && infos[f].compression_opt == CLDN_COMP_LZ4));
    }
  }
  cldn_b200_mixed_encoder_destroy(m);
  if (bad) return 1;
  puts("encode_mixed_racecheck: done");
  return 0;
}
