// TEST INFRASTRUCTURE ONLY — ThreadSanitizer driver for cldn_b200_viz_lossy_preprocess_batch_async
// (tests/test_gpu_viz_async.py). One prepared shape of viz XYZI clouds with two frame slots more than the call uses, so
// that empty frame slots run through every kernel; frames of partial last tiles (2049, 4097 points), an empty one, an
// all-duplicate one, and three refused ones (NULL cloud, one byte short, more points than prepared). Every CUDA thread is
// a TSAN fiber; statuses, counts, survivors and encode descriptors are checked against cldn_b200_viz_lossy_preprocess of
// each frame (the oracle comparisons live in the pytest file).
#include <cmath>
#include <cstdio>
#include <cstring>
#include <vector>

#include <cuda_runtime.h>  // the cusim shim (this file is only ever compiled against it)

#include "cloudini_b200_ros.h"

static uint32_t rng_state = 7331;
static uint32_t rnd() { rng_state = rng_state * 1664525u + 1013904223u; return rng_state >> 8; }

int main() {
  cldn_info_t info;
  cldn_b200_info_init(&info);
  info.width = 0; info.height = 1; info.point_step = 16; info.compression_opt = CLDN_COMP_NONE;
  const char* names[4] = {"x", "y", "z", "intensity"};
  for (int k = 0; k < 4; ++k) {
    cldn_field_t& f = info.fields[info.n_fields++];
    memset(&f, 0, sizeof(f));
    strncpy(f.name, names[k], CLDN_MAX_NAME - 1);
    f.offset = 4 * k; f.type = CLDN_FLOAT32; f.has_resolution = 1; f.resolution = k < 3 ? 0.01f : 0.1f;
  }
  const uint32_t max_points = 5000;
  const uint32_t sizes[] = {4097, 0, 2049, 300, 1, 700, 800, max_points + 1};
  const size_t n = sizeof(sizes) / sizeof(sizes[0]);
  cldn_preproc_t* pp = nullptr;
  if (cldn_b200_preproc_create(-1, nullptr, &pp) || cldn_b200_preproc_prepare_batch(pp, &info, n + 2, max_points, nullptr)) {
    printf("create failed: %s\n", cldn_b200_last_error());
    return 1;
  }
  std::vector<std::vector<float>> clouds(n);
  std::vector<std::vector<uint8_t>> outs(n);
  std::vector<cldn_viz_desc_t> desc(n);
  for (size_t f = 0; f < n; ++f) {
    clouds[f].resize(4 * static_cast<size_t>(sizes[f]) + 4);
    for (size_t i = 0; i < sizes[f]; ++i) {
      float* p = &clouds[f][4 * i];
      if (f == 3) { p[0] = 1.0f; p[1] = 2.0f; p[2] = 3.0f; }  // one voxel
      else if (i % 5 == 1) { p[0] = p[-4]; p[1] = p[-3]; p[2] = p[-2]; }  // the previous point's voxel
      else for (int k = 0; k < 3; ++k) p[k] = (static_cast<int>(rnd() % 2001) - 1000) * 0.01f;
      if (i % 37 == 3) p[1] = NAN;
      p[3] = static_cast<float>(i);
    }
    outs[f].assign(16 * static_cast<size_t>(sizes[f]) + 8, 0x5A);
    desc[f] = {clouds[f].data(), 16ull * sizes[f], outs[f].data(), 16ull * sizes[f]};
  }
  desc[5].cloud = nullptr;   // NULL cloud with bytes
  desc[6].capacity -= 1;     // one byte short
  std::vector<int32_t> status(n, 99), applied(n, 55);
  std::vector<uint64_t> kept(n, 7);
  std::vector<cldn_cloud_desc_t> enc(n);
  if (cldn_b200_viz_lossy_preprocess_batch_async(pp, n, desc.data(), status.data(), kept.data(), applied.data(), enc.data()) ||
      cldn_b200_preproc_sync(pp)) {
    printf("call failed: %s\n", cldn_b200_last_error());
    return 1;
  }
  int bad = 0;
  for (size_t f = 0; f < n; ++f) {
    std::vector<uint8_t> alone(outs[f].size(), 0x5A);
    cldn_info_t fi = info;
    size_t k1 = 0;
    int a1 = 0;
    int rc = cldn_b200_viz_lossy_preprocess(pp, &fi, desc[f].cloud, desc[f].cloud_bytes, alone.data(), desc[f].capacity, &k1, &a1,
                                            CLDN_MEM_DEVICE);
    if (f == 5) { k1 = sizes[f]; a1 = 0; }  // the single call refuses a NULL cloud before it sets them
    if (f == 7) {  // more points than prepared: refused, output untouched
      rc = CLDN_ERR_UNSUPPORTED; k1 = sizes[f]; a1 = 0;
      alone.assign(alone.size(), 0x5A);
    }
    const bool same = status[f] == rc && kept[f] == k1 && applied[f] == a1 && alone == outs[f];
    const bool enc_ok = rc ? (enc[f].cloud == nullptr && enc[f].cloud_bytes == 1)
                           : (enc[f].cloud == (a1 ? desc[f].out : desc[f].cloud) && enc[f].cloud_bytes == (a1 ? 16ull * k1 : desc[f].cloud_bytes));
    printf("frame %zu: status %d kept %llu applied %d (single call %d %zu %d)%s\n", f, status[f],
           static_cast<unsigned long long>(kept[f]), applied[f], rc, k1, a1, same && enc_ok ? "" : " MISMATCH");
    bad += !(same && enc_ok);
  }
  cldn_b200_preproc_destroy(pp);
  if (bad) return 1;
  puts("viz_async_racecheck: done");
  return 0;
}
