// TEST INFRASTRUCTURE ONLY — ThreadSanitizer driver for cldn_b200_viz_lossy_preprocess_batch and cldn_b200_encode_blobs
// (tests/test_gpu_encode_blobs.py). One viz batch over clouds of mixed sizes (empty, one point, several tiles), then one
// encode_blobs of the survivors, both with device pointers. Every CUDA thread is a TSAN fiber; the results are
// sanity-checked only (the byte-exact comparisons live in the pytest file).
#include <cmath>
#include <cstdio>
#include <cstring>
#include <vector>

#include <cuda_runtime.h>  // the cusim shim (this file is only ever compiled against it)

#include "cloudini_b200.h"
#include "cloudini_b200_ros.h"

static uint32_t rng_state = 4242;
static uint32_t rnd() { rng_state = rng_state * 1664525u + 1013904223u; return rng_state >> 8; }

int main() {
  cldn_info_t info;
  cldn_b200_info_init(&info);
  info.point_step = 16; info.compression_opt = CLDN_COMP_NONE;
  const char* names[4] = {"x", "y", "z", "intensity"};
  for (int k = 0; k < 4; ++k) {
    cldn_field_t& f = info.fields[info.n_fields++];
    memset(&f, 0, sizeof(f));
    strncpy(f.name, names[k], CLDN_MAX_NAME - 1);
    f.offset = 4 * k; f.type = CLDN_FLOAT32; f.has_resolution = 1; f.resolution = 0.01f;
  }
  const uint32_t sizes[] = {40000, 0, 1, 9000, 33000};
  const size_t n = sizeof(sizes) / sizeof(sizes[0]);
  std::vector<std::vector<float>> clouds(n);
  std::vector<std::vector<uint8_t>> mid(n), blobs(n);
  std::vector<const void*> in(n), mid_in(n);
  std::vector<void*> mid_out(n), out(n);
  std::vector<size_t> in_b(n), mid_cap(n), kept(n), caps(n), written(n);
  std::vector<int> applied(n);
  for (size_t f = 0; f < n; ++f) {
    clouds[f].resize(4 * static_cast<size_t>(sizes[f]) + 4);
    float w = 0;
    for (size_t i = 0; i < 4 * static_cast<size_t>(sizes[f]); ++i) {
      w += (static_cast<int>(rnd() % 2001) - 1000) * 1e-4f;
      clouds[f][i] = (rnd() % 50 == 0) ? NAN : w;   // NaNs are dropped, near repeats share voxels
    }
    in[f] = clouds[f].data();
    in_b[f] = 16 * static_cast<size_t>(sizes[f]);
    mid[f].assign(in_b[f] + 16, 0);
    mid_out[f] = mid[f].data();
    mid_cap[f] = in_b[f];
  }
  cldn_preproc_t* pp = nullptr;
  if (cldn_b200_preproc_create(-1, nullptr, &pp)) { printf("create failed: %s\n", cldn_b200_last_error()); return 1; }
  if (cldn_b200_viz_lossy_preprocess_batch(pp, &info, n, in.data(), in_b.data(), mid_out.data(), mid_cap.data(), kept.data(),
                                           applied.data(), nullptr, CLDN_MEM_DEVICE)) {
    printf("viz batch failed: %s\n", cldn_b200_last_error());
    return 1;
  }
  int bad = 0;
  for (size_t f = 0; f < n; ++f) {
    printf("viz frame %zu: %zu of %u points kept, applied %d\n", f, kept[f], sizes[f], applied[f]);
    bad += (applied[f] != (sizes[f] > 0)) || kept[f] > sizes[f] || (sizes[f] > 1000 && kept[f] == 0);
    mid_in[f] = mid[f].data();
    in_b[f] = 16 * kept[f];
    caps[f] = cldn_b200_max_compressed_size(&info, kept[f], 0) + 4096;
    blobs[f].assign(caps[f], 0);
    out[f] = blobs[f].data();
  }
  cldn_b200_preproc_destroy(pp);
  cldn_encoder_t* enc = nullptr;
  if (cldn_b200_encoder_create(&info, -1, nullptr, &enc)) { printf("create failed: %s\n", cldn_b200_last_error()); return 1; }
  if (cldn_b200_encode_blobs(enc, n, mid_in.data(), in_b.data(), nullptr, nullptr, out.data(), caps.data(), written.data(),
                             CLDN_MEM_DEVICE)) {
    printf("encode_blobs failed: %s\n", cldn_b200_last_error());
    return 1;
  }
  for (size_t f = 0; f < n; ++f) {
    cldn_info_t h;
    size_t hdr = 0;
    const int rc = cldn_b200_decode_header(blobs[f].data(), written[f], &h, &hdr);
    printf("blob %zu: %zu bytes, header %d, width %u\n", f, written[f], rc, h.width);
    bad += rc != 0 || h.width != kept[f] || written[f] < hdr;
  }
  cldn_b200_encoder_destroy(enc);
  if (bad) return 1;
  puts("encode_blobs_racecheck: done");
  return 0;
}
