// TEST INFRASTRUCTURE ONLY — ThreadSanitizer driver for cldn_b200_decode_blobs (tests/test_gpu_decode_blobs.py).
// One call with device pointers over a mixed, damaged batch: XYZI frames of different sizes without stage 2, ZSTD and
// LZ4 frames (one fused group each, stage 2 by the device kernels), a frame with a forged chunk prefix (its error goes
// to its own word while the other frames of its group decode) and one with a damaged header line. Every CUDA thread is a
// TSAN fiber; the statuses are sanity-checked only (the byte-exact comparisons live in the pytest file).
#include <cmath>
#include <cstdio>
#include <cstring>
#include <vector>

#include <cuda_runtime.h>  // the cusim shim (this file is only ever compiled against it)

#include "cloudini_b200.h"

static uint32_t rng_state = 777;
static uint32_t rnd() { rng_state = rng_state * 1664525u + 1013904223u; return rng_state >> 8; }

static cldn_info_t xyzi(uint32_t n, uint8_t compression) {
  cldn_info_t info;
  cldn_b200_info_init(&info);
  info.width = n; info.height = 1; info.point_step = 16; info.compression_opt = compression;
  const char* names[4] = {"x", "y", "z", "intensity"};
  for (int k = 0; k < 4; ++k) {
    cldn_field_t& f = info.fields[info.n_fields++];
    memset(&f, 0, sizeof(f));
    strncpy(f.name, names[k], CLDN_MAX_NAME - 1);
    f.offset = 4 * k; f.type = 7; f.has_resolution = 1; f.resolution = 0.001f;
  }
  return info;
}

static std::vector<uint8_t> blob_of(uint32_t n, uint8_t compression) {
  cldn_info_t info = xyzi(n, compression);
  std::vector<float> cloud(4 * static_cast<size_t>(n));
  float w = 0;
  for (auto& v : cloud) { w += (static_cast<int>(rnd() % 2001) - 1000) * 1e-5f; v = w; }
  cldn_encoder_t* enc = nullptr;
  std::vector<uint8_t> blob(cldn_b200_max_compressed_size(&info, n, 1) + 16);
  size_t written = 0;
  if (cldn_b200_encoder_create(&info, -1, nullptr, &enc) ||
      cldn_b200_encode(enc, cloud.data(), cloud.size() * 4, blob.data(), blob.size(), 1, &written, CLDN_MEM_HOST)) {
    printf("encode failed: %s\n", cldn_b200_last_error());
    blob.clear();
  }
  cldn_b200_encoder_destroy(enc);
  blob.resize(written);
  return blob;
}

int main() {
  const uint32_t sizes[] = {40000, 1, 33000, 20000, 35000, 20000, 20000};
  const uint8_t comps[] = {0, 0, 0, 2, 2, 1, 1};
  std::vector<std::vector<uint8_t>> blobs;
  for (int k = 0; k < 7; ++k) blobs.push_back(blob_of(sizes[k], comps[k]));
  for (auto& b : blobs) if (b.empty()) return 1;
  // frame 2: forged first chunk prefix; frame 6: damaged header line
  cldn_info_t info;
  size_t hdr = 0;
  cldn_b200_decode_header(blobs[2].data(), blobs[2].size(), &info, &hdr);
  memset(blobs[2].data() + hdr, 0xFF, 3);
  blobs[6][3] = 'X';
  const size_t n = blobs.size();
  std::vector<const void*> in(n);
  std::vector<size_t> in_b(n), caps(n);
  std::vector<std::vector<uint8_t>> outs(n);
  std::vector<void*> out(n);
  for (size_t f = 0; f < n; ++f) {
    in[f] = blobs[f].data();
    in_b[f] = blobs[f].size();
    caps[f] = 16 * static_cast<size_t>(sizes[f]);
    outs[f].assign(caps[f], 0);
    out[f] = outs[f].data();
  }
  cldn_decoder_t* dec = nullptr;
  if (cldn_b200_decoder_create(-1, nullptr, &dec)) { printf("create failed: %s\n", cldn_b200_last_error()); return 1; }
  std::vector<int32_t> status(n);
  cldn_b200_decode_blobs(dec, n, in.data(), in_b.data(), out.data(), caps.data(), CLDN_MEM_DEVICE, status.data(), nullptr);
  int bad = 0;
  for (size_t f = 0; f < n; ++f) {
    const int32_t want = f == 2 ? CLDN_ERR_CORRUPT_DATA : f == 6 ? CLDN_ERR_BAD_HEADER : CLDN_OK;
    printf("frame %zu: status %d (%s)\n", f, status[f], cldn_b200_decoder_frame_error(dec, f));
    bad += status[f] != want;
  }
  cldn_b200_decoder_destroy(dec);
  if (bad) return 1;
  puts("blobs_racecheck: done");
  return 0;
}
