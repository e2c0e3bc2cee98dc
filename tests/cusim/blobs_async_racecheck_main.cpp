// TEST INFRASTRUCTURE ONLY — ThreadSanitizer driver for cldn_b200_decode_blobs_async (tests/test_gpu_decode_blobs_async.py).
// One prepared shape per compression (NONE, LZ4, ZSTD): a call with fewer frames than prepared (empty tables and chunk
// slots), frames of 1 .. 33000 points (empty slots inside frames), a forged chunk prefix and a header of another size
// spelling. Every CUDA thread is a TSAN fiber; the statuses are sanity-checked only (the byte-exact comparisons live in
// the pytest file).
#include <algorithm>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include <cuda_runtime.h>  // the cusim shim (this file is only ever compiled against it)

#include "cloudini_b200.h"

static uint32_t rng_state = 4242;
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
  std::vector<float> cloud(4 * static_cast<size_t>(n) + 4);
  float w = 0;
  for (auto& v : cloud) { w += (static_cast<int>(rnd() % 2001) - 1000) * 1e-5f; v = w; }
  cldn_encoder_t* enc = nullptr;
  std::vector<uint8_t> blob(cldn_b200_max_compressed_size(&info, n, 1) + 16);
  size_t written = 0;
  if (cldn_b200_encoder_create(&info, -1, nullptr, &enc) ||
      cldn_b200_encode(enc, cloud.data(), 16 * static_cast<size_t>(n), blob.data(), blob.size(), 1, &written, CLDN_MEM_HOST)) {
    printf("encode failed: %s\n", cldn_b200_last_error());
    blob.clear();
  }
  cldn_b200_encoder_destroy(enc);
  blob.resize(written);
  return blob;
}

int main() {
  int bad = 0;
  for (uint8_t comp = 0; comp <= 2; ++comp) {
    const uint32_t sizes[] = {33000, 1, 20000, 5000};
    std::vector<std::vector<uint8_t>> blobs;
    for (uint32_t n : sizes) blobs.push_back(blob_of(n, comp));
    for (auto& b : blobs) if (b.empty()) return 1;
    cldn_info_t info;
    size_t hdr = 0;
    cldn_b200_decode_header(blobs[2].data(), blobs[2].size(), &info, &hdr);
    memset(blobs[2].data() + hdr, 0xFF, 3);  // frame 2: forged first chunk prefix
    const std::string w = "\nwidth: ";       // frame 3: "width: 05000"
    auto at = std::search(blobs[3].begin(), blobs[3].end(), w.begin(), w.end()) + w.size();
    blobs[3].insert(at, '0');
    const size_t n = blobs.size();
    std::vector<cldn_blob_desc_t> desc(n);
    std::vector<std::vector<uint8_t>> outs(n);
    for (size_t f = 0; f < n; ++f) {
      outs[f].assign(16 * static_cast<size_t>(sizes[f]), 0);
      desc[f] = {blobs[f].data(), blobs[f].size(), outs[f].data(), outs[f].size()};
    }
    cldn_decoder_t* dec = nullptr;
    if (cldn_b200_decoder_create(-1, nullptr, &dec)) { printf("create failed: %s\n", cldn_b200_last_error()); return 1; }
    std::vector<int32_t> status(n, 99);
    std::vector<uint64_t> decoded(n, 7);
    if (cldn_b200_decoder_prepare_blobs(dec, &info, n + 2, 40000) ||
        cldn_b200_decode_blobs_async(dec, n, desc.data(), status.data(), decoded.data()) || cldn_b200_decoder_sync(dec)) {
      printf("call failed: %s\n", cldn_b200_last_error());
      return 1;
    }
    for (size_t f = 0; f < n; ++f) {
      const int32_t want = f == 2 ? CLDN_ERR_CORRUPT_DATA : f == 3 ? CLDN_ERR_BAD_HEADER : CLDN_OK;
      printf("compression %d frame %zu: status %d decoded %llu\n", comp, f, status[f], static_cast<unsigned long long>(decoded[f]));
      bad += status[f] != want || decoded[f] != (want == CLDN_OK ? 16ull * sizes[f] : 0ull);
    }
    cldn_b200_decoder_destroy(dec);
  }
  if (bad) return 1;
  puts("blobs_async_racecheck: done");
  return 0;
}
