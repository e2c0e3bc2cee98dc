// TEST INFRASTRUCTURE ONLY — ThreadSanitizer driver for stage 2 on the device (cldn_b200_encoder_set_stage2_on_device,
// tests/test_gpu_zstd_encode.py): encode_blobs of clouds of mixed sizes with ZSTD and LZ4 for CLDN_MEM_DEVICE and
// CLDN_MEM_HOST, so that the block compressor (cldn_zstd_enc.cu), the LZ4 compressor and the shared pack run with every
// CUDA thread a TSAN fiber. The blobs are decoded back and compared with the clouds' stage-1 round trip (NONE).
#include <cstdio>
#include <cstring>
#include <vector>

#include <cuda_runtime.h>  // the cusim shim (this file is only ever compiled against it)

#include "cloudini_b200.h"

static uint32_t rng_state = 777;
static uint32_t rnd() { rng_state = rng_state * 1664525u + 1013904223u; return rng_state >> 8; }

int main() {
  cldn_info_t info;
  cldn_b200_info_init(&info);
  info.point_step = 16;
  const char* names[4] = {"x", "y", "z", "intensity"};
  for (int k = 0; k < 4; ++k) {
    cldn_field_t& f = info.fields[info.n_fields++];
    memset(&f, 0, sizeof(f));
    strncpy(f.name, names[k], CLDN_MAX_NAME - 1);
    f.offset = 4 * k; f.type = CLDN_FLOAT32; f.has_resolution = 1; f.resolution = 0.01f;
  }
  const uint32_t sizes[] = {40000, 0, 1, 9000};
  const size_t n = sizeof(sizes) / sizeof(sizes[0]);
  std::vector<std::vector<float>> clouds(n);
  std::vector<const void*> in(n);
  std::vector<size_t> in_b(n);
  for (size_t f = 0; f < n; ++f) {
    clouds[f].resize(4 * static_cast<size_t>(sizes[f]) + 4);
    float w = 0;
    for (size_t i = 0; i < 4 * static_cast<size_t>(sizes[f]); ++i) {
      w += (static_cast<int>(rnd() % 2001) - 1000) * 1e-4f;
      clouds[f][i] = w;
    }
    in[f] = clouds[f].data();
    in_b[f] = 16 * static_cast<size_t>(sizes[f]);
  }
  int bad = 0;
  const int comps[2] = {CLDN_COMP_ZSTD, CLDN_COMP_LZ4};
  const int mems[2] = {CLDN_MEM_DEVICE, CLDN_MEM_HOST};
  std::vector<std::vector<uint8_t>> first(n);
  for (int c = 0; c < 2; ++c) {
    info.compression_opt = static_cast<uint8_t>(comps[c]);
    cldn_encoder_t* enc = nullptr;
    if (cldn_b200_encoder_create(&info, -1, nullptr, &enc)) { printf("create failed: %s\n", cldn_b200_last_error()); return 1; }
    if (cldn_b200_encoder_set_stage2_on_device(enc, 1)) { printf("policy failed: %s\n", cldn_b200_last_error()); return 1; }
    for (int m = 0; m < 2; ++m) {
      std::vector<std::vector<uint8_t>> blobs(n);
      std::vector<void*> out(n);
      std::vector<size_t> caps(n), written(n);
      for (size_t f = 0; f < n; ++f) {
        caps[f] = cldn_b200_max_compressed_size(&info, sizes[f], 0) + 4096;
        blobs[f].assign(caps[f], 0);
        out[f] = blobs[f].data();
      }
      if (cldn_b200_encode_blobs(enc, n, in.data(), in_b.data(), nullptr, nullptr, out.data(), caps.data(), written.data(), mems[m])) {
        printf("encode_blobs failed: %s\n", cldn_b200_last_error());
        return 1;
      }
      cldn_decoder_t* dec = nullptr;
      if (cldn_b200_decoder_create(-1, nullptr, &dec)) { printf("decoder failed\n"); return 1; }
      for (size_t f = 0; f < n; ++f) {
        blobs[f].resize(written[f]);
        if (m == 0) first[f] = blobs[f];
        bad += blobs[f] != first[f];
        cldn_info_t h;
        size_t hdr = 0;
        int rc = cldn_b200_decode_header(blobs[f].data(), written[f], &h, &hdr);
        std::vector<uint8_t> pts(16 * static_cast<size_t>(sizes[f]) + 16, 0);
        if (!rc && sizes[f]) rc = cldn_b200_decode(dec, &h, blobs[f].data() + hdr, written[f] - hdr, pts.data(), pts.size(), CLDN_MEM_HOST);
        // lossy floats: within half a resolution step
        for (size_t i = 0; !rc && i < 4 * static_cast<size_t>(sizes[f]); ++i) {
          float v;
          memcpy(&v, pts.data() + 4 * i, 4);
          if (!(v - clouds[f][i] <= 0.0051f && clouds[f][i] - v <= 0.0051f)) { rc = 1; break; }
        }
        printf("comp %d mem %d blob %zu: %zu bytes, decode %d\n", comps[c], mems[m], f, written[f], rc);
        bad += rc != 0;
      }
      cldn_b200_decoder_destroy(dec);
    }
    cldn_b200_encoder_destroy(enc);
  }
  if (bad) return 1;
  puts("zstd_encode_racecheck: done");
  return 0;
}
