// TEST INFRASTRUCTURE ONLY — runs the device ZSTD decompressor (cloudini_b200/csrc/cldn_zstd.cu) on chunk bodies from a
// file, under the cusim emulation (plain, AddressSanitizer or ThreadSanitizer build; tests/test_cusim_zstd.py builds it).
//   input   u32 count, then per case: u32 cap, u32 size, size bytes (one chunk body, as ZSTD_decompress would receive it)
//   output  per case: u32 ok (1 = decompressed), u32 size, size bytes
// Every case is one launch of the chunk kernel + the re-framing kernel, exactly as the decoder issues them (one frame of
// one chunk), so the result is what the library would hand to the stage-1 decode.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include <cuda_runtime.h>  // the cusim shim (this file is only ever compiled against it)

#include "cldn_device.cuh"
#include "cldn_kernels.h"

namespace cldn {  // launch counting lives in the encoder's translation unit, which this driver does not link
void count_launch(int) {}
}  // namespace cldn

using namespace cldn;

static bool rd(FILE* f, void* p, size_t n) { return fread(p, 1, n, f) == n; }

int main(int argc, char** argv) {
  if (argc != 3) { fprintf(stderr, "usage: %s cases.bin results.bin\n", argv[0]); return 2; }
  FILE* in = fopen(argv[1], "rb");
  FILE* out = fopen(argv[2], "wb");
  if (!in || !out) return 2;
  uint32_t count = 0;
  if (!rd(in, &count, 4)) return 2;
  for (uint32_t i = 0; i < count; ++i) {
    uint32_t cap = 0, size = 0;
    if (!rd(in, &cap, 4) || !rd(in, &size, 4)) return 2;
    std::vector<uint8_t> payload(4 + size);
    memcpy(payload.data(), &size, 4);
    if (size && !rd(in, payload.data() + 4, size)) return 2;
    const uint32_t stride = (cap + 15u) & ~15u;
    const size_t plain_cap = (static_cast<size_t>(stride) + 4u + 255u) & ~size_t(255);
    uint8_t *d_payload = nullptr, *d_slot = nullptr, *d_lit = nullptr, *d_plain = nullptr;
    uint32_t *d_sizes = nullptr, *d_frame_of = nullptr, *d_err = nullptr;
    uint64_t* d_total = nullptr;
    Lz4Frame* d_frames = nullptr;
    cudaMalloc(&d_payload, payload.size());
    cudaMalloc(&d_slot, stride ? stride : 16);
    cudaMalloc(&d_lit, zstd_warps_per_cta() * zstd_lit_scratch_bytes(cap));
    cudaMalloc(&d_plain, plain_cap);
    cudaMalloc(&d_sizes, 4);
    cudaMalloc(&d_frame_of, 4);
    cudaMalloc(&d_err, 4);
    cudaMalloc(&d_total, 8);
    cudaMalloc(&d_frames, sizeof(Lz4Frame));
    cudaMemcpy(d_payload, payload.data(), payload.size(), cudaMemcpyHostToDevice);
    cudaMemset(d_frame_of, 0, 4);
    cudaMemset(d_err, 0, 4);
    Lz4Frame F;
    memset(&F, 0, sizeof(F));
    F.packed_in = d_payload;
    F.packed_in_bytes = payload.size();
    F.plain_out = d_plain;
    F.plain_cap = plain_cap;
    F.n_chunks = 1;
    cudaMemcpy(d_frames, &F, sizeof(F), cudaMemcpyHostToDevice);
    ZstdLaunch Z;
    memset(&Z, 0, sizeof(Z));
    Z.L.frames = d_frames;
    Z.L.n_frames = 1;
    Z.L.n_chunks_total = 1;
    Z.L.chunk_frame = d_frame_of;
    Z.L.scratch = d_slot;
    Z.L.slot_stride = stride;
    Z.L.chunk_sizes = d_sizes;
    Z.L.sizes = d_total;
    Z.L.err = d_err;
    Z.body_cap = cap;
    Z.n_ctas = 1;
    Z.lit_scratch = d_lit;
    launch_zstd_decompress(Z, nullptr);
    cudaDeviceSynchronize();
    uint32_t err = 0;
    uint64_t total = 0;
    cudaMemcpy(&err, d_err, 4, cudaMemcpyDeviceToHost);
    cudaMemcpy(&total, d_total, 8, cudaMemcpyDeviceToHost);
    std::vector<uint8_t> plain(total);
    if (total) cudaMemcpy(plain.data(), d_plain, total, cudaMemcpyDeviceToHost);
    uint32_t ok = err == DEV_OK ? 1u : 0u, n = 0;
    if (ok) {  // [u32 size][bytes], as the re-framing kernel writes it
      memcpy(&n, plain.data(), 4);
      if (total != 4u + n) { fprintf(stderr, "case %u: re-framed size %llu for %u bytes\n", i, (unsigned long long)total, n); return 3; }
    } else if (err != DEV_ERR_ZSTD) {
      fprintf(stderr, "case %u: unexpected device error %u\n", i, err);
      return 3;
    }
    fwrite(&ok, 4, 1, out);
    fwrite(&n, 4, 1, out);
    if (n) fwrite(plain.data() + 4, 1, n, out);
    cudaFree(d_payload); cudaFree(d_slot); cudaFree(d_lit); cudaFree(d_plain); cudaFree(d_sizes); cudaFree(d_frame_of);
    cudaFree(d_err); cudaFree(d_total); cudaFree(d_frames);
  }
  fclose(out);
  printf("zstd_main: done %u\n", count);
  return 0;
}
