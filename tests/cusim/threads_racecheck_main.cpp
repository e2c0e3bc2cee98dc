// TEST INFRASTRUCTURE ONLY — ThreadSanitizer driver for distinct handles on concurrent host threads
// (tests/test_gpu_concurrency.py). Four host threads each own an encoder, a decoder and a preprocessor for their own
// layout: XYZI (the fast paths), Velodyne XYZIRT, C3 with padding and V5 sections, and Livox raw uint8 fields with a
// Gorilla FLOAT64 stamp. Each runs host- and device-pointer encodes and decodes, device LZ4, host LZ4 / ZSTD where the
// libraries load, viz preprocessing and decode_blobs; every output and the launch count must equal those of the same
// calls made alone on the main thread. The library's host code is instrumented; a data race on process-wide state (the launch counter,
// lazily initialised statics, the dynamic shared memory limits, the stage-2 library loader) is a report.
#include <cmath>
#include <cstdio>
#include <cstring>
#include <thread>
#include <vector>

#include <cuda_runtime.h>  // the cusim shim (this file is only ever compiled against it)

#include "cloudini_b200.h"
#include "cloudini_b200_ros.h"

typedef std::vector<uint8_t> Bytes;

// --control-racy: every job also bumps this plain counter, a race between the host threads the detector must report
static bool g_control_racy = false;
static long g_control_counter = 0;

static void add_field(cldn_info_t* info, const char* name, uint32_t offset, uint8_t type, float res) {
  cldn_field_t& f = info->fields[info->n_fields++];
  memset(&f, 0, sizeof(f));
  strncpy(f.name, name, CLDN_MAX_NAME - 1);
  f.offset = offset; f.type = type; f.has_resolution = res > 0; f.resolution = res;
}

struct Layout {
  cldn_info_t info;
  Bytes cloud;
};

static Layout make_layout(int k, uint32_t n) {
  enum { U8 = 2, U16 = 4, U32 = 6, F32 = 7, F64 = 8 };
  Layout L;
  cldn_b200_info_init(&L.info);
  cldn_info_t& I = L.info;
  I.width = n; I.height = 1; I.compression_opt = 0; I.use_threads = 0;
  const char* xyz[3] = {"x", "y", "z"};
  for (int a = 0; a < 3; ++a) add_field(&I, xyz[a], 4 * a, F32, 0.001f);
  if (k != 2) add_field(&I, "intensity", 12, F32, 0.001f);
  if (k == 0) I.point_step = 16;
  if (k == 1) { add_field(&I, "ring", 16, U16, 0); add_field(&I, "time", 18, F32, 1e-5f); I.point_step = 22; }
  if (k == 2) { add_field(&I, "rgba", 16, U32, 0); add_field(&I, "ring", 20, U16, 0); I.point_step = 32; }
  if (k == 3) { add_field(&I, "tag", 16, U8, 0); add_field(&I, "line", 17, U8, 0); add_field(&I, "stamp", 18, F64, 0); I.point_step = 26; }
  L.cloud.assign(static_cast<size_t>(n) * I.point_step, 0xCD);
  uint32_t rng = 1234567u + 77u * k;
  auto rnd = [&] { rng = rng * 1664525u + 1013904223u; return rng >> 8; };
  float w[3] = {1.f, 2.f, 0.5f};
  for (uint32_t p = 0; p < n; ++p) {
    uint8_t* pt = L.cloud.data() + static_cast<size_t>(p) * I.point_step;
    for (int a = 0; a < 3; ++a) {
      w[a] += (static_cast<int>(rnd() % 2001) - 1000) * 1e-4f;
      float v = (p % 97 == 5 && a == 1) ? NAN : w[a];
      if (p % 5 == 0) v = w[a] - (a == 0 ? 0.0001f : 0.f);           // near-duplicates for the viz voxels
      memcpy(pt + 4 * a, &v, 4);
    }
    if (k != 2) { const float in = static_cast<float>(rnd() % 256); memcpy(pt + 12, &in, 4); }
    if (k == 1) { const uint16_t ring = p % 64; const float t = p * 1e-5f; memcpy(pt + 16, &ring, 2); memcpy(pt + 18, &t, 4); }
    if (k == 2) { const uint32_t rgba = 0xFF000000u | (rnd() % 8) * 0x101010u; const uint16_t ring = p % 64; memcpy(pt + 16, &rgba, 4); memcpy(pt + 20, &ring, 2); }
    if (k == 3) { pt[16] = static_cast<uint8_t>(rnd()); pt[17] = static_cast<uint8_t>(rnd()); const double s = 1.7e9 + p * 1e-5 + (p % 13 == 0 ? 0.25 : 0.0); memcpy(pt + 18, &s, 8); }
  }
  return L;
}

// Everything one thread does with its own handles; the outputs are concatenated into `out`.
static bool job(const Layout& L, Bytes* out) {
  auto put = [&](const void* p, size_t n) { const uint8_t* b = static_cast<const uint8_t*>(p); out->insert(out->end(), b, b + n); };
  auto put_int = [&](long long v) { put(&v, sizeof(v)); };
  const cldn_info_t& info = L.info;
  const size_t nbytes = L.cloud.size();
  if (g_control_racy) ++g_control_counter;
  cldn_encoder_t* enc = nullptr;
  cldn_decoder_t* dec = nullptr;
  cldn_preproc_t* pp = nullptr;
  if (cldn_b200_encoder_create(&info, -1, nullptr, &enc) || cldn_b200_decoder_create(-1, nullptr, &dec) || cldn_b200_preproc_create(-1, nullptr, &pp)) {
    printf("create failed: %s\n", cldn_b200_last_error());
    return false;
  }
  const size_t cap = cldn_b200_max_compressed_size(&info, info.width, 1);
  // host pointers
  Bytes blob(cap);
  size_t written = 0;
  if (cldn_b200_encode(enc, L.cloud.data(), nbytes, blob.data(), cap, 1, &written, CLDN_MEM_HOST)) { printf("encode: %s\n", cldn_b200_last_error()); return false; }
  blob.resize(written);
  put(blob.data(), blob.size());
  cldn_info_t hinfo;
  size_t hdr = 0;
  if (cldn_b200_decode_header(blob.data(), blob.size(), &hinfo, &hdr)) return false;
  Bytes pts(nbytes, 0x5A);
  put_int(cldn_b200_decode(dec, &hinfo, blob.data() + hdr, blob.size() - hdr, pts.data(), nbytes, CLDN_MEM_HOST));
  put(pts.data(), pts.size());
  // device pointers ("device" memory is host memory in the emulation): a batch of two frames, asynchronous, then synchronised
  Bytes d_out[2] = {Bytes(cap), Bytes(cap)};
  const void* ins[2] = {L.cloud.data(), L.cloud.data()};
  const size_t in_b[2] = {nbytes, nbytes}, caps[2] = {cap, cap};
  void* outs[2] = {d_out[0].data(), d_out[1].data()};
  put_int(cldn_b200_encode_batch(enc, 2, ins, in_b, outs, caps, 1, nullptr, CLDN_MEM_DEVICE));
  put_int(cldn_b200_encoder_sync(enc));
  for (auto& o : d_out) put(o.data(), written);
  Bytes d_pts[2] = {Bytes(nbytes, 0x5A), Bytes(nbytes, 0x5A)};
  const void* pl[2] = {d_out[0].data() + hdr, d_out[1].data() + hdr};
  const size_t pl_b[2] = {written - hdr, written - hdr}, pcap[2] = {nbytes, nbytes};
  void* pout[2] = {d_pts[0].data(), d_pts[1].data()};
  put_int(cldn_b200_decode_batch(dec, &hinfo, 2, pl, pl_b, pout, pcap, CLDN_MEM_DEVICE, 0));
  put_int(cldn_b200_decoder_sync(dec));
  for (auto& p : d_pts) put(p.data(), p.size());
  // stage 2: device LZ4, and host LZ4 / ZSTD when the libraries load (the status is part of the output)
  std::vector<Bytes> blobs{blob};
  for (int comp = 1; comp <= 2; ++comp) {
    cldn_info_t ci = info;
    ci.compression_opt = static_cast<uint8_t>(comp);
    cldn_encoder_t* e2 = nullptr;
    const int rc = cldn_b200_encoder_create(&ci, -1, nullptr, &e2);
    put_int(rc);
    if (rc) continue;
    const size_t c2 = cldn_b200_max_compressed_size(&ci, ci.width, 1);
    for (int mem = 0; mem <= (comp == 1 ? 1 : 0); ++mem) {
      Bytes b(c2);
      size_t w2 = 0;
      const int r2 = cldn_b200_encode(e2, L.cloud.data(), nbytes, b.data(), c2, 1, &w2, mem);
      put_int(r2);
      if (r2) continue;
      b.resize(w2);
      put(b.data(), b.size());
      blobs.push_back(b);
    }
    cldn_b200_encoder_destroy(e2);
  }
  // viz preprocessing
  {
    cldn_info_t vi = info;
    Bytes kept(nbytes, 0x5A);
    size_t n_kept = 0;
    int applied = 0;
    put_int(cldn_b200_viz_lossy_preprocess(pp, &vi, L.cloud.data(), nbytes, kept.data(), nbytes, &n_kept, &applied, CLDN_MEM_HOST));
    put_int(static_cast<long long>(n_kept));
    put_int(applied);
    put(kept.data(), kept.size());
  }
  // decode_blobs: every blob above, plus one with a forged chunk prefix
  {
    Bytes bad = blob;
    memset(bad.data() + hdr, 0xFF, 3);
    blobs.push_back(bad);
    const size_t n = blobs.size();
    std::vector<const void*> bi(n);
    std::vector<size_t> bb(n), bc(n, nbytes);
    std::vector<Bytes> bo(n, Bytes(nbytes, 0x5A));
    std::vector<void*> bp(n);
    for (size_t f = 0; f < n; ++f) { bi[f] = blobs[f].data(); bb[f] = blobs[f].size(); bp[f] = bo[f].data(); }
    std::vector<int32_t> status(n);
    put_int(cldn_b200_decode_blobs(dec, n, bi.data(), bb.data(), bp.data(), bc.data(), CLDN_MEM_DEVICE, status.data(), nullptr));
    put(status.data(), n * sizeof(int32_t));
    for (auto& o : bo) put(o.data(), o.size());
  }
  cldn_b200_preproc_destroy(pp);
  cldn_b200_decoder_destroy(dec);
  cldn_b200_encoder_destroy(enc);
  if (g_control_racy) ++g_control_counter;
  return true;
}

int main(int argc, char** argv) {
  g_control_racy = argc > 1 && strcmp(argv[1], "--control-racy") == 0;
  const uint32_t sizes[4] = {40000, 9000, 9000, 9000};   // XYZI: 40 tiles of the persistent encoder
  std::vector<Layout> layouts;
  for (int k = 0; k < 4; ++k) layouts.push_back(make_layout(k, sizes[k]));
  // concurrently first, while the library's lazily initialised state is still untouched; then every job alone on this
  // thread; then concurrently once more (everything initialised). Both concurrent runs must give what the jobs give alone.
  std::vector<Bytes> alone(4), first(4), second(4);
  auto concurrently = [&](std::vector<Bytes>& out, uint64_t* launches) {
    const uint64_t before = cldn_b200_kernel_launch_count();
    bool ok[4] = {false, false, false, false};
    std::vector<std::thread> threads;
    for (int k = 0; k < 4; ++k) threads.emplace_back([&, k] { ok[k] = job(layouts[k], &out[k]); });
    for (auto& t : threads) t.join();
    *launches = cldn_b200_kernel_launch_count() - before;
    return ok[0] && ok[1] && ok[2] && ok[3];
  };
  uint64_t l1 = 0, l2 = 0, l_alone = 0;
  const bool ok1 = concurrently(first, &l1);
  const uint64_t before = cldn_b200_kernel_launch_count();
  for (int k = 0; k < 4; ++k) if (!job(layouts[k], &alone[k])) return 1;
  l_alone = cldn_b200_kernel_launch_count() - before;
  const bool ok2 = concurrently(second, &l2);
  int bad = !ok1 || !ok2;
  for (int k = 0; k < 4; ++k) {
    const bool same = first[k] == alone[k] && second[k] == alone[k];
    printf("layout %d: %zu output bytes, %s\n", k, alone[k].size(), same ? "same as alone" : "DIFFERS");
    bad += !same;
  }
  printf("launches: %llu alone, %llu and %llu concurrently\n", static_cast<unsigned long long>(l_alone),
         static_cast<unsigned long long>(l1), static_cast<unsigned long long>(l2));
  bad += l1 != l_alone || l2 != l_alone;
  if (bad) return 1;
  puts("threads_racecheck: done");
  return 0;
}
