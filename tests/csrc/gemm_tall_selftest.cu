// gemm_tall_selftest.cu — the split-operand GEMM (sce_gemm.cuh) on 192-row output tiles (BM = kBMTall) against the
// same GEMM on 128-row tiles, in the two configurations libsce launches on tall tiles:
//   - decode: K-major f16f8 on E5M2 wgmma, EpiDecodeT with the column sums of g, the batch-major copies of g's 8-bit
//     planes and the per-row partials of r^2 (every output the epilogue has);
//   - the weight gradient: MN-major f16f8 on E5M2 wgmma from batch-major 8-bit planes, two operand sets, EpiStoreF32,
//     with set 0's B residual plane flagged all-zero (its cross term skipped) or not.
// Each case runs at cluster sizes 1 and 2 (2 where the column-tile count is even) on both tile heights, from output
// buffers filled with the same sentinel bytes. It passes when every output buffer of every run is bitwise equal to the
// 128-row run at cluster size 1: an output element's accumulation order depends on the K sweep only, and every
// epilogue share keeps the 128-row tiling's coordinates, so the loss partials, g_part, row_part and batch-major stores
// land in the same slots with the same contents (slots no share writes keep the sentinel in both). Row counts cover a
// last 192-row tile holding 64 rows (4096), ragged edges (1210, 1037) and fewer rows than one tile (33, 5), rounded up
// to 16 for the weight gradient (its rows are features: 4096, 1216, 1040, 48, 16); d = 64 has one column tile. Prints
// one PASS / FAIL line per case and exits non-zero when one fails. Build: Makefile target `selftest`.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "../../sparse_coding_b200/csrc/sce_epilogues.cuh"
#include "../../sparse_coding_b200/csrc/sce_tmap.h"

using namespace sce;

#define CK(x)                                                                         \
  do {                                                                                \
    cudaError_t e_ = (x);                                                             \
    if (e_ != cudaSuccess) {                                                          \
      printf("CUDA error %s at %s:%d\n", cudaGetErrorString(e_), __FILE__, __LINE__); \
      exit(2);                                                                        \
    }                                                                                 \
  } while (0)

constexpr int kF8 = kArithF16F8;
constexpr int BK = gemm_bk(kF8);
static int g_sms = 0;
static int g_fail = 0;

// finite fp16 / E5M2 values of either sign, |v| < 1, from a hash of the index and the seed
__global__ void fill_kernel(uint8_t* p, size_t n, int elem, uint32_t seed) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    uint32_t h = (uint32_t)i * 2654435761u ^ seed;
    h ^= h >> 15;
    h *= 2246822519u;
    h ^= h >> 13;
    if (elem == 2) reinterpret_cast<uint16_t*>(p)[i] = uint16_t((h & 0x37FFu) | (h >> 16 & 0x8000u));
    else if (elem == 1) p[i] = uint8_t((h & 0x37u) | (h >> 24 & 0x80u));
    else reinterpret_cast<float*>(p)[i] = float(int(h & 0xFFFFu) - 32768) * (1.0f / 32768.0f);
  }
}

static std::vector<void*> g_dev;
static void* dev(size_t bytes) {
  void* d = nullptr;
  CK(cudaMalloc(&d, bytes ? bytes : 16));
  g_dev.push_back(d);
  return d;
}
// elem 2: fp16, 1: e5m2, 4: fp32
static void* filled(size_t n, int elem) {
  void* d = dev(n * elem);
  fill_kernel<<<512, 256>>>(static_cast<uint8_t*>(d), n, elem, (uint32_t)g_dev.size() * 7919u + 1u);
  CK(cudaGetLastError());
  return d;
}
static void free_all() {
  for (void* d : g_dev) cudaFree(d);
  g_dev.clear();
}

struct Out {   // an output buffer of the epilogue and its size
  void* p;
  size_t bytes;
};
static void sentinel(const std::vector<Out>& outs) {
  for (const Out& o : outs) CK(cudaMemset(o.p, 0xA5, o.bytes));
}
static std::vector<std::vector<uint8_t>> fetch(const std::vector<Out>& outs) {
  std::vector<std::vector<uint8_t>> h;
  for (const Out& o : outs) {
    h.emplace_back(o.bytes);
    CK(cudaMemcpy(h.back().data(), o.p, o.bytes, cudaMemcpyDeviceToHost));
  }
  return h;
}

// Runs `launch(bm, cluster)` for (128, 1), (192, 1), and at cluster size 2 where tiles_n is even, and compares every
// output with the first run
template <class F>
static void compare_runs(const char* name, int tiles_n, const std::vector<Out>& outs, F&& launch) {
  std::vector<std::vector<uint8_t>> ref;
  int runs = 0, bad = 0;
  char sizes[64] = "";
  for (int cluster = 1; cluster <= (tiles_n % 2 == 0 ? 2 : 1); ++cluster)
    for (int bm : {kBM, kBMTall}) {
      sentinel(outs);
      CK(launch(bm, cluster));
      CK(cudaDeviceSynchronize());
      auto got = fetch(outs);
      if (ref.empty()) ref = got;
      else
        for (size_t i = 0; i < got.size(); ++i)
          if (got[i] != ref[i]) {
            ++bad;
            size_t j = 0;
            while (got[i][j] == ref[i][j]) ++j;
            printf("  %s: output %zu differs at BM %d, cluster %d, byte %zu of %zu\n", name, i, bm, cluster, j, got[i].size());
          }
      ++runs;
      snprintf(sizes + strlen(sizes), sizeof(sizes) - strlen(sizes), "%s%d/%d", runs > 1 ? ", " : "", bm, cluster);
    }
  printf("%s %s: %d runs (BM/cluster %s), %zu outputs\n", bad ? "FAIL" : "PASS", name, runs, sizes, outs.size());
  if (bad) ++g_fail;
}

// decode: A = c [models][rows][K] K-major, B = the transposed dictionary [models][d][K] K-major
static void decode_case(int models, int rows, int K, int d) {
  using E = EpiDecodeT<kF8, true, true, true>;
  const int ld_t = (rows + 15) / 16 * 16;
  const size_t na = (size_t)models * rows * K, nb = (size_t)models * d * K;
  void *a_hi = filled(na, 2), *a_lo = filled(na, 1), *a_x8 = filled(na, 1);
  void *b_hi = filled(nb, 2), *b_lo = filled(nb, 1), *b_x8 = filled(nb, 1);
  const int tiles_m = (rows + kBM - 1) / kBM, tiles_n = (d + kBN - 1) / kBN;
  typename E::Params ep;
  memset(&ep, 0, sizeof(ep));
  ep.x = static_cast<const float*>(filled((size_t)models * rows * d, 4));
  ep.x_model_stride = (long long)rows * d;
  std::vector<Out> outs = {{dev((size_t)models * rows * d * 2), (size_t)models * rows * d * 2},
                           {dev((size_t)models * rows * d), (size_t)models * rows * d},
                           {dev((size_t)models * rows * d), (size_t)models * rows * d},
                           {dev((size_t)models * rows * d * 4), (size_t)models * rows * d * 4},
                           {dev((size_t)models * tiles_m * 8 * tiles_n * 4), (size_t)models * tiles_m * 8 * tiles_n * 4},
                           {dev((size_t)models * tiles_m * 4 * d * 4), (size_t)models * tiles_m * 4 * d * 4},
                           {dev((size_t)models * rows * 2 * tiles_n * 4), (size_t)models * rows * 2 * tiles_n * 4},
                           {dev((size_t)models * d * ld_t), (size_t)models * d * ld_t},
                           {dev((size_t)models * d * ld_t), (size_t)models * d * ld_t}};
  ep.g_hi = static_cast<uint16_t*>(outs[0].p);
  ep.g_lo = static_cast<uint8_t*>(outs[1].p);
  ep.g_x8 = static_cast<uint8_t*>(outs[2].p);
  ep.x_hat = static_cast<float*>(outs[3].p);
  ep.part = static_cast<float*>(outs[4].p);
  ep.g_part = static_cast<float*>(outs[5].p);
  ep.row_part = static_cast<float*>(outs[6].p);
  ep.t_lo = static_cast<uint8_t*>(outs[7].p);
  ep.t_x8 = static_cast<uint8_t*>(outs[8].p);
  ep.t_ld = ld_t;
  ep.g_model_stride = (long long)rows * d;
  ep.xhat_model_stride = (long long)rows * d;
  ep.ld = d;
  ep.tiles_m = tiles_m;   // the epilogue's slots follow the 128-row tiling whatever the GEMM's tile height
  ep.tiles_n = tiles_n;
  ep.gscale = 1.f;
  auto params = [&](int bm) {
    GemmParams<typename E::Params> p;
    memset(&p, 0, sizeof(p));
    bool ok = make_tmap_bf16_box(&p.a_hi[0], a_hi, models, rows, K, K, (uint64_t)rows * K, BK, bm, CU_TENSOR_MAP_SWIZZLE_128B);
    ok &= make_tmap_u8_box(&p.a_lo[0], a_lo, models, rows, K, K, (uint64_t)rows * K, BK, bm, CU_TENSOR_MAP_SWIZZLE_64B);
    ok &= make_tmap_u8_box(&p.a_x8[0], a_x8, models, rows, K, K, (uint64_t)rows * K, BK, bm, CU_TENSOR_MAP_SWIZZLE_64B);
    ok &= make_tmap_bf16_box(&p.b_hi[0], b_hi, models, d, K, K, (uint64_t)d * K, BK, kBN, CU_TENSOR_MAP_SWIZZLE_128B);
    ok &= make_tmap_u8_box(&p.b_lo[0], b_lo, models, d, K, K, (uint64_t)d * K, BK, kBN, CU_TENSOR_MAP_SWIZZLE_64B);
    ok &= make_tmap_u8_box(&p.b_x8[0], b_x8, models, d, K, K, (uint64_t)d * K, BK, kBN, CU_TENSOR_MAP_SWIZZLE_64B);
    if (!ok) {
      printf("tensor map encode failed\n");
      exit(2);
    }
    p.a_batched[0] = p.b_batched[0] = 1;
    p.nsets = 1;
    p.k_total = K;
    p.passes = 3;
    p.n_models = models;
    p.m_total = rows;
    p.n_total = d;
    p.tiles_m = bm == kBM ? gemm_tiles_m<kBM>(rows) : gemm_tiles_m<kBMTall>(rows);
    p.tiles_n = tiles_n;
    p.epi = ep;
    return p;
  };
  const auto p128 = params(kBM), p192 = params(kBMTall);
  char name[128];
  snprintf(name, sizeof(name), "decode rows %d, K %d, d %d, %d models", rows, K, d, models);
  compare_runs(name, tiles_n, outs, [&](int bm, int cluster) {
    return bm == kBM ? launch_gemm_clusters<E, false, false, false, kF8, true>(p128, 0, g_sms, 0, cluster)
                     : launch_gemm_clusters<E, false, false, false, kF8, true, kBMTall>(p192, 0, g_sms, 0, cluster);
  });
  free_all();
}

// weight gradient: out[model] = sum over the K batch rows of A_set[model]^T B_set[model], two operand sets; the fp16
// planes [models][K][cols] MN-major, the 8-bit ones batch-major [models][cols][ld] K-major. x_exact: set 0's B residual
// plane is flagged all-zero.
static void dw_case(int models, int rows, int K, int d, bool x_exact) {
  using E = EpiStoreF32;
  const int ld = (K + 15) / 16 * 16;
  uint32_t* zero_flag = static_cast<uint32_t*>(dev(4));
  CK(cudaMemset(zero_flag, 0, 4));
  struct Op {
    void *hi, *lo, *x8;
  } a[2], b[2];
  for (int s = 0; s < 2; ++s) {
    a[s] = {filled((size_t)models * K * rows, 2), filled((size_t)models * rows * ld, 1), filled((size_t)models * rows * ld, 1)};
    b[s] = {filled((size_t)models * K * d, 2), filled((size_t)models * d * ld, 1), filled((size_t)models * d * ld, 1)};
  }
  std::vector<Out> outs = {{dev((size_t)models * rows * d * 4), (size_t)models * rows * d * 4}};
  E::Params ep;
  ep.out = static_cast<float*>(outs[0].p);
  ep.model_stride = (long long)rows * d;
  ep.ld = d;
  ep.scale = 0.5f;
  const int tiles_n = (d + kBN - 1) / kBN;
  auto params = [&](int bm) {
    GemmParams<E::Params> p;
    memset(&p, 0, sizeof(p));
    bool ok = true;
    auto maps = [&](const Op& o, int cols, uint32_t box, CUtensorMap* hi, CUtensorMap* lo, CUtensorMap* x8) {
      ok &= make_tmap_bf16(hi, o.hi, models, K, cols, cols, (uint64_t)K * cols, BK);
      ok &= make_tmap_u8_box(lo, o.lo, models, cols, K, ld, (uint64_t)cols * ld, BK, box, CU_TENSOR_MAP_SWIZZLE_64B);
      ok &= make_tmap_u8_box(x8, o.x8, models, cols, K, ld, (uint64_t)cols * ld, BK, box, CU_TENSOR_MAP_SWIZZLE_64B);
    };
    for (int s = 0; s < 2; ++s) {
      maps(a[s], rows, bm, &p.a_hi[s], &p.a_lo[s], &p.a_x8[s]);
      maps(b[s], d, kBN, &p.b_hi[s], &p.b_lo[s], &p.b_x8[s]);
      p.a_batched[s] = p.b_batched[s] = 1;
    }
    if (!ok) {
      printf("tensor map encode failed\n");
      exit(2);
    }
    if (x_exact) p.b_res_flag[0] = zero_flag;
    p.nsets = 2;
    p.k_total = K;
    p.passes = 3;
    p.n_models = models;
    p.m_total = rows;
    p.n_total = d;
    p.tiles_m = bm == kBM ? gemm_tiles_m<kBM>(rows) : gemm_tiles_m<kBMTall>(rows);
    p.tiles_n = tiles_n;
    p.epi = ep;
    return p;
  };
  const auto p128 = params(kBM), p192 = params(kBMTall);
  char name[128];
  snprintf(name, sizeof(name), "dw rows %d, K %d, d %d, %d models, x residual %s", rows, K, d, models,
           x_exact ? "flagged zero" : "read");
  compare_runs(name, tiles_n, outs, [&](int bm, int cluster) {
    return bm == kBM ? launch_gemm_clusters<E, true, true, false, kF8, true>(p128, 0, g_sms, 0, cluster)
                     : launch_gemm_clusters<E, true, true, false, kF8, true, kBMTall>(p192, 0, g_sms, 0, cluster);
  });
  free_all();
}

int main() {
  setvbuf(stdout, nullptr, _IOLBF, 0);
  cudaDeviceProp prop;
  CK(cudaGetDeviceProperties(&prop, 0));
  g_sms = prop.multiProcessorCount;
  for (int rows : {4096, 1210, 1037, 33, 5}) {
    decode_case(2, rows, 640, 256);
    decode_case(3, rows, 640, 64);
    // the weight gradient's rows are features, whose fp16 planes are MN-major: a multiple of 16 (TMA pitch)
    for (bool x_exact : {false, true}) {
      dw_case(2, (rows + 15) / 16 * 16, 1037, 256, x_exact);
      dw_case(2, (rows + 15) / 16 * 16, 512, 64, x_exact);
    }
  }
  // config 2's decode and weight-gradient shapes (16 models, batch 8192, n = 4096, d = 512), a few models of them
  decode_case(2, 8192, 4096, 512);
  dw_case(2, 4096, 8192, 512, true);
  printf(g_fail ? "%d FAILED\n" : "ALL PASS\n", g_fail);
  return g_fail ? 1 : 0;
}
