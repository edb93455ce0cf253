// gemm_cluster_selftest.cu — the split-operand GEMM (sce_gemm.cuh) run in clusters of two CTAs that share each A tile by
// TMA multicast, against the same GEMM in clusters of one and against double-precision products of its operand planes.
//
// Each case runs one configuration libsce launches (bf16x3: K x K, K x MN, K x MN and MN x MN with split accumulators;
// f16f8: K x K and MN x MN on E5M2 wgmma, MN x MN widened) through launch_gemm_clusters at cluster size 1 and, where
// the column-tile count is even, 2 (whatever K length launch_gemm would ask for before taking 2; never on the widened
// path, which launch_gemm runs singly), twice each. It passes when
//   - every run of the case is bitwise equal to the first (multicast changes where an A tile comes from, not a value);
//   - sampled outputs of every tile are within 1e-3 sqrt(K sets) (bf16x3) or 1e-4 sqrt(K sets) (f16f8) of the fp64
//     product of the planes, and no output is left unwritten.
// The cases cover odd and even column-tile counts, ragged M and N (tile rows whose second half lies wholly past M, where
// TMA completes the stage's bytes with zeros), two operand sets, tile counts just below and above twice the SM count,
// and a pair-indexed (kPairTiles) schedule whose pairs repeat and swap models. Prints one PASS / FAIL line per case and
// exits non-zero when one fails. Build: Makefile target `selftest`.
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include <cuda_fp16.h>
#include <cuda_fp8.h>

#include "../../sparse_coding_b200/csrc/sce_gemm.cuh"
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

constexpr int kBf = kArithBf16x3, kF8 = kArithF16F8;

static int g_sms = 0;
static std::vector<void*> g_dev;

static uint32_t rng_state = 4242u;
static float frand() {  // uniform in [-1, 1)
  rng_state = rng_state * 1664525u + 1013904223u;
  return (float)((rng_state >> 8) & 0xFFFFFF) / 8388608.0f - 1.0f;
}

static double bf16_value(uint16_t b) {
  const uint32_t u = uint32_t(b) << 16;
  float f;
  memcpy(&f, &u, 4);
  return f;
}
static double f16_value(uint16_t b) {
  __half_raw r;
  r.x = b;
  return __half2float(__half(r));
}
static double e5m2_value(uint8_t b) { return f16_value(uint16_t(b << 8)); }

// The planes of one operand [models][rows][K] drawn uniform in [-scale, scale). bf16x3: p16 = bf16(x), lo16 = bf16 of
// the rest; f16f8: p16 = fp16(x), h8 = e5m2(x), l8 = e5m2((x - fp16(x)) 2^kLoShift).
struct Operand {
  int arith, models, rows, K;
  std::vector<uint16_t> p16, lo16;
  std::vector<uint8_t> h8, l8;
  size_t at(int m, int r, int k) const { return ((size_t)m * rows + r) * K + k; }
};

static Operand make_operand(int arith, int models, int rows, int K, float scale) {
  Operand o{arith, models, rows, K};
  const size_t n = (size_t)models * rows * K;
  o.p16.resize(n);
  if (arith == kBf) o.lo16.resize(n);
  else o.h8.resize(n), o.l8.resize(n);
  for (size_t i = 0; i < n; ++i) {
    const float v = frand() * scale;
    if (arith == kBf) {
      const __nv_bfloat16 h = __float2bfloat16_rn(v);
      o.p16[i] = __nv_bfloat16_raw(h).x;
      o.lo16[i] = __nv_bfloat16_raw(__float2bfloat16_rn(v - __bfloat162float(h))).x;
    } else {
      const __half h = __float2half_rn(v);
      o.p16[i] = __half_raw(h).x;
      o.h8[i] = __nv_cvt_float_to_fp8(v, __NV_SATFINITE, __NV_E5M2);
      o.l8[i] = __nv_cvt_float_to_fp8((v - __half2float(h)) * float(1 << kLoShift), __NV_SATFINITE, __NV_E5M2);
    }
  }
  return o;
}

// one plane on the device, K-major [models][rows][pitch] or MN-major [models][K][pitch], rows padded to 16 elements
template <class T>
static const T* upload(const Operand& o, const std::vector<T>& v, bool mn, uint64_t& pitch) {
  pitch = ((mn ? o.rows : o.K) + 15) / 16 * 16;
  const size_t outer = mn ? o.K : o.rows;
  std::vector<T> buf((size_t)o.models * outer * pitch, T(0));
  for (int m = 0; m < o.models; ++m)
    for (int r = 0; r < o.rows; ++r)
      for (int k = 0; k < o.K; ++k) buf[((size_t)m * outer + (mn ? k : r)) * pitch + (mn ? r : k)] = v[o.at(m, r, k)];
  T* d = nullptr;
  CK(cudaMalloc(&d, buf.size() * sizeof(T)));
  CK(cudaMemcpy(d, buf.data(), buf.size() * sizeof(T), cudaMemcpyHostToDevice));
  g_dev.push_back(d);
  return d;
}

// the maps of one operand, laid out as libsce lays them out (see tests/csrc/gemm_selftest.cu)
static void operand_maps(const Operand& o, bool mn16, bool mn8, uint32_t box_rows, CUtensorMap* hi, CUtensorMap* lo,
                         CUtensorMap* x8) {
  const int BK = gemm_bk(o.arith);
  auto map16 = [&](CUtensorMap* t, const std::vector<uint16_t>& v) {
    uint64_t pitch;
    const void* d = upload(o, v, mn16, pitch);
    if (mn16) return make_tmap_bf16(t, d, o.models, o.K, o.rows, pitch, o.K * pitch, BK);
    return make_tmap_bf16_box(t, d, o.models, o.rows, o.K, pitch, o.rows * pitch, BK, box_rows,
                              BK == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B);
  };
  auto map8 = [&](CUtensorMap* t, const std::vector<uint8_t>& v) {
    uint64_t pitch;
    const void* d = upload(o, v, mn8, pitch);
    if (mn8) return make_tmap_u8_box(t, d, o.models, o.K, o.rows, pitch, o.K * pitch, 128, BK, CU_TENSOR_MAP_SWIZZLE_NONE);
    return make_tmap_u8_box(t, d, o.models, o.rows, o.K, pitch, o.rows * pitch, BK, box_rows, CU_TENSOR_MAP_SWIZZLE_64B);
  };
  const bool ok = o.arith == kBf ? map16(hi, o.p16) && map16(lo, o.lo16)
                                 : map16(hi, o.p16) && map8(lo, o.h8) && map8(x8, o.l8);
  if (!ok) {
    printf("tensor map encode failed\n");
    exit(2);
  }
}

// EpiStoreF32 on a pair-indexed schedule: tile index `model` is pair q, whose operands are models pairs[2q], pairs[2q+1]
struct EpiPairStore : EpiStoreF32 {
  static constexpr bool kPairTiles = true;
  struct Params : EpiStoreF32::Params {
    const int* pairs;
  };
  __device__ EpiPairStore(const Params& p, const TileCoord& t, int m, int n, uint8_t* s) : EpiStoreF32(p, t, m, n, s) {}
};

struct Case {
  const char* name;
  int models, M, N, K, nsets;
  bool a_shared = false;   // A is one operand for all models (the encoder's x)
  int pairs = 0;           // > 0: a kPairTiles schedule of this many pairs over `models` models
};

template <class Epi, bool A_MN, bool B_MN, bool SPLIT, int ARITH, bool NATIVE>
static std::vector<float> run_gemm(const Case& c, const Operand* A, const Operand* B, const std::vector<int>& pairs,
                                   int cluster) {
  typename Epi::Params ep{};
  GemmParams<typename Epi::Params> p;
  memset(&p, 0, sizeof(p));
  for (int s = 0; s < c.nsets; ++s) {
    operand_maps(A[s], A_MN, A_MN && !NATIVE, kBM, &p.a_hi[s], &p.a_lo[s], &p.a_x8[s]);
    operand_maps(B[s], B_MN, B_MN && !NATIVE, kBN, &p.b_hi[s], &p.b_lo[s], &p.b_x8[s]);
    p.a_batched[s] = A[s].models > 1;
    p.b_batched[s] = B[s].models > 1;
  }
  const int tiles_models = c.pairs ? c.pairs : c.models;
  const size_t out_elems = (size_t)tiles_models * c.M * c.N;
  float* d_out;
  CK(cudaMalloc(&d_out, out_elems * 4));
  CK(cudaMemset(d_out, 0xFF, out_elems * 4));
  if constexpr (epi_pair_tiles<Epi>::value) {
    int* d_pairs;
    CK(cudaMalloc(&d_pairs, pairs.size() * sizeof(int)));
    CK(cudaMemcpy(d_pairs, pairs.data(), pairs.size() * sizeof(int), cudaMemcpyHostToDevice));
    g_dev.push_back(d_pairs);
    ep.pairs = d_pairs;
  }
  ep.out = d_out;
  ep.model_stride = (long long)c.M * c.N;
  ep.ld = c.N;
  p.epi = ep;
  p.nsets = c.nsets;
  p.k_total = c.K;
  p.passes = 3;
  p.n_models = tiles_models;
  p.m_total = c.M;
  p.n_total = c.N;
  p.tiles_m = (c.M + kBM - 1) / kBM;
  p.tiles_n = (c.N + kBN - 1) / kBN;
  CK((launch_gemm_clusters<Epi, A_MN, B_MN, SPLIT, ARITH, NATIVE>(p, 0, g_sms, 0, cluster)));
  const cudaError_t err = cudaDeviceSynchronize();
  if (err != cudaSuccess) {
    printf("kernel failed: %s\n", cudaGetErrorString(err));
    exit(3);  // the context is dead after a device fault
  }
  std::vector<float> out(out_elems);
  CK(cudaMemcpy(out.data(), d_out, out_elems * 4, cudaMemcpyDeviceToHost));
  cudaFree(d_out);
  for (void* d : g_dev) cudaFree(d);
  g_dev.clear();
  return out;
}

static double plane_exact(const Operand* A, const Operand* B, int nsets, int am, int bm, int i, int j) {
  double hh = 0, cr = 0;
  for (int s = 0; s < nsets; ++s) {
    const Operand &a = A[s], &b = B[s];
    const int ams = a.models > 1 ? am : 0, bms = b.models > 1 ? bm : 0;
    for (int k = 0; k < a.K; ++k) {
      const size_t ia = a.at(ams, i, k), ib = b.at(bms, j, k);
      if (a.arith == kBf) {
        const double ah = bf16_value(a.p16[ia]), bh = bf16_value(b.p16[ib]);
        hh += ah * bh;
        cr += ah * bf16_value(b.lo16[ib]) + bf16_value(a.lo16[ia]) * bh;
      } else {
        hh += f16_value(a.p16[ia]) * f16_value(b.p16[ib]);
        cr += e5m2_value(a.l8[ia]) * e5m2_value(b.h8[ib]) + e5m2_value(a.h8[ia]) * e5m2_value(b.l8[ib]);
      }
    }
  }
  return A[0].arith == kBf ? hh + cr : hh + cr / double(1 << kLoShift);
}

// every index below n with a step under the tile size, and the last one: each tile of the output is sampled
static std::vector<int> samples(int n, int step) {
  std::vector<int> v;
  for (int i = 0; i < n; i += step) v.push_back(i);
  if (v.back() != n - 1) v.push_back(n - 1);
  return v;
}

template <class Epi, bool A_MN, bool B_MN, bool SPLIT, int ARITH, bool NATIVE>
static bool run_case(const char* config, const Case& c) {
  Operand A[2], B[2];
  const float sa = ARITH == kF8 ? 3.0f : 1.0f, sb = ARITH == kF8 ? 0.25f : 1.0f;
  for (int s = 0; s < c.nsets; ++s) {
    A[s] = make_operand(ARITH, c.a_shared ? 1 : c.models, c.M, c.K, sa);
    B[s] = make_operand(ARITH, c.models, c.N, c.K, sb);
  }
  std::vector<int> pairs;   // pair q: (q % models, (q * 3 + 1) % models): repeated and swapped models
  for (int q = 0; q < c.pairs; ++q) pairs.push_back(q % c.models), pairs.push_back((q * 3 + 1) % c.models);
  const int tiles_n = (c.N + kBN - 1) / kBN;
  const int tiles = (c.pairs ? c.pairs : c.models) * ((c.M + kBM - 1) / kBM) * tiles_n;
  std::vector<int> sizes = {1, 1};
  if (tiles_n % 2 == 0 && (ARITH != kF8 || NATIVE)) sizes.push_back(2), sizes.push_back(2);   // whatever launch_gemm would pick for the K loop
  const std::vector<float> first = run_gemm<Epi, A_MN, B_MN, SPLIT, ARITH, NATIVE>(c, A, B, pairs, sizes[0]);
  long long differ = 0, unwritten = 0, bad = 0;
  for (size_t r = 1; r < sizes.size(); ++r) {
    const std::vector<float> again = run_gemm<Epi, A_MN, B_MN, SPLIT, ARITH, NATIVE>(c, A, B, pairs, sizes[r]);
    differ += memcmp(again.data(), first.data(), first.size() * 4) != 0;
  }
  for (float v : first) unwritten += !(v == v);
  const double bound = (ARITH == kBf ? 1e-3 : 1e-4) * sqrt((double)c.K * c.nsets);
  double max_err = 0;
  const std::vector<int> rows = samples(c.M, 37), cols = samples(c.N, 29);
  for (int q = 0; q < (c.pairs ? c.pairs : c.models); ++q) {
    const int am = c.pairs ? pairs[2 * q] : q, bm = c.pairs ? pairs[2 * q + 1] : q;
    for (int i : rows)
      for (int j : cols) {
        double e = fabs(first[((size_t)q * c.M + i) * c.N + j] - plane_exact(A, B, c.nsets, am, bm, i, j));
        if (!(e == e)) e = 1e30;
        max_err = fmax(max_err, e);
        bad += e > bound;
      }
  }
  const bool ok = differ == 0 && unwritten == 0 && bad == 0;
  printf("[%s/%s] %s  models=%d%s M=%d N=%d K=%d sets=%d tiles=%d (%d SMs) cluster sizes %s  runs differing from the "
         "first %lld, unwritten %lld, max|err| vs plane-exact %.3e (bound %.3e)\n",
         config, c.name, ok ? "PASS" : "FAIL", c.models, c.pairs ? " (pairs)" : "", c.M, c.N, c.K, c.nsets, tiles, g_sms,
         sizes.size() > 2 ? "1, 1, 2, 2" : "1, 1", differ, unwritten, max_err, bound);
  return ok;
}

int main() {
  setvbuf(stdout, nullptr, _IOLBF, 0);
  cudaDeviceProp prop;
  CK(cudaGetDeviceProperties(&prop, 0));
  g_sms = prop.multiProcessorCount;
  printf("device: %s  sm_%d%d  SMs=%d\n", prop.name, prop.major, prop.minor, g_sms);
  // tile counts of one model with two column tiles just below and above twice the SM count
  const int below = (2 * g_sms - 2) / 2 * kBM, above = (2 * g_sms + 2) / 2 * kBM;
  const Case common[] = {
      {"even", 2, 256, 512, 192, 1},            // 4 column tiles: clusters of two
      {"odd", 2, 256, 384, 192, 1},             // 3 column tiles: clusters of one
      {"ragged_even", 3, 200, 456, 136, 1},     // rows 192..255 of the second tile row lie wholly past M
      {"ragged_odd", 3, 100, 328, 136, 1},      // one tile row, its second half wholly past M
      {"below_2sms", 1, below, 256, 64, 1},
      {"above_2sms", 1, above, 256, 64, 1},
  };
  const Case two_sets[] = {
      {"2set_even", 2, 200, 512, 320, 2},
      {"2set_odd", 2, 256, 328, 320, 2},
  };
  bool ok = true;
  for (const Case& c : common) {
    ok &= run_case<EpiStoreF32, false, false, false, kBf, false>("bf16x3 kk", c);
    ok &= run_case<EpiStoreF32, false, true, false, kBf, false>("bf16x3 kmn", c);
    ok &= run_case<EpiStoreF32, false, true, true, kBf, false>("bf16x3 kmn split", c);
    ok &= run_case<EpiStoreF32, false, false, false, kF8, true>("f16f8 kk native", c);
  }
  {
    Case shared = common[0];
    shared.name = "shared_a";
    shared.a_shared = true;
    ok &= run_case<EpiStoreF32, false, false, false, kF8, true>("f16f8 kk native", shared);
  }
  for (const Case& c : two_sets) {
    ok &= run_case<EpiStoreF32, true, true, true, kBf, false>("bf16x3 mnmn split", c);
    ok &= run_case<EpiStoreF32, true, true, false, kF8, true>("f16f8 mnmn native", c);
    ok &= run_case<EpiStoreF32, true, true, false, kF8, false>("f16f8 mnmn widened", c);
  }
  // kPairTiles: 7 pairs over 3 models, even and odd column-tile counts
  const Case pair_cases[] = {{"pairs_even", 3, 200, 512, 192, 1, false, 7}, {"pairs_odd", 3, 200, 328, 192, 1, false, 7}};
  for (const Case& c : pair_cases) {
    ok &= run_case<EpiPairStore, false, false, false, kBf, false>("bf16x3 kk", c);
    ok &= run_case<EpiPairStore, false, false, false, kF8, true>("f16f8 kk native", c);
  }
  printf(ok ? "ALL PASS\n" : "SOME FAILED\n");
  return ok ? 0 : 1;
}
