// gemm_selftest.cu — standalone check of the wgmma split-operand GEMM core (sce_gemm.cuh) against
// a double-precision CPU product, for every operand-major / K-block / pass configuration the engine
// instantiates. Build: see Makefile target `selftest` (build() makes it). Runs on one H100 and exits non-zero on
// failure; tests/test_engine_gpu.py::test_gemm_selftest runs the default case list, `--big` / `--f8big` are manual.
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

#define CK(x)                                                                    \
  do {                                                                           \
    cudaError_t e_ = (x);                                                        \
    if (e_ != cudaSuccess) {                                                     \
      printf("CUDA error %s at %s:%d\n", cudaGetErrorString(e_), __FILE__, __LINE__); \
      exit(2);                                                                   \
    }                                                                            \
  } while (0)

static uint32_t rng_state = 12345u;
static float frand() {  // uniform in [-1, 1)
  rng_state = rng_state * 1664525u + 1013904223u;
  return (float)((rng_state >> 8) & 0xFFFFFF) / 8388608.0f - 1.0f;
}

struct Split {
  std::vector<__nv_bfloat16> hi, lo;
  __nv_bfloat16 *d_hi = nullptr, *d_lo = nullptr;
};

static void split_upload(const std::vector<float>& x, Split& s) {
  s.hi.resize(x.size());
  s.lo.resize(x.size());
  for (size_t i = 0; i < x.size(); ++i) {
    s.hi[i] = __float2bfloat16_rn(x[i]);
    s.lo[i] = __float2bfloat16_rn(x[i] - __bfloat162float(s.hi[i]));
  }
  CK(cudaMalloc(&s.d_hi, x.size() * 2));
  CK(cudaMalloc(&s.d_lo, x.size() * 2));
  CK(cudaMemcpy(s.d_hi, s.hi.data(), x.size() * 2, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(s.d_lo, s.lo.data(), x.size() * 2, cudaMemcpyHostToDevice));
}
static void split_free(Split& s) {
  cudaFree(s.d_hi);
  cudaFree(s.d_lo);
}

// One logical operand: [models][rows][K] if K-major, [models][K][rows] if MN-major.
struct Operand {
  int models, rows, K;
  bool mn;
  std::vector<float> x;
  Split s;
  float at(int m, int r, int k) const {
    return mn ? x[((size_t)m * K + k) * rows + r] : x[((size_t)m * rows + r) * K + k];
  }
  float hi(int m, int r, int k) const {
    size_t i = mn ? ((size_t)m * K + k) * rows + r : ((size_t)m * rows + r) * K + k;
    return __bfloat162float(s.hi[i]);
  }
  float lo(int m, int r, int k) const {
    size_t i = mn ? ((size_t)m * K + k) * rows + r : ((size_t)m * rows + r) * K + k;
    return __bfloat162float(s.lo[i]);
  }
};

static void make_operand(Operand& o, int models, int rows, int K, bool mn) {
  o.models = models;
  o.rows = rows;
  o.K = K;
  o.mn = mn;
  o.x.resize((size_t)models * rows * K);
  for (auto& v : o.x) v = frand();
  split_upload(o.x, o.s);
}

static bool tmaps(const Operand& o, uint32_t box_rows_kmajor, int BK, CUtensorMap* hi,
                  CUtensorMap* lo) {
  if (!o.mn) {
    const CUtensorMapSwizzle sw = BK == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B;
    return make_tmap_bf16_box(hi, o.s.d_hi, o.models, o.rows, o.K, o.K, (uint64_t)o.rows * o.K, BK,
                              box_rows_kmajor, sw) &&
           make_tmap_bf16_box(lo, o.s.d_lo, o.models, o.rows, o.K, o.K, (uint64_t)o.rows * o.K, BK,
                              box_rows_kmajor, sw);
  }
  return make_tmap_bf16(hi, o.s.d_hi, o.models, o.K, o.rows, o.rows, (uint64_t)o.rows * o.K, BK) &&
         make_tmap_bf16(lo, o.s.d_lo, o.models, o.K, o.rows, o.rows, (uint64_t)o.rows * o.K, BK);
}

template <int BK, bool A_MN, bool B_MN, bool SPLIT = false>
static bool run_case(const char* name, int models, int M, int N, int K, int nsets, int passes,
                     bool a_shared, bool b_shared, int reps = 1) {
  Operand A[2], B[2];
  for (int s = 0; s < nsets; ++s) {
    make_operand(A[s], a_shared ? 1 : models, M, K, A_MN);
    make_operand(B[s], b_shared ? 1 : models, N, K, B_MN);
  }
  float* d_out;
  size_t out_elems = (size_t)models * M * N;
  CK(cudaMalloc(&d_out, out_elems * 4));
  CK(cudaMemset(d_out, 0xFF, out_elems * 4));  // NaN pattern: unwritten outputs are caught

  GemmParams<EpiStoreF32::Params> p;
  memset(&p, 0, sizeof(p));
  for (int s = 0; s < nsets; ++s) {
    if (!tmaps(A[s], kBM, BK, &p.a_hi[s], &p.a_lo[s]) ||
        !tmaps(B[s], kBN, BK, &p.b_hi[s], &p.b_lo[s])) {
      printf("[%s] tensor map encode failed\n", name);
      return false;
    }
    p.a_batched[s] = a_shared ? 0 : 1;
    p.b_batched[s] = b_shared ? 0 : 1;
  }
  p.nsets = nsets;
  p.k_total = K;
  p.passes = passes;
  p.n_models = models;
  p.m_total = M;
  p.n_total = N;
  p.tiles_m = (M + kBM - 1) / kBM;
  p.tiles_n = (N + kBN - 1) / kBN;
  p.epi.out = d_out;
  p.epi.model_stride = (long long)M * N;
  p.epi.ld = N;

  constexpr int STAGES = gemm_stages<BK, 0, kArithBf16x3>();
  using SM = GemmSmem<BK, STAGES, 0, kArithBf16x3>;
  auto kern = gemm_split_kernel<EpiStoreF32, BK, A_MN, B_MN, STAGES, SPLIT>;
  CK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SM::kBytes));
  int sms = 0;
  CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0));
  int tiles = models * p.tiles_m * p.tiles_n;
  int grid = tiles < sms ? tiles : sms;
  cudaEvent_t e0, e1;
  CK(cudaEventCreate(&e0));
  CK(cudaEventCreate(&e1));
  for (int rep = 0; rep < reps + (reps > 1 ? 2 : 0); ++rep) {
    if (rep == (reps > 1 ? 2 : 0)) CK(cudaEventRecord(e0));
    kern<<<grid, kGemmThreads, SM::kBytes>>>(p);
    CK(cudaGetLastError());
  }
  CK(cudaEventRecord(e1));
  cudaError_t err = cudaDeviceSynchronize();
  if (err != cudaSuccess) {
    printf("[%s] kernel failed: %s\n", name, cudaGetErrorString(err));
    exit(3);  // context is dead after a device fault
  }
  float ms = 0;
  CK(cudaEventElapsedTime(&ms, e0, e1));
  ms /= reps;

  std::vector<float> out(out_elems);
  CK(cudaMemcpy(out.data(), d_out, out_elems * 4, cudaMemcpyDeviceToHost));

  // Reference in double. `exact` uses the same (hi, lo) decomposition the device used so the only
  // differences are fp32 accumulation order; `full` is the true fp32-input product.
  double max_err_exact = 0, max_err_full = 0, max_ref = 0;
  long long bad = 0;
  int first_bad[3] = {-1, -1, -1};
  // sample rows/cols to keep the CPU check fast for big cases
  int rstep = M > 512 ? 37 : 1, cstep = N > 512 ? 29 : 1;
  for (int m = 0; m < models; ++m)
    for (int i = 0; i < M; i += rstep)
      for (int j = 0; j < N; j += cstep) {
        double ex = 0, fu = 0;
        for (int s = 0; s < nsets; ++s) {
          const int am = a_shared ? 0 : m, bm = b_shared ? 0 : m;
          for (int k = 0; k < K; ++k) {
            double ah = A[s].hi(am, i, k), al = A[s].lo(am, i, k);
            double bh = B[s].hi(bm, j, k), bl = B[s].lo(bm, j, k);
            ex += passes >= 3 ? (ah * bh + ah * bl + al * bh) : ah * bh;
            fu += (double)A[s].at(am, i, k) * (double)B[s].at(bm, j, k);
          }
        }
        double got = out[((size_t)m * M + i) * N + j];
        double ee = fabs(got - ex), ef = fabs(got - fu);
        if (!(ee == ee)) ee = 1e30;  // NaN
        if (ee > max_err_exact) max_err_exact = ee;
        if (ef == ef && ef > max_err_full) max_err_full = ef;
        if (fabs(ex) > max_ref) max_ref = fabs(ex);
        if (ee > 1e-3 * sqrt((double)K * nsets)) {
          if (!bad) {
            first_bad[0] = m;
            first_bad[1] = i;
            first_bad[2] = j;
          }
          ++bad;
        }
      }
  double flops = 2.0 * models * M * N * (double)K * nsets * (passes >= 3 ? 3 : 1);
  bool ok = bad == 0;
  printf("[%s] %s  models=%d M=%d N=%d K=%d sets=%d passes=%d  max|err| vs split-exact %.3e, vs fp32 "
         "product %.3e (max|ref| %.2f)  %.3f ms  %.1f TF(bf16-pass)\n",
         name, ok ? "PASS" : "FAIL", models, M, N, K, nsets, passes, max_err_exact, max_err_full,
         max_ref, ms, flops / ms * 1e-9);
  if (!ok) {
    printf("    %lld bad samples; first at model %d row %d col %d: got %.6f\n", bad, first_bad[0],
           first_bad[1], first_bad[2],
           out[((size_t)first_bad[0] * M + first_bad[1]) * N + first_bad[2]]);
    // error map by 8-row / 64-col blocks of model 0 to expose layout mistakes
    int m = first_bad[0];
    for (int i = 0; i < (M < 32 ? M : 32); i += 4) {
      printf("    row %3d:", i);
      for (int j = 0; j < (N < 256 ? N : 256); j += 16) {
        double ex = 0;
        for (int s = 0; s < nsets; ++s)
          for (int k = 0; k < K; ++k) {
            const int am = a_shared ? 0 : m, bm = b_shared ? 0 : m;
            double ah = A[s].hi(am, i, k), al = A[s].lo(am, i, k);
            double bh = B[s].hi(bm, j, k), bl = B[s].lo(bm, j, k);
            ex += passes >= 3 ? (ah * bh + ah * bl + al * bh) : ah * bh;
          }
        double got = out[((size_t)m * M + i) * N + j];
        printf(" %c", fabs(got - ex) < 1e-3 * sqrt((double)K * nsets) ? '.' : 'X');
      }
      printf("\n");
    }
  }
  for (int s = 0; s < nsets; ++s) {
    split_free(A[s].s);
    split_free(B[s].s);
  }
  cudaFree(d_out);
  return ok;
}

// ------------------------------------------------------------------------------------------------
// f16f8 arithmetic: fp16 plane + two e5m2 planes (value, scaled residual); see sce_ptx.cuh
// ------------------------------------------------------------------------------------------------
static float e5m2_to_float(uint8_t v) {
  __half_raw hr = __nv_cvt_fp8_to_halfraw(v, __NV_E5M2);
  return __half2float(__half(hr));
}
struct OperandF8 {
  int models, rows, K;
  bool mn;
  std::vector<float> x;
  std::vector<__half> h;
  std::vector<uint8_t> h8, l8;
  __half* d_h = nullptr;
  uint8_t *d_h8 = nullptr, *d_l8 = nullptr;
  int pitch;  // elements between consecutive rows (K-major) / k (MN-major): multiple of 16, TMA strides are 16-byte units
  size_t idx(int m, int r, int k) const { return mn ? ((size_t)m * K + k) * pitch + r : ((size_t)m * rows + r) * pitch + k; }
};
static void make_operand_f8(OperandF8& o, int models, int rows, int K, bool mn, float scale, bool fp16_exact = false) {
  o.models = models; o.rows = rows; o.K = K; o.mn = mn;
  o.pitch = ((mn ? rows : K) + 15) / 16 * 16;
  size_t n = (size_t)models * (mn ? K : rows) * o.pitch;
  o.x.resize(n); o.h.resize(n); o.h8.resize(n); o.l8.resize(n);
  for (size_t i = 0; i < n; ++i) {
    float v = frand() * scale;
    if (fp16_exact) v = __half2float(__float2half_rn(v));   // all-zero residual plane
    o.x[i] = v;
    o.h[i] = __float2half_rn(v);
    o.h8[i] = __nv_cvt_float_to_fp8(v, __NV_SATFINITE, __NV_E5M2);
    o.l8[i] = __nv_cvt_float_to_fp8((v - __half2float(o.h[i])) * float(1 << kLoShift), __NV_SATFINITE, __NV_E5M2);
  }
  CK(cudaMalloc(&o.d_h, n * 2)); CK(cudaMalloc(&o.d_h8, n)); CK(cudaMalloc(&o.d_l8, n));
  CK(cudaMemcpy(o.d_h, o.h.data(), n * 2, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(o.d_h8, o.h8.data(), n, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(o.d_l8, o.l8.data(), n, cudaMemcpyHostToDevice));
}
// 16-bit plane: 128-byte swizzle (K block 64); 8-bit planes unswizzled (the GEMM widens them to fp16)
static bool tmaps_f8(const OperandF8& o, uint32_t box_rows_kmajor, int BK, CUtensorMap* h, CUtensorMap* h8, CUtensorMap* l8) {
  const uint64_t mp = (uint64_t)(o.mn ? o.K : o.rows) * o.pitch;
  const CUtensorMapSwizzle sw8 = CU_TENSOR_MAP_SWIZZLE_NONE;
  if (!o.mn) {
    return make_tmap_bf16_box(h, o.d_h, o.models, o.rows, o.K, o.pitch, mp, BK, box_rows_kmajor, CU_TENSOR_MAP_SWIZZLE_128B) &&
           make_tmap_u8_box(h8, o.d_h8, o.models, o.rows, o.K, o.pitch, mp, BK, box_rows_kmajor, sw8) &&
           make_tmap_u8_box(l8, o.d_l8, o.models, o.rows, o.K, o.pitch, mp, BK, box_rows_kmajor, sw8);
  }
  return make_tmap_bf16(h, o.d_h, o.models, o.K, o.rows, o.pitch, mp, BK) &&
         make_tmap_u8_box(h8, o.d_h8, o.models, o.K, o.rows, o.pitch, mp, 128, BK, sw8) &&
         make_tmap_u8_box(l8, o.d_l8, o.models, o.K, o.rows, o.pitch, mp, 128, BK, sw8);
}

template <bool A_MN, bool B_MN>
static bool run_case_f8(const char* name, int models, int M, int N, int K, int nsets, int passes, bool a_shared,
                        bool b_shared, int reps = 1, int exact = 0 /*1: A of set 0, 2: B of set 0 is fp16-exact + flagged*/) {
  constexpr int BK = 64;
  OperandF8 A[2], B[2];
  for (int s = 0; s < nsets; ++s) {
    make_operand_f8(A[s], a_shared ? 1 : models, M, K, A_MN, 3.0f, s == 0 && exact == 1);
    make_operand_f8(B[s], b_shared ? 1 : models, N, K, B_MN, 0.25f, s == 0 && exact == 2);
  }
  uint32_t* d_flag = nullptr;   // "residual plane is all zeros" flag (GemmParams::a_res_flag / b_res_flag), value 0
  CK(cudaMalloc(&d_flag, 4));
  CK(cudaMemset(d_flag, 0, 4));
  float* d_out;
  size_t out_elems = (size_t)models * M * N;
  CK(cudaMalloc(&d_out, out_elems * 4));
  CK(cudaMemset(d_out, 0xFF, out_elems * 4));
  GemmParams<EpiStoreF32::Params> p;
  memset(&p, 0, sizeof(p));
  for (int s = 0; s < nsets; ++s) {
    if (!tmaps_f8(A[s], kBM, BK, &p.a_hi[s], &p.a_lo[s], &p.a_x8[s]) ||
        !tmaps_f8(B[s], kBN, BK, &p.b_hi[s], &p.b_lo[s], &p.b_x8[s])) {
      printf("[%s] tensor map encode failed\n", name);
      return false;
    }
    p.a_batched[s] = a_shared ? 0 : 1;
    p.b_batched[s] = b_shared ? 0 : 1;
  }
  if (exact == 1) p.a_res_flag[0] = d_flag;
  if (exact == 2) p.b_res_flag[0] = d_flag;
  p.nsets = nsets; p.k_total = K; p.passes = passes; p.n_models = models; p.m_total = M; p.n_total = N;
  p.tiles_m = (M + kBM - 1) / kBM;
  p.tiles_n = (N + kBN - 1) / kBN;
  p.epi.out = d_out; p.epi.model_stride = (long long)M * N; p.epi.ld = N;
  constexpr int STAGES = gemm_stages<BK, 0, kArithF16F8>();
  using SM = GemmSmem<BK, STAGES, 0, kArithF16F8>;
  auto kern = gemm_split_kernel<EpiStoreF32, BK, A_MN, B_MN, STAGES, false, kArithF16F8>;
  CK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SM::kBytes));
  int sms = 0;
  CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0));
  int tiles = models * p.tiles_m * p.tiles_n;
  int grid = tiles < sms ? tiles : sms;
  cudaEvent_t e0, e1;
  CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
  float ms = 0;
  for (int rep = 0; rep < reps + (reps > 1 ? 2 : 0); ++rep) {
    if (rep == (reps > 1 ? 2 : 0)) CK(cudaEventRecord(e0));
    kern<<<grid, kGemmThreads, SM::kBytes>>>(p);
    CK(cudaGetLastError());
  }
  CK(cudaEventRecord(e1));
  cudaError_t err = cudaDeviceSynchronize();
  if (err != cudaSuccess) {
    printf("[%s] kernel failed: %s\n", name, cudaGetErrorString(err));
    exit(3);
  }
  CK(cudaEventElapsedTime(&ms, e0, e1));
  ms /= reps;
  std::vector<float> out(out_elems);
  CK(cudaMemcpy(out.data(), d_out, out_elems * 4, cudaMemcpyDeviceToHost));
  double max_err_exact = 0, max_ref = 0, se_full = 0, s_full = 0;
  long long bad = 0;
  int fb[3] = {-1, -1, -1};
  int rstep = M > 512 ? 37 : 1, cstep = N > 512 ? 29 : 1;
  const double inv = 1.0 / double(1 << kLoShift);
  for (int m = 0; m < models; ++m)
    for (int i = 0; i < M; i += rstep)
      for (int j = 0; j < N; j += cstep) {
        double hh = 0, cr = 0, fu = 0;
        for (int s = 0; s < nsets; ++s) {
          const int am = a_shared ? 0 : m, bm = b_shared ? 0 : m;
          for (int k = 0; k < K; ++k) {
            size_t ia = A[s].idx(am, i, k), ib = B[s].idx(bm, j, k);
            hh += (double)__half2float(A[s].h[ia]) * (double)__half2float(B[s].h[ib]);
            cr += (double)e5m2_to_float(A[s].l8[ia]) * e5m2_to_float(B[s].h8[ib]) +
                  (double)e5m2_to_float(A[s].h8[ia]) * e5m2_to_float(B[s].l8[ib]);
            fu += (double)A[s].x[ia] * (double)B[s].x[ib];
          }
        }
        double ex = passes >= 3 ? hh + cr * inv : hh;
        double got = out[((size_t)m * M + i) * N + j];
        double ee = fabs(got - ex);
        if (!(ee == ee)) ee = 1e30;
        if (ee > max_err_exact) max_err_exact = ee;
        if (got == got) { se_full += (got - fu) * (got - fu); s_full += fu * fu; }
        if (fabs(ex) > max_ref) max_ref = fabs(ex);
        if (ee > 1e-4 * sqrt((double)K * nsets)) {
          if (!bad) { fb[0] = m; fb[1] = i; fb[2] = j; }
          ++bad;
        }
      }
  double flops = 2.0 * models * M * N * (double)K * nsets;
  bool ok = bad == 0;
  fflush(stdout);
  printf("[%s] %s  models=%d M=%d N=%d K=%d sets=%d passes=%d  max|err| vs plane-exact %.3e (max|ref| %.2f), rel. rms "
         "vs fp32 product %.2e  %.3f ms  %.1f TF algorithmic\n",
         name, ok ? "PASS" : "FAIL", models, M, N, K, nsets, passes, max_err_exact, max_ref,
         sqrt(se_full / (s_full + 1e-300)), ms, flops / ms * 1e-9);
  if (!ok) {
    printf("    %lld bad samples; first at model %d row %d col %d: got %.6f\n", bad, fb[0], fb[1], fb[2],
           out[((size_t)fb[0] * M + fb[1]) * N + fb[2]]);
  }
  for (int s = 0; s < nsets; ++s) {
    cudaFree(A[s].d_h); cudaFree(A[s].d_h8); cudaFree(A[s].d_l8);
    cudaFree(B[s].d_h); cudaFree(B[s].d_h8); cudaFree(B[s].d_l8);
  }
  cudaFree(d_out);
  cudaFree(d_flag);
  return ok;
}

int main(int argc, char** argv) {
  bool big = argc > 1 && !strcmp(argv[1], "--big");
  bool f8only = argc > 1 && !strcmp(argv[1], "--f8");
  bool f8big = argc > 1 && !strcmp(argv[1], "--f8big");
  setvbuf(stdout, nullptr, _IOLBF, 0);
  int dev = 0;
  cudaDeviceProp prop;
  CK(cudaGetDeviceProperties(&prop, dev));
  printf("device: %s  sm_%d%d  SMs=%d\n", prop.name, prop.major, prop.minor,
         prop.multiProcessorCount);
  bool ok = true;
  if (f8only || f8big || argc == 1) {
    // ---- f16f8 arithmetic: each operand-major combination the engine uses
    if (!f8big) {
    ok &= run_case_f8<false, false>("f8_kk_hh", 1, 128, 256, 64, 1, 1, false, false);
    ok &= run_case_f8<false, false>("f8_kk_k64", 1, 128, 256, 64, 1, 3, false, false);
    ok &= run_case_f8<false, false>("f8_kk_multi", 3, 384, 512, 512, 1, 3, true, false);
    ok &= run_case_f8<false, true>("f8_kmn_k64", 1, 128, 256, 64, 1, 3, false, false);
    ok &= run_case_f8<false, true>("f8_kmn_multi", 2, 256, 512, 512, 1, 3, false, false);
    ok &= run_case_f8<true, true>("f8_mnmn_k64", 1, 128, 256, 64, 1, 3, false, false);
    ok &= run_case_f8<true, true>("f8_mnmn_2set", 2, 256, 512, 320, 2, 3, false, true);
    ok &= run_case_f8<false, false>("f8_kk_ragged", 2, 200, 328, 104, 1, 3, true, false);
    ok &= run_case_f8<false, true>("f8_kmn", 2, 512, 512, 512, 1, 3, false, false);
    ok &= run_case_f8<false, true>("f8_kmn_ragged", 2, 200, 328, 104, 1, 3, false, false);
    ok &= run_case_f8<true, true>("f8_mnmn_ragged", 2, 200, 328, 104, 2, 3, false, true);
    // fp16-exact operand flagged "no residual plane": the cross term and the loads of its planes are skipped
    ok &= run_case_f8<false, false>("f8_kk_exactA", 3, 768, 512, 512, 1, 3, true, false, 1, 1);
    ok &= run_case_f8<true, true>("f8_mnmn_exactB", 2, 512, 512, 320, 2, 3, false, true, 1, 2);
    }
    if (f8big) {
      // same-GPU comparison with the bf16x3 configuration the engine uses (K block 32, 3 passes) at config-2 shapes
      ok &= run_case<32, false, false>("bf_big_encode", 4, 8192, 4096, 512, 1, 3, true, false, 10);
      ok &= run_case<32, false, true>("bf_big_decode", 4, 8192, 512, 4096, 1, 3, false, false, 10);
      ok &= run_case<32, true, true, true>("bf_big_dw", 4, 4096, 512, 8192, 2, 3, false, true, 10);
      ok &= run_case_f8<false, false>("f8_big_encode", 4, 8192, 4096, 512, 1, 3, true, false, 10);
      ok &= run_case_f8<false, true>("f8_big_decode", 4, 8192, 512, 4096, 1, 3, false, false, 10);
      ok &= run_case_f8<true, true>("f8_big_dw", 4, 4096, 512, 8192, 2, 3, false, true, 10);
      ok &= run_case_f8<false, false>("f8_big_enc_hh", 4, 8192, 4096, 512, 1, 1, true, false, 10);
      ok &= run_case_f8<false, false>("f8_big_encode_exactA", 4, 8192, 4096, 512, 1, 3, true, false, 10, 1);
      ok &= run_case_f8<true, true>("f8_big_dw_exactB", 4, 4096, 512, 8192, 2, 3, false, true, 10, 2);
    }
    if (f8only || f8big) {
      printf(ok ? "ALL PASS\n" : "SOME FAILED\n");
      return ok ? 0 : 1;
    }
  }
  // ---- K-major x K-major (encode / dC shape), increasing complexity
  ok &= run_case<64, false, false>("kk_k16", 1, 128, 256, 16, 1, 1, false, false);
  ok &= run_case<64, false, false>("kk_k64", 1, 128, 256, 64, 1, 1, false, false);
  ok &= run_case<64, false, false>("kk_k256", 1, 128, 256, 256, 1, 1, false, false);
  ok &= run_case<64, false, false>("kk_3pass", 1, 128, 256, 256, 1, 3, false, false);
  ok &= run_case<64, false, false>("kk_multi", 3, 384, 512, 512, 1, 3, true, false);
  ok &= run_case<64, false, false>("kk_ragged", 2, 200, 328, 104, 1, 3, true, false);
  ok &= run_case<64, false, false>("kk_bn128", 2, 256, 384, 256, 1, 3, true, false);
  // ---- K-major operands with the 64-byte swizzle (BK = 32, four stages)
  ok &= run_case<32, false, false>("kk32_k16", 1, 128, 256, 16, 1, 1, false, false);
  ok &= run_case<32, false, false>("kk32_k64", 1, 128, 256, 64, 1, 1, false, false);
  ok &= run_case<32, false, false>("kk32_multi", 3, 384, 512, 512, 1, 3, true, false);
  ok &= run_case<32, false, false>("kk32_ragged", 2, 200, 328, 104, 1, 3, true, false);
  ok &= run_case<32, false, false>("kk32_bn128", 2, 256, 384, 256, 1, 3, true, false);
  ok &= run_case<32, false, true>("kmn32_3pass", 2, 256, 512, 512, 1, 3, false, false);
  ok &= run_case<32, false, true>("kmn32_ragged", 2, 200, 328, 104, 1, 3, false, false);
  // ---- longer row counts, split accumulators
  ok &= run_case<64, false, false>("kk_short", 2, 100, 328, 104, 1, 3, true, false);
  ok &= run_case<32, false, true, true>("kmn_split", 2, 512, 512, 512, 1, 3, false, false);
  ok &= run_case<32, false, true, true>("kmn_ragged", 2, 200, 328, 104, 1, 3, false, false);
  ok &= run_case<32, true, true, true>("mnmn_2set", 2, 512, 512, 320, 2, 3, false, true);
  ok &= run_case<32, true, true, true>("mnmn_ragged", 2, 200, 328, 104, 2, 3, false, true);
  // ---- K-major A x MN-major B (decode shape: X^ = C W)
  ok &= run_case<64, false, true>("kmn_k16", 1, 128, 256, 16, 1, 1, false, false);
  ok &= run_case<64, false, true>("kmn_k64", 1, 128, 256, 64, 1, 1, false, false);
  ok &= run_case<64, false, true>("kmn_3pass", 2, 256, 512, 512, 1, 3, false, false);
  // ---- MN-major x MN-major (weight-gradient shape: dW = dZ^T X + C^T G), two operand sets
  ok &= run_case<64, true, true>("mnmn_k16", 1, 128, 256, 16, 1, 1, false, false);
  ok &= run_case<64, true, true>("mnmn_k64", 1, 128, 256, 64, 1, 1, false, false);
  ok &= run_case<32, true, true>("mnmn_bk32", 2, 256, 512, 320, 2, 3, false, true);
  if (big) {
    // config-2 shapes, one model's worth of each GEMM, for a first throughput reading
    ok &= run_case<64, false, false>("big_encode", 4, 8192, 4096, 512, 1, 3, true, false);
    ok &= run_case<64, false, true>("big_decode", 4, 8192, 512, 4096, 1, 3, false, false);
    ok &= run_case<32, true, true>("big_dw", 4, 4096, 512, 8192, 2, 3, false, true);
    ok &= run_case<64, true, true>("big_dw64", 4, 4096, 512, 8192, 2, 3, false, true);
    ok &= run_case<64, false, false>("big_enc1p", 4, 8192, 4096, 512, 1, 1, true, false);
    ok &= run_case<32, false, false>("big_encode32", 4, 8192, 4096, 512, 1, 3, true, false);
    ok &= run_case<32, false, true>("big_decode32", 4, 8192, 512, 4096, 1, 3, false, false);
  }
  printf(ok ? "ALL PASS\n" : "SOME FAILED\n");
  return ok ? 0 : 1;
}
