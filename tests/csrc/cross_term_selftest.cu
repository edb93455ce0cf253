// cross_term_selftest.cu — accuracy of the f16f8 cross-term accumulation in the split-operand GEMM (sce_gemm.cuh).
// The fp16 planes are zero, so the GEMM's output is exactly 2^-kLoShift times the sum of the E5M2 cross products
// A.l8 * B.h8 + A.h8 * B.l8. That sum is formed on E5M2 wgmma from the stage (F8_NATIVE, 64-byte swizzled tiles) or on
// fp16 wgmma after widening (unswizzled tiles), and compared with its fp64 value at several reduction lengths. Every
// product is exact in both paths, so the error measured is the tensor core's accumulation alone. (The native path
// promotes each K block's E5M2 sums into the fp32 accumulator: unpromoted, FP8 wgmma's reduced-precision, truncating
// accumulation drifts with the reduction length.)
// Prints one line per case and exits non-zero when a case exceeds its bound; tests/test_cross_terms_gpu.py runs it.
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

static uint32_t rng_state = 2024u;
static float frand() {  // uniform in [-1, 1)
  rng_state = rng_state * 1664525u + 1013904223u;
  return (float)((rng_state >> 8) & 0xFFFFFF) / 8388608.0f - 1.0f;
}

static double e5m2_value(uint8_t b) {   // an E5M2 byte is the high byte of the fp16 with the same value
  static double table[256];
  static bool filled = false;
  if (!filled) {
    for (int v = 0; v < 256; ++v) {
      __half_raw r;
      r.x = (unsigned short)(v << 8);
      table[v] = (double)__half2float(__half(r));
    }
    filled = true;
  }
  return table[b];
}

struct Operand {   // K-major [rows][K]: zero fp16 plane, random E5M2 value and residual planes
  std::vector<uint8_t> h8, l8;
  uint16_t* d_h = nullptr;
  uint8_t *d_h8 = nullptr, *d_l8 = nullptr;
};
static void make_operand(Operand& o, int rows, int K, bool positive) {
  const size_t n = (size_t)rows * K;
  o.h8.resize(n);
  o.l8.resize(n);
  for (size_t i = 0; i < n; ++i) {
    // value planes of one sign (e.g. codes after the ReLU) or of either sign; residual planes are rounding errors and
    // take either sign
    const float a = positive ? 0.5f * (frand() + 1.0f) : frand(), b = frand();
    o.h8[i] = __nv_cvt_float_to_fp8(a, __NV_SATFINITE, __NV_E5M2);
    o.l8[i] = __nv_cvt_float_to_fp8(b, __NV_SATFINITE, __NV_E5M2);
  }
  CK(cudaMalloc(&o.d_h, n * 2));
  CK(cudaMalloc(&o.d_h8, n));
  CK(cudaMalloc(&o.d_l8, n));
  CK(cudaMemset(o.d_h, 0, n * 2));
  CK(cudaMemcpy(o.d_h8, o.h8.data(), n, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(o.d_l8, o.l8.data(), n, cudaMemcpyHostToDevice));
}
static void free_operand(Operand& o) {
  cudaFree(o.d_h);
  cudaFree(o.d_h8);
  cudaFree(o.d_l8);
}

// the GEMM's output for both operands at reduction length K, with or without the native cross-term path
template <bool NATIVE>
static std::vector<float> run_gemm(const Operand& A, const Operand& B, int M, int N, int K) {
  constexpr int BK = 64;
  const CUtensorMapSwizzle sw8 = NATIVE ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_NONE;
  GemmParams<EpiStoreF32::Params> p;
  memset(&p, 0, sizeof(p));
  bool ok = make_tmap_bf16_box(&p.a_hi[0], A.d_h, 1, M, K, K, (uint64_t)M * K, BK, kBM, CU_TENSOR_MAP_SWIZZLE_128B) &&
            make_tmap_u8_box(&p.a_lo[0], A.d_h8, 1, M, K, K, (uint64_t)M * K, BK, kBM, sw8) &&
            make_tmap_u8_box(&p.a_x8[0], A.d_l8, 1, M, K, K, (uint64_t)M * K, BK, kBM, sw8) &&
            make_tmap_bf16_box(&p.b_hi[0], B.d_h, 1, N, K, K, (uint64_t)N * K, BK, kBN, CU_TENSOR_MAP_SWIZZLE_128B) &&
            make_tmap_u8_box(&p.b_lo[0], B.d_h8, 1, N, K, K, (uint64_t)N * K, BK, kBN, sw8) &&
            make_tmap_u8_box(&p.b_x8[0], B.d_l8, 1, N, K, K, (uint64_t)N * K, BK, kBN, sw8);
  if (!ok) {
    printf("tensor map encode failed\n");
    exit(2);
  }
  float* d_out;
  CK(cudaMalloc(&d_out, (size_t)M * N * 4));
  p.nsets = 1; p.k_total = K; p.passes = 3; p.n_models = 1; p.m_total = M; p.n_total = N;
  p.tiles_m = (M + kBM - 1) / kBM;
  p.tiles_n = (N + kBN - 1) / kBN;
  p.epi.out = d_out; p.epi.model_stride = (long long)M * N; p.epi.ld = N;
  constexpr int STAGES = gemm_stages<BK, 0, kArithF16F8, NATIVE>();
  using SM = GemmSmem<BK, STAGES, 0, kArithF16F8, NATIVE>;
  auto kern = gemm_split_kernel<EpiStoreF32, BK, false, false, STAGES, false, kArithF16F8, NATIVE>;
  CK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SM::kBytes));
  kern<<<p.tiles_m * p.tiles_n, kGemmThreads, SM::kBytes>>>(p);
  CK(cudaGetLastError());
  CK(cudaDeviceSynchronize());
  std::vector<float> out((size_t)M * N);
  CK(cudaMemcpy(out.data(), d_out, out.size() * 4, cudaMemcpyDeviceToHost));
  cudaFree(d_out);
  return out;
}

int main() {
  setvbuf(stdout, nullptr, _IOLBF, 0);
  cudaDeviceProp prop;
  CK(cudaGetDeviceProperties(&prop, 0));
  printf("device: %s\n", prop.name);
  const int M = 128, N = 128;
  const double inv = 1.0 / double(1 << kLoShift);
  bool all_ok = true;
  for (int positive = 0; positive < 2; ++positive)
    for (int K : {512, 4096, 16384}) {
      Operand A, B;
      make_operand(A, M, K, positive);
      make_operand(B, N, K, positive);
      const std::vector<float> wide = run_gemm<false>(A, B, M, N, K), nat = run_gemm<true>(A, B, M, N, K);
      // error of each path over sum_k |products| (the scale of the accumulation's rounding), max over the tile
      double err_w = 0, err_n = 0, bias_n = 0;
      for (int i = 0; i < M; ++i)
        for (int j = 0; j < N; ++j) {
          double s = 0, sa = 0;
          for (int k = 0; k < K; ++k) {
            const size_t ia = (size_t)i * K + k, ib = (size_t)j * K + k;
            const double t1 = e5m2_value(A.l8[ia]) * e5m2_value(B.h8[ib]);
            const double t2 = e5m2_value(A.h8[ia]) * e5m2_value(B.l8[ib]);
            s += t1 + t2;
            sa += fabs(t1) + fabs(t2);
          }
          s *= inv;
          sa *= inv;
          const double ew = (wide[(size_t)i * N + j] - s) / sa, en = (nat[(size_t)i * N + j] - s) / sa;
          err_w = fmax(err_w, fabs(ew));
          err_n = fmax(err_n, fabs(en));
          bias_n += en;
        }
      bias_n /= (double)M * N;
      // bounds: fp32 accumulation (widened) stays near 2^-24 K; the native accumulation is allowed 2^-12 — the
      // cross terms are 2^-11 of a GEMM's result, so that is below 2^-22 of it
      const bool ok = !(err_w > 1e-7 * K) && !(err_n > 1.0 / 4096);
      all_ok &= ok;
      printf("[%s K=%5d] %s  max |err| / sum|products|: widened %.3e, native %.3e (%.1f bits); native mean signed %.3e\n",
             positive ? "h8 >= 0" : "signed", K, ok ? "PASS" : "FAIL", err_w, err_n,
             err_n > 0 ? -log2(err_n) : 99.0, bias_n);
      free_operand(A);
      free_operand(B);
    }
  printf(all_ok ? "ALL PASS\n" : "SOME FAILED\n");
  return all_ok ? 0 : 1;
}
