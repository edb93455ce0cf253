// native_dw_selftest.cu — the f16f8 weight-gradient GEMM with mixed operand layouts (sce_gemm.cuh, F8_NATIVE with
// A_MN = B_MN = true): fp16 planes MN-major, as the batch holds them ([K][rows], K = batch), and the 8-bit planes K-major
// from batch-major copies ([rows][Kp], Kp = K rounded up to 16, only K columns exposed so the tail reads as zero), cross
// terms on E5M2 wgmma. Two operand sets, as in dW = dz^T x + c^T g; set 0's B is fp16-exact and flagged so (the x of
// fp16 activations), so its A.h8 x B.l8 term is skipped — A's value plane of set 0 is filled with E5M2 NaNs to show
// that it is not read (the engine does not write it then). M and N are not multiples of 128, K is 8192 and ragged 8155.
// Each case is checked against the fp64 value of the same planes (the bound of gemm_selftest) and against the widened
// instantiation (8-bit planes MN-major, widened to fp16 in shared memory) on the same data.
// Prints one line per case and exits non-zero when a case fails; tests/test_native_dw_gpu.py runs it.
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

static uint32_t rng_state = 7u;
static float frand() {  // uniform in [-1, 1)
  rng_state = rng_state * 1664525u + 1013904223u;
  return (float)((rng_state >> 8) & 0xFFFFFF) / 8388608.0f - 1.0f;
}
static double e5m2_value(uint8_t v) {
  __half_raw hr = __nv_cvt_fp8_to_halfraw(v, __NV_E5M2);
  return (double)__half2float(__half(hr));
}

constexpr uint8_t kE5m2NaN = 0x7F;

// one operand in the batch layout [models][K][rows] (rows % 16 == 0) plus batch-major copies of its 8-bit planes
struct Operand {
  int models, rows, K, Kp;
  std::vector<__half> h;
  std::vector<uint8_t> h8, l8;       // [models][K][rows]
  std::vector<uint8_t> h8t, l8t;     // [models][rows][Kp]
  __half* d_h = nullptr;
  uint8_t *d_h8 = nullptr, *d_l8 = nullptr, *d_h8t = nullptr, *d_l8t = nullptr;
  size_t idx(int m, int r, int k) const { return ((size_t)m * K + k) * rows + r; }
};
static void make_operand(Operand& o, int models, int rows, int K, float scale, bool fp16_exact, bool poison_h8) {
  o.models = models; o.rows = rows; o.K = K; o.Kp = (K + 15) / 16 * 16;
  const size_t n = (size_t)models * K * rows, nt = (size_t)models * rows * o.Kp;
  o.h.resize(n); o.h8.resize(n); o.l8.resize(n);
  for (size_t i = 0; i < n; ++i) {
    float v = frand() * scale;
    if (fp16_exact) v = __half2float(__float2half_rn(v));   // all-zero residual plane
    o.h[i] = __float2half_rn(v);
    o.h8[i] = poison_h8 ? kE5m2NaN : __nv_cvt_float_to_fp8(v, __NV_SATFINITE, __NV_E5M2);
    o.l8[i] = __nv_cvt_float_to_fp8((v - __half2float(o.h[i])) * float(1 << kLoShift), __NV_SATFINITE, __NV_E5M2);
  }
  // the copies' padding columns K .. Kp - 1 hold NaNs: the tensor map exposes K columns, so they must never be read
  o.h8t.assign(nt, kE5m2NaN);
  o.l8t.assign(nt, kE5m2NaN);
  for (int m = 0; m < models; ++m)
    for (int r = 0; r < rows; ++r)
      for (int k = 0; k < K; ++k) {
        const size_t t = ((size_t)m * rows + r) * o.Kp + k;
        o.h8t[t] = o.h8[o.idx(m, r, k)];
        o.l8t[t] = o.l8[o.idx(m, r, k)];
      }
  CK(cudaMalloc(&o.d_h, n * 2)); CK(cudaMalloc(&o.d_h8, n)); CK(cudaMalloc(&o.d_l8, n));
  CK(cudaMalloc(&o.d_h8t, nt)); CK(cudaMalloc(&o.d_l8t, nt));
  CK(cudaMemcpy(o.d_h, o.h.data(), n * 2, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(o.d_h8, o.h8.data(), n, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(o.d_l8, o.l8.data(), n, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(o.d_h8t, o.h8t.data(), nt, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(o.d_l8t, o.l8t.data(), nt, cudaMemcpyHostToDevice));
}
static void free_operand(Operand& o) {
  cudaFree(o.d_h); cudaFree(o.d_h8); cudaFree(o.d_l8); cudaFree(o.d_h8t); cudaFree(o.d_l8t);
}

// fp16 plane MN-major (boxes of 64 k-rows x 64 elements); 8-bit planes K-major from the copies (NATIVE: [128 rows][64 B],
// 64-byte swizzle) or MN-major and unswizzled (widened: [64 k-rows][128 B])
template <bool NATIVE>
static bool tmaps(const Operand& o, CUtensorMap* h, CUtensorMap* h8, CUtensorMap* l8) {
  constexpr int BK = 64;
  const uint64_t mp = (uint64_t)o.K * o.rows;
  bool ok = make_tmap_bf16(h, o.d_h, o.models, o.K, o.rows, o.rows, mp, BK);
  if (NATIVE) {
    const uint64_t mpt = (uint64_t)o.rows * o.Kp;
    return ok && make_tmap_u8_box(h8, o.d_h8t, o.models, o.rows, o.K, o.Kp, mpt, BK, kBM, CU_TENSOR_MAP_SWIZZLE_64B) &&
           make_tmap_u8_box(l8, o.d_l8t, o.models, o.rows, o.K, o.Kp, mpt, BK, kBM, CU_TENSOR_MAP_SWIZZLE_64B);
  }
  return ok && make_tmap_u8_box(h8, o.d_h8, o.models, o.K, o.rows, o.rows, mp, 128, BK, CU_TENSOR_MAP_SWIZZLE_NONE) &&
         make_tmap_u8_box(l8, o.d_l8, o.models, o.K, o.rows, o.rows, mp, 128, BK, CU_TENSOR_MAP_SWIZZLE_NONE);
}

template <bool NATIVE>
static std::vector<float> run_gemm(const Operand* A, const Operand* B, int nsets, const uint32_t* d_flag, int models,
                                   int M, int N, int K) {
  constexpr int BK = 64;
  GemmParams<EpiStoreF32::Params> p;
  memset(&p, 0, sizeof(p));
  for (int s = 0; s < nsets; ++s) {
    if (!tmaps<NATIVE>(A[s], &p.a_hi[s], &p.a_lo[s], &p.a_x8[s]) || !tmaps<NATIVE>(B[s], &p.b_hi[s], &p.b_lo[s], &p.b_x8[s])) {
      printf("tensor map encode failed\n");
      exit(2);
    }
    p.a_batched[s] = p.b_batched[s] = 1;
  }
  p.b_res_flag[0] = d_flag;   // set 0's B has an all-zero residual plane
  float* d_out;
  const size_t out_elems = (size_t)models * M * N;
  CK(cudaMalloc(&d_out, out_elems * 4));
  CK(cudaMemset(d_out, 0xFF, out_elems * 4));
  p.nsets = nsets; p.k_total = K; p.passes = 3; p.n_models = models; p.m_total = M; p.n_total = N;
  p.tiles_m = (M + kBM - 1) / kBM;
  p.tiles_n = (N + kBN - 1) / kBN;
  p.epi.out = d_out; p.epi.model_stride = (long long)M * N; p.epi.ld = N;
  constexpr int STAGES = gemm_stages<BK, 0, kArithF16F8, NATIVE>();
  using SM = GemmSmem<BK, STAGES, 0, kArithF16F8, NATIVE>;
  auto kern = gemm_split_kernel<EpiStoreF32, BK, true, true, STAGES, false, kArithF16F8, NATIVE>;
  CK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SM::kBytes));
  int sms = 0;
  CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0));
  const int tiles = models * p.tiles_m * p.tiles_n;
  kern<<<tiles < sms ? tiles : sms, kGemmThreads, SM::kBytes>>>(p);
  CK(cudaGetLastError());
  CK(cudaDeviceSynchronize());
  std::vector<float> out(out_elems);
  CK(cudaMemcpy(out.data(), d_out, out_elems * 4, cudaMemcpyDeviceToHost));
  cudaFree(d_out);
  return out;
}

int main() {
  setvbuf(stdout, nullptr, _IOLBF, 0);
  cudaDeviceProp prop;
  CK(cudaGetDeviceProperties(&prop, 0));
  printf("device: %s\n", prop.name);
  const int models = 2, M = 208, N = 336, nsets = 2;
  const double inv = 1.0 / double(1 << kLoShift);
  uint32_t* d_flag = nullptr;
  CK(cudaMalloc(&d_flag, 4));
  CK(cudaMemset(d_flag, 0, 4));
  bool all_ok = true;
  for (int K : {8192, 8155}) {
    Operand A[2], B[2];
    for (int s = 0; s < nsets; ++s) {
      make_operand(A[s], models, M, K, 3.0f, false, s == 0);
      make_operand(B[s], models, N, K, 0.25f, s == 0, false);
    }
    const std::vector<float> nat = run_gemm<true>(A, B, nsets, d_flag, models, M, N, K);
    const std::vector<float> wide = run_gemm<false>(A, B, nsets, d_flag, models, M, N, K);
    double err_n = 0, err_w = 0, err_nw = 0, max_ref = 0;
    long long bad = 0, checked = 0;
    const double bound = 1e-4 * sqrt((double)K * nsets);   // gemm_selftest's bound against the plane-exact value
    for (int m = 0; m < models; ++m)
      for (int i = 0; i < M; i += 3)
        for (int j = 0; j < N; j += 5) {
          double hh = 0, cr = 0;
          for (int s = 0; s < nsets; ++s)
            for (int k = 0; k < K; ++k) {
              const size_t ia = A[s].idx(m, i, k), ib = B[s].idx(m, j, k);
              hh += (double)__half2float(A[s].h[ia]) * (double)__half2float(B[s].h[ib]);
              cr += e5m2_value(A[s].l8[ia]) * e5m2_value(B[s].h8[ib]);
              if (s != 0) cr += e5m2_value(A[s].h8[ia]) * e5m2_value(B[s].l8[ib]);   // (set 0: skipped, B.l8 == 0)
            }
          const double ex = hh + cr * inv;
          const size_t o = ((size_t)m * M + i) * N + j;
          double en = fabs(nat[o] - ex), ew = fabs(wide[o] - ex), enw = fabs((double)nat[o] - (double)wide[o]);
          if (!(en == en)) en = 1e30;
          if (!(ew == ew)) ew = 1e30;
          if (!(enw == enw)) enw = 1e30;
          err_n = fmax(err_n, en);
          err_w = fmax(err_w, ew);
          err_nw = fmax(err_nw, enw);
          max_ref = fmax(max_ref, fabs(ex));
          bad += en > bound || ew > bound || enw > bound;
          ++checked;
        }
    // every output element is written (the rows / columns of the partial tiles are clipped, not dropped)
    long long unwritten = 0;
    for (size_t o = 0; o < nat.size(); ++o) unwritten += !(nat[o] == nat[o]);
    const bool ok = bad == 0 && unwritten == 0;
    all_ok &= ok;
    printf("[K=%d] %s  models=%d M=%d N=%d sets=%d  max|err| vs plane-exact: native %.3e, widened %.3e; "
           "max|native - widened| %.3e; bound %.3e (max|ref| %.2f); %lld samples, %lld NaN outputs\n",
           K, ok ? "PASS" : "FAIL", models, M, N, nsets, err_n, err_w, err_nw, bound, max_ref, checked, unwritten);
    for (int s = 0; s < nsets; ++s) {
      free_operand(A[s]);
      free_operand(B[s]);
    }
  }
  cudaFree(d_flag);
  printf(all_ok ? "ALL PASS\n" : "SOME FAILED\n");
  return all_ok ? 0 : 1;
}
