// gemm_selftest.cu — standalone check of the split-operand GEMM (sce_gemm.cuh) in the seven configurations libsce
// launches, against double-precision products of the same operand planes:
//   bf16x3 (K block 32): K x K; K x MN; K x MN and MN x MN with split accumulators;
//   f16f8 (K block 64): K x K and MN x MN with the cross terms on E5M2 wgmma (MN x MN: 8-bit planes from batch-major
//   copies), and MN x MN with the 8-bit tiles widened to fp16.
// Each configuration has one `_persist` case with more than twice as many output tiles as an H100 has SMs and ragged M,
// N and K, so that every persistent CTA runs a second tile (ring phase carried over, accumulator reset, epilogue staging
// reused) and some a partial one. The default run prints one PASS / FAIL line per case and exits non-zero when one fails
// (tests/test_engine_gpu.py::test_gemm_selftest). `--big` runs each configuration at config-2 shapes instead, for a
// kernel-level throughput reading. Build: Makefile target `selftest`.
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
constexpr uint16_t kBf16NaN = 0x7FC0, kF16NaN = 0x7E00;
constexpr uint8_t kE5m2NaN = 0x7F;

static int g_sms = 0;
static uint32_t* g_zero_flag = nullptr;   // device word 0: "this operand's residual plane is all zeros"
static std::vector<void*> g_dev;          // device buffers of the GEMM being run

static uint32_t rng_state = 12345u;
static float frand() {  // uniform in [-1, 1)
  rng_state = rng_state * 1664525u + 1013904223u;
  return (float)((rng_state >> 8) & 0xFFFFFF) / 8388608.0f - 1.0f;
}

static uint16_t bits(__half h) { return __half_raw(h).x; }
static uint16_t bits(__nv_bfloat16 h) { return __nv_bfloat16_raw(h).x; }
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
static double e5m2_value(uint8_t b) { return f16_value(uint16_t(b << 8)); }   // an E5M2 byte is an fp16's high byte

// One logical operand [models][rows][K] and its planes, in that index order. bf16x3: p16 = bf16(x), lo16 = bf16 of the
// rest. f16f8: p16 = fp16(x), h8 = e5m2(x) (value plane), l8 = e5m2((x - fp16(x)) 2^kLoShift) (residual plane).
struct Operand {
  int arith, models, rows, K;
  bool flagged;                 // f16f8: fp16-exact, flagged "no residual plane" (GemmParams::a_res_flag / b_res_flag)
  std::vector<float> x;         // the fp32 source (empty where the planes are drawn directly)
  std::vector<uint16_t> p16, lo16;
  std::vector<uint8_t> h8, l8;
  size_t at(int m, int r, int k) const { return ((size_t)m * rows + r) * K + k; }
};

// planes of an fp32 source uniform in [-scale, scale). `exact`: the source is rounded to fp16 (all-zero residual plane)
// and flagged so; `poison_h8`: the value plane holds E5M2 NaNs, for a plane the GEMM must not read.
static Operand make_operand(int arith, int models, int rows, int K, float scale, bool exact = false,
                            bool poison_h8 = false) {
  Operand o{arith, models, rows, K, exact};
  const size_t n = (size_t)models * rows * K;
  o.x.resize(n);
  o.p16.resize(n);
  if (arith == kBf) o.lo16.resize(n);
  else o.h8.resize(n), o.l8.resize(n);
  for (size_t i = 0; i < n; ++i) {
    float v = frand() * scale;
    if (exact) v = __half2float(__float2half_rn(v));
    o.x[i] = v;
    if (arith == kBf) {
      const __nv_bfloat16 h = __float2bfloat16_rn(v);
      o.p16[i] = bits(h);
      o.lo16[i] = bits(__float2bfloat16_rn(v - __bfloat162float(h)));
    } else {
      const __half h = __float2half_rn(v);
      o.p16[i] = bits(h);
      o.h8[i] = poison_h8 ? kE5m2NaN : __nv_cvt_float_to_fp8(v, __NV_SATFINITE, __NV_E5M2);
      o.l8[i] = __nv_cvt_float_to_fp8((v - __half2float(h)) * float(1 << kLoShift), __NV_SATFINITE, __NV_E5M2);
    }
  }
  return o;
}

// f16f8 planes drawn directly: a zero fp16 plane, a value plane of one sign (codes after the ReLU) or of either sign,
// and a residual plane of either sign (rounding errors)
static Operand cross_operand(int rows, int K, bool positive) {
  Operand o{kF8, 1, rows, K, false};
  const size_t n = (size_t)rows * K;
  o.p16.assign(n, 0);
  o.h8.resize(n);
  o.l8.resize(n);
  for (size_t i = 0; i < n; ++i) {
    const float a = positive ? 0.5f * (frand() + 1.0f) : frand(), b = frand();
    o.h8[i] = __nv_cvt_float_to_fp8(a, __NV_SATFINITE, __NV_E5M2);
    o.l8[i] = __nv_cvt_float_to_fp8(b, __NV_SATFINITE, __NV_E5M2);
  }
  return o;
}

// one plane on the device, K-major [models][rows][pitch] or MN-major [models][K][pitch]; rows are padded to 16 elements
// (TMA strides are 16-byte multiples) with `pad`, which no map exposes
template <class T>
static const T* upload_plane(const Operand& o, const std::vector<T>& v, bool mn, T pad, uint64_t& pitch) {
  pitch = ((mn ? o.rows : o.K) + 15) / 16 * 16;
  const size_t outer = mn ? o.K : o.rows;
  std::vector<T> buf((size_t)o.models * outer * pitch, pad);
  for (int m = 0; m < o.models; ++m)
    for (int r = 0; r < o.rows; ++r)
      for (int k = 0; k < o.K; ++k) buf[((size_t)m * outer + (mn ? k : r)) * pitch + (mn ? r : k)] = v[o.at(m, r, k)];
  T* d = nullptr;
  CK(cudaMalloc(&d, buf.size() * sizeof(T)));
  CK(cudaMemcpy(d, buf.data(), buf.size() * sizeof(T), cudaMemcpyHostToDevice));
  g_dev.push_back(d);
  return d;
}

// The maps the GEMM reads for one operand: 16-bit planes K-major (boxes of box_rows x BK, one swizzle span per row) or
// MN-major (boxes of BK x 64); f16f8 8-bit planes K-major (64-byte swizzle, as E5M2 wgmma reads them; the engine's
// batch-major copies of MN-major operands have this layout) or MN-major (unswizzled, widened by the GEMM).
static void operand_maps(const Operand& o, bool mn16, bool mn8, uint32_t box_rows, CUtensorMap* hi, CUtensorMap* lo,
                         CUtensorMap* x8) {
  const int BK = gemm_bk(o.arith);
  auto map16 = [&](CUtensorMap* t, const std::vector<uint16_t>& v, uint16_t nan) {
    uint64_t pitch;
    const void* d = upload_plane(o, v, mn16, nan, pitch);
    if (mn16) return make_tmap_bf16(t, d, o.models, o.K, o.rows, pitch, o.K * pitch, BK);
    return make_tmap_bf16_box(t, d, o.models, o.rows, o.K, pitch, o.rows * pitch, BK, box_rows,
                              BK == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B);
  };
  auto map8 = [&](CUtensorMap* t, const std::vector<uint8_t>& v) {
    uint64_t pitch;
    const void* d = upload_plane(o, v, mn8, kE5m2NaN, pitch);
    if (mn8) return make_tmap_u8_box(t, d, o.models, o.K, o.rows, pitch, o.K * pitch, 128, BK, CU_TENSOR_MAP_SWIZZLE_NONE);
    return make_tmap_u8_box(t, d, o.models, o.rows, o.K, pitch, o.rows * pitch, BK, box_rows, CU_TENSOR_MAP_SWIZZLE_64B);
  };
  const bool ok = o.arith == kBf ? map16(hi, o.p16, kBf16NaN) && map16(lo, o.lo16, kBf16NaN)
                                 : map16(hi, o.p16, kF16NaN) && map8(lo, o.h8) && map8(x8, o.l8);
  if (!ok) {
    printf("tensor map encode failed\n");
    exit(2);
  }
}

// out[model][i][j] = sum over the sets of A_s[i,:] . B_s[j,:] through launch_gemm, on freshly uploaded planes
// (unwritten outputs read as NaN). reps > 1: two warm-up launches, then `reps` timed ones (*ms = time per launch).
template <bool A_MN, bool B_MN, bool SPLIT, int ARITH, bool NATIVE>
static std::vector<float> run_gemm(const Operand* A, const Operand* B, int nsets, int models, int passes, int reps = 1,
                                   float* ms = nullptr) {
  const int M = A[0].rows, N = B[0].rows;
  GemmParams<EpiStoreF32::Params> p;
  memset(&p, 0, sizeof(p));
  for (int s = 0; s < nsets; ++s) {
    operand_maps(A[s], A_MN, A_MN && !NATIVE, kBM, &p.a_hi[s], &p.a_lo[s], &p.a_x8[s]);
    operand_maps(B[s], B_MN, B_MN && !NATIVE, kBN, &p.b_hi[s], &p.b_lo[s], &p.b_x8[s]);
    p.a_batched[s] = A[s].models > 1;
    p.b_batched[s] = B[s].models > 1;
    if (A[s].flagged) p.a_res_flag[s] = g_zero_flag;
    if (B[s].flagged) p.b_res_flag[s] = g_zero_flag;
  }
  const size_t out_elems = (size_t)models * M * N;
  float* d_out;
  CK(cudaMalloc(&d_out, out_elems * 4));
  CK(cudaMemset(d_out, 0xFF, out_elems * 4));
  p.nsets = nsets;
  p.k_total = A[0].K;
  p.passes = passes;
  p.n_models = models;
  p.m_total = M;
  p.n_total = N;
  p.tiles_m = (M + kBM - 1) / kBM;
  p.tiles_n = (N + kBN - 1) / kBN;
  p.epi.out = d_out;
  p.epi.model_stride = (long long)M * N;
  p.epi.ld = N;
  cudaEvent_t e0, e1;
  CK(cudaEventCreate(&e0));
  CK(cudaEventCreate(&e1));
  const int warm = reps > 1 ? 2 : 0;
  for (int rep = 0; rep < warm + reps; ++rep) {
    if (rep == warm) CK(cudaEventRecord(e0));
    CK((launch_gemm<EpiStoreF32, A_MN, B_MN, SPLIT, ARITH, NATIVE>(p, 0, g_sms, 0)));
  }
  CK(cudaEventRecord(e1));
  const cudaError_t err = cudaDeviceSynchronize();
  if (err != cudaSuccess) {
    printf("kernel failed: %s\n", cudaGetErrorString(err));
    exit(3);  // the context is dead after a device fault
  }
  float t = 0;
  CK(cudaEventElapsedTime(&t, e0, e1));
  if (ms) *ms = t / reps;
  std::vector<float> out(out_elems);
  CK(cudaMemcpy(out.data(), d_out, out_elems * 4, cudaMemcpyDeviceToHost));
  CK(cudaEventDestroy(e0));
  CK(cudaEventDestroy(e1));
  cudaFree(d_out);
  for (void* d : g_dev) cudaFree(d);
  g_dev.clear();
  return out;
}

// fp64 value of out[m][i][j] from the planes the GEMM multiplies. f16f8: a flagged operand's cross term is skipped, as
// the GEMM skips it (its residual plane is zero, and the other operand's value plane may be poisoned).
static double plane_exact(const Operand* A, const Operand* B, int nsets, int m, int i, int j, int passes) {
  double hh = 0, cr = 0;
  for (int s = 0; s < nsets; ++s) {
    const Operand &a = A[s], &b = B[s];
    const int am = a.models > 1 ? m : 0, bm = b.models > 1 ? m : 0;
    for (int k = 0; k < a.K; ++k) {
      const size_t ia = a.at(am, i, k), ib = b.at(bm, j, k);
      if (a.arith == kBf) {
        const double ah = bf16_value(a.p16[ia]), bh = bf16_value(b.p16[ib]);
        hh += ah * bh;
        if (passes >= 3) cr += ah * bf16_value(b.lo16[ib]) + bf16_value(a.lo16[ia]) * bh;
      } else {
        hh += f16_value(a.p16[ia]) * f16_value(b.p16[ib]);
        if (passes >= 3 && !a.flagged) cr += e5m2_value(a.l8[ia]) * e5m2_value(b.h8[ib]);
        if (passes >= 3 && !b.flagged) cr += e5m2_value(a.h8[ia]) * e5m2_value(b.l8[ib]);
      }
    }
  }
  return A[0].arith == kBf ? hh + cr : hh + cr / double(1 << kLoShift);
}

struct Case {
  const char* name;
  int models, M, N, K, nsets, passes;
  bool a_shared = false, b_shared = false;
  int exact = 0;   // f16f8: 1 = A of set 0, 2 = B of set 0 is fp16-exact and flagged so
};

static void make_case(const Case& c, int arith, Operand* A, Operand* B) {
  const float sa = arith == kF8 ? 3.0f : 1.0f, sb = arith == kF8 ? 0.25f : 1.0f;
  for (int s = 0; s < c.nsets; ++s) {
    A[s] = make_operand(arith, c.a_shared ? 1 : c.models, c.M, c.K, sa, s == 0 && c.exact == 1);
    B[s] = make_operand(arith, c.b_shared ? 1 : c.models, c.N, c.K, sb, s == 0 && c.exact == 2);
  }
}

// Every index of [0, n) up to 512, else every step-th one, and always the last one (the partial tile's edge).
static std::vector<int> sample_indices(int n, int step) {
  std::vector<int> v;
  for (int i = 0; i < n; i += n > 512 ? step : 1) v.push_back(i);
  if (v.back() != n - 1) v.push_back(n - 1);
  return v;
}

// Checks a case's output against plane_exact at 1e-3 sqrt(K sets) (bf16x3) or 1e-4 sqrt(K sets) (f16f8); rows and
// columns are sampled beyond 512, the last row and column always. Prints the PASS / FAIL line with the number of output
// tiles (beyond the SM count, persistent CTAs run more than one) and, on failure, a map of the failing 4 x 16 blocks.
static bool check_case(const Case& c, const char* path, const Operand* A, const Operand* B, const std::vector<float>& out,
                       float ms) {
  const int arith = A[0].arith, M = c.M, N = c.N;
  const double bound = (arith == kBf ? 1e-3 : 1e-4) * sqrt((double)c.K * c.nsets);
  double max_err = 0, max_ref = 0, se_full = 0, s_full = 0;
  long long bad = 0;
  int fb[3] = {-1, -1, -1};
  const int tiles = c.models * ((M + kBM - 1) / kBM) * ((N + kBN - 1) / kBN);
  const std::vector<int> rows = sample_indices(M, 37), cols = sample_indices(N, 29);
  for (int m = 0; m < c.models; ++m)
    for (int i : rows)
      for (int j : cols) {
        const double ex = plane_exact(A, B, c.nsets, m, i, j, c.passes), got = out[((size_t)m * M + i) * N + j];
        double fu = 0;   // the fp32 operands' product
        for (int s = 0; s < c.nsets; ++s)
          for (int k = 0; k < c.K; ++k)
            fu += (double)A[s].x[A[s].at(A[s].models > 1 ? m : 0, i, k)] * B[s].x[B[s].at(B[s].models > 1 ? m : 0, j, k)];
        double e = fabs(got - ex);
        if (!(e == e)) e = 1e30;
        max_err = fmax(max_err, e);
        max_ref = fmax(max_ref, fabs(ex));
        if (got == got) se_full += (got - fu) * (got - fu), s_full += fu * fu;
        if (e > bound && !bad++) fb[0] = m, fb[1] = i, fb[2] = j;
      }
  const bool ok = bad == 0;
  const double flops = 2.0 * c.models * M * N * (double)c.K * c.nsets * (arith == kBf && c.passes >= 3 ? 3 : 1);
  printf("[%s%s%s] %s  models=%d M=%d N=%d K=%d sets=%d passes=%d tiles=%d  max|err| vs plane-exact %.3e (bound %.3e, "
         "max|ref| %.2f), rel. rms vs fp32 product %.2e  %.3f ms  %.1f TF(%s)\n",
         c.name, *path ? "/" : "", path, ok ? "PASS" : "FAIL", c.models, M, N, c.K, c.nsets, c.passes, tiles, max_err,
         bound, max_ref, sqrt(se_full / (s_full + 1e-300)), ms, flops / ms * 1e-9,
         arith == kBf ? "bf16 passes" : "algorithmic");
  if (!ok) {
    printf("    %lld bad samples; first at model %d row %d col %d: got %.6f\n", bad, fb[0], fb[1], fb[2],
           out[((size_t)fb[0] * M + fb[1]) * N + fb[2]]);
    for (int i = 0; i < (M < 32 ? M : 32); i += 4) {   // rows 0..31, columns 0..255 of the first failing model
      printf("    row %3d:", i);
      for (int j = 0; j < (N < 256 ? N : 256); j += 16) {
        const double e = fabs(out[((size_t)fb[0] * M + i) * N + j] - plane_exact(A, B, c.nsets, fb[0], i, j, c.passes));
        printf(" %c", e <= bound ? '.' : 'X');
      }
      printf("\n");
    }
  }
  return ok;
}

template <bool A_MN, bool B_MN, bool SPLIT, int ARITH, bool NATIVE>
static bool run_case(const Case& c, int reps = 1) {
  Operand A[2], B[2];
  make_case(c, ARITH, A, B);
  float ms = 0;
  const std::vector<float> out = run_gemm<A_MN, B_MN, SPLIT, ARITH, NATIVE>(A, B, c.nsets, c.models, c.passes, reps, &ms);
  return check_case(c, "", A, B, out, ms);
}

// f16f8 MN x MN on the same data both ways: native (8-bit planes from batch-major copies) and widened
static bool run_case_f8_mnmn(const Case& c, int reps = 1) {
  Operand A[2], B[2];
  make_case(c, kF8, A, B);
  float ms = 0;
  std::vector<float> out = run_gemm<true, true, false, kF8, true>(A, B, c.nsets, c.models, c.passes, reps, &ms);
  bool ok = check_case(c, "native", A, B, out, ms);
  out = run_gemm<true, true, false, kF8, false>(A, B, c.nsets, c.models, c.passes, reps, &ms);
  ok &= check_case(c, "widened", A, B, out, ms);
  return ok;
}

// f16f8 cross-term accumulation. The fp16 planes are zero, so the output is exactly 2^-kLoShift times the sum of the E5M2
// products A.l8 B.h8 + A.h8 B.l8, each of them exact on either path: what is measured is the tensor core's accumulation
// alone, relative to the sum of |products| (the scale of its rounding). Native (K x K): E5M2 wgmma, each K block's sums
// promoted into the fp32 accumulator, since FP8 wgmma accumulates with fewer bits than fp32 and truncates, and its sums
// would drift with their length; bound 2^-12, below 2^-22 of a GEMM's result, of which the cross terms are 2^-11.
// Widened (the MN-major layout of the same data, the only one libsce widens): fp32 accumulation, bound 1e-7 K.
static bool cross_terms() {
  const int M = 128, N = 128;
  const double inv = 1.0 / double(1 << kLoShift);
  bool all_ok = true;
  for (int positive = 0; positive < 2; ++positive)
    for (int K : {512, 4096, 16384}) {
      const Operand A = cross_operand(M, K, positive), B = cross_operand(N, K, positive);
      const std::vector<float> nat = run_gemm<false, false, false, kF8, true>(&A, &B, 1, 1, 3);
      const std::vector<float> wide = run_gemm<true, true, false, kF8, false>(&A, &B, 1, 1, 3);
      double err_w = 0, err_n = 0, bias_n = 0;
      for (int i = 0; i < M; ++i)
        for (int j = 0; j < N; ++j) {
          double s = 0, sa = 0;
          for (int k = 0; k < K; ++k) {
            const size_t ia = A.at(0, i, k), ib = B.at(0, j, k);
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
      const bool ok = !(err_w > 1e-7 * K) && !(err_n > 1.0 / 4096);
      all_ok &= ok;
      printf("[cross_terms %s K=%5d] %s  max |err| / sum|products|: widened %.3e, native %.3e (%.1f bits); native mean "
             "signed %.3e\n",
             positive ? "h8>=0" : "signed", K, ok ? "PASS" : "FAIL", err_w, err_n, err_n > 0 ? -log2(err_n) : 99.0, bias_n);
    }
  return all_ok;
}

// The f16f8 weight gradient with mixed operand layouts: fp16 planes MN-major as the batch holds them ([K][rows], K =
// batch), 8-bit planes K-major from batch-major copies whose padding past K holds NaNs. Two operand sets as in
// dW = dz^T x + c^T g; set 0's B is fp16-exact and flagged (the x of fp16 activations), so its A.h8 x B.l8 term is
// skipped, and A's value plane of set 0 holds NaNs to show it is not read. M and N are not multiples of 128, K is 8192
// and a ragged 8155. Native and widened are each checked against the plane-exact value and against each other.
static bool mixed_dw() {
  const int models = 2, M = 208, N = 336, nsets = 2;
  bool all_ok = true;
  for (int K : {8192, 8155}) {
    Operand A[2], B[2];
    for (int s = 0; s < nsets; ++s) {
      A[s] = make_operand(kF8, models, M, K, 3.0f, false, s == 0);
      B[s] = make_operand(kF8, models, N, K, 0.25f, s == 0);
    }
    const std::vector<float> nat = run_gemm<true, true, false, kF8, true>(A, B, nsets, models, 3);
    const std::vector<float> wide = run_gemm<true, true, false, kF8, false>(A, B, nsets, models, 3);
    double err_n = 0, err_w = 0, err_nw = 0, max_ref = 0;
    long long bad = 0, checked = 0;
    const double bound = 1e-4 * sqrt((double)K * nsets);
    auto nan_big = [](double e) { return e == e ? e : 1e30; };
    for (int m = 0; m < models; ++m)
      for (int i = 0; i < M; i += 3)
        for (int j = 0; j < N; j += 5) {
          const double ex = plane_exact(A, B, nsets, m, i, j, 3);
          const size_t o = ((size_t)m * M + i) * N + j;
          const double en = nan_big(fabs(nat[o] - ex)), ew = nan_big(fabs(wide[o] - ex));
          const double enw = nan_big(fabs((double)nat[o] - (double)wide[o]));
          err_n = fmax(err_n, en);
          err_w = fmax(err_w, ew);
          err_nw = fmax(err_nw, enw);
          max_ref = fmax(max_ref, fabs(ex));
          bad += en > bound || ew > bound || enw > bound;
          ++checked;
        }
    long long unwritten = 0;   // every output is written: partial tiles are clipped, not dropped
    for (size_t o = 0; o < nat.size(); ++o) unwritten += !(nat[o] == nat[o]) + !(wide[o] == wide[o]);
    const bool ok = bad == 0 && unwritten == 0;
    all_ok &= ok;
    printf("[mixed_dw K=%d] %s  models=%d M=%d N=%d sets=%d  max|err| vs plane-exact: native %.3e, widened %.3e; "
           "max|native - widened| %.3e; bound %.3e (max|ref| %.2f); %lld samples, %lld NaN outputs\n",
           K, ok ? "PASS" : "FAIL", models, M, N, nsets, err_n, err_w, err_nw, bound, max_ref, checked, unwritten);
  }
  return all_ok;
}

int main(int argc, char** argv) {
  const bool big = argc > 1 && !strcmp(argv[1], "--big");
  setvbuf(stdout, nullptr, _IOLBF, 0);
  cudaDeviceProp prop;
  CK(cudaGetDeviceProperties(&prop, 0));
  g_sms = prop.multiProcessorCount;
  printf("device: %s  sm_%d%d  SMs=%d\n", prop.name, prop.major, prop.minor, g_sms);
  CK(cudaMalloc(&g_zero_flag, 4));
  CK(cudaMemset(g_zero_flag, 0, 4));
  bool ok = true;
  if (big) {
    // config-2 shapes, one model's worth of each GEMM
    ok &= run_case<false, false, false, kBf, false>({"big_encode", 4, 8192, 4096, 512, 1, 3, true}, 10);
    ok &= run_case<false, true, false, kBf, false>({"big_decode", 4, 8192, 512, 4096, 1, 3}, 10);
    ok &= run_case<false, true, true, kBf, false>({"big_decode_split", 4, 8192, 512, 4096, 1, 3}, 10);
    ok &= run_case<true, true, true, kBf, false>({"big_dw", 4, 4096, 512, 8192, 2, 3, false, true}, 10);
    ok &= run_case<false, false, false, kF8, true>({"f8_big_encode", 4, 8192, 4096, 512, 1, 3, true}, 10);
    ok &= run_case<false, false, false, kF8, true>({"f8_big_decode", 4, 8192, 512, 4096, 1, 3}, 10);
    ok &= run_case_f8_mnmn({"f8_big_dw", 4, 4096, 512, 8192, 2, 3, false, true}, 10);
  } else {
    // ---- bf16x3, K x K (encode, scores, centring, dcode, similarity)
    const Case kk[] = {{"kk_k16", 1, 128, 256, 16, 1, 1},          {"kk_k64", 1, 128, 256, 64, 1, 1},
                       {"kk_k256", 1, 128, 256, 256, 1, 1},        {"kk_3pass", 1, 128, 256, 256, 1, 3},
                       {"kk_multi", 3, 384, 512, 512, 1, 3, true}, {"kk_ragged", 2, 200, 328, 104, 1, 3, true},
                       {"kk_bn128", 2, 256, 384, 256, 1, 3, true}, {"kk_short", 2, 100, 328, 104, 1, 3, true},
                       {"kk_persist", 4, 1000, 1040, 400, 1, 3, true}};
    for (const Case& c : kk) ok &= run_case<false, false, false, kBf, false>(c);
    // ---- bf16x3, K x MN (decode: X^ = C W), without and with split accumulators
    const Case kmn[] = {{"kmn_k16", 1, 128, 256, 16, 1, 1}, {"kmn_k64", 1, 128, 256, 64, 1, 1},
                        {"kmn_3pass", 2, 256, 512, 512, 1, 3}, {"kmn_ragged", 2, 200, 328, 104, 1, 3},
                        {"kmn_persist", 4, 1000, 1040, 400, 1, 3}};
    for (const Case& c : kmn) ok &= run_case<false, true, false, kBf, false>(c);
    const Case kmn_split[] = {{"kmn_split", 2, 512, 512, 512, 1, 3}, {"kmn_split_ragged", 2, 200, 328, 104, 1, 3},
                              {"kmn_split_persist", 4, 1000, 1040, 400, 1, 3}};
    for (const Case& c : kmn_split) ok &= run_case<false, true, true, kBf, false>(c);
    // ---- bf16x3, MN x MN with split accumulators (weight gradient: dW = dZ^T X + C^T G), up to two operand sets
    const Case mnmn[] = {{"mnmn_k16", 1, 128, 256, 16, 1, 1},
                         {"mnmn_k64", 1, 128, 256, 64, 1, 1},
                         {"mnmn_2set", 2, 512, 512, 320, 2, 3, false, true},
                         {"mnmn_2set_m256", 2, 256, 512, 320, 2, 3, false, true},
                         {"mnmn_ragged", 2, 200, 328, 104, 2, 3, false, true},
                         {"mnmn_persist", 4, 1000, 1040, 400, 2, 3, false, true}};
    for (const Case& c : mnmn) ok &= run_case<true, true, true, kBf, false>(c);
    // ---- f16f8 native K x K (the f8_kmn cases: decode, which reads the transposed dictionary K-major)
    const Case f8_kk[] = {{"f8_kk_hh", 1, 128, 256, 64, 1, 1},
                          {"f8_kk_k64", 1, 128, 256, 64, 1, 3},
                          {"f8_kk_multi", 3, 384, 512, 512, 1, 3, true},
                          {"f8_kk_ragged", 2, 200, 328, 104, 1, 3, true},
                          {"f8_kk_exactA", 3, 768, 512, 512, 1, 3, true, false, 1},
                          {"f8_kmn_k64", 1, 128, 256, 64, 1, 3},
                          {"f8_kmn_multi", 2, 256, 512, 512, 1, 3},
                          {"f8_kmn", 2, 512, 512, 512, 1, 3},
                          {"f8_kmn_ragged", 2, 200, 328, 104, 1, 3},
                          {"f8_kk_persist", 4, 1000, 1040, 400, 1, 3, true}};
    for (const Case& c : f8_kk) ok &= run_case<false, false, false, kF8, true>(c);
    // ---- f16f8 MN x MN (weight gradient), native and widened
    const Case f8_mnmn[] = {{"f8_mnmn_k64", 1, 128, 256, 64, 1, 3},
                            {"f8_mnmn_2set", 2, 256, 512, 320, 2, 3, false, true},
                            {"f8_mnmn_ragged", 2, 200, 328, 104, 2, 3, false, true},
                            {"f8_mnmn_exactB", 2, 512, 512, 320, 2, 3, false, true, 2},
                            {"f8_mnmn_persist", 4, 1000, 1040, 400, 2, 3, false, true}};
    for (const Case& c : f8_mnmn) ok &= run_case_f8_mnmn(c);
    ok &= cross_terms();
    ok &= mixed_dw();
  }
  cudaFree(g_zero_flag);
  printf(ok ? "ALL PASS\n" : "SOME FAILED\n");
  return ok ? 0 : 1;
}
