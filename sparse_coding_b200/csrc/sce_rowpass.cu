// sce_rowpass.cu — the sliced row passes of the PCA, ICA and NMF baselines: second moments, the FastICA pass, the NMF
// projection, Grams, coordinate-descent sweep and residual.
#include <algorithm>

#include "sce_engine.cuh"

// ------------------------------------------------------------------------------------------------
// sliced row passes: second moments (sce_second_moments, for BatchedPCA), the FastICA pass (sce_ica_pass) and the NMF
// projection and Grams (sce_nmf_project, sce_nmf_grams, for NMFEncoder)
// ------------------------------------------------------------------------------------------------
// Each splits the rows x, shifted by a vector (clamped at 0 for NMF), into operand planes (moment_split_kernel). All
// but the projection end in a reduction over the rows, A^T V for the shifted rows V: the Gram matrix V^T V, FastICA's
// T^T V, or NMF's W^T W and W^T V. It is
// the weight gradient's GEMM (MN-major 16-bit planes, K = rows; f16f8 cross terms on E5M2 wgmma from batch-major copies
// of the 8-bit planes, EpiStoreF32). The rows are cut into S slices of R rows, run as the GEMM's models, so that an
// output of few tiles still fills the SMs; each slice leaves an fp32 partial, and the partials are added in slice order
// in fp64.
// Rows one slice accumulates in fp32. The tensor cores' fp32 accumulation truncates, and the Gram diagonal is a sum of
// squares, so its bias grows with K: 8192-row slices (the training weight gradient's K) left config 5's width 1.1e-5
// (bf16x3) and 1.7e-5 (f16f8) from fp64 in Frobenius norm, against a 2e-5 bar. 2048 rows leave a quarter of that, for
// a few more fp32 partials.
constexpr int kMomRowsMax = 2048;
constexpr int kMomTargetTiles = 528;   // output tiles a launch aims for (4 waves of 132 SMs; fixed, so results do not
                                       // depend on the device)
constexpr int kMomSliceMin = 256;      // no slice shorter than this, unless the call is
constexpr int kMomBlockRows = 64;      // rows per block of the split kernel (one column-sum partial each)
constexpr int kMomCallRowsMax = 1 << 21;

struct Slices {   // a call's rows as S slices of R rows (R a multiple of 64, the f16f8 K block, and at most kMomRowsMax)
  int S, R;
};
// the slices of a call of B rows of width d
static Slices mom_slices(int d, int B) {
  const int tiles = ((d + kBM - 1) / kBM) * ((d + kBN - 1) / kBN);
  const int s_rows = (B + kMomRowsMax - 1) / kMomRowsMax;
  int s = (kMomTargetTiles + tiles - 1) / tiles;
  const int s_short = (B + kMomSliceMin - 1) / kMomSliceMin;
  if (s > s_short) s = s_short;
  if (s < s_rows) s = s_rows;
  const int R = ((B + s - 1) / s + kMomBlockRows - 1) / kMomBlockRows * kMomBlockRows;
  return {(B + R - 1) / R, R};
}

// the (d, B) of a row pass: rows of width d, a multiple of 8 in [8, 8192], and 1 <= B <= kMomCallRowsMax rows per call
static bool row_shape_ok(int d, int B) { return d >= 8 && d % 8 == 0 && d <= 8192 && B >= 1 && B <= kMomCallRowsMax; }
// the component count n of a pass over rows of width d (ICA's n, NMF's k): a multiple of 8 in [8, d]
static bool components_ok(int n, int d) { return n >= 8 && n % 8 == 0 && n <= d; }

// The rows a pass reads and where it runs: x [B][d] (fp16 when half, else fp32), shift [d], the f16f8 range flag (set
// when a shifted row, or a matrix split beside them, holds a value the fp16 plane cannot), the device and its SMs
struct RowArgs {
  const void* x;
  bool half;
  int B, d;
  const float* shift;
  uint32_t* range_flag;
  int device, sms;
};

enum RowPass { kPassMoments, kPassIca, kPassNmfProject, kPassNmfGrams };

// The buffers of the row passes; each pass takes its own (row_carve). The projection runs one model of B rows padded
// to kMomBlockRows (S = 1) and takes no batch-major copies.
struct RowCarve {
  Planes x, xt;      // the shifted rows [S * R][d] (zero beyond B); f16f8: batch-major 8-bit copies [S][d][R]
  Planes t, tt;      // ICA: t [S * R][n]; NMF Grams: W [S * R][k]; f16f8: batch-major 8-bit copies [S][n][R]
  Planes mat;        // ICA: unmix [n][d]; NMF projection: M [k][d]
  float* part;       // [S][n, or d][d] fp32 slice partials; NMF projection: [ceil(B / 32)][2][k] column-norm partials
  float* part_g;     // NMF Grams: [S][k][k] fp32 slice partials of W^T W
  double* col_part;  // [S * R / kMomBlockRows][d]: the split kernel's column sums (second moments; ICA leaves them unread)
  float* g_part;     // ICA: [S * R / 32][n] g' partials
  uint32_t* flags;   // ICA, NMF: kFlagWords, the f16f8 range check of the matrix
};
// Carves the buffers `pass` takes, for S slices of `rows` (= S R) padded rows of a call of B rows with n components,
// in the order of RowCarve; a buffer a pass does not take has no elements and carves nothing. The workspace query
// carves upper bounds of S and rows instead, which never decrease with B: the exact S is not monotone in B (at d = 512,
// B = 64000 takes 33 slices of 1984 rows, B = 65536 32 of 2048), and a caller sizes one workspace for its longest call.
static size_t row_carve(uint8_t* base, RowPass pass, bool f8, int d, int n, int B, size_t S, size_t rows, RowCarve* out) {
  const size_t dd = (size_t)d, nn = (size_t)n, col = rows / kMomBlockRows * dd;
  struct {
    size_t t, mat, part, part_g, col_part, g_part, flags;
    bool copies;
  } z{};
  switch (pass) {   // t, mat, part, part_g, col_part, g_part, flags, copies
    case kPassMoments: z = {0, 0, S * dd * dd, 0, col, 0, 0, true}; break;
    case kPassIca: z = {rows * nn, nn * dd, S * nn * dd, 0, col, rows / 32 * nn, kFlagWords, true}; break;
    case kPassNmfProject: z = {0, nn * dd, ((size_t)B + 31) / 32 * 2 * nn, 0, 0, 0, kFlagWords, false}; break;
    case kPassNmfGrams: z = {rows * nn, 0, S * nn * dd, S * nn * nn, 0, 0, kFlagWords, true}; break;
  }
  Carve c{base, 0};
  RowCarve w{};
  w.x = c.planes(rows * dd, f8);
  w.t = c.planes(z.t, f8);
  if (f8 && z.copies) {
    w.xt = c.copies(rows * dd);
    w.tt = c.copies(z.t);
  }
  w.mat = c.planes(z.mat, f8);
  w.part = c.take<float>(z.part);
  w.part_g = c.take<float>(z.part_g);
  w.col_part = c.take<double>(z.col_part);
  w.g_part = c.take<float>(z.g_part);
  w.flags = c.take<uint32_t>(z.flags);
  if (out) *out = w;
  return align_up(c.off, 1024);
}
static size_t padded_rows(int B) { return ((size_t)B + kMomBlockRows - 1) / kMomBlockRows * kMomBlockRows; }
// The workspace of a row pass, for both arithmetics; 0 when d, B or n is out of range. The sliced passes carve the
// bounds of mom_slices, non-decreasing in B: S <= max(min(target, ceil(B / 256)), ceil(B / 2048)) (the s it starts
// from), and S R < B + R <= B + 2048 with S R <= S kMomRowsMax; rows are a multiple of kMomBlockRows.
static size_t row_pass_workspace(RowPass pass, int d, int n, int B) {
  if (!row_shape_ok(d, B) || (pass != kPassMoments && !components_ok(n, d))) return 0;
  size_t S = 1, rows = padded_rows(B);
  if (pass != kPassNmfProject) {
    const int tiles = ((d + kBM - 1) / kBM) * ((d + kBN - 1) / kBN);
    const size_t s_target = (kMomTargetTiles + tiles - 1) / tiles, s_short = (B + kMomSliceMin - 1) / kMomSliceMin;
    const size_t s_rows = (B + kMomRowsMax - 1) / kMomRowsMax;
    S = std::max(std::min(s_target, s_short), s_rows);
    rows = std::min(rows + kMomRowsMax, S * kMomRowsMax);
  }
  return std::max(row_carve(nullptr, pass, false, d, n, B, S, rows, nullptr),
                  row_carve(nullptr, pass, true, d, n, B, S, rows, nullptr));
}

// rows r0 .. r0 + 63 of the call (grid.y), four columns per thread (grid.x covers d / 4 threads):
//   v = x - shift (fp32) -> operand planes; rows >= B are stored as zero in every plane, so that the padded tail of the
//   last slice adds nothing to the Gram matrix (0 - shift would add shift shift^T per row)
//   col_part[blockIdx.y][c] = sum of v over the block's rows, in row order in fp64
//   f16f8: range_flag = 1 when some |v| >= 65520 or v is NaN (the fp16 plane cannot hold it)
// CLAMP (the NMF passes): v = max(x - shift, 0) instead (NaN stays NaN), and no column sums (col_part is not read)
template <int ARITH, class InT, bool CLAMP = false>
__global__ void __launch_bounds__(128) moment_split_kernel(const InT* __restrict__ x, int B, int d,
                                                           const float* __restrict__ shift, void* __restrict__ hi,
                                                           void* __restrict__ lo, void* __restrict__ x8,
                                                           double* __restrict__ col_part, uint32_t* __restrict__ range_flag) {
  const int c = (blockIdx.x * blockDim.x + threadIdx.x) * 4;
  if (c >= d) return;
  const float4 sh = __ldg(reinterpret_cast<const float4*>(shift + c));
  double s0 = 0.0, s1 = 0.0, s2 = 0.0, s3 = 0.0;
  bool bad = false;
  const int r0 = blockIdx.y * kMomBlockRows;
#pragma unroll 4
  for (int i = 0; i < kMomBlockRows; ++i) {
    const int r = r0 + i;
    float v[4] = {0.f, 0.f, 0.f, 0.f};
    if (r < B) {
      const long long e = (long long)r * d + c;
      if constexpr (sizeof(InT) == 2) {
        const uint2 raw = __ldg(reinterpret_cast<const uint2*>(x + e));
        const __half2 a = *reinterpret_cast<const __half2*>(&raw.x);
        const __half2 b = *reinterpret_cast<const __half2*>(&raw.y);
        v[0] = __low2float(a) - sh.x;
        v[1] = __high2float(a) - sh.y;
        v[2] = __low2float(b) - sh.z;
        v[3] = __high2float(b) - sh.w;
      } else {
        const float4 f = __ldg(reinterpret_cast<const float4*>(x + e));
        v[0] = f.x - sh.x;
        v[1] = f.y - sh.y;
        v[2] = f.z - sh.z;
        v[3] = f.w - sh.w;
      }
      if constexpr (CLAMP) {
#pragma unroll
        for (int q = 0; q < 4; ++q) v[q] = v[q] < 0.f ? 0.f : v[q];
      }
      s0 += v[0];
      s1 += v[1];
      s2 += v[2];
      s3 += v[3];
      if constexpr (ARITH == kArithF16F8)
        bad |= !(fabsf(v[0]) < 65520.f && fabsf(v[1]) < 65520.f && fabsf(v[2]) < 65520.f && fabsf(v[3]) < 65520.f);
    }
    store_planes4<ARITH>(v, hi, lo, x8, ((long long)r * d + c) / 4);
  }
  if constexpr (!CLAMP) {
    double* o = col_part + (long long)blockIdx.y * d + c;
    o[0] = s0;
    o[1] = s1;
    o[2] = s2;
    o[3] = s3;
  }
  if (bad && range_flag) *range_flag = 1u;   // benign race: all write 1
}

// gram[i] += sum over the slices s, in order, of part[s][i] (an n x d output: n4 = n d / 4, n d >= 4 d; none with
// n4 = 0); with col_part, col_sum[j] += sum over the row blocks b, in order, of col_part[b][j] (j < d); with vec_part
// (fp32 row-block partials: sce_ica_pass's g' sums per 32 rows, sce_nmf_project's column norms), vec_sum[j] += the
// same over its vec_blocks row blocks (j < n). fp64 throughout; four Gram entries per thread.
__global__ void __launch_bounds__(256) gram_reduce_kernel(const float* __restrict__ part, int S, long long n4,
                                                            double* __restrict__ gram, const double* __restrict__ col_part,
                                                            int blocks, int d, double* __restrict__ col_sum,
                                                            const float* __restrict__ vec_part, int vec_blocks, int n,
                                                            double* __restrict__ vec_sum) {
  const long long stride = (long long)gridDim.x * blockDim.x, end = n4 > n ? n4 : n;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < end; i += stride) {
    if (i < n4) {
      double a0 = 0.0, a1 = 0.0, a2 = 0.0, a3 = 0.0;
      for (int s = 0; s < S; ++s) {
        const float4 v = __ldg(reinterpret_cast<const float4*>(part) + (long long)s * n4 + i);
        a0 += v.x;
        a1 += v.y;
        a2 += v.z;
        a3 += v.w;
      }
      double2* g = reinterpret_cast<double2*>(gram) + 2 * i;
      const double2 g0 = g[0], g1 = g[1];
      g[0] = make_double2(g0.x + a0, g0.y + a1);
      g[1] = make_double2(g1.x + a2, g1.y + a3);
    }
    if (col_part && i < d) {
      double t = 0.0;
      for (int b = 0; b < blocks; ++b) t += col_part[(long long)b * d + i];
      col_sum[i] += t;
    }
    if (vec_part && i < n) {
      double t = 0.0;
      for (int b = 0; b < vec_blocks; ++b) t += vec_part[(long long)b * n + i];
      vec_sum[i] += t;
    }
  }
}

// gram_reduce_kernel: out += the S slice partials `part` of n4 float4s, col_sum [d] += the column sums col_part of
// `blocks` row blocks, vec_sum [n] += the vec_blocks row-block partials vec_part (each only where given)
static int reduce_partials(Launcher& L, const float* part, int S, long long n4, double* out,
                           const double* col_part = nullptr, int blocks = 0, int d = 0, double* col_sum = nullptr,
                           const float* vec_part = nullptr, int vec_blocks = 0, int n = 0, double* vec_sum = nullptr) {
  const long long items = n4 > n ? n4 : n;
  const int rblocks = (int)((items + 255) / 256 < 2048 ? (items + 255) / 256 : 2048);
  return L.launch(gram_reduce_kernel, rblocks, 256, 0, part, S, n4, out, col_part, blocks, d, col_sum, vec_part,
                  vec_blocks, n, vec_sum);
}

// moment_split_kernel over the S R rows of a call: the shifted rows into the planes of w.x, the column-sum partials
// (not with CLAMP) and, with f16f8, the range flag
template <int AR, bool CLAMP = false>
static int launch_row_split(Launcher& L, const RowArgs& a, const Slices& sl, const RowCarve& w) {
  const dim3 grid((a.d / 4 + 127) / 128, sl.S * sl.R / kMomBlockRows);
  uint32_t* flag = AR == kArithF16F8 ? a.range_flag : nullptr;
  auto split = [&](auto* x) {
    return L.launch(moment_split_kernel<AR, std::decay_t<decltype(*x)>, CLAMP>, grid, 128, 0, x, a.B, a.d, a.shift,
                    w.x.hi, w.x.lo, w.x.x8, CLAMP ? nullptr : w.col_part, flag);
  };
  return a.half ? split(static_cast<const __half*>(a.x)) : split(static_cast<const float*>(a.x));
}

__global__ void set_flag_if_kernel(const uint32_t* __restrict__ src, uint32_t* __restrict__ dst) {
  if (*src) *dst = 1u;
}

// fp32 matrix [count / its width] -> planes; f16f8: its range check joins the rows' in range_flag
template <int AR>
static int split_matrix(Launcher& L, const float* m, const Planes& planes, long long count, uint32_t* flags,
                        uint32_t* range_flag) {
  if (AR == kArithF16F8 && range_flag) {
    CUDA_TRY(cudaMemsetAsync(flags, 0, kFlagWords * sizeof(uint32_t), L.st));
    TRY(launch_split_rows<AR>(L, m, planes, count / 4, flags));
    return L.launch(set_flag_if_kernel, 1, 1, 0, flags + kBadWord, range_flag);
  }
  return launch_split_rows<AR>(L, m, planes, count / 4, nullptr);
}

// part[s] = A_s^T V_s (fp32 [S][m][d]) for the slices s of R rows of A [S R][m] and V [S R][d]: the weight gradient's
// GEMM, one slice per model. f16f8: first the batch-major copies At and Vt of their 8-bit planes (one when A is V; none
// of A with a_copied, when an earlier call of the same rows made At).
template <int AR>
static int sliced_gemm_t(Launcher& L, const Slices& sl, const Planes& A, const Planes& At, int m, const Planes& V,
                         const Planes& Vt, int d, float* part, int device, int sms, bool a_copied = false) {
  constexpr bool f8 = AR == kArithF16F8;
  const bool a_is_v = A.hi == V.hi;
  const int S = sl.S, R = sl.R;
  if constexpr (f8) {
    if (!a_copied) TRY(batch_major(L, A, At, S, R, m, (long long)R * m, R));
    if (!a_is_v) TRY(batch_major(L, V, Vt, S, R, d, (long long)R * d, R));
  }
  const int bk = gemm_bk(AR);
  GemmMaps maps{};
  bool ok = dw_operand_maps(maps.a[0], A, f8 ? &At : nullptr, S, R, m, (uint64_t)R * m, R, bk);
  if (a_is_v) maps.b[0] = maps.a[0];
  else ok = ok && dw_operand_maps(maps.b[0], V, f8 ? &Vt : nullptr, S, R, d, (uint64_t)R * d, R, bk);
  if (!ok) return fail(SCE_ERR_CUDA, "cuTensorMapEncodeTiled failed (row pass: %d x %d, %d slices of %d rows)", m, d, S, R);
  EpiStoreF32::Params sp;
  sp.out = part;
  sp.model_stride = (long long)m * d;
  sp.ld = d;
  sp.scale = 1.f;
  return launch_dw_t<AR>(L, f8, false, S, device, sms, maps, 1, kOnes, kOnes, R, 3, m, d, sp);
}

template <int AR>
static int run_moments_t(Launcher& L, const RowArgs& a, const Slices& sl, const RowCarve& w, double* col_sum,
                         double* gram) {
  TRY(launch_row_split<AR>(L, a, sl, w));
  TRY(sliced_gemm_t<AR>(L, sl, w.x, w.xt, a.d, w.x, w.xt, a.d, w.part, a.device, a.sms));
  return reduce_partials(L, w.part, sl.S, (long long)a.d * a.d / 4, gram, w.col_part,
                         (a.B + kMomBlockRows - 1) / kMomBlockRows, a.d, col_sum);
}

// ------------------------------------------------------------------------------------------------
// FastICA pass (sce_ica_pass): one iteration's data pass of sklearn's parallel FastICA with logcosh, for ICAEncoder
// ------------------------------------------------------------------------------------------------
// For v = x - shift and t = tanh(alpha unmix v): g_sum += sum_b alpha (1 - t_b^2), gx += sum_b t_b v_b^T. The rows are
// split and sliced as for the second moments (launch_row_split: zero padding rows, the range flag). GEMM 1, U = V
// unmix^T, is the encode geometry (both operands K-major over d) as one model of S R rows, with EpiIcaT writing the
// planes of t and the g' partials; GEMM 2, gx = T^T V per slice, is sliced_gemm_t with T in place of the first V.
template <int AR>
static int run_ica_t(Launcher& L, const RowArgs& a, const Slices& sl, const RowCarve& w, const float* unmix, int n,
                     float alpha, double* g_sum, double* gx) {
  constexpr bool f8 = AR == kArithF16F8;
  const int rows = sl.S * sl.R, d = a.d;
  TRY(launch_row_split<AR>(L, a, sl, w));
  TRY(split_matrix<AR>(L, unmix, w.mat, (long long)n * d, w.flags, a.range_flag));   // sce_similarity's raw split
  const uint64_t rows64 = rows, d64 = d, n64 = n;
  const int bk = gemm_bk(AR);
  // ---- GEMM 1: U = V unmix^T, t = tanh(alpha U) -> planes of t, g' partials
  GemmMaps m1{};
  typename EpiIcaT<AR>::Params ep;
  bool ok = operand_maps(m1.a[0], w.x, 1, rows64, d64, rows64 * d64, kBM, bk) &&
            operand_maps(m1.b[0], w.mat, 1, n64, d64, n64 * d64, kBN, bk) &&
            make_tmap_bf16_store32(&ep.out_hi, w.t.hi, 1, rows64, n64, rows64 * n64);
  if constexpr (f8)
    ok = ok && make_tmap_u8_box(&ep.out_lo, w.t.lo, 1, rows64, n64, n64, rows64 * n64, 32, 32, CU_TENSOR_MAP_SWIZZLE_32B) &&
         make_tmap_u8_box(&ep.out_x8, w.t.x8, 1, rows64, n64, n64, rows64 * n64, 32, 32, CU_TENSOR_MAP_SWIZZLE_32B);
  else
    ok = ok && make_tmap_bf16_store32(&ep.out_lo, w.t.lo, 1, rows64, n64, rows64 * n64);
  if (!ok) return fail(SCE_ERR_CUDA, "cuTensorMapEncodeTiled failed (ica pass: d=%d, n=%d, %d rows)", d, n, rows);
  ep.g_part = w.g_part;
  ep.alpha = alpha;
  ep.rows_valid = a.B;
  TRY((launch_gemm_t<EpiIcaT<AR>, false, false, false, AR, f8>(L, 1, a.device, a.sms, m1, 1, kOnes, kOnes, d, 3, rows, n,
                                                                 ep)));
  // ---- GEMM 2: gx partials [S][n][d] = T^T V per slice
  TRY(sliced_gemm_t<AR>(L, sl, w.t, w.tt, n, w.x, w.xt, d, w.part, a.device, a.sms));
  return reduce_partials(L, w.part, sl.S, (long long)n * d / 4, gx, nullptr, 0, 0, nullptr, w.g_part, (a.B + 31) / 32, n,
                         g_sum);
}

// The checks the row passes share, made before any CUDA call: the rows x [B][d], fp16 or fp32, and shift [d], 16-byte
// aligned; the arithmetic (with n components, 0 for the second moments). With `mat_name`, also the fp32 matrix `mat`
// with n rows or columns (ICA's unmix [n][d], NMF's M [k][d] or W [B][k]): present and 16-byte aligned, and n (named
// `n_name`) a multiple of 8 in [8, d].
static int check_row_pass(const char* prefix, const void* x, int x_is_half, int B, int d, const float* shift, int arith,
                          int n = 0, const char* n_name = nullptr, const float* mat = nullptr,
                          const char* mat_name = nullptr) {
  if (!x || !shift) return fail(SCE_ERR_INVALID, "%sx and shift are required", prefix);
  if (x_is_half != 0 && x_is_half != 1) return fail(SCE_ERR_INVALID, "%sx_is_half must be 0 or 1", prefix);
  if (!row_shape_ok(d, B))
    return row_shape_ok(8, B) ? fail(SCE_ERR_INVALID, "%sd (%d) must be a multiple of 8 in [8, 8192]", prefix, d)
                              : fail(SCE_ERR_INVALID, "%sB = %d outside [1, %d]", prefix, B, kMomCallRowsMax);
  if (arith < SCE_ARITH_AUTO || arith > SCE_ARITH_F16F8) return fail(SCE_ERR_INVALID, "%sunknown arith %d", prefix, arith);
  if (arith == SCE_ARITH_F16F8 && (d % 16 || n % 16))
    return n ? fail(SCE_ERR_INVALID, "%sarith = F16F8 needs d (%d) and n (%d) to be multiples of 16", prefix, d, n)
             : fail(SCE_ERR_INVALID, "%sarith = F16F8 needs d (%d) to be a multiple of 16", prefix, d);
  if (reinterpret_cast<uintptr_t>(x) % 16 || reinterpret_cast<uintptr_t>(shift) % 16)
    return fail(SCE_ERR_INVALID, "%sx and shift must be 16-byte aligned", prefix);
  if (mat_name) {
    if (!mat) return fail(SCE_ERR_INVALID, "%s%s is required", prefix, mat_name);
    if (!components_ok(n, d))
      return fail(SCE_ERR_INVALID, "%s%s (%d) must be a multiple of 8 in [8, d = %d]", prefix, n_name, n, d);
    if (reinterpret_cast<uintptr_t>(mat) % 16) return fail(SCE_ERR_INVALID, "%s%s must be 16-byte aligned", prefix, mat_name);
  }
  return SCE_OK;
}

// The prologue every row pass runs after its argument checks: the device, the arithmetic (AUTO: bf16x3, the fp32 range
// and no range check, as sce_similarity), the slices (the projection: one of B rows padded to kMomBlockRows) and the
// carve of the workspace. Then body(AR, L, a, sl, w), with the arithmetic as a compile-time constant.
template <class F>
static int row_pass(RowPass pass, RowArgs a, int n, int arith, void* workspace, void* stream, F&& body) {
  TRY(query_device(&a.device, &a.sms));
  Launcher L{static_cast<cudaStream_t>(stream)};
  const bool f8 = arith == SCE_ARITH_F16F8;
  const Slices sl = pass == kPassNmfProject ? Slices{1, (int)padded_rows(a.B)} : mom_slices(a.d, a.B);
  RowCarve w;
  row_carve(static_cast<uint8_t*>(workspace), pass, f8, a.d, n, a.B, sl.S, (size_t)sl.S * sl.R, &w);
  return with_arith(f8 ? kArithF16F8 : kArithBf16x3, [&](auto ar) { return body(ar, L, a, sl, w); });
}

// ------------------------------------------------------------------------------------------------
// NMF (sce_nmf_project, sce_nmf_grams, sce_nmf_cd_sweep): sklearn's NMF() with the coordinate-descent solver, for
// NMFEncoder
// ------------------------------------------------------------------------------------------------
// Projection: for v = max(x - shift, 0) and an fp32 M [k][d], P = v M^T, fp32 [B][k]. The rows are split as for the row
// passes (CLAMP) into one model of B rows padded to kMomBlockRows; the GEMM is the encode geometry (both operands K-major
// over d), its epilogue EpiNmfProject stores P and, optionally, the per-32-row partials of the squared positive and
// negative parts of each column, which gram_reduce_kernel adds up over the row blocks in order in fp64.
template <int AR>
static int run_nmf_project_t(Launcher& L, const RowArgs& a, const Slices& sl, const RowCarve& w, const float* m, int k,
                             float* p, double* norms) {
  constexpr bool f8 = AR == kArithF16F8;
  const int B = a.B, d = a.d;
  TRY((launch_row_split<AR, true>(L, a, sl, w)));
  TRY(split_matrix<AR>(L, m, w.mat, (long long)k * d, w.flags, a.range_flag));
  const int bk = gemm_bk(AR);
  GemmMaps maps{};
  EpiNmfProject::Params ep;
  bool ok = operand_maps(maps.a[0], w.x, 1, (uint64_t)B, (uint64_t)d, (uint64_t)B * d, kBM, bk) &&
            operand_maps(maps.b[0], w.mat, 1, (uint64_t)k, (uint64_t)d, (uint64_t)k * d, kBN, bk) &&
            make_tmap_f32_store32(&ep.out, p, 1, (uint64_t)B, (uint64_t)k, (uint64_t)B * k);
  if (!ok) return fail(SCE_ERR_CUDA, "cuTensorMapEncodeTiled failed (nmf project: d=%d, k=%d, B=%d)", d, k, B);
  ep.part = norms ? w.part : nullptr;
  TRY((launch_gemm_t<EpiNmfProject, false, false, false, AR, f8>(L, 1, a.device, a.sms, maps, 1, kOnes, kOnes, d, 3, B,
                                                                   k, ep)));
  if (!norms) return SCE_OK;
  return reduce_partials(L, nullptr, 0, 0, nullptr, nullptr, 0, 0, nullptr, w.part, (B + 31) / 32, 2 * k, norms);
}

// Gram matrices: for v as above and an fp32 W [B][k], wtw += W^T W and wtv += W^T v (fp64). The sliced row reduction of
// the second moments: v and W are split into the planes of S slices of R rows (padding rows zero), each slice's two
// products run on the weight gradient's GEMM (sliced_gemm_t: W^T W with A = V = W, then W^T v), and gram_reduce_kernel
// adds the slice partials in slice order in fp64.
template <int AR>
static int run_nmf_grams_t(Launcher& L, const RowArgs& a, const Slices& sl, const RowCarve& w, const float* wm, int k,
                           double* wtw, double* wtv) {
  const long long rows = (long long)sl.S * sl.R;
  TRY((launch_row_split<AR, true>(L, a, sl, w)));
  TRY(split_matrix<AR>(L, wm, w.t, (long long)a.B * k, w.flags, a.range_flag));
  if (rows > a.B) CUDA_TRY(w.t.at((size_t)a.B * k).zero((size_t)(rows - a.B) * k, L.st));
  TRY(sliced_gemm_t<AR>(L, sl, w.t, w.tt, k, w.t, w.tt, k, w.part_g, a.device, a.sms));
  TRY(sliced_gemm_t<AR>(L, sl, w.t, w.tt, k, w.x, w.xt, a.d, w.part, a.device, a.sms, true));   // W's copies: made above
  TRY(reduce_partials(L, w.part_g, sl.S, (long long)k * k / 4, wtw));
  return reduce_partials(L, w.part, sl.S, (long long)k * a.d / 4, wtv);
}


// One coordinate-descent sweep (sklearn's _update_cdnmf_fast, coordinates in order, no regularisation) over the rows
// of W [R][k], with G [k][k] and L [R][k] fixed: for t = 0 .. k-1, per row i,
//   grad = sum_r G[t][r] W[i][r] - L[i][t];  pg = W[i][t] == 0 ? min(grad, 0) : grad;  violation += |pg|
//   G[t][t] != 0: W[i][t] = max(W[i][t] - grad / G[t][t], 0)
// The rows are independent, so each is swept by one warp, which keeps the row and its gradient g = W G - L in
// registers: lane l holds the columns VW l + 32 VW q + e (q < KPL / VW, e < VW; VW = min(KPL, 4) consecutive columns,
// so that a lane reads its share of a row of G as one 16-byte load). Per coordinate, the owning lane takes the step and
// broadcasts the change delta with one shuffle; only when delta != 0 (a code entry that stays at 0 changes nothing) do
// the lanes add delta G[t][:] to g. g starts as -L plus W[r] G[r][:] for the non-zero W[r] (skipped for a block whose
// rows are all zero, as transform's first sweep). The blocks' kCdWarps warps share rows of G, staged in shared memory
// `tb` rows at a time. T is the arithmetic of W, G, L and g; the violation is fp64. No atomics: each lane sums its
// coordinates in order, the warp and the block add in a fixed order, and nmf_violation_kernel adds the block partials
// in block order.
// With n_iter (transform's loop), a sweep is a no-op once the stop rule held after the previous one.
constexpr int kCdWarps = 8;
constexpr int kCdMaxK = 2048;

__device__ __forceinline__ bool nmf_stopped(const double* viol, const int* n_iter, double tol) {
  if (!n_iter || *n_iter < 1) return false;
  return viol[0] == 0.0 || viol[1] / viol[0] <= tol;
}

template <class T, int VW>
__device__ __forceinline__ void load_vec(const T* p, T (&v)[VW]) {
  if constexpr (VW == 4 && sizeof(T) == 4) {
    const float4 a = *reinterpret_cast<const float4*>(p);
    v[0] = a.x, v[1] = a.y, v[2] = a.z, v[3] = a.w;
  } else if constexpr (VW >= 2 && VW % 2 == 0 && sizeof(T) == 8) {
#pragma unroll
    for (int e = 0; e < VW; e += 2) {
      const double2 a = *reinterpret_cast<const double2*>(p + e);
      v[e] = a.x, v[e + 1] = a.y;
    }
  } else {
#pragma unroll
    for (int e = 0; e < VW; ++e) v[e] = p[e];
  }
}

// g += a row[:] over the lane's columns (row: a staged row of G, 32 KPL entries)
template <class T, int KPL>
__device__ __forceinline__ void cd_axpy(T (&g)[KPL], T a, const T* row, int lane) {
  constexpr int VW = KPL < 4 ? KPL : 4;
#pragma unroll
  for (int q = 0; q < KPL / VW; ++q) {
    T v[VW];
    load_vec<T, VW>(row + 32 * VW * q + VW * lane, v);
#pragma unroll
    for (int e = 0; e < VW; ++e) g[q * VW + e] = fma(a, v[e], g[q * VW + e]);
  }
}

template <class T, int KPL>
__global__ void __launch_bounds__(kCdWarps * 32) nmf_cd_sweep_kernel(T* __restrict__ w, int R, int k,
                                                                    const T* __restrict__ G, const T* __restrict__ Lm,
                                                                    int tb, double* __restrict__ part,
                                                                    const double* __restrict__ viol,
                                                                    const int* __restrict__ n_iter, double tol) {
  if (nmf_stopped(viol, n_iter, tol)) return;   // (block-uniform)
  constexpr int VW = KPL < 4 ? KPL : 4, KP = 32 * KPL;
  extern __shared__ __align__(16) unsigned char cd_smem[];
  T* gs = reinterpret_cast<T*>(cd_smem);   // [tb][KP]: rows t0 .. t0 + tb - 1 of G, zero beyond k
  __shared__ double wsum[kCdWarps];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long long row = (long long)blockIdx.x * kCdWarps + warp;
  const bool live = row < R;
  T wr[KPL], g[KPL];
  bool nonzero = false;
#pragma unroll
  for (int q = 0; q < KPL / VW; ++q)
#pragma unroll
    for (int e = 0; e < VW; ++e) {
      const int j = 32 * VW * q + VW * lane + e;
      const bool ok = live && j < k;
      wr[q * VW + e] = ok ? w[row * k + j] : T(0);
      g[q * VW + e] = ok ? -Lm[row * k + j] : T(0);
      nonzero |= wr[q * VW + e] != T(0);
    }
  auto stage = [&](int t0) {
    __syncthreads();
    for (int i = threadIdx.x; i < tb * KP; i += blockDim.x) {
      const int t = t0 + i / KP, c = i % KP;
      gs[i] = t < k && c < k ? G[(long long)t * k + c] : T(0);
    }
    __syncthreads();
  };
  const int sb = tb / VW;   // lane groups per staged block (tb is a multiple of VW and divides 32 VW)
  // ---- g = W G - L
  if (__syncthreads_or(nonzero)) {
#pragma unroll
    for (int q = 0; q < KPL / VW; ++q) {
      for (int s0 = 0; s0 < 32 && 32 * VW * q + VW * s0 < k; s0 += sb) {
        const int t0 = 32 * VW * q + VW * s0;
        stage(t0);
        for (int s = s0; s < s0 + sb; ++s) {
#pragma unroll
          for (int e = 0; e < VW; ++e) {
            const T a = __shfl_sync(0xffffffffu, wr[q * VW + e], s);
            if (a != T(0)) cd_axpy<T, KPL>(g, a, gs + (VW * (s - s0) + e) * KP, lane);
          }
        }
      }
    }
  }
  // ---- the sweep
  double v = 0.0;
#pragma unroll
  for (int q = 0; q < KPL / VW; ++q) {
    for (int s0 = 0; s0 < 32 && 32 * VW * q + VW * s0 < k; s0 += sb) {
      const int t0 = 32 * VW * q + VW * s0;
      stage(t0);
      for (int s = s0; s < s0 + sb; ++s) {
#pragma unroll
        for (int e = 0; e < VW; ++e) {
          const T* grow = gs + (VW * (s - s0) + e) * KP;
          const int t = t0 + VW * (s - s0) + e;
          const T hess = grow[t];   // G[t][t] (t < KP)
          T delta = T(0);
          if (lane == s) {
            const T gt = g[q * VW + e], wt = wr[q * VW + e];
            const T pg = wt == T(0) ? (gt < T(0) ? gt : T(0)) : gt;
            v += fabs((double)pg);
            if (hess != T(0)) {
              const T u = wt - gt / hess;
              const T wn = u > T(0) ? u : T(0);
              delta = wn - wt;
              wr[q * VW + e] = wn;
            }
          }
          delta = __shfl_sync(0xffffffffu, delta, s);
          if (delta != T(0)) cd_axpy<T, KPL>(g, delta, grow, lane);
        }
      }
    }
  }
  if (live) {
#pragma unroll
    for (int q = 0; q < KPL / VW; ++q)
#pragma unroll
      for (int e = 0; e < VW; ++e) {
        const int j = 32 * VW * q + VW * lane + e;
        if (j < k) w[row * k + j] = wr[q * VW + e];
      }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if (lane == 0) wsum[warp] = v;
  __syncthreads();
  if (threadIdx.x == 0) {
    double b = 0.0;
#pragma unroll
    for (int i = 0; i < kCdWarps; ++i) b += wsum[i];
    part[blockIdx.x] = b;
  }
}

// The sweep's violation: the block partials added in block order. Without n_iter, violation[0] += it. With n_iter
// (transform's loop): unless the stop rule already held, ++n_iter, violation[1] = it and, on the first sweep,
// violation[0] = it.
__global__ void __launch_bounds__(256) nmf_violation_kernel(const double* __restrict__ part, int blocks, double* viol,
                                                            int* n_iter, double tol) {
  if (nmf_stopped(viol, n_iter, tol)) return;
  __shared__ double s[256];
  double a = 0.0;
  for (int i = threadIdx.x; i < blocks; i += 256) a += part[i];
  s[threadIdx.x] = a;
  __syncthreads();
  for (int h = 128; h > 0; h >>= 1) {
    if (threadIdx.x < h) s[threadIdx.x] += s[threadIdx.x + h];
    __syncthreads();
  }
  if (threadIdx.x) return;
  if (!n_iter) {
    viol[0] += s[0];
    return;
  }
  const int it = *n_iter + 1;
  *n_iter = it;
  if (it == 1) viol[0] = s[0];
  viol[1] = s[0];
}

// Residual (sce_nmf_residual): sum over the rows of ||max(x - shift, 0) - w h||^2 for W [B][k] and H [k][d] fp32, the fit's
// reconstruction_err_. A plain fp32 SIMT product, not the split-operand GEMM: at a good fit the residual is ~1e-3 of
// the rows, and products good to 2^-16 (bf16x3) would leave its square with no correct digit. Block tile 64 rows x 64
// columns, 4 x 4 per thread, k in steps of 16 through shared memory; squares in fp64, one partial per block (added in
// block order by nmf_violation_kernel).
constexpr int kResTile = 64, kResK = 16;
template <class InT>
__global__ void __launch_bounds__(256) nmf_residual_kernel(const InT* __restrict__ x, int B, int d,
                                                           const float* __restrict__ shift, const float* __restrict__ w,
                                                           int k, const float* __restrict__ h, double* __restrict__ part) {
  __shared__ float ws[kResK][kResTile + 4];
  __shared__ float hs[kResK][kResTile];
  __shared__ double red[8];
  const int tx = threadIdx.x % 16, ty = threadIdx.x / 16;
  const long long r0 = (long long)blockIdx.y * kResTile;
  const int c0 = blockIdx.x * kResTile;
  float acc[4][4] = {};
  for (int k0 = 0; k0 < k; k0 += kResK) {
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int i = threadIdx.x + 256 * q;
      const int wr = i / kResK, wk = i % kResK, hk = i / kResTile, hc = i % kResTile;
      const long long r = r0 + wr;
      ws[wk][wr] = r < B && k0 + wk < k ? w[r * k + k0 + wk] : 0.f;
      hs[hk][hc] = k0 + hk < k && c0 + hc < d ? h[(long long)(k0 + hk) * d + c0 + hc] : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < kResK; ++kk) {
      float a[4], b[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) a[i] = ws[kk][ty * 4 + i], b[i] = hs[kk][tx * 4 + i];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }
  double s = 0.0;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const long long r = r0 + ty * 4 + i;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int c = c0 + tx * 4 + j;
      if (r < B && c < d) {
        float v = (float)x[r * d + c] - shift[c];
        v = v < 0.f ? 0.f : v;
        const double e = (double)v - (double)acc[i][j];
        s += e * e;
      }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
#pragma unroll
    for (int i = 0; i < 8; ++i) t += red[i];
    part[(long long)blockIdx.y * gridDim.x + blockIdx.x] = t;
  }
}

// the shared-memory rows of G per staged block: a power of two, a multiple of VW, at most 32 VW, within 48 KB where VW
// rows fit
static int cd_stage_rows(int kpl, size_t elem) {
  const int vw = kpl < 4 ? kpl : 4;
  const size_t row = (size_t)32 * kpl * elem;
  int tb = vw;
  while (tb * 2 <= 32 * vw && (size_t)tb * 2 * row <= 48 * 1024) tb *= 2;
  return tb;
}

template <class T, int KPL>
static int launch_cd_t(Launcher& L, T* w, int R, int k, const T* G, const T* Lm, double* part, double* viol, int* n_iter,
                       double tol) {
  const int tb = cd_stage_rows(KPL, sizeof(T));
  const size_t smem = (size_t)tb * 32 * KPL * sizeof(T);
  if (smem > 48 * 1024)
    CUDA_TRY(cudaFuncSetAttribute(nmf_cd_sweep_kernel<T, KPL>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const int blocks = (R + kCdWarps - 1) / kCdWarps;
  TRY(L.launch(nmf_cd_sweep_kernel<T, KPL>, blocks, kCdWarps * 32, smem, w, R, k, G, Lm, tb, part, viol, n_iter, tol));
  return L.launch(nmf_violation_kernel, 1, 256, 0, part, blocks, viol, n_iter, tol);
}

// columns per lane: ceil(k / 32) rounded up to a power of two
template <class T>
static int launch_cd(Launcher& L, T* w, int R, int k, const T* G, const T* Lm, double* part, double* viol, int* n_iter,
                     double tol) {
  const int c = (k + 31) / 32;
  if (c <= 1) return launch_cd_t<T, 1>(L, w, R, k, G, Lm, part, viol, n_iter, tol);
  if (c <= 2) return launch_cd_t<T, 2>(L, w, R, k, G, Lm, part, viol, n_iter, tol);
  if (c <= 4) return launch_cd_t<T, 4>(L, w, R, k, G, Lm, part, viol, n_iter, tol);
  if (c <= 8) return launch_cd_t<T, 8>(L, w, R, k, G, Lm, part, viol, n_iter, tol);
  if (c <= 16) return launch_cd_t<T, 16>(L, w, R, k, G, Lm, part, viol, n_iter, tol);
  if (c <= 32) return launch_cd_t<T, 32>(L, w, R, k, G, Lm, part, viol, n_iter, tol);
  return launch_cd_t<T, 64>(L, w, R, k, G, Lm, part, viol, n_iter, tol);
}

extern "C" {

size_t sce_second_moments_workspace_bytes(int d, int B) { return row_pass_workspace(kPassMoments, d, 0, B); }

int sce_second_moments(const void* x, int x_is_half, int B, int d, const float* shift, int arith, double* col_sum,
                       double* gram, unsigned int* range_flag, void* workspace, size_t workspace_bytes, void* stream) {
  // ---- arguments (all checked before any CUDA call)
  if (!col_sum || !gram) return fail(SCE_ERR_INVALID, "second_moments: col_sum and gram are required");
  TRY(check_row_pass("second_moments: ", x, x_is_half, B, d, shift, arith));
  if (reinterpret_cast<uintptr_t>(gram) % 16) return fail(SCE_ERR_INVALID, "second_moments: gram must be 16-byte aligned");
  TRY(check_workspace(workspace, workspace_bytes, sce_second_moments_workspace_bytes(d, B), "second_moments: "));
  return row_pass(kPassMoments, {x, x_is_half == 1, B, d, shift, range_flag}, 0, arith, workspace, stream,
                  [&](auto ar, auto&... r) { return run_moments_t<decltype(ar)::value>(r..., col_sum, gram); });
}

size_t sce_ica_pass_workspace_bytes(int d, int n, int B) { return row_pass_workspace(kPassIca, d, n, B); }

int sce_ica_pass(const void* x, int x_is_half, int B, int d, const float* shift, const float* unmix, int n, float alpha,
                 int arith, double* g_sum, double* gx, unsigned int* range_flag, void* workspace, size_t workspace_bytes,
                 void* stream) {
  // ---- arguments (all checked before any CUDA call)
  if (!g_sum || !gx) return fail(SCE_ERR_INVALID, "ica_pass: g_sum and gx are required");
  TRY(check_row_pass("ica_pass: ", x, x_is_half, B, d, shift, arith, n, "n", unmix, "unmix"));
  if (!(alpha >= 1.f && alpha <= 2.f)) return fail(SCE_ERR_INVALID, "ica_pass: alpha (%g) must be in [1, 2]", (double)alpha);
  if (reinterpret_cast<uintptr_t>(gx) % 16 || reinterpret_cast<uintptr_t>(g_sum) % 8)
    return fail(SCE_ERR_INVALID, "ica_pass: gx must be 16-byte aligned, g_sum 8-byte aligned");
  TRY(check_workspace(workspace, workspace_bytes, sce_ica_pass_workspace_bytes(d, n, B), "ica_pass: "));
  return row_pass(kPassIca, {x, x_is_half == 1, B, d, shift, range_flag}, n, arith, workspace, stream,
                  [&](auto ar, auto&... r) { return run_ica_t<decltype(ar)::value>(r..., unmix, n, alpha, g_sum, gx); });
}

size_t sce_nmf_project_workspace_bytes(int d, int k, int B) { return row_pass_workspace(kPassNmfProject, d, k, B); }

int sce_nmf_project(const void* x, int x_is_half, int B, int d, const float* shift, const float* m, int k, int arith,
                    float* p, double* norms, unsigned int* range_flag, void* workspace, size_t workspace_bytes,
                    void* stream) {
  // ---- arguments (all checked before any CUDA call)
  if (!p) return fail(SCE_ERR_INVALID, "nmf_project: p is required");
  TRY(check_row_pass("nmf_project: ", x, x_is_half, B, d, shift, arith, k, "k", m, "m"));
  if (reinterpret_cast<uintptr_t>(p) % 16 || reinterpret_cast<uintptr_t>(norms) % 8)
    return fail(SCE_ERR_INVALID, "nmf_project: p must be 16-byte aligned, norms 8-byte aligned");
  TRY(check_workspace(workspace, workspace_bytes, sce_nmf_project_workspace_bytes(d, k, B), "nmf_project: "));
  return row_pass(kPassNmfProject, {x, x_is_half == 1, B, d, shift, range_flag}, k, arith, workspace, stream,
                  [&](auto ar, auto&... r) { return run_nmf_project_t<decltype(ar)::value>(r..., m, k, p, norms); });
}

size_t sce_nmf_grams_workspace_bytes(int d, int k, int B) { return row_pass_workspace(kPassNmfGrams, d, k, B); }

int sce_nmf_grams(const void* x, int x_is_half, int B, int d, const float* shift, const float* w, int k, int arith,
                  double* wtw, double* wtv, unsigned int* range_flag, void* workspace, size_t workspace_bytes,
                  void* stream) {
  // ---- arguments (all checked before any CUDA call)
  if (!wtw || !wtv) return fail(SCE_ERR_INVALID, "nmf_grams: wtw and wtv are required");
  TRY(check_row_pass("nmf_grams: ", x, x_is_half, B, d, shift, arith, k, "k", w, "w"));
  if (reinterpret_cast<uintptr_t>(wtw) % 16 || reinterpret_cast<uintptr_t>(wtv) % 16)
    return fail(SCE_ERR_INVALID, "nmf_grams: wtw and wtv must be 16-byte aligned");
  TRY(check_workspace(workspace, workspace_bytes, sce_nmf_grams_workspace_bytes(d, k, B), "nmf_grams: "));
  return row_pass(kPassNmfGrams, {x, x_is_half == 1, B, d, shift, range_flag}, k, arith, workspace, stream,
                  [&](auto ar, auto&... r) { return run_nmf_grams_t<decltype(ar)::value>(r..., w, k, wtw, wtv); });
}

size_t sce_nmf_cd_sweep_workspace_bytes(int k, int R) {
  if (k < 1 || k > kCdMaxK || R < 1) return 0;
  return align_up((size_t)((R + kCdWarps - 1) / kCdWarps) * sizeof(double), 1024);
}

int sce_nmf_cd_sweep(void* w, int w_is_f64, int R, int k, const void* g, const void* l, int max_sweeps, double tol,
                     double* violation, int* n_iter, void* workspace, size_t workspace_bytes, void* stream) {
  // ---- arguments (all checked before any CUDA call)
  if (!w || !g || !l || !violation) return fail(SCE_ERR_INVALID, "nmf_cd_sweep: w, g, l and violation are required");
  if (w_is_f64 != 0 && w_is_f64 != 1) return fail(SCE_ERR_INVALID, "nmf_cd_sweep: w_is_f64 must be 0 or 1");
  if (R < 1) return fail(SCE_ERR_INVALID, "nmf_cd_sweep: R (%d) must be >= 1", R);
  if (k < 1 || k > kCdMaxK) return fail(SCE_ERR_INVALID, "nmf_cd_sweep: k (%d) must be in [1, %d]", k, kCdMaxK);
  if (max_sweeps < 1 || (!n_iter && max_sweeps != 1))
    return fail(SCE_ERR_INVALID, "nmf_cd_sweep: max_sweeps (%d) must be 1 without n_iter, >= 1 with it", max_sweeps);
  if (!(tol >= 0.0 && tol <= 1e300)) return fail(SCE_ERR_INVALID, "nmf_cd_sweep: tol must be finite and >= 0");
  const size_t elem = w_is_f64 ? 8 : 4;
  if (reinterpret_cast<uintptr_t>(w) % elem || reinterpret_cast<uintptr_t>(g) % elem ||
      reinterpret_cast<uintptr_t>(l) % elem || reinterpret_cast<uintptr_t>(violation) % 8 ||
      reinterpret_cast<uintptr_t>(n_iter) % 4)
    return fail(SCE_ERR_INVALID, "nmf_cd_sweep: w, g, l, violation and n_iter must be aligned to their elements");
  TRY(check_workspace(workspace, workspace_bytes, sce_nmf_cd_sweep_workspace_bytes(k, R), "nmf_cd_sweep: "));

  // ---- device
  Launcher L{static_cast<cudaStream_t>(stream)};
  double* part = static_cast<double*>(workspace);
  if (n_iter) {
    CUDA_TRY(cudaMemsetAsync(violation, 0, 2 * sizeof(double), L.st));
    CUDA_TRY(cudaMemsetAsync(n_iter, 0, sizeof(int), L.st));
  }
  for (int s = 0; s < max_sweeps; ++s) {
    if (w_is_f64)
      TRY(launch_cd(L, static_cast<double*>(w), R, k, static_cast<const double*>(g), static_cast<const double*>(l), part,
                    violation, n_iter, tol));
    else
      TRY(launch_cd(L, static_cast<float*>(w), R, k, static_cast<const float*>(g), static_cast<const float*>(l), part,
                    violation, n_iter, tol));
  }
  return SCE_OK;
}


size_t sce_nmf_residual_workspace_bytes(int d, int B) {
  if (!row_shape_ok(d, B)) return 0;
  return align_up((size_t)((d + kResTile - 1) / kResTile) * ((B + kResTile - 1) / kResTile) * sizeof(double), 1024);
}

int sce_nmf_residual(const void* x, int x_is_half, int B, int d, const float* shift, const float* w, int k,
                     const float* h, double* sum, void* workspace, size_t workspace_bytes, void* stream) {
  // ---- arguments (all checked before any CUDA call)
  if (!h || !sum) return fail(SCE_ERR_INVALID, "nmf_residual: h and sum are required");
  TRY(check_row_pass("nmf_residual: ", x, x_is_half, B, d, shift, SCE_ARITH_AUTO, k, "k", w, "w"));
  if (reinterpret_cast<uintptr_t>(h) % 16 || reinterpret_cast<uintptr_t>(sum) % 8)
    return fail(SCE_ERR_INVALID, "nmf_residual: h must be 16-byte aligned, sum 8-byte aligned");
  TRY(check_workspace(workspace, workspace_bytes, sce_nmf_residual_workspace_bytes(d, B), "nmf_residual: "));

  // ---- device
  Launcher L{static_cast<cudaStream_t>(stream)};
  double* part = static_cast<double*>(workspace);
  const dim3 grid((d + kResTile - 1) / kResTile, (B + kResTile - 1) / kResTile);
  if (x_is_half)
    TRY(L.launch(nmf_residual_kernel<__half>, grid, 256, 0, static_cast<const __half*>(x), B, d, shift, w, k, h, part));
  else
    TRY(L.launch(nmf_residual_kernel<float>, grid, 256, 0, static_cast<const float*>(x), B, d, shift, w, k, h, part));
  return L.launch(nmf_violation_kernel, 1, 256, 0, part, (int)(grid.x * grid.y), sum, nullptr, 0.0);
}

}  // extern "C"
