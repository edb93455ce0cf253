// sce_correlation.cu — the cross-code moments of two plans' last calls (sce_cross_moments) and the correlation,
// covariance and best matches they give (sce_correlation_finish).
#include <math.h>

#include "sce_plan.cuh"

// ------------------------------------------------------------------------------------------------
// cross-code moments: acc[i][j] += C_a[i]^T C_b[j] over the rows of the two plans' last calls
// ------------------------------------------------------------------------------------------------
// The operands are the code planes each plan's encode epilogue (top-k: its selection) wrote, [M][batch_max][n] row-major:
// for a reduction over the rows that is the weight gradient's MN-major geometry (K = rows), so the product runs on its
// GEMM, with f16f8's 8-bit tiles widened to fp16 as in the top-k plans' weight gradient. The rows are cut into slices of
// at most kCrossRowsMax. Each slice is summed in fp32 on the tensor cores into one fp32 partial [n_a][n_b], which
// cross_add_kernel adds into the fp64 accumulator before the next slice runs: the truncation bias of fp32 tensor-core
// accumulation grows with K, and a sum of products of non-negative codes never cancels it (see sce_rowpass.cu). One
// partial, reused slice after slice, keeps the workspace at 4 n_a n_b bytes whatever B; the slices and pairs run in a
// fixed order, so results are bitwise repeatable.
constexpr int kCrossRowsMax = 2048;
constexpr int kCrossSliceAlign = 64;   // slice starts stay 16-byte aligned in every plane (n % 8 == 0; f16f8 n % 16 == 0)

// acc[i] += part[i] in fp64, four entries per thread (n4 float4s)
__global__ void __launch_bounds__(256) cross_add_kernel(const float* __restrict__ part, long long n4, double* __restrict__ acc) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
    const float4 v = __ldg(reinterpret_cast<const float4*>(part) + i);
    double* a = acc + 4 * i;
    a[0] += v.x;
    a[1] += v.y;
    a[2] += v.z;
    a[3] += v.w;
  }
}

// The two plans of a cross-moments call and of its workspace query: each evaluable, one arithmetic, one device
static int check_cross_plans(const sce_plan* a, const sce_plan* b) {
  TRY(check_evaluable(a, "cross_moments: plan_a: "));
  TRY(check_evaluable(b, "cross_moments: plan_b: "));
  if (a->cfg.arith != b->cfg.arith)
    return fail(SCE_ERR_INVALID, "cross_moments: the two plans resolved to different arithmetics");
  if (a->device != b->device) return fail(SCE_ERR_INVALID, "cross_moments: the two plans live on different devices");
  return SCE_OK;
}

template <int AR>
static int run_cross_t(Launcher& L, const sce_plan* pa, const sce_plan* pb, int B, double* acc, float* part) {
  const int na = pa->d.n, nb = pb->d.n, bk = gemm_bk(AR);
  const int S = (B + kCrossRowsMax - 1) / kCrossRowsMax;
  const int R = ((B + S - 1) / S + kCrossSliceAlign - 1) / kCrossSliceAlign * kCrossSliceAlign;
  const long long n4 = (long long)na * nb / 4;
  const int blocks = (int)((n4 + 255) / 256 < 2048 ? (n4 + 255) / 256 : 2048);
  EpiStoreF32::Params sp;
  sp.out = part;
  sp.model_stride = (long long)na * nb;
  sp.ld = nb;
  sp.scale = 1.f;
  for (int i = 0; i < pa->d.n_models; ++i)
    for (int j = 0; j < pb->d.n_models; ++j) {
      double* out = acc + ((long long)i * pb->d.n_models + j) * na * nb;
      for (int r0 = 0; r0 < B; r0 += R) {
        const int rows = B - r0 < R ? B - r0 : R;
        const Planes A = pa->c.at(((size_t)i * pa->d.batch_max + r0) * na);
        const Planes Bp = pb->c.at(((size_t)j * pb->d.batch_max + r0) * nb);
        GemmMaps maps{};
        if (!dw_operand_maps(maps.a[0], A, nullptr, 1, rows, na, (uint64_t)rows * na, 0, bk) ||
            !dw_operand_maps(maps.b[0], Bp, nullptr, 1, rows, nb, (uint64_t)rows * nb, 0, bk))
          return fail(SCE_ERR_CUDA, "cuTensorMapEncodeTiled failed (cross moments: %d x %d, %d rows)", na, nb, rows);
        TRY(launch_dw_t<AR>(L, false, false, 1, pa->device, pa->sms, maps, 1, kOnes, kOnes, rows, 3, na, nb, sp));
        TRY(L.launch(cross_add_kernel, blocks, 256, 0, part, n4, out));
      }
    }
  return SCE_OK;
}

// ------------------------------------------------------------------------------------------------
// correlation from the fp64 sums, and each feature's best match on the other side
// ------------------------------------------------------------------------------------------------
// Population moments over `rows` rows in fp64: mean = s1 / N, var = s2 / N - mean^2, cov = s_ab / N - mean_a mean_b,
// corr = cov / sqrt(var_a var_b), NaN unless both variances are positive. Both reductions below evaluate this one
// function, so the maxima equal the stored correlation entries.
struct CorrArgs {
  const double* acc;        // [n_a][lda]
  int n_a, n_b, lda;
  const double* sums_a;     // [n_a][4] moment sums (s1 at [4 j], s2 at [4 j + 1])
  const double* sums_b;     // [n_b][4]
  double n;                // rows, N
};

__device__ __forceinline__ void feature_moments(const double* sums, int j, double n, double& mean, double& var) {
  mean = sums[4 * (long long)j] / n;
  var = sums[4 * (long long)j + 1] / n - mean * mean;
}

__device__ __forceinline__ double corr_entry(const CorrArgs& a, double s, double ma, double va, double mb, double vb,
                                             double& cov) {
  cov = s / a.n - ma * mb;
  return va > 0.0 && vb > 0.0 ? cov / sqrt(va * vb) : (double)NAN;
}

// (v, i) replaces (bv, bi) when v is larger, or equal with a lower index; NaN never does, and bi = -1 is empty
__device__ __forceinline__ void better(double v, long long i, double& bv, long long& bi) {
  if (isnan(v) || i < 0) return;
  if (bi < 0 || v > bv || (v == bv && i < bi)) {
    bv = v;
    bi = i;
  }
}

// One block per row r of a: corr[r][:] and cov[r][:] (each where given) and the row's best column
__global__ void __launch_bounds__(256) corr_rows_kernel(CorrArgs a, float* __restrict__ corr, float* __restrict__ cov,
                                                        float* __restrict__ max_ab, long long* __restrict__ arg_ab) {
  __shared__ double sv[8];
  __shared__ long long si[8];
  const int r = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  double ma, va;
  feature_moments(a.sums_a, r, a.n, ma, va);
  double bv = 0.0;
  long long bi = -1;
  for (int c = threadIdx.x; c < a.n_b; c += blockDim.x) {
    double mb, vb, cv;
    feature_moments(a.sums_b, c, a.n, mb, vb);
    const double v = corr_entry(a, a.acc[(long long)r * a.lda + c], ma, va, mb, vb, cv);
    if (corr) corr[(long long)r * a.n_b + c] = (float)v;
    if (cov) cov[(long long)r * a.n_b + c] = (float)cv;
    better(v, c, bv, bi);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const double ov = __shfl_xor_sync(0xffffffffu, bv, o);
    const long long oi = __shfl_xor_sync(0xffffffffu, bi, o);
    better(ov, oi, bv, bi);
  }
  if (lane == 0) sv[warp] = bv, si[warp] = bi;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < 8; ++w) better(sv[w], si[w], bv, bi);
    max_ab[r] = bi < 0 ? NAN : (float)bv;
    arg_ab[r] = bi;
  }
}

// 32 columns of b per block, 8 warps over the rows of a (warp w: rows w, w + 8, ...): each column's best row
__global__ void __launch_bounds__(256) corr_cols_kernel(CorrArgs a, float* __restrict__ max_ba, long long* __restrict__ arg_ba) {
  __shared__ double sv[8][32];
  __shared__ long long si[8][32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, c = blockIdx.x * 32 + lane;
  double bv = 0.0;
  long long bi = -1;
  if (c < a.n_b) {
    double mb, vb;
    feature_moments(a.sums_b, c, a.n, mb, vb);
    for (int r = warp; r < a.n_a; r += 8) {
      double ma, va, cv;
      feature_moments(a.sums_a, r, a.n, ma, va);
      better(corr_entry(a, a.acc[(long long)r * a.lda + c], ma, va, mb, vb, cv), r, bv, bi);
    }
  }
  sv[warp][lane] = bv;
  si[warp][lane] = bi;
  __syncthreads();
  if (warp == 0 && c < a.n_b) {
    for (int w = 1; w < 8; ++w) better(sv[w][lane], si[w][lane], bv, bi);
    max_ba[c] = bi < 0 ? NAN : (float)bv;
    arg_ba[c] = bi;
  }
}

extern "C" {

size_t sce_cross_moments_workspace_bytes(const sce_plan* a, const sce_plan* b, int B) {
  if (!a || !b || check_cross_plans(a, b) || B < 1 || B > a->d.batch_max || B > b->d.batch_max) return 0;
  return align_up((size_t)a->d.n * b->d.n * sizeof(float), 1024);
}

int sce_cross_moments(sce_plan* a, sce_plan* b, int B, double* acc, void* workspace, size_t workspace_bytes,
                      void* stream) {
  // ---- arguments (all checked before any CUDA call)
  if (!a || !b || !acc) return fail(SCE_ERR_INVALID, "cross_moments: plan_a, plan_b and acc are required");
  TRY(check_cross_plans(a, b));
  TRY(check_rows(a, B, "cross_moments: plan_a: "));
  TRY(check_rows(b, B, "cross_moments: plan_b: "));
  TRY(check_forward_code(a, "cross_moments: plan_a: "));
  TRY(check_forward_code(b, "cross_moments: plan_b: "));
  if (reinterpret_cast<uintptr_t>(acc) % 8) return fail(SCE_ERR_INVALID, "cross_moments: acc must be 8-byte aligned");
  TRY(check_workspace(workspace, workspace_bytes, sce_cross_moments_workspace_bytes(a, b, B), "cross_moments: "));

  // ---- device
  Launcher L{static_cast<cudaStream_t>(stream)};
  float* part = static_cast<float*>(workspace);
  return with_arith(a->cfg.arith, [&](auto ar) { return run_cross_t<decltype(ar)::value>(L, a, b, B, acc, part); });
}

int sce_correlation_finish(const double* acc, int n_a, int n_b, int lda, const double* sums_a, const double* sums_b,
                           long long rows, float* corr, float* cov, float* max_ab, long long* arg_ab, float* max_ba,
                           long long* arg_ba, void* stream) {
  // ---- arguments (all checked before any CUDA call)
  if (!acc || !sums_a || !sums_b || !max_ab || !arg_ab || !max_ba || !arg_ba)
    return fail(SCE_ERR_INVALID, "correlation_finish: acc, sums_a, sums_b and the four maxima outputs are required");
  if (n_a < 1 || n_b < 1 || lda < n_b)
    return fail(SCE_ERR_INVALID, "correlation_finish: need n_a, n_b >= 1 and lda >= n_b (got %d, %d, %d)", n_a, n_b, lda);
  if (rows < 1) return fail(SCE_ERR_INVALID, "correlation_finish: rows (%lld) must be >= 1", rows);

  // ---- device
  Launcher L{static_cast<cudaStream_t>(stream)};
  const CorrArgs args{acc, n_a, n_b, lda, sums_a, sums_b, (double)rows};
  TRY(L.launch(corr_rows_kernel, n_a, 256, 0, args, corr, cov, max_ab, arg_ab));
  return L.launch(corr_cols_kernel, (n_b + 31) / 32, 256, 0, args, max_ba, arg_ba);
}

}  // extern "C"
