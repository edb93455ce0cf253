// sce_plan.cu — the plan and its training step: the entry points of include/sce.h that create, prepare, step and
// inspect an sce_plan, on top of the wgmma GEMM core and the streaming kernels. One `sce_plan` = one stacked ensemble
// (FunctionalEnsemble, autoencoders/ensemble.py:68-97). The entry points that read a call's code back are in
// sce_eval.cu, dead-feature tracking is in sce_track.cu, and what the three files share is in sce_plan.cuh.
//
// One training step (tied variant; untied and top-k differ as noted; "planes" are the operand planes of the plan's
// arithmetic, see Planes: fp16 + two E5M2 planes with f16f8, a bf16 pair with bf16x3) is
//   split_rows      x -> x planes  [+ residual-plane flag, input range monitor]
//   GEMM encode     z = x W^T (+b) -> relu -> c planes, activity masks, sum|c|, nnz   [M x B x n, K = d]
//   GEMM decode     x^ = c W -> r = x^ - x, sum r^2, g = 2r/(Bd) -> g planes  [M x B x d, K = n]
//   GEMM dcode      dz = (g W^T + alpha/B [c>0]) [z>=0] -> dz planes, db partials
//   GEMM dW         dW = dz^T x + c^T g                                            [M x n x d, K = 2B]
//   bias_norm, finalize (losses), dict_rows<ADAM> (Jacobian + Adam + renormalise + re-split), bias<ADAM>
// Top-k variant: the encode GEMM stores fp32 scores; topk_select2_kernel keeps k per row; with the k-sparse path
// (sce_topk.cuh) decode and dcode are a gather kernel over the k selected dictionary rows instead of two dense GEMMs.
// Learned-centre variant (tied in every other respect): center_sub_kernel forms x - center[m] first, the decode epilogue
// also writes column sums of g, and before the Adam update three kernels form the centre gradient sum_b g - db W
// (center_coef / center_gemv / center_grad) and update the centre.
// Non-negative tied plans (desc.encoder_nonneg, desc.input_shift; FunctionalPositiveTiedSAE) are tied plans whose batch
// split also forms x + input_shift, and whose dict_rows kernels build the dictionary from max(E, 0).
#include <cmath>
#include <new>
#include <vector>

#include "sce_plan.cuh"
#include "sce_topk.cuh"

// The training step's kernels that are not templates (see sce_kernels.cuh)
namespace sce {

// ------------------------------------------------------------------------------------------------
// learned centre (FunctionalTiedCenteredSAE.center, sae_ensemble.py:198-200): out[m] = x[m] - center[m], fp32 [M][B][d];
// x is [B][d] shared by the models (x_model_stride = 0) or [M][B][d]. grid.y = model.
// ------------------------------------------------------------------------------------------------
__global__ void center_sub_kernel(const float* __restrict__ x, long long x_model_stride, const float* __restrict__ center,
                                  float* __restrict__ out, int B, int d) {
  const int model = blockIdx.y;
  const int d4 = d >> 2;
  const long long n4 = (long long)B * d4;
  const float4* xs = reinterpret_cast<const float4*>(x + (long long)model * x_model_stride);
  const float4* cs = reinterpret_cast<const float4*>(center + (long long)model * d);
  float4* o = reinterpret_cast<float4*>(out + (long long)model * B * d);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    const float4 v = xs[i];
    const float4 c = __ldg(cs + (int)(i % d4));
    o[i] = make_float4(v.x - c.x, v.y - c.y, v.z - c.z, v.w - c.w);
  }
}

// ------------------------------------------------------------------------------------------------
// transpose_batch_u8_kernel (its layout: sce_engine.cuh)
// ------------------------------------------------------------------------------------------------
// rows a, b, c, d of four bytes each (byte = column) -> column v of the four rows in o[v]
__device__ __forceinline__ void transpose4x4_u8(uint32_t a, uint32_t b, uint32_t c, uint32_t d, uint32_t (&o)[4]) {
  const uint32_t t0 = __byte_perm(a, b, 0x5140), t1 = __byte_perm(a, b, 0x7362);   // a0 b0 a1 b1 / a2 b2 a3 b3
  const uint32_t t2 = __byte_perm(c, d, 0x5140), t3 = __byte_perm(c, d, 0x7362);
  o[0] = __byte_perm(t0, t2, 0x5410);
  o[1] = __byte_perm(t0, t2, 0x7632);
  o[2] = __byte_perm(t1, t3, 0x5410);
  o[3] = __byte_perm(t1, t3, 0x7632);
}
__global__ void __launch_bounds__(256) transpose_batch_u8_kernel(BatchPlanes t, int models, int rows, int cols,
                                                                 long long src_model_pitch, int ld) {
  // 128 source rows of 128 bytes; 16-byte piece k of row r is stored at k ^ ((r >> 4) & 7), so that the column reads
  // below (8 groups of 16 rows x 4 words per warp) hit 32 different banks
  __shared__ uint4 tile[128][8];
  const int plane = blockIdx.z / models, m = blockIdx.z - plane * models;
  const uint8_t* src = (plane ? t.src[1] : t.src[0]) + (long long)m * src_model_pitch;   // (no dynamic index into the
  uint8_t* dst = (plane ? t.dst[1] : t.dst[0]) + (long long)m * cols * ld;                // parameter struct: no local copy)
  const int r0 = blockIdx.y * 128, c0 = blockIdx.x * 128;
#pragma unroll
  for (int i = threadIdx.x; i < 1024; i += 256) {
    const int r = i >> 3, k = i & 7;
    uint4 v = make_uint4(0u, 0u, 0u, 0u);
    if (r0 + r < rows && c0 + 16 * k < cols) v = __ldg(reinterpret_cast<const uint4*>(src + (long long)(r0 + r) * cols + c0 + 16 * k));
    tile[r][k ^ ((r >> 4) & 7)] = v;
  }
  __syncthreads();
  // source rows 16 g .. + 15, source word q (columns 4 q .. + 3) -> output rows c0 + 4 q + v, bytes r0 + 16 g .. + 15
  const int g = threadIdx.x & 7, q = threadIdx.x >> 3;
  if (r0 + 16 * g >= rows) return;
  const uint32_t* tw = reinterpret_cast<const uint32_t*>(&tile[0][0]);
  uint32_t w[16];
#pragma unroll
  for (int u = 0; u < 16; ++u) w[u] = tw[(16 * g + u) * 32 + (((q >> 2) ^ g) << 2) + (q & 3)];
  uint32_t o[4][4];   // [quad of rows][column v]
#pragma unroll
  for (int h = 0; h < 4; ++h) transpose4x4_u8(w[4 * h], w[4 * h + 1], w[4 * h + 2], w[4 * h + 3], o[h]);
#pragma unroll
  for (int v = 0; v < 4; ++v) {
    const int j = c0 + 4 * q + v;
    if (j < cols)
      *reinterpret_cast<uint4*>(dst + (long long)j * ld + r0 + 16 * g) = make_uint4(o[0][v], o[1][v], o[2][v], o[3][v]);
  }
}


// ------------------------------------------------------------------------------------------------
// per-model ||bias||_2 (bias-decay loss term and its gradient; sae_ensemble.py:73, :150)
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) bias_norm_kernel(const float* __restrict__ bias, int n,
                                                        float* __restrict__ out) {
  __shared__ double red[8];
  const float* b = bias + (long long)blockIdx.x * n;
  double acc = 0.0;
  for (int i = threadIdx.x; i < n; i += 256) acc += (double)b[i] * (double)b[i];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0;
    for (int i = 0; i < 8; ++i) t += red[i];
    out[blockIdx.x] = (float)sqrt(t);
  }
}

// ------------------------------------------------------------------------------------------------
// Gradient of the learned centre: d_center = sum_b g_b - db W, W = E / max(||E_n||, floor) (the dictionary the step
// used: these kernels run before dict_rows_kernel<MODE_ADAM> rewrites E). Three passes, no atomics: bitwise repeatable.
// ------------------------------------------------------------------------------------------------
constexpr int kCenterCoefRows = 32;    // dictionary rows per block of center_coef_kernel
constexpr int kCenterChunkRows = 64;   // dictionary rows per partial of center_gemv_kernel

// coef[m][n] = db[m][n] / max(||E[m][n]||, floor), db summed from the dcode epilogue's partials in the order bias_kernel
// uses (the same fp32 value) times part_scale. Grid (ceil(n / 32), M), 256 threads: thread t < 32 sums row t's db,
// warp w takes the norms of rows w, w + 8, ...
__global__ void __launch_bounds__(256) center_coef_kernel(const float* __restrict__ e, const float* __restrict__ db_part,
                                                          int n_part, int n, int d, float floor, float part_scale,
                                                          float* __restrict__ coef) {
  __shared__ float sdb[kCenterCoefRows], snorm[kCenterCoefRows];
  const int model = blockIdx.y, j0 = blockIdx.x * kCenterCoefRows;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (threadIdx.x < kCenterCoefRows && j0 + threadIdx.x < n) {
    const float* p = db_part + (long long)model * n_part * n + j0 + threadIdx.x;
    float g = 0.f;
    for (int k = 0; k < n_part; ++k) g += p[(long long)k * n];
    sdb[threadIdx.x] = g * part_scale;
  }
  for (int r = warp; r < kCenterCoefRows; r += 8) {
    if (j0 + r >= n) break;   // warp-uniform
    const float* row = e + ((long long)model * n + j0 + r) * d;
    float ss = 0.f;
    for (int c = lane * 4; c < d; c += 128) {
      const float4 v = *reinterpret_cast<const float4*>(row + c);
      ss += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
    }
    ss = warp_sum(ss);
    if (lane == 0) {
      const float nrm = sqrtf(ss);
      snorm[r] = floor > 0.f && nrm < floor ? floor : nrm;
    }
  }
  __syncthreads();
  if (threadIdx.x < kCenterCoefRows && j0 + threadIdx.x < n)
    coef[(long long)model * n + j0 + threadIdx.x] = sdb[threadIdx.x] / snorm[threadIdx.x];
}

// part[m][chunk][c] = sum over the chunk's rows, in order, of coef[m][j] E[m][j][c]. Grid (ceil(d / 512), chunks, M),
// 128 threads of four columns each.
__global__ void __launch_bounds__(128) center_gemv_kernel(const float* __restrict__ e, const float* __restrict__ coef, int n,
                                                          int d, float* __restrict__ part) {
  const int model = blockIdx.z, chunk = blockIdx.y;
  const int c = (blockIdx.x * 128 + threadIdx.x) * 4;
  if (c >= d) return;
  const int j0 = chunk * kCenterChunkRows, j1 = min(n, j0 + kCenterChunkRows);
  const float* kp = coef + (long long)model * n;
  const float* ep = e + (long long)model * n * d + c;
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 4
  for (int j = j0; j < j1; ++j) {
    const float k = __ldg(kp + j);
    const float4 v = __ldg(reinterpret_cast<const float4*>(ep + (long long)j * d));
    acc.x += k * v.x;
    acc.y += k * v.y;
    acc.z += k * v.z;
    acc.w += k * v.w;
  }
  *reinterpret_cast<float4*>(part + ((long long)model * gridDim.y + chunk) * d + c) = acc;
}

// grad[m][c] = g_scale * sum_k g_part[m][k][c] - sum_chunk part[m][chunk][c] (both in index order); MODE_ADAM then
// applies Adam to center / center_m / center_v, unless the step is bad (kBadWord, as bias_kernel).
template <int MODE>
__global__ void center_grad_kernel(const float* __restrict__ g_part, int n_gpart, float g_scale,
                                   const float* __restrict__ part, int n_chunks, int M, int d, float* __restrict__ grad,
                                   float* __restrict__ center, float* __restrict__ m, float* __restrict__ v, AdamHyper h,
                                   const uint32_t* __restrict__ health) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)M * d) return;
  const int model = int(i / d), c = int(i - (long long)model * d);
  const float* gp = g_part + (long long)model * n_gpart * d + c;
  float gs = 0.f;
  for (int k = 0; k < n_gpart; ++k) gs += gp[(long long)k * d];
  const float* pp = part + (long long)model * n_chunks * d + c;
  float dw = 0.f;
  for (int k = 0; k < n_chunks; ++k) dw += pp[(long long)k * d];
  const float g = __fmaf_rn(gs, g_scale, -dw);   // (explicit: MODE_GRAD and MODE_ADAM round it alike)
  grad[i] = g;
  if (MODE == MODE_ADAM) {
    if (step_is_bad(health)) return;
    float mm = m[i], vv = v[i];
    center[i] = adam_apply(center[i], g, mm, vv, h);
    m[i] = mm;
    v[i] = vv;
  }
}

// ------------------------------------------------------------------------------------------------
// losses: deterministic reduction of the GEMM epilogues' per-warp partials
//   out[m] = {loss, l_reconstruction, l_l1, l_bias_decay}, nnz[m] = mean_b count_nonzero(c)
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) finalize_kernel(const float* __restrict__ enc_part, int n_enc,
                                                       const float* __restrict__ dec_part, int n_dec,
                                                       const float* __restrict__ l1_alpha,
                                                       const float* __restrict__ bias_decay,
                                                       const float* __restrict__ bnorm, int B, int d,
                                                       float* __restrict__ out, float* __restrict__ nnz,
                                                       uint32_t* __restrict__ health) {
  __shared__ double red[3][8];
  const int model = blockIdx.x;
  double l1 = 0, cnt = 0, sq = 0;
  if (enc_part) {
    const float* e = enc_part + (long long)model * n_enc * 2;
    for (int i = threadIdx.x; i < n_enc; i += 256) {
      l1 += e[2 * i];
      cnt += e[2 * i + 1];
    }
  }
  const float* dp = dec_part + (long long)model * n_dec;
  for (int i = threadIdx.x; i < n_dec; i += 256) sq += dp[i];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    l1 += __shfl_xor_sync(0xffffffffu, l1, o);
    cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
    sq += __shfl_xor_sync(0xffffffffu, sq, o);
  }
  if ((threadIdx.x & 31) == 0) {
    red[0][threadIdx.x >> 5] = l1;
    red[1][threadIdx.x >> 5] = cnt;
    red[2][threadIdx.x >> 5] = sq;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    double a = 0, b = 0, c = 0;
    for (int i = 0; i < 8; ++i) {
      a += red[0][i];
      b += red[1][i];
      c += red[2][i];
    }
    const float l_rec = (float)(c / ((double)B * d));
    const float l_l1 = l1_alpha ? (float)(l1_alpha[model] * (a / B)) : 0.f;
    const float l_bd = (bias_decay && bnorm) ? bias_decay[model] * bnorm[model] : 0.f;
    if (health && !isfinite(l_rec + l_l1 + l_bd)) health[kBadWord] = 1u;   // the Adam kernels of this step skip
    if (out) {
      out[model * 4 + 0] = l_rec + l_l1 + l_bd;
      out[model * 4 + 1] = l_rec;
      out[model * 4 + 2] = l_l1;
      out[model * 4 + 3] = l_bd;
    }
    if (nnz) nnz[model] = (float)(b / B);
  }
}

}  // namespace sce

// desc.variant without its forward-only modifiers
static int base_variant(const sce_desc& d) { return d.variant & ~(SCE_CODE_LINEAR | SCE_DECODER_RAW); }

int validate(const sce_desc* d) {
  if (!d) return fail(SCE_ERR_INVALID, "desc is NULL");
  const int variant = base_variant(*d);
  if (variant < SCE_TIED || variant > SCE_TIED_LEARNED_CENTER) return fail(SCE_ERR_INVALID, "unknown variant %d", d->variant);
  if (variant != SCE_UNTIED && variant != d->variant)
    return fail(SCE_ERR_INVALID, "SCE_CODE_LINEAR / SCE_DECODER_RAW are defined for SCE_UNTIED only (variant %d)", d->variant);
  if (d->n_models < 1 || d->batch_max < 1) return fail(SCE_ERR_INVALID, "n_models and batch_max must be >= 1");
  if (d->d < 8 || d->d % 8 || d->n < 8 || d->n % 8)
    return fail(SCE_ERR_INVALID, "d (%d) and n (%d) must be positive multiples of 8", d->d, d->n);
  if (d->d > 8192) return fail(SCE_ERR_INVALID, "d = %d > 8192 is not supported by the row kernels", d->d);
  if ((d->fwd_passes != 1 && d->fwd_passes != 3) || (d->bwd_passes != 1 && d->bwd_passes != 3))
    return fail(SCE_ERR_INVALID, "fwd_passes / bwd_passes must be 1 or 3");
  if (d->centering < 0 || d->centering > 2) return fail(SCE_ERR_INVALID, "centering must be 0, 1 or 2");
  if (d->centering && !d->x_per_model) return fail(SCE_ERR_INVALID, "centering needs x_per_model = 1 (the centred batch differs per model)");
  if (d->centering && d->variant == SCE_TIED_LEARNED_CENTER)
    return fail(SCE_ERR_INVALID, "the learned-centre variant centres the batch itself: desc.centering must be 0");
  if (d->encoder_nonneg != 0 && d->encoder_nonneg != 1) return fail(SCE_ERR_INVALID, "encoder_nonneg must be 0 or 1");
  if (!std::isfinite(d->input_shift)) return fail(SCE_ERR_INVALID, "input_shift must be finite");
  if ((d->encoder_nonneg || d->input_shift != 0.f) && d->variant != SCE_TIED)
    return fail(SCE_ERR_INVALID, "encoder_nonneg / input_shift are defined for SCE_TIED only (variant %d)", d->variant);
  if (d->input_shift != 0.f && d->centering)
    return fail(SCE_ERR_INVALID, "input_shift cannot be combined with centering");
  if (d->arith < SCE_ARITH_AUTO || d->arith > SCE_ARITH_F16F8) return fail(SCE_ERR_INVALID, "unknown arith %d", d->arith);
  if (d->arith == SCE_ARITH_F16F8 && (d->d % 16 || d->n % 16))
    return fail(SCE_ERR_INVALID, "arith = F16F8 needs d (%d) and n (%d) to be multiples of 16 (TMA pitch of the 8-bit planes)",
                d->d, d->n);
  return SCE_OK;
}

// one call's rows: 1 <= B <= batch_max (`prefix` names the entry point in the message, "" for the training calls)
int check_rows(const sce_plan* p, int B, const char* prefix) {
  if (B < 1 || B > p->d.batch_max)
    return fail(SCE_ERR_INVALID, "%sB = %d outside [1, batch_max = %d]", prefix, B, p->d.batch_max);
  return SCE_OK;
}

// the forward-only passes: plans whose forward is that of their export (a TiedSAE)
int check_evaluable(const sce_plan* p, const char* prefix) {
  if (!p->cfg.evaluable)
    return fail(SCE_ERR_INVALID, "%snot available for the learned-centre variant or with encoder_nonneg / input_shift; "
                                 "evaluate the exported dictionaries (TiedSAE)", prefix);
  return SCE_OK;
}

// the passes that read the code of the plan's last forward call: a dw_native training step leaves its residual plane
// batch-major only (code_batch_major)
int check_forward_code(const sce_plan* p, const char* prefix) {
  if (p->code_batch_major)
    return fail(SCE_ERR_INVALID, "%sa plan's last call was a training step; follow sce_forward_stats", prefix);
  return SCE_OK;
}

// the training entry points (sce_step, sce_step_host, sce_grads, sce_step_tracked, sce_resample), before any device call
int check_trainable(const sce_plan* p, const char* prefix) {
  if (p->cfg.forward_only)
    return fail(SCE_ERR_INVALID, "%sa plan with SCE_CODE_LINEAR or SCE_DECODER_RAW is forward-only: it cannot train", prefix);
  return SCE_OK;
}

// desc.arith -> kArithBf16x3 / kArithF16F8. AUTO (unless pinned to bf16x3): f16f8 where the 8-bit planes can be
// addressed by TMA (row pitches of 16 bytes), bf16x3 otherwise; validate holds an explicit F16F8 to such shapes.
static int resolve_arith(const sce_desc& d) {
  if ((d.arith == SCE_ARITH_AUTO ? env_arith() : d.arith) == SCE_ARITH_BF16X3) return kArithBf16x3;
  return d.d % 16 == 0 && d.n % 16 == 0 ? kArithF16F8 : kArithBf16x3;
}

// topk_sparse_kernel: dynamic shared memory for `slices` slices of the activation width (see there), and the slice
// count a plan uses: the smallest of 2, 4, 8 whose slice fits (two blocks per SM); 0 when none does (the plan then runs
// the dense GEMMs)
constexpr int kTopkMaxSlices = 8;
static size_t topk_sparse_smem(const sce_desc& d, size_t krows, int slices) {
  const size_t ds = d.d / slices;
  return krows * ds * sizeof(float) + 9 * ds * sizeof(float) + krows * 8 + 128;
}
static int topk_slices(const sce_desc& d, size_t kmax) {
  int best = 0;
  for (int s = 2; s <= kTopkMaxSlices; s *= 2) {
    if (d.d % (4 * s) || d.d / s > 512) continue;   // (16-byte aligned slices for the bulk copies)
    const size_t b = topk_sparse_smem(d, kmax, s);
    if (b <= 112 * 1024) return s;   // fewest slices that fit: the kernel's time goes with the number of blocks
  }
  return best;
}

// The configuration of a plan for a validated descriptor
PlanConfig plan_config(const sce_desc& d) {
  PlanConfig c{};
  c.arith = resolve_arith(d);
  c.untied = base_variant(d) == SCE_UNTIED;
  c.topk = d.variant == SCE_TOPK;
  c.learned = d.variant == SCE_TIED_LEARNED_CENTER;
  c.linear = (d.variant & SCE_CODE_LINEAR) != 0;
  c.raw_decoder = (d.variant & SCE_DECODER_RAW) != 0;
  c.forward_only = c.linear || c.raw_decoder;
  // (the learned-centre variant always holds M centred batches, whatever the caller's layout)
  c.x_models = d.x_per_model || c.learned;
  c.xm = c.x_models ? d.n_models : 1;
  c.input_models = c.learned ? (d.x_per_model ? d.n_models : 1) : d.centering == 1 ? 1 : c.xm;
  c.nonneg = d.encoder_nonneg != 0;
  c.shift = d.input_shift;
  c.evaluable = !c.learned && !c.nonneg && c.shift == 0.f;
  c.bpad = (d.batch_max + 15) / 16 * 16;
  // top-k lists hold the largest k of the ensemble (desc.topk_k_max, supplied by the host mirror, which knows
  // buffers["sparsity"]) rounded up to 8; none when it is unknown or too large for the gather kernel (dense path)
  if (c.topk && d.topk_k_max >= 1 && d.topk_k_max <= 256) {
    c.tk_kmax = (d.topk_k_max + 7) / 8 * 8;
    c.tk_slices = topk_slices(d, c.tk_kmax);
    // Worth it where the dictionary is large against k: the dense decode + dcode GEMMs cost ~ n per row, the gather
    // kernel ~ k (it is bound by the latency chain of a block, not by bytes): the gather path is used where n >= 96 k.
    c.topk_sparse = c.tk_slices > 0 && d.n >= 96 * c.tk_kmax;
  }
  // ~30 M B n d tensor FLOPs are issued per step; below ~3e11 (a fifth of a millisecond) launches dominate, and the
  // step is replayed as a CUDA graph (sce_step)
  const bool launch_bound = 30.0 * d.n_models * (double)d.batch_max * d.n * d.d < 3e11;
  c.use_graph = launch_bound;
  // Dense f16f8 plans with split backward GEMMs keep batch-major copies of the 8-bit planes of x, c, g and dz, from
  // which the weight gradient forms its cross terms on E5M2 wgmma. Top-k plans do not: their code and (k-sparse)
  // code-gradient planes are written by the selection / scatter kernels, row-major only, so their weight gradient widens
  // the 8-bit tiles. Nor do launch-bound plans: there the weight gradient takes microseconds either way, and the copies
  // would add a launch per step (x's transpose pass) and a third to the workspace.
  c.dw_native = c.arith == kArithF16F8 && !c.topk && d.bwd_passes >= 3 && !launch_bound;
  // The same plans run decode and the native weight gradient on 192-row tiles (kBMTall, sce_gemm.cuh): both have long
  // K loops fed from L2, and a taller tile reads 22 % fewer operand bytes per MMA. Encode and dcode overlap their
  // epilogue, which leaves no registers for a third consumer warpgroup; the widened weight gradient, bf16x3, top-k and
  // launch-bound plans keep 128-row tiles.
  c.tall_tiles = c.dw_native;
  // The truncation bias of a single accumulation chain grows with the reduction length; n > 4096 splits the decode
  // GEMM's cross terms into their own accumulator (config 5's width, n = 32768, needs it for the 1e-4 bar; the parity
  // tests cover both sides). Splitting doubles the decode GEMM's accumulator registers, so it is used where needed.
  c.split_decode = d.n > 4096;
  return c;
}

// Carves the workspace into `w` (buffers the plan does not use stay null); with base == nullptr only measures it.
static size_t carve(PlanBuffers& w, const sce_desc& d, const PlanConfig& cfg, uint8_t* base) {
  Carve c{base, 0};
  const size_t M = d.n_models, B = d.batch_max, n = d.n, dd = d.d;
  const size_t xm = cfg.xm;
  const size_t tiles_mB = (B + kBM - 1) / kBM;
  const size_t tiles_nN = (n + kBN - 1) / kBN;
  const size_t tiles_nD = (dd + kBN - 1) / kBN;
  const bool f8 = cfg.arith == kArithF16F8;
  w.x_stage = c.take<float>(xm * B * dd);
  w.x = c.planes(xm * B * dd, f8);
  w.wenc = c.planes(M * n * dd, f8);
  w.wdec = cfg.untied ? c.planes(M * n * dd, f8) : w.wenc;
  if (f8) w.wdt = c.planes(M * n * dd, f8);
  const bool tdw = cfg.dw_native;
  const size_t Bp = cfg.bpad;
  const size_t dz8 = tdw ? M * n * Bp : M * B * n;   // bytes of one 8-bit plane of dz
  if (!tdw) {
    w.c = c.planes(M * B * n, f8);
  } else {
    // the code's row-major 8-bit planes are read by the decode GEMM only, which runs before dcode writes dz: they live in
    // dz's 8-bit planes (below), and the code's own 8-bit space holds the batch-major copies the weight gradient reads
    w.c.hi = c.take<uint16_t>(M * B * n);
    w.ct = c.copies(dz8);
  }
  w.g = c.planes(M * B * dd, f8);
  // all planes contiguous, 4 B / element (the top-k scores alias them); with tdw the 8-bit ones are [M][n][Bp]
  uint8_t* dz = c.take<uint8_t>(2 * (M * B * n + dz8));
  w.dz = Planes{dz, dz + 2 * M * B * n, f8 ? dz + 2 * M * B * n + dz8 : nullptr, f8};
  if (tdw) {
    w.c.lo = w.dz.lo;
    w.c.x8 = w.dz.x8;
    w.xt = c.copies(xm * dd * Bp);
    w.gt = c.copies(M * dd * Bp);
    w.c.f8 = true;
  }
  w.dw_enc = c.take<float>(M * n * dd);
  w.dw_dec = cfg.untied ? c.take<float>(M * n * dd) : w.dw_enc;
  const size_t enc_parts = cfg.topk ? B : tiles_mB * 8 * tiles_nN;
  w.part_enc = c.take<float>(M * enc_parts * 2);
  const size_t dec_parts = tiles_mB * 8 * tiles_nD;   // top-k: up to kTopkMaxSlices partials per row from the gather kernel
  w.part_dec = c.take<float>(M * (cfg.topk && dec_parts < kTopkMaxSlices * B ? kTopkMaxSlices * B : dec_parts));
  w.db_part = c.take<float>(M * tiles_mB * 4 * n);
  w.bnorm = c.take<float>(M);
  w.l1_over_b = c.take<float>(M);
  w.loss_stage = c.take<float>(M * 4);
  w.nnz_stage = c.take<float>(M);
  const size_t n_chunks = (n + 31) / 32;
  w.act_pos = c.take<uint32_t>(M * n_chunks * B);
  w.act_zero = c.take<uint32_t>(M * n_chunks * B);
  // top-k: scores of their own (the code-gradient planes must keep their scattered zeros) and the k-sparse lists
  if (cfg.topk) {
    const size_t kmax = cfg.tk_kmax;
    w.scores = c.take<float>(M * B * n);
    w.tk_cmax = c.take<uint32_t>(M * B * n_chunks);
    if (kmax) {
      w.tk_col = c.take<int>(M * B * kmax);
      w.tk_val = c.take<float>(M * B * kmax);
      w.tk_cnt = c.take<int>(M * B);
      w.tk_models = c.take<int>(M);
      w.tk_dots = c.take<float>(M * B * kmax * kTopkMaxSlices);
      w.wn_f32 = c.take<float>(M * n * dd);
    }
  }
  if (d.centering) {
    w.rot = c.planes(M * dd * dd, f8);
    w.x_centered = c.take<float>(M * B * dd);
  }
  if (cfg.learned) {
    w.x_centered = c.take<float>(M * B * dd);
    w.g_part = c.take<float>(M * tiles_mB * 4 * dd);
    w.center_coef = c.take<float>(M * n);
    w.center_part = c.take<float>(M * ((n + kCenterChunkRows - 1) / kCenterChunkRows) * dd);
    w.center_grad = c.take<float>(M * dd);
  }
  if (cfg.shift != 0.f) w.x_shifted = c.take<float>(xm * B * dd);
  w.res_flags = c.take<uint32_t>(kFlagWords);   // [0] residual flag, [kAbsmaxWord] input range monitor, [kBadWord] health (separate 128-byte lines)
  return align_up(c.off, 1024);
}

// ------------------------------------------------------------------------------------------------
// tensor maps for one batch size
// ------------------------------------------------------------------------------------------------
static int build_maps(sce_plan* p, int B, BatchMaps** out) {
  auto it = p->maps->find(B);
  if (it != p->maps->end()) {
    *out = it->second;
    return SCE_OK;
  }
  BatchMaps* m = new (std::nothrow) BatchMaps;
  if (!m) return fail(SCE_ERR_INVALID, "out of host memory");
  memset(m, 0, sizeof(*m));
  const sce_desc& d = p->d;
  const PlanConfig& cfg = p->cfg;
  const uint64_t M = d.n_models, n = d.n, dd = d.d, xm = cfg.xm, Bm = d.batch_max;
  // NOTE: activations are laid out with the plan's batch_max pitch between models; only `B` rows are
  // visible through the map, so rows >= B read as zero (TMA out-of-bounds fill).
  const bool f8 = cfg.arith == kArithF16F8;
  const int bk = gemm_bk(cfg.arith);
  // activations [models][B of batch_max][cols] as the A operand: K-major tiles [128 rows][bk]
  auto act_a = [&](OperandMaps& o, const Planes& P, uint64_t models, uint64_t cols) {
    return operand_maps(o, P, models, (uint64_t)B, cols, Bm * cols, kBM, bk);
  };
  // dictionary [M][n][d] as the B operand: K-major tiles [box_rows][bk] (box_rows = the tile's B rows), or MN-major
  auto dict_b = [&](OperandMaps& o, const Planes& P, uint32_t box_rows, int kmajor_bk) {
    return operand_maps(o, P, M, n, dd, n * dd, box_rows, kmajor_bk);
  };
  bool ok = true;
  // encode: A = x [xm,B,d] K-major, B = Wenc [M,n,d] K-major
  ok &= act_a(m->encode.a[0], p->x, xm, dd);
  ok &= dict_b(m->encode.b[0], p->wenc, kBN, bk);
  if (d.centering) {
    // centring: A = (x - trans) planes in the X planes (the encode A maps), B = rot [M,d,d] K-major, output d columns
    m->center.a[0] = m->encode.a[0];
    ok &= operand_maps(m->center.b[0], p->rot, M, dd, dd, dd * dd, kBN, bk);
  }
  // decode: A = c [M,B,n] K-major, B = Wdec [M,n,d] MN-major (bk k-rows per box); f16f8: its transposed copy [M,d,n] K-major
  ok &= cfg.tall_tiles ? operand_maps(m->decode.a[0], p->c, M, (uint64_t)B, n, Bm * n, kBMTall, bk)
                        : act_a(m->decode.a[0], p->c, M, n);
  ok &= f8 ? operand_maps(m->decode.b[0], p->wdt, M, dd, n, dd * n, kBN, bk) : dict_b(m->decode.b[0], p->wdec, bk, 0);
  // dcode: A = g [M,B,d] K-major, B = Wdec K-major
  ok &= act_a(m->dcode.a[0], p->g, M, dd);
  ok &= dict_b(m->dcode.b[0], p->wdec, kBN, bk);
  // weight gradients: reduction over the batch rows; dw_native: the 8-bit planes from the batch-major copies [models][cols][Bp]
  const uint64_t Bp = (uint64_t)cfg.bpad;
  // (t_rows: the tile's rows on this side, the launch's BM for A)
  auto dw_operand = [&](OperandMaps& o, const Planes& P, const Planes& T, uint64_t models, uint64_t cols, uint32_t t_rows) {
    return dw_operand_maps(o, P, cfg.dw_native ? &T : nullptr, models, (uint64_t)B, cols, Bm * cols, Bp, bk, t_rows);
  };
  const uint32_t dw_bm = cfg.tall_tiles ? kBMTall : kBM;
  // dz^T x, then c^T g: a second GEMM of the decoder (untied) or a second operand set of the one dictionary's
  // (dz's own 8-bit planes are batch-major in dw_native plans)
  GemmMaps& cg = cfg.untied ? m->dw_dec : m->dw_enc;
  const int cg_set = cfg.untied ? 0 : 1;
  ok &= dw_operand(m->dw_enc.a[0], p->dz, p->dz, M, n, dw_bm) && dw_operand(m->dw_enc.b[0], p->x, p->xt, xm, dd, kBN);
  ok &= dw_operand(cg.a[cg_set], p->c, p->ct, M, n, dw_bm) && dw_operand(cg.b[cg_set], p->g, p->gt, M, dd, kBN);
  ok &= make_tmap_bf16_store32(&m->st_c.hi, p->c.hi, M, (uint64_t)B, n, Bm * n);
  ok &= make_tmap_bf16_store32(&m->st_dz.hi, p->dz.hi, M, (uint64_t)B, n, Bm * n);
  if (f8) {
    auto st8 = [&](CUtensorMap* t, const void* base) {
      return make_tmap_u8_box(t, base, M, (uint64_t)B, n, n, Bm * n, 32, 32, CU_TENSOR_MAP_SWIZZLE_32B);
    };
    // dw_native: dz's 8-bit planes [M][n][Bp], boxes of 32 features x 32 batch bytes (EpiDcodeT<f16f8, true>)
    auto st8t = [&](CUtensorMap* t, const void* base) {
      return make_tmap_u8_box(t, base, M, n, (uint64_t)B, Bp, n * Bp, 32, 32, CU_TENSOR_MAP_SWIZZLE_NONE);
    };
    ok &= st8(&m->st_c.lo, p->c.lo) && st8(&m->st_c.x8, p->c.x8);
    ok &= cfg.dw_native ? st8t(&m->st_dz.lo, p->dz.lo) && st8t(&m->st_dz.x8, p->dz.x8)
                        : st8(&m->st_dz.lo, p->dz.lo) && st8(&m->st_dz.x8, p->dz.x8);
  } else {
    ok &= make_tmap_bf16_store32(&m->st_c.lo, p->c.lo, M, (uint64_t)B, n, Bm * n);
    ok &= make_tmap_bf16_store32(&m->st_dz.lo, p->dz.lo, M, (uint64_t)B, n, Bm * n);
  }
  if (cfg.topk) ok &= make_tmap_f32_store32(&m->st_scores, p->scores, M, (uint64_t)B, n, Bm * n);
  if (!ok) {
    delete m;
    return fail(SCE_ERR_CUDA, "cuTensorMapEncodeTiled failed (B=%d, M=%d, n=%d, d=%d)", B, d.n_models, d.n, d.d);
  }
  (*p->maps)[B] = m;
  *out = m;
  return SCE_OK;
}


// ------------------------------------------------------------------------------------------------
// helpers shared by step / forward / grads
// ------------------------------------------------------------------------------------------------
static AdamHyper hyper_for(const sce_plan* p, long long t) {
  AdamHyper h;
  h.lr = p->d.lr;
  h.b1 = p->d.beta1;
  h.b2 = p->d.beta2;
  h.eps = p->d.eps;
  h.eps_root = p->d.eps_root;
  const double tt = p->d.adam_count_mode == SCE_ADAM_FROZEN_T1 ? 1.0 : (double)t;
  h.bc1 = (float)(1.0 - pow((double)h.b1, tt));
  h.bc2 = (float)(1.0 - pow((double)h.b2, tt));
  return h;
}

// One dictionary of the plan: its weights, their gradient, Adam moments, operand planes and row normalisation
struct DictSide {
  float *w, *dw, *m, *v;
  Planes planes;
  int normalize;
  float floor;
};
// The plan's dictionaries, encoder first: one for tied and top-k plans, which normalise it; two for untied plans, whose
// decoder alone is normalised. Returns the count.
static int dict_sides(const sce_plan* p, DictSide out[2]) {
  const sce_buffers& b = p->b;
  if (!p->cfg.untied) {
    out[0] = {b.encoder, p->dw_enc, b.encoder_m, b.encoder_v, p->wenc, 1, p->d.norm_floor};
    return 1;
  }
  out[0] = {b.encoder, p->dw_enc, b.encoder_m, b.encoder_v, p->wenc, 0, 0.f};
  out[1] = {b.decoder, p->dw_dec, b.decoder_m, b.decoder_v, p->wdec, 1, p->d.norm_floor};
  return 2;
}

// MODE_PREPARE reads the weights and writes the planes; MODE_ADAM also reads dW and updates the moments; MODE_GRAD
// reads the weights and dW and writes `grad_out` only
template <int MODE>
static int launch_dict_rows(Launcher& L, const sce_plan* p, const DictSide& s, float* grad_out, AdamHyper h) {
  const long long rows = (long long)p->d.n_models * p->d.n;
  const float* dw = MODE == MODE_PREPARE ? nullptr : s.dw;
  float* m = MODE == MODE_ADAM ? s.m : nullptr;
  float* v = MODE == MODE_ADAM ? s.v : nullptr;
  const Planes w = MODE == MODE_GRAD ? Planes{} : s.planes;
  float* wf = (MODE != MODE_GRAD && p->cfg.topk_sparse) ? p->wn_f32 : nullptr;   // (top-k plans have one dictionary)
  return with_arith(p->cfg.arith, [&](auto arith) {
    auto run = [&](auto nonneg) {
      return launch_dict_rows_t<MODE, decltype(arith)::value, decltype(nonneg)::value>(
          L, s.w, dw, m, v, w, grad_out, rows, p->d.d, s.normalize, s.floor, h, p->res_flags, wf);
    };
    return p->cfg.nonneg ? run(std::true_type{}) : run(std::false_type{});   // (nonneg: tied plans only, one side)
  });
}

// f16f8: the decoder's planes -> their transposed copy, which the decode GEMM reads K-major (nothing to do where the
// decode runs without the GEMM: k-sparse top-k plans)
static int transpose_dict(Launcher& L, const sce_plan* p) {
  if (p->cfg.arith != kArithF16F8 || p->cfg.topk_sparse) return SCE_OK;
  const sce_desc& d = p->d;
  const dim3 grid((d.d + 63) / 64, (d.n + 63) / 64, d.n_models);
  TRY(L.launch(transpose_kernel<uint16_t>, grid, 256, 0, static_cast<const uint16_t*>(p->wdec.hi),
               static_cast<uint16_t*>(p->wdt.hi), d.n, d.d));
  TRY(L.launch(transpose_kernel<uint8_t>, grid, 256, 0, static_cast<const uint8_t*>(p->wdec.lo),
               static_cast<uint8_t*>(p->wdt.lo), d.n, d.d));
  return L.launch(transpose_kernel<uint8_t>, grid, 256, 0, p->wdec.x8, p->wdt.x8, d.n, d.d);
}

// The normalised operand planes of every dictionary side from the fp32 parameters (sce_prepare, sce_resample)
int prepare_dict(Launcher& L, const sce_plan* p) {
  DictSide sides[2];
  for (int s = 0, ns = dict_sides(p, sides); s < ns; ++s) {
    if (s == 1 && p->cfg.raw_decoder) {
      // SCE_DECODER_RAW: sce_similarity's split of a raw operand; f16f8 judges its range with the batch split's flags
      const long long n4 = (long long)p->d.n_models * p->d.n * p->d.d / 4;
      TRY(with_arith(p->cfg.arith, [&](auto arith) {
        constexpr int AR = decltype(arith)::value;
        return launch_split_rows<AR>(L, sides[s].w, sides[s].planes, n4, AR == kArithF16F8 ? p->res_flags : nullptr);
      }));
      continue;
    }
    TRY(launch_dict_rows<MODE_PREPARE>(L, p, sides[s], nullptr, hyper_for(p, 1)));
  }
  return transpose_dict(L, p);
}

// f16f8 runs the backward pass on the residual r instead of g = 2r/(B d) (EpiDecodeT): weight- and bias-gradient
// outputs are multiplied by 2/(B d) on the way out, the sparsity term enters dcode as alpha d / 2.
static float grad_out_scale(const sce_plan* p, int B) {
  return p->cfg.arith == kArithF16F8 ? 2.0f / ((float)B * (float)p->d.d) : 1.0f;
}

__global__ void l1_over_b_kernel(const float* __restrict__ alpha, float* __restrict__ out, int M, float invB) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < M) out[i] = alpha ? alpha[i] * invB : 0.f;
}

template <class T>
struct TypeTag {
  using type = T;
};

// ------------------------------------------------------------------------------------------------
// the pipeline: the phases of a forward pass and its backward GEMMs, in launch order (run_pipeline_t)
// ------------------------------------------------------------------------------------------------
// the activity masks [c > 0] / [z == 0] that encode (or the top-k selection) writes and the code gradient reads
// (top-k: relu semantics, no gradient at exactly 0, no [z == 0] mask)
static ActMask act_mask(const sce_plan* p) {
  return {p->act_pos, p->cfg.topk ? nullptr : p->act_zero, (p->d.n + 31) / 32, p->d.batch_max};
}

// top-k: the k-sparse lists the selection writes and the gather and scatter kernels read
static TopkLists topk_lists(const sce_plan* p) {
  return {p->tk_col, p->tk_val, p->tk_cnt, p->cfg.tk_kmax, p->d.batch_max};
}

// Input: centring or the learned centre's subtraction, the batch split (with the input shift), the batch-major copy of
// x (`tdw`: a native weight gradient follows) and alpha / B. Points `x` at the fp32 batch the later phases read.
template <int AR>
static int input_phase(PlanCall& c, const float*& x, bool tdw) {
  constexpr bool f8 = AR == kArithF16F8;
  sce_plan* const p = c.p;
  const sce_desc& d = p->d;
  const PlanConfig& cfg = p->cfg;
  const int B = c.B, M = d.n_models, dd = d.d;
  const long long Bm = d.batch_max;
  const long long n4 = (long long)B * dd / 4;   // (the centring kernels: float4s of one model's batch, <= 1024 blocks)
  const int blocks = (int)((n4 + 255) / 256 < 1024 ? (n4 + 255) / 256 : 1024);
  if (d.centering) {
    // ---- centring (sae_ensemble.py:126-128): (x - trans[m]) -> planes, GEMM with rot[m] (all split passes), * scale[m]
    // -> the per-model fp32 batch every kernel below reads as `x`
    TRY(c.launch(center_split_kernel<AR>, dim3(blocks, M), 256, 0, x, d.centering == 2 ? (long long)B * dd : 0,
                 p->b.center_trans, p->x.hi, p->x.lo, p->x.x8, Bm * dd, B, dd));
    EpiCenter::Params cp;
    cp.out = p->x_centered;
    cp.model_stride = (long long)B * dd;
    cp.ld = dd;
    cp.col_scale = p->b.center_scale;
    TRY((c.gemm<EpiCenter, false, false, false, AR>(c.maps->center, 1, kOnes, kOnes, dd, 3, B, dd, cp)));
    x = p->x_centered;
  } else if (cfg.learned) {
    // ---- learned centre (sae_ensemble.py:198-200): x - center[m] -> the per-model fp32 batch every kernel below reads
    TRY(c.launch(center_sub_kernel, dim3(blocks, M), 256, 0, x, d.x_per_model ? (long long)B * dd : 0, p->b.center,
                 p->x_centered, B, dd));
    x = p->x_centered;
  }
  // ---- x -> (hi, lo): per model slabs are batch_max apart in the workspace. input_shift (mlp_tests.py:104): the split
  // forms x + shift once, as the caller laid the batch out, and every kernel below reads that shifted batch
  if constexpr (f8) CUDA_TRY(cudaMemsetAsync(p->res_flags, 0, sizeof(uint32_t), c.st));
  for (int m = 0; m < cfg.xm; ++m)
    TRY(launch_split_rows<AR>(c, x + (long long)m * B * dd, p->x.at(m * Bm * dd), (long long)B * dd / 4,
                              f8 ? p->res_flags : nullptr, cfg.shift,
                              cfg.shift != 0.f ? p->x_shifted + (long long)m * B * dd : nullptr));
  if (cfg.shift != 0.f) x = p->x_shifted;
  if (tdw) TRY(batch_major(c, p->x, p->xt, cfg.xm, B, dd, Bm * dd, cfg.bpad));
  p->code_batch_major = tdw ? 1 : 0;
  // alpha / B, or (f16f8, backward on r = g B d / 2) alpha d / 2
  return c.launch(l1_over_b_kernel, (M + 127) / 128, 128, 0, p->b.l1_alpha, p->l1_over_b, M,
                  f8 ? 0.5f * (float)dd : 1.0f / (float)B);
}

// Encode: z = x W^T (+b) -> relu -> code planes, activity masks and loss partials in the epilogue (with `mom_part`,
// also the moment partials of EpiEncodeT<AR, true>); top-k: the scores, then the per-row selection
template <int AR>
static int encode_phase(PlanCall& c, bool tdw, float* mom_part) {
  sce_plan* const p = c.p;
  const sce_desc& d = p->d;
  const PlanConfig& cfg = p->cfg;
  const int B = c.B, M = d.n_models, n = d.n;
  const int xb[2] = {cfg.x_models ? 1 : 0, 1};
  const ActMask act = act_mask(p);
  ResFlags x_is_a;   // the batch's residual-plane flag, for the GEMM that reads x as its A operand
  if constexpr (AR == kArithF16F8) x_is_a.a[0] = p->res_flags;
  if (!cfg.topk) {
    auto fill = [&](auto& ep) {
      ep.out_hi = c.maps->st_c.hi;
      ep.out_lo = c.maps->st_c.lo;
      ep.out_x8 = c.maps->st_c.x8;
      ep.bias = p->b.encoder_bias;
      ep.mask = p->b.coef_mask;
      ep.part = p->part_enc;
      ep.tiles_m = (B + kBM - 1) / kBM;
      ep.flag_zero = 1;
      ep.act = act;
      ep.tiles_n = (n + kBN - 1) / kBN;
    };
    // (forward-only plans: a forward pass, with or without the moment partials)
    auto stats = [&](auto linear) {
      using EpiStats = EpiEncodeT<AR, true, false, decltype(linear)::value>;
      typename EpiStats::Params ep;
      fill(ep);
      ep.mom_part = mom_part;
      ep.row_blocks = (B + 31) / 32;
      return c.gemm<EpiStats, false, false, false, AR>(c.maps->encode, 1, xb, kOnes, d.d, d.fwd_passes, B, n, ep, x_is_a);
    };
    if (cfg.linear) {
      if (mom_part) return stats(std::true_type{});
      using EpiLinear = EpiEncodeT<AR, false, false, true>;
      typename EpiLinear::Params ep;
      fill(ep);
      return c.gemm<EpiLinear, false, false, false, AR>(c.maps->encode, 1, xb, kOnes, d.d, d.fwd_passes, B, n, ep, x_is_a);
    }
    if (mom_part) return stats(std::false_type{});
    if constexpr (AR == kArithF16F8) {
      if (tdw) {   // the epilogue also writes the batch-major copies of the code's 8-bit planes the weight gradient reads
        using EpiT8 = EpiEncodeT<AR, false, true>;
        typename EpiT8::Params ep;
        fill(ep);
        ep.t_lo = static_cast<uint8_t*>(p->ct.lo);
        ep.t_x8 = p->ct.x8;
        ep.t_ld = cfg.bpad;
        return c.gemm<EpiT8, false, false, false, AR>(c.maps->encode, 1, xb, kOnes, d.d, d.fwd_passes, B, n, ep, x_is_a);
      }
    }
    typename EpiEncodeT<AR>::Params ep;
    fill(ep);
    return c.gemm<EpiEncodeT<AR>, false, false, false, AR>(c.maps->encode, 1, xb, kOnes, d.d, d.fwd_passes, B, n, ep,
                                                          x_is_a);
  }
  // scores -> fp32 and the chunk maxima of every row, then per-row selection (code planes, activity mask, k-sparse
  // lists) from the chunk maxima (the kernel reads whole rows where they cannot bound the k-th largest score)
  EpiScoresTma::Params sp;
  sp.out = c.maps->st_scores;
  sp.cmax = p->tk_cmax;
  sp.n_chunks = act.n_chunks;
  sp.cmax_model_stride = (long long)d.batch_max * act.n_chunks;
  TRY((c.gemm<EpiScoresTma, false, false, false, AR>(c.maps->encode, 1, xb, kOnes, d.d, d.fwd_passes, B, n, sp, x_is_a)));
  // one block per (row, model); scores / codes of model m start at m * batch_max * n
  return c.launch(topk_select2_kernel<AR>, dim3(B, M), 256, 0, p->scores, p->b.sparsity, p->c.hi, p->c.lo, p->c.x8,
                  cfg.topk_sparse ? p->dz.hi : nullptr, p->dz.lo, p->dz.x8, act, topk_lists(p), p->part_enc, B, n,
                  (long long)d.batch_max * n, p->tk_cmax);
}

// Decode: x^ = c W -> r = x^ - x, loss partials and the g planes (learned centre: + column sums of g), as the dense GEMM
// or, in k-sparse top-k plans, as the gather kernel per k class (which also forms the code gradient's shares, `backward`)
template <int AR>
static int decode_phase(PlanCall& c, const float* x, float* x_hat, bool backward, bool tdw) {
  constexpr bool f8 = AR == kArithF16F8;
  sce_plan* const p = c.p;
  const sce_desc& d = p->d;
  const PlanConfig& cfg = p->cfg;
  const int B = c.B, n = d.n, dd = d.d;
  const float gscale = f8 ? 1.0f : 2.0f / ((float)B * (float)dd);
  if (cfg.topk_sparse) {
    CUDA_TRY(opt_in_smem<topk_sparse_kernel<AR>>(112 * 1024, p->device));
    // one launch per k class (sce_prepare sorted the models): a block's shared memory goes with ITS models' k, so the
    // k = 16 and k = 32 models of a mixed ensemble run at 5 and 3 blocks per SM instead of the 2 that k_max = 64 allows
    for (int g = 0; g < p->tk_groups; ++g) {
      const int cnt = p->tk_group_off[g + 1] - p->tk_group_off[g];
      if (cnt == 0) continue;
      TRY(c.launch(topk_sparse_kernel<AR>, dim3(B, cnt, cfg.tk_slices), 256,
                   topk_sparse_smem(d, p->tk_group_krows[g], cfg.tk_slices), topk_lists(p), p->b.sparsity, p->wn_f32, x,
                   d.x_per_model ? (long long)B * dd : 0, p->g.hi, p->g.lo, p->g.x8, x_hat, p->part_dec,
                   backward ? p->tk_dots : nullptr, B, n, dd, gscale, p->tk_models + p->tk_group_off[g],
                   p->tk_group_krows[g]));
    }
    return SCE_OK;
  }
  auto decode = [&](auto tag) {
    using E = typename decltype(tag)::type;
    typename E::Params dp;
    dp.x = x;
    dp.x_model_stride = cfg.x_models ? (long long)B * dd : 0;
    dp.g_hi = static_cast<uint16_t*>(p->g.hi);
    dp.g_lo = static_cast<uint8_t*>(p->g.lo);
    dp.g_x8 = p->g.x8;
    dp.x_hat = x_hat;
    dp.part = p->part_dec;
    dp.g_model_stride = (long long)d.batch_max * dd;
    dp.xhat_model_stride = (long long)B * dd;
    dp.ld = dd;
    dp.tiles_m = (B + kBM - 1) / kBM;
    dp.gscale = gscale;
    dp.tiles_n = (dd + kBN - 1) / kBN;
    if constexpr (std::is_base_of<DecodeGsumParams<true>, typename E::Params>::value) dp.g_part = p->g_part;
    if constexpr (std::is_base_of<DecodeRowErrParams<true>, typename E::Params>::value) dp.row_part = c.row_part;
    if constexpr (std::is_base_of<BatchMajorParams<true>, typename E::Params>::value) {
      dp.t_lo = static_cast<uint8_t*>(p->gt.lo);
      dp.t_x8 = p->gt.x8;
      dp.t_ld = cfg.bpad;
    }
    if constexpr (f8) {
      if (cfg.tall_tiles)
        return c.gemm<E, false, false, false, AR, true, kBMTall>(c.maps->decode, 1, kOnes, kOnes, n, d.fwd_passes, B, dd, dp);
      return c.gemm<E, false, false, false, AR>(c.maps->decode, 1, kOnes, kOnes, n, d.fwd_passes, B, dd, dp);
    }
    else if (cfg.split_decode)
      return c.gemm<E, false, true, true, AR>(c.maps->decode, 1, kOnes, kOnes, n, d.fwd_passes, B, dd, dp);
    else
      return c.gemm<E, false, true, false, AR>(c.maps->decode, 1, kOnes, kOnes, n, d.fwd_passes, B, dd, dp);
  };
  // tdw: the epilogue also writes the batch-major copies of g's 8-bit planes the weight gradient reads; with row_part
  // (tracked steps) also the per-row partials of r^2
  auto pick = [&](auto rowerr) {
    constexpr bool RE = decltype(rowerr)::value;
    if constexpr (f8)
      if (tdw)
        return cfg.learned ? decode(TypeTag<EpiDecodeT<AR, true, true, RE>>{}) : decode(TypeTag<EpiDecodeT<AR, false, true, RE>>{});
    return cfg.learned ? decode(TypeTag<EpiDecodeT<AR, true, false, RE>>{}) : decode(TypeTag<EpiDecodeT<AR, false, false, RE>>{});
  };
  return c.row_part ? pick(std::true_type{}) : pick(std::false_type{});
}

// Losses: the bias norm (bias decay), then the loss columns and nnz from the partials of encode and decode
static int losses_phase(PlanCall& c, float* out_losses, float* out_nnz) {
  sce_plan* const p = c.p;
  const sce_desc& d = p->d;
  const int B = c.B, M = d.n_models, tiles_mB = (B + kBM - 1) / kBM;
  const int n_enc_parts = p->cfg.topk ? B : tiles_mB * 8 * ((d.n + kBN - 1) / kBN);
  const int n_dec_parts = p->cfg.topk_sparse ? p->cfg.tk_slices * B : tiles_mB * 8 * ((d.d + kBN - 1) / kBN);
  if (p->b.encoder_bias && p->b.bias_decay) TRY(c.launch(bias_norm_kernel, M, 256, 0, p->b.encoder_bias, d.n, p->bnorm));
  return c.launch(finalize_kernel, M, 256, 0, p->part_enc, n_enc_parts, p->part_dec, n_dec_parts, p->b.l1_alpha,
                  p->b.encoder_bias ? p->b.bias_decay : nullptr, p->bnorm, B, d.d, out_losses, out_nnz, p->res_flags);
}

// Backward: the code gradient (dcode GEMM, or the k-sparse scatter), then the weight gradients into p->dw_enc /
// p->dw_dec
template <int AR>
static int backward_phase(PlanCall& c) {
  constexpr bool f8 = AR == kArithF16F8;
  sce_plan* const p = c.p;
  const sce_desc& d = p->d;
  const PlanConfig& cfg = p->cfg;
  const int B = c.B, M = d.n_models, n = d.n, dd = d.d;
  const int xb[2] = {cfg.x_models ? 1 : 0, 1};
  if (cfg.topk_sparse) {
    // ---- code gradient planes: zero the rows, scatter the k entries
    TRY(c.launch(topk_dz_scatter_kernel<AR>, dim3(B, M), 64, 0, topk_lists(p), p->tk_dots, cfg.tk_slices, p->dz.hi,
                 p->dz.lo, p->dz.x8, n));
  } else {
    // ---- dcode
    auto dcode = [&](auto tag) {
      using E = typename decltype(tag)::type;
      typename E::Params zp;
      zp.out_hi = c.maps->st_dz.hi;
      zp.out_lo = c.maps->st_dz.lo;
      zp.out_x8 = c.maps->st_dz.x8;
      zp.act = act_mask(p);
      zp.l1_over_b = p->l1_over_b;
      zp.db_part = p->b.encoder_bias ? p->db_part : nullptr;
      zp.tiles_m = (B + kBM - 1) / kBM;
      zp.planes = d.bwd_passes >= 3 ? 3 : 0;
      // the only reader of dz's value plane is the dz^T x term of the weight gradient, against x's residual plane
      // (per-model batches carry one flag for all of them, so the same test holds)
      zp.x_res_flag = f8 ? p->res_flags : nullptr;
      return c.gemm<E, false, false, false, AR>(c.maps->dcode, 1, kOnes, kOnes, dd, d.bwd_passes, B, n, zp);
    };
    // dw_native: dz's 8-bit planes are written batch-major, as the native weight gradient reads them
    if constexpr (f8) TRY(cfg.dw_native ? dcode(TypeTag<EpiDcodeT<AR, true>>{}) : dcode(TypeTag<EpiDcodeT<AR>>{}));
    else TRY(dcode(TypeTag<EpiDcodeT<AR>>{}));
  }

  // ---- weight gradients
  c.mark(SCE_PHASE_DW);
  auto dw = [&](const GemmMaps& gm, int nsets, const int* ab, const int* bb, float* out, const ResFlags& rf) -> int {
    EpiStoreF32::Params sp;
    sp.out = out;
    sp.model_stride = (long long)n * dd;
    sp.ld = dd;
    sp.scale = grad_out_scale(p, B);
    return launch_dw_t<AR>(c, cfg.dw_native, cfg.tall_tiles, M, p->device, p->sms, gm, nsets, ab, bb, B, d.bwd_passes, n, dd, sp, rf);
  };
  ResFlags x_is_b;   // the batch's residual-plane flag, for the GEMM that reads x as its B operand (set 0)
  if constexpr (f8) x_is_b.b[0] = p->res_flags;
  if (!cfg.untied) {
    const int bb[2] = {xb[0], 1};
    return dw(c.maps->dw_enc, 2, kOnes, bb, p->dw_enc, x_is_b);
  }
  TRY(dw(c.maps->dw_enc, 1, kOnes, xb, p->dw_enc, x_is_b));
  return dw(c.maps->dw_dec, 1, kOnes, kOnes, p->dw_dec, ResFlags());
}

// The forward pass on the rows of `x` (+ the backward GEMMs, which leave dW in p->dw_enc / p->dw_dec, when `backward`),
// with the profile marks at its phase boundaries. `mom_part` (forward only, SAE variants): the encode epilogue also
// writes the moment partials of EpiEncodeT<AR, true>.
template <int AR>
static int run_pipeline_t(PlanCall& c, const float* x, float* x_hat, bool backward, float* out_losses, float* out_nnz,
                          float* mom_part) {
  const bool tdw = AR == kArithF16F8 && backward && c.p->cfg.dw_native;
  c.mark(SCE_PHASE_SPLIT);
  TRY(input_phase<AR>(c, x, tdw));
  c.mark(SCE_PHASE_ENCODE);
  TRY(encode_phase<AR>(c, tdw, mom_part));
  c.mark(SCE_PHASE_DECODE);
  TRY(decode_phase<AR>(c, x, x_hat, backward, tdw));
  c.mark(SCE_PHASE_LOSSES);
  TRY(losses_phase(c, out_losses, out_nnz));
  c.mark(SCE_PHASE_DCODE);
  if (backward) TRY(backward_phase<AR>(c));
  c.mark(SCE_PHASE_ADAM);
  return SCE_OK;
}

// Opens call `c` of plan `p` on `st` for the B rows of `x` (checks them, finds or builds the batch's tensor maps) and
// runs the pipeline in it
int run_pipeline(PlanCall& c, sce_plan* p, const float* x, int B, cudaStream_t st, float* x_hat, bool backward,
                 float* out_losses, float* out_nnz, float* mom_part, float* row_part) {
  TRY(check_rows(p, B, ""));
  if (!x) return fail(SCE_ERR_INVALID, "x is NULL");
  c = PlanCall{{st}, p, nullptr, B, row_part};
  TRY(build_maps(p, B, &c.maps));
  return with_arith(p->cfg.arith, [&](auto arith) {
    return run_pipeline_t<decltype(arith)::value>(c, x, x_hat, backward, out_losses, out_nnz, mom_part);
  });
}

// Learned-centre plans: the centre gradient of the last backward pass into p->center_grad (sum_b g - db W, with db and
// W those of this step: it runs before dict_rows_kernel<MODE_ADAM> rewrites the encoder), and with MODE_ADAM the Adam
// update of the centre
template <int MODE>
static int center_grad_launches(PlanCall& c, const AdamHyper& h) {
  sce_plan* const p = c.p;
  const sce_desc& d = p->d;
  const int M = d.n_models, n = d.n, dd = d.d;
  const int n_part = ((c.B + kBM - 1) / kBM) * 4;
  const int chunks = (n + kCenterChunkRows - 1) / kCenterChunkRows;
  const float scale = grad_out_scale(p, c.B);
  TRY(c.launch(center_coef_kernel, dim3((n + kCenterCoefRows - 1) / kCenterCoefRows, M), 256, 0, p->b.encoder, p->db_part,
               n_part, n, dd, d.norm_floor, scale, p->center_coef));
  TRY(c.launch(center_gemv_kernel, dim3((dd + 511) / 512, chunks, M), 128, 0, p->b.encoder, p->center_coef, n, dd,
               p->center_part));
  const long long tot = (long long)M * dd;
  return c.launch(center_grad_kernel<MODE>, (unsigned)((tot + 255) / 256), 256, 0, p->g_part, n_part, scale,
                  p->center_part, chunks, M, dd, p->center_grad, MODE == MODE_ADAM ? p->b.center : nullptr,
                  MODE == MODE_ADAM ? p->b.center_m : nullptr, MODE == MODE_ADAM ? p->b.center_v : nullptr, h,
                  MODE == MODE_ADAM ? p->res_flags : nullptr);
}

// What follows the backward pass, in order: the centre gradient (learned centre), dict_rows per dictionary side, the
// decoder's transposed planes (MODE_ADAM) and the bias kernel. MODE_ADAM updates the parameters; MODE_GRAD writes the
// gradients to grad_out[side] and d_bias, skipping a launch whose output is null.
template <int MODE>
static int train_tail(PlanCall& c, const AdamHyper& h, float* const* grad_out, float* d_bias) {
  constexpr bool adam = MODE == MODE_ADAM;
  sce_plan* const p = c.p;
  if (p->cfg.learned) TRY(center_grad_launches<MODE>(c, h));
  DictSide sides[2];
  for (int s = 0, ns = dict_sides(p, sides); s < ns; ++s)
    if (adam || grad_out[s]) TRY(launch_dict_rows<MODE>(c, p, sides[s], adam ? nullptr : grad_out[s], h));
  if (adam) TRY(transpose_dict(c, p));
  if (!p->b.encoder_bias || !(adam || d_bias)) return SCE_OK;
  const sce_desc& d = p->d;
  const long long tot = (long long)d.n_models * d.n;
  const int n_part = ((c.B + kBM - 1) / kBM) * 4;
  return c.launch(bias_kernel<MODE>, (unsigned)((tot + 255) / 256), 256, 0, p->b.encoder_bias,
                  adam ? p->b.bias_m : nullptr, adam ? p->b.bias_v : nullptr, p->db_part, n_part, d.n, d.n_models,
                  p->b.bias_decay, p->bnorm, adam ? nullptr : d_bias, h, grad_out_scale(p, c.B),
                  adam ? p->res_flags : nullptr);
}

// every launch of one optimisation step, in order, on `st` (also what gets captured into a CUDA graph), counted in `c`
static int step_launches(PlanCall& c, sce_plan* p, const float* x, int B, float* out_losses, float* out_nnz, long long t,
                         cudaStream_t st, float* row_part = nullptr) {
  TRY(run_pipeline(c, p, x, B, st, nullptr, true, out_losses, out_nnz, nullptr, row_part));
  TRY(train_tail<MODE_ADAM>(c, hyper_for(p, t), nullptr, nullptr));
  c.mark(SCE_PHASE_COUNT);
  return SCE_OK;
}

// Launch-bound shapes (a step of ~10 kernels that each run a few microseconds, e.g. BASELINE config 1) replay the
// step as one CUDA graph: the batch is first copied into the plan's staging buffer so that every kernel argument is
// stable, the graph is captured on the second step at a given batch size (the first one runs eagerly and performs
// the one-off cudaFuncSetAttribute calls); the captured kernels write the plan's staging outputs, which are copied to
// the caller's buffers after the launch.
static bool graph_eligible(const sce_plan* p) {
  if (p->prof_on) return false;                                   // per-phase events are recorded eagerly
  if (p->d.adam_count_mode != SCE_ADAM_FROZEN_T1) return false;   // bias correction is a kernel argument that moves
  return p->cfg.use_graph;
}

// sce_step; with row_part (sce_step_tracked) the step also leaves its per-row partials there, and runs eagerly
int step_impl(sce_plan* p, const float* x, int B, float* out_losses, float* out_nnz, cudaStream_t st, float* row_part) {
  if (int rc = check_rows(p, B, "")) return rc;
  if (!x) return fail(SCE_ERR_INVALID, "x is NULL");
  PlanCall c;
  int rc;
  if (row_part || !graph_eligible(p)) {
    rc = step_launches(c, p, x, B, out_losses, out_nnz, p->step + 1, st, row_part);
  } else {
    BatchMaps* maps = nullptr;
    rc = build_maps(p, B, &maps);
    if (rc) return rc;
    const size_t bytes = (size_t)p->cfg.input_models * B * p->d.d * sizeof(float);
    if (x != p->x_stage) CUDA_TRY(cudaMemcpyAsync(p->x_stage, x, bytes, cudaMemcpyDeviceToDevice, st));
    // the captured kernels write the plan's own staging outputs (stable addresses: callers may pass fresh tensors
    // every step, as the reference returns them); the results are copied out below
    float* const cap_losses = p->loss_stage;
    float* const cap_nnz = p->nnz_stage;
    if (maps->graph) {
      CUDA_TRY(cudaGraphLaunch(maps->graph, st));
      c.count = maps->graph_launches;
    } else if (maps->eager_steps == 0) {
      maps->eager_steps = 1;
      rc = step_launches(c, p, p->x_stage, B, cap_losses, cap_nnz, 1, st);
    } else {
      // capture on a private stream (the caller's may be the legacy default stream, which cannot be captured);
      // capturing records the launches without running them, the instantiated graph is launched on `st`
      cudaGraph_t g = nullptr;
      if (!p->cap_stream) CUDA_TRY(cudaStreamCreateWithFlags(&p->cap_stream, cudaStreamNonBlocking));
      CUDA_TRY(cudaStreamBeginCapture(p->cap_stream, cudaStreamCaptureModeThreadLocal));
      rc = step_launches(c, p, p->x_stage, B, cap_losses, cap_nnz, 1, p->cap_stream);
      cudaError_t ce = cudaStreamEndCapture(p->cap_stream, &g);
      if (rc == SCE_OK && ce == cudaSuccess && g) {
        cudaGraphExec_t ge = nullptr;
        ce = cudaGraphInstantiate(&ge, g, 0);
        cudaGraphDestroy(g);
        if (ce != cudaSuccess) return fail(SCE_ERR_CUDA, "cudaGraphInstantiate failed: %s", cudaGetErrorString(ce));
        maps->graph = ge;
        maps->graph_launches = c.count;
        CUDA_TRY(cudaGraphLaunch(maps->graph, st));
      } else {
        if (g) cudaGraphDestroy(g);
        cudaGetLastError();
        if (rc == SCE_OK) return fail(SCE_ERR_CUDA, "stream capture of the step failed: %s", cudaGetErrorString(ce));
      }
    }
    if (rc == SCE_OK && out_losses && out_losses != cap_losses)
      CUDA_TRY(cudaMemcpyAsync(out_losses, cap_losses, (size_t)p->d.n_models * SCE_LOSS_COLS * sizeof(float),
                               cudaMemcpyDeviceToDevice, st));
    if (rc == SCE_OK && out_nnz && out_nnz != cap_nnz)
      CUDA_TRY(cudaMemcpyAsync(out_nnz, cap_nnz, (size_t)p->d.n_models * sizeof(float), cudaMemcpyDeviceToDevice, st));
  }
  if (rc) return rc;
  p->last_launches = c.count;   // every launch of the step, eager or replayed
  p->step += 1;
  if (p->prof_on && p->prof_steps < kProfMaxSteps) p->prof_steps += 1;
  return SCE_OK;
}

// ------------------------------------------------------------------------------------------------
// C ABI
// ------------------------------------------------------------------------------------------------
extern "C" {

static size_t plan_workspace(const sce_desc& d, const PlanConfig& cfg) {
  PlanBuffers w{};
  return carve(w, d, cfg, nullptr);
}

size_t sce_workspace_bytes(const sce_desc* desc) {
  if (validate(desc)) return 0;
  return plan_workspace(*desc, plan_config(*desc));
}

int sce_plan_create(const sce_desc* desc, const sce_buffers* buffers, sce_plan** out_plan) {
  if (!out_plan) return fail(SCE_ERR_INVALID, "out_plan is NULL");
  *out_plan = nullptr;
  int rc = validate(desc);
  if (rc) return rc;
  if (!buffers) return fail(SCE_ERR_INVALID, "buffers is NULL");
  const sce_buffers& b = *buffers;
  if (!b.encoder || !b.encoder_m || !b.encoder_v) return fail(SCE_ERR_INVALID, "encoder / encoder_m / encoder_v are required");
  if (base_variant(*desc) == SCE_UNTIED && (!b.decoder || !b.decoder_m || !b.decoder_v))
    return fail(SCE_ERR_INVALID, "untied variant needs decoder / decoder_m / decoder_v");
  if (desc->variant != SCE_TOPK && (!b.encoder_bias || !b.bias_m || !b.bias_v))
    return fail(SCE_ERR_INVALID, "encoder_bias / bias_m / bias_v are required for SAE variants");
  if (desc->variant == SCE_TOPK && !b.sparsity) return fail(SCE_ERR_INVALID, "top-k variant needs the sparsity buffer");
  if (desc->variant == SCE_TIED_LEARNED_CENTER && (!b.center || !b.center_m || !b.center_v))
    return fail(SCE_ERR_INVALID, "the learned-centre variant needs center / center_m / center_v");
  if (b.coef_mask && (desc->encoder_nonneg || desc->input_shift != 0.f))
    return fail(SCE_ERR_INVALID, "encoder_nonneg / input_shift cannot be combined with coef_mask");
  const PlanConfig cfg = plan_config(*desc);
  rc = check_workspace(b.workspace, b.workspace_bytes, plan_workspace(*desc, cfg), "");
  if (rc) return rc;
  int dev = 0, sms = 0;
  rc = query_device(&dev, &sms);
  if (rc) return rc;
  sce_plan* p = new (std::nothrow) sce_plan;
  if (!p) return fail(SCE_ERR_INVALID, "out of host memory");
  memset(p, 0, sizeof(*p));
  p->d = *desc;
  p->b = b;
  p->cfg = cfg;
  p->sms = sms;
  p->device = dev;
  p->maps = new std::map<int, BatchMaps*>();
  carve(*p, *desc, cfg, static_cast<uint8_t*>(b.workspace));
  *out_plan = p;
  return SCE_OK;
}

int sce_plan_destroy(sce_plan* plan) {
  if (!plan) return SCE_OK;
  for (auto& kv : *plan->maps) {
    if (kv.second->graph) cudaGraphExecDestroy(kv.second->graph);
    delete kv.second;
  }
  delete plan->maps;
  if (plan->cap_stream) cudaStreamDestroy(plan->cap_stream);
  if (plan->prof_ev) {
    for (int i = 0; i < kProfMaxSteps * (SCE_PHASE_COUNT + 1); ++i) cudaEventDestroy(plan->prof_ev[i]);
    free(plan->prof_ev);
  }
  delete plan;
  return SCE_OK;
}

int sce_prepare(sce_plan* p, void* stream) {
  if (!p) return fail(SCE_ERR_INVALID, "plan is NULL");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  CUDA_TRY(cudaMemsetAsync(p->res_flags, 0, kFlagWords * sizeof(uint32_t), st));   // residual flag, input range monitor, health
  const sce_desc& d = p->d;
  const int kmax = p->cfg.tk_kmax;   // (top-k plans only)
  std::vector<long long> ks;
  if (p->cfg.topk) {
    // the selection scatters k entries into the code planes but records (and clears on the next call) at most the list
    // capacity of them, and a k below 1 leaves its bound undefined: hold every k to [1, n] and, with lists, to topk_k_max
    ks.resize(d.n_models);
    CUDA_TRY(cudaMemcpyAsync(ks.data(), p->b.sparsity, ks.size() * sizeof(long long), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    for (int m = 0; m < d.n_models; ++m) {
      if (ks[m] < 1 || ks[m] > d.n)
        return fail(SCE_ERR_INVALID, "sparsity of model %d = %lld outside [1, n = %d]", m, ks[m], d.n);
      if (kmax && ks[m] > d.topk_k_max)
        return fail(SCE_ERR_INVALID, "sparsity of model %d = %lld exceeds desc.topk_k_max = %d, the top-k list capacity the "
                    "plan was created with", m, ks[m], d.topk_k_max);
    }
  }
  if (kmax) {
    // the top-k selection keeps the code planes (and, in k-sparse plans, the code-gradient planes) all-zero except for
    // the entries its lists record: start them zeroed, with empty lists
    const size_t el = (size_t)d.n_models * d.batch_max * d.n;
    CUDA_TRY(p->c.zero(el, st));
    CUDA_TRY(cudaMemsetAsync(p->dz.hi, 0, el * 4, st));   // (the code-gradient planes are one contiguous block, 4 B / element)
    CUDA_TRY(cudaMemsetAsync(p->act_pos, 0, (size_t)d.n_models * ((d.n + 31) / 32) * d.batch_max * sizeof(uint32_t), st));
    CUDA_TRY(cudaMemsetAsync(p->tk_cnt, 0, (size_t)d.n_models * d.batch_max * sizeof(int), st));
    // k classes for the gather kernel: rows of shared memory in {8, 16, 32, 64, ...} capped at the list capacity
    const int caps[4] = {16, 32, 64, kmax};
    std::vector<int> order;
    p->tk_groups = 0;
    p->tk_group_off[0] = 0;
    int lo = 0;
    for (int g = 0; g < 4; ++g) {
      const int cap = caps[g] < kmax ? caps[g] : kmax;
      if (g > 0 && cap <= lo) continue;
      for (int m = 0; m < d.n_models; ++m) {
        if (ks[m] > lo && ks[m] <= cap) order.push_back(m);   // (1 <= k <= topk_k_max <= kmax: checked above)
      }
      p->tk_group_krows[p->tk_groups] = cap;
      p->tk_group_off[++p->tk_groups] = (int)order.size();
      lo = cap;
      if (cap == kmax) break;
    }
    if ((int)order.size() != d.n_models) return fail(SCE_ERR_INVALID, "top-k classes: %d of %d models placed", (int)order.size(), d.n_models);
    CUDA_TRY(cudaMemcpyAsync(p->tk_models, order.data(), order.size() * sizeof(int), cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaStreamSynchronize(st));   // (`order` is a local)
  }
  Launcher L{st};
  if (d.centering) {
    if (!p->b.center_trans || !p->b.center_rot || !p->b.center_scale)
      return fail(SCE_ERR_INVALID, "centering needs the center_trans / center_rot / center_scale buffers");
    const long long n4 = (long long)d.n_models * d.d * d.d / 4;
    TRY(with_arith(p->cfg.arith, [&](auto arith) {
      return launch_split_rows<decltype(arith)::value>(L, p->b.center_rot, p->rot, n4, nullptr);
    }));
  }
  return prepare_dict(L, p);
}

int sce_forward(sce_plan* p, const float* x, int B, float* x_hat, float* out_losses, float* out_nnz, void* stream) {
  if (!p) return fail(SCE_ERR_INVALID, "plan is NULL");
  PlanCall c;
  TRY(run_pipeline(c, p, x, B, static_cast<cudaStream_t>(stream), x_hat, false, out_losses, out_nnz));
  p->last_launches = c.count;
  return SCE_OK;
}

int sce_step(sce_plan* p, const float* x, int B, float* out_losses, float* out_nnz, void* stream) {
  if (!p) return fail(SCE_ERR_INVALID, "plan is NULL");
  TRY(check_trainable(p, ""));
  return step_impl(p, x, B, out_losses, out_nnz, static_cast<cudaStream_t>(stream), nullptr);
}

int sce_grads(sce_plan* p, const float* x, int B, float* d_encoder, float* d_bias, float* d_decoder,
              float* out_losses, float* out_nnz, void* stream) {
  if (!p) return fail(SCE_ERR_INVALID, "plan is NULL");
  TRY(check_trainable(p, ""));
  PlanCall c;
  TRY(run_pipeline(c, p, x, B, static_cast<cudaStream_t>(stream), nullptr, true, out_losses, out_nnz));
  p->last_launches = c.count;   // the pipeline's: the gradient kernels below are not counted
  float* const grad_out[2] = {d_encoder, d_decoder};
  return train_tail<MODE_GRAD>(c, hyper_for(p, 1), grad_out, d_bias);
}

int sce_step_host(sce_plan* p, const float* x_host, int B, float* out_losses_host, float* out_nnz_host,
                  void* stream) {
  if (!p) return fail(SCE_ERR_INVALID, "plan is NULL");
  TRY(check_trainable(p, ""));
  if (!x_host) return fail(SCE_ERR_INVALID, "x_host is NULL");
  if (int rc = check_rows(p, B, "")) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const size_t bytes = (size_t)p->cfg.input_models * B * p->d.d * sizeof(float);
  CUDA_TRY(cudaMemcpyAsync(p->x_stage, x_host, bytes, cudaMemcpyHostToDevice, st));
  int rc = sce_step(p, p->x_stage, B, p->loss_stage, p->nnz_stage, st);
  if (rc) return rc;
  if (out_losses_host)
    CUDA_TRY(cudaMemcpyAsync(out_losses_host, p->loss_stage, (size_t)p->d.n_models * 4 * sizeof(float),
                             cudaMemcpyDeviceToHost, st));
  if (out_nnz_host)
    CUDA_TRY(cudaMemcpyAsync(out_nnz_host, p->nnz_stage, (size_t)p->d.n_models * sizeof(float), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaStreamSynchronize(st));
  return SCE_OK;
}

int sce_read_center_grad(sce_plan* p, float* d_center, void* stream) {
  if (!p || !d_center) return fail(SCE_ERR_INVALID, "plan / d_center is NULL");
  if (!p->cfg.learned) return fail(SCE_ERR_INVALID, "read_center_grad: the plan has no learned centre");
  CUDA_TRY(cudaMemcpyAsync(d_center, p->center_grad, (size_t)p->d.n_models * p->d.d * sizeof(float),
                           cudaMemcpyDeviceToDevice, static_cast<cudaStream_t>(stream)));
  return SCE_OK;
}


int sce_last_launch_count(const sce_plan* plan) { return plan ? plan->last_launches : 0; }
int sce_input_absmax(sce_plan* plan, float* out_host, void* stream) {
  if (!plan || !out_host) return fail(SCE_ERR_INVALID, "plan / out_host is NULL");
  *out_host = 0.f;
  if (plan->cfg.arith != kArithF16F8) return SCE_OK;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  uint32_t bits = 0;
  CUDA_TRY(cudaMemcpyAsync(&bits, plan->res_flags + kAbsmaxWord, sizeof(bits), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaStreamSynchronize(st));
  memcpy(out_host, &bits, sizeof(bits));
  return SCE_OK;
}
int sce_health(sce_plan* plan, int* bad_out, float* absmax_out, void* stream) {
  if (!plan) return fail(SCE_ERR_INVALID, "plan is NULL");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  uint32_t words[kFlagWords];
  CUDA_TRY(cudaMemcpyAsync(words, plan->res_flags, sizeof(words), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaStreamSynchronize(st));
  if (bad_out) *bad_out = words[kBadWord] != 0u;
  if (absmax_out) {
    *absmax_out = 0.f;
    if (plan->cfg.arith == kArithF16F8) memcpy(absmax_out, &words[kAbsmaxWord], sizeof(float));
  }
  return SCE_OK;
}
int sce_clear_health(sce_plan* plan, void* stream) {
  if (!plan) return fail(SCE_ERR_INVALID, "plan is NULL");
  CUDA_TRY(cudaMemsetAsync(plan->res_flags + kBadWord, 0, sizeof(uint32_t), static_cast<cudaStream_t>(stream)));
  return SCE_OK;
}

int sce_plan_arith(const sce_plan* plan) {
  return !plan ? 0 : plan->cfg.arith == kArithF16F8 ? SCE_ARITH_F16F8 : SCE_ARITH_BF16X3;
}

int sce_profile_begin(sce_plan* p) {
  if (!p) return fail(SCE_ERR_INVALID, "plan is NULL");
  if (!p->prof_ev) {
    const int n = kProfMaxSteps * (SCE_PHASE_COUNT + 1);
    p->prof_ev = static_cast<cudaEvent_t*>(calloc(n, sizeof(cudaEvent_t)));
    if (!p->prof_ev) return fail(SCE_ERR_INVALID, "out of host memory");
    for (int i = 0; i < n; ++i) CUDA_TRY(cudaEventCreate(&p->prof_ev[i]));
  }
  p->prof_steps = 0;
  p->prof_on = true;
  return SCE_OK;
}

int sce_profile_end(sce_plan* p, float* phase_ms, int* steps_recorded) {
  if (!p || !phase_ms) return fail(SCE_ERR_INVALID, "plan / phase_ms is NULL");
  p->prof_on = false;
  for (int k = 0; k < SCE_PHASE_COUNT; ++k) phase_ms[k] = 0.f;
  for (int s = 0; s < p->prof_steps; ++s) {
    cudaEvent_t* ev = p->prof_ev + s * (SCE_PHASE_COUNT + 1);
    CUDA_TRY(cudaEventSynchronize(ev[SCE_PHASE_COUNT]));
    for (int k = 0; k < SCE_PHASE_COUNT; ++k) {
      float ms = 0.f;
      CUDA_TRY(cudaEventElapsedTime(&ms, ev[k], ev[k + 1]));
      phase_ms[k] += ms;
    }
  }
  if (steps_recorded) *steps_recorded = p->prof_steps;
  return SCE_OK;
}

long long sce_get_step_count(const sce_plan* plan) { return plan ? plan->step : 0; }
int sce_set_step_count(sce_plan* plan, long long steps_taken) {
  if (!plan || steps_taken < 0) return fail(SCE_ERR_INVALID, "bad arguments to sce_set_step_count");
  plan->step = steps_taken;
  return SCE_OK;
}

}  // extern "C"
