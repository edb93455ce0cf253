// sce_engine.cu — libsce.so: the C ABI of include/sce.h on top of the wgmma GEMM core and the
// streaming kernels. One `sce_plan` = one stacked ensemble (FunctionalEnsemble, autoencoders/ensemble.py:68-97).
//
// One training step (tied variant; untied and top-k differ as noted; "(hi, lo)" stands for the operand planes of the
// plan's arithmetic: fp16 + two E5M2 planes with f16f8, a bf16 pair with bf16x3) is
//   split_rows      x -> (x_hi, x_lo)  [+ residual-plane flag, input range monitor]
//   GEMM encode     z = x W^T (+b) -> relu -> (c_hi, c_lo), activity masks, sum|c|, nnz   [M x B x n, K = d]
//   GEMM decode     x^ = c W -> r = x^ - x, sum r^2, g = 2r/(Bd) -> (g_hi, g_lo)  [M x B x d, K = n]
//   GEMM dcode      dz = (g W^T + alpha/B [c>0]) [z>=0] -> (dz_hi, dz_lo), db partials
//   GEMM dW         dW = dz^T x + c^T g                                            [M x n x d, K = 2B]
//   bias_norm, finalize (losses), dict_rows<ADAM> (Jacobian + Adam + renormalise + re-split), bias<ADAM>
// Top-k variant: the encode GEMM stores fp32 scores; topk_select2_kernel keeps k per row; with the k-sparse path
// (sce_topk.cuh) decode and dcode are a gather kernel over the k selected dictionary rows instead of two dense GEMMs.
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <vector>
#include <new>

#include "../../include/sce.h"
#include "sce_epilogues.cuh"
#include "sce_gemm.cuh"
#include "sce_kernels.cuh"
#include "sce_synth.cuh"
#include "sce_topk.cuh"
#include "sce_tmap.h"

using namespace sce;

// ------------------------------------------------------------------------------------------------
// errors
// ------------------------------------------------------------------------------------------------
static thread_local char g_err[512] = "";
static int fail(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}
#define CUDA_TRY(x)                                                                            \
  do {                                                                                         \
    cudaError_t e_ = (x);                                                                      \
    if (e_ != cudaSuccess) return fail(SCE_ERR_CUDA, "%s failed: %s", #x, cudaGetErrorString(e_)); \
  } while (0)

// ------------------------------------------------------------------------------------------------
// plan
// ------------------------------------------------------------------------------------------------
struct GemmMaps {  // tensor maps of one GEMM for one batch size (x8: third plane of the f16f8 arithmetic)
  CUtensorMap a_hi[kMaxSets], a_lo[kMaxSets], b_hi[kMaxSets], b_lo[kMaxSets];
  CUtensorMap a_x8[kMaxSets], b_x8[kMaxSets];
};
struct BatchMaps {
  GemmMaps encode, decode, dcode, dw_enc, dw_dec;
  GemmMaps center;             // centring: A = (x - trans) planes [M,B,d], B = rot planes [M,d,d], both K-major
  CUtensorMap st_c_hi, st_c_lo, st_c_x8, st_dz_hi, st_dz_lo, st_dz_x8;  // epilogue TMA-store maps
  CUtensorMap st_scores;                                                // top-k: fp32 scores
  cudaGraphExec_t graph;       // captured step for this batch size (launch-bound shapes), or nullptr
  int graph_launches, eager_steps;
};

struct sce_plan {
  sce_desc d;
  sce_buffers b;
  int sms;
  int device;  // CUDA device the plan was created on (the caller keeps it current for every call)
  int xm;  // number of distinct input batches (1 shared, or M)
  // workspace carve-up
  // Operand planes. bf16x3: hi, lo = bf16 planes (2 B / element each), x8 unused. f16f8: hi = fp16 plane, lo =
  // e5m2 plane of the values, x8 = e5m2 plane of the scaled residuals (1 B / element each): 4 B / element either way.
  int arith;                      // kArithBf16x3 or kArithF16F8 (resolved from desc.arith / env SCE_ARITH / the shape)
  float* x_stage;                 // [xm, Bmax, d] staging for host-fed steps
  __nv_bfloat16 *x_hi, *x_lo;     // [xm, Bmax, d]
  __nv_bfloat16 *wenc_hi, *wenc_lo, *wdec_hi, *wdec_lo;  // [M, n, d] (tied: dec aliases enc)
  __nv_bfloat16 *c_hi, *c_lo;     // [M, Bmax, n]
  __nv_bfloat16 *g_hi, *g_lo;     // [M, Bmax, d]
  __nv_bfloat16 *dz_hi, *dz_lo;   // [M, Bmax, n]   (top-k: fp32 scores alias these planes; dw_native: 8-bit planes [M, n, Bp])
  uint8_t *x_x8, *wenc_x8, *wdec_x8, *c_x8, *g_x8, *dz_x8;
  // dw_native (dense f16f8 plans): batch-major copies of the 8-bit planes of x, c and g, [xm or M, cols, Bp] with Bp =
  // batch_max rounded up to 16 (TMA pitch): the weight gradient reads them K-major over the batch (E5M2 wgmma).
  // dz's 8-bit planes are written in that layout in the first place (EpiDcodeT<f16f8, true>).
  uint8_t *xt_lo, *xt_x8, *ct_lo, *ct_x8, *gt_lo, *gt_x8;
  int bpad;                        // Bp
  int code_batch_major;            // 1: the last call was a dw_native backward, which left the code's residual plane
                                   // only in its batch-major copy (ct_x8): dcode overwrote the row-major one (carve)
  int dw_native;                   // 1: the weight gradient's cross terms run on E5M2 wgmma (see native_dw_layout)
  // f16f8: the decoder's planes transposed, [M, d, n]: the decode GEMM's B operand, K-major (transpose_dict)
  __nv_bfloat16 *wdt_hi, *wdt_lo;
  uint8_t* wdt_x8;
  __nv_bfloat16 *rot_hi, *rot_lo;  // centring: operand planes of buffers["center_rot"] [M, d, d]
  uint8_t* rot_x8;
  float* x_centered;              // centring: the centred batch [M, B, d] (B, not Bmax, rows per model: what a caller's [M,B,d] looks like)
  float* scores;                  // top-k: fp32 scores [M, Bmax, n] of the encode GEMM
  int* tk_models;                 // top-k gather kernel: the models sorted into k classes (device copy of tk_group_models)
  int tk_groups, tk_group_off[5], tk_group_krows[4];   // classes: models [off[g], off[g+1]) need at most krows[g] rows
  uint32_t* tk_cmax;              // top-k: largest key per 32-column chunk of the scores [M, Bmax, n_chunks] (EpiScoresTma)
  int topk_cmax;                  // 1: the selection works from the chunk maxima (SCE_TOPK_CMAX=0 turns it off)
  int *tk_col, *tk_cnt;           // top-k lists (TopkLists): selected columns [M, Bmax, kmax], entries per row [M, Bmax]
  float *tk_val, *tk_dots;        // their values [M, Bmax, kmax]; per-slice shares of g . W_j [M, Bmax, kmax, slices]
  float* wn_f32;                  // top-k: fp32 copy of the normalised dictionary [M, n, d] the gather kernel reads
  int tk_slices;                  // slices of the activation width topk_sparse_kernel runs per row
  int tk_kmax;                    // list capacity per row (desc.topk_k_max rounded up to 8; 0: no lists)
  int topk_sparse;                // 1: decode / dcode of the top-k variant run as the k-sparse gather kernels
  uint32_t *act_pos, *act_zero;   // activity masks [M][ceil(n/32)][Bmax]: bit 31-j of a word = column 32*chunk + j (ActMask)
  uint32_t* res_flags;            // [0]: the batch has a non-zero residual plane (f16f8; written by the batch split)
  float *dw_enc, *dw_dec;         // [M, n, d]
  float *part_enc, *part_dec, *db_part, *bnorm, *l1_over_b, *loss_stage, *nnz_stage;
  int tiles_mB_max;
  std::map<int, BatchMaps*>* maps;
  cudaStream_t cap_stream;  // private stream the step is captured on
  int dcode_passes, dw_passes;  // tensor passes of the two backward GEMMs (default: desc.bwd_passes)
  int use_graph;     // 1: replay the step as a CUDA graph (launch-bound shapes; env SCE_GRAPH overrides)
  int split_decode;  // 1: separate accumulators for hi*hi and the cross terms in the decode GEMM
  int last_launches;
  long long step;  // number of optimiser steps taken
  // optional per-phase device timing (sce_profile_*): events bracket each phase of a step
  bool prof_on;
  int prof_steps;                          // steps recorded since sce_profile_begin
  cudaEvent_t* prof_ev;                    // [kProfMaxSteps][SCE_PHASE_COUNT + 1]
};

constexpr int kProfMaxSteps = 64;
static inline void prof_mark(sce_plan* p, int idx, cudaStream_t st) {
  if (p->prof_on && p->prof_steps < kProfMaxSteps)
    cudaEventRecord(p->prof_ev[p->prof_steps * (SCE_PHASE_COUNT + 1) + idx], st);
}

static size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

struct Carve {
  uint8_t* base;
  size_t off;
  template <class T>
  T* take(size_t count) {
    off = align_up(off, 1024);
    T* p = base ? reinterpret_cast<T*>(base + off) : nullptr;
    off += count * sizeof(T);
    return p;
  }
};

static int validate(const sce_desc* d) {
  if (!d) return fail(SCE_ERR_INVALID, "desc is NULL");
  if (d->variant < SCE_TIED || d->variant > SCE_TOPK) return fail(SCE_ERR_INVALID, "unknown variant %d", d->variant);
  if (d->n_models < 1 || d->batch_max < 1) return fail(SCE_ERR_INVALID, "n_models and batch_max must be >= 1");
  if (d->d < 8 || d->d % 8 || d->n < 8 || d->n % 8)
    return fail(SCE_ERR_INVALID, "d (%d) and n (%d) must be positive multiples of 8", d->d, d->n);
  if (d->d > 8192) return fail(SCE_ERR_INVALID, "d = %d > 8192 is not supported by the row kernels", d->d);
  if ((d->fwd_passes != 1 && d->fwd_passes != 3) || (d->bwd_passes != 1 && d->bwd_passes != 3))
    return fail(SCE_ERR_INVALID, "fwd_passes / bwd_passes must be 1 or 3");
  if (d->centering < 0 || d->centering > 2) return fail(SCE_ERR_INVALID, "centering must be 0, 1 or 2");
  if (d->centering && !d->x_per_model) return fail(SCE_ERR_INVALID, "centering needs x_per_model = 1 (the centred batch differs per model)");
  if (d->arith < SCE_ARITH_AUTO || d->arith > SCE_ARITH_F16F8) return fail(SCE_ERR_INVALID, "unknown arith %d", d->arith);
  if (d->arith == SCE_ARITH_F16F8 && (d->d % 16 || d->n % 16))
    return fail(SCE_ERR_INVALID, "arith = F16F8 needs d (%d) and n (%d) to be multiples of 16 (TMA pitch of the 8-bit planes)",
                d->d, d->n);
  return SCE_OK;
}

// one call's rows: 1 <= B <= batch_max (`prefix` names the entry point in the message, "" for the training calls)
static int check_rows(const sce_plan* p, int B, const char* prefix) {
  if (B < 1 || B > p->d.batch_max)
    return fail(SCE_ERR_INVALID, "%sB = %d outside [1, batch_max = %d]", prefix, B, p->d.batch_max);
  return SCE_OK;
}

// a caller's workspace: at least `need` bytes at a 1024-byte aligned address (the carves align their buffers to it)
static int check_workspace(const void* ws, size_t have, size_t need, const char* prefix) {
  if (!ws || have < need)
    return fail(SCE_ERR_WORKSPACE, "%sworkspace too small: have %zu bytes, need %zu", prefix, have, need);
  if (reinterpret_cast<uintptr_t>(ws) % 1024) return fail(SCE_ERR_WORKSPACE, "%sworkspace must be 1024-byte aligned", prefix);
  return SCE_OK;
}

// the current device and its SM count, if libsce runs on it: sm_90, with the driver's tensor-map encoder
static int query_device(int* device, int* sm_count) {
  int dev = 0, major = 0, sms = 0;
  CUDA_TRY(cudaGetDevice(&dev));
  CUDA_TRY(cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev));
  CUDA_TRY(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  if (major != 9) return fail(SCE_ERR_NO_DEVICE, "libsce needs an sm_90 device (found compute capability %d.x)", major);
  if (!get_encode_fn()) return fail(SCE_ERR_NO_DEVICE, "cuTensorMapEncodeTiled driver entry point not available");
  *device = dev;
  *sm_count = sms;
  return SCE_OK;
}

// fp32 rows -> the operand planes of arithmetic AR: n4 float4s, grid-stride over at most 2048 blocks
template <int AR>
static void launch_split_rows(const float* x, void* hi, void* lo, void* x8, long long n4, uint32_t* flags, cudaStream_t st) {
  const int blocks = (int)((n4 + 255) / 256 < 2048 ? (n4 + 255) / 256 : 2048);
  split_rows_kernel<AR><<<blocks, 256, 0, st>>>(x, hi, lo, x8, n4, flags);
}

// desc.arith -> kArithBf16x3 / kArithF16F8. AUTO: f16f8 where the 8-bit planes can be addressed by TMA
// (row pitches of 16 bytes), bf16x3 otherwise; the environment may pin AUTO to one of them (A/B runs).
static int resolve_arith(const sce_desc& d) {
  if (d.arith == SCE_ARITH_BF16X3) return kArithBf16x3;
  if (d.arith == SCE_ARITH_F16F8) return kArithF16F8;
  const bool shape_ok = d.d % 16 == 0 && d.n % 16 == 0;
  if (const char* v = getenv("SCE_ARITH")) {
    if (!strcmp(v, "bf16x3")) return kArithBf16x3;
    if (!strcmp(v, "f16f8") && shape_ok) return kArithF16F8;
  }
  return shape_ok ? kArithF16F8 : kArithBf16x3;
}

// capacity per row of the top-k lists: the largest k of the ensemble (desc.topk_k_max, supplied by the host mirror, which
// knows buffers["sparsity"]) rounded up to 8; 0 = unknown or too large for the gather kernel -> dense path, no lists
static size_t topk_kmax(const sce_desc& d) {
  if (d.variant != SCE_TOPK || d.topk_k_max < 1 || d.topk_k_max > 256) return 0;
  return (size_t)(d.topk_k_max + 7) / 8 * 8;
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
    if (d.d % (4 * s) || d.d / s > 512) continue;
    const size_t b = topk_sparse_smem(d, kmax, s);
    if (b <= 112 * 1024) return s;   // fewest slices that fit: the kernel's time goes with the number of blocks
  }
  return best;
}

// ~30 M B n d tensor FLOPs are issued per step; below ~3e11 (a fifth of a millisecond) launches dominate
static bool launch_bound(const sce_desc& d) {
  return 30.0 * d.n_models * (double)d.batch_max * d.n * d.d < 3e11;
}
// Dense f16f8 plans with split backward GEMMs keep batch-major copies of the 8-bit planes of x, c, g and dz, from which the
// weight gradient forms its cross terms on E5M2 wgmma. Top-k plans do not: their code and (k-sparse) code-gradient planes
// are written by the selection / scatter kernels, row-major only, so their weight gradient widens the 8-bit tiles. Nor do
// launch-bound plans: there the weight gradient takes microseconds either way, and the copies would add three launches
// per step and a third to the workspace.
static bool native_dw_layout(const sce_desc& d) {
  return resolve_arith(d) == kArithF16F8 && d.variant != SCE_TOPK && d.bwd_passes >= 3 && !launch_bound(d);
}
static size_t batch_pad(const sce_desc& d) { return ((size_t)d.batch_max + 15) / 16 * 16; }

// Carves the workspace; with base == nullptr only measures it.
static size_t carve(sce_plan* p, const sce_desc& d, uint8_t* base) {
  Carve c{base, 0};
  const size_t M = d.n_models, B = d.batch_max, n = d.n, dd = d.d;
  const size_t xm = d.x_per_model ? M : 1;
  const size_t tiles_mB = (B + kBM - 1) / kBM;
  const size_t tiles_nN = (n + kBN - 1) / kBN;
  const size_t tiles_nD = (dd + kBN - 1) / kBN;
  const bool f8 = resolve_arith(d) == kArithF16F8;
  // the planes of one operand tensor: 16-bit, then (bf16x3) a second 16-bit plane or (f16f8) two 8-bit planes
  auto planes = [&](size_t count, __nv_bfloat16*& hi, __nv_bfloat16*& lo, uint8_t*& x8) {
    hi = c.take<__nv_bfloat16>(count);
    if (f8) {
      lo = reinterpret_cast<__nv_bfloat16*>(c.take<uint8_t>(count));
      x8 = c.take<uint8_t>(count);
    } else {
      lo = c.take<__nv_bfloat16>(count);
      x8 = nullptr;
    }
  };
  auto X = c.take<float>(xm * B * dd);
  __nv_bfloat16 *xh, *xl, *weh, *wel, *ch, *cl, *gh, *gl;
  uint8_t *x8, *we8, *c8, *g8;
  planes(xm * B * dd, xh, xl, x8);
  planes(M * n * dd, weh, wel, we8);
  __nv_bfloat16 *wdh = weh, *wdl = wel;
  uint8_t* wd8 = we8;
  if (d.variant == SCE_UNTIED) planes(M * n * dd, wdh, wdl, wd8);
  __nv_bfloat16 *wth = nullptr, *wtl = nullptr;
  uint8_t* wt8 = nullptr;
  if (f8) planes(M * n * dd, wth, wtl, wt8);
  const bool tdw = native_dw_layout(d);
  const size_t Bp = batch_pad(d);
  const size_t dz8 = tdw ? M * n * Bp : M * B * n;   // bytes of one 8-bit plane of dz
  uint8_t *xtl = nullptr, *xtx = nullptr, *ctl = nullptr, *ctx = nullptr, *gtl = nullptr, *gtx = nullptr;
  if (!tdw) {
    planes(M * B * n, ch, cl, c8);
  } else {
    // the code's row-major 8-bit planes are read by the decode GEMM only, which runs before dcode writes dz: they live in
    // dz's 8-bit planes (below), and the code's own 8-bit space holds the batch-major copies the weight gradient reads
    ch = c.take<__nv_bfloat16>(M * B * n);
    ctl = c.take<uint8_t>(dz8);
    ctx = c.take<uint8_t>(dz8);
  }
  planes(M * B * dd, gh, gl, g8);
  // all planes contiguous, 4 B / element (the top-k scores alias them); with tdw the 8-bit ones are [M][n][Bp]
  auto dzh = c.take<__nv_bfloat16>(M * B * n + dz8);
  if (tdw) {
    cl = reinterpret_cast<__nv_bfloat16*>(reinterpret_cast<uint8_t*>(dzh) + 2 * M * B * n);
    c8 = reinterpret_cast<uint8_t*>(dzh) + 2 * M * B * n + dz8;
    xtl = c.take<uint8_t>(xm * dd * Bp);
    xtx = c.take<uint8_t>(xm * dd * Bp);
    gtl = c.take<uint8_t>(M * dd * Bp);
    gtx = c.take<uint8_t>(M * dd * Bp);
  }
  auto dwe = c.take<float>(M * n * dd);
  float* dwd = dwe;
  if (d.variant == SCE_UNTIED) dwd = c.take<float>(M * n * dd);
  const size_t enc_parts = d.variant == SCE_TOPK ? B : tiles_mB * 8 * tiles_nN;
  auto pe = c.take<float>(M * enc_parts * 2);
  const size_t dec_parts = tiles_mB * 8 * tiles_nD;   // top-k: up to kTopkMaxSlices partials per row from the gather kernel
  auto pd = c.take<float>(M * (d.variant == SCE_TOPK && dec_parts < kTopkMaxSlices * B ? kTopkMaxSlices * B : dec_parts));
  auto dbp = c.take<float>(M * tiles_mB * 4 * n);
  auto bn = c.take<float>(M);
  auto lob = c.take<float>(M);
  auto ls = c.take<float>(M * 4);
  auto ns = c.take<float>(M);
  const size_t n_chunks = (n + 31) / 32;
  auto apos = c.take<uint32_t>(M * n_chunks * B);
  auto azero = c.take<uint32_t>(M * n_chunks * B);
  // top-k: scores of their own (the code-gradient planes must keep their scattered zeros) and the k-sparse lists
  const size_t kmax = topk_kmax(d);
  float* sc = nullptr;
  int *tkc = nullptr, *tkn = nullptr, *tkm = nullptr;
  float *tkv = nullptr, *tkd = nullptr, *wnf = nullptr;
  uint32_t* tcm = nullptr;
  if (d.variant == SCE_TOPK) {
    sc = c.take<float>(M * B * n);
    tcm = c.take<uint32_t>(M * B * n_chunks);
    if (kmax) {
      tkc = c.take<int>(M * B * kmax);
      tkv = c.take<float>(M * B * kmax);
      tkn = c.take<int>(M * B);
      tkm = c.take<int>(M);
      tkd = c.take<float>(M * B * kmax * kTopkMaxSlices);
      wnf = c.take<float>(M * n * dd);
    }
  }
  __nv_bfloat16 *roth = nullptr, *rotl = nullptr;
  uint8_t* rot8 = nullptr;
  float* xcen = nullptr;
  if (d.centering) {
    planes(M * dd * dd, roth, rotl, rot8);
    xcen = c.take<float>(M * B * dd);
  }
  auto rf = c.take<uint32_t>(kFlagWords);   // [0] residual flag, [kAbsmaxWord] input range monitor, [kBadWord] health (separate 128-byte lines)
  if (p) {
    p->x_stage = X;
    p->x_hi = xh;
    p->x_lo = xl;
    p->wenc_hi = weh;
    p->wenc_lo = wel;
    p->wdec_hi = wdh;
    p->wdec_lo = wdl;
    p->c_hi = ch;
    p->c_lo = cl;
    p->g_hi = gh;
    p->g_lo = gl;
    p->dz_hi = dzh;
    p->dz_lo = dzh + M * B * n;
    p->dz_x8 = f8 ? reinterpret_cast<uint8_t*>(dzh) + 2 * M * B * n + dz8 : nullptr;
    p->xt_lo = xtl;
    p->xt_x8 = xtx;
    p->ct_lo = ctl;
    p->ct_x8 = ctx;
    p->gt_lo = gtl;
    p->gt_x8 = gtx;
    p->bpad = (int)Bp;
    p->x_x8 = x8;
    p->wenc_x8 = we8;
    p->wdec_x8 = wd8;
    p->wdt_hi = wth;
    p->wdt_lo = wtl;
    p->wdt_x8 = wt8;
    p->c_x8 = c8;
    p->g_x8 = g8;
    p->dw_enc = dwe;
    p->dw_dec = dwd;
    p->part_enc = pe;
    p->part_dec = pd;
    p->db_part = dbp;
    p->bnorm = bn;
    p->l1_over_b = lob;
    p->loss_stage = ls;
    p->nnz_stage = ns;
    p->res_flags = rf;
    p->rot_hi = roth;
    p->rot_lo = rotl;
    p->rot_x8 = rot8;
    p->x_centered = xcen;
    p->scores = sc;
    p->tk_cmax = tcm;
    p->tk_models = tkm;
    p->tk_col = tkc;
    p->tk_val = tkv;
    p->tk_cnt = tkn;
    p->tk_dots = tkd;
    p->wn_f32 = wnf;
    p->tk_kmax = (int)kmax;
    p->act_pos = apos;
    p->act_zero = azero;
    p->tiles_mB_max = (int)tiles_mB;
  }
  return align_up(c.off, 1024);
}

// ------------------------------------------------------------------------------------------------
// tensor maps for one batch size
// ------------------------------------------------------------------------------------------------
static int tune_flag(const char* env, int dflt) {
  const char* v = getenv(env);
  return v ? (atoi(v) != 0) : dflt;
}
// K-major 16-bit tiles [rows][bk], bk = gemm_bk(arith): the swizzle span is one tile row of 2 bk bytes
static CUtensorMapSwizzle swizzle_for_bk(int bk) {
  return bk * 2 == 64 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_128B;
}

// The planes of one operand [models][rows][cols] (cols contiguous, `mpitch` elements between models) as GEMM operand
// maps. kmajor_bk != 0: K-major tiles [box_rows][kmajor_bk]; else MN-major tiles of `box_rows` k-rows by 64 (16-bit)
// / 128 (8-bit) contiguous elements. K-major 8-bit tiles (64-byte rows in f16f8) carry the 64-byte swizzle E5M2 wgmma
// reads; MN-major ones arrive unswizzled and the GEMM widens them to fp16 (widen_tile).
static bool operand_maps(int arith, CUtensorMap* hi, CUtensorMap* lo, CUtensorMap* x8, const void* phi, const void* plo,
                         const void* px8, uint64_t models, uint64_t rows, uint64_t cols, uint64_t mpitch,
                         uint32_t box_rows, int kmajor_bk) {
  bool ok;
  if (kmajor_bk) {
    ok = make_tmap_bf16_box(hi, phi, models, rows, cols, cols, mpitch, kmajor_bk, box_rows, swizzle_for_bk(kmajor_bk));
    if (arith == kArithF16F8)
      ok = ok && make_tmap_u8_box(lo, plo, models, rows, cols, cols, mpitch, kmajor_bk, box_rows, CU_TENSOR_MAP_SWIZZLE_64B) &&
           make_tmap_u8_box(x8, px8, models, rows, cols, cols, mpitch, kmajor_bk, box_rows, CU_TENSOR_MAP_SWIZZLE_64B);
    else
      ok = ok && make_tmap_bf16_box(lo, plo, models, rows, cols, cols, mpitch, kmajor_bk, box_rows, swizzle_for_bk(kmajor_bk));
  } else {
    ok = make_tmap_bf16(hi, phi, models, rows, cols, cols, mpitch, box_rows);
    if (arith == kArithF16F8)
      ok = ok && make_tmap_u8_box(lo, plo, models, rows, cols, cols, mpitch, 128, box_rows, CU_TENSOR_MAP_SWIZZLE_NONE) &&
           make_tmap_u8_box(x8, px8, models, rows, cols, cols, mpitch, 128, box_rows, CU_TENSOR_MAP_SWIZZLE_NONE);
    else
      ok = ok && make_tmap_bf16(lo, plo, models, rows, cols, cols, mpitch, box_rows);
  }
  return ok;
}

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
  const uint64_t M = d.n_models, n = d.n, dd = d.d, xm = p->xm, Bm = d.batch_max;
  // NOTE: activations are laid out with the plan's batch_max pitch between models; only `B` rows are
  // visible through the map, so rows >= B read as zero (TMA out-of-bounds fill).
  const int ar = p->arith;
  const bool f8 = ar == kArithF16F8;
  const int bk = gemm_bk(ar);
  struct Pl { const void *hi, *lo, *x8; };
  const Pl X{p->x_hi, p->x_lo, p->x_x8}, WE{p->wenc_hi, p->wenc_lo, p->wenc_x8}, WD{p->wdec_hi, p->wdec_lo, p->wdec_x8},
      C{p->c_hi, p->c_lo, p->c_x8}, G{p->g_hi, p->g_lo, p->g_x8}, DZ{p->dz_hi, p->dz_lo, p->dz_x8};
  // activations [models][B of batch_max][cols]: K-major A tiles [128 rows][bk] / MN-major tiles of bk batch rows
  auto actk = [&](GemmMaps& g, int set, const Pl& P, uint64_t models, uint64_t cols) {
    return operand_maps(ar, &g.a_hi[set], &g.a_lo[set], &g.a_x8[set], P.hi, P.lo, P.x8, models, (uint64_t)B, cols, Bm * cols, kBM, bk);
  };
  auto act_a = [&](GemmMaps& g, int set, const Pl& P, uint64_t models, uint64_t cols) {
    return operand_maps(ar, &g.a_hi[set], &g.a_lo[set], &g.a_x8[set], P.hi, P.lo, P.x8, models, (uint64_t)B, cols, Bm * cols, bk, 0);
  };
  auto act_b = [&](GemmMaps& g, int set, const Pl& P, uint64_t models, uint64_t cols) {
    return operand_maps(ar, &g.b_hi[set], &g.b_lo[set], &g.b_x8[set], P.hi, P.lo, P.x8, models, (uint64_t)B, cols, Bm * cols, bk, 0);
  };
  // dictionary [M][n][d] as the B operand: K-major tiles [box_rows][bk] (box_rows = the tile's B rows), or MN-major
  auto dict_b = [&](GemmMaps& g, const Pl& P, uint32_t box_rows, int kmajor_bk) {
    return operand_maps(ar, &g.b_hi[0], &g.b_lo[0], &g.b_x8[0], P.hi, P.lo, P.x8, M, n, dd, n * dd, box_rows, kmajor_bk);
  };
  bool ok = true;
  // encode: A = x [xm,B,d] K-major, B = Wenc [M,n,d] K-major
  ok &= actk(m->encode, 0, X, xm, dd);
  ok &= dict_b(m->encode, WE, kBN, bk);
  if (d.centering) {
    // centring: A = (x - trans) planes in the X planes (the encode A maps), B = rot [M,d,d] K-major, output d columns
    m->center.a_hi[0] = m->encode.a_hi[0];
    m->center.a_lo[0] = m->encode.a_lo[0];
    m->center.a_x8[0] = m->encode.a_x8[0];
    ok &= operand_maps(ar, &m->center.b_hi[0], &m->center.b_lo[0], &m->center.b_x8[0], p->rot_hi, p->rot_lo, p->rot_x8, M, dd, dd,
                       dd * dd, kBN, bk);
  }
  // decode: A = c [M,B,n] K-major, B = Wdec [M,n,d] MN-major (bk k-rows per box); f16f8: its transposed copy [M,d,n] K-major
  ok &= actk(m->decode, 0, C, M, n);
  if (f8)
    ok &= operand_maps(ar, &m->decode.b_hi[0], &m->decode.b_lo[0], &m->decode.b_x8[0], p->wdt_hi, p->wdt_lo, p->wdt_x8, M, dd, n,
                       dd * n, kBN, bk);
  else
    ok &= dict_b(m->decode, WD, bk, 0);
  // dcode: A = g [M,B,d] K-major, B = Wdec K-major
  ok &= actk(m->dcode, 0, G, M, dd);
  ok &= dict_b(m->dcode, WD, kBN, bk);
  // weight gradients: everything MN-major, reduction over the batch rows. dw_native: the 8-bit planes come from the
  // batch-major copies [models][rows][Bp] instead, K-major tiles [128 rows][64 B] with the 64-byte swizzle; only B
  // columns are exposed, so the tail of a short batch reads as zero
  const uint64_t Bp = (uint64_t)p->bpad;
  struct Pt { const uint8_t *lo, *x8; };
  const Pt XT{p->xt_lo, p->xt_x8}, CT{p->ct_lo, p->ct_x8}, GT{p->gt_lo, p->gt_x8},
      DZT{reinterpret_cast<const uint8_t*>(p->dz_lo), p->dz_x8};
  auto kmaj8 = [&](CUtensorMap* lo, CUtensorMap* x8, const Pt& T, uint64_t models, uint64_t rows) {
    return make_tmap_u8_box(lo, T.lo, models, rows, (uint64_t)B, Bp, rows * Bp, bk, kBM, CU_TENSOR_MAP_SWIZZLE_64B) &&
           make_tmap_u8_box(x8, T.x8, models, rows, (uint64_t)B, Bp, rows * Bp, bk, kBM, CU_TENSOR_MAP_SWIZZLE_64B);
  };
  auto dw_set = [&](GemmMaps& g, int set, const Pl& A, const Pt& AT, uint64_t am, const Pl& Bo, const Pt& BT, uint64_t bm,
                    uint64_t bcols) {
    bool r = act_a(g, set, A, am, n) && act_b(g, set, Bo, bm, bcols);
    if (p->dw_native) r = r && kmaj8(&g.a_lo[set], &g.a_x8[set], AT, am, n) && kmaj8(&g.b_lo[set], &g.b_x8[set], BT, bm, bcols);
    return r;
  };
  if (d.variant == SCE_UNTIED) {
    ok &= dw_set(m->dw_enc, 0, DZ, DZT, M, X, XT, xm, dd);
    ok &= dw_set(m->dw_dec, 0, C, CT, M, G, GT, M, dd);
  } else {
    ok &= dw_set(m->dw_enc, 0, DZ, DZT, M, X, XT, xm, dd);
    ok &= dw_set(m->dw_enc, 1, C, CT, M, G, GT, M, dd);
  }
  ok &= make_tmap_bf16_store32(&m->st_c_hi, p->c_hi, M, (uint64_t)B, n, Bm * n);
  ok &= make_tmap_bf16_store32(&m->st_dz_hi, p->dz_hi, M, (uint64_t)B, n, Bm * n);
  if (f8) {
    auto st8 = [&](CUtensorMap* t, const void* base) {
      return make_tmap_u8_box(t, base, M, (uint64_t)B, n, n, Bm * n, 32, 32, CU_TENSOR_MAP_SWIZZLE_32B);
    };
    // dw_native: dz's 8-bit planes [M][n][Bp], boxes of 32 features x 32 batch bytes (EpiDcodeT<f16f8, true>)
    auto st8t = [&](CUtensorMap* t, const void* base) {
      return make_tmap_u8_box(t, base, M, n, (uint64_t)B, Bp, n * Bp, 32, 32, CU_TENSOR_MAP_SWIZZLE_NONE);
    };
    ok &= st8(&m->st_c_lo, p->c_lo) && st8(&m->st_c_x8, p->c_x8);
    ok &= p->dw_native ? st8t(&m->st_dz_lo, p->dz_lo) && st8t(&m->st_dz_x8, p->dz_x8)
                       : st8(&m->st_dz_lo, p->dz_lo) && st8(&m->st_dz_x8, p->dz_x8);
  } else {
    ok &= make_tmap_bf16_store32(&m->st_c_lo, p->c_lo, M, (uint64_t)B, n, Bm * n);
    ok &= make_tmap_bf16_store32(&m->st_dz_lo, p->dz_lo, M, (uint64_t)B, n, Bm * n);
  }
  if (d.variant == SCE_TOPK) ok &= make_tmap_f32_store32(&m->st_scores, p->scores, M, (uint64_t)B, n, Bm * n);
  if (!ok) {
    delete m;
    return fail(SCE_ERR_CUDA, "cuTensorMapEncodeTiled failed (B=%d, M=%d, n=%d, d=%d)", B, d.n_models, d.n, d.d);
  }
  (*p->maps)[B] = m;
  *out = m;
  return SCE_OK;
}

// ------------------------------------------------------------------------------------------------
// GEMM launcher
// ------------------------------------------------------------------------------------------------
// device flags "this operand's residual plane is all zeros" (f16f8; GemmParams::a_res_flag), nullptr = unknown
struct ResFlags {
  const uint32_t* a[kMaxSets] = {nullptr, nullptr};
  const uint32_t* b[kMaxSets] = {nullptr, nullptr};
};

// NATIVE (f16f8): the cross terms run on E5M2 wgmma, which needs K-major 8-bit maps (A_MN / B_MN then describe the fp16
// planes alone); K-major GEMMs always have them, the weight gradient where the plan keeps batch-major copies.
template <class Epi, bool A_MN, bool B_MN, bool SPLIT_ACC, int ARITH, bool NATIVE = ARITH == kArithF16F8 && !A_MN>
static int launch_gemm_t(const sce_plan* p, const GemmMaps& maps, int nsets, const int* a_batched,
                         const int* b_batched, int k_total, int passes, int m_total, int n_total,
                         const typename Epi::Params& epi, cudaStream_t st, const ResFlags& rf = ResFlags()) {
  GemmParams<typename Epi::Params> gp;
  memset(&gp, 0, sizeof(gp));
  for (int s = 0; s < nsets; ++s) {
    gp.a_hi[s] = maps.a_hi[s];
    gp.a_lo[s] = maps.a_lo[s];
    gp.b_hi[s] = maps.b_hi[s];
    gp.b_lo[s] = maps.b_lo[s];
    gp.a_x8[s] = maps.a_x8[s];
    gp.b_x8[s] = maps.b_x8[s];
    gp.a_batched[s] = a_batched[s];
    gp.b_batched[s] = b_batched[s];
    gp.a_res_flag[s] = rf.a[s];
    gp.b_res_flag[s] = rf.b[s];
  }
  gp.nsets = nsets;
  gp.k_total = k_total;
  gp.passes = passes;
  gp.n_models = p->d.n_models;
  gp.m_total = m_total;
  gp.n_total = n_total;
  gp.tiles_m = (m_total + kBM - 1) / kBM;
  gp.tiles_n = (n_total + kBN - 1) / kBN;
  gp.epi = epi;
  CUDA_TRY((launch_gemm<Epi, A_MN, B_MN, SPLIT_ACC, ARITH, NATIVE>(gp, p->device, p->sms, st)));
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

template <int MODE, int ARITH>
static int launch_dict_rows_t(float* e, const float* dw, float* m, float* v, void* hi, void* lo, void* x8,
                              float* grad_out, long long rows, int d, int normalize, float floor, AdamHyper h,
                              const uint32_t* health, float* w_f32, cudaStream_t st) {
  const int nv = (d + 511) / 512;
  if (nv == 1)
    dict_rows_kernel<1, MODE, ARITH><<<(unsigned)rows, 128, 0, st>>>(e, dw, m, v, hi, lo, x8, grad_out, d, normalize, floor, h, health, w_f32);
  else if (nv == 2)
    dict_rows_kernel<2, MODE, ARITH><<<(unsigned)rows, 128, 0, st>>>(e, dw, m, v, hi, lo, x8, grad_out, d, normalize, floor, h, health, w_f32);
  else if (nv <= 4)
    dict_rows_kernel<4, MODE, ARITH><<<(unsigned)rows, 128, 0, st>>>(e, dw, m, v, hi, lo, x8, grad_out, d, normalize, floor, h, health, w_f32);
  else if (nv <= 8)    // d <= 4096 (Pythia-6.9b residual width)
    dict_rows_kernel<8, MODE, ARITH><<<(unsigned)rows, 128, 0, st>>>(e, dw, m, v, hi, lo, x8, grad_out, d, normalize, floor, h, health, w_f32);
  else                 // d <= 8192
    dict_rows_kernel<16, MODE, ARITH><<<(unsigned)rows, 128, 0, st>>>(e, dw, m, v, hi, lo, x8, grad_out, d, normalize, floor, h, health, w_f32);
  CUDA_TRY(cudaGetLastError());
  return SCE_OK;
}
// `which`: 0 = the encoder's operand planes, 1 = the decoder's
template <int MODE>
static int launch_dict_rows(const sce_plan* p, int which, float* e, const float* dw, float* m, float* v, float* grad_out,
                            long long rows, int d, int normalize, float floor, AdamHyper h, cudaStream_t st) {
  void* hi = which ? (void*)p->wdec_hi : (void*)p->wenc_hi;
  void* lo = which ? (void*)p->wdec_lo : (void*)p->wenc_lo;
  void* x8 = which ? (void*)p->wdec_x8 : (void*)p->wenc_x8;
  if (MODE == MODE_GRAD) hi = lo = x8 = nullptr;
  float* wf = (MODE != MODE_GRAD && p->topk_sparse) ? p->wn_f32 : nullptr;   // (top-k plans have one dictionary)
  return p->arith == kArithF16F8
             ? launch_dict_rows_t<MODE, kArithF16F8>(e, dw, m, v, hi, lo, x8, grad_out, rows, d, normalize, floor, h, p->res_flags, wf, st)
             : launch_dict_rows_t<MODE, kArithBf16x3>(e, dw, m, v, hi, lo, x8, grad_out, rows, d, normalize, floor, h, p->res_flags, wf, st);
}

// f16f8: the decoder's planes -> their transposed copy, which the decode GEMM reads K-major (nothing to do where the
// decode runs without the GEMM: k-sparse top-k plans). Adds its launches to `launches`.
static int transpose_dict(const sce_plan* p, cudaStream_t st, int& launches) {
  if (p->arith != kArithF16F8 || p->topk_sparse) return SCE_OK;
  const sce_desc& d = p->d;
  const dim3 grid((d.d + 63) / 64, (d.n + 63) / 64, d.n_models);
  transpose_kernel<uint16_t><<<grid, 256, 0, st>>>(reinterpret_cast<const uint16_t*>(p->wdec_hi),
                                                   reinterpret_cast<uint16_t*>(p->wdt_hi), d.n, d.d);
  transpose_kernel<uint8_t><<<grid, 256, 0, st>>>(reinterpret_cast<const uint8_t*>(p->wdec_lo),
                                                  reinterpret_cast<uint8_t*>(p->wdt_lo), d.n, d.d);
  transpose_kernel<uint8_t><<<grid, 256, 0, st>>>(p->wdec_x8, p->wdt_x8, d.n, d.d);
  CUDA_TRY(cudaGetLastError());
  launches += 3;
  return SCE_OK;
}

// f16f8 runs the backward pass on the residual r instead of g = 2r/(B d) (EpiDecodeT): weight- and bias-gradient
// outputs are multiplied by 2/(B d) on the way out, the sparsity term enters dcode as alpha d / 2.
static float grad_out_scale(const sce_plan* p, int B) {
  return p->arith == kArithF16F8 ? 2.0f / ((float)B * (float)p->d.d) : 1.0f;
}

__global__ void l1_over_b_kernel(const float* __restrict__ alpha, float* __restrict__ out, int M, float invB) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < M) out[i] = alpha ? alpha[i] * invB : 0.f;
}

template <class T>
struct TypeTag {
  using type = T;
};

// forward (+ optional backward GEMMs). Leaves dW in p->dw_enc / p->dw_dec when `backward`.
// `mom_part` (forward only, SAE variants): the encode epilogue also writes the moment partials of EpiEncodeT<AR, true>.
template <int AR>
static int run_pipeline_t(sce_plan* p, const float* x, int B, float* x_hat, bool backward, float* out_losses,
                          float* out_nnz, cudaStream_t st, float* mom_part = nullptr) {
  using EpiEnc = EpiEncodeT<AR>;
  using EpiDec = EpiDecodeT<AR>;
  using EpiDco = EpiDcodeT<AR>;
  constexpr bool f8 = AR == kArithF16F8;
  const sce_desc& d = p->d;
  if (int rc = check_rows(p, B, "")) return rc;
  if (!x) return fail(SCE_ERR_INVALID, "x is NULL");
  BatchMaps* maps = nullptr;
  int rc = build_maps(p, B, &maps);
  if (rc) return rc;
  int launches = 0;
  const int M = d.n_models, n = d.n, dd = d.d;
  const long long Bm = d.batch_max;
  const int one[2] = {1, 1};
  const int xb[2] = {d.x_per_model ? 1 : 0, 1};
  const int tiles_mB = (B + kBM - 1) / kBM;

  prof_mark(p, SCE_PHASE_SPLIT, st);
  if (d.centering) {
    // ---- centring (sae_ensemble.py:126-128): (x - trans[m]) -> planes, GEMM with rot[m] (all split passes), * scale[m]
    // -> the per-model fp32 batch every kernel below reads as `x`
    const long long n4 = (long long)B * dd / 4;
    const int blocks = (int)((n4 + 255) / 256 < 1024 ? (n4 + 255) / 256 : 1024);
    center_split_kernel<AR><<<dim3(blocks, M), 256, 0, st>>>(
        x, d.centering == 2 ? (long long)B * dd : 0, p->b.center_trans, p->x_hi, p->x_lo, p->x_x8, Bm * dd, B, dd);
    CUDA_TRY(cudaGetLastError());
    EpiCenter::Params cp;
    cp.out = p->x_centered;
    cp.model_stride = (long long)B * dd;
    cp.ld = dd;
    cp.col_scale = p->b.center_scale;
    rc = launch_gemm_t<EpiCenter, false, false, false, AR>(p, maps->center, 1, one, one, dd, 3, B, dd, cp, st);
    if (rc) return rc;
    launches += 2;
    x = p->x_centered;
  }
  // ---- x -> (hi, lo): per model slabs are batch_max apart in the workspace
  if constexpr (f8) CUDA_TRY(cudaMemsetAsync(p->res_flags, 0, sizeof(uint32_t), st));
  for (int m = 0; m < p->xm; ++m) {
    // (bf16x3: the lo plane is 2 B / element; f16f8: lo and x8 are 1 B / element)
    launch_split_rows<AR>(x + (long long)m * B * dd, p->x_hi + m * Bm * dd,
                          f8 ? (void*)(reinterpret_cast<uint8_t*>(p->x_lo) + m * Bm * dd) : (void*)(p->x_lo + m * Bm * dd),
                          f8 ? (void*)(p->x_x8 + m * Bm * dd) : nullptr, (long long)B * dd / 4, f8 ? p->res_flags : nullptr, st);
    ++launches;
  }
  CUDA_TRY(cudaGetLastError());
  // dw_native: batch-major copies of the 8-bit planes of x, c and g for the weight gradient (dz's are written so by dcode)
  const bool tdw = f8 && backward && p->dw_native;
  auto batch_major = [&](const void* lo, const uint8_t* x8, uint8_t* tlo, uint8_t* tx8, int models, int cols) {
    const BatchPlanes t{{static_cast<const uint8_t*>(lo), x8}, {tlo, tx8}};
    transpose_batch_u8_kernel<<<dim3((cols + 127) / 128, (B + 127) / 128, 2 * models), 256, 0, st>>>(t, models, B, cols,
                                                                                                 Bm * cols, p->bpad);
    ++launches;
    return cudaGetLastError();
  };
  if (tdw) CUDA_TRY(batch_major(p->x_lo, p->x_x8, p->xt_lo, p->xt_x8, p->xm, dd));
  p->code_batch_major = tdw ? 1 : 0;
  // alpha / B, or (f16f8, backward on r = g B d / 2) alpha d / 2
  l1_over_b_kernel<<<(M + 127) / 128, 128, 0, st>>>(p->b.l1_alpha, p->l1_over_b, M, f8 ? 0.5f * (float)dd : 1.0f / (float)B);
  ++launches;
  // the batch's residual-plane flag, for the GEMMs that read x as their A (encode) or B (weight gradient, set 0) operand
  ResFlags x_is_a, x_is_b;
  if constexpr (f8) {
    x_is_a.a[0] = p->res_flags;
    x_is_b.b[0] = p->res_flags;
  }
  ActMask act;
  act.pos = p->act_pos;
  act.zero = p->act_zero;
  act.n_chunks = (n + 31) / 32;
  act.batch_max = d.batch_max;
  if (d.variant == SCE_TOPK) act.zero = nullptr;   // relu semantics: no gradient at exactly 0
  // ---- encode
  prof_mark(p, SCE_PHASE_ENCODE, st);
  int n_enc_parts;
  TopkLists tk = {nullptr, nullptr, nullptr, 0, 0};
  if (d.variant != SCE_TOPK) {
    auto fill = [&](auto& ep) {
      ep.out_hi = maps->st_c_hi;
      ep.out_lo = maps->st_c_lo;
      ep.out_x8 = maps->st_c_x8;
      ep.bias = p->b.encoder_bias;
      ep.mask = p->b.coef_mask;
      ep.part = p->part_enc;
      ep.tiles_m = tiles_mB;
      ep.flag_zero = 1;
      ep.act = act;
      ep.tiles_n = (n + kBN - 1) / kBN;
    };
    if (mom_part) {
      using EpiStats = EpiEncodeT<AR, true>;
      typename EpiStats::Params ep;
      fill(ep);
      ep.mom_part = mom_part;
      ep.row_blocks = (B + 31) / 32;
      rc = launch_gemm_t<EpiStats, false, false, false, AR>(p, maps->encode, 1, xb, one, dd, d.fwd_passes, B, n, ep, st, x_is_a);
    } else {
      typename EpiEnc::Params ep;
      fill(ep);
      rc = launch_gemm_t<EpiEnc, false, false, false, AR>(p, maps->encode, 1, xb, one, dd, d.fwd_passes, B, n, ep, st, x_is_a);
    }
    if (rc) return rc;
    ++launches;
    n_enc_parts = tiles_mB * 8 * ((n + kBN - 1) / kBN);
    if (tdw) CUDA_TRY(batch_major(p->c_lo, p->c_x8, p->ct_lo, p->ct_x8, M, n));
  } else {
    // scores -> fp32, then per-row selection (code planes, activity mask, k-sparse lists)
    EpiScoresTma::Params sp;
    sp.out = maps->st_scores;
    if (p->topk_cmax) {
      sp.cmax = p->tk_cmax;
      sp.n_chunks = act.n_chunks;
      sp.cmax_model_stride = (long long)Bm * act.n_chunks;
    }
    rc = launch_gemm_t<EpiScoresTma, false, false, false, AR>(p, maps->encode, 1, xb, one, dd, d.fwd_passes, B, n, sp, st, x_is_a);
    if (rc) return rc;
    ++launches;
    CUDA_TRY(opt_in_smem<topk_sparse_kernel<AR>>(112 * 1024, p->device));
    tk.col = p->tk_col;
    tk.val = p->tk_val;
    tk.cnt = p->tk_cnt;
    tk.kmax = p->tk_kmax;
    tk.batch_max = d.batch_max;
    // one block per (row, model); scores / codes of model m start at m * batch_max * n
    topk_select2_kernel<AR><<<dim3(B, M), 256, 0, st>>>(
        p->scores, p->b.sparsity, p->c_hi, p->c_lo, p->c_x8, p->topk_sparse ? (void*)p->dz_hi : nullptr, p->dz_lo, p->dz_x8,
        act, tk, p->part_enc, B, n, Bm * n, p->topk_cmax ? p->tk_cmax : nullptr);
    ++launches;
    CUDA_TRY(cudaGetLastError());
    n_enc_parts = B;
  }

  const bool sparse = d.variant == SCE_TOPK && p->topk_sparse;
  int n_dec_parts;
  prof_mark(p, SCE_PHASE_DECODE, st);
  if (sparse) {
    // ---- k-sparse decode + residual + loss partial + g planes + the code gradient at the selected entries
    const float gscale = f8 ? 1.0f : 2.0f / ((float)B * (float)dd);
    // one launch per k class (sce_prepare sorted the models): a block's shared memory goes with ITS models' k, so the
    // k = 16 and k = 32 models of a mixed ensemble run at 5 and 3 blocks per SM instead of the 2 that k_max = 64 allows
    for (int g = 0; g < p->tk_groups; ++g) {
      const int cnt = p->tk_group_off[g + 1] - p->tk_group_off[g];
      if (cnt == 0) continue;
      topk_sparse_kernel<AR><<<dim3(B, cnt, p->tk_slices), 256, topk_sparse_smem(d, p->tk_group_krows[g], p->tk_slices), st>>>(
          tk, p->b.sparsity, p->wn_f32, x, d.x_per_model ? (long long)B * dd : 0, p->g_hi, p->g_lo, p->g_x8, x_hat, p->part_dec,
          backward ? p->tk_dots : nullptr, B, n, dd, gscale, p->tk_models + p->tk_group_off[g], p->tk_group_krows[g]);
      ++launches;
    }
    CUDA_TRY(cudaGetLastError());
    n_dec_parts = p->tk_slices * B;
  } else {
  // ---- decode (+ residual, loss partial, g)
  typename EpiDec::Params dp;
  dp.x = x;
  dp.x_model_stride = d.x_per_model ? (long long)B * dd : 0;
  dp.g_hi = reinterpret_cast<uint16_t*>(p->g_hi);
  dp.g_lo = reinterpret_cast<uint8_t*>(p->g_lo);
  dp.g_x8 = p->g_x8;
  dp.x_hat = x_hat;
  dp.part = p->part_dec;
  dp.g_model_stride = Bm * dd;
  dp.xhat_model_stride = (long long)B * dd;
  dp.ld = dd;
  dp.tiles_m = tiles_mB;
  dp.gscale = f8 ? 1.0f : 2.0f / ((float)B * (float)dd);
  dp.tiles_n = (dd + kBN - 1) / kBN;
  if constexpr (f8)
    rc = launch_gemm_t<EpiDec, false, false, false, AR>(p, maps->decode, 1, one, one, n, d.fwd_passes, B, dd, dp, st);
  else if (p->split_decode)
    rc = launch_gemm_t<EpiDec, false, true, true, AR>(p, maps->decode, 1, one, one, n, d.fwd_passes, B, dd, dp, st);
  else
    rc = launch_gemm_t<EpiDec, false, true, false, AR>(p, maps->decode, 1, one, one, n, d.fwd_passes, B, dd, dp, st);
  if (rc) return rc;
  ++launches;
  n_dec_parts = tiles_mB * 8 * dp.tiles_n;
  if (tdw) CUDA_TRY(batch_major(p->g_lo, p->g_x8, p->gt_lo, p->gt_x8, M, dd));
  }

  // ---- losses
  prof_mark(p, SCE_PHASE_LOSSES, st);
  if (p->b.encoder_bias && p->b.bias_decay) {
    bias_norm_kernel<<<M, 256, 0, st>>>(p->b.encoder_bias, n, p->bnorm);
    ++launches;
  }
  finalize_kernel<<<M, 256, 0, st>>>(p->part_enc, n_enc_parts, p->part_dec, n_dec_parts, p->b.l1_alpha,
                                     p->b.encoder_bias ? p->b.bias_decay : nullptr, p->bnorm, B, dd, out_losses, out_nnz,
                                     p->res_flags);
  ++launches;
  CUDA_TRY(cudaGetLastError());

  prof_mark(p, SCE_PHASE_DCODE, st);
  if (backward) {
    if (sparse) {
      // ---- code gradient planes: zero the rows, scatter the k entries
      topk_dz_scatter_kernel<AR><<<dim3(B, M), 64, 0, st>>>(tk, p->tk_dots, p->tk_slices, p->dz_hi, p->dz_lo, p->dz_x8, n);
      ++launches;
      CUDA_TRY(cudaGetLastError());
    } else {
    // ---- dcode
    auto dcode = [&](auto tag) {
      using E = typename decltype(tag)::type;
      typename E::Params zp;
      zp.out_hi = maps->st_dz_hi;
      zp.out_lo = maps->st_dz_lo;
      zp.out_x8 = maps->st_dz_x8;
      zp.act = act;
      zp.l1_over_b = p->l1_over_b;
      zp.db_part = p->b.encoder_bias ? p->db_part : nullptr;
      zp.tiles_m = tiles_mB;
      zp.planes = p->dw_passes >= 3 ? 3 : 0;
      // the only reader of dz's value plane is the dz^T x term of the weight gradient, against x's residual plane
      // (per-model batches carry one flag for all of them, so the same test holds)
      zp.x_res_flag = f8 ? p->res_flags : nullptr;
      return launch_gemm_t<E, false, false, false, AR>(p, maps->dcode, 1, one, one, dd, p->dcode_passes, B, n, zp, st);
    };
    // dw_native: dz's 8-bit planes are written batch-major, as the native weight gradient reads them
    if constexpr (f8) rc = p->dw_native ? dcode(TypeTag<EpiDcodeT<AR, true>>{}) : dcode(TypeTag<EpiDco>{});
    else rc = dcode(TypeTag<EpiDco>{});
    if (rc) return rc;
    ++launches;
    }

    // ---- weight gradients
    prof_mark(p, SCE_PHASE_DW, st);
    auto dw = [&](const GemmMaps& gm, int nsets, const int* ab, const int* bb, float* out, const ResFlags& rf) -> int {
      EpiStoreF32::Params sp;
      sp.out = out;
      sp.model_stride = (long long)n * dd;
      sp.ld = dd;
      sp.scale = grad_out_scale(p, B);
      // reduction over the batch: split accumulators for bf16x3 (f16f8 rescales inside one). dw_native: fp16 planes
      // MN-major, 8-bit planes K-major from their batch-major copies, cross terms on E5M2 wgmma; else widened
      if constexpr (f8)
        if (p->dw_native)
          return launch_gemm_t<EpiStoreF32, true, true, false, AR, true>(p, gm, nsets, ab, bb, B, p->dw_passes, n, dd, sp, st, rf);
      return launch_gemm_t<EpiStoreF32, true, true, !f8, AR>(p, gm, nsets, ab, bb, B, p->dw_passes, n, dd, sp, st, rf);
    };
    if (d.variant == SCE_UNTIED) {
      rc = dw(maps->dw_enc, 1, one, xb, p->dw_enc, x_is_b);
      if (rc) return rc;
      rc = dw(maps->dw_dec, 1, one, one, p->dw_dec, ResFlags());
      if (rc) return rc;
      launches += 2;
    } else {
      const int bb[2] = {xb[0], 1};
      rc = dw(maps->dw_enc, 2, one, bb, p->dw_enc, x_is_b);
      if (rc) return rc;
      ++launches;
    }
  }
  prof_mark(p, SCE_PHASE_ADAM, st);
  p->last_launches = launches;
  return SCE_OK;
}

static int run_pipeline(sce_plan* p, const float* x, int B, float* x_hat, bool backward, float* out_losses,
                        float* out_nnz, cudaStream_t st, float* mom_part = nullptr) {
  return p->arith == kArithF16F8 ? run_pipeline_t<kArithF16F8>(p, x, B, x_hat, backward, out_losses, out_nnz, st, mom_part)
                                 : run_pipeline_t<kArithBf16x3>(p, x, B, x_hat, backward, out_losses, out_nnz, st, mom_part);
}

// ------------------------------------------------------------------------------------------------
// evaluation statistics (sce_forward_stats): per-feature moments and segment activity counts
// ------------------------------------------------------------------------------------------------
// Top-k plans: moment partials from the fp32 scores and the activity mask the selection left in the workspace, in the
// layout of EncodeMomentParams ([M][row_blocks][4][n]): the code is relu(score) where the mask bit is set, 0 elsewhere.
// One warp per (32-column chunk, row block): lane j sums column 32 chunk + j over the 32 rows in order.
__global__ void __launch_bounds__(256) topk_moment_kernel(const float* __restrict__ scores, const uint32_t* __restrict__ pos,
                                                          int n_chunks, int batch_max, int B, int n, int row_blocks,
                                                          float* __restrict__ part) {
  const int chunk = blockIdx.x, model = blockIdx.z, lane = threadIdx.x & 31;
  const int rb = blockIdx.y * 8 + (threadIdx.x >> 5);
  if (rb >= row_blocks) return;
  const int col = chunk * 32 + lane;
  const uint32_t* pw = pos + ((long long)model * n_chunks + chunk) * batch_max;
  const float* s = scores + (long long)model * batch_max * n;
  float a1 = 0.f, a2 = 0.f, a3 = 0.f, a4 = 0.f;
  const int r_end = min(B, rb * 32 + 32);
  for (int r = rb * 32; r < r_end; ++r) {
    const uint32_t w = __ldg(pw + r);
    if (col < n && ((w >> (31 - lane)) & 1u)) {
      const float c = fmaxf(__ldg(s + (long long)r * n + col), 0.f), c2 = c * c;
      a1 += c;
      a2 += c2;
      a3 += c2 * c;
      a4 += c2 * c2;
    }
  }
  if (col < n) {
    float* o = part + ((long long)model * row_blocks + rb) * 4 * n + col;
    o[0] = a1;
    o[n] = a2;
    o[2 * (long long)n] = a3;
    o[3 * (long long)n] = a4;
  }
}

// sums[m][j][p] += sum over the row blocks, in order, of part[m][rb][p][j] (fp64): bitwise repeatable, no atomics
__global__ void moment_reduce_kernel(const float* __restrict__ part, int row_blocks, int n, double* __restrict__ sums) {
  const int col = blockIdx.x * blockDim.x + threadIdx.x, model = blockIdx.y;
  if (col >= n) return;
  double a[4] = {0.0, 0.0, 0.0, 0.0};
  for (int rb = 0; rb < row_blocks; ++rb) {
    const float* o = part + ((long long)model * row_blocks + rb) * 4 * n + col;
#pragma unroll
    for (int q = 0; q < 4; ++q) a[q] += (double)__ldg(o + (long long)q * n);
  }
  double* out = sums + ((long long)model * n + col) * 4;
#pragma unroll
  for (int q = 0; q < 4; ++q) out[q] += a[q];
}

// Segment activity counts (calc_moments_streaming's times_active, standard_metrics.py:482-511): the rows are cut into
// segments of `seg`; counts[m][j] += number of segments that END in this call in which some row has [c > 0] in column j.
// `phase` rows of the first segment were seen by earlier calls, whose activity is carried in open[m][j] (0 / 1); the
// flag of a segment that stays open past this call is written back there. One block per (32-column chunk, model); warp
// w takes the segments w, w + 8, ...; lanes OR 32 rows' mask words at a time, so lane j ends with column j's flag.
__global__ void __launch_bounds__(256) segment_count_kernel(const uint32_t* __restrict__ pos, int n_chunks, int batch_max,
                                                            int B, int n, int seg, int phase, int* __restrict__ counts,
                                                            int* __restrict__ open) {
  __shared__ int red[8][32];
  const int chunk = blockIdx.x, model = blockIdx.y;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint32_t* p = pos + ((long long)model * n_chunks + chunk) * batch_max;
  const int col = chunk * 32 + lane;
  const long long oi = (long long)model * n + col;
  const int carried = col < n ? open[oi] : 0;
  __syncthreads();   // every read of open[] precedes the write below
  const long long K = ((long long)B + phase + seg - 1) / seg;   // segments this call touches
  int mine = 0;
  for (long long k = warp; k < K; k += 8) {
    const long long lo = k == 0 ? 0 : k * seg - phase;
    const long long end = (k + 1) * seg - phase;
    const long long hi = end < B ? end : B;
    uint32_t any = 0u;
    for (long long r = lo + lane; r < hi; r += 32) any |= __ldg(p + r);
    any = __reduce_or_sync(0xffffffffu, any);
    int act = (int)((any >> (31 - lane)) & 1u);
    if (k == 0) act |= carried;
    if (end <= B) {
      mine += act;
      if (k == K - 1 && col < n) open[oi] = 0;
    } else if (col < n) {
      open[oi] = act;   // (only the last segment can stay open)
    }
  }
  red[warp][lane] = mine;
  __syncthreads();
  if (warp == 0) {
    int t = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) t += red[i][lane];
    if (col < n) counts[oi] += t;
  }
}

// moment partials of one forward call: [M][ceil(B / 32)][4][n] fp32
static size_t stats_workspace(const sce_desc& d, int B) {
  return align_up((size_t)d.n_models * ((B + 31) / 32) * 4 * d.n * sizeof(float), 1024);
}

// ------------------------------------------------------------------------------------------------
// top-activating and random activating fragments (sce_forward_fragments; interpret.py:82-212 record tables,
// :265-321 record selection): fragment g of a call is rows g L .. g L + L - 1.
// ------------------------------------------------------------------------------------------------
struct FragCode {             // the code of the last forward, as the engine holds it
  const void* hi;             // c_hi plane [M][batch_max][n] (bf16 or fp16)
  const void* lo;             // bf16x3: c_lo plane
  const uint8_t* x8;          // f16f8: E5M2 plane of the scaled residuals
  const float* scores;        // top-k: fp32 scores [M][batch_max][n]
  const uint32_t* pos;        // activity mask [M][n_chunks][batch_max]
  int n_chunks, batch_max, n;
};

// One element c[m, r, j] of the code: SAE variants join the operand planes exactly as join_code_kernel does (-0 -> +0);
// top-k is relu(score) under the activity mask.
template <int ARITH, bool TOPK>
__device__ __forceinline__ float frag_code_value(const FragCode& c, int m, int r, int j) {
  const long long idx = ((long long)m * c.batch_max + r) * c.n + j;
  float v;
  if constexpr (TOPK) {
    const uint32_t w = __ldg(c.pos + ((long long)m * c.n_chunks + (j >> 5)) * c.batch_max + r);
    v = ((w >> (31 - (j & 31))) & 1u) ? fmaxf(__ldg(c.scores + idx), 0.f) : 0.f;
  } else if constexpr (ARITH == kArithF16F8) {
    constexpr float kInv = 1.f / float(1 << kLoShift);
    v = __half2float(static_cast<const __half*>(c.hi)[idx]) + e5m2_to_float(c.x8[idx]) * kInv;
  } else {
    v = __bfloat162float(static_cast<const __nv_bfloat16*>(c.hi)[idx]) +
        __bfloat162float(static_cast<const __nv_bfloat16*>(c.lo)[idx]);
  }
  return v == 0.f ? 0.f : v;
}

// fmax[m][g][j] = max over the L rows of fragment g of c[m, r, j]; active[m][g][j] = 1 where the activity mask has
// c > 0 on some row of it. One block per (32-column chunk, fragment, model): lane j reads column 32 chunk + j, so every
// row is read coalesced over the features; warp w takes the rows w, w + 8, ... and the 8 warps meet in shared memory.
template <int ARITH, bool TOPK>
__global__ void __launch_bounds__(256) fragment_max_kernel(FragCode c, int L, int G, float* __restrict__ fmax,
                                                           uint8_t* __restrict__ active) {
  __shared__ float smax[8][32];
  __shared__ uint32_t sact[8][32];
  const int chunk = blockIdx.x, g = blockIdx.y, m = blockIdx.z;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int j = chunk * 32 + lane;
  const uint32_t* pw = c.pos + ((long long)m * c.n_chunks + chunk) * c.batch_max;
  float mx = 0.f;
  uint32_t any = 0u;
  for (int t = warp; t < L; t += 8) {
    const int r = g * L + t;
    any |= __ldg(pw + r);
    if (j < c.n) mx = fmaxf(mx, frag_code_value<ARITH, TOPK>(c, m, r, j));
  }
  smax[warp][lane] = mx;
  sact[warp][lane] = (any >> (31 - lane)) & 1u;
  __syncthreads();
  if (warp == 0 && j < c.n) {
    float v = smax[0][lane];
    uint32_t a = sact[0][lane];
#pragma unroll
    for (int w = 1; w < 8; ++w) {
      v = fmaxf(v, smax[w][lane]);
      a |= sact[w][lane];
    }
    const long long o = ((long long)m * G + g) * c.n + j;
    fmax[o] = v;
    active[o] = (uint8_t)a;
  }
}

// splitmix64 (Steele, Lea & Flood 2014): the priority of fragment `frag` for feature `feature` under `seed` is
// mix(mix(mix(seed) ^ feature) ^ frag) >> 1, a 63-bit key that depends on nothing but these three numbers
__device__ __forceinline__ uint64_t splitmix64(uint64_t z) {
  z += 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

// list order: (key descending, fragment ascending); an entry with fragment < 0 is empty and below every other
template <class K>
__device__ __forceinline__ bool frag_above(K k, long long f, K k2, long long f2) {
  return f2 < 0 || (f >= 0 && (k > k2 || (k == k2 && f < f2)));
}
template <class K>
__device__ __forceinline__ int frag_lowest(const K* key, const long long* frag, int cap) {
  int w = 0;
  for (int i = 1; i < cap; ++i)
    if (frag_above(key[w], frag[w], key[i], frag[i])) w = i;
  return w;
}

// One thread per (feature, model) walks the call's fragments in order and keeps two lists of `cap` entries that persist
// across calls: (fragment maximum, fragment) over all fragments, and (priority, fragment) over the active ones. A
// candidate replaces the list's lowest entry when it is above it, and then its L code values are copied into that
// entry's row of top_act / rnd_act. The lists are sets (sorted by the caller after the last call): the result depends
// on nothing but the fragments seen, with no atomics.
template <int ARITH, bool TOPK>
__global__ void __launch_bounds__(128) fragment_merge_kernel(FragCode c, int L, int G, long long frag0,
                                                             const float* __restrict__ fmax,
                                                             const uint8_t* __restrict__ active, int n_top, int n_random,
                                                             unsigned long long seed, float* top_val, long long* top_frag,
                                                             float* top_act, long long* rnd_key, long long* rnd_frag,
                                                             float* rnd_act) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x, m = blockIdx.y;
  if (j >= c.n) return;
  const long long list = (long long)m * c.n + j;
  float* tv = top_val + list * n_top;
  long long* tf = top_frag + list * n_top;
  long long* rk = rnd_key + list * n_random;
  long long* rf = rnd_frag + list * n_random;
  const uint64_t h_feat = splitmix64(splitmix64(seed) ^ (uint64_t)j);
  int tlow = n_top ? frag_lowest(tv, tf, n_top) : 0;
  int rlow = n_random ? frag_lowest(rk, rf, n_random) : 0;
  for (int g = 0; g < G; ++g) {
    const long long o = ((long long)m * G + g) * c.n + j, frag = frag0 + g;
    if (n_top) {
      const float v = __ldg(fmax + o);
      if (frag_above(v, frag, tv[tlow], tf[tlow])) {
        tv[tlow] = v;
        tf[tlow] = frag;
        if (top_act) {
          float* dst = top_act + (list * n_top + tlow) * L;
          for (int t = 0; t < L; ++t) dst[t] = frag_code_value<ARITH, TOPK>(c, m, g * L + t, j);
        }
        tlow = frag_lowest(tv, tf, n_top);
      }
    }
    if (n_random && __ldg(active + o)) {
      const long long k = (long long)(splitmix64(h_feat ^ (uint64_t)frag) >> 1);
      if (frag_above(k, frag, rk[rlow], rf[rlow])) {
        rk[rlow] = k;
        rf[rlow] = frag;
        if (rnd_act) {
          float* dst = rnd_act + (list * n_random + rlow) * L;
          for (int t = 0; t < L; ++t) dst[t] = frag_code_value<ARITH, TOPK>(c, m, g * L + t, j);
        }
        rlow = frag_lowest(rk, rf, n_random);
      }
    }
  }
}

constexpr int kFragMaxList = 64;   // largest n_top / n_random

static bool frag_len_ok(int L) { return L >= 32 && L <= 8192 && L % 32 == 0; }

// fragment maxima [M][B/L][n] fp32, activity flags [M][B/L][n] u8, open-segment flags [M][n] int32
static size_t frag_workspace(const sce_desc& d, int B, int L, size_t* off_active, size_t* off_open) {
  const size_t cells = (size_t)d.n_models * (B / L) * d.n;
  const size_t a = align_up(cells * sizeof(float), 1024), o = a + align_up(cells, 1024);
  if (off_active) *off_active = a;
  if (off_open) *off_open = o;
  return o + align_up((size_t)d.n_models * d.n * sizeof(int), 1024);
}

template <int ARITH, bool TOPK>
static void launch_fragments(const FragCode& c, int M, int L, int G, long long frag0, float* fmax, uint8_t* active,
                             int n_top, int n_random, unsigned long long seed, float* top_val, long long* top_frag,
                             float* top_act, long long* rnd_key, long long* rnd_frag, float* rnd_act, cudaStream_t st) {
  fragment_max_kernel<ARITH, TOPK><<<dim3(c.n_chunks, G, M), 256, 0, st>>>(c, L, G, fmax, active);
  fragment_merge_kernel<ARITH, TOPK><<<dim3((c.n + 127) / 128, M), 128, 0, st>>>(
      c, L, G, frag0, fmax, active, n_top, n_random, seed, top_val, top_frag, top_act, rnd_key, rnd_frag, rnd_act);
}

// ------------------------------------------------------------------------------------------------
// dictionary similarity (sce_similarity): cosine maxima and capacity over a list of dictionary pairs
// ------------------------------------------------------------------------------------------------
// maxima keys (EpiSimilarity) -> floats, in place; key 0 (no valid entry: an atom beyond rows[m]) becomes NaN
__global__ void key_to_float_kernel(uint32_t* __restrict__ v, long long n) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const uint32_t k = v[i];
    v[i] = (k & 0x80000000u) ? (k & 0x7FFFFFFFu) : ~k;
  }
}

// capacity_per_feature (standard_metrics.py:356-362) of every self-pair (m, m): diag(S^2) / rowsum(S^2), the row sum
// taken over the partials of EpiSimilarity in a fixed order. Atoms beyond rows[m] get NaN. A zero row gives 0 / 0 = NaN,
// as in the reference.
__global__ void capacity_kernel(const int* __restrict__ pairs, const int* __restrict__ rows, const float* __restrict__ sq_part,
                                const float* __restrict__ diag, int na, int parts, float* __restrict__ out) {
  const int q = blockIdx.y;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int m = pairs[2 * q];
  if (i >= na || m != pairs[2 * q + 1]) return;
  float* o = out + (long long)m * na + i;
  if (i >= rows[m]) {
    *o = __int_as_float(0x7FFFFFFF);
    return;
  }
  const float* s = sq_part + ((long long)q * na + i) * parts;
  float sum = 0.f;
  for (int t = 0; t < parts; ++t) sum += s[t];
  const float dg = diag[(long long)q * na + i];
  *o = dg * dg / sum;
}

struct SimOperand {   // one side of sce_similarity
  const float* w;
  int models, rows;
  int normalize;
  float floor;
};

// Workspace of one call: operand planes (4 B per element), the pair list and valid-row counts, the range flags of the
// f16f8 split, and (capacity) the sum-of-squares partials [P][na][2 tiles_n] and diagonal [P][na]. With base == nullptr
// only measures; `f8` only changes the order of the planes, not the bytes.
struct SimCarve {
  void *a_hi, *a_lo, *a_x8, *b_hi, *b_lo, *b_x8;
  int *pairs, *a_rows, *b_rows;
  uint32_t* flags;
  float *sq_part, *diag;
};
static size_t sim_carve(uint8_t* base, bool f8, long long ma, long long na, long long mb, long long nb, long long d,
                        long long n_pairs, bool capacity, SimCarve* out) {
  Carve c{base, 0};
  auto planes = [&](size_t count, void*& hi, void*& lo, void*& x8) {
    hi = c.take<__nv_bfloat16>(count);
    if (f8) {
      lo = c.take<uint8_t>(count);
      x8 = c.take<uint8_t>(count);
    } else {
      lo = c.take<__nv_bfloat16>(count);
      x8 = nullptr;
    }
  };
  SimCarve s;
  memset(&s, 0, sizeof(s));
  planes((size_t)(ma * na * d), s.a_hi, s.a_lo, s.a_x8);
  if (mb > 0) planes((size_t)(mb * nb * d), s.b_hi, s.b_lo, s.b_x8);
  s.pairs = c.take<int>((size_t)(2 * n_pairs));
  s.a_rows = c.take<int>((size_t)ma);
  s.b_rows = mb > 0 ? c.take<int>((size_t)mb) : s.a_rows;
  s.flags = c.take<uint32_t>(kFlagWords);
  if (capacity) {
    const long long tiles_n = (na + kBN - 1) / kBN;
    s.sq_part = c.take<float>((size_t)(n_pairs * na * 2 * tiles_n));
    s.diag = c.take<float>((size_t)(n_pairs * na));
  }
  if (out) *out = s;
  return align_up(c.off, 1024);
}
static size_t sim_workspace(long long ma, long long na, long long mb, long long nb, long long d, long long n_pairs, bool capacity) {
  const size_t a = sim_carve(nullptr, false, ma, na, mb, nb, d, n_pairs, capacity, nullptr);
  const size_t b = sim_carve(nullptr, true, ma, na, mb, nb, d, n_pairs, capacity, nullptr);
  return a > b ? a : b;
}

// fp32 operand -> planes: normalised rows (dict_rows_kernel<MODE_PREPARE>, LearnedDict.get_learned_dict) or the matrix
// as given (split_rows_kernel; f16f8: sets the range flags when a value does not fit fp16)
template <int AR>
static int sim_planes(const SimOperand& o, int d, void* hi, void* lo, void* x8, uint32_t* flags, cudaStream_t st) {
  const long long rows = (long long)o.models * o.rows;
  if (o.normalize)
    return launch_dict_rows_t<MODE_PREPARE, AR>(const_cast<float*>(o.w), nullptr, nullptr, nullptr, hi, lo, x8, nullptr, rows, d,
                                                 1, o.floor, AdamHyper{}, nullptr, nullptr, st);
  launch_split_rows<AR>(o.w, hi, lo, x8, rows * d / 4, AR == kArithF16F8 ? flags : nullptr, st);
  CUDA_TRY(cudaGetLastError());
  return SCE_OK;
}

template <int AR>
static int run_similarity_t(const SimOperand& A, const SimOperand& B, bool b_is_a, int d, int n_pairs, const SimCarve& w,
                            float* row_max, float* col_max, float* capacity, int device, int sms, cudaStream_t st) {
  int rc = sim_planes<AR>(A, d, w.a_hi, w.a_lo, w.a_x8, w.flags, st);
  if (rc) return rc;
  if (!b_is_a) {
    rc = sim_planes<AR>(B, d, w.b_hi, w.b_lo, w.b_x8, w.flags, st);
    if (rc) return rc;
  }
  const void* const b_hi = b_is_a ? w.a_hi : w.b_hi;
  const void* const b_lo = b_is_a ? w.a_lo : w.b_lo;
  const void* const b_x8 = b_is_a ? w.a_x8 : w.b_x8;
  GemmParams<EpiSimilarity::Params> gp;
  memset(&gp, 0, sizeof(gp));
  // both operands are dictionary rows, K-major over d: the encode GEMM's B-operand geometry on both sides
  bool ok = operand_maps(AR, &gp.a_hi[0], &gp.a_lo[0], &gp.a_x8[0], w.a_hi, w.a_lo, w.a_x8, A.models, A.rows, d,
                         (uint64_t)A.rows * d, kBM, gemm_bk(AR));
  ok = ok && operand_maps(AR, &gp.b_hi[0], &gp.b_lo[0], &gp.b_x8[0], b_hi, b_lo, b_x8, B.models, B.rows, d,
                          (uint64_t)B.rows * d, kBN, gemm_bk(AR));
  if (!ok) return fail(SCE_ERR_CUDA, "cuTensorMapEncodeTiled failed (similarity: na=%d, nb=%d, d=%d)", A.rows, B.rows, d);
  gp.a_batched[0] = gp.b_batched[0] = 1;
  gp.nsets = 1;
  gp.k_total = d;
  gp.passes = 3;
  gp.n_models = n_pairs;
  gp.m_total = A.rows;
  gp.n_total = B.rows;
  gp.tiles_m = (A.rows + kBM - 1) / kBM;
  gp.tiles_n = (B.rows + kBN - 1) / kBN;
  gp.epi.pairs = w.pairs;
  gp.epi.a_rows = w.a_rows;
  gp.epi.b_rows = w.b_rows;
  gp.epi.row_max = reinterpret_cast<uint32_t*>(row_max);
  gp.epi.col_max = reinterpret_cast<uint32_t*>(col_max);
  gp.epi.sq_part = capacity ? w.sq_part : nullptr;
  gp.epi.diag = w.diag;
  gp.epi.tiles_n = gp.tiles_n;
  if (row_max) CUDA_TRY(cudaMemsetAsync(row_max, 0, (size_t)n_pairs * A.rows * sizeof(float), st));
  if (col_max) CUDA_TRY(cudaMemsetAsync(col_max, 0, (size_t)n_pairs * B.rows * sizeof(float), st));
  CUDA_TRY((launch_gemm<EpiSimilarity, false, false, false, AR, AR == kArithF16F8>(gp, device, sms, st)));
  auto to_float = [&](float* v, long long n) -> int {
    const int blocks = (int)((n + 255) / 256 < 1024 ? (n + 255) / 256 : 1024);
    key_to_float_kernel<<<blocks, 256, 0, st>>>(reinterpret_cast<uint32_t*>(v), n);
    CUDA_TRY(cudaGetLastError());
    return SCE_OK;
  };
  if (row_max && (rc = to_float(row_max, (long long)n_pairs * A.rows))) return rc;
  if (col_max && (rc = to_float(col_max, (long long)n_pairs * B.rows))) return rc;
  if (capacity) {
    capacity_kernel<<<dim3((A.rows + 255) / 256, n_pairs), 256, 0, st>>>(w.pairs, w.a_rows, w.sq_part, w.diag, A.rows,
                                                                       2 * gp.tiles_n, capacity);
    CUDA_TRY(cudaGetLastError());
  }
  return SCE_OK;
}

// ------------------------------------------------------------------------------------------------
// C ABI
// ------------------------------------------------------------------------------------------------
extern "C" {

int sce_version(void) { return SCE_VERSION; }
const char* sce_last_error(void) { return g_err; }

size_t sce_workspace_bytes(const sce_desc* desc) {
  if (validate(desc)) return 0;
  return carve(nullptr, *desc, nullptr);
}

int sce_plan_create(const sce_desc* desc, const sce_buffers* buffers, sce_plan** out_plan) {
  if (!out_plan) return fail(SCE_ERR_INVALID, "out_plan is NULL");
  *out_plan = nullptr;
  int rc = validate(desc);
  if (rc) return rc;
  if (!buffers) return fail(SCE_ERR_INVALID, "buffers is NULL");
  const sce_buffers& b = *buffers;
  if (!b.encoder || !b.encoder_m || !b.encoder_v) return fail(SCE_ERR_INVALID, "encoder / encoder_m / encoder_v are required");
  if (desc->variant == SCE_UNTIED && (!b.decoder || !b.decoder_m || !b.decoder_v))
    return fail(SCE_ERR_INVALID, "untied variant needs decoder / decoder_m / decoder_v");
  if (desc->variant != SCE_TOPK && (!b.encoder_bias || !b.bias_m || !b.bias_v))
    return fail(SCE_ERR_INVALID, "encoder_bias / bias_m / bias_v are required for SAE variants");
  if (desc->variant == SCE_TOPK && !b.sparsity) return fail(SCE_ERR_INVALID, "top-k variant needs the sparsity buffer");
  rc = check_workspace(b.workspace, b.workspace_bytes, carve(nullptr, *desc, nullptr), "");
  if (rc) return rc;
  int dev = 0, sms = 0;
  rc = query_device(&dev, &sms);
  if (rc) return rc;
  sce_plan* p = new (std::nothrow) sce_plan;
  if (!p) return fail(SCE_ERR_INVALID, "out of host memory");
  memset(p, 0, sizeof(*p));
  p->d = *desc;
  p->b = b;
  p->sms = sms;
  p->device = dev;
  p->xm = desc->x_per_model ? desc->n_models : 1;
  p->arith = resolve_arith(*desc);
  // The truncation bias of a single accumulation chain grows with the reduction length; n > 4096 splits the decode
  // GEMM's cross terms into their own accumulator (config 5's width, n = 32768, needs it for the 1e-4 bar; the parity
  // tests cover both sides). Splitting doubles the decode GEMM's accumulator registers, so it is used where needed.
  p->split_decode = tune_flag("SCE_TUNE_SPLIT_DECODE", desc->n > 4096 ? 1 : 0);
  p->dcode_passes = desc->bwd_passes;
  p->dw_passes = desc->bwd_passes;
  if (const char* v = getenv("SCE_TUNE_DCODE_PASSES")) p->dcode_passes = atoi(v) == 1 ? 1 : 3;
  if (const char* v = getenv("SCE_TUNE_DW_PASSES")) p->dw_passes = atoi(v) == 1 ? 1 : 3;
  p->dw_native = native_dw_layout(*desc) && p->dw_passes >= 3;
  p->use_graph = tune_flag("SCE_GRAPH", launch_bound(*desc) ? 1 : 0);
  {
    // k-sparse decode / dcode of the top-k variant: lists known (topk_k_max), bulk-copy alignment of the dictionary
    // half rows (16 bytes in every plane), shared memory of the gather kernel
    const size_t kmax = topk_kmax(*desc);
    p->tk_slices = kmax ? topk_slices(*desc, kmax) : 0;
    if (const char* v = getenv("SCE_TOPK_SLICES")) {
      const int sl = atoi(v);
      if (kmax && (sl == 2 || sl == 4 || sl == 8) && desc->d % (4 * sl) == 0 && desc->d / sl <= 512 &&
          topk_sparse_smem(*desc, kmax, sl) <= 112 * 1024)
        p->tk_slices = sl;
    }
    // Worth it where the dictionary is large against k: the dense decode + dcode GEMMs cost ~ n per row, the gather
    // kernel ~ k (it is bound by the latency chain of a block, not by bytes): the gather path is used where n >= 96 k.
    // SCE_TOPK_SPARSE = 1 / 0 forces it on / off.
    const int heuristic = (long long)desc->n >= 96ll * (long long)(kmax ? kmax : 1);
    p->topk_sparse = desc->variant == SCE_TOPK && kmax > 0 && p->tk_slices > 0 && tune_flag("SCE_TOPK_SPARSE", heuristic);
    // selection from the per-chunk maxima the scores epilogue writes; 0 = read every row twice
    p->topk_cmax = desc->variant == SCE_TOPK && tune_flag("SCE_TOPK_CMAX", 1);
  }
  p->maps = new std::map<int, BatchMaps*>();
  carve(p, *desc, static_cast<uint8_t*>(b.workspace));
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
  const long long rows = (long long)d.n_models * d.n;
  if (d.variant == SCE_TOPK && p->tk_kmax) {
    // the top-k selection keeps the code planes (and, in k-sparse plans, the code-gradient planes) all-zero except for
    // the entries its lists record: start them zeroed, with empty lists
    const size_t el = (size_t)d.n_models * d.batch_max * d.n;
    const bool f8 = p->arith == kArithF16F8;
    CUDA_TRY(cudaMemsetAsync(p->c_hi, 0, el * 2, st));
    CUDA_TRY(cudaMemsetAsync(p->c_lo, 0, el * (f8 ? 1 : 2), st));
    if (f8) CUDA_TRY(cudaMemsetAsync(p->c_x8, 0, el, st));
    CUDA_TRY(cudaMemsetAsync(p->dz_hi, 0, el * 4, st));   // (the code-gradient planes are one contiguous block, 4 B / element)
    CUDA_TRY(cudaMemsetAsync(p->act_pos, 0, (size_t)d.n_models * ((d.n + 31) / 32) * d.batch_max * sizeof(uint32_t), st));
    CUDA_TRY(cudaMemsetAsync(p->tk_cnt, 0, (size_t)d.n_models * d.batch_max * sizeof(int), st));
    // k classes for the gather kernel: rows of shared memory in {8, 16, 32, 64, ...} capped at the list capacity
    std::vector<long long> ks(d.n_models);
    CUDA_TRY(cudaMemcpyAsync(ks.data(), p->b.sparsity, ks.size() * sizeof(long long), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    const int caps[4] = {16, 32, 64, p->tk_kmax};
    std::vector<int> order;
    p->tk_groups = 0;
    p->tk_group_off[0] = 0;
    int lo = 0;
    for (int g = 0; g < 4; ++g) {
      const int cap = caps[g] < p->tk_kmax ? caps[g] : p->tk_kmax;
      if (g > 0 && cap <= lo) continue;
      for (int m = 0; m < d.n_models; ++m) {
        const long long k = ks[m] < 1 ? 1 : (ks[m] > p->tk_kmax ? (long long)p->tk_kmax : ks[m]);   // (kernels clip k the same way)
        if (k > lo && k <= cap) order.push_back(m);
      }
      p->tk_group_krows[p->tk_groups] = cap;
      p->tk_group_off[++p->tk_groups] = (int)order.size();
      lo = cap;
      if (cap == p->tk_kmax) break;
    }
    if ((int)order.size() != d.n_models) return fail(SCE_ERR_INVALID, "top-k classes: %d of %d models placed", (int)order.size(), d.n_models);
    CUDA_TRY(cudaMemcpyAsync(p->tk_models, order.data(), order.size() * sizeof(int), cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaStreamSynchronize(st));   // (`order` is a local)
  }
  if (d.centering) {
    if (!p->b.center_trans || !p->b.center_rot || !p->b.center_scale)
      return fail(SCE_ERR_INVALID, "centering needs the center_trans / center_rot / center_scale buffers");
    const long long n4 = (long long)d.n_models * d.d * d.d / 4;
    if (p->arith == kArithF16F8)
      launch_split_rows<kArithF16F8>(p->b.center_rot, p->rot_hi, p->rot_lo, p->rot_x8, n4, nullptr, st);
    else
      launch_split_rows<kArithBf16x3>(p->b.center_rot, p->rot_hi, p->rot_lo, nullptr, n4, nullptr, st);
    CUDA_TRY(cudaGetLastError());
  }
  AdamHyper h = hyper_for(p, 1);
  int rc;
  if (d.variant == SCE_UNTIED) {
    rc = launch_dict_rows<MODE_PREPARE>(p, 0, p->b.encoder, nullptr, nullptr, nullptr, nullptr, rows, d.d, 0, 0.f, h, st);
    if (rc) return rc;
    rc = launch_dict_rows<MODE_PREPARE>(p, 1, p->b.decoder, nullptr, nullptr, nullptr, nullptr, rows, d.d, 1, d.norm_floor, h, st);
  } else {
    rc = launch_dict_rows<MODE_PREPARE>(p, 0, p->b.encoder, nullptr, nullptr, nullptr, nullptr, rows, d.d, 1, d.norm_floor, h, st);
  }
  if (rc) return rc;
  int launches = 0;
  return transpose_dict(p, st, launches);
}

int sce_forward(sce_plan* p, const float* x, int B, float* x_hat, float* out_losses, float* out_nnz, void* stream) {
  if (!p) return fail(SCE_ERR_INVALID, "plan is NULL");
  return run_pipeline(p, x, B, x_hat, false, out_losses, out_nnz, static_cast<cudaStream_t>(stream));
}

// models' worth of rows in the caller's batch: 1 when it is shared ([B,d]; also with centering = 1), else M
static int input_models(const sce_plan* p) { return p->d.centering == 1 ? 1 : p->xm; }

// every launch of one optimisation step, in order, on `st` (also what gets captured into a CUDA graph)
static int step_launches(sce_plan* p, const float* x, int B, float* out_losses, float* out_nnz, long long t,
                         cudaStream_t st) {
  int rc = run_pipeline(p, x, B, nullptr, true, out_losses, out_nnz, st);
  if (rc) return rc;
  const sce_desc& d = p->d;
  const long long rows = (long long)d.n_models * d.n;
  const AdamHyper h = hyper_for(p, t);
  int launches = p->last_launches;
  if (d.variant == SCE_UNTIED) {
    rc = launch_dict_rows<MODE_ADAM>(p, 0, p->b.encoder, p->dw_enc, p->b.encoder_m, p->b.encoder_v, nullptr, rows, d.d, 0,
                                     0.f, h, st);
    if (rc) return rc;
    rc = launch_dict_rows<MODE_ADAM>(p, 1, p->b.decoder, p->dw_dec, p->b.decoder_m, p->b.decoder_v, nullptr, rows, d.d, 1,
                                     d.norm_floor, h, st);
    if (rc) return rc;
    launches += 2;
  } else {
    rc = launch_dict_rows<MODE_ADAM>(p, 0, p->b.encoder, p->dw_enc, p->b.encoder_m, p->b.encoder_v, nullptr, rows, d.d, 1,
                                     d.norm_floor, h, st);
    if (rc) return rc;
    ++launches;
  }
  rc = transpose_dict(p, st, launches);
  if (rc) return rc;
  if (p->b.encoder_bias) {
    const long long tot = (long long)d.n_models * d.n;
    const int n_part = ((B + kBM - 1) / kBM) * 4;
    bias_kernel<MODE_ADAM><<<(unsigned)((tot + 255) / 256), 256, 0, st>>>(
        p->b.encoder_bias, p->b.bias_m, p->b.bias_v, p->db_part, n_part, d.n, d.n_models, p->b.bias_decay, p->bnorm,
        nullptr, h, grad_out_scale(p, B), p->res_flags);
    CUDA_TRY(cudaGetLastError());
    ++launches;
  }
  prof_mark(p, SCE_PHASE_COUNT, st);
  p->last_launches = launches;
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
  return p->use_graph != 0;
}

int sce_step(sce_plan* p, const float* x, int B, float* out_losses, float* out_nnz, void* stream) {
  if (!p) return fail(SCE_ERR_INVALID, "plan is NULL");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (int rc = check_rows(p, B, "")) return rc;
  if (!x) return fail(SCE_ERR_INVALID, "x is NULL");
  int rc;
  if (!graph_eligible(p)) {
    rc = step_launches(p, x, B, out_losses, out_nnz, p->step + 1, st);
  } else {
    BatchMaps* maps = nullptr;
    rc = build_maps(p, B, &maps);
    if (rc) return rc;
    const size_t bytes = (size_t)input_models(p) * B * p->d.d * sizeof(float);
    if (x != p->x_stage) CUDA_TRY(cudaMemcpyAsync(p->x_stage, x, bytes, cudaMemcpyDeviceToDevice, st));
    // the captured kernels write the plan's own staging outputs (stable addresses: callers may pass fresh tensors
    // every step, as the reference returns them); the results are copied out below
    float* const cap_losses = p->loss_stage;
    float* const cap_nnz = p->nnz_stage;
    if (maps->graph) {
      CUDA_TRY(cudaGraphLaunch(maps->graph, st));
      p->last_launches = maps->graph_launches;
      rc = SCE_OK;
    } else if (maps->eager_steps == 0) {
      maps->eager_steps = 1;
      rc = step_launches(p, p->x_stage, B, cap_losses, cap_nnz, 1, st);
    } else {
      // capture on a private stream (the caller's may be the legacy default stream, which cannot be captured);
      // capturing records the launches without running them, the instantiated graph is launched on `st`
      cudaGraph_t g = nullptr;
      if (!p->cap_stream) CUDA_TRY(cudaStreamCreateWithFlags(&p->cap_stream, cudaStreamNonBlocking));
      CUDA_TRY(cudaStreamBeginCapture(p->cap_stream, cudaStreamCaptureModeThreadLocal));
      rc = step_launches(p, p->x_stage, B, cap_losses, cap_nnz, 1, p->cap_stream);
      cudaError_t ce = cudaStreamEndCapture(p->cap_stream, &g);
      if (rc == SCE_OK && ce == cudaSuccess && g) {
        cudaGraphExec_t ge = nullptr;
        ce = cudaGraphInstantiate(&ge, g, 0);
        cudaGraphDestroy(g);
        if (ce != cudaSuccess) return fail(SCE_ERR_CUDA, "cudaGraphInstantiate failed: %s", cudaGetErrorString(ce));
        maps->graph = ge;
        maps->graph_launches = p->last_launches;
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
  p->step += 1;
  if (p->prof_on && p->prof_steps < kProfMaxSteps) p->prof_steps += 1;
  return SCE_OK;
}

int sce_grads(sce_plan* p, const float* x, int B, float* d_encoder, float* d_bias, float* d_decoder,
              float* out_losses, float* out_nnz, void* stream) {
  if (!p) return fail(SCE_ERR_INVALID, "plan is NULL");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  int rc = run_pipeline(p, x, B, nullptr, true, out_losses, out_nnz, st);
  if (rc) return rc;
  const sce_desc& d = p->d;
  const long long rows = (long long)d.n_models * d.n;
  const AdamHyper h = hyper_for(p, 1);
  if (d.variant == SCE_UNTIED) {
    if (d_encoder) {
      rc = launch_dict_rows<MODE_GRAD>(p, 0, p->b.encoder, p->dw_enc, nullptr, nullptr, d_encoder, rows, d.d, 0, 0.f, h, st);
      if (rc) return rc;
    }
    if (d_decoder) {
      rc = launch_dict_rows<MODE_GRAD>(p, 1, p->b.decoder, p->dw_dec, nullptr, nullptr, d_decoder, rows, d.d, 1, d.norm_floor,
                                       h, st);
      if (rc) return rc;
    }
  } else if (d_encoder) {
    rc = launch_dict_rows<MODE_GRAD>(p, 0, p->b.encoder, p->dw_enc, nullptr, nullptr, d_encoder, rows, d.d, 1, d.norm_floor, h,
                                     st);
    if (rc) return rc;
  }
  if (p->b.encoder_bias && d_bias) {
    const long long tot = (long long)d.n_models * d.n;
    const int n_part = ((B + kBM - 1) / kBM) * 4;
    bias_kernel<MODE_GRAD><<<(unsigned)((tot + 255) / 256), 256, 0, st>>>(
        p->b.encoder_bias, nullptr, nullptr, p->db_part, n_part, d.n, d.n_models, p->b.bias_decay, p->bnorm, d_bias, h,
        grad_out_scale(p, B), nullptr);
    CUDA_TRY(cudaGetLastError());
  }
  return SCE_OK;
}

int sce_step_host(sce_plan* p, const float* x_host, int B, float* out_losses_host, float* out_nnz_host,
                  void* stream) {
  if (!p) return fail(SCE_ERR_INVALID, "plan is NULL");
  if (!x_host) return fail(SCE_ERR_INVALID, "x_host is NULL");
  if (int rc = check_rows(p, B, "")) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const size_t bytes = (size_t)input_models(p) * B * p->d.d * sizeof(float);
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

int sce_read_code(sce_plan* p, int B, float* out_code, void* stream) {
  if (!p || !out_code) return fail(SCE_ERR_INVALID, "plan / out_code is NULL");
  if (int rc = check_rows(p, B, "")) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const long long per = (long long)B * p->d.n;
  if (p->code_batch_major) {
    const long long total = (long long)p->d.n_models * per;
    join_code_batch_major_kernel<<<(unsigned)((total + 255) / 256 < 4096 ? (total + 255) / 256 : 4096), 256, 0, st>>>(
        reinterpret_cast<const __half*>(p->c_hi), p->ct_x8, out_code, B, p->d.n, p->d.batch_max, p->bpad, total);
    CUDA_TRY(cudaGetLastError());
    return SCE_OK;
  }
  for (int m = 0; m < p->d.n_models; ++m) {
    const long long src = (long long)m * p->d.batch_max * p->d.n;
    if (p->arith == kArithF16F8)
      join_code_kernel<kArithF16F8><<<1024, 256, 0, st>>>(p->c_hi + src, nullptr, p->c_x8 + src, out_code + (long long)m * per, per / 2);
    else
      join_code_kernel<kArithBf16x3><<<1024, 256, 0, st>>>(p->c_hi + src, p->c_lo + src, nullptr, out_code + (long long)m * per, per / 2);
  }
  CUDA_TRY(cudaGetLastError());
  return SCE_OK;
}

int sce_gather_rows(const void* chunk, int chunk_is_half, long long n_rows, int d, const long long* idx, int B,
                    const float* sub, float* out, void* stream) {
  if (!chunk || !out || B < 1 || d < 4 || d % 4) return fail(SCE_ERR_INVALID, "bad arguments to sce_gather_rows");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int blocks = (B + 7) / 8;
  if (chunk_is_half)
    gather_rows_kernel<__half><<<blocks, 256, 0, st>>>(static_cast<const __half*>(chunk), n_rows, d, idx, B, sub, out);
  else
    gather_rows_kernel<float><<<blocks, 256, 0, st>>>(static_cast<const float*>(chunk), n_rows, d, idx, B, sub, out);
  CUDA_TRY(cudaGetLastError());
  return SCE_OK;
}

int sce_last_launch_count(const sce_plan* plan) { return plan ? plan->last_launches : 0; }
int sce_input_absmax(sce_plan* plan, float* out_host, void* stream) {
  if (!plan || !out_host) return fail(SCE_ERR_INVALID, "plan / out_host is NULL");
  *out_host = 0.f;
  if (plan->arith != kArithF16F8) return SCE_OK;
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
    if (plan->arith == kArithF16F8) memcpy(absmax_out, &words[kAbsmaxWord], sizeof(float));
  }
  return SCE_OK;
}
int sce_clear_health(sce_plan* plan, void* stream) {
  if (!plan) return fail(SCE_ERR_INVALID, "plan is NULL");
  CUDA_TRY(cudaMemsetAsync(plan->res_flags + kBadWord, 0, sizeof(uint32_t), static_cast<cudaStream_t>(stream)));
  return SCE_OK;
}

int sce_active_counts(sce_plan* plan, int B, int* counts, void* stream) {
  if (!plan || !counts) return fail(SCE_ERR_INVALID, "plan / counts is NULL");
  if (int rc = check_rows(plan, B, "")) return rc;
  const int n_chunks = (plan->d.n + 31) / 32;
  active_count_kernel<<<dim3(n_chunks, plan->d.n_models), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      plan->act_pos, n_chunks, plan->d.batch_max, B, plan->d.n, counts);
  CUDA_TRY(cudaGetLastError());
  return SCE_OK;
}

size_t sce_forward_stats_workspace_bytes(const sce_desc* desc, int B) {
  if (validate(desc) || B < 1 || B > desc->batch_max) return 0;
  return stats_workspace(*desc, B);
}

int sce_forward_stats(sce_plan* p, const float* x, int B, int seg, int seg_phase, float* x_hat, float* out_losses,
                      float* out_nnz, double* moment_sums, int* seg_counts, int* seg_open, void* workspace,
                      size_t workspace_bytes, void* stream) {
  if (!p) return fail(SCE_ERR_INVALID, "forward_stats: plan is NULL");
  if (int rc = check_rows(p, B, "forward_stats: ")) return rc;
  if (!x) return fail(SCE_ERR_INVALID, "forward_stats: x is NULL");
  if (seg < 1) return fail(SCE_ERR_INVALID, "forward_stats: seg = %d must be >= 1", seg);
  if (seg_phase < 0 || seg_phase >= seg)
    return fail(SCE_ERR_INVALID, "forward_stats: seg_phase = %d outside [0, seg = %d)", seg_phase, seg);
  if (!out_losses || !out_nnz || !moment_sums || !seg_counts)
    return fail(SCE_ERR_INVALID, "forward_stats: out_losses, out_nnz, moment_sums and seg_counts are required");
  if (seg > 1 && !seg_open) return fail(SCE_ERR_INVALID, "forward_stats: seg > 1 needs the seg_open flags");
  if (int rc = check_workspace(workspace, workspace_bytes, stats_workspace(p->d, B), "forward_stats: ")) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const sce_desc& d = p->d;
  const bool topk = d.variant == SCE_TOPK;
  float* part = static_cast<float*>(workspace);
  int rc = run_pipeline(p, x, B, x_hat, false, out_losses, out_nnz, st, topk ? nullptr : part);
  if (rc) return rc;
  const int n_chunks = (d.n + 31) / 32, row_blocks = (B + 31) / 32;
  if (topk) {
    topk_moment_kernel<<<dim3(n_chunks, (row_blocks + 7) / 8, d.n_models), 256, 0, st>>>(p->scores, p->act_pos, n_chunks,
                                                                                        d.batch_max, B, d.n, row_blocks, part);
    CUDA_TRY(cudaGetLastError());
  }
  moment_reduce_kernel<<<dim3((d.n + 255) / 256, d.n_models), 256, 0, st>>>(part, row_blocks, d.n, moment_sums);
  CUDA_TRY(cudaGetLastError());
  if (seg == 1)
    active_count_kernel<<<dim3(n_chunks, d.n_models), 256, 0, st>>>(p->act_pos, n_chunks, d.batch_max, B, d.n, seg_counts);
  else
    segment_count_kernel<<<dim3(n_chunks, d.n_models), 256, 0, st>>>(p->act_pos, n_chunks, d.batch_max, B, d.n, seg,
                                                                     seg_phase, seg_counts, seg_open);
  CUDA_TRY(cudaGetLastError());
  return SCE_OK;
}

size_t sce_fragments_workspace_bytes(const sce_desc* desc, int B, int L) {
  if (validate(desc) || B < 1 || B > desc->batch_max || !frag_len_ok(L) || B % L) return 0;
  return frag_workspace(*desc, B, L, nullptr, nullptr);
}

int sce_forward_fragments(sce_plan* p, const float* x, int B, int L, long long frag0, int n_top, int n_random,
                          unsigned long long seed, float* top_val, long long* top_frag, float* top_act,
                          long long* rnd_key, long long* rnd_frag, float* rnd_act, int* n_active, void* workspace,
                          size_t workspace_bytes, void* stream) {
  if (!p) return fail(SCE_ERR_INVALID, "forward_fragments: plan is NULL");
  if (int rc = check_rows(p, B, "forward_fragments: ")) return rc;
  if (!x) return fail(SCE_ERR_INVALID, "forward_fragments: x is NULL");
  if (!frag_len_ok(L)) return fail(SCE_ERR_INVALID, "forward_fragments: L = %d must be a multiple of 32 in [32, 8192]", L);
  if (B % L) return fail(SCE_ERR_INVALID, "forward_fragments: B = %d is not a multiple of L = %d", B, L);
  if (frag0 < 0) return fail(SCE_ERR_INVALID, "forward_fragments: frag0 = %lld must be >= 0", frag0);
  if (n_top < 0 || n_top > kFragMaxList || n_random < 0 || n_random > kFragMaxList || n_top + n_random == 0)
    return fail(SCE_ERR_INVALID, "forward_fragments: n_top = %d and n_random = %d must lie in [0, %d], not both 0", n_top,
                n_random, kFragMaxList);
  if (n_top && (!top_val || !top_frag)) return fail(SCE_ERR_INVALID, "forward_fragments: n_top > 0 needs top_val and top_frag");
  if (n_random && (!rnd_key || !rnd_frag))
    return fail(SCE_ERR_INVALID, "forward_fragments: n_random > 0 needs rnd_key and rnd_frag");
  if (!n_active) return fail(SCE_ERR_INVALID, "forward_fragments: n_active is required");
  size_t off_active, off_open;
  const size_t need = frag_workspace(p->d, B, L, &off_active, &off_open);
  if (int rc = check_workspace(workspace, workspace_bytes, need, "forward_fragments: ")) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const sce_desc& d = p->d;
  int rc = run_pipeline(p, x, B, nullptr, false, nullptr, nullptr, st);
  if (rc) return rc;
  uint8_t* ws = static_cast<uint8_t*>(workspace);
  float* fmax = reinterpret_cast<float*>(ws);
  uint8_t* active = ws + off_active;
  int* open = reinterpret_cast<int*>(ws + off_open);
  const int n_chunks = (d.n + 31) / 32, G = B / L;
  const FragCode c{p->c_hi, p->c_lo, p->c_x8, p->scores, p->act_pos, n_chunks, d.batch_max, d.n};
  if (d.variant == SCE_TOPK)
    launch_fragments<kArithBf16x3, true>(c, d.n_models, L, G, frag0, fmax, active, n_top, n_random, seed, top_val,
                                         top_frag, top_act, rnd_key, rnd_frag, rnd_act, st);
  else if (p->arith == kArithF16F8)
    launch_fragments<kArithF16F8, false>(c, d.n_models, L, G, frag0, fmax, active, n_top, n_random, seed, top_val,
                                         top_frag, top_act, rnd_key, rnd_frag, rnd_act, st);
  else
    launch_fragments<kArithBf16x3, false>(c, d.n_models, L, G, frag0, fmax, active, n_top, n_random, seed, top_val,
                                          top_frag, top_act, rnd_key, rnd_frag, rnd_act, st);
  CUDA_TRY(cudaGetLastError());
  // active fragments: segments of L rows, cut at fragment boundaries (phase 0, no segment stays open)
  CUDA_TRY(cudaMemsetAsync(open, 0, (size_t)d.n_models * d.n * sizeof(int), st));
  segment_count_kernel<<<dim3(n_chunks, d.n_models), 256, 0, st>>>(p->act_pos, n_chunks, d.batch_max, B, d.n, L, 0,
                                                                   n_active, open);
  CUDA_TRY(cudaGetLastError());
  return SCE_OK;
}

int sce_plan_arith(const sce_plan* plan) {
  return !plan ? 0 : plan->arith == kArithF16F8 ? SCE_ARITH_F16F8 : SCE_ARITH_BF16X3;
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

size_t sce_similarity_workspace_bytes(int ma, int na, int mb, int nb, int d, int n_pairs, int want_capacity) {
  if (ma < 1 || na < 1 || mb < 0 || (mb > 0 && nb < 1) || d < 8 || n_pairs < 1) return 0;
  return sim_workspace(ma, na, mb, mb > 0 ? nb : 0, d, n_pairs, want_capacity != 0);
}

int sce_similarity(const float* a, int ma, int na, const int* a_rows, float a_norm_floor, int a_normalize,
                   const float* b, int mb, int nb, const int* b_rows, float b_norm_floor, int b_normalize,
                   int d, const int* pairs, int n_pairs, int arith, float* row_max, float* col_max, float* capacity,
                   void* workspace, size_t workspace_bytes, void* stream) {
  // ---- arguments (all checked before any CUDA call)
  if (!a) return fail(SCE_ERR_INVALID, "similarity: a is NULL");
  if (ma < 1 || na < 1) return fail(SCE_ERR_INVALID, "similarity: ma (%d) and na (%d) must be >= 1", ma, na);
  if (d < 8 || d % 8) return fail(SCE_ERR_INVALID, "similarity: d (%d) must be a positive multiple of 8", d);
  if (d > 8192) return fail(SCE_ERR_INVALID, "similarity: d = %d > 8192 is not supported by the row kernels", d);
  if ((a_normalize != 0 && a_normalize != 1) || (b && b_normalize != 0 && b_normalize != 1))
    return fail(SCE_ERR_INVALID, "similarity: a_normalize / b_normalize must be 0 or 1");
  const bool b_is_a = b == nullptr;
  if (!b_is_a && (mb < 1 || nb < 1)) return fail(SCE_ERR_INVALID, "similarity: mb (%d) and nb (%d) must be >= 1", mb, nb);
  const int Mb = b_is_a ? ma : mb, Nb = b_is_a ? na : nb;
  if (!pairs || n_pairs < 1) return fail(SCE_ERR_INVALID, "similarity: need at least one pair (pairs NULL or n_pairs = %d)", n_pairs);
  if (arith < SCE_ARITH_AUTO || arith > SCE_ARITH_F16F8) return fail(SCE_ERR_INVALID, "similarity: unknown arith %d", arith);
  if (arith == SCE_ARITH_F16F8 && d % 16)
    return fail(SCE_ERR_INVALID, "similarity: arith = F16F8 needs d (%d) to be a multiple of 16", d);
  if (!row_max && !col_max && !capacity) return fail(SCE_ERR_INVALID, "similarity: no output requested");
  if (capacity && !b_is_a) return fail(SCE_ERR_INVALID, "similarity: capacity is defined for self-pairs of one stack (b must be NULL)");
  const long long tiles = (long long)n_pairs * ((na + kBM - 1) / kBM) * ((Nb + kBN - 1) / kBN);
  if (tiles > 0x7FFFFFFFll) return fail(SCE_ERR_INVALID, "similarity: %lld tiles exceed the 32-bit tile index", tiles);
  std::vector<int> pv(pairs, pairs + 2 * (size_t)n_pairs);
  for (int q = 0; q < n_pairs; ++q)
    if (pv[2 * q] < 0 || pv[2 * q] >= ma || pv[2 * q + 1] < 0 || pv[2 * q + 1] >= Mb)
      return fail(SCE_ERR_INVALID, "similarity: pair %d = (%d, %d) outside [0, %d) x [0, %d)", q, pv[2 * q], pv[2 * q + 1], ma, Mb);
  std::vector<int> rows(ma + (b_is_a ? 0 : mb));
  for (int m = 0; m < ma; ++m) rows[m] = a_rows ? a_rows[m] : na;
  for (int m = 0; !b_is_a && m < mb; ++m) rows[ma + m] = b_rows ? b_rows[m] : nb;
  for (int m = 0; m < (int)rows.size(); ++m) {
    const int n = m < ma ? na : nb;
    if (rows[m] < 1 || rows[m] > n)
      return fail(SCE_ERR_INVALID, "similarity: rows[%d] of %s = %d outside [1, %d]", m < ma ? m : m - ma, m < ma ? "a" : "b", rows[m], n);
  }
  const size_t need = sim_workspace(ma, na, b_is_a ? 0 : mb, b_is_a ? 0 : nb, d, n_pairs, capacity != nullptr);
  if (int rc = check_workspace(workspace, workspace_bytes, need, "similarity: ")) return rc;

  // ---- device
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  int dev = 0, sms = 0;
  if (int rc = query_device(&dev, &sms)) return rc;
  const SimOperand A{a, ma, na, a_normalize, a_norm_floor};
  const SimOperand B = b_is_a ? A : SimOperand{b, mb, nb, b_normalize, b_norm_floor};
  // AUTO: bf16x3. Unlike the training GEMMs, whose epilogues write operand planes and which are bound by the SM's data
  // paths, this GEMM's epilogue is light, and the widening of the E5M2 tiles made f16f8 the slower arithmetic here (H100,
  // config 2: 30.1 ms against 23.9 ms per pass) as well as the less accurate one (5e-6 against 1.3e-6 from fp64).
  // SCE_ARITH=f16f8 pins AUTO to f16f8 where d % 16 == 0. f16f8 splits a raw operand first and reads its range flag back
  // (one 4-byte copy + synchronise): a value fp16 cannot hold (|v| >= 65520 or NaN) moves a pinned AUTO to bf16x3 and
  // is an error under explicit F16F8.
  const char* env = getenv("SCE_ARITH");
  bool f8 = arith == SCE_ARITH_F16F8 || (arith == SCE_ARITH_AUTO && env && !strcmp(env, "f16f8") && d % 16 == 0);
  const bool raw = !A.normalize || (!b_is_a && !B.normalize);
  SimCarve w;
  if (f8 && raw) {
    sim_carve(static_cast<uint8_t*>(workspace), true, ma, na, b_is_a ? 0 : mb, b_is_a ? 0 : nb, d, n_pairs, capacity != nullptr, &w);
    CUDA_TRY(cudaMemsetAsync(w.flags, 0, kFlagWords * sizeof(uint32_t), st));
    int rc = SCE_OK;
    if (!A.normalize) rc = sim_planes<kArithF16F8>(A, d, w.a_hi, w.a_lo, w.a_x8, w.flags, st);
    if (!rc && !b_is_a && !B.normalize) rc = sim_planes<kArithF16F8>(B, d, w.b_hi, w.b_lo, w.b_x8, w.flags, st);
    if (rc) return rc;
    uint32_t bad = 0;
    CUDA_TRY(cudaMemcpyAsync(&bad, w.flags + kBadWord, sizeof(bad), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    if (bad) {
      if (arith == SCE_ARITH_F16F8)
        return fail(SCE_ERR_INVALID, "similarity: a raw operand holds a value fp16 cannot (|v| >= 65520 or NaN); use "
                                     "arith = BF16X3 or AUTO");
      f8 = false;
    }
  }
  sim_carve(static_cast<uint8_t*>(workspace), f8, ma, na, b_is_a ? 0 : mb, b_is_a ? 0 : nb, d, n_pairs, capacity != nullptr, &w);
  // the pair list and row counts are host locals: copies from pageable memory are staged before cudaMemcpyAsync returns
  CUDA_TRY(cudaMemcpyAsync(w.pairs, pv.data(), pv.size() * sizeof(int), cudaMemcpyHostToDevice, st));
  CUDA_TRY(cudaMemcpyAsync(w.a_rows, rows.data(), (size_t)ma * sizeof(int), cudaMemcpyHostToDevice, st));
  if (!b_is_a) CUDA_TRY(cudaMemcpyAsync(w.b_rows, rows.data() + ma, (size_t)mb * sizeof(int), cudaMemcpyHostToDevice, st));
  // (a raw operand split above for the range check is split again here: the planes of the arithmetic that runs)
  return f8 ? run_similarity_t<kArithF16F8>(A, B, b_is_a, d, n_pairs, w, row_max, col_max, capacity, dev, sms, st)
            : run_similarity_t<kArithBf16x3>(A, B, b_is_a, d, n_pairs, w, row_max, col_max, capacity, dev, sms, st);
}

int sce_synth_rows(const float* feats, int n_gt, int d, const float* probs, int group_rows, long long row0, int B,
                   unsigned long long seed, int zero_row_rule, float noise_scale, void* out, int out_half, int* row_nnz,
                   int* code_idx, float* code_val, int code_cap, void* stream) {
  // ---- arguments (all checked before any CUDA call)
  if (!feats || !probs || !out) return fail(SCE_ERR_INVALID, "synth_rows: feats, probs and out are required");
  if (n_gt < 1 || B < 1) return fail(SCE_ERR_INVALID, "synth_rows: n_gt (%d) and B (%d) must be >= 1", n_gt, B);
  if (d < 8 || d % 8) return fail(SCE_ERR_INVALID, "synth_rows: d (%d) must be a positive multiple of 8", d);
  if (d > 8192) return fail(SCE_ERR_INVALID, "synth_rows: d = %d > 8192 is not supported by the row kernels", d);
  if (group_rows < 1) return fail(SCE_ERR_INVALID, "synth_rows: group_rows (%d) must be >= 1", group_rows);
  if (row0 < 0) return fail(SCE_ERR_INVALID, "synth_rows: row0 (%lld) must be >= 0", row0);
  if ((zero_row_rule != 0 && zero_row_rule != 1) || (out_half != 0 && out_half != 1))
    return fail(SCE_ERR_INVALID, "synth_rows: zero_row_rule and out_half must be 0 or 1");
  if (!(noise_scale >= 0.f && noise_scale <= 3.0e38f))
    return fail(SCE_ERR_INVALID, "synth_rows: noise_scale must be finite and >= 0");
  if (!code_idx != !code_val) return fail(SCE_ERR_INVALID, "synth_rows: code_idx and code_val go together");
  if (code_idx && code_cap < 1) return fail(SCE_ERR_INVALID, "synth_rows: code_cap (%d) must be >= 1 with code lists", code_cap);
  if (reinterpret_cast<uintptr_t>(out) % 16 || reinterpret_cast<uintptr_t>(feats) % 16)
    return fail(SCE_ERR_INVALID, "synth_rows: out and feats must be 16-byte aligned");

  // ---- device
  SynthArgs a{feats, probs, n_gt, d, group_rows, B, row0, (uint32_t)seed, (uint32_t)(seed >> 32), zero_row_rule,
              noise_scale, out, out_half, row_nnz, code_idx, code_val, code_idx ? code_cap : 0};
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const unsigned rows8 = (unsigned)((B + 7) / 8);
  if (d <= 128) synth_rows_kernel<1, false><<<rows8, 256, 0, st>>>(a);
  else if (d <= 256) synth_rows_kernel<2, false><<<rows8, 256, 0, st>>>(a);
  else if (d <= 512) synth_rows_kernel<4, false><<<rows8, 256, 0, st>>>(a);
  else if (d <= 1024) synth_rows_kernel<8, false><<<rows8, 256, 0, st>>>(a);
  else synth_rows_kernel<8, true><<<(unsigned)B, 32 * ((d + 1023) / 1024), 0, st>>>(a);
  CUDA_TRY(cudaGetLastError());
  return SCE_OK;
}

}  // extern "C"
