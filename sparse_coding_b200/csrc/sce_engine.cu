// sce_engine.cu — libsce.so: the C ABI of include/sce.h on top of the wgmma GEMM core and the
// streaming kernels. One `sce_plan` = one stacked ensemble (FunctionalEnsemble, autoencoders/ensemble.py:68-97).
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
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <algorithm>
#include <cstring>
#include <map>
#include <vector>
#include <new>
#include <utility>

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
// returns the SCE_ERR_* code of a failed call
#define TRY(x)                       \
  do {                               \
    if (int rc_ = (x)) return rc_;   \
  } while (0)

// The kernel launches of one call on one stream. Every launch goes through launch() (or launch_gemm_t), which checks
// it and counts it; the entry points that report their launches (sce_last_launch_count) read `count`.
struct Launcher {
  cudaStream_t st;
  int count = 0;
  template <class... P, class... A>
  int launch(void (*kernel)(P...), dim3 grid, dim3 block, size_t smem, A&&... args) {
    kernel<<<grid, block, smem, st>>>(std::forward<A>(args)...);
    CUDA_TRY(cudaGetLastError());
    ++count;
    return SCE_OK;
  }
};

// ------------------------------------------------------------------------------------------------
// plan
// ------------------------------------------------------------------------------------------------
// The planes of one operand tensor. bf16x3: hi, lo = bf16 planes (2 B / element each), x8 = nullptr. f16f8: hi = fp16
// plane, lo = E5M2 plane of the values, x8 = E5M2 plane of the scaled residuals (1 B / element each): 4 B / element
// either way. The batch-major 8-bit copies of native dW are Planes without a 16-bit plane.
struct Planes {
  void* hi;
  void* lo;
  uint8_t* x8;
  bool f8;
  size_t lo_size() const { return f8 ? 1 : 2; }   // bytes per element of lo (and of x8)
  // the planes from element `e` on (a model's slab)
  Planes at(size_t e) const {
    return {hi ? static_cast<uint8_t*>(hi) + 2 * e : nullptr, lo ? static_cast<uint8_t*>(lo) + lo_size() * e : nullptr,
            x8 ? x8 + e : nullptr, f8};
  }
  // zero the first `count` elements of every plane
  cudaError_t zero(size_t count, cudaStream_t st) const {
    cudaError_t e = cudaMemsetAsync(hi, 0, 2 * count, st);
    if (e == cudaSuccess) e = cudaMemsetAsync(lo, 0, lo_size() * count, st);
    if (e == cudaSuccess && x8) e = cudaMemsetAsync(x8, 0, count, st);
    return e;
  }
};

struct OperandMaps {   // tensor maps of one operand's planes
  CUtensorMap hi, lo, x8;
};
struct GemmMaps {      // tensor maps of one GEMM for one batch size
  OperandMaps a[kMaxSets], b[kMaxSets];
};
struct BatchMaps {
  GemmMaps encode, decode, dcode, dw_enc, dw_dec;
  GemmMaps center;             // centring: A = (x - trans) planes [M,B,d], B = rot planes [M,d,d], both K-major
  OperandMaps st_c, st_dz;     // epilogue TMA-store maps
  CUtensorMap st_scores;       // top-k: fp32 scores
  cudaGraphExec_t graph;       // captured step for this batch size (launch-bound shapes), or nullptr
  int graph_launches, eager_steps;
};

// The plan's workspace buffers, in carve order (carve)
struct PlanBuffers {
  float* x_stage;                 // [xm, Bmax, d] staging for host-fed steps
  Planes x;                       // [xm, Bmax, d]
  Planes wenc, wdec;              // [M, n, d] (tied: wdec is a copy of wenc)
  Planes wdt;                     // f16f8: the decoder's planes transposed, [M, d, n]: the decode GEMM's B operand, K-major (transpose_dict)
  Planes c;                       // [M, Bmax, n]   (dw_native: the 8-bit planes are dz's, see carve)
  Planes g;                       // [M, Bmax, d]
  Planes dz;                      // [M, Bmax, n], one contiguous block of 4 B / element (top-k: fp32 scores alias it);
                                  // dw_native: the 8-bit planes are [M, n, Bp]
  // dw_native (dense f16f8 plans): batch-major copies of the 8-bit planes of x, c and g, [xm or M, cols, Bp] with Bp =
  // batch_max rounded up to 16 (TMA pitch): the weight gradient reads them K-major over the batch (E5M2 wgmma).
  // dz's 8-bit planes are written in that layout in the first place (EpiDcodeT<f16f8, true>).
  Planes xt, ct, gt;
  Planes rot;                     // centring: operand planes of buffers["center_rot"] [M, d, d]
  float* x_centered;              // centring, learned centre: the centred batch [M, B, d] (B, not Bmax, rows per model: what a caller's [M,B,d] looks like)
  // learned centre: column sums of g [M, tiles_m*4, d] (EpiDecodeT<AR, true>), db / ||E_n|| [M, n], the GEMV partials
  // [M, ceil(n / kCenterChunkRows), d] and the centre gradient [M, d] (sce_read_center_grad)
  float *g_part, *center_coef, *center_part, *center_grad;
  float* x_shifted;               // input_shift: x + input_shift [xm, B, d], written by the batch split
  float* scores;                  // top-k: fp32 scores [M, Bmax, n] of the encode GEMM
  int* tk_models;                 // top-k gather kernel: the models sorted into k classes (device copy of tk_group_models)
  uint32_t* tk_cmax;              // top-k: largest key per 32-column chunk of the scores [M, Bmax, n_chunks] (EpiScoresTma)
  int *tk_col, *tk_cnt;           // top-k lists (TopkLists): selected columns [M, Bmax, kmax], entries per row [M, Bmax]
  float *tk_val, *tk_dots;        // their values [M, Bmax, kmax]; per-slice shares of g . W_j [M, Bmax, kmax, slices]
  float* wn_f32;                  // top-k: fp32 copy of the normalised dictionary [M, n, d] the gather kernel reads
  uint32_t *act_pos, *act_zero;   // activity masks [M][ceil(n/32)][Bmax]: bit 31-j of a word = column 32*chunk + j (ActMask)
  uint32_t* res_flags;            // [0]: the batch has a non-zero residual plane (f16f8; written by the batch split)
  float *dw_enc, *dw_dec;         // [M, n, d]
  float *part_enc, *part_dec, *db_part, *bnorm, *l1_over_b, *loss_stage, *nnz_stage;
};

// What a plan decides from its descriptor, once (plan_config): the workspace carve and every launch follow from it
struct PlanConfig {
  int arith;           // kArithBf16x3 or kArithF16F8
  bool untied;         // SCE_UNTIED: a decoder of its own, a second dictionary side
  bool topk;           // SCE_TOPK
  bool learned;        // SCE_TIED_LEARNED_CENTER: the step centres the batch on params["center"] and trains the centre
  bool x_models;       // the batch the kernels read holds one slab per model (x_per_model, or always with a learned centre)
  int xm;              // number of distinct input batches (1 shared, or M)
  int input_models;    // models' worth of rows in the caller's batch: 1 when it is shared ([B,d]; also centering = 1), else M
  bool evaluable;      // the forward-only passes may run it: not plans whose export (a TiedSAE) differs from their forward
  int bpad;            // Bp: batch_max rounded up to 16 (TMA pitch of the batch-major 8-bit planes)
  int tk_kmax;         // top-k list capacity per row (desc.topk_k_max rounded up to 8; 0: no lists)
  int tk_slices;       // slices of the activation width topk_sparse_kernel runs per row (0: none fits)
  bool topk_sparse;    // decode / dcode of the top-k variant run as the k-sparse gather kernels
  bool dw_native;      // the weight gradient's cross terms run on E5M2 wgmma from batch-major copies (carve)
  bool split_decode;   // separate accumulators for hi*hi and the cross terms in the decode GEMM (bf16x3)
  bool use_graph;      // replay the step as a CUDA graph
  bool nonneg;         // desc.encoder_nonneg: the dictionary rows are built from max(E, 0) (dict_rows_kernel<..., true>)
  float shift;         // desc.input_shift; non-zero: the batch split also writes x + shift, which the step reads
};

struct sce_plan : PlanBuffers {
  sce_desc d;
  sce_buffers b;
  PlanConfig cfg;
  int sms;
  int device;  // CUDA device the plan was created on (the caller keeps it current for every call)
  int code_batch_major;            // 1: the last call was a dw_native backward, which left the code's residual plane
                                   // only in its batch-major copy (ct.x8): dcode overwrote the row-major one (carve)
  int tk_groups, tk_group_off[5], tk_group_krows[4];   // classes: models [off[g], off[g+1]) need at most krows[g] rows
  std::map<int, BatchMaps*>* maps;
  cudaStream_t cap_stream;  // private stream the step is captured on
  int last_launches;
  long long step;  // number of optimiser steps taken
  // optional per-phase device timing (sce_profile_*): events bracket each phase of a step
  bool prof_on;
  int prof_steps;                          // steps recorded since sce_profile_begin
  cudaEvent_t* prof_ev;                    // [kProfMaxSteps][SCE_PHASE_COUNT + 1]
};

constexpr int kProfMaxSteps = 64;

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
  // the planes of `count` elements of one operand tensor: 16-bit, then a second 16-bit plane (bf16x3) or two 8-bit ones
  Planes planes(size_t count, bool f8) {
    Planes p{take<uint16_t>(count), nullptr, nullptr, f8};
    if (f8) {
      p.lo = take<uint8_t>(count);
      p.x8 = take<uint8_t>(count);
    } else {
      p.lo = take<uint16_t>(count);
    }
    return p;
  }
  // the batch-major copies of the two 8-bit planes of `count` elements (f16f8), which have no 16-bit plane
  Planes copies(size_t count) { return {nullptr, take<uint8_t>(count), take<uint8_t>(count), true}; }
};

static int validate(const sce_desc* d) {
  if (!d) return fail(SCE_ERR_INVALID, "desc is NULL");
  if (d->variant < SCE_TIED || d->variant > SCE_TIED_LEARNED_CENTER) return fail(SCE_ERR_INVALID, "unknown variant %d", d->variant);
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

// fp32 rows -> the operand planes of arithmetic AR: n4 float4s, grid-stride over at most 2048 blocks. With `xs`, the
// rows are shifted by `shift` first and the shifted fp32 rows are written to `xs` as well (input_shift plans).
template <int AR>
static int launch_split_rows(Launcher& L, const float* x, const Planes& w, long long n4, uint32_t* flags,
                             float shift = 0.f, float* xs = nullptr) {
  const int blocks = (int)((n4 + 255) / 256 < 2048 ? (n4 + 255) / 256 : 2048);
  if (xs) return L.launch(split_rows_kernel<AR, true>, blocks, 256, 0, x, w.hi, w.lo, w.x8, n4, flags, shift, xs);
  return L.launch(split_rows_kernel<AR>, blocks, 256, 0, x, w.hi, w.lo, w.x8, n4, flags, 0.f, nullptr);
}

// SCE_ARITH=bf16x3|f16f8: the arithmetic the environment pins arith = AUTO to (include/sce.h), else SCE_ARITH_AUTO
static int env_arith() {
  const char* v = getenv("SCE_ARITH");
  if (v && !strcmp(v, "bf16x3")) return SCE_ARITH_BF16X3;
  if (v && !strcmp(v, "f16f8")) return SCE_ARITH_F16F8;
  return SCE_ARITH_AUTO;
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
static PlanConfig plan_config(const sce_desc& d) {
  PlanConfig c{};
  c.arith = resolve_arith(d);
  c.untied = d.variant == SCE_UNTIED;
  c.topk = d.variant == SCE_TOPK;
  c.learned = d.variant == SCE_TIED_LEARNED_CENTER;
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
  // would add three launches per step and a third to the workspace.
  c.dw_native = c.arith == kArithF16F8 && !c.topk && d.bwd_passes >= 3 && !launch_bound;
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
// K-major 16-bit tiles [rows][bk], bk = gemm_bk(arith): the swizzle span is one tile row of 2 bk bytes
static CUtensorMapSwizzle swizzle_for_bk(int bk) {
  return bk * 2 == 64 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_128B;
}

// The planes of one operand [models][rows][cols] (cols contiguous, `mpitch` elements between models) as GEMM operand
// maps. kmajor_bk != 0: K-major tiles [box_rows][kmajor_bk]; else MN-major tiles of `box_rows` k-rows by 64 (16-bit)
// / 128 (8-bit) contiguous elements. K-major 8-bit tiles (64-byte rows in f16f8) carry the 64-byte swizzle E5M2 wgmma
// reads; MN-major ones arrive unswizzled and the GEMM widens them to fp16 (widen_tile).
static bool operand_maps(OperandMaps& m, const Planes& P, uint64_t models, uint64_t rows, uint64_t cols, uint64_t mpitch,
                         uint32_t box_rows, int kmajor_bk) {
  bool ok;
  if (kmajor_bk) {
    ok = make_tmap_bf16_box(&m.hi, P.hi, models, rows, cols, cols, mpitch, kmajor_bk, box_rows, swizzle_for_bk(kmajor_bk));
    if (P.f8)
      ok = ok && make_tmap_u8_box(&m.lo, P.lo, models, rows, cols, cols, mpitch, kmajor_bk, box_rows, CU_TENSOR_MAP_SWIZZLE_64B) &&
           make_tmap_u8_box(&m.x8, P.x8, models, rows, cols, cols, mpitch, kmajor_bk, box_rows, CU_TENSOR_MAP_SWIZZLE_64B);
    else
      ok = ok && make_tmap_bf16_box(&m.lo, P.lo, models, rows, cols, cols, mpitch, kmajor_bk, box_rows, swizzle_for_bk(kmajor_bk));
  } else {
    ok = make_tmap_bf16(&m.hi, P.hi, models, rows, cols, cols, mpitch, box_rows);
    if (P.f8)
      ok = ok && make_tmap_u8_box(&m.lo, P.lo, models, rows, cols, cols, mpitch, 128, box_rows, CU_TENSOR_MAP_SWIZZLE_NONE) &&
           make_tmap_u8_box(&m.x8, P.x8, models, rows, cols, cols, mpitch, 128, box_rows, CU_TENSOR_MAP_SWIZZLE_NONE);
    else
      ok = ok && make_tmap_bf16(&m.lo, P.lo, models, rows, cols, cols, mpitch, box_rows);
  }
  return ok;
}

// The weight gradient's operand P [models][k_rows][cols] (`mpitch` elements between models), reduced over its k_rows:
// MN-major tiles of bk rows. With T, the 8-bit planes come from P's batch-major copies T [models][cols][t_pitch] instead
// (batch_major), K-major tiles [128 rows][64 B] with the 64-byte swizzle E5M2 wgmma reads; only k_rows columns of T are
// exposed, so the tail of a short batch reads as zero.
static bool dw_operand_maps(OperandMaps& m, const Planes& P, const Planes* T, uint64_t models, uint64_t k_rows,
                            uint64_t cols, uint64_t mpitch, uint64_t t_pitch, int bk) {
  if (!T) return operand_maps(m, P, models, k_rows, cols, mpitch, bk, 0);
  return make_tmap_bf16(&m.hi, P.hi, models, k_rows, cols, cols, mpitch, bk) &&
         make_tmap_u8_box(&m.lo, T->lo, models, cols, k_rows, t_pitch, cols * t_pitch, bk, kBM, CU_TENSOR_MAP_SWIZZLE_64B) &&
         make_tmap_u8_box(&m.x8, T->x8, models, cols, k_rows, t_pitch, cols * t_pitch, bk, kBM, CU_TENSOR_MAP_SWIZZLE_64B);
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
  ok &= act_a(m->decode.a[0], p->c, M, n);
  ok &= f8 ? operand_maps(m->decode.b[0], p->wdt, M, dd, n, dd * n, kBN, bk) : dict_b(m->decode.b[0], p->wdec, bk, 0);
  // dcode: A = g [M,B,d] K-major, B = Wdec K-major
  ok &= act_a(m->dcode.a[0], p->g, M, dd);
  ok &= dict_b(m->dcode.b[0], p->wdec, kBN, bk);
  // weight gradients: reduction over the batch rows; dw_native: the 8-bit planes from the batch-major copies [models][cols][Bp]
  const uint64_t Bp = (uint64_t)cfg.bpad;
  auto dw_operand = [&](OperandMaps& o, const Planes& P, const Planes& T, uint64_t models, uint64_t cols) {
    return dw_operand_maps(o, P, cfg.dw_native ? &T : nullptr, models, (uint64_t)B, cols, Bm * cols, Bp, bk);
  };
  // dz^T x, then c^T g: a second GEMM of the decoder (untied) or a second operand set of the one dictionary's
  // (dz's own 8-bit planes are batch-major in dw_native plans)
  GemmMaps& cg = cfg.untied ? m->dw_dec : m->dw_enc;
  const int cg_set = cfg.untied ? 0 : 1;
  ok &= dw_operand(m->dw_enc.a[0], p->dz, p->dz, M, n) && dw_operand(m->dw_enc.b[0], p->x, p->xt, xm, dd);
  ok &= dw_operand(cg.a[cg_set], p->c, p->ct, M, n) && dw_operand(cg.b[cg_set], p->g, p->gt, M, dd);
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
// GEMM launcher
// ------------------------------------------------------------------------------------------------
// device flags "this operand's residual plane is all zeros" (f16f8; GemmParams::a_res_flag), nullptr = unknown
struct ResFlags {
  const uint32_t* a[kMaxSets] = {nullptr, nullptr};
  const uint32_t* b[kMaxSets] = {nullptr, nullptr};
};

// the tensor maps of operand set `s` into the kernel's parameters
template <class EpiParams>
static void set_operand_maps(GemmParams<EpiParams>& gp, int s, const OperandMaps& a, const OperandMaps& b) {
  gp.a_hi[s] = a.hi;
  gp.a_lo[s] = a.lo;
  gp.a_x8[s] = a.x8;
  gp.b_hi[s] = b.hi;
  gp.b_lo[s] = b.lo;
  gp.b_x8[s] = b.x8;
}

// a_batched / b_batched of the operand sets that hold one slab per model
static const int kOnes[2] = {1, 1};

// One GEMM over `n_models` models on `device` (with `sms` SMs), launched and counted by L
template <class Epi, bool A_MN, bool B_MN, bool SPLIT_ACC, int ARITH, bool NATIVE>
static int launch_gemm_t(Launcher& L, int n_models, int device, int sms, const GemmMaps& maps, int nsets,
                         const int* a_batched, const int* b_batched, int k_total, int passes, int m_total, int n_total,
                         const typename Epi::Params& epi, const ResFlags& rf = ResFlags()) {
  GemmParams<typename Epi::Params> gp;
  memset(&gp, 0, sizeof(gp));
  for (int s = 0; s < nsets; ++s) {
    set_operand_maps(gp, s, maps.a[s], maps.b[s]);
    gp.a_batched[s] = a_batched[s];
    gp.b_batched[s] = b_batched[s];
    gp.a_res_flag[s] = rf.a[s];
    gp.b_res_flag[s] = rf.b[s];
  }
  gp.nsets = nsets;
  gp.k_total = k_total;
  gp.passes = passes;
  gp.n_models = n_models;
  gp.m_total = m_total;
  gp.n_total = n_total;
  gp.tiles_m = (m_total + kBM - 1) / kBM;
  gp.tiles_n = (n_total + kBN - 1) / kBN;
  gp.epi = epi;
  CUDA_TRY((launch_gemm<Epi, A_MN, B_MN, SPLIT_ACC, ARITH, NATIVE>(gp, device, sms, L.st)));
  ++L.count;
  return SCE_OK;
}

// The weight gradient's GEMM (launch_gemm_t's arguments after L): a reduction over rows, both operands as
// dw_operand_maps builds them, fp32 out. bf16x3 keeps split accumulators (f16f8 rescales inside one). `native` (f16f8,
// 8-bit planes from batch-major copies): the cross terms run on E5M2 wgmma; else the 8-bit tiles are widened to fp16.
template <int AR, class... A>
static int launch_dw_t(Launcher& L, bool native, const A&... args) {
  constexpr bool f8 = AR == kArithF16F8;
  if constexpr (f8)
    if (native) return launch_gemm_t<EpiStoreF32, true, true, false, AR, true>(L, args...);
  return launch_gemm_t<EpiStoreF32, true, true, !f8, AR, false>(L, args...);
}

// One call of a plan: its launches, and the batch of B rows and its tensor maps (run_pipeline opens it)
struct PlanCall : Launcher {
  sce_plan* p;
  BatchMaps* maps;
  int B;
  // one GEMM of the plan. NATIVE (f16f8): the cross terms run on E5M2 wgmma, which needs K-major 8-bit maps (A_MN / B_MN
  // then describe the fp16 planes alone); K-major GEMMs always have them, the weight gradient where the plan keeps
  // batch-major copies.
  template <class Epi, bool A_MN, bool B_MN, bool SPLIT_ACC, int AR, bool NATIVE = AR == kArithF16F8 && !A_MN, class... A>
  int gemm(const A&... args) {
    return launch_gemm_t<Epi, A_MN, B_MN, SPLIT_ACC, AR, NATIVE>(*this, p->d.n_models, p->device, p->sms, args...);
  }
  // with sce_profile_begin: the event at the start of phase `idx` of this step (SCE_PHASE_COUNT: the step's end)
  void mark(int idx) {
    if (p->prof_on && p->prof_steps < kProfMaxSteps)
      cudaEventRecord(p->prof_ev[p->prof_steps * (SCE_PHASE_COUNT + 1) + idx], st);
  }
};

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

// Calls f(arith) with the plan's arithmetic as a compile-time constant (std::integral_constant<int, AR>)
template <class F>
static auto with_arith(int arith, F&& f) {
  return arith == kArithF16F8 ? f(std::integral_constant<int, kArithF16F8>{}) : f(std::integral_constant<int, kArithBf16x3>{});
}

// Calls f(nv) with the float4s per thread that dict_rows_kernel needs for rows of d values, ceil(d / 512) rounded up
// to 1, 2, 4, 8 or 16, as a compile-time constant
template <class F>
static auto with_row_vectors(int d, F&& f) {
  const int nv = (d + 511) / 512;
  if (nv == 1) return f(std::integral_constant<int, 1>{});
  if (nv == 2) return f(std::integral_constant<int, 2>{});
  if (nv <= 4) return f(std::integral_constant<int, 4>{});
  if (nv <= 8) return f(std::integral_constant<int, 8>{});   // d <= 4096 (Pythia-6.9b residual width)
  return f(std::integral_constant<int, 16>{});                // d <= 8192
}

template <int MODE, int ARITH, bool NONNEG = false>
static int launch_dict_rows_t(Launcher& L, float* e, const float* dw, float* m, float* v, const Planes& w,
                              float* grad_out, long long rows, int d, int normalize, float floor, AdamHyper h,
                              const uint32_t* health, float* w_f32) {
  return with_row_vectors(d, [&](auto nv) {
    return L.launch(dict_rows_kernel<decltype(nv)::value, MODE, ARITH, NONNEG>, (unsigned)rows, 128, 0, e, dw, m, v,
                    w.hi, w.lo, w.x8, grad_out, d, normalize, floor, h, health, w_f32);
  });
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

// The batch-major copy T [models][cols][ld] of the 8-bit planes of P [models][rows][cols] (`src_pitch` elements between
// models), from which the native weight gradient reads them (dw_operand_maps; dz's are written so by dcode)
static int batch_major(Launcher& L, const Planes& P, const Planes& T, int models, int rows, int cols, long long src_pitch,
                       int ld) {
  const BatchPlanes t{{static_cast<const uint8_t*>(P.lo), P.x8}, {static_cast<uint8_t*>(T.lo), T.x8}};
  return L.launch(transpose_batch_u8_kernel, dim3((cols + 127) / 128, (rows + 127) / 128, 2 * models), 256, 0, t, models,
                  rows, cols, src_pitch, ld);
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
    if (mom_part) {
      using EpiStats = EpiEncodeT<AR, true>;
      typename EpiStats::Params ep;
      fill(ep);
      ep.mom_part = mom_part;
      ep.row_blocks = (B + 31) / 32;
      TRY((c.gemm<EpiStats, false, false, false, AR>(c.maps->encode, 1, xb, kOnes, d.d, d.fwd_passes, B, n, ep, x_is_a)));
    } else {
      typename EpiEncodeT<AR>::Params ep;
      fill(ep);
      TRY((c.gemm<EpiEncodeT<AR>, false, false, false, AR>(c.maps->encode, 1, xb, kOnes, d.d, d.fwd_passes, B, n, ep,
                                                           x_is_a)));
    }
    return tdw ? batch_major(c, p->c, p->ct, M, B, n, (long long)d.batch_max * n, cfg.bpad) : SCE_OK;
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
  const int B = c.B, M = d.n_models, n = d.n, dd = d.d;
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
    if constexpr (!std::is_same<E, EpiDecodeT<AR>>::value) dp.g_part = p->g_part;
    if constexpr (f8)
      return c.gemm<E, false, false, false, AR>(c.maps->decode, 1, kOnes, kOnes, n, d.fwd_passes, B, dd, dp);
    else if (cfg.split_decode)
      return c.gemm<E, false, true, true, AR>(c.maps->decode, 1, kOnes, kOnes, n, d.fwd_passes, B, dd, dp);
    else
      return c.gemm<E, false, true, false, AR>(c.maps->decode, 1, kOnes, kOnes, n, d.fwd_passes, B, dd, dp);
  };
  TRY(cfg.learned ? decode(TypeTag<EpiDecodeT<AR, true>>{}) : decode(TypeTag<EpiDecodeT<AR>>{}));
  return tdw ? batch_major(c, p->g, p->gt, M, B, dd, (long long)d.batch_max * dd, cfg.bpad) : SCE_OK;
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
    return launch_dw_t<AR>(c, cfg.dw_native, M, p->device, p->sms, gm, nsets, ab, bb, B, d.bwd_passes, n, dd, sp, rf);
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
static int run_pipeline(PlanCall& c, sce_plan* p, const float* x, int B, cudaStream_t st, float* x_hat, bool backward,
                        float* out_losses, float* out_nnz, float* mom_part = nullptr) {
  TRY(check_rows(p, B, ""));
  if (!x) return fail(SCE_ERR_INVALID, "x is NULL");
  c = PlanCall{{st}, p, nullptr, B};
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
  const void* hi;             // the code's 16-bit plane [M][batch_max][n] (bf16 or fp16)
  const void* lo;             // bf16x3: its second bf16 plane
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
static int launch_fragments(Launcher& launcher, const FragCode& c, int M, int L, int G, long long frag0, float* fmax,
                            uint8_t* active, int n_top, int n_random, unsigned long long seed, float* top_val,
                            long long* top_frag, float* top_act, long long* rnd_key, long long* rnd_frag, float* rnd_act) {
  TRY(launcher.launch(fragment_max_kernel<ARITH, TOPK>, dim3(c.n_chunks, G, M), 256, 0, c, L, G, fmax, active));
  return launcher.launch(fragment_merge_kernel<ARITH, TOPK>, dim3((c.n + 127) / 128, M), 128, 0, c, L, G, frag0, fmax,
                         active, n_top, n_random, seed, top_val, top_frag, top_act, rnd_key, rnd_frag, rnd_act);
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
  Planes a, b;
  int *pairs, *a_rows, *b_rows;
  uint32_t* flags;
  float *sq_part, *diag;
};
static size_t sim_carve(uint8_t* base, bool f8, long long ma, long long na, long long mb, long long nb, long long d,
                        long long n_pairs, bool capacity, SimCarve* out) {
  Carve c{base, 0};
  SimCarve s{};
  s.a = c.planes((size_t)(ma * na * d), f8);
  if (mb > 0) s.b = c.planes((size_t)(mb * nb * d), f8);
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
static int sim_planes(Launcher& L, const SimOperand& o, int d, const Planes& w, uint32_t* flags) {
  const long long rows = (long long)o.models * o.rows;
  if (o.normalize)
    return launch_dict_rows_t<MODE_PREPARE, AR>(L, const_cast<float*>(o.w), nullptr, nullptr, nullptr, w, nullptr, rows, d,
                                                 1, o.floor, AdamHyper{}, nullptr, nullptr);
  return launch_split_rows<AR>(L, o.w, w, rows * d / 4, AR == kArithF16F8 ? flags : nullptr);
}

template <int AR>
static int run_similarity_t(Launcher& L, const SimOperand& A, const SimOperand& B, bool b_is_a, int d, int n_pairs,
                            const SimCarve& w, float* row_max, float* col_max, float* capacity, int device, int sms) {
  TRY(sim_planes<AR>(L, A, d, w.a, w.flags));
  if (!b_is_a) TRY(sim_planes<AR>(L, B, d, w.b, w.flags));
  // both operands are dictionary rows, K-major over d: the encode GEMM's B-operand geometry on both sides
  GemmMaps maps{};
  bool ok = operand_maps(maps.a[0], w.a, A.models, A.rows, d, (uint64_t)A.rows * d, kBM, gemm_bk(AR));
  ok = ok && operand_maps(maps.b[0], b_is_a ? w.a : w.b, B.models, B.rows, d, (uint64_t)B.rows * d, kBN, gemm_bk(AR));
  if (!ok) return fail(SCE_ERR_CUDA, "cuTensorMapEncodeTiled failed (similarity: na=%d, nb=%d, d=%d)", A.rows, B.rows, d);
  const int tiles_n = (B.rows + kBN - 1) / kBN;
  const EpiSimilarity::Params ep{w.pairs, w.a_rows, w.b_rows, reinterpret_cast<uint32_t*>(row_max),
                                 reinterpret_cast<uint32_t*>(col_max), capacity ? w.sq_part : nullptr, w.diag, tiles_n};
  if (row_max) CUDA_TRY(cudaMemsetAsync(row_max, 0, (size_t)n_pairs * A.rows * sizeof(float), L.st));
  if (col_max) CUDA_TRY(cudaMemsetAsync(col_max, 0, (size_t)n_pairs * B.rows * sizeof(float), L.st));
  TRY((launch_gemm_t<EpiSimilarity, false, false, false, AR, AR == kArithF16F8>(L, n_pairs, device, sms, maps, 1, kOnes,
                                                                                  kOnes, d, 3, A.rows, B.rows, ep)));
  auto to_float = [&](float* v, long long n) {
    const int blocks = (int)((n + 255) / 256 < 1024 ? (n + 255) / 256 : 1024);
    return L.launch(key_to_float_kernel, blocks, 256, 0, reinterpret_cast<uint32_t*>(v), n);
  };
  if (row_max) TRY(to_float(row_max, (long long)n_pairs * A.rows));
  if (col_max) TRY(to_float(col_max, (long long)n_pairs * B.rows));
  if (!capacity) return SCE_OK;
  return L.launch(capacity_kernel, dim3((A.rows + 255) / 256, n_pairs), 256, 0, w.pairs, w.a_rows, w.sq_part, w.diag,
                  A.rows, 2 * tiles_n, capacity);
}

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
  return launch_dw_t<AR>(L, f8, S, device, sms, maps, 1, kOnes, kOnes, R, 3, m, d, sp);
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

// ------------------------------------------------------------------------------------------------
// C ABI
// ------------------------------------------------------------------------------------------------
extern "C" {

int sce_version(void) { return SCE_VERSION; }
const char* sce_last_error(void) { return g_err; }

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
  if (desc->variant == SCE_UNTIED && (!b.decoder || !b.decoder_m || !b.decoder_v))
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
  DictSide sides[2];
  for (int s = 0, ns = dict_sides(p, sides); s < ns; ++s)
    TRY(launch_dict_rows<MODE_PREPARE>(L, p, sides[s], nullptr, hyper_for(p, 1)));
  return transpose_dict(L, p);
}

int sce_forward(sce_plan* p, const float* x, int B, float* x_hat, float* out_losses, float* out_nnz, void* stream) {
  if (!p) return fail(SCE_ERR_INVALID, "plan is NULL");
  PlanCall c;
  TRY(run_pipeline(c, p, x, B, static_cast<cudaStream_t>(stream), x_hat, false, out_losses, out_nnz));
  p->last_launches = c.count;
  return SCE_OK;
}

// every launch of one optimisation step, in order, on `st` (also what gets captured into a CUDA graph), counted in `c`
static int step_launches(PlanCall& c, sce_plan* p, const float* x, int B, float* out_losses, float* out_nnz, long long t,
                         cudaStream_t st) {
  TRY(run_pipeline(c, p, x, B, st, nullptr, true, out_losses, out_nnz));
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

int sce_step(sce_plan* p, const float* x, int B, float* out_losses, float* out_nnz, void* stream) {
  if (!p) return fail(SCE_ERR_INVALID, "plan is NULL");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (int rc = check_rows(p, B, "")) return rc;
  if (!x) return fail(SCE_ERR_INVALID, "x is NULL");
  PlanCall c;
  int rc;
  if (!graph_eligible(p)) {
    rc = step_launches(c, p, x, B, out_losses, out_nnz, p->step + 1, st);
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

int sce_grads(sce_plan* p, const float* x, int B, float* d_encoder, float* d_bias, float* d_decoder,
              float* out_losses, float* out_nnz, void* stream) {
  if (!p) return fail(SCE_ERR_INVALID, "plan is NULL");
  PlanCall c;
  TRY(run_pipeline(c, p, x, B, static_cast<cudaStream_t>(stream), nullptr, true, out_losses, out_nnz));
  p->last_launches = c.count;   // the pipeline's: the gradient kernels below are not counted
  float* const grad_out[2] = {d_encoder, d_decoder};
  return train_tail<MODE_GRAD>(c, hyper_for(p, 1), grad_out, d_bias);
}

int sce_step_host(sce_plan* p, const float* x_host, int B, float* out_losses_host, float* out_nnz_host,
                  void* stream) {
  if (!p) return fail(SCE_ERR_INVALID, "plan is NULL");
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

int sce_read_code(sce_plan* p, int B, float* out_code, void* stream) {
  if (!p || !out_code) return fail(SCE_ERR_INVALID, "plan / out_code is NULL");
  if (int rc = check_rows(p, B, "")) return rc;
  Launcher L{static_cast<cudaStream_t>(stream)};
  const long long per = (long long)B * p->d.n;
  if (p->code_batch_major) {
    const long long total = (long long)p->d.n_models * per;
    return L.launch(join_code_batch_major_kernel, (unsigned)((total + 255) / 256 < 4096 ? (total + 255) / 256 : 4096), 256,
                    0, static_cast<const __half*>(p->c.hi), p->ct.x8, out_code, B, p->d.n, p->d.batch_max, p->cfg.bpad,
                    total);
  }
  for (int m = 0; m < p->d.n_models; ++m) {
    const Planes c = p->c.at((size_t)m * p->d.batch_max * p->d.n);
    TRY(with_arith(p->cfg.arith, [&](auto arith) {   // (each arithmetic reads its own planes)
      return L.launch(join_code_kernel<decltype(arith)::value>, 1024, 256, 0, c.hi, c.lo, c.x8, out_code + (long long)m * per,
                      per / 2);
    }));
  }
  return SCE_OK;
}

int sce_read_center_grad(sce_plan* p, float* d_center, void* stream) {
  if (!p || !d_center) return fail(SCE_ERR_INVALID, "plan / d_center is NULL");
  if (!p->cfg.learned) return fail(SCE_ERR_INVALID, "read_center_grad: the plan has no learned centre");
  CUDA_TRY(cudaMemcpyAsync(d_center, p->center_grad, (size_t)p->d.n_models * p->d.d * sizeof(float),
                           cudaMemcpyDeviceToDevice, static_cast<cudaStream_t>(stream)));
  return SCE_OK;
}

int sce_gather_rows(const void* chunk, int chunk_is_half, long long n_rows, int d, const long long* idx, int B,
                    const float* sub, float* out, void* stream) {
  if (!chunk || !out || B < 1 || d < 4 || d % 4) return fail(SCE_ERR_INVALID, "bad arguments to sce_gather_rows");
  Launcher L{static_cast<cudaStream_t>(stream)};
  const int blocks = (B + 7) / 8;
  if (chunk_is_half)
    return L.launch(gather_rows_kernel<__half>, blocks, 256, 0, static_cast<const __half*>(chunk), n_rows, d, idx, B, sub,
                    out);
  return L.launch(gather_rows_kernel<float>, blocks, 256, 0, static_cast<const float*>(chunk), n_rows, d, idx, B, sub, out);
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

int sce_active_counts(sce_plan* plan, int B, int* counts, void* stream) {
  if (!plan || !counts) return fail(SCE_ERR_INVALID, "plan / counts is NULL");
  if (int rc = check_rows(plan, B, "")) return rc;
  const int n_chunks = (plan->d.n + 31) / 32;
  Launcher L{static_cast<cudaStream_t>(stream)};
  return L.launch(active_count_kernel, dim3(n_chunks, plan->d.n_models), 256, 0, plan->act_pos, n_chunks,
                  plan->d.batch_max, B, plan->d.n, counts);
}

// The checks that open sce_forward_stats and sce_forward_fragments; `prefix` names the entry point in the messages
static int check_forward_only(const sce_plan* p, const float* x, int B, const char* prefix) {
  if (!p) return fail(SCE_ERR_INVALID, "%splan is NULL", prefix);
  if (!p->cfg.evaluable)
    return fail(SCE_ERR_INVALID, "%snot available for the learned-centre variant or with encoder_nonneg / input_shift; "
                                 "evaluate the exported dictionaries (TiedSAE)", prefix);
  TRY(check_rows(p, B, prefix));
  if (!x) return fail(SCE_ERR_INVALID, "%sx is NULL", prefix);
  return SCE_OK;
}

size_t sce_forward_stats_workspace_bytes(const sce_desc* desc, int B) {
  if (validate(desc) || B < 1 || B > desc->batch_max || !plan_config(*desc).evaluable) return 0;
  return stats_workspace(*desc, B);
}

int sce_forward_stats(sce_plan* p, const float* x, int B, int seg, int seg_phase, float* x_hat, float* out_losses,
                      float* out_nnz, double* moment_sums, int* seg_counts, int* seg_open, void* workspace,
                      size_t workspace_bytes, void* stream) {
  TRY(check_forward_only(p, x, B, "forward_stats: "));
  if (seg < 1) return fail(SCE_ERR_INVALID, "forward_stats: seg = %d must be >= 1", seg);
  if (seg_phase < 0 || seg_phase >= seg)
    return fail(SCE_ERR_INVALID, "forward_stats: seg_phase = %d outside [0, seg = %d)", seg_phase, seg);
  if (!out_losses || !out_nnz || !moment_sums || !seg_counts)
    return fail(SCE_ERR_INVALID, "forward_stats: out_losses, out_nnz, moment_sums and seg_counts are required");
  if (seg > 1 && !seg_open) return fail(SCE_ERR_INVALID, "forward_stats: seg > 1 needs the seg_open flags");
  if (int rc = check_workspace(workspace, workspace_bytes, stats_workspace(p->d, B), "forward_stats: ")) return rc;
  const sce_desc& d = p->d;
  float* part = static_cast<float*>(workspace);
  PlanCall c;
  TRY(run_pipeline(c, p, x, B, static_cast<cudaStream_t>(stream), x_hat, false, out_losses, out_nnz,
                   p->cfg.topk ? nullptr : part));
  p->last_launches = c.count;   // the pipeline's: the statistics kernels below are not counted
  const int n_chunks = (d.n + 31) / 32, row_blocks = (B + 31) / 32;
  if (p->cfg.topk)
    TRY(c.launch(topk_moment_kernel, dim3(n_chunks, (row_blocks + 7) / 8, d.n_models), 256, 0, p->scores, p->act_pos,
                 n_chunks, d.batch_max, B, d.n, row_blocks, part));
  TRY(c.launch(moment_reduce_kernel, dim3((d.n + 255) / 256, d.n_models), 256, 0, part, row_blocks, d.n, moment_sums));
  if (seg == 1)
    return c.launch(active_count_kernel, dim3(n_chunks, d.n_models), 256, 0, p->act_pos, n_chunks, d.batch_max, B, d.n,
                    seg_counts);
  return c.launch(segment_count_kernel, dim3(n_chunks, d.n_models), 256, 0, p->act_pos, n_chunks, d.batch_max, B, d.n, seg,
                  seg_phase, seg_counts, seg_open);
}

size_t sce_fragments_workspace_bytes(const sce_desc* desc, int B, int L) {
  if (validate(desc) || B < 1 || B > desc->batch_max || !frag_len_ok(L) || B % L || !plan_config(*desc).evaluable) return 0;
  return frag_workspace(*desc, B, L, nullptr, nullptr);
}

int sce_forward_fragments(sce_plan* p, const float* x, int B, int L, long long frag0, int n_top, int n_random,
                          unsigned long long seed, float* top_val, long long* top_frag, float* top_act,
                          long long* rnd_key, long long* rnd_frag, float* rnd_act, int* n_active, void* workspace,
                          size_t workspace_bytes, void* stream) {
  TRY(check_forward_only(p, x, B, "forward_fragments: "));
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
  const sce_desc& d = p->d;
  PlanCall call;
  TRY(run_pipeline(call, p, x, B, static_cast<cudaStream_t>(stream), nullptr, false, nullptr, nullptr));
  p->last_launches = call.count;   // the pipeline's: the fragment kernels below are not counted
  uint8_t* ws = static_cast<uint8_t*>(workspace);
  float* fmax = reinterpret_cast<float*>(ws);
  uint8_t* active = ws + off_active;
  int* open = reinterpret_cast<int*>(ws + off_open);
  const int n_chunks = (d.n + 31) / 32, G = B / L;
  const FragCode c{p->c.hi, p->c.lo, p->c.x8, p->scores, p->act_pos, n_chunks, d.batch_max, d.n};
  if (p->cfg.topk)
    TRY((launch_fragments<kArithBf16x3, true>(call, c, d.n_models, L, G, frag0, fmax, active, n_top, n_random, seed,
                                              top_val, top_frag, top_act, rnd_key, rnd_frag, rnd_act)));
  else
    TRY(with_arith(p->cfg.arith, [&](auto ar) {
      return launch_fragments<decltype(ar)::value, false>(call, c, d.n_models, L, G, frag0, fmax, active, n_top, n_random,
                                                          seed, top_val, top_frag, top_act, rnd_key, rnd_frag, rnd_act);
    }));
  // active fragments: segments of L rows, cut at fragment boundaries (phase 0, no segment stays open)
  CUDA_TRY(cudaMemsetAsync(open, 0, (size_t)d.n_models * d.n * sizeof(int), call.st));
  return call.launch(segment_count_kernel, dim3(n_chunks, d.n_models), 256, 0, p->act_pos, n_chunks, d.batch_max, B, d.n,
                     L, 0, n_active, open);
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
  Launcher L{st};
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
  bool f8 = arith == SCE_ARITH_F16F8 || (arith == SCE_ARITH_AUTO && env_arith() == SCE_ARITH_F16F8 && d % 16 == 0);
  const bool raw = !A.normalize || (!b_is_a && !B.normalize);
  SimCarve w;
  if (f8 && raw) {
    sim_carve(static_cast<uint8_t*>(workspace), true, ma, na, b_is_a ? 0 : mb, b_is_a ? 0 : nb, d, n_pairs, capacity != nullptr, &w);
    CUDA_TRY(cudaMemsetAsync(w.flags, 0, kFlagWords * sizeof(uint32_t), st));
    int rc = SCE_OK;
    if (!A.normalize) rc = sim_planes<kArithF16F8>(L, A, d, w.a, w.flags);
    if (!rc && !b_is_a && !B.normalize) rc = sim_planes<kArithF16F8>(L, B, d, w.b, w.flags);
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
  return f8 ? run_similarity_t<kArithF16F8>(L, A, B, b_is_a, d, n_pairs, w, row_max, col_max, capacity, dev, sms)
            : run_similarity_t<kArithBf16x3>(L, A, B, b_is_a, d, n_pairs, w, row_max, col_max, capacity, dev, sms);
}

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
  Launcher L{static_cast<cudaStream_t>(stream)};
  const unsigned rows8 = (unsigned)((B + 7) / 8);
  if (d <= 128) return L.launch(synth_rows_kernel<1, false>, rows8, 256, 0, a);
  if (d <= 256) return L.launch(synth_rows_kernel<2, false>, rows8, 256, 0, a);
  if (d <= 512) return L.launch(synth_rows_kernel<4, false>, rows8, 256, 0, a);
  if (d <= 1024) return L.launch(synth_rows_kernel<8, false>, rows8, 256, 0, a);
  return L.launch(synth_rows_kernel<8, true>, (unsigned)B, 32 * ((d + 1023) / 1024), 0, a);
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
