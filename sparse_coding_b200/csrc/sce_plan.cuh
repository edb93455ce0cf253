// sce_plan.cuh — what the three translation units of the entry points that take an sce_plan share (internal): the plan
// and its configuration, workspace buffers, tensor maps and calls, the activity-count block of evaluation and tracking,
// and the functions of sce_plan.cu that sce_eval.cu and sce_track.cu call.
#pragma once
#include <map>

#include "sce_engine.cuh"

namespace sce {

// ------------------------------------------------------------------------------------------------
// per-feature activation counts (standard_metrics.py:305-308 `(c != 0).float().mean(0)` and :441-454
// `n_active_count += (c != 0).sum(0)`; "ever active" = count > threshold): column sums of the [c > 0] activity-mask
// plane over the batch rows. One block per (32-column chunk, model): every lane holds the mask word of one row, a
// ballot per bit position counts 32 rows at once. counts[model][32 chunk + j] += sum_r bit(31 - j) of
// pos[model][chunk][r], accumulated across calls so a held-out set can be streamed through in batches. Reads B words
// per block, coalesced (the plane is chunk-major); the dense code is never touched.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void active_count_block(const uint32_t* __restrict__ pos, int n_chunks, int batch_max, int B,
                                                   int n, int* __restrict__ counts, int chunk, int model) {
  __shared__ int red[8][32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint32_t* p = pos + ((long long)model * n_chunks + chunk) * batch_max;
  int mine = 0;   // lane j accumulates the count of column j of the chunk
  for (int r0 = warp * 32; r0 < B; r0 += 256) {
    const int r = r0 + lane;
    const uint32_t w = r < B ? __ldg(p + r) : 0u;
#pragma unroll
    for (int j = 0; j < 32; ++j) {
      const int c = __popc(__ballot_sync(0xffffffffu, (w >> (31 - j)) & 1u));
      if (lane == j) mine += c;
    }
  }
  red[warp][lane] = mine;
  __syncthreads();
  if (warp == 0) {
    int t = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) t += red[i][lane];
    const int col = chunk * 32 + lane;
    if (col < n) counts[(long long)model * n + col] += t;
  }
}

}  // namespace sce

// ------------------------------------------------------------------------------------------------
// plan
// ------------------------------------------------------------------------------------------------
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
  // x's are made by a transpose pass (batch_major); the epilogues that produce c and g write their copies besides the
  // row-major planes (EpiEncodeT / EpiDecodeT with T8), and dz's 8-bit planes exist only in that layout (EpiDcodeT<f16f8, true>).
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
  bool tall_tiles;     // decode and the native weight gradient run on kBMTall-row output tiles (f16f8, see plan_config)
  bool split_decode;   // separate accumulators for hi*hi and the cross terms in the decode GEMM (bf16x3)
  bool use_graph;      // replay the step as a CUDA graph
  bool nonneg;         // desc.encoder_nonneg: the dictionary rows are built from max(E, 0) (dict_rows_kernel<..., true>)
  float shift;         // desc.input_shift; non-zero: the batch split also writes x + shift, which the step reads
  bool linear;         // SCE_CODE_LINEAR: the encode epilogue keeps the signed code (EpiEncodeT<..., LINEAR = true>)
  bool raw_decoder;    // SCE_DECODER_RAW: the decoder's planes are split from it as given (prepare_dict)
  bool forward_only;   // either modifier: the training entry points refuse the plan
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

// One call of a plan: its launches, and the batch of B rows and its tensor maps (run_pipeline opens it)
struct PlanCall : Launcher {
  sce_plan* p;
  BatchMaps* maps;
  int B;
  float* row_part = nullptr;   // tracked steps: the decode epilogue's per-row partials of r^2 (EpiDecodeT<..., true>)
  // one GEMM of the plan. NATIVE (f16f8): the cross terms run on E5M2 wgmma, which needs K-major 8-bit maps (A_MN / B_MN
  // then describe the fp16 planes alone); K-major GEMMs always have them, the weight gradient where the plan keeps
  // batch-major copies.
  // BM: rows of the output tile (kBMTall where the plan takes tall tiles and the maps are built for them).
  template <class Epi, bool A_MN, bool B_MN, bool SPLIT_ACC, int AR, bool NATIVE = AR == kArithF16F8 && !A_MN, int BM = kBM,
            class... A>
  int gemm(const A&... args) {
    return launch_gemm_t<Epi, A_MN, B_MN, SPLIT_ACC, AR, NATIVE, BM>(*this, p->d.n_models, p->device, p->sms, args...);
  }
  // with sce_profile_begin: the event at the start of phase `idx` of this step (SCE_PHASE_COUNT: the step's end)
  void mark(int idx) {
    if (p->prof_on && p->prof_steps < kProfMaxSteps)
      cudaEventRecord(p->prof_ev[p->prof_steps * (SCE_PHASE_COUNT + 1) + idx], st);
  }
};

// Defined in sce_plan.cu. Hidden, as fail is: libsce's own, not exports.
__attribute__((visibility("hidden"))) int validate(const sce_desc* d);
__attribute__((visibility("hidden"))) PlanConfig plan_config(const sce_desc& d);
__attribute__((visibility("hidden"))) int check_rows(const sce_plan* p, int B, const char* prefix);
__attribute__((visibility("hidden"))) int check_evaluable(const sce_plan* p, const char* prefix);
__attribute__((visibility("hidden"))) int check_forward_code(const sce_plan* p, const char* prefix);
__attribute__((visibility("hidden"))) int check_trainable(const sce_plan* p, const char* prefix);
__attribute__((visibility("hidden"))) int run_pipeline(PlanCall& c, sce_plan* p, const float* x, int B, cudaStream_t st,
                                                       float* x_hat, bool backward, float* out_losses, float* out_nnz,
                                                       float* mom_part = nullptr, float* row_part = nullptr);
__attribute__((visibility("hidden"))) int step_impl(sce_plan* p, const float* x, int B, float* out_losses, float* out_nnz,
                                                    cudaStream_t st, float* row_part);
__attribute__((visibility("hidden"))) int prepare_dict(Launcher& L, const sce_plan* p);
