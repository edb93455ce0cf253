/* sce.h — C ABI of the H100-native ensemble sparse-autoencoder training engine (libsce.so).
 *
 * The reference (HoagyC/sparse_coding @ 69c5ae0) has no FFI layer: its boundary for this path is the Python
 * protocol DictSignature / FunctionalEnsemble (autoencoders/ensemble.py:15-22, 68-193). This library sits
 * UNDERNEATH that protocol: sparse_coding_b200.FunctionalEnsemble keeps the reference's Python surface and
 * forwards the arithmetic of `step_batch` to the entry points below through ctypes (see INTEGRATION.md for the
 * binding a maintainer of the reference would add).
 *
 * Conventions: plain pointers and sizes only (no torch types); device pointers are borrowed — the caller (torch)
 * owns parameters, optimiser moments and the workspace, which are updated IN PLACE exactly as
 * FunctionalEnsemble.step_batch does (ensemble.py:182-191); no device allocation and no C++ exception crosses
 * the ABI; every call returns 0 on success or a negative sce_status, with a thread-local message available from
 * sce_last_error(); work is enqueued asynchronously on the caller's CUDA stream (`stream` is a cudaStream_t
 * passed as void*); calls on different plans are re-entrant, calls on the same plan are not thread-safe.
 */
#ifndef SCE_H_
#define SCE_H_

#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

/* 201 also covers the additive extension for FunctionalTiedCenteredSAE: the enum value SCE_TIED_LEARNED_CENTER, the
 * center / center_m / center_v fields appended to sce_buffers, and sce_read_center_grad. Nothing earlier moved, so a
 * caller built against the earlier 201 header keeps working unchanged.
 * 201 also covers the additive extension for FunctionalPositiveTiedSAE: encoder_nonneg and input_shift appended to the
 * descriptor struct; the signature is SCE_TIED plus these two fields, as the masked variants are SCE_TIED plus coef_mask.
 * Zero in both is the earlier behaviour. Unlike the extension above, this one lengthens the descriptor, and the library
 * reads both fields: a caller compiled against the earlier 201 header passes a shorter struct and must be rebuilt (with
 * the two fields zeroed) before it uses this library.
 * 201 also covers the additive entry points sce_second_moments_workspace_bytes / sce_second_moments (BatchedPCA). They
 * are plan-less and change nothing above. So are sce_ica_pass_workspace_bytes / sce_ica_pass (ICAEncoder), added
 * under 201 as well, and the NMF entry points sce_nmf_project, sce_nmf_grams, sce_nmf_residual and sce_nmf_cd_sweep
 * with their *_workspace_bytes queries (NMFEncoder).
 * 201 also covers the additive dead-feature tracking entry points sce_track_workspace_bytes, sce_step_tracked and
 * sce_resample with the struct sce_track they take. sce_step and every other entry point are unchanged, and a plan that
 * never sees sce_step_tracked launches exactly the kernels it did before.
 * 201 also covers the forward-only modifiers SCE_CODE_LINEAR and SCE_DECODER_RAW, or'ed into desc.variant of an SCE_UNTIED
 * plan (ICAEncoder, RandomDict). They live in bits the variant word never used, so the descriptor keeps its layout and a
 * caller built against the earlier 201 header keeps working unchanged.
 * 201 also covers the additive entry points sce_forward_split_workspace_bytes / sce_forward_split (the top- and
 * rest-feature FVU) and the constant SCE_SPLIT_MAX_TOP. Every other entry point is unchanged.
 * 201 also covers the additive entry points sce_interference_workspace_bytes / sce_code_interference and
 * sce_expected_interference_workspace_bytes / sce_expected_interference (the expected interference).
 * 201 also covers the additive entry points sce_cross_moments_workspace_bytes / sce_cross_moments and
 * sce_correlation_finish (the correlation of two dictionaries' codes). Every other entry point is unchanged. */
#define SCE_VERSION 201 /* major*10000 + minor*100 + patch */

typedef enum sce_status {
  SCE_OK = 0,
  SCE_ERR_INVALID = -1,    /* bad argument / unsupported shape */
  SCE_ERR_CUDA = -2,       /* a CUDA runtime or driver call failed */
  SCE_ERR_WORKSPACE = -3,  /* workspace too small / misaligned */
  SCE_ERR_NO_DEVICE = -4   /* no sm_90 device / driver entry point missing */
} sce_status;

/* Which reference signature the plan reproduces. */
typedef enum sce_variant {
  SCE_TIED = 0,   /* FunctionalTiedSAE.loss   (sae_ensemble.py:135-162); + coef_mask = FunctionalMaskedTiedSAE (:347-373);
                     + desc.encoder_nonneg = 1, input_shift = 0.18 = FunctionalPositiveTiedSAE (mlp_tests.py:68-125) */
  SCE_UNTIED = 1, /* FunctionalSAE.loss       (sae_ensemble.py:53-78);   + coef_mask = FunctionalMaskedSAE     (:418-444) */
  SCE_TOPK = 2,   /* TopKEncoder.loss         (topk_encoder.py:29-40) */
  SCE_TIED_LEARNED_CENTER = 3 /* FunctionalTiedCenteredSAE.loss, sae_ensemble.py:204-230: tied, on x - center[m] with the
                                 centre a trained parameter (sce_buffers.center). x_per_model only says how the caller's
                                 batch is laid out: the plan always holds M centred batches. No bias decay; needs
                                 desc.centering = 0. */
} sce_variant;

/* Forward-only modifiers of SCE_UNTIED, or'ed into desc.variant (desc.variant & 0xff is the variant). A plan with either is
 * a scoring plan for a baseline dictionary, not a training plan: sce_step, sce_step_host, sce_grads, sce_step_tracked and
 * sce_resample return SCE_ERR_INVALID before any device call; sce_forward, sce_forward_stats, sce_forward_fragments,
 * sce_read_code and sce_active_counts run. Any other bit, or either bit with another variant, is SCE_ERR_INVALID.
 *   SCE_CODE_LINEAR  the code is c = x E^T + b with no clamp (ICAEncoder's signed code; autoencoders/ica.py). Masked and
 *                    padding columns are 0. The activity mask is [c != 0] (no [z == 0] plane is written), so out_nnz is
 *                    the mean count of c != 0 per row, sce_active_counts and the segment counts count rows / segments on
 *                    which c != 0, and the moment sums of sce_forward_stats are those of the signed c. l_l1 is 0 (give
 *                    l1_alpha = NULL). sce_forward_fragments takes each fragment's maximum of the signed code, which may be
 *                    negative, and calls a fragment active where c != 0 on some row of it.
 *   SCE_DECODER_RAW  the decoder's operand planes are split from sce_buffers.decoder as given, without row normalisation
 *                    (RandomDict decodes with its raw rows; learned_dict.py:107-127). Under F16F8 a decoder entry fp16 cannot
 *                    hold sets the health word, as an out-of-range batch does, and counts in sce_input_absmax. */
enum { SCE_CODE_LINEAR = 1 << 8, SCE_DECODER_RAW = 1 << 9 };

/* How the Adam step counter behaves (SURVEY.md Q2). */
typedef enum sce_adam_count {
  SCE_ADAM_FROZEN_T1 = 0, /* the reference: step_batch drops torchopt's incremented count (ensemble.py:185-189) */
  SCE_ADAM_STANDARD = 1   /* bias correction with the true step number */
} sce_adam_count;

/* How an fp32 GEMM operand is carried to the tensor cores (DESIGN.md section 2). Both reach the reference's fp32
 * results within the 1e-4 bar; they differ in cost and in the range of values they can hold.
 *   BF16X3: x = hi + lo, two bf16 planes; product = hi*hi + hi*lo + lo*hi, three bf16 passes. fp32 range.
 *   F16F8 : x = h + l, h = fp16(x); the dominant h*h runs as one fp16 pass, the two cross terms (which need
 *           ~3 significant bits) are carried on E5M2 planes (1 byte each) and run as two E5M2 passes (in the weight
 *           gradient of top-k and launch-bound plans, widened to fp16 for two fp16 passes).
 *           Operand values must fit fp16 (|v| < 65504; magnitudes below ~1e-4 lose relative precision) — true for
 *           language-model activations, which the reference itself stores as fp16 (activation_dataset.py:294-299, 364, 404-412).
 *           Needs d % 16 == 0 and n % 16 == 0.
 *   AUTO  : F16F8 when the shape allows it, else BF16X3 (env SCE_ARITH=bf16x3|f16f8 overrides AUTO). */
typedef enum sce_arith { SCE_ARITH_AUTO = 0, SCE_ARITH_BF16X3 = 1, SCE_ARITH_F16F8 = 2 } sce_arith;

/* Static description of one stacked ensemble (FunctionalEnsemble.__init__, ensemble.py:69-97). */
typedef struct sce_desc {
  int variant;          /* sce_variant, with SCE_UNTIED optionally or'ed with SCE_CODE_LINEAR / SCE_DECODER_RAW */
  int n_models;         /* M: models stacked on dim 0 */
  int d;                /* activation width, multiple of 8 */
  int n;                /* dictionary rows (stack size for masked variants), multiple of 8 */
  int batch_max;        /* largest batch this plan will see (the last batch of a chunk may be shorter, Q7) */
  int x_per_model;      /* 0: one [B,d] batch shared by all models (expand_dims=True); 1: [M,B,d] */
  float lr, beta1, beta2, eps, eps_root; /* torchopt.adam hyper-parameters */
  int adam_count_mode;  /* sce_adam_count */
  int fwd_passes;       /* 3: split operands (~fp32 accuracy; default), 1: the 16-bit plane only (bf16 or fp16) */
  int bwd_passes;       /* same for the three backward GEMMs */
  float norm_floor;     /* clamp floor of the row norms: 1e-8 (SAE variants); <= 0 disables it (TopK) */
  int arith;            /* enum sce_arith; 0 = AUTO */
  int topk_k_max;       /* SCE_TOPK: the largest buffers["sparsity"] of the ensemble (1..256) enables the k-sparse decode /
                           code-gradient kernels; 0 = unknown: dense GEMMs on the k-sparse code, as the reference does */
  int centering;        /* FunctionalTiedSAE.center (sae_ensemble.py:126-128) applied to the batch on the device:
                           x_c[m] = (rot[m] (x - trans[m])) * scale[m]. 0 = off (identity centring); 1 = the batch is one
                           [B,d] array shared by all models; 2 = [M,B,d]. Needs x_per_model = 1 (the centred batch differs per
                           model) and the three center_* buffers. */
  int encoder_nonneg;   /* SCE_TIED only, 0 or 1. 1: the dictionary is built from the encoder clamped at 0,
                           W = max(E, 0) / max(||max(E, 0)||, norm_floor) (mlp_tests.py:100-102). The encoder gradient is
                           the one with respect to max(E, 0), applied to E without an [E >= 0] mask (straight-through, as
                           the reference's loss gives it); Adam updates the raw E, so negative entries keep moving. */
  float input_shift;    /* SCE_TIED only; not with centering. Non-zero: the plan encodes and reconstructs x + input_shift
                           (fp32 add, once per step on the batch as the caller laid it out; mlp_tests.py:104, :110), so
                           the f16f8 range checks judge the shifted values and sce_forward's x_hat is in the shifted
                           space (x_hat - input_shift reconstructs x). Neither field is allowed with coef_mask, nor in
                           sce_forward_stats / sce_forward_fragments (exports of such dictionaries are plain TiedSAE
                           objects of the raw encoder, evaluated as such). */
} sce_desc;

/* Device pointers owned by the caller; all fp32 unless noted. Unused ones are NULL. */
typedef struct sce_buffers {
  float* encoder;       /* [M,n,d]  params["encoder"] (tied/untied) or params["dict"] (topk) */
  float* encoder_bias;  /* [M,n]    params["encoder_bias"]; NULL for topk */
  float* decoder;       /* [M,n,d]  params["decoder"]; untied only */
  float* encoder_m;     /* Adam first moment of encoder, same shape; likewise below */
  float* encoder_v;
  float* bias_m;
  float* bias_v;
  float* decoder_m;
  float* decoder_v;
  const float* l1_alpha;          /* [M]   buffers["l1_alpha"]; NULL = 0 (topk) */
  const float* bias_decay;        /* [M]   buffers["bias_decay"]; NULL = 0 */
  const unsigned char* coef_mask; /* [M,n] buffers["coef_mask"] (1 = unused coefficient) or NULL */
  const long long* sparsity;      /* [M]   buffers["sparsity"] (topk k) or NULL */
  void* workspace;                /* >= sce_workspace_bytes(desc), 1024-byte aligned */
  size_t workspace_bytes;
  const float* center_trans;      /* [M,d]   buffers["center_trans"]  (desc.centering != 0; else NULL) */
  const float* center_rot;        /* [M,d,d] buffers["center_rot"]    */
  const float* center_scale;      /* [M,d]   buffers["center_scale"]  */
  float* center;                  /* [M,d]   params["center"] (SCE_TIED_LEARNED_CENTER; else NULL), updated in place by
                                             sce_step like the other parameters */
  float* center_m;                /* its Adam moments, same shape */
  float* center_v;
} sce_buffers;

typedef struct sce_plan sce_plan;

/* Loss columns written by sce_step: out_losses[m*SCE_LOSS_COLS + k]. */
enum { SCE_LOSS_TOTAL = 0, SCE_LOSS_RECONSTRUCTION = 1, SCE_LOSS_L1 = 2, SCE_LOSS_BIAS_DECAY = 3, SCE_LOSS_COLS = 4 };

int sce_version(void);
const char* sce_last_error(void);

/* Bytes of device scratch a plan needs (operand planes — 4 bytes per element — of the dictionary, the batch, the code, the
 * residual and the code gradient; fp32 weight gradients; reduction partials). */
size_t sce_workspace_bytes(const sce_desc* desc);

/* Builds the TMA descriptors and kernel launch plan. Does not touch device memory. */
int sce_plan_create(const sce_desc* desc, const sce_buffers* buffers, sce_plan** out_plan);
int sce_plan_destroy(sce_plan* plan);

/* (Re)derive the normalised operand planes of the dictionaries from the fp32 parameters. Must be
 * called once before the first step and again whenever the caller modified the parameters itself.
 * SCE_TOPK: also reads the sparsity buffer and returns SCE_ERR_INVALID when some k lies outside [1, n] or, with
 * topk_k_max in 1..256, above topk_k_max (a larger k needs a new plan). */
int sce_prepare(sce_plan* plan, void* stream);

/* One optimisation step for all M models on one batch == FunctionalEnsemble.step_batch (ensemble.py:175-193):
 * forward, losses, backward, Adam, in-place parameter update.
 *   x          device fp32, [B,d] (x_per_model = 0) or [M,B,d]
 *   out_losses device fp32 [M, SCE_LOSS_COLS]
 *   out_nnz    device fp32 [M]: mean over the batch of count_nonzero(c, -1)  (big_sweep.py:171)            */
int sce_step(sce_plan* plan, const float* x, int B, float* out_losses, float* out_nnz, void* stream);

/* Same step, fed from HOST memory the way the reference loop feeds it (big_sweep.py:168): copies `x_host`
 * (pinned or pageable fp32) to the device, steps, copies the [M,SCE_LOSS_COLS] losses and [M] nnz back, and
 * synchronises the stream before returning. */
int sce_step_host(sce_plan* plan, const float* x_host, int B, float* out_losses_host, float* out_nnz_host,
                  void* stream);

/* Forward only (evaluation; LearnedDict.predict semantics on already-centred inputs): writes x_hat
 * [M,B,d] fp32 if non-NULL and the same losses / nnz as sce_step, without touching parameters. SCE_TIED_LEARNED_CENTER:
 * x_hat is in the centred space (x_hat + center[m] is the reconstruction of x). desc.input_shift != 0: x_hat is in the
 * shifted space (x_hat - input_shift is the reconstruction of x). */
int sce_forward(sce_plan* plan, const float* x, int B, float* x_hat, float* out_losses, float* out_nnz,
                void* stream);

/* Materialise the fp32 code tensor aux["c"] [M,B,n] of the most recent step/forward (compat path for callers
 * that really want the dense tensor the reference returns, ensemble.py:193). */
int sce_read_code(sce_plan* plan, int B, float* out_code, void* stream);

/* Materialise the fp32 parameter gradients of the most recent sce_grads call (parity tests). */
int sce_grads(sce_plan* plan, const float* x, int B, float* d_encoder, float* d_bias, float* d_decoder,
              float* out_losses, float* out_nnz, void* stream);

/* SCE_TIED_LEARNED_CENTER: copy the gradient of params["center"] that the most recent sce_grads or sce_step computed,
 * d_center = sum_b g_b - db W (g = dL/dx_hat, db the bias gradient, W the normalised dictionary), to the device fp32
 * array d_center [M,d]. Asynchronous on `stream`. SCE_ERR_INVALID for the other variants. */
int sce_read_center_grad(sce_plan* plan, float* d_center, void* stream);

/* Split a row-gathered, optionally mean-centred batch out of a resident activation chunk:
 *   out[r,:] = float(chunk[idx[r],:]) - sub[:]      chunk fp16 or fp32 [N,d]; idx int64 [B] or NULL (identity)
 * (big_sweep.py:168 `dataset[batch_idxs]`, :359-364 centring) */
int sce_gather_rows(const void* chunk, int chunk_is_half, long long n_rows, int d, const long long* idx, int B,
                    const float* sub, float* out, void* stream);

/* Per-phase device timing of sce_step, measured with CUDA events recorded on the caller's stream between the
 * kernels of a step (bench.py's roofline). Between sce_profile_begin and sce_profile_end up to 64 steps are
 * recorded; sce_profile_end synchronises and returns the summed milliseconds of each phase. */
enum {
  SCE_PHASE_SPLIT = 0,  /* batch -> (hi, lo) */
  SCE_PHASE_ENCODE = 1, /* encode GEMM (+ top-k selection) */
  SCE_PHASE_DECODE = 2, /* decode GEMM + residual */
  SCE_PHASE_LOSSES = 3, /* bias norm + loss finalisation */
  SCE_PHASE_DCODE = 4,  /* code-gradient GEMM */
  SCE_PHASE_DW = 5,     /* weight-gradient GEMM(s) */
  SCE_PHASE_ADAM = 6,   /* Jacobian + Adam + renormalise + re-split, bias Adam */
  SCE_PHASE_COUNT = 7
};
int sce_profile_begin(sce_plan* plan);
int sce_profile_end(sce_plan* plan, float* phase_ms /*[SCE_PHASE_COUNT]*/, int* steps_recorded);

/* Optimiser step counter (number of sce_step calls so far); settable so a resumed run keeps the bias correction
 * of SCE_ADAM_STANDARD continuous. */
long long sce_get_step_count(const sce_plan* plan);
int sce_set_step_count(sce_plan* plan, long long steps_taken);

/* Number of kernels the most recent sce_step / sce_forward on this plan launched. */
int sce_last_launch_count(const sce_plan* plan);

/* F16F8 plans: the largest |x| over every batch fed since the last sce_prepare (NaN if a batch held one), read back
 * with one 4-byte copy and a stream synchronise — a monitor for the fp16 range the arithmetic assumes (values beyond
 * 65504 become inf/NaN in the losses, magnitudes far below 1e-3 lose relative precision: use SCE_ARITH_BF16X3 for
 * such data). BF16X3 plans report 0. */
int sce_input_absmax(sce_plan* plan, float* out_host, void* stream);

/* Health of the run. *bad_out = 1 when some step since the last sce_prepare / sce_clear_health saw a batch the fp16
 * operand plane cannot hold (F16F8: |x| >= 65520 or NaN) or produced a non-finite loss. From that step on the Adam
 * kernels leave parameters, moments and operand planes UNTOUCHED (the update is skipped on the device, so a bad chunk
 * cannot write NaN into the caller's tensors before the host looks); the caller decides: raise, or rebuild the plan
 * with SCE_ARITH_BF16X3. *absmax_out as sce_input_absmax. One 512-byte copy and a stream synchronise. */
int sce_health(sce_plan* plan, int* bad_out, float* absmax_out, void* stream);
int sce_clear_health(sce_plan* plan, void* stream);

/* Per-feature activation counts of the most recent step / forward: counts[m][j] += number of the B rows whose code
 * c[m, r, j] is non-zero (device int32 [M, n], ACCUMULATED so that a held-out set can be streamed through in batches).
 * This is the reference's `(c != 0).sum(0)` (standard_metrics.py:441-454, "features ever active" = count > threshold)
 * and, divided by the rows, its `(c != 0).float().mean(0)` (:305-308). Reads only the activity-mask plane the encode
 * epilogue / top-k selection wrote (B/8 bytes per feature chunk): the dense code is never materialised. */
int sce_active_counts(sce_plan* plan, int B, int* counts, void* stream);

/* Evaluation of a set of activations (standard_metrics.py:305-314 fraction_variance_unexplained /
 * mean_nonzero_activations, :446-454 batched_calc_feature_n_ever_active, :482-511 calc_moments_streaming): sce_forward,
 * plus per-feature statistics of the code c [M,B,n], without ever materialising it.
 *   moment_sums  device fp64 [M,n,4], ACCUMULATED: += sum over the B rows of c, c^2, c^3, c^4 per feature. The encode
 *                epilogue (SAE variants) or a pass over the top-k scores and activity mask (TOPK) sums 32 rows in fp32 from
 *                the exact fp32 code; those partials are added over the rows in a fixed order in fp64: bitwise repeatable.
 *   seg_counts   device int32 [M,n], ACCUMULATED: += number of segments of `seg` rows, ending in this call, in which the
 *                feature is non-zero on some row. seg = 1: rows, exactly as sce_active_counts.
 *   seg_phase    rows of the first segment that earlier calls already saw, in [0, seg)
 *   seg_open     device int32 [M,n] (seg > 1; may be NULL for seg = 1): 1 where the feature fired in the segment that
 *                is still open; read at the start, written at the end, so a segment may span any number of calls
 *                (zero it before the first call)
 *   workspace    >= sce_forward_stats_workspace_bytes(desc, B), 1024-byte aligned: the moment partials,
 *                M * ceil(B/32) * 4 * n fp32 (config 2, M = 16, n = 4096, B = 8192: 256 MiB; M = 1, n = 32768,
 *                B = 4096: 64 MiB). sce_forward_stats_workspace_bytes is host-only; it returns 0 for an invalid
 *                desc or B outside [1, batch_max].
 * Not available for SCE_TIED_LEARNED_CENTER (the size query returns 0, the call SCE_ERR_INVALID): evaluate its exported
 * dictionaries, which are TiedSAE objects with the centre as their translation. Nor with desc.encoder_nonneg or
 * desc.input_shift set (likewise): evaluate the exported TiedSAE of the raw encoder.
 * x_hat, out_losses and out_nnz are those of sce_forward (x_hat optional). Asynchronous on `stream`. */
size_t sce_forward_stats_workspace_bytes(const sce_desc* desc, int B);
int sce_forward_stats(sce_plan* plan, const float* x, int B, int seg, int seg_phase, float* x_hat, float* out_losses,
                      float* out_nnz, double* moment_sums, int* seg_counts, int* seg_open, void* workspace,
                      size_t workspace_bytes, void* stream);

/* Record selection for reading what features mean (interpret.py:82-212 make_feature_activation_dataset, :265-321
 * interpret): sce_forward on B rows cut into B / L fragments of L consecutive rows (fragment frag0 + g is rows
 * g L .. g L + L - 1 of this call), then, per model m and feature j, two lists that ACCUMULATE over calls:
 *   top    (fragment maximum max_t c[m, gL + t, j], fragment) over every fragment: the n_top largest by
 *          (maximum descending, fragment ascending)
 *   random (priority, fragment) over the ACTIVE fragments (the activity mask has c > 0 on some row; c != 0 with
 *          SCE_CODE_LINEAR, whose maxima start at -inf and may be negative): the n_random
 *          largest by (priority descending, fragment ascending), priority = splitmix64(splitmix64(splitmix64(seed) ^ j)
 *          ^ fragment) >> 1 — a uniform draw without replacement that depends on nothing but (seed, j, fragment)
 * The code values are those the engine holds: the joined operand planes (as sce_read_code) for the SAE variants,
 * relu(score) under the activity mask for TOPK; the maximum is taken over the same values, so top_val equals the
 * maximum of its top_act row bitwise.
 *   L            fragment length: a multiple of 32 in [32, 8192], dividing B
 *   frag0        index of this call's first fragment (>= 0); the fragments of a pass must be distinct
 *   n_top, n_random  list lengths in [0, 64], not both 0
 *   top_val      device fp32  [M,n,n_top]  \  the lists, in no particular order within a list: sort each by the order
 *   top_frag     device int64 [M,n,n_top]   | above after the last call. Initialise every *_frag entry to -1 (an
 *   rnd_key      device int64 [M,n,n_random]| empty entry, below every other) before the first call; the values and
 *   rnd_frag     device int64 [M,n,n_random]/ keys of empty entries are never read. NULL when the list length is 0.
 *   top_act, rnd_act  device fp32 [M,n,n_top,L] / [M,n,n_random,L] or NULL: entry i's L code values, written when a
 *                fragment enters the list at position i
 *   n_active     device int32 [M,n], ACCUMULATED: += the active fragments of this call (segment counts of
 *                sce_forward_stats with seg = L)
 *   workspace    >= sce_fragments_workspace_bytes(desc, B, L), 1024-byte aligned: fragment maxima and activity flags,
 *                M (B/L) n (4 + 1) bytes, and M n int32 (config 2, M = 16, n = 4096, B = 8192, L = 64: 40 MiB).
 *                sce_fragments_workspace_bytes is host-only; it returns 0 for an invalid desc, B outside
 *                [1, batch_max] or an invalid L.
 * Not available for SCE_TIED_LEARNED_CENTER, nor with desc.encoder_nonneg or desc.input_shift, as sce_forward_stats.
 * Deterministic (no atomics) and asynchronous on `stream`. */
size_t sce_fragments_workspace_bytes(const sce_desc* desc, int B, int L);
int sce_forward_fragments(sce_plan* plan, const float* x, int B, int L, long long frag0, int n_top, int n_random,
                          unsigned long long seed, float* top_val, long long* top_frag, float* top_act,
                          long long* rnd_key, long long* rnd_frag, float* rnd_act, int* n_active, void* workspace,
                          size_t workspace_bytes, void* stream);

/* The top- and rest-feature reconstruction errors (standard_metrics.py:316-342 fraction_variance_unexplained_top_activating):
 * sce_forward on B rows, then, per model m, with T_m = top_cols[m] (n_top chosen features), t = the decode of the code
 * restricted to T_m (sum over s of c[m, r, T_m[s]] times dictionary row T_m[s], normalised as the plan normalises it:
 * tied and untied with the norm floor, TOPK without, SCE_DECODER_RAW as given) and x_hat the plan's reconstruction:
 *   sq_top[m]   device fp64 [M], ACCUMULATED: += sum over the B rows and d columns of (x - t)^2
 *   sq_rest[m]  device fp64 [M], ACCUMULATED: += sum of (x - (x_hat - t))^2, the decode of the code without T_m
 * with x the batch as the plan reads it ([B,d], or [M,B,d] with x_per_model). Both are fp32 partials per 32 rows, added
 * in a fixed order in fp64: bitwise repeatable. The dense code is never formed.
 *   n_top       1 .. SCE_SPLIT_MAX_TOP
 *   top_cols    device int32 [M, n_top]: distinct columns in [0, n) per model. They are copied to the host and checked
 *               before any launch, so the call synchronises `stream` once.
 *   x_hat       optional device fp32 [M,B,d]: sce_forward's reconstruction (else it is kept in the workspace)
 *   x_hat_top   optional device fp32 [M,B,d]: t
 * Centred plans (desc.centering != 0) reconstruct the centred batch, so the sums above are not the reference's (which
 * compares center(t) and center(x_hat - t) with the raw batch): they need x_hat and x_hat_top and leave sq_top / sq_rest
 * untouched (they may be NULL), and the caller forms the residuals. Every other plan needs sq_top and sq_rest.
 *   workspace   >= sce_forward_split_workspace_bytes(desc, B, n_top), 1024-byte aligned: x_hat, the chosen code columns
 *               and dictionary rows, and the partials, M (B d + B n_top + n_top d + 2 ceil(B/32)) fp32 (config 2, M = 16,
 *               d = 512, B = 8192, n_top = 2: 257 MiB). Host-only; returns 0 for an invalid desc, B outside [1, batch_max],
 *               n_top outside [1, SCE_SPLIT_MAX_TOP] or n_top > n.
 * Not available for SCE_TIED_LEARNED_CENTER, nor with desc.encoder_nonneg or desc.input_shift, as sce_forward_stats.
 * Asynchronous on `stream` after the check of top_cols. */
#define SCE_SPLIT_MAX_TOP 64
size_t sce_forward_split_workspace_bytes(const sce_desc* desc, int B, int n_top);
int sce_forward_split(sce_plan* plan, const float* x, int B, int n_top, const int* top_cols, double* sq_top,
                      double* sq_rest, float* x_hat, float* x_hat_top, void* workspace, size_t workspace_bytes,
                      void* stream);

/* Expected interference (big_sweep.py:43-57 calc_expected_interference), per model m, of the code c [B, n] of the plan's
 * LAST sce_forward / sce_forward_stats call (its B rows) and the dictionary the plan decodes with (tied and top-k: the
 * encoder, untied: the decoder), as stored. With W_i = row i / max(||row i||, 1e-8) for every kind (whatever the plan's
 * own decode normalises; SURVEY Q15) and A_r = {j : c[r, j] != 0}:
 *   totals[r, i] = sum over j in A_r of (W_i . W_j)^2 c[r, j]      (fp32 FMA dot products)
 *   cap[r, i]    = c[r, i] / max(totals[r, i], 1e-8)                 (i in A_r; 0 elsewhere)
 *   cap_sums[m]  device fp64 [M, n], ACCUMULATED: += sum over the B rows of cap[r, j]
 *   nz_counts[m] device int64 [M, n], ACCUMULATED: += number of rows with c[r, j] != 0
 * The reference's result is cap_sums / max(nz_counts, 1) over all rows. Only the Gram of each row's active dictionary
 * rows is formed (O(|A_r|^2 d) per row, the active set tiled 64 at a time, any size up to n); the [n, n] cosine matrix
 * never is. Per-feature partials of 32 rows are added in a fixed order in fp64: bitwise repeatable.
 *   workspace   >= sce_interference_workspace_bytes(desc, B), 1024-byte aligned: the normalised dictionary and the
 *               partials, M (n ceil(d / 32) 32 + 2 n ceil(B / 32)) fp32 (config 2, M = 16, n = 4096, d = 512, B = 8192:
 *               256 MiB). Host-only; returns 0 for an invalid desc or B outside [1, batch_max].
 * Not available for SCE_TIED_LEARNED_CENTER, nor with desc.encoder_nonneg or desc.input_shift, as sce_forward_stats.
 * Refuses a plan whose last call was a training step, as sce_cross_moments does.
 * Asynchronous on `stream`. */
size_t sce_interference_workspace_bytes(const sce_desc* desc, int B);
int sce_code_interference(sce_plan* plan, int B, double* cap_sums, long long* nz_counts, void* workspace,
                          size_t workspace_bytes, void* stream);

/* The same for a caller-held code, without a plan: dict device fp32 [n, d], code device fp32 [B, n] (any n, d >= 1),
 * cap_sums device fp64 [n] and nz_counts device int64 [n], ACCUMULATED. The workspace (>= the query's bytes, 1024-byte
 * aligned) grows with B; call once per slice of rows to bound it. The query returns 0 for n, d or B < 1. */
size_t sce_expected_interference_workspace_bytes(int n, int d, int B);
int sce_expected_interference(const float* dict, int n, int d, const float* code, int B, double* cap_sums,
                              long long* nz_counts, void* workspace, size_t workspace_bytes, void* stream);

/* Cross-code moments of two plans (inter_dict_connections.ipynb's covariance cell): after a sce_forward_stats call of
 * each plan on the same B paired rows (row r of plan_a's batch paired with row r of plan_b's), for every model pair
 * (i, j), with C_a[i] [B, n_a] and C_b[j] [B, n_b] the codes those calls left in the plans,
 *   acc[i][j][p][q]  device fp64 [M_a][M_b][n_a][n_b], ACCUMULATED: += sum over the B rows of C_a[i][r, p] C_b[j][r, q]
 * The operands are the code planes the plans hold (the dense code never reaches memory); the product runs on the weight
 * gradient's GEMM over slices of at most 2048 rows, each summed in fp32 on the tensor cores and added in fp64 in slice
 * order: bitwise repeatable. Padding columns of a plan (coef_mask) hold 0 and add 0. The per-feature sums and sums of
 * squares are the moment sums sce_forward_stats already made. plan_a may be plan_b.
 *   B            in [1, min(batch_max)]: the rows of both plans' last calls
 *   workspace    >= sce_cross_moments_workspace_bytes(plan_a, plan_b, B), 1024-byte aligned: one fp32 partial
 *                n_a n_b 4 bytes (n = 4096: 64 MiB). Host-only; returns 0 unless both plans are evaluable, resolved to the
 *                same arithmetic on the same device, and B fits both.
 * Not available for SCE_TIED_LEARNED_CENTER, nor with desc.encoder_nonneg or desc.input_shift, as sce_forward_stats;
 * nor after a training step (the call must follow sce_forward_stats). Asynchronous on `stream`. */
size_t sce_cross_moments_workspace_bytes(const sce_plan* plan_a, const sce_plan* plan_b, int B);
int sce_cross_moments(sce_plan* plan_a, sce_plan* plan_b, int B, double* acc, void* workspace, size_t workspace_bytes,
                      void* stream);

/* The correlation of one model pair from its fp64 sums over N = rows rows, without a plan: with mean = s1 / N,
 * var = s2 / N - mean^2 per feature and cov[p][q] = acc[p * lda + q] / N - mean_a[p] mean_b[q] (fp64),
 *   corr[p][q] = cov[p][q] / sqrt(var_a[p] var_b[q]), NaN unless both variances are > 0
 *   corr, cov      device fp32 [n_a][n_b], each optional (NULL: not written)
 *   max_ab[p], arg_ab[p]  device fp32 / int64 [n_a]: the largest corr[p][:] and its column; NaN entries are skipped, equal
 *                  values go to the lower index, and a row with no defined entry gets NaN and -1
 *   max_ba, arg_ba device fp32 / int64 [n_b]: the same over the columns corr[:][q]
 *   sums_a, sums_b device fp64 [n_a][4] / [n_b][4]: sce_forward_stats' moment sums of one model (s1, s2 read)
 *   lda            >= n_b: the row pitch of acc (a plan's padded n_b; only the first n_b columns are read)
 * The maxima are taken in fp64 over the values corr holds before rounding. Deterministic; asynchronous on `stream`. */
int sce_correlation_finish(const double* acc, int n_a, int n_b, int lda, const double* sums_a, const double* sums_b,
                           long long rows, float* corr, float* cov, float* max_ab, long long* arg_ab, float* max_ba,
                           long long* arg_ba, void* stream);

/* Dead-feature resampling (experiments/huge_batch_size.py:120-146 WorstIndices, :189-250 process_reinit), per model m,
 * over a WINDOW of tracked steps (the sce_step_tracked calls since the caller emptied the lists, or since sce_resample):
 *   e_r        mean over d of (x_hat - x)^2 for row r, in the space the plan reconstructs (centred, x - center[m],
 *              x + input_shift), from the same fp32 residuals whose sum is l_reconstruction
 *   list       the N rows of the window with the largest e, by (e descending, window serial ascending); an entry holds e,
 *              the row's serial (row number within the window) and a bitwise copy of the row of `x` as the caller passed
 *              it (x[m] when x_per_model, the shared row otherwise)
 *   counts     per feature, the rows of the window whose code is non-zero (as sce_active_counts)
 * A step whose update was skipped (the health word is set, see sce_health) enters nothing and counts nothing.
 * sce_track: caller-owned device arrays, kept between calls (start a window with filled and counts zeroed and
 * next_serial = 0):
 *   err [M,N] fp32, serial [M,N] int64, rows [M,N,d] fp32 (16-byte aligned): the lists, entries 0 .. filled[m] - 1
 *              valid, in no particular order
 *   filled [M] int32, counts [M,n] int32
 *   next_serial  window serial of this call's first row (the caller adds B after each call); next_serial + B must stay
 *              below 2^32 - 1
 *   n_worst    N, in [1, n]
 *   workspace  >= sce_track_workspace_bytes(desc, N), 1024-byte aligned: scratch of one call (nothing in it is kept).
 *              Host-only; 0 for an invalid desc or N. Config 2 (M = 16, B = 8192, d = 512, n = N = 4096): 7 MiB.
 * sce_step_tracked: sce_step, then one merge kernel (row errors from the decode epilogue's per-row partials or the top-k
 *   gather kernel's, the list merge as a radix select over 64-bit keys (e bits, inverted serial), the window's counts)
 *   and one kernel copying the entering rows. No host synchronisation, no atomics whose order matters: bitwise
 *   repeatable. The step itself computes exactly what sce_step computes; launch-bound plans run it without their CUDA
 *   graph.
 * sce_resample: for the dead features j_1 < j_2 < ... (count 0 over the window; masked padding, coef_mask = 1, is never
 *   dead) and the list sorted as above, v_1, v_2, ...: for i <= min(#dead, filled), row j_i of the dictionary parameter
 *   (encoder; dict for SCE_TOPK) becomes v_i * (ratio / mu), mu the mean L2 norm of the model's valid rows before the
 *   replacement (fp64, fixed order), and the Adam moments of that row of the encoder, of the decoder (untied) and of its
 *   bias entry become 0. Bias values, decoder rows, the centre, the step count, the health and range words and every
 *   other row stay as they are. The operand planes of the dictionary are re-derived as sce_prepare does. Writes
 *   n_dead[m], n_replaced[m] (device int32 [M]) and replaced (device uint8 [M,n], 1 = row replaced), then restarts the
 *   window on the device (filled and counts zeroed; the caller sets next_serial = 0).
 * Argument errors (NULL pointers, N outside [1, n], a small or misaligned workspace, misaligned rows) are reported
 * before any device call. Asynchronous on `stream`. */
typedef struct sce_track {
  float* err;
  long long* serial;
  float* rows;
  int* filled;
  int* counts;
  long long next_serial;
  int n_worst;
  void* workspace;
  size_t workspace_bytes;
} sce_track;
size_t sce_track_workspace_bytes(const sce_desc* desc, int n_worst);
int sce_step_tracked(sce_plan* plan, const float* x, int B, float* out_losses, float* out_nnz, const sce_track* track,
                     void* stream);
int sce_resample(sce_plan* plan, const sce_track* track, float ratio, int* n_dead, int* n_replaced,
                 unsigned char* replaced, void* stream);

/* The arithmetic the plan resolved to: SCE_ARITH_BF16X3 or SCE_ARITH_F16F8. */
int sce_plan_arith(const sce_plan* plan);

/* Dictionary similarity without a plan (standard_metrics.py:270-303 mmcs / mcs_duplicates / mcs_to_fixed /
 * representedness, :356-362 capacity_per_feature). For each pair q = (i, j) of `pairs` it forms S = A_i B_j^T on the
 * split-operand GEMM and keeps only reductions of it — the [na, nb] matrix never reaches memory:
 *   row_max[q][r] = max over valid atoms c of B_j of S[r, c]   (each atom of A_i: its best match in B_j)
 *   col_max[q][c] = max over valid atoms r of A_i of S[r, c]   (each atom of B_j: its best match in A_i)
 *   capacity[i][r] = S[r, r]^2 / sum_c S[r, c]^2             for the self-pairs (i, i); needs b == NULL
 * Entries of atoms beyond rows[m] are NaN; so is the capacity of a zero row (0 / 0, as in the reference).
 *   a, b        device fp32 [ma, na, d] / [mb, nb, d] stacks of dictionaries; b == NULL: B = A (mb, nb, b_* ignored)
 *   *_rows      HOST int32 [ma] / [mb]: valid atoms of each model (masked stacks export encoder[:dict_size]), each in
 *               [1, n]; NULL = all
 *   *_normalize 1: rows divided by max(||row||, floor) on the device (floor <= 0: no clamp — TopK), the
 *               get_learned_dict of the SAE and TopK signatures; 0: the matrix as given (a raw truth matrix)
 *   pairs       HOST int32 [n_pairs][2]: (model of A, model of B)
 *   arith       sce_arith. AUTO: BF16X3 (the faster and more accurate of the two on this GEMM; env SCE_ARITH=f16f8 pins
 *               AUTO to F16F8 where d % 16 == 0). Under F16F8 a raw operand fp16 cannot hold (|v| >= 65520 or NaN) is
 *               SCE_ERR_INVALID (a pinned AUTO runs it on BF16X3); finding out costs one 4-byte copy and a stream
 *               synchronise for calls with a raw operand.
 *   row_max, col_max, capacity  device fp32 outputs, each optional (at least one)
 *   workspace   >= sce_similarity_workspace_bytes(...), 1024-byte aligned: operand planes (4 B per element) and, with
 *               capacity, sum-of-squares partials [n_pairs][na][2 ceil(na / 128)] — never O(na nb).
 * Bitwise repeatable: maxima are exact, sums are reduced in a fixed order. Asynchronous on `stream` otherwise. */
size_t sce_similarity_workspace_bytes(int ma, int na, int mb /* 0: B = A */, int nb, int d, int n_pairs, int want_capacity);
int sce_similarity(const float* a, int ma, int na, const int* a_rows, float a_norm_floor, int a_normalize,
                   const float* b, int mb, int nb, const int* b_rows, float b_norm_floor, int b_normalize,
                   int d, const int* pairs, int n_pairs, int arith, float* row_max, float* col_max, float* capacity,
                   void* workspace, size_t workspace_bytes, void* stream);

/* Synthetic sparse-mixture rows (sc_datasets/random_dataset.py:191-245 generate_correlated_dataset, :160-188
 * generate_rand_dataset, :145-157 generate_noise_dataset with the identity covariance), without a dense code:
 *   active(i, j) = u_thresh(i, j) <= probs[i / group_rows][j]                      (a p > 1 is always on)
 *   coef(i, j)   = u_val(i, j) * u_strength(i, j)          in fp32, for the active j
 *   zero-row rule (zero_row_rule = 1): a row with no active component gets component z(i) with coef 1.0 * u_strength(i, z(i))
 *   out[i, :]    = fma(noise_scale, n(i, :), sum over active j, ascending, of coef(i, j) feats[j, :])   fp32 FMAs;
 *                  stored as fp32 (out_half = 0) or rounded to nearest fp16 (out_half = 1)
 *   feats        device fp32 [n_gt, d], row-major, 16-byte aligned; d a multiple of 8 in [8, 8192]; n_gt >= 1
 *   probs        device fp32 [ceil(B / group_rows), n_gt]: local row i belongs to group i / group_rows
 *   row0         global index of local row 0 (>= 0); every draw of local row i is keyed by the global row row0 + i
 *   out          device [B, d] fp32 or fp16, 16-byte aligned
 *   row_nnz      device int32 [B] or NULL: the number of active components of each row (1 for a zero-row fill)
 *   code_idx, code_val  device int32 / fp32 [B, code_cap] or both NULL: each row's active components in ascending j
 *                and their coef, the ground-truth code; entries beyond code_cap are dropped (row_nnz still counts them)
 * Random numbers: Philox4x32-10 with key (seed & 0xffffffff, seed >> 32) and counter (c0, global row & 0xffffffff,
 * global row >> 32, tag); a word x gives the uniform (x >> 8) 2^-24 in [0, 1).
 *   tag 0 threshold, 1 value, 2 strength: c0 = j / 4, word j % 4
 *   tag 3 zero-row component: c0 = 0, z(i) = (word 0 * n_gt) >> 32
 *   tag 4 noise: c0 = k / 4 for columns k .. k + 3 (k % 4 = 0); Box-Muller on the word pairs (0, 1) -> columns k, k + 1
 *         and (2, 3) -> k + 2, k + 3: u1 = ((a >> 8) + 1) 2^-24, u2 = (b >> 8) 2^-24, r = sqrt(-2 ln u1),
 *         n = (r cos 2 pi u2, r sin 2 pi u2)
 *   tag 5 is left to the caller for per-group Gaussians (with the group index in the row words; see
 *         sparse_coding_b200/synthetic.py), so that they never share a stream with a row's draws.
 * The active sets, coefficients, row_nnz and lists are therefore a function of (seed, global row, probs) alone, bitwise:
 * independent of the launch, of how rows are split over calls, and of the GPU. out is that function up to the rounding
 * of fp32 FMAs in a fixed order, deterministic run to run. Asynchronous on `stream`. */
int sce_synth_rows(const float* feats, int n_gt, int d, const float* probs, int group_rows, long long row0, int B,
                   unsigned long long seed, int zero_row_rule, float noise_scale, void* out, int out_half, int* row_nnz,
                   int* code_idx, float* code_val, int code_cap, void* stream);

/* Streaming second moments of shifted rows without a plan (autoencoders/pca.py:54-64 BatchedPCA.train_batch, as one Gram
 * matrix instead of a [B, d, d] outer-product tensor): for the B rows x_b of x and v_b = x_b - shift (fp32),
 *   col_sum[j]    += sum_b v_b[j]
 *   gram[i * d + j] += sum_b v_b[i] v_b[j]
 *   x            device [B, d] row-major, fp16 (x_is_half = 1, read as it is) or fp32; 16-byte aligned
 *   shift        device fp32 [d], 16-byte aligned (BatchedPCA: the first batch's column mean, so that the sums stay small
 *                against the offset of the data and the covariance needs no large cancellation)
 *   col_sum, gram  device fp64 [d] / [d, d] (gram 16-byte aligned), ACCUMULATED
 *   arith        sce_arith. AUTO: BF16X3 (the fp32 range, no range check), as sce_similarity. F16F8 needs d % 16 == 0.
 *   range_flag   device uint32 or NULL: F16F8 sets it to 1 when some v does not fit the fp16 plane (|v| >= 65520 or
 *                NaN); the sums are then not meaningful. The caller zeroes it.
 *   d            a multiple of 8 in [8, 8192];  B in [1, 2^21]
 *   workspace    >= sce_second_moments_workspace_bytes(d, B), 1024-byte aligned: the operand planes of the rows (6 B per
 *                element), the fp32 Gram partials of the row slices, S d^2 4 B, and the column-sum partials. Host-only;
 *                0 for invalid arguments. Never decreases with B, so a workspace sized for the longest call serves
 *                every shorter one.
 * The Gram matrix runs on the weight gradient's GEMM. The rows are cut into S slices of at most 2048 rows (S chosen from d
 * and B only), each slice's product is summed in fp32 on the tensor cores, and the slices are added in fp64 in slice order;
 * the column sums are fp64 from fp32 v. No atomics: results are bitwise repeatable. Asynchronous on `stream`. */
size_t sce_second_moments_workspace_bytes(int d, int B);
int sce_second_moments(const void* x, int x_is_half, int B, int d, const float* shift, int arith, double* col_sum,
                       double* gram, unsigned int* range_flag, void* workspace, size_t workspace_bytes, void* stream);

/* One data pass of FastICA's parallel update with the logcosh nonlinearity, without a plan (autoencoders/ica.py's
 * FastICA().fit, one iteration's two GEMMs): for the B rows x_b of x, v_b = x_b - shift and t_b = tanh(alpha unmix v_b),
 *   g_sum[i]        += sum_b alpha (1 - t_b[i]^2)
 *   gx[i * d + j]   += sum_b t_b[i] v_b[j]
 *   x            device [B, d] row-major, fp16 (x_is_half = 1) or fp32; 16-byte aligned
 *   shift        device fp32 [d], 16-byte aligned (ICAEncoder: the fp32 column mean)
 *   unmix        device fp32 [n, d] row-major, 16-byte aligned. ICAEncoder folds the whitening into it, unmix = W Kw, so
 *                that no whitened copy of the rows is written; gx Kw^T then is the whitened rows' G X1^T.
 *   alpha        in [1, 2] (sklearn's fun_args alpha)
 *   g_sum, gx    device fp64 [n] / [n, d] (gx 16-byte aligned), ACCUMULATED
 *   arith        sce_arith. AUTO: BF16X3 (the fp32 range, no range check). F16F8 needs d % 16 == 0 and n % 16 == 0.
 *   range_flag   device uint32 or NULL: F16F8 sets it to 1 when some v or some unmix entry does not fit the fp16 plane
 *                (|v| >= 65520 or NaN); the sums are then not meaningful. The caller zeroes it.
 *   d            a multiple of 8 in [8, 8192];  n a multiple of 8 in [8, d];  B in [1, 2^21]
 *   workspace    >= sce_ica_pass_workspace_bytes(d, n, B), 1024-byte aligned: the planes of v, of t and of unmix, the
 *                fp32 gx partials of the row slices (S n d 4 B) and the g' partials. Host-only; 0 for invalid arguments.
 *                Never decreases with B.
 * The rows are sliced as in sce_second_moments. U = V unmix^T runs on the encode GEMM, whose epilogue writes the planes
 * of t = tanhf(alpha U) (the accurate tanh) and fp32 partials of g' per 32 rows; gx runs on the weight gradient's GEMM per
 * slice. Partials are added in fp64 in a fixed order. No atomics: results are bitwise repeatable. Asynchronous on
 * `stream`. */
size_t sce_ica_pass_workspace_bytes(int d, int n, int B);
int sce_ica_pass(const void* x, int x_is_half, int B, int d, const float* shift, const float* unmix, int n, float alpha,
                 int arith, double* g_sum, double* gx, unsigned int* range_flag, void* workspace, size_t workspace_bytes,
                 void* stream);

/* NMF with sklearn's coordinate-descent solver (autoencoders/nmf.py's NMF().fit and transform), without a plan. For the B
 * rows x_b of x, v_b = max(x_b - shift, 0) (fp32; NaN stays NaN):
 *
 * sce_nmf_project: p[b * k + j] = sum_i m[j * d + i] v_b[i], fp32 [B, k] (transform's X H^T with m = H, or NNDSVD's
 * X V^T with m = the right singular vectors), and with norms (device fp64 [2][k], ACCUMULATED, or NULL)
 *   norms[j]     += sum_b max(p_bj, 0)^2,   norms[k + j] += sum_b min(p_bj, 0)^2
 * It runs on the encode GEMM; its epilogue stores p and fp32 partials of the norms per 32 rows, added in fp64 in row-block
 * order.
 *
 * sce_nmf_grams: for w [B, k] fp32 (rows of the codes W),
 *   wtw[i * k + j] += sum_b w_bi w_bj,   wtv[i * d + j] += sum_b w_bi v_b[j]     (device fp64, 16-byte aligned)
 * The rows are sliced as in sce_second_moments; both products run on the weight gradient's GEMM per slice, and the
 * slices are added in fp64 in slice order.
 *
 * For both:
 *   x            device [B, d] row-major, fp16 (x_is_half = 1, read as it is) or fp32; 16-byte aligned
 *   shift        device fp32 [d], 16-byte aligned
 *   m / w        device fp32, 16-byte aligned; p device fp32 [B, k], 16-byte aligned
 *   arith        sce_arith. AUTO: BF16X3. F16F8 needs d % 16 == 0 and k % 16 == 0.
 *   range_flag   device uint32 or NULL: F16F8 sets it to 1 when some v, m or w entry does not fit the fp16 plane
 *                (|v| >= 65520 or NaN); the results are then not meaningful. The caller zeroes it.
 *   d            a multiple of 8 in [8, 8192];  k a multiple of 8 in [8, d];  B in [1, 2^21]
 *   workspace    >= the matching *_workspace_bytes(d, k, B), 1024-byte aligned: the planes of the operands and the
 *                fp32 partials. Host-only; 0 for invalid arguments. Never decreases with B.
 *
 * sce_nmf_cd_sweep: coordinate-descent sweeps of sklearn's _update_cdnmf_fast (no regularisation, coordinates in order
 * 0 .. k-1) over the R rows of w [R, k] (in/out), with g [k, k] (HH^T or W^T W) and l [R, k] (XH^T or X^T W) fixed:
 *   for t in 0 .. k-1, per row i:  grad = sum_r g[t][r] w[i][r] - l[i][t];  pg = w[i][t] == 0 ? min(grad, 0) : grad;
 *   violation += |pg|;  if g[t][t] != 0: w[i][t] = max(w[i][t] - grad / g[t][t], 0)
 *   g            must be symmetric (H H^T and W^T W are in exact arithmetic; NMFEncoder symmetrises both): the kernel
 *                keeps the gradient as sum_r w[i][r] g[r][t] and so reads row t of g where the loop above names its
 *                column t
 *   w_is_f64     0: w, g and l are fp32 (NMFEncoder's W-update and transform), 1: fp64 (its H-update)
 *   k            in [1, 2048];  R >= 1
 *   n_iter NULL  one sweep (max_sweeps = 1): violation[0] (device fp64) += its violation
 *   n_iter       device int: transform's loop. violation[0..1] and n_iter are zeroed, then up to max_sweeps sweeps are
 *                queued; sweep s is a no-op once the stop rule held after sweep s - 1 (violation[0] == 0, or
 *                violation[1] / violation[0] <= tol), so n_iter ends as sklearn's iteration count, violation[0] as the
 *                first sweep's violation and violation[1] as the last one's. No host read.
 *   workspace    >= sce_nmf_cd_sweep_workspace_bytes(k, R), 1024-byte aligned: one fp64 partial per 8 rows.
 * One warp sweeps one row, with the row and its gradient in registers and rows of g staged in shared memory; a coordinate
 * whose step is zero costs no gradient update. Violations are fp64, added in a fixed order.
 * No atomics anywhere: results are bitwise repeatable. All three are asynchronous on `stream`. */
size_t sce_nmf_project_workspace_bytes(int d, int k, int B);
int sce_nmf_project(const void* x, int x_is_half, int B, int d, const float* shift, const float* m, int k, int arith,
                    float* p, double* norms, unsigned int* range_flag, void* workspace, size_t workspace_bytes,
                    void* stream);
size_t sce_nmf_grams_workspace_bytes(int d, int k, int B);
int sce_nmf_grams(const void* x, int x_is_half, int B, int d, const float* shift, const float* w, int k, int arith,
                  double* wtw, double* wtv, unsigned int* range_flag, void* workspace, size_t workspace_bytes,
                  void* stream);
/* sce_nmf_residual: sum[0] += sum_b ||v_b - w_b h||^2 (device fp64, ACCUMULATED) for w [B, k] and h [k, d], both fp32
 * and 16-byte aligned, with v_b as above (the fit's reconstruction_err_). A plain fp32 product on the CUDA cores, not the
 * split-operand GEMM: at a good fit the residual is a small fraction of the rows, which products good to 2^-16 would
 * not resolve. d, k and B as for sce_nmf_project; workspace >= sce_nmf_residual_workspace_bytes(d, B) (one fp64
 * partial per 64 x 64 tile), 1024-byte aligned. Squares are fp64, added in a fixed order. */
size_t sce_nmf_residual_workspace_bytes(int d, int B);
int sce_nmf_residual(const void* x, int x_is_half, int B, int d, const float* shift, const float* w, int k,
                     const float* h, double* sum, void* workspace, size_t workspace_bytes, void* stream);
size_t sce_nmf_cd_sweep_workspace_bytes(int k, int R);
int sce_nmf_cd_sweep(void* w, int w_is_f64, int R, int k, const void* g, const void* l, int max_sweeps, double tol,
                     double* violation, int* n_iter, void* workspace, size_t workspace_bytes, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* SCE_H_ */
