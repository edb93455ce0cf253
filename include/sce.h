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
  SCE_TIED = 0,   /* FunctionalTiedSAE.loss   (sae_ensemble.py:135-162); + coef_mask = FunctionalMaskedTiedSAE (:347-373) */
  SCE_UNTIED = 1, /* FunctionalSAE.loss       (sae_ensemble.py:53-78);   + coef_mask = FunctionalMaskedSAE     (:418-444) */
  SCE_TOPK = 2    /* TopKEncoder.loss         (topk_encoder.py:29-40) */
} sce_variant;

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
  int variant;          /* sce_variant */
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
 * called once before the first step and again whenever the caller modified the parameters itself. */
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
 * [M,B,d] fp32 if non-NULL and the same losses / nnz as sce_step, without touching parameters. */
int sce_forward(sce_plan* plan, const float* x, int B, float* x_hat, float* out_losses, float* out_nnz,
                void* stream);

/* Materialise the fp32 code tensor aux["c"] [M,B,n] of the most recent step/forward (compat path for callers
 * that really want the dense tensor the reference returns, ensemble.py:193). */
int sce_read_code(sce_plan* plan, int B, float* out_code, void* stream);

/* Materialise the fp32 parameter gradients of the most recent sce_grads call (parity tests). */
int sce_grads(sce_plan* plan, const float* x, int B, float* d_encoder, float* d_bias, float* d_decoder,
              float* out_losses, float* out_nnz, void* stream);

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
 *   random (priority, fragment) over the ACTIVE fragments (the activity mask has c > 0 on some row): the n_random
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
 * Deterministic (no atomics) and asynchronous on `stream`. */
size_t sce_fragments_workspace_bytes(const sce_desc* desc, int B, int L);
int sce_forward_fragments(sce_plan* plan, const float* x, int B, int L, long long frag0, int n_top, int n_random,
                          unsigned long long seed, float* top_val, long long* top_frag, float* top_act,
                          long long* rnd_key, long long* rnd_frag, float* rnd_act, int* n_active, void* workspace,
                          size_t workspace_bytes, void* stream);

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

#ifdef __cplusplus
}
#endif
#endif /* SCE_H_ */
