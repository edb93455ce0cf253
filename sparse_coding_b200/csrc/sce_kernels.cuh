// sce_kernels.cuh — the HBM-bound streaming kernels around the GEMMs of one training step:
// batch split, dictionary normalise+split, row-norm Jacobian + Adam + re-split, bias Adam,
// top-k selection, chunk row gather.
// Each is a single pass over its data with 16-byte accesses; algorithmic bytes per element are
// listed in DESIGN.md.
// Every translation unit of libsce.so includes this header, so every kernel here is a template: a kernel that is not
// one is defined in the one .cu that owns it (the loss finalisation, centre gradient and batch-major transpose of the
// training step: sce_plan.cu; the activity counts: sce_eval.cu), or each includer would define it again.
#pragma once
#include "sce_epilogues.cuh"

namespace sce {

// ------------------------------------------------------------------------------------------------
// batch split: x fp32 [rows, d] -> operand planes. bf16x3: (hi, lo) bf16. f16f8: fp16 plane `hi`, value-e5m2
// plane `lo` (1 B / element), residual-e5m2 plane `x8`.
// ------------------------------------------------------------------------------------------------
// Four consecutive values -> the operand planes at element offset 4 * i4 (shared by every producer of operands).
template <int ARITH>
__device__ __forceinline__ void store_planes4(const float (&v)[4], void* hi, void* lo, void* x8, long long i4) {
  if constexpr (ARITH == kArithF16F8) {
    uint2 h16;
    uint32_t h8, l8;
    split4_f16f8(v, h16, h8, l8);
    reinterpret_cast<uint2*>(hi)[i4] = h16;
    reinterpret_cast<uint32_t*>(lo)[i4] = h8;
    reinterpret_cast<uint32_t*>(x8)[i4] = l8;
  } else {
    __nv_bfloat16 h[4], l[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) split_bf16(v[u], h[u], l[u]);
    reinterpret_cast<uint2*>(hi)[i4] = make_uint2(pack_bf16(h[0], h[1]), pack_bf16(h[2], h[3]));
    reinterpret_cast<uint2*>(lo)[i4] = make_uint2(pack_bf16(l[0], l[1]), pack_bf16(l[2], l[3]));
  }
}

// f16f8: `res_flag` (zeroed by the caller) is set to 1 when any element has a non-zero residual plane entry, i.e. is
// not exactly representable in fp16; the GEMMs that read x skip the corresponding cross term while it stays 0.
// res_flag[kAbsmaxWord] accumulates the bit pattern of the largest |x| seen since the plan was prepared (a monitor for
// the fp16 range this arithmetic assumes; sce_input_absmax reads it). It lives in its own 128-byte line: next to the
// flag word, every warp's store to the flag would bounce the line the monitor's read needs (measured: 0.29 ms
// instead of 0.03 ms for the 16 MB batch split on inexact data).
constexpr int kAbsmaxWord = 32;
// res_flag[kBadWord] != 0: "this step must not update the parameters" — the batch split saw a value the fp16 operand
// plane cannot hold (|x| >= 65520 or NaN), or the loss finalisation saw a non-finite loss. The Adam kernels read it
// and leave parameters, moments and operand planes untouched, so an out-of-range chunk cannot poison the run before
// the host looks (sce_health); sticky until sce_prepare / sce_clear_health. Own 128-byte line, like the monitor.
constexpr int kBadWord = 64;
constexpr int kFlagWords = 128;
__device__ __forceinline__ bool step_is_bad(const uint32_t* __restrict__ flags) {
  return flags != nullptr && *reinterpret_cast<const volatile uint32_t*>(flags + kBadWord) != 0u;
}
// SHIFT (input_shift plans): the planes are those of x + shift (fp32 add), and the shifted fp32 values are also written
// to `xs`, the batch every later kernel of the step reads; the flags above judge the shifted values.
template <int ARITH, bool SHIFT = false>
__global__ void split_rows_kernel(const float* __restrict__ x, void* __restrict__ hi, void* __restrict__ lo,
                                  void* __restrict__ x8, long long n4, uint32_t* __restrict__ res_flag, float shift,
                                  float* __restrict__ xs) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  uint32_t any = 0;
  float amax = 0.f;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
    float4 v = reinterpret_cast<const float4*>(x)[i];
    if constexpr (SHIFT) {
      v = make_float4(v.x + shift, v.y + shift, v.z + shift, v.w + shift);
      reinterpret_cast<float4*>(xs)[i] = v;
    }
    const float vv[4] = {v.x, v.y, v.z, v.w};
    if constexpr (ARITH == kArithF16F8) {
      amax = fmaxf(fmaxf(amax, fmaxf(fabsf(v.x), fabsf(v.y))), fmaxf(fabsf(v.z), fabsf(v.w)));
      uint2 h16;
      uint32_t h8, l8;
      split4_f16f8(vv, h16, h8, l8);
      reinterpret_cast<uint2*>(hi)[i] = h16;
      reinterpret_cast<uint32_t*>(lo)[i] = h8;
      reinterpret_cast<uint32_t*>(x8)[i] = l8;
      any |= l8 & 0x7F7F7F7Fu;   // (a residual of -0 is still zero)
    } else {
      store_planes4<ARITH>(vv, hi, lo, x8, i);
    }
  }
  if constexpr (ARITH == kArithF16F8) {
    if (res_flag && __any_sync(0xffffffffu, any != 0u) && (threadIdx.x & 31) == 0) *res_flag = 1u;  // benign race: all write 1
    if (res_flag) {
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
      // non-negative floats order like their bit patterns (a NaN input has the largest pattern and sticks)
      if ((threadIdx.x & 31) == 0 && __float_as_uint(amax) > res_flag[kAbsmaxWord])
        atomicMax(res_flag + kAbsmaxWord, __float_as_uint(amax));
      // 65520 is the smallest magnitude that rounds to inf in fp16; a NaN has a larger bit pattern still
      if ((threadIdx.x & 31) == 0 && __float_as_uint(amax) >= 0x477FF000u) res_flag[kBadWord] = 1u;
    }
  }
}

// ------------------------------------------------------------------------------------------------
// centring, first half: (x - trans[m]) -> operand planes of model m (the A operand of the rotation GEMM, EpiCenter).
// x: [B][d] shared by the models (x_model_stride = 0) or [M][B][d]; planes of model m start at m * plane_model_stride.
// ------------------------------------------------------------------------------------------------
template <int ARITH>
__global__ void center_split_kernel(const float* __restrict__ x, long long x_model_stride, const float* __restrict__ trans,
                                    void* __restrict__ hi, void* __restrict__ lo, void* __restrict__ x8,
                                    long long plane_model_stride, int B, int d) {
  const int model = blockIdx.y;
  const int d4 = d >> 2;
  const long long n4 = (long long)B * d4;
  const float4* xs = reinterpret_cast<const float4*>(x + (long long)model * x_model_stride);
  const float4* ts = reinterpret_cast<const float4*>(trans + (long long)model * d);
  const long long p4 = (long long)model * plane_model_stride / 4;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    const float4 v = xs[i];
    const float4 t = __ldg(ts + (int)(i % d4));
    const float vv[4] = {v.x - t.x, v.y - t.y, v.z - t.z, v.w - t.w};
    store_planes4<ARITH>(vv, hi, lo, x8, p4 + i);
  }
}

// ------------------------------------------------------------------------------------------------
// chunk row gather (+ fp16 -> fp32, + mean-centring): out[r,:] = float(chunk[idx[r],:]) - sub
// one warp per row; big_sweep.py:168 and :359-364
// ------------------------------------------------------------------------------------------------
template <typename InT>
__global__ void gather_rows_kernel(const InT* __restrict__ chunk, long long n_rows, int d,
                                   const long long* __restrict__ idx, int B,
                                   const float* __restrict__ sub, float* __restrict__ out) {
  const int warps_per_block = blockDim.x >> 5;
  const int lane = threadIdx.x & 31;
  for (int r = blockIdx.x * warps_per_block + (threadIdx.x >> 5); r < B; r += gridDim.x * warps_per_block) {
    long long src = idx ? idx[r] : r;
    if (src < 0) src += n_rows;
    const InT* s = chunk + src * d;
    float* o = out + (long long)r * d;
    for (int c = lane * 4; c < d; c += 128) {
      float v[4];
      if constexpr (sizeof(InT) == 2) {
        const uint2 raw = *reinterpret_cast<const uint2*>(s + c);
        const __half2 a = *reinterpret_cast<const __half2*>(&raw.x);
        const __half2 b = *reinterpret_cast<const __half2*>(&raw.y);
        v[0] = __low2float(a);
        v[1] = __high2float(a);
        v[2] = __low2float(b);
        v[3] = __high2float(b);
      } else {
        const float4 f = *reinterpret_cast<const float4*>(s + c);
        v[0] = f.x;
        v[1] = f.y;
        v[2] = f.z;
        v[3] = f.w;
      }
      if (sub) {
        const float4 m = *reinterpret_cast<const float4*>(sub + c);
        v[0] -= m.x;
        v[1] -= m.y;
        v[2] -= m.z;
        v[3] -= m.w;
      }
      *reinterpret_cast<float4*>(o + c) = make_float4(v[0], v[1], v[2], v[3]);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// block-wide sum over 128 threads (two values at once)
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void block_sum2(float& a, float& b, float* red /*[8]*/) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    a += __shfl_xor_sync(0xffffffffu, a, o);
    b += __shfl_xor_sync(0xffffffffu, b, o);
  }
  const int w = threadIdx.x >> 5;
  __syncthreads();
  if ((threadIdx.x & 31) == 0) {
    red[w] = a;
    red[4 + w] = b;
  }
  __syncthreads();
  a = red[0] + red[1] + red[2] + red[3];
  b = red[4] + red[5] + red[6] + red[7];
}

struct AdamHyper {
  float lr, b1, b2, eps, eps_root;
  float bc1, bc2;  // 1 - b1^t, 1 - b2^t
};

__device__ __forceinline__ float adam_apply(float p, float g, float& m, float& v, const AdamHyper& h) {
  m = h.b1 * m + (1.f - h.b1) * g;
  v = h.b2 * v + (1.f - h.b2) * g * g;
  const float mh = m / h.bc1;
  const float vh = v / h.bc2;
  return p - h.lr * (mh / (sqrtf(vh + h.eps_root) + h.eps));
}

// ------------------------------------------------------------------------------------------------
// Dictionary rows: one 128-thread block per (model, row).
//   MODE_PREPARE : w = e / max(||e||, floor) -> (w_hi, w_lo)                     (sce_prepare)
//   MODE_ADAM    : de = J(dw); Adam on e; then as PREPARE for the updated row     (sce_step)
//   MODE_GRAD    : de = J(dw) -> grad_out                                         (sce_grads)
// J is the Jacobian of the row normalisation, de = (dw - w <w, dw>) / s (sae_ensemble.py:136-137
// differentiated); with `normalize == 0` (untied encoder) J = I and the split is of e itself.
// NONNEG (desc.encoder_nonneg, mlp_tests.py:100-102): the norm, w, J and the emitted planes use e+ = max(e, 0), formed
// in place from the raw row as it is read; de = J(dw) is the gradient with respect to e+, which MODE_GRAD returns and
// MODE_ADAM applies to the raw e, read again for the update (straight-through: no [e >= 0] mask, as the reference's
// gradient).
// NV = ceil(d / 512) float4 per thread.
// ------------------------------------------------------------------------------------------------
enum { MODE_PREPARE = 0, MODE_ADAM = 1, MODE_GRAD = 2 };

__device__ __forceinline__ float4 nonneg4(const float4& e) {
  return make_float4(fmaxf(e.x, 0.f), fmaxf(e.y, 0.f), fmaxf(e.z, 0.f), fmaxf(e.w, 0.f));
}
// The row sums and the Jacobian in explicitly rounded steps: every instantiation then rounds them alike, which free
// contraction does not guarantee (MODE_GRAD and MODE_ADAM of one width had fused different products). So the gradient
// MODE_ADAM applies is bitwise the one MODE_GRAD returns (sce_grads). dot4_rn is the order the step's kernels were
// compiled to. NONNEG rows take the sum of squares as sumsq4_rn, so that the norm MODE_ADAM re-splits the updated row
// with and the one MODE_PREPARE derives from the same row are bitwise equal (a resumed run prepares its planes afresh).
__device__ __forceinline__ float dot4_rn(const float4& a, const float4& b) {
  return __fmaf_rn(a.w, b.w, __fmaf_rn(a.z, b.z, __fmaf_rn(a.x, b.x, __fmul_rn(a.y, b.y))));
}
__device__ __forceinline__ float sumsq4_rn(const float4& v) {
  return __fmaf_rn(v.w, v.w, __fmaf_rn(v.z, v.z, __fmaf_rn(v.y, v.y, __fmul_rn(v.x, v.x))));
}

template <int NV, int MODE, int ARITH, bool NONNEG = false>
__global__ void __launch_bounds__(128) dict_rows_kernel(float* __restrict__ e, const float* __restrict__ dw,
                                                        float* __restrict__ m, float* __restrict__ v,
                                                        void* __restrict__ w_hi, void* __restrict__ w_lo,
                                                        void* __restrict__ w_x8, float* __restrict__ grad_out, int d,
                                                        int normalize, float floor, AdamHyper h,
                                                        const uint32_t* __restrict__ health,
                                                        float* __restrict__ w_f32 /*optional fp32 copy of w (top-k gather)*/) {
  __shared__ float red[8];
  if (MODE == MODE_ADAM && step_is_bad(health)) return;   // block-uniform: see kBadWord
  const long long row = blockIdx.x;
  const long long base = row * d;
  float4 ev[NV], gv[NV];
  float ss = 0.f, dot = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int c = (i * 128 + threadIdx.x) * 4;
    ev[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    gv[i] = ev[i];
    if (c < d) {
      ev[i] = *reinterpret_cast<const float4*>(e + base + c);
      if (MODE != MODE_PREPARE) gv[i] = *reinterpret_cast<const float4*>(dw + base + c);
      if constexpr (NONNEG) ev[i] = nonneg4(ev[i]);
    }
    if constexpr (NONNEG) ss = __fadd_rn(ss, sumsq4_rn(ev[i]));
    else ss = __fadd_rn(ss, dot4_rn(ev[i], ev[i]));
    dot = __fadd_rn(dot, dot4_rn(ev[i], gv[i]));
  }
  float s = 1.f;
  if (normalize) {
    block_sum2(ss, dot, red);
    const float nrm = sqrtf(ss);
    const bool clamped = floor > 0.f && nrm < floor;
    s = clamped ? floor : nrm;
    if (MODE != MODE_PREPARE) {
      // <w, dw> = <e, dw> / s ;  de = (dw - w <w,dw>) / s = dw / s - e * <e,dw> / s^3
      const float inv = 1.f / s;
      const float k = clamped ? 0.f : dot * inv * inv * inv;  // clamp active: d s / d e = 0
#pragma unroll
      for (int i = 0; i < NV; ++i) {
        gv[i].x = __fmaf_rn(gv[i].x, inv, -__fmul_rn(ev[i].x, k));
        gv[i].y = __fmaf_rn(gv[i].y, inv, -__fmul_rn(ev[i].y, k));
        gv[i].z = __fmaf_rn(gv[i].z, inv, -__fmul_rn(ev[i].z, k));
        gv[i].w = __fmaf_rn(gv[i].w, inv, -__fmul_rn(ev[i].w, k));
      }
    }
  }
  if (MODE == MODE_GRAD) {
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int c = (i * 128 + threadIdx.x) * 4;
      if (c < d) *reinterpret_cast<float4*>(grad_out + base + c) = gv[i];
    }
    return;
  }
  if (MODE == MODE_ADAM) {
    float ss2 = 0.f, dummy = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int c = (i * 128 + threadIdx.x) * 4;
      if (c < d) {
        float4 mv = *reinterpret_cast<const float4*>(m + base + c);
        float4 vv = *reinterpret_cast<const float4*>(v + base + c);
        if constexpr (NONNEG) ev[i] = *reinterpret_cast<const float4*>(e + base + c);   // Adam moves the raw entries
        ev[i].x = adam_apply(ev[i].x, gv[i].x, mv.x, vv.x, h);
        ev[i].y = adam_apply(ev[i].y, gv[i].y, mv.y, vv.y, h);
        ev[i].z = adam_apply(ev[i].z, gv[i].z, mv.z, vv.z, h);
        ev[i].w = adam_apply(ev[i].w, gv[i].w, mv.w, vv.w, h);
        *reinterpret_cast<float4*>(m + base + c) = mv;
        *reinterpret_cast<float4*>(v + base + c) = vv;
        *reinterpret_cast<float4*>(e + base + c) = ev[i];
        if constexpr (NONNEG) {
          ev[i] = nonneg4(ev[i]);
          ss2 = __fadd_rn(ss2, sumsq4_rn(ev[i]));
        } else {
          ss2 += ev[i].x * ev[i].x + ev[i].y * ev[i].y + ev[i].z * ev[i].z + ev[i].w * ev[i].w;
        }
      }
    }
    if (normalize) {
      block_sum2(ss2, dummy, red);
      const float nrm = sqrtf(ss2);
      s = (floor > 0.f && nrm < floor) ? floor : nrm;
    }
  }
  // emit the operand copy the next step's GEMMs read
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int c = (i * 128 + threadIdx.x) * 4;
    if (c < d) {
      const float w[4] = {ev[i].x / s, ev[i].y / s, ev[i].z / s, ev[i].w / s};
      store_planes4<ARITH>(w, w_hi, w_lo, w_x8, (base + c) >> 2);
      if (w_f32) *reinterpret_cast<float4*>(w_f32 + base + c) = make_float4(w[0], w[1], w[2], w[3]);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// [models][rows][cols] -> [models][cols][rows] through 64 x 64 tiles in shared memory (grid: column tiles, row tiles,
// models). f16f8 runs it on the decoder's planes after every rewrite, so that the decode GEMM reads the dictionary
// K-major (its reduction runs over the dictionary rows) and forms its cross terms on E5M2 wgmma.
// ------------------------------------------------------------------------------------------------
template <class T>
__global__ void __launch_bounds__(256) transpose_kernel(const T* __restrict__ src, T* __restrict__ dst, int rows, int cols) {
  __shared__ T tile[64][65];
  const long long off = (long long)blockIdx.z * rows * cols;
  const int r0 = blockIdx.y * 64, c0 = blockIdx.x * 64, tx = threadIdx.x & 63, ty = threadIdx.x >> 6;
  for (int i = ty; i < 64; i += 4)
    if (r0 + i < rows && c0 + tx < cols) tile[i][tx] = src[off + (long long)(r0 + i) * cols + c0 + tx];
  __syncthreads();
  for (int i = ty; i < 64; i += 4)
    if (c0 + i < cols && r0 + tx < rows) dst[off + (long long)(c0 + i) * rows + r0 + tx] = tile[tx][i];
}

// ------------------------------------------------------------------------------------------------
// bias gradient = sum of the per-warp column partials (+ bias decay), then Adam or plain output
// ------------------------------------------------------------------------------------------------
template <int MODE>
__global__ void bias_kernel(float* __restrict__ bias, float* __restrict__ m, float* __restrict__ v,
                            const float* __restrict__ db_part, int n_part, int n, int n_models,
                            const float* __restrict__ bias_decay, const float* __restrict__ bnorm,
                            float* __restrict__ grad_out, AdamHyper h, float part_scale,
                            const uint32_t* __restrict__ health) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)n_models * n) return;
  if (MODE == MODE_ADAM && step_is_bad(health)) return;
  const int model = int(i / n);
  const int j = int(i - (long long)model * n);
  const float* p = db_part + (long long)model * n_part * n + j;
  float g = 0.f;
  for (int k = 0; k < n_part; ++k) g += p[(long long)k * n];
  g = __fmul_rn(g, part_scale);  // f16f8: the partials are sums of dz * B d / 2 (see EpiDecodeT); not fused with the
                                 // decay term, so that MODE_GRAD and MODE_ADAM round it alike
  const float b = bias[i];
  if (bias_decay) {
    const float bd = bias_decay[model], nb = bnorm[model];
    if (bd != 0.f && nb > 0.f) g += bd * b / nb;
  }
  if (MODE == MODE_GRAD) {
    grad_out[i] = g;
  } else {
    float mm = m[i], vv = v[i];
    bias[i] = adam_apply(b, g, mm, vv, h);
    m[i] = mm;
    v[i] = vv;
  }
}

// ------------------------------------------------------------------------------------------------
// TopK selection helpers (topk_encoder.py:19-27; the kernels are in sce_topk.cuh): order-preserving keys, a
// warp-aggregated histogram and a block-wide bin pick for the 8-bit radix select.
// Ties at the k-th value are broken by lowest column index (torch.topk leaves this unspecified, Q8).
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t f2key(float f) {
  const uint32_t u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);  // ascending float order == ascending uint order
}

// warp-aggregated shared-memory histogram increment: lanes with the same bin elect one to add their count
// (Gaussian-like scores share sign+exponent bits, so a naive atomicAdd serialises on two or three hot bins)
__device__ __forceinline__ void hist_add(uint32_t* hist, uint32_t bin, bool active) {
  const uint32_t act = __ballot_sync(0xffffffffu, active);
  if (!active) return;
  const uint32_t peers = __match_any_sync(act, bin);
  if ((threadIdx.x & 31) == (__ffs(peers) - 1)) atomicAdd(&hist[bin], (uint32_t)__popc(peers));
}

// block-wide (256 threads, one per bin): find the bin holding the `rem`-th largest element by a parallel
// suffix scan of the histogram (a serial walk by one thread costs ~250 dependent shared-memory reads per pass).
// Updates sh_prefix / sh_remaining; ends with a __syncthreads().
__device__ __forceinline__ void pick_bin(const uint32_t* hist, uint32_t* sh_prefix, uint32_t* sh_remaining,
                                         uint32_t* warp_tot /*[8]*/, int shift, uint32_t* count_in_bin) {
  const int r = threadIdx.x;            // reversed bin index: bin = 255 - r, so a PREFIX sum counts bins >= bin
  const uint32_t h = hist[255 - r];
  uint32_t p = h;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t v = __shfl_up_sync(0xffffffffu, p, o);
    if ((r & 31) >= o) p += v;
  }
  if ((r & 31) == 31) warp_tot[r >> 5] = p;
  __syncthreads();
  uint32_t off = 0;
  for (int w = 0; w < (r >> 5); ++w) off += warp_tot[w];
  p += off;                              // elements in bins >= this one
  const uint32_t rem = *sh_remaining;
  __syncthreads();                       // everyone has read sh_remaining before the winner rewrites it
  if (p >= rem && p - h < rem) {         // exactly one bin satisfies this (rem >= 1, total >= rem)
    *sh_prefix |= uint32_t(255 - r) << shift;
    *sh_remaining = rem - (p - h);
    if (count_in_bin) *count_in_bin = h;
  }
  __syncthreads();
}

__device__ __forceinline__ float key2relu(uint32_t key) {  // relu(float behind an order-preserving key)
  return key > 0x80000000u ? __uint_as_float(key & 0x7FFFFFFFu) : 0.f;
}

}  // namespace sce
