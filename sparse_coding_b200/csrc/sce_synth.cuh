// sce_synth.cuh — synthetic sparse-mixture rows (sc_datasets/random_dataset.py generate_correlated_dataset /
// generate_rand_dataset / generate_noise_dataset) generated on the device, one row at a time, without the dense
// [rows, n_gt] code the reference materialises three times per send.
//
// Every draw is a pure function of (seed, global row, component, stream tag) under Philox4x32-10 (include/sce.h spells
// the contract out), so a row is the same whichever call, launch geometry or GPU produced it.
//
// One row: the thresholds u_thresh(j) <= p_j of all n_gt components, four per Philox call, one warp stepping through
// windows of 128 components; the active set is compacted in ascending j (a warp scan of the per-lane counts) into a
// shared-memory list of (j, u_val * u_strength), with the value and strength words drawn only by lanes that hold an
// active component. When the list could overflow in the next window, and at the end of the row, the row's warps
// accumulate coef * feats[j, :] into fp32 registers in ascending j, reading the feature rows as float4 from L2. A row
// with no active component gets the zero-row component when the caller asks for it. Then the Box-Muller noise is added
// and the row is stored as fp32 or round-to-nearest fp16.
//   d <= 1024: a warp per row, eight rows per 256-thread block, V float4 per lane (V = 1, 2, 4, 8).
//   d  > 1024: one row per block of ceil(d / 1024) warps that share the list (the first warp builds it), 8 float4 per lane.
#pragma once
#include <cuda_fp16.h>
#include <stdint.h>

namespace sce {

enum : uint32_t { kSynthThresh = 0, kSynthValue = 1, kSynthStrength = 2, kSynthZero = 3, kSynthNoise = 4 };
constexpr int kSynthList = 256;   // list entries per row held in shared memory between two gathers
constexpr int kSynthWindow = 128; // components one warp tests per step (32 lanes x one Philox call)

struct Philox4 { uint32_t x, y, z, w; };

// Philox4x32-10 (Salmon et al., SC'11; the Random123 constants).
__device__ __forceinline__ Philox4 philox4x32_10(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t k0,
                                                 uint32_t k1) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
    c0 = hi1 ^ c1 ^ k0;
    c2 = hi0 ^ c3 ^ k1;
    c1 = lo1;
    c3 = lo0;
    k0 += 0x9E3779B9u;
    k1 += 0xBB67AE85u;
  }
  return {c0, c1, c2, c3};
}

__device__ __forceinline__ float synth_uniform(uint32_t x) { return (float)(x >> 8) * 0x1p-24f; }
__device__ __forceinline__ uint32_t synth_word(const Philox4& r, int k) {
  return k == 0 ? r.x : k == 1 ? r.y : k == 2 ? r.z : r.w;
}

// One Box-Muller pair: u1 = ((a >> 8) + 1) 2^-24 in (0, 1], u2 = (b >> 8) 2^-24; r = sqrt(-2 ln u1);
// (r cos 2 pi u2, r sin 2 pi u2).
__device__ __forceinline__ void synth_box_muller(uint32_t a, uint32_t b, float& z0, float& z1) {
  const float u1 = (float)((a >> 8) + 1u) * 0x1p-24f;
  const float u2 = (float)(b >> 8) * 0x1p-24f;
  const float r = sqrtf(-2.f * logf(u1));
  float s, c;
  sincospif(2.f * u2, &s, &c);
  z0 = r * c;
  z1 = r * s;
}

struct SynthArgs {
  const float* feats;  // [n_gt, d]
  const float* probs;  // [ceil(B / group_rows), n_gt]
  int n_gt, d, group_rows, B;
  long long row0;
  uint32_t k0, k1;
  int zero_row_rule;
  float noise_scale;
  void* out;
  int out_half;
  int* row_nnz;
  int* code_idx;
  float* code_val;
  int code_cap;
};

// acc[v] += coef[e] * feats[idx[e], 4 c4 .. 4 c4 + 3] for e in [0, count), ascending, c4 = col0 + stride4 * v.
template <int V>
__device__ __forceinline__ void synth_gather(const SynthArgs& a, const int* idx, const float* coef, int count, int col0,
                                             int stride4, float4 (&acc)[V]) {
  const float4* f4 = reinterpret_cast<const float4*>(a.feats);
  const int d4 = a.d >> 2;
#pragma unroll 2
  for (int e = 0; e < count; ++e) {
    const float c = coef[e];
    const float4* row = f4 + (long long)idx[e] * d4;
#pragma unroll
    for (int v = 0; v < V; ++v) {
      const int c4 = col0 + stride4 * v;
      if (c4 < d4) {
        const float4 f = __ldg(row + c4);
        acc[v].x = fmaf(c, f.x, acc[v].x);
        acc[v].y = fmaf(c, f.y, acc[v].y);
        acc[v].z = fmaf(c, f.z, acc[v].z);
        acc[v].w = fmaf(c, f.w, acc[v].w);
      }
    }
  }
}

// TEAM = false: blockDim 256, warp w of block b makes local row 8 b + w. TEAM = true: blockDim 32 G (G <= 8), block b
// makes local row b; warp 0 builds the list, the count reaches the other warps through shared memory.
template <int V, bool TEAM>
__global__ void __launch_bounds__(256) synth_rows_kernel(SynthArgs a) {
  constexpr int kLists = TEAM ? 1 : 8;
  __shared__ int s_idx[kLists][kSynthList];
  __shared__ float s_coef[kLists][kSynthList];
  __shared__ int s_cnt[3];  // TEAM: list length after even / odd windows, and after the zero-row rule
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int i = TEAM ? (int)blockIdx.x : (int)blockIdx.x * 8 + warp;
  if (!TEAM && i >= a.B) return;  // whole warps: nothing synchronises across warps in this mode
  const bool builder = !TEAM || warp == 0;
  const long long grow = a.row0 + i;
  const uint32_t rlo = (uint32_t)grow, rhi = (uint32_t)((unsigned long long)grow >> 32);
  const float* p = a.probs + (long long)(i / a.group_rows) * a.n_gt;
  int* s_i = s_idx[TEAM ? 0 : warp];
  float* s_c = s_coef[TEAM ? 0 : warp];
  const int col0 = TEAM ? (int)threadIdx.x : lane;
  const int stride4 = TEAM ? (int)blockDim.x : 32;
  const long long code0 = (long long)i * a.code_cap;
  float4 acc[V];
#pragma unroll
  for (int v = 0; v < V; ++v) acc[v] = make_float4(0.f, 0.f, 0.f, 0.f);

  int total = 0;  // active components of the row so far (builder warp)
  int count = 0;  // entries in the list (every thread of the row)
  for (int base = 0, w = 0; base < a.n_gt; base += kSynthWindow, ++w) {
    if (builder) {
      const int j0 = base + 4 * lane;
      const uint32_t q = (uint32_t)(j0 >> 2);
      uint32_t bits = 0;
      if (j0 < a.n_gt) {
        const Philox4 t = philox4x32_10(q, rlo, rhi, kSynthThresh, a.k0, a.k1);
#pragma unroll
        for (int k = 0; k < 4; ++k)
          if (j0 + k < a.n_gt && synth_uniform(synth_word(t, k)) <= __ldg(p + j0 + k)) bits |= 1u << k;
      }
      const int mine = __popc(bits);
      int incl = mine;
#pragma unroll
      for (int off = 1; off < 32; off <<= 1) {
        const int o = __shfl_up_sync(0xffffffffu, incl, off);
        if (lane >= off) incl += o;
      }
      const int window = __shfl_sync(0xffffffffu, incl, 31);
      if (bits) {
        const Philox4 val = philox4x32_10(q, rlo, rhi, kSynthValue, a.k0, a.k1);
        const Philox4 str = philox4x32_10(q, rlo, rhi, kSynthStrength, a.k0, a.k1);
        int pos = incl - mine;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          if (bits >> k & 1u) {
            const float c = synth_uniform(synth_word(val, k)) * synth_uniform(synth_word(str, k));
            s_i[count + pos] = j0 + k;
            s_c[count + pos] = c;
            if (a.code_idx && total + pos < a.code_cap) {
              a.code_idx[code0 + total + pos] = j0 + k;
              a.code_val[code0 + total + pos] = c;
            }
            ++pos;
          }
        }
      }
      count += window;
      total += window;
      if (TEAM && lane == 0) s_cnt[w & 1] = count;
    }
    if (TEAM) {
      __syncthreads();
      count = s_cnt[w & 1];  // rewritten two windows later, after a barrier every thread passes only after this read
    } else {
      __syncwarp();
    }
    if (count > kSynthList - kSynthWindow) {  // the next window could overflow the list: gather it now
      synth_gather<V>(a, s_i, s_c, count, col0, stride4, acc);
      count = 0;
      if (TEAM) __syncthreads(); else __syncwarp();
    }
  }
  if (builder && total == 0 && a.zero_row_rule) {  // generate_correlated_dataset: no row without a component
    const Philox4 z = philox4x32_10(0u, rlo, rhi, kSynthZero, a.k0, a.k1);
    const int j = (int)(((unsigned long long)z.x * (unsigned)a.n_gt) >> 32);
    const Philox4 str = philox4x32_10((uint32_t)(j >> 2), rlo, rhi, kSynthStrength, a.k0, a.k1);
    const float c = 1.0f * synth_uniform(synth_word(str, j & 3));
    if (lane == 0) {
      s_i[0] = j;
      s_c[0] = c;
      if (a.code_idx) {
        a.code_idx[code0] = j;
        a.code_val[code0] = c;
      }
    }
    count = 1;
    total = 1;
  }
  if (TEAM) {
    if (warp == 0 && lane == 0) s_cnt[2] = count;
    __syncthreads();
    count = s_cnt[2];
  } else {
    __syncwarp();
  }
  if (count) synth_gather<V>(a, s_i, s_c, count, col0, stride4, acc);
  if (builder && lane == 0 && a.row_nnz) a.row_nnz[i] = total;

  const int d4 = a.d >> 2;
#pragma unroll
  for (int v = 0; v < V; ++v) {
    const int c4 = col0 + stride4 * v;
    if (c4 >= d4) continue;
    float4 x = acc[v];
    if (a.noise_scale != 0.f) {
      const Philox4 r = philox4x32_10((uint32_t)c4, rlo, rhi, kSynthNoise, a.k0, a.k1);
      float z0, z1, z2, z3;
      synth_box_muller(r.x, r.y, z0, z1);
      synth_box_muller(r.z, r.w, z2, z3);
      x.x = fmaf(a.noise_scale, z0, x.x);
      x.y = fmaf(a.noise_scale, z1, x.y);
      x.z = fmaf(a.noise_scale, z2, x.z);
      x.w = fmaf(a.noise_scale, z3, x.w);
    }
    const long long o4 = (long long)i * d4 + c4;
    if (a.out_half) {
      const __half2 h0 = __floats2half2_rn(x.x, x.y), h1 = __floats2half2_rn(x.z, x.w);
      uint2 u;
      u.x = *reinterpret_cast<const uint32_t*>(&h0);
      u.y = *reinterpret_cast<const uint32_t*>(&h1);
      reinterpret_cast<uint2*>(a.out)[o4] = u;
    } else {
      reinterpret_cast<float4*>(a.out)[o4] = x;
    }
  }
}

}  // namespace sce
