// sce_epilogues.cuh — the fused epilogues of the four GEMMs of one ensemble training step.
// Each functor is constructed per (thread, tile) by gemm_split_kernel, receives the fp32
// accumulator of its row in 32-column chunks, and writes what the next GEMM
// needs — as operand planes (fp16 + two E5M2 planes, or a (hi, lo) bf16 pair; 4 bytes per element either way) — so
// the fp32 code tensor [M,B,n] never exists in HBM.
//
// Reference arithmetic being fused (HoagyC/sparse_coding @ 69c5ae0):
//   encode  c = clamp(x W^T + b, min=0) [masked_fill]        autoencoders/sae_ensemble.py:141-143, 356
//   decode  x^ = c W ; l_rec = mean((x^ - x)^2)               :145, :148
//   l1      alpha * mean_b sum_n |c|                          :149
//   dcode   backward of the above (SURVEY.md §8 a4)
#pragma once
#include "sce_gemm.cuh"

namespace sce {

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Store 32 consecutive bf16 (64 B) from packed registers.
__device__ __forceinline__ void store_bf16x32(__nv_bfloat16* dst, const uint32_t (&w)[16], int ncols_valid) {
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    if (j * 8 < ncols_valid) {  // host guarantees n % 8 == 0
      uint4 v = make_uint4(w[4 * j], w[4 * j + 1], w[4 * j + 2], w[4 * j + 3]);
      *reinterpret_cast<uint4*>(dst + j * 8) = v;
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Epilogue output staging: each epilogue warp owns two 2 KB shared-memory tiles (hi, lo) of 32 rows x
// 32 bf16 (64-byte rows, TMA 64-byte swizzle: 16-byte chunk index ^= (row >> 1) & 3). A thread writes its
// own row with four conflict-free 16-byte stores; one lane then hands the tile to the TMA engine, which
// writes full lines to HBM and clips rows/columns outside the tensor. Replaces 32-line scattered STG.128
// (the r01b profile had the encode/dcode epilogues bound by L1 line requests, ~16 k per tile).
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void stage_row32(uint8_t* tile, int lane, const uint32_t (&w)[16]) {
  const int sw = (lane >> 1) & 3;
#pragma unroll
  for (int q = 0; q < 4; ++q)
    *reinterpret_cast<uint4*>(tile + lane * 64 + ((q ^ sw) << 4)) =
        make_uint4(w[4 * q], w[4 * q + 1], w[4 * q + 2], w[4 * q + 3]);
}
// 8-bit plane tile: 32 rows x 32 bytes, TMA 32-byte swizzle (16-byte chunk index ^= (row >> 2) & 1)
__device__ __forceinline__ void stage_row32_u8(uint8_t* tile, int lane, const uint32_t* w /*[8]*/) {
  const int sw = (lane >> 2) & 1;
#pragma unroll
  for (int q = 0; q < 2; ++q)
    *reinterpret_cast<uint4*>(tile + lane * 32 + ((q ^ sw) << 4)) = make_uint4(w[4 * q], w[4 * q + 1], w[4 * q + 2], w[4 * q + 3]);
}
// 8-bit plane tile TRANSPOSED: 32 columns x 32 rows, 32-byte rows, no swizzle. The lane's row becomes byte `lane` of
// each of the 32 tile rows. A lane holds one row of each 4 x 4 byte block (4 columns of the 4 rows of its lane quad), so
// the blocks are transposed across the quad in two exchanges: lanes 2 apart swap byte pairs, then lanes 1 apart single
// bytes, the halves of two words per shuffle. Lane 4 a + s then holds bytes 4 a .. + 3 of the tile rows 4 w + s and
// writes them as words; the 32 lanes of each store hit 32 different banks.
__device__ __forceinline__ void stage_col32_u8(uint8_t* tile, int lane, const uint32_t* w /*[8]*/) {
  const bool h = lane & 2, l = lane & 1;
  // PRMT selectors of this lane's place in its quad: what it sends, and how it joins what it keeps with what it receives
  const uint32_t s1_send = h ? 0x5410 : 0x7632, s1_lo = h ? 0x3254 : 0x5410, s1_hi = h ? 0x3276 : 0x7610;
  const uint32_t s2_send = l ? 0x6420 : 0x7531, s2_lo = l ? 0x3514 : 0x5240, s2_hi = l ? 0x3716 : 0x7260;
  uint32_t* out = reinterpret_cast<uint32_t*>(tile) + (lane & 3) * 8 + (lane >> 2);
#pragma unroll
  for (int q = 0; q < 4; ++q) {   // words 2 q and 2 q + 1: tile rows 8 q + s and 8 q + 4 + s
    const uint32_t x0 = w[2 * q], x1 = w[2 * q + 1];
    uint32_t t = __shfl_xor_sync(0xffffffffu, __byte_perm(x0, x1, s1_send), 2);
    const uint32_t z0 = __byte_perm(x0, t, s1_lo), z1 = __byte_perm(x1, t, s1_hi);
    t = __shfl_xor_sync(0xffffffffu, __byte_perm(z0, z1, s2_send), 1);
    out[(2 * q) * 32] = __byte_perm(z0, t, s2_lo);
    out[(2 * q + 1) * 32] = __byte_perm(z1, t, s2_hi);
  }
}
// The same transpose stored straight to global memory, without staging: tile row j (a column of the 32-row block) goes
// to dst + j * ld, each store instruction writing four whole 32-byte segments. Only tile rows below `cols` (a multiple
// of 16, as f16f8 shapes are) and words whose first byte lies below `rows` are written; a word that crosses `rows` writes
// up to three bytes beyond it, which stay inside the row pitch ld (a multiple of 16 at least `rows`) and which no reader
// of the copy looks at. (Its own copy of the exchange: sharing one with stage_col32_u8 moved the dcode kernel's
// instruction schedule.)
__device__ __forceinline__ void store_col32_u8(uint8_t* dst, int ld, int lane, const uint32_t* w /*[8]*/, int rows,
                                               int cols) {
  const bool h = lane & 2, l = lane & 1;
  const uint32_t s1_send = h ? 0x5410 : 0x7632, s1_lo = h ? 0x3254 : 0x5410, s1_hi = h ? 0x3276 : 0x7610;
  const uint32_t s2_send = l ? 0x6420 : 0x7531, s2_lo = l ? 0x3514 : 0x5240, s2_hi = l ? 0x3716 : 0x7260;
  const bool lo_ok = 4 * (lane >> 2) < rows, hi_ok = lo_ok && cols > 16;   // tile rows 0 .. 15, 16 .. 31
  uint8_t* out = dst + (lane & 3) * ld + 4 * (lane >> 2);
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const uint32_t x0 = w[2 * q], x1 = w[2 * q + 1];
    uint32_t t = __shfl_xor_sync(0xffffffffu, __byte_perm(x0, x1, s1_send), 2);
    const uint32_t z0 = __byte_perm(x0, t, s1_lo), z1 = __byte_perm(x1, t, s1_hi);
    t = __shfl_xor_sync(0xffffffffu, __byte_perm(z0, z1, s2_send), 1);
    st_global_u32_if(out + 8 * q * ld, __byte_perm(z0, t, s2_lo), q < 2 ? lo_ok : hi_ok);
    st_global_u32_if(out + (8 * q + 4) * ld, __byte_perm(z1, t, s2_hi), q < 2 ? lo_ok : hi_ok);
  }
}
// whole warp: wait until the share's staging tiles may be written (staging_wait), write them, launch their stores.
// bf16x3: whi / wx are the hi / lo planes. f16f8: whi is the fp16 plane, wx[0..7] the value-e5m2 plane and
// wx[8..15] the residual-e5m2 plane (maps m_lo / m_x8).
// `planes`: which of the f16f8 8-bit planes a consumer will read (bit 0: value plane, bit 1: residual plane); planes
// nobody reads are neither staged nor stored (warp-uniform). bf16x3 always writes both of its planes.
// T8 (f16f8): the 8-bit planes go to batch-major copies [model][col][row] (maps m_lo / m_x8 of box 32 rows x 32 bytes).
template <int ARITH, bool T8 = false>
__device__ __forceinline__ void stage_and_store(uint8_t* stage, const TileCoord& t, const uint32_t (&whi)[16],
                                                const uint32_t (&wx)[16], const CUtensorMap* m_hi,
                                                const CUtensorMap* m_lo, const CUtensorMap* m_x8, int col, int row0,
                                                int model, int planes = 3) {
  static_assert(!T8 || ARITH == kArithF16F8, "transposed 8-bit planes are f16f8 only");
  const int lane = t.lane;
  staging_wait(t);
  stage_row32(stage, lane, whi);
  if constexpr (T8) {
    if (planes & 1) stage_col32_u8(stage + 2048, lane, &wx[0]);
    if (planes & 2) stage_col32_u8(stage + 3072, lane, &wx[8]);
  } else if constexpr (ARITH == kArithF16F8) {
    if (planes & 1) stage_row32_u8(stage + 2048, lane, &wx[0]);
    if (planes & 2) stage_row32_u8(stage + 3072, lane, &wx[8]);
  } else {
    stage_row32(stage + 2048, lane, wx);
  }
  fence_proxy_async_smem();
  __syncwarp();
  if (lane == 0) {
    tma_store_3d(m_hi, stage, col, row0, model);
    if constexpr (T8) {
      if (planes & 1) tma_store_3d(m_lo, stage + 2048, row0, col, model);
      if (planes & 2) tma_store_3d(m_x8, stage + 3072, row0, col, model);
    } else if constexpr (ARITH == kArithF16F8) {
      if (planes & 1) tma_store_3d(m_lo, stage + 2048, col, row0, model);
      if (planes & 2) tma_store_3d(m_x8, stage + 3072, col, row0, model);
    } else {
      tma_store_3d(m_lo, stage + 2048, col, row0, model);
    }
    tma_store_commit();
  }
}

// ------------------------------------------------------------------------------------------------
// (hi, lo) split of two fp32 values into packed bf16x2 words: one packed conversion per pair for hi
// and one for lo (cvt.rn.bf16x2.f32), the residual formed on the fp32 pipe.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void split2(float a, float b, uint32_t& hi2, uint32_t& lo2) {
  const __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
  hi2 = *reinterpret_cast<const uint32_t*>(&h);
  const float ha = __uint_as_float(hi2 << 16), hb = __uint_as_float(hi2 & 0xFFFF0000u);
  const __nv_bfloat162 l = __floats2bfloat162_rn(a - ha, b - hb);
  lo2 = *reinterpret_cast<const uint32_t*>(&l);
}

// Pair `i` (0..15, compile-time after unrolling; pairs are produced in increasing order) of a 32-column chunk into
// the packed plane words the stores take.
template <int ARITH>
__device__ __forceinline__ void split_pair(float a, float b, int i, uint32_t (&whi)[16], uint32_t (&wx)[16]) {
  if constexpr (ARITH == kArithF16F8) {
    uint32_t h8, l8;
    split2_f16f8(a, b, whi[i], h8, l8);
    if (i & 1) {
      wx[i >> 1] |= h8 << 16;
      wx[8 + (i >> 1)] |= l8 << 16;
    } else {
      wx[i >> 1] = h8;
      wx[8 + (i >> 1)] = l8;
    }
  } else {
    split2(a, b, whi[i], wx[i]);
  }
}

// ------------------------------------------------------------------------------------------------
// Activity masks: what the backward pass needs to know about the forward pass per coefficient is two bits —
// [c > 0] (the sparsity term and the ReLU gate) and [z == 0] (clamp(min=0) passes the gradient at exactly 0, SURVEY
// Q4). encode (and the top-k selection) write them as two planes of 32-column words laid out CHUNK-major,
// word(model, chunk, row) at ((model * n_chunks + chunk) * batch_max + row): the 32 lanes of an epilogue warp own 32
// consecutive rows, so one coalesced 128-byte request per chunk replaces the 32 scattered 64-byte reads of the code's
// 16-bit plane the dcode epilogue used to make (1 GB per step at config 2; same-box timing without those reads: -12 %
// on dcode). Bit (31 - j) of a word is column 32 * chunk + j.
// ------------------------------------------------------------------------------------------------
struct ActMask {
  uint32_t* pos;    // [M][n_chunks][batch_max]
  uint32_t* zero;   // same shape: z == 0 exactly; nullptr with relu semantics (top-k), where it would stay empty
  int n_chunks, batch_max;
  __device__ __forceinline__ long long at(int model, int chunk, int row) const {
    return ((long long)model * n_chunks + chunk) * batch_max + row;
  }
};

// transpose-reduce: 32 lanes x 32 columns -> lane j holds op over the warp's rows of column j (31 shuffles). The inner
// loop runs a fixed 16 steps and skips those at or beyond `half`: with a trip count of `half` it is not unrolled before
// the outer loop, and v, indexed at run time, would live in local memory.
template <class T, class Op>
__device__ __forceinline__ T warp_column_reduce(T (&v)[32], int lane, Op op) {
#pragma unroll
  for (int half = 16; half >= 1; half >>= 1) {
    const bool upper = (lane & half) != 0;
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      if (i < half) {
        const T send = upper ? v[i] : v[i + half];
        const T keep = upper ? v[i + half] : v[i];
        v[i] = op(keep, __shfl_xor_sync(0xffffffffu, send, half));
      }
    }
  }
  return v[0];
}
__device__ __forceinline__ float warp_column_sum(float (&v)[32], int lane) {
  return warp_column_reduce(v, lane, [](float a, float b) { return a + b; });
}

// the same for W < 32 columns: lanes j, j + W, j + 2W, ... all end with the sum of column j over the warp's rows
template <int W>
__device__ __forceinline__ float warp_column_sum_part(float (&v)[W], int lane) {
#pragma unroll
  for (int half = W / 2; half >= 1; half >>= 1) {
    const bool upper = (lane & half) != 0;
#pragma unroll
    for (int i = 0; i < half; ++i) {
      const float send = upper ? v[i] : v[i + half];
      const float keep = upper ? v[i + half] : v[i];
      v[i] = keep + __shfl_xor_sync(0xffffffffu, send, half);
    }
  }
#pragma unroll
  for (int o = W; o < 32; o <<= 1) v[0] += __shfl_xor_sync(0xffffffffu, v[0], o);
  return v[0];
}

// Per-feature moments of the code (EpiEncodeT<ARITH, true>, evaluation only): each epilogue warp writes the column sums
// of c, c^2, c^3, c^4 over its 32 rows as fp32 partials [M][row_blocks][4][n], row block = global row / 32; a second
// kernel (moment_reduce_kernel) adds them up over the row blocks in a fixed order in fp64.
template <bool STATS>
struct EncodeMomentParams {};
template <>
struct EncodeMomentParams<true> {
  float* mom_part;   // [M][row_blocks][4][n]
  int row_blocks;    // ceil(B / 32)
};

// Batch-major copies of an epilogue's two 8-bit planes (T8 of EpiEncodeT and EpiDecodeT, f16f8 plans whose weight
// gradient runs native): [M][cols][ld], ld = batch_max rounded up to 16, as the weight gradient reads them (K-major over
// the batch). Written besides the row-major planes, straight from the epilogue's registers (store_col32_u8).
template <bool T8>
struct BatchMajorParams {};
template <>
struct BatchMajorParams<true> {
  uint8_t* t_lo;   // value-e5m2 plane
  uint8_t* t_x8;   // residual-e5m2 plane
  int t_ld;
};

// the batch-major copies of the 8-bit planes wx of the warp's 32 rows from row0 and 32 columns from col (T8)
__device__ __forceinline__ void store_batch_major(const BatchMajorParams<true>& P, const TileCoord& t, const uint32_t (&wx)[16],
                                                  int col, int row0, int m_total, int n_total) {
  const long long off = ((long long)t.model * n_total + col) * P.t_ld + row0;
  store_col32_u8(P.t_lo + off, P.t_ld, t.lane, &wx[0], m_total - row0, n_total - col);
  store_col32_u8(P.t_x8 + off, P.t_ld, t.lane, &wx[8], m_total - row0, n_total - col);
}

// ------------------------------------------------------------------------------------------------
// encode:  c = relu(acc + bias) -> (c_hi, c_lo);  per-tile partial sums of |c| and count(c > 0)
// [c > 0] and [z == 0] (clamp(min=0)'s gradient of 1 at exactly 0, SURVEY.md Q4) go to the activity masks, so the
// backward pass needs neither z nor the code.
// STATS (compile-time, evaluation only) adds the moment partials of EncodeMomentParams; the training instantiations
// (STATS = false) compile to the same code as without the switch.
// T8 (f16f8 training steps with a native weight gradient) also writes the batch-major copies of BatchMajorParams; the
// row-major planes are stored as without it (the decode GEMM reads the 8-bit ones).
// ------------------------------------------------------------------------------------------------
template <int ARITH, bool STATS = false, bool T8 = false>
struct EpiEncodeT {
  static_assert(!T8 || (ARITH == kArithF16F8 && !STATS), "batch-major copies: f16f8 training steps only");
  static constexpr int kCols = 32;
  static constexpr int kWarpStageBytes = 4096;
  static constexpr bool kInline = STATS;   // the moment sums do not fit the epilogue warpgroup's registers (sce_gemm.cuh)
  struct Params : EncodeMomentParams<STATS>, BatchMajorParams<T8> {
    CUtensorMap out_hi, out_lo, out_x8;  // store maps of the code planes: [M][B][n], box 32 x 32
    const float* bias;             // [M, n] or nullptr
    const unsigned char* mask;     // [M, n] (1 = coefficient unused) or nullptr
    float* part;                   // [M][tiles_m*8][tiles_n][2]  (sum c, nnz)
    int tiles_m, tiles_n;
    int flag_zero;                 // 1: record z == 0 (clamp semantics), 0: relu semantics
    ActMask act;                   // activity masks for the backward pass
  };
  const Params& P;
  const TileCoord& T;
  int m_total, n_total;
  uint8_t* stage;
  float l1 = 0.f;
  int nnz = 0;
  __device__ EpiEncodeT(const Params& p, const TileCoord& t, int m, int n, uint8_t* st)
      : P(p), T(t), m_total(m), n_total(n), stage(st) {}

  __device__ __forceinline__ void chunk(int c, const uint32_t (&r)[32]) {
    const int col = T.col0 + c;
    if (col >= n_total) return;  // warp-uniform
    const bool row_ok = T.row < m_total;
    uint32_t whi[16], wlo[16];
    const float* bias = P.bias ? P.bias + (long long)T.model * n_total + col : nullptr;
    float ls = 0.f;
    uint32_t pos = 0, zero = 0;   // activity-mask words of this row and chunk: bit (31 - j) is column j
    float cs[32];                 // STATS: the code of this row's chunk, 0 for rows beyond the batch
    if (col + 32 <= n_total && !P.mask && bias) {
      // fast path: whole chunk in range, no coefficient mask; bias fetched as 8 uniform float4.
      // Lean on purpose (this GEMM is bound by the SM's data paths, not by the tensor pipe): relu as max, the sign
      // bits shifted into one word, and ONE tracker — the smallest |z| — for the rare exact zeros, resolved after the loop
      float zmin = 1.f;
      uint32_t neg = 0;
#pragma unroll
      for (int j = 0; j < 32; j += 4) {
        const float4 b4 = __ldg(reinterpret_cast<const float4*>(bias + j));
        const float bb[4] = {b4.x, b4.y, b4.z, b4.w};
#pragma unroll
        for (int u = 0; u < 4; u += 2) {
          const float z0 = __uint_as_float(r[j + u]) + bb[u], z1 = __uint_as_float(r[j + u + 1]) + bb[u + 1];
          zmin = fminf(zmin, fminf(fabsf(z0), fabsf(z1)));
          neg = __funnelshift_l(__float_as_uint(z1), __funnelshift_l(__float_as_uint(z0), neg, 1), 1);
          const float c0 = fmaxf(z0, 0.f), c1 = fmaxf(z1, 0.f);
          split_pair<ARITH>(c0, c1, (j + u) >> 1, whi, wlo);
          ls += c0 + c1;
          if constexpr (STATS) {
            cs[j + u] = row_ok ? c0 : 0.f;
            cs[j + u + 1] = row_ok ? c1 : 0.f;
          }
        }
      }
      pos = ~neg;  // no zero among the 32 scores: positive <=> sign bit clear
      if (zmin == 0.f) {  // some score is exactly +-0: not positive; recorded for the clamp semantics
#pragma unroll
        for (int j = 0; j < 32; ++j) {
          const float z = __uint_as_float(r[j]) + __ldg(bias + j);
          if (z == 0.f) {
            pos &= ~(0x80000000u >> j);
            if (P.flag_zero) zero |= 0x80000000u >> j;
          }
        }
      }
    } else {
      const unsigned char* mask = P.mask ? P.mask + (long long)T.model * n_total + col : nullptr;
#pragma unroll
      for (int j = 0; j < 32; j += 2) {
        float cv[2];
#pragma unroll
        for (int u = 0; u < 2; ++u) {
          const bool col_ok = col + j + u < n_total;
          const float z = __uint_as_float(r[j + u]) + ((bias && col_ok) ? __ldg(bias + j + u) : 0.f);
          const bool masked = !col_ok || (mask && __ldg(mask + j + u));
          cv[u] = (z > 0.f && !masked) ? z : 0.f;
          if (cv[u] > 0.f) pos |= 0x80000000u >> (j + u);
          if (P.flag_zero && z == 0.f && !masked) zero |= 0x80000000u >> (j + u);
          ls += cv[u];
          if constexpr (STATS) cs[j + u] = row_ok ? cv[u] : 0.f;
        }
        split_pair<ARITH>(cv[0], cv[1], j >> 1, whi, wlo);
      }
    }
    if (row_ok) {
      l1 += ls;
      nnz += __popc(pos);
      const long long w = P.act.at(T.model, col >> 5, T.row);   // 32 lanes = 32 consecutive rows: coalesced
      P.act.pos[w] = pos;
      if (P.act.zero) P.act.zero[w] = zero;
    }
    stage_and_store<ARITH>(stage, T, whi, wlo, &P.out_hi, &P.out_lo, &P.out_x8, col, T.m_blk * kBM + T.warp_q * 32,
                           T.model);
    if constexpr (T8) store_batch_major(P, T, wlo, col, T.m_blk * kBM + T.warp_q * 32, m_total, n_total);
    if constexpr (STATS) {
      if (T.m_blk * kBM + T.warp_q * 32 < m_total) {   // warp-uniform: some row of this warp is in the batch
        float* o = P.mom_part + ((long long)T.model * P.row_blocks + T.m_blk * 4 + T.warp_q) * 4 * n_total + col + T.lane;
        const bool col_ok = col + T.lane < n_total;
#pragma unroll
        for (int p = 0; p < 4; ++p) {
          float v[32];
#pragma unroll
          for (int j = 0; j < 32; ++j) {
            const float c = cs[j], c2 = c * c;
            v[j] = p == 0 ? c : p == 1 ? c2 : p == 2 ? c2 * c : c2 * c2;
          }
          const float sum = warp_column_sum(v, T.lane);
          if (col_ok) o[(long long)p * n_total] = sum;
        }
      }
    }
  }
  __device__ __forceinline__ void finish() {
    if (T.lane == 0) tma_store_wait_read();  // the staging tiles must outlive their bulk stores
    const float a = warp_sum(l1), b = warp_sum(float(nnz));
    if (T.lane == 0 && T.m_blk * kBM < m_total) {
      float* o = P.part +
                 ((((long long)T.model * P.tiles_m + T.m_blk) * 8 + T.grp * 4 + T.warp_q) * P.tiles_n + T.n_blk) * 2;
      o[0] = a;
      o[1] = b;
    }
  }
};

// Column sums of g (EpiDecodeT<ARITH, true>, learned-centre variant only): each epilogue warp writes the sums of its 32
// rows of g = r * gscale per column as fp32 partials [M][tiles_m*4][d], laid out like the bias-gradient partials of
// EpiDcodeT; center_grad_kernel adds them up over the row blocks in a fixed order (sum_b g_b of the centre gradient).
template <bool GSUM>
struct DecodeGsumParams {};
template <>
struct DecodeGsumParams<true> {
  float* g_part;   // [M][tiles_m*4][d]
};

// Per-row squared residuals (EpiDecodeT<ARITH, GSUM, T8, true>, tracked training steps): each thread stores the sum of
// r^2 over its 64 columns of the tile before the warp reduction, [M][B][2 tiles_n] (index 2 n_blk + grp), so that
// sum_p row_part[m][r][p] / d is row r's error e_r, made of the same fp32 residuals whose sum is l_reconstruction.
template <bool ROWERR>
struct DecodeRowErrParams {};
template <>
struct DecodeRowErrParams<true> {
  float* row_part;   // [M][B][2 tiles_n]
};

// ------------------------------------------------------------------------------------------------
// decode:  r = acc - x;  partial sum r^2;  g = r * gscale -> planes of g;  optional x^ store
// bf16x3: gscale = 2/(B d) (g is the loss gradient). f16f8: gscale = 1 — the fp16 plane could not hold 2r/(Bd)
// (~1e-7), so the backward pass runs on the residual itself and its consumers carry the factor (dcode adds
// alpha d/2 instead of alpha/B; the weight- and bias-gradient outputs are multiplied by 2/(B d)).
// GSUM (compile-time) adds the column sums of DecodeGsumParams; there rows beyond the batch stay in the warp (as zeros)
// for the transpose-reduce. T8 (f16f8 training steps with a native weight gradient) also writes the batch-major copies
// of g's 8-bit planes (BatchMajorParams), through a lane-quad transpose for which the rows beyond the batch stay in the
// warp as well. ROWERR also stores each thread's partial sum of r^2 per row (DecodeRowErrParams). The instantiations
// without the switches compile to the same code as without them.
// ------------------------------------------------------------------------------------------------
template <int ARITH, bool GSUM = false, bool T8 = false, bool ROWERR = false>
struct EpiDecodeT {
  static_assert(!T8 || ARITH == kArithF16F8, "batch-major copies: f16f8 only");
  static constexpr int kCols = 32;
  static constexpr int kWarpStageBytes = 0;
  static constexpr bool kInline = true;   // a few percent of a tile beside a K = n main loop (sce_gemm.cuh)
  static constexpr bool kWarpRows = GSUM || T8;   // rows beyond the batch run the chunk with the warp (as zeros)
  struct Params : DecodeGsumParams<GSUM>, BatchMajorParams<T8>, DecodeRowErrParams<ROWERR> {
    const float* x;                // [B, d] (x_model_stride = 0) or [M, B, d]
    long long x_model_stride;
    uint16_t* g_hi;                // [M, B, d] 16-bit plane
    uint8_t* g_lo;                 // bf16x3: lo plane (2 B / element); f16f8: value-e5m2 plane
    uint8_t* g_x8;                 // f16f8: residual-e5m2 plane
    float* x_hat;                  // optional [M, B, d] fp32 (evaluation / parity tests)
    float* part;                   // [M][tiles_m*8][tiles_n]  (sum r^2)
    long long g_model_stride;      // batch_max*d (workspace pitch)
    long long xhat_model_stride;   // B*d (caller's tensor)
    int ld;                        // d
    int tiles_m, tiles_n;
    float gscale;                  // 2 / (B * d), or 1 (f16f8)
  };
  const Params& P;
  const TileCoord& T;
  int m_total, n_total;
  float sq = 0.f;
  float4 xn[8];  // the input row's next 32 columns, fetched one chunk ahead (hides the L2 latency of x behind
                 // the tail of the main loop / the previous chunk; with SPLIT_ACC the epilogue is on the critical path)
  __device__ __forceinline__ void fetch_x(int c) {
    const int col = T.col0 + c;
    const bool row_ok = T.row < m_total;
    const float* x = P.x + (long long)T.model * P.x_model_stride + (long long)T.row * P.ld + col;
#pragma unroll
    for (int j = 0; j < 8; ++j)
      xn[j] = (row_ok && col + 4 * j < n_total) ? __ldg(reinterpret_cast<const float4*>(x + 4 * j))
                                               : make_float4(0.f, 0.f, 0.f, 0.f);
  }
  __device__ EpiDecodeT(const Params& p, const TileCoord& t, int m, int n, uint8_t*) : P(p), T(t), m_total(m), n_total(n) {
    fetch_x(T.grp * 32);
  }

  __device__ __forceinline__ void chunk(int c, const uint32_t (&r)[32]) {
    const int col = T.col0 + c;
    float4 xc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) xc[j] = xn[j];
    fetch_x(c + 64);  // this warp's next chunk (harmless past the tile: predicated on n_total, unused)
    if constexpr (kWarpRows) {
      if (col >= n_total) return;  // warp-uniform
    } else {
      if (col >= n_total || T.row >= m_total) return;
    }
    const bool row_ok = !kWarpRows || T.row < m_total;
    const long long off = (long long)T.model * P.g_model_stride + (long long)T.row * P.ld + col;
    uint32_t whi[16], wlo[16];
    // GSUM: every row block of a tile in the batch writes its column sums (as EpiDcodeT's db_part); warp-uniform. They are
    // reduced 8 columns at a time as the loop goes, so that few values are live beside the split decode's accumulators
    const bool gsum = GSUM && T.m_blk * kBM < m_total;
    float gv[8], gs = 0.f;
#pragma unroll
    for (int j = 0; j < 32; j += 4) {
      const float4 xv = xc[j >> 2];
      const bool ok = row_ok && col + j < n_total;  // d % 4 == 0
      const float r0 = ok ? __uint_as_float(r[j]) - xv.x : 0.f, r1 = ok ? __uint_as_float(r[j + 1]) - xv.y : 0.f;
      const float r2 = ok ? __uint_as_float(r[j + 2]) - xv.z : 0.f, r3 = ok ? __uint_as_float(r[j + 3]) - xv.w : 0.f;
      sq += r0 * r0 + r1 * r1 + r2 * r2 + r3 * r3;
      split_pair<ARITH>(r0 * P.gscale, r1 * P.gscale, j >> 1, whi, wlo);
      split_pair<ARITH>(r2 * P.gscale, r3 * P.gscale, (j >> 1) + 1, whi, wlo);
      if constexpr (GSUM) {
        gv[j & 7] = r0 * P.gscale;   // this row's g as split, 0 outside the batch and the matrix
        gv[(j & 7) + 1] = r1 * P.gscale;
        gv[(j & 7) + 2] = r2 * P.gscale;
        gv[(j & 7) + 3] = r3 * P.gscale;
        if ((j & 7) == 4 && gsum) {   // columns j - 4 .. j + 3 -> lanes j - 4 .. j + 3 (and their copies)
          const float t = warp_column_sum_part<8>(gv, T.lane);
          if ((T.lane >> 3) == (j >> 3)) gs = t;
        }
      }
      if (P.x_hat && ok)
        *reinterpret_cast<float4*>(P.x_hat + (long long)T.model * P.xhat_model_stride + (long long)T.row * P.ld + col + j) =
            make_float4(__uint_as_float(r[j]), __uint_as_float(r[j + 1]), __uint_as_float(r[j + 2]),
                        __uint_as_float(r[j + 3]));
    }
    if (row_ok) {
      store_bf16x32(reinterpret_cast<__nv_bfloat16*>(P.g_hi) + off, whi, n_total - col);
      if constexpr (ARITH == kArithF16F8) {
#pragma unroll
        for (int q = 0; q < 2; ++q)
          if (q * 16 < n_total - col) {  // d % 16 == 0 in this arithmetic
            *reinterpret_cast<uint4*>(P.g_lo + off + q * 16) = make_uint4(wlo[4 * q], wlo[4 * q + 1], wlo[4 * q + 2], wlo[4 * q + 3]);
            *reinterpret_cast<uint4*>(P.g_x8 + off + q * 16) = make_uint4(wlo[8 + 4 * q], wlo[9 + 4 * q], wlo[10 + 4 * q], wlo[11 + 4 * q]);
          }
      } else {
        store_bf16x32(reinterpret_cast<__nv_bfloat16*>(P.g_lo) + off, wlo, n_total - col);
      }
    }
    if constexpr (T8) store_batch_major(P, T, wlo, col, T.m_blk * kBM + T.warp_q * 32, m_total, n_total);
    if constexpr (GSUM) {
      if (gsum && col + T.lane < n_total)
        P.g_part[(((long long)T.model * P.tiles_m + T.m_blk) * 4 + T.warp_q) * n_total + col + T.lane] = gs;
    }
  }
  __device__ __forceinline__ void finish() {
    if constexpr (ROWERR) {
      if (T.row < m_total) P.row_part[((long long)T.model * m_total + T.row) * (2 * P.tiles_n) + 2 * T.n_blk + T.grp] = sq;
    }
    const float a = warp_sum(sq);
    if (T.lane == 0 && T.m_blk * kBM < m_total)
      P.part[(((long long)T.model * P.tiles_m + T.m_blk) * 8 + T.grp * 4 + T.warp_q) * P.tiles_n + T.n_blk] = a;
  }
};

// ------------------------------------------------------------------------------------------------
// dcode:  dz = (acc + (alpha/B) [c > 0]) * [z >= 0]  -> (dz_hi, dz_lo);
//         per-warp column sums of dz (32 rows) -> bias-gradient partials
// T8 (f16f8): dz's 8-bit planes are written batch-major, [M][n][batch] (out_lo / out_x8 map that layout), which is
// how the weight gradient's native E5M2 path reads them (K-major over the batch); the fp16 plane stays row-major.
// ------------------------------------------------------------------------------------------------
template <int ARITH, bool T8 = false>
struct EpiDcodeT {
  static constexpr int kCols = 32;
  static constexpr int kWarpStageBytes = 4096;
  struct Params {
    CUtensorMap out_hi, out_lo, out_x8;  // store maps of the dz planes: [M][B][n] (T8: 8-bit ones [M][n][B]), box 32 x 32
    ActMask act;                  // [c > 0] / [z == 0] written by encode (or the top-k selection)
    const float* l1_over_b;        // [M]: alpha_m / B (f16f8: alpha_m d / 2, see EpiDecodeT)
    float* db_part;                // [M][tiles_m*4][n] or nullptr (no bias)
    int tiles_m;
    // f16f8: the 8-bit planes of dz the weight-gradient GEMM will read. dz meets x there (dz^T x): its value plane
    // multiplies x's RESIDUAL plane, which is all zeros for fp16-exact activations (*x_res_flag == 0: that cross term
    // is skipped, GemmParams::b_res_flag) — and with single-pass backward GEMMs neither 8-bit plane is read at all.
    const uint32_t* x_res_flag;    // device flag written by the batch split, or nullptr (unknown: write the plane)
    int planes;                    // planes the consumer reads at most (3, or 0 with single-pass backward)
  };
  const Params& P;
  const TileCoord& T;
  int m_total, n_total;
  uint8_t* stage;
  float aB;
  int planes;              // 8-bit planes of dz to write (see Params)
  uint32_t pos_n, zero_n;  // the mask words of this warp's next chunk, fetched one chunk ahead
  __device__ __forceinline__ void fetch_mask(int c) {
    const int col = T.col0 + c;
    pos_n = zero_n = 0u;
    if (T.row < m_total && col < n_total) {
      const long long w = P.act.at(T.model, col >> 5, T.row);
      pos_n = __ldg(P.act.pos + w);
      if (P.act.zero) zero_n = __ldg(P.act.zero + w);
    }
  }
  __device__ EpiDcodeT(const Params& p, const TileCoord& t, int m, int n, uint8_t* st)
      : P(p), T(t), m_total(m), n_total(n), stage(st) {
    aB = __ldg(P.l1_over_b + T.model);
    planes = P.planes;
    if (P.x_res_flag && __ldg(P.x_res_flag) == 0u) planes &= ~1;
    fetch_mask(T.grp * 32);
  }

  __device__ __forceinline__ void chunk(int c, const uint32_t (&r)[32]) {
    const int col = T.col0 + c;
    const uint32_t pos = pos_n, zero = zero_n;
    fetch_mask(c + 64);  // this warp's next chunk
    if (col >= n_total) return;  // warp-uniform
    float dz[32];
    uint32_t whi[16], wlo[16];
    if (zero == 0u) {   // the common case: gradient passes exactly where the coefficient is active
#pragma unroll
      for (int j = 0; j < 32; j += 2) {
        const float v0 = (pos & (0x80000000u >> j)) ? __uint_as_float(r[j]) + aB : 0.f;
        const float v1 = (pos & (0x40000000u >> j)) ? __uint_as_float(r[j + 1]) + aB : 0.f;
        dz[j] = v0;
        dz[j + 1] = v1;
        split_pair<ARITH>(v0, v1, j >> 1, whi, wlo);
      }
    } else {            // some z == 0: clamp passes the reconstruction gradient there, without the sparsity term
      const uint32_t gate = pos | zero;
#pragma unroll
      for (int j = 0; j < 32; j += 2) {
        const float v0 = (gate & (0x80000000u >> j)) ? __uint_as_float(r[j]) + ((pos & (0x80000000u >> j)) ? aB : 0.f) : 0.f;
        const float v1 = (gate & (0x40000000u >> j)) ? __uint_as_float(r[j + 1]) + ((pos & (0x40000000u >> j)) ? aB : 0.f) : 0.f;
        dz[j] = v0;
        dz[j + 1] = v1;
        split_pair<ARITH>(v0, v1, j >> 1, whi, wlo);
      }
    }
    stage_and_store<ARITH, T8>(stage, T, whi, wlo, &P.out_hi, &P.out_lo, &P.out_x8, col,
                               T.m_blk * kBM + T.warp_q * 32, T.model, planes);
    if (P.db_part && T.m_blk * kBM < m_total) {  // warp-uniform
      const float s = warp_column_sum(dz, T.lane);   // lane j: the sum of column j over the warp's rows
      if (col + T.lane < n_total)
        P.db_part[(((long long)T.model * P.tiles_m + T.m_blk) * 4 + T.warp_q) * n_total + col + T.lane] = s;
    }
  }
  __device__ __forceinline__ void finish() {
    if (T.lane == 0) tma_store_wait_read();
  }
};

// ------------------------------------------------------------------------------------------------
// scores of the top-k variant: acc -> fp32 [M][B][n] through the same staging + bulk-store path as the code planes
// (each epilogue warp owns a 4 KB tile of 32 rows x 128 B, 128-byte swizzle: a thread writes its row with eight
// conflict-free 16-byte stores, one lane hands the tile to the TMA engine, which writes full lines and clips the
// ragged edges). The plain per-thread stores of EpiStoreF32 touch 32 different lines per instruction — fine for
// the small weight-gradient output, but the scores GEMM (K = d only, 4 B per element out) was bound by them.
// ------------------------------------------------------------------------------------------------
struct EpiScoresTma {
  static constexpr int kCols = 32;
  static constexpr int kWarpStageBytes = 4096;
  struct Params {
    CUtensorMap out;   // [M][B][n] fp32, box 32 x 32
    // optional: largest order-preserving key (f2key) of every 32-column chunk of every row, [M][batch_max][n_chunks] —
    // the selection then reads these (1/32 of the scores) and only the chunks that can hold one of the k largest
    uint32_t* cmax = nullptr;
    int n_chunks = 0;
    long long cmax_model_stride = 0;   // batch_max * n_chunks
  };
  const Params& P;
  const TileCoord& T;
  int m_total, n_total;
  uint8_t* stage;
  __device__ EpiScoresTma(const Params& p, const TileCoord& t, int m, int n, uint8_t* st)
      : P(p), T(t), m_total(m), n_total(n), stage(st) {}
  __device__ __forceinline__ void chunk(int c, const uint32_t (&r)[32]) {
    const int col = T.col0 + c;
    if (col >= n_total) return;   // warp-uniform
    staging_wait(T);
    const int sw = T.lane & 7;
#pragma unroll
    for (int q = 0; q < 8; ++q)
      *reinterpret_cast<uint4*>(stage + T.lane * 128 + ((q ^ sw) << 4)) = make_uint4(r[4 * q], r[4 * q + 1], r[4 * q + 2], r[4 * q + 3]);
    fence_proxy_async_smem();
    __syncwarp();
    if (T.lane == 0) {
      tma_store_3d(&P.out, stage, col, T.m_blk * kBM + T.warp_q * 32, T.model);
      tma_store_commit();
    }
    if (P.cmax) {   // (kernel-uniform)
      const int valid = n_total - col;   // columns of this chunk inside the matrix (a multiple of 8)
      uint32_t mx = 0;
#pragma unroll
      for (int j = 0; j < 32; ++j) {
        const uint32_t u = r[j];
        const uint32_t key = u ^ ((uint32_t)((int32_t)u >> 31) | 0x80000000u);   // == f2key
        if (valid >= 32 || j < valid) mx = max(mx, key);
      }
      if (T.row < m_total)
        P.cmax[(long long)T.model * P.cmax_model_stride + (long long)T.row * P.n_chunks + (col >> 5)] = mx;
    }
  }
  __device__ __forceinline__ void finish() {
    if (T.lane == 0) tma_store_wait_read();
  }
};

// ------------------------------------------------------------------------------------------------
// centring GEMM (FunctionalTiedSAE.center, sae_ensemble.py:126-128): acc = rot (x - trans); out = acc * scale[col], fp32
// [M][B][d] — the per-model batch every later kernel of the step reads (split into operand planes by split_rows_kernel,
// subtracted from x^ by the decode epilogue).
// ------------------------------------------------------------------------------------------------
struct EpiCenter {
  static constexpr int kCols = 32;
  static constexpr int kWarpStageBytes = 0;
  struct Params {
    float* out;                // [M][B][ld]
    long long model_stride;    // elements between models of `out`
    int ld;
    const float* col_scale;    // [M][ld]
  };
  const Params& P;
  const TileCoord& T;
  int m_total, n_total;
  __device__ EpiCenter(const Params& p, const TileCoord& t, int m, int n, uint8_t*) : P(p), T(t), m_total(m), n_total(n) {}
  __device__ __forceinline__ void chunk(int c, const uint32_t (&r)[32]) {
    if (T.row >= m_total) return;
    const int col = T.col0 + c;
    float* o = P.out + (long long)T.model * P.model_stride + (long long)T.row * P.ld + col;
    const float* sc = P.col_scale + (long long)T.model * P.ld + col;
#pragma unroll
    for (int j = 0; j < 32; j += 4) {
      if (col + j < n_total) {   // n_total % 4 == 0
        const float4 s4 = __ldg(reinterpret_cast<const float4*>(sc + j));
        *reinterpret_cast<float4*>(o + j) = make_float4(__uint_as_float(r[j]) * s4.x, __uint_as_float(r[j + 1]) * s4.y,
                                                        __uint_as_float(r[j + 2]) * s4.z, __uint_as_float(r[j + 3]) * s4.w);
      }
    }
  }
  __device__ __forceinline__ void finish() {}
};

// ------------------------------------------------------------------------------------------------
// dictionary similarity (standard_metrics.py:270-303, 356-362): acc = <a_i, b_j> for the pair (model_a, model_b) of the
// tile (kPairTiles). The [na, nb] matrix never reaches HBM; per tile the epilogue leaves
//   row maxima   max over valid j of acc (each A atom's best match in B)       -> row_max keys [P][na]
//   column maxima max over valid i of acc (each B atom's best match in A)      -> col_max keys [P][nb]
//   self-pairs (model_a == model_b, capacity): the row sum of acc^2 of this tile's 64 columns of each group ->
//   sq_part [P][na][2 tiles_n], and the diagonal element -> diag [P][na]
// Maxima go through integer atomicMax on order-preserving keys (f2key): exact and independent of the order tiles finish
// in. The sums of squares are partials reduced in a fixed order afterwards (capacity_kernel), so a result is bitwise
// repeatable. Atoms at index >= rows[model] (masked stacks, and the zero rows TMA fills in beyond na / nb) enter no
// maximum and no sum: a zero row has cosine 0 and would win where every real cosine is negative.
// ------------------------------------------------------------------------------------------------
struct EpiSimilarity {
  static constexpr int kCols = 32;
  static constexpr int kWarpStageBytes = 0;
  static constexpr bool kPairTiles = true;
  struct Params {
    const int* pairs;      // [P][2]: model of A, model of B
    const int* a_rows;     // [Ma] valid atoms of each A model
    const int* b_rows;     // [Mb]
    uint32_t* row_max;     // [P][na] keys, zeroed by the caller; or nullptr
    uint32_t* col_max;     // [P][nb] keys, zeroed by the caller; or nullptr
    float* sq_part;        // [P][na][2 tiles_n] or nullptr (no capacity)
    float* diag;           // [P][na]
    int tiles_n;
  };
  const Params& P;
  const TileCoord& T;
  int m_total, n_total;
  int ra, rb;              // valid atoms of this pair's A and B models
  bool self;               // capacity partials wanted for this tile (self-pair)
  uint32_t rkey = 0u;      // this thread's row maximum over its chunks (key 0 is below every float)
  float sq = 0.f;
  __device__ EpiSimilarity(const Params& p, const TileCoord& t, int m, int n, uint8_t*) : P(p), T(t), m_total(m), n_total(n) {
    const int ma = __ldg(P.pairs + 2 * T.model), mb = __ldg(P.pairs + 2 * T.model + 1);
    ra = __ldg(P.a_rows + ma);
    rb = __ldg(P.b_rows + mb);
    self = P.sq_part != nullptr && ma == mb;
  }
  static __device__ __forceinline__ uint32_t key(uint32_t u) { return u ^ ((uint32_t)((int32_t)u >> 31) | 0x80000000u); }  // == f2key

  __device__ __forceinline__ void chunk(int c, const uint32_t (&r)[32]) {
    const int col = T.col0 + c;
    if (col >= rb) return;   // warp-uniform: no valid column in this chunk
    const int valid = rb - col;
    const bool row_ok = T.row < ra;
    uint32_t ck[32];
#pragma unroll
    for (int j = 0; j < 32; ++j) {
      const bool ok = row_ok && (valid >= 32 || j < valid);
      const uint32_t k = ok ? key(r[j]) : 0u;
      rkey = max(rkey, k);
      ck[j] = k;
      if (self && ok) {
        const float v = __uint_as_float(r[j]);
        sq += v * v;
        if (col + j == T.row) P.diag[(long long)T.model * m_total + T.row] = v;
      }
    }
    if (P.col_max && T.m_blk * kBM + T.warp_q * 32 < ra) {   // warp-uniform: some row of this warp is valid
      // lane j: the maximum of column j over the warp's rows
      const uint32_t m = warp_column_reduce(ck, T.lane, [](uint32_t a, uint32_t b) { return max(a, b); });
      if (T.lane < valid) atomicMax(P.col_max + (long long)T.model * n_total + col + T.lane, m);
    }
  }
  __device__ __forceinline__ void finish() {
    if (P.row_max && T.row < ra) atomicMax(P.row_max + (long long)T.model * m_total + T.row, rkey);
    if (self && T.row < m_total)
      P.sq_part[((long long)T.model * m_total + T.row) * (2 * P.tiles_n) + 2 * T.n_blk + T.grp] = sq;
  }
};

// ------------------------------------------------------------------------------------------------
// FastICA pass (sce_ica_pass, sklearn's logcosh nonlinearity): acc = u = unmix v of one row;
//   t = tanh(alpha u) -> (t_hi, t_lo), [rows][n], as EpiEncodeT writes the code
//   per warp of 32 rows, the column sums of g' = alpha (1 - t^2) over the rows < rows_valid -> g_part [row_block][n]
//   (row block = global row / 32; a second kernel adds them over the row blocks in a fixed order in fp64)
// The accurate tanhf, not tanh.approx.f32: its 2^-11 error would reach gx = sum t v unreduced. The padding rows of the
// last slice are zero (u = 0, t = 0 adds nothing to gx), but g' = alpha there: they are kept out of the sums.
// ------------------------------------------------------------------------------------------------
template <int ARITH>
struct EpiIcaT {
  static constexpr int kCols = 32;
  static constexpr int kWarpStageBytes = 4096;
  struct Params {
    CUtensorMap out_hi, out_lo, out_x8;  // store maps of the t planes: [1][rows][n], box 32 x 32
    float* g_part;                       // [ceil(rows_valid / 32)][n]
    float alpha;
    int rows_valid;                      // B: rows at or beyond it are padding
  };
  const Params& P;
  const TileCoord& T;
  int m_total, n_total;
  uint8_t* stage;
  __device__ EpiIcaT(const Params& p, const TileCoord& t, int m, int n, uint8_t* st)
      : P(p), T(t), m_total(m), n_total(n), stage(st) {}

  __device__ __forceinline__ void chunk(int c, const uint32_t (&r)[32]) {
    const int col = T.col0 + c;
    if (col >= n_total) return;  // warp-uniform
    const bool row_ok = T.row < P.rows_valid;
    uint32_t whi[16], wlo[16];
    float g[32];
#pragma unroll
    for (int j = 0; j < 32; j += 2) {
      const float t0 = tanhf(P.alpha * __uint_as_float(r[j])), t1 = tanhf(P.alpha * __uint_as_float(r[j + 1]));
      split_pair<ARITH>(t0, t1, j >> 1, whi, wlo);
      g[j] = row_ok ? P.alpha * (1.f - t0 * t0) : 0.f;
      g[j + 1] = row_ok ? P.alpha * (1.f - t1 * t1) : 0.f;
    }
    const int row0 = T.m_blk * kBM + T.warp_q * 32;
    stage_and_store<ARITH>(stage, T, whi, wlo, &P.out_hi, &P.out_lo, &P.out_x8, col, row0, T.model);
    if (row0 < P.rows_valid) {   // warp-uniform: some row of this warp is in the batch
      const float s = warp_column_sum(g, T.lane);
      if (col + T.lane < n_total) P.g_part[(long long)(row0 >> 5) * n_total + col + T.lane] = s;
    }
  }
  __device__ __forceinline__ void finish() {
    if (T.lane == 0) tma_store_wait_read();  // the staging tiles must outlive their bulk stores
  }
};

// ------------------------------------------------------------------------------------------------
// NMF projection (sce_nmf_project): acc = p = M v of one row -> fp32 [rows][k] through EpiScoresTma's staging and bulk
// stores; with `part`, per warp of 32 rows the column sums of max(p, 0)^2 and min(p, 0)^2 over the rows < m_total ->
// part [row_block][2][k] (fp32; a second kernel adds them over the row blocks in a fixed order in fp64). NNDSVD reads
// the norms of the positive and negative parts of X v_j from them.
// ------------------------------------------------------------------------------------------------
struct EpiNmfProject {
  static constexpr int kCols = 32;
  static constexpr int kWarpStageBytes = 4096;
  struct Params {
    CUtensorMap out;   // [1][rows][k] fp32, box 32 x 32
    float* part;       // [ceil(rows / 32)][2][k], or nullptr
  };
  const Params& P;
  const TileCoord& T;
  int m_total, n_total;
  uint8_t* stage;
  __device__ EpiNmfProject(const Params& p, const TileCoord& t, int m, int n, uint8_t* st)
      : P(p), T(t), m_total(m), n_total(n), stage(st) {}
  __device__ __forceinline__ void chunk(int c, const uint32_t (&r)[32]) {
    const int col = T.col0 + c;
    if (col >= n_total) return;   // warp-uniform
    const int row0 = T.m_blk * kBM + T.warp_q * 32;
    staging_wait(T);
    const int sw = T.lane & 7;
#pragma unroll
    for (int q = 0; q < 8; ++q)
      *reinterpret_cast<uint4*>(stage + T.lane * 128 + ((q ^ sw) << 4)) = make_uint4(r[4 * q], r[4 * q + 1], r[4 * q + 2], r[4 * q + 3]);
    fence_proxy_async_smem();
    __syncwarp();
    if (T.lane == 0) {
      tma_store_3d(&P.out, stage, col, row0, T.model);
      tma_store_commit();
    }
    if (P.part && row0 < m_total) {   // (warp-uniform) some row of this warp is in the batch
      const bool row_ok = T.row < m_total;
      float* o = P.part + (long long)(row0 >> 5) * 2 * n_total + col + T.lane;
      float s[32];
#pragma unroll
      for (int j = 0; j < 32; ++j) {
        const float v = row_ok ? __uint_as_float(r[j]) : 0.f;
        s[j] = v > 0.f ? v * v : 0.f;
      }
      const float sp = warp_column_sum(s, T.lane);
#pragma unroll
      for (int j = 0; j < 32; ++j) {
        const float v = row_ok ? __uint_as_float(r[j]) : 0.f;
        s[j] = v < 0.f ? v * v : 0.f;
      }
      const float sn = warp_column_sum(s, T.lane);
      if (col + T.lane < n_total) {
        o[0] = sp;
        o[n_total] = sn;
      }
    }
  }
  __device__ __forceinline__ void finish() {
    if (T.lane == 0) tma_store_wait_read();
  }
};

using EpiEncode = EpiEncodeT<kArithBf16x3>;
using EpiDecode = EpiDecodeT<kArithBf16x3>;
using EpiDcode = EpiDcodeT<kArithBf16x3>;

}  // namespace sce
