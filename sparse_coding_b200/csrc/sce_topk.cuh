// sce_topk.cuh — the k-sparse path of the TopK variant (TopKEncoder, autoencoders/topk_encoder.py:19-40).
//
// The reference's code is exactly k-sparse (k <= 64 of n = 3072 .. 12288 columns: <= 2 % dense), but it multiplies it as
// a dense matrix three more times (decode, code gradient, weight gradient). Here, after the scores GEMM:
//   topk_select2_kernel   per row: the k largest signed scores (ties by lowest column), ReLU -> (column, value) list,
//                         the dense operand planes of the code as "zero the row, scatter k entries", activity mask,
//                         per-row sum / count partials
//   topk_sparse_kernel    per row and slice of the activation width: x^ = sum_j c_j W_j from the k gathered rows of the
//                         normalised dictionary (fp32 copy, staged ONCE in shared memory by cp.async), the residual
//                         r = x^ - x, its square sum, the planes of g, and the k dot products g . W_j that are the
//                         code gradient at the selected entries                    (replaces two dense GEMMs)
//   topk_dz_scatter_kernel  sums the slices' dot products and writes the dense planes of the code gradient as
//                         "zero the row, scatter k entries" for the (dense, tensor-core) weight-gradient GEMM.
// Per model and step the sparse kernels move B k d 4 bytes of dictionary rows (L2-resident) instead of issuing
// 2 x 2 B n d tensor FLOPs twice over; the weight gradient stays a dense GEMM — at these densities (k/n ~ 0.5 %) a
// gather-based sparse dW moves as many bytes as the dense GEMM takes time (DESIGN.md section 4).
#pragma once
#include "sce_kernels.cuh"

namespace sce {

// one value -> its operand-plane entries at element offset `i` (scatter form of store_planes4)
template <int ARITH>
__device__ __forceinline__ void store_plane1(float v, void* hi, void* lo, void* x8, long long i) {
  if constexpr (ARITH == kArithF16F8) {
    uint32_t h16, h8, l8;
    split2_f16f8(v, 0.f, h16, h8, l8);
    reinterpret_cast<uint16_t*>(hi)[i] = (uint16_t)(h16 & 0xFFFFu);
    reinterpret_cast<uint8_t*>(lo)[i] = (uint8_t)(h8 & 0xFFu);
    reinterpret_cast<uint8_t*>(x8)[i] = (uint8_t)(l8 & 0xFFu);
  } else {
    __nv_bfloat16 h, l;
    split_bf16(v, h, l);
    reinterpret_cast<__nv_bfloat16*>(hi)[i] = h;
    reinterpret_cast<__nv_bfloat16*>(lo)[i] = l;
  }
}

// one element of every plane back to zero
template <int ARITH>
__device__ __forceinline__ void store_plane_zero(void* hi, void* lo, void* x8, long long i) {
  reinterpret_cast<uint16_t*>(hi)[i] = 0;
  if constexpr (ARITH == kArithF16F8) {
    reinterpret_cast<uint8_t*>(lo)[i] = 0;
    reinterpret_cast<uint8_t*>(x8)[i] = 0;
  } else {
    reinterpret_cast<uint16_t*>(lo)[i] = 0;
  }
}

// zero `count` consecutive elements (count % 8 == 0, offset % 8 == 0) of every plane with 16-byte stores, block-wide
template <int ARITH>
__device__ __forceinline__ void zero_planes_row(void* hi, void* lo, void* x8, long long off, int count) {
  const uint4 z = make_uint4(0u, 0u, 0u, 0u);
  uint4* h = reinterpret_cast<uint4*>(reinterpret_cast<uint16_t*>(hi) + off);
  for (int i = threadIdx.x; i < count / 8; i += blockDim.x) h[i] = z;
  if constexpr (ARITH == kArithF16F8) {
    // 8-bit planes: 16 elements per 16-byte store (n % 16 == 0 in this arithmetic)
    uint4* a = reinterpret_cast<uint4*>(reinterpret_cast<uint8_t*>(lo) + off);
    uint4* b = reinterpret_cast<uint4*>(reinterpret_cast<uint8_t*>(x8) + off);
    for (int i = threadIdx.x; i < count / 16; i += blockDim.x) {
      a[i] = z;
      b[i] = z;
    }
  } else {
    uint4* a = reinterpret_cast<uint4*>(reinterpret_cast<uint16_t*>(lo) + off);
    for (int i = threadIdx.x; i < count / 8; i += blockDim.x) a[i] = z;
  }
}

// k-sparse lists of one plan: entry e of row r of model m at ((m * batch_max + r) * kmax + e)
struct TopkLists {
  int* col;        // selected column, in the order the selection produced it
  float* val;      // relu(score) of that column (0 for a selected negative score: L0 < k, topk_encoder.py:24-27)
  int* cnt;        // [M][batch_max]: entries of the row (min(k, n))
  int kmax;        // capacity per row (0: lists not kept)
  int batch_max;
};

// ------------------------------------------------------------------------------------------------
// selection. One 256-thread block per (row, model). The row is read twice with 16-byte loads — the second time out
// of L2 — instead of being parked in shared memory: 9 KB of shared memory per block keep eight blocks on an SM
// (with the keys in shared memory, 24-49 KB per row, the kernel sat at 37 % warp occupancy and 44 % of the DRAM rate).
//   1. first pass over the row: per-thread maximum of the order-preserving keys. Meanwhile the row of the code planes
//      and of the activity mask is returned to all-zero: with lists (the plan knows k) by clearing the entries the
//      PREVIOUS call scattered — the planes start zeroed (sce_prepare) and every write to them is recorded in the
//      row's list, so k clears replace rewriting n zeros (half of this kernel's DRAM traffic) —, else by zeroing it.
//      In k-sparse plans the code-gradient planes are kept the same way (topk_dz_scatter_kernel only scatters).
//   2. a lower bound of the k-th largest key: every warp sorts its 32 thread maxima, takes its ceil(k/8)-th largest;
//      the minimum over the 8 warps has at least k elements at or above it
//   3. second pass: the keys >= bound (typically 1-3 k of them) are compacted into a candidate list
//   4. exact rank of every candidate by counting (keys made unique by the column: ties go to the lowest column):
//      rank < k <=> selected, and rank is its slot in the list               — no sort, no radix passes
//      (more candidates than the list holds — k > 256, many equal scores — : 4-pass radix select re-reading the row
//      each pass, then an ordered compaction, as the first version of this kernel did for every row from shared memory)
//   5. scatter the k entries into the zeroed planes, activity-mask bits, (column, value) list, per-row partials
// With the chunk maxima of the scores epilogue (`cmax`: the largest key of every 32-column chunk of the row, written by
// EpiScoresTma) steps 1 and 3 do not read the row: the thread maxima of step 1 are taken over the chunk maxima (chunk i
// belongs to thread i % 256; the bound of step 2 then uses the warps whose 32 lanes all own a chunk), and step 3 lists the
// chunks whose maximum reaches the bound and reads only those, a warp per 128-byte chunk. Rows with fewer than 32 chunks,
// or with k beyond 32 per such warp, take the two full passes.
// ------------------------------------------------------------------------------------------------
constexpr int kTopkCand = 1024;
__device__ __forceinline__ unsigned long long pack_cand(uint32_t key, int col) {
  return ((unsigned long long)key << 32) | (uint32_t)(0x7FFFFFFF - col);
}
__device__ __forceinline__ uint32_t cand_key_of(unsigned long long c) { return (uint32_t)(c >> 32); }
__device__ __forceinline__ int cand_col_of(unsigned long long c) { return 0x7FFFFFFF - (int)(uint32_t)c; }
constexpr int kTopkChunkList = 2048;   // 32-column chunks of a row the chunk-maxima path can list (n <= 65536)

template <int ARITH>
__global__ void __launch_bounds__(256) topk_select2_kernel(const float* __restrict__ scores,
                                                           const long long* __restrict__ sparsity,
                                                           void* __restrict__ c_hi, void* __restrict__ c_lo,
                                                           void* __restrict__ c_x8, void* __restrict__ dz_hi,
                                                           void* __restrict__ dz_lo, void* __restrict__ dz_x8,
                                                           ActMask act, TopkLists lists,
                                                           float* __restrict__ part /*[M][B][2]*/, int B, int n,
                                                           long long model_stride /*elements between models*/,
                                                           const uint32_t* __restrict__ cmax /*[M][batch_max][n_chunks] or nullptr*/) {
  constexpr int UNROLL = 4;
  __shared__ uint16_t chunk_list[kTopkChunkList];
  __shared__ uint32_t sh_nchunk;
  // candidates as one 64-bit word: key in the high half, (0x7FFFFFFF - column) in the low half — a strict order in which
  // "larger" means larger key, or equal key and lower column (ties go to the lowest column)
  __shared__ unsigned long long cand[kTopkCand];
  __shared__ int cand_rank[kTopkCand];
  __shared__ uint32_t hist[256];
  __shared__ uint32_t sh_prefix, sh_remaining, sh_ncand, sh_neq, sh_kept, sh_ties;
  __shared__ uint32_t warp_cnt[8], warp_cnt2[8], warp_bound[8];
  __shared__ float redf[16];
  const int model = blockIdx.y;
  const int row = blockIdx.x;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long long base = (long long)model * model_stride + (long long)row * n;
  const int n4 = n >> 2;
  int k = (int)sparsity[model];
  if (k > n) k = n;
  if (threadIdx.x == 0) {
    sh_ncand = 0;
    sh_kept = 0;
    sh_ties = 0;
    sh_nchunk = 0;
  }
  // Chunk maxima from the scores epilogue (EpiScoresTma): chunk i belongs to thread i % 256, so the first
  // n_chunks / 32 warps hold a real element of the row in every lane. The bound below is then taken over those warps
  // only: `full_warps` warps x their j-th largest maximum, j = ceil(k / full_warps) <= 32, are >= k elements.
  const int n_chunks = act.n_chunks;
  const int full_warps = min(8, n_chunks >> 5);
  const int j_pick = full_warps ? (k + full_warps - 1) / full_warps : 33;
  const bool fused = cmax != nullptr && k <= 256 && j_pick <= 32 && n_chunks <= kTopkChunkList;   // block-uniform
  const uint32_t* cm = fused ? cmax + ((long long)model * act.batch_max + row) * n_chunks : nullptr;
  // ---- 1. first pass over the row: per-thread maximum; meanwhile clear this row of the outputs
  uint32_t my_max = 0;
  const float4* src4 = reinterpret_cast<const float4*>(scores + base);
  auto key4 = [&](int i) {   // keys of elements 4i .. 4i+3 (i < n4)
    const float4 v = __ldg(src4 + i);
    return make_uint4(f2key(v.x), f2key(v.y), f2key(v.z), f2key(v.w));
  };
  if (fused) {
    for (int i = threadIdx.x; i < n_chunks; i += 256) my_max = max(my_max, __ldg(cm + i));
  } else
  for (int i0 = 0; i0 < n4; i0 += 256 * UNROLL) {
    float4 v[UNROLL];
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) {
      const int i = i0 + u * 256 + threadIdx.x;
      v[u] = i < n4 ? __ldg(src4 + i) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) {
      const int i = i0 + u * 256 + threadIdx.x;
      if (i < n4) {
        const uint4 kk = make_uint4(f2key(v[u].x), f2key(v[u].y), f2key(v[u].z), f2key(v[u].w));
        my_max = max(max(my_max, kk.x), max(kk.y, max(kk.z, kk.w)));
      }
    }
  }
  const long long lbase = lists.kmax ? ((long long)model * lists.batch_max + row) * lists.kmax : 0;
  if (lists.kmax) {
    // clear what the previous call left in this row (dz_* != nullptr: k-sparse plan, same entries in the code gradient)
    const int old = lists.cnt[(long long)model * lists.batch_max + row];
    for (int j = threadIdx.x; j < old; j += 256) {
      const int col = lists.col[lbase + j];
      store_plane_zero<ARITH>(c_hi, c_lo, c_x8, base + col);
      if (dz_hi) store_plane_zero<ARITH>(dz_hi, dz_lo, dz_x8, base + col);
      act.pos[act.at(model, col >> 5, row)] = 0u;   // (several old entries may share the word: they all write 0)
    }
  } else {
    zero_planes_row<ARITH>(c_hi, c_lo, c_x8, base, n);
    for (int ch = threadIdx.x; ch < act.n_chunks; ch += 256) act.pos[act.at(model, ch, row)] = 0u;
  }
  // ---- 2. lower bound of the k-th largest key
  uint32_t bound = 0;   // k > 256: every key is a candidate (the radix path below takes over)
  if (k <= 256) {
    uint32_t v = my_max;   // bitonic sort of the warp's 32 maxima, descending by lane
#pragma unroll
    for (int size = 2; size <= 32; size <<= 1) {
#pragma unroll
      for (int stride = size >> 1; stride > 0; stride >>= 1) {
        const uint32_t o = __shfl_xor_sync(0xffffffffu, v, stride);
        const bool up = ((lane & size) == 0) == ((lane & stride) == 0);   // this lane keeps the larger of the pair
        v = up ? max(v, o) : min(v, o);
      }
    }
    // 8 warps x j elements >= their j-th largest: at least k elements >= the minimum (fused: the full warps only)
    const int j = fused ? j_pick : (k + 7) >> 3;
    if (lane == j - 1) warp_bound[warp] = v;
  }
  __syncthreads();
  if (k <= 256) {
    const int nw = fused ? full_warps : 8;
    bound = warp_bound[0];
    for (int w = 1; w < nw; ++w) bound = min(bound, warp_bound[w]);
  }
  // ---- 3. candidates
  if (fused) {
    // only the chunks whose maximum reaches the bound can hold a candidate: list them, then a warp per listed chunk
    // reads its 128 bytes (four chunks in flight per warp)
    for (int i = threadIdx.x; i < n_chunks; i += 256)
      if (__ldg(cm + i) >= bound) chunk_list[atomicAdd(&sh_nchunk, 1u)] = (uint16_t)i;
    __syncthreads();
    const int nch = (int)sh_nchunk;
    for (int c0 = warp * 4; c0 < nch; c0 += 32) {
      float v[4];
      int col[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        col[u] = c0 + u < nch ? (int)chunk_list[c0 + u] * 32 + lane : n;
        v[u] = col[u] < n ? __ldg(scores + base + col[u]) : 0.f;
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const uint32_t kv = f2key(v[u]);
        if (col[u] < n && kv >= bound) {
          const uint32_t slot = atomicAdd(&sh_ncand, 1u);
          if (slot < kTopkCand) cand[slot] = pack_cand(kv, col[u]);
        }
      }
    }
  } else
  // (second pass over the row, L2-resident)
  for (int i0 = 0; i0 < n4; i0 += 256 * UNROLL) {
    float4 v[UNROLL];
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) {
      const int i = i0 + u * 256 + threadIdx.x;
      v[u] = i < n4 ? __ldg(src4 + i) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) {
      const int i = i0 + u * 256 + threadIdx.x;
      if (i >= n4) continue;
      const uint32_t kv[4] = {f2key(v[u].x), f2key(v[u].y), f2key(v[u].z), f2key(v[u].w)};
#pragma unroll
      for (int e = 0; e < 4; ++e)
        if (kv[e] >= bound) {
          const uint32_t slot = atomicAdd(&sh_ncand, 1u);
          if (slot < kTopkCand) cand[slot] = pack_cand(kv[e], 4 * i + e);
        }
    }
  }
  __syncthreads();
  const int ncand = (int)sh_ncand;
  float l1 = 0.f, cnt = 0.f;
  auto emit = [&](int slot, int col, uint32_t key) {   // entry `slot` of the selection: column `col`
    const float v = key2relu(key);
    store_plane1<ARITH>(v, c_hi, c_lo, c_x8, base + col);
    if (v > 0.f) {
      atomicOr(&act.pos[act.at(model, col >> 5, row)], 0x80000000u >> (col & 31));
      l1 += v;
      cnt += 1.f;
    }
    if (lists.kmax && slot < lists.kmax) {
      lists.col[lbase + slot] = col;
      lists.val[lbase + slot] = v;
    }
  };
  if (ncand <= kTopkCand) {
    // ---- 4. exact ranks by counting: rank = candidates above this one; rank < k <=> selected, and rank is its slot.
    // The ncand^2 comparisons are the bulk of this kernel's instructions: one 64-bit
    // broadcast load and compare per pair, and every candidate's count is split over `parts` threads so that all 256
    // threads count (typically ncand = 2-3 k < 256).
    const int parts = ncand >= kTopkCand ? 1 : min(8, (kTopkCand + ncand - 1) / max(ncand, 1));
    if (parts == 1) {
      for (int i = threadIdx.x; i < ncand; i += 256) {
        const unsigned long long ci = cand[i];
        int rank = 0;
#pragma unroll 8
        for (int j = 0; j < ncand; ++j) rank += cand[j] > ci ? 1 : 0;
        if (rank < k) emit(rank, cand_col_of(ci), cand_key_of(ci));
      }
    } else {
      for (int i = threadIdx.x; i < ncand; i += 256) cand_rank[i] = 0;
      __syncthreads();
      const int seg = (ncand + parts - 1) / parts;
      for (int w = threadIdx.x; w < ncand * parts; w += 256) {
        const int part = w / ncand, i = w - part * ncand;
        const int j0 = part * seg, j1 = min(ncand, j0 + seg);
        const unsigned long long ci = cand[i];
        int cntp = 0;
#pragma unroll 8
        for (int j = j0; j < j1; ++j) cntp += cand[j] > ci ? 1 : 0;
        atomicAdd(&cand_rank[i], cntp);
      }
      __syncthreads();
      for (int i = threadIdx.x; i < ncand; i += 256) {
        const int rank = cand_rank[i];
        const unsigned long long ci = cand[i];
        if (rank < k) emit(rank, cand_col_of(ci), cand_key_of(ci));
      }
    }
  } else {
    // ---- 4'. exact 4-pass 8-bit radix select over the keys >= bound, then an ordered compaction (column order)
    if (threadIdx.x == 0) {
      sh_prefix = 0;
      sh_remaining = (uint32_t)k;
    }
    for (int pass = 0; pass < 4; ++pass) {
      const int shift = 24 - 8 * pass;
      hist[threadIdx.x] = 0;
      __syncthreads();
      const uint32_t prefix = sh_prefix;
      const uint32_t pmask = pass == 0 ? 0u : (0xFFFFFFFFu << (shift + 8));
      for (int i0 = 0; i0 < n; i0 += 256) {
        const int i = i0 + threadIdx.x;
        const uint32_t kk = i < n ? f2key(__ldg(scores + base + i)) : 0u;
        hist_add(hist, (kk >> shift) & 0xFF, i < n && kk >= bound && (kk & pmask) == prefix);
      }
      __syncthreads();
      pick_bin(hist, &sh_prefix, &sh_remaining, warp_cnt, shift, pass == 3 ? &sh_neq : nullptr);
    }
    const uint32_t kth = sh_prefix;           // exact key of the k-th largest
    const uint32_t take_ties = sh_remaining;  // how many of the elements == kth to keep (the lowest columns)
    for (int i0 = 0; i0 < n4; i0 += 256) {
      const int i = i0 + threadIdx.x;
      uint4 kk = make_uint4(0, 0, 0, 0);
      if (i < n4) kk = key4(i);
      const uint32_t kv[4] = {kk.x, kk.y, kk.z, kk.w};
      int ties = 0, greater = 0;
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        ties += (i < n4 && kv[u] == kth) ? 1 : 0;
        greater += (i < n4 && kv[u] > kth) ? 1 : 0;
      }
      // exclusive prefixes over the block, in element order (thread t owns elements 4i .. 4i+3)
      int inc_t = ties, inc_g = greater;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int a = __shfl_up_sync(0xffffffffu, inc_t, o), b = __shfl_up_sync(0xffffffffu, inc_g, o);
        if (lane >= o) {
          inc_t += a;
          inc_g += b;
        }
      }
      if (lane == 31) {
        warp_cnt[warp] = (uint32_t)inc_t;
        warp_cnt2[warp] = (uint32_t)inc_g;
      }
      __syncthreads();
      uint32_t ties_before = sh_ties + (uint32_t)(inc_t - ties), greater_before = sh_kept + (uint32_t)(inc_g - greater);
      for (int w = 0; w < warp; ++w) {
        ties_before += warp_cnt[w];
        greater_before += warp_cnt2[w];
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        if (i >= n4) break;
        const bool tie = kv[u] == kth, gt = kv[u] > kth;
        if (gt || (tie && ties_before < take_ties)) {
          // slot: elements kept before this one = greater ones before + min(ties before, take_ties)
          emit((int)(greater_before + (ties_before < take_ties ? ties_before : take_ties)), 4 * i + u, kv[u]);
        }
        if (tie) ++ties_before;
        if (gt) ++greater_before;
      }
      __syncthreads();
      if (threadIdx.x == 0) {
        uint32_t a = 0, b = 0;
        for (int w = 0; w < 8; ++w) {
          a += warp_cnt[w];
          b += warp_cnt2[w];
        }
        sh_ties += a;
        sh_kept += b;
      }
      __syncthreads();
    }
  }
  if (lists.kmax && threadIdx.x == 0) lists.cnt[(long long)model * lists.batch_max + row] = k < lists.kmax ? k : lists.kmax;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    l1 += __shfl_xor_sync(0xffffffffu, l1, o);
    cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
  }
  if (lane == 0) {
    redf[warp] = l1;
    redf[8 + warp] = cnt;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    float a = 0, b = 0;
    for (int w = 0; w < 8; ++w) {
      a += redf[w];
      b += redf[8 + w];
    }
    part[((long long)model * B + row) * 2] = a;
    part[((long long)model * B + row) * 2 + 1] = b;
  }
}

// ------------------------------------------------------------------------------------------------
// sparse decode + residual + code gradient at the selected entries. One 256-thread block per (row, model, slice of the
// activation width; the plan picks 2 or 4 slices so that several blocks fit an SM). The k selected rows of the
// NORMALISED dictionary (an fp32 copy kept by the dictionary-row kernel for these plans: no unpacking in the inner
// loops) are fetched ONCE into shared memory with 16-byte cp.async; warp w then owns the entries w, w+8, ... and its
// lanes the column groups.
//   pass 1  x^ = sum_j c_j W_j (per-warp partial sums, added in a fixed order), r = x^ - x, sum r^2 -> part[row][slice],
//           g = r * gscale -> operand planes of g (what the dense weight-gradient GEMM reads), optional fp32 x^
//   pass 2  dots[row][j][slice] = sum_t g_t W_jt   (topk_dz_scatter_kernel adds the slices)
// Shared memory: kmax * ds * 4 bytes of dictionary rows, 8 * ds floats of partial sums, ds floats of g.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gsrc) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(smem_dst)), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() {
  asm volatile("cp.async.commit_group;\n\tcp.async.wait_group 0;" ::: "memory");
}

template <int ARITH>
__global__ void __launch_bounds__(256) topk_sparse_kernel(TopkLists lists, const long long* __restrict__ sparsity,
                                                          const float* __restrict__ wn /*[M][n][d]*/,
                                                          const float* __restrict__ x, long long x_model_stride,
                                                          void* __restrict__ g_hi, void* __restrict__ g_lo,
                                                          void* __restrict__ g_x8, float* __restrict__ x_hat,
                                                          float* __restrict__ part /*[M][B][slices]*/,
                                                          float* __restrict__ dots /*[M][batch_max][kmax][slices]*/,
                                                          int B, int n, int d, float gscale,
                                                          const int* __restrict__ models /*this launch's models or nullptr*/,
                                                          int krows /*shared-memory rows: >= the k of every model of the launch*/) {
  extern __shared__ __align__(128) uint8_t smem_b[];
  __shared__ float red[8];
  // (a launch covers the models of one k class, so that its blocks take k x slice bytes of shared memory, not k_max x)
  const int row = blockIdx.x, model = models ? __ldg(models + blockIdx.y) : (int)blockIdx.y, slice = blockIdx.z, slices = gridDim.z;
  const int ds = d / slices, groups = ds >> 2;   // this block's columns, float4 groups of them
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int kmax = lists.kmax;
  float* s_w = reinterpret_cast<float*>(smem_b);            // [krows][ds]
  float* s_part = s_w + (size_t)krows * ds;                  // [8][ds]
  float* s_g = s_part + 8 * ds;                              // [ds]
  float* s_val = s_g + ds;                                   // [krows]
  const long long lrow = (long long)model * lists.batch_max + row;
  // entries of the row = min(k, n, kmax), as the selection wrote them (no dependent load of lists.cnt)
  int cnt = (int)min((long long)min(min(n, kmax), krows), __ldg(sparsity + model));
  // ---- gather: entry j, 16-byte piece q of its slice; every thread reads the column of its entry itself (one
  // dependent global load before the copies are in flight, not two), values and the x row are fetched alongside
  // (warp per entry: ONE column load and one base address per dictionary row, lanes stride its 16-byte pieces — the first
  //  version spread the pieces over all threads and paid an integer division, 64-bit address arithmetic and a dependent
  //  column load per PIECE)
  {
    const float* wn_slice = wn + (long long)model * n * d + (long long)slice * ds;
    const int* cols = lists.col + lrow * kmax;
#pragma unroll 4
    for (int j = warp; j < cnt; j += 8) {
      const float* src = wn_slice + (long long)__ldg(cols + j) * d;
      float* dst = s_w + (size_t)j * ds;
      for (int q = lane; q < groups; q += 32) cp_async16(dst + 4 * q, src + 4 * q);
    }
  }
  for (int j = threadIdx.x; j < cnt; j += 256) s_val[j] = __ldg(lists.val + lrow * kmax + j);
  float4 xv_pre = make_float4(0.f, 0.f, 0.f, 0.f);   // (groups <= 128 < 256 threads: one column group per thread)
  if (threadIdx.x < groups)
    xv_pre = __ldg(reinterpret_cast<const float4*>(x + (long long)model * x_model_stride + (long long)row * d +
                                                   (long long)slice * ds + 4 * threadIdx.x));
  cp_async_wait_all();
  __syncthreads();
  // ---- pass 1: partial x^ of this warp's entries
  constexpr int GP = 4;   // column groups per lane held in registers (ds <= 4 * 32 * GP = 512 columns per slice)
  float4 acc[GP];
#pragma unroll
  for (int i = 0; i < GP; ++i) acc[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int j = warp; j < cnt; j += 8) {
    const float c = s_val[j];
    if (c == 0.f) continue;   // (warp-uniform) a selected negative score
    const float4* w4 = reinterpret_cast<const float4*>(s_w + (size_t)j * ds);
#pragma unroll
    for (int i = 0; i < GP; ++i) {
      const int g = lane + 32 * i;
      if (g < groups) {
        const float4 w = w4[g];
        acc[i].x = fmaf(c, w.x, acc[i].x);
        acc[i].y = fmaf(c, w.y, acc[i].y);
        acc[i].z = fmaf(c, w.z, acc[i].z);
        acc[i].w = fmaf(c, w.w, acc[i].w);
      }
    }
  }
#pragma unroll
  for (int i = 0; i < GP; ++i) {
    const int g = lane + 32 * i;
    if (g < groups) reinterpret_cast<float4*>(s_part + warp * ds)[g] = acc[i];
  }
  __syncthreads();
  float sq = 0.f;
  for (int g = threadIdx.x; g < groups; g += 256) {
    float4 xh = reinterpret_cast<const float4*>(s_part)[g];
#pragma unroll
    for (int w = 1; w < 8; ++w) {   // fixed order: bit-identical from run to run
      const float4 pw = reinterpret_cast<const float4*>(s_part + w * ds)[g];
      xh.x += pw.x;
      xh.y += pw.y;
      xh.z += pw.z;
      xh.w += pw.w;
    }
    const long long col = (long long)slice * ds + 4 * g;
    const float4 xv = xv_pre;   // g == threadIdx.x
    const float4 r = make_float4(xh.x - xv.x, xh.y - xv.y, xh.z - xv.z, xh.w - xv.w);
    sq += r.x * r.x + r.y * r.y + r.z * r.z + r.w * r.w;
    const float gv[4] = {r.x * gscale, r.y * gscale, r.z * gscale, r.w * gscale};
    reinterpret_cast<float4*>(s_g)[g] = make_float4(gv[0], gv[1], gv[2], gv[3]);
    store_planes4<ARITH>(gv, g_hi, g_lo, g_x8, (lrow * d + col) >> 2);
    if (x_hat) *reinterpret_cast<float4*>(x_hat + ((long long)model * B + row) * d + col) = xh;
  }
  sq = warp_sum(sq);
  if (lane == 0) red[warp] = sq;
  __syncthreads();
  if (threadIdx.x == 0)
    part[((long long)model * B + row) * slices + slice] =
        ((red[0] + red[1]) + (red[2] + red[3])) + ((red[4] + red[5]) + (red[6] + red[7]));
  // ---- pass 2: this slice's share of g . W_j for the warp's entries
  if (dots) {
    float4 gr[GP];
#pragma unroll
    for (int i = 0; i < GP; ++i) {
      const int g = lane + 32 * i;
      gr[i] = g < groups ? reinterpret_cast<const float4*>(s_g)[g] : make_float4(0.f, 0.f, 0.f, 0.f);
    }
    for (int j = warp; j < cnt; j += 8) {
      const float4* w4 = reinterpret_cast<const float4*>(s_w + (size_t)j * ds);
      float dot = 0.f;
#pragma unroll
      for (int i = 0; i < GP; ++i) {
        const int g = lane + 32 * i;
        if (g < groups) {
          const float4 w = w4[g];
          dot = fmaf(gr[i].x, w.x, fmaf(gr[i].y, w.y, fmaf(gr[i].z, w.z, fmaf(gr[i].w, w.w, dot))));
        }
      }
      dot = warp_sum(dot);
      if (lane == 0) dots[(lrow * kmax + j) * slices + slice] = dot;
    }
  }
}

// dense operand planes of the code gradient for the weight-gradient GEMM: scatter the k entries into the zeroed row
//   dz[row][col_j] = [c_j > 0] * sum_slices dots[row][j][slice]              (relu: no gradient at exactly 0)
template <int ARITH>
__global__ void __launch_bounds__(64) topk_dz_scatter_kernel(TopkLists lists, const float* __restrict__ dots, int slices,
                                                              void* __restrict__ dz_hi, void* __restrict__ dz_lo,
                                                              void* __restrict__ dz_x8, int n) {
  const int row = blockIdx.x, model = blockIdx.y;
  const long long lrow = (long long)model * lists.batch_max + row;
  const int cnt = lists.cnt[lrow];   // (the row is all-zero: the selection cleared the previous step's entries)
  for (int j = threadIdx.x; j < cnt; j += 64) {
    const long long e = lrow * lists.kmax + j;
    if (lists.val[e] > 0.f) {
      float v = 0.f;
      for (int sidx = 0; sidx < slices; ++sidx) v += dots[e * slices + sidx];   // fixed order
      store_plane1<ARITH>(v, dz_hi, dz_lo, dz_x8, lrow * n + lists.col[e]);
    }
  }
}

}  // namespace sce
