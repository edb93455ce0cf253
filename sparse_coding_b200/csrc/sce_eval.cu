// sce_eval.cu — the entry points that read a plan's call back: the dense code (sce_read_code), activation counts
// (sce_active_counts), the evaluation statistics of a forward pass (sce_forward_stats), its top-activating and
// random activating fragments (sce_forward_fragments), the top- and rest-feature errors (sce_forward_split) and the
// expected interference of its code (sce_code_interference; sce_expected_interference for a caller-held code).
#include "sce_plan.cuh"

namespace sce {
__global__ void __launch_bounds__(256) active_count_kernel(const uint32_t* __restrict__ pos, int n_chunks, int batch_max,
                                                           int B, int n, int* __restrict__ counts) {
  active_count_block(pos, n_chunks, batch_max, B, n, counts, blockIdx.x, blockIdx.y);
}
}  // namespace sce

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
// segments of `seg`; counts[m][j] += number of segments that END in this call in which some row has [c > 0] in column j
// ([c != 0] for SCE_CODE_LINEAR plans, whose activity mask holds that; the reference tests the segment's mean of c for
// != 0, standard_metrics.py:498, which differs only where a segment's non-zero values cancel exactly).
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

// The workspace of one forward-stats call: the moment partials [M][ceil(B / 32)][4][n] fp32. With base == nullptr only
// measures it.
static size_t stats_carve(uint8_t* base, const sce_desc& d, int B, float** part) {
  Carve c{base, 0};
  float* mp = c.take<float>((size_t)d.n_models * ((B + 31) / 32) * 4 * d.n);
  if (part) *part = mp;
  return align_up(c.off, 1024);
}

// ------------------------------------------------------------------------------------------------
// the code of the plan's last call, as the engine holds it (sce_read_code, sce_forward_fragments)
// ------------------------------------------------------------------------------------------------
// Where a CodeView reads the code from. The row-major operand planes are numbered by their arithmetic (with_arith).
enum CodeSource {
  kCodeBf16x3 = kArithBf16x3,   // the bf16 pair hi + lo
  kCodeF16F8 = kArithF16F8,     // the fp16 plane hi + the E5M2 plane of the residuals x8, scaled by 2^-kLoShift
  kCodeBatchMajor,              // f16f8 after a dw_native backward (sce_plan::code_batch_major): hi + x8 as above, with x8
                                // the residuals' batch-major copy [M][n][ld], since dcode overwrote the row-major plane
  kCodeScores,                  // top-k: relu(score) where the activity mask has the bit, else 0
};

// W adjacent elements of a plane, loaded as one
template <class T, int W>
struct alignas(W * sizeof(T)) Adjacent {
  T e[W];
};
template <class T, int W>
__device__ __forceinline__ Adjacent<T, W> adjacent(const void* plane, long long idx) {
  return *reinterpret_cast<const Adjacent<T, W>*>(static_cast<const T*>(plane) + idx);
}

// The code c[m, r, j] read from source SRC, the one decoder of the planes' format: -0 (the [z == 0] flag) reads as +0.
template <int SRC>
struct CodeView {
  const void* hi;             // the code's 16-bit plane [M][batch_max][n] (bf16 or fp16)
  const void* lo;             // bf16x3: its second bf16 plane
  const uint8_t* x8;          // f16f8: E5M2 plane of the scaled residuals, [M][batch_max][n] or (kCodeBatchMajor) [M][n][ld]
  const float* scores;        // top-k: fp32 scores [M][batch_max][n]
  const uint32_t* pos;        // activity mask [M][n_chunks][batch_max]
  int n_chunks, batch_max, n, ld;

  // c[m, r, j + u] for u < W; with W = 2 (j even) one load reads both values of a row-major plane
  template <int W>
  __device__ __forceinline__ void get(int m, int r, int j, float (&v)[W]) const {
    const long long idx = ((long long)m * batch_max + r) * n + j;
    if constexpr (SRC == kCodeScores) {
      const uint32_t w = __ldg(pos + ((long long)m * n_chunks + (j >> 5)) * batch_max + r);
#pragma unroll
      for (int u = 0; u < W; ++u) v[u] = ((w >> (31 - ((j + u) & 31))) & 1u) ? fmaxf(__ldg(scores + idx + u), 0.f) : 0.f;
    } else if constexpr (SRC == kCodeBf16x3) {
      const Adjacent<__nv_bfloat16, W> h = adjacent<__nv_bfloat16, W>(hi, idx), l = adjacent<__nv_bfloat16, W>(lo, idx);
#pragma unroll
      for (int u = 0; u < W; ++u) v[u] = __bfloat162float(h.e[u]) + __bfloat162float(l.e[u]);
    } else {
      constexpr float kInv = 1.f / float(1 << kLoShift);
      const Adjacent<__half, W> h = adjacent<__half, W>(hi, idx);
      Adjacent<uint8_t, W> res;
      if constexpr (SRC == kCodeF16F8) {
        res = adjacent<uint8_t, W>(x8, idx);
      } else {
#pragma unroll
        for (int u = 0; u < W; ++u) res.e[u] = x8[((long long)m * n + j + u) * ld + r];
      }
#pragma unroll
      for (int u = 0; u < W; ++u) v[u] = __half2float(h.e[u]) + e5m2_to_float(res.e[u]) * kInv;
    }
#pragma unroll
    for (int u = 0; u < W; ++u) v[u] = v[u] == 0.f ? 0.f : v[u];
  }
  __device__ __forceinline__ float at(int m, int r, int j) const {
    float v[1];
    get(m, r, j, v);
    return v[0];
  }
};

// The view of the code of p's last call from source SRC
template <int SRC>
static CodeView<SRC> code_view(const sce_plan* p) {
  return {p->c.hi, p->c.lo, SRC == kCodeBatchMajor ? p->ct.x8 : p->c.x8, p->scores, p->act_pos, (p->d.n + 31) / 32,
          p->d.batch_max, p->d.n, p->cfg.bpad};
}

// out [M][B][n] fp32 = the code of the B rows of the last call. Grid (<= 1024, M), two adjacent columns per thread.
template <int SRC>
__global__ void __launch_bounds__(256) read_code_kernel(CodeView<SRC> c, int B, float* __restrict__ out) {
  const int m = blockIdx.y, row_pairs = c.n / 2;
  const long long pairs = (long long)B * row_pairs;
  float2* o = reinterpret_cast<float2*>(out + (long long)m * B * c.n);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < pairs; i += (long long)gridDim.x * blockDim.x) {
    const int r = (int)(i / row_pairs);
    float v[2];
    c.get(m, r, 2 * (int)(i - (long long)r * row_pairs), v);
    o[i] = make_float2(v[0], v[1]);
  }
}

// ------------------------------------------------------------------------------------------------
// top-activating and random activating fragments (sce_forward_fragments; interpret.py:82-212 record tables,
// :265-321 record selection): fragment g of a call is rows g L .. g L + L - 1.
// ------------------------------------------------------------------------------------------------
// fmax[m][g][j] = max over the L rows of fragment g of c[m, r, j]; active[m][g][j] = 1 where the activity mask has
// c > 0 on some row of it. One block per (32-column chunk, fragment, model): lane j reads column 32 chunk + j, so every
// row is read coalesced over the features; warp w takes the rows w, w + 8, ... and the 8 warps meet in shared memory.
// grid.y is capped at kMaxGridY: a block takes the fragments blockIdx.y, blockIdx.y + gridDim.y, ... (one when G fits).
// SIGNED (SCE_CODE_LINEAR plans): the maximum starts at -inf, not 0, so a fragment whose code is negative on every row
// keeps its negative maximum; "active" stays the OR of the activity mask, there c != 0 on some row. (The reference's
// interpret.py:309 tests the maximum for 0 instead: the two differ for a fragment whose maximum is exactly 0 while some
// row is negative.)
constexpr int kMaxGridY = 65535;
template <int SRC, bool SIGNED = false>
__global__ void __launch_bounds__(256) fragment_max_kernel(CodeView<SRC> c, int L, int G, float* __restrict__ fmax,
                                                           uint8_t* __restrict__ active) {
  __shared__ float smax[8][32];
  __shared__ uint32_t sact[8][32];
  const int chunk = blockIdx.x, m = blockIdx.z;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int j = chunk * 32 + lane;
  const uint32_t* pw = c.pos + ((long long)m * c.n_chunks + chunk) * c.batch_max;
  for (int g = blockIdx.y; g < G; g += gridDim.y) {
    float mx = SIGNED ? -INFINITY : 0.f;
    uint32_t any = 0u;
    for (int t = warp; t < L; t += 8) {
      const int r = g * L + t;
      any |= __ldg(pw + r);
      if (j < c.n) mx = fmaxf(mx, c.at(m, r, j));
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
    __syncthreads();   // warp 0 has read smax / sact before the next fragment overwrites them
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
template <int SRC>
__global__ void __launch_bounds__(128) fragment_merge_kernel(CodeView<SRC> c, int L, int G, long long frag0,
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
          for (int t = 0; t < L; ++t) dst[t] = c.at(m, g * L + t, j);
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
          for (int t = 0; t < L; ++t) dst[t] = c.at(m, g * L + t, j);
        }
        rlow = frag_lowest(rk, rf, n_random);
      }
    }
  }
}

constexpr int kFragMaxList = 64;   // largest n_top / n_random

static bool frag_len_ok(int L) { return L >= 32 && L <= 8192 && L % 32 == 0; }

// The workspace of one fragments call: fragment maxima [M][B/L][n] fp32, activity flags [M][B/L][n] u8, open-segment
// flags [M][n] int32. With base == nullptr only measures it.
struct FragCarve {
  float* fmax;
  uint8_t* active;
  int* open;
};
static size_t frag_carve(uint8_t* base, const sce_desc& d, int B, int L, FragCarve* out) {
  const size_t cells = (size_t)d.n_models * (B / L) * d.n;
  Carve c{base, 0};
  FragCarve w;
  w.fmax = c.take<float>(cells);
  w.active = c.take<uint8_t>(cells);
  w.open = c.take<int>((size_t)d.n_models * d.n);
  if (out) *out = w;
  return align_up(c.off, 1024);
}

template <int SRC>
static int launch_fragments(Launcher& launcher, const CodeView<SRC>& c, bool linear, int M, int L, int G, long long frag0,
                            float* fmax, uint8_t* active, int n_top, int n_random, unsigned long long seed, float* top_val,
                            long long* top_frag, float* top_act, long long* rnd_key, long long* rnd_frag, float* rnd_act) {
  const dim3 grid(c.n_chunks, G < kMaxGridY ? G : kMaxGridY, M);
  bool signed_max = false;
  if constexpr (SRC != kCodeScores) signed_max = linear;   // (top-k plans have no linear code)
  if (signed_max) {
    if constexpr (SRC != kCodeScores) TRY(launcher.launch(fragment_max_kernel<SRC, true>, grid, 256, 0, c, L, G, fmax, active));
  } else {
    TRY(launcher.launch(fragment_max_kernel<SRC>, grid, 256, 0, c, L, G, fmax, active));
  }
  return launcher.launch(fragment_merge_kernel<SRC>, dim3((c.n + 127) / 128, M), 128, 0, c, L, G, frag0, fmax,
                         active, n_top, n_random, seed, top_val, top_frag, top_act, rnd_key, rnd_frag, rnd_act);
}

// ------------------------------------------------------------------------------------------------
// top- and rest-feature reconstruction errors (sce_forward_split; standard_metrics.py:316-342
// fraction_variance_unexplained_top_activating): with t the decode of the code on the chosen columns alone, the
// residuals x - t and x - (x^ - t), summed per 32 rows. The decode of the rest is x^ - t, so only the n_top chosen
// columns of the code and rows of the dictionary are ever read besides x^.
// ------------------------------------------------------------------------------------------------
// c_top[m][r][s] = c[m, r, cols[m][s]], the code as the engine holds it. Grid (<= 1024, M).
template <int SRC>
__global__ void __launch_bounds__(256) code_columns_kernel(CodeView<SRC> c, int B, int n_top, const int* __restrict__ cols,
                                                           float* __restrict__ c_top) {
  const int m = blockIdx.y;
  const long long cells = (long long)B * n_top;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < cells; i += (long long)gridDim.x * blockDim.x) {
    const int r = (int)(i / n_top), s = (int)(i - (long long)r * n_top);
    c_top[(long long)m * cells + i] = c.at(m, r, __ldg(cols + m * n_top + s));
  }
}

// d_top[m][s] = dictionary row cols[m][s] of w [M][n][d], divided by max(||row||, floor) (floor <= 0: by ||row||) where
// `normalize`, as given otherwise. The norm is summed in dict_rows_kernel's order, so the row is bitwise the fp32 row the
// plan splits into its planes. One block of 128 threads per (s, m); d % 4 == 0.
__global__ void __launch_bounds__(128) chosen_rows_kernel(const float* __restrict__ w, const int* __restrict__ cols, int n,
                                                          int d, int n_top, int normalize, float floor,
                                                          float* __restrict__ d_top) {
  __shared__ float red[8];
  const int s = blockIdx.x, m = blockIdx.y;
  const float* e = w + ((long long)m * n + __ldg(cols + m * n_top + s)) * d;
  float* o = d_top + ((long long)m * n_top + s) * d;
  float sc = 1.f;
  if (normalize) {
    float ss = 0.f, unused = 0.f;
    for (int c = threadIdx.x * 4; c < d; c += 512) {
      const float4 v = *reinterpret_cast<const float4*>(e + c);
      ss = __fadd_rn(ss, dot4_rn(v, v));
    }
    block_sum2(ss, unused, red);
    const float nrm = sqrtf(ss);
    sc = (floor > 0.f && nrm < floor) ? floor : nrm;
  }
  for (int c = threadIdx.x * 4; c < d; c += 512) {
    const float4 v = *reinterpret_cast<const float4*>(e + c);
    *reinterpret_cast<float4*>(o + c) = make_float4(v.x / sc, v.y / sc, v.z / sc, v.w / sc);
  }
}

// Per block of 32 rows and model: t = sum_s c_top[r][s] d_top[s] (fp32, s ascending), x_hat_top = t where given, and
// with `part` the fp32 sums of (x - t)^2 and (x - (x^ - t))^2 over the block's rows to part[m][rb][0 / 1]. Warp w takes
// the rows w, w + 8, ..., lane l the columns 4 l + 128 i; the 8 warps' sums are added in warp order: no atomics.
__global__ void __launch_bounds__(256) split_residual_kernel(const float* __restrict__ x, long long x_model_stride,
                                                             const float* __restrict__ x_hat,
                                                             const float* __restrict__ c_top,
                                                             const float* __restrict__ d_top, int B, int d, int n_top,
                                                             float* __restrict__ x_hat_top, float* __restrict__ part) {
  __shared__ float red[2][8];
  const int rb = blockIdx.x, m = blockIdx.y, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const float* dt = d_top + (long long)m * n_top * d;
  float a = 0.f, b = 0.f;
  const int r_end = min(B, rb * 32 + 32);
  for (int r = rb * 32 + warp; r < r_end; r += 8) {
    const float* ct = c_top + ((long long)m * B + r) * n_top;
    const float* xr = x + m * x_model_stride + (long long)r * d;
    const long long row = ((long long)m * B + r) * d;
    for (int col = 4 * lane; col < d; col += 128) {
      float t[4] = {0.f, 0.f, 0.f, 0.f};
      for (int s = 0; s < n_top; ++s) {
        const float cs = __ldg(ct + s);
        const float4 dv = __ldg(reinterpret_cast<const float4*>(dt + (long long)s * d + col));
        t[0] = fmaf(cs, dv.x, t[0]);
        t[1] = fmaf(cs, dv.y, t[1]);
        t[2] = fmaf(cs, dv.z, t[2]);
        t[3] = fmaf(cs, dv.w, t[3]);
      }
      if (x_hat_top) *reinterpret_cast<float4*>(x_hat_top + row + col) = make_float4(t[0], t[1], t[2], t[3]);
      if (part) {
        const float4 xv = __ldg(reinterpret_cast<const float4*>(xr + col));
        const float4 hv = __ldg(reinterpret_cast<const float4*>(x_hat + row + col));
        const float xs[4] = {xv.x, xv.y, xv.z, xv.w}, hs[4] = {hv.x, hv.y, hv.z, hv.w};
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const float rt = xs[u] - t[u], rr = xs[u] - (hs[u] - t[u]);
          a = fmaf(rt, rt, a);
          b = fmaf(rr, rr, b);
        }
      }
    }
  }
  if (!part) return;   // (grid-uniform)
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    a += __shfl_xor_sync(0xffffffffu, a, o);
    b += __shfl_xor_sync(0xffffffffu, b, o);
  }
  if (lane == 0) {
    red[0][warp] = a;
    red[1][warp] = b;
  }
  __syncthreads();
  if (threadIdx.x < 2) {
    float v = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) v += red[threadIdx.x][w];
    part[((long long)m * gridDim.x + rb) * 2 + threadIdx.x] = v;
  }
}

// sq_top[m] += sum over the row blocks, in order, of part[m][rb][0] (fp64); sq_rest likewise from part[m][rb][1]
__global__ void split_reduce_kernel(const float* __restrict__ part, int row_blocks, int M, double* __restrict__ sq_top,
                                    double* __restrict__ sq_rest) {
  const int m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= M) return;
  double a = 0.0, b = 0.0;
  for (int rb = 0; rb < row_blocks; ++rb) {
    a += (double)part[((long long)m * row_blocks + rb) * 2];
    b += (double)part[((long long)m * row_blocks + rb) * 2 + 1];
  }
  sq_top[m] += a;
  sq_rest[m] += b;
}

static bool split_top_ok(const sce_desc& d, int n_top) { return n_top >= 1 && n_top <= SCE_SPLIT_MAX_TOP && n_top <= d.n; }

// The workspace of one split call: x^ [M][B][d], the chosen code columns [M][B][n_top] and dictionary rows
// [M][n_top][d], and the residual partials [M][ceil(B / 32)][2], fp32. With base == nullptr only measures it.
struct SplitCarve {
  float *x_hat, *c_top, *d_top, *part;
};
static size_t split_carve(uint8_t* base, const sce_desc& d, int B, int n_top, SplitCarve* out) {
  const size_t M = d.n_models;
  Carve c{base, 0};
  SplitCarve w;
  w.x_hat = c.take<float>(M * B * d.d);
  w.c_top = c.take<float>(M * B * n_top);
  w.d_top = c.take<float>(M * n_top * d.d);
  w.part = c.take<float>(M * ((B + 31) / 32) * 2);
  if (out) *out = w;
  return align_up(c.off, 1024);
}

// ------------------------------------------------------------------------------------------------
// expected interference (sce_code_interference, sce_expected_interference; big_sweep.py:43-57
// calc_expected_interference): with W the dictionary rows divided by max(||row||, 1e-8) and A_r the features with
// c[r, j] != 0, totals[r, i] = sum over j in A_r of (W_i . W_j)^2 c[r, j] and cap[r, i] = c[r, i] / max(totals, 1e-8)
// for i in A_r (0 elsewhere). Only the Gram of each row's active dictionary rows is formed, O(|A_r|^2 d) per row,
// tiled by kIfTile features, so the active set may be any size.
// ------------------------------------------------------------------------------------------------
constexpr int kCodeDense = kCodeScores + 1;   // a caller-held fp32 code [B][n] (sce_expected_interference)
constexpr int kIfTile = 64;                   // active features per Gram tile
constexpr int kIfK = 32;                      // dictionary columns per staged chunk
constexpr int kIfRows = 32;                   // rows per block, added in order into the block's partials
constexpr int kIfLd = kIfTile + 4;            // (16-byte aligned rows of the staged chunks)

// wn[m][j][0 .. dp) = w[m][j] / max(||w[m][j]||, 1e-8), zero from d on. One block of 128 threads per (j, m).
__global__ void __launch_bounds__(128) clamp_rows_kernel(const float* __restrict__ w, int n, int d, int dp,
                                                         float* __restrict__ wn) {
  __shared__ float red[8];
  const int j = blockIdx.x, m = blockIdx.y;
  const float* e = w + ((long long)m * n + j) * d;
  float* o = wn + ((long long)m * n + j) * dp;
  float ss = 0.f, unused = 0.f;
  for (int c = threadIdx.x; c < d; c += 128) ss = fmaf(e[c], e[c], ss);
  block_sum2(ss, unused, red);
  const float nrm = sqrtf(ss), sc = nrm < 1e-8f ? 1e-8f : nrm;
  for (int c = threadIdx.x; c < dp; c += 128) o[c] = c < d ? e[c] / sc : 0.f;
}

// c[m, r, j]: the plan's code through its CodeView, or the dense code
template <int SRC>
__device__ __forceinline__ float if_code(const CodeView<SRC>& c, const float* dense, int m, int r, int j) {
  if constexpr (SRC == kCodeDense) return __ldg(dense + (long long)r * c.n + j);
  else return c.at(m, r, j);
}

// The column of the k-th candidate of a row (k < the row's count): mask[w] bit l is column 32 w + l, before[w] the
// candidates in the words below w
__device__ __forceinline__ int if_column(const uint32_t* mask, const int* before, int n_chunks, int k) {
  int lo = 0, hi = n_chunks - 1;   // the last word w with before[w] <= k
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (before[mid] <= k) lo = mid;
    else hi = mid - 1;
  }
  return 32 * lo + (int)__fns(mask[lo], 0, k - before[lo] + 1);
}

// Per block of kIfRows rows and model, rows in order: part[m][rb][0][j] = sum of cap[r, j], part[m][rb][1][j] = number of
// rows with c[r, j] != 0. The candidates of a row are its activity-mask bits (plan code; exactly its c != 0 set) or its
// non-zero entries (dense code); a candidate whose value reads 0 adds nothing. The I and J tiles of kIfTile candidates
// are staged kIfK dictionary columns at a time; thread (ty, tx) forms the Gram entries (4 ty + u, 4 tx + v) in fp32 FMA,
// then totals[i] gets sum over v of g^2 c_j, added over the 16 tx lanes and the J tiles in a fixed order.
// Dynamic shared memory: 2 ceil(n / 32) + 1 words (the row's mask and the ranks before each word).
template <int SRC>
__global__ void __launch_bounds__(256, 2) interference_kernel(CodeView<SRC> c, const float* __restrict__ dense,
                                                           const float* __restrict__ wn, int dp, int B,
                                                           float* __restrict__ part) {
  extern __shared__ uint32_t if_words[];
  __shared__ __align__(16) float sa[kIfK][kIfLd];
  __shared__ __align__(16) float sb[kIfK][kIfLd];
  __shared__ int col_i[kIfTile], col_j[kIfTile];
  __shared__ float val_i[kIfTile], val_j[kIfTile], tot[kIfTile];
  const int n = c.n, n_chunks = (n + 31) / 32;
  uint32_t* mask = if_words;
  int* before = reinterpret_cast<int*>(if_words + n_chunks);
  const int rb = blockIdx.x, m = blockIdx.y, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int tx = tid & 15, ty = tid >> 4;
  float* pc = part + ((long long)m * gridDim.x + rb) * 2 * n;
  for (int j = tid; j < 2 * n; j += 256) pc[j] = 0.f;
  const float* wm = wn + (long long)m * n * dp;
  const int r_end = min(B, rb * kIfRows + kIfRows);
  // the k-th candidate of the row and its code value, or (-1, 0) past the last
  auto candidate = [&](int r, int k, int L, int* col, float* val) {
    int j = -1;
    float v = 0.f;
    if (k < L) {
      j = if_column(mask, before, n_chunks, k);
      v = if_code(c, dense, m, r, j);
    }
    *col = j;
    *val = v;
  };
  for (int r = rb * kIfRows; r < r_end; ++r) {
    __syncthreads();   // the previous row (and the zeroing of pc) is done
    if constexpr (SRC == kCodeDense) {
      for (int w = warp; w < n_chunks; w += 8) {
        const int j = 32 * w + lane;
        const uint32_t bits = __ballot_sync(0xffffffffu, j < n && __ldg(dense + (long long)r * n + j) != 0.f);
        if (lane == 0) mask[w] = bits;
      }
    } else {
      for (int w = tid; w < n_chunks; w += 256) {
        uint32_t bits = __brev(__ldg(c.pos + ((long long)m * n_chunks + w) * c.batch_max + r));
        if (32 * w + 32 > n) bits &= (1u << (n - 32 * w)) - 1u;
        mask[w] = bits;
      }
    }
    __syncthreads();
    if (warp == 0) {   // exclusive ranks of the words, 32 at a time
      int carry = 0;
      for (int w0 = 0; w0 < n_chunks; w0 += 32) {
        const int w = w0 + lane, v = w < n_chunks ? __popc(mask[w]) : 0;
        int s = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
          const int t = __shfl_up_sync(0xffffffffu, s, o);
          if (lane >= o) s += t;
        }
        if (w < n_chunks) before[w] = carry + s - v;
        carry += __shfl_sync(0xffffffffu, s, 31);
      }
      if (lane == 0) before[n_chunks] = carry;
    }
    __syncthreads();
    const int L = before[n_chunks];
    for (int i0 = 0; i0 < L; i0 += kIfTile) {
      if (tid < kIfTile) {
        candidate(r, i0 + tid, L, &col_i[tid], &val_i[tid]);
        tot[tid] = 0.f;
      }
      for (int j0 = 0; j0 < L; j0 += kIfTile) {
        const bool same = j0 == i0;
        if (!same && tid < kIfTile) candidate(r, j0 + tid, L, &col_j[tid], &val_j[tid]);
        __syncthreads();
        const int* cj = same ? col_i : col_j;
        const float* vj = same ? val_i : val_j;
        float acc[4][4];
#pragma unroll
        for (int u = 0; u < 4; ++u)
#pragma unroll
          for (int v = 0; v < 4; ++v) acc[u][v] = 0.f;
        for (int k0 = 0; k0 < dp; k0 += kIfK) {
          for (int q = tid; q < kIfTile * kIfK / 4; q += 256) {
            const int t = q >> 3, k = (q & 7) * 4;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (col_i[t] >= 0) v = __ldg(reinterpret_cast<const float4*>(wm + (long long)col_i[t] * dp + k0 + k));
            sa[k][t] = v.x;
            sa[k + 1][t] = v.y;
            sa[k + 2][t] = v.z;
            sa[k + 3][t] = v.w;
            if (!same) {
              v = make_float4(0.f, 0.f, 0.f, 0.f);
              if (cj[t] >= 0) v = __ldg(reinterpret_cast<const float4*>(wm + (long long)cj[t] * dp + k0 + k));
              sb[k][t] = v.x;
              sb[k + 1][t] = v.y;
              sb[k + 2][t] = v.z;
              sb[k + 3][t] = v.w;
            }
          }
          __syncthreads();
          const float(*bt)[kIfLd] = same ? sa : sb;
#pragma unroll 8
          for (int k = 0; k < kIfK; ++k) {
            const float4 a = *reinterpret_cast<const float4*>(&sa[k][4 * ty]);
            const float4 b = *reinterpret_cast<const float4*>(&bt[k][4 * tx]);
            const float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
            for (int u = 0; u < 4; ++u)
#pragma unroll
              for (int v = 0; v < 4; ++v) acc[u][v] = fmaf(av[u], bv[v], acc[u][v]);
          }
          __syncthreads();
        }
        float s[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          s[u] = 0.f;
#pragma unroll
          for (int v = 0; v < 4; ++v) s[u] = fmaf(acc[u][v] * acc[u][v], vj[4 * tx + v], s[u]);
#pragma unroll
          for (int o = 8; o > 0; o >>= 1) s[u] += __shfl_xor_sync(0xffffffffu, s[u], o);
        }
        if (tx == 0)
#pragma unroll
          for (int u = 0; u < 4; ++u) tot[4 * ty + u] += s[u];
        __syncthreads();   // tot is complete; col_j / val_j may be replaced
      }
      if (tid < kIfTile && col_i[tid] >= 0 && val_i[tid] != 0.f) {
        const float t = tot[tid];
        pc[col_i[tid]] += val_i[tid] / (t < 1e-8f ? 1e-8f : t);   // (a NaN total stays NaN, as torch.clamp keeps it)
        pc[n + col_i[tid]] += 1.f;
      }
      __syncthreads();   // before the next I tile replaces col_i / val_i / tot
    }
  }
}

// cap_sums[m][j] += sum over the row blocks, in order, of part[m][rb][0][j] (fp64); nz_counts[m][j] += those of [1][j]
__global__ void interference_reduce_kernel(const float* __restrict__ part, int row_blocks, int n,
                                           double* __restrict__ cap_sums, long long* __restrict__ nz_counts) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x, m = blockIdx.y;
  if (j >= n) return;
  double a = 0.0;
  long long k = 0;
  for (int rb = 0; rb < row_blocks; ++rb) {
    const float* o = part + ((long long)m * row_blocks + rb) * 2 * n + j;
    a += (double)__ldg(o);
    k += (long long)__ldg(o + n);
  }
  cap_sums[(long long)m * n + j] += a;
  nz_counts[(long long)m * n + j] += k;
}

// The workspace of one interference call: the clamp-normalised dictionary [M][n][dp] (dp = d rounded up to kIfK) and the
// row-block partials [M][ceil(B / kIfRows)][2][n], fp32. With base == nullptr only measures it.
struct IfCarve {
  float *wn, *part;
};
static int if_width(int d) { return (d + kIfK - 1) / kIfK * kIfK; }
static size_t if_carve(uint8_t* base, size_t M, size_t n, int d, int B, IfCarve* out) {
  Carve c{base, 0};
  IfCarve w;
  w.wn = c.take<float>(M * n * if_width(d));
  w.part = c.take<float>(M * ((B + kIfRows - 1) / kIfRows) * 2 * n);
  if (out) *out = w;
  return align_up(c.off, 1024);
}

// clamp_rows_kernel, interference_kernel<SRC> and the reduction on `dict` [M][n][d] and the code of view `c`
template <int SRC>
static int launch_interference(Launcher& L, const CodeView<SRC>& c, const float* dense, const float* dict, int M, int d,
                               int B, const IfCarve& w, double* cap_sums, long long* nz_counts) {
  const int n = c.n, dp = if_width(d), row_blocks = (B + kIfRows - 1) / kIfRows;
  TRY(L.launch(clamp_rows_kernel, dim3(n, M), 128, 0, dict, n, d, dp, w.wn));
  const size_t smem = sizeof(uint32_t) * (2 * ((n + 31) / 32) + 1);
  CUDA_TRY(cudaFuncSetAttribute(interference_kernel<SRC>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  TRY(L.launch(interference_kernel<SRC>, dim3(row_blocks, M), 256, smem, c, dense, w.wn, dp, B, w.part));
  return L.launch(interference_reduce_kernel, dim3((n + 255) / 256, M), 256, 0, w.part, row_blocks, n, cap_sums, nz_counts);
}

// ------------------------------------------------------------------------------------------------
// C ABI
// ------------------------------------------------------------------------------------------------
extern "C" {

int sce_read_code(sce_plan* p, int B, float* out_code, void* stream) {
  if (!p || !out_code) return fail(SCE_ERR_INVALID, "plan / out_code is NULL");
  if (int rc = check_rows(p, B, "")) return rc;
  Launcher L{static_cast<cudaStream_t>(stream)};
  const long long blocks = ((long long)B * p->d.n / 2 + 255) / 256;   // per model
  auto read = [&](auto src) {
    constexpr int SRC = decltype(src)::value;
    return L.launch(read_code_kernel<SRC>, dim3((unsigned)(blocks < 1024 ? blocks : 1024), p->d.n_models), 256, 0,
                    code_view<SRC>(p), B, out_code);
  };
  // (top-k plans too: the selection writes their code planes)
  if (p->code_batch_major) return read(std::integral_constant<int, kCodeBatchMajor>{});
  return with_arith(p->cfg.arith, read);
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
  return stats_carve(nullptr, *desc, B, nullptr);
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
  float* part;
  const size_t need = stats_carve(static_cast<uint8_t*>(workspace), p->d, B, &part);
  if (int rc = check_workspace(workspace, workspace_bytes, need, "forward_stats: ")) return rc;
  const sce_desc& d = p->d;
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
  return frag_carve(nullptr, *desc, B, L, nullptr);
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
  FragCarve w;
  const size_t need = frag_carve(static_cast<uint8_t*>(workspace), p->d, B, L, &w);
  if (int rc = check_workspace(workspace, workspace_bytes, need, "forward_fragments: ")) return rc;
  const sce_desc& d = p->d;
  PlanCall call;
  TRY(run_pipeline(call, p, x, B, static_cast<cudaStream_t>(stream), nullptr, false, nullptr, nullptr));
  p->last_launches = call.count;   // the pipeline's: the fragment kernels below are not counted
  const int n_chunks = (d.n + 31) / 32, G = B / L;
  auto fragments = [&](auto src) {
    constexpr int SRC = decltype(src)::value;
    return launch_fragments<SRC>(call, code_view<SRC>(p), p->cfg.linear, d.n_models, L, G, frag0, w.fmax, w.active, n_top, n_random,
                                 seed, top_val, top_frag, top_act, rnd_key, rnd_frag, rnd_act);
  };
  // (a forward pass leaves the code planes row-major)
  TRY(p->cfg.topk ? fragments(std::integral_constant<int, kCodeScores>{}) : with_arith(p->cfg.arith, fragments));
  // active fragments: segments of L rows, cut at fragment boundaries (phase 0, no segment stays open)
  CUDA_TRY(cudaMemsetAsync(w.open, 0, (size_t)d.n_models * d.n * sizeof(int), call.st));
  return call.launch(segment_count_kernel, dim3(n_chunks, d.n_models), 256, 0, p->act_pos, n_chunks, d.batch_max, B, d.n,
                     L, 0, n_active, w.open);
}

size_t sce_forward_split_workspace_bytes(const sce_desc* desc, int B, int n_top) {
  if (validate(desc) || B < 1 || B > desc->batch_max || !split_top_ok(*desc, n_top) || !plan_config(*desc).evaluable)
    return 0;
  return split_carve(nullptr, *desc, B, n_top, nullptr);
}

int sce_forward_split(sce_plan* p, const float* x, int B, int n_top, const int* top_cols, double* sq_top, double* sq_rest,
                      float* x_hat, float* x_hat_top, void* workspace, size_t workspace_bytes, void* stream) {
  TRY(check_forward_only(p, x, B, "forward_split: "));
  const sce_desc& d = p->d;
  if (!split_top_ok(d, n_top))
    return fail(SCE_ERR_INVALID, "forward_split: n_top = %d must lie in [1, min(n = %d, %d)]", n_top, d.n, SCE_SPLIT_MAX_TOP);
  if (!top_cols) return fail(SCE_ERR_INVALID, "forward_split: top_cols is NULL");
  const bool centred = d.centering != 0;
  if (centred && (!x_hat || !x_hat_top))
    return fail(SCE_ERR_INVALID, "forward_split: a centred plan needs x_hat and x_hat_top (the caller forms its residuals)");
  if (!centred && (!sq_top || !sq_rest)) return fail(SCE_ERR_INVALID, "forward_split: sq_top and sq_rest are required");
  SplitCarve w;
  const size_t need = split_carve(static_cast<uint8_t*>(workspace), d, B, n_top, &w);
  if (int rc = check_workspace(workspace, workspace_bytes, need, "forward_split: ")) return rc;
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  // the columns are checked on the host before anything is launched
  const int M = d.n_models;
  int* cols = static_cast<int*>(std::malloc(sizeof(int) * M * n_top));
  if (!cols) return fail(SCE_ERR_INVALID, "forward_split: out of host memory");
  cudaError_t e = cudaMemcpyAsync(cols, top_cols, sizeof(int) * M * n_top, cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  int bad = e == cudaSuccess ? SCE_OK : fail(SCE_ERR_CUDA, "forward_split: reading top_cols: %s", cudaGetErrorString(e));
  for (int m = 0; m < M && !bad; ++m)
    for (int s = 0; s < n_top && !bad; ++s) {
      const int j = cols[m * n_top + s];
      if (j < 0 || j >= d.n)
        bad = fail(SCE_ERR_INVALID, "forward_split: top_cols[%d][%d] = %d outside [0, n = %d)", m, s, j, d.n);
      for (int s2 = 0; s2 < s && !bad; ++s2)
        if (cols[m * n_top + s2] == j)
          bad = fail(SCE_ERR_INVALID, "forward_split: column %d appears twice in top_cols[%d]", j, m);
    }
  std::free(cols);
  if (bad) return bad;
  PlanCall c;
  float* xh = x_hat ? x_hat : w.x_hat;
  TRY(run_pipeline(c, p, x, B, st, xh, false, nullptr, nullptr));
  p->last_launches = c.count;   // the pipeline's: the split kernels below are not counted
  const PlanConfig& cfg = p->cfg;
  // the decoding dictionary, normalised as the plan's planes are (SCE_DECODER_RAW: as given)
  const float* dict = cfg.untied ? p->b.decoder : p->b.encoder;
  TRY(c.launch(chosen_rows_kernel, dim3(n_top, M), 128, 0, dict, top_cols, d.n, d.d, n_top, cfg.raw_decoder ? 0 : 1,
               d.norm_floor, w.d_top));
  const long long blocks = ((long long)B * n_top + 255) / 256;
  auto columns = [&](auto src) {
    constexpr int SRC = decltype(src)::value;
    return c.launch(code_columns_kernel<SRC>, dim3((unsigned)(blocks < 1024 ? blocks : 1024), M), 256, 0, code_view<SRC>(p),
                    B, n_top, top_cols, w.c_top);
  };
  // (a forward pass leaves the code planes row-major)
  TRY(cfg.topk ? columns(std::integral_constant<int, kCodeScores>{}) : with_arith(cfg.arith, columns));
  const int row_blocks = (B + 31) / 32;
  TRY(c.launch(split_residual_kernel, dim3(row_blocks, M), 256, 0, x, cfg.x_models ? (long long)B * d.d : 0LL, xh, w.c_top,
               w.d_top, B, d.d, n_top, x_hat_top, centred ? nullptr : w.part));
  if (centred) return SCE_OK;
  return c.launch(split_reduce_kernel, dim3((M + 127) / 128), 128, 0, w.part, row_blocks, M, sq_top, sq_rest);
}

size_t sce_interference_workspace_bytes(const sce_desc* desc, int B) {
  if (validate(desc) || B < 1 || B > desc->batch_max || !plan_config(*desc).evaluable) return 0;
  return if_carve(nullptr, desc->n_models, desc->n, desc->d, B, nullptr);
}

int sce_code_interference(sce_plan* p, int B, double* cap_sums, long long* nz_counts, void* workspace,
                          size_t workspace_bytes, void* stream) {
  if (!p) return fail(SCE_ERR_INVALID, "code_interference: plan is NULL");
  if (!p->cfg.evaluable)
    return fail(SCE_ERR_INVALID, "code_interference: not available for the learned-centre variant or with encoder_nonneg / "
                                 "input_shift; evaluate the exported dictionaries (TiedSAE)");
  TRY(check_rows(p, B, "code_interference: "));
  if (!cap_sums || !nz_counts) return fail(SCE_ERR_INVALID, "code_interference: cap_sums and nz_counts are required");
  const sce_desc& d = p->d;
  IfCarve w;
  const size_t need = if_carve(static_cast<uint8_t*>(workspace), d.n_models, d.n, d.d, B, &w);
  if (int rc = check_workspace(workspace, workspace_bytes, need, "code_interference: ")) return rc;
  Launcher L{static_cast<cudaStream_t>(stream)};
  // the dictionary the plan decodes with, as stored: every kind is normalised here with the clamp alone
  const float* dict = p->cfg.untied ? p->b.decoder : p->b.encoder;
  auto run = [&](auto src) {
    constexpr int SRC = decltype(src)::value;
    return launch_interference<SRC>(L, code_view<SRC>(p), nullptr, dict, d.n_models, d.d, B, w, cap_sums, nz_counts);
  };
  if (p->cfg.topk) return run(std::integral_constant<int, kCodeScores>{});
  if (p->code_batch_major) return run(std::integral_constant<int, kCodeBatchMajor>{});
  return with_arith(p->cfg.arith, run);
}

size_t sce_expected_interference_workspace_bytes(int n, int d, int B) {
  if (n < 1 || d < 1 || B < 1) return 0;
  return if_carve(nullptr, 1, n, d, B, nullptr);
}

int sce_expected_interference(const float* dict, int n, int d, const float* code, int B, double* cap_sums,
                              long long* nz_counts, void* workspace, size_t workspace_bytes, void* stream) {
  if (!dict || !code) return fail(SCE_ERR_INVALID, "expected_interference: dict / code is NULL");
  if (n < 1 || d < 1 || B < 1)
    return fail(SCE_ERR_INVALID, "expected_interference: n = %d, d = %d and B = %d must be >= 1", n, d, B);
  if (!cap_sums || !nz_counts) return fail(SCE_ERR_INVALID, "expected_interference: cap_sums and nz_counts are required");
  IfCarve w;
  const size_t need = if_carve(static_cast<uint8_t*>(workspace), 1, n, d, B, &w);
  if (int rc = check_workspace(workspace, workspace_bytes, need, "expected_interference: ")) return rc;
  Launcher L{static_cast<cudaStream_t>(stream)};
  const CodeView<kCodeDense> c{nullptr, nullptr, nullptr, nullptr, nullptr, (n + 31) / 32, B, n, 0};
  return launch_interference<kCodeDense>(L, c, code, dict, 1, d, B, w, cap_sums, nz_counts);
}

}  // extern "C"
