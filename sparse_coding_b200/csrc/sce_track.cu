// sce_track.cu — dead-feature tracking (sce_track_workspace_bytes, sce_step_tracked, sce_resample;
// experiments/huge_batch_size.py:120-146 WorstIndices, :189-250): each model's worst-reconstructed rows and the
// features' activity over a window of tracked steps, and the resample that reinitialises the features that never fired.
#include <cmath>

#include "sce_plan.cuh"

namespace sce {

constexpr int kTrackThreads = 256;   // every tracking kernel; active_count_block needs 8 warps

// The list order as one 64-bit key, larger = earlier in the list: the bits of e (>= 0, so they order as the values do)
// above the inverted window serial (e descending, serial ascending). Every real key is >= 1 (serial < 2^32 - 1).
__device__ __forceinline__ unsigned long long track_key(float e, long long serial) {
  return ((unsigned long long)__float_as_uint(e) << 32) | (unsigned long long)(0xFFFFFFFFu - (uint32_t)serial);
}

// Exclusive prefix count of `flag` over the block's threads in thread order, and the block's total. Every thread calls.
__device__ __forceinline__ int block_prefix(bool flag, int* total) {
  __shared__ int warp_cnt[kTrackThreads / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint32_t bal = __ballot_sync(0xffffffffu, flag);
  if (lane == 0) warp_cnt[warp] = __popc(bal);
  __syncthreads();
  int before = 0, all = 0;
#pragma unroll
  for (int w = 0; w < kTrackThreads / 32; ++w) {
    before += w < warp ? warp_cnt[w] : 0;
    all += warp_cnt[w];
  }
  __syncthreads();   // (warp_cnt is reused by the next call)
  *total = all;
  return before + __popc(bal & ((1u << lane) - 1u));
}

__device__ __forceinline__ unsigned long long block_min_u64(unsigned long long v) {
  __shared__ unsigned long long red[kTrackThreads / 32];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = min(v, __shfl_xor_sync(0xffffffffu, v, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  unsigned long long r = red[0];
#pragma unroll
  for (int w = 1; w < kTrackThreads / 32; ++w) r = min(r, red[w]);
  __syncthreads();
  return r;
}

// One tracked step's view of the caller's lists and of its scratch (TrackCarve)
struct TrackArgs {
  float* err;                  // [M][N]
  long long* serial;           // [M][N]
  float* rows;                 // [M][N][d]
  int* filled;                 // [M]
  int* counts;                 // [M][n]
  long long next_serial;
  int N;
  const float* part;           // [M][B][n_part] partial sums of r^2 per row
  int n_part;
  unsigned long long* keys;    // [M][N + batch_max]: the list's keys (slots), then the rows' (0: not a candidate)
  int *enter_row, *enter_slot; // [M][cap]: the rows entering the list, in row order, and the slots they take
  int* enter_cnt;              // [M]
  int cap;                     // min(N, batch_max)
  const float* x;              // the caller's batch; model m's rows start at x + m x_model_stride
  long long x_model_stride;
};

// The key of rank `want` (1 = largest) among the non-zero keys of keys[0, n_list) and keys[N, N + B): a most-significant-
// digit radix select, 8 bits per pass, with a 256-bin histogram in shared memory (integer counts: any order of the adds
// gives the same result). Keys are distinct, so exactly one key equals the result.
__device__ unsigned long long track_select(const unsigned long long* keys, int n_list, int N, int B, int want) {
  __shared__ int hist[256];
  __shared__ unsigned long long s_prefix;
  __shared__ int s_want;
  unsigned long long prefix = 0ull, mask = 0ull;
  for (int shift = 56; shift >= 0; shift -= 8) {
    for (int i = threadIdx.x; i < 256; i += kTrackThreads) hist[i] = 0;
    __syncthreads();
    for (int i = threadIdx.x; i < n_list + B; i += kTrackThreads) {
      const unsigned long long k = keys[i < n_list ? i : N + (i - n_list)];
      if (k != 0ull && (k & mask) == prefix) atomicAdd(&hist[(int)((k >> shift) & 255ull)], 1);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      int b = 255;
      for (; b > 0; --b) {
        if (want <= hist[b]) break;
        want -= hist[b];
      }
      s_prefix = prefix | ((unsigned long long)b << shift);
      s_want = want;
    }
    __syncthreads();
    prefix = s_prefix;
    want = s_want;
    mask |= 255ull << shift;
    __syncthreads();
  }
  return prefix;
}

// Merge of one tracked step. Block (0, m): model m's list; blocks (1 + chunk, m): the window's activity counts of a
// 32-feature chunk (active_count_block). Nothing happens when the step's update was skipped (kBadWord).
// List merge: e_r = (sum of row r's partials, in order) / d; rows whose key is not above the N-th key of a full list
// drop out; the cut K is the N-th largest key of list and candidates (track_select, only when they overflow N); list
// entries below K leave, candidates at or above K enter: the i-th entering row (row order) takes the i-th free slot
// (slot order: vacated slots and slots past filled), and track_copy_kernel copies its d values.
__global__ void __launch_bounds__(kTrackThreads) track_merge_kernel(TrackArgs t, const uint32_t* __restrict__ pos,
                                                                    int n_chunks, int batch_max, int B, int n, int d,
                                                                    const uint32_t* __restrict__ health) {
  const int m = blockIdx.y;
  if (step_is_bad(health)) {
    if (blockIdx.x == 0 && threadIdx.x == 0) t.enter_cnt[m] = 0;
    return;
  }
  if (blockIdx.x > 0) {
    active_count_block(pos, n_chunks, batch_max, B, n, t.counts, blockIdx.x - 1, m);
    return;
  }
  const int N = t.N;
  float* err = t.err + (long long)m * N;
  long long* ser = t.serial + (long long)m * N;
  unsigned long long* keys = t.keys + (long long)m * (N + batch_max);
  int* enter_row = t.enter_row + (long long)m * t.cap;
  int* enter_slot = t.enter_slot + (long long)m * t.cap;
  const int filled = t.filled[m];
  unsigned long long lo = ~0ull;
  for (int s = threadIdx.x; s < filled; s += kTrackThreads) {
    const unsigned long long k = track_key(err[s], ser[s]);
    keys[s] = k;
    lo = min(lo, k);
  }
  lo = block_min_u64(lo);
  const unsigned long long thr = filled == N ? lo : 0ull;
  const float* part = t.part + (long long)m * B * t.n_part;
  int mine = 0;
  for (int r = threadIdx.x; r < B; r += kTrackThreads) {
    float sq = 0.f;
    for (int q = 0; q < t.n_part; ++q) sq += part[(long long)r * t.n_part + q];
    unsigned long long k = track_key(sq / (float)d, t.next_serial + r);
    if (k <= thr) k = 0ull;
    else ++mine;
    keys[N + r] = k;
  }
  int cand;
  block_prefix(mine > 0, &cand);   // (only whether some thread has one)
  __syncthreads();                 // keys[] complete for every thread
  if (cand == 0) {
    if (threadIdx.x == 0) t.enter_cnt[m] = 0;
    return;
  }
  // candidates in total (an integer sum: order-independent)
  __shared__ int s_total;
  if (threadIdx.x == 0) s_total = 0;
  __syncthreads();
  if (mine) atomicAdd(&s_total, mine);
  __syncthreads();
  const int C = s_total;
  const unsigned long long cut = filled + C > N ? track_select(keys, filled, N, B, N) : 1ull;
  const int new_filled = filled + C < N ? filled + C : N;
  int n_in = 0, n_free = 0;
  for (int r0 = 0; r0 < B; r0 += kTrackThreads) {
    const int r = r0 + threadIdx.x;
    const bool in = r < B && keys[N + r] >= cut;
    int tot;
    const int at = block_prefix(in, &tot);
    if (in) enter_row[n_in + at] = r;
    n_in += tot;
  }
  for (int s0 = 0; s0 < new_filled; s0 += kTrackThreads) {
    const int s = s0 + threadIdx.x;
    const bool fr = s < new_filled && (s >= filled || keys[s] < cut);
    int tot;
    const int at = block_prefix(fr, &tot);
    if (fr) enter_slot[n_free + at] = s;
    n_free += tot;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < n_in; i += kTrackThreads) {
    const int r = enter_row[i], s = enter_slot[i];
    err[s] = __uint_as_float((uint32_t)(keys[N + r] >> 32));
    ser[s] = t.next_serial + r;
  }
  if (threadIdx.x == 0) {
    t.enter_cnt[m] = n_in;   // (== n_free)
    t.filled[m] = new_filled;
  }
}

// The d values of each row that entered model blockIdx.y's list, from the caller's batch into its slot
__global__ void __launch_bounds__(kTrackThreads) track_copy_kernel(TrackArgs t, int d) {
  const int m = blockIdx.y, cnt = t.enter_cnt[m], d4 = d >> 2;
  for (int i = blockIdx.x; i < cnt; i += gridDim.x) {
    const int r = t.enter_row[(long long)m * t.cap + i], s = t.enter_slot[(long long)m * t.cap + i];
    const float4* src = reinterpret_cast<const float4*>(t.x + m * t.x_model_stride + (long long)r * d);
    float4* dst = reinterpret_cast<float4*>(t.rows + ((long long)m * t.N + s) * d);
    for (int c = threadIdx.x; c < d4; c += kTrackThreads) dst[c] = src[c];
  }
}

// norms[m][j] = ||W[m][j]|| in fp64 (squares summed per lane in column order, then across the warp in a fixed tree).
// One warp per row, grid (ceil(n / 8), M).
__global__ void __launch_bounds__(kTrackThreads) track_norm_kernel(const float* __restrict__ w, int n, int d,
                                                                   double* __restrict__ norms) {
  const int m = blockIdx.y, j = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (j >= n) return;
  const float* row = w + ((long long)m * n + j) * d;
  double ss = 0.0;
  for (int c = lane; c < d; c += 32) ss += (double)row[c] * (double)row[c];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
  if (lane == 0) norms[(long long)m * n + j] = sqrt(ss);
}

// order[m][rank] = slot: the rank of each filled entry in the list order, by counting the entries above it (keys are
// distinct). Grid (ceil(N / 256), M).
__global__ void __launch_bounds__(kTrackThreads) track_rank_kernel(const float* __restrict__ err,
                                                                   const long long* __restrict__ serial,
                                                                   const int* __restrict__ filled, int N,
                                                                   int* __restrict__ order) {
  __shared__ unsigned long long tile[kTrackThreads];
  const int m = blockIdx.y, f = filled[m], s = blockIdx.x * kTrackThreads + threadIdx.x;
  const float* e = err + (long long)m * N;
  const long long* sr = serial + (long long)m * N;
  const unsigned long long k = s < f ? track_key(e[s], sr[s]) : 0ull;
  int rank = 0;
  for (int u0 = 0; u0 < f; u0 += kTrackThreads) {
    const int u = u0 + threadIdx.x;
    tile[threadIdx.x] = u < f ? track_key(e[u], sr[u]) : 0ull;
    __syncthreads();
    const int lim = f - u0 < kTrackThreads ? f - u0 : kTrackThreads;
    for (int q = 0; q < lim; ++q) rank += tile[q] > k;
    __syncthreads();
  }
  if (s < f) order[(long long)m * N + rank] = s;
}

// Per model (one block): the dead set j_1 < j_2 < ... in dead[m] (count 0, not masked), mu = mean of the valid rows'
// norms (fp64, each thread's columns in order, then the threads in order), scale[m] = ratio / mu, the outputs n_dead,
// n_replaced = min(n_dead, filled) and replaced; then the window restarts (filled and counts zeroed).
__global__ void __launch_bounds__(kTrackThreads) track_dead_kernel(int* __restrict__ counts, int* __restrict__ filled,
                                                                   const unsigned char* __restrict__ mask,
                                                                   const double* __restrict__ norms, int n, float ratio,
                                                                   int* __restrict__ dead, int* __restrict__ n_rep,
                                                                   float* __restrict__ scale, int* __restrict__ n_dead_out,
                                                                   int* __restrict__ n_rep_out,
                                                                   unsigned char* __restrict__ replaced) {
  __shared__ double red[kTrackThreads];
  __shared__ int red_valid[kTrackThreads];
  const int m = blockIdx.x;
  int* cnt = counts + (long long)m * n;
  const unsigned char* mk = mask ? mask + (long long)m * n : nullptr;
  int n_dead = 0;
  for (int j0 = 0; j0 < n; j0 += kTrackThreads) {
    const int j = j0 + threadIdx.x;
    const bool dd = j < n && cnt[j] == 0 && !(mk && mk[j]);
    int tot;
    const int at = block_prefix(dd, &tot);
    if (dd) dead[(long long)m * n + n_dead + at] = j;
    n_dead += tot;
  }
  double acc = 0.0;
  int valid = 0;
  for (int j = threadIdx.x; j < n; j += kTrackThreads)
    if (!(mk && mk[j])) {
      acc += norms[(long long)m * n + j];
      ++valid;
    }
  red[threadIdx.x] = acc;
  red_valid[threadIdx.x] = valid;
  __syncthreads();
  const int f = filled[m];
  const int nr = n_dead < f ? n_dead : f;
  for (int j = threadIdx.x; j < n; j += kTrackThreads) replaced[(long long)m * n + j] = 0;
  __syncthreads();
  for (int i = threadIdx.x; i < nr; i += kTrackThreads) replaced[(long long)m * n + dead[(long long)m * n + i]] = 1;
  for (int j = threadIdx.x; j < n; j += kTrackThreads) cnt[j] = 0;
  if (threadIdx.x == 0) {
    double sum = 0.0;
    int nv = 0;
    for (int i = 0; i < kTrackThreads; ++i) {
      sum += red[i];
      nv += red_valid[i];
    }
    scale[m] = (float)((double)ratio / (sum / nv));
    n_rep[m] = nr;
    n_dead_out[m] = n_dead;
    n_rep_out[m] = nr;
    filled[m] = 0;
  }
}

// Row dead[m][i] of the dictionary parameter <- rows[m][order[m][i]] * scale[m] for i < n_rep[m]; the Adam moments of that
// row (encoder, decoder) and of its bias entry <- 0. Grid (<= n, M).
__global__ void __launch_bounds__(kTrackThreads) track_write_kernel(const float* __restrict__ rows,
                                                                    const int* __restrict__ order,
                                                                    const int* __restrict__ dead,
                                                                    const int* __restrict__ n_rep,
                                                                    const float* __restrict__ scale, int N, int n, int d,
                                                                    float* w, float* w_m, float* w_v, float* dec_m,
                                                                    float* dec_v, float* b_m, float* b_v) {
  const int m = blockIdx.y, cnt = n_rep[m];
  const float sc = scale[m];
  for (int i = blockIdx.x; i < cnt; i += gridDim.x) {
    const int j = dead[(long long)m * n + i], s = order[(long long)m * N + i];
    const float* src = rows + ((long long)m * N + s) * d;
    const long long o = ((long long)m * n + j) * d;
    for (int c = threadIdx.x; c < d; c += kTrackThreads) {
      w[o + c] = src[c] * sc;
      w_m[o + c] = 0.f;
      w_v[o + c] = 0.f;
      if (dec_m) {
        dec_m[o + c] = 0.f;
        dec_v[o + c] = 0.f;
      }
    }
    if (threadIdx.x == 0 && b_m) {
      b_m[(long long)m * n + j] = 0.f;
      b_v[(long long)m * n + j] = 0.f;
    }
  }
}

}  // namespace sce

// The scratch of one tracked step or resample (sce_track.workspace). With base == nullptr only measures it.
struct TrackCarve {
  float* row_part;              // [M][batch_max][2 tiles_n] decode epilogue partials (unused by k-sparse top-k plans)
  unsigned long long* keys;     // [M][N + batch_max]
  int *enter_row, *enter_slot;  // [M][cap]
  int* enter_cnt;               // [M]
  int cap;                      // min(N, batch_max)
  double* norms;                // [M][n]
  int *order, *dead;            // [M][N], [M][n]
  int* n_rep;                   // [M]
  float* scale;                 // [M]
};
static size_t track_carve(uint8_t* base, const sce_desc& d, int N, TrackCarve* out) {
  const size_t M = d.n_models, Bm = d.batch_max, n = d.n;
  Carve c{base, 0};
  TrackCarve w;
  w.cap = N < d.batch_max ? N : d.batch_max;
  w.row_part = c.take<float>(M * Bm * 2 * ((d.d + kBN - 1) / kBN));
  w.keys = c.take<unsigned long long>(M * (N + Bm));
  w.enter_row = c.take<int>(M * w.cap);
  w.enter_slot = c.take<int>(M * w.cap);
  w.enter_cnt = c.take<int>(M);
  w.norms = c.take<double>(M * n);
  w.order = c.take<int>(M * N);
  w.dead = c.take<int>(M * n);
  w.n_rep = c.take<int>(M);
  w.scale = c.take<float>(M);
  if (out) *out = w;
  return align_up(c.off, 1024);
}

// The checks of sce_step_tracked / sce_resample that come before any device call. Those on the track alone come first,
// then the plan and what depends on it; carves the workspace into `w`.
static int check_track(const sce_plan* p, const sce_track* t, const char* prefix, TrackCarve* w) {
  if (!t) return fail(SCE_ERR_INVALID, "%strack is NULL", prefix);
  if (!t->err || !t->serial || !t->rows || !t->filled || !t->counts)
    return fail(SCE_ERR_INVALID, "%strack: err, serial, rows, filled and counts are required", prefix);
  if (reinterpret_cast<uintptr_t>(t->rows) % 16) return fail(SCE_ERR_INVALID, "%strack: rows must be 16-byte aligned", prefix);
  if (t->n_worst < 1) return fail(SCE_ERR_INVALID, "%strack: n_worst = %d must be >= 1", prefix, t->n_worst);
  if (!p) return fail(SCE_ERR_INVALID, "%splan is NULL", prefix);
  TRY(check_trainable(p, prefix));
  if (t->n_worst > p->d.n) return fail(SCE_ERR_INVALID, "%strack: n_worst = %d outside [1, n = %d]", prefix, t->n_worst, p->d.n);
  const size_t need = track_carve(static_cast<uint8_t*>(t->workspace), p->d, t->n_worst, w);
  return check_workspace(t->workspace, t->workspace_bytes, need, prefix);
}

// ------------------------------------------------------------------------------------------------
// C ABI
// ------------------------------------------------------------------------------------------------
extern "C" {

size_t sce_track_workspace_bytes(const sce_desc* desc, int n_worst) {
  if (validate(desc)) return 0;
  if (n_worst < 1 || n_worst > desc->n) {
    fail(SCE_ERR_INVALID, "track: n_worst = %d outside [1, n = %d]", n_worst, desc->n);
    return 0;
  }
  return track_carve(nullptr, *desc, n_worst, nullptr);
}

int sce_step_tracked(sce_plan* p, const float* x, int B, float* out_losses, float* out_nnz, const sce_track* track,
                     void* stream) {
  TrackCarve w;
  TRY(check_track(p, track, "step_tracked: ", &w));
  TRY(check_rows(p, B, "step_tracked: "));
  if (track->next_serial < 0 || track->next_serial + B >= 0xFFFFFFFFll)
    return fail(SCE_ERR_INVALID, "step_tracked: next_serial = %lld with B = %d leaves [0, 2^32 - 1)", track->next_serial, B);
  const sce_desc& d = p->d;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  TRY(step_impl(p, x, B, out_losses, out_nnz, st, p->cfg.topk_sparse ? nullptr : w.row_part));
  sce::TrackArgs t{track->err, track->serial, track->rows, track->filled, track->counts, track->next_serial,
                   track->n_worst, p->cfg.topk_sparse ? p->part_dec : w.row_part,
                   p->cfg.topk_sparse ? p->cfg.tk_slices : 2 * ((d.d + kBN - 1) / kBN), w.keys, w.enter_row, w.enter_slot,
                   w.enter_cnt, w.cap, x, p->cfg.input_models == 1 ? 0 : (long long)B * d.d};
  Launcher L{st};
  const int n_chunks = (d.n + 31) / 32;
  TRY(L.launch(track_merge_kernel, dim3(1 + n_chunks, d.n_models), kTrackThreads, 0, t, p->act_pos, n_chunks,
               d.batch_max, B, d.n, d.d, p->res_flags));
  return L.launch(track_copy_kernel, dim3(w.cap < 1024 ? w.cap : 1024, d.n_models), kTrackThreads, 0, t, d.d);
}

int sce_resample(sce_plan* p, const sce_track* track, float ratio, int* n_dead, int* n_replaced, unsigned char* replaced,
                 void* stream) {
  TrackCarve w;
  TRY(check_track(p, track, "resample: ", &w));
  if (!(ratio > 0.f) || !std::isfinite(ratio)) return fail(SCE_ERR_INVALID, "resample: ratio must be positive and finite");
  if (!n_dead || !n_replaced || !replaced) return fail(SCE_ERR_INVALID, "resample: n_dead, n_replaced and replaced are required");
  const sce_desc& d = p->d;
  const sce_buffers& b = p->b;
  const int M = d.n_models, n = d.n, N = track->n_worst;
  Launcher L{static_cast<cudaStream_t>(stream)};
  TRY(L.launch(track_norm_kernel, dim3((n + 7) / 8, M), kTrackThreads, 0, b.encoder, n, d.d, w.norms));
  TRY(L.launch(track_rank_kernel, dim3((N + kTrackThreads - 1) / kTrackThreads, M), kTrackThreads, 0, track->err,
               track->serial, track->filled, N, w.order));
  TRY(L.launch(track_dead_kernel, M, kTrackThreads, 0, track->counts, track->filled, b.coef_mask, w.norms, n, ratio,
               w.dead, w.n_rep, w.scale, n_dead, n_replaced, replaced));
  const int cap = N < n ? N : n;
  TRY(L.launch(track_write_kernel, dim3(cap < 1024 ? cap : 1024, M), kTrackThreads, 0, track->rows, w.order, w.dead, w.n_rep,
               w.scale, N, n, d.d, b.encoder, b.encoder_m, b.encoder_v, p->cfg.untied ? b.decoder_m : nullptr,
               p->cfg.untied ? b.decoder_v : nullptr, b.bias_m, b.bias_v));
  return prepare_dict(L, p);
}


}  // extern "C"
