// gemm_overlap_probe.cu — main-loop-only time of the split-operand GEMM (sce_gemm.cuh) at the four config-2 GEMMs of a
// training step (16 tied SAEs, d = 512, n = 4096, batch 8192, f16f8, fp16-exact activations).
//
// Each GEMM runs in the configuration libsce launches it in (layouts, operand sets, passes, skipped cross terms,
// persistent grid), but with an epilogue that does nothing with the accumulators beyond reading them from the staging
// tile. It declares the staging bytes of the engine's epilogue, so the stage ring is as deep. The time per launch is
// the main loop alone: the engine's kernel time for the same GEMM minus this one is what its epilogue adds. Each GEMM
// runs in clusters of each size given on the command line, in that order: 1 (every CTA loads its own A tiles), 2 (two
// CTAs along N share each A tile by multicast) or 0 (the size launch_gemm takes, as libsce launches it: 2 for decode and
// the weight gradient, 1 for encode and dcode). Without sizes, 0. Each JSON line names the size run ("cluster") and the
// size launch_gemm takes ("engine_cluster"). tools/gemm_overlap_probe.py reads them from stdout. Build: Makefile target
// `probe`. Decode and the weight gradient also run on tall tiles (192 rows, BM = kBMTall) at each size, right after the
// 128-row tiles; each JSON line names its tile height ("bm").
//
//   build/gemm_overlap_probe [reps] [cluster sizes ...]
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "../sparse_coding_b200/csrc/sce_gemm.cuh"
#include "../sparse_coding_b200/csrc/sce_tmap.h"

using namespace sce;

#define CK(x)                                                                         \
  do {                                                                                \
    cudaError_t e_ = (x);                                                             \
    if (e_ != cudaSuccess) {                                                          \
      printf("CUDA error %s at %s:%d\n", cudaGetErrorString(e_), __FILE__, __LINE__); \
      exit(2);                                                                        \
    }                                                                                 \
  } while (0)

// Reads every accumulator of its chunks and stores nothing (the never-taken store keeps the reads). INLINE: run in line
// by the consumers, as the engine epilogue it stands for (kInline in sce_gemm.cuh).
template <int STAGE_BYTES, bool INLINE>
struct EpiNoop {
  static constexpr int kCols = 32;
  static constexpr int kWarpStageBytes = STAGE_BYTES;
  static constexpr bool kInline = INLINE;
  struct Params {
    uint32_t* sink;
  };
  const Params& P;
  uint32_t x = 0;
  __device__ EpiNoop(const Params& p, const TileCoord&, int, int, uint8_t*) : P(p) {}
  __device__ __forceinline__ void chunk(int, const uint32_t (&r)[32]) {
#pragma unroll
    for (int j = 0; j < 32; ++j) x ^= r[j];
  }
  __device__ __forceinline__ void finish() {
    if (x == 0x7FC00001u) *P.sink = x;
  }
};

// finite fp16 / E5M2 values of either sign, |v| < 1, from a hash of the index: the tensor cores switch as they do on
// real operands
__global__ void fill_kernel(uint8_t* p, size_t bytes, int elem, uint32_t seed) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < bytes / elem; i += (size_t)gridDim.x * blockDim.x) {
    uint32_t h = (uint32_t)i * 2654435761u ^ seed;
    h ^= h >> 15;
    h *= 2246822519u;
    h ^= h >> 13;
    if (elem == 2) reinterpret_cast<uint16_t*>(p)[i] = uint16_t((h & 0x37FFu) | (h >> 16 & 0x8000u));
    else p[i] = uint8_t((h & 0x37u) | (h >> 24 & 0x80u));
  }
}

static std::vector<void*> g_dev;
static void* plane(size_t bytes, int elem) {
  void* d = nullptr;
  CK(cudaMalloc(&d, bytes));
  fill_kernel<<<1024, 256>>>(static_cast<uint8_t*>(d), bytes, elem, (uint32_t)g_dev.size() * 7919u + 1u);
  CK(cudaGetLastError());
  g_dev.push_back(d);
  return d;
}

// The planes of one operand [models][rows][K]: fp16, value-e5m2 and residual-e5m2, filled with hashed values
struct Planes3 {
  void *hi, *lo, *x8;
};
static Planes3 planes(int models, int rows, int K) {
  const size_t n = (size_t)models * rows * K;
  return {plane(2 * n, 2), plane(n, 1), plane(n, 1)};
}

// The maps of one operand [models][rows][K]: the fp16 plane K-major (box rows x 64, 128-byte swizzle) or MN-major
// ([models][K][rows], boxes 64 x 64); the two 8-bit planes always K-major (64-byte swizzle), as the native cross terms
// read them (the weight gradient's are the batch-major copies).
static void operand(const Planes3& P, int models, int rows, int K, bool mn, uint32_t box_rows, CUtensorMap* hi,
                    CUtensorMap* lo, CUtensorMap* x8) {
  constexpr int BK = gemm_bk(kArithF16F8);
  bool ok = mn ? make_tmap_bf16(hi, P.hi, models, K, rows, rows, (uint64_t)K * rows, BK)
               : make_tmap_bf16_box(hi, P.hi, models, rows, K, K, (uint64_t)rows * K, BK, box_rows,
                                    CU_TENSOR_MAP_SWIZZLE_128B);
  ok &= make_tmap_u8_box(lo, P.lo, models, rows, K, K, (uint64_t)rows * K, BK, box_rows, CU_TENSOR_MAP_SWIZZLE_64B);
  ok &= make_tmap_u8_box(x8, P.x8, models, rows, K, K, (uint64_t)rows * K, BK, box_rows, CU_TENSOR_MAP_SWIZZLE_64B);
  if (!ok) {
    printf("tensor map encode failed\n");
    exit(2);
  }
}

struct Shape {
  const char* name;
  int a_models, b_models, M, N, K, nsets;
  bool b0_exact;   // set 0's B operand (x) is fp16-exact: its residual plane is flagged all-zero
  bool a0_exact;   // set 0's A operand (x) is fp16-exact
};

// The GEMM's parameters for output tiles of BM rows, on operand planes pa / pb per set
template <class Epi, int BM>
static GemmParams<typename Epi::Params> params(const Shape& s, int models, bool mn, const Planes3* pa, const Planes3* pb,
                                               uint32_t* zero_flag, uint32_t* sink) {
  GemmParams<typename Epi::Params> p;
  memset(&p, 0, sizeof(p));
  for (int set = 0; set < s.nsets; ++set) {
    const int bm = set == 0 ? s.b_models : models;   // the weight gradient's second set (c^T g) is per model on both sides
    operand(pa[set], s.a_models, s.M, s.K, mn, BM, &p.a_hi[set], &p.a_lo[set], &p.a_x8[set]);
    operand(pb[set], bm, s.N, s.K, mn, kBN, &p.b_hi[set], &p.b_lo[set], &p.b_x8[set]);
    p.a_batched[set] = s.a_models > 1;
    p.b_batched[set] = bm > 1;
  }
  if (s.a0_exact) p.a_res_flag[0] = zero_flag;
  if (s.b0_exact) p.b_res_flag[0] = zero_flag;
  p.nsets = s.nsets;
  p.k_total = s.K;
  p.passes = 3;
  p.n_models = models;
  p.m_total = s.M;
  p.n_total = s.N;
  p.tiles_m = gemm_tiles_m<BM>(s.M);
  p.tiles_n = (s.N + kBN - 1) / kBN;
  p.epi.sink = sink;
  return p;
}

// Times the GEMM at each asked cluster size; TALL: at each, also with tall tiles (BM = kBMTall) right after the kBM
// tiles, on the same operands, so that the two alternate in the session
template <int STAGE_BYTES, bool INLINE, bool MN, bool NATIVE, bool TALL = false>
static void run(const Shape& s, int models, int sms, uint32_t* zero_flag, uint32_t* sink, int reps,
                const std::vector<int>& clusters) {
  using Epi = EpiNoop<STAGE_BYTES, INLINE>;
  Planes3 pa[kMaxSets], pb[kMaxSets];
  for (int set = 0; set < s.nsets; ++set) {
    pa[set] = planes(s.a_models, s.M, s.K);
    pb[set] = planes(set == 0 ? s.b_models : models, s.N, s.K);
  }
  const auto p = params<Epi, kBM>(s, models, MN, pa, pb, zero_flag, sink);
  const auto pt = params<Epi, kBMTall>(s, models, MN, pa, pb, zero_flag, sink);
  cudaEvent_t e0, e1;
  CK(cudaEventCreate(&e0));
  CK(cudaEventCreate(&e1));
  const int engine_cluster = gemm_launch_cluster<kArithF16F8, NATIVE>(p);
  // resident(): the clusters resident at once, asked after the launches have opted the kernel in to its shared memory
  auto time = [&](int bm, int cluster, auto launch, int tiles, int stages, auto resident) {
    for (int rep = 0; rep < 3; ++rep) CK(launch());
    CK(cudaEventRecord(e0));
    for (int rep = 0; rep < reps; ++rep) CK(launch());
    CK(cudaEventRecord(e1));
    CK(cudaDeviceSynchronize());
    float ms = 0;
    CK(cudaEventElapsedTime(&ms, e0, e1));
    const double flops = 2.0 * models * s.M * s.N * (double)s.K * s.nsets;
    printf("{\"gemm\": \"%s\", \"bm\": %d, \"cluster\": %d, \"engine_cluster\": %d, \"resident_clusters\": %d, "
           "\"main_loop_ms\": %.4f, \"tiles\": %d, \"stages\": %d, \"reps\": %d, \"tflops\": %.1f}\n",
           s.name, bm, cluster, engine_cluster, resident(), ms / reps, tiles, stages, reps, flops / (ms / reps) * 1e-9);
  };
  for (int asked : clusters) {
    const int cluster = asked == 0 ? engine_cluster : asked;
    {
      using SM = GemmSmem<STAGE_BYTES, kArithF16F8, NATIVE>;
      constexpr auto kern2 = gemm_split_kernel<Epi, MN, MN, false, kArithF16F8, NATIVE, 2>;
      auto resident = [&] {
        return cluster == 1 ? sms : max_active_clusters<kern2>(2, gemm_threads<Epi, kArithF16F8, NATIVE>(), SM::kBytes, 0);
      };
      time(kBM, cluster, [&] { return launch_gemm_clusters<Epi, MN, MN, false, kArithF16F8, NATIVE>(p, 0, sms, 0, cluster); },
           models * p.tiles_m * p.tiles_n, SM::kStages, resident);
    }
    if constexpr (TALL) {
      using SM = GemmSmem<STAGE_BYTES, kArithF16F8, NATIVE, kBMTall>;
      constexpr auto kern2 = gemm_split_kernel<Epi, MN, MN, false, kArithF16F8, NATIVE, 2, kBMTall>;
      auto resident = [&] {
        return cluster == 1 ? sms
                            : max_active_clusters<kern2>(2, gemm_threads<Epi, kArithF16F8, NATIVE, kBMTall>(), SM::kBytes, 0);
      };
      time(kBMTall, cluster,
           [&] { return launch_gemm_clusters<Epi, MN, MN, false, kArithF16F8, NATIVE, kBMTall>(pt, 0, sms, 0, cluster); },
           models * pt.tiles_m * pt.tiles_n, SM::kStages, resident);
    }
  }
  CK(cudaEventDestroy(e0));
  CK(cudaEventDestroy(e1));
  for (void* d : g_dev) cudaFree(d);
  g_dev.clear();
}

int main(int argc, char** argv) {
  const int reps = argc > 1 ? atoi(argv[1]) : 20;
  std::vector<int> clusters;
  for (int i = 2; i < argc; ++i) clusters.push_back(atoi(argv[i]));
  if (clusters.empty()) clusters.push_back(0);
  setvbuf(stdout, nullptr, _IOLBF, 0);
  cudaDeviceProp prop;
  CK(cudaGetDeviceProperties(&prop, 0));
  uint32_t *zero_flag, *sink;
  CK(cudaMalloc(&zero_flag, 4));
  CK(cudaMemset(zero_flag, 0, 4));
  CK(cudaMalloc(&sink, 4));
  const int M = 16, d = 512, n = 4096, B = 8192, sms = prop.multiProcessorCount;
  // encode: z = x W_enc^T, x shared and fp16-exact (its cross term skipped); EpiEncodeT stages 4 KB per warp
  run<4096, false, false, true>({"encode", 1, M, B, n, d, 1, false, true}, M, sms, zero_flag, sink, reps, clusters);
  // the same with 6 KB per warp, what staging the code's batch-major copies as well would take: one ring stage fewer
  run<6144, false, false, true>({"encode_6k", 1, M, B, n, d, 1, false, true}, M, sms, zero_flag, sink, reps, clusters);
  // decode: x^ = c W_dec, both operands per model; EpiDecodeT stages nothing and runs in line
  run<0, true, false, true, true>({"decode", M, M, B, d, n, 1, false, false}, M, sms, zero_flag, sink, reps, clusters);
  // dcode: g W_dec^T; EpiDcodeT stages 4 KB per warp
  run<4096, false, false, true>({"dcode", M, M, B, n, d, 1, false, false}, M, sms, zero_flag, sink, reps, clusters);
  // weight gradient: dz^T x + c^T g, reduction over the batch, fp16 planes MN-major, 8-bit ones from batch-major copies;
  // x (set 0's B) fp16-exact; EpiStoreF32 runs in line
  run<0, true, true, true, true>({"dw", M, 1, n, d, B, 2, true, false}, M, sms, zero_flag, sink, reps, clusters);
  cudaFree(zero_flag);
  cudaFree(sink);
  return 0;
}
