// sce_gemm.cuh — persistent, warp-specialised, batched split-operand GEMM on wgmma / TMA / mbarrier (sm_90a).
//
//   D[model][i][j] = sum_set sum_k A_set[model][i,k] * B_set[model][j,k]            (fp32 accumulators)
//
// This is how the engine reaches the reference's true-FP32 results (SURVEY.md H1) on the 16-bit tensor cores.
// Every fp32 operand is carried as operand planes and the product formed from partial products:
//   ARITH = bf16x3: x ~= hi + lo (two bf16 planes); hi*hi + hi*lo + lo*hi, three bf16 passes (~2^-16);
//   ARITH = f16f8 : x ~= h + l, h = fp16(x); h*h on the fp16 planes, the two cross terms on E5M2 planes, rescaled in
//                   the accumulator (see sce_ptx.cuh) — the default.
// `passes == 1` keeps only the 16-bit plane product. Operands may be K-major (reduction index contiguous in HBM) or
// MN-major (row/column index contiguous); f16f8 GEMMs are one or the other on both sides. The f16f8 cross terms run on
// E5M2 wgmma (F8_NATIVE), which reads K-major 8-bit tiles only: A_MN / B_MN then describe the fp16 planes alone, and an
// MN-major GEMM (the weight gradient) reads batch-major copies of its 8-bit planes. Without those copies (top-k and
// launch-bound plans) the MN-major weight gradient widens its 8-bit tiles to fp16 in shared memory instead.
//
// One CTA per SM, 512 threads in four warpgroups, each setting its registers with setmaxnreg: warpgroup 0 = TMA
// producer (one thread), warpgroups 1 and 2 = wgmma consumers (rows 0..63 and 64..127 of the 128 x 128 tile),
// warpgroup 3 = the fused epilogue. The consumers write the accumulators into a padded fp32 tile in shared memory
// (acc_stage) and arrive on the mbarrier acc_full; the epilogue warpgroup reads the tile, arrives on acc_empty, and
// runs the epilogue while the consumers run the next tile's main loop (they wait on acc_empty only before writing
// acc_stage again). Each epilogue thread owns one output row and 32 consecutive columns. A tile's epilogue has eight
// shares (q, g): rows 32 q .. +31 and the 32-column chunks with chunk % 2 == g; epilogue warp q runs (q, 0) and (q, 1)
// chunk by chunk, alternating between their staging tiles. Where the epilogue does not overlap (gemm_overlap: kInline
// epilogues, the widened path) the kernel runs 384 threads without the epilogue warpgroup, and the eight consumer warps
// run it in line after the main loop, warp w taking share (w % 4, w / 4). The outputs are the same either way.
//
// Where a model's column-tile count is even and the K loop long, the CTAs run in clusters of two along N (launch_gemm,
// gemm_cluster_size): the pair works on the two columns of one tile row at a time, so both need the same A tile at
// every K block, and one of them loads it for both with a TMA multicast. That cuts the operand bytes read from L2 per
// MMA by a quarter (A and B tiles are the same size). Each stage then holds bytes written by both CTAs, so it is free
// only once the consumers of both have released it. Nothing about the arithmetic, its order or the epilogues depends on
// the cluster size.
#pragma once
#include <type_traits>
#include "sce_ptx.cuh"

namespace sce {

constexpr int kBM = 128;        // rows of the output tile
constexpr int kBN = 128;        // columns of the output tile
constexpr int kEpiWarps = 8;    // epilogue shares of a tile (warp quarter x column group), each with its own staging
// Launches that overlap the epilogue run 512 threads, and each warpgroup sets its per-thread registers with setmaxnreg:
// producer, each of the two consumers, epilogue. They add up to the 65536 registers of the SM over 128 threads each
// (the launch count of 128 per thread at 512 threads). In-line launches run 384 threads without setmaxnreg.
constexpr int kProducerRegs = 40, kConsumerRegs = 168, kEpilogueRegs = 136;
static_assert(kProducerRegs + 2 * kConsumerRegs + kEpilogueRegs == 65536 / 128, "register split of the four warpgroups");
// Tall tiles (BM = kBMTall, see gemm_split_kernel): 512 threads, a producer warpgroup and three consumer warpgroups. A
// native f16f8 consumer holds acc[64] and accx[64] and compiles to about 153 registers, so a fourth consumer warpgroup
// (256 rows) would leave it 122 and spill; three fit at 160.
constexpr int kBMTall = 192;
constexpr int kTallProducerRegs = 32, kTallConsumerRegs = 160;
static_assert(kTallProducerRegs + 3 * kTallConsumerRegs <= 65536 / 128, "register split of the tall-tile warpgroups");
constexpr int kMaxSets = 2;
constexpr int kSmemLimit = 232448;  // 227 KB of shared memory one CTA may use on sm_90

// What the epilogue functor sees for each tile.
struct TileCoord {
  int model;    // ensemble index (pair index for epilogues with kPairTiles)
  int m_blk;    // tile row index
  int n_blk;    // tile column index
  int row;      // global output row owned by this thread (may be >= m_total: predicate!)
  int col0;     // first global output column of the tile
  int warp_q;   // epilogue warp quarter 0..3 (rows 32*warp_q .. +31 of the tile)
  int grp;      // epilogue warp group 0..1 (handles the 32-column chunks with chunk % 2 == grp)
  int lane;
  // The warp runs this share chunk by chunk alternately with its other share (the epilogue warpgroup), so the bulk
  // store issued just before a chunk read the other share's staging tile, not this one's.
  bool alternate;
};

// Whole warp, before a chunk writes its share's staging tile: wait until the bulk stores that read that tile are done
// with it. Where the warp alternates between two shares' tiles, the most recent store may still be reading the other.
// Each share's last chunk is followed by its epilogue's finish(), which waits for every store (the staging tiles must
// outlive them), so the next tile's first chunk never meets a store of this tile.
__device__ __forceinline__ void staging_wait(const TileCoord& t) {
  if (t.lane == 0) {
    if (t.alternate) tma_store_wait_read<1>();
    else tma_store_wait_read<0>();
  }
  __syncwarp();
}

template <class EpiParams>
struct GemmParams {
  // bf16x3: (hi, lo) bf16 planes. f16f8: hi = fp16 plane, lo = e5m2(x) plane, x8 = e5m2((x - fp16(x)) * 2^kLoShift) plane.
  CUtensorMap a_hi[kMaxSets], a_lo[kMaxSets], b_hi[kMaxSets], b_lo[kMaxSets];
  CUtensorMap a_x8[kMaxSets], b_x8[kMaxSets];
  // f16f8: optional device flags, one per operand: *flag == 0 says "the residual plane (x8) of this operand is all
  // zeros for this launch" (e.g. activations that are exactly fp16, the reference's chunk format). The cross term that
  // multiplies that plane is then skipped together with the loads of its two planes: 25 % fewer operand bytes and
  // cross-term instructions for that operand pair, bit-identical results. nullptr = no such knowledge.
  const uint32_t* a_res_flag[kMaxSets];
  const uint32_t* b_res_flag[kMaxSets];
  int a_batched[kMaxSets], b_batched[kMaxSets];  // 0: operand shared by all models
  int nsets;      // number of (A,B) operand pairs accumulated into the same tile
  int k_total;    // reduction length of each pair
  int passes;     // 3: hi*hi + hi*lo + lo*hi (f16f8: fp16 hh + two cross terms), 1: hi*hi
  int n_models, m_total, n_total;
  int tiles_m, tiles_n;
  EpiParams epi;
};

constexpr int kArithBf16x3 = 0, kArithF16F8 = 1;

// K block of every GEMM of an arithmetic; a K-major 16-bit tile row is then one swizzle span (64 or 128 bytes).
// bf16x3: 32 (a stage of the four bf16 planes is 32 KB, so several stages fit beside the accumulator tile).
// f16f8: 64 (a stage holds one 16-bit plane per operand, or the four 8-bit planes in the same bytes).
__host__ __device__ constexpr int gemm_bk(int arith) { return arith == kArithF16F8 ? 64 : 32; }

constexpr int align1k(int v) { return (v + 1023) / 1024 * 1024; }

// Shared memory of one CTA. F8_NATIVE (f16f8): the cross terms run on E5M2 wgmma from the stage, nothing is widened.
// BM: rows of the output tile. The accumulator tile holds kBM rows either way (a tall tile's epilogue runs in two
// rounds through it), so at BM = kBMTall four 40 KB stages fill the 227 KB exactly.
template <int EPI_WARP_BYTES, int ARITH, bool F8_NATIVE, int BM = kBM>
struct GemmSmem {
  static constexpr int kBK = gemm_bk(ARITH);
  static constexpr int kATile = BM * kBK * 2;   // bytes of one 16-bit A tile
  static constexpr int kBTile = kBN * kBK * 2;
  // bf16x3: hi and lo planes of A and B. f16f8: either the fp16 planes or the four 8-bit planes (same bytes).
  static constexpr int kStage = ARITH == kArithBf16x3 ? 2 * kATile + 2 * kBTile : kATile + kBTile;
  static constexpr int kAccLd = kBN + 1;         // padded row of the fp32 accumulator tile (conflict-free both ways)
  static constexpr int kAccBytes = kBM * kAccLd * 4;
  // f16f8: the four 8-bit tiles of a stage widened to fp16 (shares the space of the accumulator tile: never live together)
  static constexpr int kWideBytes = ARITH == kArithF16F8 && !F8_NATIVE ? 2 * kATile + 2 * kBTile : 0;
  static constexpr int kAccRegion = align1k(kAccBytes > kWideBytes ? kAccBytes : kWideBytes);
  static constexpr int kFixed = kAccRegion + kEpiWarps * EPI_WARP_BYTES + 1024 /*barriers*/ + 1024 /*align slack*/;
  // pipeline depth: as many stages as fit beside the accumulator tile and the epilogue staging (at most 8)
  static constexpr int kStages = (kSmemLimit - kFixed) / kStage > 8 ? 8 : (kSmemLimit - kFixed) / kStage;
  static constexpr int kAccOff = kStages * kStage;
  static constexpr int kEpiOff = kAccOff + kAccRegion;
  static constexpr int kBarOff = kEpiOff + kEpiWarps * EPI_WARP_BYTES;
  static constexpr int kBytes = kBarOff + 1024 + 1024;
  static_assert(kBytes <= kSmemLimit, "exceeds the 227 KB of shared memory one CTA may use");
};

// epilogues may declare `static constexpr bool kPairTiles = true`: the tile's `model` index is then a PAIR index, and the
// operand models of pair q are read from the device list Epi::Params::pairs ([q][2] = model of A, model of B) instead of
// following a_batched / b_batched. One persistent launch then runs any set of (model_a, model_b) products.
template <class Epi, class = void>
struct epi_pair_tiles : std::false_type {};
template <class Epi>
struct epi_pair_tiles<Epi, std::void_t<decltype(Epi::kPairTiles)>> : std::bool_constant<Epi::kPairTiles> {};

// epilogues may declare `static constexpr bool kInline = true`: the consumers then run them in line after each tile's
// main loop, in the 384-thread kernel without an epilogue warpgroup. For epilogues whose state needs more than the
// epilogue warpgroup's kEpilogueRegs registers, and for light ones beside a long main loop, where the overlap has
// nothing to win and its epilogue traffic during the main loop measured slower (decode, the fp32 store of dW).
template <class Epi, class = void>
struct epi_inline : std::false_type {};
template <class Epi>
struct epi_inline<Epi, std::void_t<decltype(Epi::kInline)>> : std::bool_constant<Epi::kInline> {};

// Whether the epilogue warpgroup runs a tile's epilogue while the consumers run the next tile's main loop. Not for
// kInline epilogues, nor on the widened f16f8 path (MN-major 8-bit tiles without F8_NATIVE), which widens into the space
// of the accumulator tile, so that tile cannot be held for the epilogue during the main loop there. A region of its own
// would cost two of its five ring stages, and the plans on that path (top-k, launch-bound shapes) run it for the weight
// gradient only, whose fp32 store epilogue is in line anyway.
template <class Epi, int ARITH, bool F8_NATIVE>
__host__ __device__ constexpr bool gemm_overlap() {
  return (ARITH != kArithF16F8 || F8_NATIVE) && !epi_inline<Epi>::value;
}
template <class Epi, int ARITH, bool F8_NATIVE, int BM = kBM>
__host__ __device__ constexpr int gemm_threads() {
  return gemm_overlap<Epi, ARITH, F8_NATIVE>() || BM == kBMTall ? 512 : 384;
}

// Output-tile rows of the GEMM's launch over m_total rows. Tall tiles cover at least the rows of the kBM tiling, so that
// every epilogue share of that tiling (whose slots the epilogues fill, rows beyond m_total included) is run.
template <int BM>
__host__ __device__ constexpr int gemm_tiles_m(int m_total) {
  return ((m_total + kBM - 1) / kBM * kBM + BM - 1) / BM;
}

// f16f8 without F8_NATIVE (MN-major operands): an MN-major 8-bit tile as TMA delivers it without swizzle, [BK][ROWS]
// bytes, widened to the fp16 tile the 16-bit loads of the same operand produce, [ROWS / 64][BK][64] with the 128-byte
// swizzle. 256 consumer threads, 16 bytes each per round.
template <int ROWS>
__device__ __forceinline__ void widen_tile(const uint8_t* src, uint8_t* dst, int tid) {
  constexpr int BK = gemm_bk(kArithF16F8);
  constexpr int kPieces = ROWS * BK / 16;
#pragma unroll 2
  for (int q = tid; q < kPieces; q += 256) {
    const uint4 v = *reinterpret_cast<const uint4*>(src + q * 16);
    uint4 w0, w1;
    widen_e5m2x4(v.x, w0.x, w0.y);
    widen_e5m2x4(v.y, w0.z, w0.w);
    widen_e5m2x4(v.z, w1.x, w1.y);
    widen_e5m2x4(v.w, w1.z, w1.w);
    const int k = q / (ROWS / 16), m0 = (q % (ROWS / 16)) * 16;
    const int base = (m0 >> 6) * (BK * 128) + k * 128, j = (m0 & 63) >> 3;
    *reinterpret_cast<uint4*>(dst + base + ((j ^ (k & 7)) << 4)) = w0;
    *reinterpret_cast<uint4*>(dst + base + (((j + 1) ^ (k & 7)) << 4)) = w1;
  }
}

// ------------------------------------------------------------------------------------------------
// The kernel
// ------------------------------------------------------------------------------------------------
// SPLIT_ACC: keep the dominant hi*hi products and the small cross terms (hi*lo, lo*hi) in two separate
// accumulators (summed in the epilogue). The tensor core's fp32 accumulation truncates, which biases a
// result by a small amount per accumulated MMA; the cross terms are 2^-8 of the total, so moving them out
// shortens the chain that matters 3x. Used where the reduction is long: the decode GEMM at large n and the
// weight gradient (K = batch).
//
// ARITH = kArithF16F8 (see sce_ptx.cuh, "fp16 + fp8 arithmetic"): a tile makes TWO sweeps over K. Sweep 1 streams the
// 8-bit planes (a stage holds A.h8, A.l8, B.h8, B.l8 — the same bytes as A.f16 + B.f16) and accumulates the cross terms;
// the accumulator is then scaled by 2^-kLoShift; sweep 2 streams the fp16 planes and adds hh. F8_NATIVE (8-bit tiles
// K-major, loaded with the 64-byte swizzle): sweep 1 runs E5M2 wgmma on the stage itself; A_MN / B_MN describe the fp16
// planes only (sweep 2), because E5M2 wgmma reads no layout but K-major. Otherwise (MN-major operands) the 8-bit tiles
// arrive unswizzled and MN-major, and are widened to fp16 in shared memory first.
//
// CLUSTER (1 or 2): the CTAs of the launch run in clusters of that many along N, sharing each A tile (see the top of the
// file). A compile-time value, so that a launch in clusters of one runs the kernel without any of the pairing.
//
// BM (kBM or kBMTall): rows of the output tile. Tall tiles (192 rows) read (96 + 128) operand elements per k for 192 x
// 128 outputs in pairs, against (64 + 128) for 128 x 128: 22 % fewer L2 bytes per MMA, for GEMMs whose main loop is
// fed from L2 rather than bound by the tensor pipe (decode and the weight gradient). Only for in-line epilogues on the
// native f16f8 path: 512 threads, the producer warpgroup and three consumer warpgroups of 64 rows each (setmaxnreg
// kTallProducerRegs / kTallConsumerRegs). The epilogue runs in two rounds through the kBM-row acc_stage: rows 0..127
// from consumers 0 and 1, then rows 128..191 from consumer 2 (while 0 and 1 start the next tile). Every share keeps the
// TileCoord of the kBM tiling (m_blk = row / kBM, warp_q = row % kBM / 32), and each output's accumulation order
// depends on the K sweep only, so the outputs are bitwise those of BM = kBM.
template <class Epi, bool A_MN, bool B_MN, bool SPLIT_ACC, int ARITH, bool F8_NATIVE, int CLUSTER, int BM = kBM>
__global__ void __launch_bounds__(gemm_threads<Epi, ARITH, F8_NATIVE, BM>(), 1)
gemm_split_kernel(const __grid_constant__ GemmParams<typename Epi::Params> p) {
  constexpr bool F8 = ARITH == kArithF16F8;
  constexpr int BN = kBN;
  static_assert(!F8 || !SPLIT_ACC, "f16f8 rescales in the accumulator; no split accumulators");
  static_assert(!F8_NATIVE || F8, "F8_NATIVE is an f16f8 path");
  static_assert(!F8 || A_MN == B_MN, "f16f8 GEMMs are K-major or MN-major on both sides");
  static_assert(!F8 || F8_NATIVE || (A_MN && B_MN), "the widened f16f8 path is MN-major on both sides");
  static_assert(CLUSTER == 1 || CLUSTER == 2, "clusters of one or two CTAs");
  static_assert(CLUSTER == 1 || !F8 || F8_NATIVE, "the widened f16f8 path runs in clusters of one");
  constexpr bool TALL = BM == kBMTall;
  static_assert(BM == kBM || TALL, "tiles of 128 or 192 rows");
  static_assert(!TALL || (F8_NATIVE && epi_inline<Epi>::value && Epi::kWarpStageBytes == 0),
                "tall tiles: native f16f8, in-line epilogues without staging");
  constexpr int kWGs = BM / 64;   // consumer warpgroups
  using SM = GemmSmem<Epi::kWarpStageBytes, ARITH, F8_NATIVE, BM>;
  constexpr int BK = SM::kBK;
  constexpr int STAGES = SM::kStages;
  constexpr int EC = Epi::kCols;  // accumulator columns handed to the epilogue per call
  static_assert(EC == 32, "epilogue chunk is 32 columns");
  constexpr bool OVERLAP = gemm_overlap<Epi, ARITH, F8_NATIVE>();

  // Aligned by an offset from smem_raw, not by a round trip through an integer: a pointer derived from smem_raw stays
  // in the shared address space, so every access through it compiles to LDS / STS, not to generic LD / ST.
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + SM::kBarOff);
  uint64_t* empty_bar = full_bar + STAGES;
  uint64_t* acc_full = empty_bar + STAGES;   // OVERLAP: acc_stage holds a tile for the epilogue warpgroup
  uint64_t* acc_empty = acc_full + 1;        // OVERLAP: the epilogue warpgroup has read acc_stage
  float* acc_stage = reinterpret_cast<float*>(smem + SM::kAccOff);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  // Tile schedule: CTA b runs tiles b, b + gridDim.x, ... The launch groups the CTAs in clusters of CLUSTER consecutive
  // CTAs, and takes CLUSTER = 2 only where tiles_n is even (launch_gemm_clusters). The two CTAs of a cluster then run
  // tiles 2 u and 2 u + 1 at every step: the two columns of one model and tile row, with the same operand sets and K
  // loop, and the same A tile (for kPairTiles epilogues too: the A model is the tile's pair).
  [[maybe_unused]] const int cta_rank = CLUSTER == 2 ? int(cluster_ctarank()) : 0;
  const int num_tiles = p.n_models * p.tiles_m * p.tiles_n;
  auto decode_tile = [&](int tile, int& model, int& tile_m, int& tile_n) {
    model = tile / (p.tiles_m * p.tiles_n);
    const int rem = tile - model * (p.tiles_m * p.tiles_n);
    tile_m = rem / p.tiles_n;
    tile_n = rem % p.tiles_n;
  };
  // operand models of operand pair `set` for the tile's model (or pair) index
  auto operand_models = [&](int model, int set, int& am, int& bm) {
    if constexpr (epi_pair_tiles<Epi>::value) {
      am = __ldg(p.epi.pairs + 2 * model);
      bm = __ldg(p.epi.pairs + 2 * model + 1);
    } else {
      am = p.a_batched[set] ? model : 0;
      bm = p.b_batched[set] ? model : 0;
    }
  };
  const int kblocks = (p.k_total + BK - 1) / BK;
  const bool three = p.passes >= 3;

  if (threadIdx.x == 0) {
    for (int s = 0; s < p.nsets; ++s) {
      tma_prefetch_desc(&p.a_hi[s]);
      tma_prefetch_desc(&p.b_hi[s]);
      if (three) {
        tma_prefetch_desc(&p.a_lo[s]);
        tma_prefetch_desc(&p.b_lo[s]);
        if constexpr (F8) {
          tma_prefetch_desc(&p.a_x8[s]);
          tma_prefetch_desc(&p.b_x8[s]);
        }
      }
    }
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], kWGs * CLUSTER);   // one arrival per consumer warpgroup of each CTA of the cluster
    }
    if constexpr (OVERLAP) {
      mbar_init(acc_full, 256);      // every consumer thread, after its accumulators are in acc_stage
      mbar_init(acc_empty, 128);     // every epilogue thread, after its last read of acc_stage
    }
    fence_mbar_init();
  }
  // in a pair, the barriers of both CTAs are initialised before either multicasts into the other or arrives on its
  // barriers
  if constexpr (CLUSTER == 2) cluster_sync();
  else __syncthreads();
  // f16f8: which cross terms each operand pair needs (see GemmParams::a_res_flag), bit s for operand pair s; the same
  // for every CTA of the launch. Bit masks, not arrays: an array indexed by the run-time pair would live in local memory.
  [[maybe_unused]] uint32_t term_lh = 0u, term_hl = 0u;
  if constexpr (F8) {
#pragma unroll
    for (int s = 0; s < kMaxSets; ++s) {
      term_lh |= uint32_t(s < p.nsets && (p.a_res_flag[s] == nullptr || __ldg(p.a_res_flag[s]) != 0u)) << s;
      term_hl |= uint32_t(s < p.nsets && (p.b_res_flag[s] == nullptr || __ldg(p.b_res_flag[s]) != 0u)) << s;
    }
  }

  // One epilogue share (warp_q, grp) of the tile in acc_stage: rows 32 warp_q .. +31 and the 32-column chunks grp,
  // grp + 2, ... (column group g takes the chunks g, g + 2, ...), with its own epilogue object and staging tile.
  auto share_coord = [&](int model, int tile_m, int tile_n, int warp_q, int grp, bool alternate) {
    TileCoord tc;
    tc.model = model;
    tc.m_blk = tile_m;
    tc.n_blk = tile_n;
    tc.col0 = tile_n * BN;
    tc.warp_q = warp_q;
    tc.grp = grp;
    tc.lane = lane;
    tc.row = tc.m_blk * kBM + tc.warp_q * 32 + lane;
    tc.alternate = alternate;
    return tc;
  };
  // Tall tiles: the share of the tile's rows 32 q .. +31 (q = 0..5) under the kBM tiling's coordinates
  [[maybe_unused]] auto tall_share_coord = [&](int model, int tile_m, int tile_n, int q, int grp) {
    const int quarter = tile_m * (BM / 32) + q;   // 32-row quarter of the output rows
    return share_coord(model, quarter >> 2, tile_n, quarter & 3, grp, false);
  };
  auto share_staging = [&](int warp_q, int grp) { return smem + SM::kEpiOff + (grp * 4 + warp_q) * Epi::kWarpStageBytes; };
  constexpr int kChunks = BN / EC;
  static_assert(kChunks % 2 == 0, "the two column groups alternate chunks");
  // chunk c of this thread's row of acc_stage, in its rows 32 q .. +31
  auto read_chunk = [&](int q, int c, uint32_t (&r)[EC]) {
    const float* src = acc_stage + (q * 32 + lane) * SM::kAccLd + c * EC;
#pragma unroll
    for (int j = 0; j < EC; ++j) r[j] = __float_as_uint(src[j]);
  };

  if (warp < 4) {
    // ======================= TMA producer =======================
    if constexpr (OVERLAP) reg_dealloc<kProducerRegs>();
    if constexpr (TALL) reg_dealloc<kTallProducerRegs>();
    if (threadIdx.x == 0) {
      const uint32_t stage_bytes = (three && !F8) ? uint32_t(SM::kStage) : uint32_t(SM::kATile + SM::kBTile);
      int stage = 0;
      uint32_t phase = 0;
      auto next = [&]() {
        if (++stage == STAGES) {
          stage = 0;
          phase ^= 1;
        }
      };
      // A tiles. In a cluster of two both CTAs need the same A tile at every K block: the CTA of rank kb % 2 loads it
      // for both (multicast), so each A tile crosses from L2 once per cluster. B tiles are loaded by each CTA for itself.
      // Every CTA's full barrier still expects the whole stage.
      auto load_a = [&](void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2, int kb) {
        if constexpr (CLUSTER == 1) tma_load_3d(dst, m, bar, c0, c1, c2);
        else if ((kb & 1) == cta_rank) tma_load_3d_multicast(dst, m, bar, c0, c1, c2, uint16_t(0x3));
      };
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        int model, tile_m, tile_n;
        decode_tile(tile, model, tile_m, tile_n);
        const int a_row0 = tile_m * BM, b_row0 = tile_n * BN;
        if constexpr (F8) {
          // sweep 1: the 8-bit planes (skipped for passes == 1); sweep 2: the fp16 planes
          for (int sweep = three ? 0 : 1; sweep < 2; ++sweep)
            for (int set = 0; set < p.nsets; ++set) {
              int am, bm;
              operand_models(model, set, am, bm);
              // cross terms of this operand pair: t_lh = A.l8 x B.h8 (needs A's residual), t_hl = A.h8 x B.l8
              const bool t_lh = (term_lh >> set) & 1u, t_hl = (term_hl >> set) & 1u;
              if (sweep == 0 && !t_lh && !t_hl) continue;
              const uint32_t bytes = sweep == 1 ? stage_bytes : (uint32_t(t_lh) + uint32_t(t_hl)) * (stage_bytes / 2);
              for (int kb = 0; kb < kblocks; ++kb) {
                mbar_wait(&empty_bar[stage], phase ^ 1);
                uint8_t* st = smem + stage * SM::kStage;
                uint64_t* bar = &full_bar[stage];
                mbar_expect_tx(bar, bytes);
                const int k0 = kb * BK;
                if (sweep == 1) {
                  uint8_t* sa = st;
                  uint8_t* sb = st + SM::kATile;
                  if constexpr (!A_MN) load_a(sa, &p.a_hi[set], bar, k0, a_row0, am, kb);
                  else {
#pragma unroll
                    for (int j = 0; j < BM / 64; ++j) load_a(sa + j * (BK * 128), &p.a_hi[set], bar, a_row0 + j * 64, k0, am, kb);
                  }
                  if constexpr (!B_MN) tma_load_3d(sb, &p.b_hi[set], bar, k0, b_row0, bm);
                  else {
#pragma unroll
                    for (int j = 0; j < BN / 64; ++j) tma_load_3d(sb + j * (BK * 128), &p.b_hi[set], bar, b_row0 + j * 64, k0, bm);
                  }
                } else {
                  // 8-bit tiles: F8_NATIVE K-major [rows][BK] bytes (64-byte swizzle), else MN-major [BK][128] bytes
                  // (unswizzled)
                  uint8_t* sa_h = st;
                  uint8_t* sa_l = st + SM::kATile / 2;
                  uint8_t* sb_h = st + SM::kATile;
                  uint8_t* sb_l = sb_h + SM::kBTile / 2;
                  const int ac0 = F8_NATIVE ? k0 : a_row0, ac1 = F8_NATIVE ? a_row0 : k0;
                  const int bc0 = F8_NATIVE ? k0 : b_row0, bc1 = F8_NATIVE ? b_row0 : k0;
                  if (t_hl) load_a(sa_h, &p.a_lo[set], bar, ac0, ac1, am, kb);
                  if (t_lh) load_a(sa_l, &p.a_x8[set], bar, ac0, ac1, am, kb);
                  if (t_lh) tma_load_3d(sb_h, &p.b_lo[set], bar, bc0, bc1, bm);
                  if (t_hl) tma_load_3d(sb_l, &p.b_x8[set], bar, bc0, bc1, bm);
                }
                next();
              }
            }
        } else {
          for (int set = 0; set < p.nsets; ++set) {
            int am, bm;
            operand_models(model, set, am, bm);
            for (int kb = 0; kb < kblocks; ++kb) {
              mbar_wait(&empty_bar[stage], phase ^ 1);
              uint8_t* sa_hi = smem + stage * SM::kStage;
              uint8_t* sa_lo = sa_hi + SM::kATile;
              uint8_t* sb_hi = sa_lo + SM::kATile;
              uint8_t* sb_lo = sb_hi + SM::kBTile;
              uint64_t* bar = &full_bar[stage];
              mbar_expect_tx(bar, stage_bytes);
              const int k0 = kb * BK;
              if constexpr (!A_MN) {
                load_a(sa_hi, &p.a_hi[set], bar, k0, a_row0, am, kb);
                if (three) load_a(sa_lo, &p.a_lo[set], bar, k0, a_row0, am, kb);
              } else {
#pragma unroll
                for (int j = 0; j < BM / 64; ++j) {
                  load_a(sa_hi + j * (BK * 128), &p.a_hi[set], bar, a_row0 + j * 64, k0, am, kb);
                  if (three) load_a(sa_lo + j * (BK * 128), &p.a_lo[set], bar, a_row0 + j * 64, k0, am, kb);
                }
              }
              if constexpr (!B_MN) {
                tma_load_3d(sb_hi, &p.b_hi[set], bar, k0, b_row0, bm);
                if (three) tma_load_3d(sb_lo, &p.b_lo[set], bar, k0, b_row0, bm);
              } else {
#pragma unroll
                for (int j = 0; j < BN / 64; ++j) {
                  tma_load_3d(sb_hi + j * (BK * 128), &p.b_hi[set], bar, b_row0 + j * 64, k0, bm);
                  if (three) tma_load_3d(sb_lo + j * (BK * 128), &p.b_lo[set], bar, b_row0 + j * 64, k0, bm);
                }
              }
              next();
            }
          }
        }
      }
    }
  } else if (!OVERLAP || warp < 12) {
    // ======================= wgmma consumers (+ the epilogue where !OVERLAP) =======================
    if constexpr (OVERLAP) reg_alloc<kConsumerRegs>();
    if constexpr (TALL) reg_alloc<kTallConsumerRegs>();
    const int ctid = threadIdx.x - 128;      // 0..255 (tall tiles: 0..383)
    const int wg = ctid >> 7;                // rows 64 wg .. +63 of the tile
    const int wl = ctid & 127;               // thread within the warpgroup
    auto consumer_sync = [] { named_sync(1, 256); };
    // descriptor geometry: K-major rows of BK * 2 bytes (128B swizzle at BK = 64, 64B at BK = 32); MN-major 64-element
    // rows of 128 B, 64-element blocks BK * 128 B apart
    constexpr uint32_t a_sw = (A_MN || BK == 64) ? 1 : 2, b_sw = (B_MN || BK == 64) ? 1 : 2;
    constexpr uint32_t a_lbo = A_MN ? BK * 128 : 16, b_lbo = B_MN ? BK * 128 : 16;
    constexpr uint32_t a_sbo = (A_MN || BK == 64) ? 1024 : 512, b_sbo = (B_MN || BK == 64) ? 1024 : 512;
    constexpr uint32_t a_kstep = A_MN ? 2048 : 32, b_kstep = B_MN ? 2048 : 32;   // bytes per K = 16 slice
    const uint32_t a_wg = A_MN ? uint32_t(wg) * (BK * 128) : uint32_t(wg) * (64 * BK * 2);  // this warpgroup's 64 rows
    auto adesc = [&](uint32_t tile, int k) { return make_wgmma_desc(tile + a_wg + k * a_kstep, a_lbo, a_sbo, a_sw); };
    auto bdesc = [&](uint32_t tile, int k) { return make_wgmma_desc(tile + k * b_kstep, b_lbo, b_sbo, b_sw); };
    constexpr bool F16 = F8;   // f16f8 multiplies fp16 (and widened e5m2) planes; bf16x3 bf16 planes

    float acc[64];
    float accx[SPLIT_ACC || F8_NATIVE ? 64 : 1];   // split cross-term accumulator / one K block of E5M2 cross terms
    int stage = 0;
    uint32_t phase = 0;
    uint32_t acc_phase = 0;   // OVERLAP: parity of the tiles handed to the epilogue warpgroup
    auto next = [&]() {
      if (++stage == STAGES) {
        stage = 0;
        phase ^= 1;
      }
    };
    // A stage is free once the consumers of every CTA of the cluster are done with it: the peer's multicast writes this
    // CTA's stage as well as its own
    auto release = [&](int s) {
      if (wl == 0) {
        mbar_arrive(&empty_bar[s]);
        if constexpr (CLUSTER == 2) mbar_arrive_cluster(&empty_bar[s], uint32_t(cta_rank ^ 1));
      }
    };

    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      int model, tile_m, tile_n;
      decode_tile(tile, model, tile_m, tile_n);
#pragma unroll
      for (int i = 0; i < 64; ++i) acc[i] = 0.f;
      if constexpr (SPLIT_ACC || F8_NATIVE) {
#pragma unroll
        for (int i = 0; i < 64; ++i) accx[i] = 0.f;
      }
      if constexpr (F8) {
        // sweep 1 over one operand pair with a compile-time choice of cross terms (LH: A.l8 x B.h8, HL: A.h8 x B.l8), so
        // that no wgmma sits behind a run-time branch between fence and commit
        auto cross_sweep = [&](auto lh, auto hl) {
          constexpr bool LH = decltype(lh)::value, HL = decltype(hl)::value;
          for (int kb = 0; kb < kblocks; ++kb) {
            mbar_wait(&full_bar[stage], phase);
            const uint8_t* st = smem + stage * SM::kStage;
            if constexpr (F8_NATIVE) {
              // K-major 8-bit tiles [rows][64 B] with the 64-byte swizzle: the geometry of a bf16 tile at K block 32
              // (8-row groups 512 B apart, 32 B per k32 slice)
              const uint32_t sa_h = smem_u32(st) + uint32_t(wg) * (64 * BK), sa_l = sa_h + SM::kATile / 2;
              const uint32_t sb_h = smem_u32(st + SM::kATile), sb_l = sb_h + SM::kBTile / 2;
              auto d8 = [](uint32_t tile, int k) { return make_wgmma_desc(tile + k * 32, 16, 512, 2); };
              wgmma_fence();
#pragma unroll
              for (int k = 0; k < BK / 32; ++k) {
                if constexpr (LH) wgmma_n128_e5m2(accx, d8(sa_l, k), d8(sb_h, k));
                if constexpr (HL) wgmma_n128_e5m2(accx, d8(sa_h, k), d8(sb_l, k));
              }
              wgmma_commit();
              wgmma_wait<0>();
              release(stage);
              next();
              // FP8 wgmma adds with fewer bits than fp32 and truncates, so its sums drift with their length: each K
              // block's cross terms are promoted into the fp32 accumulator
#pragma unroll
              for (int i = 0; i < 64; ++i) {
                acc[i] += accx[i];
                accx[i] = 0.f;
              }
            } else {
              uint8_t* wide = smem + SM::kAccOff;   // widened tiles: A.h8, A.l8, B.h8, B.l8 (fp16)
              const uint32_t wa_h = smem_u32(wide), wa_l = wa_h + SM::kATile, wb_h = wa_l + SM::kATile,
                             wb_l = wb_h + SM::kBTile;
              consumer_sync();   // both warpgroups are done with the widened tiles (and the previous epilogue)
              if constexpr (HL) widen_tile<kBM>(st, wide, ctid);
              if constexpr (LH) widen_tile<kBM>(st + SM::kATile / 2, wide + SM::kATile, ctid);
              if constexpr (LH) widen_tile<BN>(st + SM::kATile, wide + 2 * SM::kATile, ctid);
              if constexpr (HL) widen_tile<BN>(st + SM::kATile + SM::kBTile / 2, wide + 2 * SM::kATile + SM::kBTile, ctid);
              fence_proxy_async_smem();   // generic-proxy writes -> visible to wgmma
              consumer_sync();
              release(stage);
              next();
              wgmma_fence();
#pragma unroll
              for (int k = 0; k < BK / 16; ++k) {
                if constexpr (LH) wgmma_n128<true, A_MN, B_MN>(acc, adesc(wa_l, k), bdesc(wb_h, k));
                if constexpr (HL) wgmma_n128<true, A_MN, B_MN>(acc, adesc(wa_h, k), bdesc(wb_l, k));
              }
              wgmma_commit();
              wgmma_wait<0>();
            }
          }
        };
        if (three) {
          for (int set = 0; set < p.nsets; ++set) {
            const bool t_lh = (term_lh >> set) & 1u, t_hl = (term_hl >> set) & 1u;
            if (t_lh && t_hl) cross_sweep(std::true_type{}, std::true_type{});
            else if (t_lh) cross_sweep(std::true_type{}, std::false_type{});
            else if (t_hl) cross_sweep(std::false_type{}, std::true_type{});
          }
          constexpr float kDown = 1.0f / float(1 << kLoShift);
#pragma unroll
          for (int i = 0; i < 64; ++i) acc[i] *= kDown;   // exact: the cross terms were accumulated at 2^kLoShift
        }
        for (int it = 0; it < p.nsets * kblocks; ++it) {
          mbar_wait(&full_bar[stage], phase);
          const uint32_t sa = smem_u32(smem + stage * SM::kStage);
          const uint32_t sb = sa + SM::kATile;
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < BK / 16; ++k) wgmma_n128<true, A_MN, B_MN>(acc, adesc(sa, k), bdesc(sb, k));
          wgmma_commit();
          wgmma_wait<0>();
          release(stage);
          next();
        }
      } else {
        for (int it = 0; it < p.nsets * kblocks; ++it) {
          mbar_wait(&full_bar[stage], phase);
          const uint32_t sa_hi = smem_u32(smem + stage * SM::kStage);
          const uint32_t sa_lo = sa_hi + SM::kATile;
          const uint32_t sb_hi = sa_lo + SM::kATile;
          const uint32_t sb_lo = sb_hi + SM::kBTile;
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < BK / 16; ++k) {
            if (three) {
              // small cross terms first, then the dominant hi*hi term
              if constexpr (SPLIT_ACC) {
                wgmma_n128<F16, A_MN, B_MN>(accx, adesc(sa_lo, k), bdesc(sb_hi, k));
                wgmma_n128<F16, A_MN, B_MN>(accx, adesc(sa_hi, k), bdesc(sb_lo, k));
              } else {
                wgmma_n128<F16, A_MN, B_MN>(acc, adesc(sa_lo, k), bdesc(sb_hi, k));
                wgmma_n128<F16, A_MN, B_MN>(acc, adesc(sa_hi, k), bdesc(sb_lo, k));
              }
            }
            wgmma_n128<F16, A_MN, B_MN>(acc, adesc(sa_hi, k), bdesc(sb_hi, k));
          }
          wgmma_commit();
          wgmma_wait<0>();
          release(stage);
          next();
        }
        if constexpr (SPLIT_ACC) {
#pragma unroll
          for (int i = 0; i < 64; ++i) acc[i] += accx[i];
        }
      }

      if constexpr (TALL) {
        // ---- epilogue in two rounds through acc_stage: rows 0..127 of the tile from consumers 0 and 1 (eight warps, warp w
        // plays quarter w % 4, group w / 4, as in line below), then rows 128..191 from consumer 2 (warp w: quarter 4 + w % 2,
        // group w / 2) in acc_stage rows 0..63. Named barriers: kBarRound1Read (0, 1 -> 2: round 1 read, acc_stage free
        // for round 2), kBarRound2Read (2 -> 0, 1: round 2 read, free for the next tile's round 1; 0 and 1 run the next
        // main loop meanwhile), kBarRound1Full / kBarRound2Full (written -> read, within each round).
        constexpr uint32_t kBarRound1Full = 2, kBarRound2Full = 3, kBarRound1Read = 4, kBarRound2Read = 5;
        const bool round2 = wg == 2;
        if (round2) named_sync(kBarRound1Read, 384);
        else if (tile != int(blockIdx.x)) named_sync(kBarRound2Read, 384);
        {
          const int w = wl >> 5, l = wl & 31;
          const int r0 = (wg & 1) * 64 + w * 16 + (l >> 2);
#pragma unroll
          for (int i = 0; i < 64; ++i) {
            const int row = r0 + 8 * ((i >> 1) & 1);
            const int col = 8 * (i >> 2) + 2 * (l & 3) + (i & 1);
            acc_stage[row * SM::kAccLd + col] = acc[i];
          }
        }
        if (round2) named_sync(kBarRound2Full, 128);
        else named_sync(kBarRound1Full, 256);
        const int cw = (ctid >> 5) & 7;
        const int sq = round2 ? cw & 1 : cw & 3;        // quarter of acc_stage
        const int grp = round2 ? cw >> 1 : cw >> 2;
        const TileCoord tc = tall_share_coord(model, tile_m, tile_n, round2 ? 4 + sq : sq, grp);
        Epi epi(p.epi, tc, p.m_total, p.n_total, nullptr);
#pragma unroll 1
        for (int c = grp; c < kChunks; c += 2) {
          uint32_t r[EC];
          read_chunk(sq, c, r);
          epi.chunk(c * EC, r);
        }
        epi.finish();
        if (!round2) named_arrive(kBarRound1Read, 384);
        else if (tile + int(gridDim.x) < num_tiles) named_arrive(kBarRound2Read, 384);
        continue;
      }
      // ---- accumulators -> padded fp32 tile (row-per-thread view for the epilogue)
      // OVERLAP: the epilogue warpgroup has read the previous tile (it ran under this tile's main loop). Otherwise both
      // consumer warpgroups are past their previous epilogue and the widened tiles.
      if constexpr (OVERLAP) mbar_wait(acc_empty, acc_phase ^ 1);
      else consumer_sync();
      {
        const int w = wl >> 5, l = wl & 31;
        const int r0 = wg * 64 + w * 16 + (l >> 2);
#pragma unroll
        for (int i = 0; i < 64; ++i) {
          const int row = r0 + 8 * ((i >> 1) & 1);
          const int col = 8 * (i >> 2) + 2 * (l & 3) + (i & 1);
          acc_stage[row * SM::kAccLd + col] = acc[i];
        }
      }
      if constexpr (OVERLAP) {
        mbar_arrive(acc_full);
        acc_phase ^= 1;
      } else {
        // ======================= epilogue in line: eight warps, warp w plays (w % 4, w / 4) =======================
        consumer_sync();
        const int cw = ctid >> 5, warp_q = cw & 3, grp = cw >> 2;
        const TileCoord tc = share_coord(model, tile_m, tile_n, warp_q, grp, false);
        Epi epi(p.epi, tc, p.m_total, p.n_total, share_staging(warp_q, grp));
#pragma unroll 1
        for (int c = grp; c < kChunks; c += 2) {
          uint32_t r[EC];
          read_chunk(warp_q, c, r);
          epi.chunk(c * EC, r);
        }
        epi.finish();
      }
    }
  } else if constexpr (OVERLAP) {
    // ======================= epilogue warpgroup =======================
    // Warp q plays both of the in-line epilogue's warps (q, 0) and (q, 1), chunk by chunk: chunks 0, 2, ... go to share
    // (q, 0) and chunks 1, 3, ... to share (q, 1). Each share's sums, partial-sum slots, staging and chunk order are
    // those of the in-line mapping, so the outputs do not depend on which warps run them. Consecutive chunks write
    // different staging tiles, so a chunk does not wait for the bulk store issued just before it (staging_wait).
    reg_alloc<kEpilogueRegs>();
    const int warp_q = warp - 12;
    uint32_t acc_phase = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      int model, tile_m, tile_n;
      decode_tile(tile, model, tile_m, tile_n);
      mbar_wait(acc_full, acc_phase);
      acc_phase ^= 1;
      const TileCoord tc0 = share_coord(model, tile_m, tile_n, warp_q, 0, true);
      const TileCoord tc1 = share_coord(model, tile_m, tile_n, warp_q, 1, true);
      Epi epi0(p.epi, tc0, p.m_total, p.n_total, share_staging(warp_q, 0));
      Epi epi1(p.epi, tc1, p.m_total, p.n_total, share_staging(warp_q, 1));
#pragma unroll 1
      for (int c = 0; c < kChunks; c += 2) {
        uint32_t r[EC];
        read_chunk(warp_q, c, r);
        epi0.chunk(c * EC, r);
        read_chunk(warp_q, c + 1, r);
        if (c + 2 == kChunks) mbar_arrive(acc_empty);   // the warp's last read of acc_stage for this tile
        epi1.chunk((c + 1) * EC, r);
      }
      epi0.finish();
      epi1.finish();
    }
  }
  // no CTA of a pair leaves while its peer may still arrive on its barriers
  if constexpr (CLUSTER == 2) cluster_sync();
}

// ------------------------------------------------------------------------------------------------
// Host side
// ------------------------------------------------------------------------------------------------
// Opts the kernel KERN in to `bytes` of dynamic shared memory (above the default 48 KB). The opt-in is per device and
// per kernel, so each instantiation remembers the devices it has made it on.
template <auto KERN>
inline cudaError_t opt_in_smem(int bytes, int device) {
  static bool configured[64] = {};
  if (device >= 0 && device < 64 && configured[device]) return cudaSuccess;
  const cudaError_t e = cudaFuncSetAttribute(KERN, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  if (e == cudaSuccess && device >= 0 && device < 64) configured[device] = true;
  return e;
}

// The most clusters of `cluster` CTAs of the kernel KERN that can be resident on `device` at once (0: none), queried
// once per device and cluster size.
template <auto KERN>
inline int max_active_clusters(int cluster, int threads, int bytes, int device) {
  static int known[64][2] = {};   // [device][cluster - 1]: the count + 1 once queried
  if (device >= 0 && device < 64 && known[device][cluster - 1]) return known[device][cluster - 1] - 1;
  cudaLaunchConfig_t cfg = {};
  cudaLaunchAttribute attr;
  attr.id = cudaLaunchAttributeClusterDimension;
  attr.val.clusterDim.x = cluster;
  attr.val.clusterDim.y = 1;
  attr.val.clusterDim.z = 1;
  cfg.gridDim = dim3(cluster);
  cfg.blockDim = dim3(threads);
  cfg.dynamicSmemBytes = bytes;
  cfg.attrs = &attr;
  cfg.numAttrs = 1;
  int n = 0;
  if (cudaOccupancyMaxActiveClusters(&n, KERN, &cfg) != cudaSuccess) n = 0;
  if (device >= 0 && device < 64) known[device][cluster - 1] = n + 1;
  return n;
}

// Cluster size of a launch: two CTAs along N, which share each A tile, where a model's column-tile count is even (a
// column pair never straddles two tile rows) and each tile's K loop runs at least kClusterMinKBlocks K blocks over its
// operand sets; one otherwise, and on the widened f16f8 path. The pair reads a quarter fewer operand bytes from L2 but
// runs in lockstep, each stage waiting for both CTAs' consumers. On an H100 at 700 W the main loop alone (config 2
// shapes) got 13-21 % shorter in pairs at 64 K blocks (decode) and 2 x 64 (the weight gradient), and no shorter at 8
// (encode, dcode). Only those lengths were measured: where between 8 and 64 blocks pairs start to pay is not known, and
// 64 is the shortest loop they were seen to pay on.
constexpr int kClusterMinKBlocks = 64;
inline int gemm_cluster_size(int tiles_n, int k_blocks, bool widened) {
  return tiles_n % 2 == 0 && k_blocks >= kClusterMinKBlocks && !widened ? 2 : 1;
}

// Launches gemm_split_kernel<..., CLUSTER> on `st` as a persistent grid of clusters of CLUSTER CTAs (2 only where
// p.tiles_n is even): one cluster per column group of CLUSTER tiles, at most as many as are resident at once, and at
// most one CTA per SM (`sms` of them on `device`, the current device). BM: rows of the output tile; p.tiles_m must be
// gemm_tiles_m<BM>(p.m_total).
template <class Epi, bool A_MN, bool B_MN, bool SPLIT_ACC, int ARITH, bool F8_NATIVE, int CLUSTER, int BM = kBM>
cudaError_t launch_gemm_cluster_t(const GemmParams<typename Epi::Params>& p, int device, int sms, cudaStream_t st) {
  constexpr auto kern = gemm_split_kernel<Epi, A_MN, B_MN, SPLIT_ACC, ARITH, F8_NATIVE, CLUSTER, BM>;
  constexpr int bytes = GemmSmem<Epi::kWarpStageBytes, ARITH, F8_NATIVE, BM>::kBytes;
  constexpr int threads = gemm_threads<Epi, ARITH, F8_NATIVE, BM>();
  if (p.tiles_n % CLUSTER != 0) return cudaErrorInvalidValue;
  if (BM != kBM && p.tiles_m != gemm_tiles_m<BM>(p.m_total)) return cudaErrorInvalidValue;
  cudaError_t e = opt_in_smem<kern>(bytes, device);
  if (e != cudaSuccess) return e;
  long long slots = sms / CLUSTER;
  if constexpr (CLUSTER > 1) {
    const int resident = max_active_clusters<kern>(CLUSTER, threads, bytes, device);
    if (resident <= 0) return cudaErrorInvalidConfiguration;
    if (resident < slots) slots = resident;
  }
  const long long units = (long long)p.n_models * p.tiles_m * (p.tiles_n / CLUSTER);
  cudaLaunchConfig_t cfg = {};
  cudaLaunchAttribute attr;
  attr.id = cudaLaunchAttributeClusterDimension;
  attr.val.clusterDim.x = CLUSTER;
  attr.val.clusterDim.y = 1;
  attr.val.clusterDim.z = 1;
  cfg.gridDim = dim3((unsigned)(CLUSTER * (units < slots ? units : slots)));
  cfg.blockDim = dim3(threads);
  cfg.dynamicSmemBytes = bytes;
  cfg.stream = st;
  cfg.attrs = &attr;
  cfg.numAttrs = CLUSTER > 1 ? 1 : 0;
  e = cudaLaunchKernelEx(&cfg, kern, p);
  return e != cudaSuccess ? e : cudaGetLastError();
}

// The same with the cluster size given at run time (1 or 2; always 1 on the widened f16f8 path).
template <class Epi, bool A_MN, bool B_MN, bool SPLIT_ACC, int ARITH, bool F8_NATIVE, int BM = kBM>
cudaError_t launch_gemm_clusters(const GemmParams<typename Epi::Params>& p, int device, int sms, cudaStream_t st,
                                 int cluster) {
  if (cluster == 1) return launch_gemm_cluster_t<Epi, A_MN, B_MN, SPLIT_ACC, ARITH, F8_NATIVE, 1, BM>(p, device, sms, st);
  if constexpr (ARITH != kArithF16F8 || F8_NATIVE) {
    if (cluster == 2) return launch_gemm_cluster_t<Epi, A_MN, B_MN, SPLIT_ACC, ARITH, F8_NATIVE, 2, BM>(p, device, sms, st);
  }
  return cudaErrorInvalidValue;
}

// The cluster size launch_gemm takes for p's shape on this path (gemm_cluster_size).
template <int ARITH, bool F8_NATIVE, class EpiParams>
inline int gemm_launch_cluster(const GemmParams<EpiParams>& p) {
  const int k_blocks = p.nsets * ((p.k_total + gemm_bk(ARITH) - 1) / gemm_bk(ARITH));
  return gemm_cluster_size(p.tiles_n, k_blocks, ARITH == kArithF16F8 && !F8_NATIVE);
}

// Launches gemm_split_kernel in the cluster size that p's shape and path take.
template <class Epi, bool A_MN, bool B_MN, bool SPLIT_ACC, int ARITH, bool F8_NATIVE, int BM = kBM>
cudaError_t launch_gemm(const GemmParams<typename Epi::Params>& p, int device, int sms, cudaStream_t st) {
  return launch_gemm_clusters<Epi, A_MN, B_MN, SPLIT_ACC, ARITH, F8_NATIVE, BM>(p, device, sms, st,
                                                                                gemm_launch_cluster<ARITH, F8_NATIVE>(p));
}

// ------------------------------------------------------------------------------------------------
// Epilogue: plain fp32 store  out[model][row][col] = acc   (dW tiles; self-test)
// ------------------------------------------------------------------------------------------------
struct EpiStoreF32 {
  static constexpr int kCols = 32;
  static constexpr int kWarpStageBytes = 0;
  static constexpr bool kInline = true;   // a few percent of a weight-gradient tile (K = batch)
  struct Params {
    float* out;
    long long model_stride;  // elements
    int ld;                  // elements
    float scale;             // out = acc * scale (0 is read as 1: zero-initialised params keep working)
  };
  const Params& P;
  const TileCoord& T;
  int m_total, n_total;
  __device__ EpiStoreF32(const Params& p, const TileCoord& t, int m, int n, uint8_t*)
      : P(p), T(t), m_total(m), n_total(n) {}
  __device__ __forceinline__ void chunk(int c, const uint32_t (&r)[32]) {
    if (T.row >= m_total) return;
    float* o = P.out + (long long)T.model * P.model_stride + (long long)T.row * P.ld + T.col0 + c;
    const float sc = P.scale == 0.f ? 1.f : P.scale;
#pragma unroll
    for (int j = 0; j < 32; j += 4) {
      if (T.col0 + c + j < n_total) {  // n_total % 4 == 0 is required by the host
        float4 v = make_float4(__uint_as_float(r[j]) * sc, __uint_as_float(r[j + 1]) * sc,
                               __uint_as_float(r[j + 2]) * sc, __uint_as_float(r[j + 3]) * sc);
        *reinterpret_cast<float4*>(o + j) = v;
      }
    }
  }
  __device__ __forceinline__ void finish() {}
};

}  // namespace sce
