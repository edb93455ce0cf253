// sce_engine.cuh — what the translation units of libsce.so share (internal; the ABI is include/sce.h): the error
// state, the launcher, operand planes and the workspace carve, the GEMM operand maps and launchers, and the launchers
// of the row kernels that more than one family of entry points runs.
#pragma once
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <type_traits>
#include <utility>

#include "../../include/sce.h"
#include "sce_gemm.cuh"
#include "sce_kernels.cuh"
#include "sce_tmap.h"

using namespace sce;

// ------------------------------------------------------------------------------------------------
// errors and launches
// ------------------------------------------------------------------------------------------------
// Records the message of a failing call for sce_last_error (one per thread, whichever file failed) and returns `code`
// (sce_abi.cu). Hidden: it is libsce's own, not an export.
__attribute__((visibility("hidden"))) int fail(int code, const char* fmt, ...);
#define CUDA_TRY(x)                                                                            \
  do {                                                                                         \
    cudaError_t e_ = (x);                                                                      \
    if (e_ != cudaSuccess) return fail(SCE_ERR_CUDA, "%s failed: %s", #x, cudaGetErrorString(e_)); \
  } while (0)
// returns the SCE_ERR_* code of a failed call
#define TRY(x)                       \
  do {                               \
    if (int rc_ = (x)) return rc_;   \
  } while (0)

// The kernel launches of one call on one stream. Every launch goes through launch() (or launch_gemm_t), which checks
// it and counts it; the entry points that report their launches (sce_last_launch_count) read `count`.
struct Launcher {
  cudaStream_t st;
  int count = 0;
  template <class... P, class... A>
  int launch(void (*kernel)(P...), dim3 grid, dim3 block, size_t smem, A&&... args) {
    kernel<<<grid, block, smem, st>>>(std::forward<A>(args)...);
    CUDA_TRY(cudaGetLastError());
    ++count;
    return SCE_OK;
  }
};

// ------------------------------------------------------------------------------------------------
// operand planes and workspaces
// ------------------------------------------------------------------------------------------------
// The planes of one operand tensor. bf16x3: hi, lo = bf16 planes (2 B / element each), x8 = nullptr. f16f8: hi = fp16
// plane, lo = E5M2 plane of the values, x8 = E5M2 plane of the scaled residuals (1 B / element each): 4 B / element
// either way. The batch-major 8-bit copies of native dW are Planes without a 16-bit plane.
struct Planes {
  void* hi;
  void* lo;
  uint8_t* x8;
  bool f8;
  size_t lo_size() const { return f8 ? 1 : 2; }   // bytes per element of lo (and of x8)
  // the planes from element `e` on (a model's slab)
  Planes at(size_t e) const {
    return {hi ? static_cast<uint8_t*>(hi) + 2 * e : nullptr, lo ? static_cast<uint8_t*>(lo) + lo_size() * e : nullptr,
            x8 ? x8 + e : nullptr, f8};
  }
  // zero the first `count` elements of every plane
  cudaError_t zero(size_t count, cudaStream_t st) const {
    cudaError_t e = cudaMemsetAsync(hi, 0, 2 * count, st);
    if (e == cudaSuccess) e = cudaMemsetAsync(lo, 0, lo_size() * count, st);
    if (e == cudaSuccess && x8) e = cudaMemsetAsync(x8, 0, count, st);
    return e;
  }
};

static size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

struct Carve {
  uint8_t* base;
  size_t off;
  template <class T>
  T* take(size_t count) {
    off = align_up(off, 1024);
    T* p = base ? reinterpret_cast<T*>(base + off) : nullptr;
    off += count * sizeof(T);
    return p;
  }
  // the planes of `count` elements of one operand tensor: 16-bit, then a second 16-bit plane (bf16x3) or two 8-bit ones
  Planes planes(size_t count, bool f8) {
    Planes p{take<uint16_t>(count), nullptr, nullptr, f8};
    if (f8) {
      p.lo = take<uint8_t>(count);
      p.x8 = take<uint8_t>(count);
    } else {
      p.lo = take<uint16_t>(count);
    }
    return p;
  }
  // the batch-major copies of the two 8-bit planes of `count` elements (f16f8), which have no 16-bit plane
  Planes copies(size_t count) { return {nullptr, take<uint8_t>(count), take<uint8_t>(count), true}; }
};

// a caller's workspace: at least `need` bytes at a 1024-byte aligned address (the carves align their buffers to it)
static int check_workspace(const void* ws, size_t have, size_t need, const char* prefix) {
  if (!ws || have < need)
    return fail(SCE_ERR_WORKSPACE, "%sworkspace too small: have %zu bytes, need %zu", prefix, have, need);
  if (reinterpret_cast<uintptr_t>(ws) % 1024) return fail(SCE_ERR_WORKSPACE, "%sworkspace must be 1024-byte aligned", prefix);
  return SCE_OK;
}

// ------------------------------------------------------------------------------------------------
// device and arithmetic
// ------------------------------------------------------------------------------------------------
// the current device and its SM count, if libsce runs on it: sm_90, with the driver's tensor-map encoder
static int query_device(int* device, int* sm_count) {
  int dev = 0, major = 0, sms = 0;
  CUDA_TRY(cudaGetDevice(&dev));
  CUDA_TRY(cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev));
  CUDA_TRY(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  if (major != 9) return fail(SCE_ERR_NO_DEVICE, "libsce needs an sm_90 device (found compute capability %d.x)", major);
  if (!get_encode_fn()) return fail(SCE_ERR_NO_DEVICE, "cuTensorMapEncodeTiled driver entry point not available");
  *device = dev;
  *sm_count = sms;
  return SCE_OK;
}

// SCE_ARITH=bf16x3|f16f8: the arithmetic the environment pins arith = AUTO to (include/sce.h), else SCE_ARITH_AUTO
static int env_arith() {
  const char* v = getenv("SCE_ARITH");
  if (v && !strcmp(v, "bf16x3")) return SCE_ARITH_BF16X3;
  if (v && !strcmp(v, "f16f8")) return SCE_ARITH_F16F8;
  return SCE_ARITH_AUTO;
}

// Calls f(arith) with the plan's arithmetic as a compile-time constant (std::integral_constant<int, AR>)
template <class F>
static auto with_arith(int arith, F&& f) {
  return arith == kArithF16F8 ? f(std::integral_constant<int, kArithF16F8>{}) : f(std::integral_constant<int, kArithBf16x3>{});
}

// ------------------------------------------------------------------------------------------------
// GEMM operand maps and launchers
// ------------------------------------------------------------------------------------------------
struct OperandMaps {   // tensor maps of one operand's planes
  CUtensorMap hi, lo, x8;
};
struct GemmMaps {      // tensor maps of one GEMM for one batch size
  OperandMaps a[kMaxSets], b[kMaxSets];
};

// K-major 16-bit tiles [rows][bk], bk = gemm_bk(arith): the swizzle span is one tile row of 2 bk bytes
static CUtensorMapSwizzle swizzle_for_bk(int bk) {
  return bk * 2 == 64 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_128B;
}

// The planes of one operand [models][rows][cols] (cols contiguous, `mpitch` elements between models) as GEMM operand
// maps. kmajor_bk != 0: K-major tiles [box_rows][kmajor_bk]; else MN-major tiles of `box_rows` k-rows by 64 (16-bit)
// / 128 (8-bit) contiguous elements. K-major 8-bit tiles (64-byte rows in f16f8) carry the 64-byte swizzle E5M2 wgmma
// reads; MN-major ones arrive unswizzled and the GEMM widens them to fp16 (widen_tile).
static bool operand_maps(OperandMaps& m, const Planes& P, uint64_t models, uint64_t rows, uint64_t cols, uint64_t mpitch,
                         uint32_t box_rows, int kmajor_bk) {
  bool ok;
  if (kmajor_bk) {
    ok = make_tmap_bf16_box(&m.hi, P.hi, models, rows, cols, cols, mpitch, kmajor_bk, box_rows, swizzle_for_bk(kmajor_bk));
    if (P.f8)
      ok = ok && make_tmap_u8_box(&m.lo, P.lo, models, rows, cols, cols, mpitch, kmajor_bk, box_rows, CU_TENSOR_MAP_SWIZZLE_64B) &&
           make_tmap_u8_box(&m.x8, P.x8, models, rows, cols, cols, mpitch, kmajor_bk, box_rows, CU_TENSOR_MAP_SWIZZLE_64B);
    else
      ok = ok && make_tmap_bf16_box(&m.lo, P.lo, models, rows, cols, cols, mpitch, kmajor_bk, box_rows, swizzle_for_bk(kmajor_bk));
  } else {
    ok = make_tmap_bf16(&m.hi, P.hi, models, rows, cols, cols, mpitch, box_rows);
    if (P.f8)
      ok = ok && make_tmap_u8_box(&m.lo, P.lo, models, rows, cols, cols, mpitch, 128, box_rows, CU_TENSOR_MAP_SWIZZLE_NONE) &&
           make_tmap_u8_box(&m.x8, P.x8, models, rows, cols, cols, mpitch, 128, box_rows, CU_TENSOR_MAP_SWIZZLE_NONE);
    else
      ok = ok && make_tmap_bf16(&m.lo, P.lo, models, rows, cols, cols, mpitch, box_rows);
  }
  return ok;
}

// The weight gradient's operand P [models][k_rows][cols] (`mpitch` elements between models), reduced over its k_rows:
// MN-major tiles of bk rows. With T, the 8-bit planes come from P's batch-major copies T [models][cols][t_pitch] instead
// (batch_major), K-major tiles [t_rows][64 B] with the 64-byte swizzle E5M2 wgmma reads (t_rows: the tile's rows on
// this side, kBN for B, the launch's BM for A); only k_rows columns of T are exposed, so the tail of a short batch reads
// as zero.
static bool dw_operand_maps(OperandMaps& m, const Planes& P, const Planes* T, uint64_t models, uint64_t k_rows,
                            uint64_t cols, uint64_t mpitch, uint64_t t_pitch, int bk, uint32_t t_rows = kBM) {
  if (!T) return operand_maps(m, P, models, k_rows, cols, mpitch, bk, 0);
  return make_tmap_bf16(&m.hi, P.hi, models, k_rows, cols, cols, mpitch, bk) &&
         make_tmap_u8_box(&m.lo, T->lo, models, cols, k_rows, t_pitch, cols * t_pitch, bk, t_rows, CU_TENSOR_MAP_SWIZZLE_64B) &&
         make_tmap_u8_box(&m.x8, T->x8, models, cols, k_rows, t_pitch, cols * t_pitch, bk, t_rows, CU_TENSOR_MAP_SWIZZLE_64B);
}

// device flags "this operand's residual plane is all zeros" (f16f8; GemmParams::a_res_flag), nullptr = unknown
struct ResFlags {
  const uint32_t* a[kMaxSets] = {nullptr, nullptr};
  const uint32_t* b[kMaxSets] = {nullptr, nullptr};
};

// the tensor maps of operand set `s` into the kernel's parameters
template <class EpiParams>
static void set_operand_maps(GemmParams<EpiParams>& gp, int s, const OperandMaps& a, const OperandMaps& b) {
  gp.a_hi[s] = a.hi;
  gp.a_lo[s] = a.lo;
  gp.a_x8[s] = a.x8;
  gp.b_hi[s] = b.hi;
  gp.b_lo[s] = b.lo;
  gp.b_x8[s] = b.x8;
}

// a_batched / b_batched of the operand sets that hold one slab per model
static const int kOnes[2] = {1, 1};

// One GEMM over `n_models` models on `device` (with `sms` SMs) on output tiles of BM rows (kBMTall: the maps' A boxes
// must be that tall), launched and counted by L
template <class Epi, bool A_MN, bool B_MN, bool SPLIT_ACC, int ARITH, bool NATIVE, int BM = kBM>
static int launch_gemm_t(Launcher& L, int n_models, int device, int sms, const GemmMaps& maps, int nsets,
                         const int* a_batched, const int* b_batched, int k_total, int passes, int m_total, int n_total,
                         const typename Epi::Params& epi, const ResFlags& rf = ResFlags()) {
  GemmParams<typename Epi::Params> gp;
  memset(&gp, 0, sizeof(gp));
  for (int s = 0; s < nsets; ++s) {
    set_operand_maps(gp, s, maps.a[s], maps.b[s]);
    gp.a_batched[s] = a_batched[s];
    gp.b_batched[s] = b_batched[s];
    gp.a_res_flag[s] = rf.a[s];
    gp.b_res_flag[s] = rf.b[s];
  }
  gp.nsets = nsets;
  gp.k_total = k_total;
  gp.passes = passes;
  gp.n_models = n_models;
  gp.m_total = m_total;
  gp.n_total = n_total;
  gp.tiles_m = gemm_tiles_m<BM>(m_total);
  gp.tiles_n = (n_total + kBN - 1) / kBN;
  gp.epi = epi;
  CUDA_TRY((launch_gemm<Epi, A_MN, B_MN, SPLIT_ACC, ARITH, NATIVE, BM>(gp, device, sms, L.st)));
  ++L.count;
  return SCE_OK;
}

// The weight gradient's GEMM (launch_gemm_t's arguments after L): a reduction over rows, both operands as
// dw_operand_maps builds them, fp32 out. bf16x3 keeps split accumulators (f16f8 rescales inside one). `native` (f16f8,
// 8-bit planes from batch-major copies): the cross terms run on E5M2 wgmma; else the 8-bit tiles are widened to fp16.
// `tall` (native only): on kBMTall-row tiles, from maps whose A-side 8-bit boxes are that tall.
template <int AR, class... A>
static int launch_dw_t(Launcher& L, bool native, bool tall, const A&... args) {
  constexpr bool f8 = AR == kArithF16F8;
  if constexpr (f8)
    if (native) {
      if (tall) return launch_gemm_t<EpiStoreF32, true, true, false, AR, true, kBMTall>(L, args...);
      return launch_gemm_t<EpiStoreF32, true, true, false, AR, true>(L, args...);
    }
  return launch_gemm_t<EpiStoreF32, true, true, !f8, AR, false>(L, args...);
}

// ------------------------------------------------------------------------------------------------
// row kernels
// ------------------------------------------------------------------------------------------------
// fp32 rows -> the operand planes of arithmetic AR: n4 float4s, grid-stride over at most 2048 blocks. With `xs`, the
// rows are shifted by `shift` first and the shifted fp32 rows are written to `xs` as well (input_shift plans).
template <int AR>
static int launch_split_rows(Launcher& L, const float* x, const Planes& w, long long n4, uint32_t* flags,
                             float shift = 0.f, float* xs = nullptr) {
  const int blocks = (int)((n4 + 255) / 256 < 2048 ? (n4 + 255) / 256 : 2048);
  if (xs) return L.launch(split_rows_kernel<AR, true>, blocks, 256, 0, x, w.hi, w.lo, w.x8, n4, flags, shift, xs);
  return L.launch(split_rows_kernel<AR>, blocks, 256, 0, x, w.hi, w.lo, w.x8, n4, flags, 0.f, nullptr);
}

// Calls f(nv) with the float4s per thread that dict_rows_kernel needs for rows of d values, ceil(d / 512) rounded up
// to 1, 2, 4, 8 or 16, as a compile-time constant
template <class F>
static auto with_row_vectors(int d, F&& f) {
  const int nv = (d + 511) / 512;
  if (nv == 1) return f(std::integral_constant<int, 1>{});
  if (nv == 2) return f(std::integral_constant<int, 2>{});
  if (nv <= 4) return f(std::integral_constant<int, 4>{});
  if (nv <= 8) return f(std::integral_constant<int, 8>{});   // d <= 4096 (Pythia-6.9b residual width)
  return f(std::integral_constant<int, 16>{});                // d <= 8192
}

template <int MODE, int ARITH, bool NONNEG = false>
static int launch_dict_rows_t(Launcher& L, float* e, const float* dw, float* m, float* v, const Planes& w,
                              float* grad_out, long long rows, int d, int normalize, float floor, AdamHyper h,
                              const uint32_t* health, float* w_f32) {
  return with_row_vectors(d, [&](auto nv) {
    return L.launch(dict_rows_kernel<decltype(nv)::value, MODE, ARITH, NONNEG>, (unsigned)rows, 128, 0, e, dw, m, v,
                    w.hi, w.lo, w.x8, grad_out, d, normalize, floor, h, health, w_f32);
  });
}

namespace sce {
// f16f8 weight gradient: the two 8-bit planes of a batch operand [models][batch_max][cols] (rows 0 .. rows - 1 valid) ->
// batch-major copies [models][cols][ld], ld = batch_max rounded up to 16, so that the weight-gradient GEMM reads them
// K-major over the batch and forms its cross terms on E5M2 wgmma. 128 x 128-byte tiles through shared memory, 16-byte
// loads and stores (cols and ld are multiples of 16): a thread gathers one 4-byte word of 16 source rows and turns it
// into 16 bytes of four output rows with 4 x 4 byte transposes in registers. Grid: (cols / 128, rows / 128, 2 models),
// z = plane * models + model.
struct BatchPlanes {
  const uint8_t* src[2];
  uint8_t* dst[2];
};
// Defined once, in sce_plan.cu; the row passes launch it through its host stub
__global__ void __launch_bounds__(256) transpose_batch_u8_kernel(BatchPlanes t, int models, int rows, int cols,
                                                                 long long src_model_pitch, int ld);
}  // namespace sce

// The batch-major copy T [models][cols][ld] of the 8-bit planes of P [models][rows][cols] (`src_pitch` elements between
// models), from which the native weight gradient reads them (dw_operand_maps; the code's, g's and dz's are written so
// by the encode, decode and dcode epilogues)
static int batch_major(Launcher& L, const Planes& P, const Planes& T, int models, int rows, int cols, long long src_pitch,
                       int ld) {
  const BatchPlanes t{{static_cast<const uint8_t*>(P.lo), P.x8}, {static_cast<uint8_t*>(T.lo), T.x8}};
  return L.launch(transpose_batch_u8_kernel, dim3((cols + 127) / 128, (rows + 127) / 128, 2 * models), 256, 0, t, models,
                  rows, cols, src_pitch, ld);
}
