// sce_ptx.cuh — thin inline-PTX wrappers for the sm_90a features the engine uses:
// mbarrier, thread block clusters, TMA (cp.async.bulk.tensor, multicast included), wgmma (warpgroup MMA from shared
// memory, accumulators in registers) and the shared-memory matrix descriptors wgmma consumes.
//
// Nothing here is specific to sparse autoencoders; sce_gemm.cuh builds the split-operand
// batched GEMM on top of it.
#pragma once
#include <cstdint>
#include <cuda.h>
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_fp8.h>

namespace sce {

// ----------------------------------------------------------------------------------------------
// small utilities
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// named barrier over `count` threads (id 0 is __syncthreads)
__device__ __forceinline__ void named_sync(uint32_t id, uint32_t count) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory");
}
// arrives on named barrier `id` without waiting: the threads that named_sync on it (count in all) go on once the
// arrivals are in, and see this thread's memory accesses from before the arrival
__device__ __forceinline__ void named_arrive(uint32_t id, uint32_t count) {
  asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(count) : "memory");
}

// setmaxnreg: sets the per-thread register count of the executing warpgroup to N (a multiple of 8 in 24..256). Every
// thread of the warpgroup executes it. `dec` hands registers back to the CTA's pool; `inc` waits until the pool has
// them. The kernel's launch register count (from __launch_bounds__) times its threads is the pool.
template <uint32_t N>
__device__ __forceinline__ void reg_dealloc() {
  asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N));
}
template <uint32_t N>
__device__ __forceinline__ void reg_alloc() {
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N));
}

// ----------------------------------------------------------------------------------------------
// mbarrier
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t"
      "}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}

// ----------------------------------------------------------------------------------------------
// thread block clusters
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ uint32_t cluster_nctarank() {
  uint32_t n;
  asm("mov.u32 %0, %%cluster_nctarank;" : "=r"(n));
  return n;
}
// Every thread of every CTA of the cluster arrives, then waits for all of them; release / acquire order the shared
// memory and mbarrier operations before it against those after it, across the cluster. Also a barrier of the CTA.
__device__ __forceinline__ void cluster_sync() {
  asm volatile("barrier.cluster.arrive.release;\n\tbarrier.cluster.wait.acquire;" ::: "memory");
}
// Arrives on the mbarrier at the same shared-memory offset as `bar` in CTA `cta` of the cluster.
__device__ __forceinline__ void mbar_arrive_cluster(uint64_t* bar, uint32_t cta) {
  uint32_t remote;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(remote) : "r"(smem_u32(bar)), "r"(cta));
  asm volatile("mbarrier.arrive.shared::cluster.b64 _, [%0];" ::"r"(remote) : "memory");
}

// ----------------------------------------------------------------------------------------------
// TMA: 3-D tiled tensor map load, global -> shared, completion on an mbarrier
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* smem_dst, const CUtensorMap* m, uint64_t* bar,
                                            int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes "
      "[%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}

// The same load multicast to the CTAs of the cluster in `cta_mask`: the box lands at the same shared-memory offset in
// each of them and completes its bytes on the mbarrier at the same offset in each.
__device__ __forceinline__ void tma_load_3d_multicast(void* smem_dst, const CUtensorMap* m, uint64_t* bar,
                                                      int c0, int c1, int c2, uint16_t cta_mask) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster "
      "[%0], [%1, {%3, %4, %5}], [%2], %6;"
      ::"r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "h"(cta_mask)
      : "memory");
}

// TMA store: shared -> global through a tiled tensor map (bulk async-group completion). Elements of the
// box that fall outside the tensor are clipped, so ragged tile edges need no predication.
__device__ __forceinline__ void tma_store_3d(const CUtensorMap* m, const void* smem_src, int c0, int c1, int c2) {
  asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%2, %3, %4}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(m)),
               "r"(smem_u32(smem_src)), "r"(c0), "r"(c1), "r"(c2)
               : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// all committed bulk stores of this thread but the N most recent have finished READING shared memory (it may be
// rewritten)
template <int N = 0>
__device__ __forceinline__ void tma_store_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}

// A 4-byte global store made only where `ok`, as one predicated instruction. Where an epilogue writes words under
// conditions that differ per word (store_col32_u8), a C++ `if` around each store costs branches and registers: the encode
// kernel spilled at its 128-register launch bound with them, and does not with this.
__device__ __forceinline__ void st_global_u32_if(void* p, uint32_t v, bool ok) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %2, 0;\n\t@p st.global.b32 [%0], %1;\n\t}" ::"l"(p), "r"(v),
               "r"((uint32_t)ok)
               : "memory");
}

// ----------------------------------------------------------------------------------------------
// wgmma shared-memory matrix descriptor (sm_90). Fields (PTX ISA "Matrix Descriptor Format"):
// [0,14) start address >> 4, [16,30) leading byte offset >> 4, [32,46) stride byte offset >> 4,
// [62,64) swizzle mode (1 = 128B, 2 = 64B, 3 = 32B). Tiles are 1024-byte aligned, so the base offset is 0.
//
//  * K-major operand (reduction index contiguous): rows of 128 B (128B swizzle, 64 16-bit elements) or 64 B
//    (64B swizzle, 32 elements); 8-row groups are SBO = 1024 / 512 B apart; LBO unused. A K=16 slice is 32 B
//    inside the row: advance the start address by 32 B per slice (the hardware applies the XOR swizzle).
//  * MN-major operand (row/column index contiguous, 128B swizzle): one 128-B row holds 64 consecutive M (or N)
//    elements of ONE k; 8 consecutive k make a 1024-B group, the next 8 k are SBO bytes further; the next 64 M/N
//    elements are LBO bytes further. A K=16 slice is two groups: 2048 B.
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ uint64_t make_wgmma_desc(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes,
                                                    uint32_t swizzle_mode) {
  uint64_t d = 0;
  d |= uint64_t((smem_addr & 0x3FFFFu) >> 4);
  d |= uint64_t((lbo_bytes >> 4) & 0x3FFFu) << 16;
  d |= uint64_t((sbo_bytes >> 4) & 0x3FFFu) << 32;
  d |= uint64_t(swizzle_mode) << 62;
  return d;
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}

// ----------------------------------------------------------------------------------------------
// wgmma m64n128k16, fp32 accumulators in registers: d += A(64 x 16) * B(16 x 128).
// F16: operands are fp16 (else bf16). TA / TB: operand is MN-major (transposed) in shared memory.
// Accumulator fragment of thread t of the warpgroup (warp w = t / 32, lane l): d[i] is row
// 16 w + l / 4 + 8 ((i / 2) % 2), column 8 (i / 4) + 2 (l % 4) + i % 2.
// ----------------------------------------------------------------------------------------------
#define SCE_WGMMA_N128(TYPE)                                                                                         \
  asm volatile(                                                                                                      \
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"                                                               \
      "wgmma.mma_async.sync.aligned.m64n128k16.f32." TYPE "." TYPE " "                                               \
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, "   \
      "%23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, "    \
      "%44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "        \
      "%64, %65, p, 1, 1, %66, %67;\n\t}\n"                                                                          \
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),              \
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),        \
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),      \
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),      \
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),      \
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),      \
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),      \
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])       \
      : "l"(adesc), "l"(bdesc), "n"(int(TA)), "n"(int(TB)))

template <bool F16, bool TA, bool TB>
__device__ __forceinline__ void wgmma_n128(float (&d)[64], uint64_t adesc, uint64_t bdesc) {
  if constexpr (F16) SCE_WGMMA_N128("f16");
  else SCE_WGMMA_N128("bf16");
}
#undef SCE_WGMMA_N128

// wgmma m64n128k32 on E5M2 operands, both K-major in shared memory (the fp8 forms have no transpose): d += A(64 x 32) *
// B(32 x 128). Same accumulator fragment as wgmma_n128.
__device__ __forceinline__ void wgmma_n128_e5m2(float (&d)[64], uint64_t adesc, uint64_t bdesc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k32.f32.e5m2.e5m2 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, "
      "%23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, "
      "%44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "%64, %65, p, 1, 1;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(adesc), "l"(bdesc));
}

// ----------------------------------------------------------------------------------------------
// fp16 + fp8 arithmetic ("f16f8"): x ~= h + l with h = fp16(x) (11 significant bits) and l = x - h, |l| <= 2^-11 |x|.
// The product a*b = ah*bh + (al*bh + ah*bl) + O(2^-22): the dominant term is formed on the fp16 planes, the two cross
// terms need only ~3 significant bits and are carried as 8-bit E5M2 planes: h8 = e5m2(x) and l8 = e5m2(l * 2^kLoShift)
// (1 byte / element in HBM: 4 bytes per operand element in all). The cross terms are accumulated FIRST (they carry the
// factor 2^kLoShift), the accumulator is then scaled by 2^-kLoShift (exact) and the hh products are added.
// Where both operands are K-major the cross terms run on E5M2 wgmma straight from the TMA stage. FP8 wgmma cannot read
// MN-major operands: there the GEMM widens the 8-bit tiles to fp16 in shared memory (exactly: an E5M2 byte is the high
// byte of the fp16 with the same value) and forms the cross terms with fp16 wgmma. The products are exact either way;
// only the accumulation of the cross-term sum differs.
// ----------------------------------------------------------------------------------------------
constexpr int kLoShift = 11;  // |l| * 2^11 <= |x|: the scaled residual has the range of x itself (fits E5M2 when x fits fp16)

// four e5m2 bytes -> four fp16 (two packed words): byte b becomes the fp16 with bits b << 8
__device__ __forceinline__ void widen_e5m2x4(uint32_t w, uint32_t& lo, uint32_t& hi) {
  lo = __byte_perm(w, 0u, 0x1404);
  hi = __byte_perm(w, 0u, 0x3424);
}

// ----------------------------------------------------------------------------------------------
// bf16 hi/lo split: x ~= hi + lo with hi = bf16(x), lo = bf16(x - hi); |x - hi - lo| <= 2^-17 |x|.
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void split_bf16(float x, __nv_bfloat16& hi, __nv_bfloat16& lo) {
  hi = __float2bfloat16_rn(x);
  lo = __float2bfloat16_rn(x - __bfloat162float(hi));
}
__device__ __forceinline__ uint32_t pack_bf16(__nv_bfloat16 a, __nv_bfloat16 b) {
  return uint32_t(__bfloat16_as_ushort(a)) | (uint32_t(__bfloat16_as_ushort(b)) << 16);
}

// f16f8 planes of a pair of values: packed fp16x2 (low half = a), packed e5m2x2 of the values and of the scaled
// residuals. Values beyond the fp16 range become inf in the fp16 plane (and NaN in the products): visible, not silent.
__device__ __forceinline__ void split2_f16f8(float a, float b, uint32_t& h16x2, uint32_t& h8x2, uint32_t& l8x2) {
  const __half2 h = __floats2half2_rn(a, b);
  h16x2 = *reinterpret_cast<const uint32_t*>(&h);
  const float2 hf = __half22float2(h);
  constexpr float kS = float(1 << kLoShift);
  l8x2 = __nv_cvt_float2_to_fp8x2(make_float2((a - hf.x) * kS, (b - hf.y) * kS), __NV_SATFINITE, __NV_E5M2);
  h8x2 = __nv_cvt_float2_to_fp8x2(make_float2(a, b), __NV_SATFINITE, __NV_E5M2);
}
// four consecutive values -> 8 B of the fp16 plane, 4 B of each 8-bit plane
__device__ __forceinline__ void split4_f16f8(const float (&v)[4], uint2& h16, uint32_t& h8, uint32_t& l8) {
  uint32_t a8, al, b8, bl;
  split2_f16f8(v[0], v[1], h16.x, a8, al);
  split2_f16f8(v[2], v[3], h16.y, b8, bl);
  h8 = a8 | (b8 << 16);
  l8 = al | (bl << 16);
}
__device__ __forceinline__ float e5m2_to_float(uint32_t byte) {  // e5m2 is the high byte of an fp16
  return __half2float(__ushort_as_half((unsigned short)(byte << 8)));
}

}  // namespace sce
