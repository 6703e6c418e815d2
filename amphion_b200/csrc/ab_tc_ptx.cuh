// mbarrier / bulk-copy (TMA 1-D) / wgmma PTX wrappers shared by the tensor-core kernels (sm_90a).
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/amphion_b200.h"

namespace ab {
namespace tcx {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ uint32_t mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(bar), "r"(parity)
      : "memory");
  return ok;
}
// Bounded wait: a protocol bug traps (-> cudaErrorLaunchFailure) instead of hanging the GPU.  No printf here: a
// call inside the MMA loop would make ptxas serialise the wgmma pipeline.
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (++spins > (1u << 24)) __trap();
  }
}
// generic-proxy shared-memory writes -> visible to the async proxy (wgmma operand reads, bulk copies)
__device__ __forceinline__ void fence_proxy_async() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst),
      "l"(src), "r"(bytes), "r"(bar)
      : "memory");
}
// Ampere-style async copies: src_bytes = 0 zero-fills the 16-byte destination (out-of-range rows).
__device__ __forceinline__ void cp_async16(uint32_t dst_smem, const void* src, uint32_t src_bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst_smem), "l"(src), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }

// warpgroup MMA ordering: fence before the first wgmma that touches the accumulator registers, commit after a
// batch, wait until at most N batches are in flight
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wg_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}

// Operand tiles are K-major without swizzle, in 8-row x 16-byte core matrices:
//   [c8][row][8 x 16 bit]  — unit (c8, row) at (c8 * rows + row) * 16 bytes.
// Rows are linear in memory, so a tap shift of s time steps is a +16*s byte move of the descriptor start, and one
// resident activation tile serves every tap.  Consecutive rows of one c8 are consecutive 16-byte units: the
// row-per-lane loaders and epilogues write 512 contiguous bytes per warp.
__device__ __forceinline__ uint32_t unit_offset(int rows, int c8, int row) {
  return ((uint32_t)c8 * (uint32_t)rows + (uint32_t)row) * 16u;
}
// sm_90 matrix descriptor for that layout: start >> 4 @0, leading byte offset (next core matrix along K =
// rows * 16 B) >> 4 @16, stride byte offset (next 8 rows = 128 B) >> 4 @32, no swizzle (0 @62).
__device__ __forceinline__ uint64_t make_desc(uint32_t saddr, uint32_t rows) {
  return (uint64_t)((saddr >> 4) & 0x3FFFu) | ((uint64_t)(rows & 0x3FFFu) << 16) | ((uint64_t)(128u >> 4) << 32);
}

// two fp32 -> packed 16-bit pair (first argument in the low half = lower address), round to nearest,
// saturating to the largest finite value: operands must never become inf (DESIGN.md §5).  One F2FP.
template <int BF16>
__device__ __forceinline__ uint32_t pack2t(float lo, float hi) {
  uint32_t r;
  if (BF16) asm("cvt.rn.satfinite.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
  else asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
  return r;
}
__device__ __forceinline__ uint32_t pack2(float lo, float hi, int bf16) {
  return bf16 ? pack2t<1>(lo, hi) : pack2t<0>(lo, hi);
}

// leaky_relu for 0 <= slope <= 1 (slope 1 = identity): max(v, slope*v)
__device__ __forceinline__ float lrelu(float v, float slope) { return fmaxf(v, v * slope); }

}  // namespace tcx
}  // namespace ab
