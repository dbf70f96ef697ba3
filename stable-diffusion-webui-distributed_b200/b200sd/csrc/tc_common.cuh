// tc_common.cuh — sm_90a building blocks shared by the tensor-core kernels:
// mbarrier, TMA (cp.async.bulk.tensor), wgmma fences and shared-memory descriptors.
// Inline PTX only; no CUTLASS dependency.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include "../../../include/b200sd.h"

namespace b200sd {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ float fast_exp2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// ----------------------------------------------------------------------------------------------
// mbarrier
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// Every wait carries a suspend-time hint (B200SD_WAIT_HINT_NS): the waiting thread sleeps in hardware and is woken by
// barrier traffic instead of re-issuing the poll back to back, so waiting warps leave their issue slots to the warps
// doing the math.
#ifndef B200SD_WAIT_HINT_NS
#define B200SD_WAIT_HINT_NS 20000
#endif
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t"
      ".reg .pred P;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2, %3;\n\t"
      "selp.b32 %0, 1, 0, P;\n\t"
      "}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity), "r"(static_cast<uint32_t>(B200SD_WAIT_HINT_NS))
      : "memory");
  return ok != 0;
}
// Bounded wait: a protocol bug traps (CUDA error on the host) instead of hanging the GPU.  No printf here: a call in
// the kernel would make ptxas serialise the wgmma pipeline and spill the accumulators around it.
#ifndef B200SD_SPIN_LIMIT
#define B200SD_SPIN_LIMIT (1u << 22)
#endif
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (++spins > B200SD_SPIN_LIMIT) __trap();
  }
}
// Unbounded wait, for code after a setmaxnreg.inc whose budget is above the launch's register count: ptxas holds a
// branch that contains a trap to the launch's count (128 registers at 512 threads) and spills the rest.  A warp-
// specialised kernel uses it where the barrier is completed by TMA loads its producer issues after bounded waits of its
// own, so a stuck ring still traps there.
__device__ __forceinline__ void mbar_wait_unbounded(uint64_t* bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}

// ----------------------------------------------------------------------------------------------
// TMA loads (tile mode). Coordinates innermost first. OOB elements are zero-filled.
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2,
                                            int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], "
      "[%2];" ::"r"(smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}

// generic-proxy smem writes -> visible to the async proxy (tensor core / TMA reads)
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ----------------------------------------------------------------------------------------------
// wgmma (sm_90a warpgroup MMA): the four warps of a warpgroup issue together; operands are read from shared memory
// through descriptors (or A from registers), the fp32 accumulator lives in the warpgroup's registers.
// ----------------------------------------------------------------------------------------------
// registers / shared memory written before this point are visible to the wgmma instructions issued after it
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
// all but the newest N committed wgmma groups of this warpgroup have completed
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// per-thread register budget of the executing warpgroup, changed at run time (warp-specialised kernels hand the producer's
// registers to the math warpgroups); every warp of the warpgroup executes it
template <int N>
__device__ __forceinline__ void setmaxnreg_inc() {
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N) : "memory");
}
template <int N>
__device__ __forceinline__ void setmaxnreg_dec() {
  asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N) : "memory");
}
// Register split of the 384-thread warp-specialised kernels (two math warpgroups + one TMA producer warpgroup): the
// producer keeps 40 registers per thread and the math warpgroups take 232 (2 x 128 x 232 + 128 x 40 <= 64 K).
__device__ __forceinline__ void producer_warpgroup_regs() { setmaxnreg_dec<40>(); }
__device__ __forceinline__ void consumer_warpgroup_regs() { setmaxnreg_inc<232>(); }
// Keeps the compiler from moving reads / writes of an accumulator across a wgmma fence, commit or wait.
template <int N>
__device__ __forceinline__ void reg_fence(float (&d)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// Shared-memory matrix descriptor (wgmma), SWIZZLE_128B:
//  [0,14) start>>4  [16,30) LBO>>4  [32,46) SBO>>4  [62,64) layout (1 = SWIZZLE_128B)
// K-major tile (rows x 64 halfs, 128 B per row, TMA SWIZZLE_128B): SBO = 1024 B (8-row group), LBO unused (1).
// Advancing K by 16 elements inside the 128-byte row adds 32 B to the start address.
// MN-major tile (k-rows x 64 halfs of MN): SBO = 1024 B (8 k-rows), LBO = byte distance between 64-wide MN chunks.
__device__ __forceinline__ uint64_t make_gdesc_sw128(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFF) >> 4);
  d |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= static_cast<uint64_t>((sbo_bytes >> 4) & 0x3FFF) << 32;
  d |= static_cast<uint64_t>(1) << 62;
  return d;
}

// Byte offset of 16-byte chunk `chunk16` (0..7) of row `row` inside a K-major SWIZZLE_128B tile whose
// base is 1024-byte aligned and whose rows are 128 B (64 halfs).  Swizzle<3,4,3>: chunk ^= row % 8.
__host__ __device__ __forceinline__ uint32_t sw128_offset(uint32_t row, uint32_t chunk16) {
  return row * 128u + (((chunk16 ^ (row & 7u)) & 7u) << 4);
}

// Same for a SWIZZLE_64B tile with 64-byte rows (32 halfs), chunk16 in 0..3.  Swizzle<2,4,3>: chunk ^= (row/2) % 4.
__host__ __device__ __forceinline__ uint32_t sw64_offset(uint32_t row, uint32_t chunk16) {
  return row * 64u + (((chunk16 ^ ((row >> 1) & 3u)) & 3u) << 4);
}

// ----------------------------------------------------------------------------------------------
// TMA stores (shared -> global, bulk-group completion).  OOB parts of the box are clipped.
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* m, const void* src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(m)),
               "r"(smem_u32(src)), "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void tma_store_4d(const CUtensorMap* m, const void* src, int c0, int c1, int c2, int c3) {
  asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(m)),
               "r"(smem_u32(src)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
               : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// all but the newest N bulk groups of this thread have finished READING their shared-memory source
template <int N>
__device__ __forceinline__ void bulk_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
// ... have completed entirely (global writes performed)
template <int N>
__device__ __forceinline__ void bulk_wait() {
  asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory");
}

// ----------------------------------------------------------------------------------------------
// Host side: tensor-map encoding through the driver entry point (no link-time libcuda dependency)
// ----------------------------------------------------------------------------------------------

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
PFN_encodeTiled get_encode_tiled();

// fp16/bf16 tensor, rank 2..4, SWIZZLE_128B, inner box = 64 elements (128 B).
// dims/strides innermost first; strides[i] = byte stride of dim i+1. Returns B200SD_* code.
int make_tmap_sw128(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                    const uint32_t* box, const uint32_t* elem_strides);
// same, SWIZZLE_64B with a 32-element (64 B) inner box: the epilogue staging tiles of the GEMM kernel
int make_tmap_sw64(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                   const uint32_t* box, const uint32_t* elem_strides);

}  // namespace b200sd
