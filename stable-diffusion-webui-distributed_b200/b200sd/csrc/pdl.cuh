// pdl.cuh — programmatic dependent launch (PDL) for the kernel chains of one UNet evaluation / VAE pass.
//
// A UNet evaluation is ~350 kernels on one stream (replayed from a CUDA graph).  Back to back, every boundary costs the
// launch latency of the next grid plus its prologue (mbarrier init, tensor-map prefetch) — a few
// microseconds each, i.e. 1-2 ms per evaluation whatever the batch, which is 2 % of an evaluation at the benchmark batch
// and a quarter of it at one image per GPU.  With PDL the next grid's CTAs become resident as soon as every CTA of the
// running grid has executed `griddepcontrol.launch_dependents` (placed at kernel entry) and SM resources free up; they run
// their prologue and then block in `griddepcontrol.wait` until the previous grid has COMPLETED and its memory is visible.
//
// Rules every kernel launched through launch_pdl() follows (they make the chain transitively safe):
//   * pdl_wait() is executed by every thread before the first global-memory access (read OR write) of the kernel;
//   * nothing before pdl_wait() touches global memory (shared memory, barriers, descriptor prefetch only).
// Kernels launched the ordinary way are unaffected (griddepcontrol.* are no-ops for them), and B200SD_PDL=0 turns the
// launch attribute off at run time.
//
// With every SM busy there is no tail to hide a prologue in, and early-resident dependents can cost more than the launch
// gap they save.  Hence the rule in launch_pdl(): the attribute is set only on grids that do not fill the machine (fewer
// CTAs than SMs) — the latency-bound regime of small batches, where boundaries are a visible share of the time.
// B200SD_PDL=2 forces it on every launch.
#pragma once
#include <cuda_runtime.h>
#include <stdlib.h>

namespace b200sd {

__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

constexpr int kNumSms = 132;  // H100 SXM: sizes the grids of the grid-stride and persistent kernels
constexpr unsigned kPdlMaxCtas = kNumSms;  // grids below one CTA per SM

inline int pdl_mode() {  // 0 off, 1 small grids only (default), 2 every launch
  static const int mode = [] {
    const char* e = getenv("B200SD_PDL");
    return e == nullptr ? 1 : (e[0] == '0' ? 0 : (e[0] == '2' ? 2 : 1));
  }();
  return mode;
}

template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream,
                              Args&&... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  const int mode = pdl_mode();
  cfg.numAttrs = (mode == 2 || (mode == 1 && grid.x * grid.y * grid.z < kPdlMaxCtas)) ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

}  // namespace b200sd
