// norm_kernels.cu — HBM-bound normalisation kernels (NHWC, 16-byte vector loads, fp32 statistics).
//
//   groupnorm_stats  : per-(image, group) sum / sum-of-squares            1 read
//   groupnorm_apply  : y = (x - mean) * rstd * gamma + beta [, SiLU]       1 read + 1 write
//   layernorm        : one warp per token row, two passes in registers     1 read + 1 write
//
// All three keep several independent 16-byte loads in flight per thread (unrolled pixel / row loops) and run at
// high occupancy: they are latency-bound otherwise (ncu round 1: 17-20 % of HBM peak with one load in flight).
//
// Upstream: ldm GroupNorm32 (ResBlock.in_layers/out_layers, out), Normalize (SpatialTransformer.norm, VAE),
// BasicTransformerBlock.norm1/2/3 (SURVEY.md §8 a-ext x3, x9; not in /root/reference).
#include "pdl.cuh"
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <cstdlib>
#include <map>
#include <mutex>
#include <tuple>
#include "../../../include/b200sd.h"
#include "tc_common.cuh"

namespace b200sd {

template <bool kBf16>
__device__ __forceinline__ void unpack8(const uint4& u, float (&f)[8]) {
  const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    float2 t;
    if constexpr (kBf16) t = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&w[i]));
    else t = __half22float2(*reinterpret_cast<const __half2*>(&w[i]));
    f[2 * i] = t.x;
    f[2 * i + 1] = t.y;
  }
}
template <bool kBf16>
__device__ __forceinline__ uint4 pack8(const float (&f)[8]) {
  uint32_t w[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    if constexpr (kBf16) {
      __nv_bfloat162 v = __floats2bfloat162_rn(f[2 * i], f[2 * i + 1]);
      w[i] = *reinterpret_cast<uint32_t*>(&v);
    } else {
      __half2 v = __floats2half2_rn(f[2 * i], f[2 * i + 1]);
      w[i] = *reinterpret_cast<uint32_t*>(&v);
    }
  }
  return make_uint4(w[0], w[1], w[2], w[3]);
}

// Pairs of fp32 lanes.  sm_90 has no packed fp32 pipe, so each pair op is two scalar round-to-nearest ops — the
// same per-lane results the packed form gives.
struct F2 { float x, y; };
__device__ __forceinline__ F2 f2_make(float x, float y) { return F2{x, y}; }
__device__ __forceinline__ void f2_get(F2 a, float& x, float& y) {
  x = a.x;
  y = a.y;
}
__device__ __forceinline__ F2 f2_add(F2 a, F2 b) { return F2{__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)}; }
__device__ __forceinline__ F2 f2_mul(F2 a, F2 b) { return F2{__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)}; }
__device__ __forceinline__ F2 f2_fma(F2 a, F2 b, F2 c) { return F2{__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y)}; }
template <bool kBf16>
__device__ __forceinline__ void unpack4x2(const uint4& u, F2 (&f)[4]) {
  const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    float2 t;
    if constexpr (kBf16) t = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&w[i]));
    else t = __half22float2(*reinterpret_cast<const __half2*>(&w[i]));
    f[i] = f2_make(t.x, t.y);
  }
}
template <bool kBf16>
__device__ __forceinline__ uint32_t pack2(F2 a) {
  float x, y;
  f2_get(a, x, y);
  if constexpr (kBf16) {
    __nv_bfloat162 v = __floats2bfloat162_rn(x, y);
    return *reinterpret_cast<uint32_t*>(&v);
  } else {
    __half2 v = __floats2half2_rn(x, y);
    return *reinterpret_cast<uint32_t*>(&v);
  }
}

__device__ __forceinline__ float __frcp_rn_fast(float x) {
  float y;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

constexpr int kGnUnroll = 4;

// block = (C/8, PY): thread (v, py) owns channels [8v, 8v+8) for pixels p0+py, p0+py+PY, ... of its pixel range.
// Per-thread partials go to smem [PY][2C] (no atomics), are summed over PY, folded into groups, and one global
// atomicAdd per (group, stat) and block lands in stats[n][g][2].
template <bool kBf16>
__global__ void groupnorm_stats_kernel(const uint8_t* __restrict__ X, long long pitch, int HW, int C, int G,
                                       int pix_per_cta, float* __restrict__ stats, int reverse) {
  extern __shared__ float sh[];  // [PY][2C] partials, then [2C] channel totals reuse row 0
  pdl_trigger();
  pdl_wait();  // X is the previous kernel's output; the shared stats / ticket buffer is reused from GroupNorm to GroupNorm
  // `reverse`: the grid walks the tensor from its END.  The producer wrote it front to back and the apply kernel reads it
  // front to back, so of a tensor larger than the L2 the statistics pass finds the producer's last ~L2-size bytes still
  // cached, and leaves the FIRST ones cached for the apply pass (front-to-back twice evicts everything before its reuse).
  // Which CTA owns which slab is unchanged — only the order in which they are scheduled — so every bit of the result is.
  const int n = reverse ? static_cast<int>(gridDim.y - 1 - blockIdx.y) : static_cast<int>(blockIdx.y);
  const int bx = reverse ? static_cast<int>(gridDim.x - 1 - blockIdx.x) : static_cast<int>(blockIdx.x);
  const int v = threadIdx.x;
  const int py = threadIdx.y;
  const int PY = blockDim.y;
  const int p0 = bx * pix_per_cta;
  const int p1 = min(HW, p0 + pix_per_cta);
  F2 s2[4], q2[4];  // packed fp32 pairs: channel pairs (8v+2i, 8v+2i+1)
#pragma unroll
  for (int i = 0; i < 4; ++i) { s2[i] = f2_make(0.f, 0.f); q2[i] = s2[i]; }
  const uint8_t* base = X + (static_cast<long long>(n) * HW) * pitch * 2 + static_cast<long long>(v) * 16;
  const long long rowb = pitch * 2;
  int p = p0 + py;
  for (; p + (kGnUnroll - 1) * PY < p1; p += kGnUnroll * PY) {
    uint4 u[kGnUnroll];
#pragma unroll
    for (int k = 0; k < kGnUnroll; ++k) u[k] = __ldg(reinterpret_cast<const uint4*>(base + (p + k * PY) * rowb));
#pragma unroll
    for (int k = 0; k < kGnUnroll; ++k) {
      F2 f[4];
      unpack4x2<kBf16>(u[k], f);
#pragma unroll
      for (int i = 0; i < 4; ++i) { s2[i] = f2_add(s2[i], f[i]); q2[i] = f2_fma(f[i], f[i], q2[i]); }
    }
  }
  for (; p < p1; p += PY) {
    const uint4 u = __ldg(reinterpret_cast<const uint4*>(base + p * rowb));
    F2 f[4];
    unpack4x2<kBf16>(u, f);
#pragma unroll
    for (int i = 0; i < 4; ++i) { s2[i] = f2_add(s2[i], f[i]); q2[i] = f2_fma(f[i], f[i], q2[i]); }
  }
  float s[8], q[8];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    f2_get(s2[i], s[2 * i], s[2 * i + 1]);
    f2_get(q2[i], q[2 * i], q[2 * i + 1]);
  }
  float* mine = sh + static_cast<size_t>(py) * 2 * C;
  *reinterpret_cast<float4*>(mine + v * 8) = make_float4(s[0], s[1], s[2], s[3]);
  *reinterpret_cast<float4*>(mine + v * 8 + 4) = make_float4(s[4], s[5], s[6], s[7]);
  *reinterpret_cast<float4*>(mine + C + v * 8) = make_float4(q[0], q[1], q[2], q[3]);
  *reinterpret_cast<float4*>(mine + C + v * 8 + 4) = make_float4(q[4], q[5], q[6], q[7]);
  __syncthreads();
  const int tid = py * blockDim.x + v;
  const int nthreads = blockDim.x * PY;
  for (int i = tid; i < 2 * C; i += nthreads) {
    float a = 0.f;
    for (int k = 0; k < PY; ++k) a += sh[static_cast<size_t>(k) * 2 * C + i];
    sh[i] = a;  // row 0 is only read at index i by this same thread: no hazard
  }
  __syncthreads();
  // Deterministic cross-CTA reduction (no float atomics): every CTA publishes its 2G group partials; the CTA that
  // arrives last for image n (integer ticket) adds all of them in CTA-index order and writes stats[n].  The ticket
  // counter is left at zero again, so the scratch area needs zeroing only once, at allocation.
  const int cpg = C / G;
  const int parts = gridDim.x;
  float* out_stats = stats + static_cast<long long>(n) * G * 2;
  unsigned int* tickets = reinterpret_cast<unsigned int*>(stats + static_cast<long long>(gridDim.y) * G * 2);
  float* partials = stats + static_cast<long long>(gridDim.y) * G * 2 + gridDim.y + 1 +  // +1: the fused kernel's work counter
                    static_cast<long long>(n) * parts * 2 * G;
  for (int g = tid; g < 2 * G; g += nthreads) {
    const int grp = g >> 1, st = g & 1;
    float a = 0.f;
    for (int c = grp * cpg; c < (grp + 1) * cpg; ++c) a += sh[st * C + c];
    if (parts == 1) out_stats[g] = a;
    else __stcg(&partials[static_cast<long long>(bx) * 2 * G + g], a);
  }
  if (parts == 1) return;
  __shared__ unsigned int s_last;
  __threadfence();
  __syncthreads();
  if (tid == 0) s_last = (atomicAdd(&tickets[n], 1u) == static_cast<unsigned int>(parts - 1)) ? 1u : 0u;
  __syncthreads();
  if (s_last == 0u) return;
  __threadfence();
  // slices of the CTA-index range are summed by different threads, then combined in slice order: still a fixed order
  const int items = 2 * G;
  const int slices = max(1, min(nthreads / items, 8));
  float* red = sh;  // [slices][items], the channel totals are dead by now
  for (int idx = tid; idx < slices * items; idx += nthreads) {
    const int item = idx % items, sl = idx / items;
    const int per = (parts + slices - 1) / slices;
    const int lo = sl * per, hi = min(parts, lo + per);
    float a = 0.f;
    for (int k = lo; k < hi; ++k) a += __ldcg(&partials[static_cast<long long>(k) * items + item]);
    red[sl * items + item] = a;
  }
  __syncthreads();
  for (int g = tid; g < items; g += nthreads) {
    float a = 0.f;
    for (int sl = 0; sl < slices; ++sl) a += red[sl * items + g];
    out_stats[g] = a;
  }
  if (tid == 0) tickets[n] = 0u;
}

template <bool kBf16>
__global__ void groupnorm_apply_kernel(const uint8_t* __restrict__ X, long long pitch_x, uint8_t* __restrict__ Y,
                                       long long pitch_y, int HW, int C, int G, int pix_per_cta,
                                       const float* __restrict__ stats, const float* __restrict__ gamma,
                                       const float* __restrict__ beta, float eps, int silu) {
  pdl_trigger();
  pdl_wait();  // stats come from groupnorm_stats_kernel, X from the kernel before it
  const int n = blockIdx.y;
  const int v = threadIdx.x;
  const int PY = blockDim.y;
  const int p0 = blockIdx.x * pix_per_cta;
  const int p1 = min(HW, p0 + pix_per_cta);
  const int cpg = C / G;
  const float inv_cnt = 1.0f / (static_cast<float>(cpg) * static_cast<float>(HW));
  float a[8], b[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int c = v * 8 + i;
    const int g = c / cpg;
    const float sum = stats[(static_cast<long long>(n) * G + g) * 2];
    const float sq = stats[(static_cast<long long>(n) * G + g) * 2 + 1];
    const float mean = sum * inv_cnt;
    const float var = fmaxf(sq * inv_cnt - mean * mean, 0.f);
    const float rstd = rsqrtf(var + eps);
    a[i] = rstd * gamma[c];
    b[i] = beta[c] - mean * a[i];
  }
  const uint8_t* xb = X + (static_cast<long long>(n) * HW) * pitch_x * 2 + static_cast<long long>(v) * 16;
  uint8_t* yb = Y + (static_cast<long long>(n) * HW) * pitch_y * 2 + static_cast<long long>(v) * 16;
  const long long rx = pitch_x * 2, ry = pitch_y * 2;
  F2 a2[4], b2[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    a2[i] = f2_make(a[2 * i], a[2 * i + 1]);
    b2[i] = f2_make(b[2 * i], b[2 * i + 1]);
  }
  const F2 nlog2e = f2_make(-1.4426950408889634f, -1.4426950408889634f), one2 = f2_make(1.0f, 1.0f);
  auto emit = [&](const uint4& u, int p) {
    F2 f[4];
    unpack4x2<kBf16>(u, f);
    uint32_t w[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      F2 t = f2_fma(f[i], a2[i], b2[i]);
      if (silu) {  // t / (1 + exp(-t)): the two MUFU operations per element stay scalar, the arithmetic around them is packed
        float ex, ey;
        f2_get(f2_mul(t, nlog2e), ex, ey);
        float dx, dy;
        f2_get(f2_add(f2_make(fast_exp2(ex), fast_exp2(ey)), one2), dx, dy);
        t = f2_mul(t, f2_make(__frcp_rn_fast(dx), __frcp_rn_fast(dy)));
      }
      w[i] = pack2<kBf16>(t);
    }
    *reinterpret_cast<uint4*>(yb + p * ry) = make_uint4(w[0], w[1], w[2], w[3]);
  };
  int p = p0 + threadIdx.y;
  for (; p + (kGnUnroll - 1) * PY < p1; p += kGnUnroll * PY) {
    uint4 u[kGnUnroll];
#pragma unroll
    for (int k = 0; k < kGnUnroll; ++k) u[k] = __ldg(reinterpret_cast<const uint4*>(xb + (p + k * PY) * rx));
#pragma unroll
    for (int k = 0; k < kGnUnroll; ++k) emit(u[k], p + k * PY);
  }
  for (; p < p1; p += PY) emit(__ldg(reinterpret_cast<const uint4*>(xb + p * rx)), p);
}

// ---- one-pass GroupNorm ------------------------------------------------------------------------------------------
// stats + apply read the tensor twice (6 bytes per element with the write).  Here a CTA keeps its slab of one image
// (~48 KB: `ppc` pixels x C channels) in shared memory while the image's statistics are agreed on across CTAs, then
// normalises from shared memory: 1 read + 1 write (4 bytes per element).
//
// Cross-CTA protocol per image n (one 32-bit word, tickets[n], zero at rest):
//   arrive  : a CTA publishes its 2G group partials, fences, adds 1.  The CTA that brings the word to `parts` adds all
//             partials in slab order (the same sliced, fixed-order sum as groupnorm_stats_kernel), writes stats[n], fences,
//             adds 1 more (parts + 1 = "statistics ready");
//   wait    : the other CTAs spin (ld.acquire) until the word is >= parts + 1, then read stats[n];
//   depart  : every CTA adds 1 after it has read them; the one that sees 2 * parts resets the word to 0.
// A waiting CTA needs its siblings to RUN: slabs are handed out through an atomic work counter (not blockIdx), so the
// slabs started so far always form a prefix of the (image-major) order and every image whose first slab is running has
// all its slabs running or startable as long as `parts` CTAs fit on the device at once — the launcher checks that and
// falls back to the two-kernel path otherwise (huge VAE tensors).  The spin is bounded: a protocol failure traps instead
// of hanging the device.  tests/test_gn_protocol_cpu.py model-checks exactly this protocol under random interleavings.
__device__ __forceinline__ unsigned int ld_acquire_u32(const unsigned int* p) {
  unsigned int v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

#ifndef B200SD_GN_FUSED_DEFAULT
#define B200SD_GN_FUSED_DEFAULT 0
#endif
constexpr int kGnFusedThreads = 256;
constexpr int kGnMaxGroups = 64;

template <bool kBf16>
__global__ void __launch_bounds__(kGnFusedThreads, 3)
groupnorm_fused_kernel(const uint8_t* __restrict__ X, long long pitch_x, uint8_t* __restrict__ Y, long long pitch_y,
                       int NB, int HW, int C, int G, int ppc, int parts, float* __restrict__ stats,
                       const float* __restrict__ gamma, const float* __restrict__ beta, float eps, int silu) {
  extern __shared__ __align__(16) uint8_t gn_smem[];
  __shared__ float g_mean[kGnMaxGroups], g_rstd[kGnMaxGroups];
  __shared__ unsigned int s_item, s_last;
  pdl_trigger();
  pdl_wait();  // X is the previous kernel's output; the counters are left at zero by the previous GroupNorm
  const int v = threadIdx.x;
  const int py = threadIdx.y;
  const int vx = blockDim.x;
  const int PY = blockDim.y;
  const int tid = py * vx + v;
  const int nthreads = vx * PY;
  unsigned int* tickets = reinterpret_cast<unsigned int*>(stats + static_cast<long long>(NB) * G * 2);
  unsigned int* work = tickets + NB;
  if (tid == 0) {
    const unsigned int it = atomicAdd(work, 1u);
    if (it == gridDim.x - 1) atomicExch(work, 0u);  // the last slab handed out: nobody else touches the counter
    s_item = it;
  }
  __syncthreads();
  const int item = static_cast<int>(s_item);
  const int n = item / parts;
  const int part = item - n * parts;
  const int p0 = part * ppc;
  const int p1 = min(HW, p0 + ppc);
  uint4* slab = reinterpret_cast<uint4*>(gn_smem);                                            // [ppc][vx]
  float* sh = reinterpret_cast<float*>(gn_smem + static_cast<size_t>(ppc) * vx * 16);        // [PY][2C]

  // ---- pass over global memory: accumulate and keep
  F2 s2[4], q2[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) { s2[i] = f2_make(0.f, 0.f); q2[i] = s2[i]; }
  const uint8_t* xb = X + (static_cast<long long>(n) * HW) * pitch_x * 2 + static_cast<long long>(v) * 16;
  const long long rx = pitch_x * 2;
  int p = p0 + py;
  for (; p + (kGnUnroll - 1) * PY < p1; p += kGnUnroll * PY) {
    uint4 u[kGnUnroll];
#pragma unroll
    for (int k = 0; k < kGnUnroll; ++k) u[k] = __ldg(reinterpret_cast<const uint4*>(xb + (p + k * PY) * rx));
#pragma unroll
    for (int k = 0; k < kGnUnroll; ++k) {
      F2 f[4];
      unpack4x2<kBf16>(u[k], f);
#pragma unroll
      for (int i = 0; i < 4; ++i) { s2[i] = f2_add(s2[i], f[i]); q2[i] = f2_fma(f[i], f[i], q2[i]); }
      slab[static_cast<size_t>(p + k * PY - p0) * vx + v] = u[k];
    }
  }
  for (; p < p1; p += PY) {
    const uint4 u = __ldg(reinterpret_cast<const uint4*>(xb + p * rx));
    F2 f[4];
    unpack4x2<kBf16>(u, f);
#pragma unroll
    for (int i = 0; i < 4; ++i) { s2[i] = f2_add(s2[i], f[i]); q2[i] = f2_fma(f[i], f[i], q2[i]); }
    slab[static_cast<size_t>(p - p0) * vx + v] = u;
  }
  {
    float s[8], q[8];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      f2_get(s2[i], s[2 * i], s[2 * i + 1]);
      f2_get(q2[i], q[2 * i], q[2 * i + 1]);
    }
    float* mine = sh + static_cast<size_t>(py) * 2 * C;
    *reinterpret_cast<float4*>(mine + v * 8) = make_float4(s[0], s[1], s[2], s[3]);
    *reinterpret_cast<float4*>(mine + v * 8 + 4) = make_float4(s[4], s[5], s[6], s[7]);
    *reinterpret_cast<float4*>(mine + C + v * 8) = make_float4(q[0], q[1], q[2], q[3]);
    *reinterpret_cast<float4*>(mine + C + v * 8 + 4) = make_float4(q[4], q[5], q[6], q[7]);
  }
  __syncthreads();
  for (int i = tid; i < 2 * C; i += nthreads) {
    float a = 0.f;
    for (int k = 0; k < PY; ++k) a += sh[static_cast<size_t>(k) * 2 * C + i];
    sh[i] = a;  // row 0, index i: written by the only thread that reads it
  }
  __syncthreads();

  // ---- agree on the image's statistics
  const int cpg = C / G;
  const int items = 2 * G;
  float* out_stats = stats + static_cast<long long>(n) * items;
  float* partials = stats + static_cast<long long>(NB) * items + NB + 1 + static_cast<long long>(n) * parts * items;
  float* fin = sh + max(PY * 2 * C, 8 * items);  // [items] final sums, behind the scratch (the launcher sizes both)
  for (int g = tid; g < items; g += nthreads) {
    const int grp = g >> 1, st = g & 1;
    float a = 0.f;
    for (int c = grp * cpg; c < (grp + 1) * cpg; ++c) a += sh[st * C + c];
    if (parts == 1) { fin[g] = a; out_stats[g] = a; }
    else __stcg(&partials[static_cast<long long>(part) * items + g], a);
  }
  if (parts > 1) {
    __threadfence();
    __syncthreads();
    if (tid == 0) s_last = (atomicAdd(&tickets[n], 1u) == static_cast<unsigned int>(parts - 1)) ? 1u : 0u;
    __syncthreads();
    if (s_last != 0u) {
      __threadfence();
      const int slices = max(1, min(nthreads / items, 8));
      float* red = sh;  // [slices][items] <= 2C floats: the channel totals are dead by now
      for (int idx = tid; idx < slices * items; idx += nthreads) {
        const int it = idx % items, sl = idx / items;
        const int per = (parts + slices - 1) / slices;
        const int lo = sl * per, hi = min(parts, lo + per);
        float a = 0.f;
#pragma unroll 8
        for (int k = lo; k < hi; ++k) a += __ldcg(&partials[static_cast<long long>(k) * items + it]);
        red[sl * items + it] = a;
      }
      __syncthreads();
      for (int g = tid; g < items; g += nthreads) {
        float a = 0.f;
        for (int sl = 0; sl < slices; ++sl) a += red[sl * items + g];
        fin[g] = a;
        __stcg(&out_stats[g], a);
      }
      __threadfence();
      __syncthreads();
      if (tid == 0) atomicAdd(&tickets[n], 1u);  // parts + 1: statistics ready
    } else {
      if (tid == 0) {
        const unsigned int ready = static_cast<unsigned int>(parts) + 1u;
        unsigned int spins = 0;
        while (ld_acquire_u32(&tickets[n]) < ready) {
          __nanosleep(64);
          if (++spins > (1u << 24)) __trap();  // seconds: a sibling slab never ran — fail loudly, never hang
        }
      }
      __syncthreads();
      for (int g = tid; g < items; g += nthreads) fin[g] = __ldcg(&out_stats[g]);
    }
    __syncthreads();
    if (tid == 0) {
      if (atomicAdd(&tickets[n], 1u) == 2u * static_cast<unsigned int>(parts)) atomicExch(&tickets[n], 0u);
    }
  } else {
    __syncthreads();
  }
  const float inv_cnt = 1.0f / (static_cast<float>(cpg) * static_cast<float>(HW));
  for (int g = tid; g < G; g += nthreads) {
    const float mean = fin[2 * g] * inv_cnt;
    const float var = fmaxf(fin[2 * g + 1] * inv_cnt - mean * mean, 0.f);
    g_mean[g] = mean;
    g_rstd[g] = rsqrtf(var + eps);
  }
  __syncthreads();

  // ---- normalise from shared memory
  F2 a2[4], b2[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    float a[2], b[2];
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const int c = v * 8 + 2 * i + j;
      const int g = c / cpg;
      a[j] = g_rstd[g] * gamma[c];
      b[j] = beta[c] - g_mean[g] * a[j];
    }
    a2[i] = f2_make(a[0], a[1]);
    b2[i] = f2_make(b[0], b[1]);
  }
  uint8_t* yb = Y + (static_cast<long long>(n) * HW) * pitch_y * 2 + static_cast<long long>(v) * 16;
  const long long ry = pitch_y * 2;
  const F2 nlog2e = f2_make(-1.4426950408889634f, -1.4426950408889634f), one2 = f2_make(1.0f, 1.0f);
  for (p = p0 + py; p < p1; p += PY) {
    const uint4 u = slab[static_cast<size_t>(p - p0) * vx + v];
    F2 f[4];
    unpack4x2<kBf16>(u, f);
    uint32_t w[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      F2 t = f2_fma(f[i], a2[i], b2[i]);
      if (silu) {
        float ex, ey;
        f2_get(f2_mul(t, nlog2e), ex, ey);
        float dx, dy;
        f2_get(f2_add(f2_make(fast_exp2(ex), fast_exp2(ey)), one2), dx, dy);
        t = f2_mul(t, f2_make(__frcp_rn_fast(dx), __frcp_rn_fast(dy)));
      }
      w[i] = pack2<kBf16>(t);
    }
    *reinterpret_cast<uint4*>(yb + p * ry) = make_uint4(w[0], w[1], w[2], w[3]);
  }
}

// LPR lanes (a power of two, 4..32) share one row and 32/LPR rows share a warp, so every lane carries data whatever C is
// (C = 320 is 40 vectors: 8 lanes x 5, four rows per warp — one row per warp would leave 3/8 of the load slots empty);
// VPT 16-byte vectors per lane, all in flight before the first reduction; gamma/beta staged in smem once per CTA;
// persistent CTAs stride over rows so the staging is amortised and many rows are in flight per SM.
template <bool kBf16, int VPT>
__global__ void __launch_bounds__(256)
layernorm_kernel(const uint8_t* __restrict__ X, long long ldx, uint8_t* __restrict__ Y, long long ldy, int rows, int C,
                 const float* __restrict__ gamma, const float* __restrict__ beta, float eps, int lpr) {
  extern __shared__ float gb[];  // gamma[C], beta[C]
  pdl_trigger();
  for (int i = threadIdx.x; i < C; i += blockDim.x) {  // weights: immutable after model load, safe ahead of pdl_wait
    gb[i] = gamma[i];
    gb[C + i] = beta[i];
  }
  __syncthreads();
  pdl_wait();
  const int lane = threadIdx.x & 31;
  const int sub = lane & (lpr - 1);   // my position among the lanes of my row
  const int rpw = 32 / lpr;           // rows per warp
  const int wrow = lane / lpr;        // which of the warp's rows is mine
  const int warps_per_cta = blockDim.x >> 5;
  const int nvec = C / 8;
  const float inv_c = 1.0f / static_cast<float>(C);
  const int row_step = gridDim.x * warps_per_cta * rpw;
  for (int row0 = (blockIdx.x * warps_per_cta + (threadIdx.x >> 5)) * rpw; row0 < rows; row0 += row_step) {
    const int row = row0 + wrow;
    const bool live = row < rows;     // whole-warp shuffles below: dead rows just carry zeros
    const uint8_t* xr = X + static_cast<long long>(live ? row : 0) * ldx * 2;
    uint8_t* yr = Y + static_cast<long long>(live ? row : 0) * ldy * 2;
    float f[VPT][8];
    float sum = 0.f;
#pragma unroll
    for (int it = 0; it < VPT; ++it) {
      const int vec = it * lpr + sub;
      if (live && vec < nvec) {
        const uint4 u = __ldg(reinterpret_cast<const uint4*>(xr + static_cast<long long>(vec) * 16));
        unpack8<kBf16>(u, f[it]);
#pragma unroll
        for (int i = 0; i < 8; ++i) sum += f[it][i];
      } else {
#pragma unroll
        for (int i = 0; i < 8; ++i) f[it][i] = 0.f;
      }
    }
    for (int o = lpr >> 1; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    const float mean = sum * inv_c;
    float var = 0.f;
#pragma unroll
    for (int it = 0; it < VPT; ++it) {
      if (it * lpr + sub < nvec) {
#pragma unroll
        for (int i = 0; i < 8; ++i) { const float d = f[it][i] - mean; var = fmaf(d, d, var); }
      }
    }
    for (int o = lpr >> 1; o > 0; o >>= 1) var += __shfl_xor_sync(0xffffffffu, var, o);
    const float rstd = rsqrtf(var * inv_c + eps);
#pragma unroll
    for (int it = 0; it < VPT; ++it) {
      const int vec = it * lpr + sub;
      if (live && vec < nvec) {
        float o8[8];
        const float4 g0 = *reinterpret_cast<const float4*>(gb + vec * 8);
        const float4 g1 = *reinterpret_cast<const float4*>(gb + vec * 8 + 4);
        const float4 b0 = *reinterpret_cast<const float4*>(gb + C + vec * 8);
        const float4 b1 = *reinterpret_cast<const float4*>(gb + C + vec * 8 + 4);
        const float gg[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
        const float bb[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
        for (int i = 0; i < 8; ++i) o8[i] = fmaf((f[it][i] - mean) * rstd, gg[i], bb[i]);
        *reinterpret_cast<uint4*>(yr + static_cast<long long>(vec) * 16) = pack8<kBf16>(o8);
      }
    }
  }
}

// ---- TMA-staged LayerNorm ------------------------------------------------------------------------------------
// The register version above keeps rows in flight with threads (79 registers -> 24 warps per SM, every warp idle for a
// DRAM round trip per row: ncu 46 % of the measured HBM bandwidth).  Here every warp is its own pipeline: lane 0 streams
// the warp's row groups (32 / lpr rows, 2.5 KB for the UNet's widths) through a private ring of shared-memory stages
// with 1-D bulk copies (cp.async.bulk: the TMA engine without a tensor map), the normalised rows leave through two
// private output stages by bulk stores, and nothing but __syncwarp and the warp's own mbarriers synchronises — a first
// version with one producer warp and CTA-wide barriers per 20 KB tile spent 2.3 us per tile in hand-offs (2.6 TB/s with
// one CTA per SM whatever the ring depth).  The arithmetic runs on pairs of
// values with two accumulators (F2 above; two scalar ops per pair on sm_90).
constexpr int kLnWarps = 16;
constexpr int kLnThreads = 32 * kLnWarps;
constexpr int kLnInDefault = 3, kLnOutDefault = 2;  // input / output stages per warp (B200SD_LN_STAGES="in,out")

__device__ __forceinline__ void bulk_load_1d(uint32_t dst_smem, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst_smem),
               "l"(src), "r"(bytes), "r"(bar)
               : "memory");
}
__device__ __forceinline__ void bulk_store_1d(void* dst, uint32_t src_smem, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst), "r"(src_smem), "r"(bytes)
               : "memory");
}

template <bool kBf16, int VPT>
__global__ void __launch_bounds__(kLnThreads)
layernorm_staged_kernel(const uint8_t* __restrict__ X, long long ldx, uint8_t* __restrict__ Y, long long ldy, int rows,
                        int C, const float* __restrict__ gamma, const float* __restrict__ beta, float eps, int lpr,
                        int n_in, int n_out) {
  extern __shared__ __align__(128) uint8_t ln_smem[];
  const int rpw = 32 / lpr;                // rows per warp and tile
  const uint32_t row_bytes = static_cast<uint32_t>(C) * 2u;
  const uint32_t tile_bytes = static_cast<uint32_t>(rpw) * row_bytes;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float* gb = reinterpret_cast<float*>(ln_smem);                                  // gamma[C], beta[C]
  uint64_t* bars = reinterpret_cast<uint64_t*>(gb + 2 * C);                       // [kLnWarps][8]
  uint8_t* stages = reinterpret_cast<uint8_t*>(bars + kLnWarps * 8);              // [kLnWarps][n_in + n_out][tile]
  uint8_t* in_st = stages + static_cast<size_t>(warp) * (n_in + n_out) * tile_bytes;
  uint8_t* out_st = in_st + static_cast<size_t>(n_in) * tile_bytes;
  uint64_t* full = bars + warp * 8;
  pdl_trigger();
  if (lane == 0) {
    for (int s = 0; s < n_in; ++s) mbar_init(&full[s], 1);
    fence_mbar_init();
  }
  for (int i = threadIdx.x; i < C; i += blockDim.x) {  // weights: immutable after model load, safe ahead of pdl_wait
    gb[i] = gamma[i];
    gb[C + i] = beta[i];
  }
  __syncthreads();
  pdl_wait();  // X is the previous kernel's output
  const int num_tiles = (rows + rpw - 1) / rpw;
  const int tile_step = gridDim.x * kLnWarps;
  const int tile0 = blockIdx.x * kLnWarps + warp;
  auto load_tile = [&](int tile, int s) {  // lane 0
    const int r0 = tile * rpw, nr = min(rpw, rows - r0);
    mbar_arrive_expect_tx(&full[s], static_cast<uint32_t>(nr) * row_bytes);
    const uint32_t dst = smem_u32(in_st + s * tile_bytes), bar = smem_u32(&full[s]);
    const uint8_t* src = X + static_cast<long long>(r0) * ldx * 2;
    if (ldx == C) {
      bulk_load_1d(dst, src, static_cast<uint32_t>(nr) * row_bytes, bar);
    } else {
      for (int r = 0; r < nr; ++r) bulk_load_1d(dst + r * row_bytes, src + static_cast<long long>(r) * ldx * 2, row_bytes, bar);
    }
  };
  if (lane == 0)
    for (int s = 0; s < n_in; ++s)
      if (tile0 + s * tile_step < num_tiles) load_tile(tile0 + s * tile_step, s);
  const int sub = lane & (lpr - 1);   // my position among the lanes of my row
  const int wrow = lane / lpr;        // which of the warp's rows is mine
  const int nvec = C / 8;
  const float inv_c = 1.0f / static_cast<float>(C);
  int s = 0, o = 0;
  uint32_t par = 0;
  for (int tile = tile0; tile < num_tiles; tile += tile_step) {
    const int r0 = tile * rpw, nr = min(rpw, rows - r0);
    const bool live = wrow < nr;      // whole-warp shuffles below: dead rows just carry zeros
    mbar_wait(&full[s], par);
    const uint8_t* xr = in_st + s * tile_bytes + static_cast<uint32_t>(wrow) * row_bytes;
    F2 f[VPT][4];                      // my 8 * VPT elements as fp32 pairs
    F2 acc0 = f2_make(0.f, 0.f), acc1 = acc0;
#pragma unroll
    for (int it = 0; it < VPT; ++it) {
      const int vec = it * lpr + sub;
      if (live && vec < nvec) {
        unpack4x2<kBf16>(*reinterpret_cast<const uint4*>(xr + vec * 16), f[it]);
        acc0 = f2_add(acc0, f2_add(f[it][0], f[it][2]));
        acc1 = f2_add(acc1, f2_add(f[it][1], f[it][3]));
      } else {
#pragma unroll
        for (int i = 0; i < 4; ++i) f[it][i] = f2_make(0.f, 0.f);
      }
    }
    // the inputs are in registers: refill this stage with the tile n_in steps ahead
    __syncwarp();
    if (lane == 0 && tile + n_in * tile_step < num_tiles) load_tile(tile + n_in * tile_step, s);
    float sa, sb;
    f2_get(f2_add(acc0, acc1), sa, sb);
    float sum = sa + sb;
    for (int d = lpr >> 1; d > 0; d >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, d);
    const float mean = sum * inv_c;
    const F2 nmean = f2_make(-mean, -mean);
    acc0 = f2_make(0.f, 0.f);
    acc1 = acc0;
#pragma unroll
    for (int it = 0; it < VPT; ++it) {
      if (it * lpr + sub < nvec) {
#pragma unroll
        for (int i = 0; i < 4; ++i) f[it][i] = f2_add(f[it][i], nmean);   // keep the centred values
        acc0 = f2_fma(f[it][0], f[it][0], acc0);
        acc1 = f2_fma(f[it][1], f[it][1], acc1);
        acc0 = f2_fma(f[it][2], f[it][2], acc0);
        acc1 = f2_fma(f[it][3], f[it][3], acc1);
      }
    }
    f2_get(f2_add(acc0, acc1), sa, sb);
    float var = sa + sb;
    for (int d = lpr >> 1; d > 0; d >>= 1) var += __shfl_xor_sync(0xffffffffu, var, d);
    const float rstd = rsqrtf(var * inv_c + eps);
    const F2 rstd2 = f2_make(rstd, rstd);
    // out_st[o] was the source of the store issued n_out tiles ago: lane 0 has waited for it to be read (below)
    uint8_t* yr = out_st + o * tile_bytes + static_cast<uint32_t>(wrow) * row_bytes;
#pragma unroll
    for (int it = 0; it < VPT; ++it) {
      const int vec = it * lpr + sub;
      if (live && vec < nvec) {
        const float4 g0 = *reinterpret_cast<const float4*>(gb + vec * 8);
        const float4 g1 = *reinterpret_cast<const float4*>(gb + vec * 8 + 4);
        const float4 b0 = *reinterpret_cast<const float4*>(gb + C + vec * 8);
        const float4 b1 = *reinterpret_cast<const float4*>(gb + C + vec * 8 + 4);
        const F2 gg[4] = {{g0.x, g0.y}, {g0.z, g0.w}, {g1.x, g1.y}, {g1.z, g1.w}};
        const F2 bb[4] = {{b0.x, b0.y}, {b0.z, b0.w}, {b1.x, b1.y}, {b1.z, b1.w}};
        uint32_t w[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) w[i] = pack2<kBf16>(f2_fma(f2_mul(f[it][i], rstd2), gg[i], bb[i]));
        *reinterpret_cast<uint4*>(yr + vec * 16) = make_uint4(w[0], w[1], w[2], w[3]);
      }
    }
    fence_proxy_async_smem();  // my generic-proxy writes -> visible to the bulk store
    __syncwarp();
    if (lane == 0) {
      const uint32_t src = smem_u32(out_st + o * tile_bytes);
      uint8_t* dst = Y + static_cast<long long>(r0) * ldy * 2;
      if (ldy == C) {
        bulk_store_1d(dst, src, static_cast<uint32_t>(nr) * row_bytes);
      } else {
        for (int r = 0; r < nr; ++r) bulk_store_1d(dst + static_cast<long long>(r) * ldy * 2, src + r * row_bytes, row_bytes);
      }
      bulk_commit();
      if (n_out == 2) bulk_wait_read<1>();  // the stage the next tile writes has been read by its store
      else bulk_wait_read<2>();
    }
    __syncwarp();
    if (++s == n_in) {
      s = 0;
      par ^= 1u;
    }
    if (++o == n_out) o = 0;
  }
  if (lane == 0) bulk_wait<0>();
}

// KB of one image a statistics CTA owns (B200SD_GN_STATS_KB overrides): the per-CTA epilogue (shared-memory reduction,
// group fold, partial store, fence, ticket) is amortised over this much streaming.  Measured at the bench batch (sum over
// the UNet's shapes, stats + apply): 48 KB 1.33 ms, 96 KB 1.24, 192 KB 1.20, 384 KB 1.20; 96 keeps a single image
// (batch 1 x CFG) spread over enough CTAs.
static int gn_stats_kb() {
  static int kb = 0;
  if (kb == 0) {
    const char* e = std::getenv("B200SD_GN_STATS_KB");
    kb = e ? std::atoi(e) : 96;
    if (kb < 16 || kb > 1024) kb = 96;
  }
  return kb;
}

static int g_gn_stats_reverse = -1;  // B200SD_GN_REVERSE (default 1): the statistics grid walks the tensor back to front
static int gn_stats_reverse() {
  if (g_gn_stats_reverse < 0) {
    const char* e = std::getenv("B200SD_GN_REVERSE");
    g_gn_stats_reverse = e ? (std::atoi(e) != 0 ? 1 : 0) : 1;
  }
  return g_gn_stats_reverse;
}

static int gn_geometry(int NB, int HW, int C, dim3& block, dim3& grid, int& pix_per_cta, int chunk_kb = 48) {
  if (C % 8 != 0 || C / 8 > 1024) return B200SD_ERR_INVALID;
  const int vx = C / 8;
  int py = 512 / vx;
  if (py < 1) py = 1;
  if (py > HW) py = HW;
  block = dim3(vx, py, 1);
  // A CTA owns ~48 KB of one image (a multiple of py*unroll pixels).  The split depends on the image's shape only,
  // NOT on how many images are in the batch: the partial sums of an image — and therefore every bit of its result —
  // are the same whether it is processed alone, in a batch of 32, or on another GPU of a sharded request.
  (void)NB;
  const int quantum = py * kGnUnroll;
  int ppc = (chunk_kb * 1024 / (2 * C) + quantum - 1) / quantum * quantum;
  if (ppc < quantum) ppc = quantum;
  pix_per_cta = ppc;
  grid = dim3((HW + ppc - 1) / ppc, NB, 1);
  return B200SD_OK;
}

// One-pass GroupNorm geometry: 256 threads as (C/8, PY); a slab of ~B200SD_GN_FUSED_KB (default 48) KB per CTA, rounded DOWN
// to whole unrolled rounds so that slab + scratch stay below 1/3 of an SM's shared memory (3 CTAs per SM).  Like
// gn_geometry it depends on the image's shape only — never on the batch — so an image's bits do not depend on how a
// request was sharded.
struct GnFused {
  dim3 block;
  int ppc, parts;
  size_t smem;
};
static int g_gn_fused_kb = 0;  // 0 = not read yet
static int gn_fused_kb() {
  if (g_gn_fused_kb == 0) {
    const char* e = std::getenv("B200SD_GN_FUSED_KB");
    int kb = e ? std::atoi(e) : 48;
    if (kb < 8 || kb > 160) kb = 48;
    g_gn_fused_kb = kb;
  }
  return g_gn_fused_kb;
}
static int gn_fused_mode() {  // B200SD_GN_FUSED: 0 never, 1 (default) where eligible
  static int mode = -1;
  if (mode < 0) {
    const char* e = std::getenv("B200SD_GN_FUSED");
    mode = e ? (std::atoi(e) != 0 ? 1 : 0) : B200SD_GN_FUSED_DEFAULT;
  }
  return mode;
}
static bool gn_fused_geometry(int HW, int C, int G, GnFused& f) {
  if (C % 8 != 0 || G <= 0 || G > kGnMaxGroups || C % G != 0) return false;
  const int vx = C / 8;
  if (vx > kGnFusedThreads) return false;
  int py = kGnFusedThreads / vx;
  if (py > HW) py = HW;
  const int quantum = py * kGnUnroll;
  int ppc = (gn_fused_kb() * 1024 / (2 * C)) / quantum * quantum;
  if (ppc < quantum) ppc = quantum;
  f.block = dim3(vx, py, 1);
  f.ppc = ppc;
  f.parts = (HW + ppc - 1) / ppc;
  const size_t scratch = static_cast<size_t>(py) * 2 * C > static_cast<size_t>(16 * G) ? static_cast<size_t>(py) * 2 * C : 16 * G;
  f.smem = static_cast<size_t>(ppc) * C * 2 + (scratch + 2 * G) * sizeof(float);
  return f.smem <= 72 * 1024;
}
// CTAs of the fused kernel that are resident at once on the current device (occupancy x SMs), cached per device and
// shared-memory size class; 0 = unknown (treated as "not eligible")
template <bool kBf16>
static int gn_fused_capacity(const GnFused& f) {
  static std::mutex mu;
  static std::map<std::tuple<int, size_t, unsigned>, int> cache;  // (device, smem, threads) -> resident CTAs
  static int sms[64] = {};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 0;
  const unsigned threads = f.block.x * f.block.y;
  std::lock_guard<std::mutex> lock(mu);
  auto key = std::make_tuple(dev, f.smem, threads);
  auto hit = cache.find(key);
  if (hit != cache.end()) return hit->second;  // in particular: no CUDA API calls while a stream is being captured
  if (sms[dev] == 0) {
    if (cudaFuncSetAttribute(groupnorm_fused_kernel<kBf16>, cudaFuncAttributeMaxDynamicSharedMemorySize, 72 * 1024) != cudaSuccess)
      return 0;
    int n = 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) return 0;
    sms[dev] = n;
  }
  int per_sm = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, groupnorm_fused_kernel<kBf16>, static_cast<int>(threads),
                                                    f.smem) != cudaSuccess)
    return 0;
  cache[key] = per_sm * sms[dev];
  return per_sm * sms[dev];
}
template <bool kBf16>
static int launch_gn_fused(const GnFused& f, cudaStream_t st, const uint8_t* X, long long pitch_x, uint8_t* Y, long long pitch_y,
                           int NB, int HW, int C, int G, float* stats, const float* gamma, const float* beta, float eps,
                           int silu) {
  launch_pdl(groupnorm_fused_kernel<kBf16>, dim3(static_cast<unsigned>(NB) * f.parts), f.block, f.smem, st, X, pitch_x, Y,
             pitch_y, NB, HW, C, G, f.ppc, f.parts, stats, gamma, beta, eps, silu);
  return cudaGetLastError() == cudaSuccess ? B200SD_OK : B200SD_ERR_CUDA;
}

template <bool kBf16, int V>
static void launch_ln_staged_v(int n_in, int n_out, int lpr, int blocks, size_t sh, cudaStream_t st, const uint8_t* X, long long ldx, uint8_t* Y,
                               long long ldy, int rows, int C, const float* gamma, const float* beta, float eps) {
  static bool ready[64] = {};  // per-device opt-in to large dynamic shared memory; first call is outside graph capture
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev >= 0 && dev < 64 && !ready[dev]) {
    cudaFuncSetAttribute(layernorm_staged_kernel<kBf16, V>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    ready[dev] = true;
  }
  launch_pdl(layernorm_staged_kernel<kBf16, V>, dim3(blocks), dim3(kLnThreads), sh, st, X, ldx, Y, ldy, rows, C, gamma, beta,
             eps, lpr, n_in, n_out);
}

template <bool kBf16>
static void launch_ln_staged(int n_in, int n_out, int vpt, int lpr, int blocks, size_t sh, cudaStream_t st, const uint8_t* X, long long ldx,
                             uint8_t* Y, long long ldy, int rows, int C, const float* gamma, const float* beta, float eps) {
  switch (vpt) {
    case 1: launch_ln_staged_v<kBf16, 1>(n_in, n_out, lpr, blocks, sh, st, X, ldx, Y, ldy, rows, C, gamma, beta, eps); break;
    case 2: launch_ln_staged_v<kBf16, 2>(n_in, n_out, lpr, blocks, sh, st, X, ldx, Y, ldy, rows, C, gamma, beta, eps); break;
    case 3: launch_ln_staged_v<kBf16, 3>(n_in, n_out, lpr, blocks, sh, st, X, ldx, Y, ldy, rows, C, gamma, beta, eps); break;
    case 4: launch_ln_staged_v<kBf16, 4>(n_in, n_out, lpr, blocks, sh, st, X, ldx, Y, ldy, rows, C, gamma, beta, eps); break;
    case 5: launch_ln_staged_v<kBf16, 5>(n_in, n_out, lpr, blocks, sh, st, X, ldx, Y, ldy, rows, C, gamma, beta, eps); break;
    default: launch_ln_staged_v<kBf16, 8>(n_in, n_out, lpr, blocks, sh, st, X, ldx, Y, ldy, rows, C, gamma, beta, eps); break;
  }
}

template <bool kBf16>
static void launch_ln(int vpt, int lpr, int blocks, size_t sh, cudaStream_t st, const uint8_t* X, long long ldx, uint8_t* Y,
                      long long ldy, int rows, int C, const float* gamma, const float* beta, float eps) {
  switch (vpt) {
    case 1: launch_pdl(layernorm_kernel<kBf16, 1>, dim3(blocks), dim3(256), sh, st, X, ldx, Y, ldy, rows, C, gamma, beta, eps, lpr); break;
    case 2: launch_pdl(layernorm_kernel<kBf16, 2>, dim3(blocks), dim3(256), sh, st, X, ldx, Y, ldy, rows, C, gamma, beta, eps, lpr); break;
    case 3: launch_pdl(layernorm_kernel<kBf16, 3>, dim3(blocks), dim3(256), sh, st, X, ldx, Y, ldy, rows, C, gamma, beta, eps, lpr); break;
    case 4: launch_pdl(layernorm_kernel<kBf16, 4>, dim3(blocks), dim3(256), sh, st, X, ldx, Y, ldy, rows, C, gamma, beta, eps, lpr); break;
    case 5: launch_pdl(layernorm_kernel<kBf16, 5>, dim3(blocks), dim3(256), sh, st, X, ldx, Y, ldy, rows, C, gamma, beta, eps, lpr); break;
    default: launch_pdl(layernorm_kernel<kBf16, 8>, dim3(blocks), dim3(256), sh, st, X, ldx, Y, ldy, rows, C, gamma, beta, eps, lpr); break;
  }
}

}  // namespace b200sd

using namespace b200sd;

extern "C" long long b200sd_groupnorm_stats_floats(int NB, int HW, int C, int G) {
  if (NB <= 0 || HW <= 0 || G <= 0) return 0;
  dim3 block, grid;
  int ppc;
  if (gn_geometry(NB, HW, C, block, grid, ppc, gn_stats_kb()) != B200SD_OK) return -1;
  // [NB][G][2] results | NB arrival tickets + 1 work counter | [NB][CTAs per image][2G] partial sums (the larger of the
  // two-kernel and the one-pass geometry)
  long long parts = grid.x;
  GnFused f;
  if (gn_fused_geometry(HW, C, G, f) && f.parts > parts) parts = f.parts;
  return static_cast<long long>(NB) * G * 2 + NB + 1 + static_cast<long long>(NB) * parts * 2 * G;
}

extern "C" int b200sd_groupnorm_stats(const void* X, long long pitch, int NB, int HW, int C, int G, float* stats,
                                      int dtype, void* stream) {
  if (NB <= 0 || HW <= 0) return B200SD_OK;
  if (G <= 0 || C % G != 0 || pitch % 8 != 0 || (reinterpret_cast<uintptr_t>(X) & 15)) return B200SD_ERR_INVALID;
  dim3 block, grid;
  int ppc;
  int rc = gn_geometry(NB, HW, C, block, grid, ppc, gn_stats_kb());
  if (rc != B200SD_OK) return rc;
  const size_t sh = static_cast<size_t>(block.y) * 2 * C * sizeof(float);
  if (sh > 48 * 1024) return B200SD_ERR_UNSUPPORTED;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int rev = gn_stats_reverse();
  if (dtype == B200SD_BF16)
    launch_pdl(groupnorm_stats_kernel<true>, grid, block, sh, st, static_cast<const uint8_t*>(X), pitch, HW, C, G, ppc, stats, rev);
  else
    launch_pdl(groupnorm_stats_kernel<false>, grid, block, sh, st, static_cast<const uint8_t*>(X), pitch, HW, C, G, ppc, stats, rev);
  return cudaGetLastError() == cudaSuccess ? B200SD_OK : B200SD_ERR_CUDA;
}

extern "C" int b200sd_groupnorm_apply(const void* X, long long pitch_x, void* Y, long long pitch_y, int NB, int HW,
                                      int C, int G, const float* stats, const float* gamma, const float* beta,
                                      float eps, int silu, int dtype, void* stream) {
  if (NB <= 0 || HW <= 0) return B200SD_OK;
  if (G <= 0 || C % G != 0 || pitch_x % 8 != 0 || pitch_y % 8 != 0 ||
      ((reinterpret_cast<uintptr_t>(X) | reinterpret_cast<uintptr_t>(Y)) & 15))
    return B200SD_ERR_INVALID;
  dim3 block, grid;
  int ppc;
  int rc = gn_geometry(NB, HW, C, block, grid, ppc);
  if (rc != B200SD_OK) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (dtype == B200SD_BF16)
    launch_pdl(groupnorm_apply_kernel<true>, grid, block, 0, st, static_cast<const uint8_t*>(X), pitch_x,
               static_cast<uint8_t*>(Y), pitch_y, HW, C, G, ppc, stats, gamma, beta, eps, silu);
  else
    launch_pdl(groupnorm_apply_kernel<false>, grid, block, 0, st, static_cast<const uint8_t*>(X), pitch_x,
               static_cast<uint8_t*>(Y), pitch_y, HW, C, G, ppc, stats, gamma, beta, eps, silu);
  return cudaGetLastError() == cudaSuccess ? B200SD_OK : B200SD_ERR_CUDA;
}

extern "C" int b200sd_groupnorm(const void* X, long long pitch_x, void* Y, long long pitch_y, int NB, int HW, int C, int G,
                                float* stats, const float* gamma, const float* beta, float eps, int silu, int mode,
                                int dtype, void* stream) {
  if (NB <= 0 || HW <= 0) return B200SD_OK;
  if (G <= 0 || C % G != 0 || pitch_x % 8 != 0 || pitch_y % 8 != 0 ||
      ((reinterpret_cast<uintptr_t>(X) | reinterpret_cast<uintptr_t>(Y)) & 15))
    return B200SD_ERR_INVALID;
  if (mode < 0 || mode > 2) return B200SD_ERR_INVALID;
  GnFused f;
  bool fused = mode == 2 || (mode == 0 && gn_fused_mode() == 1);
  if (fused) {
    fused = gn_fused_geometry(HW, C, G, f);
    if (fused) {
      // every slab of one image must be able to run at the same time (the kernel's header explains why)
      const int cap = dtype == B200SD_BF16 ? gn_fused_capacity<true>(f) : gn_fused_capacity<false>(f);
      fused = f.parts <= cap && static_cast<long long>(NB) * f.parts < (1ll << 31);
    }
    if (!fused && mode == 2) return B200SD_ERR_UNSUPPORTED;
  }
  if (fused) {
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    return dtype == B200SD_BF16
               ? launch_gn_fused<true>(f, st, static_cast<const uint8_t*>(X), pitch_x, static_cast<uint8_t*>(Y), pitch_y, NB, HW, C,
                                       G, stats, gamma, beta, eps, silu)
               : launch_gn_fused<false>(f, st, static_cast<const uint8_t*>(X), pitch_x, static_cast<uint8_t*>(Y), pitch_y, NB, HW,
                                        C, G, stats, gamma, beta, eps, silu);
  }
  int rc = b200sd_groupnorm_stats(X, pitch_x, NB, HW, C, G, stats, dtype, stream);
  if (rc != B200SD_OK) return rc;
  return b200sd_groupnorm_apply(X, pitch_x, Y, pitch_y, NB, HW, C, G, stats, gamma, beta, eps, silu, dtype, stream);
}

/* tools/norm_sweep.py: slab size of the one-pass kernel (0 = keep) and scheduling order of the statistics kernel
 * (-1 = keep) for the calls that follow; scratch sizes change with the slab size */
extern "C" int b200sd_debug_gn_config(int slab_kb, int reverse_stats) {
  if (slab_kb != 0 && (slab_kb < 8 || slab_kb > 160)) return B200SD_ERR_INVALID;
  if (slab_kb != 0) g_gn_fused_kb = slab_kb;
  if (reverse_stats >= 0) g_gn_stats_reverse = reverse_stats != 0 ? 1 : 0;
  return B200SD_OK;
}

/* 1 when b200sd_groupnorm(mode 0 / 2) would take the one-pass kernel for this shape on the current device */
extern "C" int b200sd_groupnorm_is_fused(int NB, int HW, int C, int G, int dtype) {
  GnFused f;
  if (NB <= 0 || !gn_fused_geometry(HW, C, G, f)) return 0;
  const int cap = dtype == B200SD_BF16 ? gn_fused_capacity<true>(f) : gn_fused_capacity<false>(f);
  return f.parts <= cap ? 1 : 0;
}

extern "C" int b200sd_layernorm(const void* X, long long ldx, void* Y, long long ldy, int rows, int C,
                                const float* gamma, const float* beta, float eps, int dtype, void* stream) {
  if (rows <= 0) return B200SD_OK;
  if (C % 8 != 0 || C > 2048 || ldx % 8 != 0 || ldy % 8 != 0 ||
      ((reinterpret_cast<uintptr_t>(X) | reinterpret_cast<uintptr_t>(Y)) & 15))
    return B200SD_ERR_INVALID;
  // lanes per row: the fewest (power of two >= 4) that keep the per-lane vector count at 5 or below
  const int nvec = C / 8;
  int lpr = 4;
  while (lpr < 32 && (nvec + lpr - 1) / lpr > 5) lpr <<= 1;
  int vpt = (nvec + lpr - 1) / lpr;
  if (vpt > 5) vpt = 8;
  const int rows_per_block = 8 * (32 / lpr);
  int blocks = (rows + rows_per_block - 1) / rows_per_block;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  static int staged = -1;  // B200SD_LN_STAGED=0: the register version
  if (staged < 0) {
    const char* e = std::getenv("B200SD_LN_STAGED");
    staged = e ? std::atoi(e) : 1;
  }
  static int n_in = kLnInDefault, n_out = kLnOutDefault, ctas_per_sm = 0;
  static bool env_read = false;
  if (!env_read) {
    if (const char* e = std::getenv("B200SD_LN_STAGES")) {
      n_in = std::atoi(e);
      const char* c = e;
      while (*c && *c != ',') ++c;
      n_out = *c ? std::atoi(c + 1) : 2;
      if (n_in < 2 || n_in > 8) n_in = kLnInDefault;
      if (n_out < 2 || n_out > 3) n_out = kLnOutDefault;
    }
    if (const char* e = std::getenv("B200SD_LN_CTAS")) ctas_per_sm = std::atoi(e);
    env_read = true;
  }
  const size_t tile_bytes = static_cast<size_t>(32 / lpr) * C * 2;   // one warp's row group
  const size_t sh_staged = 2 * static_cast<size_t>(C) * sizeof(float) + kLnWarps * 8 * sizeof(uint64_t) +
                           static_cast<size_t>(kLnWarps) * (n_in + n_out) * tile_bytes;
  if (staged && sh_staged <= 227 * 1024 && (ldx * 2) % 16 == 0 && (ldy * 2) % 16 == 0) {
    // persistent CTAs of 16 autonomous warps
    blocks = (rows + (32 / lpr) * kLnWarps - 1) / ((32 / lpr) * kLnWarps);
    int per_sm = sh_staged + 1024 <= 113 * 1024 ? 2 : 1;
    if (ctas_per_sm > 0) per_sm = ctas_per_sm;
    if (blocks > kNumSms * per_sm) blocks = kNumSms * per_sm;
    if (dtype == B200SD_BF16)
      launch_ln_staged<true>(n_in, n_out, vpt, lpr, blocks, sh_staged, st, static_cast<const uint8_t*>(X), ldx,
                             static_cast<uint8_t*>(Y), ldy, rows, C, gamma, beta, eps);
    else
      launch_ln_staged<false>(n_in, n_out, vpt, lpr, blocks, sh_staged, st, static_cast<const uint8_t*>(X), ldx,
                              static_cast<uint8_t*>(Y), ldy, rows, C, gamma, beta, eps);
    return cudaGetLastError() == cudaSuccess ? B200SD_OK : B200SD_ERR_CUDA;
  }
  if (blocks > kNumSms * 8) blocks = kNumSms * 8;
  const size_t sh = 2 * static_cast<size_t>(C) * sizeof(float);
  if (dtype == B200SD_BF16)
    launch_ln<true>(vpt, lpr, blocks, sh, st, static_cast<const uint8_t*>(X), ldx, static_cast<uint8_t*>(Y), ldy, rows, C,
                    gamma, beta, eps);
  else
    launch_ln<false>(vpt, lpr, blocks, sh, st, static_cast<const uint8_t*>(X), ldx, static_cast<uint8_t*>(Y), ldy, rows, C,
                     gamma, beta, eps);
  return cudaGetLastError() == cudaSuccess ? B200SD_OK : B200SD_ERR_CUDA;
}
