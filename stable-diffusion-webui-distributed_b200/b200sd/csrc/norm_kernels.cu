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

// The GroupNorm kernels and the staged LayerNorm spell their fp32 arithmetic with __fadd_rn / __fmul_rn / __fmaf_rn:
// nvcc never contracts those into a fused multiply-add, so every rounding step, and so every output bit, is the one the
// source states.

__device__ __forceinline__ float rcp_approx(float x) {
  float y;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

constexpr int kGnUnroll = 4;

// block = (C/8, PY): thread (v, py) owns channels [8v, 8v+8) for pixels p0+py, p0+py+PY, ... of its pixel range.
// Per-thread partials go to smem [PY][2C] (no atomics), are summed over PY, folded into groups, and one global
// atomicAdd per (group, stat) and block lands in stats[n][g][2].
// A block has at most 768 threads: wider rows need more than the 48 KB of shared memory b200sd_groupnorm_stats allows.
// Two such blocks per SM cap the kernel at 40 registers, so three 480-thread blocks share an SM at the UNet's widths, and
// ptxas issues the kGnUnroll loads of a round back to back (at 44 registers it did not, and the kernel ran 14 % slower
// over the SD1.5 UNet's shapes at batch 128 on an H100 80GB HBM3 at 400 W).
template <bool kBf16>
__global__ void __launch_bounds__(768, 2)
groupnorm_stats_kernel(const uint8_t* __restrict__ X, long long pitch, int HW, int C, int G, int pix_per_cta,
                       float* __restrict__ stats) {
  extern __shared__ float sh[];  // [PY][2C] partials, then [2C] channel totals reuse row 0
  pdl_trigger();
  pdl_wait();  // X is the previous kernel's output; the shared stats / ticket buffer is reused from GroupNorm to GroupNorm
  // The grid walks the tensor from its END.  The producer wrote it front to back and the apply kernel reads it front to
  // back, so of a tensor larger than the L2 the statistics pass finds the producer's last ~L2-size bytes still cached,
  // and leaves the FIRST ones cached for the apply pass (front-to-back twice evicts everything before its reuse).  Which
  // CTA owns which slab does not depend on the order in which they are scheduled, so neither does any bit of the result.
  const int n = static_cast<int>(gridDim.y - 1 - blockIdx.y);
  const int bx = static_cast<int>(gridDim.x - 1 - blockIdx.x);
  const int v = threadIdx.x;
  const int py = threadIdx.y;
  const int PY = blockDim.y;
  const int p0 = bx * pix_per_cta;
  const int p1 = min(HW, p0 + pix_per_cta);
  float s[8], q[8];  // channels 8v .. 8v+7
#pragma unroll
  for (int i = 0; i < 8; ++i) { s[i] = 0.f; q[i] = 0.f; }
  const long long rowb = pitch * 2;
  int p = p0 + py;
  const uint8_t* base = X + (static_cast<long long>(n) * HW + p) * rowb + static_cast<long long>(v) * 16;
  const long long step = PY * rowb;
  for (; p + (kGnUnroll - 1) * PY < p1; p += kGnUnroll * PY, base += kGnUnroll * step) {
    uint4 u[kGnUnroll];
#pragma unroll
    for (int k = 0; k < kGnUnroll; ++k) u[k] = __ldg(reinterpret_cast<const uint4*>(base + k * step));
#pragma unroll
    for (int k = 0; k < kGnUnroll; ++k) {
      float f[8];
      unpack8<kBf16>(u[k], f);
#pragma unroll
      for (int i = 0; i < 8; ++i) { s[i] = __fadd_rn(s[i], f[i]); q[i] = __fmaf_rn(f[i], f[i], q[i]); }
    }
  }
  for (; p < p1; p += PY, base += step) {
    const uint4 u = __ldg(reinterpret_cast<const uint4*>(base));
    float f[8];
    unpack8<kBf16>(u, f);
#pragma unroll
    for (int i = 0; i < 8; ++i) { s[i] = __fadd_rn(s[i], f[i]); q[i] = __fmaf_rn(f[i], f[i], q[i]); }
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
  float* partials = stats + static_cast<long long>(gridDim.y) * G * 2 + gridDim.y + static_cast<long long>(n) * parts * 2 * G;
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
  auto emit = [&](const uint4& u, int p) {
    float f[8];
    unpack8<kBf16>(u, f);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      float t = __fmaf_rn(f[i], a[i], b[i]);
      if (silu)  // t / (1 + exp(-t))
        t = __fmul_rn(t, rcp_approx(__fadd_rn(fast_exp2(__fmul_rn(t, -1.4426950408889634f)), 1.0f)));
      f[i] = t;
    }
    *reinterpret_cast<uint4*>(yb + p * ry) = pack8<kBf16>(f);
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
// one CTA per SM whatever the ring depth).  The sums run in four accumulators per lane, combined in a fixed order.
constexpr int kLnWarps = 16;
constexpr int kLnThreads = 32 * kLnWarps;
constexpr int kLnIn = 3, kLnOut = 2;  // input / output stages per warp

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
                        int C, const float* __restrict__ gamma, const float* __restrict__ beta, float eps, int lpr) {
  extern __shared__ __align__(128) uint8_t ln_smem[];
  const int rpw = 32 / lpr;                // rows per warp and tile
  const uint32_t row_bytes = static_cast<uint32_t>(C) * 2u;
  const uint32_t tile_bytes = static_cast<uint32_t>(rpw) * row_bytes;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float* gb = reinterpret_cast<float*>(ln_smem);                                  // gamma[C], beta[C]
  uint64_t* bars = reinterpret_cast<uint64_t*>(gb + 2 * C);                       // [kLnWarps][8]
  uint8_t* stages = reinterpret_cast<uint8_t*>(bars + kLnWarps * 8);              // [kLnWarps][kLnIn + kLnOut][tile]
  uint8_t* in_st = stages + static_cast<size_t>(warp) * (kLnIn + kLnOut) * tile_bytes;
  uint8_t* out_st = in_st + static_cast<size_t>(kLnIn) * tile_bytes;
  uint64_t* full = bars + warp * 8;
  pdl_trigger();
  if (lane == 0) {
    for (int s = 0; s < kLnIn; ++s) mbar_init(&full[s], 1);
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
    for (int s = 0; s < kLnIn; ++s)
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
    float f[VPT][8];                   // my 8 * VPT elements
    float acc[4] = {0.f, 0.f, 0.f, 0.f};  // acc[j] sums elements j and j + 4 of every vector
#pragma unroll
    for (int it = 0; it < VPT; ++it) {
      const int vec = it * lpr + sub;
      if (live && vec < nvec) {
        unpack8<kBf16>(*reinterpret_cast<const uint4*>(xr + vec * 16), f[it]);
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[j] = __fadd_rn(acc[j], __fadd_rn(f[it][j], f[it][j + 4]));
      } else {
#pragma unroll
        for (int i = 0; i < 8; ++i) f[it][i] = 0.f;
      }
    }
    // the inputs are in registers: refill this stage with the tile kLnIn steps ahead
    __syncwarp();
    if (lane == 0 && tile + kLnIn * tile_step < num_tiles) load_tile(tile + kLnIn * tile_step, s);
    float sum = __fadd_rn(acc[0], acc[2]) + __fadd_rn(acc[1], acc[3]);
    for (int d = lpr >> 1; d > 0; d >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, d);
    const float mean = sum * inv_c;
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[j] = 0.f;
#pragma unroll
    for (int it = 0; it < VPT; ++it) {
      if (it * lpr + sub < nvec) {
#pragma unroll
        for (int i = 0; i < 8; ++i) f[it][i] = __fadd_rn(f[it][i], -mean);   // keep the centred values
#pragma unroll
        for (int i = 0; i < 8; ++i) acc[i & 3] = __fmaf_rn(f[it][i], f[it][i], acc[i & 3]);
      }
    }
    float var = __fadd_rn(acc[0], acc[2]) + __fadd_rn(acc[1], acc[3]);
    for (int d = lpr >> 1; d > 0; d >>= 1) var += __shfl_xor_sync(0xffffffffu, var, d);
    const float rstd = rsqrtf(var * inv_c + eps);
    // out_st[o] was the source of the store issued kLnOut tiles ago: lane 0 has waited for it to be read (below)
    uint8_t* yr = out_st + o * tile_bytes + static_cast<uint32_t>(wrow) * row_bytes;
#pragma unroll
    for (int it = 0; it < VPT; ++it) {
      const int vec = it * lpr + sub;
      if (live && vec < nvec) {
        const float4 g0 = *reinterpret_cast<const float4*>(gb + vec * 8);
        const float4 g1 = *reinterpret_cast<const float4*>(gb + vec * 8 + 4);
        const float4 b0 = *reinterpret_cast<const float4*>(gb + C + vec * 8);
        const float4 b1 = *reinterpret_cast<const float4*>(gb + C + vec * 8 + 4);
        const float gg[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
        const float bb[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
        float o8[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) o8[i] = __fmaf_rn(__fmul_rn(f[it][i], rstd), gg[i], bb[i]);
        *reinterpret_cast<uint4*>(yr + vec * 16) = pack8<kBf16>(o8);
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
      bulk_wait_read<kLnOut - 1>();  // the stage the next tile writes has been read by its store
    }
    __syncwarp();
    if (++s == kLnIn) {
      s = 0;
      par ^= 1u;
    }
    if (++o == kLnOut) o = 0;
  }
  if (lane == 0) bulk_wait<0>();
}

// KB of one image a statistics CTA owns: the per-CTA epilogue (shared-memory reduction, group fold, partial store,
// fence, ticket) is amortised over this much streaming.  Measured at the bench batch (sum over the UNet's shapes,
// stats + apply): 48 KB 1.33 ms, 96 KB 1.24, 192 KB 1.20, 384 KB 1.20; 96 keeps a single image (batch 1 x CFG) spread
// over enough CTAs.
constexpr int kGnStatsKb = 96;

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

template <bool kBf16, int V>
static void launch_ln_staged_v(int lpr, int blocks, size_t sh, cudaStream_t st, const uint8_t* X, long long ldx, uint8_t* Y,
                               long long ldy, int rows, int C, const float* gamma, const float* beta, float eps) {
  static bool ready[64] = {};  // per-device opt-in to large dynamic shared memory; first call is outside graph capture
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev >= 0 && dev < 64 && !ready[dev]) {
    cudaFuncSetAttribute(layernorm_staged_kernel<kBf16, V>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    ready[dev] = true;
  }
  launch_pdl(layernorm_staged_kernel<kBf16, V>, dim3(blocks), dim3(kLnThreads), sh, st, X, ldx, Y, ldy, rows, C, gamma, beta,
             eps, lpr);
}

template <bool kBf16>
static void launch_ln_staged(int vpt, int lpr, int blocks, size_t sh, cudaStream_t st, const uint8_t* X, long long ldx,
                             uint8_t* Y, long long ldy, int rows, int C, const float* gamma, const float* beta, float eps) {
  switch (vpt) {
    case 1: launch_ln_staged_v<kBf16, 1>(lpr, blocks, sh, st, X, ldx, Y, ldy, rows, C, gamma, beta, eps); break;
    case 2: launch_ln_staged_v<kBf16, 2>(lpr, blocks, sh, st, X, ldx, Y, ldy, rows, C, gamma, beta, eps); break;
    case 3: launch_ln_staged_v<kBf16, 3>(lpr, blocks, sh, st, X, ldx, Y, ldy, rows, C, gamma, beta, eps); break;
    case 4: launch_ln_staged_v<kBf16, 4>(lpr, blocks, sh, st, X, ldx, Y, ldy, rows, C, gamma, beta, eps); break;
    case 5: launch_ln_staged_v<kBf16, 5>(lpr, blocks, sh, st, X, ldx, Y, ldy, rows, C, gamma, beta, eps); break;
    default: launch_ln_staged_v<kBf16, 8>(lpr, blocks, sh, st, X, ldx, Y, ldy, rows, C, gamma, beta, eps); break;
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
  if (gn_geometry(NB, HW, C, block, grid, ppc, kGnStatsKb) != B200SD_OK) return -1;
  // [NB][G][2] results | NB arrival tickets | [NB][CTAs per image][2G] partial sums
  return static_cast<long long>(NB) * G * 2 + NB + static_cast<long long>(NB) * grid.x * 2 * G;
}

extern "C" int b200sd_groupnorm_stats(const void* X, long long pitch, int NB, int HW, int C, int G, float* stats,
                                      int dtype, void* stream) {
  if (NB <= 0 || HW <= 0) return B200SD_OK;
  if (G <= 0 || C % G != 0 || pitch % 8 != 0 || (reinterpret_cast<uintptr_t>(X) & 15)) return B200SD_ERR_INVALID;
  dim3 block, grid;
  int ppc;
  int rc = gn_geometry(NB, HW, C, block, grid, ppc, kGnStatsKb);
  if (rc != B200SD_OK) return rc;
  const size_t sh = static_cast<size_t>(block.y) * 2 * C * sizeof(float);
  if (sh > 48 * 1024) return B200SD_ERR_UNSUPPORTED;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (dtype == B200SD_BF16)
    launch_pdl(groupnorm_stats_kernel<true>, grid, block, sh, st, static_cast<const uint8_t*>(X), pitch, HW, C, G, ppc, stats);
  else
    launch_pdl(groupnorm_stats_kernel<false>, grid, block, sh, st, static_cast<const uint8_t*>(X), pitch, HW, C, G, ppc, stats);
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
                                float* stats, const float* gamma, const float* beta, float eps, int silu, int dtype,
                                void* stream) {
  if (NB <= 0 || HW <= 0) return B200SD_OK;
  // everything the apply kernel checks, before the statistics kernel is launched: a failed call launches nothing
  if (G <= 0 || C % G != 0 || pitch_x % 8 != 0 || pitch_y % 8 != 0 ||
      ((reinterpret_cast<uintptr_t>(X) | reinterpret_cast<uintptr_t>(Y)) & 15))
    return B200SD_ERR_INVALID;
  int rc = b200sd_groupnorm_stats(X, pitch_x, NB, HW, C, G, stats, dtype, stream);
  if (rc != B200SD_OK) return rc;
  return b200sd_groupnorm_apply(X, pitch_x, Y, pitch_y, NB, HW, C, G, stats, gamma, beta, eps, silu, dtype, stream);
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
  const size_t tile_bytes = static_cast<size_t>(32 / lpr) * C * 2;   // one warp's row group
  const size_t sh_staged = 2 * static_cast<size_t>(C) * sizeof(float) + kLnWarps * 8 * sizeof(uint64_t) +
                           static_cast<size_t>(kLnWarps) * (kLnIn + kLnOut) * tile_bytes;
  // the staged rings fit in shared memory up to C = 1376; wider rows take the register version
  if (sh_staged <= 227 * 1024 && (ldx * 2) % 16 == 0 && (ldy * 2) % 16 == 0) {
    // persistent CTAs of 16 autonomous warps
    blocks = (rows + (32 / lpr) * kLnWarps - 1) / ((32 / lpr) * kLnWarps);
    const int per_sm = sh_staged + 1024 <= 113 * 1024 ? 2 : 1;
    if (blocks > kNumSms * per_sm) blocks = kNumSms * per_sm;
    if (dtype == B200SD_BF16)
      launch_ln_staged<true>(vpt, lpr, blocks, sh_staged, st, static_cast<const uint8_t*>(X), ldx,
                             static_cast<uint8_t*>(Y), ldy, rows, C, gamma, beta, eps);
    else
      launch_ln_staged<false>(vpt, lpr, blocks, sh_staged, st, static_cast<const uint8_t*>(X), ldx,
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
