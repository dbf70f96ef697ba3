// gemm_conv_tc.cu — persistent warp-specialised wgmma GEMM / implicit-GEMM convolution for sm_90a.
//
//   D[M, N] = epilogue( A[M, K] * Wt[N, K]^T )          fp16 or bf16 operands, fp32 accumulation in registers
//
// mode GEMM : A is a row-major [M, K] matrix (row pitch lda), loaded by 2-D TMA tiles {64 x 128}.
//             Covers every Linear layer and every 1x1 convolution of the UNet / VAE (NHWC activations).
// mode CONV : A is never materialised.  The activation is an NHWC tensor seen through a 4-D tensor map
//             {C, W, H, N}; one M-tile is a box of bw x bh x bn output pixels (bw*bh*bn <= 128) and the
//             K loop runs over (tap, 64-channel block): tap (dy, dx) is the same box shifted by
//             (dx - pad, dy - pad) — TMA's out-of-bounds zero fill is the convolution padding, and
//             elementStrides = 2 gives the stride-2 Downsample.  Weights are packed [Cout][tap][Cin].
//
// Roles (384 threads): warps 0-7 are two consumer warpgroups, warpgroup 2 is the TMA producer, which releases registers
// to the consumers at run time (setmaxnreg 40 / 232).  ptxas still allocates against the 168-register launch budget of
// 12 warps, so BN = 192 / 224 / 256 (96-128 accumulator registers) spill 64-304 bytes per thread: those widths are kept
// for callers that pass an explicit block_n and are correct, but ops.pick_block_n never chooses them.  Warpgroup w owns rows
// [64w, 64w+64) of the 128 x BN tile: it issues m64nBNk16 wgmma on the shared-memory stages (A and B K-major,
// SWIZZLE_128B) and keeps the fp32 accumulator in registers.  The producer fills a ring of stages (A 16 KB + B BN x 128 B)
// that runs ahead into the next tile while the consumers are in their epilogue.  Epilogue, in 32-column chunks:
// registers -> (+bias, GEGLU, +residual, SiLU) -> fp16 -> a SWIZZLE_64B staging tile in shared memory -> one TMA store
// of the whole 128-row box.  The residual arrives the same way (TMA load into a staging tile, two chunks ahead), so all
// global traffic of the kernel is bulk and asynchronous; out-of-range rows (M tail, partial pixel boxes) are clipped /
// zero-filled by the tensor maps instead of predicated.
//
// Upstream ops this kernel stands in for: ldm ResBlock conv3x3 / skip 1x1, Up/Downsample conv, SpatialTransformer
// proj_in/out, CrossAttention to_q/k/v/out, FeedForward GEGLU + out, AutoencoderKL decoder convs
// (SURVEY.md §8 a-ext x1,x2,x5,x7,x8,x9,x11).
#include <math.h>
#include <stddef.h>
#include <stdlib.h>
#include "tc_common.cuh"
#include "wgmma.cuh"
#include "b200sd_internal.h"
#include "pdl.cuh"

namespace b200sd {

constexpr int kBlockM = 128;
constexpr int kBlockK = 64;   // 64 halfs = 128 B = one SWIZZLE_128B row
constexpr int kMmaK = 16;
constexpr int kConsumerThreads = 256;                 // two warpgroups of 64 rows each
constexpr int kGemmThreads = kConsumerThreads + 128;  // + the producer warpgroup (one thread issues the TMA loads)
constexpr int kMaxStages = 8;
constexpr int kChunkCols = 32;
constexpr uint32_t kStageTileBytes = kBlockM * kChunkCols * 2;  // 8 KB: 128 rows x 32 halfs, SWIZZLE_64B
constexpr uint32_t kATileBytes = kBlockM * kBlockK * 2;         // 16 KB

struct GemmKernelParams {
  int M, N, K;
  int block_n;
  int num_m_tiles, num_n_tiles, num_k_blocks, num_stages;
  uint32_t a_bytes, b_bytes, d_bytes;  // d_bytes: bytes one staging box moves (rows of the tile actually stored)
  int mode;                        // 0 = GEMM, 1 = CONV
  int H, W, NB;                    // CONV: output height / width / images
  int bw, bh, bn;                  // CONV: output-pixel box
  int tiles_x, tiles_y;            // CONV: boxes per row / column
  int taps, cblocks, stride, pad;  // CONV
  const float* bias;               // [groups][N] fp32 or nullptr
  int bias_group_rows;             // rows (output pixels) sharing one bias row; <= 0 -> single row
  int has_residual;
  int flags;                       // B200SD_EPI_*
};

struct __align__(8) GemmBarriers {
  uint64_t full[kMaxStages];   // stage landed (TMA transaction bytes)
  uint64_t empty[kMaxStages];  // stage consumed: one arrival per consumer warpgroup
  uint64_t res_full[2];        // residual staging tile landed
};

// gelu(x) = 0.5 x (1 + erf(x / sqrt 2)), erf by Abramowitz-Stegun 7.1.28: erf(z) = 1 - (1 + a1 z + ... + a6 z^6)^-16 for
// z >= 0, |error| < 3e-7 (gelu: 9e-7 absolute over [-12, 12], far below the fp16 output rounding): one MUFU op (the
// reciprocal; the 16th power is four squarings).  An overflow of the 16th power (z > ~15) gives rcp(inf) = 0, i.e.
// erf = 1, which is the right limit.
__device__ __forceinline__ float rcp_approx(float x) {
  float y;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float gelu_erf(float x) {
  const float z = __fmul_rn(fabsf(x), 0.70710678118654752440f);
  float q = __fmaf_rn(0.0000430638f, z, 0.0002765672f);
  q = __fmaf_rn(q, z, 0.0001520143f);
  q = __fmaf_rn(q, z, 0.0092705272f);
  q = __fmaf_rn(q, z, 0.0422820123f);
  q = __fmaf_rn(q, z, 0.0705230784f);
  q = __fmaf_rn(q, z, 1.0f);
  q = __fmul_rn(q, q);
  q = __fmul_rn(q, q);
  q = __fmul_rn(q, q);
  q = __fmul_rn(q, q);
  const float h = __fmaf_rn(0.5f, copysignf(1.0f - rcp_approx(q), x), 0.5f);
  return __fmul_rn(x, h);
}

template <bool kBf16>
__device__ __forceinline__ uint32_t pack2(float a, float b) {
  if constexpr (kBf16) {
    __nv_bfloat162 v = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&v);
  } else {
    __half2 v = __floats2half2_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&v);
  }
}
template <bool kBf16>
__device__ __forceinline__ float2 unpack2(uint32_t u) {
  if constexpr (kBf16) {
    return __bfloat1622float2(*reinterpret_cast<__nv_bfloat162*>(&u));
  } else {
    return __half22float2(*reinterpret_cast<__half2*>(&u));
  }
}

__device__ __forceinline__ void consumer_bar_sync() {  // named barrier 1: the 256 consumer threads
  asm volatile("bar.sync 1, %0;" ::"n"(kConsumerThreads) : "memory");
}

struct TileCoord {
  int c1, c2, c3;  // coordinates of the tile's first output row in the D / residual tensor maps (after the column)
};

__device__ __forceinline__ TileCoord tile_coord(const GemmKernelParams& p, int m_tile) {
  TileCoord t;
  if (p.mode == 0) {
    t.c1 = m_tile * kBlockM; t.c2 = 0; t.c3 = 0;
  } else {
    t.c1 = (m_tile % p.tiles_x) * p.bw;
    t.c2 = ((m_tile / p.tiles_x) % p.tiles_y) * p.bh;
    t.c3 = (m_tile / (p.tiles_x * p.tiles_y)) * p.bn;
  }
  return t;
}

// global output row of tile row r (0 when r lies outside the problem: only used to pick a per-image bias row)
__device__ __forceinline__ long long tile_row(const GemmKernelParams& p, const TileCoord& tc, int m_tile, int r) {
  if (p.mode == 0) {
    const long long row = static_cast<long long>(m_tile) * kBlockM + r;
    return row < p.M ? row : 0;
  }
  const int x = tc.c1 + r % p.bw, y = tc.c2 + (r / p.bw) % p.bh, n = tc.c3 + r / (p.bw * p.bh);
  return (x < p.W && y < p.H && n < p.NB && r < p.bw * p.bh * p.bn) ? (static_cast<long long>(n) * p.H + y) * p.W + x : 0;
}

__device__ __forceinline__ void load_residual(const GemmKernelParams& p, const CUtensorMap* tmR, GemmBarriers* bars,
                                              uint8_t* stage_r, const TileCoord& tc, int n_tile, int out_bn, int c) {
  const int buf = c & 1;
  mbar_arrive_expect_tx(&bars->res_full[buf], p.d_bytes);
  const int col = n_tile * out_bn + c * kChunkCols;
  uint8_t* dst = stage_r + buf * kStageTileBytes;
  if (p.mode == 0) tma_load_2d(dst, tmR, &bars->res_full[buf], col, tc.c1);
  else tma_load_4d(dst, tmR, &bars->res_full[buf], col, tc.c1, tc.c2, tc.c3);
}

template <int BN, bool kBf16>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_conv_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                    const __grid_constant__ CUtensorMap tmD, const __grid_constant__ CUtensorMap tmR,
                    const GemmKernelParams p) {
  constexpr uint32_t kStageBytes = kATileBytes + BN * 128u;
  extern __shared__ uint8_t smem_raw[];
  // SWIZZLE_128B tiles need 1024-byte alignment.
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* stage_d = smem + static_cast<size_t>(p.num_stages) * kStageBytes;  // 2 output staging tiles
  uint8_t* stage_r = stage_d + 2 * kStageTileBytes;                            // 2 residual staging tiles (if any)
  GemmBarriers* bars = reinterpret_cast<GemmBarriers*>(stage_r + (p.has_residual ? 2 * kStageTileBytes : 0));

  pdl_trigger();  // the next kernel of the chain may start its prologue as SMs free up (pdl.cuh)
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int num_items = p.num_m_tiles * p.num_n_tiles;

  if (threadIdx.x == kConsumerThreads) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    tma_prefetch_desc(&tmD);
    if (p.has_residual) tma_prefetch_desc(&tmR);
    for (int s = 0; s < p.num_stages; ++s) {
      mbar_init(&bars->full[s], 1);
      mbar_init(&bars->empty[s], kConsumerThreads / 128);
    }
    mbar_init(&bars->res_full[0], 1);
    mbar_init(&bars->res_full[1], 1);
    fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();  // prologue done; from here on the kernel reads what its predecessors wrote

  if (warp >= kConsumerThreads / 32) {
    // ------------------------------- TMA producer (one thread) -------------------------------
    // The (tap, channel-block) position of the conv K loop is advanced by counters, not divisions.
    producer_warpgroup_regs();
    if (threadIdx.x == kConsumerThreads) {
      const int nkb = p.num_k_blocks, nstages = p.num_stages, cblocks = p.cblocks;
      const bool conv = p.mode == 1, taps9 = p.taps == 9;
      const uint32_t tx_bytes = p.a_bytes + p.b_bytes;
      int stage = 0;
      uint32_t phase = 0;
      for (int item = blockIdx.x; item < num_items; item += gridDim.x) {
        const int n_tile = item % p.num_n_tiles;
        const int m_tile = item / p.num_n_tiles;
        int cx = 0, cy = 0, cn = 0;
        if (conv) {
          const int tx = m_tile % p.tiles_x;
          const int ty = (m_tile / p.tiles_x) % p.tiles_y;
          cn = (m_tile / (p.tiles_x * p.tiles_y)) * p.bn;
          cx = tx * p.bw * p.stride - p.pad;
          cy = ty * p.bh * p.stride - p.pad;
        }
        const int b_row = n_tile * BN;
        const int a_row = m_tile * kBlockM;
        int cb = 0, dx = 0, dy = 0;  // conv: channel block within the tap, tap offsets
        for (int kb = 0; kb < nkb; ++kb) {
          mbar_wait(&bars->empty[stage], phase ^ 1u);
          uint8_t* sA = smem + static_cast<size_t>(stage) * kStageBytes;
          uint8_t* sB = sA + kATileBytes;
          uint64_t* full_bar = &bars->full[stage];
          mbar_arrive_expect_tx(full_bar, tx_bytes);
          if (!conv) tma_load_2d(sA, &tmA, full_bar, kb * kBlockK, a_row);
          else tma_load_4d(sA, &tmA, full_bar, cb * kBlockK, cx + dx, cy + dy, cn);
          tma_load_2d(sB, &tmB, full_bar, kb * kBlockK, b_row);
          if (++cb == cblocks) {  // next tap (1x1 convs have a single tap: dx, dy never move)
            cb = 0;
            if (taps9 && ++dx == 3) { dx = 0; ++dy; }
          }
          if (++stage == nstages) { stage = 0; phase ^= 1u; }
        }
      }
    }
    return;
  }

  // ------------------------------- consumer warpgroups -------------------------------
  consumer_warpgroup_regs();
  const int wg = warp >> 2;
  const int row0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);  // this thread's accumulator rows: row0, row0 + 8
  const int colq = (lane & 3) * 2;                            // and columns 8g + colq, 8g + colq + 1
  const bool signaller = (threadIdx.x & 127) == 0;            // releases stages for its warpgroup
  const bool leader = threadIdx.x == 0;                       // issues the epilogue's TMA stores / residual loads
  const bool geglu = (p.flags & B200SD_EPI_GEGLU) != 0;
  const int out_bn = geglu ? BN / 2 : BN;
  const int nchunks = out_bn / kChunkCols;
  const uint32_t smem0 = smem_u32(smem);
  float acc[BN / 2];
  int stage = 0;
  uint32_t phase = 0;
  uint32_t res_uses[2] = {0u, 0u};
  uint32_t d_slot = 0;

  for (int item = blockIdx.x; item < num_items; item += gridDim.x) {
    const int n_tile = item % p.num_n_tiles;
    const int m_tile = item / p.num_n_tiles;
    const TileCoord tc = tile_coord(p, m_tile);
    // residual chunks 0 and 1 are fetched while the main loop runs (both buffers are free: every read of the previous
    // tile's residual is behind the consumer barrier of its last chunk)
    if (p.has_residual && leader) {
      load_residual(p, &tmR, bars, stage_r, tc, n_tile, out_bn, 0);
      if (nchunks > 1) load_residual(p, &tmR, bars, stage_r, tc, n_tile, out_bn, 1);
    }

    // main loop: one wgmma group per k-block; a stage is released once the group after it has been waited for
    int prev_stage = 0;
    for (int kb = 0; kb < p.num_k_blocks; ++kb) {
      mbar_wait(&bars->full[stage], phase);
      const uint32_t a_addr = smem0 + static_cast<uint32_t>(stage) * kStageBytes + static_cast<uint32_t>(wg) * 8192u;
      const uint32_t b_addr = smem0 + static_cast<uint32_t>(stage) * kStageBytes + kATileBytes;
      reg_fence(acc);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < kBlockK / kMmaK; ++k)
        Wgmma<BN, kBf16>::ss(acc, make_gdesc_sw128(a_addr + 32u * k, 16, 1024), make_gdesc_sw128(b_addr + 32u * k, 16, 1024),
                             (kb | k) != 0 ? 1u : 0u);
      wgmma_commit();
      reg_fence(acc);
      wgmma_wait<1>();
      if (kb > 0 && signaller) mbar_arrive(&bars->empty[prev_stage]);
      prev_stage = stage;
      if (++stage == p.num_stages) { stage = 0; phase ^= 1u; }
    }
    wgmma_wait<0>();
    reg_fence(acc);
    if (signaller) mbar_arrive(&bars->empty[prev_stage]);

    // epilogue
    const float* bias_r[2] = {p.bias, p.bias};
    if (p.bias != nullptr && p.bias_group_rows > 0) {
#pragma unroll
      for (int h = 0; h < 2; ++h) bias_r[h] = p.bias + (tile_row(p, tc, m_tile, row0 + 8 * h) / p.bias_group_rows) * p.N;
    }
#pragma unroll
    for (int c = 0; c < BN / kChunkCols; ++c) {
      if (c < nchunks) {
        float f[2][4][2];  // [row half][8-column group][column]
#pragma unroll
        for (int g = 0; g < 4; ++g) {
          const int col = n_tile * BN + c * kChunkCols + g * 8 + colq;  // column in the [N] space of the GEMM
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            float2 b = make_float2(0.f, 0.f), bg = make_float2(0.f, 0.f);
            if (p.bias != nullptr) {
              b = __ldg(reinterpret_cast<const float2*>(bias_r[h] + col));
              if (geglu) bg = __ldg(reinterpret_cast<const float2*>(bias_r[h] + col + BN / 2));
            }
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int idx = 4 * (4 * c + g) + 2 * h + e;
              float v = acc[idx] + (e ? b.y : b.x);
              if (geglu) {
                constexpr int kGate = BN / 4;  // accumulator index distance of column + BN/2
                v *= gelu_erf(acc[(idx + kGate) % (BN / 2)] + (e ? bg.y : bg.x));
              }
              f[h][g][e] = v;
            }
          }
        }
        if (p.has_residual) {
          const int buf = c & 1;
          mbar_wait(&bars->res_full[buf], res_uses[buf] & 1u);
          res_uses[buf]++;
          const uint8_t* rt = stage_r + buf * kStageTileBytes;
#pragma unroll
          for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int g = 0; g < 4; ++g) {
              const float2 t = unpack2<kBf16>(*reinterpret_cast<const uint32_t*>(rt + sw64_offset(row0 + 8 * h, g) + colq * 2));
              f[h][g][0] += t.x;
              f[h][g][1] += t.y;
            }
        }
        if (p.flags & B200SD_EPI_SILU) {
#pragma unroll
          for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int g = 0; g < 4; ++g)
#pragma unroll
              for (int e = 0; e < 2; ++e) f[h][g][e] = __fdividef(f[h][g][e], 1.0f + __expf(-f[h][g][e]));
        }
        uint8_t* dt = stage_d + d_slot * kStageTileBytes;
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int g = 0; g < 4; ++g)
            *reinterpret_cast<uint32_t*>(dt + sw64_offset(row0 + 8 * h, g) + colq * 2) = pack2<kBf16>(f[h][g][0], f[h][g][1]);
        fence_proxy_async_smem();  // my staging writes (and residual reads) -> visible / ordered for the async proxy
        // the buffer the next chunk is staged into was last read by the previous store: it must be done reading
        if (leader) bulk_wait_read<0>();
        consumer_bar_sync();
        if (leader) {
          const int col = n_tile * out_bn + c * kChunkCols;
          if (p.mode == 0) tma_store_2d(&tmD, dt, col, tc.c1);
          else tma_store_4d(&tmD, dt, col, tc.c1, tc.c2, tc.c3);
          bulk_commit();
          if (p.has_residual && c + 2 < nchunks) load_residual(p, &tmR, bars, stage_r, tc, n_tile, out_bn, c + 2);
        }
        d_slot ^= 1u;
      }
    }
  }
  if (leader) bulk_wait<0>();  // the TMA stores must have completed before the CTA (and its smem) goes away
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
typedef void (*GemmKernel)(CUtensorMap, CUtensorMap, CUtensorMap, CUtensorMap, GemmKernelParams);

template <bool kBf16>
static GemmKernel kernel_for(int block_n) {
  switch (block_n) {
    case 32: return gemm_conv_tc_kernel<32, kBf16>;
    case 64: return gemm_conv_tc_kernel<64, kBf16>;
    case 96: return gemm_conv_tc_kernel<96, kBf16>;
    case 128: return gemm_conv_tc_kernel<128, kBf16>;
    case 160: return gemm_conv_tc_kernel<160, kBf16>;
    case 192: return gemm_conv_tc_kernel<192, kBf16>;
    case 224: return gemm_conv_tc_kernel<224, kBf16>;
    case 256: return gemm_conv_tc_kernel<256, kBf16>;
    default: return nullptr;
  }
}
static GemmKernel kernel_for(int block_n, int is_bf16) {
  return is_bf16 ? kernel_for<true>(block_n) : kernel_for<false>(block_n);
}

static int g_num_sms = 0;
static int g_max_smem = 0;
static bool g_dev_ready[64] = {};
// per-device one-time setup (the dynamic-smem opt-in is per context): safe to call from several host threads
// that each drive their own device, and must first happen OUTSIDE any stream capture (warm-up run).
static int device_props() {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return B200SD_ERR_CUDA;
  if (dev < 0 || dev >= 64) return B200SD_ERR_UNSUPPORTED;
  if (!g_dev_ready[dev]) {
    int sms = 0, smem = 0;
    if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) return B200SD_ERR_CUDA;
    if (cudaDeviceGetAttribute(&smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev) != cudaSuccess)
      return B200SD_ERR_CUDA;
    for (int bn = 32; bn <= 256; bn += 32)
      for (int bf = 0; bf < 2; ++bf)
        if (cudaFuncSetAttribute(kernel_for(bn, bf), cudaFuncAttributeMaxDynamicSharedMemorySize, smem) != cudaSuccess)
          return B200SD_ERR_CUDA;
    g_num_sms = sms;
    g_max_smem = smem;
    g_dev_ready[dev] = true;
  }
  return B200SD_OK;
}

static int launch(const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmD, const CUtensorMap& tmR,
                  GemmKernelParams& p, int is_bf16, int max_ctas, cudaStream_t stream) {
  const uint32_t stage_bytes = kATileBytes + static_cast<uint32_t>(p.block_n) * 128u;
  const int staging = (p.has_residual ? 4 : 2) * static_cast<int>(kStageTileBytes);
  const int budget = g_max_smem - 1024 /*align*/ - staging - static_cast<int>(sizeof(GemmBarriers));
  int stages = budget / static_cast<int>(stage_bytes);
  if (stages > kMaxStages) stages = kMaxStages;
  if (stages < 2) return B200SD_ERR_UNSUPPORTED;
  p.num_stages = stages;
  const size_t smem = 1024 + static_cast<size_t>(stages) * stage_bytes + staging + sizeof(GemmBarriers);
  const int num_tiles = p.num_m_tiles * p.num_n_tiles;
  int grid = num_tiles < g_num_sms ? num_tiles : g_num_sms;
  if (max_ctas > 0 && grid > max_ctas) grid = max_ctas;
  if (grid <= 0) return B200SD_OK;
  GemmKernel k = kernel_for(p.block_n, is_bf16);
  if (k == nullptr) return B200SD_ERR_INVALID;
  launch_pdl(k, dim3(grid), dim3(kGemmThreads), smem, stream, tmA, tmB, tmD, tmR, p);
  return cudaGetLastError() == cudaSuccess ? B200SD_OK : B200SD_ERR_CUDA;
}

struct OutSpec {
  void* D;
  long long ldd;
  const void* residual;
  long long ldr;
  int n_out;
};

static int fill_common(GemmKernelParams& p, OutSpec& o, int M, int N, int K, int block_n, const b200sd_epilogue* epi,
                       void* D, long long ldd, int is_bf16) {
  if (block_n < 32 || block_n > 256 || block_n % 32 != 0 || N % block_n != 0 || K % kBlockK != 0) return B200SD_ERR_INVALID;
  p.M = M; p.N = N; p.K = K; p.block_n = block_n;
  p.num_n_tiles = N / block_n;
  p.num_k_blocks = K / kBlockK;
  p.b_bytes = static_cast<uint32_t>(block_n) * 128u;
  p.bias = epi ? epi->bias : nullptr;
  p.bias_group_rows = epi ? epi->bias_group_rows : 0;
  p.flags = epi ? epi->flags : 0;
  o.D = D; o.ldd = ldd;
  o.residual = epi ? epi->residual : nullptr;
  o.ldr = epi ? epi->ldr : 0;
  p.has_residual = o.residual != nullptr ? 1 : 0;
  const bool geglu = (p.flags & B200SD_EPI_GEGLU) != 0;
  if (geglu && block_n % 64 != 0) return B200SD_ERR_INVALID;
  o.n_out = geglu ? N / 2 : N;
  if (ldd % 8 != 0 || (reinterpret_cast<uintptr_t>(D) & 15) != 0) return B200SD_ERR_INVALID;
  if (o.residual && (o.ldr % 8 != 0 || (reinterpret_cast<uintptr_t>(o.residual) & 15) != 0)) return B200SD_ERR_INVALID;
  if (p.bias && (reinterpret_cast<uintptr_t>(p.bias) & 15) != 0) return B200SD_ERR_INVALID;
  return B200SD_OK;
}

// tensor maps of the output (store) and residual (load): same geometry as the tile's rows, 32-column SWIZZLE_64B boxes
static int make_out_maps(const GemmKernelParams& p, const OutSpec& o, CUtensorMap* tmD, CUtensorMap* tmR) {
  int rc;
  for (int which = 0; which < 2; ++which) {
    const void* base = which == 0 ? o.D : o.residual;
    const long long ld = which == 0 ? o.ldd : o.ldr;
    CUtensorMap* out = which == 0 ? tmD : tmR;
    if (base == nullptr) {  // no residual: a valid (unused) map keeps the kernel signature fixed
      *tmR = *tmD;
      continue;
    }
    if (p.mode == 0) {
      const uint64_t dims[2] = {static_cast<uint64_t>(o.n_out), static_cast<uint64_t>(p.M)};
      const uint64_t strides[1] = {static_cast<uint64_t>(ld) * 2};
      const uint32_t box[2] = {kChunkCols, kBlockM};
      const uint32_t es[2] = {1, 1};
      rc = make_tmap_sw64(out, base, 2, dims, strides, box, es);
    } else {
      const uint64_t dims[4] = {static_cast<uint64_t>(o.n_out), static_cast<uint64_t>(p.W), static_cast<uint64_t>(p.H),
                                static_cast<uint64_t>(p.NB)};
      const uint64_t strides[3] = {static_cast<uint64_t>(ld) * 2, static_cast<uint64_t>(ld) * 2 * p.W,
                                   static_cast<uint64_t>(ld) * 2 * p.W * p.H};
      const uint32_t box[4] = {kChunkCols, static_cast<uint32_t>(p.bw), static_cast<uint32_t>(p.bh),
                               static_cast<uint32_t>(p.bn)};
      const uint32_t es[4] = {1, 1, 1, 1};
      rc = make_tmap_sw64(out, base, 4, dims, strides, box, es);
    }
    if (rc != B200SD_OK) return rc;
  }
  return B200SD_OK;
}

int gemm_tc(const void* A, long long lda, const void* Wt, void* D, long long ldd, int M, int N, int K, int block_n,
            const b200sd_epilogue* epi, int is_bf16, int max_ctas, cudaStream_t stream) {
  if (M <= 0) return B200SD_OK;
  GemmKernelParams p{};
  OutSpec o{};
  int rc = fill_common(p, o, M, N, K, block_n, epi, D, ldd, is_bf16);
  if (rc != B200SD_OK) return rc;
  if (lda % 8 != 0 || (reinterpret_cast<uintptr_t>(A) & 15) != 0 || (reinterpret_cast<uintptr_t>(Wt) & 15) != 0)
    return B200SD_ERR_INVALID;
  p.mode = 0;
  p.num_m_tiles = (M + kBlockM - 1) / kBlockM;
  p.a_bytes = 16384u;
  p.d_bytes = kStageTileBytes;
  rc = device_props();
  if (rc != B200SD_OK) return rc;
  CUtensorMap tmA, tmB, tmD, tmR;
  {
    const uint64_t dims[2] = {static_cast<uint64_t>(K), static_cast<uint64_t>(M)};
    const uint64_t strides[1] = {static_cast<uint64_t>(lda) * 2};
    const uint32_t box[2] = {kBlockK, kBlockM};
    const uint32_t es[2] = {1, 1};
    rc = make_tmap_sw128(&tmA, A, 2, dims, strides, box, es);
    if (rc != B200SD_OK) return rc;
  }
  {
    const uint64_t dims[2] = {static_cast<uint64_t>(K), static_cast<uint64_t>(N)};
    const uint64_t strides[1] = {static_cast<uint64_t>(K) * 2};
    const uint32_t box[2] = {kBlockK, static_cast<uint32_t>(block_n)};
    const uint32_t es[2] = {1, 1};
    rc = make_tmap_sw128(&tmB, Wt, 2, dims, strides, box, es);
    if (rc != B200SD_OK) return rc;
  }
  rc = make_out_maps(p, o, &tmD, &tmR);
  if (rc != B200SD_OK) return rc;
  return launch(tmA, tmB, tmD, tmR, p, is_bf16, max_ctas, stream);
}

int conv_tc(const void* X, long long pitch_c, int NB, int Hin, int Win, int C, const void* Wt, int ksize, int stride,
            int pad, int pad_end, void* D, long long ldd, int Cout, int block_n, const b200sd_epilogue* epi,
            int is_bf16, int max_ctas, cudaStream_t stream) {
  if (NB <= 0) return B200SD_OK;
  if ((ksize != 3 && ksize != 1) || (stride != 1 && stride != 2) || C % kBlockK != 0) return B200SD_ERR_INVALID;
  if (pitch_c % 8 != 0 || (reinterpret_cast<uintptr_t>(X) & 15) != 0 || (reinterpret_cast<uintptr_t>(Wt) & 15) != 0)
    return B200SD_ERR_INVALID;
  const int taps = ksize * ksize;
  // pad = zeros before the first row/column, pad_end = zeros after the last (the VAE encoder pads (0,1,0,1))
  const int Ho = (Hin + pad + pad_end - ksize) / stride + 1;
  const int Wo = (Win + pad + pad_end - ksize) / stride + 1;
  if (Ho <= 0 || Wo <= 0) return B200SD_ERR_INVALID;
  GemmKernelParams p{};
  OutSpec o{};
  int rc = fill_common(p, o, NB * Ho * Wo, Cout, taps * C, block_n, epi, D, ldd, is_bf16);
  if (rc != B200SD_OK) return rc;
  p.mode = 1;
  p.H = Ho; p.W = Wo; p.NB = NB;
  p.taps = taps; p.cblocks = C / kBlockK; p.stride = stride; p.pad = pad;
  // output-pixel box: as much of a row as fits, then rows, then images (all <= 128 pixels)
  p.bw = Wo < kBlockM ? Wo : kBlockM;
  p.bh = kBlockM / p.bw; if (p.bh > Ho) p.bh = Ho; if (p.bh < 1) p.bh = 1;
  p.bn = kBlockM / (p.bw * p.bh); if (p.bn > NB) p.bn = NB; if (p.bn < 1) p.bn = 1;
  p.tiles_x = (Wo + p.bw - 1) / p.bw;
  p.tiles_y = (Ho + p.bh - 1) / p.bh;
  const int tiles_n = (NB + p.bn - 1) / p.bn;
  p.num_m_tiles = p.tiles_x * p.tiles_y * tiles_n;
  p.a_bytes = static_cast<uint32_t>(p.bw * p.bh * p.bn) * 128u;
  p.d_bytes = static_cast<uint32_t>(p.bw * p.bh * p.bn) * kChunkCols * 2u;
  rc = device_props();
  if (rc != B200SD_OK) return rc;
  CUtensorMap tmA, tmB, tmD, tmR;
  {
    const uint64_t dims[4] = {static_cast<uint64_t>(C), static_cast<uint64_t>(Win), static_cast<uint64_t>(Hin),
                              static_cast<uint64_t>(NB)};
    const uint64_t strides[3] = {static_cast<uint64_t>(pitch_c) * 2, static_cast<uint64_t>(pitch_c) * 2 * Win,
                                 static_cast<uint64_t>(pitch_c) * 2 * Win * Hin};
    // with elementStrides s the box extent is given in input elements: s * (#loaded elements)
    const uint32_t box[4] = {kBlockK, static_cast<uint32_t>(p.bw * stride), static_cast<uint32_t>(p.bh * stride),
                             static_cast<uint32_t>(p.bn)};
    const uint32_t es[4] = {1, static_cast<uint32_t>(stride), static_cast<uint32_t>(stride), 1};
    if (box[1] > 256 || box[2] > 256) return B200SD_ERR_UNSUPPORTED;
    rc = make_tmap_sw128(&tmA, X, 4, dims, strides, box, es);
    if (rc != B200SD_OK) return rc;
  }
  {
    const uint64_t K = static_cast<uint64_t>(taps) * C;
    const uint64_t dims[2] = {K, static_cast<uint64_t>(Cout)};
    const uint64_t strides[1] = {K * 2};
    const uint32_t box[2] = {kBlockK, static_cast<uint32_t>(block_n)};
    const uint32_t es[2] = {1, 1};
    rc = make_tmap_sw128(&tmB, Wt, 2, dims, strides, box, es);
    if (rc != B200SD_OK) return rc;
  }
  rc = make_out_maps(p, o, &tmD, &tmR);
  if (rc != B200SD_OK) return rc;
  return launch(tmA, tmB, tmD, tmR, p, is_bf16, max_ctas, stream);
}

}  // namespace b200sd
