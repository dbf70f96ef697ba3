// attention_tc.cu — flash-attention forward (non-causal) on wgmma for sm_90a.
//
//   O[b, s, h, :] = softmax(Q[b, s, h, :] . K[b, :, h, :]^T * scale) . V[b, :, h, :]
//
// Covers the UNet's self-attention (S = 4096/1024/256/64, d = 40/80/160) and cross-attention (77 context
// tokens) — upstream ldm CrossAttention (SURVEY.md §8 a-ext x6, x7).
//
// Layout: Q/K/V rows are tokens; every head owns d_pad (multiple of 16) consecutive halfs, the first d of which are
// data and the rest zero (the projection GEMM produces this directly from zero-padded weight rows).  Shared-memory tiles
// are whole 64-column chunks, each one TMA SWIZZLE_128B box; a box that runs past its head reads the next head's first
// columns (never used: Q.K^T stops at d16, and P.V columns >= d are not stored) or, for the last head, the tensor map's
// zero fill.  O is written unpadded ([b, s, h*d]) because it feeds the out-projection GEMM as a plain K-major A operand.
//
// One CTA = one 128-row Q tile of one (batch, head); 256 threads = two warpgroups, warpgroup w owns Q rows
// [64w, 64w+64).  K / V are consumed in tiles of 64 rows through a ring of `stages` shared-memory slots that thread 0
// refills by TMA (a slot is refilled once both warpgroups have released it).  Per kv tile and warpgroup:
//   S = Q K^T        wgmma m64n64k16, A = Q and B = K both K-major in shared memory, S in registers
//   online softmax   exact running maximum per row (the four threads of a row agree through two shuffles), P = 2^(S*scale*log2 e - m)
//   O += P V         wgmma m64n(64*chunks)k16 with A = P from registers (the S accumulator fragment is the A fragment)
//                    and B = V MN-major in shared memory
// The row sums are accumulated in fp32 registers, so the ones column a caller may place in V (v_ones_col) is not needed
// and its output column is not stored.
#include <cstddef>
#include <cstdlib>

#include "tc_common.cuh"
#include "wgmma.cuh"
#include "b200sd_internal.h"
#include "pdl.cuh"

namespace b200sd {

constexpr int kAttnThreads = 256;                    // two warpgroups
constexpr int kQTile = 128;
constexpr int kKv = 64;                              // kv rows per tile
constexpr int kMaxStages = 3;
constexpr uint32_t kQChunkBytes = kQTile * 128;      // 128 rows x 64 halfs
constexpr uint32_t kKvChunkBytes = kKv * 128;        // 64 rows x 64 halfs

struct AttnParams {
  int B, heads, Sq, Skv, d, d_pad;
  int d16;           // d rounded up to 16 (MMA K of Q.K^T)
  int chunks;        // 64-column chunks per head tile
  int stages;        // K / V ring slots
  float scale_log2;  // softmax scale * log2(e)
  void* O;
  long long ldo;
};

struct __align__(8) AttnShared {
  uint64_t q_full;
  uint64_t kv_full[kMaxStages];
  uint64_t kv_empty[kMaxStages];  // one arrival per warpgroup
};

template <bool kBf16>
__device__ __forceinline__ uint32_t pack_h2(float a, float b) {
  if constexpr (kBf16) {
    __nv_bfloat162 v = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&v);
  } else {
    __half2 v = __floats2half2_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&v);
  }
}

template <int kChunks, bool kBf16>
__global__ void __launch_bounds__(kAttnThreads, 1)
attention_tc_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                    const __grid_constant__ CUtensorMap tmV, const AttnParams p) {
  constexpr int kDv = 64 * kChunks;  // MMA N of P.V
  constexpr uint32_t kKvBytes = kChunks * kKvChunkBytes;
  extern __shared__ uint8_t smem_raw[];
  pdl_trigger();  // pdl.cuh: the next kernel's prologue may overlap this kernel's tail
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sQ = smem;                                   // chunks x (128 rows x 64)
  uint8_t* sK = sQ + kChunks * kQChunkBytes;            // stages x chunks x (64 rows x 64)
  uint8_t* sV = sK + p.stages * kKvBytes;
  AttnShared* sh = reinterpret_cast<AttnShared*>(sV + p.stages * kKvBytes);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int wg = warp >> 2;
  const int qt = blockIdx.x;
  const int head = blockIdx.y;
  const int b = blockIdx.z;
  const int nkv = (p.Skv + kKv - 1) / kKv;
  const int col0 = head * p.d_pad;
  const bool loader = threadIdx.x == 0;

  if (loader) {
    tma_prefetch_desc(&tmQ);
    tma_prefetch_desc(&tmK);
    tma_prefetch_desc(&tmV);
    mbar_init(&sh->q_full, 1);
    for (int s = 0; s < kMaxStages; ++s) {
      mbar_init(&sh->kv_full[s], 1);
      mbar_init(&sh->kv_empty[s], 2);
    }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();  // Q / K / V come from the preceding projection GEMM

  auto load_kv = [&](int t) {  // tile t into slot t % stages (the slot is free)
    const int s = t % p.stages;
    mbar_arrive_expect_tx(&sh->kv_full[s], 2 * kKvBytes);
#pragma unroll
    for (int c = 0; c < kChunks; ++c) {
      tma_load_3d(sK + s * kKvBytes + c * kKvChunkBytes, &tmK, &sh->kv_full[s], col0 + c * 64, t * kKv, b);
      tma_load_3d(sV + s * kKvBytes + c * kKvChunkBytes, &tmV, &sh->kv_full[s], col0 + c * 64, t * kKv, b);
    }
  };
  if (loader) {
    mbar_arrive_expect_tx(&sh->q_full, kChunks * kQChunkBytes);
#pragma unroll
    for (int c = 0; c < kChunks; ++c) tma_load_3d(sQ + c * kQChunkBytes, &tmQ, &sh->q_full, col0 + c * 64, qt * kQTile, b);
    for (int t = 0; t < p.stages && t < nkv; ++t) load_kv(t);
  }

  const int colq = (lane & 3) * 2;  // accumulator columns 8g + colq, +1 of rows r0 (h = 0) and r0 + 8 (h = 1)
  const uint32_t sQ_a = smem_u32(sQ) + static_cast<uint32_t>(wg) * 8192u;
  const uint32_t sK_a = smem_u32(sK), sV_a = smem_u32(sV);
  float o[kDv / 2];
#pragma unroll
  for (int i = 0; i < kDv / 2; ++i) o[i] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
  mbar_wait(&sh->q_full, 0);

  for (int t = 0; t < nkv; ++t) {
    // refill the slot of tile t-1 with tile t-1+stages once both warpgroups are done with it
    if (loader && t > 0 && t - 1 + p.stages < nkv) {
      const int s = (t - 1) % p.stages;
      mbar_wait(&sh->kv_empty[s], static_cast<uint32_t>((t - 1) / p.stages) & 1u);
      load_kv(t - 1 + p.stages);
    }
    const int s = t % p.stages;
    mbar_wait(&sh->kv_full[s], static_cast<uint32_t>(t / p.stages) & 1u);

    // S = Q K^T
    float sacc[32];
    const uint32_t k_a = sK_a + static_cast<uint32_t>(s) * kKvBytes;
    wgmma_fence();
    for (int ks = 0; ks < p.d16 / 16; ++ks) {
      const uint32_t off = static_cast<uint32_t>(ks & 3) * 32u;  // k16 step inside the 128-byte swizzled row
      Wgmma<64, kBf16>::ss(sacc, make_gdesc_sw128(sQ_a + static_cast<uint32_t>(ks >> 2) * kQChunkBytes + off, 16, 1024),
                           make_gdesc_sw128(k_a + static_cast<uint32_t>(ks >> 2) * kKvChunkBytes + off, 16, 1024),
                           ks != 0 ? 1u : 0u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(sacc);

    // online softmax (scaled logits in log2 units); kv columns >= Skv are masked
    const int valid = p.Skv - t * kKv;
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int g = 0; g < 8; ++g)
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          float& v = sacc[4 * g + 2 * h + e];
          v = (8 * g + colq + e < valid) ? v * p.scale_log2 : -INFINITY;
          mx[h] = fmaxf(mx[h], v);
        }
    float alpha[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 1));
      mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 2));
      const float m_new = fmaxf(m_run[h], mx[h]);  // finite: every kv tile has at least one valid column
      alpha[h] = fast_exp2(m_run[h] - m_new);      // 2^(-inf) = 0 on the first tile
      m_run[h] = m_new;
      l_run[h] *= alpha[h];
    }
#pragma unroll
    for (int i = 0; i < kDv / 2; ++i) o[i] *= alpha[(i >> 1) & 1];
    uint32_t pa[4][4];  // P as the A fragments of the four k16 steps of P.V
#pragma unroll
    for (int g = 0; g < 8; ++g)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const float p0 = fast_exp2(sacc[4 * g + 2 * h] - m_run[h]);
        const float p1 = fast_exp2(sacc[4 * g + 2 * h + 1] - m_run[h]);
        l_run[h] += p0 + p1;
        pa[g >> 1][(g & 1) * 2 + h] = pack_h2<kBf16>(p0, p1);
      }

    // O += P V
    const uint32_t v_a = sV_a + static_cast<uint32_t>(s) * kKvBytes;
    reg_fence(o);
    wgmma_fence();
#pragma unroll
    for (int j = 0; j < 4; ++j)
      Wgmma<kDv, kBf16>::rs_tb(o, pa[j], make_gdesc_sw128(v_a + static_cast<uint32_t>(j) * 2048u, kKvChunkBytes, 1024), 1u);
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(o);
    if ((threadIdx.x & 127) == 0) mbar_arrive(&sh->kv_empty[s]);
  }

  // O / l -> global (rows < Sq, columns < d)
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    l_run[h] += __shfl_xor_sync(0xffffffffu, l_run[h], 1);
    l_run[h] += __shfl_xor_sync(0xffffffffu, l_run[h], 2);
  }
  const int r0 = qt * kQTile + wg * 64 + (warp & 3) * 16 + (lane >> 2);
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int row = r0 + 8 * h;
    if (row >= p.Sq) continue;
    const float inv = 1.0f / l_run[h];
    uint8_t* orow = static_cast<uint8_t*>(p.O) + ((static_cast<long long>(b) * p.Sq + row) * p.ldo +
                                                  static_cast<long long>(head) * p.d) * 2;
#pragma unroll
    for (int g = 0; g < kDv / 8; ++g) {
      const int col = 8 * g + colq;
      if (col < p.d)
        *reinterpret_cast<uint32_t*>(orow + col * 2) = pack_h2<kBf16>(o[4 * g + 2 * h] * inv, o[4 * g + 2 * h + 1] * inv);
    }
  }
}

// ------------------------------------------------------------------------------------------------
typedef void (*AttnKernel)(CUtensorMap, CUtensorMap, CUtensorMap, AttnParams);

static AttnKernel attn_kernel_for(int chunks, int is_bf16) {
  switch (chunks * 2 + (is_bf16 ? 1 : 0)) {
    case 2: return attention_tc_kernel<1, false>;
    case 3: return attention_tc_kernel<1, true>;
    case 4: return attention_tc_kernel<2, false>;
    case 5: return attention_tc_kernel<2, true>;
    case 6: return attention_tc_kernel<3, false>;
    case 7: return attention_tc_kernel<3, true>;
    default: return nullptr;
  }
}

static int g_attn_max_smem = 0;
static bool g_attn_dev_ready[64] = {};

int attention_tc(const void* Q, long long ldq, const void* K, long long ldk, const void* V, long long ldv, void* O,
                 long long ldo, int B, int heads, int Sq, int Skv, int d, int d_pad, float scale, int v_ones_col,
                 int is_bf16, cudaStream_t stream) {
  if (B <= 0 || heads <= 0 || Sq <= 0) return B200SD_OK;
  // d_pad: the head pitch in Q / K / V, a multiple of 16
  if (Skv <= 0 || d <= 0 || d % 8 != 0 || d_pad % 16 != 0 || d_pad < d) return B200SD_ERR_INVALID;
  if (ldq % 8 || ldk % 8 || ldv % 8 || ldo % 8) return B200SD_ERR_INVALID;
  if ((reinterpret_cast<uintptr_t>(Q) | reinterpret_cast<uintptr_t>(K) | reinterpret_cast<uintptr_t>(V) |
       reinterpret_cast<uintptr_t>(O)) & 15)
    return B200SD_ERR_INVALID;
  if (ldq < static_cast<long long>(heads) * d_pad || ldk < static_cast<long long>(heads) * d_pad ||
      ldv < static_cast<long long>(heads) * d_pad || ldo < static_cast<long long>(heads) * d)
    return B200SD_ERR_INVALID;
  if (v_ones_col && d >= d_pad) return B200SD_ERR_INVALID;  // the ones column needs a free pad column
  const int chunks = (d_pad + 63) / 64;
  if (chunks > 3) return B200SD_ERR_UNSUPPORTED;
  {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return B200SD_ERR_CUDA;
    if (dev < 0 || dev >= 64) return B200SD_ERR_UNSUPPORTED;
    if (!g_attn_dev_ready[dev]) {  // per-device opt-in to large dynamic smem; first call must be outside capture
      int smem = 0;
      if (cudaDeviceGetAttribute(&smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev) != cudaSuccess)
        return B200SD_ERR_CUDA;
      for (int c = 1; c <= 3; ++c)
        for (int bf = 0; bf < 2; ++bf)
          if (cudaFuncSetAttribute(attn_kernel_for(c, bf), cudaFuncAttributeMaxDynamicSharedMemorySize, smem) !=
              cudaSuccess)
            return B200SD_ERR_CUDA;
      g_attn_max_smem = smem;
      g_attn_dev_ready[dev] = true;
    }
  }
  AttnParams p{};
  p.B = B; p.heads = heads; p.Sq = Sq; p.Skv = Skv; p.d = d; p.d_pad = d_pad;
  p.d16 = (d + 15) & ~15;
  p.chunks = chunks;
  p.scale_log2 = scale * 1.4426950408889634f;
  p.O = O; p.ldo = ldo;
  const int nkv = (Skv + kKv - 1) / kKv;
  const size_t qt = static_cast<size_t>(chunks) * kQChunkBytes;
  const size_t kvt = 2 * static_cast<size_t>(chunks) * kKvChunkBytes;  // K and V of one slot
  p.stages = nkv < kMaxStages ? nkv : kMaxStages;
  const size_t smem = 1024 + qt + static_cast<size_t>(p.stages) * kvt + sizeof(AttnShared);
  if (smem > static_cast<size_t>(g_attn_max_smem)) return B200SD_ERR_UNSUPPORTED;
  CUtensorMap tmQ, tmK, tmV;
  const uint32_t es[3] = {1, 1, 1};
  int rc;
  {
    const uint32_t box[3] = {64, kQTile, 1};
    const uint64_t dims[3] = {static_cast<uint64_t>(heads) * d_pad, static_cast<uint64_t>(Sq), static_cast<uint64_t>(B)};
    const uint64_t st[2] = {static_cast<uint64_t>(ldq) * 2, static_cast<uint64_t>(ldq) * 2 * Sq};
    if ((rc = make_tmap_sw128(&tmQ, Q, 3, dims, st, box, es)) != B200SD_OK) return rc;
  }
  const uint32_t kvbox[3] = {64, kKv, 1};
  {
    const uint64_t dims[3] = {static_cast<uint64_t>(heads) * d_pad, static_cast<uint64_t>(Skv), static_cast<uint64_t>(B)};
    const uint64_t st[2] = {static_cast<uint64_t>(ldk) * 2, static_cast<uint64_t>(ldk) * 2 * Skv};
    if ((rc = make_tmap_sw128(&tmK, K, 3, dims, st, kvbox, es)) != B200SD_OK) return rc;
  }
  {
    const uint64_t dims[3] = {static_cast<uint64_t>(heads) * d_pad, static_cast<uint64_t>(Skv), static_cast<uint64_t>(B)};
    const uint64_t st[2] = {static_cast<uint64_t>(ldv) * 2, static_cast<uint64_t>(ldv) * 2 * Skv};
    if ((rc = make_tmap_sw128(&tmV, V, 3, dims, st, kvbox, es)) != B200SD_OK) return rc;
  }
  dim3 grid((Sq + kQTile - 1) / kQTile, heads, B);
  launch_pdl(attn_kernel_for(chunks, is_bf16), grid, dim3(kAttnThreads), smem, stream, tmQ, tmK, tmV, p);
  return cudaGetLastError() == cudaSuccess ? B200SD_OK : B200SD_ERR_CUDA;
}

}  // namespace b200sd
