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
// One CTA = one Q tile of one (batch, head), warp-specialised like the GEMM: 64 * W rows on W math warpgroups and one
// producer warpgroup, 128 * (W + 1) threads.
//   * warpgroup W is the producer: one thread loads Q and runs the K / V ring (`stages` shared-memory slots of one kv
//     tile each), refilling a slot once every math warpgroup has released it;
//   * warpgroups 0 .. W-1 do the math, warpgroup w on Q rows [64w, 64w+64).
// Heads of one 64-column chunk (d <= 64) run W = 3 (192-row tiles, a four-slot ring, 24 / 160 registers per producer /
// math thread); two and three chunks run W = 2 (128-row tiles, three slots, 40 / 232 registers).  With two math
// warpgroups a one-chunk head stalls on the dependency chains of its softmax with two warps per SM sub-partition: the
// third warpgroup gives each sub-partition a third independent instruction stream.  On one H100 80GB HBM3 at a 700 W
// power limit (SM clock about 1.70 GHz), SD1.5 self-attention 4096/d40 at UNet batch 64 takes 4.26 ms per call with
// three warpgroups against 5.55 ms with two (56 % of the MUFU.EX2 peak), with bitwise equal output.
// A kv tile is kKv = 128 rows for heads of one 64-column chunk (d <= 64) and 64 rows for two or three chunks, whose
// wider O accumulator leaves no registers for a 128-wide S.  Per kv tile t and math warpgroup:
//   S_t = Q K_t^T        wgmma m64n(kKv)k16, A = Q and B = K both K-major in shared memory, S in registers
//   O += P_{t-1} V_{t-1} wgmma m64n(64*chunks)k16, A = P from registers (the S accumulator fragment is the A fragment),
//                        B = V MN-major in shared memory; issued right behind S_t, so it runs during the softmax of S_t
//   online softmax       exact running maximum of the raw logits per row (the four threads of a row agree through two
//                        shuffles), P = 2^(S * c - m * c) with c = scale * log2 e, one FFMA and one MUFU.EX2 per element;
//                        the columns >= Skv of a ragged last tile are masked (a separate instantiation of the loop body)
//   O *= alpha           once P_{t-1} V_{t-1} has completed, outside any wgmma fence -> commit window
// The math warpgroups take turns at issuing their wgmma in a fixed rotation (named barriers 2 .. 1 + W), so the tensor
// core works for one warpgroup while the others run their softmax.  The row sums are accumulated in fp32 registers, so
// the ones column a caller may place in V (v_ones_col) is not needed and its output column is not stored.  Rows >= Sq
// (zero-filled Q) are computed like the others and only their stores are skipped, so every warpgroup runs the same
// number of turns.
//
// Varlen mode (b200sd_attention_varlen, kVarlen): batch row b attends to keys [0, kv_len[b]) of a K/V buffer that is Skv
// rows long; kv_len is a device array, so one captured graph serves any split of lengths.  A CTA walks only the
// ceil(kv_len[b] / kKv) tiles it needs and masks columns >= kv_len[b] as the ragged tail of a plain call.  Tile walk and
// reduction order are those of a plain call with Skv = kv_len[b], so the results are bitwise equal to it as long as the
// buffer rows in [kv_len[b], kKv * ceil(kv_len[b] / kKv)) hold finite values (they get P = 0, where a plain call reads
// the tensor map's zero fill).
#include <cstddef>
#include <cstdlib>

#include "tc_common.cuh"
#include "wgmma.cuh"
#include "b200sd_internal.h"
#include "pdl.cuh"

namespace b200sd {

constexpr int kMaxStages = 4;
__host__ __device__ constexpr int kv_tile(int chunks) { return chunks == 1 ? 128 : 64; }
__host__ __device__ constexpr int math_warpgroups(int chunks) { return chunks == 1 ? 3 : 2; }
__host__ __device__ constexpr int q_tile(int chunks) { return 64 * math_warpgroups(chunks); }
__host__ __device__ constexpr int attn_threads(int chunks) { return 128 * (math_warpgroups(chunks) + 1); }
// K / V ring depth: four slots of 32 KB next to the 24 KB Q tile for one chunk; the wider heads keep three
__host__ __device__ constexpr int max_stages(int chunks) { return chunks == 1 ? kMaxStages : 3; }

struct AttnParams {
  int B, heads, Sq, Skv, d, d_pad;
  int d16;           // d rounded up to 16 (MMA K of Q.K^T)
  int chunks;        // 64-column chunks per head tile
  int stages;        // K / V ring slots
  float scale_log2;  // softmax scale * log2(e)
  void* O;
  long long ldo;
  const int* kv_len;  // varlen: [B] key counts on the device, clamped to [1, Skv]
};

struct __align__(8) AttnShared {
  uint64_t q_full;
  uint64_t kv_full[kMaxStages];
  uint64_t kv_empty[kMaxStages];  // one arrival per math warpgroup
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

// Rotation of the math warpgroups: warpgroup w issues its wgmma between turn_wait (bar.sync 2 + w) and turn_pass
// (bar.arrive on the barrier of warpgroup (w + 1) % kMathWg).  Each barrier counts the 128 threads that wait on it and
// the 128 that pass to it.  Ids 2..4 stay clear of __syncthreads (0) and of the GEMM's consumer barrier (1).
__device__ __forceinline__ void turn_wait(int wg) {
  asm volatile("bar.sync %0, %1;" ::"r"(2 + wg), "n"(256) : "memory");
}
template <int kMathWg>
__device__ __forceinline__ void turn_pass(int wg) {
  asm volatile("bar.arrive %0, %1;" ::"r"(2 + (wg + 1) % kMathWg), "n"(256) : "memory");
}

// Online softmax of one kv tile in place: s (the S accumulator, raw logits) becomes P = 2^(s * c - m * c) in fp32,
// m_run / l_run advance, alpha = 2^((m_old - m_new) * c) is the factor O still has to be rescaled by.  kMask: columns
// >= valid are -inf (the ragged last tile only).  The row maximum runs as four independent chains, combined at the end
// (fmaxf is exact, so the order does not change it); the row sum keeps its one serial order.
template <int kKv, bool kMask>
__device__ __forceinline__ void softmax_tile(float (&s)[kKv / 2], float (&m_run)[2], float (&l_run)[2],
                                             float (&alpha)[2], float c, int valid, int colq) {
  float mp[2][4];
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int j = 0; j < 4; ++j) mp[h][j] = -INFINITY;
#pragma unroll
  for (int g = 0; g < kKv / 8; ++g)
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        float& v = s[4 * g + 2 * h + e];
        if constexpr (kMask) v = (8 * g + colq + e < valid) ? v : -INFINITY;
        float& m = mp[h][2 * (g & 1) + e];
        m = fmaxf(m, v);
      }
  float mx[2], mc[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    mx[h] = fmaxf(fmaxf(mp[h][0], mp[h][1]), fmaxf(mp[h][2], mp[h][3]));
    mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 1));
    mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 2));
    const float m_new = fmaxf(m_run[h], mx[h]);     // finite: every kv tile has at least one valid column
    alpha[h] = fast_exp2((m_run[h] - m_new) * c);  // 2^(-inf) = 0 on the first tile; exactly 1 while the max holds
    m_run[h] = m_new;
    mc[h] = m_new * c;
    l_run[h] *= alpha[h];
  }
#pragma unroll
  for (int g = 0; g < kKv / 8; ++g)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float& p0 = s[4 * g + 2 * h];
      float& p1 = s[4 * g + 2 * h + 1];
      p0 = fast_exp2(fmaf(p0, c, -mc[h]));
      p1 = fast_exp2(fmaf(p1, c, -mc[h]));
      l_run[h] += p0 + p1;
    }
}

// S = Q K^T over kSteps k16 steps of the head dimension.  The count is a compile-time constant: ptxas serialises wgmma
// issued from a run-time loop.
// The descriptors of the later steps are those of step 0 plus the byte offset / 16 (start-address field, no carry: shared
// memory ends below 256 KB).
template <int kSteps, int kKv, uint32_t kQChunkBytes, bool kBf16>
__device__ __forceinline__ void qk_tile(float (&s)[kKv / 2], uint64_t dq, uint64_t dk) {
#pragma unroll
  for (int ks = 0; ks < kSteps; ++ks) {
    const uint32_t off = static_cast<uint32_t>(ks & 3) * 32u;  // k16 step inside the 128-byte swizzled row
    Wgmma<kKv, kBf16>::ss(s, dq + ((static_cast<uint32_t>(ks >> 2) * kQChunkBytes + off) >> 4),
                          dk + ((static_cast<uint32_t>(ks >> 2) * (kKv * 128u) + off) >> 4), ks != 0 ? 1u : 0u);
  }
}

template <int kChunks, bool kBf16, bool kVarlen>
__global__ void __launch_bounds__(attn_threads(kChunks), 1)
attention_tc_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                    const __grid_constant__ CUtensorMap tmV, const AttnParams p) {
  constexpr int kKv = kv_tile(kChunks);
  constexpr int kMathWg = math_warpgroups(kChunks);
  constexpr int kMathThreads = 128 * kMathWg;
  constexpr int kQTile = q_tile(kChunks);
  constexpr uint32_t kQChunkBytes = kQTile * 128;        // kQTile rows x 64 halfs
  constexpr int kDv = 64 * kChunks;                      // MMA N of P.V
  // P_{t-1} V_{t-1} runs during the softmax of S_t; three chunks have no registers for S_t and P_{t-1} next to O
  constexpr bool kOverlap = kChunks < 3;
  constexpr uint32_t kKvChunkBytes = kKv * 128;          // kKv rows x 64 halfs
  constexpr uint32_t kKvBytes = kChunks * kKvChunkBytes;
  extern __shared__ uint8_t smem_raw[];
  pdl_trigger();  // pdl.cuh: the next kernel's prologue may overlap this kernel's tail
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sQ = smem;                                   // chunks x (kQTile rows x 64)
  uint8_t* sK = sQ + kChunks * kQChunkBytes;            // stages x chunks x (kKv rows x 64)
  uint8_t* sV = sK + p.stages * kKvBytes;
  AttnShared* sh = reinterpret_cast<AttnShared*>(sV + p.stages * kKvBytes);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int qt = blockIdx.x;
  const int head = blockIdx.y;
  const int b = blockIdx.z;
  const int col0 = head * p.d_pad;

  if (threadIdx.x == kMathThreads) {
    tma_prefetch_desc(&tmQ);
    tma_prefetch_desc(&tmK);
    tma_prefetch_desc(&tmV);
    mbar_init(&sh->q_full, 1);
    for (int s = 0; s < kMaxStages; ++s) {
      mbar_init(&sh->kv_full[s], 1);
      mbar_init(&sh->kv_empty[s], kMathWg);
    }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();  // Q / K / V come from the preceding projection GEMM
  const int skv = kVarlen ? min(max(p.kv_len[b], 1), p.Skv) : p.Skv;  // keys this batch row attends to
  const int nkv = (skv + kKv - 1) / kKv;

  if (warp >= kMathThreads / 32) {
    // ------------------------------- producer (one thread) -------------------------------
    // 128 x 24 + 384 x 160 and 128 x 40 + 256 x 232 registers fit the 64 K of the SM
    setmaxnreg_dec<kMathWg == 3 ? 24 : 40>();
    if (threadIdx.x == kMathThreads) {
      mbar_arrive_expect_tx(&sh->q_full, kChunks * kQChunkBytes);
#pragma unroll
      for (int c = 0; c < kChunks; ++c)
        tma_load_3d(sQ + c * kQChunkBytes, &tmQ, &sh->q_full, col0 + c * 64, qt * kQTile, b);
      int s = 0;           // slot of tile t
      uint32_t phase = 0;  // parity of its use t / stages
      for (int t = 0; t < nkv; ++t) {
        // wait for the release of the slot's previous use
        if (t >= p.stages) mbar_wait(&sh->kv_empty[s], phase ^ 1u);
        mbar_arrive_expect_tx(&sh->kv_full[s], 2 * kKvBytes);
#pragma unroll
        for (int c = 0; c < kChunks; ++c) {
          tma_load_3d(sK + s * kKvBytes + c * kKvChunkBytes, &tmK, &sh->kv_full[s], col0 + c * 64, t * kKv, b);
          tma_load_3d(sV + s * kKvBytes + c * kKvChunkBytes, &tmV, &sh->kv_full[s], col0 + c * 64, t * kKv, b);
        }
        if (++s == p.stages) { s = 0; phase ^= 1u; }
      }
    }
    return;
  }

  // ------------------------------- math warpgroups -------------------------------
  setmaxnreg_inc<kMathWg == 3 ? 160 : 232>();
  const int wg = warp >> 2;
  const int colq = (lane & 3) * 2;  // accumulator columns 8g + colq, +1 of rows r0 (h = 0) and r0 + 8 (h = 1)
  const bool signaller = (threadIdx.x & 127) == 0;  // releases ring slots for its warpgroup
  const float c = p.scale_log2;
  const bool ragged = skv % kKv != 0;
  const uint32_t sQ_a = smem_u32(sQ) + static_cast<uint32_t>(wg) * 8192u;
  const uint32_t sK_a = smem_u32(sK), sV_a = smem_u32(sV);
  float o[kDv / 2];
#pragma unroll
  for (int i = 0; i < kDv / 2; ++i) o[i] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f}, alpha[2];
  float sacc[kKv / 2];
  uint32_t pa[kKv / 16][4];  // P of the previous tile as the A fragments of the k16 steps of P.V

  auto issue_qk = [&](int s) {  // S = Q K^T of the tile in slot s; d16 / 16 lies in [4 kChunks - 3, 4 kChunks]
    const uint64_t dq = make_gdesc_sw128(sQ_a, 16, 1024);
    const uint64_t dk = make_gdesc_sw128(sK_a + static_cast<uint32_t>(s) * kKvBytes, 16, 1024);
    switch (p.d16 / 16 - 4 * kChunks) {
      case -3: qk_tile<4 * kChunks - 3, kKv, kQChunkBytes, kBf16>(sacc, dq, dk); break;
      case -2: qk_tile<4 * kChunks - 2, kKv, kQChunkBytes, kBf16>(sacc, dq, dk); break;
      case -1: qk_tile<4 * kChunks - 1, kKv, kQChunkBytes, kBf16>(sacc, dq, dk); break;
      default: qk_tile<4 * kChunks, kKv, kQChunkBytes, kBf16>(sacc, dq, dk); break;
    }
    wgmma_commit();
  };
  auto issue_pv = [&](int s) {  // O += P V of the tile in slot s
    const uint64_t dv = make_gdesc_sw128(sV_a + static_cast<uint32_t>(s) * kKvBytes, kKvChunkBytes, 1024);
#pragma unroll
    for (int j = 0; j < kKv / 16; ++j) Wgmma<kDv, kBf16>::rs_tb(o, pa[j], dv + static_cast<uint32_t>(j) * (2048u >> 4), 1u);
    wgmma_commit();
  };
  auto softmax = [&](int t) {
    if (ragged && t == nkv - 1) softmax_tile<kKv, true>(sacc, m_run, l_run, alpha, c, skv - t * kKv, colq);
    else softmax_tile<kKv, false>(sacc, m_run, l_run, alpha, c, 0, colq);
  };
  auto pack_p = [&]() {
#pragma unroll
    for (int g = 0; g < kKv / 8; ++g)
#pragma unroll
      for (int h = 0; h < 2; ++h) pa[g >> 1][(g & 1) * 2 + h] = pack_h2<kBf16>(sacc[4 * g + 2 * h], sacc[4 * g + 2 * h + 1]);
  };

  // Turns go round warpgroups 0, 1, .., kMathWg - 1: the last one passes once up front, so warpgroup 0 goes first.
  // Each warpgroup takes nkv + 1 turns (S_0; S_t with P_{t-1} V_{t-1}; the last P V) and passes after each; the last
  // warpgroup skips its final pass, which nobody waits for.
  if (wg == kMathWg - 1) turn_pass<kMathWg>(wg);
  int s = 0;           // slot of tile t
  uint32_t phase = 0;  // parity of its use t / stages
  mbar_wait_unbounded(&sh->q_full, 0);
  mbar_wait_unbounded(&sh->kv_full[0], 0);
  turn_wait(wg);
  wgmma_fence();
  issue_qk(0);
  turn_pass<kMathWg>(wg);
  wgmma_wait<0>();
  reg_fence(sacc);
  softmax(0);
  pack_p();

  for (int t = 1; t < nkv; ++t) {
    const int s_prev = s;
    if (++s == p.stages) { s = 0; phase ^= 1u; }
    mbar_wait_unbounded(&sh->kv_full[s], phase);
    turn_wait(wg);
    reg_fence(o);
    wgmma_fence();
    if constexpr (kOverlap) {
      issue_qk(s);
      issue_pv(s_prev);
    } else {
      issue_pv(s_prev);
      wgmma_wait<0>();  // P is dead: S_t may take its registers
      reg_fence(o);
      wgmma_fence();
      issue_qk(s);
    }
    turn_pass<kMathWg>(wg);
    wgmma_wait<kOverlap ? 1 : 0>();  // S_t has landed; with kOverlap, P_{t-1} V_{t-1} is still running
    reg_fence(sacc);
    softmax(t);
    wgmma_wait<0>();
    reg_fence(o);
    if (signaller) mbar_arrive(&sh->kv_empty[s_prev]);
#pragma unroll
    for (int i = 0; i < kDv / 2; ++i) o[i] *= alpha[(i >> 1) & 1];
    pack_p();
  }

  turn_wait(wg);
  reg_fence(o);
  wgmma_fence();
  issue_pv(s);
  if (wg != kMathWg - 1) turn_pass<kMathWg>(wg);
  wgmma_wait<0>();
  reg_fence(o);
  if (signaller) mbar_arrive(&sh->kv_empty[s]);

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

template <bool kVarlen>
static AttnKernel attn_kernel_for(int chunks, int is_bf16) {
  switch (chunks * 2 + (is_bf16 ? 1 : 0)) {
    case 2: return attention_tc_kernel<1, false, kVarlen>;
    case 3: return attention_tc_kernel<1, true, kVarlen>;
    case 4: return attention_tc_kernel<2, false, kVarlen>;
    case 5: return attention_tc_kernel<2, true, kVarlen>;
    case 6: return attention_tc_kernel<3, false, kVarlen>;
    case 7: return attention_tc_kernel<3, true, kVarlen>;
    default: return nullptr;
  }
}

static int g_attn_max_smem = 0;
static bool g_attn_dev_ready[64] = {};

int attention_tc(const void* Q, long long ldq, const void* K, long long ldk, const void* V, long long ldv, void* O,
                 long long ldo, int B, int heads, int Sq, int Skv, const int* kv_len, int d, int d_pad, float scale,
                 int v_ones_col, int is_bf16, cudaStream_t stream) {
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
  if (kv_len && (reinterpret_cast<uintptr_t>(kv_len) & 3)) return B200SD_ERR_INVALID;
  const int chunks = (((d + 15) & ~15) + 63) / 64;  // 64-column chunks that hold the d16 columns the MMAs read
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
          if (cudaFuncSetAttribute(attn_kernel_for<false>(c, bf), cudaFuncAttributeMaxDynamicSharedMemorySize, smem) !=
                  cudaSuccess ||
              cudaFuncSetAttribute(attn_kernel_for<true>(c, bf), cudaFuncAttributeMaxDynamicSharedMemorySize, smem) !=
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
  p.kv_len = kv_len;
  const int kv = kv_tile(chunks);
  const int nkv = (Skv + kv - 1) / kv;
  const int qtile = q_tile(chunks);
  const size_t qt = static_cast<size_t>(chunks) * qtile * 128;
  const size_t kvt = 2 * static_cast<size_t>(chunks) * kv * 128;  // K and V of one slot
  p.stages = nkv < max_stages(chunks) ? nkv : max_stages(chunks);
  const size_t smem = 1024 + qt + static_cast<size_t>(p.stages) * kvt + sizeof(AttnShared);
  if (smem > static_cast<size_t>(g_attn_max_smem)) return B200SD_ERR_UNSUPPORTED;
  CUtensorMap tmQ, tmK, tmV;
  const uint32_t es[3] = {1, 1, 1};
  int rc;
  {
    const uint32_t box[3] = {64, static_cast<uint32_t>(qtile), 1};
    const uint64_t dims[3] = {static_cast<uint64_t>(heads) * d_pad, static_cast<uint64_t>(Sq), static_cast<uint64_t>(B)};
    const uint64_t st[2] = {static_cast<uint64_t>(ldq) * 2, static_cast<uint64_t>(ldq) * 2 * Sq};
    if ((rc = make_tmap_sw128(&tmQ, Q, 3, dims, st, box, es)) != B200SD_OK) return rc;
  }
  const uint32_t kvbox[3] = {64, static_cast<uint32_t>(kv), 1};
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
  dim3 grid((Sq + qtile - 1) / qtile, heads, B);
  launch_pdl(kv_len ? attn_kernel_for<true>(chunks, is_bf16) : attn_kernel_for<false>(chunks, is_bf16), grid,
             dim3(attn_threads(chunks)), smem, stream, tmQ, tmK, tmV, p);
  return cudaGetLastError() == cudaSuccess ? B200SD_OK : B200SD_ERR_CUDA;
}

}  // namespace b200sd
