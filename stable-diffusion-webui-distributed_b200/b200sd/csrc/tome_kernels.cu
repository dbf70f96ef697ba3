// tome_kernels.cu — token merging (tomesd 0.1.3 as sdwui applies it: bipartite soft matching on the 2x2 grid, no
// random dst choice) for the self-attention of the UNet's full-resolution transformer blocks.
//
// Tokens are the h*w latent pixels of one batch row, t = y*w + x (h and w even).  The top-left token of every 2x2 block
// is a dst token, dst index j = (y/2) * (w/2) + x/2; the other 3/4 are src tokens, numbered a = 0.. in ascending token
// order.  With r merged tokens the merged sequence has Nm = N - r slots: slots [0, Ns - r) are the unmerged src tokens in
// ascending token order, slot Ns - r + j is dst token j together with every src token merged into it.
//
// b200sd_tome_match, per batch row:
//   1. tome_normalize: metric = x / ||x|| rounded to fp16 (tomesd normalises in the model dtype), gathered into a src
//      and a dst matrix in the workspace.
//   2. tome_argmax: node_max[a], node_idx[a] = max / argmax over dst b of metric_a . metric_b.  wgmma m64n64k16 with
//      fp32 accumulation: a CTA holds 128 src rows in shared memory and streams the dst rows through a TMA ring of 64-row
//      tiles; each thread keeps a running (max, argmax) of its accumulator columns, no score matrix is written.  Ties go
//      to the lowest dst index.
//   3. tome_select: the r src tokens with the largest keys (node_max desc, src index asc) — an exact top-r by an MSB-first
//      radix select over the order-preserving 32-bit image of node_max, then the first ties by index — and the partition
//      slot[N] / members[N] / seg[Nm + 1] (members ordered by slot, ascending token index within a slot).
// b200sd_tome_merge: Y[s] = fp32 mean of X over members of slot s (ascending token order), rounded once.
// b200sd_tome_unmerge_add: out[t] = round(R[t] + Y[slot[t]]).
#include <cstddef>

#include "tc_common.cuh"
#include "wgmma.cuh"

namespace b200sd {

constexpr int kTomeSrcTile = 128;             // src rows per CTA (two math warpgroups of 64)
constexpr int kTomeDstTile = 64;              // dst rows per ring slot (MMA N)
constexpr int kTomeMaxStages = 4;
constexpr int kTomeMathThreads = 256;
constexpr int kTomeThreads = kTomeMathThreads + 32;   // + one producer warp
constexpr uint32_t kTomeSrcChunkBytes = kTomeSrcTile * 128;   // 128 rows x 64 halfs
constexpr uint32_t kTomeDstChunkBytes = kTomeDstTile * 128;
constexpr int kTomeSelectThreads = 1024;

struct TomeDims {
  int B, H, W, C, N, Ns, Nd, r;
};

__host__ __device__ inline size_t tome_align(size_t v) { return (v + 255) & ~static_cast<size_t>(255); }

// workspace: src metric fp16 [B][Ns][C], dst metric fp16 [B][Nd][C], node_max f32 [B][Ns], node_idx i32 [B][Ns],
// per-dst counters i32 [B][Nd]
struct TomeWorkspace {
  size_t msrc, mdst, nmax, nidx, cnt, total;
};

__host__ __device__ inline TomeWorkspace tome_workspace(long long B, long long Ns, long long Nd, long long C) {
  TomeWorkspace w;
  w.msrc = 0;
  w.mdst = tome_align(w.msrc + static_cast<size_t>(B * Ns * C * 2));
  w.nmax = tome_align(w.mdst + static_cast<size_t>(B * Nd * C * 2));
  w.nidx = tome_align(w.nmax + static_cast<size_t>(B * Ns * 4));
  w.cnt = tome_align(w.nidx + static_cast<size_t>(B * Ns * 4));
  w.total = tome_align(w.cnt + static_cast<size_t>(B * Nd * 4));
  return w;
}

// token of src index a: every pair of rows (2p, 2p+1) holds w/2 src tokens of the even row (odd x) then w of the odd row
__device__ __forceinline__ int tome_src_token(int a, int w) {
  const int per = w + w / 2;
  const int p = a / per, rem = a - p * per;
  return rem < w / 2 ? (2 * p) * w + 2 * rem + 1 : (2 * p + 1) * w + (rem - w / 2);
}

// ---------------------------------------------------------------------------------------------- 1. normalise + gather
// one warp per token; C % 8 == 0
__global__ void tome_normalize_kernel(const __half* __restrict__ X, long long pitch, TomeDims d, __half* __restrict__ msrc,
                                      __half* __restrict__ mdst) {
  const long long gw = (blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (gw >= static_cast<long long>(d.B) * d.N) return;
  const int b = static_cast<int>(gw / d.N), t = static_cast<int>(gw - static_cast<long long>(b) * d.N);
  const int y = t / d.W, x = t - y * d.W;
  const uint4* row = reinterpret_cast<const uint4*>(X + (static_cast<long long>(b) * d.N + t) * pitch);
  const int nv = d.C / 8;
  float ss = 0.f;
  for (int v = lane; v < nv; v += 32) {
    uint4 u = row[v];
    const __half2* h = reinterpret_cast<const __half2*>(&u);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 f = __half22float2(h[i]);
      ss = fmaf(f.x, f.x, ss);
      ss = fmaf(f.y, f.y, ss);
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
  const float nrm = __half2float(__float2half_rn(sqrtf(ss)));   // ||x|| in the model dtype
  __half* dst;
  if ((y & 1) == 0 && (x & 1) == 0) {
    dst = mdst + (static_cast<long long>(b) * d.Nd + (y / 2) * (d.W / 2) + x / 2) * d.C;
  } else {
    const int a = t - ((y + 1) / 2) * (d.W / 2) - ((y & 1) == 0 ? (x + 1) / 2 : 0);
    dst = msrc + (static_cast<long long>(b) * d.Ns + a) * d.C;
  }
  uint4* out = reinterpret_cast<uint4*>(dst);
  for (int v = lane; v < nv; v += 32) {
    uint4 u = row[v];
    __half2* h = reinterpret_cast<__half2*>(&u);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 f = __half22float2(h[i]);
      h[i] = __floats2half2_rn(f.x / nrm, f.y / nrm);
    }
    out[v] = u;
  }
}

// ---------------------------------------------------------------------------------------------- 2. fused argmax
struct __align__(8) TomeShared {
  uint64_t src_full;
  uint64_t full[kTomeMaxStages];
  uint64_t empty[kTomeMaxStages];   // one arrival per math warpgroup
};

template <int kChunks>
__device__ __forceinline__ void tome_scores(float (&s)[kTomeDstTile / 2], uint64_t da, uint64_t db) {
#pragma unroll
  for (int ks = 0; ks < 4 * kChunks; ++ks) {
    const uint32_t off = static_cast<uint32_t>(ks & 3) * 32u;
    Wgmma<kTomeDstTile, false>::ss(s, da + ((static_cast<uint32_t>(ks >> 2) * kTomeSrcChunkBytes + off) >> 4),
                                   db + ((static_cast<uint32_t>(ks >> 2) * kTomeDstChunkBytes + off) >> 4),
                                   ks != 0 ? 1u : 0u);
  }
}

template <int kChunks>
__global__ void __launch_bounds__(kTomeThreads, 1)
tome_argmax_kernel(const __grid_constant__ CUtensorMap tmS, const __grid_constant__ CUtensorMap tmD, TomeDims d,
                   int stages, float* __restrict__ nmax, int* __restrict__ nidx) {
  constexpr uint32_t kStageBytes = kChunks * kTomeDstChunkBytes;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sS = smem;
  uint8_t* sD = sS + kChunks * kTomeSrcChunkBytes;
  TomeShared* sh = reinterpret_cast<TomeShared*>(sD + stages * kStageBytes);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int st = blockIdx.x, b = blockIdx.y;
  const int ntiles = (d.Nd + kTomeDstTile - 1) / kTomeDstTile;

  if (threadIdx.x == kTomeMathThreads) {
    tma_prefetch_desc(&tmS);
    tma_prefetch_desc(&tmD);
    mbar_init(&sh->src_full, 1);
    for (int s = 0; s < kTomeMaxStages; ++s) {
      mbar_init(&sh->full[s], 1);
      mbar_init(&sh->empty[s], kTomeMathThreads / 128);
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (warp == kTomeMathThreads / 32) {   // producer
    if (lane == 0) {
      mbar_arrive_expect_tx(&sh->src_full, kChunks * kTomeSrcChunkBytes);
#pragma unroll
      for (int c = 0; c < kChunks; ++c)
        tma_load_3d(sS + c * kTomeSrcChunkBytes, &tmS, &sh->src_full, c * 64, st * kTomeSrcTile, b);
      for (int t = 0; t < ntiles; ++t) {
        const int s = t % stages;
        if (t >= stages) mbar_wait(&sh->empty[s], static_cast<uint32_t>(t / stages - 1) & 1u);
        mbar_arrive_expect_tx(&sh->full[s], kStageBytes);
#pragma unroll
        for (int c = 0; c < kChunks; ++c)
          tma_load_3d(sD + s * kStageBytes + c * kTomeDstChunkBytes, &tmD, &sh->full[s], c * 64, t * kTomeDstTile, b);
      }
    }
    return;
  }

  const int wg = warp >> 2;
  const int colq = (lane & 3) * 2;
  const uint64_t da = make_gdesc_sw128(smem_u32(sS) + static_cast<uint32_t>(wg) * 8192u, 16, 1024);
  float acc[kTomeDstTile / 2];
  float best[2] = {-INFINITY, -INFINITY};
  int arg[2] = {0, 0};
  mbar_wait(&sh->src_full, 0);
  for (int t = 0; t < ntiles; ++t) {
    const int s = t % stages;
    mbar_wait(&sh->full[s], static_cast<uint32_t>(t / stages) & 1u);
    wgmma_fence();
    tome_scores<kChunks>(acc, da, make_gdesc_sw128(smem_u32(sD + s * kStageBytes), 16, 1024));
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(acc);
    if ((threadIdx.x & 127) == 0) mbar_arrive(&sh->empty[s]);
    // columns in ascending order per thread: a strict > keeps the lowest index of equal maxima
#pragma unroll
    for (int g = 0; g < kTomeDstTile / 8; ++g)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int col = t * kTomeDstTile + 8 * g + colq + e;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const float v = acc[4 * g + 2 * h + e];
          if (col < d.Nd && v > best[h]) {
            best[h] = v;
            arg[h] = col;
          }
        }
      }
  }
  // the four threads of a row: largest value, lowest index among equal ones
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int o = 1; o <= 2; o <<= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, best[h], o);
      const int oi = __shfl_xor_sync(0xffffffffu, arg[h], o);
      if (ov > best[h] || (ov == best[h] && oi < arg[h])) {
        best[h] = ov;
        arg[h] = oi;
      }
    }
  if ((lane & 3) == 0) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = st * kTomeSrcTile + wg * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * h;
      if (row < d.Ns) {
        nmax[static_cast<long long>(b) * d.Ns + row] = best[h];
        nidx[static_cast<long long>(b) * d.Ns + row] = arg[h];
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------- 3. select + partition
// order-preserving image of a float in uint32
__device__ __forceinline__ uint32_t tome_ord(float f) {
  const uint32_t u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

// exclusive block scan of v (blockDim.x == kTomeSelectThreads); *total = the block's sum
__device__ __forceinline__ int tome_block_scan(int v, int* sh, int* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int incl = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int n = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += n;
  }
  if (lane == 31) sh[warp] = incl;
  __syncthreads();
  if (warp == 0) {
    int w = sh[lane];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int n = __shfl_up_sync(0xffffffffu, w, o);
      if (lane >= o) w += n;
    }
    sh[lane] = w;
  }
  __syncthreads();
  const int res = incl - v + (warp > 0 ? sh[warp - 1] : 0);
  *total = sh[31];
  __syncthreads();
  return res;
}

__global__ void __launch_bounds__(kTomeSelectThreads)
tome_select_kernel(TomeDims d, const float* __restrict__ nmax_all, const int* __restrict__ nidx_all, int* cnt_all,
                   int* slot_all, int* members_all, int* seg_all) {
  __shared__ int hist[256];
  __shared__ int scan_sh[32];
  __shared__ int pick[2];
  const int b = blockIdx.x, tid = threadIdx.x;
  const int Ns = d.Ns, Nd = d.Nd, N = d.N, r = d.r, Nm = N - r, m0 = Ns - r;
  const float* nmax = nmax_all + static_cast<long long>(b) * Ns;
  const int* nidx = nidx_all + static_cast<long long>(b) * Ns;
  int* cnt = cnt_all + static_cast<long long>(b) * Nd;
  int* slot = slot_all + static_cast<long long>(b) * N;
  int* members = members_all + static_cast<long long>(b) * N;
  int* seg = seg_all + static_cast<long long>(b) * (Nm + 1);

  // radix select: V = the r-th largest key, k = how many of the keys equal to V are taken
  uint32_t prefix = 0, mask = 0;
  int k = r;
  for (int shift = 24; shift >= 0; shift -= 8) {
    if (tid < 256) hist[tid] = 0;
    __syncthreads();
    for (int a = tid; a < Ns; a += kTomeSelectThreads) {
      const uint32_t u = tome_ord(nmax[a]);
      if ((u & mask) == prefix) atomicAdd(&hist[(u >> shift) & 255u], 1);
    }
    __syncthreads();
    if (tid == 0) {
      int cum = 0, dg = 0;
      for (dg = 255; dg > 0; --dg) {
        if (cum + hist[dg] >= k) break;
        cum += hist[dg];
      }
      pick[0] = dg;
      pick[1] = k - cum;
    }
    __syncthreads();
    prefix |= static_cast<uint32_t>(pick[0]) << shift;
    mask |= 0xFFu << shift;
    k = pick[1];
    __syncthreads();
  }
  for (int j = tid; j < Nd; j += kTomeSelectThreads) {
    cnt[j] = 1;
    slot[(2 * (j / (d.W / 2))) * d.W + 2 * (j % (d.W / 2))] = m0 + j;
  }
  __syncthreads();
  // src tokens in index order: the first k ties are merged; the unmerged ones take slots 0.. in order
  int tie_carry = 0, unm_carry = 0;
  for (int base = 0; base < Ns; base += kTomeSelectThreads) {
    const int a = base + tid;
    const uint32_t u = a < Ns ? tome_ord(nmax[a]) : 0u;
    const bool tie = a < Ns && u == prefix;
    int tot;
    const int trank = tome_block_scan(tie ? 1 : 0, scan_sh, &tot) + tie_carry;
    tie_carry += tot;
    const bool sel = a < Ns && (u > prefix || (tie && trank < k));
    const bool unm = a < Ns && !sel;
    const int urank = tome_block_scan(unm ? 1 : 0, scan_sh, &tot) + unm_carry;
    unm_carry += tot;
    if (a < Ns) {
      const int tok = tome_src_token(a, d.W);
      if (sel) {
        const int j = nidx[a];
        slot[tok] = m0 + j;
        atomicAdd(&cnt[j], 1);
      } else {
        slot[tok] = urank;
        members[urank] = tok;
        seg[urank] = urank;
      }
    }
  }
  __syncthreads();
  // dst segments: starts by an exclusive scan of the counts; cnt becomes each segment's write cursor
  int carry = m0;
  for (int base = 0; base < Nd; base += kTomeSelectThreads) {
    const int j = base + tid;
    const int c = j < Nd ? cnt[j] : 0;
    int tot;
    const int start = tome_block_scan(c, scan_sh, &tot) + carry;
    carry += tot;
    if (j < Nd) {
      seg[m0 + j] = start;
      cnt[j] = start;
    }
  }
  if (tid == 0) seg[Nm] = N;
  __syncthreads();
  // members of the dst segments in ascending token order: one warp walks the tokens 32 at a time
  if (tid < 32) {
    for (int base = 0; base < N; base += 32) {
      const int t = base + tid;
      const int s = t < N ? slot[t] : -1;
      const int key = s >= m0 ? s - m0 : -1;
      const unsigned peers = __match_any_sync(0xffffffffu, key);
      int pos = 0;
      if (key >= 0) pos = cnt[key] + __popc(peers & ((1u << tid) - 1u));
      __syncwarp();
      if (key >= 0) {
        members[pos] = t;
        if ((__ffs(peers) - 1) == tid) cnt[key] += __popc(peers);
      }
      __syncwarp();
    }
  }
}

// ---------------------------------------------------------------------------------------------- merge / unmerge
// one thread per (slot, 8 channels)
__global__ void tome_merge_kernel(const __half* __restrict__ X, long long px, const int* __restrict__ members,
                                  const int* __restrict__ seg, __half* __restrict__ Y, long long py, int N, int Nm, int C) {
  const int cv = C / 8;
  const long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  const int b = blockIdx.y;
  if (i >= static_cast<long long>(Nm) * cv) return;
  const int s = static_cast<int>(i / cv), v = static_cast<int>(i - static_cast<long long>(s) * cv);
  const int* mem = members + static_cast<long long>(b) * N;
  const int* sg = seg + static_cast<long long>(b) * (Nm + 1);
  const int beg = sg[s], end = sg[s + 1];
  float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  for (int m = beg; m < end; ++m) {
    const uint4 u = *reinterpret_cast<const uint4*>(X + (static_cast<long long>(b) * N + mem[m]) * px + 8 * v);
    const __half2* h = reinterpret_cast<const __half2*>(&u);
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float2 f = __half22float2(h[e]);
      acc[2 * e] += f.x;
      acc[2 * e + 1] += f.y;
    }
  }
  const float n = static_cast<float>(end - beg);
  uint4 o;
  __half2* oh = reinterpret_cast<__half2*>(&o);
#pragma unroll
  for (int e = 0; e < 4; ++e) oh[e] = __floats2half2_rn(acc[2 * e] / n, acc[2 * e + 1] / n);
  *reinterpret_cast<uint4*>(Y + (static_cast<long long>(b) * Nm + s) * py + 8 * v) = o;
}

// one thread per (token, 8 channels)
__global__ void tome_unmerge_add_kernel(const __half* __restrict__ R, long long pr, const __half* __restrict__ Y,
                                        long long py, const int* __restrict__ slot, __half* __restrict__ O, long long po,
                                        int N, int Nm, int C) {
  const int cv = C / 8;
  const long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  const int b = blockIdx.y;
  if (i >= static_cast<long long>(N) * cv) return;
  const int t = static_cast<int>(i / cv), v = static_cast<int>(i - static_cast<long long>(t) * cv);
  const int s = slot[static_cast<long long>(b) * N + t];
  const uint4 ru = *reinterpret_cast<const uint4*>(R + (static_cast<long long>(b) * N + t) * pr + 8 * v);
  const uint4 yu = *reinterpret_cast<const uint4*>(Y + (static_cast<long long>(b) * Nm + s) * py + 8 * v);
  const __half2* rh = reinterpret_cast<const __half2*>(&ru);
  const __half2* yh = reinterpret_cast<const __half2*>(&yu);
  uint4 o;
  __half2* oh = reinterpret_cast<__half2*>(&o);
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    const float2 a = __half22float2(rh[e]), c = __half22float2(yh[e]);
    oh[e] = __floats2half2_rn(a.x + c.x, a.y + c.y);
  }
  *reinterpret_cast<uint4*>(O + (static_cast<long long>(b) * N + t) * po + 8 * v) = o;
}

// ---------------------------------------------------------------------------------------------- host
typedef void (*TomeArgmaxKernel)(CUtensorMap, CUtensorMap, TomeDims, int, float*, int*);

static TomeArgmaxKernel tome_argmax_for(int chunks) {
  switch (chunks) {
    case 1: return tome_argmax_kernel<1>;
    case 5: return tome_argmax_kernel<5>;
    default: return nullptr;
  }
}

static int g_tome_max_smem[64] = {};

static bool tome_shape_ok(int B, int H, int W, int C) {
  return B > 0 && H > 0 && W > 0 && H % 2 == 0 && W % 2 == 0 && (C == 64 || C == 320) &&
         static_cast<long long>(H) * W <= (1 << 24);
}

static bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

}  // namespace b200sd

using namespace b200sd;

extern "C" long long b200sd_tome_match_workspace_bytes(int B, int H, int W, int C) {
  if (!tome_shape_ok(B, H, W, C)) return -1;
  const long long N = static_cast<long long>(H) * W, Nd = N / 4;
  return static_cast<long long>(tome_workspace(B, N - Nd, Nd, C).total);
}

extern "C" int b200sd_tome_match(const void* X, long long pitch, int B, int H, int W, int C, int r, int* slot,
                                 int* members, int* seg, void* workspace, long long workspace_bytes, int dtype,
                                 void* stream) {
  if (dtype == B200SD_BF16) return B200SD_ERR_UNSUPPORTED;   // merging runs on the fp16 (SD1.x / SD 2.x) UNets only
  if (dtype != B200SD_F16) return B200SD_ERR_INVALID;
  if (!tome_shape_ok(B, H, W, C)) return (H % 2 || W % 2 || B <= 0 || H <= 0 || W <= 0) ? B200SD_ERR_INVALID
                                                                                        : B200SD_ERR_UNSUPPORTED;
  TomeDims d{};
  d.B = B; d.H = H; d.W = W; d.C = C;
  d.N = H * W; d.Nd = d.N / 4; d.Ns = d.N - d.Nd; d.r = r;
  if (r < 1 || r > d.Ns) return B200SD_ERR_INVALID;
  if (pitch < C || pitch % 8 || !aligned16(X) || !aligned16(workspace) || !slot || !members || !seg)
    return B200SD_ERR_INVALID;
  const TomeWorkspace ws = tome_workspace(B, d.Ns, d.Nd, C);
  if (workspace_bytes < static_cast<long long>(ws.total)) return B200SD_ERR_INVALID;
  uint8_t* w8 = static_cast<uint8_t*>(workspace);
  __half* msrc = reinterpret_cast<__half*>(w8 + ws.msrc);
  __half* mdst = reinterpret_cast<__half*>(w8 + ws.mdst);
  float* nmax = reinterpret_cast<float*>(w8 + ws.nmax);
  int* nidx = reinterpret_cast<int*>(w8 + ws.nidx);
  int* cnt = reinterpret_cast<int*>(w8 + ws.cnt);
  const int chunks = C / 64;
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return B200SD_ERR_CUDA;
  if (dev < 0 || dev >= 64) return B200SD_ERR_UNSUPPORTED;
  if (!g_tome_max_smem[dev]) {   // per-device opt-in to large dynamic smem; the first call must be outside capture
    int smem = 0;
    if (cudaDeviceGetAttribute(&smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev) != cudaSuccess) return B200SD_ERR_CUDA;
    for (int c : {1, 5})
      if (cudaFuncSetAttribute(tome_argmax_for(c), cudaFuncAttributeMaxDynamicSharedMemorySize, smem) != cudaSuccess)
        return B200SD_ERR_CUDA;
    g_tome_max_smem[dev] = smem;
  }
  const size_t fixed = 1024 + static_cast<size_t>(chunks) * kTomeSrcChunkBytes + sizeof(TomeShared);
  const size_t stage = static_cast<size_t>(chunks) * kTomeDstChunkBytes;
  const int ntiles = (d.Nd + kTomeDstTile - 1) / kTomeDstTile;
  int stages = static_cast<int>((static_cast<size_t>(g_tome_max_smem[dev]) - fixed) / stage);
  stages = stages < kTomeMaxStages ? stages : kTomeMaxStages;
  stages = stages < ntiles ? stages : ntiles;
  if (stages < 1) return B200SD_ERR_UNSUPPORTED;
  CUtensorMap tmS, tmD;
  const uint32_t es[3] = {1, 1, 1};
  int rc;
  {
    const uint64_t dims[3] = {static_cast<uint64_t>(C), static_cast<uint64_t>(d.Ns), static_cast<uint64_t>(B)};
    const uint64_t st[2] = {static_cast<uint64_t>(C) * 2, static_cast<uint64_t>(C) * 2 * d.Ns};
    const uint32_t box[3] = {64, kTomeSrcTile, 1};
    if ((rc = make_tmap_sw128(&tmS, msrc, 3, dims, st, box, es)) != B200SD_OK) return rc;
  }
  {
    const uint64_t dims[3] = {static_cast<uint64_t>(C), static_cast<uint64_t>(d.Nd), static_cast<uint64_t>(B)};
    const uint64_t st[2] = {static_cast<uint64_t>(C) * 2, static_cast<uint64_t>(C) * 2 * d.Nd};
    const uint32_t box[3] = {64, kTomeDstTile, 1};
    if ((rc = make_tmap_sw128(&tmD, mdst, 3, dims, st, box, es)) != B200SD_OK) return rc;
  }
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const long long warps = static_cast<long long>(B) * d.N;
  tome_normalize_kernel<<<static_cast<unsigned>((warps * 32 + 255) / 256), 256, 0, s>>>(
      static_cast<const __half*>(X), pitch, d, msrc, mdst);
  tome_argmax_for(chunks)<<<dim3((d.Ns + kTomeSrcTile - 1) / kTomeSrcTile, B), kTomeThreads,
                            fixed + static_cast<size_t>(stages) * stage, s>>>(tmS, tmD, d, stages, nmax, nidx);
  tome_select_kernel<<<B, kTomeSelectThreads, 0, s>>>(d, nmax, nidx, cnt, slot, members, seg);
  return cudaGetLastError() == cudaSuccess ? B200SD_OK : B200SD_ERR_CUDA;
}

extern "C" int b200sd_tome_merge(const void* X, long long pitch_x, const int* members, const int* seg, void* Y,
                                 long long pitch_y, int B, int N, int Nm, int C, int dtype, void* stream) {
  if (dtype == B200SD_BF16) return B200SD_ERR_UNSUPPORTED;
  if (dtype != B200SD_F16) return B200SD_ERR_INVALID;
  if (B <= 0 || N <= 0 || Nm <= 0 || Nm > N || C <= 0 || C % 8 || pitch_x < C || pitch_y < C || pitch_x % 8 ||
      pitch_y % 8 || !aligned16(X) || !aligned16(Y))
    return B200SD_ERR_INVALID;
  const long long n = static_cast<long long>(Nm) * (C / 8);
  tome_merge_kernel<<<dim3(static_cast<unsigned>((n + 255) / 256), B), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const __half*>(X), pitch_x, members, seg, static_cast<__half*>(Y), pitch_y, N, Nm, C);
  return cudaGetLastError() == cudaSuccess ? B200SD_OK : B200SD_ERR_CUDA;
}

extern "C" int b200sd_tome_unmerge_add(const void* R, long long pitch_r, const void* Y, long long pitch_y,
                                       const int* slot, void* out, long long pitch_o, int B, int N, int Nm, int C,
                                       int dtype, void* stream) {
  if (dtype == B200SD_BF16) return B200SD_ERR_UNSUPPORTED;
  if (dtype != B200SD_F16) return B200SD_ERR_INVALID;
  if (B <= 0 || N <= 0 || Nm <= 0 || Nm > N || C <= 0 || C % 8 || pitch_r < C || pitch_y < C || pitch_o < C ||
      pitch_r % 8 || pitch_y % 8 || pitch_o % 8 || !aligned16(R) || !aligned16(Y) || !aligned16(out))
    return B200SD_ERR_INVALID;
  const long long n = static_cast<long long>(N) * (C / 8);
  tome_unmerge_add_kernel<<<dim3(static_cast<unsigned>((n + 255) / 256), B), 256, 0,
                            static_cast<cudaStream_t>(stream)>>>(static_cast<const __half*>(R), pitch_r,
                                                                 static_cast<const __half*>(Y), pitch_y, slot,
                                                                 static_cast<__half*>(out), pitch_o, N, Nm, C);
  return cudaGetLastError() == cudaSuccess ? B200SD_OK : B200SD_ERR_CUDA;
}
