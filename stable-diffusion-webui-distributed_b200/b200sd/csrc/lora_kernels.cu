// lora_kernels.cu — LoRA networks merged into the packed weights (sdwui's `<lora:name:te:unet>`, networks.py
// network_apply_weights): W = round(P + U . D) for every targeted weight tensor, from its pristine copy P.
// One persistent launch walks the output tiles of every descriptor in table order; a UNet has hundreds of targets and
// one launch per tensor would cost more in launch overhead than the update itself.  Register-tiled fp32 FMA, no tensor
// cores: at rank 32 a whole SD1.5 UNet is ~55 GFLOP against ~3.4 GB of pristine reads and weight writes, so the FLOP
// bound (fp32) and the byte bound are within a factor of two of each other, and the merge runs once per change of the
// network set, never per sampler step.
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include "../../../include/b200sd.h"

namespace b200sd {

constexpr int kLoraTM = 64;       // output rows per tile
constexpr int kLoraTN = 128;      // output columns per tile
constexpr int kLoraRC = 32;       // ranks staged in shared memory per pass
constexpr int kLoraThreads = 256; // 16 x 16 threads, each 4 rows x 8 columns

template <bool kBf16>
__device__ __forceinline__ float load_w(const void* p, long long i) {
  if constexpr (kBf16) return __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(p)[i]);
  else return __half2float(reinterpret_cast<const __half*>(p)[i]);
}

template <bool kBf16>
__device__ __forceinline__ void store_w(void* p, long long i, float v) {
  if constexpr (kBf16) reinterpret_cast<__nv_bfloat16*>(p)[i] = __float2bfloat16_rn(v);
  else reinterpret_cast<__half*>(p)[i] = __float2half_rn(v);
}

__device__ __forceinline__ long long lora_tiles(const b200sd_lora_target& t) {
  return static_cast<long long>((t.rows + kLoraTM - 1) / kLoraTM) * ((t.cols + kLoraTN - 1) / kLoraTN);
}

// Block b takes global tiles b, b + gridDim.x, ... in descriptor order; its cursor over the table only moves forward.
// Every output element is s = sum_j U[i,j] D[j,k] accumulated by fmaf in ascending j from 0 (the same sequence whatever
// the tiling or the grid), then W = round(P + s), or W = P bitwise where s == 0 (R = 0 restores, zero rows of U leave
// their row pristine, signed zeros included).
template <bool kBf16>
__global__ void __launch_bounds__(kLoraThreads) lora_merge_kernel(const b200sd_lora_target* __restrict__ targets,
                                                                  int n_targets) {
  __shared__ __align__(16) float us[kLoraRC][kLoraTM + 4];   // U chunk, transposed: us[j][row] (padded: 4-way writes)
  __shared__ __align__(16) float ds[kLoraRC][kLoraTN];   // D chunk: ds[j][col]
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  int d = 0;
  long long d_start = 0;   // global index of descriptor d's first tile
  long long d_tiles = n_targets > 0 ? lora_tiles(targets[0]) : 0;
  for (long long g = blockIdx.x;; g += gridDim.x) {
    while (d < n_targets && g >= d_start + d_tiles) {
      d_start += d_tiles;
      if (++d < n_targets) d_tiles = lora_tiles(targets[d]);
    }
    if (d >= n_targets) return;
    const b200sd_lora_target t = targets[d];
    const long long local = g - d_start;
    const int col_tiles = (t.cols + kLoraTN - 1) / kLoraTN;
    const int row0 = static_cast<int>(local / col_tiles) * kLoraTM;
    const int col0 = static_cast<int>(local % col_tiles) * kLoraTN;
    float acc[4][8];
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
      for (int c = 0; c < 8; ++c) acc[r][c] = 0.0f;
    for (int j0 = 0; j0 < t.R; j0 += kLoraRC) {
      const int rc = min(kLoraRC, t.R - j0);
      __syncthreads();   // the previous chunk (or tile) is consumed
      for (int e = threadIdx.x; e < kLoraRC * kLoraTM; e += kLoraThreads) {
        const int i = e / kLoraRC, j = e % kLoraRC;   // consecutive threads read consecutive ranks of one row
        const int row = row0 + i;
        us[j][i] = (j < rc && row < t.rows) ? t.U[static_cast<long long>(row) * t.R + j0 + j] : 0.0f;
      }
      for (int e = threadIdx.x; e < kLoraRC * kLoraTN; e += kLoraThreads) {
        const int j = e / kLoraTN, k = e % kLoraTN;
        const int col = col0 + k;
        ds[j][k] = (j < rc && col < t.cols) ? t.D[static_cast<long long>(j0 + j) * t.cols + col] : 0.0f;
      }
      __syncthreads();
      for (int j = 0; j < rc; ++j) {
        const float4 u = *reinterpret_cast<const float4*>(&us[j][ty * 4]);
        float dv[8];
#pragma unroll
        for (int c = 0; c < 8; ++c) dv[c] = ds[j][tx + 16 * c];
#pragma unroll
        for (int c = 0; c < 8; ++c) {
          acc[0][c] = fmaf(u.x, dv[c], acc[0][c]);
          acc[1][c] = fmaf(u.y, dv[c], acc[1][c]);
          acc[2][c] = fmaf(u.z, dv[c], acc[2][c]);
          acc[3][c] = fmaf(u.w, dv[c], acc[3][c]);
        }
      }
    }
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const int row = row0 + ty * 4 + r;
      if (row >= t.rows) continue;
      const long long base = static_cast<long long>(row) * t.ldw;
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        const int col = col0 + tx + 16 * c;
        if (col >= t.cols) continue;
        const float s = acc[r][c];
        if (s == 0.0f) {
          if constexpr (kBf16) reinterpret_cast<__nv_bfloat16*>(t.W)[base + col] =
              reinterpret_cast<const __nv_bfloat16*>(t.P)[base + col];
          else reinterpret_cast<__half*>(t.W)[base + col] = reinterpret_cast<const __half*>(t.P)[base + col];
        } else {
          store_w<kBf16>(t.W, base + col, load_w<kBf16>(t.P, base + col) + s);
        }
      }
    }
  }
}

}  // namespace b200sd

using namespace b200sd;

extern "C" int b200sd_lora_merge(const b200sd_lora_target* targets, int n_targets, int dtype, void* stream) {
  if (dtype != B200SD_F16 && dtype != B200SD_BF16) return B200SD_ERR_INVALID;
  if (n_targets < 0 || (n_targets > 0 && targets == nullptr)) return B200SD_ERR_INVALID;
  if (n_targets == 0) return B200SD_OK;
  static int sms = 0;
  if (sms == 0) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess)
      return B200SD_ERR_CUDA;
  }
  // 24 KB of shared memory and 256 threads per block: several blocks per SM hide the staging loads of the others
  const int blocks = 4 * sms;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (dtype == B200SD_BF16) lora_merge_kernel<true><<<blocks, kLoraThreads, 0, st>>>(targets, n_targets);
  else lora_merge_kernel<false><<<blocks, kLoraThreads, 0, st>>>(targets, n_targets);
  return cudaGetLastError() == cudaSuccess ? B200SD_OK : B200SD_ERR_CUDA;
}
