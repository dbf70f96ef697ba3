// pad_kernels.cu — circular padding of NHWC activations for seamless tiling.
//
// sdwui's tiling option (model_hijack.apply_circular) sets padding_mode = 'circular' on every Conv2d of the model.
// The implicit-GEMM conv takes its zero padding from TMA's out-of-bounds fill, and TMA has no wrap mode: a circular
// 3x3 conv is this copy into a buffer p pixels larger on each side, then b200sd_conv2d with pad = pad_end = 0.
#include <cuda_runtime.h>
#include <stdint.h>
#include "../../../include/b200sd.h"
#include "pdl.cuh"

namespace b200sd {

// Y[n, yo, xo, :] = X[n, (yo - p) mod H, (xo - p) mod W, :] for yo < H + 2p, xo < W + 2p.  One CTA per output row
// (grid-stride over NB * (H + 2p) rows), its threads over the row's pixels x 16-byte channel vectors.  p <= H and
// p <= W, so one add or subtract of the extent wraps every index.
__global__ void pad_circular_kernel(const uint4* __restrict__ X, long long pitch_x_v, uint4* __restrict__ Y,
                                    long long pitch_y_v, int NB, int H, int W, int cvec, int p) {
  pdl_trigger();
  pdl_wait();
  const int Ho = H + 2 * p, Wo = W + 2 * p;
  const long long rows = static_cast<long long>(NB) * Ho;
  const int row_vecs = Wo * cvec;
  for (long long r = blockIdx.x; r < rows; r += gridDim.x) {
    const int n = static_cast<int>(r / Ho);
    int y = static_cast<int>(r - static_cast<long long>(n) * Ho) - p;
    y += y < 0 ? H : (y >= H ? -H : 0);
    const uint4* src = X + (static_cast<long long>(n) * H + y) * W * pitch_x_v;
    uint4* dst = Y + r * Wo * pitch_y_v;
    for (int i = threadIdx.x; i < row_vecs; i += blockDim.x) {
      const int xo = i / cvec;
      const int v = i - xo * cvec;
      int x = xo - p;
      x += x < 0 ? W : (x >= W ? -W : 0);
      dst[static_cast<long long>(xo) * pitch_y_v + v] = __ldg(&src[static_cast<long long>(x) * pitch_x_v + v]);
    }
  }
}

}  // namespace b200sd

using namespace b200sd;

extern "C" int b200sd_pad_circular(const void* X, long long pitch_x, void* Y, long long pitch_y, int NB, int H, int W,
                                   int C, int p, int dtype, void* stream) {
  if (dtype != B200SD_F16 && dtype != B200SD_BF16) return B200SD_ERR_INVALID;
  if (NB < 0 || H <= 0 || W <= 0 || C <= 0 || p < 0 || p > H || p > W) return B200SD_ERR_INVALID;
  if (C % 8 || pitch_x < C || pitch_y < C || pitch_x % 8 || pitch_y % 8 ||
      ((reinterpret_cast<uintptr_t>(X) | reinterpret_cast<uintptr_t>(Y)) & 15))
    return B200SD_ERR_INVALID;
  if (NB == 0) return B200SD_OK;
  long long blocks = static_cast<long long>(NB) * (H + 2 * p);
  if (blocks > kNumSms * 16) blocks = kNumSms * 16;
  launch_pdl(pad_circular_kernel, dim3(static_cast<int>(blocks)), dim3(256), 0, static_cast<cudaStream_t>(stream),
             static_cast<const uint4*>(X), pitch_x / 8, static_cast<uint4*>(Y), pitch_y / 8, NB, H, W, C / 8, p);
  return cudaGetLastError() == cudaSuccess ? B200SD_OK : B200SD_ERR_CUDA;
}
