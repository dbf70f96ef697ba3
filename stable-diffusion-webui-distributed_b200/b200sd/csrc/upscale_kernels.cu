// upscale_kernels.cu — the hires fix's upscalers around the tensor-core convolutions: Pillow-exact uint8 resampling
// (LANCZOS / NEAREST), sdwui's tile blend (images.combine_grid), ESRGAN's output quantiser and RRDB residual, and the
// table-driven latent resize of the "Latent (...)" modes.
//
// Upstream: Pillow ImagingResample (Resample.c) and paste with an "L" mask (Paste.c); sdwui images.resize_image,
// split_grid / combine_grid, upscaler_utils.upscale_pil_patch; basicsr RRDBNet; torch.nn.functional.interpolate.
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include "../../../include/b200sd.h"

namespace b200sd {
namespace {

constexpr int kPillowPrecisionBits = 22;  // Resample.c: PRECISION_BITS = 32 - 8 - 2

// one resampling pass of Pillow's ImagingResample on RGB uint8 [B, H, W, 3]: along x (horizontal) or y (vertical).
// Output position o reads `bounds[2o+1]` input positions from bounds[2o] with the fixed-point weights kk[o * ksize + k];
// the sum starts at 1 << 21 and the result is clip8(sum >> 22), as ImagingResampleHorizontal_8bpc / Vertical_8bpc.
template <bool kVertical>
__global__ void resample_u8_kernel(const uint8_t* __restrict__ in, uint8_t* __restrict__ out, int B, int Hin, int Win,
                                   int Hout, int Wout, const int* __restrict__ bounds, const int* __restrict__ kk,
                                   int ksize) {
  const long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  const long long n = static_cast<long long>(B) * Hout * Wout;
  if (i >= n) return;
  const int x = static_cast<int>(i % Wout), y = static_cast<int>((i / Wout) % Hout);
  const long long b = i / (static_cast<long long>(Wout) * Hout);
  const int o = kVertical ? y : x;
  const int first = bounds[2 * o], count = bounds[2 * o + 1];
  const int* k = kk + static_cast<long long>(o) * ksize;
  const uint8_t* src = in + (kVertical ? (b * Hin * Win + x) : ((b * Hin + y) * Win)) * 3;
  const long long step = kVertical ? static_cast<long long>(Win) * 3 : 3;
  int s0 = 1 << (kPillowPrecisionBits - 1), s1 = s0, s2 = s0;
  for (int t = 0; t < count; ++t) {
    const uint8_t* px = src + (first + t) * step;
    s0 += px[0] * k[t];
    s1 += px[1] * k[t];
    s2 += px[2] * k[t];
  }
  uint8_t* dst = out + i * 3;
  dst[0] = static_cast<uint8_t>(min(max(s0 >> kPillowPrecisionBits, 0), 255));
  dst[1] = static_cast<uint8_t>(min(max(s1 >> kPillowPrecisionBits, 0), 255));
  dst[2] = static_cast<uint8_t>(min(max(s2 >> kPillowPrecisionBits, 0), 255));
}

// Pillow's BLEND(a, out, in) of paste(..., mask=L): DIV255(out * (255 - a) + in * a), DIV255(v) = ((v+128 >> 8) + v+128) >> 8
__device__ __forceinline__ int blend255(int a, int under, int over) {
  const int t = under * (255 - a) + over * a + 128;
  return ((t >> 8) + t) >> 8;
}

// sdwui images.combine_grid on upscaled tiles [B * rows * cols, th, tw, 3]: tile (r, c) of image b lands at
// (xs[c], ys[r]).  Within a row, every tile but one at x == 0 is pasted with its first `ov` columns blended over what
// is there through mask[column]; the rows are then stacked the same way through mask[row].  Evaluated per output pixel in
// paste order, so one launch replaces the sequence of pastes.
__global__ void combine_tiles_u8_kernel(const uint8_t* __restrict__ tiles, uint8_t* __restrict__ out, int B, int H, int W,
                                        int th, int tw, int rows, int cols, const int* __restrict__ ys,
                                        const int* __restrict__ xs, const uint8_t* __restrict__ mask, int ov) {
  const long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  const long long n = static_cast<long long>(B) * H * W;
  if (i >= n) return;
  const int X = static_cast<int>(i % W), Y = static_cast<int>((i / W) % H);
  const long long b = i / (static_cast<long long>(W) * H);
  int v[3] = {0, 0, 0};
  for (int r = 0; r < rows; ++r) {
    const int y0 = ys[r];
    if (Y < y0 || Y >= y0 + th) continue;
    const int yy = Y - y0;
    int u[3] = {0, 0, 0};  // the combined row at (yy, X): starts black
    for (int c = 0; c < cols; ++c) {
      const int x0 = xs[c];
      if (X < x0 || X >= x0 + tw) continue;
      const int xx = X - x0;
      const uint8_t* t = tiles + ((((b * rows + r) * cols + c) * th + yy) * static_cast<long long>(tw) + xx) * 3;
      for (int ch = 0; ch < 3; ++ch) u[ch] = (x0 != 0 && xx < ov) ? blend255(mask[xx], u[ch], t[ch]) : t[ch];
    }
    for (int ch = 0; ch < 3; ++ch) v[ch] = (y0 != 0 && yy < ov) ? blend255(mask[yy], v[ch], u[ch]) : u[ch];
  }
  uint8_t* dst = out + i * 3;
  dst[0] = static_cast<uint8_t>(v[0]);
  dst[1] = static_cast<uint8_t>(v[1]);
  dst[2] = static_cast<uint8_t>(v[2]);
}

// network output fp16 [B, HW, pitch] (channels 0..2 in [0, 1] nominal) -> uint8 round(255 * clamp(v, 0, 1)), half to
// even (sdwui torch_bgr_to_pil_image: clamp, x 255, numpy round, astype uint8)
__global__ void quantize_unit_u8_kernel(const __half* img, long long pitch, uint8_t* out, long long npix) {
  const long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (i >= npix) return;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float v = fminf(fmaxf(__half2float(img[i * pitch + c]), 0.f), 1.f);
    out[i * 3 + c] = static_cast<uint8_t>(rintf(__fmul_rn(255.f, v)));
  }
}

// Y[r, c] = Y[r, c] + alpha * X[r, c], fp16 storage, fp32 math (basicsr RRDB: out * 0.2 + x)
__global__ void scaled_add_kernel(const __half* X, long long pitch_x, __half* Y, long long pitch_y, long long rows, int C,
                                  float alpha) {
  const long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (i >= rows * C) return;
  const long long r = i / C;
  const int c = static_cast<int>(i % C);
  Y[r * pitch_y + c] = __float2half_rn(__fmaf_rn(alpha, __half2float(X[r * pitch_x + c]), __half2float(Y[r * pitch_y + c])));
}

// y[b, oy, ox] = sum_j wy[oy, j] * (sum_i wx[ox, i] * x[b, iy[oy, j], ix[ox, i]]) on fp32 NHWC latents [B, H*W, 4]:
// each output row's horizontal sums first, then the vertical one, in tap order (torch's separable interpolation)
__global__ void resize_latent_table_kernel(const float4* __restrict__ x, float4* __restrict__ y, int B, int H, int W,
                                           int Ho, int Wo, const int* __restrict__ ix, const float* __restrict__ wx,
                                           int kx, const int* __restrict__ iy, const float* __restrict__ wy, int ky) {
  const long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  const long long n = static_cast<long long>(B) * Ho * Wo;
  if (i >= n) return;
  const int xo = static_cast<int>(i % Wo), yo = static_cast<int>((i / Wo) % Ho);
  const long long b = i / (static_cast<long long>(Wo) * Ho);
  const float4* img = x + b * H * W;
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int j = 0; j < ky; ++j) {
    const float4* row = img + static_cast<long long>(iy[yo * ky + j]) * W;
    const float4 p0 = row[ix[xo * kx]];
    const float w0 = wx[xo * kx];
    float4 h = make_float4(p0.x * w0, p0.y * w0, p0.z * w0, p0.w * w0);
    for (int t = 1; t < kx; ++t) {
      const float4 p = row[ix[xo * kx + t]];
      const float w = wx[xo * kx + t];
      h.x += p.x * w; h.y += p.y * w; h.z += p.z * w; h.w += p.w * w;
    }
    const float v = wy[yo * ky + j];
    if (j == 0) acc = make_float4(h.x * v, h.y * v, h.z * v, h.w * v);
    else { acc.x += h.x * v; acc.y += h.y * v; acc.z += h.z * v; acc.w += h.w * v; }
  }
  y[i] = acc;
}

inline int blocks_for(long long n) { return static_cast<int>((n + 255) / 256); }

}  // namespace
}  // namespace b200sd

using namespace b200sd;
#define ST(s) static_cast<cudaStream_t>(s)
#define RET_LAUNCH() return cudaGetLastError() == cudaSuccess ? B200SD_OK : B200SD_ERR_CUDA

extern "C" int b200sd_resample_u8(const unsigned char* in, unsigned char* out, int B, int Hin, int Win, int Hout,
                                  int Wout, int vertical, const int* bounds, const int* kk, int ksize, void* stream) {
  if (B <= 0) return B200SD_OK;
  if (Hin <= 0 || Win <= 0 || Hout <= 0 || Wout <= 0 || ksize <= 0 || !bounds || !kk) return B200SD_ERR_INVALID;
  if (vertical ? Wout != Win : Hout != Hin) return B200SD_ERR_INVALID;
  const long long n = static_cast<long long>(B) * Hout * Wout;
  if (vertical) resample_u8_kernel<true><<<blocks_for(n), 256, 0, ST(stream)>>>(in, out, B, Hin, Win, Hout, Wout, bounds, kk, ksize);
  else resample_u8_kernel<false><<<blocks_for(n), 256, 0, ST(stream)>>>(in, out, B, Hin, Win, Hout, Wout, bounds, kk, ksize);
  RET_LAUNCH();
}

extern "C" int b200sd_combine_tiles_u8(const unsigned char* tiles, unsigned char* out, int B, int H, int W, int th,
                                       int tw, int rows, int cols, const int* ys, const int* xs,
                                       const unsigned char* mask, int overlap, void* stream) {
  if (B <= 0) return B200SD_OK;
  if (H <= 0 || W <= 0 || th <= 0 || tw <= 0 || rows <= 0 || cols <= 0 || overlap < 0 || !ys || !xs ||
      (overlap > 0 && !mask))
    return B200SD_ERR_INVALID;
  const long long n = static_cast<long long>(B) * H * W;
  combine_tiles_u8_kernel<<<blocks_for(n), 256, 0, ST(stream)>>>(tiles, out, B, H, W, th, tw, rows, cols, ys, xs, mask,
                                                                  overlap);
  RET_LAUNCH();
}

extern "C" int b200sd_quantize_unit_u8(const void* img, long long pitch, unsigned char* out, int B, int HW, int dtype,
                                       void* stream) {
  if (B <= 0 || HW <= 0) return B200SD_OK;
  if (dtype != B200SD_F16) return B200SD_ERR_UNSUPPORTED;
  if (pitch < 3) return B200SD_ERR_INVALID;
  const long long n = static_cast<long long>(B) * HW;
  quantize_unit_u8_kernel<<<blocks_for(n), 256, 0, ST(stream)>>>(static_cast<const __half*>(img), pitch, out, n);
  RET_LAUNCH();
}

extern "C" int b200sd_scaled_add(const void* X, long long pitch_x, void* Y, long long pitch_y, long long rows, int C,
                                 float alpha, int dtype, void* stream) {
  if (rows <= 0 || C <= 0) return B200SD_OK;
  if (dtype != B200SD_F16) return B200SD_ERR_UNSUPPORTED;
  if (pitch_x < C || pitch_y < C) return B200SD_ERR_INVALID;
  scaled_add_kernel<<<blocks_for(rows * C), 256, 0, ST(stream)>>>(static_cast<const __half*>(X), pitch_x,
                                                                  static_cast<__half*>(Y), pitch_y, rows, C, alpha);
  RET_LAUNCH();
}

extern "C" int b200sd_resize_latent_table(const float* x, float* y, int B, int H, int W, int Ho, int Wo, const int* ix,
                                          const float* wx, int kx, const int* iy, const float* wy, int ky,
                                          void* stream) {
  if (B <= 0) return B200SD_OK;
  if (H <= 0 || W <= 0 || Ho <= 0 || Wo <= 0 || kx <= 0 || ky <= 0 || !ix || !wx || !iy || !wy ||
      ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(y)) & 15))
    return B200SD_ERR_INVALID;
  const long long n = static_cast<long long>(B) * Ho * Wo;
  resize_latent_table_kernel<<<blocks_for(n), 256, 0, ST(stream)>>>(reinterpret_cast<const float4*>(x),
                                                                     reinterpret_cast<float4*>(y), B, H, W, Ho, Wo, ix,
                                                                     wx, kx, iy, wy, ky);
  RET_LAUNCH();
}
