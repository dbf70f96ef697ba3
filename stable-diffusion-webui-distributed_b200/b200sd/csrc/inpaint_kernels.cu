// inpaint_kernels.cu — the image conditioning of 9-channel inpainting UNets (sd-v1-5-inpainting, 512-inpainting-ema,
// SDXL inpainting).  Such a UNet reads cat([x, mask, z_cond]): channel 4 is the inpainting mask at latent resolution,
// channels 5..8 the VAE latents of the masked init image (sdwui inpainting_image_conditioning / txt2img_image_conditioning).
// Both kernels run once per request; the per-step kernels write channels 0..3 of the UNet input only, so what is packed
// here stays in place through every step and graph replay.
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include "../../../include/b200sd.h"

namespace b200sd {

template <bool kBf16>
__device__ __forceinline__ void store_act(void* p, long long i, float v) {
  if constexpr (kBf16) reinterpret_cast<__nv_bfloat16*>(p)[i] = __float2bfloat16_rn(v);
  else reinterpret_cast<__half*>(p)[i] = __float2half_rn(v);
}

// channels 0..2 = (2x/255 - 1) * (1 - w [m >= 128]): torch.lerp(s, s * (1 - M), w) with M = round(m / 255).  The FMA is
// image_to_nhwc's own, so with M = 0 (k = 1 exactly) the output is bitwise that kernel's.
template <bool kBf16>
__global__ void masked_image_to_nhwc_kernel(const unsigned char* __restrict__ img, const unsigned char* __restrict__ mask,
                                            float weight, void* out, long long pitch, int HW, long long npix) {
  const long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (i >= npix) return;
  const bool m = mask == nullptr || mask[i % HW] >= 128;
  const float k = m ? 1.0f - weight : 1.0f;
#pragma unroll
  for (int c = 0; c < 3; ++c)
    store_act<kBf16>(out, i * pitch + c, __fmaf_rn(static_cast<float>(img[i * 3 + c]), 2.0f / 255.0f, -1.0f) * k);
}

// one thread per (image b, latent pixel): channel 4 = [mask[f i, f j] >= 128] (F.interpolate(M, size=(h, w)), nearest,
// for an integer factor f), channels 5..8 = z, into rows b and B + b ([cond | uncond] see the same conditioning)
template <bool kBf16>
__global__ void pack_image_cond_kernel(const float4* __restrict__ z, const unsigned char* __restrict__ mask, void* xin,
                                       long long pitch, int B, int h, int w, int f) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int hw = h * w;
  if (i >= B * hw) return;
  const int b = i / hw, pix = i - b * hw;
  const int y = pix / w, x = pix - y * w;
  const float m = mask == nullptr || mask[(static_cast<long long>(f) * y) * (static_cast<long long>(f) * w) + f * x] >= 128
                      ? 1.0f : 0.0f;
  const float4 v = z[i];
  uint2 pk;
  uint16_t last;
  if constexpr (kBf16) {
    __nv_bfloat162 a = __floats2bfloat162_rn(m, v.x), c = __floats2bfloat162_rn(v.y, v.z);
    __nv_bfloat16 d = __float2bfloat16_rn(v.w);
    pk.x = *reinterpret_cast<uint32_t*>(&a);
    pk.y = *reinterpret_cast<uint32_t*>(&c);
    last = *reinterpret_cast<uint16_t*>(&d);
  } else {
    __half2 a = __floats2half2_rn(m, v.x), c = __floats2half2_rn(v.y, v.z);
    __half d = __float2half_rn(v.w);
    pk.x = *reinterpret_cast<uint32_t*>(&a);
    pk.y = *reinterpret_cast<uint32_t*>(&c);
    last = *reinterpret_cast<uint16_t*>(&d);
  }
  uint16_t* base = reinterpret_cast<uint16_t*>(xin);
  for (int r = 0; r < 2; ++r) {
    uint16_t* row = base + (static_cast<long long>(b + r * B) * hw + pix) * pitch;
    *reinterpret_cast<uint2*>(row + 4) = pk;   // channels 4..7: 8-byte aligned (pitch % 4 == 0)
    row[8] = last;
  }
}

}  // namespace b200sd

using namespace b200sd;

extern "C" int b200sd_masked_image_to_nhwc(const unsigned char* img, const unsigned char* mask, float weight, void* out,
                                           long long pitch, int B, int HW, int dtype, void* stream) {
  if (dtype != B200SD_F16 && dtype != B200SD_BF16) return B200SD_ERR_INVALID;
  if (B <= 0 || HW <= 0) return B200SD_OK;
  if (pitch < 3) return B200SD_ERR_INVALID;
  const long long n = static_cast<long long>(B) * HW;
  const int blocks = static_cast<int>((n + 255) / 256);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (dtype == B200SD_BF16) masked_image_to_nhwc_kernel<true><<<blocks, 256, 0, st>>>(img, mask, weight, out, pitch, HW, n);
  else masked_image_to_nhwc_kernel<false><<<blocks, 256, 0, st>>>(img, mask, weight, out, pitch, HW, n);
  return cudaGetLastError() == cudaSuccess ? B200SD_OK : B200SD_ERR_CUDA;
}

extern "C" int b200sd_pack_image_cond(const float* z, const unsigned char* mask, void* xin, long long pitch, int B, int h,
                                      int w, int f, int dtype, void* stream) {
  if (dtype != B200SD_F16 && dtype != B200SD_BF16) return B200SD_ERR_INVALID;
  if (B < 0 || h <= 0 || w <= 0 || f <= 0) return B200SD_ERR_INVALID;
  if (pitch < 9 || pitch % 4 || (reinterpret_cast<uintptr_t>(z) & 15) || (reinterpret_cast<uintptr_t>(xin) & 7))
    return B200SD_ERR_INVALID;
  if (B == 0) return B200SD_OK;
  const long long n = static_cast<long long>(B) * h * w;
  if (n > 0x7fffffffLL) return B200SD_ERR_INVALID;
  const int blocks = static_cast<int>((n + 255) / 256);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (dtype == B200SD_BF16)
    pack_image_cond_kernel<true><<<blocks, 256, 0, st>>>(reinterpret_cast<const float4*>(z), mask, xin, pitch, B, h, w, f);
  else
    pack_image_cond_kernel<false><<<blocks, 256, 0, st>>>(reinterpret_cast<const float4*>(z), mask, xin, pitch, B, h, w, f);
  return cudaGetLastError() == cudaSuccess ? B200SD_OK : B200SD_ERR_CUDA;
}
