// elementwise.cu — small HBM/latency-bound kernels around the tensor-core ops: nearest 2x upsample,
// row softmax (VAE mid attention), SiLU, sinusoidal timestep embedding, per-step bias folding/selection,
// CFG + DDIM / Euler-ancestral latent update fused with re-packing the next UNet input, and the final
// [-1,1] -> uint8 quantisation.
//
// Upstream: ldm Upsample, timestep_embedding, ResBlock.emb_layers; sdwui CFGDenoiser,
// sd_samplers_timesteps_impl.ddim, k-diffusion sample_euler_ancestral, process_images_inner's
// clamp/255/uint8 (SURVEY.md §8 a-ext x2, x4, x10, x11 and App. C; not in /root/reference).
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include "../../../include/b200sd.h"
#include "pdl.cuh"

namespace b200sd {

template <bool kBf16>
__device__ __forceinline__ float load1(const void* p, long long i) {
  if constexpr (kBf16) return __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(p)[i]);
  else return __half2float(reinterpret_cast<const __half*>(p)[i]);
}
template <bool kBf16>
__device__ __forceinline__ void store1(void* p, long long i, float v) {
  if constexpr (kBf16) reinterpret_cast<__nv_bfloat16*>(p)[i] = __float2bfloat16_rn(v);
  else reinterpret_cast<__half*>(p)[i] = __float2half_rn(v);
}

// ---------------------------------------------------------------------------------------------
__global__ void upsample2x_kernel(const uint4* __restrict__ X, long long pitch_x_v, uint4* __restrict__ Y,
                                  long long pitch_y_v, int NB, int H, int W, int cvec) {
  pdl_trigger();
  pdl_wait();
  // one thread per (output pixel, 16-byte channel vector)
  const long long total = static_cast<long long>(NB) * (2 * H) * (2 * W) * cvec;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int v = static_cast<int>(i % cvec);
    const long long pix = i / cvec;
    const int x = static_cast<int>(pix % (2 * W));
    const int y = static_cast<int>((pix / (2 * W)) % (2 * H));
    const int n = static_cast<int>(pix / (static_cast<long long>(2 * W) * (2 * H)));
    const long long src = (static_cast<long long>(n) * H + (y >> 1)) * W + (x >> 1);
    Y[pix * pitch_y_v + v] = __ldg(&X[src * pitch_x_v + v]);
  }
}

// one CTA per row; in place; cols <= 16384
template <bool kBf16>
__global__ void softmax_rows_kernel(void* S, long long lds, int cols, float scale_log2) {
  pdl_trigger();
  pdl_wait();
  __shared__ float red[32];
  const long long row = blockIdx.x;
  uint8_t* base = reinterpret_cast<uint8_t*>(S) + row * lds * 2;
  float mx = -INFINITY;
  for (int c = threadIdx.x; c < cols; c += blockDim.x) mx = fmaxf(mx, load1<kBf16>(base, c));
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = mx;
  __syncthreads();
  mx = red[0];
  for (int w = 1; w < (blockDim.x >> 5); ++w) mx = fmaxf(mx, red[w]);
  __syncthreads();
  float sum = 0.f;
  for (int c = threadIdx.x; c < cols; c += blockDim.x) sum += exp2f((load1<kBf16>(base, c) - mx) * scale_log2);
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = sum;
  __syncthreads();
  sum = 0.f;
  for (int w = 0; w < (blockDim.x >> 5); ++w) sum += red[w];
  const float inv = 1.0f / sum;
  for (int c = threadIdx.x; c < cols; c += blockDim.x)
    store1<kBf16>(base, c, exp2f((load1<kBf16>(base, c) - mx) * scale_log2) * inv);
}

template <bool kBf16>
__global__ void silu_kernel(const void* X, void* Y, long long n) {
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float v = load1<kBf16>(X, i);
    store1<kBf16>(Y, i, v / (1.0f + __expf(-v)));
  }
}

// emb[t][0:half] = cos(t * f_k), emb[t][half:] = sin(t * f_k), f_k = exp(-ln(10000) * k / half)
template <bool kBf16>
__global__ void timestep_embedding_kernel(const float* __restrict__ t, int T, int dim, void* out, long long ldo) {
  const int half = dim / 2;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= T * half) return;
  const int row = i / half, k = i % half;
  const float freq = expf(-logf(10000.0f) * static_cast<float>(k) / static_cast<float>(half));
  const float a = t[row] * freq;
  store1<kBf16>(out, row * ldo + k, cosf(a));
  store1<kBf16>(out, row * ldo + half + k, sinf(a));
}

template <bool kBf16>
__global__ void fold_bias_kernel(const void* emb, long long lde, const float* __restrict__ bias, float* table, int T,
                                 int C) {
  const long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (i >= static_cast<long long>(T) * C) return;
  const int row = static_cast<int>(i / C), c = static_cast<int>(i % C);
  table[i] = bias[c] + load1<kBf16>(emb, row * lde + c);
}

__global__ void select_step_kernel(const float* __restrict__ table, long long row_len, const int* step, float* cur) {
  pdl_trigger();
  pdl_wait();
  const float* src = table + static_cast<long long>(*step) * row_len;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < row_len;
       i += static_cast<long long>(gridDim.x) * blockDim.x)
    cur[i] = src[i];
}

// ---------------------------------------------------------------------------------------------
// latents: x fp32 [B][HW][4]; UNet input xin [2B][HW][pitch] (channels 0..3 written, rest stay zero)
template <bool kBf16>
__device__ __forceinline__ void write_xin(void* xin, long long pitch, int B, int HW, int b, int pix, float4 v) {
  uint2 pk;
  if constexpr (kBf16) {
    __nv_bfloat162 a = __floats2bfloat162_rn(v.x, v.y), c = __floats2bfloat162_rn(v.z, v.w);
    pk.x = *reinterpret_cast<uint32_t*>(&a);
    pk.y = *reinterpret_cast<uint32_t*>(&c);
  } else {
    __half2 a = __floats2half2_rn(v.x, v.y), c = __floats2half2_rn(v.z, v.w);
    pk.x = *reinterpret_cast<uint32_t*>(&a);
    pk.y = *reinterpret_cast<uint32_t*>(&c);
  }
  uint8_t* base = reinterpret_cast<uint8_t*>(xin);
  *reinterpret_cast<uint2*>(base + ((static_cast<long long>(b) * HW + pix) * pitch) * 2) = pk;
  *reinterpret_cast<uint2*>(base + ((static_cast<long long>(b + B) * HW + pix) * pitch) * 2) = pk;
}

template <bool kBf16>
__device__ __forceinline__ float4 read_eps4(const void* eps, long long pitch, long long row) {
  const uint2 u = *reinterpret_cast<const uint2*>(reinterpret_cast<const uint8_t*>(eps) + row * pitch * 2);
  float2 a, c;
  if constexpr (kBf16) {
    a = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&u.x));
    c = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&u.y));
  } else {
    a = __half22float2(*reinterpret_cast<const __half2*>(&u.x));
    c = __half22float2(*reinterpret_cast<const __half2*>(&u.y));
  }
  return make_float4(a.x, a.y, c.x, c.y);
}

template <bool kBf16>
__global__ void pack_unet_input_kernel(const float4* __restrict__ x, void* xin, long long pitch, int B, int HW,
                                       float in_scale) {
  pdl_trigger();
  pdl_wait();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * HW) return;
  float4 v = x[i];
  v.x *= in_scale; v.y *= in_scale; v.z *= in_scale; v.w *= in_scale;
  write_xin<kBf16>(xin, pitch, B, HW, i / HW, i % HW, v);
}

// kVPred: the UNet predicts v (SD 2.x 768-v); the CFG-combined v becomes eps = sqrt(1-a_t) x + sqrt(a_t) v with the
// pre-update fp32 x, the point the UNet evaluated (sdwui CompVisTimestepsVDenoiser.predict_eps_from_z_and_v)
template <bool kBf16, bool kVPred = false>
__global__ void cfg_ddim_step_kernel(const void* eps, long long pitch_e, float4* x, void* xin, long long pitch_x, int B,
                                     int HW, float cfg, const float* __restrict__ coef, int* step_counter) {
  pdl_trigger();
  pdl_wait();
  const int step = *step_counter;
  const float sa = coef[step * 4 + 0], s1a = coef[step * 4 + 1], sap = coef[step * 4 + 2], s1ap = coef[step * 4 + 3];
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < B * HW) {
    const int b = i / HW, pix = i % HW;
    const float4 ec = read_eps4<kBf16>(eps, pitch_e, static_cast<long long>(b) * HW + pix);
    const float4 eu = read_eps4<kBf16>(eps, pitch_e, static_cast<long long>(b + B) * HW + pix);
    float4 xv = x[i];
    float e[4] = {eu.x + cfg * (ec.x - eu.x), eu.y + cfg * (ec.y - eu.y), eu.z + cfg * (ec.z - eu.z),
                  eu.w + cfg * (ec.w - eu.w)};
    float xs[4] = {xv.x, xv.y, xv.z, xv.w};
    if constexpr (kVPred) {
#pragma unroll
      for (int k = 0; k < 4; ++k) e[k] = s1a * xs[k] + sa * e[k];
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float x0 = (xs[k] - s1a * e[k]) / sa;
      xs[k] = sap * x0 + s1ap * e[k];
    }
    xv = make_float4(xs[0], xs[1], xs[2], xs[3]);
    x[i] = xv;
    write_xin<kBf16>(xin, pitch_x, B, HW, b, pix, xv);
  }
}

// coef[step] = {sigma, sigma_down, sigma_up, in_scale_next}; x lives in sigma space (x = latent * sqrt(1+sigma^2));
// the UNet input of the NEXT step is x_next * in_scale_next with in_scale_next = 1/sqrt(sigma_next^2 + 1).
// kVPred: rows of 8 floats {sigma, sigma_down, sigma_up, in_scale_next, kx, kv, 0, 0}; the CFG-combined v becomes
// eps = kx x + kv v with kx = sigma/(sigma^2+1), kv = 1/sqrt(sigma^2+1) (k-diffusion CompVisVDenoiser: to_d of its denoised)
template <bool kBf16, bool kVPred = false>
__global__ void cfg_euler_a_step_kernel(const void* eps, long long pitch_e, float4* x, const float4* __restrict__ noise,
                                        void* xin, long long pitch_x, int B, int HW, float cfg,
                                        const float* __restrict__ coef, int* step_counter) {
  pdl_trigger();
  pdl_wait();
  const int step = *step_counter;
  constexpr int ld = kVPred ? 8 : 4;
  const float sigma = coef[step * ld + 0], sdown = coef[step * ld + 1], sup = coef[step * ld + 2],
              in_next = coef[step * ld + 3];
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < B * HW) {
    const int b = i / HW, pix = i % HW;
    const float4 ec = read_eps4<kBf16>(eps, pitch_e, static_cast<long long>(b) * HW + pix);
    const float4 eu = read_eps4<kBf16>(eps, pitch_e, static_cast<long long>(b + B) * HW + pix);
    float4 xv = x[i];
    float e[4] = {eu.x + cfg * (ec.x - eu.x), eu.y + cfg * (ec.y - eu.y), eu.z + cfg * (ec.z - eu.z),
                  eu.w + cfg * (ec.w - eu.w)};
    float xs[4] = {xv.x, xv.y, xv.z, xv.w};
    if constexpr (kVPred) {
      const float kx = coef[step * ld + 4], kv = coef[step * ld + 5];
#pragma unroll
      for (int k = 0; k < 4; ++k) e[k] = kx * xs[k] + kv * e[k];
    }
    float nz[4] = {0.f, 0.f, 0.f, 0.f};
    if (noise != nullptr && sup > 0.f) {
      const float4 nv = noise[static_cast<long long>(step) * B * HW + i];
      nz[0] = nv.x; nz[1] = nv.y; nz[2] = nv.z; nz[3] = nv.w;
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      // denoised = x - sigma * eps; d = (x - denoised) / sigma = eps; x += d * (sigma_down - sigma)
      xs[k] = xs[k] + e[k] * (sdown - sigma) + nz[k] * sup;
    }
    xv = make_float4(xs[0], xs[1], xs[2], xs[3]);
    x[i] = xv;
    write_xin<kBf16>(xin, pitch_x, B, HW, b, pix,
                     make_float4(xs[0] * in_next, xs[1] * in_next, xs[2] * in_next, xs[3] * in_next));
  }
}

// DPM-Solver++(2M) (k-diffusion sample_dpmpp_2m) on an eps-prediction model:
//   denoised = x - sigma * eps;  dd = c1 * denoised - c2 * old_denoised;  x = a * x + (1 - a) * dd;  old = denoised
// with a = sigma_next / sigma = exp(-h), c1 = 1 + 1/(2r), c2 = 1/(2r), r = h_last / h (c1 = 1, c2 = 0 on the first step and
// on the step to sigma = 0).  coef row = {sigma, a, c1, c2, in_scale_next, -, -, -}.
// kVPred: columns 5, 6 hold kx, kv and the CFG-combined v becomes eps = kx x + kv v (as in the Euler (a) kernel).
template <bool kBf16, bool kVPred = false>
__global__ void cfg_dpmpp_2m_step_kernel(const void* eps, long long pitch_e, float4* x, float4* old_denoised, void* xin,
                                         long long pitch_x, int B, int HW, float cfg, const float* __restrict__ coef,
                                         int* step_counter) {
  pdl_trigger();
  pdl_wait();
  const int step = *step_counter;
  const float sigma = coef[step * 8 + 0], a = coef[step * 8 + 1], c1 = coef[step * 8 + 2], c2 = coef[step * 8 + 3],
              in_next = coef[step * 8 + 4];
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < B * HW) {
    const int b = i / HW, pix = i % HW;
    const float4 ec = read_eps4<kBf16>(eps, pitch_e, static_cast<long long>(b) * HW + pix);
    const float4 eu = read_eps4<kBf16>(eps, pitch_e, static_cast<long long>(b + B) * HW + pix);
    const float4 xv = x[i], ov = old_denoised[i];
    float e[4] = {eu.x + cfg * (ec.x - eu.x), eu.y + cfg * (ec.y - eu.y), eu.z + cfg * (ec.z - eu.z),
                  eu.w + cfg * (ec.w - eu.w)};
    const float xs[4] = {xv.x, xv.y, xv.z, xv.w}, os[4] = {ov.x, ov.y, ov.z, ov.w};
    if constexpr (kVPred) {
      const float kx = coef[step * 8 + 5], kv = coef[step * 8 + 6];
#pragma unroll
      for (int k = 0; k < 4; ++k) e[k] = kx * xs[k] + kv * e[k];
    }
    float xn[4], dn[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      dn[k] = xs[k] - sigma * e[k];
      const float dd = c2 != 0.f ? c1 * dn[k] - c2 * os[k] : dn[k];
      xn[k] = a * xs[k] + (1.0f - a) * dd;
    }
    x[i] = make_float4(xn[0], xn[1], xn[2], xn[3]);
    old_denoised[i] = make_float4(dn[0], dn[1], dn[2], dn[3]);
    write_xin<kBf16>(xin, pitch_x, B, HW, b, pix,
                     make_float4(xn[0] * in_next, xn[1] * in_next, xn[2] * in_next, xn[3] * in_next));
  }
}

__global__ void bump_step_kernel(int* step_counter) {
  pdl_trigger();
  pdl_wait(); *step_counter += 1; }

// ---- generic sampler building blocks (every k-diffusion / timestep sampler beyond the four fused ones above is a short
// list of these per model evaluation; b200sd/samplers.py holds the coefficient algebra) ----
// e[b, pix, :] (fp32) = eu + cfg * (ec - eu): sdwui CFGDenoiser's combine.  For an eps-prediction model wrapped by
// k-diffusion's CompVisDenoiser, to_d(x, sigma, denoised) = (x - denoised) / sigma is exactly this e.
template <bool kBf16>
__global__ void cfg_eps_kernel(const void* eps, long long pitch_e, float4* __restrict__ e, int B, int HW, float cfg) {
  pdl_trigger();
  pdl_wait();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * HW) return;
  const int b = i / HW, pix = i % HW;
  const float4 ec = read_eps4<kBf16>(eps, pitch_e, static_cast<long long>(b) * HW + pix);
  const float4 eu = read_eps4<kBf16>(eps, pitch_e, static_cast<long long>(b + B) * HW + pix);
  e[i] = make_float4(eu.x + cfg * (ec.x - eu.x), eu.y + cfg * (ec.y - eu.y), eu.z + cfg * (ec.z - eu.z),
                     eu.w + cfg * (ec.w - eu.w));
}

constexpr int kMaxLincomb = 8;
struct LincombParams {
  const float4* src[kMaxLincomb];
  long long idx_stride[kMaxLincomb];  // in float4 elements; != 0: the source is a stack of tensors indexed by `idx`
  int n;
};
// dst = sum_k c[k] * src_k with c = coef[row * ld + col0 ...], row = *step_counter; sources with an index stride read
// tensor (int)coef[row * ld + idx_col] of their stack (the per-step noise draws).  With xin != null the result times
// c[n] is also written as the next UNet input (both CFG halves).  dst may alias a source (same element, same thread).
template <bool kBf16>
__global__ void latent_lincomb_kernel(float4* dst, const LincombParams p, const float* __restrict__ coef, int ld,
                                      int col0, int idx_col, const int* __restrict__ step_counter, void* xin,
                                      long long pitch_x, int B, int HW) {
  pdl_trigger();
  pdl_wait();
  const int row = *step_counter;
  const float* c = coef + static_cast<long long>(row) * ld + col0;
  const long long idx = idx_col >= 0 ? static_cast<long long>(coef[static_cast<long long>(row) * ld + idx_col]) : 0;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * HW) return;
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
  for (int k = 0; k < kMaxLincomb; ++k) {
    if (k < p.n) {
      const float w = c[k];
      if (w != 0.f) {  // a zero weight must not propagate a stale buffer's NaN / Inf
        const float4 v = p.src[k][idx * p.idx_stride[k] + i];
        acc.x = fmaf(w, v.x, acc.x); acc.y = fmaf(w, v.y, acc.y); acc.z = fmaf(w, v.z, acc.z); acc.w = fmaf(w, v.w, acc.w);
      }
    }
  }
  dst[i] = acc;
  if (xin != nullptr) {
    const float s = c[p.n];
    write_xin<kBf16>(xin, pitch_x, B, HW, i / HW, i % HW, make_float4(acc.x * s, acc.y * s, acc.z * s, acc.w * s));
  }
}


template <bool kBf16>
__global__ void quantize_u8_kernel(const void* img, long long pitch, unsigned char* out, long long npix) {
  pdl_trigger();
  pdl_wait();
  const long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (i >= npix) return;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    float v = load1<kBf16>(img, i * pitch + c);
    v = fminf(fmaxf((v + 1.0f) * 0.5f, 0.f), 1.f);
    out[i * 3 + c] = static_cast<unsigned char>(255.0f * v);  // truncation, as numpy astype(uint8)
  }
}

template <bool kBf16>
__global__ void image_to_nhwc_kernel(const unsigned char* __restrict__ img, void* out, long long pitch, long long npix) {
  const long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (i >= npix) return;
#pragma unroll
  for (int c = 0; c < 3; ++c) store1<kBf16>(out, i * pitch + c, static_cast<float>(img[i * 3 + c]) * (2.0f / 255.0f) - 1.0f);
}

template <bool kBf16>
__global__ void unpack_latent_kernel(const void* m, long long pitch, float4* x, long long npix, float scale) {
  const long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (i >= npix) return;
  x[i] = make_float4(load1<kBf16>(m, i * pitch) * scale, load1<kBf16>(m, i * pitch + 1) * scale,
                     load1<kBf16>(m, i * pitch + 2) * scale, load1<kBf16>(m, i * pitch + 3) * scale);
}

// bilinear resize of NHWC fp32 latents [B, H*W, 4] -> [B, Ho*Wo, 4], half-pixel centres (align_corners = False), no
// antialiasing: torch.nn.functional.interpolate(mode="bilinear") as sdwui's "Latent" hires upscaler calls it
// inpainting: x = x * latmask + init * (1 - latmask), latmask [HW] shared by the channels and the images of the request
// (sdwui CFGDenoiser.apply_blend: current * nmask + init_latent * mask)
__global__ void blend_latent_kernel(float4* __restrict__ x, const float4* __restrict__ init, const float* __restrict__ latmask,
                                    int B, int HW) {
  pdl_trigger();
  pdl_wait();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * HW) return;
  const float m = latmask[i % HW];
  const float4 xv = x[i], iv = init[i];
  x[i] = make_float4(xv.x * m + iv.x * (1.f - m), xv.y * m + iv.y * (1.f - m), xv.z * m + iv.z * (1.f - m),
                     xv.w * m + iv.w * (1.f - m));
}

__global__ void resize_latent_bilinear_kernel(const float4* __restrict__ x, float4* __restrict__ y, int B, int H, int W,
                                              int Ho, int Wo) {
  const long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  const long long n = static_cast<long long>(B) * Ho * Wo;
  if (i >= n) return;
  const int xo = static_cast<int>(i % Wo), yo = static_cast<int>((i / Wo) % Ho), b = static_cast<int>(i / (static_cast<long long>(Wo) * Ho));
  const float sy = fmaxf((yo + 0.5f) * (static_cast<float>(H) / Ho) - 0.5f, 0.f);
  const float sx = fmaxf((xo + 0.5f) * (static_cast<float>(W) / Wo) - 0.5f, 0.f);
  const int y0 = min(static_cast<int>(sy), H - 1), x0 = min(static_cast<int>(sx), W - 1);
  const int y1 = min(y0 + 1, H - 1), x1 = min(x0 + 1, W - 1);
  const float ly = sy - y0, lx = sx - x0;
  const float4* img = x + static_cast<long long>(b) * H * W;
  const float4 a = img[y0 * W + x0], c = img[y0 * W + x1], d = img[y1 * W + x0], e = img[y1 * W + x1];
  const float w00 = (1.f - ly) * (1.f - lx), w01 = (1.f - ly) * lx, w10 = ly * (1.f - lx), w11 = ly * lx;
  y[i] = make_float4(w00 * a.x + w01 * c.x + w10 * d.x + w11 * e.x, w00 * a.y + w01 * c.y + w10 * d.y + w11 * e.y,
                     w00 * a.z + w01 * c.z + w10 * d.z + w11 * e.z, w00 * a.w + w01 * c.w + w10 * d.w + w11 * e.w);
}

}  // namespace b200sd

using namespace b200sd;
#define ST(s) static_cast<cudaStream_t>(s)
#define RET_LAUNCH() return cudaGetLastError() == cudaSuccess ? B200SD_OK : B200SD_ERR_CUDA

extern "C" int b200sd_upsample2x(const void* X, long long pitch_x, void* Y, long long pitch_y, int NB, int H, int W,
                                 int C, int dtype, void* stream) {
  (void)dtype;
  if (NB <= 0) return B200SD_OK;
  if (C % 8 || pitch_x % 8 || pitch_y % 8 || ((reinterpret_cast<uintptr_t>(X) | reinterpret_cast<uintptr_t>(Y)) & 15))
    return B200SD_ERR_INVALID;
  const long long total = static_cast<long long>(NB) * 4 * H * W * (C / 8);
  long long blocks = (total + 255) / 256;
  if (blocks > kNumSms * 16) blocks = kNumSms * 16;
  launch_pdl(upsample2x_kernel, dim3(static_cast<int>(blocks)), dim3(256), 0, ST(stream), static_cast<const uint4*>(X), pitch_x / 8, static_cast<uint4*>(Y), pitch_y / 8, NB, H, W, C / 8);
  RET_LAUNCH();
}

extern "C" int b200sd_softmax_rows(void* S, long long lds, int rows, int cols, float scale, int dtype, void* stream) {
  if (rows <= 0) return B200SD_OK;
  if (cols <= 0) return B200SD_ERR_INVALID;
  const float sl2 = scale * 1.4426950408889634f;
  if (dtype == B200SD_BF16) launch_pdl(softmax_rows_kernel<true>, dim3(rows), dim3(256), 0, ST(stream), S, lds, cols, sl2);
  else launch_pdl(softmax_rows_kernel<false>, dim3(rows), dim3(256), 0, ST(stream), S, lds, cols, sl2);
  RET_LAUNCH();
}

extern "C" int b200sd_silu(const void* X, void* Y, long long n, int dtype, void* stream) {
  if (n <= 0) return B200SD_OK;
  long long blocks = (n + 255) / 256;
  if (blocks > kNumSms * 8) blocks = kNumSms * 8;
  if (dtype == B200SD_BF16) silu_kernel<true><<<static_cast<int>(blocks), 256, 0, ST(stream)>>>(X, Y, n);
  else silu_kernel<false><<<static_cast<int>(blocks), 256, 0, ST(stream)>>>(X, Y, n);
  RET_LAUNCH();
}

extern "C" int b200sd_timestep_embedding(const float* t, int T, int dim, void* out, long long ldo, int dtype,
                                         void* stream) {
  if (T <= 0) return B200SD_OK;
  if (dim % 2) return B200SD_ERR_INVALID;
  const int n = T * (dim / 2);
  if (dtype == B200SD_BF16) timestep_embedding_kernel<true><<<(n + 127) / 128, 128, 0, ST(stream)>>>(t, T, dim, out, ldo);
  else timestep_embedding_kernel<false><<<(n + 127) / 128, 128, 0, ST(stream)>>>(t, T, dim, out, ldo);
  RET_LAUNCH();
}

extern "C" int b200sd_fold_bias(const void* emb, long long lde, const float* bias, float* table, int T, int C,
                                int dtype, void* stream) {
  if (T <= 0 || C <= 0) return B200SD_OK;
  const long long n = static_cast<long long>(T) * C;
  const int blocks = static_cast<int>((n + 255) / 256);
  if (dtype == B200SD_BF16) fold_bias_kernel<true><<<blocks, 256, 0, ST(stream)>>>(emb, lde, bias, table, T, C);
  else fold_bias_kernel<false><<<blocks, 256, 0, ST(stream)>>>(emb, lde, bias, table, T, C);
  RET_LAUNCH();
}

extern "C" int b200sd_select_step(const float* table, long long row_len, const int* step_counter, float* cur,
                                  void* stream) {
  if (row_len <= 0) return B200SD_OK;
  long long blocks = (row_len + 255) / 256;
  if (blocks > kNumSms) blocks = kNumSms;
  launch_pdl(select_step_kernel, dim3(static_cast<int>(blocks)), dim3(256), 0, ST(stream), table, row_len, step_counter, cur);
  RET_LAUNCH();
}

extern "C" int b200sd_pack_unet_input(const float* x, void* xin, long long pitch, int B, int HW, float in_scale,
                                      int dtype, void* stream) {
  if (B <= 0) return B200SD_OK;
  if (pitch % 4) return B200SD_ERR_INVALID;
  const int n = B * HW;
  if (dtype == B200SD_BF16)
    launch_pdl(pack_unet_input_kernel<true>, dim3((n + 255) / 256), dim3(256), 0, ST(stream), reinterpret_cast<const float4*>(x), xin, pitch, B, HW, in_scale);
  else
    launch_pdl(pack_unet_input_kernel<false>, dim3((n + 255) / 256), dim3(256), 0, ST(stream), reinterpret_cast<const float4*>(x), xin, pitch, B, HW, in_scale);
  RET_LAUNCH();
}

template <bool kVPred>
static int cfg_ddim_step(const void* eps, long long pitch_e, float* x, void* xin, long long pitch_x, int B, int HW,
                         float cfg_scale, const float* coef, int* step_counter, int dtype, void* stream) {
  if (B <= 0) return B200SD_OK;
  if (pitch_e % 4 || pitch_x % 4) return B200SD_ERR_INVALID;
  const int n = B * HW;
  if (dtype == B200SD_BF16)
    launch_pdl(cfg_ddim_step_kernel<true, kVPred>, dim3((n + 255) / 256), dim3(256), 0, ST(stream), eps, pitch_e, reinterpret_cast<float4*>(x), xin, pitch_x, B, HW, cfg_scale, coef, step_counter);
  else
    launch_pdl(cfg_ddim_step_kernel<false, kVPred>, dim3((n + 255) / 256), dim3(256), 0, ST(stream), eps, pitch_e, reinterpret_cast<float4*>(x), xin, pitch_x, B, HW, cfg_scale, coef, step_counter);
  if (cudaGetLastError() != cudaSuccess) return B200SD_ERR_CUDA;
  launch_pdl(bump_step_kernel, dim3(1), dim3(1), 0, ST(stream), step_counter);
  RET_LAUNCH();
}

template <bool kVPred>
static int cfg_euler_a_step(const void* eps, long long pitch_e, float* x, const float* noise, void* xin,
                            long long pitch_x, int B, int HW, float cfg_scale, const float* coef, int* step_counter,
                            int dtype, void* stream) {
  if (B <= 0) return B200SD_OK;
  if (pitch_e % 4 || pitch_x % 4) return B200SD_ERR_INVALID;
  const int n = B * HW;
  if (dtype == B200SD_BF16)
    launch_pdl(cfg_euler_a_step_kernel<true, kVPred>, dim3((n + 255) / 256), dim3(256), 0, ST(stream), eps, pitch_e, reinterpret_cast<float4*>(x), reinterpret_cast<const float4*>(noise), xin, pitch_x, B, HW, cfg_scale, coef, step_counter);
  else
    launch_pdl(cfg_euler_a_step_kernel<false, kVPred>, dim3((n + 255) / 256), dim3(256), 0, ST(stream), eps, pitch_e, reinterpret_cast<float4*>(x), reinterpret_cast<const float4*>(noise), xin, pitch_x, B, HW, cfg_scale, coef, step_counter);
  if (cudaGetLastError() != cudaSuccess) return B200SD_ERR_CUDA;
  launch_pdl(bump_step_kernel, dim3(1), dim3(1), 0, ST(stream), step_counter);
  RET_LAUNCH();
}

template <bool kVPred>
static int cfg_dpmpp_2m_step(const void* eps, long long pitch_e, float* x, float* old_denoised, void* xin,
                             long long pitch_x, int B, int HW, float cfg_scale, const float* coef, int* step_counter,
                             int dtype, void* stream) {
  if (B <= 0) return B200SD_OK;
  if ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(old_denoised)) & 15) return B200SD_ERR_INVALID;
  const int n = B * HW;
  if (dtype == B200SD_BF16)
    launch_pdl(cfg_dpmpp_2m_step_kernel<true, kVPred>, dim3((n + 255) / 256), dim3(256), 0, ST(stream), eps, pitch_e, reinterpret_cast<float4*>(x), reinterpret_cast<float4*>(old_denoised), xin, pitch_x, B, HW, cfg_scale, coef, step_counter);
  else
    launch_pdl(cfg_dpmpp_2m_step_kernel<false, kVPred>, dim3((n + 255) / 256), dim3(256), 0, ST(stream), eps, pitch_e, reinterpret_cast<float4*>(x), reinterpret_cast<float4*>(old_denoised), xin, pitch_x, B, HW, cfg_scale, coef, step_counter);
  if (cudaGetLastError() != cudaSuccess) return B200SD_ERR_CUDA;
  launch_pdl(bump_step_kernel, dim3(1), dim3(1), 0, ST(stream), step_counter);
  RET_LAUNCH();
}

extern "C" int b200sd_cfg_ddim_step(const void* eps, long long pitch_e, float* x, void* xin, long long pitch_x, int B,
                                    int HW, float cfg_scale, const float* coef, int* step_counter, int dtype,
                                    void* stream) {
  return cfg_ddim_step<false>(eps, pitch_e, x, xin, pitch_x, B, HW, cfg_scale, coef, step_counter, dtype, stream);
}

extern "C" int b200sd_cfg_ddim_step_v(const void* eps, long long pitch_e, float* x, void* xin, long long pitch_x, int B,
                                      int HW, float cfg_scale, const float* coef, int* step_counter, int dtype,
                                      void* stream) {
  return cfg_ddim_step<true>(eps, pitch_e, x, xin, pitch_x, B, HW, cfg_scale, coef, step_counter, dtype, stream);
}

extern "C" int b200sd_cfg_euler_a_step(const void* eps, long long pitch_e, float* x, const float* noise, void* xin,
                                       long long pitch_x, int B, int HW, float cfg_scale, const float* coef,
                                       int* step_counter, int dtype, void* stream) {
  return cfg_euler_a_step<false>(eps, pitch_e, x, noise, xin, pitch_x, B, HW, cfg_scale, coef, step_counter, dtype,
                                 stream);
}

extern "C" int b200sd_cfg_euler_a_step_v(const void* eps, long long pitch_e, float* x, const float* noise, void* xin,
                                         long long pitch_x, int B, int HW, float cfg_scale, const float* coef,
                                         int* step_counter, int dtype, void* stream) {
  return cfg_euler_a_step<true>(eps, pitch_e, x, noise, xin, pitch_x, B, HW, cfg_scale, coef, step_counter, dtype,
                                stream);
}

extern "C" int b200sd_cfg_dpmpp_2m_step(const void* eps, long long pitch_e, float* x, float* old_denoised, void* xin,
                                        long long pitch_x, int B, int HW, float cfg_scale, const float* coef,
                                        int* step_counter, int dtype, void* stream) {
  return cfg_dpmpp_2m_step<false>(eps, pitch_e, x, old_denoised, xin, pitch_x, B, HW, cfg_scale, coef, step_counter,
                                  dtype, stream);
}

extern "C" int b200sd_cfg_dpmpp_2m_step_v(const void* eps, long long pitch_e, float* x, float* old_denoised, void* xin,
                                          long long pitch_x, int B, int HW, float cfg_scale, const float* coef,
                                          int* step_counter, int dtype, void* stream) {
  return cfg_dpmpp_2m_step<true>(eps, pitch_e, x, old_denoised, xin, pitch_x, B, HW, cfg_scale, coef, step_counter,
                                 dtype, stream);
}


extern "C" int b200sd_cfg_eps(const void* eps, long long pitch_e, float* e, int B, int HW, float cfg_scale, int dtype,
                              void* stream) {
  if (B <= 0 || HW <= 0) return B200SD_OK;
  if (pitch_e % 4 || (reinterpret_cast<uintptr_t>(e) & 15)) return B200SD_ERR_INVALID;
  const int n = B * HW;
  if (dtype == B200SD_BF16) launch_pdl(cfg_eps_kernel<true>, dim3((n + 255) / 256), dim3(256), 0, ST(stream), eps, pitch_e, reinterpret_cast<float4*>(e), B, HW, cfg_scale);
  else launch_pdl(cfg_eps_kernel<false>, dim3((n + 255) / 256), dim3(256), 0, ST(stream), eps, pitch_e, reinterpret_cast<float4*>(e), B, HW, cfg_scale);
  RET_LAUNCH();
}

extern "C" int b200sd_latent_lincomb(float* dst, const float* const* srcs, const long long* idx_strides, int n_src,
                                     const float* coef, int ld, int col0, int idx_col, const int* step_counter,
                                     void* xin, long long pitch_x, int B, int HW, int dtype, void* stream) {
  if (B <= 0 || HW <= 0) return B200SD_OK;
  if (n_src < 1 || n_src > kMaxLincomb || ld <= 0 || col0 < 0 || col0 + n_src + (xin != nullptr ? 1 : 0) > ld ||
      idx_col >= ld || (reinterpret_cast<uintptr_t>(dst) & 15) || (xin != nullptr && pitch_x % 4))
    return B200SD_ERR_INVALID;
  LincombParams p{};
  p.n = n_src;
  for (int k = 0; k < n_src; ++k) {
    if (srcs[k] == nullptr || (reinterpret_cast<uintptr_t>(srcs[k]) & 15) || (idx_strides != nullptr && idx_strides[k] % 4))
      return B200SD_ERR_INVALID;
    p.src[k] = reinterpret_cast<const float4*>(srcs[k]);
    p.idx_stride[k] = idx_strides != nullptr ? idx_strides[k] / 4 : 0;
    if (p.idx_stride[k] != 0 && idx_col < 0) return B200SD_ERR_INVALID;
  }
  const int n = B * HW;
  if (dtype == B200SD_BF16)
    launch_pdl(latent_lincomb_kernel<true>, dim3((n + 255) / 256), dim3(256), 0, ST(stream), reinterpret_cast<float4*>(dst), p, coef, ld, col0, idx_col, step_counter, xin, pitch_x, B, HW);
  else
    launch_pdl(latent_lincomb_kernel<false>, dim3((n + 255) / 256), dim3(256), 0, ST(stream), reinterpret_cast<float4*>(dst), p, coef, ld, col0, idx_col, step_counter, xin, pitch_x, B, HW);
  RET_LAUNCH();
}

extern "C" int b200sd_bump_step(int* step_counter, void* stream) {
  launch_pdl(bump_step_kernel, dim3(1), dim3(1), 0, ST(stream), step_counter);
  RET_LAUNCH();
}

extern "C" int b200sd_image_to_nhwc(const unsigned char* img, void* out, long long pitch, int B, int HW, int dtype,
                                    void* stream) {
  if (B <= 0) return B200SD_OK;
  if (pitch < 3) return B200SD_ERR_INVALID;
  const long long n = static_cast<long long>(B) * HW;
  const int blocks = static_cast<int>((n + 255) / 256);
  if (dtype == B200SD_BF16) image_to_nhwc_kernel<true><<<blocks, 256, 0, ST(stream)>>>(img, out, pitch, n);
  else image_to_nhwc_kernel<false><<<blocks, 256, 0, ST(stream)>>>(img, out, pitch, n);
  RET_LAUNCH();
}

extern "C" int b200sd_unpack_latent(const void* moments, long long pitch, float* x, int B, int HW, float scale,
                                    int dtype, void* stream) {
  if (B <= 0) return B200SD_OK;
  if (pitch < 4 || (reinterpret_cast<uintptr_t>(x) & 15)) return B200SD_ERR_INVALID;
  const long long n = static_cast<long long>(B) * HW;
  const int blocks = static_cast<int>((n + 255) / 256);
  if (dtype == B200SD_BF16)
    unpack_latent_kernel<true><<<blocks, 256, 0, ST(stream)>>>(moments, pitch, reinterpret_cast<float4*>(x), n, scale);
  else
    unpack_latent_kernel<false><<<blocks, 256, 0, ST(stream)>>>(moments, pitch, reinterpret_cast<float4*>(x), n, scale);
  RET_LAUNCH();
}

extern "C" int b200sd_quantize_u8(const void* img, long long pitch, unsigned char* out, int B, int HW, int dtype,
                                  void* stream) {
  if (B <= 0) return B200SD_OK;
  const long long n = static_cast<long long>(B) * HW;
  const int blocks = static_cast<int>((n + 255) / 256);
  if (dtype == B200SD_BF16) launch_pdl(quantize_u8_kernel<true>, dim3(blocks), dim3(256), 0, ST(stream), img, pitch, out, n);
  else launch_pdl(quantize_u8_kernel<false>, dim3(blocks), dim3(256), 0, ST(stream), img, pitch, out, n);
  RET_LAUNCH();
}

extern "C" int b200sd_blend_latent(float* x, const float* init, const float* latmask, int B, int HW, void* stream) {
  if (B <= 0 || HW <= 0) return B200SD_OK;
  if ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(init)) & 15) return B200SD_ERR_INVALID;
  const long long n = static_cast<long long>(B) * HW;
  launch_pdl(blend_latent_kernel, dim3(static_cast<int>((n + 255) / 256)), dim3(256), 0, ST(stream), reinterpret_cast<float4*>(x), reinterpret_cast<const float4*>(init), latmask, B, HW);
  RET_LAUNCH();
}

extern "C" int b200sd_resize_latent_bilinear(const float* x, float* y, int B, int H, int W, int Ho, int Wo, void* stream) {
  if (B <= 0) return B200SD_OK;
  if (H <= 0 || W <= 0 || Ho <= 0 || Wo <= 0 || ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(y)) & 15))
    return B200SD_ERR_INVALID;
  const long long n = static_cast<long long>(B) * Ho * Wo;
  resize_latent_bilinear_kernel<<<static_cast<int>((n + 255) / 256), 256, 0, ST(stream)>>>(
      reinterpret_cast<const float4*>(x), reinterpret_cast<float4*>(y), B, H, W, Ho, Wo);
  RET_LAUNCH();
}
