// The pieces of the SD / SDXL VAE (diffusers AutoencoderKL) that the UNet's kernels do not cover: the 3-channel
// convolutions at the image ends with the image processor's pre- / postprocess fused in, the encoder's latent head
// (conv_out + quant_conv + DiagonalGaussianDistribution + scaling_factor), the decoder's latent input
// (1 / scaling_factor + post_quant_conv) and the row softmax of the mid-block attention.  Every other VAE layer runs on
// sb200_conv3x3 / sb200_groupnorm / sb200_gemm / sb200_upsample2x.
//
// Replaces (diffusers 0.20.2): VaeImageProcessor.preprocess / postprocess + numpy_to_pil, Encoder.conv_in,
// Decoder.conv_out, Encoder.conv_out + AutoencoderKL.quant_conv + DiagonalGaussianDistribution.sample / .mode,
// AutoencoderKL.post_quant_conv, and the softmax of AttnProcessor's get_attention_scores.
#include "../../include/sb200_vae.h"
#include "common.h"
#include "ptx.cuh"

namespace sb200 {

__device__ __forceinline__ float dot8_bf16(const uint4& a, const uint4& b) {
  const uint32_t aw[4] = {a.x, a.y, a.z, a.w};
  const uint32_t bw[4] = {b.x, b.y, b.z, b.w};
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < 4; ++i) s += bf16_lo(aw[i]) * bf16_lo(bw[i]) + bf16_hi(aw[i]) * bf16_hi(bw[i]);
  return s;
}

// ------------------------------------------------------------------------------------------------
// Encoder.conv_in on uint8 pixels: x = v / 255 * 2 - 1 (fp32, VaeImageProcessor.preprocess), 3x3 pad 1, 3 -> Cout.
// thread = (pixel, 8 output channels); weights transposed to [27][Cout] in shared memory.
// ------------------------------------------------------------------------------------------------
__global__ void vae_conv_in_u8_kernel(const uint8_t* __restrict__ img, const __nv_bfloat16* __restrict__ w,
                                      const __nv_bfloat16* __restrict__ bias, __nv_bfloat16* __restrict__ out, int B,
                                      int H, int W, int Cout) {
  extern __shared__ __align__(16) __nv_bfloat16 wsh[];
  for (int i = threadIdx.x; i < Cout * 27; i += blockDim.x) {
    const int co = i / 27, k = i - co * 27;
    wsh[k * Cout + co] = w[i];
  }
  __syncthreads();
  const int ovec = Cout >> 3;
  const size_t total = static_cast<size_t>(B) * H * W * ovec;
  for (size_t idx = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int ov = static_cast<int>(idx % ovec);
    const size_t pix = idx / ovec;
    const int wq = static_cast<int>(pix % W);
    const int hq = static_cast<int>((pix / W) % H);
    const int b = static_cast<int>(pix / (static_cast<size_t>(W) * H));
    float patch[27];  // [kh][kw][c]
#pragma unroll
    for (int kh = 0; kh < 3; ++kh)
#pragma unroll
      for (int kw = 0; kw < 3; ++kw) {
        const int hh = hq + kh - 1, ww = wq + kw - 1;
        const bool ok = hh >= 0 && hh < H && ww >= 0 && ww < W;
#pragma unroll
        for (int c = 0; c < 3; ++c)
          patch[(kh * 3 + kw) * 3 + c] =
              ok ? static_cast<float>(img[((static_cast<size_t>(b) * H + hh) * W + ww) * 3 + c]) / 255.f * 2.f - 1.f
                 : 0.f;
      }
    float acc[8];
#pragma unroll
    for (int o = 0; o < 8; ++o) acc[o] = bias ? __bfloat162float(bias[ov * 8 + o]) : 0.f;
#pragma unroll
    for (int k = 0; k < 27; ++k) {
      const uint4 wv = *reinterpret_cast<const uint4*>(wsh + k * Cout + ov * 8);
      const uint32_t ww4[4] = {wv.x, wv.y, wv.z, wv.w};
#pragma unroll
      for (int o = 0; o < 4; ++o) {
        acc[2 * o] += patch[k] * bf16_lo(ww4[o]);
        acc[2 * o + 1] += patch[k] * bf16_hi(ww4[o]);
      }
    }
    uint4 o4;
    o4.x = pack_bf16x2(acc[0], acc[1]);
    o4.y = pack_bf16x2(acc[2], acc[3]);
    o4.z = pack_bf16x2(acc[4], acc[5]);
    o4.w = pack_bf16x2(acc[6], acc[7]);
    *reinterpret_cast<uint4*>(out + pix * Cout + ov * 8) = o4;
  }
}

// ------------------------------------------------------------------------------------------------
// 3x3 pad 1 conv, Cin -> NO outputs of one pixel, summed over a group of G lanes (G divides 32): the dot products of
// Decoder.conv_out (NO = 3) and Encoder.conv_out (NO = 8).  wsh: [NO][9][Cin] bf16.  On return every lane of the group
// holds all NO sums (without bias).
// ------------------------------------------------------------------------------------------------
template <int NO, int G>
__device__ __forceinline__ void conv3x3_pixel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* wsh, int b,
                                              int hq, int wq, int H, int W, int Cin, int sub, float (&acc)[NO]) {
#pragma unroll
  for (int o = 0; o < NO; ++o) acc[o] = 0.f;
  const int nvec = Cin >> 3;
  for (int tap = 0; tap < 9; ++tap) {
    const int hh = hq + tap / 3 - 1, ww = wq + tap % 3 - 1;
    if (hh < 0 || hh >= H || ww < 0 || ww >= W) continue;  // uniform over the group
    const __nv_bfloat16* xr = x + ((static_cast<size_t>(b) * H + hh) * W + ww) * Cin;
    for (int v = sub; v < nvec; v += G) {
      const uint4 xv = __ldg(reinterpret_cast<const uint4*>(xr + v * 8));
#pragma unroll
      for (int o = 0; o < NO; ++o)
        acc[o] += dot8_bf16(xv, *reinterpret_cast<const uint4*>(wsh + (o * 9 + tap) * Cin + v * 8));
    }
  }
#pragma unroll
  for (int o = 0; o < NO; ++o) {
#pragma unroll
    for (int s = G / 2; s > 0; s >>= 1) acc[o] += __shfl_xor_sync(0xffffffffu, acc[o], s);
  }
}

// Decoder.conv_out (Cin -> 3) + VaeImageProcessor.postprocess + numpy_to_pil: u8 = rint(clamp(y / 2 + 0.5, 0, 1) * 255)
// (numpy's round is half to even, as rintf).  Half a warp per pixel.  y_f32: optional fp32 NCHW copy of y.
constexpr int kOutLanes = 16;
__global__ void vae_conv_out_u8_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ w,
                                       const __nv_bfloat16* __restrict__ bias, uint8_t* __restrict__ img,
                                       float* __restrict__ y_f32, int B, int H, int W, int Cin) {
  extern __shared__ __align__(16) __nv_bfloat16 wsh[];  // [3][9][Cin]
  for (int i = threadIdx.x; i < 27 * Cin; i += blockDim.x) wsh[i] = w[i];
  __syncthreads();
  const int groups_per_block = blockDim.x / kOutLanes;
  const int sub = threadIdx.x % kOutLanes;
  const size_t npix = static_cast<size_t>(B) * H * W;
  // every group runs the same number of iterations, so the full-warp shuffles see all 32 lanes
  const size_t stride = static_cast<size_t>(gridDim.x) * groups_per_block;
  for (size_t base = blockIdx.x * static_cast<size_t>(groups_per_block); base < npix; base += stride) {
    const size_t pix = base + threadIdx.x / kOutLanes;
    const bool live = pix < npix;
    const size_t pp = live ? pix : npix - 1;
    const int wq = static_cast<int>(pp % W);
    const int hq = static_cast<int>((pp / W) % H);
    const int b = static_cast<int>(pp / (static_cast<size_t>(W) * H));
    float acc[3];
    conv3x3_pixel<3, kOutLanes>(x, wsh, b, hq, wq, H, W, Cin, sub, acc);
    if (live && sub < 3) {
      const float y = (sub == 0 ? acc[0] : sub == 1 ? acc[1] : acc[2]) + (bias ? __bfloat162float(bias[sub]) : 0.f);
      if (y_f32) y_f32[((static_cast<size_t>(b) * 3 + sub) * H + hq) * W + wq] = y;
      const float t = fminf(fmaxf(y * 0.5f + 0.5f, 0.f), 1.f);
      img[pp * 3 + sub] = static_cast<uint8_t>(rintf(t * 255.f));
    }
  }
}

// Encoder.conv_out (Cin -> 8) + quant_conv (1x1, 8 -> 8, fp32) + DiagonalGaussianDistribution: mean = m[0:4],
// logvar = clamp(m[4:8], -30, 20), z = (mean + exp(0.5 logvar) * eps) * scaling  (eps NULL: z = mean * scaling).
// One warp per pixel; lanes 0-3 write channel `lane` of the fp32 NCHW latent.
__global__ void vae_moments_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ w,
                                   const __nv_bfloat16* __restrict__ bias, const float* __restrict__ qw,
                                   const float* __restrict__ qb, const float* __restrict__ eps, float scaling,
                                   float* __restrict__ z, int B, int H, int W, int Cin) {
  extern __shared__ __align__(16) __nv_bfloat16 wsh[];  // [8][9][Cin]
  for (int i = threadIdx.x; i < 72 * Cin; i += blockDim.x) wsh[i] = w[i];
  __syncthreads();
  const int warps_per_block = blockDim.x >> 5;
  const int lane = threadIdx.x & 31;
  const size_t npix = static_cast<size_t>(B) * H * W;
  for (size_t pix = blockIdx.x * static_cast<size_t>(warps_per_block) + (threadIdx.x >> 5); pix < npix;
       pix += static_cast<size_t>(gridDim.x) * warps_per_block) {
    const int wq = static_cast<int>(pix % W);
    const int hq = static_cast<int>((pix / W) % H);
    const int b = static_cast<int>(pix / (static_cast<size_t>(W) * H));
    float h[8];
    conv3x3_pixel<8, 32>(x, wsh, b, hq, wq, H, W, Cin, lane, h);
    if (lane < 4) {
      float mean = qb[lane], logvar = qb[lane + 4];
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const float hk = h[k] + (bias ? __bfloat162float(bias[k]) : 0.f);
        mean += qw[lane * 8 + k] * hk;
        logvar += qw[(lane + 4) * 8 + k] * hk;
      }
      const size_t o = ((static_cast<size_t>(b) * 4 + lane) * H + hq) * W + wq;
      float v = mean;
      if (eps) v += expf(0.5f * fminf(fmaxf(logvar, -30.f), 20.f)) * eps[o];
      z[o] = v * scaling;
    }
  }
}

// AutoencoderKL.decode's input: out[b, c] = post_quant_conv(z / scaling)[b, c] over fp32 NCHW [B, 4, HW].
__global__ void vae_post_quant_kernel(const float* __restrict__ z, const float* __restrict__ pw,
                                      const float* __restrict__ pb, float scaling, float* __restrict__ out, int B,
                                      int HW) {
  const size_t total = static_cast<size_t>(B) * HW;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const size_t b = i / HW, p = i - b * HW;
    const float* zb = z + b * 4 * HW + p;
    float v[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) v[k] = zb[k * HW] / scaling;
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      float s = pb[c];
#pragma unroll
      for (int k = 0; k < 4; ++k) s += pw[c * 4 + k] * v[k];
      out[b * 4 * HW + c * HW + p] = s;
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Row softmax of fp32 attention scores: P[r, :] = bf16(exp(scale (s - max)) / sum).  One block per row; an online
// (max, sum) pass and a write pass over the row, both in fp32.
// ------------------------------------------------------------------------------------------------
constexpr int kSmThreads = 256;
__device__ __forceinline__ void online_merge(float& m, float& l, float m2, float l2, float scale) {
  const float mn = fmaxf(m, m2);
  l = l * expf((m - mn) * scale) + l2 * expf((m2 - mn) * scale);
  m = mn;
}

__global__ void __launch_bounds__(kSmThreads) softmax_rows_kernel(const float* __restrict__ s, int lds,
                                                                  __nv_bfloat16* __restrict__ p, int ldp, int cols,
                                                                  float scale) {
  const float4* row = reinterpret_cast<const float4*>(s + static_cast<size_t>(blockIdx.x) * lds);
  const int nq = cols >> 2;
  float m = -INFINITY, l = 0.f;
  for (int i = threadIdx.x; i < nq; i += kSmThreads) {
    const float4 v = row[i];
    const float vm = fmaxf(fmaxf(v.x, v.y), fmaxf(v.z, v.w));
    if (vm > m) {
      l *= expf((m - vm) * scale);
      m = vm;
    }
    l += expf((v.x - m) * scale) + expf((v.y - m) * scale) + expf((v.z - m) * scale) + expf((v.w - m) * scale);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float m2 = __shfl_xor_sync(0xffffffffu, m, o), l2 = __shfl_xor_sync(0xffffffffu, l, o);
    if (m2 != -INFINITY) online_merge(m, l, m2, l2, scale);
  }
  __shared__ float red[2][kSmThreads / 32];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) red[0][warp] = m, red[1][warp] = l;
  __syncthreads();
  m = red[0][0], l = red[1][0];
  for (int i = 1; i < kSmThreads / 32; ++i)
    if (red[0][i] != -INFINITY) online_merge(m, l, red[0][i], red[1][i], scale);
  const float inv = 1.f / l;
  uint2* prow = reinterpret_cast<uint2*>(p + static_cast<size_t>(blockIdx.x) * ldp);
  for (int i = threadIdx.x; i < nq; i += kSmThreads) {
    const float4 v = row[i];
    prow[i] = make_uint2(pack_bf16x2(expf((v.x - m) * scale) * inv, expf((v.y - m) * scale) * inv),
                         pack_bf16x2(expf((v.z - m) * scale) * inv, expf((v.w - m) * scale) * inv));
  }
}

}  // namespace sb200

using namespace sb200;

extern "C" int sb200_vae_conv_in_u8(void* handle, void* stream, const uint8_t* img, const void* w, const void* bias,
                                    void* out, int B, int H, int W, int Cout) {
  Ctx* ctx = as_ctx(handle);
  SB200_REQUIRE(ctx && img && w && out, "vae_conv_in_u8: NULL argument");
  SB200_REQUIRE(B > 0 && H > 0 && W > 0, "vae_conv_in_u8: dims %dx%dx%d", B, H, W);
  SB200_REQUIRE(Cout % 8 == 0 && Cout > 0 && Cout * 27 * 2 <= 48 * 1024, "vae_conv_in_u8: Cout=%d unsupported", Cout);
  const size_t smem = static_cast<size_t>(Cout) * 27 * 2;
  vae_conv_in_u8_kernel<<<grid_cap(ctx, static_cast<size_t>(B) * H * W * (Cout / 8), 256, 8), 256, smem,
                          static_cast<cudaStream_t>(stream)>>>(img, static_cast<const __nv_bfloat16*>(w),
                                                               static_cast<const __nv_bfloat16*>(bias),
                                                               static_cast<__nv_bfloat16*>(out), B, H, W, Cout);
  SB200_CUDA_CHECK(cudaGetLastError());
  return 0;
}

extern "C" int sb200_vae_conv_out_u8(void* handle, void* stream, const void* x, const void* w, const void* bias,
                                     uint8_t* img, float* y_f32, int B, int H, int W, int Cin) {
  Ctx* ctx = as_ctx(handle);
  SB200_REQUIRE(ctx && x && w && img, "vae_conv_out_u8: NULL argument");
  SB200_REQUIRE(B > 0 && H > 0 && W > 0, "vae_conv_out_u8: dims %dx%dx%d", B, H, W);
  SB200_REQUIRE(Cin % 8 == 0 && Cin > 0 && Cin * 27 * 2 <= 48 * 1024, "vae_conv_out_u8: Cin=%d unsupported", Cin);
  const size_t smem = static_cast<size_t>(Cin) * 27 * 2;
  vae_conv_out_u8_kernel<<<grid_cap(ctx, static_cast<size_t>(B) * H * W, 256 / kOutLanes, 8), 256, smem,
                           static_cast<cudaStream_t>(stream)>>>(
      static_cast<const __nv_bfloat16*>(x), static_cast<const __nv_bfloat16*>(w),
      static_cast<const __nv_bfloat16*>(bias), img, y_f32, B, H, W, Cin);
  SB200_CUDA_CHECK(cudaGetLastError());
  return 0;
}

extern "C" int sb200_vae_moments(void* handle, void* stream, const void* x, const void* w, const void* bias,
                                 const float* quant_w, const float* quant_b, const float* eps, float scaling, float* z,
                                 int B, int H, int W, int Cin) {
  Ctx* ctx = as_ctx(handle);
  SB200_REQUIRE(ctx && x && w && quant_w && quant_b && z, "vae_moments: NULL argument");
  SB200_REQUIRE(B > 0 && H > 0 && W > 0, "vae_moments: dims %dx%dx%d", B, H, W);
  const size_t smem = static_cast<size_t>(Cin) * 72 * 2;
  SB200_REQUIRE(Cin % 8 == 0 && Cin > 0 && smem <= static_cast<size_t>(ctx->smem_optin),
                "vae_moments: Cin=%d unsupported", Cin);
  if (smem > 48 * 1024)
    SB200_CUDA_CHECK(cudaFuncSetAttribute(vae_moments_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                          static_cast<int>(smem)));
  vae_moments_kernel<<<grid_cap(ctx, static_cast<size_t>(B) * H * W, 8, 2), 256, smem,
                       static_cast<cudaStream_t>(stream)>>>(
      static_cast<const __nv_bfloat16*>(x), static_cast<const __nv_bfloat16*>(w),
      static_cast<const __nv_bfloat16*>(bias), quant_w, quant_b, eps, scaling, z, B, H, W, Cin);
  SB200_CUDA_CHECK(cudaGetLastError());
  return 0;
}

extern "C" int sb200_vae_post_quant(void* handle, void* stream, const float* z, const float* post_w,
                                    const float* post_b, float scaling, float* out, int B, int HW) {
  Ctx* ctx = as_ctx(handle);
  SB200_REQUIRE(ctx && z && post_w && post_b && out, "vae_post_quant: NULL argument");
  SB200_REQUIRE(B > 0 && HW > 0 && scaling != 0.f, "vae_post_quant: B=%d HW=%d scaling=%g", B, HW, scaling);
  vae_post_quant_kernel<<<grid_cap(ctx, static_cast<size_t>(B) * HW, 256, 8), 256, 0,
                          static_cast<cudaStream_t>(stream)>>>(z, post_w, post_b, scaling, out, B, HW);
  SB200_CUDA_CHECK(cudaGetLastError());
  return 0;
}

extern "C" int sb200_softmax_rows(void* handle, void* stream, const float* s, int lds, void* p, int ldp, int rows,
                                  int cols, float scale) {
  Ctx* ctx = as_ctx(handle);
  SB200_REQUIRE(ctx && s && p, "softmax_rows: NULL argument");
  SB200_REQUIRE(rows > 0 && cols > 0 && cols % 4 == 0 && lds % 4 == 0 && ldp % 4 == 0 && lds >= cols && ldp >= cols,
                "softmax_rows: rows=%d cols=%d lds=%d ldp=%d (cols and leading dims multiples of 4)", rows, cols, lds,
                ldp);
  SB200_REQUIRE((reinterpret_cast<uintptr_t>(s) & 15) == 0 && (reinterpret_cast<uintptr_t>(p) & 7) == 0,
                "softmax_rows: s must be 16-byte and p 8-byte aligned");
  SB200_REQUIRE(scale > 0.f, "softmax_rows: scale %g must be positive", scale);
  softmax_rows_kernel<<<rows, kSmThreads, 0, static_cast<cudaStream_t>(stream)>>>(
      s, lds, static_cast<__nv_bfloat16*>(p), ldp, cols, scale);
  SB200_CUDA_CHECK(cudaGetLastError());
  return 0;
}
