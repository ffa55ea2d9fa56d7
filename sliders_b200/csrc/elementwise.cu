// Latency-class pieces of the UNet denoise step: sinusoidal embeddings, the small dense layers of the
// time / add-embedding MLPs and time_emb_proj (M <= 64 rows, weight-bandwidth bound), conv_in / conv_out
// (4 <-> C channels, NCHW latent <-> NHWC activations), nearest x2 upsample, and the fused CFG + DDIM update.
//
// Replaces (reference): diffusers Timesteps / TimestepEmbedding, conv_in / conv_out, Upsample2D's
// F.interpolate, and trainscripts/textsliders/train_util.py:250-253 (CFG) + scheduler.step (:291).
#include "common.h"
#include "ptx.cuh"

namespace sb200 {

// ------------------------------------------------------------------------------------------------
__global__ void sinusoid_kernel(const float* __restrict__ values, int n, int dim,
                                __nv_bfloat16* __restrict__ out, int ldo) {
  const int half = dim >> 1;
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n * half) return;
  const int i = idx / half, j = idx - i * half;
  // f_j = exp(-ln(10000) * j / half)   (downscale_freq_shift = 0, flip_sin_to_cos = True -> [cos | sin])
  const float freq = expf(-9.210340371976184f * static_cast<float>(j) / static_cast<float>(half));
  const float arg = values[i] * freq;
  out[static_cast<size_t>(i) * ldo + j] = __float2bfloat16(cosf(arg));
  out[static_cast<size_t>(i) * ldo + half + j] = __float2bfloat16(sinf(arg));
}

// ------------------------------------------------------------------------------------------------
// small_linear: out[M, N] = act_out(act_in(x) W^T + b) (+ scale * (act_in(x) down^T) up^T)
// block = 8 warps, each warp owns kColsPerWarp output columns; x rows are read through L1.
// ------------------------------------------------------------------------------------------------
constexpr int kSlWarps = 8;
constexpr int kSlColsPerWarp = 1;  // more, smaller blocks: M <= 64 rows, the kernel is latency-bound (53 -> ~15 us at N = 1280)
constexpr int kSlMaxM = 64;
constexpr int kSlMaxR = 8;

struct SmallLinearArgs {
  const __nv_bfloat16* x;
  int ldx;
  const __nv_bfloat16* w;
  int ldw;
  const __nv_bfloat16* bias;
  const __nv_bfloat16* resid;
  __nv_bfloat16* out;
  int ldo;
  int M, N, K;
  int act_in, act_out;
  const __nv_bfloat16* down;  // [rt, K]
  const float* up;            // [N, r] fp32
  int r, group_n;
  float scale;
  const float* scale_dev;
};

__device__ __forceinline__ float dot8(const uint4& a, const uint4& b, bool silu_a) {
  const uint32_t aw[4] = {a.x, a.y, a.z, a.w};
  const uint32_t bw[4] = {b.x, b.y, b.z, b.w};
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    float a0 = bf16_lo(aw[i]), a1 = bf16_hi(aw[i]);
    if (silu_a) {
      // the reference applies SiLU in bf16: round like torch would before the matmul
      a0 = __bfloat162float(__float2bfloat16(silu_f(a0)));
      a1 = __bfloat162float(__float2bfloat16(silu_f(a1)));
    }
    s += a0 * bf16_lo(bw[i]) + a1 * bf16_hi(bw[i]);
  }
  return s;
}

__global__ void __launch_bounds__(kSlWarps * 32) small_linear_kernel(SmallLinearArgs a) {
  pdl_trigger();
  pdl_wait();
  __shared__ float t_sh[kSlMaxM][kSlMaxR * 4];  // LoRA down-projection of every row: [M][groups*r]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nvec = a.K >> 3;
  const bool silu_in = a.act_in == 1;
  const int n_block = blockIdx.x * kSlWarps * kSlColsPerWarp;
  int lora_cols = 0;
  if (a.down) {
    // columns of this block may span several groups; compute T for the groups it touches
    const int g_lo = n_block / a.group_n;
    const int n_hi = min(n_block + kSlWarps * kSlColsPerWarp, a.N) - 1;
    const int g_hi = n_hi / a.group_n;
    lora_cols = (g_hi - g_lo + 1) * a.r;
    for (int idx = warp; idx < lora_cols * a.M; idx += kSlWarps) {
      const int m = idx / lora_cols, j = idx - m * lora_cols;
      const __nv_bfloat16* dr = a.down + static_cast<size_t>(g_lo * a.r + j) * a.K;
      const __nv_bfloat16* xr = a.x + static_cast<size_t>(m) * a.ldx;
      float s = 0.f;
      for (int v = lane; v < nvec; v += 32)
        s += dot8(__ldg(reinterpret_cast<const uint4*>(xr + v * 8)),
                  __ldg(reinterpret_cast<const uint4*>(dr + v * 8)), silu_in);
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
      if (lane == 0) t_sh[m][j] = s;
    }
    __syncthreads();
  }
  for (int cidx = 0; cidx < kSlColsPerWarp; ++cidx) {
    const int n = n_block + warp * kSlColsPerWarp + cidx;
    if (n >= a.N) break;
    const __nv_bfloat16* wr = a.w + static_cast<size_t>(n) * a.ldw;
    for (int m0 = 0; m0 < a.M; m0 += 8) {
      float acc[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) acc[i] = 0.f;
      for (int v = lane; v < nvec; v += 32) {
        const uint4 wv = __ldg(reinterpret_cast<const uint4*>(wr + v * 8));
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          if (m0 + i < a.M) {
            const uint4 xv = __ldg(reinterpret_cast<const uint4*>(a.x + static_cast<size_t>(m0 + i) * a.ldx + v * 8));
            acc[i] += dot8(xv, wv, silu_in);
          }
        }
      }
#pragma unroll
      for (int i = 0; i < 8; ++i) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) acc[i] += __shfl_xor_sync(0xffffffffu, acc[i], o);
      }
      if (lane == 0) {
        const float bv = a.bias ? __bfloat162float(a.bias[n]) : 0.f;
        for (int i = 0; i < 8 && m0 + i < a.M; ++i) {
          float y = acc[i] + bv;
          if (a.down) {
            const int g_lo = n_block / a.group_n;
            const int gj = (n / a.group_n - g_lo) * a.r;
            float l = 0.f;
            for (int j = 0; j < a.r; ++j)
              l += t_sh[m0 + i][gj + j] * a.up[static_cast<size_t>(n) * a.r + j];
            y += (a.scale_dev ? a.scale * __ldg(a.scale_dev) : a.scale) * l;
          }
          if (a.act_out == 1) y = silu_f(y);
          if (a.resid) y += __bfloat162float(a.resid[static_cast<size_t>(m0 + i) * a.N + n]);
          // act_out == 2: SiLU of the rounded sum (emb = t_emb + aug_emb is a bf16 tensor in the reference
          // before ResnetBlock2D applies its nonlinearity)
          if (a.act_out == 2) y = silu_f(__bfloat162float(__float2bfloat16(y)));
          a.out[static_cast<size_t>(m0 + i) * a.ldo + n] = __float2bfloat16(y);
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// conv_in: 3x3, 4 -> Cout. thread = (pixel, 8 output channels).
// ------------------------------------------------------------------------------------------------
template <typename TIn>
__global__ void conv_in_kernel(const TIn* __restrict__ x, const __nv_bfloat16* __restrict__ w,
                               const __nv_bfloat16* __restrict__ bias, __nv_bfloat16* __restrict__ out,
                               int B, int H, int W, int Cout) {
  // weights transposed to [36][Cout] so that a thread's 8 output channels of one tap element are a single
  // 16-byte word and neighbouring threads (neighbouring channel octets) hit neighbouring banks
  extern __shared__ __align__(16) __nv_bfloat16 wsh[];
  for (int i = threadIdx.x; i < Cout * 36; i += blockDim.x) {
    const int co = i / 36, k = i - co * 36;
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
    float patch[36];  // [kh][kw][c]
#pragma unroll
    for (int kh = 0; kh < 3; ++kh)
#pragma unroll
      for (int kw = 0; kw < 3; ++kw) {
        const int hh = hq + kh - 1, ww = wq + kw - 1;
        const bool ok = hh >= 0 && hh < H && ww >= 0 && ww < W;
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          float v = 0.f;
          if (ok) {
            v = static_cast<float>(x[((static_cast<size_t>(b) * 4 + c) * H + hh) * W + ww]);
            v = __bfloat162float(__float2bfloat16(v));  // model dtype is bf16 (reference casts latents)
          }
          patch[(kh * 3 + kw) * 4 + c] = v;
        }
      }
    float acc[8];
#pragma unroll
    for (int o = 0; o < 8; ++o) acc[o] = bias ? __bfloat162float(bias[ov * 8 + o]) : 0.f;
#pragma unroll
    for (int k = 0; k < 36; ++k) {
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
// conv_out: 3x3, Cin -> 4 on NHWC bf16; one warp per output pixel, lanes split the channels.
// ------------------------------------------------------------------------------------------------
template <typename TOut>
__global__ void conv_out_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ w,
                                const __nv_bfloat16* __restrict__ bias, TOut* __restrict__ out, int B, int H,
                                int W, int Cin) {
  extern __shared__ __nv_bfloat16 wsh[];  // [4][9][Cin]
  for (int i = threadIdx.x; i < 36 * Cin; i += blockDim.x) wsh[i] = w[i];
  __syncthreads();
  const int warps_per_block = blockDim.x >> 5;
  const int lane = threadIdx.x & 31;
  const int nvec = Cin >> 3;
  const size_t npix = static_cast<size_t>(B) * H * W;
  for (size_t pix = blockIdx.x * static_cast<size_t>(warps_per_block) + (threadIdx.x >> 5); pix < npix;
       pix += static_cast<size_t>(gridDim.x) * warps_per_block) {
    const int wq = static_cast<int>(pix % W);
    const int hq = static_cast<int>((pix / W) % H);
    const int b = static_cast<int>(pix / (static_cast<size_t>(W) * H));
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    for (int tap = 0; tap < 9; ++tap) {
      const int hh = hq + tap / 3 - 1, ww = wq + tap % 3 - 1;
      if (hh < 0 || hh >= H || ww < 0 || ww >= W) continue;  // warp-uniform
      const __nv_bfloat16* xr = x + ((static_cast<size_t>(b) * H + hh) * W + ww) * Cin;
      for (int v = lane; v < nvec; v += 32) {
        const uint4 xv = __ldg(reinterpret_cast<const uint4*>(xr + v * 8));
#pragma unroll
        for (int o = 0; o < 4; ++o) {
          const uint4 wv = *reinterpret_cast<const uint4*>(wsh + (o * 9 + tap) * Cin + v * 8);
          acc[o] += dot8(xv, wv, false);
        }
      }
    }
#pragma unroll
    for (int o = 0; o < 4; ++o) {
#pragma unroll
      for (int s = 16; s > 0; s >>= 1) acc[o] += __shfl_xor_sync(0xffffffffu, acc[o], s);
    }
    if (lane < 4) {
      const float y = acc[lane] + (bias ? __bfloat162float(bias[lane]) : 0.f);
      out[((static_cast<size_t>(b) * 4 + lane) * H + hq) * W + wq] = static_cast<TOut>(y);
    }
  }
}

// ------------------------------------------------------------------------------------------------
__global__ void upsample2x_kernel(const uint4* __restrict__ x, uint4* __restrict__ out, int B, int H, int W,
                                  int cvec) {
  const size_t total = static_cast<size_t>(B) * (2 * H) * (2 * W) * cvec;
  for (size_t idx = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int cv = static_cast<int>(idx % cvec);
    size_t pix = idx / cvec;
    const int wo = static_cast<int>(pix % (2 * W));
    pix /= (2 * W);
    const int ho = static_cast<int>(pix % (2 * H));
    const int b = static_cast<int>(pix / (2 * H));
    out[idx] = __ldg(x + ((static_cast<size_t>(b) * H + (ho >> 1)) * W + (wo >> 1)) * cvec + cv);
  }
}

// ------------------------------------------------------------------------------------------------
template <typename TE, typename TO>
__global__ void cfg_ddim_kernel(const TE* __restrict__ eps2, float g, const TO* __restrict__ x, float a_t,
                                float a_prev, TO* __restrict__ x_prev, TO* __restrict__ eps_out, int64_t n,
                                int affine) {
  // affine: (a_t, a_prev) are the coefficients (cx, ce) of x_prev = cx x + ce eps (Euler-discrete step: cx = 1,
  // ce = sigma_next - sigma); otherwise the DDIM update from the two alpha-bar values
  const float sa = affine ? 1.f : sqrtf(a_t), sb = affine ? 0.f : sqrtf(1.f - a_t);
  const float pa = affine ? a_t : sqrtf(a_prev), pb = affine ? a_prev : sqrtf(1.f - a_prev);
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const float eu = static_cast<float>(eps2[i]);
    const float ec = (g != 0.f) ? static_cast<float>(eps2[n + i]) : eu;  // g == 0: plain DDIM step on eps
    const float e = eu + g * (ec - eu);
    if (eps_out) eps_out[i] = static_cast<TO>(e);
    if (x) {
      const float xv = static_cast<float>(x[i]);
      const float x0 = (xv - sb * e) / sa;
      x_prev[i] = static_cast<TO>(pa * x0 + pb * e);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// null-text inversion inner-step loss: x_rec = cx x + ce (eps_u + g (eps_c - eps_u)), loss = mean((x_rec - target)^2)
constexpr int kLossThreads = 256;

__device__ __forceinline__ float guided_residual(const float* eps_u, const float* eps_c, float g, const float* x,
                                                 float cx, float ce, const float* target, int64_t i) {
  const float eu = eps_u[i];
  const float e = eu + g * (eps_c[i] - eu);
  return cx * x[i] + ce * e - target[i];
}

// mode 0: block b sums the squared residuals of its grid-stride share into ws[b] (fixed order: strided per thread,
// then a shared-memory tree); mode 1: d_eps_u = dloss (1 - g) ce 2 r / n
__global__ void __launch_bounds__(kLossThreads) guided_loss_kernel(const float* __restrict__ eps_u,
                                                                    const float* __restrict__ eps_c, float g,
                                                                    const float* __restrict__ x, float cx, float ce,
                                                                    const float* __restrict__ target, int64_t n,
                                                                    int mode, float* __restrict__ ws,
                                                                    const float* __restrict__ dloss,
                                                                    float* __restrict__ d_eps_u) {
  pdl_trigger();
  pdl_wait();
  const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
  if (mode == 1) {
    const float k = __ldg(dloss) * (1.f - g) * ce * 2.f / static_cast<float>(n);
    for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < n; i += stride)
      d_eps_u[i] = k * guided_residual(eps_u, eps_c, g, x, cx, ce, target, i);
    return;
  }
  float acc = 0.f;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < n; i += stride) {
    const float r = guided_residual(eps_u, eps_c, g, x, cx, ce, target, i);
    acc = fmaf(r, r, acc);
  }
  __shared__ float red[kLossThreads];
  red[threadIdx.x] = acc;
  __syncthreads();
  for (int w = kLossThreads / 2; w > 0; w >>= 1) {
    if (threadIdx.x < w) red[threadIdx.x] += red[threadIdx.x + w];
    __syncthreads();
  }
  if (threadIdx.x == 0) ws[blockIdx.x] = red[0];
}

__global__ void __launch_bounds__(kLossThreads) guided_loss_finalize_kernel(const float* __restrict__ ws, int parts,
                                                                             int64_t n, float* __restrict__ loss) {
  pdl_trigger();
  pdl_wait();
  __shared__ float red[kLossThreads];
  red[threadIdx.x] = threadIdx.x < parts ? ws[threadIdx.x] : 0.f;
  __syncthreads();
  for (int w = kLossThreads / 2; w > 0; w >>= 1) {
    if (threadIdx.x < w) red[threadIdx.x] += red[threadIdx.x + w];
    __syncthreads();
  }
  if (threadIdx.x == 0) *loss = red[0] / static_cast<float>(n);
}

}  // namespace sb200

using namespace sb200;

extern "C" int sb200_guided_step_loss(void* handle, void* stream, const float* eps_u, const float* eps_c, float g,
                                      const float* x, float cx, float ce, const float* target, int64_t n, int mode,
                                      float* loss, float* ws, const float* dloss, float* d_eps_u) {
  pdl_hint() = true;
  SB200_REQUIRE(handle && eps_u && eps_c && x && target && n > 0, "guided_step_loss: NULL argument");
  SB200_REQUIRE(mode == 0 ? (loss && ws) : (mode == 1 && dloss && d_eps_u), "guided_step_loss: mode %d outputs", mode);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int parts = SB200_GUIDED_LOSS_BLOCKS(n);
  const int blocks = mode == 0 ? parts : static_cast<int>((n + kLossThreads - 1) / kLossThreads < 1024
                                                               ? (n + kLossThreads - 1) / kLossThreads : 1024);
  SB200_CUDA_CHECK(launch_pdl(guided_loss_kernel, dim3(blocks), dim3(kLossThreads), 0, s, eps_u, eps_c, g, x, cx, ce,
                              target, n, mode, ws, dloss, d_eps_u));
  if (mode == 0)
    SB200_CUDA_CHECK(launch_pdl(guided_loss_finalize_kernel, dim3(1), dim3(kLossThreads), 0, s,
                                static_cast<const float*>(ws), parts, n, loss));
  SB200_CUDA_CHECK(cudaGetLastError());
  return 0;
}

extern "C" int sb200_sinusoid(void* handle, void* stream, const float* values, int n, int dim, void* out,
                              int ldo) {
  pdl_hint() = true;
  SB200_REQUIRE(handle && values && out, "sinusoid: NULL argument");
  SB200_REQUIRE(n > 0 && dim > 0 && dim % 2 == 0 && ldo >= dim, "sinusoid: dims");
  const int total = n * (dim / 2);
  sinusoid_kernel<<<(total + 255) / 256, 256, 0, static_cast<cudaStream_t>(stream)>>>(
      values, n, dim, static_cast<__nv_bfloat16*>(out), ldo);
  SB200_CUDA_CHECK(cudaGetLastError());
  return 0;
}

extern "C" int sb200_small_linear(void* handle, void* stream, const void* x, int ldx, const void* w, int ldw,
                                  const void* bias, void* out, int ldo, int M, int N, int K, int act_in,
                                  int act_out, const sb200_lora* lora, const void* resid) {
  pdl_hint() = true;
  SB200_REQUIRE(handle && x && w && out, "small_linear: NULL argument");
  SB200_REQUIRE(M > 0 && M <= kSlMaxM, "small_linear: M=%d must be in [1, %d]", M, kSlMaxM);
  SB200_REQUIRE(N > 0 && K > 0 && K % 8 == 0 && ldx % 8 == 0 && ldw % 8 == 0, "small_linear: dims");
  SmallLinearArgs a;
  memset(&a, 0, sizeof(a));
  a.x = static_cast<const __nv_bfloat16*>(x);
  a.ldx = ldx;
  a.w = static_cast<const __nv_bfloat16*>(w);
  a.ldw = ldw;
  a.bias = static_cast<const __nv_bfloat16*>(bias);
  a.resid = static_cast<const __nv_bfloat16*>(resid);
  a.out = static_cast<__nv_bfloat16*>(out);
  a.ldo = ldo;
  a.M = M;
  a.N = N;
  a.K = K;
  a.act_in = act_in;
  a.act_out = act_out;
  if (lora) {
    SB200_REQUIRE(lora->down && lora->up && lora->r > 0 && lora->r <= kSlMaxR, "small_linear: lora rank");
    SB200_REQUIRE(lora->group_n >= kSlWarps * kSlColsPerWarp, "small_linear: lora group_n too small");
    a.down = static_cast<const __nv_bfloat16*>(lora->down);
    a.up = static_cast<const float*>(lora->up);
    a.r = lora->r;
    a.group_n = lora->group_n;
    a.scale = lora->scale;
    a.scale_dev = lora->scale_dev;
  }
  const int cols_per_block = kSlWarps * kSlColsPerWarp;
  SB200_CUDA_CHECK(launch_pdl(small_linear_kernel, dim3((N + cols_per_block - 1) / cols_per_block),
                              dim3(kSlWarps * 32), 0, static_cast<cudaStream_t>(stream), a));
  return 0;
}

extern "C" int sb200_conv_in(void* handle, void* stream, const void* latent_nchw, int latent_is_f32,
                             const void* w, const void* bias, void* out, int B, int H, int W, int Cout) {
  pdl_hint() = true;
  Ctx* ctx = as_ctx(handle);
  SB200_REQUIRE(ctx && latent_nchw && w && out, "conv_in: NULL argument");
  SB200_REQUIRE(Cout % 8 == 0 && Cout * 36 * 2 <= 48 * 1024, "conv_in: Cout=%d unsupported", Cout);
  const size_t total = static_cast<size_t>(B) * H * W * (Cout / 8);
  int blocks = static_cast<int>((total + 255) / 256);
  if (blocks > ctx->num_sms * 8) blocks = ctx->num_sms * 8;
  const size_t smem = static_cast<size_t>(Cout) * 36 * 2;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (latent_is_f32)
    conv_in_kernel<float><<<blocks, 256, smem, s>>>(static_cast<const float*>(latent_nchw),
                                                    static_cast<const __nv_bfloat16*>(w),
                                                    static_cast<const __nv_bfloat16*>(bias),
                                                    static_cast<__nv_bfloat16*>(out), B, H, W, Cout);
  else
    conv_in_kernel<__nv_bfloat16><<<blocks, 256, smem, s>>>(
        static_cast<const __nv_bfloat16*>(latent_nchw), static_cast<const __nv_bfloat16*>(w),
        static_cast<const __nv_bfloat16*>(bias), static_cast<__nv_bfloat16*>(out), B, H, W, Cout);
  SB200_CUDA_CHECK(cudaGetLastError());
  return 0;
}

extern "C" int sb200_conv_out(void* handle, void* stream, const void* x, const void* w, const void* bias,
                              void* out, int out_is_f32, int B, int H, int W, int Cin) {
  pdl_hint() = true;
  Ctx* ctx = as_ctx(handle);
  SB200_REQUIRE(ctx && x && w && out, "conv_out: NULL argument");
  SB200_REQUIRE(Cin % 8 == 0 && Cin * 36 * 2 <= 48 * 1024, "conv_out: Cin=%d unsupported", Cin);
  const size_t npix = static_cast<size_t>(B) * H * W;
  int blocks = static_cast<int>((npix + 7) / 8);
  if (blocks > ctx->num_sms * 8) blocks = ctx->num_sms * 8;
  const size_t smem = static_cast<size_t>(Cin) * 36 * 2;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (out_is_f32)
    conv_out_kernel<float><<<blocks, 256, smem, s>>>(static_cast<const __nv_bfloat16*>(x),
                                                     static_cast<const __nv_bfloat16*>(w),
                                                     static_cast<const __nv_bfloat16*>(bias),
                                                     static_cast<float*>(out), B, H, W, Cin);
  else
    conv_out_kernel<__nv_bfloat16><<<blocks, 256, smem, s>>>(
        static_cast<const __nv_bfloat16*>(x), static_cast<const __nv_bfloat16*>(w),
        static_cast<const __nv_bfloat16*>(bias), static_cast<__nv_bfloat16*>(out), B, H, W, Cin);
  SB200_CUDA_CHECK(cudaGetLastError());
  return 0;
}

extern "C" int sb200_upsample2x(void* handle, void* stream, const void* x, void* out, int B, int H, int W,
                                int C) {
  pdl_hint() = true;
  Ctx* ctx = as_ctx(handle);
  SB200_REQUIRE(ctx && x && out, "upsample2x: NULL argument");
  SB200_REQUIRE(C % 8 == 0, "upsample2x: C=%d must be a multiple of 8", C);
  const size_t total = static_cast<size_t>(B) * 4 * H * W * (C / 8);
  int blocks = static_cast<int>((total + 255) / 256);
  if (blocks > ctx->num_sms * 16) blocks = ctx->num_sms * 16;
  upsample2x_kernel<<<blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const uint4*>(x), static_cast<uint4*>(out), B, H, W, C / 8);
  SB200_CUDA_CHECK(cudaGetLastError());
  return 0;
}

static int launch_cfg(void* handle, void* stream, const void* eps2, int eps_is_f32, float g, const void* x,
                      float a_t, float a_prev, void* x_prev, void* eps_out, int out_is_f32, int64_t n, int affine);

extern "C" int sb200_cfg_ddim(void* handle, void* stream, const void* eps2, int eps_is_f32, float g,
                              const void* x, float a_t, float a_prev, void* x_prev, void* eps_out,
                              int out_is_f32, int64_t n) {
  return launch_cfg(handle, stream, eps2, eps_is_f32, g, x, a_t, a_prev, x_prev, eps_out, out_is_f32, n, 0);
}

extern "C" int sb200_cfg_step(void* handle, void* stream, const void* eps2, int eps_is_f32, float g,
                              const void* x, float cx, float ce, void* x_prev, void* eps_out, int out_is_f32,
                              int64_t n) {
  return launch_cfg(handle, stream, eps2, eps_is_f32, g, x, cx, ce, x_prev, eps_out, out_is_f32, n, 1);
}

static int launch_cfg(void* handle, void* stream, const void* eps2, int eps_is_f32, float g, const void* x,
                      float a_t, float a_prev, void* x_prev, void* eps_out, int out_is_f32, int64_t n, int affine) {
  pdl_hint() = true;
  Ctx* ctx = as_ctx(handle);
  SB200_REQUIRE(ctx && eps2 && n > 0, "cfg_ddim: bad arguments");
  SB200_REQUIRE(x || eps_out, "cfg_ddim: nothing to write");
  SB200_REQUIRE(!x || x_prev, "cfg_ddim: x without x_prev");
  int blocks = static_cast<int>((n + 255) / 256);
  if (blocks > ctx->num_sms * 8) blocks = ctx->num_sms * 8;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
#define SB200_LAUNCH_CFG(TE, TO)                                                                     \
  cfg_ddim_kernel<TE, TO><<<blocks, 256, 0, s>>>(static_cast<const TE*>(eps2), g,                    \
                                                 static_cast<const TO*>(x), a_t, a_prev,             \
                                                 static_cast<TO*>(x_prev), static_cast<TO*>(eps_out), n, \
                                                 affine)
  if (eps_is_f32 && out_is_f32)
    SB200_LAUNCH_CFG(float, float);
  else if (eps_is_f32 && !out_is_f32)
    SB200_LAUNCH_CFG(float, __nv_bfloat16);
  else if (!eps_is_f32 && out_is_f32)
    SB200_LAUNCH_CFG(__nv_bfloat16, float);
  else
    SB200_LAUNCH_CFG(__nv_bfloat16, __nv_bfloat16);
#undef SB200_LAUNCH_CFG
  SB200_CUDA_CHECK(cudaGetLastError());
  return 0;
}
