// HBM-bound pieces of the backward-to-LoRA pass (loss.backward() in trainscripts/textsliders/train_lora_xl.py:345,
// train_lora-scale-xl.py:340,372): GroupNorm(+SiLU) / LayerNorm / GEGLU backward, the rank-r LoRA weight-gradient
// reductions and the rank-r input-gradient updates, nearest-x2 / stride-2 helpers, conv_out backward, and the
// bf16 AdamW step (train_util.py:362-363).  The dense input-gradient products reuse gemm_kernel / the implicit
// GEMM conv with transposed weights; attention backward lives in attention_bwd.cu.
// Everything is deterministic: reductions are two-stage (per-chunk partials, fixed-order final sum), no atomics.
#include "common.h"
#include "ptx.cuh"

namespace sb200 {

__device__ __forceinline__ void unpack8(const uint4& v, float* f) {
  const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    f[2 * i] = bf16_lo(w[i]);
    f[2 * i + 1] = bf16_hi(w[i]);
  }
}
__device__ __forceinline__ uint4 pack8(const float* f) {
  uint4 o;
  o.x = pack_bf16x2(f[0], f[1]);
  o.y = pack_bf16x2(f[2], f[3]);
  o.z = pack_bf16x2(f[4], f[5]);
  o.w = pack_bf16x2(f[6], f[7]);
  return o;
}
__device__ __forceinline__ float silu_grad(float z) {
  const float s = 1.f / (1.f + __expf(-z));
  return s * (1.f + z * (1.f - s));
}

// ------------------------------------------------------------------------------------------------
// GroupNorm (+SiLU) backward.  y = act(z), z = gamma * xhat + beta, xhat = (x - mean) * rstd.
//   dz = dy * act'(z);  per (batch, group): m1 = mean(dz gamma), m2 = mean(dz gamma xhat)
//   dx = rstd * (dz gamma - m1 - xhat m2) (+ add)
// Same chunked layout as the forward (norm.cu): grid (chunks, B), thread = (row lane, 8-channel vector).
// ------------------------------------------------------------------------------------------------
struct GnBwdArgs {
  const __nv_bfloat16* x0;
  const __nv_bfloat16* x1;
  int ld0, ld1, C0, C;
  int HW, groups, cpg, rows_per_block;
  const __nv_bfloat16* gamma;
  const __nv_bfloat16* beta;
  const __nv_bfloat16* dy;
  int lddy;
  const __nv_bfloat16* add;  // optional, same layout as dx
  int ldadd;
  __nv_bfloat16* dx;
  int lddx;
  const float* stats;  // [B][G][2] (mean, rstd) from the forward
  int silu;
};

__device__ __forceinline__ void gn_bwd_load(const GnBwdArgs& a, int b, int c, const float*& st,
                                            const __nv_bfloat16*& src, int& ld, int& cc, float* gm, float* bt,
                                            float* mean, float* rstd) {
  if (c < a.C0) {
    src = a.x0, ld = a.ld0, cc = c;
  } else {
    src = a.x1, ld = a.ld1, cc = c - a.C0;
  }
  unpack8(__ldg(reinterpret_cast<const uint4*>(a.gamma + c)), gm);
  unpack8(__ldg(reinterpret_cast<const uint4*>(a.beta + c)), bt);
  st = a.stats + static_cast<size_t>(b) * 2 * a.groups;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int g = (c + i) / a.cpg;
    mean[i] = st[2 * g];
    rstd[i] = st[2 * g + 1];
  }
}

__global__ void gn_bwd_stats_kernel(GnBwdArgs a, float* __restrict__ partial) {
  pdl_trigger();
  pdl_wait();
  extern __shared__ float sh[];  // [rows_par][C][2]
  const int nvec = a.C >> 3;
  const int cv = threadIdx.x % nvec, r0 = threadIdx.x / nvec, rows_par = blockDim.x / nvec;
  const int b = blockIdx.y, c = cv << 3;
  const float* st;
  const __nv_bfloat16* src;
  int ld, cc;
  float gm[8], bt[8], mean[8], rstd[8];
  gn_bwd_load(a, b, c, st, src, ld, cc, gm, bt, mean, rstd);
  float s1[8], s2[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) s1[i] = s2[i] = 0.f;
  const int row_begin = blockIdx.x * a.rows_per_block;
  const int row_end = min(row_begin + a.rows_per_block, a.HW);
  for (int r = row_begin + r0; r < row_end; r += rows_par) {
    const size_t pix = static_cast<size_t>(b) * a.HW + r;
    float x[8], g[8];
    unpack8(__ldg(reinterpret_cast<const uint4*>(src + pix * ld + cc)), x);
    unpack8(__ldg(reinterpret_cast<const uint4*>(a.dy + pix * a.lddy + c)), g);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float xh = (x[i] - mean[i]) * rstd[i];
      float dz = g[i];
      if (a.silu) dz *= silu_grad(fmaf(gm[i], xh, bt[i]));
      const float dg = dz * gm[i];
      s1[i] += dg;
      s2[i] += dg * xh;
    }
  }
  float* mine = sh + (static_cast<size_t>(r0) * a.C + c) * 2;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    mine[2 * i] = s1[i];
    mine[2 * i + 1] = s2[i];
  }
  __syncthreads();
  for (int g = threadIdx.x; g < a.groups; g += blockDim.x) {
    float S1 = 0.f, S2 = 0.f;
    for (int r = 0; r < rows_par; ++r) {
      const float* row = sh + (static_cast<size_t>(r) * a.C + g * a.cpg) * 2;
      for (int ci = 0; ci < a.cpg; ++ci) {
        S1 += row[2 * ci];
        S2 += row[2 * ci + 1];
      }
    }
    float* out = partial + ((static_cast<size_t>(b) * gridDim.x + blockIdx.x) * a.groups + g) * 2;
    out[0] = S1;
    out[1] = S2;
  }
}

__global__ void gn_bwd_finalize_kernel(const float* __restrict__ partial, float* __restrict__ final_m, int chunks,
                                       int groups, float inv_n) {
  pdl_trigger();
  pdl_wait();
  const int b = blockIdx.x, lane = threadIdx.x & 31;
  for (int g = threadIdx.x >> 5; g < groups; g += blockDim.x >> 5) {
    float S1 = 0.f, S2 = 0.f;
    for (int k = lane; k < chunks; k += 32) {
      const float2 pp = *reinterpret_cast<const float2*>(partial + ((static_cast<size_t>(b) * chunks + k) * groups + g) * 2);
      S1 += pp.x;
      S2 += pp.y;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      S1 += __shfl_xor_sync(0xffffffffu, S1, o);
      S2 += __shfl_xor_sync(0xffffffffu, S2, o);
    }
    if (lane == 0) {
      final_m[(static_cast<size_t>(b) * groups + g) * 2] = S1 * inv_n;
      final_m[(static_cast<size_t>(b) * groups + g) * 2 + 1] = S2 * inv_n;
    }
  }
}

__global__ void gn_bwd_apply_kernel(GnBwdArgs a, const float* __restrict__ final_m) {
  pdl_trigger();
  pdl_wait();
  const int nvec = a.C >> 3;
  const int cv = threadIdx.x % nvec, r0 = threadIdx.x / nvec, rows_par = blockDim.x / nvec;
  const int b = blockIdx.y, c = cv << 3;
  const float* st;
  const __nv_bfloat16* src;
  int ld, cc;
  float gm[8], bt[8], mean[8], rstd[8], m1[8], m2[8];
  gn_bwd_load(a, b, c, st, src, ld, cc, gm, bt, mean, rstd);
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int g = (c + i) / a.cpg;
    m1[i] = final_m[(static_cast<size_t>(b) * a.groups + g) * 2];
    m2[i] = final_m[(static_cast<size_t>(b) * a.groups + g) * 2 + 1];
  }
  const int row_begin = blockIdx.x * a.rows_per_block;
  const int row_end = min(row_begin + a.rows_per_block, a.HW);
  for (int r = row_begin + r0; r < row_end; r += rows_par) {
    const size_t pix = static_cast<size_t>(b) * a.HW + r;
    float x[8], g[8], o[8];
    unpack8(__ldg(reinterpret_cast<const uint4*>(src + pix * ld + cc)), x);
    unpack8(__ldg(reinterpret_cast<const uint4*>(a.dy + pix * a.lddy + c)), g);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float xh = (x[i] - mean[i]) * rstd[i];
      float dz = g[i];
      if (a.silu) dz *= silu_grad(fmaf(gm[i], xh, bt[i]));
      o[i] = rstd[i] * (dz * gm[i] - m1[i] - xh * m2[i]);
    }
    if (a.add) {
      float ad[8];
      unpack8(__ldg(reinterpret_cast<const uint4*>(a.add + pix * a.ldadd + c)), ad);
#pragma unroll
      for (int i = 0; i < 8; ++i) o[i] += ad[i];
    }
    *reinterpret_cast<uint4*>(a.dx + pix * a.lddx + c) = pack8(o);
  }
}

// ------------------------------------------------------------------------------------------------
// LayerNorm backward: one warp per row; x row and dy*gamma row live in registers.
//   dx = rstd * (dy gamma - mean(dy gamma) - xhat * mean(dy gamma xhat)) (+ add)
// ------------------------------------------------------------------------------------------------
template <int NV>
__global__ void layernorm_bwd_kernel(const __nv_bfloat16* __restrict__ x, int ldx,
                                     const __nv_bfloat16* __restrict__ gamma,
                                     const __nv_bfloat16* __restrict__ dy, int lddy,
                                     const __nv_bfloat16* __restrict__ add, int ldadd,
                                     __nv_bfloat16* __restrict__ dx, int lddx, int M, int C, float eps) {
  pdl_trigger();
  pdl_wait();
  const int wpb = blockDim.x >> 5, lane = threadIdx.x & 31, nvec = C >> 3;
  for (int row = blockIdx.x * wpb + (threadIdx.x >> 5); row < M; row += gridDim.x * wpb) {
    const __nv_bfloat16* xr = x + static_cast<size_t>(row) * ldx;
    const __nv_bfloat16* gr = dy + static_cast<size_t>(row) * lddy;
    float f[NV][8], dg[NV][8];
    float sum = 0.f;
#pragma unroll
    for (int k = 0; k < NV; ++k) {
      const int v = lane + k * 32;
      if (v < nvec) {
        unpack8(__ldg(reinterpret_cast<const uint4*>(xr + v * 8)), f[k]);
#pragma unroll
        for (int i = 0; i < 8; ++i) sum += f[k][i];
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    const float mean = sum / C;
    float var = 0.f;
#pragma unroll
    for (int k = 0; k < NV; ++k)
      if (lane + k * 32 < nvec) {
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const float d = f[k][i] - mean;
          var += d * d;
        }
      }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) var += __shfl_xor_sync(0xffffffffu, var, o);
    const float rstd = rsqrtf(var / C + eps);
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int k = 0; k < NV; ++k) {
      const int v = lane + k * 32;
      if (v < nvec) {
        float g[8], gm[8];
        unpack8(__ldg(reinterpret_cast<const uint4*>(gr + v * 8)), g);
        unpack8(__ldg(reinterpret_cast<const uint4*>(gamma + v * 8)), gm);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          f[k][i] = (f[k][i] - mean) * rstd;  // xhat
          dg[k][i] = g[i] * gm[i];
          s1 += dg[k][i];
          s2 += dg[k][i] * f[k][i];
        }
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      s1 += __shfl_xor_sync(0xffffffffu, s1, o);
      s2 += __shfl_xor_sync(0xffffffffu, s2, o);
    }
    const float m1 = s1 / C, m2 = s2 / C;
#pragma unroll
    for (int k = 0; k < NV; ++k) {
      const int v = lane + k * 32;
      if (v < nvec) {
        float o[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) o[i] = rstd * (dg[k][i] - m1 - f[k][i] * m2);
        if (add) {
          float ad[8];
          unpack8(__ldg(reinterpret_cast<const uint4*>(add + static_cast<size_t>(row) * ldadd + v * 8)), ad);
#pragma unroll
          for (int i = 0; i < 8; ++i) o[i] += ad[i];
        }
        *reinterpret_cast<uint4*>(dx + static_cast<size_t>(row) * lddx + v * 8) = pack8(o);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// GEGLU (unfused training forward) and its backward.  pre = [a | g] (each F wide).
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ float gelu_grad(float x) {
  // d/dx [x Phi(x)] = Phi(x) + x phi(x)
  const float cdf = 0.5f * (1.f + erff(x * 0.7071067811865475f));
  const float pdf = 0.3989422804014327f * __expf(-0.5f * x * x);
  return cdf + x * pdf;
}

__global__ void geglu_kernel(const __nv_bfloat16* __restrict__ pre, int ldp, __nv_bfloat16* __restrict__ out,
                             int ldo, int M, int F) {
  pdl_trigger();
  pdl_wait();
  const int nvec = F >> 3;
  const size_t total = static_cast<size_t>(M) * nvec;
  for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const size_t m = i / nvec;
    const int c = static_cast<int>(i % nvec) << 3;
    float a[8], g[8], o[8];
    unpack8(__ldg(reinterpret_cast<const uint4*>(pre + m * ldp + c)), a);
    unpack8(__ldg(reinterpret_cast<const uint4*>(pre + m * ldp + F + c)), g);
#pragma unroll
    for (int k = 0; k < 8; ++k) o[k] = a[k] * gelu_erf_f(g[k]);
    *reinterpret_cast<uint4*>(out + m * ldo + c) = pack8(o);
  }
}

__global__ void geglu_bwd_kernel(const __nv_bfloat16* __restrict__ pre, int ldp,
                                 const __nv_bfloat16* __restrict__ dout, int lddo,
                                 __nv_bfloat16* __restrict__ dpre, int lddp, int M, int F) {
  pdl_trigger();
  pdl_wait();
  const int nvec = F >> 3;
  const size_t total = static_cast<size_t>(M) * nvec;
  for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const size_t m = i / nvec;
    const int c = static_cast<int>(i % nvec) << 3;
    float a[8], g[8], d[8], da[8], dg[8];
    unpack8(__ldg(reinterpret_cast<const uint4*>(pre + m * ldp + c)), a);
    unpack8(__ldg(reinterpret_cast<const uint4*>(pre + m * ldp + F + c)), g);
    unpack8(__ldg(reinterpret_cast<const uint4*>(dout + m * lddo + c)), d);
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      da[k] = d[k] * gelu_erf_f(g[k]);
      dg[k] = d[k] * a[k] * gelu_grad(g[k]);
    }
    *reinterpret_cast<uint4*>(dpre + m * lddp + c) = pack8(da);
    *reinterpret_cast<uint4*>(dpre + m * lddp + F + c) = pack8(dg);
  }
}

// ------------------------------------------------------------------------------------------------
// out = a + b (+ c), 2-D bf16 with row strides (gradient accumulation at residual / skip joins)
// ------------------------------------------------------------------------------------------------
__global__ void add_kernel(const __nv_bfloat16* __restrict__ a, int lda, const __nv_bfloat16* __restrict__ b,
                           int ldb, const __nv_bfloat16* __restrict__ c3, int ldc, __nv_bfloat16* __restrict__ out,
                           int ldo, int M, int C) {
  pdl_trigger();
  pdl_wait();
  const int nvec = C >> 3;
  const size_t total = static_cast<size_t>(M) * nvec;
  for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const size_t m = i / nvec;
    const int c = static_cast<int>(i % nvec) << 3;
    float x[8], y[8];
    unpack8(__ldg(reinterpret_cast<const uint4*>(a + m * lda + c)), x);
    unpack8(__ldg(reinterpret_cast<const uint4*>(b + m * ldb + c)), y);
#pragma unroll
    for (int k = 0; k < 8; ++k) x[k] += y[k];
    if (c3) {
      unpack8(__ldg(reinterpret_cast<const uint4*>(c3 + m * ldc + c)), y);
#pragma unroll
      for (int k = 0; k < 8; ++k) x[k] += y[k];
    }
    *reinterpret_cast<uint4*>(out + m * ldo + c) = pack8(x);
  }
}

// nearest x2 upsample backward: dx[b,y,x,:] = sum of the 2x2 block of dy
__global__ void upsample2x_bwd_kernel(const __nv_bfloat16* __restrict__ dy, __nv_bfloat16* __restrict__ dx, int B,
                                      int H, int W, int C) {
  pdl_trigger();
  pdl_wait();
  const int nvec = C >> 3;
  const size_t total = static_cast<size_t>(B) * H * W * nvec;
  for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int c = static_cast<int>(i % nvec) << 3;
    size_t pix = i / nvec;
    const int x = static_cast<int>(pix % W);
    pix /= W;
    const int y = static_cast<int>(pix % H);
    const size_t b = pix / H;
    float acc[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) acc[k] = 0.f;
#pragma unroll
    for (int dyy = 0; dyy < 2; ++dyy)
#pragma unroll
      for (int dxx = 0; dxx < 2; ++dxx) {
        float v[8];
        unpack8(__ldg(reinterpret_cast<const uint4*>(
                    dy + ((b * 2 * H + 2 * y + dyy) * 2 * W + 2 * x + dxx) * C + c)), v);
#pragma unroll
        for (int k = 0; k < 8; ++k) acc[k] += v[k];
      }
    *reinterpret_cast<uint4*>(dx + ((b * H + y) * W + x) * C + c) = pack8(acc);
  }
}

// stride-2 conv input gradient helper: z[b, 2i, 2j, :] = dy[b, i, j, :], zero elsewhere ([B,2Ho,2Wo,C])
__global__ void zero_stuff_kernel(const __nv_bfloat16* __restrict__ dy, __nv_bfloat16* __restrict__ z, int B, int Ho,
                                  int Wo, int C) {
  pdl_trigger();
  pdl_wait();
  const int nvec = C >> 3;
  const size_t total = static_cast<size_t>(B) * 2 * Ho * 2 * Wo * nvec;
  for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int c = static_cast<int>(i % nvec) << 3;
    size_t pix = i / nvec;
    const int x = static_cast<int>(pix % (2 * Wo));
    pix /= 2 * Wo;
    const int y = static_cast<int>(pix % (2 * Ho));
    const size_t b = pix / (2 * Ho);
    uint4 v = make_uint4(0, 0, 0, 0);
    if (((x | y) & 1) == 0)
      v = __ldg(reinterpret_cast<const uint4*>(dy + ((b * Ho + (y >> 1)) * Wo + (x >> 1)) * C + c));
    *reinterpret_cast<uint4*>(z + i * 8) = v;
  }
}

// conv_out backward: dx[b,y,x,c] = sum_{o,tap} d_eps[b,o,y-dy+1... ] w[o][tap][c]   (d_eps NCHW fp32 or bf16)
__global__ void conv_out_bwd_kernel(const void* __restrict__ deps, int deps_f32,
                                    const __nv_bfloat16* __restrict__ w /*[4][3][3][C]*/,
                                    __nv_bfloat16* __restrict__ dx, int B, int H, int W, int C) {
  pdl_trigger();
  pdl_wait();
  const int nvec = C >> 3;
  const size_t total = static_cast<size_t>(B) * H * W * nvec;
  for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int c = static_cast<int>(i % nvec) << 3;
    size_t pix = i / nvec;
    const int x = static_cast<int>(pix % W);
    pix /= W;
    const int y = static_cast<int>(pix % H);
    const size_t b = pix / H;
    float acc[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) acc[k] = 0.f;
    // forward: out[o, yo, xo] = sum_{a,bb,c} in[yo+a-1, xo+bb-1, c] w[o][a][bb][c]  ->  in[y,x] feeds out[y-a+1, x-bb+1]
    for (int a = 0; a < 3; ++a) {
      const int yo = y - a + 1;
      if (yo < 0 || yo >= H) continue;
      for (int bb = 0; bb < 3; ++bb) {
        const int xo = x - bb + 1;
        if (xo < 0 || xo >= W) continue;
#pragma unroll
        for (int o = 0; o < 4; ++o) {
          const size_t di = ((b * 4 + o) * H + yo) * W + xo;
          const float g = deps_f32 ? static_cast<const float*>(deps)[di]
                                   : __bfloat162float(static_cast<const __nv_bfloat16*>(deps)[di]);
          float wv[8];
          unpack8(__ldg(reinterpret_cast<const uint4*>(w + ((o * 3 + a) * 3 + bb) * C + c)), wv);
#pragma unroll
          for (int k = 0; k < 8; ++k) acc[k] = fmaf(g, wv[k], acc[k]);
        }
      }
    }
    *reinterpret_cast<uint4*>(dx + i * 8) = pack8(acc);
  }
}

// per-batch column sum: out[b, c] = sum_hw dy[b, hw, c]   (gradient of the time-embedding row bias)
// grid (C/8 / vec_per_block, B); block = (vec_per_block, rows_par)
__global__ void colsum_kernel(const __nv_bfloat16* __restrict__ dy, int ld, float* __restrict__ out, int HW, int C) {
  pdl_trigger();
  pdl_wait();
  extern __shared__ float sh[];  // [rows_par][vpb*8]
  const int vpb = blockDim.x, rows_par = blockDim.y;
  const int cv = blockIdx.x * vpb + threadIdx.x;
  const int b = blockIdx.y;
  float acc[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) acc[k] = 0.f;
  if (cv * 8 < C) {
    for (int r = threadIdx.y; r < HW; r += rows_par) {
      float v[8];
      unpack8(__ldg(reinterpret_cast<const uint4*>(dy + (static_cast<size_t>(b) * HW + r) * ld + cv * 8)), v);
#pragma unroll
      for (int k = 0; k < 8; ++k) acc[k] += v[k];
    }
  }
  float* mine = sh + (static_cast<size_t>(threadIdx.y) * vpb + threadIdx.x) * 8;
#pragma unroll
  for (int k = 0; k < 8; ++k) mine[k] = acc[k];
  __syncthreads();
  if (threadIdx.y == 0 && cv * 8 < C) {
    for (int r = 1; r < rows_par; ++r) {
      const float* o = sh + (static_cast<size_t>(r) * vpb + threadIdx.x) * 8;
#pragma unroll
      for (int k = 0; k < 8; ++k) acc[k] += o[k];
    }
#pragma unroll
    for (int k = 0; k < 8; ++k) out[static_cast<size_t>(b) * C + cv * 8 + k] = acc[k];
  }
}

// ------------------------------------------------------------------------------------------------
// LoRA rank-r helpers (r = 4, 8 or 16).  Matrices: A [M, C] bf16 activations or gradients (row stride lda).
// ------------------------------------------------------------------------------------------------
constexpr int kMaxR = 16;
constexpr int kVB = 32;  // 8-channel vectors per block in the wgrad / rank-update kernels (block = kVB x 4 row lanes)

// T[m, j] = sum_c A[m, c] * Bt[j, c]     (Bt: [r][C] bf16, row stride ldb)  -> T fp32 [M, r]
__global__ void lora_proj_kernel(const __nv_bfloat16* __restrict__ A, int lda, const __nv_bfloat16* __restrict__ Bt,
                                 int ldb, float* __restrict__ T, int M, int C, int r, int accumulate) {
  pdl_trigger();
  pdl_wait();
  const int wpb = blockDim.x >> 5, lane = threadIdx.x & 31, nvec = C >> 3;
  for (int row = blockIdx.x * wpb + (threadIdx.x >> 5); row < M; row += gridDim.x * wpb) {
    float acc[kMaxR];
#pragma unroll
    for (int j = 0; j < kMaxR; ++j) acc[j] = 0.f;
    for (int v = lane; v < nvec; v += 32) {
      float a[8];
      unpack8(__ldg(reinterpret_cast<const uint4*>(A + static_cast<size_t>(row) * lda + v * 8)), a);
#pragma unroll
      for (int j = 0; j < kMaxR; ++j) {
        if (j < r) {
          float w[8];
          unpack8(__ldg(reinterpret_cast<const uint4*>(Bt + static_cast<size_t>(j) * ldb + v * 8)), w);
#pragma unroll
          for (int k = 0; k < 8; ++k) acc[j] = fmaf(a[k], w[k], acc[j]);
        }
      }
    }
#pragma unroll
    for (int j = 0; j < kMaxR; ++j) {
      if (j < r) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) acc[j] += __shfl_xor_sync(0xffffffffu, acc[j], o);
      }
    }
    if (lane == 0) {
      for (int j = 0; j < r; ++j) {
        float* t = T + static_cast<size_t>(row) * r + j;
        *t = accumulate ? *t + acc[j] : acc[j];
      }
    }
  }
}

// partial[chunk][c][j] = sum_{m in chunk} A[m, c] * T[m, j];   grid (chunks, ceil(C/8/kVB), halves), block (kVB vectors,
// 4 row lanes).  Each z slice owns R consecutive columns j of T and partial, whose rows are halves * R wide: rank 16
// runs as two R = 8 slices (R = 16 would need 64 KB of static shared memory and 128 accumulators per thread).
template <int R>
__global__ void lora_wgrad_kernel(const __nv_bfloat16* __restrict__ A, int lda, const float* __restrict__ T,
                                  float* __restrict__ partial, int M, int C, int rows_per_block) {
  pdl_trigger();
  pdl_wait();
  __shared__ float sh[4][kVB][8 * R];
  const int cv = blockIdx.y * kVB + threadIdx.x;
  const int nvec = C >> 3;
  const int ldt = gridDim.z * R, j0 = blockIdx.z * R;  // row stride of T and partial, first column of this slice
  float acc[8][R];
#pragma unroll
  for (int k = 0; k < 8; ++k)
#pragma unroll
    for (int j = 0; j < R; ++j) acc[k][j] = 0.f;
  const int row_begin = blockIdx.x * rows_per_block;
  const int row_end = min(row_begin + rows_per_block, M);
  if (cv < nvec) {
    for (int m = row_begin + threadIdx.y; m < row_end; m += 4) {
      float a[8], t[R];
      unpack8(__ldg(reinterpret_cast<const uint4*>(A + static_cast<size_t>(m) * lda + cv * 8)), a);
#pragma unroll
      for (int j = 0; j < R; j += 4) {
        const float4 t4 = __ldg(reinterpret_cast<const float4*>(T + static_cast<size_t>(m) * ldt + j0 + j));
        t[j] = t4.x, t[j + 1] = t4.y, t[j + 2] = t4.z, t[j + 3] = t4.w;
      }
#pragma unroll
      for (int k = 0; k < 8; ++k)
#pragma unroll
        for (int j = 0; j < R; ++j) acc[k][j] = fmaf(a[k], t[j], acc[k][j]);
    }
  }
#pragma unroll
  for (int k = 0; k < 8; ++k)
#pragma unroll
    for (int j = 0; j < R; ++j) sh[threadIdx.y][threadIdx.x][k * R + j] = acc[k][j];
  __syncthreads();
  if (threadIdx.y == 0 && cv < nvec) {
    float* out = partial + (static_cast<size_t>(blockIdx.x) * C + cv * 8) * ldt + j0;
#pragma unroll
    for (int e = 0; e < 8 * R; ++e)
      out[(e / R) * ldt + e % R] =
          sh[0][threadIdx.x][e] + sh[1][threadIdx.x][e] + sh[2][threadIdx.x][e] + sh[3][threadIdx.x][e];
  }
}

// G[c * gs_c + j * gs_r] (+)= scale * sum_chunks partial[chunk][c][j]
__global__ void lora_wgrad_reduce_kernel(const float* __restrict__ partial, float* __restrict__ G, int chunks, int C,
                                         int r, int gs_c, int gs_r, float scale, int accumulate) {
  pdl_trigger();
  pdl_wait();
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= C * r) return;
  float s = 0.f;
  for (int k = 0; k < chunks; ++k) s += partial[static_cast<size_t>(k) * C * r + idx];
  const int c = idx / r, j = idx - c * r;
  float* g = G + static_cast<size_t>(c) * gs_c + static_cast<size_t>(j) * gs_r;
  *g = accumulate ? *g + s * scale : s * scale;
}

// dX[m, c] += scale * sum_j U[m, j] * D[j, c]     (D: [r][C] bf16)
template <int R>
__global__ void lora_rank_update_kernel(__nv_bfloat16* __restrict__ dX, int ldx, const float* __restrict__ U,
                                        const __nv_bfloat16* __restrict__ D, int ldd, float scale, int M, int C,
                                        int rows_per_block) {
  pdl_trigger();
  pdl_wait();
  const int nvec = C >> 3;
  const int cv = blockIdx.y * kVB + threadIdx.x;
  if (cv >= nvec) return;
  float d[R][8];
#pragma unroll
  for (int j = 0; j < R; ++j) {
    unpack8(__ldg(reinterpret_cast<const uint4*>(D + static_cast<size_t>(j) * ldd + cv * 8)), d[j]);
#pragma unroll
    for (int k = 0; k < 8; ++k) d[j][k] *= scale;
  }
  const int row_begin = blockIdx.x * rows_per_block;
  const int row_end = min(row_begin + rows_per_block, M);
  for (int m = row_begin + threadIdx.y; m < row_end; m += 4) {
    float x[8], u[R];
    uint4* px = reinterpret_cast<uint4*>(dX + static_cast<size_t>(m) * ldx + cv * 8);
    unpack8(*px, x);
#pragma unroll
    for (int j = 0; j < R; j += 4) {
      const float4 t4 = __ldg(reinterpret_cast<const float4*>(U + static_cast<size_t>(m) * R + j));
      u[j] = t4.x, u[j + 1] = t4.y, u[j + 2] = t4.z, u[j + 3] = t4.w;
    }
#pragma unroll
    for (int j = 0; j < R; ++j)
#pragma unroll
      for (int k = 0; k < 8; ++k) x[k] = fmaf(u[j], d[j][k], x[k]);
    *px = pack8(x);
  }
}

// ---- 3x3 conv LoRA (down is a 3x3 conv to r channels with the leaf's stride / pad 1, up is 1x1) ----------------
struct ConvGeom {
  const __nv_bfloat16* x0;
  const __nv_bfloat16* x1;
  int ld0, ld1, C0, C;  // channels-last sources (concat)
  int B, H, W, Ho, Wo, stride;
};

__device__ __forceinline__ const __nv_bfloat16* conv_src(const ConvGeom& g, size_t pix, int c) {
  return c < g.C0 ? g.x0 + pix * g.ld0 + c : g.x1 + pix * g.ld1 + (c - g.C0);
}

// T[p, j] = sum_{tap, c} x[p*stride + tap - 1, c] * D[j][tap][c]    one warp per output pixel
__global__ void lora_conv_proj_kernel(ConvGeom g, const __nv_bfloat16* __restrict__ D /*[r][3][3][C]*/,
                                      float* __restrict__ T, int r) {
  pdl_trigger();
  pdl_wait();
  const int wpb = blockDim.x >> 5, lane = threadIdx.x & 31, nvec = g.C >> 3;
  const int P = g.B * g.Ho * g.Wo;
  for (int p = blockIdx.x * wpb + (threadIdx.x >> 5); p < P; p += gridDim.x * wpb) {
    const int xo = p % g.Wo, yo = (p / g.Wo) % g.Ho, b = p / (g.Wo * g.Ho);
    float acc[kMaxR];
#pragma unroll
    for (int j = 0; j < kMaxR; ++j) acc[j] = 0.f;
    for (int tap = 0; tap < 9; ++tap) {
      const int y = yo * g.stride + tap / 3 - 1, x = xo * g.stride + tap % 3 - 1;
      if (y < 0 || y >= g.H || x < 0 || x >= g.W) continue;
      const size_t pix = (static_cast<size_t>(b) * g.H + y) * g.W + x;
      for (int v = lane; v < nvec; v += 32) {
        float a[8];
        unpack8(__ldg(reinterpret_cast<const uint4*>(conv_src(g, pix, v * 8))), a);
#pragma unroll
        for (int j = 0; j < kMaxR; ++j) {
          if (j < r) {
            float w[8];
            unpack8(__ldg(reinterpret_cast<const uint4*>(D + (static_cast<size_t>(j) * 9 + tap) * g.C + v * 8)), w);
#pragma unroll
            for (int k = 0; k < 8; ++k) acc[j] = fmaf(a[k], w[k], acc[j]);
          }
        }
      }
    }
#pragma unroll
    for (int j = 0; j < kMaxR; ++j) {
      if (j < r) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) acc[j] += __shfl_xor_sync(0xffffffffu, acc[j], o);
      }
    }
    if (lane == 0)
      for (int j = 0; j < r; ++j) T[static_cast<size_t>(p) * r + j] = acc[j];
  }
}

// partial[chunk][tap][c][j] = sum_{p in chunk} U[p, j] * x[p*stride + tap - 1, c];  grid (chunks, ceil(C/8/kVB),
// 9 * halves): z = half * 9 + tap, the column slices as in lora_wgrad_kernel
template <int R>
__global__ void lora_conv_wgrad_kernel(ConvGeom g, const float* __restrict__ U, float* __restrict__ partial,
                                       int rows_per_block) {
  pdl_trigger();
  pdl_wait();
  __shared__ float sh[4][kVB][8 * R];
  const int cv = blockIdx.y * kVB + threadIdx.x, nvec = g.C >> 3, tap = blockIdx.z % 9;
  const int ldt = (gridDim.z / 9) * R, j0 = (blockIdx.z / 9) * R;  // row stride of U and partial, first column
  const int P = g.B * g.Ho * g.Wo;
  float acc[8][R];
#pragma unroll
  for (int k = 0; k < 8; ++k)
#pragma unroll
    for (int j = 0; j < R; ++j) acc[k][j] = 0.f;
  const int row_begin = blockIdx.x * rows_per_block;
  const int row_end = min(row_begin + rows_per_block, P);
  if (cv < nvec) {
    for (int p = row_begin + threadIdx.y; p < row_end; p += 4) {
      const int xo = p % g.Wo, yo = (p / g.Wo) % g.Ho, b = p / (g.Wo * g.Ho);
      const int y = yo * g.stride + tap / 3 - 1, x = xo * g.stride + tap % 3 - 1;
      if (y < 0 || y >= g.H || x < 0 || x >= g.W) continue;
      const size_t pix = (static_cast<size_t>(b) * g.H + y) * g.W + x;
      float a[8], t[R];
      unpack8(__ldg(reinterpret_cast<const uint4*>(conv_src(g, pix, cv * 8))), a);
#pragma unroll
      for (int j = 0; j < R; j += 4) {
        const float4 t4 = __ldg(reinterpret_cast<const float4*>(U + static_cast<size_t>(p) * ldt + j0 + j));
        t[j] = t4.x, t[j + 1] = t4.y, t[j + 2] = t4.z, t[j + 3] = t4.w;
      }
#pragma unroll
      for (int k = 0; k < 8; ++k)
#pragma unroll
        for (int j = 0; j < R; ++j) acc[k][j] = fmaf(a[k], t[j], acc[k][j]);
    }
  }
#pragma unroll
  for (int k = 0; k < 8; ++k)
#pragma unroll
    for (int j = 0; j < R; ++j) sh[threadIdx.y][threadIdx.x][k * R + j] = acc[k][j];
  __syncthreads();
  if (threadIdx.y == 0 && cv < nvec) {
    // partial layout: [chunk][tap*C + c][j]  (= lora_wgrad_reduce_kernel's layout with "C" = 9*C)
    float* out = partial + ((static_cast<size_t>(blockIdx.x) * 9 + tap) * g.C + cv * 8) * ldt + j0;
#pragma unroll
    for (int e = 0; e < 8 * R; ++e)
      out[(e / R) * ldt + e % R] =
          sh[0][threadIdx.x][e] + sh[1][threadIdx.x][e] + sh[2][threadIdx.x][e] + sh[3][threadIdx.x][e];
  }
}

// dX[b,y,x,c] += scale * sum_{tap,j} U[(y - a + 1)/s, (x - bb + 1)/s ; j] * D[j][tap][c]   (dX: [B,H,W,C] contiguous)
template <int R>
__global__ void lora_conv_rank_update_kernel(__nv_bfloat16* __restrict__ dX, int B, int H, int W, int C, int Ho,
                                             int Wo, int stride, const float* __restrict__ U,
                                             const __nv_bfloat16* __restrict__ D, float scale) {
  pdl_trigger();
  pdl_wait();
  const int nvec = C >> 3;
  const size_t total = static_cast<size_t>(B) * H * W * nvec;
  for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int c = static_cast<int>(i % nvec) << 3;
    size_t pix = i / nvec;
    const int x = static_cast<int>(pix % W);
    pix /= W;
    const int y = static_cast<int>(pix % H);
    const size_t b = pix / H;
    float acc[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) acc[k] = 0.f;
    for (int a = 0; a < 3; ++a) {
      const int ys = y - a + 1;
      if (ys < 0 || ys % stride) continue;
      const int yo = ys / stride;
      if (yo >= Ho) continue;
      for (int bb = 0; bb < 3; ++bb) {
        const int xs = x - bb + 1;
        if (xs < 0 || xs % stride) continue;
        const int xo = xs / stride;
        if (xo >= Wo) continue;
        const float* u = U + ((b * Ho + yo) * Wo + xo) * R;
#pragma unroll
        for (int j = 0; j < R; ++j) {
          const float uj = __ldg(u + j);
          float w[8];
          unpack8(__ldg(reinterpret_cast<const uint4*>(D + (static_cast<size_t>(j) * 9 + a * 3 + bb) * C + c)), w);
#pragma unroll
          for (int k = 0; k < 8; ++k) acc[k] = fmaf(uj, w[k], acc[k]);
        }
      }
    }
    uint4* px = reinterpret_cast<uint4*>(dX + i * 8);
    float xv[8];
    unpack8(*px, xv);
#pragma unroll
    for (int k = 0; k < 8; ++k) xv[k] = fmaf(scale, acc[k], xv[k]);
    *px = pack8(xv);
  }
}

// ------------------------------------------------------------------------------------------------
// AdamW on bf16 parameters with bf16 moments (torch.optim.AdamW semantics, every intermediate that torch
// materialises as a bf16 tensor is rounded to bf16 here too).  One launch over a table of tensors.
// ------------------------------------------------------------------------------------------------
struct AdamTensor {
  __nv_bfloat16* p;
  const __nv_bfloat16* g;
  __nv_bfloat16* m;
  __nv_bfloat16* v;
  long long n;
};

__device__ __forceinline__ float rbf(float x) { return __bfloat162float(__float2bfloat16(x)); }

__global__ void adamw_kernel(const AdamTensor* __restrict__ table, float decay, float one_m_beta1, float beta2,
                             float one_m_beta2, float eps, float neg_step_size, float bc2_sqrt) {
  pdl_trigger();
  pdl_wait();
  const AdamTensor t = table[blockIdx.y];
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < t.n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float g = __bfloat162float(t.g[i]);
    float p = __bfloat162float(t.p[i]);
    float m = __bfloat162float(t.m[i]);
    float v = __bfloat162float(t.v[i]);
    p = rbf(p * decay);                                  // param.mul_(1 - lr * weight_decay)
    m = rbf(m + one_m_beta1 * (g - m));               // exp_avg.lerp_(grad, 1 - beta1)
    v = rbf(v * beta2);                                 // exp_avg_sq.mul_(beta2)
    v = rbf(v + one_m_beta2 * (g * g));                //            .addcmul_(grad, grad, value = 1 - beta2)
    float denom = rbf(sqrtf(v));                        // exp_avg_sq.sqrt()
    denom = rbf(denom / bc2_sqrt);                      //   / bias_correction2_sqrt
    denom = rbf(denom + eps);                           //   .add_(eps)
    p = rbf(p + neg_step_size * (m / denom));          // param.addcdiv_(exp_avg, denom, value = -step_size)
    t.p[i] = __float2bfloat16(p);
    t.m[i] = __float2bfloat16(m);
    t.v[i] = __float2bfloat16(v);
  }
}

// torch.optim.Adam (foreach / single-tensor, amsgrad off) on fp32 parameters and moments: the null-text embedding
struct AdamTensorF32 {
  float* p;
  const float* g;
  float* m;
  float* v;
  long long n;
};

__global__ void adam_f32_kernel(const AdamTensorF32* __restrict__ table, float weight_decay, float one_m_beta1,
                                float beta2, float one_m_beta2, float eps, float neg_step_size, float bc2_sqrt) {
  pdl_trigger();
  pdl_wait();
  const AdamTensorF32 t = table[blockIdx.y];
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < t.n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    float p = t.p[i];
    const float g = t.g[i] + weight_decay * p;          // grad.add(param, alpha=weight_decay)
    const float m = t.m[i] + one_m_beta1 * (g - t.m[i]);  // exp_avg.lerp_(grad, 1 - beta1)
    const float v = t.v[i] * beta2 + one_m_beta2 * g * g; // exp_avg_sq.mul_(beta2).addcmul_(grad, grad, 1 - beta2)
    const float denom = sqrtf(v) / bc2_sqrt + eps;       // (exp_avg_sq.sqrt() / bias_correction2_sqrt).add_(eps)
    p += neg_step_size * (m / denom);                    // param.addcdiv_(exp_avg, denom, value=-step_size)
    t.p[i] = p;
    t.m[i] = m;
    t.v[i] = v;
  }
}

}  // namespace sb200

using namespace sb200;
typedef __nv_bfloat16 bf;

extern "C" int sb200_groupnorm_bwd(void* handle, void* stream, const void* x0, int ldx0, int C0, const void* x1,
                                   int ldx1, int C1, const void* gamma, const void* beta, const void* dy, int lddy,
                                   const void* add, int ldadd, void* dx, int lddx, int B, int HW, int groups,
                                   int silu, const float* fwd_stats, float* ws) {
  Ctx* ctx = as_ctx(handle);
  SB200_REQUIRE(ctx, "groupnorm_bwd: NULL handle");
  if (!x1) C1 = 0;
  const int C = C0 + C1;
  SB200_REQUIRE(B > 0 && HW > 0 && C0 > 0 && C0 % 8 == 0 && C1 % 8 == 0 && C % groups == 0, "groupnorm_bwd: dims");
  SB200_REQUIRE(ldx0 % 8 == 0 && lddy % 8 == 0 && lddx % 8 == 0 && (C1 == 0 || ldx1 % 8 == 0) &&
                    (!add || ldadd % 8 == 0),
                "groupnorm_bwd: leading dims");
  SB200_REQUIRE(fwd_stats && ws && gamma && beta && dy && dx, "groupnorm_bwd: arguments");
  // the stats kernel keeps [rows_par][C][2] fp32 partials in dynamic shared memory without opting in above 48 KB
  SB200_REQUIRE(gn_stats_smem_ok(C), "groupnorm_bwd: C=%d too large", C);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  GnBwdArgs a;
  a.x0 = static_cast<const bf*>(x0);
  a.x1 = static_cast<const bf*>(x1);
  a.ld0 = ldx0, a.ld1 = ldx1, a.C0 = C0, a.C = C, a.HW = HW, a.groups = groups, a.cpg = C / groups;
  a.gamma = static_cast<const bf*>(gamma);
  a.beta = static_cast<const bf*>(beta);
  a.dy = static_cast<const bf*>(dy);
  a.lddy = lddy;
  a.add = static_cast<const bf*>(add);
  a.ldadd = ldadd;
  a.dx = static_cast<bf*>(dx);
  a.lddx = lddx;
  a.stats = fwd_stats;
  a.silu = silu;
  const GnShape g = gn_shape(ctx, B, HW, C);
  // above C = 4096 a block has C/8 > 512 threads; the stats / apply kernels' register use caps the block size
  int max_threads = 1024;
  for (const void* fn : {reinterpret_cast<const void*>(gn_bwd_stats_kernel), reinterpret_cast<const void*>(gn_bwd_apply_kernel)}) {
    cudaFuncAttributes attr;
    SB200_CUDA_CHECK(cudaFuncGetAttributes(&attr, fn));
    if (attr.maxThreadsPerBlock < max_threads) max_threads = attr.maxThreadsPerBlock;
  }
  SB200_REQUIRE(g.threads <= max_threads, "groupnorm_bwd: C=%d too large (%d threads per block, at most %d)", C, g.threads,
                max_threads);
  a.rows_per_block = g.rows_per_block;
  float* final_m = ws + SB200_GN_STATS_OFFSET(B, groups);
  SB200_CUDA_CHECK(launch_pdl(gn_bwd_stats_kernel, dim3(g.chunks, B), dim3(g.threads), sizeof(float) * 2 * C * g.rows_par, s, true, a, ws));
  SB200_CUDA_CHECK(launch_pdl(gn_bwd_finalize_kernel, dim3(B), dim3(1024), 0, s, true, ws, final_m, g.chunks, groups, 1.f / (static_cast<float>(HW) * a.cpg)));
  SB200_CUDA_CHECK(launch_pdl(gn_bwd_apply_kernel, dim3(g.chunks, B), dim3(g.threads), 0, s, true, a, final_m));
  return 0;
}

extern "C" int sb200_layernorm_bwd(void* handle, void* stream, const void* x, int ldx, const void* gamma,
                                   const void* dy, int lddy, const void* add, int ldadd, void* dx, int lddx, int M,
                                   int C, float eps) {
  Ctx* ctx = as_ctx(handle);
  SB200_REQUIRE(ctx, "layernorm_bwd: NULL handle");
  SB200_REQUIRE(M > 0 && C > 0 && C % 8 == 0 && C <= 2048, "layernorm_bwd: C=%d unsupported", C);
  SB200_REQUIRE(ldx % 8 == 0 && lddy % 8 == 0 && lddx % 8 == 0 && (!add || ldadd % 8 == 0), "layernorm_bwd: leading dims");
  const int warps = 8;
  const int blocks = grid_cap(ctx, M, warps, 16);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
#define SB200_LNB(NV)                                                                                           \
  layernorm_bwd_kernel<NV><<<blocks, warps * 32, 0, st>>>(static_cast<const bf*>(x), ldx,                        \
                                                          static_cast<const bf*>(gamma), static_cast<const bf*>(dy), \
                                                          lddy, static_cast<const bf*>(add), ldadd,               \
                                                          static_cast<bf*>(dx), lddx, M, C, eps)
  if (C <= 256)
    SB200_LNB(1);
  else if (C <= 768)
    SB200_LNB(3);
  else if (C <= 1280)
    SB200_LNB(5);
  else
    SB200_LNB(8);
#undef SB200_LNB
  SB200_CUDA_CHECK(cudaGetLastError());
  return 0;
}

extern "C" int sb200_geglu(void* handle, void* stream, const void* pre, int ldp, void* out, int ldo, int M, int F) {
  Ctx* ctx = as_ctx(handle);
  SB200_REQUIRE(ctx && M > 0 && F > 0 && F % 8 == 0 && ldp % 8 == 0 && ldo % 8 == 0, "geglu: arguments");
  SB200_CUDA_CHECK(launch_pdl(geglu_kernel, dim3(grid_cap(ctx, static_cast<size_t>(M) * F / 8, 256, 16, true)), dim3(256), 0,
                              static_cast<cudaStream_t>(stream), true, static_cast<const bf*>(pre), ldp, static_cast<bf*>(out), ldo, M, F));
  return 0;
}

extern "C" int sb200_geglu_bwd(void* handle, void* stream, const void* pre, int ldp, const void* dout, int lddo,
                               void* dpre, int lddp, int M, int F) {
  Ctx* ctx = as_ctx(handle);
  SB200_REQUIRE(ctx && M > 0 && F > 0 && F % 8 == 0 && ldp % 8 == 0 && lddo % 8 == 0 && lddp % 8 == 0,
                "geglu_bwd: arguments");
  SB200_CUDA_CHECK(launch_pdl(geglu_bwd_kernel, dim3(grid_cap(ctx, static_cast<size_t>(M) * F / 8, 256, 16, true)), dim3(256), 0,
                              static_cast<cudaStream_t>(stream), true, static_cast<const bf*>(pre), ldp,
                                                          static_cast<const bf*>(dout), lddo, static_cast<bf*>(dpre),
                                                          lddp, M, F));
  return 0;
}

extern "C" int sb200_add(void* handle, void* stream, const void* a, int lda, const void* b, int ldb, const void* c,
                         int ldc, void* out, int ldo, int M, int C) {
  Ctx* ctx = as_ctx(handle);
  SB200_REQUIRE(ctx && a && b && out && M > 0 && C > 0 && C % 8 == 0 && lda % 8 == 0 && ldb % 8 == 0 &&
                    ldo % 8 == 0 && (!c || ldc % 8 == 0),
                "add: arguments");
  SB200_CUDA_CHECK(launch_pdl(add_kernel, dim3(grid_cap(ctx, static_cast<size_t>(M) * C / 8, 256, 16, true)), dim3(256), 0,
                              static_cast<cudaStream_t>(stream), true, static_cast<const bf*>(a), lda, static_cast<const bf*>(b), ldb,
                                                    static_cast<const bf*>(c), ldc, static_cast<bf*>(out), ldo, M, C));
  return 0;
}

extern "C" int sb200_upsample2x_bwd(void* handle, void* stream, const void* dy, void* dx, int B, int H, int W, int C) {
  Ctx* ctx = as_ctx(handle);
  SB200_REQUIRE(ctx && dy && dx && B > 0 && H > 0 && W > 0 && C % 8 == 0, "upsample2x_bwd: arguments");
  SB200_CUDA_CHECK(launch_pdl(upsample2x_bwd_kernel, dim3(grid_cap(ctx, static_cast<size_t>(B) * H * W * C / 8, 256, 16, true)), dim3(256), 0,
                              static_cast<cudaStream_t>(stream), true, static_cast<const bf*>(dy), static_cast<bf*>(dx), B, H, W, C));
  return 0;
}

extern "C" int sb200_zero_stuff(void* handle, void* stream, const void* dy, void* z, int B, int Ho, int Wo, int C) {
  Ctx* ctx = as_ctx(handle);
  SB200_REQUIRE(ctx && dy && z && B > 0 && Ho > 0 && Wo > 0 && C % 8 == 0, "zero_stuff: arguments");
  SB200_CUDA_CHECK(launch_pdl(zero_stuff_kernel, dim3(grid_cap(ctx, static_cast<size_t>(B) * 4 * Ho * Wo * C / 8, 256, 16, true)), dim3(256), 0,
                              static_cast<cudaStream_t>(stream), true, static_cast<const bf*>(dy), static_cast<bf*>(z), B, Ho, Wo, C));
  return 0;
}

extern "C" int sb200_conv_out_bwd(void* handle, void* stream, const void* deps, int deps_f32, const void* w, void* dx,
                                  int B, int H, int W, int C) {
  Ctx* ctx = as_ctx(handle);
  SB200_REQUIRE(ctx && deps && w && dx && B > 0 && H > 0 && W > 0 && C % 8 == 0, "conv_out_bwd: arguments");
  SB200_CUDA_CHECK(launch_pdl(conv_out_bwd_kernel, dim3(grid_cap(ctx, static_cast<size_t>(B) * H * W * C / 8, 256, 16, true)), dim3(256), 0,
                              static_cast<cudaStream_t>(stream), true, deps, deps_f32, static_cast<const bf*>(w),
                                                             static_cast<bf*>(dx), B, H, W, C));
  return 0;
}

extern "C" int sb200_colsum(void* handle, void* stream, const void* dy, int ld, float* out, int B, int HW, int C) {
  Ctx* ctx = as_ctx(handle);
  SB200_REQUIRE(ctx && dy && out && B > 0 && HW > 0 && C % 8 == 0 && ld % 8 == 0, "colsum: arguments");
  const int vpb = 8, rows_par = 64;  // 64 channels per block: many blocks, each streams 128-byte row pieces
  dim3 grid((C / 8 + vpb - 1) / vpb, B), block(vpb, rows_par);
  SB200_CUDA_CHECK(launch_pdl(colsum_kernel, dim3(grid), dim3(block), sizeof(float) * rows_par * vpb * 8, static_cast<cudaStream_t>(stream), true, 
      static_cast<const bf*>(dy), ld, out, HW, C));
  return 0;
}

extern "C" int sb200_lora_proj(void* handle, void* stream, const void* A, int lda, const void* Bt, int ldb, float* T,
                               int M, int C, int r, int accumulate) {
  Ctx* ctx = as_ctx(handle);
  SB200_REQUIRE(ctx && A && Bt && T && M > 0 && C % 8 == 0 && lda % 8 == 0 && ldb % 8 == 0 &&
                    (r == 4 || r == 8 || r == 16),
                "lora_proj: arguments (r=%d)", r);
  const int blocks = grid_cap(ctx, M, 8, 16);
  SB200_CUDA_CHECK(launch_pdl(lora_proj_kernel, dim3(blocks), dim3(256), 0, static_cast<cudaStream_t>(stream), true, static_cast<const bf*>(A), lda,
                                                                          static_cast<const bf*>(Bt), ldb, T, M, C, r, accumulate));
  return 0;
}

static int wgrad_chunks(int rows, int cblocks, int* rows_per_block) {
  int chunks = (264 + cblocks - 1) / cblocks;  // two per SM of an H100, fixed (not num_sms-derived) so callers can size `ws`: see sb200.h
  if (chunks > 256) chunks = 256;
  int rpb = (rows + chunks - 1) / chunks;
  if (rpb < 32) rpb = 32;
  *rows_per_block = rpb;
  return (rows + rpb - 1) / rpb;
}

/* ws must hold SB200_WGRAD_WS_FLOATS(C, r) floats */
extern "C" int sb200_lora_wgrad(void* handle, void* stream, const void* A, int lda, const float* T, float* G,
                                int gs_c, int gs_r, float scale, int accumulate, int M, int C, int r, float* ws) {
  Ctx* ctx = as_ctx(handle);
  SB200_REQUIRE(ctx && A && T && G && ws && M > 0 && C % 8 == 0 && lda % 8 == 0 && (r == 4 || r == 8 || r == 16),
                "lora_wgrad: arguments (r=%d)", r);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int cblocks = (C / 8 + kVB - 1) / kVB;
  int rpb;
  const int chunks = wgrad_chunks(M, cblocks, &rpb);
  dim3 grid(chunks, cblocks, r == 16 ? 2 : 1), block(kVB, 4);
  if (r == 4)
    SB200_CUDA_CHECK(launch_pdl(lora_wgrad_kernel<4>, dim3(grid), dim3(block), 0, s, true, static_cast<const bf*>(A), lda, T, ws, M, C, rpb));
  else
    SB200_CUDA_CHECK(launch_pdl(lora_wgrad_kernel<8>, dim3(grid), dim3(block), 0, s, true, static_cast<const bf*>(A), lda, T, ws, M, C, rpb));
  SB200_CUDA_CHECK(launch_pdl(lora_wgrad_reduce_kernel, dim3((C * r + 255) / 256), dim3(256), 0, s, true, ws, G, chunks, C, r, gs_c, gs_r, scale, accumulate));
  return 0;
}

extern "C" int sb200_lora_rank_update(void* handle, void* stream, void* dX, int ldx, const float* U, const void* D,
                                      int ldd, float scale, int M, int C, int r) {
  Ctx* ctx = as_ctx(handle);
  SB200_REQUIRE(ctx && dX && U && D && M > 0 && C % 8 == 0 && ldx % 8 == 0 && ldd % 8 == 0 &&
                    (r == 4 || r == 8 || r == 16),
                "lora_rank_update: arguments (r=%d)", r);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int cblocks = (C / 8 + kVB - 1) / kVB;
  int rpb;
  const int chunks = wgrad_chunks(M, cblocks, &rpb);
  dim3 grid(chunks, cblocks), block(kVB, 4);
  if (r == 4)
    SB200_CUDA_CHECK(launch_pdl(lora_rank_update_kernel<4>, dim3(grid), dim3(block), 0, s, true, static_cast<bf*>(dX), ldx, U, static_cast<const bf*>(D), ldd,
                                                     scale, M, C, rpb));
  else if (r == 8)
    SB200_CUDA_CHECK(launch_pdl(lora_rank_update_kernel<8>, dim3(grid), dim3(block), 0, s, true, static_cast<bf*>(dX), ldx, U, static_cast<const bf*>(D), ldd,
                                                     scale, M, C, rpb));
  else
    SB200_CUDA_CHECK(launch_pdl(lora_rank_update_kernel<16>, dim3(grid), dim3(block), 0, s, true, static_cast<bf*>(dX), ldx, U, static_cast<const bf*>(D), ldd,
                                                     scale, M, C, rpb));
  return 0;
}

static int fill_geom(ConvGeom* g, const void* x0, int ldx0, int C0, const void* x1, int ldx1, int C1, int B, int H,
                     int W, int stride) {
  g->x0 = static_cast<const bf*>(x0);
  g->x1 = static_cast<const bf*>(x1);
  g->ld0 = ldx0, g->ld1 = ldx1, g->C0 = C0, g->C = C0 + (x1 ? C1 : 0);
  g->B = B, g->H = H, g->W = W, g->stride = stride, g->Ho = H / stride, g->Wo = W / stride;
  return 0;
}

extern "C" int sb200_lora_conv_proj(void* handle, void* stream, const void* x0, int ldx0, int C0, const void* x1,
                                    int ldx1, int C1, const void* D, float* T, int B, int H, int W, int stride, int r) {
  Ctx* ctx = as_ctx(handle);
  SB200_REQUIRE(ctx && x0 && D && T && C0 % 8 == 0 && (!x1 || C1 % 8 == 0) && (stride == 1 || stride == 2) &&
                    (r == 4 || r == 8 || r == 16),
                "lora_conv_proj: arguments");
  ConvGeom g;
  fill_geom(&g, x0, ldx0, C0, x1, ldx1, C1, B, H, W, stride);
  const int P = B * g.Ho * g.Wo;
  const int blocks = grid_cap(ctx, P, 8, 16);
  SB200_CUDA_CHECK(launch_pdl(lora_conv_proj_kernel, dim3(blocks), dim3(256), 0, static_cast<cudaStream_t>(stream), true, g, static_cast<const bf*>(D), T, r));
  return 0;
}

/* G: [r][3][3][C] fp32 (the lora_down.weight gradient in the packed tap-major layout); ws: SB200_WGRAD_WS_FLOATS(9*C, r) */
extern "C" int sb200_lora_conv_wgrad(void* handle, void* stream, const void* x0, int ldx0, int C0, const void* x1,
                                     int ldx1, int C1, const float* U, float* G, float scale, int accumulate, int B,
                                     int H, int W, int stride, int r, float* ws) {
  Ctx* ctx = as_ctx(handle);
  SB200_REQUIRE(ctx && x0 && U && G && ws && C0 % 8 == 0 && (!x1 || C1 % 8 == 0) && (stride == 1 || stride == 2) &&
                    (r == 4 || r == 8 || r == 16),
                "lora_conv_wgrad: arguments");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  ConvGeom g;
  fill_geom(&g, x0, ldx0, C0, x1, ldx1, C1, B, H, W, stride);
  const int P = B * g.Ho * g.Wo;
  const int cblocks = (g.C / 8 + kVB - 1) / kVB;
  int rpb;
  const int chunks = wgrad_chunks(P, cblocks * 9, &rpb);
  dim3 grid(chunks, cblocks, r == 16 ? 18 : 9), block(kVB, 4);
  if (r == 4)
    SB200_CUDA_CHECK(launch_pdl(lora_conv_wgrad_kernel<4>, dim3(grid), dim3(block), 0, s, true, g, U, ws, rpb));
  else
    SB200_CUDA_CHECK(launch_pdl(lora_conv_wgrad_kernel<8>, dim3(grid), dim3(block), 0, s, true, g, U, ws, rpb));
  const int C9 = 9 * g.C;
  // G[j][tap*C + c]: gs_c = 1, gs_r = 9*C
  SB200_CUDA_CHECK(launch_pdl(lora_wgrad_reduce_kernel, dim3((C9 * r + 255) / 256), dim3(256), 0, s, true, ws, G, chunks, C9, r, 1, C9, scale, accumulate));
  return 0;
}

extern "C" int sb200_lora_conv_rank_update(void* handle, void* stream, void* dX, const float* U, const void* D,
                                           float scale, int B, int H, int W, int C, int stride, int r) {
  Ctx* ctx = as_ctx(handle);
  SB200_REQUIRE(ctx && dX && U && D && C % 8 == 0 && (stride == 1 || stride == 2) &&
                    (r == 4 || r == 8 || r == 16),
                "lora_conv_rank_update: arguments");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int blocks = grid_cap(ctx, static_cast<size_t>(B) * H * W * C / 8, 256, 16, true);
  if (r == 4)
    SB200_CUDA_CHECK(launch_pdl(lora_conv_rank_update_kernel<4>, dim3(blocks), dim3(256), 0, s, true, static_cast<bf*>(dX), B, H, W, C, H / stride, W / stride,
                                                          stride, U, static_cast<const bf*>(D), scale));
  else if (r == 8)
    SB200_CUDA_CHECK(launch_pdl(lora_conv_rank_update_kernel<8>, dim3(blocks), dim3(256), 0, s, true, static_cast<bf*>(dX), B, H, W, C, H / stride, W / stride,
                                                          stride, U, static_cast<const bf*>(D), scale));
  else
    SB200_CUDA_CHECK(launch_pdl(lora_conv_rank_update_kernel<16>, dim3(blocks), dim3(256), 0, s, true, static_cast<bf*>(dX), B, H, W, C, H / stride, W / stride,
                                                          stride, U, static_cast<const bf*>(D), scale));
  return 0;
}

/* table: device array of n_tensors {p, g, m, v (device pointers), n (int64)} records (5 x 8 bytes each) */
extern "C" int sb200_adamw(void* handle, void* stream, const void* table, int n_tensors, long long max_numel,
                           double lr, double beta1, double beta2, double eps, double weight_decay, int step) {
  Ctx* ctx = as_ctx(handle);
  SB200_REQUIRE(ctx && table && n_tensors > 0 && max_numel > 0 && step >= 1, "adamw: arguments");
  SB200_REQUIRE(n_tensors <= 65535, "adamw: %d tensors exceed the grid's 65535 y-blocks", n_tensors);
  static_assert(sizeof(AdamTensor) == 40, "AdamTensor layout");
  const double bc1 = 1.0 - pow(beta1, static_cast<double>(step));
  const double bc2 = 1.0 - pow(beta2, static_cast<double>(step));
  int bx = static_cast<int>((max_numel + 255) / 256);
  if (bx > 64) bx = 64;
  SB200_CUDA_CHECK(launch_pdl(adamw_kernel, dim3(dim3(bx, n_tensors)), dim3(256), 0, static_cast<cudaStream_t>(stream), true, 
      static_cast<const AdamTensor*>(table), static_cast<float>(1.0 - lr * weight_decay),
      static_cast<float>(1.0 - beta1), static_cast<float>(beta2), static_cast<float>(1.0 - beta2),
      static_cast<float>(eps), static_cast<float>(-(lr / bc1)), static_cast<float>(sqrt(bc2))));
  return 0;
}

extern "C" int sb200_adam_f32(void* handle, void* stream, const void* table, int n_tensors, long long max_numel,
                              double lr, double beta1, double beta2, double eps, double weight_decay, int step) {
  Ctx* ctx = as_ctx(handle);
  SB200_REQUIRE(ctx && table && n_tensors > 0 && max_numel > 0 && step >= 1, "adam_f32: arguments");
  SB200_REQUIRE(n_tensors <= 65535, "adam_f32: %d tensors exceed the grid's 65535 y-blocks", n_tensors);
  const double bc1 = 1.0 - pow(beta1, step), bc2 = 1.0 - pow(beta2, step);
  const int bx = grid_cap(ctx, static_cast<size_t>(max_numel), 256, 16, true);
  SB200_CUDA_CHECK(launch_pdl(adam_f32_kernel, dim3(bx, n_tensors), dim3(256), 0, static_cast<cudaStream_t>(stream), true,
                              static_cast<const AdamTensorF32*>(table), static_cast<float>(weight_decay),
                              static_cast<float>(1.0 - beta1), static_cast<float>(beta2),
                              static_cast<float>(1.0 - beta2), static_cast<float>(eps), static_cast<float>(-lr / bc1),
                              static_cast<float>(sqrt(bc2))));
  SB200_CUDA_CHECK(cudaGetLastError());
  return 0;
}
