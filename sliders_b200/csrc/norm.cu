// GroupNorm(+SiLU) and LayerNorm for channels-last bf16 activations (HBM-bound kernels: 16-byte vector
// loads, fp32 statistics, warp-shuffle / shared-memory reductions).
//
// Replaces torch.nn.GroupNorm + SiLU in diffusers ResnetBlock2D / Transformer2DModel / conv_norm_out and
// torch.nn.LayerNorm in BasicTransformerBlock (called under trainscripts/textsliders/train_util.py:242-247).
#include "common.h"
#include "ptx.cuh"

namespace sb200 {

// ------------------------------------------------------------------------------------------------
// GroupNorm statistics over (HW x C/G) elements per (batch, group); the input may be the
// channel concat of two NHWC sources.
// grid (chunks, B); block = (C/8) * rows_par threads: thread (r, cv) owns channel vector cv and walks
// rows r, r + rows_par, ... of its chunk.
// ------------------------------------------------------------------------------------------------
struct GnArgs {
  const __nv_bfloat16* x0;
  const __nv_bfloat16* x1;
  int ld0, ld1, C0, C;
  int HW, groups, cpg;
  int rows_per_block;
};

// Deterministic (atomic-free) reduction: per-thread partials -> shared memory -> one thread per group sums
// its channels in a fixed order -> partial[b][chunk][g] in global; gn_finalize_kernel sums the chunks in order.
__global__ void gn_stats_kernel(GnArgs a, float* __restrict__ partial) {
  pdl_trigger();
  pdl_wait();
  extern __shared__ float sh[];  // [rows_par][C][2]
  const int nvec = a.C >> 3;
  const int cv = threadIdx.x % nvec;
  const int r0 = threadIdx.x / nvec;
  const int rows_par = blockDim.x / nvec;
  const int b = blockIdx.y;
  const int c = cv << 3;
  const __nv_bfloat16* src;
  int ld, cc;
  if (c < a.C0) {
    src = a.x0, ld = a.ld0, cc = c;
  } else {
    src = a.x1, ld = a.ld1, cc = c - a.C0;
  }
  const int row_begin = blockIdx.x * a.rows_per_block;
  const int row_end = min(row_begin + a.rows_per_block, a.HW);
  float s[8], ss[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) s[i] = ss[i] = 0.f;
#pragma unroll 4  // independent 16-byte loads in flight per thread: the loop is latency-bound otherwise (2.4 TB/s)
  for (int r = row_begin + r0; r < row_end; r += rows_par) {
    const uint4 v = __ldg(reinterpret_cast<const uint4*>(src + (static_cast<size_t>(b) * a.HW + r) * ld + cc));
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float lo = bf16_lo(w[i]), hi = bf16_hi(w[i]);
      s[2 * i] += lo;
      ss[2 * i] += lo * lo;
      s[2 * i + 1] += hi;
      ss[2 * i + 1] += hi * hi;
    }
  }
  float* mine = sh + (static_cast<size_t>(r0) * a.C + c) * 2;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    mine[2 * i] = s[i];
    mine[2 * i + 1] = ss[i];
  }
  __syncthreads();
  for (int g = threadIdx.x; g < a.groups; g += blockDim.x) {
    float S = 0.f, SS = 0.f;
    for (int r = 0; r < rows_par; ++r) {
      const float* row = sh + (static_cast<size_t>(r) * a.C + g * a.cpg) * 2;
      for (int ci = 0; ci < a.cpg; ++ci) {
        S += row[2 * ci];
        SS += row[2 * ci + 1];
      }
    }
    float* out = partial + ((static_cast<size_t>(b) * gridDim.x + blockIdx.x) * a.groups + g) * 2;
    out[0] = S;
    out[1] = SS;
  }
}

// final[b][g] = {mean, rstd}; one warp per group, fixed-order lane-strided sum + shuffle tree (deterministic)
__global__ void gn_finalize_kernel(const float* __restrict__ partial, float* __restrict__ final_stats,
                                   int chunks, int groups, float inv_n, float eps) {
  pdl_trigger();
  pdl_wait();
  const int b = blockIdx.x;
  const int lane = threadIdx.x & 31;
  for (int g = threadIdx.x >> 5; g < groups; g += blockDim.x >> 5) {
    float S = 0.f, SS = 0.f;
    for (int k = lane; k < chunks; k += 32) {
      const float2 pp = *reinterpret_cast<const float2*>(partial + ((static_cast<size_t>(b) * chunks + k) * groups + g) * 2);
      S += pp.x;
      SS += pp.y;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      S += __shfl_xor_sync(0xffffffffu, S, o);
      SS += __shfl_xor_sync(0xffffffffu, SS, o);
    }
    if (lane == 0) {
      const float mean = S * inv_n;
      const float var = fmaxf(SS * inv_n - mean * mean, 0.f);
      final_stats[(static_cast<size_t>(b) * groups + g) * 2] = mean;
      final_stats[(static_cast<size_t>(b) * groups + g) * 2 + 1] = rsqrtf(var + eps);
    }
  }
}

struct GnApplyArgs {
  GnArgs in;
  const __nv_bfloat16* gamma;
  const __nv_bfloat16* beta;
  __nv_bfloat16* out;
  int ldo;
  int B;
  float eps;
  int silu;
};

// grid (chunks, B), block = (C/8) * rows_par threads like gn_stats_kernel: a thread owns one 8-channel vector,
// folds (mean, rstd, gamma, beta) into scale/shift once and then streams its rows: 16 B in, 8 FMA (+SiLU), 16 B out.
__global__ void gn_apply_kernel(GnApplyArgs a, const float* __restrict__ stats) {
  pdl_trigger();
  pdl_wait();
  const GnArgs& in = a.in;
  const int nvec = in.C >> 3;
  const int cv = threadIdx.x % nvec;
  const int r0 = threadIdx.x / nvec;
  const int rows_par = blockDim.x / nvec;
  const int b = blockIdx.y;
  const int c = cv << 3;
  const __nv_bfloat16* src;
  int ld, cc;
  if (c < in.C0) {
    src = in.x0, ld = in.ld0, cc = c;
  } else {
    src = in.x1, ld = in.ld1, cc = c - in.C0;
  }
  float sc[8], sh[8];
  {
    const uint4 gv = __ldg(reinterpret_cast<const uint4*>(a.gamma + c));
    const uint4 bv = __ldg(reinterpret_cast<const uint4*>(a.beta + c));
    const uint32_t gw[4] = {gv.x, gv.y, gv.z, gv.w};
    const uint32_t bw[4] = {bv.x, bv.y, bv.z, bv.w};
    const float* st = stats + static_cast<size_t>(b) * 2 * in.groups;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int g = (c + i) / in.cpg;
      const float mean = st[2 * g], rstd = st[2 * g + 1];
      const float gm = (i & 1) ? bf16_hi(gw[i >> 1]) : bf16_lo(gw[i >> 1]);
      const float bt = (i & 1) ? bf16_hi(bw[i >> 1]) : bf16_lo(bw[i >> 1]);
      sc[i] = rstd * gm;
      sh[i] = bt - mean * rstd * gm;
    }
  }
  const int row_begin = blockIdx.x * in.rows_per_block;
  const int row_end = min(row_begin + in.rows_per_block, in.HW);
#pragma unroll 4
  for (int r = row_begin + r0; r < row_end; r += rows_par) {
    const size_t pix = static_cast<size_t>(b) * in.HW + r;
    const uint4 v = __ldg(reinterpret_cast<const uint4*>(src + pix * ld + cc));
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
    float f[8];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      f[2 * i] = fmaf(bf16_lo(w[i]), sc[2 * i], sh[2 * i]);
      f[2 * i + 1] = fmaf(bf16_hi(w[i]), sc[2 * i + 1], sh[2 * i + 1]);
    }
    if (a.silu) {
#pragma unroll
      for (int i = 0; i < 8; ++i) f[i] = silu_f(f[i]);
    }
    uint4 o;
    o.x = pack_bf16x2(f[0], f[1]);
    o.y = pack_bf16x2(f[2], f[3]);
    o.z = pack_bf16x2(f[4], f[5]);
    o.w = pack_bf16x2(f[6], f[7]);
    *reinterpret_cast<uint4*>(a.out + pix * a.ldo + c) = o;
  }
}

// ------------------------------------------------------------------------------------------------
// LayerNorm: one warp per row, the row lives in registers between the mean and variance passes.
// ------------------------------------------------------------------------------------------------
constexpr int kLnMaxVec = 8;  // C <= 8 * 32 * 8 = 2048

template <int NV>  // 16-byte vectors per lane: C <= NV * 256
__global__ void layernorm_kernel(const __nv_bfloat16* __restrict__ x, int ldx,
                                 const __nv_bfloat16* __restrict__ gamma,
                                 const __nv_bfloat16* __restrict__ beta, __nv_bfloat16* __restrict__ out,
                                 int ldo, int M, int C, float eps) {
  pdl_trigger();
  // gamma / beta staged once per block (frozen parameters: readable before the predecessor grid has finished), so the
  // 8 rows of a block do not each re-read 2 x C x 2 bytes through L1 / L2 — that doubled the kernel's memory traffic
  extern __shared__ uint4 gb_sh[];  // [2][C / 8]
  const int warps_per_block = blockDim.x >> 5;
  const int lane = threadIdx.x & 31;
  const int nvec = C >> 3;
  for (int v = threadIdx.x; v < nvec; v += blockDim.x) {
    gb_sh[v] = __ldg(reinterpret_cast<const uint4*>(gamma) + v);
    gb_sh[nvec + v] = __ldg(reinterpret_cast<const uint4*>(beta) + v);
  }
  __syncthreads();
  pdl_wait();
  for (int row = blockIdx.x * warps_per_block + (threadIdx.x >> 5); row < M;
       row += gridDim.x * warps_per_block) {
    const __nv_bfloat16* xr = x + static_cast<size_t>(row) * ldx;
    float f[NV][8];
    float sum = 0.f;
#pragma unroll
    for (int k = 0; k < NV; ++k) {
      const int v = lane + k * 32;
      if (v < nvec) {
        const uint4 u = __ldg(reinterpret_cast<const uint4*>(xr + v * 8));
        const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          f[k][2 * i] = bf16_lo(w[i]);
          f[k][2 * i + 1] = bf16_hi(w[i]);
          sum += f[k][2 * i] + f[k][2 * i + 1];
        }
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    const float mean = sum / C;
    float var = 0.f;
#pragma unroll
    for (int k = 0; k < NV; ++k) {
      if (lane + k * 32 < nvec) {
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const float d = f[k][i] - mean;
          var += d * d;
        }
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) var += __shfl_xor_sync(0xffffffffu, var, o);
    const float rstd = rsqrtf(var / C + eps);
    __nv_bfloat16* orow = out + static_cast<size_t>(row) * ldo;
#pragma unroll
    for (int k = 0; k < NV; ++k) {
      const int v = lane + k * 32;
      if (v < nvec) {
        const uint4 gv = gb_sh[v];
        const uint4 bv = gb_sh[nvec + v];
        const uint32_t gw[4] = {gv.x, gv.y, gv.z, gv.w};
        const uint32_t bw[4] = {bv.x, bv.y, bv.z, bv.w};
        uint32_t o[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float y0 = (f[k][2 * i] - mean) * rstd * bf16_lo(gw[i]) + bf16_lo(bw[i]);
          const float y1 = (f[k][2 * i + 1] - mean) * rstd * bf16_hi(gw[i]) + bf16_hi(bw[i]);
          o[i] = pack_bf16x2(y0, y1);
        }
        *reinterpret_cast<uint4*>(orow + v * 8) = make_uint4(o[0], o[1], o[2], o[3]);
      }
    }
  }
}

}  // namespace sb200

using namespace sb200;

extern "C" int sb200_groupnorm(void* handle, void* stream, const void* x0, int ldx0, int C0, const void* x1,
                               int ldx1, int C1, const void* gamma, const void* beta, void* out, int ldo,
                               int B, int HW, int groups, float eps, int silu, float* stats_ws) {
  Ctx* ctx = as_ctx(handle);
  SB200_REQUIRE(ctx, "groupnorm: NULL handle");
  if (!x1) C1 = 0;
  const int C = C0 + C1;
  SB200_REQUIRE(B > 0 && HW > 0 && C0 > 0 && C0 % 8 == 0 && C1 % 8 == 0, "groupnorm: dims (C0=%d C1=%d)", C0, C1);
  SB200_REQUIRE(groups > 0 && C % groups == 0, "groupnorm: C=%d not divisible by groups=%d", C, groups);
  SB200_REQUIRE(ldx0 % 8 == 0 && ldo % 8 == 0 && (C1 == 0 || ldx1 % 8 == 0), "groupnorm: leading dims");
  // the stats kernel keeps [rows_par][C][2] fp32 partials in dynamic shared memory without opting in above 48 KB
  SB200_REQUIRE(gn_stats_smem_ok(C), "groupnorm: C=%d too large", C);
  SB200_REQUIRE(stats_ws && gamma && beta, "groupnorm: NULL argument");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const bool pdl = static_cast<long long>(B) * HW * C <= (16LL << 20);
  GnArgs a;
  a.x0 = static_cast<const __nv_bfloat16*>(x0);
  a.x1 = static_cast<const __nv_bfloat16*>(x1);
  a.ld0 = ldx0;
  a.ld1 = ldx1;
  a.C0 = C0;
  a.C = C;
  a.HW = HW;
  a.groups = groups;
  a.cpg = C / groups;
  const GnShape g = gn_shape(ctx, B, HW, C);
  a.rows_per_block = g.rows_per_block;
  // workspace: partial[B][chunks][G][2] followed by final[B][G][2]
  float* final_stats = stats_ws + SB200_GN_STATS_OFFSET(B, groups);
  SB200_CUDA_CHECK(launch_pdl(gn_stats_kernel, dim3(g.chunks, B), dim3(g.threads), sizeof(float) * 2 * C * g.rows_par,
                              s, pdl, a, stats_ws));
  SB200_CUDA_CHECK(launch_pdl(gn_finalize_kernel, dim3(B), dim3(1024), 0, s, pdl, stats_ws, final_stats, g.chunks,
                              groups, 1.f / (static_cast<float>(HW) * a.cpg), eps));
  GnApplyArgs ap;
  ap.in = a;
  ap.gamma = static_cast<const __nv_bfloat16*>(gamma);
  ap.beta = static_cast<const __nv_bfloat16*>(beta);
  ap.out = static_cast<__nv_bfloat16*>(out);
  ap.ldo = ldo;
  ap.B = B;
  ap.eps = eps;
  ap.silu = silu;
  SB200_CUDA_CHECK(launch_pdl(gn_apply_kernel, dim3(g.chunks, B), dim3(g.threads), 0, s, pdl, ap, final_stats));
  return 0;
}

extern "C" int sb200_layernorm(void* handle, void* stream, const void* x, int ldx, const void* gamma,
                               const void* beta, void* out, int ldo, int M, int C, float eps) {
  Ctx* ctx = as_ctx(handle);
  SB200_REQUIRE(ctx, "layernorm: NULL handle");
  SB200_REQUIRE(M > 0 && C > 0 && C % 8 == 0 && C <= kLnMaxVec * 256, "layernorm: C=%d unsupported", C);
  SB200_REQUIRE(ldx % 8 == 0 && ldo % 8 == 0, "layernorm: leading dims");
  const int warps = 8;
  const int blocks = grid_cap(ctx, M, warps, 16);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const bool pdl = static_cast<long long>(M) * C <= (8LL << 20);
#define SB200_LN(NV)                                                                                      \
  SB200_CUDA_CHECK(launch_pdl(layernorm_kernel<NV>, dim3(blocks), dim3(warps * 32), static_cast<size_t>(C) * 4, st, pdl, \
                              static_cast<const __nv_bfloat16*>(x), ldx, static_cast<const __nv_bfloat16*>(gamma), \
                              static_cast<const __nv_bfloat16*>(beta), static_cast<__nv_bfloat16*>(out), ldo, M, C, \
                              eps))
  if (C <= 256)
    SB200_LN(1);
  else if (C <= 768)
    SB200_LN(3);
  else if (C <= 1280)
    SB200_LN(5);
  else
    SB200_LN(8);
#undef SB200_LN
  SB200_CUDA_CHECK(cudaGetLastError());
  return 0;
}
