// Flash-attention backward for sm_90a (wgmma + TMA), the gradient path of
//   loss.backward()  (trainscripts/textsliders/train_lora_xl.py:345; train_lora-scale-xl.py:340,372)
// through diffusers' Attention (xformers memory_efficient_attention backward in the reference).
//
// With S = scale * Q K^T, P = softmax(S), O = P V and D[q] = sum_d dO[q,d] O[q,d]:
//   dV = P^T dO          dP = dO V^T          dS = P o (dP - D)          dQ = scale dS K      dK = scale dS^T Q
// One kernel template, three launches.  Each CTA keeps a 128-row "resident" pair of tiles (64 rows per consumer
// warpgroup) and streams kT-row tiles:
//   mode 0 (dQ)  resident R1 = Q, R2 = dO   streamed T1 = K_j, T2 = V_j    out = dQ += dS T1
//   mode 1 (dV)  resident R1 = K            streamed T1 = Q_i, T2 = dO_i   out = dV += P^T T2
//   mode 2 (dK)  resident R1 = K, R2 = V    streamed T1 = Q_i, T2 = dO_i   out = dK += dS^T T1
// so that in every mode
//   S'  = R1 T1^T   and   dP' = R2 T2^T   (wgmma m64 x kT x 16 from shared memory, fp32 in registers)
//   p = exp2(s * scale * log2e - lse), ds = p (dp - D) scale, packed to bf16 in place as the A operand of
//   out += {P | dS} . T   (wgmma m64 x 64 x 16 per 64 head columns, A from registers, the streamed tile MN-major).
// dV and dK come from separate launches so that one accumulator holds the registers of a thread.
// The log-sum-exp comes from the forward kernel (attention.cu, `lse`), D from attn_bwd_prep_kernel.  Modes 1 / 2 read
// lse / D per streamed column, mode 0 per resident row.  Head dim padded to ND x 64 columns by TMA zero fill as in
// the forward.  Deterministic: no atomics (each output tile has one owner CTA).
//
// Query split (sb200_attention_bwd_ws): cross-attention has one 77-row resident tile per (head, batch), so modes 1 / 2
// would run heads x B CTAs (8 for SD1.x at batch 1) that each stream every query.  With a scratch buffer, modes 1 / 2
// instead run a (nsplit, heads, B) grid: CTA s streams queries [s q_split, (s + 1) q_split) and stores its fp32 partial
// dV / dK tile to the scratch; attn_bwd_reduce_kernel sums the nsplit partials in split order into the bf16 outputs.
#include "common.h"
#include "ptx.cuh"

namespace sb200 {

constexpr int kBwdThreads = 288;        // two consumer warpgroups + the TMA warp
constexpr uint32_t kRTile = 128 * 128;  // 128 rows x 64 bf16, SWIZZLE_128B

template <int ND>
struct AttnBwdCfg {
  static constexpr int kT = ND == 3 ? 32 : 64;  // streamed rows per tile (the output accumulator takes the registers)
  static constexpr int kStages = 2;
  static constexpr uint32_t kTChunk = kT * 128;  // 64 head columns of a streamed tile
  static constexpr uint32_t kRBytes = kRTile * ND;
  static constexpr uint32_t kTBytes = kTChunk * ND;
  static constexpr int kSmem = 2 * kRBytes + kStages * 2 * kTBytes + 1024 /*barriers*/ + 1024 /*align*/;
};

struct AttnBwdParams {
  CUtensorMap tmR1, tmR2, tmT1, tmT2;
  __nv_bfloat16* out;
  int ld;
  const float* lse;   // [B, heads, Sq]
  const float* dsum;  // [B, heads, Sq]
  int Sq;
  int n_res;     // valid resident rows in total (mode 0: Sq, modes 1 / 2: Skv)
  int n_stream;  // valid streamed rows in total (mode 0: Skv, modes 1 / 2: Sq)
  int d;
  int mode;
  float scale_log2, scale;
  float* ws;    // modes 1 / 2 query split: [nsplit][B * n_res][ld_ws] fp32 partials (NULL: one CTA per resident tile)
  int q_split;  // streamed rows per split (a multiple of 64)
  int ld_ws;    // heads * d
};

__device__ __forceinline__ float bwd_exp2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

template <int kN>
__device__ __forceinline__ void wgmma_ss_t(float* d, uint64_t a, uint64_t b, uint32_t acc) {
  if constexpr (kN == 64)
    wgmma_ss_n64(d, a, b, acc);
  else
    wgmma_ss_n32(d, a, b, acc);
}

template <int ND>
__global__ void __launch_bounds__(kBwdThreads, 1) attention_bwd_kernel(const __grid_constant__ AttnBwdParams p) {
  constexpr int kT = AttnBwdCfg<ND>::kT;
  constexpr int kStages = AttnBwdCfg<ND>::kStages;
  constexpr uint32_t kRBytes = AttnBwdCfg<ND>::kRBytes;
  constexpr uint32_t kTBytes = AttnBwdCfg<ND>::kTBytes;
  constexpr uint32_t kTChunk = AttnBwdCfg<ND>::kTChunk;
  pdl_trigger();
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_addr = smem_u32(smem_raw);
  const uint32_t base = (raw_addr + 1023u) & ~1023u;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const bool split = p.ws != nullptr;
  const int rt = split ? 0 : blockIdx.x, head = blockIdx.y, b = blockIdx.z;
  const int q0 = split ? blockIdx.x * p.q_split : 0;                       // first streamed row
  const int n_str = split ? min(p.q_split, p.n_stream - q0) : p.n_stream;  // streamed rows of this CTA
  const int mode = p.mode;
  const bool need_dp = mode != 1;

  const uint32_t sR1 = base;
  const uint32_t sR2 = sR1 + kRBytes;
  const uint32_t sT1 = sR2 + kRBytes;            // kStages x kTBytes
  const uint32_t sT2 = sT1 + kStages * kTBytes;  // kStages x kTBytes
  const uint32_t bars = sT2 + kStages * kTBytes;
  const uint32_t bar_r = bars;
  const uint32_t bar_full = bars + 8;  // kStages
  const uint32_t bar_empty = bar_full + 8 * kStages;

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&p.tmR1);
    tma_prefetch_desc(&p.tmR2);
    tma_prefetch_desc(&p.tmT1);
    tma_prefetch_desc(&p.tmT2);
  }
  if (warp == 1 && lane == 0) {
    mbar_init(bar_r, 1);
    for (int i = 0; i < kStages; ++i) {
      mbar_init(bar_full + 8 * i, 1);
      mbar_init(bar_empty + 8 * i, 2);  // one arrival per consumer warpgroup
    }
    fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();
  const int n = (n_str + kT - 1) / kT;
  const size_t stat_base = (static_cast<size_t>(b) * gridDim.y + head) * p.Sq;

  if (warp == 8) {
    // ------------------------------------------------------------------ TMA producer, converged warp
    if (elect_one()) {
      mbar_expect_tx(bar_r, need_dp ? 2 * kRBytes : kRBytes);
#pragma unroll
      for (int i = 0; i < ND; ++i) {
        tma_load_4d(sR1 + i * kRTile, &p.tmR1, bar_r, i * 64, head, rt * 128, b);
        if (need_dp) tma_load_4d(sR2 + i * kRTile, &p.tmR2, bar_r, i * 64, head, rt * 128, b);
      }
    }
    __syncwarp();
    for (int t = 0; t < n; ++t) {
      const int s = t % kStages;
      const uint32_t ph = (t / kStages) & 1;
      mbar_wait(bar_empty + 8 * s, ph ^ 1u);
      if (elect_one()) {
        mbar_expect_tx(bar_full + 8 * s, 2 * kTBytes);
#pragma unroll
        for (int i = 0; i < ND; ++i) {
          tma_load_4d(sT1 + s * kTBytes + i * kTChunk, &p.tmT1, bar_full + 8 * s, i * 64, head, q0 + t * kT, b);
          tma_load_4d(sT2 + s * kTBytes + i * kTChunk, &p.tmT2, bar_full + 8 * s, i * 64, head, q0 + t * kT, b);
        }
      }
      __syncwarp();
    }
    return;
  }

  // ------------------------------------------------------------------ consumer warpgroups
  const int wg = warp >> 2, wl = warp & 3;
  const bool signal = (threadIdx.x & 127) == 0;
  const int dsteps = (p.d + 15) >> 4;
  const uint32_t roff = static_cast<uint32_t>(wg) * 64u * 128u;  // this warpgroup's 64 resident rows
  const int row0 = rt * 128 + wg * 64 + wl * 16 + (lane >> 2);   // resident rows row0 and row0 + 8 of this thread
  float lse_r[2] = {INFINITY, INFINITY}, d_r[2] = {0.f, 0.f};
  if (mode == 0) {
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      if (row0 + 8 * r < p.n_res) {
        lse_r[r] = __ldg(p.lse + stat_base + row0 + 8 * r);
        d_r[r] = __ldg(p.dsum + stat_base + row0 + 8 * r);
      }
    }
  }
  float acc[ND * 32];
#pragma unroll
  for (int i = 0; i < ND * 32; ++i) acc[i] = 0.f;
  mbar_wait(bar_r, 0);
  for (int t = 0; t < n; ++t) {
    const int s = t % kStages;
    const uint32_t ph = (t / kStages) & 1;
    const int left = n_str - t * kT;  // valid streamed rows in this tile
    // per-column statistics of the streamed queries (modes 1 / 2): columns 8 e + 2 (lane % 4) + {0, 1}
    float lse_c[kT / 4], d_c[kT / 4];
    if (mode != 0) {
#pragma unroll
      for (int e = 0; e < kT / 8; ++e)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int col = 8 * e + 2 * (lane & 3) + h;
          lse_c[2 * e + h] = col < left ? __ldg(p.lse + stat_base + q0 + t * kT + col) : INFINITY;
          d_c[2 * e + h] = col < left ? __ldg(p.dsum + stat_base + q0 + t * kT + col) : 0.f;
        }
    }
    float sc[kT / 2], dp[kT / 2];
    mbar_wait(bar_full + 8 * s, ph);
    wgmma_fence();
    for (int k = 0; k < dsteps; ++k) {
      const uint32_t ro = static_cast<uint32_t>(k >> 2) * kRTile + roff + static_cast<uint32_t>(k & 3) * 32;
      const uint32_t to = static_cast<uint32_t>(k >> 2) * kTChunk + static_cast<uint32_t>(k & 3) * 32;
      wgmma_ss_t<kT>(sc, gmma_desc_sw128(sR1 + ro), gmma_desc_sw128(sT1 + s * kTBytes + to), k != 0);
    }
    if (need_dp) {
      for (int k = 0; k < dsteps; ++k) {
        const uint32_t ro = static_cast<uint32_t>(k >> 2) * kRTile + roff + static_cast<uint32_t>(k & 3) * 32;
        const uint32_t to = static_cast<uint32_t>(k >> 2) * kTChunk + static_cast<uint32_t>(k & 3) * 32;
        wgmma_ss_t<kT>(dp, gmma_desc_sw128(sR2 + ro), gmma_desc_sw128(sT2 + s * kTBytes + to), k != 0);
      }
    }
    wgmma_commit();
    wgmma_wait<0>();
#pragma unroll
    for (int i = 0; i < kT / 2; ++i) {
      reg_fence(sc[i]);
      reg_fence(dp[i]);
    }
    uint32_t pa[kT / 16][4];  // P (mode 1) or dS as bf16 A fragments, one group of four registers per 16 streamed rows
#pragma unroll
    for (int i = 0; i < kT / 2; i += 2) {
      const int r = (i >> 1) & 1;
      const int cp = 2 * (i >> 2);  // index of this pair's first column in lse_c / d_c
      float v[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int col = 8 * (i >> 2) + 2 * (lane & 3) + h;
        float pv, dv;
        if (mode == 0) {
          pv = col < left ? bwd_exp2(fmaf(sc[i + h], p.scale_log2, -lse_r[r])) : 0.f;  // keys beyond Skv
          dv = d_r[r];
        } else {
          pv = bwd_exp2(fmaf(sc[i + h], p.scale_log2, -lse_c[cp + h]));  // lse = inf beyond Sq: p = 0
          dv = d_c[cp + h];
        }
        v[h] = mode == 1 ? pv : pv * (dp[i + h] - dv) * p.scale;
      }
      pa[i >> 3][(i >> 1) & 3] = pack_bf16x2(v[0], v[1]);
    }
    const uint32_t sB = (mode == 1 ? sT2 : sT1) + s * kTBytes;
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < kT / 16; ++kk) {
#pragma unroll
      for (int c = 0; c < ND; ++c) wgmma_rs_n64_tb(acc + 32 * c, pa[kk], gmma_desc_sw128(sB + c * kTChunk + kk * 2048), 1u);
    }
    wgmma_commit();
    wgmma_wait<0>();
#pragma unroll
    for (int i = 0; i < ND * 32; ++i) reg_fence(acc[i]);
    if (signal) mbar_arrive(bar_empty + 8 * s);
  }

  // ---- write the accumulator (first d columns of each padded head)
  if (split) {
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int grow = row0 + 8 * r;
      if (grow >= p.n_res) continue;
      float* wp = p.ws + ((static_cast<size_t>(blockIdx.x) * gridDim.z + b) * p.n_res + grow) * p.ld_ws +
                  static_cast<size_t>(head) * p.d;
#pragma unroll
      for (int c = 0; c < ND; ++c) {
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          const int col = c * 64 + 8 * e + 2 * (lane & 3);
          if (col < p.d) {
            const int i = 32 * c + 4 * e + 2 * r;
            *reinterpret_cast<float2*>(wp + col) = make_float2(acc[i], acc[i + 1]);
          }
        }
      }
    }
    return;
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int grow = row0 + 8 * r;
    if (grow >= p.n_res) continue;
    __nv_bfloat16* op = p.out + (static_cast<size_t>(b) * p.n_res + grow) * p.ld + static_cast<size_t>(head) * p.d;
#pragma unroll
    for (int c = 0; c < ND; ++c) {
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const int col = c * 64 + 8 * e + 2 * (lane & 3);
        if (col < p.d) {
          const int i = 32 * c + 4 * e + 2 * r;
          *reinterpret_cast<uint32_t*>(op + col) = pack_bf16x2(acc[i], acc[i + 1]);
        }
      }
    }
  }
}

// D[b, head, q] = sum_d dO[q, head*d + i] * O[q, head*d + i]; one thread per (row, head)
__global__ void attn_bwd_prep_kernel(const __nv_bfloat16* __restrict__ o, int ldo,
                                     const __nv_bfloat16* __restrict__ dout, int lddo, float* __restrict__ dsum,
                                     int B, int heads, int Sq, int d) {
  pdl_trigger();
  pdl_wait();
  const size_t idx = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  const size_t total = static_cast<size_t>(B) * Sq * heads;
  if (idx >= total) return;
  const int h = static_cast<int>(idx % heads);
  const size_t rowi = idx / heads;  // b * Sq + q
  const __nv_bfloat16* po = o + rowi * ldo + h * d;
  const __nv_bfloat16* pd = dout + rowi * lddo + h * d;
  float acc = 0.f;
  for (int i = 0; i < d; i += 8) {
    const uint4 a = __ldg(reinterpret_cast<const uint4*>(po + i));
    const uint4 g = __ldg(reinterpret_cast<const uint4*>(pd + i));
    const uint32_t aw[4] = {a.x, a.y, a.z, a.w}, gw[4] = {g.x, g.y, g.z, g.w};
#pragma unroll
    for (int k = 0; k < 4; ++k) acc += bf16_lo(aw[k]) * bf16_lo(gw[k]) + bf16_hi(aw[k]) * bf16_hi(gw[k]);
  }
  const int bq = static_cast<int>(rowi / Sq);
  const int qi = static_cast<int>(rowi % Sq);
  dsum[(static_cast<size_t>(bq) * heads + h) * Sq + qi] = acc;
}

// out[row, j] = sum over s (in order) of ws[s][row][j]; blockIdx.y: 0 = dV (first half of the scratch), 1 = dK.
// Four columns per thread (cols is a multiple of 8).
__global__ void attn_bwd_reduce_kernel(const float* __restrict__ ws, int nsplit, int rows, int cols,
                                       __nv_bfloat16* __restrict__ dv, int lddv, __nv_bfloat16* __restrict__ dk,
                                       int lddk) {
  pdl_trigger();
  pdl_wait();
  const size_t part = static_cast<size_t>(rows) * cols;
  const size_t idx = (static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x) * 4;
  if (idx >= part) return;
  const float* src = ws + static_cast<size_t>(blockIdx.y) * nsplit * part + idx;
  float4 a = __ldg(reinterpret_cast<const float4*>(src));
  for (int s = 1; s < nsplit; ++s) {
    const float4 v = __ldg(reinterpret_cast<const float4*>(src + s * part));
    a.x += v.x;
    a.y += v.y;
    a.z += v.z;
    a.w += v.w;
  }
  const int row = static_cast<int>(idx / cols), col = static_cast<int>(idx % cols);
  __nv_bfloat16* o =
      blockIdx.y == 0 ? dv + static_cast<size_t>(row) * lddv + col : dk + static_cast<size_t>(row) * lddk + col;
  *reinterpret_cast<uint2*>(o) = make_uint2(pack_bf16x2(a.x, a.y), pack_bf16x2(a.z, a.w));
}

template <int ND>
static int launch_attention_bwd(cudaStream_t stream, const AttnBwdParams& p, dim3 grid) {
  static bool attr_set = false;
  if (!attr_set) {
    SB200_CUDA_CHECK(cudaFuncSetAttribute(attention_bwd_kernel<ND>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                          AttnBwdCfg<ND>::kSmem));
    attr_set = true;
  }
  SB200_CUDA_CHECK(launch_pdl(attention_bwd_kernel<ND>, grid, dim3(kBwdThreads), AttnBwdCfg<ND>::kSmem, stream, p));
  SB200_CUDA_CHECK(cudaGetLastError());
  return 0;
}

static int launch_attention_bwd_d(cudaStream_t stream, const AttnBwdParams& p, dim3 grid) {
  if (p.d <= 64) return launch_attention_bwd<1>(stream, p, grid);
  if (p.d <= 128) return launch_attention_bwd<2>(stream, p, grid);
  return launch_attention_bwd<3>(stream, p, grid);
}

static int streamed_rows(int head_dim) {
  return head_dim <= 64 ? AttnBwdCfg<1>::kT : (head_dim <= 128 ? AttnBwdCfg<2>::kT : AttnBwdCfg<3>::kT);
}

static int make_map(Ctx* ctx, CUtensorMap* m, const void* ptr, int ld, int d, int heads, int S, int B, uint32_t rows) {
  const uint64_t dims[4] = {static_cast<uint64_t>(d), static_cast<uint64_t>(heads), static_cast<uint64_t>(S),
                            static_cast<uint64_t>(B)};
  const uint64_t strides[3] = {static_cast<uint64_t>(d) * 2, static_cast<uint64_t>(ld) * 2,
                               static_cast<uint64_t>(ld) * 2 * S};
  const uint32_t box[4] = {64, 1, rows, 1};
  return make_tmap_bf16(ctx, m, ptr, 4, dims, strides, box);
}

// Query splits of the dK / dV launches (include/sb200.h: SB200_ATTN_BWD_SPLITS bounds the result, which sizes the
// scratch); *q_split receives the streamed rows per split.  1 = no split.
static int attention_bwd_nsplit(int B, int heads, int Sq, int Skv, int* q_split) {
  const int want = SB200_ATTN_BWD_SPLITS(B, heads, Sq, Skv);
  if (want <= 1) return 1;
  const int per = ((Sq + want - 1) / want + 63) / 64 * 64;
  *q_split = per;
  return (Sq + per - 1) / per;
}

}  // namespace sb200

using namespace sb200;

static int attention_bwd_impl(void* handle, void* stream, const void* q, int ldq, const void* k, int ldk,
                              const void* v, int ldv, const void* o, int ldo, const void* dout, int lddo,
                              const float* lse, float* dsum, void* dq, int lddq, void* dk, int lddk, void* dv,
                              int lddv, int B, int heads, int Sq, int Skv, int head_dim, float scale, float* ws,
                              size_t ws_floats) {
  pdl_hint() = true;
  Ctx* ctx = as_ctx(handle);
  SB200_REQUIRE(ctx, "attention_bwd: NULL handle");
  SB200_REQUIRE(B > 0 && heads > 0 && Sq > 0 && Skv > 0, "attention_bwd: bad dims");
  SB200_REQUIRE(head_dim >= 8 && head_dim <= 192 && head_dim % 8 == 0, "attention_bwd: head dim %d unsupported",
                head_dim);
  SB200_REQUIRE(q && k && v && o && dout && lse && dsum && dq, "attention_bwd: NULL argument");
  SB200_REQUIRE((dk == nullptr) == (dv == nullptr), "attention_bwd: dk and dv must be given together");
  SB200_REQUIRE(ldq % 8 == 0 && ldk % 8 == 0 && ldv % 8 == 0 && ldo % 8 == 0 && lddo % 8 == 0 && lddq % 8 == 0 &&
                    (!dk || (lddk % 8 == 0 && lddv % 8 == 0)),
                "attention_bwd: leading dims must be multiples of 8");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  {
    const size_t total = static_cast<size_t>(B) * Sq * heads;
    SB200_CUDA_CHECK(launch_pdl(attn_bwd_prep_kernel, dim3(static_cast<unsigned>((total + 255) / 256)), dim3(256), 0, s,
                                static_cast<const __nv_bfloat16*>(o), ldo, static_cast<const __nv_bfloat16*>(dout), lddo,
                                dsum, B, heads, Sq, head_dim));
    SB200_CUDA_CHECK(cudaGetLastError());
  }
  int st;
  AttnBwdParams p;
  memset(&p, 0, sizeof(p));
  p.lse = lse;
  p.dsum = dsum;
  p.Sq = Sq;
  p.d = head_dim;
  p.scale = scale;
  p.scale_log2 = scale * 1.4426950408889634f;
  const uint32_t trows = static_cast<uint32_t>(streamed_rows(head_dim));
  // ---- dQ: resident (Q, dO) tiles, streamed (K, V)
  p.mode = 0;
  p.n_res = Sq;
  p.n_stream = Skv;
  p.out = static_cast<__nv_bfloat16*>(dq);
  p.ld = lddq;
  if ((st = make_map(ctx, &p.tmR1, q, ldq, head_dim, heads, Sq, B, 128))) return st;
  if ((st = make_map(ctx, &p.tmR2, dout, lddo, head_dim, heads, Sq, B, 128))) return st;
  if ((st = make_map(ctx, &p.tmT1, k, ldk, head_dim, heads, Skv, B, trows))) return st;
  if ((st = make_map(ctx, &p.tmT2, v, ldv, head_dim, heads, Skv, B, trows))) return st;
  if ((st = launch_attention_bwd_d(s, p, dim3((Sq + 127) / 128, heads, B))) || !dk) return st;
  // ---- dV, then dK: resident (K, V) tiles, streamed (Q, dO)
  p.n_res = Skv;
  p.n_stream = Sq;
  if ((st = make_map(ctx, &p.tmR1, k, ldk, head_dim, heads, Skv, B, 128))) return st;
  if ((st = make_map(ctx, &p.tmR2, v, ldv, head_dim, heads, Skv, B, 128))) return st;
  if ((st = make_map(ctx, &p.tmT1, q, ldq, head_dim, heads, Sq, B, trows))) return st;
  if ((st = make_map(ctx, &p.tmT2, dout, lddo, head_dim, heads, Sq, B, trows))) return st;
  const int nsplit = ws ? attention_bwd_nsplit(B, heads, Sq, Skv, &p.q_split) : 1;
  if (nsplit > 1) {
    const size_t part = static_cast<size_t>(nsplit) * B * Skv * heads * head_dim;
    SB200_REQUIRE(ws_floats >= 2 * part, "attention_bwd: scratch of %zu floats, %zu needed", ws_floats, 2 * part);
    const dim3 gs(nsplit, heads, B);
    p.ld_ws = heads * head_dim;
    p.mode = 1;
    p.ws = ws;
    if ((st = launch_attention_bwd_d(s, p, gs))) return st;
    p.mode = 2;
    p.ws = ws + part;
    if ((st = launch_attention_bwd_d(s, p, gs))) return st;
    const size_t quads = static_cast<size_t>(B) * Skv * heads * head_dim / 4;
    SB200_CUDA_CHECK(launch_pdl(attn_bwd_reduce_kernel, dim3(static_cast<unsigned>((quads + 255) / 256), 2), dim3(256),
                                0, s, static_cast<const float*>(ws), nsplit, B * Skv, heads * head_dim,
                                static_cast<__nv_bfloat16*>(dv), lddv, static_cast<__nv_bfloat16*>(dk), lddk));
    SB200_CUDA_CHECK(cudaGetLastError());
    return 0;
  }
  const dim3 gk((Skv + 127) / 128, heads, B);
  p.mode = 1;
  p.out = static_cast<__nv_bfloat16*>(dv);
  p.ld = lddv;
  if ((st = launch_attention_bwd_d(s, p, gk))) return st;
  p.mode = 2;
  p.out = static_cast<__nv_bfloat16*>(dk);
  p.ld = lddk;
  return launch_attention_bwd_d(s, p, gk);
}

extern "C" int sb200_attention_bwd(void* handle, void* stream, const void* q, int ldq, const void* k, int ldk,
                                   const void* v, int ldv, const void* o, int ldo, const void* dout, int lddo,
                                   const float* lse, float* dsum, void* dq, int lddq, void* dk, int lddk, void* dv,
                                   int lddv, int B, int heads, int Sq, int Skv, int head_dim, float scale) {
  return attention_bwd_impl(handle, stream, q, ldq, k, ldk, v, ldv, o, ldo, dout, lddo, lse, dsum, dq, lddq, dk, lddk,
                            dv, lddv, B, heads, Sq, Skv, head_dim, scale, nullptr, 0);
}

extern "C" int sb200_attention_bwd_ws(void* handle, void* stream, const void* q, int ldq, const void* k, int ldk,
                                      const void* v, int ldv, const void* o, int ldo, const void* dout, int lddo,
                                      const float* lse, float* dsum, void* dq, int lddq, void* dk, int lddk, void* dv,
                                      int lddv, int B, int heads, int Sq, int Skv, int head_dim, float scale, float* ws,
                                      size_t ws_floats) {
  SB200_REQUIRE(ws || ws_floats == 0, "attention_bwd_ws: NULL scratch");
  return attention_bwd_impl(handle, stream, q, ldq, k, ldk, v, ldv, o, ldo, dout, lddo, lse, dsum, dq, lddq, dk, lddk,
                            dv, lddv, B, heads, Sq, Skv, head_dim, scale, ws, ws_floats);
}
