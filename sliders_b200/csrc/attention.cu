// Flash-attention forward for sm_90a:  O = softmax(Q K^T * scale) V  per (batch, head), head dim d <= 192
// (SDXL: 64; SD1.x: 40 / 80 / 160).  The head dim is padded to ND x 64 columns by TMA's out-of-bounds zero
// fill: Q/K/V are addressed through 4-D descriptors (d, heads, tokens, batch), so a 64-wide box that sticks out
// of a 40- or 80-wide head reads zeros, never the neighbouring head.
//
// One CTA per (128-query tile, head, batch), 288 threads:
//   warp 8      TMA producer: Q tile once, then K / V tiles (KV keys x ND x 64) through a ring of stages
//   warps 0..7  two consumer warpgroups, 64 query rows each:
//                 S = Q K^T   wgmma m64 x KV x 16 from shared memory, fp32 in registers
//                 online softmax on the accumulator fragment (each thread holds two rows; a row's max / sum is
//                 reduced over the four threads of a quad), P packed to bf16 in place as the A operand of
//                 O += P V   wgmma m64 x 64 x 16 per 64 columns of the head, A from registers, V MN-major from smem
// The two warpgroups run independently, so one's softmax overlaps the other's tensor work.  KV = 128 keys for
// d <= 64 and 64 keys for wider heads (the O accumulator takes the registers).  Keys beyond Skv are masked to -inf;
// TMA zero-fills the out-of-range rows.
//
// Replaces the attention processor that diffusers' Attention calls (xformers memory_efficient_attention /
// torch SDPA; reference: trainscripts/textsliders/train_lora_xl.py:79-80, train_lora.py:68).
#include "common.h"
#include "ptx.cuh"

namespace sb200 {

constexpr int kAttnThreads = 288;       // two consumer warpgroups + the TMA warp
constexpr int kQTileBytes = 128 * 128;  // 128 rows x 64 bf16

__device__ __forceinline__ float fast_exp2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

template <int ND>
struct AttnCfg {
  static constexpr int kKV = ND == 1 ? 128 : 64;  // keys per K / V tile
  static constexpr int kStages = 2;
  static constexpr uint32_t kKVBytes = kKV * 128 * ND;  // one K or V tile
  static constexpr int kSmem = kQTileBytes * ND + 2 * kStages * kKVBytes + 1024 /*barriers*/ + 1024 /*align*/;
};

struct AttnParams {
  CUtensorMap tmQ, tmK, tmV;
  __nv_bfloat16* o;
  float* lse;      // optional [B, heads, Sq]: log2-domain log-sum-exp of scale*log2(e)*S (for attention_bwd.cu)
  int ldo;
  int Sq, Skv;
  int d;           // head dim (multiple of 8)
  int n_kv_tiles;
  float scale_log2;  // scale * log2(e)
};

template <int ND>
__global__ void __launch_bounds__(kAttnThreads, 1) attention_kernel(const __grid_constant__ AttnParams p) {
  constexpr int kKV = AttnCfg<ND>::kKV;
  constexpr int kStages = AttnCfg<ND>::kStages;
  constexpr uint32_t kKVBytes = AttnCfg<ND>::kKVBytes;
  constexpr uint32_t kKVChunk = kKV * 128;  // 64 head columns of a K / V tile
  pdl_trigger();
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_addr = smem_u32(smem_raw);
  const uint32_t base = (raw_addr + 1023u) & ~1023u;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int qt = blockIdx.x, head = blockIdx.y, b = blockIdx.z;

  const uint32_t sQ = base;
  const uint32_t sK = base + kQTileBytes * ND;
  const uint32_t sV = sK + kStages * kKVBytes;
  const uint32_t bars = sV + kStages * kKVBytes;
  const uint32_t bar_q = bars;
  const uint32_t bar_kfull = bars + 8;                   // kStages
  const uint32_t bar_kempty = bar_kfull + 8 * kStages;   // kStages
  const uint32_t bar_vfull = bar_kempty + 8 * kStages;
  const uint32_t bar_vempty = bar_vfull + 8 * kStages;

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&p.tmQ);
    tma_prefetch_desc(&p.tmK);
    tma_prefetch_desc(&p.tmV);
  }
  if (warp == 1 && lane == 0) {
    mbar_init(bar_q, 1);
    for (int i = 0; i < kStages; ++i) {
      mbar_init(bar_kfull + 8 * i, 1);
      mbar_init(bar_kempty + 8 * i, 2);  // one arrival per consumer warpgroup
      mbar_init(bar_vfull + 8 * i, 1);
      mbar_init(bar_vempty + 8 * i, 2);
    }
    fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();
  const int n = p.n_kv_tiles;

  if (warp == 8) {
    // ------------------------------------------------------------------ TMA producer, converged warp
    if (elect_one()) {
      mbar_expect_tx(bar_q, kQTileBytes * ND);
#pragma unroll
      for (int i = 0; i < ND; ++i) tma_load_4d(sQ + i * kQTileBytes, &p.tmQ, bar_q, i * 64, head, qt * 128, b);
    }
    __syncwarp();
    for (int j = 0; j < n; ++j) {
      const int s = j % kStages;
      const uint32_t ph = (j / kStages) & 1;
      mbar_wait(bar_kempty + 8 * s, ph ^ 1u);
      if (elect_one()) {
        mbar_expect_tx(bar_kfull + 8 * s, kKVBytes);
#pragma unroll
        for (int i = 0; i < ND; ++i)
          tma_load_4d(sK + s * kKVBytes + i * kKVChunk, &p.tmK, bar_kfull + 8 * s, i * 64, head, j * kKV, b);
      }
      __syncwarp();
      mbar_wait(bar_vempty + 8 * s, ph ^ 1u);
      if (elect_one()) {
        mbar_expect_tx(bar_vfull + 8 * s, kKVBytes);
#pragma unroll
        for (int i = 0; i < ND; ++i)
          tma_load_4d(sV + s * kKVBytes + i * kKVChunk, &p.tmV, bar_vfull + 8 * s, i * 64, head, j * kKV, b);
      }
      __syncwarp();
    }
    return;
  }

  // ------------------------------------------------------------------ consumer warpgroups
  const int wg = warp >> 2;
  const bool signal = (threadIdx.x & 127) == 0;
  const int dsteps = (p.d + 15) >> 4;  // 16-wide k-steps of the Q K^T contraction that hold data
  const uint32_t sQw = sQ + static_cast<uint32_t>(wg) * 64u * 128u;  // this warpgroup's 64 query rows
  float o[ND * 32];
#pragma unroll
  for (int i = 0; i < ND * 32; ++i) o[i] = 0.f;
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};  // rows lane / 4 and lane / 4 + 8 of the warp's 16
  mbar_wait(bar_q, 0);
  for (int j = 0; j < n; ++j) {
    const int s = j % kStages;
    const uint32_t ph = (j / kStages) & 1;
    float sc[kKV / 2];
    mbar_wait(bar_kfull + 8 * s, ph);
    wgmma_fence();
    for (int k = 0; k < dsteps; ++k) {
      const uint32_t qoff = static_cast<uint32_t>(k >> 2) * kQTileBytes + static_cast<uint32_t>(k & 3) * 32;
      const uint32_t koff = static_cast<uint32_t>(k >> 2) * kKVChunk + static_cast<uint32_t>(k & 3) * 32;
      if constexpr (kKV == 128)
        wgmma_ss<128>(sc, gmma_desc_sw128(sQw + qoff), gmma_desc_sw128(sK + s * kKVBytes + koff), k != 0);
      else
        wgmma_ss<64>(sc, gmma_desc_sw128(sQw + qoff), gmma_desc_sw128(sK + s * kKVBytes + koff), k != 0);
    }
    wgmma_commit();
    wgmma_wait<0>();
#pragma unroll
    for (int i = 0; i < kKV / 2; ++i) reg_fence(sc[i]);
    if (signal) mbar_arrive(bar_kempty + 8 * s);

    // ---- online softmax in the log2 domain: x = s * scale * log2(e)
    const int left = p.Skv - j * kKV;  // valid keys in this tile
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int i = 0; i < kKV / 2; ++i) {
      const int col = 8 * (i >> 2) + 2 * (lane & 3) + (i & 1);
      sc[i] = col < left ? sc[i] * p.scale_log2 : -INFINITY;
      mx[(i >> 1) & 1] = fmaxf(mx[(i >> 1) & 1], sc[i]);
    }
    float alpha[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
      const float mn = fmaxf(m[r], mx[r]);  // finite: every tile holds at least one valid key
      alpha[r] = fast_exp2(m[r] - mn);
      m[r] = mn;
      l[r] *= alpha[r];
    }
    uint32_t pa[kKV / 16][4];  // P as bf16 A fragments, one group of four registers per 16 keys
#pragma unroll
    for (int i = 0; i < kKV / 2; i += 2) {
      const int r = (i >> 1) & 1;
      const float p0 = fast_exp2(sc[i] - m[r]), p1 = fast_exp2(sc[i + 1] - m[r]);
      l[r] += p0 + p1;
      pa[i >> 3][(i >> 1) & 3] = pack_bf16x2(p0, p1);
    }
#pragma unroll
    for (int i = 0; i < ND * 32; ++i) o[i] *= alpha[(i >> 1) & 1];

    mbar_wait(bar_vfull + 8 * s, ph);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < kKV / 16; ++kk) {
#pragma unroll
      for (int c = 0; c < ND; ++c)
        wgmma_rs_n64_tb(o + 32 * c, pa[kk], gmma_desc_sw128(sV + s * kKVBytes + c * kKVChunk + kk * 2048), 1u);
    }
    wgmma_commit();
    wgmma_wait<0>();
#pragma unroll
    for (int i = 0; i < ND * 32; ++i) reg_fence(o[i]);
    if (signal) mbar_arrive(bar_vempty + 8 * s);
  }

  // ---- normalise and write O (first d columns of each padded head), log-sum-exp for the backward pass
  const int wl = warp & 3;
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    l[r] += __shfl_xor_sync(0xffffffffu, l[r], 1);
    l[r] += __shfl_xor_sync(0xffffffffu, l[r], 2);
  }
  const int heads = gridDim.y;
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int q = qt * 128 + wg * 64 + wl * 16 + (lane >> 2) + 8 * r;
    if (q >= p.Sq) continue;
    const float inv = 1.f / l[r];
    __nv_bfloat16* orow = p.o + (static_cast<size_t>(b) * p.Sq + q) * p.ldo + static_cast<size_t>(head) * p.d;
#pragma unroll
    for (int c = 0; c < ND; ++c) {
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const int col = c * 64 + 8 * e + 2 * (lane & 3);
        if (col < p.d) {
          const int i = 32 * c + 4 * e + 2 * r;
          *reinterpret_cast<uint32_t*>(orow + col) = pack_bf16x2(o[i] * inv, o[i + 1] * inv);
        }
      }
    }
    if (p.lse != nullptr && (lane & 3) == 0)
      p.lse[(static_cast<size_t>(b) * heads + head) * p.Sq + q] = m[r] + __log2f(l[r]);
  }
}

template <int ND>
static int launch_attention(cudaStream_t stream, const AttnParams& p, dim3 grid, bool pdl) {
  static bool attr_set = false;
  if (!attr_set) {
    SB200_CUDA_CHECK(
        cudaFuncSetAttribute(attention_kernel<ND>, cudaFuncAttributeMaxDynamicSharedMemorySize, AttnCfg<ND>::kSmem));
    attr_set = true;
  }
  SB200_CUDA_CHECK(launch_pdl(attention_kernel<ND>, grid, dim3(kAttnThreads), AttnCfg<ND>::kSmem, stream, pdl, p));
  SB200_CUDA_CHECK(cudaGetLastError());
  return 0;
}

}  // namespace sb200

using namespace sb200;

extern "C" int sb200_attention(void* handle, void* stream, const void* q, int ldq, const void* k, int ldk,
                               const void* v, int ldv, void* o, int ldo, int B, int heads, int Sq, int Skv,
                               int head_dim, float scale, float* lse) {
  Ctx* ctx = as_ctx(handle);
  SB200_REQUIRE(ctx, "attention: NULL handle");
  SB200_REQUIRE(B > 0 && heads > 0 && Sq > 0 && Skv > 0, "attention: bad dims");
  SB200_REQUIRE(head_dim >= 8 && head_dim <= 192 && head_dim % 8 == 0,
                "attention: head dim %d unsupported (multiple of 8, <= 192)", head_dim);
  SB200_REQUIRE(ldq % 8 == 0 && ldk % 8 == 0 && ldv % 8 == 0 && ldo % 8 == 0,
                "attention: leading dims must be multiples of 8");
  SB200_REQUIRE(ldq >= heads * head_dim && ldk >= heads * head_dim && ldv >= heads * head_dim &&
                    ldo >= heads * head_dim,
                "attention: heads=%d x head_dim=%d exceeds a row", heads, head_dim);
  const int kv = head_dim <= 64 ? AttnCfg<1>::kKV : AttnCfg<2>::kKV;
  AttnParams p;
  memset(&p, 0, sizeof(p));
  int st;
  const uint64_t hs = static_cast<uint64_t>(head_dim) * 2;  // byte stride between heads
  {
    const uint32_t box[4] = {64, 1, 128, 1};
    const uint64_t dims[4] = {static_cast<uint64_t>(head_dim), static_cast<uint64_t>(heads),
                              static_cast<uint64_t>(Sq), static_cast<uint64_t>(B)};
    const uint64_t strides[3] = {hs, static_cast<uint64_t>(ldq) * 2, static_cast<uint64_t>(ldq) * 2 * Sq};
    if ((st = make_tmap_bf16(ctx, &p.tmQ, q, 4, dims, strides, box))) return st;
  }
  {
    const uint32_t box[4] = {64, 1, static_cast<uint32_t>(kv), 1};
    const uint64_t dims[4] = {static_cast<uint64_t>(head_dim), static_cast<uint64_t>(heads),
                              static_cast<uint64_t>(Skv), static_cast<uint64_t>(B)};
    const uint64_t sk[3] = {hs, static_cast<uint64_t>(ldk) * 2, static_cast<uint64_t>(ldk) * 2 * Skv};
    const uint64_t sv[3] = {hs, static_cast<uint64_t>(ldv) * 2, static_cast<uint64_t>(ldv) * 2 * Skv};
    if ((st = make_tmap_bf16(ctx, &p.tmK, k, 4, dims, sk, box))) return st;
    if ((st = make_tmap_bf16(ctx, &p.tmV, v, 4, dims, sv, box))) return st;
  }
  p.o = static_cast<__nv_bfloat16*>(o);
  p.lse = lse;
  p.ldo = ldo;
  p.Sq = Sq;
  p.Skv = Skv;
  p.d = head_dim;
  p.n_kv_tiles = (Skv + kv - 1) / kv;
  p.scale_log2 = scale * 1.4426950408889634f;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  dim3 grid((Sq + 127) / 128, heads, B);
  const bool pdl = pdl_small_grid(ctx, static_cast<long long>(grid.x) * grid.y * grid.z);
  if (head_dim <= 64) return launch_attention<1>(s, p, grid, pdl);
  if (head_dim <= 128) return launch_attention<2>(s, p, grid, pdl);
  return launch_attention<3>(s, p, grid, pdl);
}
