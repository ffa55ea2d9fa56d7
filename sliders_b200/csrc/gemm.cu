// LoRA-fused bf16 GEMM / implicit-GEMM 3x3 convolution for sm_90a.
//
//   out[M, N] = epilogue( A[M, K] . W[N, K]^T  [+ scale * (A . down^T) . up^T] )
//
// One CTA per 128 x BN output tile (BN = 64 or 128: a template parameter, picked on the host), 288 threads:
//   warp 8      TMA producer — streams A / W / LoRA-down tiles (64-deep k-blocks) through an mbarrier ring of smem stages
//   warps 0..7  two consumer warpgroups, rows 0..63 and 64..127 of the tile: wgmma m64 x BN x 16 from shared memory
//               into registers; then the epilogue
// The LoRA down-projection rides in the same k-block loop: its rows are staged right behind the W rows of the stage and
// one more wgmma (N = rt) per k-step accumulates t = A . down^T.
// Epilogue: both warpgroups park their accumulators in shared memory as an fp32 [128 x (BN + rt)] tile (over the stage
// ring, which is free once the main loop has ended).  Each thread then owns one row: rank-r LoRA up-projection,
// LayerNorm fold, bias / time-embedding row bias / GEGLU / residual; residual tiles come in by cp.async and results
// leave through a swizzled smem staging tile so that global accesses are coalesced.
// CTA pairs (kCtas = 2): a cluster of two CTAs on consecutive 128-row tiles of the same N tile.  Each CTA loads half
// of the W (and LoRA-down) rows of a stage and multicasts them to both, which halves the weight traffic from L2.
//
// A-operand addressing modes:
//   plain   2-D [M, K], optionally split along K over two sources (skip-connection concat, conv_shortcut)
//   conv    4-D NHWC box per filter tap (implicit GEMM): a tile is a bb x bh x bw patch of output pixels (<= 128), the
//           box start is shifted by (kh-1, kw-1) and TMA's out-of-bounds zero fill provides the padding AND the ragged
//           edges of patches that overhang the image, so any H x W works; two sources along C give the concat
//   conv/2  stride-2 conv: four parity-plane descriptors (even/odd rows x even/odd columns)
//
// Replaces (reference): every nn.Linear / nn.Conv2d leaf that diffusers' UNet2DConditionModel executes under
// trainscripts/textsliders/train_util.py:242-247 together with the LoRA hook trainscripts/textsliders/lora.py:108-112.
#include <stdlib.h>

#include "common.h"
#include "ptx.cuh"

namespace sb200 {

constexpr int kBM = 128;  // rows per CTA
constexpr int kBK = 64;
constexpr int kEpiWarps = 8;                   // the two consumer warpgroups
constexpr int kEpiPerQuarter = kEpiWarps / 4;  // epilogue warps sharing one 32-row quarter; slabs are dealt round-robin
constexpr int kProducerWarp = kEpiWarps;
constexpr int kGemmThreads = 32 * (kEpiWarps + 1);
constexpr int kMaxStages = 8;
constexpr int kSmemBudget = 227 * 1024;
constexpr int kBarRegion = 1024;
constexpr int kLoraCols = 32;         // accumulator columns kept for t = A . down^T (rt <= 32)
constexpr int kSlab = 32;             // output columns staged per epilogue-warp iteration
constexpr int kEpiBufBytes = 32 * 64; // [32 rows x 32 cols] bf16
constexpr int kEpiBytes = kEpiWarps * kEpiBufBytes;  // + kEpiWarps x [32 cols][r] fp32 of lora_up rows with LoRA
constexpr int kConsumerBar = 5;       // named barrier of the 256 consumer threads (1..4: row-statistics reduction)

// fp32 accumulator tile in shared memory: row stride BN + kLoraCols + 4 floats, so that the 32 rows a warp reads at
// one column fall into distinct 16-byte bank groups
__host__ __device__ constexpr int acc_stride(int bn) { return bn + kLoraCols + 4; }
__host__ __device__ constexpr int acc_tile_bytes(int bn) { return kBM * acc_stride(bn) * 4; }

struct GemmParams {
  CUtensorMap tmA[4];
  CUtensorMap tmB;
  CUtensorMap tmL;
  int M, N, K;
  int bn;           // output columns of W per tile (the kernel's BN)
  int ncols_out;    // output columns per tile (bn, or bn/2 with GEGLU)
  int Nout;         // output columns overall (N, or N/2 with GEGLU)
  int num_m_tiles, num_n_tiles;  // tiles of (128 * kCtas) x bn
  int num_sub;      // 128-row sub-tiles along M (a CTA of a pair whose sub-tile index is >= num_sub computes zeros)
  int kblocks;      // K / 64 (conv: 9 * cb_total)
  int stages;
  int stage_bytes;  // bytes of one smem stage
  int ring_bytes;   // stage ring, also holds the fp32 accumulator tile after the main loop
  int a_tx;         // bytes one A load deposits (box bytes; < 16 KB for conv patches smaller than 128 pixels)
  int b_rows;       // W rows one CTA loads per k-block (bn / kCtas)
  int l_rows;       // LoRA-down rows one CTA loads per k-block (rt / kCtas)
  int up_buf_bytes; // per-warp staging of one slab's lora_up rows: 32 * r * 4 (0 without LoRA)
  int n_fast;       // tile order: 1 = consecutive CTAs share the A row-tile and walk the N tiles (A is read from
                    // DRAM once, W stays L2-resident); 0 = M fastest (A re-streamed once per N tile when it exceeds L2)
  int a_mode;       // 0 plain, 1 conv3x3 stride 1, 2 conv3x3 stride 2
  int kb_split;     // k-blocks (per tap) that come from source 0
  int cb_total;     // k-blocks per tap
  int B, H, W;      // conv OUTPUT dims
  int bw, bh, bb;   // conv patch of one sub-tile (bw * bh * bb <= 128 pixels)
  int tiles_w, tiles_h;
  int flags;
  const __nv_bfloat16* bias;
  const __nv_bfloat16* rowbias;
  int rows_per_batch;
  const __nv_bfloat16* resid;
  int ldr;
  __nv_bfloat16* out;
  int ldo;
  const float* lora_up;  // [N, r] fp32
  int lora_r, lora_rt, lora_group_n;
  float lora_scale;
  const float* lora_scale_dev;
  // LayerNorm folded into this projection (struct sb200_lnfold) / row statistics left for the next one
  const float* ln_stats;
  int ln_parts;
  float ln_inv_c, ln_eps;
  const float* ln_c;
  const float* ln_d;
  const float* ln_cl;
  const float* ln_dl;
  float* rs_out;
  int rs_parts;
  // split-K (sb200_gemm_splitk_f32): grid y = split index; split s runs k-blocks [s * sk_kb, (s + 1) * sk_kb) and stores
  // its raw fp32 tile to sk_ws[s][M][N] instead of running the epilogue
  float* sk_ws;
  int sk_kb, sk_splits;
};

__device__ __forceinline__ void add_bf16x16(float* f, const __nv_bfloat16* src) {
  const uint4* bp = reinterpret_cast<const uint4*>(src);
  const uint4 b0 = __ldg(bp), b1 = __ldg(bp + 1);
  const uint32_t bw[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    f[2 * i] += bf16_lo(bw[i]);
    f[2 * i + 1] += bf16_hi(bw[i]);
  }
}

template <int R>
__device__ __forceinline__ void lora_apply(float* f, const float* t, uint32_t up_rows) {
  // up_rows: shared-memory address of 16 consecutive rows of [N, R] fp32 (same address for the whole warp: broadcast)
#pragma unroll
  for (int i = 0; i < 16; ++i) {
    const uint4 a = ld_shared_v4(up_rows + i * R * 4);
    f[i] += t[0] * __uint_as_float(a.x) + t[1] * __uint_as_float(a.y) + t[2] * __uint_as_float(a.z) +
            t[3] * __uint_as_float(a.w);
    if constexpr (R == 8) {
      const uint4 b = ld_shared_v4(up_rows + i * R * 4 + 16);
      f[i] += t[4] * __uint_as_float(b.x) + t[5] * __uint_as_float(b.y) + t[6] * __uint_as_float(b.z) +
              t[7] * __uint_as_float(b.w);
    }
  }
}

// n consecutive fp32 of the shared accumulator tile (n multiple of 4)
template <int n>
__device__ __forceinline__ void ld_acc(uint32_t addr, uint32_t* v) {
#pragma unroll
  for (int i = 0; i < n / 4; ++i) {
    const uint4 a = ld_shared_v4(addr + 16 * i);
    v[4 * i] = a.x;
    v[4 * i + 1] = a.y;
    v[4 * i + 2] = a.z;
    v[4 * i + 3] = a.w;
  }
}

// accumulator fragment of one warpgroup (m64 x N, see wgmma.cuh) -> rows row0.. of the shared fp32 tile
template <int N>
__device__ __forceinline__ void store_frag(const float* d, uint32_t tile, int row0, int col0, int stride) {
  const int lane = threadIdx.x & 31, w = (threadIdx.x >> 5) & 3;
  const int r = row0 + w * 16 + (lane >> 2);
#pragma unroll
  for (int i = 0; i < N / 2; i += 2) {
    const int row = r + 8 * ((i >> 1) & 1);
    const int col = col0 + 8 * (i >> 2) + 2 * (lane & 3);
    asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(tile + (row * stride + col) * 4), "f"(d[i]), "f"(d[i + 1])
                 : "memory");
  }
}

template <int BN>
__device__ __forceinline__ void wgmma_main(float* d, uint64_t a, uint64_t b) {
  if constexpr (BN == 64)
    wgmma_ss_n64(d, a, b, 1u);
  else
    wgmma_ss_n128(d, a, b, 1u);
}

// First output pixel (b0, h0, w0) of conv sub-tile `st` (w fastest, then h, then batch).
__device__ __forceinline__ void conv_origin(const GemmParams& p, int st, int& b0, int& h0, int& w0) {
  const int tw = st % p.tiles_w;
  const int r = st / p.tiles_w;
  const int th = r % p.tiles_h;
  w0 = tw * p.bw;
  h0 = th * p.bh;
  b0 = (r / p.tiles_h) * p.bb;
}

template <int BN, int kCtas, int RT>
__global__ void __launch_bounds__(kGemmThreads, 1) gemm_kernel(const __grid_constant__ GemmParams p) {
  pdl_trigger();
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_addr = smem_u32(smem_raw);
  const uint32_t base = (raw_addr + 1023u) & ~1023u;  // SWIZZLE_128B tiles need 1024 B alignment

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const uint32_t cta_rank = kCtas == 2 ? cluster_ctarank() : 0u;
  const int S = p.stages;
  const uint32_t bar_full = base;            // S barriers
  const uint32_t bar_empty = base + 8u * S;  // S barriers
  const uint32_t tiles = base + kBarRegion;
  const bool has_lora = (p.flags & SB200_EPI_LORA) != 0;
  const bool geglu = (p.flags & SB200_EPI_GEGLU) != 0;
  constexpr int rt = RT;  // LoRA-down rows of a stage (0 without LoRA)

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&p.tmA[0]);
    tma_prefetch_desc(&p.tmB);
    if (has_lora) tma_prefetch_desc(&p.tmL);
  }
  if (warp == 1 && lane == 0) {
    for (int i = 0; i < S; ++i) {
      mbar_init(bar_full + 8u * i, 1);
      mbar_init(bar_empty + 8u * i, 2 * kCtas);  // one arrival per consumer warpgroup of every CTA the stage feeds
    }
    fence_barrier_init();
  }
  if constexpr (kCtas == 2) {
    cluster_sync_all();
  } else {
    __syncthreads();
  }
  pdl_wait();  // everything above overlapped the previous kernel's tail; global memory is touched only below

  const int t = blockIdx.x / kCtas;  // this CTA's (pair's) output tile
  const int num_n_tiles = p.num_n_tiles, num_m_tiles = p.num_m_tiles;
  const int mt = p.n_fast ? t / num_n_tiles : t % num_m_tiles;
  const int nt = p.n_fast ? t % num_n_tiles : t / num_m_tiles;
  const int st = mt * kCtas + static_cast<int>(cta_rank);  // this CTA's 128-row sub-tile
  const int kb_lo = p.sk_ws ? static_cast<int>(blockIdx.y) * p.sk_kb : 0;
  const int kb_hi = p.sk_ws ? min(p.kblocks, kb_lo + p.sk_kb) : p.kblocks;
  const uint32_t stage_bytes = static_cast<uint32_t>(p.stage_bytes);
  const uint32_t a_bytes = kBM * 128;
  const uint32_t b_bytes = static_cast<uint32_t>(BN) * 128;  // W rows of a stage (both halves for a pair)

  if (warp == kProducerWarp) {
    // ------------------------------------------------------------------ TMA producer, converged warp
    const int a_mode = p.a_mode, kb_split = p.kb_split, cb_total = p.cb_total;
    const uint32_t tx = static_cast<uint32_t>(p.a_tx) + b_bytes + static_cast<uint32_t>(rt) * 128u;
    const int m0 = st * kBM;
    int b0 = 0, h0 = 0, w0 = 0;
    if (a_mode != 0) {
      if (st < p.num_sub)
        conv_origin(p, st, b0, h0, w0);
      else
        b0 = p.B;  // phantom sub-tile of an odd pair: every box is out of bounds -> zero fill
    }
    // W rows this CTA loads (a pair: half each, multicast to both)
    int brow;
    if (geglu) {
      const int half = BN >> 1;
      brow = (kCtas == 2 && cta_rank == 1) ? (p.N >> 1) + nt * half : nt * half;
    } else {
      brow = nt * BN + static_cast<int>(cta_rank) * p.b_rows;
    }
    int stage = 0;
    uint32_t phase = 0;
    for (int kb = kb_lo; kb < kb_hi; ++kb) {
      const uint32_t full_bar = bar_full + 8u * stage, empty_bar = bar_empty + 8u * stage;
      mbar_wait(empty_bar, phase ^ 1u);
      if (elect_one()) {
        mbar_expect_tx(full_bar, tx);
        const uint32_t sA = tiles + static_cast<uint32_t>(stage) * stage_bytes;
        const uint32_t sB = sA + a_bytes;
        if (a_mode == 0) {
          const int src = kb < kb_split ? 0 : 1;
          tma_load_2d(sA, &p.tmA[src], full_bar, (src ? kb - kb_split : kb) * kBK, m0);
        } else {
          const int tap = kb / cb_total;  // filter tap and channel block of this k-block
          const int cb = kb - tap * cb_total;
          const int kh = tap / 3;
          const int kw = tap - kh * 3;
          if (a_mode == 1) {
            const int src = cb < kb_split ? 0 : 1;
            tma_load_4d(sA, &p.tmA[src], full_bar, (src ? cb - kb_split : cb) * kBK, w0 + kw - 1, h0 + kh - 1, b0);
          } else {
            // input row 2*ho + kh - 1: kh=0 -> odd plane, row ho-1; kh=1 -> even plane, row ho; kh=2 -> odd plane, row ho
            const int ph = (kh == 1) ? 0 : 1;
            const int pwl = (kw == 1) ? 0 : 1;
            tma_load_4d(sA, &p.tmA[ph * 2 + pwl], full_bar, cb * kBK, w0 + ((kw == 0) ? -1 : 0),
                        h0 + ((kh == 0) ? -1 : 0), b0);
          }
        }
        if constexpr (kCtas == 2) {
          const uint32_t boff = cta_rank * static_cast<uint32_t>(p.b_rows) * 128u;
          tma_load_2d_mc(sB + boff, &p.tmB, full_bar, kb * kBK, brow, 3);
          if (has_lora)
            tma_load_2d_mc(sB + b_bytes + cta_rank * static_cast<uint32_t>(p.l_rows) * 128u, &p.tmL, full_bar, kb * kBK,
                           static_cast<int>(cta_rank) * p.l_rows, 3);
        } else {
          tma_load_2d(sB, &p.tmB, full_bar, kb * kBK, brow);
          if (geglu) tma_load_2d(sB + (b_bytes >> 1), &p.tmB, full_bar, kb * kBK, (p.N >> 1) + nt * (BN >> 1));
          if (has_lora) tma_load_2d(sB + b_bytes, &p.tmL, full_bar, kb * kBK, 0);
        }
      }
      __syncwarp();
      if (++stage == S) {
        stage = 0;
        phase ^= 1u;
      }
    }
  } else {
    // ------------------------------------------------------------------ consumers: main loop
    const int wg = warp >> 2;
    float acc[BN / 2];
    float accl[16];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
#pragma unroll
    for (int i = 0; i < 16; ++i) accl[i] = 0.f;
    const bool signal = (threadIdx.x & 127) == 0;
    const uint32_t peer_empty = kCtas == 2 ? mapa_u32(bar_empty, cta_rank ^ 1u) : 0u;
    int stage = 0, prev = 0;
    uint32_t phase = 0;
    for (int kb = kb_lo; kb < kb_hi; ++kb) {
      mbar_wait(bar_full + 8u * stage, phase);
      const uint32_t sA = tiles + static_cast<uint32_t>(stage) * stage_bytes + static_cast<uint32_t>(wg) * 64u * 128u;
      const uint32_t sB = tiles + static_cast<uint32_t>(stage) * stage_bytes + a_bytes;
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < kBK / 16; ++k) {
        const uint64_t adesc = gmma_desc_sw128(sA + 32u * k);
        wgmma_main<BN>(acc, adesc, gmma_desc_sw128(sB + 32u * k));
        if constexpr (rt == 16)
          wgmma_ss_n16(accl, adesc, gmma_desc_sw128(sB + b_bytes + 32u * k), 1u);
        else if constexpr (rt == 32)
          wgmma_ss_n32(accl, adesc, gmma_desc_sw128(sB + b_bytes + 32u * k), 1u);
      }
      wgmma_commit();
      wgmma_wait<1>();  // the previous k-block's products have read their stage: hand it back to the producer(s)
      if (kb > kb_lo && signal) {
        mbar_arrive(bar_empty + 8u * prev);
        if (kCtas == 2) mbar_arrive_cluster(peer_empty + 8u * prev);
      }
      prev = stage;
      if (++stage == S) {
        stage = 0;
        phase ^= 1u;
      }
    }
    wgmma_wait<0>();
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) reg_fence(acc[i]);
#pragma unroll
    for (int i = 0; i < 16; ++i) reg_fence(accl[i]);

    // ------------------------------------------------------------------ epilogue
    const uint32_t accs = tiles;  // fp32 accumulator tile, over the stage ring
    constexpr int kStride = acc_stride(BN);
    asm volatile("bar.sync %0, %1;" ::"n"(kConsumerBar), "n"(32 * kEpiWarps) : "memory");  // both warpgroups done reading
    store_frag<BN>(acc, accs, wg * 64, 0, kStride);
    if constexpr (rt == 16)
      store_frag<16>(accl, accs, wg * 64, BN, kStride);
    else if constexpr (rt == 32)
      store_frag<32>(accl, accs, wg * 64, BN, kStride);
    asm volatile("bar.sync %0, %1;" ::"n"(kConsumerBar), "n"(32 * kEpiWarps) : "memory");
    if (p.sk_ws != nullptr) {
      // split-K: this split's raw fp32 tile, row-coalesced; sb200_gemm_splitk_f32's reduction sums the splits
      float* dst = p.sk_ws + static_cast<size_t>(blockIdx.y) * p.M * p.N;
      constexpr int kQuads = BN / 4;
      for (int idx = threadIdx.x; idx < kBM * kQuads; idx += 32 * kEpiWarps) {
        const int row = idx / kQuads, c = (idx - row * kQuads) * 4;
        const int m = st * kBM + row, n = nt * BN + c;
        if (m < p.M && n < p.N)
          *reinterpret_cast<uint4*>(dst + static_cast<size_t>(m) * p.N + n) =
              ld_shared_v4(accs + static_cast<uint32_t>(row * kStride + c) * 4u);
      }
      return;
    }

    const int q = warp & 3;      // 32-row quarter of the tile this warp writes
    const int hsel = warp >> 2;  // which of the kEpiPerQuarter warps of this quarter (slab index mod that)
    const float lscale =
        has_lora ? (p.lora_scale_dev ? p.lora_scale * __ldg(p.lora_scale_dev) : p.lora_scale) : 0.f;
    const bool has_resid = (p.flags & SB200_EPI_RESID) != 0;
    // per-warp staging buffer ([32 rows x 32 cols] bf16, 64 B rows, 16-byte chunks XOR-swizzled by (row >> 1) & 3):
    // residual tiles arrive here by cp.async with coalesced global reads, results leave from here with coalesced global
    // writes; in between every thread touches only its own row.
    const uint32_t ebuf = tiles + static_cast<uint32_t>(p.ring_bytes) +
                          static_cast<uint32_t>(warp) * (kEpiBufBytes + p.up_buf_bytes);
    const uint32_t ubuf = ebuf + kEpiBufBytes;  // p.up_buf_bytes of lora_up rows
    const uint32_t arow = accs + static_cast<uint32_t>((q * 32 + lane) * kStride) * 4u;
    // output row of this thread's accumulator row (q * 32 + lane), or -1 (padding row of the tile)
    int my_row = -1, my_batch = 0;
    {
      const int r = q * 32 + lane;
      if (p.a_mode == 0) {
        const int m = st * kBM + r;
        if (m < p.M) my_row = m;
        my_batch = (p.flags & SB200_EPI_ROWBIAS) ? m / p.rows_per_batch : 0;
      } else if (st < p.num_sub) {
        int b0, h0, w0;
        conv_origin(p, st, b0, h0, w0);
        const int iw = r % p.bw;
        const int t2 = r / p.bw;
        const int ih = t2 % p.bh;
        const int ib = t2 / p.bh;
        const int b = b0 + ib, h = h0 + ih, w = w0 + iw;
        if (ib < p.bb && b < p.B && h < p.H && w < p.W) my_row = (b * p.H + h) * p.W + w;
        my_batch = b;
      }
    }
    const bool row_ok = my_row >= 0;
    // LayerNorm fold: (mean, rstd) of this thread's row of x from the producer's partial sums, part-major
    // [parts][M][2]: the 32 rows of a warp read consecutive addresses
    float ln_rstd = 1.f, ln_rm = 0.f;
    if (p.ln_stats != nullptr && row_ok) {
      const float2* ln_sp = reinterpret_cast<const float2*>(p.ln_stats) + my_row;
      float s1 = 0.f, s2 = 0.f;
      for (int i = 0; i < p.ln_parts; ++i) {
        const float2 v2 = __ldg(ln_sp + static_cast<size_t>(i) * p.M);
        s1 += v2.x;
        s2 += v2.y;
      }
      const float mean = s1 * p.ln_inv_c;
      ln_rstd = rsqrtf(fmaxf(s2 * p.ln_inv_c - mean * mean, 0.f) + p.ln_eps);
      ln_rm = ln_rstd * mean;
    }
    float rs1 = 0.f, rs2 = 0.f;  // row statistics of what this warp writes in this tile
    const int n_base = nt * p.ncols_out;
    const int ncols_valid = min(p.ncols_out, p.Nout - n_base);
    const int nslabs = (ncols_valid + kSlab - 1) / kSlab;
    const int my_slabs = (nslabs - hsel + kEpiPerQuarter - 1) / kEpiPerQuarter;  // slabs hsel, hsel + kEpiPerQuarter, ...
    auto prefetch_resid = [&](int col0, int sw) {
      const int cpr = sw >> 3;  // 16-byte chunks per row
      if (has_resid) {
        for (int idx = lane; idx < 32 * cpr; idx += 32) {
          const int row = cpr == 4 ? idx >> 2 : idx / cpr;
          const int ch = idx - row * cpr;
          const int mr = __shfl_sync(0xffffffffu, my_row, row);
          if (mr >= 0)
            cp_async_16(ebuf + row * 64 + ((ch ^ ((row >> 1) & 3)) << 4),
                        p.resid + static_cast<size_t>(mr) * p.ldr + n_base + col0 + ch * 8);
        }
      }
      if (has_lora && lane < sw) {
        // this slab's lora_up rows ([r] fp32 per output column) travel with the residual: the rank-r update then
        // reads them from shared memory instead of taking an L2 round trip per 16 columns inside the loop
        const uint32_t ub = ubuf + lane * p.lora_r * 4;
        const float* src = p.lora_up + static_cast<size_t>(n_base + col0 + lane) * p.lora_r;
        cp_async_16(ub, src);
        if (p.lora_r == 8) cp_async_16(ub + 16, src + 4);
      }
      cp_async_commit();
    };
    const bool staged = has_resid || has_lora;
    if (staged && my_slabs > 0) prefetch_resid(hsel * kSlab, min(kSlab, ncols_valid - hsel * kSlab));
    const __nv_bfloat16* rb =
        (p.flags & SB200_EPI_ROWBIAS) ? p.rowbias + static_cast<size_t>(row_ok ? my_batch : 0) * p.Nout : nullptr;
    float tl[8];
    int group_lo = 0, group_hi = 0;  // output-column range of the adaptor whose t = A.down^T is held in tl
    const uint32_t swz = static_cast<uint32_t>((lane >> 1) & 3);
    for (int k = 0; k < my_slabs; ++k) {
      const int col0 = (hsel + kEpiPerQuarter * k) * kSlab;
      const int sw = min(kSlab, ncols_valid - col0);
      const bool more = k + 1 < my_slabs;
      for (int sub = 0; sub * 16 < sw; ++sub) {
        const int c = col0 + sub * 16;
        const int n = n_base + c;
        uint32_t v[16];
        uint32_t g[16];
        ld_acc<16>(arow + c * 4, v);
        if (geglu) ld_acc<16>(arow + ((BN >> 1) + c) * 4, g);
        if (has_lora && (n < group_lo || n >= group_hi)) {
          const int grp = n / p.lora_group_n;
          group_lo = grp * p.lora_group_n;
          group_hi = group_lo + p.lora_group_n;
          uint32_t tv[8];
          const int j = grp * p.lora_r;
          ld_acc<8>(arow + (BN + j) * 4, tv);
          if (p.ln_cl != nullptr) {
#pragma unroll
            for (int jj = 0; jj < 8; ++jj)
              tl[jj] = (jj < p.lora_r) ? fmaf(__uint_as_float(tv[jj]), ln_rstd,
                                              fmaf(-ln_rm, __ldg(p.ln_cl + j + jj), __ldg(p.ln_dl + j + jj))) * lscale
                                       : 0.f;
          } else {
#pragma unroll
            for (int jj = 0; jj < 8; ++jj) tl[jj] = __uint_as_float(tv[jj]) * lscale;
          }
        }
        float f[16];
#pragma unroll
        for (int j = 0; j < 16; ++j) f[j] = __uint_as_float(v[j]);
        if (p.ln_stats != nullptr) {
          // LN(x) . W^T + b = rstd * acc - rstd * mean * c[n] + d[n]
#pragma unroll
          for (int j4 = 0; j4 < 4; ++j4) {
            const float4 cc = __ldg(reinterpret_cast<const float4*>(p.ln_c + n) + j4);
            const float4 dd = __ldg(reinterpret_cast<const float4*>(p.ln_d + n) + j4);
            f[4 * j4 + 0] = fmaf(f[4 * j4 + 0], ln_rstd, fmaf(-ln_rm, cc.x, dd.x));
            f[4 * j4 + 1] = fmaf(f[4 * j4 + 1], ln_rstd, fmaf(-ln_rm, cc.y, dd.y));
            f[4 * j4 + 2] = fmaf(f[4 * j4 + 2], ln_rstd, fmaf(-ln_rm, cc.z, dd.z));
            f[4 * j4 + 3] = fmaf(f[4 * j4 + 3], ln_rstd, fmaf(-ln_rm, cc.w, dd.w));
          }
        }
        if (staged && sub == 0) {  // this slab's residual / lora_up rows have landed
          cp_async_wait<0>();
          __syncwarp();
        }
        if (has_lora) {
          const uint32_t up = ubuf + sub * 16 * p.lora_r * 4;
          if (p.lora_r == 4)
            lora_apply<4>(f, tl, up);
          else
            lora_apply<8>(f, tl, up);
        }
        if (p.flags & SB200_EPI_BIAS) add_bf16x16(f, p.bias + n);
        if (rb) add_bf16x16(f, rb + n);
        if (geglu) {
          float gb[16];
#pragma unroll
          for (int j = 0; j < 16; ++j) gb[j] = __uint_as_float(g[j]);
          if (p.ln_stats != nullptr) {
#pragma unroll
            for (int j = 0; j < 16; ++j)
              gb[j] = fmaf(gb[j], ln_rstd, fmaf(-ln_rm, __ldg(p.ln_c + p.Nout + n + j), __ldg(p.ln_d + p.Nout + n + j)));
          }
          if (p.flags & SB200_EPI_BIAS) add_bf16x16(gb, p.bias + p.Nout + n);
#pragma unroll
          for (int j = 0; j < 16; ++j) f[j] *= gelu_erf_f(gb[j]);
        }
        const uint32_t a0 = ebuf + lane * 64 + (((2 * sub) ^ swz) << 4);
        const uint32_t a1 = ebuf + lane * 64 + (((2 * sub + 1) ^ swz) << 4);
        uint32_t o[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = pack_bf16x2(f[2 * j], f[2 * j + 1]);
        if (has_resid && row_ok) {
          // the residual is added to the ROUNDED projection, in bf16, like the reference's separate elementwise
          // `hidden_states = attn_output + hidden_states` on two bf16 tensors
          const uint4 r0 = ld_shared_v4(a0), r1 = ld_shared_v4(a1);
          const uint32_t rw[8] = {r0.x, r0.y, r0.z, r0.w, r1.x, r1.y, r1.z, r1.w};
#pragma unroll
          for (int j = 0; j < 8; ++j) o[j] = add_bf16x2(o[j], rw[j]);
        }
        if (p.rs_out != nullptr) {
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const float lo = bf16_lo(o[j]), hi = bf16_hi(o[j]);
            rs1 += lo + hi;
            rs2 = fmaf(lo, lo, fmaf(hi, hi, rs2));
          }
        }
        st_shared_v4(a0, make_uint4(o[0], o[1], o[2], o[3]));
        st_shared_v4(a1, make_uint4(o[4], o[5], o[6], o[7]));
      }
      __syncwarp();
      {  // coalesced copy-out of the staged [32 x sw] tile
        const int cpr = sw >> 3;
        for (int idx = lane; idx < 32 * cpr; idx += 32) {
          const int row = cpr == 4 ? idx >> 2 : idx / cpr;
          const int ch = idx - row * cpr;
          const int mr = __shfl_sync(0xffffffffu, my_row, row);
          const uint4 val = ld_shared_v4(ebuf + row * 64 + ((ch ^ ((row >> 1) & 3)) << 4));
          if (mr >= 0)
            *reinterpret_cast<uint4*>(p.out + static_cast<size_t>(mr) * p.ldo + n_base + col0 + ch * 8) = val;
        }
      }
      __syncwarp();
      if (staged && more) {  // the next slab's residual / lora_up rows replace what was just copied out
        const int ncol0 = col0 + kEpiPerQuarter * kSlab;
        prefetch_resid(ncol0, min(kSlab, ncols_valid - ncol0));
      }
    }
    if (p.rs_out != nullptr) {
      // The kEpiPerQuarter warps of a quarter hold partial sums of the SAME 32 rows (different slabs): combine them
      // through the quarter's first warp's staging buffer (free after its last copy-out), so that a row has one slot
      // per N tile.  Named barrier 1 + q, 32 * kEpiPerQuarter threads.
      const uint32_t red = tiles + static_cast<uint32_t>(p.ring_bytes) +
                           static_cast<uint32_t>(q) * (kEpiBufBytes + p.up_buf_bytes);
      asm volatile("bar.sync %0, %1;" ::"r"(1 + q), "r"(32 * kEpiPerQuarter) : "memory");  // first warp done with its buffer
      if (hsel != 0)
        asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(red + ((hsel - 1) * 32 + lane) * 8), "f"(rs1), "f"(rs2)
                     : "memory");
      asm volatile("bar.sync %0, %1;" ::"r"(1 + q), "r"(32 * kEpiPerQuarter) : "memory");
      if (hsel == 0) {
#pragma unroll
        for (int w = 0; w < kEpiPerQuarter - 1; ++w) {
          float a, b;
          asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(a), "=f"(b) : "r"(red + (w * 32 + lane) * 8));
          rs1 += a;
          rs2 += b;
        }
        if (row_ok) reinterpret_cast<float2*>(p.rs_out)[static_cast<size_t>(nt) * p.M + my_row] = make_float2(rs1, rs2);
      }
    }
  }

  if constexpr (kCtas == 2) {
    __syncwarp();
    cluster_sync_all();  // the peer's barriers / smem must outlive every multicast and remote arrive aimed at them
  }
}

// -------------------------------------------------------------------------------------------------
// host side
// -------------------------------------------------------------------------------------------------
struct TileChoice {
  int ctas;
  int bn;
};

static int env_int(const char* name, int dflt) {
  const char* e = getenv(name);
  return (e && e[0]) ? atoi(e) : dflt;
}

// SB200_PAIR=2 runs every GEMM / conv as CTA pairs; otherwise pairs run only where the caller forces them (bit 12 of
// bn).  Pairs are opt-in: they halve the weight traffic from L2, but they never need fewer waves than single CTAs (a
// pair is two CTAs on two row tiles), and these tiles are not L2-bound: on an H100 at 400 W, 8192 x 1280 x 1280 takes
// 69 us single / 105 us paired, 8192 x 10240 x 1280 576 / 1056 us, 2048 x 640 x 640 20.5 / 21.9 us.
static bool pairs_always() {
  static const bool v = env_int("SB200_PAIR", 0) == 2;
  return v;
}

// Tile widths the kernel is instantiated for (a 256-wide accumulator does not fit the registers of 288 threads).
static bool bn_supported(int bn) { return bn == 64 || bn == 128; }

// Tile width from a cost model in SM cycles.  A 128 x bn tile's 64-deep k-block takes 4 bn cycles of tensor work (m64
// wgmmas of two warpgroups at 4096 bf16 FLOP / clk / SM) plus the LoRA columns; a tile pays ~2000 cycles of prologue
// and pipeline fill and an epilogue of ~14 cycles per output column (more with a residual / LoRA / GEGLU).  One CTA per
// SM: work is dealt in waves of num_sms tiles.
static TileChoice pick_tile(int ncols, int num_sms, int kblocks, int lora_rt, int force_ctas, int sub_tiles, int flags) {
  double best = -1;
  TileChoice bc{1, 64};
  const int ctas = force_ctas ? force_ctas : (pairs_always() ? 2 : 1);
  const bool geglu = (flags & SB200_EPI_GEGLU) != 0;
  const double epi_per_col = 14.0 + ((flags & SB200_EPI_RESID) ? 5.0 : 0.0) + (lora_rt ? 6.0 : 0.0) + (geglu ? 10.0 : 0.0);
  for (int bn = 64; bn <= 128; bn *= 2) {
    const long tiles = static_cast<long>(sub_tiles) * ((ncols + bn - 1) / bn);
    const long waves = (tiles + num_sms - 1) / num_sms;
    const double perkb = 4.0 * (bn + lora_rt) + 64.0;
    const double cost = waves * (kblocks * perkb + 2000.0 + epi_per_col * (geglu ? bn / 2 : bn));
    if (best < 0 || cost < best - 1e-9 || (cost < best + 1e-9 && bn > bc.bn)) {
      best = cost;
      bc = TileChoice{ctas, bn};
    }
  }
  return bc;
}

static bool n_fast_default() {
  static const bool v = [] {
    const char* e = getenv("SB200_TILE_ORDER");  // "m" restores the M-fastest order
    return !(e && e[0] == 'm');
  }();
  return v;
}

template <int BN, int kCtas, int RT>
static int launch_gemm_bn(Ctx* ctx, cudaStream_t stream, const GemmParams& p, int smem) {
  static bool attr_set = false;  // one flag per instantiation
  if (!attr_set) {
    SB200_CUDA_CHECK(
        cudaFuncSetAttribute(gemm_kernel<BN, kCtas, RT>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBudget));
    attr_set = true;
  }
  const int total = p.num_m_tiles * p.num_n_tiles;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(total * kCtas, p.sk_ws ? p.sk_splits : 1);
  cfg.blockDim = dim3(kGemmThreads);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[2];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = (pdl_mode() == 2 || (pdl_mode() == 1 && pdl_hint())) ? 1 : 0;
  attr[1].id = cudaLaunchAttributeClusterDimension;
  attr[1].val.clusterDim.x = kCtas;
  attr[1].val.clusterDim.y = 1;
  attr[1].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = kCtas == 2 ? 2 : 1;
  SB200_CUDA_CHECK(cudaLaunchKernelEx(&cfg, gemm_kernel<BN, kCtas, RT>, p));
  (void)ctx;
  return 0;
}

static int launch_gemm(Ctx* ctx, cudaStream_t stream, GemmParams& p, int ctas) {
  // Tile order: N fastest reads each A row-tile from DRAM once and re-reads W once per row-tile, which is free while W
  // stays in L2.  When W is the big operand and does not fit (the batched cross-attention K/V projection: 616 x 2048
  // activations against 629 MB of weights) the M-fastest order streams W once instead.
  {
    const double w_bytes = 2.0 * p.N * p.K;
    const double a_bytes_total = 2.0 * p.M * (p.a_mode == 0 ? p.K : p.K / 9);
    p.n_fast = (n_fast_default() && !(w_bytes > a_bytes_total && w_bytes > 32e6)) ? 1 : 0;
  }
  const bool has_lora = p.flags & SB200_EPI_LORA;
  p.b_rows = p.bn / ctas;
  p.l_rows = has_lora ? p.lora_rt / ctas : 0;
  p.stage_bytes = kBM * 128 + p.bn * 128 + (has_lora ? p.lora_rt * 128 : 0);
  p.up_buf_bytes = has_lora ? kSlab * p.lora_r * 4 : 0;
  const int epi_bytes = kEpiBytes + kEpiWarps * p.up_buf_bytes;
  int stages = (kSmemBudget - kBarRegion - 1024 - epi_bytes) / p.stage_bytes;
  if (stages > kMaxStages) stages = kMaxStages;
  if (stages < 2) return set_error(SB200_ERR_INVALID, "gemm: tile does not fit shared memory");
  p.stages = stages;
  p.ring_bytes = stages * p.stage_bytes;
  if (p.ring_bytes < acc_tile_bytes(p.bn)) p.ring_bytes = acc_tile_bytes(p.bn);
  const int smem = kBarRegion + 1024 + p.ring_bytes + epi_bytes;
  if (smem > kSmemBudget) return set_error(SB200_ERR_INVALID, "gemm: tile does not fit shared memory");
  pdl_hint() = p.num_m_tiles * p.num_n_tiles * ctas * (p.sk_ws ? p.sk_splits : 1) <= 2 * ctx->num_sms;
  const int rt = has_lora ? p.lora_rt : 0;
  const int variant = (ctas == 2 ? 6 : 0) + (p.bn == 128 ? 3 : 0) + (rt == 16 ? 1 : (rt == 32 ? 2 : 0));
  cudaStream_t s = stream;
  int st;
  switch (variant) {
    case 0: st = launch_gemm_bn<64, 1, 0>(ctx, s, p, smem); break;
    case 1: st = launch_gemm_bn<64, 1, 16>(ctx, s, p, smem); break;
    case 2: st = launch_gemm_bn<64, 1, 32>(ctx, s, p, smem); break;
    case 3: st = launch_gemm_bn<128, 1, 0>(ctx, s, p, smem); break;
    case 4: st = launch_gemm_bn<128, 1, 16>(ctx, s, p, smem); break;
    case 5: st = launch_gemm_bn<128, 1, 32>(ctx, s, p, smem); break;
    case 6: st = launch_gemm_bn<64, 2, 0>(ctx, s, p, smem); break;
    case 7: st = launch_gemm_bn<64, 2, 16>(ctx, s, p, smem); break;
    case 8: st = launch_gemm_bn<64, 2, 32>(ctx, s, p, smem); break;
    case 9: st = launch_gemm_bn<128, 2, 0>(ctx, s, p, smem); break;
    case 10: st = launch_gemm_bn<128, 2, 16>(ctx, s, p, smem); break;
    default: st = launch_gemm_bn<128, 2, 32>(ctx, s, p, smem); break;
  }
  if (st) return st;
  SB200_CUDA_CHECK(cudaGetLastError());
  return 0;
}

static int check_lora(const sb200_lora* l, int N) {
  SB200_REQUIRE(l->down && l->up, "lora: NULL weights");
  SB200_REQUIRE(l->r == 4 || l->r == 8, "lora: rank %d unsupported by the fused epilogue (4 or 8)", l->r);
  SB200_REQUIRE(l->rt == 16 || l->rt == 32, "lora: rt must be 16 or 32");
  SB200_REQUIRE(l->group_n > 0 && l->group_n % 16 == 0, "lora: group_n must be a multiple of 16");
  const int groups = (N + l->group_n - 1) / l->group_n;
  SB200_REQUIRE(groups * l->r <= l->rt, "lora: %d groups of rank %d exceed rt=%d", groups, l->r, l->rt);
  return 0;
}

// bn encodes an explicit choice when > 0: low 12 bits = tile width, bit 12 set = force CTA pairs, bit 13 set = force
// single CTAs (used by the tests to cover both).
static void decode_bn(int bn_arg, int* bn, int* force_ctas) {
  *force_ctas = (bn_arg > 0 && (bn_arg & 0x1000)) ? 2 : ((bn_arg > 0 && (bn_arg & 0x2000)) ? 1 : 0);
  *bn = bn_arg > 0 ? (bn_arg & 0xFFF) : 0;
}

static void fill_lora(GemmParams& p, const sb200_lora* lora) {
  p.lora_up = static_cast<const float*>(lora->up);
  p.lora_r = lora->r;
  p.lora_rt = lora->rt;
  p.lora_group_n = lora->group_n;
  p.lora_scale = lora->scale;
  p.lora_scale_dev = lora->scale_dev;
}

// out[m, n] = sum over s (in order) of ws[s][m][n]; four columns per thread
__global__ void splitk_reduce_kernel(const float* __restrict__ ws, int splits, int M, int N, float* __restrict__ out,
                                     int ldo) {
  pdl_trigger();
  pdl_wait();
  const size_t part = static_cast<size_t>(M) * N;
  const size_t idx = (static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x) * 4;
  if (idx >= part) return;
  float4 a = __ldg(reinterpret_cast<const float4*>(ws + idx));
  for (int s = 1; s < splits; ++s) {
    const float4 v = __ldg(reinterpret_cast<const float4*>(ws + s * part + idx));
    a.x += v.x;
    a.y += v.y;
    a.z += v.z;
    a.w += v.w;
  }
  const size_t m = idx / N, n = idx % N;
  *reinterpret_cast<float4*>(out + m * ldo + n) = a;
}

}  // namespace sb200

using namespace sb200;

extern "C" int sb200_gemm_splitk_f32(void* handle, void* stream, const void* x, int ldx, const void* w, int ldw,
                                     float* out, int ldo, int M, int N, int K, float* ws, size_t ws_floats) {
  Ctx* ctx = as_ctx(handle);
  SB200_REQUIRE(ctx && x && w && out && ws, "gemm_splitk_f32: NULL argument");
  SB200_REQUIRE(M > 0 && N > 0 && K > 0 && N % 16 == 0, "gemm_splitk_f32: bad dims M=%d N=%d K=%d", M, N, K);
  SB200_REQUIRE(K % 8 == 0 && ldx % 8 == 0 && ldw % 8 == 0 && ldo % 4 == 0,
                "gemm_splitk_f32: K and the bf16 leading dims must be multiples of 8, ldo of 4");
  const size_t need = SB200_GEMM_SPLITK_WS_FLOATS(M, N, K);
  SB200_REQUIRE(ws_floats >= need, "gemm_splitk_f32: scratch of %zu floats, %zu needed", ws_floats, need);
  GemmParams p;
  memset(&p, 0, sizeof(p));
  p.M = M;
  p.N = N;
  p.K = K;
  p.Nout = N;
  p.kblocks = (K + kBK - 1) / kBK;
  p.kb_split = p.kblocks;
  p.cb_total = p.kblocks;
  p.a_tx = kBM * 128;
  p.num_sub = (M + kBM - 1) / kBM;
  p.bn = N % 128 == 0 ? 128 : 64;
  p.ncols_out = p.bn;
  p.num_m_tiles = p.num_sub;
  p.num_n_tiles = (N + p.bn - 1) / p.bn;
  p.sk_ws = ws;
  p.sk_kb = SB200_GEMM_SPLITK_KB(M, N, K);
  p.sk_splits = SB200_GEMM_SPLITK_SPLITS(M, N, K);
  int st;
  {
    const uint64_t dims[2] = {static_cast<uint64_t>(K), static_cast<uint64_t>(M)};
    const uint64_t strides[1] = {static_cast<uint64_t>(ldx) * 2};
    const uint32_t box[2] = {kBK, kBM};
    if ((st = make_tmap_bf16(ctx, &p.tmA[0], x, 2, dims, strides, box))) return st;
  }
  {
    const uint64_t dims[2] = {static_cast<uint64_t>(K), static_cast<uint64_t>(N)};
    const uint64_t strides[1] = {static_cast<uint64_t>(ldw) * 2};
    const uint32_t box[2] = {kBK, static_cast<uint32_t>(p.bn)};
    if ((st = make_tmap_bf16(ctx, &p.tmB, w, 2, dims, strides, box))) return st;
  }
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if ((st = launch_gemm(ctx, s, p, 1))) return st;
  const size_t quads = static_cast<size_t>(M) * N / 4;
  SB200_CUDA_CHECK(launch_pdl(splitk_reduce_kernel, dim3(static_cast<unsigned>((quads + 255) / 256)), dim3(256), 0, s,
                              static_cast<const float*>(ws), p.sk_splits, M, N, out, ldo));
  SB200_CUDA_CHECK(cudaGetLastError());
  return 0;
}

extern "C" int sb200_gemm(void* handle, void* stream, const void* x0, int ldx0, const void* x1, int ldx1,
                          int K0, const void* w, int ldw, void* out, int ldo, int M, int N, int K,
                          int flags, const void* bias, const void* rowbias, int rows_per_batch,
                          const void* resid, int ldr, const sb200_lora* lora, int bn_arg) {
  return sb200_gemm_ln(handle, stream, x0, ldx0, x1, ldx1, K0, w, ldw, out, ldo, M, N, K, flags, bias, rowbias,
                       rows_per_batch, resid, ldr, lora, bn_arg, nullptr, nullptr, 0, nullptr);
}

extern "C" int sb200_gemm_ln(void* handle, void* stream, const void* x0, int ldx0, const void* x1, int ldx1,
                             int K0, const void* w, int ldw, void* out, int ldo, int M, int N, int K,
                             int flags, const void* bias, const void* rowbias, int rows_per_batch,
                             const void* resid, int ldr, const sb200_lora* lora, int bn_arg,
                             const sb200_lnfold* ln, float* rowstats, int rowstats_cap, int* rowstats_parts) {
  Ctx* ctx = as_ctx(handle);
  SB200_REQUIRE(ctx, "gemm: NULL handle");
  SB200_REQUIRE(M > 0 && N > 0 && K > 0, "gemm: bad dims M=%d N=%d K=%d", M, N, K);
  SB200_REQUIRE(N % 16 == 0, "gemm: N=%d must be a multiple of 16", N);
  SB200_REQUIRE(K % 8 == 0 && ldx0 % 8 == 0 && ldw % 8 == 0 && ldo % 8 == 0,
                "gemm: K and leading dims must be multiples of 8 elements");
  const bool split = x1 != nullptr;
  if (!split) K0 = K;
  SB200_REQUIRE(!split || (K0 % 64 == 0 && K0 > 0 && K0 < K && ldx1 % 8 == 0),
                "gemm: split K0=%d must be a multiple of 64 inside (0, K)", K0);
  const bool geglu = flags & SB200_EPI_GEGLU;
  const bool has_lora = flags & SB200_EPI_LORA;
  SB200_REQUIRE(!(geglu && has_lora), "gemm: GEGLU and LORA cannot be combined");
  SB200_REQUIRE(!geglu || N % 32 == 0, "gemm: GEGLU needs N %% 32 == 0");
  SB200_REQUIRE(!(flags & SB200_EPI_BIAS) || bias, "gemm: BIAS without bias");
  SB200_REQUIRE(!(flags & SB200_EPI_ROWBIAS) || (rowbias && rows_per_batch > 0), "gemm: ROWBIAS args");
  SB200_REQUIRE(!(flags & SB200_EPI_RESID) || (resid && ldr % 8 == 0), "gemm: RESID args");
  SB200_REQUIRE(!has_lora || lora, "gemm: LORA without sb200_lora");

  GemmParams p;
  memset(&p, 0, sizeof(p));
  p.M = M;
  p.N = N;
  p.K = K;
  p.flags = flags;
  p.Nout = geglu ? N / 2 : N;
  p.kblocks = (K + kBK - 1) / kBK;
  p.a_mode = 0;
  p.kb_split = split ? K0 / kBK : p.kblocks;
  p.cb_total = p.kblocks;
  p.a_tx = kBM * 128;
  p.num_sub = (M + kBM - 1) / kBM;
  if (has_lora) {
    int st = check_lora(lora, N);
    if (st) return st;
    fill_lora(p, lora);
  }
  int bn, force_ctas;
  decode_bn(bn_arg, &bn, &force_ctas);
  TileChoice tc = pick_tile(N, ctx->num_sms, p.kblocks, has_lora ? lora->rt : 0, force_ctas, p.num_sub, flags);
  if (bn > 0) tc.bn = bn;
  if (force_ctas) tc.ctas = force_ctas;
  SB200_REQUIRE(bn_supported(tc.bn), "gemm: bn=%d invalid (64 or 128)", tc.bn);
  p.bn = tc.bn;
  p.ncols_out = geglu ? tc.bn / 2 : tc.bn;
  p.num_m_tiles = (p.num_sub + tc.ctas - 1) / tc.ctas;
  p.num_n_tiles = (p.Nout + p.ncols_out - 1) / p.ncols_out;
  p.bias = static_cast<const __nv_bfloat16*>(bias);
  p.rowbias = static_cast<const __nv_bfloat16*>(rowbias);
  p.rows_per_batch = rows_per_batch;
  p.resid = static_cast<const __nv_bfloat16*>(resid);
  p.ldr = ldr;
  p.out = static_cast<__nv_bfloat16*>(out);
  p.ldo = ldo;
  if (ln != nullptr) {
    SB200_REQUIRE(ln->stats && ln->parts > 0 && ln->C == K && ln->c && ln->d, "gemm: lnfold arguments (C must equal K)");
    SB200_REQUIRE(!(flags & SB200_EPI_BIAS), "gemm: with lnfold the bias lives in d[]");
    SB200_REQUIRE(!has_lora || (ln->c_lora && ln->d_lora), "gemm: lnfold with LoRA needs c_lora / d_lora");
    p.ln_stats = ln->stats;
    p.ln_parts = ln->parts;
    p.ln_inv_c = 1.0f / static_cast<float>(ln->C);
    p.ln_eps = ln->eps;
    p.ln_c = ln->c;
    p.ln_d = ln->d;
    p.ln_cl = has_lora ? ln->c_lora : nullptr;
    p.ln_dl = has_lora ? ln->d_lora : nullptr;
  }
  if (rowstats != nullptr) {
    SB200_REQUIRE(!geglu, "gemm: rowstats of a GEGLU output are not supported");
    p.rs_parts = p.num_n_tiles;
    SB200_REQUIRE(p.rs_parts <= rowstats_cap, "gemm: rowstats needs %d slots per row, capacity %d", p.rs_parts, rowstats_cap);
    p.rs_out = rowstats;
    if (rowstats_parts) *rowstats_parts = p.rs_parts;
  }

  int st;
  {
    const uint64_t dims[2] = {static_cast<uint64_t>(K0), static_cast<uint64_t>(M)};
    const uint64_t strides[1] = {static_cast<uint64_t>(ldx0) * 2};
    const uint32_t box[2] = {kBK, kBM};
    if ((st = make_tmap_bf16(ctx, &p.tmA[0], x0, 2, dims, strides, box))) return st;
  }
  if (split) {
    const uint64_t dims[2] = {static_cast<uint64_t>(K - K0), static_cast<uint64_t>(M)};
    const uint64_t strides[1] = {static_cast<uint64_t>(ldx1) * 2};
    const uint32_t box[2] = {kBK, kBM};
    if ((st = make_tmap_bf16(ctx, &p.tmA[1], x1, 2, dims, strides, box))) return st;
  }
  {
    const uint64_t dims[2] = {static_cast<uint64_t>(K), static_cast<uint64_t>(N)};
    const uint64_t strides[1] = {static_cast<uint64_t>(ldw) * 2};
    const int brows = (geglu || tc.ctas == 2) ? tc.bn / 2 : tc.bn;
    const uint32_t box[2] = {kBK, static_cast<uint32_t>(brows)};
    if ((st = make_tmap_bf16(ctx, &p.tmB, w, 2, dims, strides, box))) return st;
  }
  if (has_lora) {
    const uint64_t dims[2] = {static_cast<uint64_t>(K), static_cast<uint64_t>(lora->rt)};
    const uint64_t strides[1] = {static_cast<uint64_t>(K) * 2};
    const uint32_t box[2] = {kBK, static_cast<uint32_t>(lora->rt / tc.ctas)};
    if ((st = make_tmap_bf16(ctx, &p.tmL, lora->down, 2, dims, strides, box))) return st;
  }
  return launch_gemm(ctx, static_cast<cudaStream_t>(stream), p, tc.ctas);
}

// Patch of output pixels one 128-row sub-tile covers: bw x bh x bb with bw * bh * bb <= 128, chosen to minimise the
// number of sub-tiles (ties: the widest patch row, i.e. the longest contiguous TMA runs).  bb > 1 only for whole images.
static void pick_patch(int B, int H, int W, int* bw_o, int* bh_o, int* bb_o) {
  long best = -1;
  int sel_w = 1, sel_h = 1, sel_b = 1;
  for (int bw = (W < 128 ? W : 128); bw >= 1; --bw) {
    int bh = 128 / bw;
    if (bh > H) bh = H;
    int bb = 1;
    if (bw == W && bh == H) {
      bb = 128 / (bw * bh);
      if (bb > B) bb = B;
      if (bb < 1) bb = 1;
    }
    const long tiles = static_cast<long>((W + bw - 1) / bw) * ((H + bh - 1) / bh) * ((B + bb - 1) / bb);
    if (best < 0 || tiles < best) {
      best = tiles;
      sel_w = bw, sel_h = bh, sel_b = bb;
    }
  }
  *bw_o = sel_w, *bh_o = sel_h, *bb_o = sel_b;
}

extern "C" int sb200_conv3x3(void* handle, void* stream, const void* x0, int ldx0, const void* x1,
                             int ldx1, int C0, int C1, const void* w, void* out, int ldo, int B, int Hin,
                             int Win, int Cout, int stride, int flags, const void* bias,
                             const void* rowbias, const void* resid, int ldr, const sb200_lora* lora,
                             int bn_arg) {
  Ctx* ctx = as_ctx(handle);
  SB200_REQUIRE(ctx, "conv3x3: NULL handle");
  SB200_REQUIRE(stride == 1 || stride == 2, "conv3x3: stride %d", stride);
  SB200_REQUIRE(B > 0 && Hin > 0 && Win > 0 && Hin % stride == 0 && Win % stride == 0,
                "conv3x3: %dx%d input with stride %d (stride 2 needs even dims)", Hin, Win, stride);
  if (!x1) C1 = 0;
  SB200_REQUIRE(C0 > 0 && C0 % 64 == 0 && C1 % 64 == 0, "conv3x3: C0=%d C1=%d must be multiples of 64", C0,
                C1);
  SB200_REQUIRE(Cout % 16 == 0, "conv3x3: Cout=%d must be a multiple of 16", Cout);
  SB200_REQUIRE(!(flags & SB200_EPI_GEGLU), "conv3x3: GEGLU unsupported");
  SB200_REQUIRE(stride == 1 || C1 == 0, "conv3x3: stride 2 takes a single source");
  SB200_REQUIRE(ldx0 % 8 == 0 && ldo % 8 == 0 && (C1 == 0 || ldx1 % 8 == 0), "conv3x3: leading dims");
  const bool has_lora = flags & SB200_EPI_LORA;
  SB200_REQUIRE(!has_lora || lora, "conv3x3: LORA without sb200_lora");
  SB200_REQUIRE(!(flags & SB200_EPI_BIAS) || bias, "conv3x3: BIAS without bias");
  SB200_REQUIRE(!(flags & SB200_EPI_ROWBIAS) || rowbias, "conv3x3: ROWBIAS without rowbias");
  SB200_REQUIRE(!(flags & SB200_EPI_RESID) || (resid && ldr % 8 == 0), "conv3x3: RESID args");
  const int H = Hin / stride, W = Win / stride;
  int bw, bh, bb;
  pick_patch(B, H, W, &bw, &bh, &bb);
  const int Cin = C0 + C1;
  const int M = B * H * W;

  GemmParams p;
  memset(&p, 0, sizeof(p));
  p.M = M;
  p.N = Cout;
  p.K = 9 * Cin;
  p.flags = flags;
  p.Nout = Cout;
  p.cb_total = Cin / kBK;
  p.kblocks = 9 * p.cb_total;
  p.a_mode = stride == 1 ? 1 : 2;
  p.kb_split = C0 / kBK;
  p.B = B;
  p.H = H;
  p.W = W;
  p.bw = bw;
  p.bh = bh;
  p.bb = bb;
  p.tiles_w = (W + bw - 1) / bw;
  p.tiles_h = (H + bh - 1) / bh;
  p.num_sub = p.tiles_w * p.tiles_h * ((B + bb - 1) / bb);
  p.a_tx = bw * bh * bb * 128;
  if (has_lora) {
    int st = check_lora(lora, Cout);
    if (st) return st;
    fill_lora(p, lora);
  }
  int bn, force_ctas;
  decode_bn(bn_arg, &bn, &force_ctas);
  TileChoice tc = pick_tile(Cout, ctx->num_sms, p.kblocks, has_lora ? lora->rt : 0, force_ctas, p.num_sub, flags);
  if (bn > 0) tc.bn = bn;
  if (force_ctas) tc.ctas = force_ctas;
  SB200_REQUIRE(bn_supported(tc.bn), "conv3x3: bn=%d invalid (64 or 128)", tc.bn);
  p.bn = tc.bn;
  p.ncols_out = tc.bn;
  p.num_m_tiles = (p.num_sub + tc.ctas - 1) / tc.ctas;
  p.num_n_tiles = (Cout + tc.bn - 1) / tc.bn;
  p.bias = static_cast<const __nv_bfloat16*>(bias);
  p.rowbias = static_cast<const __nv_bfloat16*>(rowbias);
  p.rows_per_batch = H * W;
  p.resid = static_cast<const __nv_bfloat16*>(resid);
  p.ldr = ldr;
  p.out = static_cast<__nv_bfloat16*>(out);
  p.ldo = ldo;

  int st;
  const uint32_t box[4] = {kBK, static_cast<uint32_t>(bw), static_cast<uint32_t>(bh),
                           static_cast<uint32_t>(bb)};
  if (stride == 1) {
    const void* src[2] = {x0, x1};
    const int ld[2] = {ldx0, ldx1};
    const int cs[2] = {C0, C1};
    for (int s = 0; s < (C1 ? 2 : 1); ++s) {
      const uint64_t dims[4] = {static_cast<uint64_t>(cs[s]), static_cast<uint64_t>(Win),
                                static_cast<uint64_t>(Hin), static_cast<uint64_t>(B)};
      const uint64_t pix = static_cast<uint64_t>(ld[s]) * 2;
      const uint64_t strides[3] = {pix, pix * Win, pix * Win * Hin};
      if ((st = make_tmap_bf16(ctx, &p.tmA[s], src[s], 4, dims, strides, box))) return st;
    }
  } else {
    // parity planes: plane (ph, pw) holds input pixels (2*hh + ph, 2*ww + pw)
    for (int ph = 0; ph < 2; ++ph)
      for (int pw = 0; pw < 2; ++pw) {
        const uint64_t pix = static_cast<uint64_t>(ldx0) * 2;
        const uint8_t* basep = static_cast<const uint8_t*>(x0) + (static_cast<uint64_t>(ph) * Win + pw) * pix;
        const uint64_t dims[4] = {static_cast<uint64_t>(C0), static_cast<uint64_t>(W),
                                  static_cast<uint64_t>(H), static_cast<uint64_t>(B)};
        const uint64_t strides[3] = {pix * 2, pix * Win * 2, pix * Win * Hin};
        if ((st = make_tmap_bf16(ctx, &p.tmA[ph * 2 + pw], basep, 4, dims, strides, box))) return st;
      }
  }
  {
    const uint64_t dims[2] = {static_cast<uint64_t>(p.K), static_cast<uint64_t>(Cout)};
    const uint64_t strides[1] = {static_cast<uint64_t>(p.K) * 2};
    const uint32_t wbox[2] = {kBK, static_cast<uint32_t>(tc.bn / tc.ctas)};
    if ((st = make_tmap_bf16(ctx, &p.tmB, w, 2, dims, strides, wbox))) return st;
  }
  if (has_lora) {
    const uint64_t dims[2] = {static_cast<uint64_t>(p.K), static_cast<uint64_t>(lora->rt)};
    const uint64_t strides[1] = {static_cast<uint64_t>(p.K) * 2};
    const uint32_t lbox[2] = {kBK, static_cast<uint32_t>(lora->rt / tc.ctas)};
    if ((st = make_tmap_bf16(ctx, &p.tmL, lora->down, 2, dims, strides, lbox))) return st;
  }
  return launch_gemm(ctx, static_cast<cudaStream_t>(stream), p, tc.ctas);
}
