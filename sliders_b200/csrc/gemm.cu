// LoRA-fused bf16 GEMM / implicit-GEMM 3x3 convolution for sm_90a.
//
//   out[M, N] = epilogue( A[M, K] . W[N, K]^T  [+ scale * (A . down^T) . up^T] )
//
// One CTA per 128 x BN output tile (BN = 64 or 128: a template parameter, picked on the host), 288 threads:
//   warp 8      TMA producer — streams A / W / LoRA-down tiles (64-deep k-blocks) through an mbarrier ring of smem stages
//   warps 0..7  two consumer warpgroups, rows 0..63 and 64..127 of the tile: wgmma m64 x BN x 16 from shared memory
//               into registers; then the epilogue
// The LoRA down-projection rides in the same k-block loop: its rows are staged right behind the W rows of the stage and
// the same wgmma (N = BN + rt) accumulates t = A . down^T in the tail of the fragment (lora_folded).
// Epilogue: both warpgroups park their accumulators in shared memory as an fp32 [128 x (BN + rt)] tile (over the stage
// ring, which is free once the main loop has ended).  Each thread then owns one row: rank-r LoRA up-projection,
// bias / time-embedding row bias / GEGLU / residual; residual tiles come in by cp.async and results leave through a
// swizzled smem staging tile (also in the ring, behind the accumulator tile) so that global accesses are coalesced.
// Residency: two CTAs per SM wherever 96 registers per thread hold the accumulators without spills (BN = 64 with up
// to 32 LoRA rows, or no LoRA), so one CTA's prologue and epilogue run while the other's wgmmas keep the tensor cores
// busy; BN = 128 with LoRA needs ~120 registers and runs one CTA per SM, as do the 64 LoRA rows (rank-16 q|k|v) at
// either width.  Each CTA's ring is sized from its share of the SM's shared memory.
// CTA pairs (kCtas = 2): a cluster of two CTAs on consecutive 128-row tiles of the same N tile.  Each CTA loads half
// of the W (and LoRA-down) rows of a stage and multicasts them to both, which halves the weight traffic from L2.
// The ring protocol is written once for this kernel and gemm_wide_kernel below: gemm_prologue (descriptor prefetch,
// barrier init, sync), produce (the producer's k-block loop, CTA-pair multicast included) and consume (the consumers'
// k-block loop and stage handback); tile_coords maps a tile index to its (mt, nt) and tile_out_row a tile row to its
// output row.  On the host the three entry points fill in their A operand and hand over to plan_and_launch (epilogue
// and LoRA checks, tile choice, W / LoRA-down maps), launch_gemm (ring sizing) and launch_checked (the launch).
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

#include <algorithm>

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
constexpr int kBarRegion = 1024;
constexpr int kAlignSlack = 1024;     // the dynamic smem base is rounded up to 1024 B
constexpr int kSlab = 32;             // output columns staged per epilogue-warp iteration
constexpr int kEpiBufBytes = 32 * 64; // [32 rows x 32 cols] bf16
constexpr int kEpiBytes = kEpiWarps * kEpiBufBytes;  // + kEpiWarps x [32 cols][r] fp32 of lora_up rows with LoRA
constexpr int kConsumerBar = 1;       // named barrier of the 256 consumer threads

// CTAs per SM an instantiation is compiled for (its launch bounds): under two, ptxas caps a thread at 96 registers,
// which holds BN = 64 with up to 32 LoRA rows and BN = 128 without them; BN = 128 with LoRA, and 64 LoRA rows at any
// width, would spill and serialise their wgmmas (DESIGN §4a)
__host__ __device__ constexpr int gemm_slots(int bn, int rt) { return rt == 64 ? 1 : (bn == 64 || rt == 0) ? 2 : 1; }

// fp32 accumulator tile in shared memory: row stride BN + rt + 4 floats (an odd multiple of 16 bytes), so that the 32
// rows a warp reads at one column fall into distinct 16-byte bank groups.  The 4 padding floats also absorb the
// 8-float read of the last rank-4 adaptor's t columns.
__host__ __device__ constexpr int acc_stride(int bn, int rt) { return bn + rt + 4; }
__host__ __device__ constexpr int acc_tile_bytes(int bn, int rt) { return kBM * acc_stride(bn, rt) * 4; }

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
  int ring_bytes;   // stage ring; after the main loop: fp32 accumulator tile, then the epilogue staging buffers
  int a_tx;         // bytes one A load deposits (box bytes; < 16 KB for conv patches smaller than 128 pixels)
  int b_rows;       // W rows one CTA loads per k-block (bn / kCtas)
  int l_rows;       // LoRA-down rows one CTA loads per k-block (rt / kCtas)
  int up_buf_bytes; // per-warp staging of one slab's lora_up rows: 32 * r * 4 (0 without LoRA)
  int n_fast;       // tile order: 1 = consecutive CTAs share the A row-tile and walk the N tiles (A is read from
                    // DRAM once, W stays L2-resident); 0 = M fastest (A re-streamed once per N tile when it exceeds L2)
  int a_mode;       // 0 plain, 1 conv3x3 stride 1, 2 conv3x3 stride 2, 3 stride 2 padded at the bottom / right
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
  const float* lora_sample_scale;  // per-sample factors (NULL = none): row m uses [m / lora_rows_per_sample]
  int lora_rows_per_sample;
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

// f[i] += t . up[i] over NQ groups of four ranks (all R of them by default), four terms at a time in rank order.
// up_rows: shared-memory address of the first of those ranks in 16 consecutive rows of [N, R] fp32 (same address for
// the whole warp: broadcast)
template <int R, int NQ = R / 4>
__device__ __forceinline__ void lora_apply(float* f, const float* t, uint32_t up_rows) {
#pragma unroll
  for (int i = 0; i < 16; ++i) {
#pragma unroll
    for (int q = 0; q < NQ; ++q) {
      const uint4 a = ld_shared_v4(up_rows + i * R * 4 + 16 * q);
      f[i] += t[4 * q] * __uint_as_float(a.x) + t[4 * q + 1] * __uint_as_float(a.y) +
              t[4 * q + 2] * __uint_as_float(a.z) + t[4 * q + 3] * __uint_as_float(a.w);
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

// The RT LoRA-down rows of a stage sit right behind its BN W rows, so [BN + RT, 64] is one K-major SW128 operand:
// wherever one wgmma can take it (N <= 256) each k-step issues a single m64 x (BN + RT) product and t = A.down^T is the
// tail of the accumulator fragment (registers BN/2 ..).  BN = 256 keeps a second product (N = RT) into its own fragment.
__host__ __device__ constexpr bool lora_folded(int bn, int rt) { return rt != 0 && bn + rt <= 256; }
__host__ __device__ constexpr int acc_regs(int bn, int rt) { return (lora_folded(bn, rt) ? bn + rt : bn) / 2; }
__host__ __device__ constexpr int accl_regs(int bn, int rt) { return (rt == 0 || lora_folded(bn, rt)) ? 1 : rt / 2; }

// Output tile t of the launch order -> its row tile mt and N tile nt
__device__ __forceinline__ void tile_coords(const GemmParams& p, int t, int& mt, int& nt) {
  mt = p.n_fast ? t / p.num_n_tiles : t % p.num_m_tiles;
  nt = p.n_fast ? t % p.num_n_tiles : t / p.num_m_tiles;
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

// Where the A operand of 128-row sub-tile st starts: its first row (plain) or its first output pixel (conv)
struct AOrigin {
  int m0, b0, h0, w0;
};
__device__ __forceinline__ AOrigin a_origin(const GemmParams& p, int st) {
  AOrigin o{st * kBM, 0, 0, 0};
  if (p.a_mode != 0) {
    if (st < p.num_sub)
      conv_origin(p, st, o.b0, o.h0, o.w0);
    else
      o.b0 = p.B;  // phantom sub-tile of an odd pair: every box is out of bounds -> zero fill
  }
  return o;
}

// TMA load of k-block kb of the A tile at `o` into sA (128 rows x 64 k, or the conv patch), completing on `bar`
__device__ __forceinline__ void load_a(const GemmParams& p, const AOrigin& o, int kb, uint32_t sA, uint32_t bar) {
  const int a_mode = p.a_mode, kb_split = p.kb_split, cb_total = p.cb_total;
  if (a_mode == 0) {
    const int src = kb < kb_split ? 0 : 1;
    tma_load_2d(sA, &p.tmA[src], bar, (src ? kb - kb_split : kb) * kBK, o.m0);
  } else {
    const int tap = kb / cb_total;  // filter tap and channel block of this k-block
    const int cb = kb - tap * cb_total;
    const int kh = tap / 3;
    const int kw = tap - kh * 3;
    if (a_mode == 1) {
      const int src = cb < kb_split ? 0 : 1;
      tma_load_4d(sA, &p.tmA[src], bar, (src ? cb - kb_split : cb) * kBK, o.w0 + kw - 1, o.h0 + kh - 1, o.b0);
    } else if (a_mode == 2) {
      // input row 2*ho + kh - 1: kh=0 -> odd plane, row ho-1; kh=1 -> even plane, row ho; kh=2 -> odd plane, row ho
      const int ph = (kh == 1) ? 0 : 1;
      const int pwl = (kw == 1) ? 0 : 1;
      tma_load_4d(sA, &p.tmA[ph * 2 + pwl], bar, cb * kBK, o.w0 + ((kw == 0) ? -1 : 0), o.h0 + ((kh == 0) ? -1 : 0),
                  o.b0);
    } else {
      // SB200_CONV_PAD_BR: input row 2*ho + kh: kh=0 -> even plane, row ho; kh=1 -> odd plane, row ho; kh=2 -> even
      // plane, row ho+1 (past the last row for ho = Ho-1: the TMA zero fill is the bottom / right pad)
      tma_load_4d(sA, &p.tmA[(kh & 1) * 2 + (kw & 1)], bar, cb * kBK, o.w0 + (kw >> 1), o.h0 + (kh >> 1), o.b0);
    }
  }
}

// Output row of row r of 128-row sub-tile st (the conv patch mapping of conv_origin), or -1 for a padding row (the
// phantom sub-tile of an odd pair has only padding rows)
__device__ __forceinline__ int tile_out_row(const GemmParams& p, int st, int r) {
  if (p.a_mode == 0) {
    const int m = st * kBM + r;
    return m < p.M ? m : -1;
  }
  int b0, h0, w0;
  conv_origin(p, st, b0, h0, w0);
  const int iw = r % p.bw;
  const int t2 = r / p.bw;
  const int ih = t2 % p.bh;
  const int ib = t2 / p.bh;
  const int b = b0 + ib, h = h0 + ih, w = w0 + iw;
  return (ib < p.bb && b < p.B && h < p.H && w < p.W) ? (b * p.H + h) * p.W + w : -1;
}

// The stage ring in shared memory: `stages` stages of stage_bytes from `tiles` on, each with a full barrier (its TMA
// bytes have landed) and an empty barrier (every consumer warpgroup of every CTA the stage feeds is done reading it)
struct Ring {
  uint32_t full, empty, tiles, stage_bytes;
  int stages;
};

// Prologue of both GEMM kernels: descriptor prefetch and barrier init, which overlap the previous kernel's tail, then
// the block / cluster sync and pdl_wait; global memory is touched only after it
template <int kCtas>
__device__ __forceinline__ Ring gemm_prologue(const GemmParams& p, bool has_lora) {
  pdl_trigger();
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;  // SWIZZLE_128B tiles need 1024 B alignment
  const Ring ring{base, base + 8u * p.stages, base + kBarRegion, static_cast<uint32_t>(p.stage_bytes), p.stages};
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&p.tmA[0]);
    tma_prefetch_desc(&p.tmB);
    if (has_lora) tma_prefetch_desc(&p.tmL);
  }
  if (threadIdx.x == 32) {
    // stage i's full barrier, then its empty one: one arrival per consumer warpgroup of every CTA the stage feeds
    for (int i = 0; i < ring.stages; ++i)
#pragma unroll
      for (int e = 0; e < 2; ++e) mbar_init((e ? ring.empty : ring.full) + 8u * i, e ? 2 * kCtas : 1);
    fence_barrier_init();
  }
  if constexpr (kCtas == 2) {
    cluster_sync_all();
  } else {
    __syncthreads();
  }
  pdl_wait();
  return ring;
}

// TMA producer, one converged warp: k-blocks [kb_lo, kb_hi) of the tile at A origin `ao` and N tile nt into the ring;
// `stage` and `phase` run on across calls.  A stage holds the A tile, the tile's kBRows W rows (GEGLU: its value rows,
// then the matching gate rows from row N/2 on) and RT LoRA-down rows.  In a CTA pair each CTA loads half of the W and
// LoRA-down rows (GEGLU: CTA 1 the gate rows) and multicasts them to both.
template <int kBRows, int RT, int kCtas>
__device__ __forceinline__ void produce(const GemmParams& p, const Ring& ring, const AOrigin& ao, int nt,
                                        uint32_t cta_rank, bool geglu, bool has_lora, int kb_lo, int kb_hi,
                                        int& stage, uint32_t& phase) {
  constexpr uint32_t a_bytes = kBM * 128, b_bytes = kBRows * 128;
  const uint32_t tx = static_cast<uint32_t>(p.a_tx) + b_bytes + static_cast<uint32_t>(RT) * 128u;
  int brow;  // the first W row this CTA loads
  if (geglu) {
    const int half = kBRows >> 1;
    brow = (kCtas == 2 && cta_rank == 1) ? (p.N >> 1) + nt * half : nt * half;
  } else {
    brow = nt * kBRows + static_cast<int>(cta_rank) * p.b_rows;
  }
  for (int kb = kb_lo; kb < kb_hi; ++kb) {
    const uint32_t full_bar = ring.full + 8u * stage;
    mbar_wait(ring.empty + 8u * stage, phase ^ 1u);
    if (elect_one()) {
      mbar_expect_tx(full_bar, tx);
      const uint32_t sA = ring.tiles + static_cast<uint32_t>(stage) * ring.stage_bytes;
      const uint32_t sB = sA + a_bytes;
      load_a(p, ao, kb, sA, full_bar);
      if constexpr (kCtas == 2) {
        const uint32_t boff = cta_rank * static_cast<uint32_t>(p.b_rows) * 128u;
        tma_load_2d_mc(sB + boff, &p.tmB, full_bar, kb * kBK, brow, 3);
        if (has_lora)
          tma_load_2d_mc(sB + b_bytes + cta_rank * static_cast<uint32_t>(p.l_rows) * 128u, &p.tmL, full_bar, kb * kBK,
                         static_cast<int>(cta_rank) * p.l_rows, 3);
      } else {
        tma_load_2d(sB, &p.tmB, full_bar, kb * kBK, brow);
        if (geglu) tma_load_2d(sB + (b_bytes >> 1), &p.tmB, full_bar, kb * kBK, (p.N >> 1) + nt * (kBRows >> 1));
        if (has_lora) tma_load_2d(sB + b_bytes, &p.tmL, full_bar, kb * kBK, 0);
      }
    }
    __syncwarp();
    if (++stage == ring.stages) {
      stage = 0;
      phase ^= 1u;
    }
  }
}

// reg_fence over an accumulator array, once its wgmmas have completed
template <int N>
__device__ __forceinline__ void fence_regs(float (&r)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) reg_fence(r[i]);
}

// Main loop of consumer warpgroup wg (rows wg * 64 ..) over k-blocks [kb_lo, kb_hi): zeroes acc (m64 x BN, with t =
// A.down^T in its tail where lora_folded) and accl (t otherwise, m64 x RT), issues each k-block's wgmmas with one
// k-block's group kept in flight, and hands each stage back (to both CTAs of a pair) once the products reading it are
// done.  On return every product has completed; the caller fences the registers (fence_regs).  Returns the stage of
// the last k-block, which it has not handed back.
template <int BN, int RT, int kCtas>
__device__ __forceinline__ int consume(float (&acc)[acc_regs(BN, RT)], float (&accl)[accl_regs(BN, RT)],
                                       const Ring& ring, int wg, uint32_t cta_rank, int kb_lo, int kb_hi, int& stage,
                                       uint32_t& phase) {
  constexpr uint32_t a_bytes = kBM * 128, b_bytes = BN * 128;
  constexpr bool folded = lora_folded(BN, RT);
#pragma unroll
  for (int i = 0; i < acc_regs(BN, RT); ++i) acc[i] = 0.f;
#pragma unroll
  for (int i = 0; i < accl_regs(BN, RT); ++i) accl[i] = 0.f;
  const bool signal = (threadIdx.x & 127) == 0;
  const uint32_t peer_empty = kCtas == 2 ? mapa_u32(ring.empty, cta_rank ^ 1u) : 0u;
  int prev = 0;
  for (int kb = kb_lo; kb < kb_hi; ++kb) {
    mbar_wait(ring.full + 8u * stage, phase);
    const uint32_t stage_base = ring.tiles + static_cast<uint32_t>(stage) * ring.stage_bytes;
    const uint32_t sA = stage_base + static_cast<uint32_t>(wg) * 64u * 128u;
    const uint32_t sB = stage_base + a_bytes;
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < kBK / 16; ++k) {
      const uint64_t adesc = gmma_desc_sw128(sA + 32u * k);
      if constexpr (folded) {
        wgmma_ss<BN + RT>(acc, adesc, gmma_desc_sw128(sB + 32u * k), 1u);
      } else {
        wgmma_ss<BN>(acc, adesc, gmma_desc_sw128(sB + 32u * k), 1u);
        if constexpr (RT != 0) wgmma_ss<RT>(accl, adesc, gmma_desc_sw128(sB + b_bytes + 32u * k), 1u);
      }
    }
    wgmma_commit();
    wgmma_wait<1>();  // the previous k-block's products have read their stage: hand it back to the producer(s)
    if (kb > kb_lo && signal) {
      mbar_arrive(ring.empty + 8u * prev);
      if (kCtas == 2) mbar_arrive_cluster(peer_empty + 8u * prev);
    }
    prev = stage;
    if (++stage == ring.stages) {
      stage = 0;
      phase ^= 1u;
    }
  }
  wgmma_wait<0>();
  return prev;
}

template <int BN, int kCtas, int RT>
__global__ void __launch_bounds__(kGemmThreads, gemm_slots(BN, RT)) gemm_kernel(const __grid_constant__ GemmParams p) {
  // launch_gemm runs every LoRA call on an RT > 0 instantiation, so the RT = 0 ones carry no LoRA code; GEGLU never
  // comes with LoRA (sb200_gemm refuses it), so the RT > 0 ones carry no GEGLU code, whose gate registers would
  // otherwise stay live across the LoRA update and spill the 96-register instantiations
  const bool has_lora = RT != 0 && (p.flags & SB200_EPI_LORA) != 0;
  const bool geglu = RT == 0 && (p.flags & SB200_EPI_GEGLU) != 0;
  const Ring ring = gemm_prologue<kCtas>(p, has_lora);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const uint32_t cta_rank = kCtas == 2 ? cluster_ctarank() : 0u;
  int mt, nt;
  tile_coords(p, blockIdx.x / kCtas, mt, nt);  // this CTA's (pair's) output tile
  const int st = mt * kCtas + static_cast<int>(cta_rank);  // this CTA's 128-row sub-tile
  const int kb_lo = p.sk_ws ? static_cast<int>(blockIdx.y) * p.sk_kb : 0;
  const int kb_hi = p.sk_ws ? min(p.kblocks, kb_lo + p.sk_kb) : p.kblocks;
  int stage = 0;
  uint32_t phase = 0;

  if (warp == kProducerWarp) {
    produce<BN, RT, kCtas>(p, ring, a_origin(p, st), nt, cta_rank, geglu, has_lora, kb_lo, kb_hi, stage, phase);
  } else {
    // ------------------------------------------------------------------ consumers: main loop
    const int wg = warp >> 2;
    static_assert(RT == 0 || lora_folded(BN, RT), "gemm_kernel keeps t = A.down^T in the accumulator's tail");
    float acc[acc_regs(BN, RT)];
    float accl[accl_regs(BN, RT)];
    consume<BN, RT, kCtas>(acc, accl, ring, wg, cta_rank, kb_lo, kb_hi, stage, phase);
    fence_regs(acc);
    fence_regs(accl);

    // ------------------------------------------------------------------ epilogue
    const uint32_t accs = ring.tiles;  // fp32 accumulator tile, over the stage ring
    constexpr int kStride = acc_stride(BN, RT);
    asm volatile("bar.sync %0, %1;" ::"n"(kConsumerBar), "n"(32 * kEpiWarps) : "memory");  // both warpgroups done reading
    store_frag<BN + RT>(acc, accs, wg * 64, 0, kStride);  // t = A.down^T lands in columns BN ..
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
    const bool has_resid = (p.flags & SB200_EPI_RESID) != 0;
    // per-warp staging buffer ([32 rows x 32 cols] bf16, 64 B rows, 16-byte chunks XOR-swizzled by (row >> 1) & 3):
    // residual tiles arrive here by cp.async with coalesced global reads, results leave from here with coalesced global
    // writes; in between every thread touches only its own row.  The buffers sit in the ring behind the accumulator
    // tile: every k-block's loads have landed (this CTA waited on each full barrier, whose byte count includes the
    // peer's multicast) and both warpgroups have passed kConsumerBar, so nothing else writes or reads there.
    const uint32_t epi = accs + static_cast<uint32_t>(acc_tile_bytes(BN, RT));
    const uint32_t ebuf = epi + static_cast<uint32_t>(warp) * (kEpiBufBytes + p.up_buf_bytes);
    const uint32_t ubuf = ebuf + kEpiBufBytes;  // p.up_buf_bytes of lora_up rows
    const uint32_t arow = accs + static_cast<uint32_t>((q * 32 + lane) * kStride) * 4u;
    const int my_row = tile_out_row(p, st, q * 32 + lane);  // output row of this thread's accumulator row, or -1
    const bool row_ok = my_row >= 0;
    float lscale = has_lora ? (p.lora_scale_dev ? p.lora_scale * __ldg(p.lora_scale_dev) : p.lora_scale) : 0.f;
    // this thread's row factor, read once per tile; without a vector nothing is loaded and lscale keeps its bits
    if (has_lora && p.lora_sample_scale != nullptr && row_ok)
      lscale *= __ldg(p.lora_sample_scale + my_row / p.lora_rows_per_sample);
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
        if (p.lora_r >= 8) cp_async_16(ub + 16, src + 4);
        if (p.lora_r == 16) {
          cp_async_16(ub + 32, src + 8);
          cp_async_16(ub + 48, src + 12);
        }
      }
      cp_async_commit();
    };
    const bool staged = has_resid || has_lora;
    if (staged && my_slabs > 0) prefetch_resid(hsel * kSlab, min(kSlab, ncols_valid - hsel * kSlab));
    const __nv_bfloat16* rb =
        (p.flags & SB200_EPI_ROWBIAS) ? p.rowbias + static_cast<size_t>(row_ok ? my_row / p.rows_per_batch : 0) * p.Nout
                                      : nullptr;
    float tl[8];
    int group_lo = 0, group_hi = 0;  // output-column range of the adaptor whose t = A.down^T is held in tl
    // tl = lscale * t, from the 8 t columns of this row starting at column j; rank 4 uses the first 4 (the row's 4
    // padding floats cover the last adaptor's read)
    auto load_t8 = [&](int j) {
      uint32_t tv[8];
      ld_acc<8>(arow + (BN + j) * 4, tv);
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) tl[jj] = __uint_as_float(tv[jj]) * lscale;
    };
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
        if (has_lora && p.lora_r != 16 && (n < group_lo || n >= group_hi)) {
          const int grp = n / p.lora_group_n;
          group_lo = grp * p.lora_group_n;
          group_hi = group_lo + p.lora_group_n;
          load_t8(grp * p.lora_r);
        }
        float f[16];
#pragma unroll
        for (int j = 0; j < 16; ++j) f[j] = __uint_as_float(v[j]);
        if (staged && sub == 0) {  // this slab's residual / lora_up rows have landed
          cp_async_wait<0>();
          __syncwarp();
        }
        if (has_lora) {
          const uint32_t up = ubuf + sub * 16 * p.lora_r * 4;
          if (p.lora_r == 4) {
            lora_apply<4>(f, tl, up);
          } else if (p.lora_r == 8) {
            lora_apply<8>(f, tl, up);
          } else {
            // rank 16: t is re-read for every 16 columns, ranks 0..7 then 8..15, so that the epilogue holds no more
            // registers than at rank 8 (the 96-register instantiations would spill); each element still adds its
            // terms in rank order.  The __syncwarp keeps ptxas from hoisting the second half's shared-memory loads
            // over the first half's FMAs, which would hold both halves live again.
            const int j = (n / p.lora_group_n) * 16;
            load_t8(j);
            lora_apply<16, 2>(f, tl, up);
            __syncwarp();
            load_t8(j + 8);
            lora_apply<16, 2>(f, tl, up + 32);
          }
        }
        if (p.flags & SB200_EPI_BIAS) add_bf16x16(f, p.bias + n);
        if (rb) add_bf16x16(f, rb + n);
        if (geglu) {
          float gb[16];
#pragma unroll
          for (int j = 0; j < 16; ++j) gb[j] = __uint_as_float(g[j]);
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
  }

  if constexpr (kCtas == 2) {
    __syncwarp();
    cluster_sync_all();  // the peer's barriers / smem must outlive every multicast and remote arrive aimed at them
  }
}

// -------------------------------------------------------------------------------------------------
// Wide tiles: a persistent kernel for layers whose W has a multiple of 160 or 256 rows
// -------------------------------------------------------------------------------------------------
// gemm_wide_kernel<BN, RT, GEGLU>: 128 x BN tiles, BN = 256 (GEGLU: 256 W rows, 128 output columns) or 160 (every
// width the SD / SDXL UNets run is a multiple of 320, so 160 tiles their 320- and 640-wide layers with no ragged
// tile, and 160 + 32 LoRA rows still fit one wgmma), 384 threads, one CTA per SM,
// each CTA walking the tiles blockIdx.x, blockIdx.x + gridDim.x, ... in launch_gemm's order:
//   warpgroup 2    producer: gives its registers to the consumers (setmaxnreg 40); one elected thread of warp 8 issues
//                  the TMA loads, running ahead into the next tile while the consumers finish the current epilogue
//   warpgroups 0/1 consumers (setmaxnreg 232): rows 0..63 / 64..127, an m64 x BN accumulator of BN / 2 registers
// The k-loop, its barrier protocol and the LoRA-down rows behind the W rows are gemm_kernel's (gemm_prologue, produce
// and consume, called once per tile); the ring's stage and phase run on across tiles, and the consumers hand each
// tile's last stage back once its wgmmas are done.  The epilogue works on the accumulator registers: per element it applies, in gemm_kernel's
// order and with its expressions, the LoRA update, bias, row bias and GEGLU, rounds to bf16, adds the residual in bf16,
// and leaves through a swizzled staging buffer (two per warpgroup, 64 rows x wide_chunk columns each) with coalesced
// stores.
// Only t = A.down^T and the tile's lora_up rows are staged in shared memory.  No split-K or CTA pairs: those stay on
// gemm_kernel.  GEGLU is a template parameter (only with RT = 0: GEGLU never comes with LoRA) rather than a flag: with
// a runtime flag every element's gate code sat between the plain path's instructions and the chunk loop spanned
// ~29 KB of SASS; a chunk took 2 000-2 500 cycles for 32 elements per thread with no global access on the way (clock64
// stamps per phase on an H100 SXM at 700 W), far above its instruction count and in line with instruction fetch from
// a loop that does not stay in the instruction cache.  Split, and with 16-byte output stores, a plain tile's epilogue
// takes half the cycles (DESIGN §8 item 1).
constexpr int kWideThreads = 384;
constexpr int kWideBarBase = 1;  // named barriers 1, 2: one per consumer warpgroup

// Output columns per staging buffer: 64 where they divide the tile (128 B rows, 16-byte chunks XOR-swizzled by row & 7),
// else 32 (BN = 160: 64 B rows swizzled by (row >> 1) & 3, gemm_kernel's layout).  Either way the 8 rows a warp stores
// to at once, and the 2 or 1 rows a quarter-warp copies out, fall into distinct banks.
__host__ __device__ constexpr int wide_chunk(int bn) { return bn % 64 == 0 ? 64 : 32; }
__host__ __device__ constexpr int wide_stg_bytes(int bn) { return 64 * wide_chunk(bn) * 2; }  // [64 rows x chunk] bf16

// Shared memory of one consumer warpgroup's epilogue: two staging buffers, then with LoRA its 64 rows of t
// (row stride rt + 4 floats) and the tile's bn lora_up rows.
__host__ __device__ constexpr int wide_t_bytes(int rt) { return rt ? 64 * (rt + 4) * 4 : 0; }
__host__ __device__ constexpr int wide_epi_bytes(int bn, int rt, int r) {
  return 2 * wide_stg_bytes(bn) + wide_t_bytes(rt) + (rt ? bn * r * 4 : 0);
}

// t = A.down^T of a consumer warpgroup's rows: the accumulator's tail where the LoRA rows ride in the main wgmma
template <int BN, int RT>
__device__ __forceinline__ const float* t_frag(const float (&acc)[acc_regs(BN, RT)],
                                               const float (&accl)[accl_regs(BN, RT)]) {
  if constexpr (lora_folded(BN, RT))
    return acc + BN / 2;
  else
    return accl;
}

template <int BN, int RT, bool GEGLU>
__global__ void __launch_bounds__(kWideThreads, 1) gemm_wide_kernel(const __grid_constant__ GemmParams p) {
  static_assert(!GEGLU || (BN % 256 == 0 && RT == 0), "GEGLU runs on 256-wide tiles without LoRA");
  const Ring ring = gemm_prologue<1>(p, RT != 0);
  const int warp = threadIdx.x >> 5;
  constexpr bool geglu = GEGLU;
  const int num_tiles = p.num_m_tiles * p.num_n_tiles;
  int stage = 0;
  uint32_t phase = 0;

  if (warp >= 8) {
    // ------------------------------------------------------------------ TMA producer
    setmaxnreg_dec<40>();
    if (warp != 8) return;
    for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
      int mt, nt;
      tile_coords(p, t, mt, nt);
      produce<BN, RT, 1>(p, ring, a_origin(p, mt), nt, 0u, geglu, RT != 0, 0, p.kblocks, stage, phase);
    }
    return;
  }

  // ------------------------------------------------------------------ consumers
  setmaxnreg_inc<232>();
  const int wg = warp >> 2;
  const int tid = threadIdx.x & 127;
  const int lane = threadIdx.x & 31;
  const int q = lane & 3;
  const int fr0 = (warp & 3) * 16 + (lane >> 2);  // accumulator rows of this thread: fr0 and fr0 + 8 (of 64)
  const bool has_lora = RT != 0;
  const bool has_resid = (p.flags & SB200_EPI_RESID) != 0;
  const bool has_bias = (p.flags & SB200_EPI_BIAS) != 0;
  const bool has_rb = (p.flags & SB200_EPI_ROWBIAS) != 0;
  const int r = has_lora ? p.lora_r : 0;
  const float lscale = has_lora ? (p.lora_scale_dev ? p.lora_scale * __ldg(p.lora_scale_dev) : p.lora_scale) : 0.f;
  constexpr int kChunk = wide_chunk(BN);
  constexpr int kCpr = kChunk / 8;          // 16-byte chunks per staging row = 8-column accumulator blocks per chunk
  constexpr int kPitch = kChunk * 2;        // bytes per staging row
  constexpr int kCopyRows = 128 / kCpr;     // staging rows the warpgroup moves per pass
  constexpr int kPasses = 64 / kCopyRows;
  constexpr int nchunks = (GEGLU ? BN / 2 : BN) / kChunk;  // p.ncols_out / kChunk
  auto swz = [](int row) { return kChunk == 64 ? (row & 7) : ((row >> 1) & 3); };
  const uint32_t epi = ring.tiles + static_cast<uint32_t>(ring.stages) * ring.stage_bytes +
                       static_cast<uint32_t>(wg) * static_cast<uint32_t>(wide_epi_bytes(BN, RT, r));
  const uint32_t tbuf = epi + 2 * wide_stg_bytes(BN);  // [64][RT + 4] fp32: t of this warpgroup's rows
  const uint32_t ubuf = tbuf + wide_t_bytes(RT);        // [BN][r] fp32: the tile's lora_up rows
  constexpr int kTStride = RT + 4;
  // rows / 16-byte chunk this thread moves between a staging buffer and global memory: rows crow + kCopyRows i, chunk cch
  const int crow = tid / kCpr, cch = tid % kCpr;
  const uint32_t bar_id = kWideBarBase + wg;
  auto wg_sync = [&]() { asm volatile("bar.sync %0, 128;" ::"r"(bar_id) : "memory"); };

  for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
    int st, nt;
    tile_coords(p, t, st, nt);
    const int n_base = nt * p.ncols_out;
    int orow[kPasses];  // output rows this thread copies
#pragma unroll
    for (int i = 0; i < kPasses; ++i) orow[i] = tile_out_row(p, st, wg * 64 + crow + kCopyRows * i);
    auto prefetch_resid = [&](int c, uint32_t buf) {
#pragma unroll
      for (int i = 0; i < kPasses; ++i) {
        const int row = crow + kCopyRows * i;
        if (orow[i] >= 0)
          cp_async_16(buf + row * kPitch + ((cch ^ swz(row)) << 4),
                      p.resid + static_cast<size_t>(orow[i]) * p.ldr + n_base + c * kChunk + cch * 8);
      }
      cp_async_commit();
    };
    // The tile's lora_up rows and its first residual chunk are loaded while its k-blocks run, so that the epilogue
    // does not start with a global-memory round trip.  Their buffers are free once every thread of the warpgroup is
    // done with the previous tile's epilogue.
    wg_sync();
    if constexpr (RT != 0) {
      const float* up_src = p.lora_up + static_cast<size_t>(n_base) * r;
      for (int i = tid; i < BN * r / 4; i += 128) cp_async_16(ubuf + i * 16, up_src + i * 4);
      cp_async_commit();
    }
    if (has_resid) prefetch_resid(0, epi);
    float acc[acc_regs(BN, RT)];
    float accl[accl_regs(BN, RT)];
    const int last = consume<BN, RT, 1>(acc, accl, ring, wg, 0u, 0, p.kblocks, stage, phase);
    if (tid == 0) mbar_arrive(ring.empty + 8u * last);  // the last stage of the tile, for the producer's next tile
    fence_regs(acc);
    fence_regs(accl);

    // ------------------------------------------------------------------ epilogue
    if constexpr (RT != 0) {
      // t = A.down^T of this warpgroup's rows (fragment layout as in wgmma.cuh)
      const float* tf = t_frag<BN, RT>(acc, accl);
#pragma unroll
      for (int i = 0; i < RT / 2; i += 2) {
        const int row = fr0 + 8 * ((i >> 1) & 1);
        const int col = 8 * (i >> 2) + 2 * q;
        asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(tbuf + (row * kTStride + col) * 4), "f"(tf[i]),
                     "f"(tf[i + 1])
                     : "memory");
      }
    }
    if (has_resid || has_lora) {
      cp_async_wait<0>();
      wg_sync();
    }
    const __nv_bfloat16* rb[2] = {nullptr, nullptr};
    if (has_rb) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int orw = tile_out_row(p, st, wg * 64 + fr0 + 8 * h);
        rb[h] = p.rowbias + static_cast<size_t>(orw >= 0 ? orw / p.rows_per_batch : 0) * p.Nout;
      }
    }
    // lscale with the per-sample factors of rows fr0 and fr0 + 8, read once per tile outside the chunk loop
    float lsc[2] = {lscale, lscale};
    if (RT != 0 && p.lora_sample_scale != nullptr) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int orw = tile_out_row(p, st, wg * 64 + fr0 + 8 * h);
        if (orw >= 0) lsc[h] *= __ldg(p.lora_sample_scale + orw / p.lora_rows_per_sample);
      }
    }
    float tl[2][8];  // lsc * t of the current adaptor, rows fr0 and fr0 + 8
    int cur_grp = -1;
    // A runtime loop over the chunks keeps one copy of the epilogue code (unrolled it outgrows the instruction cache);
    // each pass first selects its chunk's accumulator registers (and with GEGLU its gate registers).
#pragma unroll 1
    for (int c = 0; c < nchunks; ++c) {
      {
        constexpr int kChunkRegs = kChunk / 2;  // accumulator registers per thread and chunk
        float v[kChunkRegs], gv[kChunkRegs];
#pragma unroll
        for (int k = 0; k < kChunkRegs; ++k) {
          v[k] = acc[k];
#pragma unroll
          for (int cc = 1; cc < nchunks; ++cc) v[k] = c == cc ? acc[cc * kChunkRegs + k] : v[k];
          if constexpr (GEGLU) {  // column + BN / 2, the gate half
            gv[k] = acc[nchunks * kChunkRegs + k];
#pragma unroll
            for (int cc = 1; cc < nchunks; ++cc) gv[k] = c == cc ? acc[(nchunks + cc) * kChunkRegs + k] : gv[k];
          }
        }
        const uint32_t buf = epi + static_cast<uint32_t>(c & 1) * wide_stg_bytes(BN);
        uint32_t o[kCpr][2];
#pragma unroll
        for (int jj = 0; jj < kCpr; ++jj) {
          const int j = c * kCpr + jj;  // 8-column block of the accumulator
          const int n = n_base + 8 * j + 2 * q;
          float up[2][8];
          if constexpr (RT != 0) {
            const int grp = n / p.lora_group_n;
            if (grp != cur_grp) {
              cur_grp = grp;
#pragma unroll
              for (int h = 0; h < 2; ++h) {
                const uint32_t ta = tbuf + ((fr0 + 8 * h) * kTStride + grp * r) * 4;
                const uint4 a = ld_shared_v4(ta);
                const uint4 b = r == 8 ? ld_shared_v4(ta + 16) : make_uint4(0, 0, 0, 0);
                const uint32_t tv[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
#pragma unroll
                for (int jt = 0; jt < 8; ++jt) tl[h][jt] = __uint_as_float(tv[jt]) * lsc[h];
              }
            }
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const uint32_t ua = ubuf + (8 * j + 2 * q + e) * r * 4;
              const uint4 a = ld_shared_v4(ua);
              const uint4 b = r == 8 ? ld_shared_v4(ua + 16) : make_uint4(0, 0, 0, 0);
              const uint32_t uv[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
#pragma unroll
              for (int ju = 0; ju < 8; ++ju) up[e][ju] = __uint_as_float(uv[ju]);
            }
          }
          const uint32_t bw = has_bias ? __ldg(reinterpret_cast<const uint32_t*>(p.bias + n)) : 0u;
          const uint32_t gbw = (has_bias && geglu) ? __ldg(reinterpret_cast<const uint32_t*>(p.bias + p.Nout + n)) : 0u;
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const uint32_t rbw = has_rb ? __ldg(reinterpret_cast<const uint32_t*>(rb[h] + n)) : 0u;
            float f[2];
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int i = 4 * jj + 2 * h + e;
              f[e] = v[i];
              if constexpr (RT != 0) {
                // gemm_kernel's lora_apply, term for term
                f[e] += tl[h][0] * up[e][0] + tl[h][1] * up[e][1] + tl[h][2] * up[e][2] + tl[h][3] * up[e][3];
                if (r == 8)
                  f[e] += tl[h][4] * up[e][4] + tl[h][5] * up[e][5] + tl[h][6] * up[e][6] + tl[h][7] * up[e][7];
              }
              if (has_bias) f[e] += e ? bf16_hi(bw) : bf16_lo(bw);
              if (has_rb) f[e] += e ? bf16_hi(rbw) : bf16_lo(rbw);
              if (geglu) {
                float gb = gv[i];
                if (has_bias) gb += e ? bf16_hi(gbw) : bf16_lo(gbw);
                f[e] *= gelu_erf_f(gb);
              }
            }
            o[jj][h] = pack_bf16x2(f[0], f[1]);
          }
        }
        if (has_resid && c > 0) {
          cp_async_wait<0>();
          wg_sync();  // chunk c's residual has landed; chunk c - 1's copy-out from the other buffer is done
        }
        if (has_resid && c + 1 < nchunks)
          prefetch_resid(c + 1, epi + static_cast<uint32_t>((c + 1) & 1) * wide_stg_bytes(BN));
#pragma unroll
        for (int jj = 0; jj < kCpr; ++jj) {
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int row = fr0 + 8 * h;
            const uint32_t a = buf + row * kPitch + ((jj ^ swz(row)) << 4) + q * 4;
            // the residual is added to the ROUNDED projection, in bf16, as in gemm_kernel
            st_shared_u32(a, has_resid ? add_bf16x2(o[jj][h], ld_shared_u32(a)) : o[jj][h]);
          }
        }
        wg_sync();
#pragma unroll
        for (int i = 0; i < kPasses; ++i) {
          const int row = crow + kCopyRows * i;
          const uint4 v = ld_shared_v4(buf + row * kPitch + ((cch ^ swz(row)) << 4));
          if (orow[i] >= 0)
            st_global_v4(p.out + static_cast<size_t>(orow[i]) * p.ldo + n_base + c * kChunk + cch * 8, v);
        }
      }
    }
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

// Tile widths: 64 and 128 run gemm_kernel, 160 and 256 run gemm_wide_kernel (a 160- or 256-wide accumulator needs the
// registers a producer warpgroup gives up, which 288 threads do not have).
static bool is_wide(int bn) { return bn == 160 || bn == 256; }
static bool bn_supported(int bn) { return bn == 64 || bn == 128 || is_wide(bn); }

// gemm_wide_kernel takes W with a multiple of bn rows (with GEGLU, only at bn = 256: 128 rows per half, so a tile
// writes 128 output columns), single CTAs, and LoRA of rank 4 or 8 in at most 32 rows.
static bool wide_lora_ok(int lora_r, int lora_rt) { return lora_rt == 0 || (lora_rt <= 32 && lora_r <= 8); }
static bool wide_eligible(int bn, int N, int ctas, int lora_r, int lora_rt, bool geglu) {
  return N % bn == 0 && ctas == 1 && wide_lora_ok(lora_r, lora_rt) && (bn == 256 || !geglu);
}

// Tile width from a cost model in SM cycles.  A 128 x bn tile's 64-deep k-block takes 4 bn cycles of tensor work (m64
// wgmmas of two warpgroups at 4096 bf16 FLOP / clk / SM) plus the LoRA columns and ~208 cycles of per-k-block
// overhead; a tile pays ~1500 cycles of prologue and pipeline fill and an epilogue of ~21 cycles per output column
// (more with a residual / LoRA / GEGLU).  The busiest SM runs ceil(tiles / num_sms) tiles; their tensor work adds up,
// but where two CTAs share the SM (gemm_slots) one's prologue and epilogue run under the other's wgmmas, so the fixed
// cost is paid once per pair.  The constants are a least-squares fit (7 % rms) to the times of the B = 8 SDXL shapes
// with BN forced (no CTA pairs, each instantiation at its own residency) on an H100 80GB HBM3 SXM at 400 W, in us
// (BN 64 / 128): 8192 x 10240 x 1280 GEGLU 683 / 551,
// 8192 x 1280 x 5120 + residual 293 / 245, 8192 x 3840 x 1280 LoRA 299 / 241, 32768 x 5120 x 640 GEGLU 833 / 625,
// 32768 x 1920 x 640 LoRA 361 / 315, 32768 x 640 x 640 LoRA + residual 137 / 131, 616 x 153600 x 2048 1225 / 949,
// LoRA convs 32x32 1280 -> 1280 850 / 620, 64x64 640 -> 640 831 / 630, 128x128 320 -> 320 881 / 832 (B = 8).
// gemm_wide_kernel in the same units: 4 (bn + rt) cycles per k-block, a LoRA term more with LoRA, and a per-tile term
// (epilogue and pipeline refill; the wide epilogue does not overlap the tensor cores): kWideLoraPerKb / kWideTile at
// bn = 256, kW160LoraPerKb / kW160Tile at bn = 160, where the LoRA-down rows ride in the main wgmma (lora_folded) and a
// LoRA k-block costs less than half as much.  The 256 constants were fitted earlier (its LoRA k-block costs more than
// its 16 extra columns); the 160 ones are the grid-search optimum over the times below, with each width forced, on an
// H100 80GB HBM3 SXM at 700 W (us, BN 64 / 128 / 160 / 256, "-" where the width does not divide N), B = 8 SDXL:
// 8192 x 10240 x 1280 GEGLU 585 / 442 / - / 387, 8192 x 1280 x 5120 + residual 277 / 217 / 155 / 170, 32768 x 5120 x
// 640 GEGLU 752 / 531 / - / 457, 616 x 153600 x 2048 1115 / 744 / 666 / 607, 8192 x 1280 x 1280 bias 72.1 / 61.7 / 50.0
// / 54.8, the same + residual 79.5 / 70.4 / 57.2 / 57.9, 8192 x 3840 x 1280 LoRA 223 / 199 / 180 / 182, 8192 x 1280 x
// 1280 LoRA + residual 84.7 / 79.1 / 63.4 / 72.3, 32768 x 1920 x 640 LoRA 274 / 262 / 231 / -, 32768 x 640 x 640 bias +
// residual 104 / 81.8 / 79.3 / -, the same with LoRA 111 / 116 / 90.7 / -, 32768 x 640 x 2560 + residual 277 / 208 /
// 175 / -, LoRA convs 32x32 1280 -> 1280 + residual 693 / 451 / 372 / 464, 2560 -> 1280 1540 / 959 / 795 / 1184, 64x64
// 640 -> 640 + residual 689 / 476 / 394 / -, 128x128 320 -> 320 + residual 732 / 757 / 450 / -, 640 -> 320 1438 / 1368
// / 779 / -; SD-1.5 at B = 1 (CFG pair): 512 x 1280 x 1280 + residual 10.1 / 13.2 / 13.0 / 18.3, 512 x 3840 x 1280
// LoRA 16.8 / 14.5 / 17.1 / 23.5, 512 x 10240 x 1280 GEGLU 46.4 / 42.4 / - / 38.3, 2048 x 5120 x 640 GEGLU 50.9 / 40.7
// / - / 39.1, convs 16x16 and 8x8 1280 -> 1280 + residual 73 / 82 / 85 / 112 and 74 / 82 / 84 / 112, 8192 x 320 x 320
// LoRA + residual 16.1 / 17.9 / 10.8 / -, 8192 x 960 x 320 LoRA 29.0 / 30.2 / 26.0 / -, 2048 x 640 x 640 LoRA +
// residual 11.8 / 11.3 / 12.0 / -, LoRA convs + residual 64x64 320 -> 320 54.2 / 55.0 / 28.9 / - and 32x32 640 -> 640
// 61.2 / 47.4 / 48.8 / -.  Single-wave grids (SD-1.5 at B = 1) stay on the narrow tiles, whose smaller tiles finish
// sooner.  The model picks the fastest width for every shape but the 512 x 10240 GEGLU, which stays at 128 (10 %
// slower than 256).
constexpr double kWideTile = 5400.0;
constexpr double kWideLoraPerKb = 370.0;
constexpr double kW160Tile = 5600.0;
constexpr double kW160LoraPerKb = 160.0;
static TileChoice pick_tile(int ncols, int num_sms, int kblocks, int lora_r, int lora_rt, int force_ctas, int sub_tiles,
                            int flags) {
  double best = -1;
  TileChoice bc{1, 64};
  const int ctas = force_ctas ? force_ctas : (pairs_always() ? 2 : 1);
  const bool geglu = (flags & SB200_EPI_GEGLU) != 0;
  const double epi_per_col = 21.0 + ((flags & SB200_EPI_RESID) ? 7.5 : 0.0) + (lora_rt ? 9.0 : 0.0) + (geglu ? 15.0 : 0.0);
  for (const int bn : {64, 128, 160, 256}) {
    if (is_wide(bn) && !wide_eligible(bn, ncols, ctas, lora_r, lora_rt, geglu)) continue;
    const long tiles = static_cast<long>(sub_tiles) * ((ncols + bn - 1) / bn);
    const long load = (tiles + num_sms - 1) / num_sms;
    const int cols_out = geglu ? bn / 2 : bn;
    double cost;
    if (is_wide(bn)) {
      // persistent, one CTA per SM
      const double lora_kb = lora_rt ? (bn == 256 ? kWideLoraPerKb : kW160LoraPerKb) : 0.0;
      cost = load * (kblocks * (4.0 * (bn + lora_rt) + lora_kb) + (bn == 256 ? kWideTile : kW160Tile));
    } else {
      const int slots = gemm_slots(bn, lora_rt);
      const double perkb = 4.0 * (bn + lora_rt) + 208.0;
      cost = load * kblocks * perkb + ((load + slots - 1) / slots) * (1500.0 + epi_per_col * cols_out);
    }
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

// Dynamic shared memory one CTA may use when `slots` CTAs are to share an SM.
static int smem_budget(const Ctx* ctx, int slots) {
  return std::min(ctx->smem_optin, ctx->smem_per_sm / slots - ctx->smem_reserved);
}

// Launches kKernel, kThreads threads per CTA and built for kSlots CTAs per SM, in clusters of `cluster` CTAs.  Its
// first launch opts it in to the SM's shared memory and checks with the occupancy calculator that kSlots CTAs fit.
template <void (*kKernel)(GemmParams), int kThreads, int kSlots>
static int launch_checked(Ctx* ctx, cudaStream_t stream, const GemmParams& p, dim3 grid, int smem, int cluster,
                          bool pdl) {
  static bool checked = false;  // one flag per instantiation
  if (!checked) {
    SB200_CUDA_CHECK(cudaFuncSetAttribute(kKernel, cudaFuncAttributeMaxDynamicSharedMemorySize, ctx->smem_optin));
    SB200_CUDA_CHECK(
        cudaFuncSetAttribute(kKernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
    int resident = 0;
    SB200_CUDA_CHECK(
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&resident, kKernel, kThreads, smem_budget(ctx, kSlots)));
    if (resident < kSlots)
      return set_error(SB200_ERR_CUDA, "gemm: bn=%d, %d CTA(s) per cluster, rt=%d: %d CTA(s) per SM fit, built for %d",
                       p.bn, cluster, p.lora_rt, resident, kSlots);
    checked = true;
  }
  SB200_CUDA_CHECK(launch_ex(kKernel, grid, dim3(kThreads), smem, stream, cluster, pdl, p));
  return 0;
}

// gemm_kernel<BN, kCtas, RT> for the call's RT
template <int BN, int kCtas>
static int launch_narrow(Ctx* ctx, cudaStream_t s, const GemmParams& p, int rt, int smem, bool pdl) {
  const dim3 grid(p.num_m_tiles * p.num_n_tiles * kCtas, p.sk_ws ? p.sk_splits : 1);
  constexpr int T = kGemmThreads;
  switch (rt) {
    case 0: return launch_checked<gemm_kernel<BN, kCtas, 0>, T, gemm_slots(BN, 0)>(ctx, s, p, grid, smem, kCtas, pdl);
    case 16: return launch_checked<gemm_kernel<BN, kCtas, 16>, T, gemm_slots(BN, 16)>(ctx, s, p, grid, smem, kCtas, pdl);
    case 32: return launch_checked<gemm_kernel<BN, kCtas, 32>, T, gemm_slots(BN, 32)>(ctx, s, p, grid, smem, kCtas, pdl);
    default: return launch_checked<gemm_kernel<BN, kCtas, 64>, T, gemm_slots(BN, 64)>(ctx, s, p, grid, smem, kCtas, pdl);
  }
}

// gemm_wide_kernel<BN, RT, GEGLU> for the call's RT and epilogue
template <int BN>
static int launch_wide(Ctx* ctx, cudaStream_t s, const GemmParams& p, int rt, dim3 grid, int smem, bool pdl) {
  constexpr int T = kWideThreads;
  if (rt == 16) return launch_checked<gemm_wide_kernel<BN, 16, false>, T, 1>(ctx, s, p, grid, smem, 1, pdl);
  if (rt != 0) return launch_checked<gemm_wide_kernel<BN, 32, false>, T, 1>(ctx, s, p, grid, smem, 1, pdl);
  if constexpr (BN == 256)
    if (p.flags & SB200_EPI_GEGLU) return launch_checked<gemm_wide_kernel<BN, 0, true>, T, 1>(ctx, s, p, grid, smem, 1, pdl);
  return launch_checked<gemm_wide_kernel<BN, 0, false>, T, 1>(ctx, s, p, grid, smem, 1, pdl);
}

// *pdl receives the launch's PDL choice
static int launch_gemm(Ctx* ctx, cudaStream_t stream, GemmParams& p, int ctas, bool* pdl) {
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
  const int rt = has_lora ? p.lora_rt : 0;
  int st;
  if (is_wide(p.bn)) {
    // one CTA per SM: the ring gets what the two warpgroups' epilogue buffers leave of the SM's shared memory
    const int budget = smem_budget(ctx, 1);
    const int epi = 2 * wide_epi_bytes(p.bn, rt, has_lora ? p.lora_r : 0);
    const int stages = std::min(kMaxStages, (budget - kBarRegion - kAlignSlack - epi) / p.stage_bytes);
    if (stages < 2) return set_error(SB200_ERR_INVALID, "gemm: tile does not fit shared memory");
    p.stages = stages;
    p.ring_bytes = stages * p.stage_bytes + epi;
    const int smem = kBarRegion + kAlignSlack + p.ring_bytes;
    *pdl = pdl_small_grid(ctx, p.num_m_tiles * p.num_n_tiles);
    const dim3 grid(std::min(p.num_m_tiles * p.num_n_tiles, ctx->num_sms));
    st = p.bn == 160 ? launch_wide<160>(ctx, stream, p, rt, grid, smem, *pdl)
                     : launch_wide<256>(ctx, stream, p, rt, grid, smem, *pdl);
  } else {
    const int grid_ctas = p.num_m_tiles * p.num_n_tiles * ctas * (p.sk_ws ? p.sk_splits : 1);
    // A grid that gives each SM at most one CTA lets that CTA have the whole SM's shared memory (a deeper ring).
    const int budget = smem_budget(ctx, grid_ctas > ctx->num_sms ? gemm_slots(p.bn, rt) : 1);
    int stages = (budget - kBarRegion - kAlignSlack) / p.stage_bytes;
    if (stages > kMaxStages) stages = kMaxStages;
    if (stages < 2) return set_error(SB200_ERR_INVALID, "gemm: tile does not fit shared memory");
    p.stages = stages;
    p.ring_bytes = std::max(stages * p.stage_bytes, acc_tile_bytes(p.bn, rt) + kEpiBytes + kEpiWarps * p.up_buf_bytes);
    const int smem = kBarRegion + kAlignSlack + p.ring_bytes;
    if (smem > budget) return set_error(SB200_ERR_INVALID, "gemm: tile does not fit shared memory");
    *pdl = pdl_small_grid(ctx, grid_ctas);
    if (p.bn == 128)
      st = ctas == 2 ? launch_narrow<128, 2>(ctx, stream, p, rt, smem, *pdl)
                     : launch_narrow<128, 1>(ctx, stream, p, rt, smem, *pdl);
    else
      st = ctas == 2 ? launch_narrow<64, 2>(ctx, stream, p, rt, smem, *pdl)
                     : launch_narrow<64, 1>(ctx, stream, p, rt, smem, *pdl);
  }
  if (st) return st;
  SB200_CUDA_CHECK(cudaGetLastError());
  return 0;
}

static int check_lora(const sb200_lora* l, int M, int N) {
  SB200_REQUIRE(l->down && l->up, "lora: NULL weights");
  SB200_REQUIRE(l->r == 4 || l->r == 8 || l->r == 16,
                "lora: slot width %d unsupported by the fused epilogue (4, 8 or 16; pad lower ranks with zeros)", l->r);
  SB200_REQUIRE(l->rt == 16 || l->rt == 32 || l->rt == 64, "lora: rt must be 16, 32 or 64");
  SB200_REQUIRE(l->group_n > 0 && l->group_n % 16 == 0, "lora: group_n must be a multiple of 16");
  const int groups = (N + l->group_n - 1) / l->group_n;
  SB200_REQUIRE(groups * l->r <= l->rt, "lora: %d groups of rank %d exceed rt=%d", groups, l->r, l->rt);
  SB200_REQUIRE(!l->sample_scale || (l->rows_per_sample > 0 && M % l->rows_per_sample == 0),
                "lora: rows_per_sample=%d must be positive and divide M=%d", l->rows_per_sample, M);
  return 0;
}

// bn encodes an explicit choice when > 0: low 12 bits = tile width, bit 12 set = force CTA pairs, bit 13 set = force
// single CTAs (used by the tests to cover both).
static void decode_bn(int bn_arg, int* bn, int* force_ctas) {
  *force_ctas = (bn_arg > 0 && (bn_arg & 0x1000)) ? 2 : ((bn_arg > 0 && (bn_arg & 0x2000)) ? 1 : 0);
  *bn = bn_arg > 0 ? (bn_arg & 0xFFF) : 0;
}

// 2-D bf16 tensor map of `rows` rows of k elements, row stride ld elements, in boxes of box_rows rows x 64 k
static int tmap_2d(Ctx* ctx, CUtensorMap* out, const void* ptr, int ld, int k, int rows, int box_rows) {
  const uint64_t dims[2] = {static_cast<uint64_t>(k), static_cast<uint64_t>(rows)};
  const uint64_t strides[1] = {static_cast<uint64_t>(ld) * 2};
  const uint32_t box[2] = {kBK, static_cast<uint32_t>(box_rows)};
  return make_tmap_bf16(ctx, out, ptr, 2, dims, strides, box);
}

// The part of a GEMM / conv / split-K launch that does not depend on how A is addressed.  The entry point `who` has
// filled in the problem (M, N, K, flags, kblocks, num_sub, split-K) and the A operand; this validates the epilogue
// flags and the LoRA, picks the tile (bn_arg as decode_bn reads it), fills in the tile counts and the epilogue
// pointers, builds the tensor maps of W ([N, K], row stride ldw) and of the LoRA down-projection, and launches.  *pdl
// (when given) receives the launch's PDL choice.
static int plan_and_launch(Ctx* ctx, cudaStream_t stream, GemmParams& p, const char* who, const void* w, int ldw,
                           const void* bias, const void* rowbias, int rows_per_batch, const void* resid, int ldr,
                           void* out, int ldo, const sb200_lora* lora, int bn_arg, bool* pdl = nullptr) {
  const int flags = p.flags;
  const bool geglu = flags & SB200_EPI_GEGLU;
  const bool has_lora = flags & SB200_EPI_LORA;
  SB200_REQUIRE(!(geglu && has_lora), "%s: GEGLU and LORA cannot be combined", who);
  SB200_REQUIRE(!geglu || p.N % 32 == 0, "%s: GEGLU needs N %% 32 == 0", who);
  SB200_REQUIRE(!(flags & SB200_EPI_BIAS) || bias, "%s: BIAS without bias", who);
  SB200_REQUIRE(!(flags & SB200_EPI_ROWBIAS) || (rowbias && rows_per_batch > 0), "%s: ROWBIAS args", who);
  SB200_REQUIRE(!(flags & SB200_EPI_RESID) || (resid && ldr % 8 == 0), "%s: RESID args", who);
  SB200_REQUIRE(!has_lora || lora, "%s: LORA without sb200_lora", who);
  if (has_lora) {
    const int st = check_lora(lora, p.M, p.N);
    if (st) return st;
    p.lora_up = static_cast<const float*>(lora->up);
    p.lora_r = lora->r;
    p.lora_rt = lora->rt;
    p.lora_group_n = lora->group_n;
    p.lora_scale = lora->scale;
    p.lora_scale_dev = lora->scale_dev;
    p.lora_sample_scale = lora->sample_scale;
    p.lora_rows_per_sample = lora->rows_per_sample;
  }
  int bn, force_ctas;
  decode_bn(bn_arg, &bn, &force_ctas);
  TileChoice tc = pick_tile(p.N, ctx->num_sms, p.kblocks, p.lora_r, p.lora_rt, force_ctas, p.num_sub, flags);
  if (bn > 0) tc.bn = bn;
  if (force_ctas) tc.ctas = force_ctas;
  SB200_REQUIRE(bn_supported(tc.bn), "%s: bn=%d invalid (64, 128, 160 or 256)", who, tc.bn);
  SB200_REQUIRE(!is_wide(tc.bn) || wide_eligible(tc.bn, p.N, tc.ctas, p.lora_r, p.lora_rt, geglu),
                "%s: bn=%d needs N %% %d == 0 and single CTAs, without LoRA of rank 16 or rt 64%s (N=%d)", who, tc.bn,
                tc.bn, tc.bn == 160 ? " or GEGLU" : "", p.N);
  p.Nout = geglu ? p.N / 2 : p.N;
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
  // a CTA's W rows per k-block: half of the tile's in a pair; with GEGLU one box of value rows and one of gate rows
  int st;
  if ((st = tmap_2d(ctx, &p.tmB, w, ldw, p.K, p.N, (geglu || tc.ctas == 2) ? tc.bn / 2 : tc.bn))) return st;
  if (has_lora && (st = tmap_2d(ctx, &p.tmL, lora->down, p.K, p.K, lora->rt, lora->rt / tc.ctas))) return st;
  bool used_pdl;
  return launch_gemm(ctx, stream, p, tc.ctas, pdl ? pdl : &used_pdl);
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
  // the split tiles store 16-byte vectors to ws and the reduction 16-byte vectors to out
  SB200_REQUIRE((reinterpret_cast<uintptr_t>(out) & 15) == 0 && (reinterpret_cast<uintptr_t>(ws) & 15) == 0,
                "gemm_splitk_f32: out and ws must be 16-byte aligned");
  const size_t need = SB200_GEMM_SPLITK_WS_FLOATS(M, N, K);
  SB200_REQUIRE(ws_floats >= need, "gemm_splitk_f32: scratch of %zu floats, %zu needed", ws_floats, need);
  GemmParams p;
  memset(&p, 0, sizeof(p));
  p.M = M;
  p.N = N;
  p.K = K;
  p.kblocks = (K + kBK - 1) / kBK;
  p.kb_split = p.kblocks;
  p.cb_total = p.kblocks;
  p.a_tx = kBM * 128;
  p.num_sub = (M + kBM - 1) / kBM;
  p.sk_ws = ws;
  p.sk_kb = SB200_GEMM_SPLITK_KB(M, N, K);
  p.sk_splits = SB200_GEMM_SPLITK_SPLITS(M, N, K);
  int st;
  if ((st = tmap_2d(ctx, &p.tmA[0], x, ldx, K, M, kBM))) return st;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  // single CTAs on tiles 128 wide where N allows, no epilogue
  const int bn_arg = (N % 128 == 0 ? 128 : 64) | 0x2000;
  bool pdl;  // the reduction launches as the GEMM did
  if ((st = plan_and_launch(ctx, s, p, "gemm_splitk_f32", w, ldw, nullptr, nullptr, 0, nullptr, 0, nullptr, 0, nullptr,
                            bn_arg, &pdl)))
    return st;
  const size_t quads = static_cast<size_t>(M) * N / 4;
  SB200_CUDA_CHECK(launch_pdl(splitk_reduce_kernel, dim3(static_cast<unsigned>((quads + 255) / 256)), dim3(256), 0, s,
                              pdl, static_cast<const float*>(ws), p.sk_splits, M, N, out, ldo));
  SB200_CUDA_CHECK(cudaGetLastError());
  return 0;
}

extern "C" int sb200_gemm(void* handle, void* stream, const void* x0, int ldx0, const void* x1, int ldx1,
                          int K0, const void* w, int ldw, void* out, int ldo, int M, int N, int K,
                          int flags, const void* bias, const void* rowbias, int rows_per_batch,
                          const void* resid, int ldr, const sb200_lora* lora, int bn_arg) {
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

  GemmParams p;
  memset(&p, 0, sizeof(p));
  p.M = M;
  p.N = N;
  p.K = K;
  p.flags = flags;
  p.kblocks = (K + kBK - 1) / kBK;
  p.a_mode = 0;
  p.kb_split = split ? K0 / kBK : p.kblocks;
  p.cb_total = p.kblocks;
  p.a_tx = kBM * 128;
  p.num_sub = (M + kBM - 1) / kBM;
  int st;
  if ((st = tmap_2d(ctx, &p.tmA[0], x0, ldx0, K0, M, kBM))) return st;
  if (split && (st = tmap_2d(ctx, &p.tmA[1], x1, ldx1, K - K0, M, kBM))) return st;
  return plan_and_launch(ctx, static_cast<cudaStream_t>(stream), p, "gemm", w, ldw, bias, rowbias, rows_per_batch,
                         resid, ldr, out, ldo, lora, bn_arg);
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
  const bool pad_br = flags & SB200_CONV_PAD_BR;
  SB200_REQUIRE(!pad_br || stride == 2, "conv3x3: CONV_PAD_BR needs stride 2");
  flags &= ~SB200_CONV_PAD_BR;
  SB200_REQUIRE(ldx0 % 8 == 0 && ldo % 8 == 0 && (C1 == 0 || ldx1 % 8 == 0), "conv3x3: leading dims");
  const int H = Hin / stride, W = Win / stride;
  int bw, bh, bb;
  pick_patch(B, H, W, &bw, &bh, &bb);
  const int Cin = C0 + C1;

  GemmParams p;
  memset(&p, 0, sizeof(p));
  p.M = B * H * W;
  p.N = Cout;
  p.K = 9 * Cin;
  p.flags = flags;
  p.cb_total = Cin / kBK;
  p.kblocks = 9 * p.cb_total;
  p.a_mode = stride == 1 ? 1 : (pad_br ? 3 : 2);
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
  // w: [Cout, 3, 3, Cin], a row of K = 9 * Cin per output channel
  return plan_and_launch(ctx, static_cast<cudaStream_t>(stream), p, "conv3x3", w, p.K, bias, rowbias, H * W, resid,
                         ldr, out, ldo, lora, bn_arg);
}
