// Host-side plumbing shared by the C-ABI entry points: error reporting, the per-device context and
// the TMA descriptor cache.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <cstdlib>
#include <stdarg.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <mutex>
#include <unordered_map>

#include "../../include/sb200.h"

namespace sb200 {

int set_error(int code, const char* fmt, ...);

#define SB200_CUDA_CHECK(expr)                                                                  \
  do {                                                                                          \
    cudaError_t _e = (expr);                                                                    \
    if (_e != cudaSuccess)                                                                      \
      return ::sb200::set_error(SB200_ERR_CUDA, "%s failed: %s (%s:%d)", #expr,                 \
                                cudaGetErrorString(_e), __FILE__, __LINE__);                    \
  } while (0)

#define SB200_REQUIRE(cond, ...)                                            \
  do {                                                                      \
    if (!(cond)) return ::sb200::set_error(SB200_ERR_INVALID, __VA_ARGS__); \
  } while (0)

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                  const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

struct TmapKey {
  uint64_t ptr;
  uint64_t dims[5];
  uint64_t strides[4];
  uint32_t box[5];
  uint32_t rank;
  bool operator==(const TmapKey& o) const { return memcmp(this, &o, sizeof(TmapKey)) == 0; }
};
struct TmapKeyHash {
  size_t operator()(const TmapKey& k) const {
    const uint64_t* w = reinterpret_cast<const uint64_t*>(&k);
    uint64_t h = 1469598103934665603ull;
    for (size_t i = 0; i < sizeof(TmapKey) / 8; ++i) {
      h ^= w[i];
      h *= 1099511628211ull;
    }
    return static_cast<size_t>(h);
  }
};

struct Ctx {
  int device = 0;
  int num_sms = 0;
  int smem_per_sm = 0;     // shared memory of one SM (bytes)
  int smem_optin = 0;      // largest dynamic shared memory one CTA may opt in to
  int smem_reserved = 0;   // shared memory the system reserves per resident CTA
  EncodeTiledFn encode = nullptr;
  std::mutex mu;
  std::unordered_map<TmapKey, CUtensorMap, TmapKeyHash> tmaps;
};

// bf16 tensor map, 128-byte swizzle, zero OOB fill. dims/box innermost first; strides (bytes) for dims
// 1..rank-1. Returns 0 or a negative status.
int make_tmap_bf16(Ctx* ctx, CUtensorMap* out, const void* ptr, int rank, const uint64_t* dims,
                   const uint64_t* strides_bytes, const uint32_t* box);

// SB200_PDL=0 disables programmatic dependent launch, 2 applies it to every launch_ex / launch_pdl whatever its size
// (same-box A/B); default 1: each launch's `pdl` argument decides
inline int pdl_mode() {
  static const int m = [] {
    const char* e = getenv("SB200_PDL");
    return e ? atoi(e) : 1;
  }();
  return m;
}

// PDL pays off for small launches (launch latency and prologue are a visible share: +3 % at 2 passes per forward) and
// costs ~1 % on machine-filling ones (8 passes), so the GEMM and attention forward use it only on grids of at most two
// CTAs per SM
inline bool pdl_small_grid(const Ctx* ctx, long long ctas) { return ctas <= 2LL * ctx->num_sms; }

// <<<grid, block, smem, stream>>> in clusters of `cluster_x` CTAs along x (1: no cluster), with the
// programmatic-stream-serialization attribute as pdl_mode() and `pdl` decide (the kernel must call pdl_wait() before
// touching global memory)
template <typename... KArgs, typename... Args>
inline cudaError_t launch_ex(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream,
                             unsigned cluster_x, bool pdl, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[2];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = (pdl_mode() == 2 || (pdl_mode() == 1 && pdl)) ? 1 : 0;
  attr[1].id = cudaLaunchAttributeClusterDimension;
  attr[1].val.clusterDim.x = cluster_x;
  attr[1].val.clusterDim.y = 1;
  attr[1].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = cluster_x > 1 ? 2 : 1;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream,
                              bool pdl, Args&&... args) {
  return launch_ex(kernel, grid, block, smem, stream, 1u, pdl, static_cast<Args&&>(args)...);
}

// Grid of a grid-stride kernel: ceil(work / per_block) blocks, at most `waves` per SM, computed in the type of `work`;
// at_least_one launches one block for empty work.
template <typename T>
inline int grid_cap(const Ctx* ctx, T work, int per_block, int waves, bool at_least_one = false) {
  T blocks = (work + per_block - 1) / per_block;
  const T cap = static_cast<T>(ctx->num_sms) * waves;
  if (blocks > cap) blocks = cap;
  return at_least_one && blocks < 1 ? 1 : static_cast<int>(blocks);
}

inline Ctx* as_ctx(void* h) { return reinterpret_cast<Ctx*>(h); }

// GroupNorm forward / backward stats kernels: block = (C/8) x rows_par threads, rows_par = max(1, 512 / (C/8)), with
// [rows_par][C][2] fp32 partials in dynamic shared memory.  They launch without opting in above the default 48 KB,
// so C may not exceed 6144 (rows_par = 1 for C > 4096).
inline int gn_rows_par(int C) {
  const int rp = 512 / (C / 8);
  return rp < 1 ? 1 : rp;
}
inline bool gn_stats_smem_ok(int C) {
  return C > 0 && sizeof(float) * 2 * static_cast<size_t>(C) * gn_rows_par(C) <= 48 * 1024;
}

// The partials of at most this many row chunks per sample precede the final (mean, rstd) block in the workspace
// (the 128 of SB200_GN_STATS_OFFSET).
constexpr int kGnMaxChunks = 128;
static_assert(SB200_GN_STATS_OFFSET(1, 1) == 2 * kGnMaxChunks, "GroupNorm workspace layout");

// GroupNorm stats / apply launch shape, forward and backward: a (chunks, B) grid of `threads`-thread blocks, each block
// walking rows_per_block of the HW rows.  Enough blocks to fill the machine, but each block walks >= 8 rows per thread.
struct GnShape {
  int rows_par, threads, chunks, rows_per_block;
};
inline GnShape gn_shape(const Ctx* ctx, int B, int HW, int C) {
  GnShape g;
  g.rows_par = gn_rows_par(C);
  g.threads = C / 8 * g.rows_par;
  int chunks = (ctx->num_sms * 4 + B - 1) / B;
  if (chunks > kGnMaxChunks) chunks = kGnMaxChunks;
  g.rows_per_block = (HW + chunks - 1) / chunks;
  if (g.rows_per_block < g.rows_par * 8) g.rows_per_block = g.rows_par * 8;
  g.chunks = (HW + g.rows_per_block - 1) / g.rows_per_block;
  return g;
}

}  // namespace sb200
