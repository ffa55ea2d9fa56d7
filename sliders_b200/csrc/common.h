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
  EncodeTiledFn encode = nullptr;
  std::mutex mu;
  std::unordered_map<TmapKey, CUtensorMap, TmapKeyHash> tmaps;
};

// bf16 tensor map, 128-byte swizzle, zero OOB fill. dims/box innermost first; strides (bytes) for dims
// 1..rank-1. Returns 0 or a negative status.
int make_tmap_bf16(Ctx* ctx, CUtensorMap* out, const void* ptr, int rank, const uint64_t* dims,
                   const uint64_t* strides_bytes, const uint32_t* box);

// SB200_PDL=0 disables programmatic dependent launch, 2 applies it to every launch whatever its size (same-box A/B;
// default 1: only launches that do not fill the machine, see pdl_hint)
inline int pdl_mode() {
  static const int m = [] {
    const char* e = getenv("SB200_PDL");
    return e ? atoi(e) : 1;
  }();
  return m;
}
inline bool pdl_enabled() { return pdl_mode() != 0; }

// Per-call hint set by the C-ABI entry points: PDL pays off for small launches (launch latency and prologue are a
// visible share: +3 % at 2 passes per forward) and costs ~1 % on machine-filling ones (8 passes), so the big shapes
// launch without it.
inline bool& pdl_hint() {
  static thread_local bool h = true;
  return h;
}

// <<<grid, block, smem, stream>>> with the programmatic-stream-serialization attribute (the kernel must call
// pdl_wait() before touching global memory)
template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream,
                              Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = (pdl_mode() == 2 || (pdl_mode() == 1 && pdl_hint())) ? 1 : 0;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

inline Ctx* as_ctx(void* h) { return reinterpret_cast<Ctx*>(h); }

}  // namespace sb200
