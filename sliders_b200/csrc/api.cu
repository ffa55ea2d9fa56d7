// Context, error reporting and TMA descriptor encoding for libsb200.so.
#include "common.h"

namespace sb200 {

static thread_local char g_err[512] = "";

int set_error(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}

int make_tmap_bf16(Ctx* ctx, CUtensorMap* out, const void* ptr, int rank, const uint64_t* dims,
                   const uint64_t* strides_bytes, const uint32_t* box) {
  TmapKey key;
  memset(&key, 0, sizeof(key));
  key.ptr = reinterpret_cast<uint64_t>(ptr);
  key.rank = static_cast<uint32_t>(rank);
  for (int i = 0; i < rank; ++i) {
    key.dims[i] = dims[i];
    key.box[i] = box[i];
    if (i < rank - 1) key.strides[i] = strides_bytes[i];
  }
  {
    std::lock_guard<std::mutex> lk(ctx->mu);
    auto it = ctx->tmaps.find(key);
    if (it != ctx->tmaps.end()) {
      *out = it->second;
      return 0;
    }
  }
  if ((key.ptr & 15) != 0) return set_error(SB200_ERR_INVALID, "TMA base %p not 16B aligned", ptr);
  for (int i = 0; i < rank - 1; ++i)
    if (strides_bytes[i] % 16 != 0)
      return set_error(SB200_ERR_INVALID, "TMA stride[%d]=%llu not a multiple of 16 bytes", i,
                       (unsigned long long)strides_bytes[i]);
  cuuint64_t gdim[5];
  cuuint64_t gstr[4];
  cuuint32_t bdim[5];
  cuuint32_t estr[5];
  for (int i = 0; i < rank; ++i) {
    gdim[i] = dims[i];
    bdim[i] = box[i];
    estr[i] = 1;
    if (i < rank - 1) gstr[i] = strides_bytes[i];
  }
  alignas(64) CUtensorMap m;
  CUresult r = ctx->encode(&m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, rank, const_cast<void*>(ptr), gdim,
                           gstr, bdim, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                           CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                           CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS)
    return set_error(SB200_ERR_CUDA,
                     "cuTensorMapEncodeTiled failed (%d): rank %d dims [%llu %llu %llu %llu] box [%u "
                     "%u %u %u] stride0 %llu",
                     (int)r, rank, (unsigned long long)dims[0],
                     (unsigned long long)(rank > 1 ? dims[1] : 0),
                     (unsigned long long)(rank > 2 ? dims[2] : 0),
                     (unsigned long long)(rank > 3 ? dims[3] : 0), box[0], rank > 1 ? box[1] : 0,
                     rank > 2 ? box[2] : 0, rank > 3 ? box[3] : 0,
                     (unsigned long long)(rank > 1 ? strides_bytes[0] : 0));
  {
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (ctx->tmaps.size() > (1u << 16)) ctx->tmaps.clear();
    ctx->tmaps.emplace(key, m);
  }
  *out = m;
  return 0;
}

}  // namespace sb200

using namespace sb200;

extern "C" {

const char* sb200_version(void) { return "sb200 0.1 sm_90a"; }

const char* sb200_last_error(void) { return g_err; }

int sb200_create(int device, void** handle) {
  if (!handle) return set_error(SB200_ERR_INVALID, "handle is NULL");
  SB200_CUDA_CHECK(cudaSetDevice(device));
  cudaDeviceProp prop;
  SB200_CUDA_CHECK(cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9 || prop.minor != 0)
    return set_error(SB200_ERR_UNSUPPORTED, "device %d is sm_%d%d; libsb200 is built for sm_90a only",
                     device, prop.major, prop.minor);
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult qres;
  SB200_CUDA_CHECK(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres));
  if (!fn || qres != cudaDriverEntryPointSuccess)
    return set_error(SB200_ERR_CUDA, "cuTensorMapEncodeTiled not available from the driver");
  Ctx* ctx = new Ctx();
  ctx->device = device;
  ctx->num_sms = prop.multiProcessorCount;
  ctx->encode = reinterpret_cast<EncodeTiledFn>(fn);
  *handle = ctx;
  return 0;
}

int sb200_destroy(void* handle) {
  delete as_ctx(handle);
  return 0;
}

}  // extern "C"
