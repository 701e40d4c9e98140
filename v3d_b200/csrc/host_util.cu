#include "host_util.cuh"

#include <atomic>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <mutex>

#include "common.cuh"
#include "v3d_b200.h"

namespace v3d {

static thread_local char g_err[512] = "";
static std::atomic<int64_t> g_launches{0};

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
void count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }

int num_sms() {
  static int sms = 0;
  if (sms == 0) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return 132;  // H100 SXM
    int v = 0;
    if (cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || v <= 0)
      return 132;  // H100 SXM
    sms = v;
  }
  return sms;
}

EncodeTiledFn get_encode_tiled() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q);
    if (e == cudaSuccess && q == cudaDriverEntryPointSuccess) fn = reinterpret_cast<EncodeTiledFn>(p);
    (void)cudaGetLastError();
  });
  return fn;
}

int make_tmap_bf16(CUtensorMap* map, const void* base, int rank, const uint64_t* dims,
                   const uint64_t* strides_bytes, const uint32_t* box, int swizzle_bytes) {
  EncodeTiledFn enc = get_encode_tiled();
  if (!enc) {
    set_error("cuTensorMapEncodeTiled unavailable (no CUDA driver?)");
    return V3D_ERR_NO_DRIVER;
  }
  cuuint64_t gdim[5];
  cuuint64_t gstr[5];
  cuuint32_t bx[5];
  cuuint32_t es[5];
  for (int i = 0; i < rank; ++i) {
    gdim[i] = dims[i];
    bx[i] = box[i];
    es[i] = 1;
    if (i + 1 < rank) gstr[i] = strides_bytes[i];
  }
  if ((reinterpret_cast<uintptr_t>(base) & 15u) != 0) {
    set_error("tensor map base %p not 16-byte aligned", base);
    return V3D_ERR_BAD_ARG;
  }
  CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, static_cast<cuuint32_t>(rank),
                   const_cast<void*>(base), gdim, gstr, bx, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   swizzle_bytes == 128  ? CU_TENSOR_MAP_SWIZZLE_128B
                   : swizzle_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B
                   : swizzle_bytes == 32 ? CU_TENSOR_MAP_SWIZZLE_32B
                                         : CU_TENSOR_MAP_SWIZZLE_NONE,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed (%d): rank %d dims [%llu,%llu,%llu,%llu] box [%u,%u,%u,%u] "
              "stride0 %llu",
              static_cast<int>(r), rank, (unsigned long long)dims[0],
              (unsigned long long)(rank > 1 ? dims[1] : 0), (unsigned long long)(rank > 2 ? dims[2] : 0),
              (unsigned long long)(rank > 3 ? dims[3] : 0), box[0], rank > 1 ? box[1] : 0,
              rank > 2 ? box[2] : 0, rank > 3 ? box[3] : 0,
              (unsigned long long)(rank > 1 ? strides_bytes[0] : 0));
    return V3D_ERR_CUDA;
  }
  return V3D_OK;
}

}  // namespace v3d

extern "C" {
int v3d_abi_version(void) { return V3D_ABI_VERSION; }
const char* v3d_last_error(void) { return v3d::g_err; }
int64_t v3d_launch_count(void) { return v3d::g_launches.load(std::memory_order_relaxed); }
}
