// Library-level pieces of the C ABI: error text, version, launch counter, driver entry point lookup, tensor-map encoding, SM count.
#include <atomic>
#include <cstdio>
#include <cstring>

#include "internal.h"

namespace cvb {

static thread_local char g_err[1024] = "";
static std::atomic<long long> g_launches{0};

int set_error(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}

void count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }

// cuTensorMapEncodeTiled resolved through the runtime (no link-time dependency on libcuda).
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_tiled() {
  static EncodeTiledFn fn = nullptr;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
    else
      (void)cudaGetLastError();
  }
  return fn;
}

int encode_map(CUtensorMap* m, CUtensorMapDataType dt, int rank, const void* base, const cuuint64_t* dims, const cuuint64_t* strides_bytes,
               const cuuint32_t* box, CUtensorMapSwizzle swz) {
  EncodeTiledFn enc = get_encode_tiled();
  if (!enc) return set_error(CVB_ERR_NO_DEVICE, "cuTensorMapEncodeTiled entry point not found (no CUDA driver?)");
  const cuuint32_t estr[5] = {1, 1, 1, 1, 1};
  const CUresult r = enc(m, dt, (cuuint32_t)rank, const_cast<void*>(base), dims, strides_bytes, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swz,
                         CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    return set_error(CVB_ERR_CUDA,
                     "cuTensorMapEncodeTiled failed (%d): rank %d dims [%llu %llu %llu %llu %llu] box [%u %u %u %u %u] base %p", (int)r,
                     rank, (unsigned long long)dims[0], (unsigned long long)(rank > 1 ? dims[1] : 0),
                     (unsigned long long)(rank > 2 ? dims[2] : 0), (unsigned long long)(rank > 3 ? dims[3] : 0),
                     (unsigned long long)(rank > 4 ? dims[4] : 0), box[0], rank > 1 ? box[1] : 0, rank > 2 ? box[2] : 0,
                     rank > 3 ? box[3] : 0, rank > 4 ? box[4] : 0, base);
  }
  return CVB_OK;
}

int sm_count() {
  struct Query {
    cudaError_t err;
    int sms;
  };
  static const Query q = [] {
    Query r{cudaSuccess, 0};
    int dev = 0;
    r.err = cudaGetDevice(&dev);
    if (r.err == cudaSuccess) r.err = cudaDeviceGetAttribute(&r.sms, cudaDevAttrMultiProcessorCount, dev);
    return r;
  }();
  if (q.err != cudaSuccess || q.sms <= 0) {
    set_error(CVB_ERR_NO_DEVICE, "no CUDA device: %s", cudaGetErrorString(q.err));
    return 0;
  }
  return q.sms;
}

}  // namespace cvb

extern "C" const char* cvb_last_error_string(void) { return cvb::g_err; }
extern "C" int cvb_version(void) { return 100; /* 0.1.0 */ }
extern "C" int64_t cvb_launch_count(void) { return cvb::g_launches.load(std::memory_order_relaxed); }
