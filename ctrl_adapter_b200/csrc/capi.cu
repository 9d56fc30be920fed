// What the extern "C" entry points share: the thread-local error message, TMA tensor-map encoding and the SM count;
// plus the three entry points that belong to no kernel.  Each other entry point is defined next to its kernel.
// cuTensorMapEncodeTiled is resolved at run time through the CUDA runtime (cudaGetDriverEntryPoint) so the library has
// no link-time dependency on libcuda and can be dlopen'ed (symbol check) on a machine without a driver.
#include <stdarg.h>
#include <stdio.h>

#include "kernels.h"

namespace ca {

namespace {

thread_local char g_err[512] = "";

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

}  // namespace

int fail(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}

int launched(cudaError_t e, const char* what) {
  return e == cudaSuccess ? CA_OK : fail(CA_ERR_CUDA, "%s: %s", what, cudaGetErrorString(e));
}

int make_tmap(CUtensorMap* m, const void* base, int rank, const cuuint64_t* dims, const cuuint64_t* strides_bytes,
              const cuuint32_t* box) {
  if ((reinterpret_cast<uintptr_t>(base) & 15) != 0) return fail(CA_ERR_INVALID, "tensor base not 16-byte aligned");
  for (int i = 0; i + 1 < rank; ++i)
    if (strides_bytes[i] % 16 != 0) return fail(CA_ERR_INVALID, "tensor stride %d (%llu B) not a multiple of 16", i + 1,
                                                (unsigned long long)strides_bytes[i]);
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) return fail(CA_ERR_CUDA, "cuTensorMapEncodeTiled unavailable (no CUDA driver?)");
  cuuint32_t estr[5] = {1, 1, 1, 1, 1};
  CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, rank, const_cast<void*>(base), dims, strides_bytes, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    return fail(CA_ERR_CUDA,
                "cuTensorMapEncodeTiled failed (%d): rank %d dims [%llu %llu %llu %llu %llu] box [%u %u %u %u %u]",
                (int)r, rank, (unsigned long long)dims[0], (unsigned long long)(rank > 1 ? dims[1] : 0),
                (unsigned long long)(rank > 2 ? dims[2] : 0), (unsigned long long)(rank > 3 ? dims[3] : 0),
                (unsigned long long)(rank > 4 ? dims[4] : 0), box[0], rank > 1 ? box[1] : 0, rank > 2 ? box[2] : 0,
                rank > 3 ? box[3] : 0, rank > 4 ? box[4] : 0);
  }
  return CA_OK;
}

int num_sms() {
  static int sms = 0;
  if (sms == 0) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return 132;
    if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || sms <= 0) sms = 132;
  }
  return sms;
}

extern "C" int ca_abi_version(void) { return CA_ABI_VERSION; }
extern "C" const char* ca_last_error(void) { return g_err; }

extern "C" int ca_device_ok(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess || n <= 0) return fail(CA_ERR_CUDA, "no CUDA device");
  int dev = 0, major = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev);
  if (major != 9) return fail(CA_ERR_UNSUPPORTED, "device compute capability %d.x, need 9.x (sm_90a)", major);
  return CA_OK;
}

}  // namespace ca
