// Internal declarations shared by the .cu translation units.  Each extern "C" entry point of
// include/ctrl_adapter_b200.h is defined in the file that holds its kernel, inside namespace ca: a function with C
// language linkage is the same function in every namespace, so it is the header's global ca_* symbol.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/ctrl_adapter_b200.h"

namespace ca {

// --- capi.cu ---
// records the message returned by ca_last_error() and returns `code`
int fail(int code, const char* fmt, ...) __attribute__((format(printf, 2, 3)));
// CA_OK for cudaSuccess, else CA_ERR_CUDA with "what: <CUDA error>"
int launched(cudaError_t e, const char* what);
// bf16 tensor map, 128B swizzle unless `swizzle` says otherwise, zero OOB fill. dims/strides fastest-first; strides
// in BYTES for dims 1..rank-1.
int make_tmap(CUtensorMap* m, const void* base, int rank, const cuuint64_t* dims, const cuuint64_t* strides_bytes,
              const cuuint32_t* box, CUtensorMapSwizzle swizzle = CU_TENSOR_MAP_SWIZZLE_128B);
int num_sms();
// argument checks: a pointer the kernel accesses in `bytes`-wide vectors (a null pointer passes), and the largest
// gridDim.y / gridDim.z a launch may have
inline bool aligned(const void* p, unsigned bytes) { return (reinterpret_cast<uintptr_t>(p) & (bytes - 1u)) == 0; }
constexpr long long kMaxGridYZ = 65535;

// --- gemm_conv.cu / gemm_conv_bn*.cu ---
struct GemmParams {
  int box[4];             // row-space box extents (product == 128)
  int ntile[4];           // tiles along each row dim
  int odim[4];            // output extents (rows outside are computed but not stored)
  long long ostride[4];   // output element strides per row dim
  long long rstride[4];   // residual / blend_src element strides per row dim
  long long vstride[4];   // rowvec element strides per row dim
  int ntaps;
  int tap_off[CA_MAX_TAPS][4];  // A-coordinate offset of each tap, per row dim
  int tap_c_off[CA_MAX_TAPS];   // A channel offset of each tap (stride-2 parity views)
  int nsrc;
  int src_c[2];           // channels taken from each A source (K extent per tap = sum)
  int src_c0_off[2];      // first channel inside each source tensor
  int k_per_tap;          // weight row elements per tap (>= src_c[0] + src_c[1], zero padded)
  int n_out;              // output columns
  int n_tiles_n;
  int act;
  int out_fp32;
  int vec_ok;             // bf16 output: out / residual / blend_src / rowvec bases and strides allow 16-byte access
  int ops_tma;            // bf16, non-GEGLU, vec_ok: residual / blend_src come through their tensor maps
  float out_scale;
  const float* bias;               // [weight rows] fp32
  const __nv_bfloat16* rowvec;     // broadcast add, indexed through vstride
  const __nv_bfloat16* residual;   // indexed through rstride
  const __nv_bfloat16* blend_src;  // AlphaBlender x_spatial, indexed through rstride
  const float* blend_alpha;        // device scalar: sigmoid(mix_factor), bf16-valued
  void* out;
};

// one per N tile width, each in its own translation unit so that the kernel instantiations compile in parallel
cudaError_t launch_gemm_bn64(const CUtensorMap& a0, const CUtensorMap& a1, const CUtensorMap& w, const CUtensorMap& res,
                             const CUtensorMap& blend, const GemmParams& p, int grid, cudaStream_t stream);
cudaError_t launch_gemm_bn128(const CUtensorMap& a0, const CUtensorMap& a1, const CUtensorMap& w, const CUtensorMap& res,
                              const CUtensorMap& blend, const GemmParams& p, int grid, cudaStream_t stream);
cudaError_t launch_gemm_bn160(const CUtensorMap& a0, const CUtensorMap& a1, const CUtensorMap& w, const CUtensorMap& res,
                              const CUtensorMap& blend, const GemmParams& p, int grid, cudaStream_t stream);
cudaError_t launch_gemm_bn256(const CUtensorMap& a0, const CUtensorMap& a1, const CUtensorMap& w, const CUtensorMap& res,
                              const CUtensorMap& blend, const GemmParams& p, int grid, cudaStream_t stream);

}  // namespace ca
