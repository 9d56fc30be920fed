// Host-side dispatch of gemm_conv_kernel to the per-BN translation units (gemm_conv_bn*.cu; split so the kernel
// instantiations compile in parallel).
#include "kernels.h"

namespace ca {

#define CA_DECL_BN(bn)                                                                                         \
  cudaError_t launch_gemm_bn##bn(const CUtensorMap& a0, const CUtensorMap& a1, const CUtensorMap& w,           \
                                 const GemmParams& p, int grid, cudaStream_t stream);
CA_DECL_BN(64)
CA_DECL_BN(128)
CA_DECL_BN(160)
CA_DECL_BN(256)
#undef CA_DECL_BN

cudaError_t launch_gemm_conv(int bn, const CUtensorMap& a0, const CUtensorMap& a1, const CUtensorMap& w,
                             const GemmParams& p, int grid, cudaStream_t stream) {
  switch (bn) {
    case 64: return launch_gemm_bn64(a0, a1, w, p, grid, stream);
    case 128: return launch_gemm_bn128(a0, a1, w, p, grid, stream);
    case 160: return launch_gemm_bn160(a0, a1, w, p, grid, stream);
    case 256: return launch_gemm_bn256(a0, a1, w, p, grid, stream);
    default: return cudaErrorInvalidValue;
  }
}

}  // namespace ca
