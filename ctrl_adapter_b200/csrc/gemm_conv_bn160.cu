// gemm_conv_kernel instantiation for BN = 160 (see gemm_conv.cu for the dispatch).
#include "gemm_conv_kernel.cuh"

namespace ca {
cudaError_t launch_gemm_bn160(const CUtensorMap& a0, const CUtensorMap& a1, const CUtensorMap& w, const CUtensorMap& res,
                              const CUtensorMap& blend, const GemmParams& p, int grid, cudaStream_t stream) {
  return launch_bn<160>(a0, a1, w, res, blend, p, grid, stream);
}
}  // namespace ca
