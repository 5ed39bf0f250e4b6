// vitron_b200 — wgmma GEMM kernel instantiations for 32-column tiles (8 smem stages); see gemm_v2.cuh.
#include "gemm_v2.cuh"

namespace vb {
int launch_gemm_v2_32(int need, bool generic, const CUtensorMap& ta, const CUtensorMap& tb, const GemmParams& p, cudaStream_t stream) {
  return dispatch_v2<32, 8>(need, generic, ta, tb, p, stream);
}
}  // namespace vb
