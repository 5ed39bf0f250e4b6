// vitron_b200 — wgmma GEMM kernel instantiations for 128-column tiles (6 smem stages); see gemm_v2.cuh.
#include "gemm_v2.cuh"

namespace vb {
int launch_gemm_v2_128(int need, bool generic, const CUtensorMap& ta, const CUtensorMap& tb, const GemmParams& p, cudaStream_t stream) {
  return dispatch_v2<128, 6>(need, generic, ta, tb, p, stream);
}
}  // namespace vb
