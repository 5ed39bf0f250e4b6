// vitron_b200 — wgmma GEMM "resident B" instantiations (small-K GEMMs: the weight n-block stays in shared memory); see gemm_v2.cuh.
#include "gemm_v2.cuh"

namespace vb {
// A-ring depth by tile width: what is left of 227 KB next to a 5 k-block B slab (K = 320) resp. 10 k-blocks at BN = 128 (K = 640)
int launch_gemm_v2_resb(int bn, int need, const CUtensorMap& ta, const CUtensorMap& tb, const GemmParams& p, cudaStream_t stream) {
  switch (bn) {
    case 256: return dispatch_v2_resb<256, 3>(need, ta, tb, p, stream);
    case 160: return dispatch_v2_resb<160, 6>(need, ta, tb, p, stream);
    case 128: return dispatch_v2_resb<128, 3>(need, ta, tb, p, stream);
    default: return VB_ERR_UNSUPPORTED;
  }
}
int resb_smem_bytes(int bn, int nkb) {
  switch (bn) {
    case 256: return gemm_smem<256, 3, true>(nkb);
    case 160: return gemm_smem<160, 6, true>(nkb);
    case 128: return gemm_smem<128, 3, true>(nkb);
    default: return 1 << 30;
  }
}
}  // namespace vb
